"""The bounds of the attention reference tests (attn_ref_util.py) accept the kernels' arithmetic and are tight enough to catch the
bugs those tests exist for.

`_emulate` restates the kernels in fp32 on the host, with their rounding points: scores fmaf(q.k, scale log2 e, bias log2 e) in
the exp2 domain, unnormalised probabilities rounded to bf16 before P V (whole-row softmax as the wgmma kernels do it, or the online
softmax of the staged and whole-head kernels: probabilities relative to the running maximum, fp32 rescales of the accumulator and
the sum when a later key block raises it, the dropout scale folded in before the rounding), the fp32 lse, bf16 ctx, D from that
bf16 ctx, probabilities recomputed from the stored lse, dS rounded to bf16 before dQ and dK, and the dropout scale
256 / (256 - round(256 p)). Every input family of the GPU tests passes: the fp32 lse and drow with a worst error / bound under
0.05, the bf16 outputs under 1 (their own final rounding alone reaches up to 2^-8 relative, the bound's first term, so they sit at
0.4-0.9 by construction). Each planted bug is the same emulation with one thing wrong, and is rejected by at least 2x in some output
on the family where it shows; most by 10-1000x."""
import math

import pytest
import torch

import attn_ref_util as R

LOG2E = 1.4426950408889634
B, A = 3, 2
P_DROP = 0.1


def _bf(x):
    return x.bfloat16().float()


def _emulate(q, k, v, bias, keep, scale, dO, online, bug=None):
    """fp32 emulation of one forward + backward in head layout ([N, S, 64] bf16 operands, bias [N, S] fp32, keep [N, S, S]
    0/1 or None). -> {name: output} as the kernels would write it."""
    N, S, _ = q.shape
    qf, kf, vf, dof = q.float(), k.float(), v.float(), dO.float()
    b2 = bias.float() * torch.tensor(LOG2E, dtype=torch.float32)
    if bug == "bias on neighbouring key":
        b2 = torch.cat([b2[:, 1:], b2[:, -1:]], 1)
    if bug == "last key of partial block dropped":
        b2 = b2.clone()
        b2[:, S - 1] = -math.inf
    sc2 = torch.tensor(0.125 * LOG2E, dtype=torch.float32)
    s2 = (qf @ kf.transpose(-1, -2)) * sc2 + b2[:, None, :]
    kp = torch.ones(N, S, S) if keep is None else keep.float()
    sd = torch.tensor(scale, dtype=torch.float32)

    # forward
    if not online:
        m = s2.amax(-1)
        e = torch.exp2(s2 - m[..., None])
        l = e.sum(-1)
        o = (_bf(e * kp) @ vf) * (sd / l)[..., None]
    else:
        m = torch.full((N, S), -math.inf)
        l = torch.zeros(N, S)
        o = torch.zeros(N, S, 64)
        for k0 in range(0, S, 64):
            blk = s2[:, :, k0:k0 + 64]
            mn = torch.maximum(m, blk.amax(-1))
            alpha = torch.exp2(m - mn)
            e = torch.exp2(blk - mn[..., None])
            l = l * alpha + e.sum(-1)
            if bug != "accumulator not rescaled":
                o = o * alpha[..., None]
            o = o + _bf(e * kp[:, :, k0:k0 + 64] * sd) @ vf[:, k0:k0 + 64]
            m = mn
        o = o / l[..., None]
    ctx = o.bfloat16()
    lse = (m + torch.log2(l)) * torch.tensor(math.log(2.0), dtype=torch.float32)

    # backward
    lse_b = lse if bug != "P from neighbouring row's lse" else torch.cat([lse[:, 1:], lse[:, :1]], 1)
    P = torch.exp2(s2 - (lse_b * torch.tensor(LOG2E, dtype=torch.float32))[..., None])
    dP = dof @ vf.transpose(-1, -2)
    D = drow = (dof * ctx.float()).sum(-1)
    if bug == "D from neighbouring row":   # drow is written right, dS reads the wrong entry
        D = torch.cat([D[:, 1:], D[:, :1]], 1)

    def dS(kk):
        return _bf(P * (torch.where(kk > 0, dP * sd, torch.zeros(())) - D[..., None]))

    kkv = kp.transpose(-1, -2) if bug == "dK/dV keep bits untransposed" else kp
    dq = (dS(kp) @ kf) * 0.125
    dk = (dS(kkv).transpose(-1, -2) @ qf) * (1.0 if bug == "dK without 1/8" else 0.125)
    Pd = _bf(P * kkv * sd * (sd if bug == "dropout scale twice in dV" else 1.0))
    dv = Pd.transpose(-1, -2) @ dof
    return dict(ctx=ctx, lse=lse, drow=drow, dq=dq.bfloat16(), dk=dk.bfloat16(), dv=dv.bfloat16())


def _case(family, S, p, seed=0):
    """Operands of one dense call of the family in head layout, with random keep bits when p > 0."""
    qkv, bias, dctx = R.inputs(family, B, S, A, torch.device("cpu"), seed=1000 * S + seed)
    q, k, v = R.dense_heads(qkv, B, S, A)
    dO = R.dense_heads(dctx, B, S, A)[0]
    bh = bias.repeat_interleave(A, 0)
    keep = None
    if p > 0:
        g = torch.Generator().manual_seed(seed + 7)
        keep = (torch.randint(0, 256, (B * A, S, S), generator=g) >= int(p * 256 + 0.5)).to(torch.uint8)
    return q, k, v, bh, keep, R.drop_scale(p), dO


def _ratios(case, online, bug=None, keep_used=None):
    q, k, v, bh, keep, scale, dO = case
    out = _emulate(q, k, v, bh, keep if keep_used is None else keep_used, scale, dO, online, bug)
    ref = R.reference(q, k, v, bh, keep, scale, dO, out["ctx"])
    worst = {}
    for n, o in out.items():
        r, bd = ref[n]
        worst[n] = float(((o.double() - r).abs() / (bd + 1e-300)).max())
    return worst, out, ref


@pytest.mark.parametrize("online", [False, True], ids=["whole", "online"])
@pytest.mark.parametrize("p", [0.0, P_DROP])
@pytest.mark.parametrize("S", [65, 200])
@pytest.mark.parametrize("family", R.FAMILIES)
def test_bound_accepts_the_kernel_arithmetic(family, S, p, online):
    case = _case(family, S, p)
    q, k, v, bh, keep, scale, dO = case
    out = _emulate(q, k, v, bh, keep, scale, dO, online)
    ref = R.reference(q, k, v, bh, keep, scale, dO, out["ctx"])
    worst = R.check_all(out, ref, f"{family} S={S} p={p}")
    assert worst["lse"] < 0.05 and worst["drow"] < 0.05, worst


# (bug, input family, dropout, softmax variant)
BUGS = [
    ("dK/dV keep bits untransposed", "unit", P_DROP, False),
    ("last key of partial block dropped", "peaked", 0.0, True),
    ("bias on neighbouring key", "bias", 0.0, False),
    ("P from neighbouring row's lse", "peaked", 0.0, False),
    ("D from neighbouring row", "rowscale", 0.0, False),
    ("accumulator not rescaled", "peaked", 0.0, True),
    ("dK without 1/8", "unit", 0.0, False),
    ("dropout scale twice in dV", "unit", P_DROP, False),
]


@pytest.mark.parametrize("bug,family,p,online", BUGS, ids=[b[0] for b in BUGS])
def test_bound_rejects_a_planted_bug(bug, family, p, online):
    for S in (65, 130):
        case = _case(family, S, p)
        good, _, _ = _ratios(case, online)
        assert max(good.values()) < 1.0, good
        worst, _, _ = _ratios(case, online, bug)
        assert max(worst.values()) > 2.0, f"{bug} S={S}: worst error / bound {worst}"


@pytest.mark.parametrize("online", [False, True], ids=["whole", "online"])
def test_bound_rejects_one_flipped_keep_bit(online):
    """The forward and backward apply one keep bit other than the stored one, on a row's largest probability: the largest
    probability dropped, or kept where it was dropped."""
    for S in (65, 200):
        case = _case("unit", S, P_DROP)
        q, k, v, bh, keep, scale, dO = case
        sc = q.double() @ k.double().transpose(-1, -2) / 8 + bh.double()[:, None, :]
        for n, i in ((0, 3), (1, S // 2), (B * A - 1, S - 1)):
            j = int(sc[n, i].argmax())
            flipped = keep.clone()
            flipped[n, i, j] ^= 1
            worst, _, _ = _ratios(case, online, keep_used=flipped)
            assert max(worst["ctx"], worst["dv"]) > 2.0, f"S={S} bit ({n}, {i}, {j}): {worst}"
