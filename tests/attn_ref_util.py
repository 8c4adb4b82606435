"""Reference arithmetic and error bounds of the attention tests (test_attention_reference_gpu.py, test_unpadded_gpu.py,
test_attention_reference_cpu.py): ctx, lse, drow, dQ, dK and dV of every attention route, dense and variable-length.

The reference is fp64 and starts from the exact operands the kernels read: the bf16 Q, K, V and dO, the fp32 key bias, the keep
bits the forward stored, and for the backward D = rowsum(dO ctx) from the kernel's own bf16 ctx (attn_delta_kernel, the EPI_DELTA
epilogue and the staged dQ kernel all read that ctx, so the ctx rounding is not part of the gradient bound; ctx is checked on its
own). Per head, with s_ij = q_i.k_j / 8 + bias_j, P = softmax(s), kd_ij = keep_ij * 256 / (256 - round(256 p)) (1 without
dropout), P_drop = P kd, dP_ij = dO_i.v_j and dS = P (kd dP - D):

    ctx = P_drop V,  lse_i = logsumexp_j s_ij,  drow_i = D_i,
    dV = P_drop^T dO,  dQ = dS K / 8,  dK = dS^T Q / 8.

An element passes when |out - ref| <= bound. Every probability carries a relative error

    eP_ij = C_P + C_S (1 + m_ij + |lse_i|),    m_ij = |q_i|.|k_j| / 8 + |bias_j|.

C_P = 2^-8 is the bf16 rounding of the unnormalised probabilities before the P V and P^T dO products (the normalisation sum is
accumulated from the unrounded fp32 values and does not carry it). C_S covers the fp32 path from scores to probabilities: the
fp32 dot product (its error is relative to |q|.|k|, not to |q.k|, hence m_ij in place of |s_ij|), fmaf(s, scale log2 e,
bias log2 e) and the subtraction of the row maximum or of the stored lse (whose roundings are relative to the operands: near
14427 in the exp2 domain for a -10000 bias, where an ulp is 2^-10), ex2.approx, log2f, the fp32 online-softmax rescales and the
fp32 lse the forward stores and the backward reads. The term is per element: a key bias only loosens the probabilities of its own
key, so the valid rows of a padded example keep a tight bound.

    ctx:     2^-8 |ctx| + (eP P_drop) |V|
    lse:     C_S (1 + |lse_i| + sum_j P_ij m_ij)        (the error of lse is the P-weighted error of the scores)
    drow:    C_SUM sum |dO| |ctx|                       (fp32 sum of bf16 products)
    dV:      2^-8 |dV| + (eP P_drop)^T |dO|
    dQ, dK:  2^-8 |ref| + mag(dS) |K| / 8,  mag(dS)^T |Q| / 8
             mag(dS) = 2^-8 |dS| + eP P (kd |dP| + |D|) + P bound(drow)

The 2^-8 |dS| term is the bf16 rounding of dS before the two MMAs; P bound(drow) is the kernel's fp32 D against the fp64 one.
2^-8 |ref| is the final bf16 rounding of each output (half an ulp of bf16 is up to 2^-8 of the value).

Choosing the constants: from the fp32 outputs of test_attention_reference_gpu.py and test_unpadded_gpu.py on an H100 SXM (80 GB
HBM3, 700 W power limit), where no bf16 rounding hides them. The largest |lse - ref| / (1 + |lse| + sum P m) was about 2^-23.3,
on the staged route (C_S = 2^-18: ~40x headroom); the largest |drow - ref| / sum |dO| |ctx| about 2^-23.4 (C_SUM = 2^-18: ~40x).
C_P and the output rounding are not measured but derived: one bf16 rounding each, so the bf16 outputs reach 0.8-0.9 of their
bound by construction. The planted bugs of test_attention_reference_cpu.py exceed these bounds by at least 2x on the input family
each shows on.
"""
import torch

REL_BF16 = 2.0 ** -8
C_P = 2.0 ** -8
C_S = 2.0 ** -18
C_SUM = 2.0 ** -18


def drop_scale(p):
    """The survivors' scale of attention dropout p: the drop probability is quantised to round(256 p) / 256."""
    if p <= 0:
        return 1.0
    return 256.0 / (256 - int(p * 256 + 0.5))


def reference(q, k, v, bias, keep, scale, dO, ctx):
    """fp64 references and bounds of one call, per head.

    q, k, v, dO, ctx: [N, S, 64] (the bf16 operands; N heads); bias: fp32 [N, S] additive key bias or None; keep: [N, S, S] 0/1
    bits the forward stored (rows = queries) or None; scale: the dropout survivors' scale (drop_scale(p)). Returns
    {name: (ref, bound)} for ctx, lse, drow, dq, dk, dv, each of the shape of the kernel output in this layout ([N, S, 64] or
    [N, S])."""
    q, k, v, dO, ctx = (x.double() for x in (q, k, v, dO, ctx))
    N, S, _ = q.shape
    b = torch.zeros(N, S, dtype=torch.float64, device=q.device) if bias is None else bias.double()
    sc = q @ k.transpose(-1, -2) / 8.0 + b[:, None, :]
    mag = q.abs() @ k.abs().transpose(-1, -2) / 8.0 + b.abs()[:, None, :]
    lse = torch.logsumexp(sc, -1)
    P = torch.exp(sc - lse[..., None])
    del sc
    kd = torch.ones_like(P) if keep is None else keep.double() * scale
    Pd = P * kd
    eP = C_P + C_S * (1.0 + mag + lse.abs()[..., None])
    out = {}
    o = Pd @ v
    ePd = eP * Pd
    out["ctx"] = (o, REL_BF16 * o.abs() + ePd @ v.abs())
    out["lse"] = (lse, C_S * (1.0 + lse.abs() + (P * mag).sum(-1)))
    del mag
    D = (dO * ctx).sum(-1)
    D_bound = C_SUM * (dO.abs() * ctx.abs()).sum(-1)
    out["drow"] = (D, D_bound)
    dv = Pd.transpose(-1, -2) @ dO
    out["dv"] = (dv, REL_BF16 * dv.abs() + ePd.transpose(-1, -2) @ dO.abs())
    del ePd, Pd
    dP = dO @ v.transpose(-1, -2)
    dS = P * (kd * dP - D[..., None])
    mds = REL_BF16 * dS.abs() + eP * P * (kd * dP.abs() + D.abs()[..., None]) + P * D_bound[..., None]
    del dP, eP, kd
    dq = dS @ k / 8.0
    dk = dS.transpose(-1, -2) @ q / 8.0
    out["dq"] = (dq, REL_BF16 * dq.abs() + mds @ k.abs() / 8.0)
    out["dk"] = (dk, REL_BF16 * dk.abs() + mds.transpose(-1, -2) @ q.abs() / 8.0)
    return out


def check(out, ref, bound, what):
    """Assert |out - ref| <= bound element by element (fp64 ref and bound of out's shape); returns the largest error / bound.
    The message names the worst element and the count outside the bound."""
    out = out.double()
    assert out.shape == ref.shape, f"{what}: shape {tuple(out.shape)} against {tuple(ref.shape)}"
    assert torch.isfinite(out).all(), f"{what}: {int((~torch.isfinite(out)).sum())} non-finite elements"
    ratio = (out - ref).abs() / (bound + 1e-300)
    worst = float(ratio.max()) if ratio.numel() else 0.0
    if worst > 1.0:
        idx = tuple(int(i) for i in torch.nonzero(ratio == ratio.max())[0])
        n_bad = int((ratio > 1).sum())
        raise AssertionError(f"{what}: {n_bad} of {ratio.numel()} elements outside the bound; worst at {idx}: "
                             f"out {float(out[idx]):.6g} ref {float(ref[idx]):.6g} bound {float(bound[idx]):.3g}")
    return worst


def check_all(outs, refs, what):
    """outs: {name: kernel output in the reference's layout}; refs: reference(). -> {name: worst error / bound}."""
    return {n: check(outs[n], *refs[n], f"{what}: {n}") for n in outs}


# ---- inputs ----------------------------------------------------------------------------------------------------------------
FAMILIES = ("unit", "peaked", "bias", "rowscale")


def inputs(family, B, S, A, dev, seed, fully_masked=False):
    """Dense-call operands of one input family: qkv [B*S, 3H] and dO [B*S, H] bf16, bias [B, S] fp32 with ragged key lengths
    (-10000 on each example's tail).

    unit:     unit-normal Q, K, V and dO; the bias is 0 or -10000.
    peaked:   Q x 4 (scores of std ~4) and +8 on one key: the last key (in the last, partial key block; these examples are
              not ragged) of even examples, so the row maximum arrives late, and key 0 of odd ones, so it arrives early.
    bias:     a general fp32 bias, N(0, 2^2) on every key plus -10000 on the tail; example 1 (B > 1) is fully masked.
    rowscale: rows of dO scaled by 2^k, k uniform in [-6, 6].
    fully_masked: example 1 gets -10000 on every key (not -inf: it attends over its raw scores)."""
    assert family in FAMILIES, family
    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    H = A * 64
    qkv = torch.randn(B * S, 3 * H, device=dev, generator=g)
    dctx = torch.randn(B * S, H, device=dev, generator=g)
    lens = torch.randint(max(1, S // 2), S + 1, (B,), device=dev, generator=g)
    bias = (torch.arange(S, device=dev)[None, :] >= lens[:, None]).float() * -10000.0
    if family == "peaked":
        qkv[:, :H] *= 4.0
        bias[0::2] = 0.0
        bias[0::2, S - 1] += 8.0
        bias[1::2, 0] += 8.0
    elif family == "bias":
        bias += 2.0 * torch.randn(B, S, device=dev, generator=g)
        fully_masked = fully_masked or B > 1
    elif family == "rowscale":
        dctx *= 2.0 ** torch.randint(-6, 7, (B * S, 1), device=dev, generator=g).float()
    if fully_masked and B > 1:
        bias[1] = torch.where(bias[1] > -5000.0, bias[1] - 10000.0, bias[1])
    return qkv.bfloat16(), bias.contiguous(), dctx.bfloat16()


# ---- layouts of the C ABI --------------------------------------------------------------------------------------------------
def dense_heads(x, B, S, A):
    """[B*S, c*A*64] rows (qkv: c = 3; ctx, dO: c = 1) -> [c, B*A, S, 64] heads."""
    c = x.shape[1] // (A * 64)
    return x.view(B, S, c, A, 64).permute(2, 0, 3, 1, 4).reshape(c, B * A, S, 64)


def varlen_heads(x, r, n, A):
    """Packed rows r .. r+n of [total, c*A*64] -> [c, A, n, 64] heads of that sequence."""
    c = x.shape[1] // (A * 64)
    return x[r:r + n].view(n, c, A, 64).permute(1, 2, 0, 3)


def keep_bits(keep, BA, S, half=0):
    """[B*A, S, S] 0/1 keep decisions from the keep buffer (laid out for S keys): half 0 = rows are queries, half 1 = its
    transpose."""
    nkb = (S + 63) // 64
    words = keep.view(torch.int64).view(2, BA, nkb * 64, nkb)[half]
    bits = (words.unsqueeze(-1) >> torch.arange(64, device=keep.device)) & 1
    return bits.reshape(BA, nkb * 64, nkb * 64)[:, :S, :S]
