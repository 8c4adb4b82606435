"""Every attention kernel against a plain fp64 restatement of the same op, through the C ABI (ctypes).

The library has three attention paths; the sequence length alone picks one:

    wgmma    S <= 192          attn_fwd_wgmma_kernel / attn_bwd_wgmma_kernel
    head     193 <= S <= 256   attn_fwd_head_kernel  / attn_bwd_head_kernel
    staged   S > 256           attn_fwd_kernel / attn_bwd_dq_kernel + attn_bwd_dkv_kernel

Each case checks ctx, lse, dQ, dK and dV separately against the reference, that every output element is written (outputs are pre-filled with NaN), that nothing is read or written
outside the tensors (they are views inside buffers whose guard bands hold NaN for inputs and a sentinel for outputs),
and that two identical calls are bit-identical. With dropout, the reference applies the bits the forward stored in the
keep buffer, so a match also shows that the forward applied exactly the stored bits.

Every output (ctx, lse, drow = rowsum(dO ctx), dQ, dK, dV) must lie within the per-element bound of attn_ref_util.py of its
fp64 reference. Besides unit-normal inputs, every route runs the input families of attn_ref_util.inputs: peaked rows (Q x 4 and a
+8 key bias that puts the row maximum in the last, partial key block or on key 0), a general fp32 key bias, and dO rows scaled
by 2^-6 .. 2^6; and the staged kernels run long key loops (S = 1024, 1025, 2049) and 16 heads (H = 1024)."""
import ctypes
import re

import pytest
import torch

import attn_ref_util as R

pytestmark = pytest.mark.gpu

GUARD_ROWS = 64    # guard rows around every [rows, cols] tensor: whole rows keep the views 16-byte aligned
GUARD_FLAT = 256   # guard elements around the [B, A, S] fp32 tensors (1 KB)
GUARD_KEEP = 1024  # guard bytes around the keep buffer
SENTINEL = -12345.0
KEEP_SENTINEL = 0xA5
P_FIRST = 0.1      # dropout of the reference comparisons (quantised to 26/256)

KERNELS = {
    "wgmma": {"attn_fwd_wgmma_kernel", "attn_delta_kernel", "attn_bwd_wgmma_kernel"},
    "head": {"attn_fwd_head_kernel", "attn_delta_kernel", "attn_bwd_head_kernel"},
    "staged": {"attn_fwd_kernel", "attn_bwd_dq_kernel", "attn_bwd_dkv_kernel"},
}


def _path(S):
    """The implementation the library picks for sequence length S."""
    return "wgmma" if S <= 192 else "head" if S <= 256 else "staged"


# sequence lengths: tile edges (1, 63/64/65, 127/128/129, 191/192), the cut-overs 192/193 and 256/257, and the staged
# kernels' stages of up to 4 key blocks: a partial and a full last block (319, 320), two stages (384), a last block of one
# row (449) and three stages (513)
SEQS = [1, 2, 17, 63, 64, 65, 100, 127, 128, 129, 164, 191, 192, 193, 200, 255, 256, 257, 319, 320, 356, 384, 449, 513]
# dropout comparisons: a partial and a full last tile per path
DROP_SEQS = [65, 128, 192, 200, 256, 257, 320, 356, 384, 513]
# persistent whole-head kernels: B*A = 288 heads, more than twice the SM count, so every CTA walks several heads
WALK = [200]
# one shape per path for the routing test
ROUTING_SEQS = [100, 200, 356]

CASES = ([(B, S, A, 0.0) for S in SEQS for B in (1, 3) for A in (1, 2, 12)]
         + [(3, S, 12, P_FIRST) for S in DROP_SEQS]
         + [(24, S, 12, p) for S in WALK for p in (0.0, P_FIRST)])
# the input families on every route: a partial and a full last key block of the wgmma and whole-head kernels, one and four
# staged key blocks with a partial last one
FAMILY_SEQS = [65, 192, 200, 256, 257, 449]
FAMILY_CASES = ([(3, S, 2, p, fam) for fam in ("peaked", "bias", "rowscale") for S in FAMILY_SEQS for p in (0.0, P_FIRST)]
                # long staged runs (16, 17 and 33 key blocks: 4, 5 and 9 stages) and 16 heads (cfg5, H = 1024)
                + [(1, 1024, 2, 0.0, "unit"), (1, 1025, 2, P_FIRST, "peaked"), (1, 2049, 2, 0.0, "peaked"),
                   (1, 2049, 2, 0.0, "bias"), (2, 164, 16, P_FIRST, "unit"), (2, 356, 16, 0.0, "unit"),
                   (2, 356, 16, P_FIRST, "peaked")])


def _setup():
    from visualbert_b200 import _lib
    return _lib, _lib.lib(), torch.device("cuda:0"), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


class _Guarded:
    """A tensor of `shape` placed in the middle of a flat buffer with `guard` elements of `fill` on each side."""

    def __init__(self, shape, dtype, guard, fill, dev):
        n = 1
        for s in shape:
            n *= s
        self.n, self.guard, self.fill = n, guard, fill
        self.buf = torch.full((n + 2 * guard,), fill, dtype=dtype, device=dev)
        self.t = self.buf[guard:guard + n].view(shape)

    def guards_intact(self):
        g = torch.cat([self.buf[:self.guard], self.buf[self.guard + self.n:]])
        if g.dtype.is_floating_point and self.fill != self.fill:
            return bool(torch.isnan(g).all())
        return torch.equal(g, torch.full_like(g, self.fill))


def _keep_bits(keep, B, S, A, half=0):
    """[B*A, S, S] 0/1 keep decisions from the keep buffer: half 0 = rows are queries, half 1 = its transpose."""
    return R.keep_bits(keep, B * A, S, half)


def _err(out, ref, scale=0.0):
    out, ref = out.double(), ref.double()
    return ((out - ref).abs().max() / max(ref.abs().max().item(), scale, 1e-30)).item()


def _inputs(B, S, A, dev, seed, fully_masked=False, family="unit"):
    """qkv, bias, dO of an input family (attn_ref_util.inputs); with `fully_masked`, example 1 has no valid key (additive
    -10000, not -inf: it attends uniformly over raw scores, M.py:1293)."""
    return R.inputs(family, B, S, A, dev, seed, fully_masked)


def _run(L, _lib, st, qkv, bias, dctx, B, S, A, p, dev, seed=99, stream=5, guarded=True):
    """One forward + backward through the C ABI. Inputs are copied into NaN-guarded buffers and outputs are NaN-filled
    views inside sentinel-guarded buffers. Returns {name: _Guarded}."""
    H = A * 64
    nan = float("nan")
    gr, gf = (GUARD_ROWS, GUARD_FLAT) if guarded else (0, 0)
    T = {
        "qkv": _Guarded((B * S, 3 * H), torch.bfloat16, gr * 3 * H, nan, dev),
        "bias": _Guarded((B, S), torch.float32, gf, nan, dev),
        "dctx": _Guarded((B * S, H), torch.bfloat16, gr * H, nan, dev),
        "ctx": _Guarded((B * S, H), torch.bfloat16, gr * H, SENTINEL, dev),
        "lse": _Guarded((B, A, S), torch.float32, gf, SENTINEL, dev),
        "dqkv": _Guarded((B * S, 3 * H), torch.bfloat16, gr * 3 * H, SENTINEL, dev),
        "drow": _Guarded((B, A, S), torch.float32, gf, SENTINEL, dev),
    }
    T["qkv"].t.copy_(qkv); T["bias"].t.copy_(bias); T["dctx"].t.copy_(dctx)
    for k in ("ctx", "lse", "dqkv", "drow"):
        T[k].t.fill_(nan)
    keep = None
    if p > 0:
        T["keep"] = _Guarded((int(L.vb_attention_keep_bytes(B, S, A)),), torch.uint8, GUARD_KEEP if guarded else 0,
                             KEEP_SENTINEL, dev)
        T["keep"].t.zero_()
        keep = T["keep"].t
    args = (ctypes.c_float(p), ctypes.c_uint64(seed), stream, st)
    P = _ptr
    _lib.check(L.vb_attention_fwd(P(T["qkv"].t), P(T["bias"].t), P(T["ctx"].t), P(T["lse"].t), P(keep), B, S, A, H, *args),
               "attn_fwd")
    _lib.check(L.vb_attention_bwd(P(T["qkv"].t), P(T["bias"].t), P(T["ctx"].t), P(T["lse"].t), P(keep), P(T["dctx"].t),
                                  P(T["dqkv"].t), P(T["drow"].t), B, S, A, H, *args), "attn_bwd")
    return T


def _check_case(B, S, A, p, seed, fully_masked, family="unit"):
    """One forward + backward against the reference, with all checks described in the module docstring. Returns the worst
    error / bound per output."""
    _lib, L, dev, st = _setup()
    H = A * 64
    where = f"{_path(S)} {family} B={B} S={S} A={A} p={p}"
    qkv, bias, dctx = _inputs(B, S, A, dev, seed, fully_masked, family)
    T = _run(L, _lib, st, qkv, bias, dctx, B, S, A, p, dev)
    T2 = _run(L, _lib, st, qkv, bias, dctx, B, S, A, p, dev, guarded=False)
    torch.cuda.synchronize()
    ctx, lse, dqkv, drow = T["ctx"].t, T["lse"].t, T["dqkv"].t, T["drow"].t

    # every element written, nothing outside the tensors read (NaN guards) or written (sentinels)
    for k in ("ctx", "lse", "dqkv", "drow"):
        assert torch.isfinite(T[k].t).all(), f"{where}: {k} has unwritten (NaN) elements"
    for k, gt in T.items():
        assert gt.guards_intact(), f"{where}: guard band of {k} changed"
    # deterministic: no atomics, so a second call gives the same bits
    for k in ("ctx", "lse", "dqkv", "drow") + (("keep",) if p > 0 else ()):
        assert torch.equal(T[k].t, T2[k].t), f"{where}: {k} differs between two identical calls"

    keep = T["keep"].t if p > 0 else None
    q, k, v = R.dense_heads(qkv, B, S, A)
    dO, c = R.dense_heads(dctx, B, S, A)[0], R.dense_heads(ctx, B, S, A)[0]
    bits = _keep_bits(keep, B, S, A) if p > 0 else None
    ref = R.reference(q, k, v, bias.repeat_interleave(A, 0), bits, R.drop_scale(p), dO, c)
    dq, dk, dv = R.dense_heads(dqkv, B, S, A)
    worst = R.check_all(dict(ctx=c, lse=lse.view(B * A, S), drow=drow.view(B * A, S), dq=dq, dk=dk, dv=dv), ref, where)
    del ref
    print(f"{where}: worst error / bound " + ", ".join(f"{n} {w:.3f}" for n, w in worst.items()))

    if p > 0:
        rate = int(p * 256 + 0.5) / 256
        if _path(S) != "staged":  # the mask kernel also writes the transpose (rows = keys); the staged path does not
            assert torch.equal(bits, _keep_bits(keep, B, S, A, half=1).transpose(1, 2)), f"{where}: transposed keep bits differ"
        assert abs(bits.float().mean().item() - (1 - rate)) < 5e-3, f"{where}: keep rate {bits.float().mean().item():.4f}"
        for kb in range((S + 63) // 64):  # per 64-key block: 6 standard deviations of a binomial rate
            blk = bits[:, :, kb * 64:(kb + 1) * 64].float()
            tol = 6 * (rate * (1 - rate) / blk.numel()) ** 0.5
            assert abs(blk.mean().item() - (1 - rate)) < tol, f"{where}: keep rate {blk.mean().item():.4f} in key block {kb}"
        o0 = R.reference(q, k, v, bias.repeat_interleave(A, 0), None, 1.0, dO, c)["ctx"][0]
        assert _err(c, o0) > 0.05, f"{where}: dropout did not change the output"
    if p > 0 and family == "unit":   # statistics sized for unit-normal rows
        # E[dropout(P)] = P: averaged over many rows the output stays close to the no-dropout one
        assert abs(c.double().mean().item() - o0.mean().item()) < 5e-3, f"{where}: mean output moved"
        # for a fixed mask the output is linear in V: <dO, O> = <dV, V>
        lhs = (dctx.double() * ctx.double()).sum().item()
        rhs = (dqkv[:, 2 * H:].double() * qkv[:, 2 * H:].double()).sum().item()
        assert abs(lhs - rhs) < 2e-2 * max(abs(lhs), 1.0) + 2.0, f"{where}: <dO, O> = {lhs} but <dV, V> = {rhs}"
    return worst


@pytest.mark.parametrize("B,S,A,p", CASES)
def test_attention_matches_reference(B, S, A, p):
    _check_case(B, S, A, p, seed=1000 * S + 10 * B + A, fully_masked=B == 3)


@pytest.mark.parametrize("B,S,A,p,family", FAMILY_CASES)
def test_attention_input_families(B, S, A, p, family):
    """Peaked rows, a general key bias and row-scaled dO on every route; long staged runs and 16 heads."""
    _check_case(B, S, A, p, seed=1000 * S + 10 * B + A + 7, fully_masked=family == "unit" and B > 1, family=family)


def test_attention_fully_masked_example_stays_finite():
    """An example whose mask is all zero gets the additive -10000 on every key (not -inf), so it attends uniformly over
    its raw scores (M.py:1293): its outputs and gradients stay finite and match the reference."""
    _check_case(2, 70, 1, 0.0, seed=6, fully_masked=True)


def test_attention_dropout_consistent_between_fwd_and_bwd():
    """p = 0.2 (quantised to 51/256): the backward applies the bits the forward stored, so dQ, dK and dV match the
    reference built from those bits; the output is linear in V for a fixed mask (<dO, O> = <dV, V>) and its mean is
    preserved."""
    _check_case(2, 100, 2, 0.2, seed=7, fully_masked=False)

@pytest.mark.parametrize("S", SEQS)
def test_attention_dropout_words_are_distinct(S):
    """At p = 0.5 a keep decision is the top bit of an 8-bit hash value, so each stored 64-bit word of a valid row
    (query < S, every key block, all 64 bits) is 64 independent random bits: two of them are equal with probability
    2^-64. A repeated word means a reused hash counter, i.e. masks that are not independent across rows or heads."""
    _lib, L, dev, st = _setup()
    B, A = 2, 2
    H = A * 64
    qkv, bias, _ = _inputs(B, S, A, dev, seed=S)
    keep = torch.zeros(int(L.vb_attention_keep_bytes(B, S, A)), device=dev, dtype=torch.uint8)
    ctx = torch.empty(B * S, H, device=dev, dtype=torch.bfloat16)
    lse = torch.empty(B, A, S, device=dev)
    P = _ptr
    _lib.check(L.vb_attention_fwd(P(qkv), P(bias), P(ctx), P(lse), P(keep), B, S, A, H, ctypes.c_float(0.5), ctypes.c_uint64(7),
                                  3, st), "attn_fwd")
    torch.cuda.synchronize()
    nkb = (S + 63) // 64
    words = keep.view(torch.int64).view(2, B * A, nkb * 64, nkb)[0, :, :S, :].reshape(-1)
    dup = words.numel() - torch.unique(words).numel()
    assert dup == 0, f"{_path(S)} S={S}: {dup} repeated keep words of {words.numel()}"
    bits = _keep_bits(keep, B, S, A).float()
    for kb in range(nkb):
        blk = bits[:, :, kb * 64:(kb + 1) * 64]
        assert abs(blk.mean().item() - 0.5) < 6 * (0.25 / blk.numel()) ** 0.5, f"S={S}: keep rate {blk.mean().item():.4f} in block {kb}"


@pytest.mark.parametrize("S", ROUTING_SEQS)
def test_attention_routing(S):
    """The kernels one forward + backward launches are those of the expected path: a change to the dispatch must not send
    every case silently to one implementation."""
    from torch.profiler import ProfilerActivity, profile
    _lib, L, dev, st = _setup()
    B, A, p = 2, 2, P_FIRST
    qkv, bias, dctx = _inputs(B, S, A, dev, seed=S)
    _run(L, _lib, st, qkv, bias, dctx, B, S, A, p, dev)   # first call: one-time setup outside the profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        _run(L, _lib, st, qkv, bias, dctx, B, S, A, p, dev)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    if not names:
        pytest.skip("torch.profiler recorded no device kernels")
    ran = {m.group(1) for n in names for m in [re.search(r"\b(attn_\w+_kernel)\b", n)] if m}
    path = _path(S)
    want = KERNELS[path] | ({"attn_keep_mask_kernel"} if path != "staged" else set())
    assert ran == want, f"S={S}: expected {sorted(want)}, ran {sorted(ran)}"

