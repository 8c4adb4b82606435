"""Reference arithmetic and the error bound of the vb_gemm tests (test_gemm_reference_gpu.py, test_gemm_reference_cpu.py).

Every reference is fp64, computed from the exact bf16 operands. An output element passes when

    |out - ref| <= REL_BF16 * |ref| + C_ACC * mag + approx

- REL_BF16 = 2^-8 is one rounding to bf16 (bf16 outputs only; 0 for fp32 outputs).
- mag is the fp64 magnitude of everything summed into the element: (|A| |B|)_ij, plus |bias|, |addend|, the prefilled |C| of an
  accumulating fp32 output, times the dropout scale or |gelu'(u)| where the epilogue multiplies. C_ACC * mag covers the fp32
  accumulation of the tensor cores, the fp32 epilogue arithmetic and, for split-K, one red.add rounding per split.
- Through the GELU epilogue the bound of u = acc + bias is multiplied by GELU_LIP >= max |gelu'| (and >= max |gelu''| for the
  stored gelu'(u)), and approx = GELU_APPROX * (1 + |u|) covers the fp32 erf approximation of the kernel.

C_ACC was chosen from the measured error: over every fp32-output case of test_gemm_reference_gpu.py on an H100 SXM (80 GB HBM3,
700 W power limit) the largest |out - ref| / mag was 3.1e-7 (about 2^-21.6, tile-edge cases with K = 3072). C_ACC = 2^-16 leaves
a factor of ~50 and still rejects, by orders of magnitude, a lost 64-wide k-slab, a misplaced 16-column chunk, a bias added
twice and a flipped dropout bit (test_gemm_reference_cpu.py).
"""
import math

import torch

REL_BF16 = 2.0 ** -8
C_ACC = 2.0 ** -16
GELU_LIP = 1.13
GELU_APPROX = 2.0 ** -17

BLOCK_M, BLOCK_K = 128, 64
EPI_GENERIC, EPI_BIAS, EPI_RESID, EPI_DROP_RESID, EPI_GELU_FWD, EPI_DGELU_BWD, EPI_GELU_FWD_T, EPI_DGELU_BWD_T, EPI_DELTA = range(9)
# the specialised 256-wide bf16 kernels vb_gemm instantiates, per B layout (A is K-major for all of them)
SPECIALISED = {0: {EPI_BIAS, EPI_RESID, EPI_DROP_RESID, EPI_GELU_FWD, EPI_GELU_FWD_T},
               1: {EPI_BIAS, EPI_RESID, EPI_DGELU_BWD, EPI_DGELU_BWD_T, EPI_DELTA}}


def bound(ref, mag, bf16_out, approx=None):
    b = C_ACC * mag
    if bf16_out:
        b = b + REL_BF16 * ref.abs()
    if approx is not None:
        b = b + approx
    return b


def check_close(out, ref, mag, bf16_out, what, approx=None):
    """Assert |out - ref| <= bound element by element (out: any float dtype; ref, mag: fp64 of the same shape).
    Returns the largest |out - ref| / bound."""
    out = out.double()
    assert torch.isfinite(out).all(), f"{what}: {int((~torch.isfinite(out)).sum())} non-finite elements"
    err = (out - ref).abs()
    b = bound(ref, mag, bf16_out, approx) + 1e-300
    ratio = err / b
    worst = float(ratio.max()) if ratio.numel() else 0.0
    if worst > 1.0:
        idx = tuple(int(i) for i in torch.nonzero(ratio == ratio.max())[0])
        n_bad = int((ratio > 1).sum())
        raise AssertionError(f"{what}: {n_bad} of {ratio.numel()} elements outside the bound; worst at {idx}: "
                             f"out {float(out[idx]):.6g} ref {float(ref[idx]):.6g} bound {float(b[idx]):.3g}")
    return worst


def check_dropout(out, acc, mag, keep, scale, addend, what):
    """Dropout epilogue D = keep ? (acc + bias) * scale + addend : addend, bf16 output. acc: fp64 acc + bias, mag: its
    magnitude, addend: the bf16 addend or None. Kept elements must be within the bound; dropped ones equal the addend bit for
    bit (0 + addend rounds to the addend; +0 without one). Returns the largest error / bound of the kept elements."""
    add64 = addend.double() if addend is not None else torch.zeros_like(acc)
    ref = acc * scale + add64
    m = mag * scale + add64.abs()
    worst = check_close(out[keep], ref[keep], m[keep], True, what + " (kept)")
    want = addend[~keep] if addend is not None else torch.zeros_like(out[~keep])
    got = out[~keep]
    n_bad = int((got.view(torch.int16) != want.view(torch.int16)).sum())
    assert n_bad == 0, f"{what}: {n_bad} of {got.numel()} dropped elements differ from the addend"
    return worst


def gelu64(u):
    return 0.5 * u * (1.0 + torch.erf(u / math.sqrt(2.0)))


def gelu_prime64(u):
    return 0.5 * (1.0 + torch.erf(u / math.sqrt(2.0))) + u * torch.exp(-0.5 * u * u) / math.sqrt(2.0 * math.pi)


def gp_tiled_ok(M, N):
    """Restatement of vb_gemm.cu::gemm_gp_tiled_ok: the shapes whose gelu'(u) can be stored tile-native."""
    return M >= 256 and M % 256 == 0 and N % 256 == 0


def untile(t, M, N):
    """tile-native gelu'(u) (vbert_b200.h, vb_gemm_args.gp_tiled) -> row-major [M, N]"""
    return t.reshape(M // 256, N // 256, 2, 2, 4, 8, 32, 16).permute(0, 2, 4, 6, 1, 3, 5, 7).reshape(M, N)


def tile_n(N):
    """vb_gemm's tile width: 256 unless N is small or padding N to a multiple of 256 wastes more than 1/8 of the columns."""
    pad = (N + 255) // 256 * 256 - N
    return 256 if N >= 256 and pad * 8 <= N else 128


def tiles(M, N):
    bn = tile_n(N)
    return ((M + BLOCK_M - 1) // BLOCK_M) * ((N + bn - 1) // bn)


def wgrad_splits(n_tiles, k_blocks, sms):
    """Restatement of vb_gemm.cu::wgrad_splits: the split-K factor of an fp32 output, the smallest s <= min(k_blocks, 32) that
    minimises waves * (k-blocks per split + 4)."""
    best, best_cost = 1, None
    for s in range(1, min(k_blocks, 32) + 1):
        cost = -(-n_tiles * s // sms) * (-(-k_blocks // s) + 4)
        if best_cost is None or cost < best_cost:
            best, best_cost = s, cost
    return best


def expected_kernel(M, N, *, a_mn=0, b_mn=0, f32=False, epi=0, add=False, drop=False, gp_tiled=False, delta=False):
    """Template arguments <A_MN, B_MN, BLOCK_N, OUT_F32, EPI> of the gemm_wgmma_kernel a vb_gemm call must launch.
    epi: 0 none, 1 GELU, 2 DGELU (VB_EPI_*)."""
    bn = tile_n(N)
    e = EPI_GENERIC
    if bn == 256 and not f32 and not a_mn:
        if delta:
            e = EPI_DELTA
        elif epi == 1:
            e = EPI_GELU_FWD_T if gp_tiled else EPI_GELU_FWD
        elif epi == 2:
            e = EPI_DGELU_BWD_T if gp_tiled else EPI_DGELU_BWD
        else:
            e = (EPI_DROP_RESID if drop else EPI_RESID) if add else (EPI_GENERIC if drop else EPI_BIAS)
        if e not in SPECIALISED[b_mn]:
            e = EPI_GENERIC
    return (bool(a_mn), bool(b_mn), bn, bool(f32), e)
