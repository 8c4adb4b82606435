"""vb_gemm against an fp64 reference, element by element, at the shapes, layouts and epilogues where a GEMM kernel goes wrong.

Each call runs through the C ABI (ctypes). The reference is fp64 on the GPU from the exact bf16 operands, and the bound is that
of gemm_ref_util.py: one bf16 rounding plus C_ACC times the magnitude summed into the element. Every output lives inside a larger
allocation (rows before and after, row stride N + 16 g) whose bands hold a NaN bit pattern that must survive the call. bf16
outputs are prefilled with the same pattern in range, so an element the kernel skips shows up as a NaN; fp32 outputs accumulate,
so they are prefilled with known random values C and must come back as C + A B (+ bias once).

torch.profiler records which gemm_wgmma_kernel<A_MN, B_MN, BLOCK_N, OUT_F32, EPI> each call launched and its grid: tiles x
split-K factor, the factor restated from vb_gemm.cu::wgrad_splits with this device's SM count. Split-K shapes are chosen at run
time so that the factor is >= 2 and does not divide the k-blocks.

Bitwise comparisons are made only where the arithmetic is identical by construction: the tile-native and row-major gelu'(u),
EPI_DELTA's D and the plain call's, dropped elements (0 + addend rounds to the addend) and two identical calls.
"""
import ctypes
import json
import re
import time

import pytest
import torch

from dropout_util import hidden_keep
from gemm_ref_util import (GELU_APPROX,GELU_LIP, check_close, check_dropout, expected_kernel, gelu64, gelu_prime64,
                           tiles, untile, wgrad_splits)

pytestmark = pytest.mark.gpu

BF, F32 = torch.bfloat16, torch.float32
NAN16, NAN32 = 0x7FA5, 0x7FBADBAD   # bf16 / fp32 NaN bit patterns of the guard bands
GELU, DGELU = 1, 2                  # VB_EPI_*
SEED_HI = 0xFEDCBA9876543210        # a dropout seed with the high bits set
WORST = {}                          # case family -> largest error / bound seen


def _dev():
    return torch.device("cuda:0")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _note(family, ratio):
    WORST[family] = max(WORST.get(family, 0.0), ratio)


def _report(families):
    print("\n" + "  ".join(f"{f}: {WORST[f]:.3g}" for f in families if f in WORST))


def _call(**kw):
    from visualbert_b200 import _lib
    a = _lib.GemmArgs()
    for k, v in kw.items():
        setattr(a, k, v)
    _lib.check(_lib.lib().vb_gemm(ctypes.byref(a), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "vb_gemm")


class Guarded:
    """rows x cols output inside a [lead + rows + tail, cols + 16 g] allocation prefilled with a NaN bit pattern; `fill`
    (if given) replaces the pattern in range."""

    def __init__(self, rows, cols, dtype, g=1, lead=2, tail=3, fill=None):
        self.ld = cols + 16 * g
        self.it, self.pat = (torch.int16, NAN16) if dtype == BF else (torch.int32, NAN32)
        self.buf = torch.full((lead + rows + tail, self.ld), self.pat, dtype=self.it, device=_dev()).view(dtype)
        self.t = self.buf[lead:lead + rows, :cols]
        if fill is not None:
            self.t.copy_(fill)
        self.inside = torch.zeros(self.buf.shape, dtype=torch.bool, device=_dev())
        self.inside[lead:lead + rows, :cols] = True

    def ptr(self):
        return self.t.data_ptr()

    def check_bands(self, what):
        n = int((self.buf.view(self.it)[~self.inside] != self.pat).sum())
        assert n == 0, f"{what}: {n} elements written outside the output"


def _operand(rows, cols, pad, scale=1.0):
    """bf16 [rows, cols] view of a [rows, ld] allocation, ld = cols rounded up to 8, plus pad."""
    ld = (cols + 7) // 8 * 8 + pad
    return (scale * torch.randn(rows, ld, device=_dev())).to(BF)[:, :cols], ld


def _sample_rows(M, n_random=256):
    if M <= 512:
        return None
    g = torch.Generator().manual_seed(M)
    mid = torch.randperm(M - 256, generator=g)[:n_random] + 128
    return torch.cat([torch.arange(128), mid.sort().values, torch.arange(M - 128, M)]).to(_dev())


# torch.profiler can lose the kernel records nearest the edges of its capture window (the first kernel of a short window,
# or the whole of one): each counted window starts after the device is idle and leaves host time at both ends
PROFILE_PAD_S = 0.05


class Launches:
    """Profiles a block of vb_gemm calls and checks, in launch order, the template arguments and grid of every
    gemm_wgmma_kernel against `expected` ((case, (A_MN, B_MN, BLOCK_N, OUT_F32, EPI), grid) per call)."""

    def __init__(self, tmp_path):
        self.expected = []
        self.trace = tmp_path / "gemm_trace.json"

    def __enter__(self):
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.synchronize()
        self.prof = profile(activities=[ProfilerActivity.CUDA])
        self.prof.__enter__()
        time.sleep(PROFILE_PAD_S)
        return self

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        time.sleep(PROFILE_PAD_S)
        self.prof.__exit__(*exc)
        if exc[0] is not None:
            return False
        self.prof.export_chrome_trace(str(self.trace))
        events = json.loads(self.trace.read_text())["traceEvents"]
        ks = sorted((e for e in events if e.get("cat") == "kernel" and "gemm_wgmma_kernel" in e.get("name", "")), key=lambda e: e["ts"])
        assert len(ks) == len(self.expected), f"{len(ks)} gemm_wgmma_kernel launches recorded for {len(self.expected)} vb_gemm calls"
        for e, (case, want, grid) in zip(ks, self.expected):
            m = re.search(r"gemm_wgmma_kernel<(\w+), (\w+), (\d+), (\w+), (\d+)>", e["name"])
            assert m, e["name"]
            got = (m.group(1) == "true", m.group(2) == "true", int(m.group(3)), m.group(4) == "true", int(m.group(5)))
            assert got == want, f"{case}: launched {got}, expected {want}"
            assert e["args"]["grid"][0] == grid, f"{case}: grid {e['args']['grid']}, expected {grid}"
        return False


def run(launches, family, M, N, K, *, a_mn=0, b_mn=0, f32=False, bias=False, add=False, epi=0, drop=None, pad=8, g=1,
        gp_tiled=False, aux_in=None, A=None, seed=0, rows="auto"):
    """One vb_gemm call checked against the fp64 reference. drop = (p, seed, stream); aux_in = (tensor, ld, row-major
    gelu'(u)) for the DGELU epilogue (random when None); A = (logical [M, K] view, lda) overrides the random A.
    Returns the outputs (and the keep mask under dropout)."""
    dev = _dev()
    torch.manual_seed(seed)
    case = f"M={M} N={N} K={K} a_mn={a_mn} b_mn={b_mn} f32={f32} bias={bias} add={add} epi={epi} drop={drop} tiled={gp_tiled}"
    if A is None:
        At, lda = _operand(K, M, pad) if a_mn else _operand(M, K, pad)
        A_log = At.t() if a_mn else At
    else:
        A_log, lda = A
    Bt, ldb = _operand(K, N, pad, 0.05) if b_mn else _operand(N, K, pad, 0.05)
    B_log = Bt.t() if b_mn else Bt
    kw = dict(A=A_log.data_ptr(), lda=lda, a_mn_major=a_mn, B=Bt.data_ptr(), ldb=ldb, b_mn_major=b_mn, M=M, N=N, K=K)
    bias_t = torch.randn(N, device=dev) if bias else None
    if bias:
        kw.update(bias=bias_t.data_ptr())
    add_t = None
    if add:
        add_t, ld_add = _operand(M, N, 16 * g)
        kw.update(addend=add_t.data_ptr(), ld_add=ld_add)
    aux_out = aux_ref = None
    if epi == GELU:
        aux_out = Guarded(M, N, BF, g)
        kw.update(epilogue=GELU, aux_out=aux_out.ptr(), ld_aux=aux_out.ld, gp_tiled=int(gp_tiled))
    elif epi == DGELU:
        if aux_in is None:
            t, ld = _operand(M, N, 16 * g)
            t.uniform_(-0.17, 1.13)
            aux_in = (t, ld, t)
        kw.update(epilogue=DGELU, aux_in=aux_in[0].data_ptr(), ld_aux=aux_in[1], gp_tiled=int(gp_tiled))
        aux_ref = aux_in[2]
    if drop is not None:
        kw.update(dropout_p=drop[0], dropout_seed=drop[1], dropout_stream=drop[2])
    C = torch.randn(M, N, device=dev) if f32 else None
    D = Guarded(M, N, F32 if f32 else BF, 0 if gp_tiled else g, fill=C)
    _call(D=D.ptr(), ldd=D.ld, d_fp32=int(f32), **kw)
    n_tiles = tiles(M, N)
    splits = wgrad_splits(n_tiles, (K + 63) // 64, _sms()) if f32 else 1
    launches.expected.append((case, expected_kernel(M, N, a_mn=a_mn, b_mn=b_mn, f32=f32, epi=epi, add=add, drop=drop is not None,
                                                    gp_tiled=gp_tiled), n_tiles * splits))
    torch.cuda.synchronize()
    D.check_bands(case + " D")
    assert torch.isfinite(D.t).all(), f"{case}: D has elements the call did not write"
    if aux_out is not None:
        aux_out.check_bands(case + " aux_out")
        assert torch.isfinite(aux_out.t).all(), f"{case}: aux_out has elements the call did not write"

    r = _sample_rows(M) if rows == "auto" else rows
    sel = (lambda t: t) if r is None else (lambda t: t[r])
    a64, b64 = sel(A_log).double(), B_log.double()
    acc, mag = a64 @ b64.t(), a64.abs() @ b64.abs().t()
    if bias:
        acc, mag = acc + bias_t.double(), mag + bias_t.double().abs()
    d_rm = untile(D.t, M, N) if gp_tiled and epi == GELU else D.t
    out = {"D": D.t, "D_rowmajor": d_rm, "aux_out": aux_out.t if aux_out is not None else None, "splits": splits}
    if f32:
        c64 = sel(C).double()
        ratio = check_close(sel(D.t), c64 + acc, c64.abs() + mag, False, case)
    elif epi == GELU:
        approx = GELU_APPROX * (1.0 + acc.abs())
        ratio = max(check_close(sel(d_rm), gelu_prime64(acc), GELU_LIP * mag, True, case + " gelu'(u)", approx),
                    check_close(sel(aux_out.t), gelu64(acc), GELU_LIP * mag, True, case + " gelu(u)", approx))
    elif epi == DGELU:
        x = sel(aux_ref).double()
        ratio = check_close(sel(D.t), acc * x, mag * x.abs(), True, case)
    elif drop is not None:
        keep, scale = hidden_keep(drop[1], drop[2], M, N, drop[0], dev)
        ratio = check_dropout(sel(D.t), acc, mag, sel(keep), scale, sel(add_t) if add else None, case)
        out["keep"] = keep
    else:
        a = sel(add_t).double() if add else 0.0
        ratio = check_close(sel(D.t), acc + a, mag + (a.abs() if add else 0.0), True, case)
    _note(family, ratio)
    return out


TILE_EDGES = [(1, 16, 8), (64, 112, 48), (127, 128, 64), (128, 144, 72), (129, 240, 200), (255, 256, 768), (300, 272, 3072),
              (1000, 384, 72), (129, 768, 8), (64, 2304, 200), (127, 3072, 48), (1000, 2304, 768), (300, 16, 3072),
              (300, 2112, 200)]   # the last: a partial last 256-wide tile


def test_tile_edges(tmp_path):
    """Every residue class of M, N and K at the 128-row tile, both tile widths and the 64-wide k-slab; bf16 output with bias and
    residual, and fp32 accumulating output with bias; operand, addend and output strides wider than their widths."""
    with Launches(tmp_path) as rec:
        for M, N, K in TILE_EDGES:
            run(rec, "tile edges bf16", M, N, K, bias=True, add=True, seed=M + N + K)
            run(rec, "tile edges fp32", M, N, K, f32=True, bias=True, seed=M + N + K + 1)
    _report(["tile edges bf16", "tile edges fp32"])


def test_every_epilogue(tmp_path):
    """Each specialised epilogue of the 256-wide tile and the generic one: bias, residual with and without bias, GELU and
    DGELU on both tile widths and both B layouts, dropout without an addend on both tile widths, residual on 128-wide tiles."""
    M, K = 300, 200
    with Launches(tmp_path) as rec:
        for b_mn in (0, 1):
            run(rec, "epilogues", M, 768, K, b_mn=b_mn, bias=True, seed=1)                       # EPI_BIAS
            run(rec, "epilogues", M, 768, K, b_mn=b_mn, bias=True, add=True, seed=2)             # EPI_RESID
            run(rec, "epilogues", M, 1024, K, b_mn=b_mn, add=True, g=2, seed=3)                  # EPI_RESID, no bias
            for N in (768, 384):
                run(rec, "gelu", M, N, K, b_mn=b_mn, bias=True, epi=GELU, seed=4)             # GELU_FWD / generic
                run(rec, "epilogues", M, N, K, b_mn=b_mn, epi=DGELU, seed=5)                 # DGELU_BWD / generic
                run(rec, "dropout kept", M, N, K, b_mn=b_mn, bias=True, drop=(0.1, SEED_HI, 9), seed=6)   # generic
            run(rec, "epilogues", M, 144, K, b_mn=b_mn, add=True, seed=7)                       # generic residual
    _report(["epilogues", "gelu", "dropout kept"])


def test_every_layout(tmp_path):
    """All four (a_mn_major, b_mn_major) layouts x bf16 / fp32 output x 128 / 256-wide tiles, with strided operands; a K-major
    A that is a column slice of a wider tensor (K of qkv, lda = 3 H)."""
    M, K = 200, 136
    with Launches(tmp_path) as rec:
        for a_mn in (0, 1):
            for b_mn in (0, 1):
                for N in (384, 512):
                    run(rec, "layouts fp32", M, N, K, a_mn=a_mn, b_mn=b_mn, f32=True, bias=N == 512, pad=24, seed=a_mn + 2 * b_mn)
                    if a_mn == 0 and N == 512:   # K-major A on 256-wide tiles: the generic kernel serves dropout alone
                        run(rec, "dropout kept", M, N, K, b_mn=b_mn, bias=True, drop=(0.5, 3, 1), pad=24, seed=4)
                    else:
                        run(rec, "layouts bf16", M, N, K, a_mn=a_mn, b_mn=b_mn, bias=True, add=True, pad=24, seed=5)
        H = 768
        qkv = torch.randn(M, 3 * H, device=_dev()).to(BF)
        for N, f32 in ((768, False), (2304, True), (384, False)):
            run(rec, "layouts bf16" if not f32 else "layouts fp32", M, N, H, A=(qkv[:, H:2 * H], 3 * H), f32=f32, bias=True, seed=6)
    _report(["layouts bf16", "layouts fp32", "dropout kept"])


def _uneven_split_k(M, N, k_lo):
    """Smallest K >= k_lo with K % 64 != 0 whose split-K factor on this device is >= 2 and leaves an uneven partition."""
    for K in range(k_lo, k_lo + 64 * 256, 8):
        kb = (K + 63) // 64
        s = wgrad_splits(tiles(M, N), kb, _sms())
        if K % 64 and s >= 2 and kb % s:
            return K
    raise AssertionError(f"no uneven split-K shape for M={M} N={N} on {_sms()} SMs")


def test_split_k(tmp_path):
    """fp32 accumulating outputs whose k-range is cut into splits: uneven partitions with a partial last k-block, bias added
    once, accumulation into a prefilled D; the weight-gradient shapes of the layer and the MLM decoder's dE."""
    table = []
    with Launches(tmp_path) as rec:
        cases = [(256, 256, 1, 1, True), (300, 144, 0, 0, False), (129, 272, 1, 0, True), (64, 768, 0, 1, True),
                 (2304, 768, 1, 1, False), (3072, 768, 1, 1, True), (768, 3072, 1, 1, False)]   # the last three: dw_qkv, dw_inter, dw_out
        for M, N, a_mn, b_mn, bias in cases:
            K = _uneven_split_k(M, N, 2000 if M * N > 10 ** 6 else 300)
            o = run(rec, "split-K", M, N, K, a_mn=a_mn, b_mn=b_mn, f32=True, bias=bias, seed=M + N)
            assert o["splits"] >= 2
            table.append((M, N, K, tiles(M, N), o["splits"]))
        for K in (5, 300):   # MLM decoder dE = dlogits^T t: A = dlogits [n, Vp] (lda = Vp), B = t [n, 768]
            o = run(rec, "split-K", 30522, 768, K, a_mn=1, b_mn=1, f32=True, pad=0, seed=K)
            table.append((30522, 768, K, tiles(30522, 768), o["splits"]))
    print(f"\n{_sms()} SMs: " + "; ".join(f"M={M} N={N} K={K}: {t} tiles x {s} splits = grid {t * s}" for M, N, K, t, s in table))
    _report(["split-K"])


@pytest.mark.parametrize("p", [1 / 256, 0.1, 0.5, 0.99])
def test_dropout_mask_is_exact_and_matches_layernorm_backward(p, tmp_path):
    """Dropout in the residual epilogue (256-wide EPI_DROP_RESID) and the generic one (128-wide): kept elements within the
    bound of (acc + bias) * scale + addend, dropped elements equal to the addend bit for bit, two identical calls bit-equal.
    vb_layernorm_bwd with the same (p, seed, stream, rows, H) regenerates the mask: its dx_drop is zero exactly where the GEMM
    dropped (and where dx itself is zero) and nowhere else."""
    from visualbert_b200 import _lib
    L = _lib.lib()
    dev = _dev()
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    M, K = 300, 200
    with Launches(tmp_path) as rec:
        for N in (768, 384):
            for stream in (0, 5, 0xFFFFFFFF):
                o = run(rec, "dropout kept", M, N, K, bias=True, add=True, drop=(p, SEED_HI, stream), seed=stream % 97)
                o2 = run(rec, "dropout kept", M, N, K, bias=True, add=True, drop=(p, SEED_HI, stream), seed=stream % 97)
                assert torch.equal(o["D"].view(torch.int16), o2["D"].view(torch.int16)), "two identical calls differ"
                keep = o["keep"]
                x = torch.randn(M, N, device=dev).to(BF)
                dy = (torch.randn(M, N, device=dev).sign() * (0.5 + torch.rand(M, N, device=dev))).to(BF)
                mean, rstd, gamma = torch.zeros(M, device=dev), torch.ones(M, device=dev), 1 + 0.1 * torch.rand(N, device=dev)
                dx, dx_drop = torch.empty(M, N, device=dev, dtype=BF), torch.empty(M, N, device=dev, dtype=BF)
                P = lambda t: ctypes.c_void_p(t.data_ptr())
                _lib.check(L.vb_layernorm_bwd(P(dy), P(x), P(mean), P(rstd), P(gamma), P(dx), P(dx_drop), None, None, None, M, N,
                                              ctypes.c_float(p), ctypes.c_uint64(SEED_HI), ctypes.c_uint32(stream), ctypes.c_float(0.0),
                                              ctypes.c_uint32(0), st), "vb_layernorm_bwd")
                torch.cuda.synchronize()
                assert (dx != 0).float().mean().item() > 0.99
                assert torch.equal(dx_drop == 0, ~keep | (dx == 0)), f"N={N} stream={stream}: the LayerNorm backward's mask differs"
    _report(["dropout kept"])


@pytest.mark.parametrize("M,N", [(768, 3072), (1024, 1024)])
def test_tile_native_gelu_prime(M, N, tmp_path):
    """gp_tiled over several 256-row and 256-column blocks: GELU_FWD_T stores the same gelu(u) as GELU_FWD and a permutation
    of its gelu'(u); DGELU_BWD_T on that permutation equals DGELU_BWD on the row-major one, bit for bit."""
    K = 768
    with Launches(tmp_path) as rec:
        f = run(rec, "gelu", M, N, K, bias=True, epi=GELU, g=0, seed=1)
        t = run(rec, "gelu", M, N, K, bias=True, epi=GELU, gp_tiled=True, g=0, seed=1)
        assert torch.equal(t["aux_out"].view(torch.int16), f["aux_out"].view(torch.int16))
        assert torch.equal(t["D_rowmajor"].view(torch.int16), f["D"].view(torch.int16))
        d = run(rec, "epilogues", M, N, K, b_mn=1, epi=DGELU, aux_in=(f["D"], N, f["D"]), seed=2)
        dt = run(rec, "epilogues", M, N, K, b_mn=1, epi=DGELU, gp_tiled=True, aux_in=(t["D"], N, f["D"]), seed=2)
        assert torch.equal(dt["D"].view(torch.int16), d["D"].view(torch.int16))
    _report(["gelu", "epilogues"])


def _delta_case(rec, Bsz, S, N, K=768, seed=0):
    """EPI_DELTA: D must equal the plain call's bit for bit, delta_out[b][h][s] the fp64 sum over the head of the STORED D
    times ctx, and nothing outside delta_out may change."""
    M, dev = Bsz * S, _dev()
    plain = run(rec, "delta D", M, N, K, b_mn=1, seed=seed)
    torch.manual_seed(seed)
    At, lda = _operand(M, K, 8)
    Bt, ldb = _operand(K, N, 8, 0.05)
    ctx = torch.randn(M, N, device=dev).to(BF)
    D = Guarded(M, N, BF)
    delta = Guarded(Bsz * (N // 64), S, F32, g=0)
    _call(A=At.data_ptr(), lda=lda, B=Bt.data_ptr(), ldb=ldb, b_mn_major=1, M=M, N=N, K=K, D=D.ptr(), ldd=D.ld,
          delta_ctx=ctx.data_ptr(), delta_out=delta.ptr(), delta_seq=S)
    case = f"delta B={Bsz} S={S} N={N}"
    rec.expected.append((case, expected_kernel(M, N, b_mn=1, delta=True), tiles(M, N)))
    torch.cuda.synchronize()
    D.check_bands(case + " D")
    delta.check_bands(case + " delta_out")
    assert torch.equal(D.t.view(torch.int16), plain["D"].view(torch.int16)), f"{case}: D differs from the plain call"
    prod = D.t.double() * ctx.double()
    ref = prod.view(Bsz, S, N // 64, 64).sum(-1).permute(0, 2, 1).reshape(Bsz * (N // 64), S)
    mag = prod.abs().view(Bsz, S, N // 64, 64).sum(-1).permute(0, 2, 1).reshape(Bsz * (N // 64), S)
    _note("delta", check_close(delta.t, ref, mag, False, case))


def test_attention_delta_epilogue(tmp_path):
    """EPI_DELTA with M not a multiple of 128, a partial last 256-wide tile (N = 1216) and the varlen form (delta_seq = M)."""
    with Launches(tmp_path) as rec:
        for Bsz, S, N in ((5, 56, 768), (3, 100, 1216), (2, 164, 768), (2, 164, 1216), (1, 300, 768), (1, 300, 1216)):
            _delta_case(rec, Bsz, S, N, seed=S + N)
    _report(["delta D", "delta"])


def test_benchmark_rows(tmp_path):
    """One call per specialised epilogue at the benchmark's M = 41 984 (256 x 164 rows); the reference covers the first and the
    last 128-row tile and 256 random rows."""
    M, H, I = 41984, 768, 3072
    with Launches(tmp_path) as rec:
        run(rec, "benchmark rows", M, 3 * H, H, bias=True, g=0, seed=1)                               # EPI_BIAS (QKV)
        run(rec, "benchmark rows", M, H, H, bias=True, add=True, seed=2)                              # EPI_RESID
        run(rec, "benchmark rows", M, H, I, bias=True, add=True, drop=(0.1, SEED_HI, 10), seed=3)     # EPI_DROP_RESID
        f = run(rec, "benchmark rows", M, I, H, bias=True, epi=GELU, g=0, seed=4)                     # EPI_GELU_FWD
        t = run(rec, "benchmark rows", M, I, H, bias=True, epi=GELU, gp_tiled=True, g=0, seed=4)      # EPI_GELU_FWD_T
        assert torch.equal(t["aux_out"].view(torch.int16), f["aux_out"].view(torch.int16))
        assert torch.equal(t["D_rowmajor"].view(torch.int16), f["D"].view(torch.int16))
        del t["aux_out"], f["aux_out"], t["D_rowmajor"]
        d = run(rec, "benchmark rows", M, I, H, b_mn=1, epi=DGELU, aux_in=(f["D"], I, f["D"]), g=0, seed=5)        # EPI_DGELU_BWD
        dt = run(rec, "benchmark rows", M, I, H, b_mn=1, epi=DGELU, gp_tiled=True, aux_in=(t["D"], I, f["D"]), g=0, seed=5)
        assert torch.equal(dt["D"].view(torch.int16), d["D"].view(torch.int16))                                  # EPI_DGELU_BWD_T
        del f, t, d, dt
        _delta_case(rec, 256, 164, H, seed=6)                                                                    # EPI_DELTA
    _report(["benchmark rows", "delta"])
