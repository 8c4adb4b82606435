"""The layer and encoder calls on the GPU, stage by stage against fp64 (layer_ref_util.check_layer): every activation, every
scratch buffer the backward leaves, every gradient (prefilled: they must come back as prefill + result) and dx.

- Single layers through vb_layer_fwd / vb_layer_bwd, every activation and scratch buffer in its own allocation between two bands
  of 0xFF bytes (a NaN in bf16 and fp32); the inside starts as the same NaN pattern, so an element no kernel wrote fails.
- Single unpadded layers through vb_encoder_fwd_varlen / _bwd_varlen, on every attention route.
- Three layers dense (with dx, and with dx NULL, where the gradient between layers travels in scratch.d_x1), three layers unpadded
  and two dense layers in deterministic mode, through vb_encoder_fwd / vb_encoder_bwd. Layer l's input is slot l-1's y. Its
  incoming gradient comes from a separate vb_encoder_bwd over the layers above it (on the arena from slot l+1, x_in = slot l's y).
  Layer l's scratch comes from a one-layer call with that gradient, and the full call's gradients of layer l are checked
  against it.

Arena and scratch start as the NaN pattern; after the calls, the 256-byte alignment gaps between arena buffers and the bands
around every allocation must still hold it. No profiler and no model: the file sorts after the tests that count kernel records
(see test_zz_checkpointing_gpu.py)."""
import ctypes
import itertools

import pytest
import torch

import gemm_ref_util as GR
from layer_ref_util import check_layer

pytestmark = pytest.mark.gpu

BF, F32 = torch.bfloat16, torch.float32
DEV = "cuda:0"
GUARD = 4096                 # bytes of 0xFF on each side of every allocation (keeps the 256-byte alignment)
SEED = 0x0FEDCBA987654321
ARENA_SIZES = lambda M, H, A, I, keep: [M * 3 * H * 2, M * H * 2, A * M * 4, M * H * 2, M * 4, M * 4, M * H * 2, M * I * 2, M * I * 2,
                                        M * H * 2, M * 4, M * 4, keep, M * H * 2]   # vb_api.cu encoder_arena_layout


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _lib():
    from visualbert_b200 import _lib
    return _lib, _lib.lib()


class GuardedBytes:
    """n bytes between two GUARD-byte bands of 0xFF; the inside starts as 0xFF too, or as a copy of `fill`."""

    def __init__(self, n, fill=None):
        self.n = n
        self.buf = torch.full((n + 2 * GUARD,), 0xFF, dtype=torch.uint8, device=DEV)
        self.t = self.buf[GUARD:GUARD + n]
        if fill is not None:
            self.t.view(fill.dtype).copy_(fill.reshape(-1))

    def ptr(self, off=0):
        return self.t.data_ptr() + off

    def view(self, dtype, off=0, nbytes=None):
        return self.t[off:off + (self.n - off if nbytes is None else nbytes)].view(dtype)

    def check_bands(self, what):
        assert bool((self.buf[:GUARD] == 0xFF).all()) and bool((self.buf[GUARD + self.n:] == 0xFF).all()), f"{what}: guard band overwritten"


def _mask_bias(B, S, fully_masked):
    valid = torch.arange(S, device=DEV)[None, :] < torch.randint(S // 2, S + 1, (B, 1), device=DEV)
    bias = (~valid).float() * -10000.0
    if fully_masked and B > 1:
        bias[1] = -10000.0
    return bias.contiguous()


def _params(H, I):
    r = lambda *s, sc=1.0: sc * torch.randn(*s, device=DEV)
    return dict(w_qkv=r(3 * H, H, sc=0.05).to(BF), b_qkv=r(3 * H, sc=0.1), w_attn_out=r(H, H, sc=0.05).to(BF), b_attn_out=r(H, sc=0.1),
                ln1_gamma=1 + r(H, sc=0.1), ln1_beta=r(H, sc=0.1), w_inter=r(I, H, sc=0.05).to(BF), b_inter=r(I, sc=0.1),
                w_out=r(H, I, sc=0.05).to(BF), b_out=r(H, sc=0.1), ln2_gamma=1 + r(H, sc=0.1), ln2_beta=r(H, sc=0.1))


def _desc(cfg, prm, layer_index):
    _l, _ = _lib()
    mb = cfg.get("mask_bias")
    return _l.LayerDesc(batch=cfg["B"], seq=cfg["S"], hidden=64 * cfg["A"], heads=cfg["A"], inter=cfg["I"], hidden_dropout=cfg["p_h"],
                        attn_dropout=cfg["p_a"], seed=SEED, layer_index=layer_index, mask_bias=0 if mb is None else mb.data_ptr(),
                        **{k: prm[k].data_ptr() for k in prm})


def _grad_shapes(H, I):
    return dict(dw_qkv=(3 * H, H), db_qkv=(3 * H,), dw_attn_out=(H, H), db_attn_out=(H,), dln1_gamma=(H,), dln1_beta=(H,),
                dw_inter=(I, H), db_inter=(I,), dw_out=(H, I), db_out=(H,), dln2_gamma=(H,), dln2_beta=(H,))


class Grads:
    """vb_layer_grads of `n` layers over guarded fp32 buffers prefilled with random values (or zeros)."""

    def __init__(self, n, H, I, random=True):
        _l, _ = _lib()
        self.arr, self.bufs, self.prefill = (_l.LayerGrads * n)(), [], []
        for l in range(n):
            pre = {k: (torch.randn if random else torch.zeros)(*s, device=DEV) for k, s in _grad_shapes(H, I).items()}
            bufs = {k: GuardedBytes(4 * v.numel(), fill=v) for k, v in pre.items()}
            for k, b in bufs.items():
                setattr(self.arr[l], k, b.ptr())
            self.bufs.append(bufs)
            self.prefill.append(pre)

    def layer(self, l):
        return {k: b.view(F32).view(self.prefill[l][k].shape) for k, b in self.bufs[l].items()}

    def check_bands(self, what):
        for l, bufs in enumerate(self.bufs):
            for k, b in bufs.items():
                b.check_bands(f"{what} layer {l} {k}")


class Scratch:
    """vb_layer_scratch over guarded buffers holding the NaN pattern; d_pre_drop is NULL without hidden dropout."""

    def __init__(self, M, H, I, A, hd):
        _l, _ = _lib()
        sizes = dict(d_pre=M * H * 2, d_pre_drop=M * H * 2 if hd else 0, d_big=M * max(I, 3 * H) * 2, d_x1=M * H * 2, d_ctx=M * H * 2,
                     drow=A * M * 4)
        self.bufs = {k: GuardedBytes(n) for k, n in sizes.items() if n}
        self.s = _l.LayerScratch(**{k: b.ptr() for k, b in self.bufs.items()})

    def views(self):
        v = {k: b.view(F32 if k == "drow" else BF) for k, b in self.bufs.items()}
        v.setdefault("d_pre_drop", None)
        return v

    def check_bands(self, what):
        for k, b in self.bufs.items():
            b.check_bands(f"{what} scratch {k}")


def _report(what, worst):
    print(f"\n{what}: " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))


WORST = {}


def _note(worst):
    for k, v in worst.items():
        WORST[k] = max(WORST.get(k, 0.0), v)


def _check_gp_restatement(M, I):
    _, L = _lib()
    assert GR.gp_tiled_ok(M, I) == bool(L.vb_gemm_gp_tiled_ok(M, I)), f"gp_tiled_ok({M}, {I}) differs from the library"


# ---- single layers through vb_layer_fwd / vb_layer_bwd -----------------------------------------------------------------------
LAYER_CASES = [  # B, S, A, p_h, p_a, layer_index
    (3, 164, 4, 0.1, 0.1, 0),     # wgmma attention, M = 492 (a partial tile), EPI_DELTA, example 1 fully masked
    (2, 128, 4, 0.1, 0.1, 5),     # M = 256, I = 1024: tile-native gelu', EPI_DELTA
    (2, 200, 2, 0.1, 0.1, 11),    # whole-head attention, attn_delta_kernel (H = 128)
    (2, 300, 2, 0.1, 0.1, 3),     # staged attention (it computes D itself)
    (2, 164, 12, 0.0, 0.0, 0),    # base width (H = 768, I = 3072), d_pre_drop NULL, no keep buffer
    (2, 164, 4, 0.1, 0.0, 2),     # hidden dropout without attention dropout
]


@pytest.mark.parametrize("B,S,A,p_h,p_a,layer_index", LAYER_CASES)
def test_layer_call_matches_fp64_stage_by_stage(B, S, A, p_h, p_a, layer_index):
    _l, L = _lib()
    torch.manual_seed(B * 1000 + S + A + layer_index)
    H, I, M = 64 * A, 256 * A, B * S
    _check_gp_restatement(M, I)
    cfg = dict(B=B, S=S, A=A, I=I, p_h=p_h, p_a=p_a, seed=SEED, layer_index=layer_index,
               mask_bias=_mask_bias(B, S, fully_masked=layer_index == 0 and p_a > 0))
    prm = _params(H, I)
    d = _desc(cfg, prm, layer_index)
    x, dy = torch.randn(M, H, device=DEV).to(BF), torch.randn(M, H, device=DEV).to(BF)
    keep_bytes = int(L.vb_attention_keep_bytes(B, S, A)) if p_a > 0 else 0
    sizes = dict(zip(_l.ARENA_NAMES, ARENA_SIZES(M, H, A, I, keep_bytes)))
    sizes["keep"] = sizes.pop("keep_mask")
    acts = {k: GuardedBytes(n) for k, n in sizes.items() if n}
    a = _l.LayerActs(**{k: acts[k].ptr() for k in _l.ARENA_NAMES[:12]}, keep_mask=acts["keep"].ptr() if p_a > 0 else None)
    _l.check(L.vb_layer_fwd(ctypes.byref(d), ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(acts["y"].ptr()), ctypes.byref(a), _st()),
             "vb_layer_fwd")
    grads, scr, dx = Grads(1, H, I), Scratch(M, H, I, A, p_h > 0), GuardedBytes(M * H * 2)
    _l.check(L.vb_layer_bwd(ctypes.byref(d), ctypes.c_void_p(x.data_ptr()), ctypes.byref(a), ctypes.c_void_p(dy.data_ptr()),
                            ctypes.c_void_p(dx.ptr()), ctypes.byref(grads.arr[0]), ctypes.byref(scr.s), _st()), "vb_layer_bwd")
    torch.cuda.synchronize()
    what = f"layer B={B} S={S} A={A} p_h={p_h} p_a={p_a} l={layer_index}"
    for k, b in acts.items():
        b.check_bands(f"{what} acts {k}")
    scr.check_bands(what)
    grads.check_bands(what)
    dx.check_bands(what + " dx")
    av = {k: b.view(torch.uint8 if k == "keep" else F32 if k in ("lse", "mean1", "rstd1", "mean2", "rstd2") else BF)
          for k, b in acts.items()}
    worst = check_layer(cfg, prm, x, dy, av, scr.views(), grads.layer(0), grads.prefill[0], dx.view(BF), what=what)
    _note(worst)
    _report(what, worst)


# ---- encoder calls: unpadded single layers, and stacks of layers -----------------------------------------------------------
def _slot_views(arena, base, off, sizes):
    names = ("qkv", "ctx", "lse", "pre1", "mean1", "rstd1", "x1", "u", "g", "pre2", "mean2", "rstd2", "keep", "y")
    v = {}
    for i, k in enumerate(names):
        if sizes[i]:
            v[k] = arena.view(torch.uint8 if k == "keep" else F32 if k in ("lse", "mean1", "rstd1", "mean2", "rstd2") else BF,
                              base + off[i], sizes[i])
    return v


def _check_arena_gaps(arena, L, stride, off, sizes, what):
    fill = torch.full((), 0xFF, dtype=torch.uint8, device=DEV)
    for l in range(L):
        for i in range(len(sizes)):
            end = off[i + 1] if i + 1 < len(sizes) else stride
            gap = arena.t[l * stride + off[i] + sizes[i]: l * stride + end]
            assert bool((gap == fill).all()), f"{what}: slot {l}: the alignment gap after arena buffer {i} was written"
    arena.check_bands(what + " arena")


def _encoder_case(B, S, A, L, p, lens=None, with_dx=True, det=False):
    _l, lib = _lib()
    torch.manual_seed(B * 1000 + S + A + L + (len(lens) if lens else 0))
    H, I = 64 * A, 256 * A
    vl = lens is not None
    M = sum(lens) if vl else B * S
    _check_gp_restatement(M, I)
    cfg = dict(B=B, S=S, A=A, I=I, p_h=p, p_a=p, seed=SEED)
    if vl:
        cfg["lens"] = tuple(lens)
        cu = torch.tensor([0] + list(itertools.accumulate(lens)), dtype=torch.int32, device=DEV)
    else:
        cfg["mask_bias"] = _mask_bias(B, S, fully_masked=False)
    prms = [_params(H, I) for _ in range(L)]
    descs = (_l.LayerDesc * L)(*[_desc(cfg, prms[l], l) for l in range(L)])
    sub = lambda lo, hi: (_l.LayerDesc * (hi - lo))(*[descs[l] for l in range(lo, hi)])
    x, dy = torch.randn(M, H, device=DEV).to(BF), torch.randn(M, H, device=DEV).to(BF)
    off = (ctypes.c_int64 * _l.VB_ENCODER_ARENA_BUFFERS)()
    drop = 1 if p > 0 else 0
    stride = int(lib.vb_encoder_arena_layout_varlen(B, S, M, H, A, I, drop, off) if vl else lib.vb_encoder_arena_layout(B, S, H, A, I, drop, off))
    sizes = ARENA_SIZES(M, H, A, I, int(lib.vb_attention_keep_bytes(B, S, A)) if drop else 0)
    what = f"encoder B={B} S={S} A={A} L={L} p={p} lens={lens} dx={with_dx} det={det}"
    P = ctypes.c_void_p

    def fwd(arena):
        if vl:
            _l.check(lib.vb_encoder_fwd_varlen(descs, L, cu.data_ptr(), M, x.data_ptr(), arena.ptr(), _st()), "vb_encoder_fwd_varlen")
        else:
            _l.check(lib.vb_encoder_fwd(descs, L, P(x.data_ptr()), P(arena.ptr()), _st()), "vb_encoder_fwd")

    def bwd(ds, n, x_in, arena_ptr, g_in, dx_ptr, grads, scr):
        if vl:
            _l.check(lib.vb_encoder_bwd_varlen(ds, n, cu.data_ptr(), M, x_in, arena_ptr, g_in, dx_ptr, grads.arr, ctypes.byref(scr.s),
                                               _st()), "vb_encoder_bwd_varlen")
        else:
            _l.check(lib.vb_encoder_bwd(ds, n, P(x_in), P(arena_ptr), P(g_in), P(dx_ptr), grads.arr, ctypes.byref(scr.s), _st()),
                     "vb_encoder_bwd")

    det_ws = None
    if det:
        det_ws = torch.empty(max(int(lib.vb_deterministic_workspace_bytes(M, H, I, 0, 0)), 256), device=DEV, dtype=torch.uint8)
        _l.check(lib.vb_set_deterministic(det_ws.data_ptr(), det_ws.numel()), "vb_set_deterministic")
    try:
        arena = GuardedBytes(L * stride)
        fwd(arena)
        grads, scr = Grads(L, H, I), Scratch(M, H, I, A, p > 0)
        dx = GuardedBytes(M * H * 2) if with_dx else None
        bwd(descs, L, x.data_ptr(), arena.ptr(), dy.data_ptr(), dx.ptr() if with_dx else None, grads, scr)
        torch.cuda.synchronize()
        _check_arena_gaps(arena, L, stride, off, sizes, what)
        grads.check_bands(what)
        scr.check_bands(what)
        if with_dx:
            dx.check_bands(what + " dx")
        y = lambda l: arena.view(BF, l * stride + off[13], M * H * 2)
        for l in range(L - 1, -1, -1):
            x_l = x if l == 0 else y(l - 1)
            if l == L - 1:
                g_l = dy
            else:   # the gradient entering layer l: the layers above it, run on their own from slot l+1
                g_buf = GuardedBytes(M * H * 2)
                bwd(sub(l + 1, L), L - 1 - l, y(l).data_ptr(), arena.ptr((l + 1) * stride), dy.data_ptr(), g_buf.ptr(), Grads(L - 1 - l, H, I, False),
                    Scratch(M, H, I, A, p > 0))
                g_l = g_buf.view(BF)
            if l == 0:   # the full call's scratch holds layer 0's buffers
                s_l, dx_l = scr, (dx.view(BF) if with_dx else None)
            else:        # layer l alone, on its slot, with that gradient: the scratch the full call had at layer l
                s_l, dx_buf = Scratch(M, H, I, A, p > 0), GuardedBytes(M * H * 2)
                bwd(sub(l, l + 1), 1, x_l.data_ptr(), arena.ptr(l * stride), g_l.data_ptr(), dx_buf.ptr(), Grads(1, H, I, False), s_l)
                dx_l = dx_buf.view(BF)
            torch.cuda.synchronize()
            cfg["layer_index"] = l
            wl = f"{what} layer {l}"
            worst = check_layer(cfg, prms[l], x_l, g_l, _slot_views(arena, l * stride, off, sizes), s_l.views(), grads.layer(l),
                                grads.prefill[l], dx_l, what=wl)
            _note(worst)
            _report(wl, worst)
    finally:
        if det:
            lib.vb_set_deterministic(None, 0)


@pytest.mark.parametrize("lens,A", [((40, 0, 97, 63), 4), ((190, 66, 0, 128), 4), ((164, 120, 1, 227), 4), ((300, 17, 150, 0), 2)])
def test_unpadded_layer_call_matches_fp64_stage_by_stage(lens, A):
    """total 200 (attn_delta_kernel, row-major gelu', wgmma attention), 384 (EPI_DELTA with delta_seq = total), 512 (tile-native
    gelu', whole-head attention), 467 (staged attention); every set has an empty sequence or one of length 1."""
    _encoder_case(len(lens), max(lens), A, 1, 0.1, lens=lens)


@pytest.mark.parametrize("with_dx", [True, False])
def test_three_dense_layers_match_fp64_stage_by_stage(with_dx):
    _encoder_case(3, 164, 2, 3, 0.1, with_dx=with_dx)


def test_three_unpadded_layers_match_fp64_stage_by_stage():
    _encoder_case(4, 97, 2, 3, 0.1, lens=(40, 0, 97, 63))


def test_two_dense_layers_in_deterministic_mode_match_fp64_stage_by_stage():
    _encoder_case(3, 164, 2, 2, 0.1, det=True)


def test_zz_report_worst_ratios():
    """The worst error / bound per buffer over every case of this file that ran before it."""
    if WORST:
        _report("worst over all cases", WORST)
