"""CPU-side checks of the forward-only encoder call (vb_encoder_infer, vb_encoder_infer_varlen, vb_encoder_infer_workspace) and
of the VB_EPI_GELU_FWD epilogue selector: exported without an ABI bump, workspace sized below one arena slot, and bad arguments
refused through vb_last_error before anything reaches a device (the pointers below are never dereferenced)."""
import ctypes

import pytest

from visualbert_b200 import _lib

FAKE = 0x10000   # 32-byte aligned, non-null
_GEMM = dict(A=0x10000, lda=256, B=0x20000, ldb=256, M=256, N=256, K=256, D=0x30000, ldd=256)


def _refused(rc, what):
    assert rc != 0
    msg = _lib.lib().vb_last_error()
    assert what in msg, msg


def test_infer_entry_points_exported_without_an_abi_bump():
    L = _lib.lib()
    names = {"vb_encoder_infer_workspace", "vb_encoder_infer", "vb_encoder_infer_varlen"}
    assert names <= set(_lib.EXPORTS) and all(hasattr(L, n) for n in names)
    assert L.vb_abi_version() == _lib.ABI_VERSION == 4
    assert _lib.VB_EPI_GELU_FWD == 4


@pytest.mark.parametrize("shape", [(4, 56, 768, 12, 3072), (256, 164, 768, 12, 3072), (64, 356, 1024, 16, 4096), (3, 17, 128, 2, 64)])
@pytest.mark.parametrize("drop", [0, 1])
def test_workspace_is_aligned_and_no_larger_than_an_arena_slot(shape, drop):
    L = _lib.lib()
    B, S, H, A, I = shape
    M = B * S
    ws = L.vb_encoder_infer_workspace(B, S, H, A, I, drop, -1)
    stride = L.vb_encoder_arena_layout(B, S, H, A, I, drop, None)
    assert ws % 256 == 0 and 0 < ws <= stride
    # qkv, ctx, one pre-LayerNorm buffer, x1, gelu(u), two ping-pong outputs (+ the keep bits): nothing else
    need = M * 3 * H * 2 + 5 * M * H * 2 + M * I * 2 + (L.vb_attention_keep_bytes(B, S, A) if drop else 0)
    assert need <= ws <= need + 8 * 256
    # packed rows: fewer rows, smaller workspace, still below the varlen arena slot
    total = M - M // 3
    wsp = L.vb_encoder_infer_workspace(B, S, H, A, I, drop, total)
    assert wsp % 256 == 0 and 0 < wsp <= L.vb_encoder_arena_layout_varlen(B, S, total, H, A, I, drop, None) and wsp < ws


def test_workspace_refuses_bad_shapes():
    L = _lib.lib()
    good = [4, 56, 768, 12, 3072]
    for i in range(5):
        for bad in (0, -1):
            a = list(good)
            a[i] = bad
            assert L.vb_encoder_infer_workspace(*a, 0, -1) == -1
            assert b"bad shape" in L.vb_last_error()
    assert L.vb_encoder_infer_workspace(*good, 0, 0) == -1 and b"bad shape" in L.vb_last_error()
    assert L.vb_encoder_infer_workspace(*good, 0, 1 << 31) == -1


def _descs(n=2):
    descs = (_lib.LayerDesc * n)()
    for d in descs:
        d.batch, d.seq, d.hidden, d.heads, d.inter = 2, 17, 128, 2, 512
        d.w_qkv = d.w_attn_out = d.w_inter = d.w_out = d.mask_bias = FAKE
    return descs


def test_encoder_infer_refuses_bad_arguments():
    L = _lib.lib()
    descs = _descs()
    _refused(L.vb_encoder_infer(descs, 0, FAKE, FAKE, FAKE, None, None, None), b"no layers")
    _refused(L.vb_encoder_infer(None, 2, FAKE, FAKE, FAKE, None, None, None), b"no layers")
    _refused(L.vb_encoder_infer(descs, 2, None, FAKE, FAKE, None, None, None), b"null x_in / workspace")
    _refused(L.vb_encoder_infer(descs, 2, FAKE, None, FAKE, None, None, None), b"null x_in / workspace")
    _refused(L.vb_encoder_infer(descs, 2, FAKE, FAKE, None, None, None, None), b"both NULL")
    _refused(L.vb_encoder_infer(descs, 2, FAKE, FAKE, FAKE, 0x800000, None, None), b"last slice")
    _refused(L.vb_encoder_infer((_lib.LayerDesc * 2)(), 2, FAKE, FAKE, FAKE, None, None, None), b"empty batch")
    descs[1].mask_bias = None
    _refused(L.vb_encoder_infer(descs, 2, FAKE, FAKE, FAKE, None, None, None), b"null mask_bias")
    descs = _descs()
    descs[1].seq = 18
    _refused(L.vb_encoder_infer(descs, 2, FAKE, FAKE, FAKE, None, None, None), b"layers differ in shape")
    _refused(L.vb_encoder_infer(descs, 2, FAKE, FAKE, None, FAKE, FAKE, None), b"layers differ in shape")   # with attention maps
    descs = _descs()
    descs[1].attn_dropout = 0.1
    _refused(L.vb_encoder_infer(descs, 2, FAKE, FAKE, FAKE, None, None, None), b"layers differ in shape")
    descs = _descs()
    descs[0].heads = descs[1].heads = 3
    _refused(L.vb_encoder_infer(descs, 2, FAKE, FAKE, FAKE, None, None, None), b"must equal heads")


def test_encoder_infer_varlen_refuses_bad_arguments():
    L = _lib.lib()
    descs = _descs()
    for d in descs:
        d.mask_bias = None   # ignored by the variable-length call
    _refused(L.vb_encoder_infer_varlen(descs, 2, None, 20, FAKE, FAKE, FAKE, None, None), b"cu_seqlens is NULL")
    _refused(L.vb_encoder_infer_varlen(descs, 2, FAKE, 0, FAKE, FAKE, FAKE, None, None), b"must be > 0")
    _refused(L.vb_encoder_infer_varlen(descs, 0, FAKE, 20, FAKE, FAKE, FAKE, None, None), b"no layers")
    _refused(L.vb_encoder_infer_varlen(descs, 2, FAKE, 20, None, FAKE, FAKE, None, None), b"null x_in / workspace")
    _refused(L.vb_encoder_infer_varlen(descs, 2, FAKE, 20, FAKE, None, FAKE, None, None), b"null x_in / workspace")
    _refused(L.vb_encoder_infer_varlen(descs, 2, FAKE, 20, FAKE, FAKE, None, None, None), b"both NULL")
    descs[1].inter = 256
    _refused(L.vb_encoder_infer_varlen(descs, 2, FAKE, 20, FAKE, FAKE, FAKE, None, None), b"layers differ in shape")
    descs[1].inter = 512
    descs[0].hidden = descs[1].hidden = 192
    _refused(L.vb_encoder_infer_varlen(descs, 2, FAKE, 20, FAKE, FAKE, FAKE, None, None), b"must equal heads")


@pytest.mark.parametrize("kw, what", [
    (dict(dropout_p=0.1, dropout_seed=1), b"take no dropout and no addend"),
    (dict(addend=0x60000, ld_add=256), b"take no dropout and no addend"),
    (dict(gp_tiled=1), b"gp_tiled needs a GELU / DGELU epilogue"),
    (dict(d_fp32=1), b"GELU_FWD epilogue needs"),
    (dict(a_mn_major=1), b"GELU_FWD epilogue needs"),
    (dict(b_mn_major=1), b"GELU_FWD epilogue needs"),
    (dict(aux_out=0x50000, ld_aux=256), b"GELU_FWD epilogue needs"),
    (dict(aux_in=0x40000, ld_aux=256), b"GELU_FWD epilogue needs"),
])
def test_gemm_gelu_fwd_epilogue_refuses_what_it_cannot_do(kw, what):
    L = _lib.lib()
    a = _lib.GemmArgs(epilogue=_lib.VB_EPI_GELU_FWD, **kw, **_GEMM)
    _refused(L.vb_gemm(ctypes.byref(a), None), what)


def test_epilogue_3_is_still_unknown():
    L = _lib.lib()
    a = _lib.GemmArgs(epilogue=3, **_GEMM)
    _refused(L.vb_gemm(ctypes.byref(a), None), b"unknown epilogue 3")
