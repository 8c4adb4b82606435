"""vb_gemm reads O of the attention-output input-gradient epilogue (delta_ctx) through a TMA tensor map, like an addend: a
delta_ctx that is not 32-byte aligned is refused before the first CUDA call, with an error that names it."""
import ctypes

import pytest

# 32-byte aligned fake device pointers: every check in vb_gemm runs before its first CUDA call
_FAKE = dict(A=0x10000, lda=256, B=0x20000, ldb=256, b_mn_major=1, M=256, N=256, K=256, D=0x30000, ldd=256,
             delta_out=0x40000, delta_seq=64)


@pytest.mark.parametrize("ctx", [0x50010, 0x50008, 0x50002])
def test_gemm_refuses_a_misaligned_delta_ctx(ctx):
    from visualbert_b200 import _lib
    L = _lib.lib()
    a = _lib.GemmArgs(delta_ctx=ctx, **_FAKE)
    assert L.vb_gemm(ctypes.byref(a), None) != 0
    assert b"delta_ctx must be 32-byte aligned" in L.vb_last_error()

