"""CPU checks of the unpadded (variable-length) interface: the varlen arena layout, argument validation through
vb_last_error, and the row bookkeeping (packing index and cu_seqlens) of ops.unpad_plan."""
import ctypes

import pytest
import torch


def test_varlen_arena_layout_is_aligned_and_sized():
    from visualbert_b200 import _lib
    L = _lib.lib()
    off = (ctypes.c_int64 * _lib.VB_ENCODER_ARENA_BUFFERS)()
    B, S, total, H, A, I = 7, 164, 613, 768, 12, 3072
    stride = L.vb_encoder_arena_layout_varlen(B, S, total, H, A, I, 1, off)
    o = list(off)
    assert o[0] == 0 and all(x % 256 == 0 for x in o) and stride % 256 == 0
    sizes = dict(zip(_lib.ARENA_NAMES, [b - a for a, b in zip(o, o[1:] + [stride])]))
    M = total
    assert sizes["qkv"] >= M * 3 * H * 2 and sizes["ctx"] >= M * H * 2 and sizes["u"] >= M * I * 2 and sizes["g"] >= M * I * 2
    assert sizes["y"] >= M * H * 2 and sizes["mean1"] >= M * 4 and sizes["lse"] >= A * total * 4
    assert sizes["keep_mask"] >= L.vb_attention_keep_bytes(B, S, A)
    assert sizes["qkv"] < 2 * M * 3 * H * 2   # sized for the packed rows, not for B * S
    stride0 = L.vb_encoder_arena_layout_varlen(B, S, total, H, A, I, 0, off)
    assert stride0 == stride - sizes["keep_mask"]
    # total = B * S gives the dense layout
    dense = (ctypes.c_int64 * _lib.VB_ENCODER_ARENA_BUFFERS)()
    assert L.vb_encoder_arena_layout(B, S, H, A, I, 1, dense) == L.vb_encoder_arena_layout_varlen(B, S, B * S, H, A, I, 1, off)
    assert list(dense) == list(off)
    assert L.vb_encoder_arena_layout_varlen(0, S, total, H, A, I, 1, off) == -1
    assert b"bad shape" in L.vb_last_error()


def _aligned_buffer(n):
    """A host buffer and a 16-byte aligned address inside it (stands in for device pointers the calls refuse before use)."""
    buf = ctypes.create_string_buffer(n + 16)
    return buf, (ctypes.addressof(buf) + 15) // 16 * 16


def test_varlen_argument_validation_reports_through_vb_last_error():
    from visualbert_b200 import _lib
    L = _lib.lib()
    buf, p = _aligned_buffer(64)
    # batch 0, max_seq 0, negative total, null cu_seqlens, head_dim != 64: refused before anything is launched
    assert L.vb_attention_fwd_varlen(p, p, p, p, None, 0, 10, 10, 1, 64, 0.0, 1, 0, None) != 0
    assert b"empty problem" in L.vb_last_error()
    assert L.vb_attention_fwd_varlen(p, p, p, p, None, 2, 0, 10, 1, 64, 0.0, 1, 0, None) != 0
    assert L.vb_attention_fwd_varlen(p, p, p, p, None, 2, 10, -1, 1, 64, 0.0, 1, 0, None) != 0
    assert b"total" in L.vb_last_error()
    assert L.vb_attention_fwd_varlen(p, None, p, p, None, 2, 10, 10, 1, 64, 0.0, 1, 0, None) != 0
    assert b"cu_seqlens" in L.vb_last_error()
    assert L.vb_attention_fwd_varlen(p, p, p, p, None, 2, 10, 10, 2, 64, 0.0, 1, 0, None) != 0
    assert b"head_dim" in L.vb_last_error()
    assert L.vb_attention_fwd_varlen(p, p, p, None, None, 2, 10, 10, 1, 64, 0.0, 1, 0, None) != 0
    assert b"lse" in L.vb_last_error()
    assert L.vb_attention_bwd_varlen(p, p, p, p, None, None, p, p, 2, 10, 10, 1, 64, 0.0, 1, 0, None) != 0
    assert b"null pointer" in L.vb_last_error()
    assert L.vb_attention_fwd_varlen(p, p, p, p, None, 2, 10, 10, 1, 64, 0.2, 1, 0, None) != 0
    assert b"keep" in L.vb_last_error()
    assert L.vb_encoder_fwd_varlen(None, 1, None, 10, None, None, None) != 0
    assert b"cu_seqlens" in L.vb_last_error()
    assert L.vb_encoder_fwd_varlen(None, 1, p, 0, None, None, None) != 0
    assert b"total" in L.vb_last_error()
    assert L.vb_encoder_bwd_varlen(None, 1, p, 5, None, None, None, None, None, None, None) != 0
    assert b"null pointer" in L.vb_last_error()


def test_attention_refuses_operands_that_are_not_16_byte_aligned():
    """Every attention route reads qkv, and in the backward ctx and dctx, in 16-byte pieces: a pointer 2 bytes off that
    alignment is refused before anything is launched."""
    from visualbert_b200 import _lib
    L = _lib.lib()
    buf, a = _aligned_buffer(64)
    p, off = ctypes.c_void_p(a), ctypes.c_void_p(a + 2)
    B, S, A, H = 2, 100, 1, 64
    tail = (B, S, A, H, ctypes.c_float(0.0), ctypes.c_uint64(1), 0, None)
    assert L.vb_attention_fwd(off, p, p, p, None, *tail) != 0
    assert b"16-byte aligned" in L.vb_last_error()
    assert L.vb_attention_bwd(off, p, p, p, None, p, p, p, *tail) != 0   # qkv
    assert b"16-byte aligned" in L.vb_last_error()
    assert L.vb_attention_bwd(p, p, off, p, None, p, p, p, *tail) != 0   # ctx
    assert b"16-byte aligned" in L.vb_last_error()
    assert L.vb_attention_bwd(p, p, p, p, None, off, p, p, *tail) != 0   # dctx
    assert b"16-byte aligned" in L.vb_last_error()
    assert L.vb_attention_fwd_varlen(a + 2, a, a, a, None, 2, 10, 10, 1, 64, 0.0, 1, 0, None) != 0
    assert b"16-byte aligned" in L.vb_last_error()
    assert L.vb_attention_bwd_varlen(a, a, a, a, None, a + 2, a, a, 2, 10, 10, 1, 64, 0.0, 1, 0, None) != 0
    assert b"16-byte aligned" in L.vb_last_error()


def _loop_plan(valid):
    B, S = valid.shape
    index, cu = [], [0]
    for b in range(B):
        rows = [b * S + s for s in range(S) if valid[b, s]]
        index += rows
        cu.append(cu[-1] + len(rows))
    lens = [cu[b + 1] - cu[b] for b in range(B)]
    return index, cu, max(lens), cu[-1]


@pytest.mark.parametrize("seed", range(6))
def test_unpad_plan_matches_python_loop(seed):
    from visualbert_b200 import ops
    g = torch.Generator().manual_seed(seed)
    B, S = int(torch.randint(1, 9, (1,), generator=g)), int(torch.randint(1, 40, (1,), generator=g))
    kind = seed % 3
    if kind == 0:      # prefixes, some empty
        lens = torch.randint(0, S + 1, (B,), generator=g)
        valid = torch.arange(S)[None, :] < lens[:, None]
    else:              # arbitrary patterns (not prefixes), one example empty
        valid = torch.rand(B, S, generator=g) < (0.3 if kind == 1 else 0.8)
        valid[0] = False
    mask = valid.long() * (1 + torch.randint(0, 3, (B, S), generator=g))  # any non-zero value is valid
    plan = ops.unpad_plan(mask != 0)
    index, cu, max_seq, total = _loop_plan(valid)
    assert plan["index"].tolist() == index
    assert plan["cu_seqlens"].tolist() == cu and plan["cu_seqlens"].dtype == torch.int32
    assert plan["max_seq"] == max_seq and plan["total"] == total and plan["batch"] == B
