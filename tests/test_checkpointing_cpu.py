"""CPU-side checks of the activation-checkpointing encoder calls (vb_encoder_ckpt_layout, vb_encoder_fwd_ckpt, vb_encoder_bwd_ckpt
and their _varlen forms): exported without an ABI bump, the checkpoint region sized and aligned as documented, and bad arguments
refused through vb_last_error before anything reaches a device (the pointers below are never dereferenced)."""
import ctypes

import pytest

from visualbert_b200 import _lib

FAKE = 0x10000   # 32-byte aligned, non-null


def _align(x):
    return (x + 255) // 256 * 256


def _refused(rc, what):
    assert rc != 0
    msg = _lib.lib().vb_last_error()
    assert what in msg, msg


def test_ckpt_entry_points_exported_without_an_abi_bump():
    L = _lib.lib()
    names = {"vb_encoder_ckpt_layout", "vb_encoder_fwd_ckpt", "vb_encoder_bwd_ckpt", "vb_encoder_fwd_ckpt_varlen",
             "vb_encoder_bwd_ckpt_varlen"}
    assert names <= set(_lib.EXPORTS) and all(hasattr(L, n) for n in names)
    assert L.vb_abi_version() == _lib.ABI_VERSION == 4
    assert _lib.CKPT_NAMES == ("y", "mean2", "rstd2")


@pytest.mark.parametrize("shape", [(4, 56, 768, 12, 3072), (256, 164, 768, 12, 3072), (64, 356, 1024, 16, 4096), (3, 17, 128, 2, 64)])
def test_ckpt_layout_is_aligned_and_sized(shape):
    L = _lib.lib()
    B, S, H, A, I = shape
    for rows in (-1, B * S - (B * S) // 3, 1):
        M = B * S if rows < 0 else rows
        off = (ctypes.c_int64 * 3)()
        stride = L.vb_encoder_ckpt_layout(B, S, H, A, I, rows, off)
        assert stride == _align(M * H * 2) + 2 * _align(M * 4)
        assert list(off) == [0, _align(M * H * 2), _align(M * H * 2) + _align(M * 4)]
        assert stride % 256 == 0 and all(o % 256 == 0 for o in off)
        assert L.vb_encoder_ckpt_layout(B, S, H, A, I, rows, None) == stride
    # a region is far smaller than the arena slot it replaces
    assert L.vb_encoder_ckpt_layout(B, S, H, A, I, -1, None) * 4 < L.vb_encoder_arena_layout(B, S, H, A, I, 0, None)


def test_ckpt_layout_at_the_benchmark_shape():
    """cfg2 (B 256, S 164, H 768): 64.8 MB per region against a 1.06 GB arena slot."""
    L = _lib.lib()
    cs = L.vb_encoder_ckpt_layout(256, 164, 768, 12, 3072, -1, None)
    assert abs(cs / 1e6 - 64.8) < 0.1
    assert L.vb_encoder_arena_layout(256, 164, 768, 12, 3072, 1, None) > 16 * cs


def test_ckpt_layout_refuses_bad_shapes():
    L = _lib.lib()
    good = [4, 56, 768, 12, 3072]
    for i in range(5):
        for bad in (0, -1):
            a = list(good)
            a[i] = bad
            assert L.vb_encoder_ckpt_layout(*a, -1, None) == -1
            assert b"bad shape" in L.vb_last_error()
    assert L.vb_encoder_ckpt_layout(*good, 0, None) == -1 and b"bad shape" in L.vb_last_error()
    assert L.vb_encoder_ckpt_layout(*good, 1 << 31, None) == -1


def _descs(n=2):
    descs = (_lib.LayerDesc * n)()
    for d in descs:
        d.batch, d.seq, d.hidden, d.heads, d.inter = 2, 17, 128, 2, 512
        d.w_qkv = d.w_attn_out = d.w_inter = d.w_out = d.mask_bias = FAKE
    return descs


def _grads(n=2):
    return (_lib.LayerGrads * n)()


def _scratch():
    return _lib.LayerScratch(d_pre=FAKE, d_pre_drop=FAKE, d_big=FAKE, d_x1=FAKE, d_ctx=FAKE, drow=FAKE)


def test_fwd_ckpt_refuses_bad_arguments():
    L = _lib.lib()
    n0 = L.vb_launch_count()
    descs = _descs()
    _refused(L.vb_encoder_fwd_ckpt(descs, 0, FAKE, FAKE, FAKE, None, None), b"no layers")
    _refused(L.vb_encoder_fwd_ckpt(None, 2, FAKE, FAKE, FAKE, None, None), b"no layers")
    _refused(L.vb_encoder_fwd_ckpt(descs, 2, FAKE, None, FAKE, None, None), b"ckpt is NULL with 2 layers")
    _refused(L.vb_encoder_fwd_ckpt(descs, 2, None, FAKE, FAKE, None, None), b"null x_in / slot")
    _refused(L.vb_encoder_fwd_ckpt(descs, 2, FAKE, FAKE, None, None, None), b"null x_in / slot")
    _refused(L.vb_encoder_fwd_ckpt((_lib.LayerDesc * 2)(), 2, FAKE, FAKE, FAKE, None, None), b"empty batch")
    descs[1].mask_bias = None
    _refused(L.vb_encoder_fwd_ckpt(descs, 2, FAKE, FAKE, FAKE, None, None), b"null mask_bias")
    for field, value in (("seq", 18), ("inter", 256), ("attn_dropout", 0.1)):
        descs = _descs()
        setattr(descs[1], field, value)
        _refused(L.vb_encoder_fwd_ckpt(descs, 2, FAKE, FAKE, FAKE, None, None), b"layers differ in shape")
        _refused(L.vb_encoder_fwd_ckpt(descs, 2, FAKE, FAKE, FAKE, FAKE, None), b"layers differ in shape")
    descs = _descs()
    descs[0].heads = descs[1].heads = 3
    _refused(L.vb_encoder_fwd_ckpt(descs, 2, FAKE, FAKE, FAKE, None, None), b"must equal heads")
    assert L.vb_launch_count() == n0


def test_bwd_ckpt_refuses_bad_arguments():
    L = _lib.lib()
    n0 = L.vb_launch_count()
    descs, g, sc = _descs(), _grads(), _scratch()
    sref = ctypes.byref(sc)
    _refused(L.vb_encoder_bwd_ckpt(descs, 0, FAKE, FAKE, FAKE, FAKE, FAKE, g, sref, None), b"no layers")
    _refused(L.vb_encoder_bwd_ckpt(descs, 2, FAKE, None, FAKE, FAKE, FAKE, g, sref, None), b"ckpt is NULL with 2 layers")
    _refused(L.vb_encoder_bwd_ckpt(descs, 2, FAKE, FAKE, None, FAKE, FAKE, g, sref, None), b"null pointer")
    _refused(L.vb_encoder_bwd_ckpt(descs, 2, FAKE, FAKE, FAKE, None, FAKE, g, sref, None), b"null pointer")
    _refused(L.vb_encoder_bwd_ckpt(descs, 2, FAKE, FAKE, FAKE, FAKE, FAKE, None, sref, None), b"null pointer")
    _refused(L.vb_encoder_bwd_ckpt(descs, 2, FAKE, FAKE, FAKE, FAKE, FAKE, g, None, None), b"null pointer")
    bad = _descs()
    bad[1].hidden = 192
    bad[1].heads = 3
    _refused(L.vb_encoder_bwd_ckpt(bad, 2, FAKE, FAKE, FAKE, FAKE, FAKE, g, sref, None), b"layers differ in shape")
    # a partly NULL LayerNorm group in the lowest layer: refused before the top layer's backward launches anything
    g = _grads()
    g[0].dln1_gamma = FAKE
    _refused(L.vb_encoder_bwd_ckpt(descs, 2, FAKE, FAKE, FAKE, FAKE, FAKE, g, sref, None), b"give all three or none")
    # hidden dropout in the lowest layer only, without the d_pre_drop scratch
    descs, sc = _descs(), _scratch()
    descs[0].hidden_dropout = 0.1
    sc.d_pre_drop = None
    _refused(L.vb_encoder_bwd_ckpt(descs, 2, FAKE, FAKE, FAKE, FAKE, FAKE, _grads(), ctypes.byref(sc), None), b"d_pre_drop")
    assert L.vb_launch_count() == n0


def test_ckpt_varlen_refuses_bad_arguments():
    L = _lib.lib()
    n0 = L.vb_launch_count()
    descs = _descs()
    for d in descs:
        d.mask_bias = None   # ignored by the variable-length calls
    sref = ctypes.byref(_scratch())
    _refused(L.vb_encoder_fwd_ckpt_varlen(descs, 2, None, 20, FAKE, FAKE, FAKE, None), b"cu_seqlens is NULL")
    _refused(L.vb_encoder_fwd_ckpt_varlen(descs, 2, FAKE, 0, FAKE, FAKE, FAKE, None), b"must be > 0")
    _refused(L.vb_encoder_fwd_ckpt_varlen(descs, 2, FAKE, 20, FAKE, None, FAKE, None), b"ckpt is NULL")
    _refused(L.vb_encoder_bwd_ckpt_varlen(descs, 2, None, 20, FAKE, FAKE, FAKE, FAKE, FAKE, _grads(), sref, None), b"cu_seqlens is NULL")
    _refused(L.vb_encoder_bwd_ckpt_varlen(descs, 2, FAKE, -1, FAKE, FAKE, FAKE, FAKE, FAKE, _grads(), sref, None), b"must be > 0")
    _refused(L.vb_encoder_bwd_ckpt_varlen(descs, 2, FAKE, 20, FAKE, None, FAKE, FAKE, FAKE, _grads(), sref, None), b"ckpt is NULL")
    descs[1].inter = 256
    _refused(L.vb_encoder_fwd_ckpt_varlen(descs, 2, FAKE, 20, FAKE, FAKE, FAKE, None), b"layers differ in shape")
    _refused(L.vb_encoder_bwd_ckpt_varlen(descs, 2, FAKE, 20, FAKE, FAKE, FAKE, FAKE, FAKE, _grads(), sref, None),
             b"layers differ in shape")
    assert L.vb_launch_count() == n0


def test_model_switch_is_off_by_default_and_reaches_the_encoder_meta():
    from visualbert_b200 import BertConfig, BertVisualModel, synthetic
    from visualbert_b200.modeling import _encoder_meta
    cfg = BertConfig.from_dict(synthetic.bert_config_dict(2, 128, 2, 512, vocab=64))
    cfg.visual_embedding_dim = 32
    m = BertVisualModel(cfg)
    assert m.encoder.activation_checkpointing is False
    assert _encoder_meta(m.encoder, m.encoder.layer, 0)["checkpoint"] is False
    assert m.set_activation_checkpointing() is m
    assert _encoder_meta(m.encoder, m.encoder.layer, 0)["checkpoint"] is True
    # a single layer's own call (the padded per-layer route) is not checkpointed
    assert _encoder_meta(m.encoder.layer[0], [m.encoder.layer[0]], 0)["checkpoint"] is False
    m.set_activation_checkpointing(False)
    assert _encoder_meta(m.encoder, m.encoder.layer, 0)["checkpoint"] is False
