"""CPU-side checks of selective FFN recomputation (set_ffn_recompute; vb_encoder_arena_layout_ffnrc, vb_encoder_fwd_ffnrc,
vb_encoder_bwd_ffnrc and their _varlen forms): exported without an ABI bump, the layout sized as documented against the arena
layout, bad arguments refused through vb_last_error before any launch (the pointers below are never dereferenced), and the
switch reaching the meta of the routes it governs."""
import ctypes

import pytest

from visualbert_b200 import _lib

FAKE = 0x10000   # 32-byte aligned, non-null
NAMES = {"vb_encoder_arena_layout_ffnrc", "vb_encoder_arena_layout_ffnrc_varlen", "vb_encoder_fwd_ffnrc", "vb_encoder_bwd_ffnrc",
         "vb_encoder_fwd_ffnrc_varlen", "vb_encoder_bwd_ffnrc_varlen"}


def _align(x):
    return (x + 255) // 256 * 256


def _refused(rc, what):
    assert rc != 0
    msg = _lib.lib().vb_last_error()
    assert what in msg, msg


def test_ffnrc_entry_points_exported_without_an_abi_bump():
    L = _lib.lib()
    assert NAMES <= set(_lib.EXPORTS) and all(hasattr(L, n) for n in NAMES)
    assert L.vb_abi_version() == _lib.ABI_VERSION == 4
    assert L.vb_encoder_arena_layout_ffnrc.restype is ctypes.c_int64
    assert L.vb_encoder_arena_layout_ffnrc_varlen.restype is ctypes.c_int64
    assert len(L.vb_encoder_arena_layout_ffnrc.argtypes) == 8 and len(L.vb_encoder_arena_layout_ffnrc_varlen.argtypes) == 9
    assert len(L.vb_encoder_fwd_ffnrc.argtypes) == 6 and len(L.vb_encoder_fwd_ffnrc_varlen.argtypes) == 8
    assert len(L.vb_encoder_bwd_ffnrc.argtypes) == 10 and len(L.vb_encoder_bwd_ffnrc_varlen.argtypes) == 12


def _layouts(B, S, H, A, I, drop, total=None):
    L = _lib.lib()
    n = _lib.VB_ENCODER_ARENA_BUFFERS
    off, roff, fb = (ctypes.c_int64 * n)(), (ctypes.c_int64 * n)(), ctypes.c_int64(-7)
    if total is None:
        ref = L.vb_encoder_arena_layout(B, S, H, A, I, drop, roff)
        stride = L.vb_encoder_arena_layout_ffnrc(B, S, H, A, I, drop, off, ctypes.byref(fb))
        assert L.vb_encoder_arena_layout_ffnrc(B, S, H, A, I, drop, None, None) == stride
    else:
        ref = L.vb_encoder_arena_layout_varlen(B, S, total, H, A, I, drop, roff)
        stride = L.vb_encoder_arena_layout_ffnrc_varlen(B, S, total, H, A, I, drop, off, ctypes.byref(fb))
        assert L.vb_encoder_arena_layout_ffnrc_varlen(B, S, total, H, A, I, drop, None, None) == stride
    return ref, list(roff), stride, list(off), fb.value


@pytest.mark.parametrize("shape", [(4, 56, 768, 12, 3072), (256, 164, 768, 12, 3072), (64, 356, 1024, 16, 4096), (3, 17, 128, 2, 64)])
@pytest.mark.parametrize("drop", [0, 1])
def test_ffnrc_layout_is_the_arena_layout_without_u_and_g(shape, drop):
    B, S, H, A, I = shape
    for total in (None, B * S - (B * S) // 3, 1, 0):
        M = B * S if total is None else total
        ref, roff, stride, off, ffn = _layouts(B, S, H, A, I, drop, total)
        u, g = 7, 8   # ARENA_NAMES
        assert _lib.ARENA_NAMES[u] == "u" and _lib.ARENA_NAMES[g] == "g"
        assert ffn == 2 * _align(M * I * 2)
        assert stride == ref - 2 * _align(M * I * 2)
        assert off[u] == off[g] == off[g + 1] == roff[u]   # u and g take no room in the slot
        assert off[:u + 1] == roff[:u + 1]
        assert [o + 2 * _align(M * I * 2) for o in off[g + 1:]] == roff[g + 1:]
        assert off[0] == 0 and stride % 256 == 0 and all(o % 256 == 0 for o in off)


def test_ffnrc_layout_at_the_benchmark_shape():
    """cfg2 (B 256, S 164, H 768, I 3072): the shared buffer is 516 MB, and the slot drops from 1.06 GB by that much."""
    ref, _, stride, _, ffn = _layouts(256, 164, 768, 12, 3072, 1)
    assert abs(ffn / 1e6 - 515.9) < 0.1
    assert ref - stride == ffn and abs(ref / 1e9 - 1.063) < 0.01
    assert 12 * ref - (12 * stride + ffn) == 11 * ffn   # the saving of a 12-layer arena


def test_ffnrc_layout_refuses_bad_shapes():
    L = _lib.lib()
    good = [4, 56, 768, 12, 3072]
    for i in range(5):
        for bad in (0, -1):
            a = list(good)
            a[i] = bad
            assert L.vb_encoder_arena_layout_ffnrc(*a, 1, None, None) == -1
            assert b"bad shape" in L.vb_last_error()
    assert L.vb_encoder_arena_layout_ffnrc_varlen(4, 56, -1, 768, 12, 3072, 1, None, None) == -1
    assert b"bad shape" in L.vb_last_error()
    assert L.vb_encoder_arena_layout_ffnrc_varlen(0, 56, 10, 768, 12, 3072, 1, None, None) == -1


def _descs(n=2):
    descs = (_lib.LayerDesc * n)()
    for d in descs:
        d.batch, d.seq, d.hidden, d.heads, d.inter = 2, 17, 128, 2, 512
        d.w_qkv = d.w_attn_out = d.w_inter = d.w_out = d.mask_bias = FAKE
    return descs


def _scratch():
    return _lib.LayerScratch(d_pre=FAKE, d_pre_drop=FAKE, d_big=FAKE, d_x1=FAKE, d_ctx=FAKE, drow=FAKE)


def test_fwd_ffnrc_refuses_bad_arguments():
    L = _lib.lib()
    n0 = L.vb_launch_count()
    descs = _descs()
    _refused(L.vb_encoder_fwd_ffnrc(descs, 0, FAKE, FAKE, FAKE, None), b"no layers")
    _refused(L.vb_encoder_fwd_ffnrc(None, 2, FAKE, FAKE, FAKE, None), b"no layers")
    _refused(L.vb_encoder_fwd_ffnrc(descs, 2, FAKE, FAKE, None, None), b"null x_in / arena / ffn")
    _refused(L.vb_encoder_fwd_ffnrc(descs, 2, None, FAKE, FAKE, None), b"null x_in / arena / ffn")
    _refused(L.vb_encoder_fwd_ffnrc(descs, 2, FAKE, None, FAKE, None), b"null x_in / arena / ffn")
    descs[1].mask_bias = None   # the top layer's descriptor is checked before layer 0 launches
    _refused(L.vb_encoder_fwd_ffnrc(descs, 2, FAKE, FAKE, FAKE, None), b"null mask_bias")
    for field, value in (("seq", 18), ("inter", 256), ("attn_dropout", 0.1)):
        descs = _descs()
        setattr(descs[1], field, value)
        _refused(L.vb_encoder_fwd_ffnrc(descs, 2, FAKE, FAKE, FAKE, None), b"layers differ in shape")
    assert L.vb_launch_count() == n0


def test_bwd_ffnrc_refuses_bad_arguments():
    L = _lib.lib()
    n0 = L.vb_launch_count()
    descs, g, sc = _descs(), (_lib.LayerGrads * 2)(), _scratch()
    sref = ctypes.byref(sc)
    _refused(L.vb_encoder_bwd_ffnrc(descs, 0, FAKE, FAKE, FAKE, FAKE, FAKE, g, sref, None), b"no layers")
    _refused(L.vb_encoder_bwd_ffnrc(descs, 2, FAKE, FAKE, None, FAKE, FAKE, g, sref, None), b"null pointer")
    _refused(L.vb_encoder_bwd_ffnrc(descs, 2, FAKE, None, FAKE, FAKE, FAKE, g, sref, None), b"null pointer")
    _refused(L.vb_encoder_bwd_ffnrc(descs, 2, FAKE, FAKE, FAKE, None, FAKE, g, sref, None), b"null pointer")
    _refused(L.vb_encoder_bwd_ffnrc(descs, 2, FAKE, FAKE, FAKE, FAKE, FAKE, None, sref, None), b"null pointer")
    _refused(L.vb_encoder_bwd_ffnrc(descs, 2, FAKE, FAKE, FAKE, FAKE, FAKE, g, None, None), b"null pointer")
    bad = _descs()
    bad[1].hidden, bad[1].heads = 192, 3
    _refused(L.vb_encoder_bwd_ffnrc(bad, 2, FAKE, FAKE, FAKE, FAKE, FAKE, g, sref, None), b"layers differ in shape")
    # a partly NULL LayerNorm group in the lowest layer: refused before the top layer's backward launches anything
    g = (_lib.LayerGrads * 2)()
    g[0].dln1_gamma = FAKE
    _refused(L.vb_encoder_bwd_ffnrc(descs, 2, FAKE, FAKE, FAKE, FAKE, FAKE, g, sref, None), b"give all three or none")
    # hidden dropout in the lowest layer only, without the d_pre_drop scratch
    descs, sc = _descs(), _scratch()
    descs[0].hidden_dropout = 0.1
    sc.d_pre_drop = None
    _refused(L.vb_encoder_bwd_ffnrc(descs, 2, FAKE, FAKE, FAKE, FAKE, FAKE, (_lib.LayerGrads * 2)(), ctypes.byref(sc), None),
             b"d_pre_drop")
    assert L.vb_launch_count() == n0


def test_ffnrc_varlen_refuses_bad_arguments():
    L = _lib.lib()
    n0 = L.vb_launch_count()
    descs = _descs()
    for d in descs:
        d.mask_bias = None   # ignored by the variable-length calls
    g, sref = (_lib.LayerGrads * 2)(), ctypes.byref(_scratch())
    _refused(L.vb_encoder_fwd_ffnrc_varlen(descs, 2, None, 20, FAKE, FAKE, FAKE, None), b"cu_seqlens is NULL")
    _refused(L.vb_encoder_fwd_ffnrc_varlen(descs, 2, FAKE, 0, FAKE, FAKE, FAKE, None), b"must be > 0")
    _refused(L.vb_encoder_fwd_ffnrc_varlen(descs, 2, FAKE, 20, FAKE, FAKE, None, None), b"null x_in / arena / ffn")
    _refused(L.vb_encoder_bwd_ffnrc_varlen(descs, 2, None, 20, FAKE, FAKE, FAKE, FAKE, FAKE, g, sref, None), b"cu_seqlens is NULL")
    _refused(L.vb_encoder_bwd_ffnrc_varlen(descs, 2, FAKE, -1, FAKE, FAKE, FAKE, FAKE, FAKE, g, sref, None), b"must be > 0")
    _refused(L.vb_encoder_bwd_ffnrc_varlen(descs, 2, FAKE, 20, FAKE, FAKE, None, FAKE, FAKE, g, sref, None), b"null pointer")
    descs[1].inter = 256
    _refused(L.vb_encoder_fwd_ffnrc_varlen(descs, 2, FAKE, 20, FAKE, FAKE, FAKE, None), b"layers differ in shape")
    _refused(L.vb_encoder_bwd_ffnrc_varlen(descs, 2, FAKE, 20, FAKE, FAKE, FAKE, FAKE, FAKE, g, sref, None), b"layers differ in shape")
    assert L.vb_launch_count() == n0


def _model(**flags):
    from visualbert_b200 import BertConfig, BertVisualModel, synthetic
    cfg = BertConfig.from_dict(synthetic.bert_config_dict(2, 128, 2, 512, vocab=64))
    cfg.visual_embedding_dim = 32
    for k, v in flags.items():
        setattr(cfg, k, v)
    return BertVisualModel(cfg)


def test_switch_is_off_by_default_and_reaches_the_encoder_meta():
    from visualbert_b200.modeling import _encoder_meta
    m = _model()
    enc = m.encoder
    meta = lambda: _encoder_meta(enc, enc.layer, 0)
    assert enc.ffn_recompute is False and meta()["ffn_recompute"] is False
    assert m.set_ffn_recompute() is m
    assert enc.ffn_recompute is True and meta()["ffn_recompute"] is True and meta()["checkpoint"] is False
    # the unpadded call and the attention-map call take their meta from the same place
    assert _encoder_meta(enc, enc.layer, 0, varlen={}, all_layers=False)["ffn_recompute"] is True
    assert _encoder_meta(enc, enc.layer, 0, attn_maps=True)["ffn_recompute"] is True
    # a single layer's own call (the padded per-layer route) is not changed
    assert _encoder_meta(enc.layer[0], [enc.layer[0]], 0)["ffn_recompute"] is False
    # full checkpointing governs when both are on; its flag stays a bool
    m.set_activation_checkpointing(True)
    assert meta()["checkpoint"] is True and meta()["ffn_recompute"] is False
    assert enc.activation_checkpointing is True and enc.ffn_recompute is True
    m.set_activation_checkpointing(False)
    assert meta()["checkpoint"] is False and meta()["ffn_recompute"] is True
    m.set_ffn_recompute(False)
    assert meta()["ffn_recompute"] is False


def test_split_encoder_parts_keep_the_switch():
    """bert_encoder's frozen-parameter split builds the upper part's meta as dict(meta, ...): the switch travels with it."""
    from visualbert_b200.modeling import _encoder_meta
    m = _model().set_ffn_recompute(True)
    meta = _encoder_meta(m.encoder, m.encoder.layer, 0)
    high = dict(meta, caches=meta["caches"][1:], plan=meta["plan"].part(1), layer_index0=1, all_layers=True)
    assert high["ffn_recompute"] is True


def test_bypass_text_encoder_is_the_switched_encoder():
    """bypass_transformer: the text positions run through model.encoder (the switched module); the additional layer is a
    single-layer call of its own and is not changed."""
    from visualbert_b200.modeling import _encoder_meta
    m = _model(bypass_transformer=True).set_ffn_recompute(True)
    assert _encoder_meta(m.encoder, m.encoder.layer, 0)["ffn_recompute"] is True
    assert _encoder_meta(m.additional_layer, [m.additional_layer], 0)["ffn_recompute"] is False

