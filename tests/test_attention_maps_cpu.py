"""CPU-side checks of the attention-map entry points: exported, counted in the ABI version, and refusing bad arguments
through vb_last_error before anything reaches a device (the pointers below are never dereferenced)."""
import ctypes

from visualbert_b200 import _lib

FAKE = 0x10000   # 16-byte aligned, non-null


def _refused(rc, what):
    assert rc != 0
    msg = _lib.lib().vb_last_error()
    assert what in msg, msg


def test_attention_probs_exported_and_version_bumped():
    L = _lib.lib()
    assert hasattr(L, "vb_attention_probs") and hasattr(L, "vb_encoder_attention_probs")
    assert {"vb_attention_probs", "vb_encoder_attention_probs"} <= set(_lib.EXPORTS)
    assert L.vb_abi_version() == _lib.ABI_VERSION == 4


def test_attention_probs_refuses_bad_arguments():
    L = _lib.lib()
    B, S, A, H = 2, 17, 2, 128
    _refused(L.vb_attention_probs(FAKE, FAKE, FAKE, 0, S, A, H, None), b"empty problem")
    _refused(L.vb_attention_probs(FAKE, FAKE, FAKE, B, 0, A, H, None), b"empty problem")
    _refused(L.vb_attention_probs(FAKE, FAKE, FAKE, B, S, -1, H, None), b"empty problem")
    _refused(L.vb_attention_probs(FAKE, FAKE, FAKE, B, S, 3, H, None), b"head_dim must be 64")
    _refused(L.vb_attention_probs(FAKE, FAKE, FAKE, B, S, A, H + 64, None), b"head_dim must be 64")
    _refused(L.vb_attention_probs(FAKE + 2, FAKE, FAKE, B, S, A, H, None), b"16-byte aligned")
    _refused(L.vb_attention_probs(FAKE, None, FAKE, B, S, A, H, None), b"null pointer")
    _refused(L.vb_attention_probs(FAKE, FAKE, None, B, S, A, H, None), b"null pointer")


def test_encoder_attention_probs_refuses_bad_arguments():
    L = _lib.lib()
    descs = (_lib.LayerDesc * 2)()
    _refused(L.vb_encoder_attention_probs(descs, 0, FAKE, FAKE, None), b"null pointer / no layers")
    _refused(L.vb_encoder_attention_probs(descs, 2, None, FAKE, None), b"null pointer / no layers")
    _refused(L.vb_encoder_attention_probs(descs, 2, FAKE, None, None), b"null pointer / no layers")
    # all-zero descriptors: an empty batch
    _refused(L.vb_encoder_attention_probs(descs, 2, FAKE, FAKE, None), b"empty batch")
    for d in descs:
        d.batch, d.seq, d.hidden, d.heads, d.inter = 2, 17, 128, 3, 512
        d.w_qkv = d.w_attn_out = d.w_inter = d.w_out = d.mask_bias = FAKE
    _refused(L.vb_encoder_attention_probs(descs, 2, FAKE, FAKE, None), b"must equal heads")
    descs[1].heads = descs[0].heads = 2
    descs[1].seq = 18
    _refused(L.vb_encoder_attention_probs(descs, 2, FAKE, FAKE, None), b"layers differ in shape")
