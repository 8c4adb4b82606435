"""ctypes binding of libvbert_b200.so (the C ABI declared in include/vbert_b200.h).

The library is the product path: there is no Python/PyTorch fallback. If the shared object is
missing or fails to load, importing any compute op raises immediately.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# VB_LIB_PATH: load another build of the same library (A/B timing of kernel variants on one GPU, scripts/build_variant.sh)
LIB_PATH = os.environ.get("VB_LIB_PATH") or os.path.join(_HERE, "lib", "libvbert_b200.so")

ABI_VERSION = 4  # == VB_ABI_VERSION of include/vbert_b200.h (tests/test_abi.py keeps the two in step)
VB_EPI_NONE, VB_EPI_GELU, VB_EPI_DGELU = 0, 1, 2
VB_EPI_GELU_FWD = 4  # 3 is retired

c_void_p, c_int, c_i64, c_f32, c_u64, c_u32 = (
    ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_float, ctypes.c_uint64, ctypes.c_uint32)


class GemmArgs(ctypes.Structure):
    """Mirror of vb_gemm_args (include/vbert_b200.h)."""
    _fields_ = [
        ("A", c_void_p), ("lda", c_i64), ("a_mn_major", c_int),
        ("B", c_void_p), ("ldb", c_i64), ("b_mn_major", c_int),
        ("M", c_int), ("N", c_int), ("K", c_int),
        ("D", c_void_p), ("ldd", c_i64),
        ("d_fp32", c_int), ("splits", c_int),
        ("bias", c_void_p),
        ("addend", c_void_p), ("ld_add", c_i64),
        ("epilogue", c_int),
        ("aux_in", c_void_p), ("aux_out", c_void_p), ("ld_aux", c_i64),
        ("dropout_p", c_f32), ("dropout_seed", c_u64), ("dropout_stream", c_u32),
        ("gp_tiled", c_int),
        ("delta_ctx", c_void_p), ("delta_out", c_void_p), ("delta_seq", c_int),
    ]


def _struct(name, fields):
    return type(name, (ctypes.Structure,), {"_fields_": fields})


_P = c_void_p
LayerDesc = _struct("LayerDesc", [
    ("batch", c_int), ("seq", c_int), ("hidden", c_int), ("heads", c_int), ("inter", c_int),
    ("hidden_dropout", c_f32), ("attn_dropout", c_f32), ("seed", c_u64), ("layer_index", c_u32),
    ("w_qkv", _P), ("w_attn_out", _P), ("w_inter", _P), ("w_out", _P),
    ("b_qkv", _P), ("b_attn_out", _P), ("ln1_gamma", _P), ("ln1_beta", _P),
    ("b_inter", _P), ("b_out", _P), ("ln2_gamma", _P), ("ln2_beta", _P), ("mask_bias", _P)])
LayerActs = _struct("LayerActs", [(n, _P) for n in (
    "qkv", "ctx", "lse", "pre1", "mean1", "rstd1", "x1", "u", "g", "pre2", "mean2", "rstd2", "keep_mask")])
LayerGrads = _struct("LayerGrads", [(n, _P) for n in (
    "dw_qkv", "db_qkv", "dw_attn_out", "db_attn_out", "dln1_gamma", "dln1_beta",
    "dw_inter", "db_inter", "dw_out", "db_out", "dln2_gamma", "dln2_beta")])
LayerScratch = _struct("LayerScratch", [(n, _P) for n in ("d_pre", "d_pre_drop", "d_big", "d_x1", "d_ctx", "drow")])
EmbedDesc = _struct("EmbedDesc", [
    ("batch", c_int), ("text_len", c_int), ("num_regions", c_int), ("hidden", c_int), ("visual_dim", c_int),
    ("vocab", c_int), ("max_pos", c_int), ("n_types", c_int),
    ("eps", c_f32), ("dropout", c_f32), ("seed", c_u64),
    ("input_ids", _P), ("token_type_ids", _P), ("visual_type", _P), ("visual_feats", _P),
    ("w_proj", _P), ("b_proj", _P),
    ("word", _P), ("pos", _P), ("type", _P), ("pos_vis", _P), ("type_vis", _P), ("gamma", _P), ("beta", _P),
    ("visual_addend", _P)])
EmbedActs = _struct("EmbedActs", [(n, _P) for n in ("vis_proj", "pre", "mean", "rstd")])
EmbedGrads = _struct("EmbedGrads", [(n, _P) for n in (
    "dword", "dpos", "dtype", "dpos_vis", "dtype_vis", "dw_proj", "db_proj", "dgamma", "dbeta",
    "d_pre", "d_vis", "d_feats")])

AdamTensor = _struct("AdamTensor", [
    ("p", _P), ("g", _P), ("m", _P), ("v", _P), ("numel", c_i64), ("lr", c_f32), ("weight_decay", c_f32),
    ("first_chunk", c_int), ("reserved", c_int)])
VB_ADAM_CHUNK = 32768
AdamGroup = _struct("AdamGroup", [
    ("lr", ctypes.c_double), ("warmup", ctypes.c_double), ("t_total", ctypes.c_double), ("cycles", ctypes.c_double),
    ("weight_decay", c_f32), ("schedule", c_int)])
VB_SCHED_CONSTANT, VB_SCHED_WARMUP_CONSTANT, VB_SCHED_WARMUP_LINEAR, VB_SCHED_WARMUP_COSINE = 0, 1, 2, 3
CastItem = _struct("CastItem", [("src", _P), ("dst", _P), ("numel", c_i64), ("first_chunk", c_int), ("dst_fp32", c_int)])
VB_CAST_CHUNK = 8192

# every symbol include/vbert_b200.h declares (checked by tests/test_abi.py without a GPU)
EXPORTS = [
    "vb_abi_version", "vb_last_error", "vb_launch_count", "vb_profile_enable", "vb_profile_read", "vb_gemm", "vb_gemm_gp_tiled_ok", "vb_gemm_delta_ok", "vb_layernorm_fwd", "vb_layernorm_bwd",
    "vb_attention_keep_bytes", "vb_attention_fwd", "vb_attention_bwd", "vb_mask_bias", "vb_cast_f32_to_bf16", "vb_cast_bf16_to_f32",
    "vb_colsum_bf16", "vb_cross_entropy_fwd", "vb_cross_entropy_bwd", "vb_layer_fwd", "vb_layer_bwd", "vb_embed_fwd", "vb_embed_bwd",
    "vb_bert_adam_step", "vb_cast_multi", "vb_encoder_arena_layout", "vb_encoder_fwd", "vb_encoder_bwd",
    "vb_attention_fwd_varlen", "vb_attention_bwd_varlen", "vb_encoder_arena_layout_varlen", "vb_encoder_fwd_varlen",
    "vb_encoder_bwd_varlen", "vb_attention_probs", "vb_encoder_attention_probs",
    "vb_encoder_infer_workspace", "vb_encoder_infer", "vb_encoder_infer_varlen",
    "vb_set_deterministic", "vb_deterministic_workspace_bytes", "vb_set_dropout_offset",
    "vb_bert_adam_step_sched", "vb_bert_adam_sched_check",
    "vb_encoder_ckpt_layout", "vb_encoder_fwd_ckpt", "vb_encoder_bwd_ckpt", "vb_encoder_fwd_ckpt_varlen", "vb_encoder_bwd_ckpt_varlen",
    "vb_encoder_arena_layout_ffnrc", "vb_encoder_arena_layout_ffnrc_varlen", "vb_encoder_fwd_ffnrc", "vb_encoder_bwd_ffnrc",
    "vb_encoder_fwd_ffnrc_varlen", "vb_encoder_bwd_ffnrc_varlen",
]
VB_ENCODER_ARENA_BUFFERS = 14
ARENA_NAMES = ("qkv", "ctx", "lse", "pre1", "mean1", "rstd1", "x1", "u", "g", "pre2", "mean2", "rstd2", "keep_mask", "y")
CKPT_NAMES = ("y", "mean2", "rstd2")   # the buffers of one checkpoint region (vb_encoder_ckpt_layout)


class VBertLibraryError(RuntimeError):
    pass


_lib = None


def lib():
    """Load (once) and return the ctypes handle; raise loudly when the CUDA library is absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise VBertLibraryError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'`. "
                "visualbert_b200 has no CPU or PyTorch fallback.")
        h = ctypes.CDLL(LIB_PATH)
        h.vb_last_error.restype = ctypes.c_char_p
        h.vb_launch_count.restype = ctypes.c_int64
        h.vb_abi_version.restype = ctypes.c_int
        h.vb_attention_keep_bytes.restype = ctypes.c_int64
        h.vb_encoder_arena_layout.restype = ctypes.c_int64
        h.vb_encoder_arena_layout_varlen.restype = ctypes.c_int64
        _P, _I, _F, _U64, _U32 = c_void_p, c_int, c_f32, c_u64, c_u32
        h.vb_attention_fwd_varlen.argtypes = [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _F, _U64, _U32, _P]
        h.vb_attention_bwd_varlen.argtypes = [_P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _F, _U64, _U32, _P]
        h.vb_encoder_arena_layout_varlen.argtypes = [_I, _I, _I, _I, _I, _I, _I, _P]
        h.vb_encoder_fwd_varlen.argtypes = [_P, _I, _P, _I, _P, _P, _P]
        h.vb_encoder_bwd_varlen.argtypes = [_P, _I, _P, _I, _P, _P, _P, _P, _P, _P, _P]
        h.vb_attention_probs.argtypes = [_P, _P, _P, _I, _I, _I, _I, _P]
        h.vb_encoder_attention_probs.argtypes = [_P, _I, _P, _P, _P]
        h.vb_encoder_infer_workspace.restype = ctypes.c_int64
        h.vb_encoder_infer_workspace.argtypes = [_I, _I, _I, _I, _I, _I, c_i64]
        h.vb_encoder_infer.argtypes = [_P, _I, _P, _P, _P, _P, _P, _P]
        h.vb_encoder_infer_varlen.argtypes = [_P, _I, _P, _I, _P, _P, _P, _P, _P]
        h.vb_set_deterministic.argtypes = [_P, c_i64]
        h.vb_deterministic_workspace_bytes.restype = ctypes.c_int64
        h.vb_deterministic_workspace_bytes.argtypes = [c_i64, _I, _I, _I, _I]
        h.vb_set_dropout_offset.argtypes = [_P]
        _D = ctypes.c_double
        h.vb_bert_adam_step_sched.argtypes = [_P, _I, _I, _P, _I, _P, _P, _P, _D, _D, _D, _D, _P]
        h.vb_bert_adam_sched_check.argtypes = [_P, _I, _I, _P, _I]
        h.vb_encoder_ckpt_layout.restype = ctypes.c_int64
        h.vb_encoder_ckpt_layout.argtypes = [_I, _I, _I, _I, _I, c_i64, _P]
        h.vb_encoder_fwd_ckpt.argtypes = [_P, _I, _P, _P, _P, _P, _P]
        h.vb_encoder_bwd_ckpt.argtypes = [_P, _I, _P, _P, _P, _P, _P, _P, _P, _P]
        h.vb_encoder_fwd_ckpt_varlen.argtypes = [_P, _I, _P, _I, _P, _P, _P, _P]
        h.vb_encoder_bwd_ckpt_varlen.argtypes = [_P, _I, _P, _I, _P, _P, _P, _P, _P, _P, _P, _P]
        h.vb_encoder_arena_layout_ffnrc.restype = ctypes.c_int64
        h.vb_encoder_arena_layout_ffnrc.argtypes = [_I, _I, _I, _I, _I, _I, _P, _P]
        h.vb_encoder_arena_layout_ffnrc_varlen.restype = ctypes.c_int64
        h.vb_encoder_arena_layout_ffnrc_varlen.argtypes = [_I, _I, _I, _I, _I, _I, _I, _P, _P]
        h.vb_encoder_fwd_ffnrc.argtypes = [_P, _I, _P, _P, _P, _P]
        h.vb_encoder_bwd_ffnrc.argtypes = [_P, _I, _P, _P, _P, _P, _P, _P, _P, _P]
        h.vb_encoder_fwd_ffnrc_varlen.argtypes = [_P, _I, _P, _I, _P, _P, _P, _P]
        h.vb_encoder_bwd_ffnrc_varlen.argtypes = [_P, _I, _P, _I, _P, _P, _P, _P, _P, _P, _P, _P]
        _lib = h
    return _lib


def check(rc, what):
    if rc != 0:
        msg = lib().vb_last_error().decode("utf-8", "replace")
        raise VBertLibraryError(f"{what} failed (status {rc}): {msg}")


def launch_count():
    return int(lib().vb_launch_count())


PROFILE_CATEGORIES = ("gemm_fwd", "gemm_dgrad", "gemm_wgrad", "attn_fwd", "attn_dq", "attn_dkv", "ln_fwd", "ln_bwd",
                      "colsum", "embed", "other")


def profile_enable(on=True):
    lib().vb_profile_enable(1 if on else 0)


def profile_read():
    """-> {category: dict(ms, work, launches)} since the previous read (synchronises the device)."""
    k = len(PROFILE_CATEGORIES)
    ms = (ctypes.c_double * k)(); work = (ctypes.c_double * k)(); n = (ctypes.c_int64 * k)()
    check(lib().vb_profile_read(ms, work, n), "vb_profile_read")
    return {c: dict(ms=ms[i], work=work[i], launches=int(n[i])) for i, c in enumerate(PROFILE_CATEGORIES)}
