"""CPU-side checks of the drop-in boundary: the shared library loads, exports every symbol the header declares,
the ctypes mirrors match the C struct sizes, and the product path refuses to run without CUDA (no CPU fallback)."""
import ctypes
import os
import re
import subprocess

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_loads_and_exports_every_declared_symbol():
    from visualbert_b200 import _lib
    L = _lib.lib()
    header = open(os.path.join(ROOT, "include", "vbert_b200.h")).read()
    declared = set(re.findall(r"\b(vb_[a-z0-9_]+)\s*\(", header))
    assert declared == set(_lib.EXPORTS), declared ^ set(_lib.EXPORTS)
    for name in declared:
        assert hasattr(L, name), name
    assert L.vb_abi_version() == _lib.ABI_VERSION == int(re.search(r"#define VB_ABI_VERSION (\d+)", header).group(1))
    assert L.vb_launch_count() == 0


def test_struct_mirrors_match_c_sizes(tmp_path):
    from visualbert_b200 import _lib
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include "vbert_b200.h"\nint main(){printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %d %d %d\\n",'
                   'sizeof(vb_gemm_args),sizeof(vb_layer_desc),sizeof(vb_layer_acts),sizeof(vb_layer_grads),'
                   'sizeof(vb_layer_scratch),sizeof(vb_embed_desc),sizeof(vb_embed_acts),sizeof(vb_embed_grads),sizeof(vb_adam_tensor),'
                   'sizeof(vb_cast_item),VB_ADAM_CHUNK,VB_CAST_CHUNK,VB_ENCODER_ARENA_BUFFERS);return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    sizes = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    mirrors = [_lib.GemmArgs, _lib.LayerDesc, _lib.LayerActs, _lib.LayerGrads, _lib.LayerScratch, _lib.EmbedDesc,
               _lib.EmbedActs, _lib.EmbedGrads, _lib.AdamTensor, _lib.CastItem]
    assert sizes == [ctypes.sizeof(m) for m in mirrors] + [_lib.VB_ADAM_CHUNK, _lib.VB_CAST_CHUNK, _lib.VB_ENCODER_ARENA_BUFFERS]
    assert len(_lib.ARENA_NAMES) == _lib.VB_ENCODER_ARENA_BUFFERS


def test_encoder_arena_layout_is_aligned_and_ordered():
    """vb_encoder_arena_layout (no GPU needed): 14 buffers per layer slot, 256-byte aligned, sized for the shapes."""
    from visualbert_b200 import _lib
    L = _lib.lib()
    off = (ctypes.c_int64 * _lib.VB_ENCODER_ARENA_BUFFERS)()
    B, S, H, A, I = 4, 56, 768, 12, 3072
    stride = L.vb_encoder_arena_layout(B, S, H, A, I, 1, off)
    o = list(off)
    M = B * S
    assert o[0] == 0 and all(x % 256 == 0 for x in o) and stride % 256 == 0
    sizes = dict(zip(_lib.ARENA_NAMES, [b - a for a, b in zip(o, o[1:] + [stride])]))
    assert sizes["qkv"] >= M * 3 * H * 2 and sizes["u"] >= M * I * 2 and sizes["y"] >= M * H * 2 and sizes["lse"] >= B * A * S * 4
    assert sizes["keep_mask"] >= L.vb_attention_keep_bytes(B, S, A)
    stride0 = L.vb_encoder_arena_layout(B, S, H, A, I, 0, off)
    assert stride0 == stride - sizes["keep_mask"]


def test_argument_validation_reports_through_vb_last_error():
    from visualbert_b200 import _lib
    L = _lib.lib()
    a = _lib.GemmArgs()  # all zero: empty problem
    rc = L.vb_gemm(ctypes.byref(a), None)
    assert rc != 0
    assert b"empty problem" in L.vb_last_error()
    assert L.vb_gemm(None, None) != 0


# 32-byte aligned fake device pointers: every check in vb_gemm runs before its first CUDA call
_FAKE = dict(A=0x10000, lda=256, B=0x20000, ldb=256, M=256, N=256, K=256, D=0x30000, ldd=256)


def test_gemm_refuses_an_unknown_epilogue():
    from visualbert_b200 import _lib
    L = _lib.lib()
    for epi in (3, -1, 9):
        a = _lib.GemmArgs(epilogue=epi, aux_in=0x40000, aux_out=0x50000, ld_aux=256, **_FAKE)
        assert L.vb_gemm(ctypes.byref(a), None) != 0
        assert b"unknown epilogue" in L.vb_last_error()


@pytest.mark.parametrize("epi", ["gelu", "dgelu"])
@pytest.mark.parametrize("extra", ["dropout", "addend"])
def test_gemm_refuses_gelu_epilogues_with_dropout_or_addend(epi, extra):
    from visualbert_b200 import _lib
    L = _lib.lib()
    kw = dict(epilogue=_lib.VB_EPI_GELU, aux_out=0x50000) if epi == "gelu" else dict(epilogue=_lib.VB_EPI_DGELU, aux_in=0x40000)
    kw.update(dict(dropout_p=0.1, dropout_seed=1) if extra == "dropout" else dict(addend=0x60000, ld_add=256))
    a = _lib.GemmArgs(ld_aux=256, **kw, **_FAKE)
    assert L.vb_gemm(ctypes.byref(a), None) != 0
    assert b"take no dropout and no addend" in L.vb_last_error()


_A, _BAD = 0x10000, 0x10008   # a 16-byte aligned and an 8-byte (not 16-byte) aligned fake device pointer


def _refused(rc, words):
    from visualbert_b200 import _lib
    assert rc != 0
    assert words.encode() in _lib.lib().vb_last_error()


def _p(v):
    return ctypes.c_void_p(v)


@pytest.mark.parametrize("bad", ["x", "y", "gamma", "beta", "ldx", "ldy", "ldx<H"])
def test_layernorm_forward_refuses_what_its_vector_loads_cannot_take(bad):
    """Every check of vb_layernorm_fwd runs before its first CUDA call: a misaligned pointer or row stride is an error."""
    from visualbert_b200 import _lib
    H = 64
    a = dict(x=_A, y=_A, gamma=_A, beta=_A, ldx=H, ldy=H)
    if bad in ("ldx", "ldy"):
        a[bad] = H + 4
    elif bad == "ldx<H":
        a["ldx"] = H - 8
    else:
        a[bad] = _BAD
    rc = _lib.lib().vb_layernorm_fwd(_p(a["x"]), ctypes.c_int64(a["ldx"]), _p(a["gamma"]), _p(a["beta"]), _p(a["y"]),
                                     ctypes.c_int64(a["ldy"]), None, None, 4, H, ctypes.c_float(1e-12), None)
    _refused(rc, "16-byte aligned" if bad in a and bad not in ("ldx", "ldy") else "must be multiples of 8 and >= H")


@pytest.mark.parametrize("bad", ["dy", "x", "gamma", "dx", "dx_drop"])
def test_layernorm_backward_refuses_a_misaligned_pointer(bad):
    from visualbert_b200 import _lib
    a = dict(dy=_A, x=_A, gamma=_A, dx=_A, dx_drop=_A)
    a[bad] = _BAD
    rc = _lib.lib().vb_layernorm_bwd(_p(a["dy"]), _p(a["x"]), _p(_A), _p(_A), _p(a["gamma"]), _p(a["dx"]), _p(a["dx_drop"]),
                                     None, None, None, 4, 64, ctypes.c_float(0.1), ctypes.c_uint64(1), ctypes.c_uint32(0),
                                     ctypes.c_float(0.0), ctypes.c_uint32(0), None)
    _refused(rc, "16-byte aligned")


@pytest.mark.parametrize("x,ld,words", [(_BAD, 64, "16-byte aligned"), (_A, 68, "multiple of 8"), (_A, 56, ">= N")])
def test_colsum_refuses_a_misaligned_pointer_or_stride(x, ld, words):
    from visualbert_b200 import _lib
    _refused(_lib.lib().vb_colsum_bf16(_p(x), ctypes.c_int64(ld), _p(_A), 5, 64, None), words)


@pytest.mark.parametrize("rows", [0, 3])
def test_cross_entropy_refuses_misaligned_logits(rows):
    from visualbert_b200 import _lib
    L = _lib.lib()
    _refused(L.vb_cross_entropy_fwd(_p(_BAD), ctypes.c_int64(16), _p(_A), rows, 9, _p(_A), _p(_A), None), "16-byte aligned")
    _refused(L.vb_cross_entropy_bwd(_p(_BAD), ctypes.c_int64(16), _p(_A), rows, 9, 16, _p(_A), _p(_A), None), "16-byte aligned")


@pytest.mark.parametrize("src,dst", [(_BAD, _A), (_A, _BAD)])
def test_casts_refuse_a_misaligned_pointer(src, dst):
    from visualbert_b200 import _lib
    L = _lib.lib()
    _refused(L.vb_cast_f32_to_bf16(_p(src), _p(dst), ctypes.c_int64(64), None), "16-byte aligned")
    _refused(L.vb_cast_bf16_to_f32(_p(src), _p(dst), ctypes.c_int64(64), None), "16-byte aligned")


@pytest.mark.parametrize("bad", ["word", "pos", "type", "pos_vis", "type_vis", "pre", "y"])
def test_embedding_forward_refuses_misaligned_tables(bad):
    """Refused before anything is launched (the projection GEMM included)."""
    from visualbert_b200 import _lib
    tabs = {k: (_BAD if k == bad else _A) for k in ("word", "pos", "type", "pos_vis", "type_vis", "pre", "y")}
    d = _lib.EmbedDesc(batch=2, text_len=4, num_regions=0, hidden=64, visual_dim=0, vocab=10, max_pos=8, n_types=2, eps=1e-12,
                       input_ids=_A, token_type_ids=_A, word=tabs["word"], pos=tabs["pos"], type=tabs["type"],
                       pos_vis=tabs["pos_vis"], type_vis=tabs["type_vis"], gamma=_A, beta=_A)
    acts = _lib.EmbedActs(vis_proj=0, pre=tabs["pre"], mean=_A, rstd=_A)
    _refused(_lib.lib().vb_embed_fwd(ctypes.byref(d), _p(tabs["y"]), ctypes.byref(acts), None), "16-byte aligned")


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU behaviour")
def test_product_path_fails_loudly_without_cuda():
    from visualbert_b200 import BertConfig, TrainVisualBERTObjective, _lib, synthetic
    cfg = BertConfig.from_dict(synthetic.bert_config_dict(1, 128, 2, 512, vocab=64))
    model = TrainVisualBERTObjective(cfg, "nlvr", visual_embedding_dim=64).eval()
    batch = synthetic.make_batch(2, 6, 3, 64, head="nlvr", vocab=64)
    with pytest.raises(_lib.VBertLibraryError):
        model(**batch)


def test_config_round_trip(tmp_path):
    from visualbert_b200 import BertConfig
    c = BertConfig(30522, hidden_size=768)
    p = tmp_path / "bert_config.json"
    p.write_text(c.to_json_string())
    c2 = BertConfig.from_json_file(str(p))
    assert c2.to_dict() == c.to_dict()
    assert BertConfig(str(p)).hidden_size == 768
    with pytest.raises(ValueError):
        BertConfig(3.5)


def test_from_pretrained_local_directory(tmp_path):
    from visualbert_b200 import BertConfig, TrainVisualBERTObjective, synthetic
    cfgd = synthetic.bert_config_dict(1, 128, 2, 512, vocab=64)
    (tmp_path / "bert_config.json").write_text(BertConfig.from_dict(cfgd).to_json_string())
    m = TrainVisualBERTObjective.from_pretrained(str(tmp_path), random_initialize=True, training_head_type="pretraining",
                                                 visual_embedding_dim=64)
    sd = {k: v + 1 for k, v in m.state_dict().items()}
    sd["bert.embeddings.LayerNorm.gamma"] = sd.pop("bert.embeddings.LayerNorm.weight")  # TF-era name (M.py:556-568)
    torch.save(sd, str(tmp_path / "pytorch_model.bin"))
    m2 = TrainVisualBERTObjective.from_pretrained(str(tmp_path), training_head_type="pretraining", visual_embedding_dim=64)
    for k, v in m.state_dict().items():
        assert torch.allclose(m2.state_dict()[k], v + 1), k
    m.bert.embeddings.special_intialize()
    assert torch.equal(m.bert.embeddings.token_type_embeddings_visual.weight, m.bert.embeddings.token_type_embeddings.weight)
    with pytest.raises(EnvironmentError):
        TrainVisualBERTObjective.from_pretrained("bert-base-uncased", training_head_type="nlvr")


def test_lazy_output_dict_defers_and_caches():
    from visualbert_b200.modeling import LazyOutputDict
    d, calls = LazyOutputDict(), []
    d.set_lazy("logits", lambda: (calls.append(1), 42)[1])
    d["loss"] = 1.5
    assert "logits" in d and list(d.keys()) == ["logits", "loss"] and not calls
    assert d["logits"] == 42 and d["logits"] == 42 and len(calls) == 1
    e = LazyOutputDict()
    e.set_lazy("x", lambda: 7)
    assert dict(e.items()) == {"x": 7} and e.get("y", 3) == 3
    e["x"] = 8
    assert e["x"] == 8


def test_documented_tile_native_layout_is_a_permutation():
    """include/vbert_b200.h documents where vb_gemm_args.gp_tiled puts element (row, col) of gelu'(u); the formula must be a bijection
    onto [0, M * N) in 16-element groups (tests/test_kernels_gpu.py checks the kernels against the same formula on the GPU)."""
    M, N = 512, 768
    row = torch.arange(M).view(M, 1).expand(M, N)
    col = torch.arange(N).view(1, N).expand(M, N)
    mb, r, q, l = row // 256, (row % 256) // 128, (row % 128) // 32, row % 32
    nb, half, k, e = col // 256, (col % 256) // 128, (col % 128) // 16, col % 16
    w = 4 * half + q
    off = ((((mb * (N // 256) + nb) * 2 + r) * 8 + w) * 8 + k) * 512 + 16 * l + e
    assert off.min() == 0 and off.max() == M * N - 1 and torch.unique(off).numel() == M * N
    # the same thing as a view / permute of the flat buffer (what the GPU test uses)
    flat = torch.empty(M * N, dtype=torch.int64)
    flat[off.reshape(-1)] = (row * N + col).reshape(-1)
    t = flat.view(M // 256, N // 256, 2, 2, 4, 8, 32, 16).permute(0, 2, 4, 6, 1, 3, 5, 7).reshape(M, N)
    assert torch.equal(t, row * N + col)
