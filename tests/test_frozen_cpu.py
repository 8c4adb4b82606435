"""Partial fine-tuning without a GPU: the plan that turns requires_grad flags into the lowest layer a backward reaches and the
NULL fields of vb_layer_grads, and the C ABI's documentation and refusals of those NULL fields."""
import ctypes
import os

import torch

from visualbert_b200 import _lib, ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = [f for f, _ in ops._GRAD_FIELDS]


def _encoder(L=3, H=64, I=128):
    from visualbert_b200 import BertConfig, modeling, synthetic
    cfg = BertConfig.from_dict(synthetic.bert_config_dict(L, H, 1, I, vocab=64))
    return modeling.BertEncoder(cfg)


def _plan(enc, input_grad=False):
    params = enc._fused_params()
    return ops.encoder_grad_plan(params, [p.requires_grad for p in params], input_grad)


def test_all_trainable_without_grad_owner_uses_buffers():
    l0, layers = _plan(_encoder())
    assert l0 == 0 and len(layers) == 3
    for direct, kinds in layers:
        assert not direct and all(kinds[f] == "buffer" for f in FIELDS)


def test_all_trainable_with_flat_grad_sync_accumulates_directly():
    from visualbert_b200 import parallel
    enc = _encoder()
    parallel.FlatGradSync(enc)
    l0, layers = _plan(enc)
    assert l0 == 0 and all(direct and all(k[f] == "grad" for f in FIELDS) for direct, k in layers)


def test_frozen_bottom_layers_set_l0():
    enc = _encoder()
    for l in enc.layer[:2]:
        l.requires_grad_(False)
    l0, layers = _plan(enc)
    assert l0 == 2 and len(layers) == 1
    assert _plan(enc, input_grad=True)[0] == 0
    enc.layer[2].requires_grad_(False)
    assert _plan(enc)[0] == 3


def test_input_gradient_only_layers_are_all_null():
    enc = _encoder()
    enc.requires_grad_(False)
    l0, layers = _plan(enc, input_grad=True)
    assert l0 == 0 and all(all(k[f] == "null" for f in FIELDS) for _, k in layers)


def test_frozen_query_weight_is_a_partial_group():
    from visualbert_b200 import parallel
    enc = _encoder()
    enc.layer[1].attention.self.query.weight.requires_grad_(False)
    parallel.FlatGradSync(enc)
    l0, layers = _plan(enc)
    assert l0 == 0
    direct, kinds = layers[1]
    assert direct and kinds["dw_qkv"] == "buffer" and kinds["db_qkv"] == "grad"
    assert all(kinds[f] == "grad" for f in FIELDS if f != "dw_qkv")
    assert all(k[f] == "grad" for _, k in (layers[0], layers[2]) for f in FIELDS)


def test_frozen_layernorm_gamma_keeps_its_group():
    enc = _encoder()
    enc.layer[0].output.LayerNorm.weight.requires_grad_(False)
    enc.layer[0].attention.output.LayerNorm.requires_grad_(False)
    enc.layer[0].attention.output.dense.bias.requires_grad_(False)
    _, layers = _plan(enc)
    kinds = layers[0][1]
    assert kinds["dln2_gamma"] == "buffer" and kinds["dln2_beta"] == "buffer" and kinds["db_out"] == "buffer"
    assert kinds["dln1_gamma"] == kinds["dln1_beta"] == kinds["db_attn_out"] == "null"


def test_layer_grads_pointers_follow_the_plan():
    enc = _encoder(L=1, H=64, I=128)
    enc.layer[0].attention.self.key.weight.requires_grad_(False)
    enc.layer[0].intermediate.dense.requires_grad_(False)
    params = enc._fused_params()
    tr = [p.requires_grad for p in params]
    _, plan = ops.encoder_grad_plan(params, tr, True)
    grads, flat, pieces = ops._layer_grads(params, tr, plan, 64, 128, "cpu")
    assert grads[0].dw_inter in (None, 0) and grads[0].db_inter in (None, 0)
    assert grads[0].dw_qkv == flat.data_ptr()
    got = {i for i, _ in pieces}
    assert 2 not in got and 10 not in got and 11 not in got and {0, 4} <= got
    assert flat.numel() == 3 * 64 * 64 + 3 * 64 + 64 * 64 + 3 * 64 + 128 * 64 + 3 * 64


def test_header_documents_null_gradient_fields():
    h = open(os.path.join(ROOT, "include", "vbert_b200.h")).read()
    assert "#define VB_ABI_VERSION 4" in h and _lib.lib().vb_abi_version() == 4
    for phrase in ("A NULL field is not computed", "dx may be NULL", "receives no scatter"):
        assert phrase in h, phrase


def test_partial_layernorm_group_is_refused():
    L = _lib.lib()
    descs = (_lib.LayerDesc * 1)()
    grads = (_lib.LayerGrads * 1)()
    grads[0].dln1_gamma = 256   # dln1_beta and db_attn_out NULL
    fake = ctypes.c_void_p(256)
    sc = _lib.LayerScratch()
    rc = L.vb_encoder_bwd(descs, 1, fake, fake, fake, None, grads, ctypes.byref(sc), None)
    assert rc != 0 and b"computed together" in L.vb_last_error()
