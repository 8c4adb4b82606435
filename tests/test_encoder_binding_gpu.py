"""The Python binding of the encoder call (ops._EncoderFn), which serves the whole stack and single layers alike.

  * a backward describes its own forward: a forward of another shape between a forward and its backward changes nothing;
  * the layer-by-layer route (output_all_encoded_layers=True in training under grad: one one-layer encoder call per layer)
    computes what the whole-encoder call computes, and its intermediate outputs are differentiable."""
import pytest
import torch

pytestmark = pytest.mark.gpu

GRAD_TOL = 1e-5   # relative; the order of the fp32 atomic adds in the weight gradients is the only difference between two runs


def _model_and_batches(batch_sizes, layers=3, hidden=256, heads=4, inter=1024, T=40, V=20, Dv=64):
    from visualbert_b200 import BertConfig, TrainVisualBERTObjective, synthetic
    dev = torch.device("cuda:0")
    cfg = synthetic.bert_config_dict(layers, hidden, heads, inter, vocab=4096)
    model = TrainVisualBERTObjective(BertConfig.from_dict(cfg), "pretraining", visual_embedding_dim=Dv)
    model.load_state_dict(synthetic.init_state_dict(cfg, "pretraining", Dv, seed=0), strict=False)
    model.to(dev).train()
    batches = []
    for i, B in enumerate(batch_sizes):
        b = synthetic.make_batch(B, T, V, Dv, head="pretraining", seed=7 + i, vocab=4096, ragged=True)
        batches.append({k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in b.items()})
    return model, batches


def _grads(module):
    return {n: (None if p.grad is None else p.grad.detach().clone()) for n, p in module.named_parameters()}


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-300)).item()


def _assert_same_grads(got, want, names=None):
    for n in (want if names is None else names):
        assert (got[n] is None) == (want[n] is None), n
        if want[n] is not None:
            assert _rel(got[n], want[n]) <= GRAD_TOL, f"{n}: {_rel(got[n], want[n]):.3g}"


def test_backward_uses_the_descriptors_of_its_own_forward():
    """Forward X, forward a batch of fewer examples, backward X: the gradients are those of forward X, backward X."""
    model, (x, y) = _model_and_batches((6, 2))
    model.bert._step = 0
    model(**x)["loss"].backward()
    want = _grads(model)
    assert any(g is not None and g.abs().max().item() > 0 for n, g in want.items() if ".encoder." in n)

    model.bert._step = 0
    model.zero_grad(set_to_none=True)
    loss_x = model(**x)["loss"]
    loss_y = model(**y)["loss"]
    loss_x.backward()
    _assert_same_grads(_grads(model), want)
    assert torch.isfinite(loss_y)


def _bert_forward(model, b, all_layers):
    mask = torch.cat((b["input_mask"], b["image_mask"]), 1)
    model.bert._step = 0
    model.zero_grad(set_to_none=True)
    return model.bert(b["input_ids"], b["token_type_ids"], mask, b["visual_embeddings"], None, b["visual_embeddings_type"],
                      None, None, output_all_encoded_layers=all_layers)


def test_layer_by_layer_route_equals_the_whole_encoder_call_and_differentiates_intermediate_outputs():
    model, (b,) = _model_and_batches((4,))
    bert = model.bert
    S, H = 60, 256
    torch.manual_seed(3)
    w_last, w_mid = torch.randn(S, H, device="cuda:0"), torch.randn(S, H, device="cuda:0")

    def loss_of(last, pooled):
        return (last.float() * w_last).sum() + pooled.sum()

    last, pooled = _bert_forward(model, b, all_layers=False)
    loss_of(last, pooled).backward()
    fused_out, fused = last.detach().clone(), _grads(bert)

    layers, pooled = _bert_forward(model, b, all_layers=True)
    assert len(layers) == 3 and all(y.requires_grad for y in layers)
    assert torch.equal(layers[-1], fused_out)
    loss_of(layers[-1], pooled).backward()
    by_layer = _grads(bert)
    _assert_same_grads(by_layer, fused)

    # a loss that also reads the first layer's output: layers 1 and 2 come after it and keep their gradients, the first
    # layer's change
    layers, pooled = _bert_forward(model, b, all_layers=True)
    (loss_of(layers[-1], pooled) + (layers[0].float() * w_mid).sum()).backward()
    both = _grads(bert)
    _assert_same_grads(both, by_layer, [n for n in by_layer if n.startswith(("encoder.layer.1.", "encoder.layer.2.", "pooler."))])
    k = "encoder.layer.0.output.dense.weight"
    assert _rel(both[k], by_layer[k]) > 1e-2
