"""Partial fine-tuning on the GPU: a parameter with requires_grad=False gets no gradient work and no kernel writes its .grad,
while the loss, the outputs and every trainable gradient keep the bits of the all-trainable run (deterministic mode) or stay
within fp32 reordering (default mode). Layers below the lowest trainable one run forward-only and take no arena slot."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(autouse=True)
def _cublas(monkeypatch):
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    yield
    torch.use_deterministic_algorithms(False)


def _model(layers, hidden, heads, inter, B, T, V, head, Dv=64, vocab=512):
    from visualbert_b200 import BertConfig, TrainVisualBERTObjective, synthetic
    cfg = synthetic.bert_config_dict(layers, hidden, heads, inter, vocab=vocab)
    model = TrainVisualBERTObjective(BertConfig.from_dict(cfg), head, visual_embedding_dim=Dv)
    model.load_state_dict(synthetic.init_state_dict(cfg, head, Dv, seed=0), strict=False)
    for m in model.modules():   # torch's own dropout in the heads draws from torch's generator: seeded per run below anyway
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    batch = synthetic.make_batch(B, T, V, Dv, head=head, seed=1234, vocab=vocab, ragged=True)
    return model.to(DEV).train(True), {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in batch.items()}


def _frozen(model, pattern, k=1):
    """Names of the parameters a pattern freezes."""
    names = [n for n, _ in model.named_parameters()]
    emb = [n for n in names if n.startswith("bert.embeddings.")]
    text = [n for n in emb if any(t in n for t in ("word_embeddings", ".position_embeddings.", ".token_type_embeddings."))]
    layer = lambda i: [n for n in names if n.startswith(f"bert.encoder.layer.{i}.")]
    L = len(model.bert.encoder.layer)
    return {
        "a": ["bert.embeddings.word_embeddings.weight"],
        "b": emb + [n for i in range(k) for n in layer(i)],
        "c": text + [n for i in range(L) for n in layer(i)],
        "d": ["bert.encoder.layer.0.attention.self.query.weight"],
        "e": [f"bert.encoder.layer.{L - 1}.attention.output.LayerNorm.weight"],
        "f": [n for n in names if n.startswith("bert.")],
    }[pattern]


def _set_frozen(model, names):
    for n, p in model.named_parameters():
        p.requires_grad_(n not in names)


def _run(model, batch, state, det, sync=None, sentinel=None):
    """One forward + backward. Returns (loss, encoder output, {name: grad} of trainable tensors, backward launches)."""
    from visualbert_b200 import _lib
    torch.use_deterministic_algorithms(det)
    try:
        torch.manual_seed(1234)
        model.bert.set_dropout_state(state)
        for n, p in model.named_parameters():
            p.grad = sentinel[n].clone() if (sentinel is not None and not p.requires_grad) else None
        if sync is not None:
            sync.zero()
        enc = []
        hook = model.bert.encoder.register_forward_hook(lambda m, i, o: enc.append(o[-1].detach().clone()))
        out = model(**batch)
        hook.remove()
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        out["loss"].backward()
        torch.cuda.synchronize()
        launches = _lib.launch_count() - n0
        # (a head's unused parameters keep no gradient)
        grads = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.requires_grad and p.grad is not None}
        return out["loss"].detach().clone(), enc[0], grads, launches
    finally:
        torch.use_deterministic_algorithms(False)


SHAPES = {
    "pretraining": dict(args=(3, 256, 4, 1024, 4, 20, 10), head="pretraining"),
    "vqa": dict(args=(2, 128, 2, 512, 4, 24, 12), head="vqa"),
}


@pytest.mark.parametrize("pattern", list("abcdef"))
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_frozen_pattern_keeps_every_trainable_bit(shape, pattern):
    from visualbert_b200 import parallel
    c = SHAPES[shape]
    model, batch = _model(*c["args"], head=c["head"])
    state = model.bert.dropout_state()
    ref = _run(model, batch, state, True)
    ref_default = _run(model, batch, state, False)
    frozen = _frozen(model, pattern)
    _set_frozen(model, frozen)
    params = dict(model.named_parameters())
    sentinel = {n: torch.full_like(params[n], 3.25) for n in frozen}
    for use_sync, sent in ((False, None), (False, sentinel), (True, None)):
        sync = parallel.FlatGradSync(model) if use_sync else None
        got = _run(model, batch, state, True, sync=sync, sentinel=sent)
        assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])
        want = {n for n in ref[2] if n not in frozen}
        assert want <= got[2].keys()
        for n in want:
            assert torch.equal(got[2][n], ref[2][n]), (pattern, use_sync, n)
        for n in frozen:
            if sent is None:
                assert params[n].grad is None, n
            else:
                assert torch.equal(params[n].grad, sentinel[n]), n
        # a frozen member of a packed output (d: query of q|k|v, e: a LayerNorm gamma) is computed and dropped, and a frozen word
        # table without the tied MLM decoder only drops the scatter inside the embedding kernel: no launch saved there
        fewer = pattern in "bcf" or (pattern == "a" and shape == "pretraining")
        assert got[3] < ref[3] if fewer else got[3] <= ref[3], (got[3], ref[3])
        for p in params.values():   # FlatGradSync's views stay attached to the parameters it saw: detach them for the next run
            p.grad = None
            p.__dict__.pop("_vb_direct_grad", None)
    got = _run(model, batch, state, False)
    assert torch.equal(got[0], ref_default[0])
    # fp32 atomics reorder the sums; the q|k|v bias gradients are sums that nearly cancel (softmax is shift-invariant), so the
    # bound takes at least 1e-4 of the model's largest gradient as the scale
    top = max(g.abs().max().item() for g in ref_default[2].values())
    for n, g in got[2].items():
        scale = ref_default[2][n].abs().max().item()
        assert (g - ref_default[2][n]).abs().max().item() <= 1e-5 * max(scale, 1e-4 * top), n


def test_frozen_bottom_layers_take_no_arena_slot():
    """Pattern (b) at 12 layers, H = 768: peak memory drops by at least k arena strides."""
    from visualbert_b200 import _lib
    model, batch = _model(12, 768, 12, 3072, 8, 32, 16, "vqa")
    state = model.bert.dropout_state()
    B, S = batch["input_ids"].shape[0], batch["input_ids"].shape[1] + batch["visual_embeddings"].shape[1]
    stride = int(_lib.lib().vb_encoder_arena_layout(B, S, 768, 12, 3072, 1, None))

    def peak():
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        r = _run(model, batch, state, True)
        return torch.cuda.max_memory_allocated() - base, r

    _run(model, batch, state, True)
    full, ref = peak()
    k = 6
    _set_frozen(model, _frozen(model, "b", k))
    _run(model, batch, state, True)
    part, got = peak()
    assert full - part >= k * stride, (full, part, stride)
    assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])
    for n, g in got[2].items():
        assert torch.equal(g, ref[2][n]), n


@pytest.mark.parametrize("pattern", ["a", "b"])
def test_frozen_unpadded(pattern):
    model, batch = _model(3, 256, 4, 1024, 4, 20, 10, "pretraining")
    model.bert.set_unpadded(True)
    state = model.bert.dropout_state()
    ref = _run(model, batch, state, True)
    _set_frozen(model, _frozen(model, pattern))
    got = _run(model, batch, state, True)
    assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])
    for n, g in got[2].items():
        assert torch.equal(g, ref[2][n]), n
    assert got[3] < ref[3]


@pytest.mark.parametrize("pattern", ["a", "b"])
def test_frozen_graphed_step_with_optimizer(pattern):
    """GraphedStep(optimizer=BertAdam) over three steps equals an eager loop with the same frozen set; toggling requires_grad
    captures a new graph."""
    from visualbert_b200 import BertAdam, graphs, parallel, synthetic
    torch.use_deterministic_algorithms(True)
    state = {"seed": 77, "step": 5}
    batches = []
    for i in range(3):
        b = synthetic.make_batch(4, 24, 16, 64, head="nlvr", seed=100 + i, vocab=512, ragged=True)
        batches.append({k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in b.items()})

    def setup():
        model, _ = _model(2, 128, 2, 256, 4, 24, 16, "nlvr")
        _set_frozen(model, _frozen(model, pattern))
        model.bert.set_dropout_state(state)
        sync = parallel.FlatGradSync(model)
        opt = BertAdam([p for p in model.parameters() if p.requires_grad], lr=1e-3, warmup=0.1, t_total=10, max_grad_norm=1.0)
        return model, sync, opt

    ref, ref_sync, ref_opt = setup()
    ref_losses = []
    for b in batches:
        ref_sync.zero()
        out = ref(**b)
        out["loss"].backward()
        ref_losses.append(out["loss"].detach().clone())
        ref_opt.step()
    model, sync, opt = setup()
    step = graphs.GraphedStep(model, sync, optimizer=opt)
    losses = [step(b)["loss"].detach().clone() for b in batches]
    assert len(step.graphs) == 1
    for a, b in zip(losses, ref_losses):
        assert torch.equal(a, b)
    for (n, p), q in zip(model.named_parameters(), ref.parameters()):
        assert torch.equal(p.detach(), q.detach()), n
    frozen = [p for p in model.parameters() if not p.requires_grad]
    frozen[0].requires_grad_(True)
    step(batches[0])   # a new trainable set: warm-up call, then a second capture
    step(batches[1])
    assert len(step.graphs) == 2
    torch.use_deterministic_algorithms(False)
