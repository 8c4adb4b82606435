"""CUDA-graph training steps on the GPU.

- Op level: every library route with its dropout seed offset in device memory (vb_set_dropout_offset) gives the bits of the same
  call with seed + offset by value — GEMM epilogues at both tile widths, LayerNorm backward with both dropouts, embeddings,
  encoder forward / backward / forward-only at S = 164 (wgmma attention), 224 (whole-head) and 356 (staged), dense and
  variable-length — for offsets that carry across bit 32. Another thread is not affected by the offset.
- Run-time read: a captured encoder forward + backward replayed with the counter changed between replays equals eager calls.
- GraphedStep: six steps of the NLVR and VQA models, BertAdam between them, bit-equal to the same steps run eagerly; fresh masks
  on every replay; two shapes interleaved and an evicted graph; a captured eval forward sees weight changes; refused cases.
"""
import ctypes
import threading

import pytest
import torch

pytestmark = pytest.mark.gpu

K = 0xA5A5A5A5FFFFFFF0                    # the low word wraps for either offset below
OFFSETS = (2 ** 32 - 1, 2 ** 32)
DEV = "cuda:0"


@pytest.fixture(autouse=True)
def _deterministic(monkeypatch):
    """Gradients are compared bit for bit: fixed-order reductions (torch's flag turns on the library's, and the heads' cuBLAS
    needs a workspace configuration for it)."""
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(False)
    from visualbert_b200 import _lib
    _lib.lib().vb_set_deterministic(None, 0)
    _lib.lib().vb_set_dropout_offset(None)


def _off(d):
    return torch.tensor([d], dtype=torch.int64, device=DEV)


def _model(head, S_text, V, layers=2, hidden=128, heads=2, inter=256, Dv=64, B=2, seed=1234, p_head=0.0):
    from visualbert_b200 import BertConfig, TrainVisualBERTObjective, synthetic
    cfg = synthetic.bert_config_dict(layers, hidden, heads, inter, vocab=512)
    sd = synthetic.init_state_dict(cfg, head, Dv, seed=0)
    model = TrainVisualBERTObjective(BertConfig.from_dict(cfg), head, visual_embedding_dim=Dv)
    model.load_state_dict(sd, strict=False)
    for m in model.modules():   # torch's own dropout draws from torch's generator, whose sequence under capture is not ours
        if isinstance(m, torch.nn.Dropout):
            m.p = p_head
    model = model.to(DEV).train(True)
    batch = synthetic.make_batch(B, S_text, V, Dv, head=head, seed=seed, vocab=512, ragged=True)
    return model, {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in batch.items()}


def _encoder_run(enc, x, bias, dy, seed, off, varlen=None, grad=True):
    from visualbert_b200 import ops
    enc.zero_grad(set_to_none=True)
    xi = x.detach().clone().requires_grad_(grad)
    with ops.forward_seed_offset(off), torch.set_grad_enabled(grad):
        y = enc(xi, bias, output_all_encoded_layers=False, seed=seed, varlen=varlen)[-1]
    if not grad:
        return [y]
    y.float().backward(dy)
    return [y.detach(), xi.grad] + [p.grad.clone() for p in enc.parameters()]


def _same(a, b):
    assert len(a) == len(b)
    for i, (u, v) in enumerate(zip(a, b)):
        assert torch.equal(u, v), i


@pytest.mark.parametrize("S", [164, 224, 356])
@pytest.mark.parametrize("varlen", [False, True])
def test_encoder_offset_equals_seed_by_value(S, varlen):
    from visualbert_b200 import ops
    model, _ = _model("nlvr", 8, 8)
    enc = model.bert.encoder
    B, H = 2, 128
    g = torch.Generator(device=DEV).manual_seed(S)
    valid = torch.ones(B, S, dtype=torch.bool, device=DEV)
    valid[1, S - 37:] = False
    if varlen:
        vl = ops.unpad_plan(valid)
        x = torch.randn(vl["total"], H, generator=g, device=DEV).bfloat16()
        bias = None
    else:
        vl = None
        x = torch.randn(B, S, H, generator=g, device=DEV).bfloat16()
        bias = ops.mask_bias(valid.long(), None)
    dy = torch.randn(x.shape, generator=g, device=DEV)
    for d in OFFSETS:
        ref = _encoder_run(enc, x, bias, dy, (K + d) % 2 ** 64, None, vl)
        _same(_encoder_run(enc, x, bias, dy, K, _off(d), vl), ref)
        _same(_encoder_run(enc, x, bias, dy, K, _off(d), vl, grad=False), ref[:1])   # forward-only route
    assert not torch.equal(ref[0], _encoder_run(enc, x, bias, dy, K, None, vl)[0])  # the offset matters


def _gemm(M, N, K_, p, seed, addend=True):
    from visualbert_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(N)
    a = torch.randn(M, K_, generator=g, device=DEV).bfloat16()
    w = torch.randn(N, K_, generator=g, device=DEV).bfloat16()
    bias = torch.randn(N, generator=g, device=DEV)
    res = torch.randn(M, N, generator=g, device=DEV).bfloat16()
    d = torch.empty(M, N, device=DEV, dtype=torch.bfloat16)
    kw = dict(addend=res.data_ptr(), ld_add=N) if addend else {}
    ops._gemm(torch.device(DEV), A=a.data_ptr(), lda=K_, B=w.data_ptr(), ldb=K_, M=M, N=N, K=K_, D=d.data_ptr(), ldd=N,
              bias=bias.data_ptr(), dropout_p=p, dropout_seed=seed, dropout_stream=7, **kw)
    return d


@pytest.mark.parametrize("N", [384, 768])    # 128- and 256-wide tiles
@pytest.mark.parametrize("addend", [False, True])
def test_gemm_offset(N, addend):
    from visualbert_b200 import ops
    for d in OFFSETS:
        ref = _gemm(300, N, 256, 0.1, (K + d) % 2 ** 64, addend)
        with ops.dropout_offset(_off(d)):
            got = _gemm(300, N, 256, 0.1, K, addend)
        assert torch.equal(got, ref)
        # a call on another thread does not see this thread's offset
        out = {}
        with ops.dropout_offset(_off(d)):
            t = threading.Thread(target=lambda: out.setdefault("y", _gemm(300, N, 256, 0.1, K, addend)))
            t.start()
            t.join()
        assert torch.equal(out["y"], _gemm(300, N, 256, 0.1, K, addend))


@pytest.mark.parametrize("H", [128, 768, 1024])
def test_layernorm_backward_offset(H):
    from visualbert_b200 import _lib, ops
    L = _lib.lib()
    rows = 333
    g = torch.Generator(device=DEV).manual_seed(H)
    dy, x = (torch.randn(rows, H, generator=g, device=DEV).bfloat16() for _ in range(2))
    mean, rstd = torch.randn(rows, generator=g, device=DEV), torch.rand(rows, generator=g, device=DEV) + 0.5
    gamma = torch.randn(H, generator=g, device=DEV)

    def run(seed):
        dx, dxd = torch.empty_like(dy), torch.empty_like(dy)
        dg, db, dbias = (torch.zeros(H, device=DEV) for _ in range(3))
        P = ctypes.c_void_p
        rc = L.vb_layernorm_bwd(P(dy.data_ptr()), P(x.data_ptr()), P(mean.data_ptr()), P(rstd.data_ptr()), P(gamma.data_ptr()),
                                P(dx.data_ptr()), P(dxd.data_ptr()), P(dg.data_ptr()), P(db.data_ptr()), P(dbias.data_ptr()), rows, H,
                                ctypes.c_float(0.1), ctypes.c_uint64(seed), ctypes.c_uint32(5), ctypes.c_float(0.1), ctypes.c_uint32(9),
                                P(torch.cuda.current_stream().cuda_stream))
        _lib.check(rc, "vb_layernorm_bwd")
        return [dx, dxd]   # (dbias: column sums by atomics outside the deterministic mode)
    for d in OFFSETS:
        ref = run((K + d) % 2 ** 64)
        with ops.dropout_offset(_off(d)):
            got = run(K)
        _same([t.view(torch.int16) for t in got], [t.view(torch.int16) for t in ref])


def test_embeddings_offset():
    from visualbert_b200 import ops
    model, batch = _model("nlvr", 20, 10)
    emb = model.bert.embeddings
    ids, tt, feats = batch["input_ids"], batch["token_type_ids"], batch["visual_embeddings"]
    dy = torch.randn(ids.shape[0], ids.shape[1] + feats.shape[1], 128, device=DEV)

    def run(seed, off):
        emb.zero_grad(set_to_none=True)
        with ops.forward_seed_offset(off):
            y = emb(ids, tt, visual_embeddings=feats, seed=seed)
        y.float().backward(dy)
        return [y.detach()] + [p.grad.clone() for p in emb.parameters() if p.grad is not None]
    for d in OFFSETS:
        _same(run(K, _off(d)), run((K + d) % 2 ** 64, None))


def test_captured_encoder_reads_the_offset_when_it_runs():
    from visualbert_b200 import ops
    model, _ = _model("nlvr", 8, 8)
    enc = model.bert.encoder
    S, H = 164, 128
    x = torch.randn(2, S, H, device=DEV).bfloat16().requires_grad_(True)
    bias = ops.mask_bias(torch.ones(2, S, dtype=torch.long, device=DEV), None)
    dy = torch.randn(2, S, H, device=DEV)
    off = _off(1)
    torch.use_deterministic_algorithms(True)
    try:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):   # warm-up: sizes the backward scratch and the deterministic workspace
            _encoder_run(enc, x, bias, dy, K, off)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        xs = x.detach().clone().requires_grad_(True)
        with torch.cuda.graph(graph):
            enc.zero_grad(set_to_none=False)
            with ops.forward_seed_offset(off):
                y = enc(xs, bias, output_all_encoded_layers=False, seed=K)[-1]
            y.float().backward(dy)
        grads = [xs.grad] + [p.grad for p in enc.parameters()]   # the tensors the graph writes
        for d in (5, 2 ** 32 - 1, 2 ** 32, 7):
            off.fill_(d)
            graph.replay()
            got = [y.detach().clone()] + [t.clone() for t in grads]
            _same(got, _encoder_run(enc, x, bias, dy, (K + d) % 2 ** 64, None))
    finally:
        torch.use_deterministic_algorithms(False)


def _eager_steps(model, batches, opt_factory, sync):
    losses = []
    opt = opt_factory(model)
    for b in batches:
        sync.zero()
        out = model(**b)
        out["loss"].backward()
        losses.append(out["loss"].detach().clone())
        opt.step()
    return losses


@pytest.mark.parametrize("head,T,V", [("nlvr", 40, 36), ("vqa", 20, 36)])
def test_graphed_steps_equal_eager_steps(head, T, V, monkeypatch):
    from visualbert_b200 import BertAdam, graphs, parallel, synthetic
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    batches = []
    for i in range(6):
        b = synthetic.make_batch(4, T, V, 64, head=head, seed=100 + i, vocab=512, ragged=True)
        batches.append({k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in b.items()})
    opt_factory = lambda m: BertAdam(m.parameters(), lr=1e-3, warmup=0.1, t_total=10, max_grad_norm=1.0)
    torch.use_deterministic_algorithms(True)
    try:
        ref_model, _ = _model(head, T, V, B=4)
        ref_model.bert.set_dropout_state({"seed": 77, "step": 2 ** 32 - 3})
        ref_sync = parallel.FlatGradSync(ref_model)
        ref = _eager_steps(ref_model, batches, opt_factory, ref_sync)
        ref_state = ref_model.bert.dropout_state()

        model, _ = _model(head, T, V, B=4)
        model.bert.set_dropout_state({"seed": 77, "step": 2 ** 32 - 3})
        sync = parallel.FlatGradSync(model)
        step = graphs.GraphedStep(model, sync)
        opt = opt_factory(model)
        losses = []
        for b in batches:
            losses.append(step(b)["loss"].detach().clone())
            opt.step()
        assert len(step.graphs) == 1
        _same(losses, ref)
        _same([p.detach() for p in model.parameters()], [p.detach() for p in ref_model.parameters()])
        assert model.bert.dropout_state() == ref_state
    finally:
        torch.use_deterministic_algorithms(False)


def test_replays_draw_fresh_masks_and_honour_set_dropout_state():
    from visualbert_b200 import graphs, parallel
    model, batch = _model("nlvr", 30, 20)
    sync = parallel.FlatGradSync(model)
    step = graphs.GraphedStep(model, sync)
    model.bert.set_dropout_state({"seed": 5, "step": 10})
    step(batch)                                   # eager warm-up, step 11
    l12 = step(batch)["loss"].item()             # capture + replay, step 12
    l13 = step(batch)["loss"].item()
    assert l12 != l13
    model.bert.set_dropout_state({"seed": 5, "step": 11})
    assert step(batch)["loss"].item() == l12      # replay at state 11 -> step 12 again
    assert model.bert.dropout_state()["step"] == 12

    ref, _ = _model("nlvr", 30, 20)
    ref.bert.set_dropout_state({"seed": 5, "step": 11})
    assert ref(**batch)["loss"].item() == l12
    assert ref(**batch)["loss"].item() == l13


def test_two_shapes_interleaved_and_eviction():
    from visualbert_b200 import graphs, parallel, synthetic
    model, a = _model("nlvr", 24, 16)
    b = {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in synthetic.make_batch(2, 32, 20, 64, head="nlvr", seed=9, vocab=512).items()}
    sync = parallel.FlatGradSync(model)
    step = graphs.GraphedStep(model, sync, max_graphs=1)
    ref, _ = _model("nlvr", 24, 16)
    ref_sync = parallel.FlatGradSync(ref)
    for batch in (a, b, a, b, a, b, a):
        got = step(batch)["loss"].item()
        ref_sync.zero()
        assert got == ref(**batch)["loss"].item()
        assert len(step.graphs) <= 1


def test_captured_eval_forward_sees_weight_changes():
    model, batch = _model("nlvr", 20, 12)
    model.eval()
    model.bert.set_graph_capturable(True)
    with torch.no_grad():
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            model(**batch)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = model(**batch)
        w = model.bert.encoder.layer[0].intermediate.dense.weight
        for scale in (1.0, 0.5):
            w.data.mul_(scale)
            graph.replay()
            assert torch.equal(out["logits"], model(**batch)["logits"])


def test_refused_cases_leave_no_graph():
    from visualbert_b200 import graphs, parallel
    model, batch = _model("nlvr", 20, 12)
    graph = torch.cuda.CUDAGraph()
    step0 = model.bert.dropout_state()["step"]
    with pytest.raises(ValueError, match="set_graph_capturable"):
        with torch.cuda.graph(graph):
            model(**batch)
    # refused before anything was captured or counted: the model is untouched and an eager step still runs
    assert model.bert.dropout_state()["step"] == step0 and model.bert._seed_offset is None and not model.bert._capturable
    model(**batch)["loss"].backward()
    torch.cuda.synchronize()
    pre, pbatch = _model("pretraining", 20, 12)
    sync = parallel.FlatGradSync(pre)
    step = graphs.GraphedStep(pre, sync)
    step(pbatch)                                   # eager: finds the rows with nonzero
    with pytest.raises(ValueError, match="masked_lm_rows"):
        step(pbatch)
    assert len(step.graphs) == 0
    adv, abatch = _model("vqa_advanced", 20, 12)
    step = graphs.GraphedStep(adv, parallel.FlatGradSync(adv), warmup=0)
    with pytest.raises(ValueError, match="vqa_advanced"):
        step(abatch)
    assert len(step.graphs) == 0


def test_default_path_launches_no_offset_kernel():
    from torch.profiler import ProfilerActivity, profile
    model, batch = _model("nlvr", 20, 12)

    def names(m):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            m(**batch)["loss"].backward()
            torch.cuda.synchronize()
        return [e.name for e in prof.events() if e.device_type.name == "CUDA"]
    default = names(model)
    assert not any("_off_kernel" in n or ", 11>" in n for n in default)
    model.bert.set_graph_capturable(True)
    captured = names(model)
    assert any("_off_kernel" in n for n in captured) and any(", 11>" in n for n in captured)
    model.bert.set_graph_capturable(False)
    assert not any("_off_kernel" in n or ", 11>" in n for n in names(model))


def test_pretraining_with_capacity_padded_rows_matches_eager():
    """Graphed pretraining steps with masked_lm_rows padded to a fixed capacity against eager steps with the plain rows: the loss
    divides by a device-side count instead of the host's row count, so they agree to fp32 reordering."""
    from visualbert_b200 import graphs, parallel, synthetic
    host = synthetic.make_batch(4, 24, 12, 64, head="pretraining", seed=21, vocab=512, ragged=True)
    plain = {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in host.items()}
    plain["masked_lm_rows"] = parallel.BatchPrefetcher.labelled_rows(host).to(DEV)
    capped = dict(plain, masked_lm_rows=parallel.BatchPrefetcher.labelled_rows(host, capacity=60).to(DEV))
    assert int((capped["masked_lm_rows"] == -1).sum()) > 0
    state = {"seed": 3, "step": 40}

    ref, _ = _model("pretraining", 24, 12)
    ref_sync = parallel.FlatGradSync(ref)
    ref.bert.set_dropout_state(state)
    ref_sync.zero()
    out = ref(**plain)
    out["loss"].backward()
    ref_loss = out["loss"].item()
    ref_norms = torch.stack([g.norm() for g in ref_sync.views])

    model, _ = _model("pretraining", 24, 12)
    sync = parallel.FlatGradSync(model)
    step = graphs.GraphedStep(model, sync)
    for _ in range(2):                 # eager warm-up, then capture + replay, each at the same dropout state
        model.bert.set_dropout_state(state)
        loss = step(capped)["loss"].item()
        norms = torch.stack([g.norm() for g in sync.views])
        loss_rel = abs(loss - ref_loss) / abs(ref_loss)
        norm_rel = ((norms - ref_norms).abs() / ref_norms.clamp(min=1e-30)).max().item()
        print(f"capacity-padded pretraining: loss rel {loss_rel:.2e}, gradient-norm rel max {norm_rel:.2e}")
        assert loss_rel <= 1e-6 and norm_rel <= 1e-5, (loss_rel, norm_rel)
    assert len(step.graphs) == 1
