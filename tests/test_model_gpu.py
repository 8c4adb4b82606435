"""End-to-end parity of the CUDA path (visualbert_b200.TrainVisualBERTObjective -> C ABI -> sm_90a kernels) against
(a) the committed reference outputs in tests/golden/ (generated from the unmodified reference, fp32 CPU) and
(b) the oracle (oracle/vb_oracle.py) run in fp32 on the same seeded weights and batches.

Stated bf16 tolerance (activations and GEMM operands are bf16, accumulation / LayerNorm / softmax statistics fp32):
  loss           |rel err| <= 1e-2
  logits/hidden  max-abs err <= 5e-2 * max|reference|
  gradients      per-tensor cosine >= 0.99 and norm ratio within 6 % (tensors whose reference norm is above noise),
                 or — for ill-conditioned tensors, e.g. the multichoice head where per-choice terms cancel — an error
                 no larger than that of the reference arithmetic itself run in bf16 (oracle with bf16 tensors)
The reference's own fp32 target (1e-3 relative) applies to an fp32 compute path; this build computes in bf16 as
BASELINE.json's north_star specifies ("stated tolerance for bf16")."""
import numpy as np
import pytest
import torch

import golden_util
import vb_oracle

pytestmark = pytest.mark.gpu

CASES = ["cfg1_pretraining", "small_ragged_pretraining", "small_vqa", "small_nlvr", "small_multichoice",
         "base3_ragged_pretraining", "small_vcr_alignment", "small_bypass_nlvr"]
LOSS_RTOL, ACT_TOL, GRAD_COS, GRAD_NORM = 1e-2, 5e-2, 0.99, 0.06


def _build(name, train=False):
    from visualbert_b200 import BertConfig, TrainVisualBERTObjective
    cfg, sd, batch, c, gold = golden_util.load(name)
    dev = torch.device("cuda:0")
    model = TrainVisualBERTObjective(BertConfig.from_dict(cfg), c["head"], visual_embedding_dim=c["Dv"], **c.get("flags", {}))
    res = model.load_state_dict(sd, strict=False)
    assert set(res.missing_keys) <= {"cls.predictions.decoder.weight"} and not res.unexpected_keys
    model.to(dev)
    model.train(train)
    batch = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in batch.items()}
    sd_dev = {k: v.to(dev) for k, v in sd.items()}
    return model, cfg, sd_dev, batch, c, gold


def _relmax(a, b):
    a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-12)


def test_state_dict_keys_match_reference_layout():
    from visualbert_b200 import synthetic
    model, cfg, sd, batch, c, gold = _build("cfg1_pretraining")
    mine = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    want = synthetic.param_shapes(cfg, c["head"], c["Dv"])
    want["cls.predictions.decoder.weight"] = want["bert.embeddings.word_embeddings.weight"]
    assert mine == {k: tuple(v) for k, v in want.items()}
    assert model.cls.predictions.decoder.weight is model.bert.embeddings.word_embeddings.weight  # tied (M.py:414)


@pytest.mark.parametrize("name", CASES)
def test_forward_backward_parity(name):
    model, cfg, sd, batch, c, gold = _build(name)
    from visualbert_b200 import _lib
    n0 = _lib.launch_count()
    out = model(**batch)
    assert _lib.launch_count() > n0, "the CUDA library did not launch anything"
    loss = out["loss"]
    # (a) reference goldens
    assert abs(loss.item() - float(gold["loss"])) <= LOSS_RTOL * abs(float(gold["loss"]))
    # (b) oracle on the same device, fp32 — and the same arithmetic in torch bf16 as the noise floor
    sdo = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    kw = {k: v for k, v in batch.items() if k != "position_embeddings_visual"}
    flags = c.get("flags", {})
    ref = vb_oracle.objective(sdo, cfg, c["head"], **kw, **flags)
    sdb = {k: v.bfloat16().clone().requires_grad_(True) for k, v in sd.items()}
    kwb = {k: (v.bfloat16() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in kw.items()}
    refb = vb_oracle.objective(sdb, cfg, c["head"], **kwb, **flags)
    if "nsp" in gold:
        # W.pooled + b can cancel to ~1e-3 (tiny models): accept bf16-level error of the reference arithmetic itself
        nsp = out["seq_relationship_score"].detach().float().cpu().numpy()
        nsp_b = refb["seq_relationship_score"].detach().float().cpu().numpy()
        assert _relmax(nsp, gold["nsp"]) < ACT_TOL or np.abs(nsp - gold["nsp"]).max() <= np.abs(nsp_b - gold["nsp"]).max()
    assert abs(loss.item() - ref["loss"].item()) <= LOSS_RTOL * abs(ref["loss"].item())
    # logits against the golden and the oracle; classifier outputs of the tiny models can cancel to ~1e-2 (w.pooled + b),
    # where bf16 rounding of the encoder output is visible: then require no more error than torch-bf16 arithmetic has
    lg, lg_ref = out["logits"].detach().float().cpu().numpy().reshape(-1), ref["logits"].detach().cpu().numpy().reshape(-1)
    lg_b = refb["logits"].detach().float().cpu().numpy().reshape(-1)
    assert _relmax(golden_util.subsample(out["logits"].float()), gold["logits_sub"]) < ACT_TOL or \
        np.abs(lg - lg_ref).max() <= np.abs(lg_b - lg_ref).max()
    assert _relmax(lg, lg_ref) < ACT_TOL or np.abs(lg - lg_ref).max() <= np.abs(lg_b - lg_ref).max()
    if flags.get("bypass_transformer"):
        # the bypass model refuses output_all_encoded_layers, like the reference (M.py:1300): hook the final layer
        with pytest.raises(AssertionError):
            model(**{**batch, "output_all_encoded_layers": True})
        keep = {}
        hook = model.bert.additional_layer.register_forward_hook(lambda m, i, o: keep.__setitem__("y", o))
        with torch.no_grad():
            model(**batch)
        hook.remove()
        last, pooled = keep["y"].float(), model.bert.pooler(keep["y"])
    else:
        enc = model(**{**batch, "output_all_encoded_layers": True})
        assert len(enc["sequence_output"]) == cfg["num_hidden_layers"]
        last, pooled = enc["sequence_output"][-1].float(), enc["pooled_output"]
    assert _relmax(last.detach().cpu().numpy(), ref["sequence_output"].detach().cpu().numpy()) < ACT_TOL
    assert _relmax(golden_util.subsample(last), gold[f"hidden{cfg['num_hidden_layers'] - 1}_sub"]) < ACT_TOL
    assert _relmax(pooled.float().detach().cpu().numpy(), gold["pooled"]) < ACT_TOL
    # gradients
    loss.backward()
    ref["loss"].backward()
    refb["loss"].float().backward()
    gold_norms = dict(zip(gold["grad_names"].tolist(), gold["grad_norms"].tolist()))
    big = max(gold_norms.values())
    checked = 0
    for k, p in model.named_parameters():
        if k == "cls.predictions.decoder.weight":
            continue
        g_ref = sdo[k].grad
        if g_ref is None:
            assert p.grad is None or p.grad.abs().max().item() == 0, k
            continue
        assert p.grad is not None, f"no gradient for {k}"
        a, b = p.grad.float().reshape(-1), g_ref.float().reshape(-1)
        nb = b.norm().item()
        if nb < 1e-3 * big:  # below bf16 noise floor of this step: only require it to stay small
            assert a.norm().item() < 3e-3 * big, k
            continue
        cos = torch.dot(a, b).item() / max(a.norm().item() * nb, 1e-30)
        err, err_bf16 = (a - b).norm().item(), (sdb[k].grad.float().reshape(-1) - b).norm().item()
        well = cos >= GRAD_COS and abs(a.norm().item() / nb - 1.0) <= GRAD_NORM
        assert well or err <= err_bf16, f"{k}: cosine {cos:.5f}, rel err {err / nb:.3e} vs torch-bf16 {err_bf16 / nb:.3e}"
        assert abs(nb - gold_norms[k]) <= 1e-3 * max(gold_norms[k], 1e-6) + 1e-6, f"oracle grad norm drifted from golden: {k}"
        checked += 1
    assert checked >= 10


def test_lazy_logits_have_reference_shape_and_values():
    model, cfg, sd, batch, c, gold = _build("small_ragged_pretraining")
    out = model(**batch)
    assert "logits" in out and "logits" in list(out.keys())
    logits = out["logits"]  # materialised on access
    B, T = batch["input_ids"].shape
    V = batch["visual_embeddings"].shape[1]
    assert logits.shape == (B, T + V, cfg["vocab_size"])
    assert _relmax(golden_util.subsample(logits.float()), gold["logits_sub"]) < ACT_TOL
    # the loss over labelled rows equals the reference's ignore_index loss over all rows
    full = torch.nn.functional.cross_entropy(
        logits.float().view(-1, cfg["vocab_size"]),
        torch.cat((batch["masked_lm_labels"], torch.full((B, V), -1, device=logits.device, dtype=torch.long)), 1).view(-1),
        ignore_index=-1)
    assert abs(full.item() - out["masked_lm_loss"].item()) < 2e-3 * abs(full.item())


def test_three_d_inputs_are_flattened_like_the_reference():
    model, cfg, sd, batch, c, gold = _build("small_multichoice")
    assert batch["input_ids"].dim() == 3 and batch["visual_embeddings"].dim() == 4
    out = model(**batch)
    assert out["logits"].shape == (batch["input_ids"].shape[0], 4)


def test_train_mode_dropout_is_active_and_seeded():
    model, cfg, sd, batch, c, gold = _build("base3_ragged_pretraining", train=True)
    model.bert._step = 0
    l1 = model(**batch)["loss"].item()
    model.bert._step = 0
    l2 = model(**batch)["loss"].item()
    l3 = model(**batch)["loss"].item()
    assert l1 == l2, "same seed must reproduce the same dropout masks"
    assert l1 != l3, "a new step must draw new masks"
    model.eval()
    le = model(**batch)["loss"].item()
    assert abs(l1 - le) > 1e-4
    # training-mode gradients exist and are finite
    model.train()
    model.zero_grad()
    model(**batch)["loss"].backward()
    for k, p in model.named_parameters():
        if p.grad is not None:
            assert torch.isfinite(p.grad).all(), k


def test_attention_weights_mode_matches_reference():
    """output_attention_weights=True (M.py:1430-1444): the analysis slow path returns one [B, A, S, S] map per layer and
    nothing else; values against the reference golden and the oracle."""
    model, cfg, sd, batch, c, gold = _build("small_attention_weights")
    out = model(**batch)
    assert out["loss"] is None and set(out) == {"attention_weights", "loss"}
    maps = out["attention_weights"]
    assert len(maps) == cfg["num_hidden_layers"] and list(maps[0].shape) == gold["attn_shape"].tolist()
    kw = {k: v for k, v in batch.items() if k != "position_embeddings_visual"}
    ref = vb_oracle.objective(sd, cfg, c["head"], **kw, **c["flags"])["attention_weights"]
    for i, w in enumerate(maps):
        assert not w.requires_grad
        assert torch.allclose(w.sum(-1), torch.ones_like(w.sum(-1)), atol=1e-4)
        assert _relmax(golden_util.subsample(w), gold[f"attn{i}_sub"]) < ACT_TOL
        assert _relmax(w.cpu().numpy(), ref[i].detach().cpu().numpy()) < ACT_TOL


def test_bypass_transformer_state_dict_has_the_additional_layer():
    from visualbert_b200 import synthetic
    model, cfg, sd, batch, c, gold = _build("small_bypass_nlvr")
    mine = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    want = synthetic.param_shapes(cfg, c["head"], c["Dv"], bypass_transformer=True)
    assert mine == {k: tuple(v) for k, v in want.items()}
    assert any(k.startswith("bert.additional_layer.") for k in mine)


def test_alignment_gradient_reaches_the_position_table():
    """VCR alignment branch: the text position embeddings receive gradient through the aligned regions as well."""
    model, cfg, sd, batch, c, gold = _build("small_vcr_alignment")
    model(**batch)["loss"].backward()
    g_with = model.bert.embeddings.position_embeddings.weight.grad.clone()
    model.zero_grad()
    model(**{k: v for k, v in batch.items() if k != "image_text_alignment"})["loss"].backward()
    g_without = model.bert.embeddings.position_embeddings.weight.grad
    assert (g_with - g_without).abs().max().item() > 1e-6


def test_direct_gradient_accumulation_matches_autograd_path():
    """FlatGradSync pre-sets p.grad to views of one flat buffer; the layer/embedding backward then accumulate in place
    (autograd receives None). Results must equal the default path (fresh buffers returned to autograd)."""
    from visualbert_b200.parallel import FlatGradSync
    model, cfg, sd, batch, c, gold = _build("base3_ragged_pretraining")
    model(**batch)["loss"].backward()
    want = {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}
    model.zero_grad(set_to_none=True)
    sync = FlatGradSync(model)
    q = model.bert.encoder.layer[0].attention.self
    assert q.query.weight.grad.data_ptr() + q.query.weight.numel() * 4 == q.key.weight.grad.data_ptr()
    for _ in range(2):  # second pass also checks zero()
        sync.zero()
        model(**batch)["loss"].backward()
        for k, p in model.named_parameters():
            if k in want:
                a, b = p.grad.float(), want[k].float()
                assert (a - b).norm().item() <= 2e-3 * b.norm().item() + 1e-7, k
    assert sync.flat.data_ptr() <= model.bert.encoder.layer[1].output.dense.weight.grad.data_ptr()


def test_large_config_shapes_match_oracle():
    """BASELINE configs[4] geometry (VisualBERT-large: H=1024, 16 heads, I=4096, 100 regions + 256 tokens => S=356, which
    takes the staged attention kernels) at a reduced depth/batch: forward + backward against the fp32 oracle on the GPU."""
    from visualbert_b200 import BertConfig, TrainVisualBERTObjective, synthetic
    dev = torch.device("cuda:0")
    cfg = synthetic.bert_config_dict(2, 1024, 16, 4096, vocab=2048)
    sd = synthetic.init_state_dict(cfg, "pretraining", 2048, seed=3)
    batch = synthetic.make_batch(3, 256, 100, 2048, head="pretraining", seed=7, vocab=2048, ragged=True)
    batch = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in batch.items()}
    model = TrainVisualBERTObjective(BertConfig.from_dict(cfg), "pretraining", visual_embedding_dim=2048)
    model.load_state_dict(sd, strict=False)
    model.to(dev).eval()
    out = model(**batch)
    out["loss"].backward()
    sdo = {k: v.to(dev).requires_grad_(True) for k, v in sd.items()}
    ref = vb_oracle.objective(sdo, cfg, "pretraining", **{k: v for k, v in batch.items() if k != "position_embeddings_visual"})
    ref["loss"].backward()
    assert abs(out["loss"].item() - ref["loss"].item()) <= LOSS_RTOL * abs(ref["loss"].item())
    for k in ("bert.encoder.layer.0.attention.self.key.weight", "bert.encoder.layer.1.intermediate.dense.weight",
              "bert.embeddings.projection.weight", "bert.encoder.layer.0.output.LayerNorm.weight"):
        a, b = dict(model.named_parameters())[k].grad.float().reshape(-1), sdo[k].grad.reshape(-1)
        cos = torch.dot(a, b).item() / (a.norm().item() * b.norm().item())
        assert cos >= GRAD_COS, f"{k}: cosine {cos:.5f}"


def test_batch_prefetcher_matches_direct_copy():
    """parallel.BatchPrefetcher: staged copies on the side stream deliver the same tensors, in order."""
    from visualbert_b200.parallel import BatchPrefetcher
    dev = torch.device("cuda:0")
    pf = BatchPrefetcher(dev)
    hosts = [{"a": torch.randn(257, 33).pin_memory(), "b": torch.arange(i, i + 1000).pin_memory(), "tag": i} for i in range(4)]
    staged = pf.stage(hosts[0])
    for i in range(4):
        batch = pf.take(staged)
        if i + 1 < 4:
            staged = pf.stage(hosts[i + 1])
        assert batch["tag"] == i
        assert torch.equal(batch["a"].cpu(), hosts[i]["a"]) and torch.equal(batch["b"].cpu(), hosts[i]["b"])


def test_masked_lm_rows_extension_gives_identical_results():
    """forward(masked_lm_rows=...) (indices found on the host by BatchPrefetcher) == the default device-side scan."""
    from visualbert_b200.parallel import BatchPrefetcher
    model, cfg, sd, batch, c, gold = _build("small_ragged_pretraining")
    host = {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in batch.items()}
    rows = BatchPrefetcher.labelled_rows(host).to("cuda:0")
    a = model(**batch)
    b = model(**batch, masked_lm_rows=rows)
    assert a["loss"].item() == b["loss"].item() and a["masked_lm_loss"].item() == b["masked_lm_loss"].item()
    staged = BatchPrefetcher("cuda:0").stage({k: (v.pin_memory() if torch.is_tensor(v) else v) for k, v in host.items()})
    c2 = model(**BatchPrefetcher("cuda:0").take(staged))
    assert c2["loss"].item() == a["loss"].item()


def test_data_updating_optimizer_is_seen_by_the_compute_weights():
    """ADVICE r1 (high): the reference BertAdam updates `p.data` in place (optimization.py:293), which does not bump
    Tensor._version. The bf16 compute copies are therefore refreshed on EVERY training-mode forward (one
    vb_cast_multi launch): a step taken through `.data` must change the next forward's loss, and must match what a
    freshly built model with the updated masters computes."""
    model, cfg, sd, batch, c, gold = _build("small_ragged_pretraining", train=True)
    model.bert._step = 100          # fixed dropout seed sequence for both models
    l0 = model(**batch)["loss"]
    l0.backward()
    v0 = {n: p._version for n, p in model.named_parameters()}
    with torch.no_grad():
        for p in model.parameters():
            if p.grad is not None:
                p.data.add_(-0.05 * p.grad.data.sign())   # sign-SGD through .data, like opt.py:293's p.data.add_
    assert all(p._version == v0[n] for n, p in model.named_parameters()), "the update was meant to be invisible to _version"
    model.zero_grad()
    model.bert._step = 100
    l1 = model(**batch)["loss"].item()
    assert abs(l1 - l0.item()) > 1e-3 * abs(l0.item()), "stale compute weights: the loss did not move after the update"
    # the same masters in a fresh model give the same loss
    from visualbert_b200 import BertConfig, TrainVisualBERTObjective
    fresh = TrainVisualBERTObjective(BertConfig.from_dict(cfg), c["head"], visual_embedding_dim=c["Dv"], **c.get("flags", {}))
    fresh.load_state_dict(model.state_dict(), strict=False)
    fresh.to(l0.device).train()
    fresh.bert.set_dropout_state(dict(model.bert.dropout_state(), step=100))
    l2 = fresh(**batch)["loss"].item()
    assert abs(l1 - l2) <= 1e-5 * abs(l2) + 1e-6
    # eval mode keeps the cache until a version changes
    model.eval()
    e0 = model(**batch)["loss"].item()
    g0 = model.bert._bank.generation
    e1 = model(**batch)["loss"].item()
    assert model.bert._bank.generation == g0 and e0 == e1
    with torch.no_grad():
        model.bert.encoder.layer[0].output.dense.weight.mul_(1.5)   # autograd-visible in-place op: version bump
    e2 = model(**batch)["loss"].item()
    assert model.bert._bank.generation == g0 + 1 and e2 != e1


def test_full_depth_base_model_parity_at_benchmark_shape():
    """VERDICT r1 item 6a: the goldens stop at 3 layers — the 12-layer, H=768, S=164 stack of the headline number is
    compared here with the fp32 oracle on the device (B=16, ragged masks): loss, last hidden state, pooled output and
    gradients of tensors at the bottom, middle and top of the stack (bf16 compute, 12 layers); the bounds are about twice
    the errors of the bf16 arithmetic."""
    from visualbert_b200 import BertConfig, TrainVisualBERTObjective, synthetic
    dev = torch.device("cuda:0")
    cfg = synthetic.bert_config_dict(12, 768, 12, 3072, vocab=8192)
    sd = synthetic.init_state_dict(cfg, "pretraining", 2048, seed=3)
    batch = synthetic.make_batch(16, 128, 36, 2048, head="pretraining", seed=77, ragged=True, vocab=8192)
    batch = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in batch.items()}
    model = TrainVisualBERTObjective(BertConfig.from_dict(cfg), "pretraining", visual_embedding_dim=2048)
    model.load_state_dict(sd, strict=False)
    model.to(dev).eval()
    out = model(**batch)
    out["loss"].backward()
    enc = model(**{**batch, "output_all_encoded_layers": True})
    sdo = {k: v.to(dev).requires_grad_(True) for k, v in sd.items()}
    kw = {k: v for k, v in batch.items() if k != "position_embeddings_visual"}
    ref = vb_oracle.objective(sdo, cfg, "pretraining", **kw)
    ref["loss"].backward()
    rel_loss = abs(out["loss"].item() - ref["loss"].item()) / abs(ref["loss"].item())
    assert rel_loss < 3e-4, f"loss {out['loss'].item()} vs oracle {ref['loss'].item()} (rel {rel_loss:.2e})"
    last = enc["sequence_output"][-1].float()
    hid = ((last - ref["sequence_output"]).abs().max() / ref["sequence_output"].abs().max()).item()
    assert hid < 4e-2, f"last hidden state: {hid:.3e} of max"
    pooled = ((enc["pooled_output"].float() - ref["pooled_output"]).abs().max() / ref["pooled_output"].abs().max()).item()
    assert pooled < 4e-2, f"pooled output: {pooled:.3e}"
    names = ["bert.encoder.layer.0.attention.self.query.weight", "bert.encoder.layer.0.output.dense.weight",
             "bert.encoder.layer.5.intermediate.dense.weight", "bert.encoder.layer.6.attention.output.dense.weight",
             "bert.encoder.layer.11.attention.self.value.weight", "bert.encoder.layer.11.output.LayerNorm.weight",
             "bert.embeddings.projection.weight", "bert.embeddings.word_embeddings.weight"]
    params = dict(model.named_parameters())
    worst = 0.0
    for k in names:
        a, b = params[k].grad.float().reshape(-1), sdo[k].grad.reshape(-1)
        r = ((a - b).norm() / b.norm()).item()
        cos = (torch.dot(a, b) / (a.norm() * b.norm())).item()
        worst = max(worst, r)
        assert r < 4e-2 and cos > 0.999, f"{k}: relative error {r:.3e}, cosine {cos:.5f}"
    print(f"12-layer parity: loss rel {rel_loss:.2e}, hidden {hid:.2e}, pooled {pooled:.2e}, worst grad rel err {worst:.2e}")
