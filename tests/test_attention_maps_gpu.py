"""Attention maps (output_attention_weights=True, M.py:1316-1324, 1430-1444) from the attention-probability kernel.

  * vb_attention_probs against softmax(QK^T / 8 + bias) in fp64 from the same bf16 qkv, at tile edges and every route's
    lengths, with ragged masks and an example whose keys are all masked; every element written, nothing outside the tensors
    read or written, two calls bit-identical;
  * the maps are the probabilities the attention kernels used: maps . V equals the ctx of vb_attention_fwd on all three routes;
  * the model serves the maps from the whole-encoder call, close to the fp32 oracle, pre-dropout in train mode, the same on
    the per-layer path, and without the fp32 score temporaries of a torch recompute."""
import ctypes

import pytest
import torch

import golden_util  # noqa: F401  (puts oracle/ on the path)
import vb_oracle

pytestmark = pytest.mark.gpu

PROB_TOL = 1e-5    # max abs error of a probability and of a row sum against fp64
SENTINEL = -12345.0
GUARD_ROWS = 64
GUARD_FLAT = 1024

SEQS = [1, 2, 17, 63, 64, 65, 127, 128, 129, 191, 192, 193, 255, 256, 257, 356, 512]
CASES = [(B, S, A) for S in SEQS for B in (1, 3) for A in (1, 2, 12)]


def _setup():
    from visualbert_b200 import _lib
    return _lib, _lib.lib(), torch.device("cuda:0"), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr())


def _guarded(n, dtype, guard, fill, dev):
    buf = torch.full((n + 2 * guard,), fill, dtype=dtype, device=dev)
    return buf, buf[guard:guard + n]


def _guards_intact(buf, guard, fill):
    g = torch.cat([buf[:guard], buf[-guard:]])
    if fill != fill:
        return bool(torch.isnan(g).all())
    return torch.equal(g, torch.full_like(g, fill))


def _inputs(B, S, A, dev, seed):
    """qkv unit normal (bf16); ragged key lengths; with B = 3 example 1 has no valid key (every bias -10000)."""
    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    qkv = torch.randn(B * S, 3 * A * 64, device=dev, generator=g).bfloat16()
    lens = torch.randint(max(1, S // 2), S + 1, (B,), device=dev, generator=g)
    bias = (torch.arange(S, device=dev)[None, :] >= lens[:, None]).float() * -10000.0
    if B == 3:
        bias[1] = -10000.0
    return qkv, bias.contiguous()


def _scores(qkv, B, S, A):
    q, k, _ = qkv.double().view(B, S, 3, A, 64).permute(2, 0, 3, 1, 4)
    return q @ k.transpose(-1, -2) / 8.0


def _probs(L, _lib, st, qkv, bias, B, S, A, dev):
    """vb_attention_probs with qkv and bias inside NaN guard bands and the NaN-filled output inside sentinel guards."""
    H = A * 64
    nan = float("nan")
    qbuf, q = _guarded(B * S * 3 * H, torch.bfloat16, GUARD_ROWS * 3 * H, nan, dev)
    bbuf, b = _guarded(B * S, torch.float32, GUARD_FLAT, nan, dev)
    pbuf, p = _guarded(B * A * S * S, torch.float32, GUARD_FLAT, SENTINEL, dev)
    q.copy_(qkv.reshape(-1))
    b.copy_(bias.reshape(-1))
    p.fill_(nan)
    _lib.check(L.vb_attention_probs(q.data_ptr(), b.data_ptr(), p.data_ptr(), B, S, A, H, st), "vb_attention_probs")
    torch.cuda.synchronize()
    assert _guards_intact(qbuf, GUARD_ROWS * 3 * H, nan) and _guards_intact(bbuf, GUARD_FLAT, nan)
    assert _guards_intact(pbuf, GUARD_FLAT, SENTINEL), "a store outside [B, A, S, S]"
    return p.view(B, A, S, S)


@pytest.mark.parametrize("B,S,A", CASES)
def test_attention_probs_match_fp64(B, S, A):
    _lib, L, dev, st = _setup()
    where = f"B={B} S={S} A={A}"
    qkv, bias = _inputs(B, S, A, dev, seed=1000 * S + 10 * B + A)
    p = _probs(L, _lib, st, qkv, bias, B, S, A, dev)
    assert torch.isfinite(p).all(), f"{where}: unwritten (NaN) elements"
    p2 = _probs(L, _lib, st, qkv, bias, B, S, A, dev)
    assert torch.equal(p, p2), f"{where}: two identical calls differ"
    sc = _scores(qkv, B, S, A)
    ref = torch.softmax(sc + bias.double()[:, None, None, :], -1)
    err = (p.double() - ref).abs().max().item()
    assert err <= PROB_TOL, f"{where}: max abs error {err:.3g}"
    rows = (p.double().sum(-1) - 1).abs().max().item()
    assert rows <= PROB_TOL, f"{where}: a row sums to 1 +- {rows:.3g}"
    masked = (bias < 0)[:, None, None, :].expand_as(p)
    if B == 3:
        # example 1: every key masked -> the reference's uniform shift leaves softmax(QK^T / 8) over all keys
        full = torch.softmax(sc[1], -1)
        e1 = (p[1].double() - full).abs().max().item()
        assert e1 <= PROB_TOL, f"{where}: fully masked example off by {e1:.3g}"
        masked = masked.clone()
        masked[1] = False
    assert (p[masked] == 0).all(), f"{where}: masked keys must get exact zeros"


@pytest.mark.parametrize("S", [100, 200, 356])
def test_maps_are_the_probabilities_the_forward_used(S):
    """maps . V (fp64) against the ctx of vb_attention_fwd (dropout 0) on the wgmma, whole-head and staged routes: equal to the
    bf16 rounding of ctx."""
    _lib, L, dev, st = _setup()
    B, A = 2, 2
    H = A * 64
    qkv, bias = _inputs(B, S, A, dev, seed=S)
    ctx = torch.empty(B * S, H, device=dev, dtype=torch.bfloat16)
    lse = torch.empty(B, A, S, device=dev)
    _lib.check(L.vb_attention_fwd(_ptr(qkv), _ptr(bias), _ptr(ctx), _ptr(lse), None, B, S, A, H, ctypes.c_float(0.0),
                                  ctypes.c_uint64(1), 0, st), "vb_attention_fwd")
    p = _probs(L, _lib, st, qkv, bias, B, S, A, dev)
    v = qkv.double().view(B, S, 3, A, 64)[:, :, 2].permute(0, 2, 1, 3)
    o = (p.double() @ v).permute(0, 2, 1, 3).reshape(B * S, H)
    err = (ctx.double() - o).abs().max().item()
    assert err <= 2.0 ** -8 * o.abs().max().item(), f"S={S}: ctx differs from maps . V by {err:.3g}"
    # and the forward's own log-sum-exp reproduces the maps' normalisation
    sc = _scores(qkv, B, S, A) + bias.double()[:, None, None, :]
    lse_maps = torch.logsumexp(sc, -1)
    assert (lse.double() - lse_maps).abs().max().item() < 1e-3


# ---------------------------------------------------------------------------------------------------------------------
# the model
# ---------------------------------------------------------------------------------------------------------------------
def _model(layers, hidden, heads, inter, B, T, V, Dv=2048, seed=0, **cfg_over):
    from visualbert_b200 import BertConfig, TrainVisualBERTObjective, synthetic
    dev = torch.device("cuda:0")
    cfg = synthetic.bert_config_dict(layers, hidden, heads, inter, vocab=4096)
    cfg.update(cfg_over)
    sd = synthetic.init_state_dict(cfg, "pretraining", Dv, seed=seed)
    model = TrainVisualBERTObjective(BertConfig.from_dict(cfg), "pretraining", visual_embedding_dim=Dv,
                                     output_attention_weights=True)
    model.load_state_dict(sd, strict=False)
    model.to(dev).eval()
    batch = synthetic.make_batch(B, T, V, Dv, head="pretraining", seed=seed + 1, vocab=4096, ragged=True)
    batch = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in batch.items()}
    return model, cfg, {k: v.to(dev) for k, v in sd.items()}, batch


def _forbid_layer_calls(monkeypatch):
    from visualbert_b200 import ops

    def _no(*a, **k):
        raise AssertionError("analysis forward took the per-layer path")
    monkeypatch.setattr(ops, "bert_layer", _no)


def test_whole_encoder_maps_match_the_oracle(monkeypatch):
    """12 layers, H = 768, S = 164, ragged: one whole-encoder call serves the maps (ops.bert_layer is never called); each
    map is within 5e-2 of max of the fp32 oracle, or no further from it than an fp32 torch recompute from the same layer
    inputs (the method this kernel replaced: fp32 Q / K projections from the masters, fp32 scores, softmax)."""
    model, cfg, sd, batch = _model(12, 768, 12, 3072, B=8, T=128, V=36)
    _forbid_layer_calls(monkeypatch)
    with torch.no_grad():
        out = model(**batch)
    maps = out["attention_weights"]
    assert out["loss"] is None and set(out) == {"attention_weights", "loss"}
    B, S, A = batch["input_ids"].shape[0], 164, 12
    assert len(maps) == 12 and all(m.shape == (B, A, S, S) and m.dtype == torch.float32 and not m.requires_grad for m in maps)
    # layer inputs of the same CUDA forward for the restated fp32 recompute
    keep = {}
    hook = model.bert.embeddings.register_forward_hook(lambda m, i, o: keep.__setitem__("x", o))
    mask = torch.cat((batch["input_mask"], batch["image_mask"]), 1)
    with torch.no_grad():
        layers, _, maps2 = model.bert(batch["input_ids"], batch["token_type_ids"], mask, batch["visual_embeddings"], None,
                                      batch["visual_embeddings_type"], None, None, output_all_encoded_layers=True)
    hook.remove()
    for a, b in zip(maps, maps2):
        assert torch.equal(a, b)
    inputs = [keep["x"]] + list(layers[:-1])
    bias = (1.0 - mask.float()) * -10000.0
    kw = {k: v for k, v in batch.items() if k != "position_embeddings_visual"}
    with torch.no_grad():
        ref = vb_oracle.objective(sd, cfg, "pretraining", **kw, output_attention_weights=True)["attention_weights"]
    for i, (m, r) in enumerate(zip(maps, ref)):
        r = r.float()
        layer = model.bert.encoder.layer[i].attention.self
        x = inputs[i].float()

        def heads(lin):
            return torch.nn.functional.linear(x, lin.weight, lin.bias).view(B, S, A, 64).permute(0, 2, 1, 3)
        with torch.no_grad():
            old = torch.softmax(heads(layer.query) @ heads(layer.key).transpose(-1, -2) / 8.0 + bias[:, None, None, :], -1)
        err, err_old = (m - r).abs().max().item(), (old - r).abs().max().item()
        assert err <= 5e-2 * r.abs().max().item() or err <= err_old, f"layer {i}: {err:.3g} (fp32 recompute {err_old:.3g})"
        assert torch.allclose(m.sum(-1), torch.ones_like(m.sum(-1)), atol=1e-5)


def test_bypass_model_with_attention_weights_runs():
    from visualbert_b200 import BertConfig, TrainVisualBERTObjective, synthetic
    dev = torch.device("cuda:0")
    cfg = synthetic.bert_config_dict(2, 128, 2, 512, vocab=64)
    model = TrainVisualBERTObjective(BertConfig.from_dict(cfg), "nlvr", visual_embedding_dim=64, bypass_transformer=True,
                                     output_attention_weights=True).to(dev).eval()
    b = synthetic.make_batch(2, 6, 3, 64, head="nlvr", vocab=64, ragged=True)
    b = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in b.items()}
    mask = torch.cat((b["input_mask"], b["image_mask"]), 1)
    with torch.no_grad():
        final, pooled = model.bert(b["input_ids"], b["token_type_ids"], mask, b["visual_embeddings"], None,
                                   b["visual_embeddings_type"], None, None, output_all_encoded_layers=False)
    assert final.shape == (2, 9, 128) and torch.isfinite(final.float()).all() and torch.isfinite(pooled).all()


def test_train_mode_maps_are_pre_dropout():
    """Hidden dropout 0, attention dropout 0.1: the first layer's maps in train mode equal eval's bit for bit (the maps are
    taken before dropout); the second layer's differ, since attention dropout changed the first layer's output."""
    model, cfg, sd, batch = _model(2, 256, 4, 1024, B=4, T=40, V=20, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.1)
    with torch.no_grad():
        ev = model(**batch)["attention_weights"]
    model.train()
    tr = model(**batch)["attention_weights"]
    assert torch.equal(tr[0], ev[0])
    assert not torch.equal(tr[1], ev[1])
    assert all(not m.requires_grad for m in tr)


def test_per_layer_path_maps_equal_whole_encoder_maps(monkeypatch):
    """output_all_encoded_layers=True in train mode under grad runs the layers one by one (gradients through intermediate
    layers); its maps, from each layer's own qkv, equal those of the whole-encoder call with the same dropout seed."""
    model, cfg, sd, batch = _model(3, 256, 4, 1024, B=4, T=40, V=20)
    model.train()
    model.bert._step = 0
    fused = model(**batch)["attention_weights"]
    model.bert._step = 0
    per_layer = model(**batch, output_all_encoded_layers=True)["attention_weights"]
    assert len(per_layer) == 3
    for a, b in zip(fused, per_layer):
        assert not b.requires_grad
        assert torch.equal(a, b)


def test_analysis_forward_memory():
    """B = 64, S = 356, 2 layers, H = 1024: the analysis forward's peak allocation stays within arena + maps + 256 MB for the
    embedding activations; the fp32 recompute's score and softmax temporaries (2 x 519 MB per layer) are gone."""
    from visualbert_b200 import _lib
    model, cfg, sd, batch = _model(2, 1024, 16, 4096, B=64, T=256, V=100)
    B, S, H, A, I, L = 64, 356, 1024, 16, 4096, 2
    off = (ctypes.c_int64 * _lib.VB_ENCODER_ARENA_BUFFERS)()
    arena = L * int(_lib.lib().vb_encoder_arena_layout(B, S, H, A, I, 0, off))
    maps = 4 * L * B * A * S * S
    with torch.no_grad():
        model(**batch)   # weight bank and first-call set-up outside the measurement
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out = model(**batch)
        torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    assert out["attention_weights"][0].shape == (B, A, S, S)
    margin = 256 << 20
    assert peak <= arena + maps + margin, f"peak {peak / 2**20:.0f} MB > arena {arena / 2**20:.0f} + maps {maps / 2**20:.0f} + 256 MB"
