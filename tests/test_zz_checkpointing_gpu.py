"""Activation checkpointing on the GPU: vb_encoder_fwd_ckpt / vb_encoder_bwd_ckpt (and the _varlen forms) against
vb_encoder_fwd / vb_encoder_bwd on the same descriptors and inputs, bit for bit on every attention route with and without
dropout; the model with set_activation_checkpointing against the model without it (loss, encoder output, every gradient, the
attention maps, frozen patterns, unpadded batches, GraphedStep with BertAdam); and the memory the mode exists for.

The file sorts after the tests that read kernel launches back from torch.profiler (test_deterministic_gpu.py,
test_gemm_reference_gpu.py, test_rowop_reference_gpu.py, ...). Those tests count kernel records, and the profiler now and
then loses one. Run ahead of them in one pytest process, these 37 tests (model steps and graph captures among them) made
that far more frequent, so they run last and leave the earlier tests' process as it was."""
import ctypes
import itertools

import pytest
import torch

import golden_util

pytestmark = pytest.mark.gpu

BF, F32 = torch.bfloat16, torch.float32
DEV = "cuda:0"
GUARD = 4096   # guard bytes on each side of a raw buffer (keeps the 256-byte alignment of the allocation)


@pytest.fixture(autouse=True)
def _cublas(monkeypatch):
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    yield
    torch.use_deterministic_algorithms(False)


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


class GuardedBytes:
    """n bytes between two GUARD-byte bands of 0xFF (a NaN pattern in bf16 and fp32); the inside starts as `fill`."""

    def __init__(self, n, fill=0xFF):
        self.n = n
        self.buf = torch.full((n + 2 * GUARD,), 0xFF, dtype=torch.uint8, device=DEV)
        self.t = self.buf[GUARD:GUARD + n]
        self.t.fill_(fill)

    def ptr(self):
        return self.t.data_ptr()

    def check_bands(self, what):
        assert bool((self.buf[:GUARD] == 0xFF).all()) and bool((self.buf[GUARD + self.n:] == 0xFF).all()), f"{what}: guard band overwritten"


def _layers(L, B, S, A, p_h, p_a, mask_bias):
    """L random layers of hidden 64 A, intermediate 256 A: (descriptor array, the tensors it points to)."""
    from visualbert_b200 import _lib
    H, I = 64 * A, 256 * A
    rnd = lambda *s, sc=1.0: sc * torch.randn(*s, device=DEV)
    descs, keep = (_lib.LayerDesc * L)(), []
    for l in range(L):
        W = [rnd(3 * H, H, sc=0.05).to(BF), rnd(H, H, sc=0.05).to(BF), rnd(I, H, sc=0.05).to(BF), rnd(H, I, sc=0.05).to(BF)]
        v = [rnd(3 * H, sc=0.1), rnd(H, sc=0.1), 1 + rnd(H, sc=0.1), rnd(H, sc=0.1), rnd(I, sc=0.1), rnd(H, sc=0.1), 1 + rnd(H, sc=0.1),
             rnd(H, sc=0.1)]
        keep += W + v
        descs[l] = _lib.LayerDesc(batch=B, seq=S, hidden=H, heads=A, inter=I, hidden_dropout=p_h, attn_dropout=p_a,
                                  seed=0x0FEDCBA987654321, layer_index=l, w_qkv=W[0].data_ptr(), w_attn_out=W[1].data_ptr(),
                                  w_inter=W[2].data_ptr(), w_out=W[3].data_ptr(), b_qkv=v[0].data_ptr(), b_attn_out=v[1].data_ptr(),
                                  ln1_gamma=v[2].data_ptr(), ln1_beta=v[3].data_ptr(), b_inter=v[4].data_ptr(), b_out=v[5].data_ptr(),
                                  ln2_gamma=v[6].data_ptr(), ln2_beta=v[7].data_ptr(),
                                  mask_bias=0 if mask_bias is None else mask_bias.data_ptr())
    return descs, keep


GRAD_SIZES = lambda H, I: dict(dw_qkv=3 * H * H, db_qkv=3 * H, dw_attn_out=H * H, db_attn_out=H, dln1_gamma=H, dln1_beta=H,
                               dw_inter=I * H, db_inter=I, dw_out=H * I, db_out=H, dln2_gamma=H, dln2_beta=H)
# frozen fields per layer of the frozen case: a NULL LayerNorm group, a NULL weight and a NULL bias, and a layer with nothing
FROZEN = [set(GRAD_SIZES(1, 1)), {"dw_qkv", "db_attn_out", "dln1_gamma", "dln1_beta"}, {"db_inter", "dw_out"}, set()]


class Grads:
    """A vb_layer_grads array over guarded fp32 buffers (zero inside); fields in `frozen[l]` are NULL."""

    def __init__(self, L, H, I, frozen=None):
        from visualbert_b200 import _lib
        self.arr, self.bufs = (_lib.LayerGrads * L)(), {}
        for l in range(L):
            for name, n in GRAD_SIZES(H, I).items():
                if frozen is not None and name in frozen[l % len(frozen)]:
                    continue
                b = GuardedBytes(4 * n, fill=0)
                self.bufs[l, name] = b
                setattr(self.arr[l], name, b.ptr())

    def values(self):
        return {k: b.t.view(F32) for k, b in self.bufs.items()}

    def check_bands(self, what):
        for k, b in self.bufs.items():
            b.check_bands(f"{what} grad {k}")


def _scratch(M, H, I, A):
    from visualbert_b200 import _lib
    t = dict(d_pre=torch.empty(M, H, device=DEV, dtype=BF), d_pre_drop=torch.empty(M, H, device=DEV, dtype=BF),
             d_big=torch.empty(M, max(I, 3 * H), device=DEV, dtype=BF), d_x1=torch.empty(M, H, device=DEV, dtype=BF),
             d_ctx=torch.empty(M, H, device=DEV, dtype=BF), drow=torch.empty(A * M, device=DEV, dtype=F32))
    return _lib.LayerScratch(**{k: v.data_ptr() for k, v in t.items()}), t


def _compare(B, S, A, L, p, lens=None, with_dx=True, frozen=None, det=True):
    """Arena calls and checkpointed calls on the same descriptors, inputs and fresh gradient buffers."""
    from visualbert_b200 import _lib
    lib = _lib.lib()
    torch.manual_seed(B * 1000 + S + L)
    H, I = 64 * A, 256 * A
    vl = lens is not None
    M = sum(lens) if vl else B * S
    drop = 1 if p > 0 else 0
    if vl:
        cu = torch.tensor([0] + list(itertools.accumulate(lens)), dtype=torch.int32, device=DEV)
        mbias = None
    else:
        valid = torch.arange(S, device=DEV)[None, :] < torch.randint(S // 2, S + 1, (B, 1), device=DEV)
        mbias = ((~valid).float() * -10000.0).contiguous()
    descs, keep = _layers(L, B, S, A, p, p, mbias)
    x = torch.randn(M, H, device=DEV).to(BF)
    dy = torch.randn(M, H, device=DEV).to(BF)
    off = (ctypes.c_int64 * _lib.VB_ENCODER_ARENA_BUFFERS)()
    coff = (ctypes.c_int64 * 3)()
    stride = int(lib.vb_encoder_arena_layout_varlen(B, S, M, H, A, I, drop, off) if vl else lib.vb_encoder_arena_layout(B, S, H, A, I, drop, off))
    cs = int(lib.vb_encoder_ckpt_layout(B, S, H, A, I, M if vl else -1, coff))
    sc, sc_keep = _scratch(M, H, I, A)
    det_ws = None
    if det:
        det_ws = torch.empty(max(int(lib.vb_deterministic_workspace_bytes(M, H, I, 0, 0)), 256), device=DEV, dtype=torch.uint8)
        _lib.check(lib.vb_set_deterministic(det_ws.data_ptr(), det_ws.numel()), "vb_set_deterministic")
    try:
        def launches(fn):
            n = _lib.launch_count()
            fn()
            return _lib.launch_count() - n

        # the arena calls
        arena = GuardedBytes(L * stride, fill=0xA5)
        g_ref = Grads(L, H, I, frozen)
        dx_ref = GuardedBytes(M * H * 2) if with_dx else None
        if vl:
            f_ref = launches(lambda: _lib.check(lib.vb_encoder_fwd_varlen(descs, L, cu.data_ptr(), M, x.data_ptr(), arena.ptr(), _st()), "fwd"))
            b_ref = launches(lambda: _lib.check(lib.vb_encoder_bwd_varlen(descs, L, cu.data_ptr(), M, x.data_ptr(), arena.ptr(), dy.data_ptr(),
                                                                          dx_ref.ptr() if with_dx else None, g_ref.arr, ctypes.byref(sc),
                                                                          _st()), "bwd"))
        else:
            f_ref = launches(lambda: _lib.check(lib.vb_encoder_fwd(descs, L, ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(arena.ptr()),
                                                                   _st()), "fwd"))
            b_ref = launches(lambda: _lib.check(lib.vb_encoder_bwd(descs, L, ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(arena.ptr()),
                                                                   ctypes.c_void_p(dy.data_ptr()),
                                                                   ctypes.c_void_p(dx_ref.ptr() if with_dx else None), g_ref.arr,
                                                                   ctypes.byref(sc), _st()), "bwd"))
        # the checkpointed calls
        ckpt = GuardedBytes((L - 1) * cs) if L > 1 else None
        slot = GuardedBytes(stride, fill=0xA5)
        g = Grads(L, H, I, frozen)
        dx = GuardedBytes(M * H * 2) if with_dx else None
        ck = ckpt.ptr() if ckpt is not None else None
        if vl:
            f = launches(lambda: _lib.check(lib.vb_encoder_fwd_ckpt_varlen(descs, L, cu.data_ptr(), M, x.data_ptr(), ck, slot.ptr(), _st()),
                                            "fwd_ckpt"))
        else:
            f = launches(lambda: _lib.check(lib.vb_encoder_fwd_ckpt(descs, L, x.data_ptr(), ck, slot.ptr(), None, _st()), "fwd_ckpt"))
        torch.cuda.synchronize()
        what = f"B={B} S={S} A={A} L={L} p={p} lens={lens} dx={with_dx} frozen={frozen is not None} det={det}"
        n = M * H * 2
        y_ref = [arena.t[l * stride + off[13]: l * stride + off[13] + n] for l in range(L)]
        for l in range(L - 1):   # every layer output, and the kept LN2 statistics
            base = l * cs
            assert torch.equal(ckpt.t[base + coff[0]: base + coff[0] + n], y_ref[l]), f"{what}: output of layer {l}"
            for i, k in ((1, 10), (2, 11)):
                assert torch.equal(ckpt.t[base + coff[i]: base + coff[i] + 4 * M], arena.t[l * stride + off[k]: l * stride + off[k] + 4 * M]), \
                    f"{what}: LN2 statistics of layer {l}"
        assert torch.equal(slot.t[off[13]: off[13] + n], y_ref[L - 1]), f"{what}: output of the top layer"
        # the top layer's slot is the arena's top slot (everything the backward reads)
        top = (L - 1) * stride
        for k in (0, 1, 3, 6, 8, 9, 12):
            size = off[k + 1] - off[k]
            assert torch.equal(slot.t[off[k]: off[k] + size], arena.t[top + off[k]: top + off[k] + size]), f"{what}: top slot buffer {k}"
        assert f == f_ref, f"{what}: forward launches {f} vs {f_ref}"

        if vl:
            b = launches(lambda: _lib.check(lib.vb_encoder_bwd_ckpt_varlen(descs, L, cu.data_ptr(), M, x.data_ptr(), ck, slot.ptr(),
                                                                           dy.data_ptr(), dx.ptr() if with_dx else None, g.arr,
                                                                           ctypes.byref(sc), _st()), "bwd_ckpt"))
        else:
            b = launches(lambda: _lib.check(lib.vb_encoder_bwd_ckpt(descs, L, x.data_ptr(), ck, slot.ptr(), dy.data_ptr(),
                                                                    dx.ptr() if with_dx else None, g.arr, ctypes.byref(sc), _st()),
                                            "bwd_ckpt"))
        torch.cuda.synchronize()
        # the recompute: each lower layer's forward launches minus its LN2 forward (the keep-mask kernel included)
        assert b - b_ref == (L - 1) * (f_ref // L - 1), f"{what}: backward launches {b} vs {b_ref}, forward {f_ref}"
        if L > 1:   # the slot now holds the recomputed layer 0: its LN2 input and keep bits are the arena's
            for k in (9, 12):
                size = off[k + 1] - off[k]
                assert torch.equal(slot.t[off[k]: off[k] + size], arena.t[off[k]: off[k] + size]), f"{what}: recomputed buffer {k}"
        if with_dx:
            if det:
                assert torch.equal(dx.t, dx_ref.t), f"{what}: dx"
            else:
                d, r = dx.t.view(BF).float(), dx_ref.t.view(BF).float()
                assert (d - r).norm().item() <= 1e-2 * r.norm().item(), f"{what}: dx"
        got, want = g.values(), g_ref.values()
        assert got.keys() == want.keys()
        for k in want:
            if det:
                assert torch.equal(got[k], want[k]), f"{what}: gradient {k}"
            else:   # fp32 red.add accumulation: the order of the partial sums is not fixed
                assert (got[k] - want[k]).norm().item() <= 1e-4 * want[k].norm().item() + 1e-6, f"{what}: gradient {k}"
        for buf, name in ((ckpt, "ckpt"), (slot, "slot"), (dx, "dx")):
            if buf is not None:
                buf.check_bands(f"{what} {name}")
        g.check_bands(what)
        if ckpt is not None:   # the backward leaves the checkpoints as the forward wrote them
            for l in range(L - 1):
                assert torch.equal(ckpt.t[l * cs + coff[0]: l * cs + coff[0] + n], y_ref[l]), f"{what}: checkpoint {l} after backward"
    finally:
        if det:
            lib.vb_set_deterministic(None, 0)
    del keep, sc_keep


@pytest.mark.parametrize("S", [164, 200, 300])          # wgmma, whole-head and staged attention
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_ckpt_calls_equal_the_arena_calls_dense(S, p):
    _compare(3, S, 2, 4, p)                              # M = 3 S is no multiple of 128


@pytest.mark.parametrize("L", [1, 2])
def test_ckpt_calls_with_one_and_two_layers(L):
    _compare(3, 164, 2, L, 0.1)


def test_ckpt_calls_with_tile_native_gelu_prime():
    """M and I multiples of 256: the training forward keeps gelu'(u) tile-native; the recompute writes it the same way."""
    _compare(4, 64, 4, 4, 0.1)


@pytest.mark.parametrize("S", [164, 300])
def test_ckpt_calls_without_dx_and_with_frozen_fields(S):
    _compare(3, S, 2, 4, 0.1, with_dx=False, frozen=FROZEN)
    _compare(3, S, 2, 4, 0.1, with_dx=True, frozen=FROZEN)


@pytest.mark.parametrize("lens", [[37, 0, 164, 5], [200, 0, 13], [300, 7, 0, 64]])
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_ckpt_calls_equal_the_arena_calls_varlen(lens, p):
    _compare(len(lens), max(lens), 2, 4, p, lens=lens)


def test_ckpt_calls_varlen_without_dx_and_with_frozen_fields():
    _compare(4, 164, 2, 4, 0.1, lens=[37, 0, 164, 5], with_dx=False, frozen=FROZEN)


@pytest.mark.parametrize("S", [164, 300])
def test_ckpt_calls_default_mode_within_reordering(S):
    _compare(3, S, 2, 4, 0.1, det=False)


# ---------------------------------------------------------------------------------------------------------------------------
# the model
# ---------------------------------------------------------------------------------------------------------------------------
def _build(name, unpadded=False):
    from visualbert_b200 import BertConfig, TrainVisualBERTObjective
    cfg, sd, batch, c, gold = golden_util.load(name)
    model = TrainVisualBERTObjective(BertConfig.from_dict(cfg), c["head"], visual_embedding_dim=c["Dv"], **c.get("flags", {}))
    model.load_state_dict(sd, strict=False)
    model.to(DEV).train(True)
    if unpadded:
        model.bert.set_unpadded(True)
    return model, {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in batch.items()}


def _step(model, batch, state, ckpt):
    """One deterministic forward + backward from a given dropout state -> (every tensor output, encoder outputs, {name: grad})."""
    torch.use_deterministic_algorithms(True)
    try:
        model.bert.set_activation_checkpointing(ckpt)
        model.bert.set_dropout_state(state)
        torch.manual_seed(7)
        model.zero_grad(set_to_none=True)
        enc = []
        hook = model.bert.encoder.register_forward_hook(lambda m, i, o: enc.append(o))
        out = model(**batch)
        hook.remove()
        res = {k: out[k] for k in list(out.keys()) if k != "logits"}
        # the attention-weights model returns maps and no loss: its backward starts from the encoder output
        loss = out["loss"] if out["loss"] is not None else enc[0][0][-1].float().square().mean()
        loss.backward()
        torch.cuda.synchronize()
        grads = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}
        return res, enc, grads
    finally:
        torch.use_deterministic_algorithms(False)
        model.bert.set_activation_checkpointing(False)


def _same(a, b, what):
    if isinstance(a, dict):
        assert a.keys() == b.keys(), what
        for k in a:
            _same(a[k], b[k], f"{what}[{k}]")
    elif torch.is_tensor(a):
        assert torch.is_tensor(b) and a.shape == b.shape and a.dtype == b.dtype, what
        assert torch.equal(a.detach(), b.detach()), f"{what} differs"
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), what
        for i, (u, v) in enumerate(zip(a, b)):
            _same(u, v, f"{what}[{i}]")
    else:
        assert a == b, what


def _check_model(model, batch, what):
    state = model.bert.dropout_state()
    want = _step(model, batch, state, False)
    got = _step(model, batch, state, True)
    _same(got[0], want[0], f"{what} outputs")
    _same(got[1], want[1], f"{what} encoder outputs")
    assert got[2].keys() == want[2].keys() and len(want[2]) > 0, what
    for k in want[2]:
        assert torch.equal(got[2][k], want[2][k]), f"{what}: gradient of {k}"
    return want


GOLDEN = [n for n, c in golden_util.cases().items() if "model" in c]


@pytest.mark.parametrize("name", GOLDEN)
def test_model_checkpointing_keeps_every_bit(name):
    """Every golden case's head in training mode with dropout (the attention-weights case compares its maps as outputs)."""
    model, batch = _build(name)
    _check_model(model, batch, name)


@pytest.mark.parametrize("name", ["small_ragged_pretraining", "base3_ragged_pretraining"])
def test_model_checkpointing_unpadded(name):
    model, batch = _build(name, unpadded=True)
    _check_model(model, batch, f"{name} unpadded")


@pytest.mark.parametrize("pattern", ["b", "c"])
def test_model_checkpointing_with_frozen_layers(pattern):
    """Patterns (b) and (c) of the frozen-parameter tests: the bottom layer frozen with the embeddings (the checkpointed call
    covers the layers above it), and every layer frozen with the text embeddings (only the input gradient flows)."""
    from visualbert_b200 import BertConfig, TrainVisualBERTObjective, synthetic
    cfg = synthetic.bert_config_dict(3, 256, 4, 1024, vocab=512)
    model = TrainVisualBERTObjective(BertConfig.from_dict(cfg), "pretraining", visual_embedding_dim=64)
    model.load_state_dict(synthetic.init_state_dict(cfg, "pretraining", 64, seed=0), strict=False)
    model.to(DEV).train(True)
    batch = synthetic.make_batch(4, 20, 10, 64, head="pretraining", seed=1234, vocab=512, ragged=True)
    batch = {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in batch.items()}
    names = [n for n, _ in model.named_parameters()]
    emb = [n for n in names if n.startswith("bert.embeddings.")]
    text = [n for n in emb if any(t in n for t in ("word_embeddings", ".position_embeddings.", ".token_type_embeddings."))]
    layers = [n for n in names if n.startswith("bert.encoder.layer.")]
    frozen = emb + [n for n in layers if n.startswith("bert.encoder.layer.0.")] if pattern == "b" else text + layers
    for n, p in model.named_parameters():
        p.requires_grad_(n not in frozen)
    want = _check_model(model, batch, f"frozen ({pattern})")
    assert not (set(frozen) & want[2].keys())


def test_checkpointed_graphed_step_with_optimizer():
    """GraphedStep(optimizer=BertAdam) with checkpointing gives the parameters of the eager step without it after three steps; its
    graph's pool is smaller than the arena path's; changing the flag captures a new graph."""
    from visualbert_b200 import BertAdam, BertConfig, TrainVisualBERTObjective, graphs, parallel, synthetic
    torch.use_deterministic_algorithms(True)
    state = {"seed": 77, "step": 5}
    batches = []
    for i in range(3):
        b = synthetic.make_batch(64, 24, 16, 64, head="nlvr", seed=100 + i, vocab=512, ragged=True)
        batches.append({k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in b.items()})

    def setup():
        cfg = synthetic.bert_config_dict(4, 256, 4, 1024, vocab=512)
        model = TrainVisualBERTObjective(BertConfig.from_dict(cfg), "nlvr", visual_embedding_dim=64)
        model.load_state_dict(synthetic.init_state_dict(cfg, "nlvr", 64, seed=0), strict=False)
        for m in model.modules():
            if isinstance(m, torch.nn.Dropout):
                m.p = 0.0
        model.to(DEV).train(True)
        model.bert.set_dropout_state(state)
        sync = parallel.FlatGradSync(model)
        opt = BertAdam(list(model.parameters()), lr=1e-3, warmup=0.1, t_total=10, max_grad_norm=1.0)
        return model, sync, opt

    ref, ref_sync, ref_opt = setup()
    ref_losses = []
    for b in batches:
        ref_sync.zero()
        out = ref(**b)
        out["loss"].backward()
        ref_losses.append(out["loss"].detach().clone())
        ref_opt.step()

    # the first capture of a process also allocates the capture stream's library workspaces inside its pool: the arena step is
    # captured once before the two captures whose pools are compared. B = 64, S = 40 makes an arena slot (21 MB) larger than
    # the allocator's 20 MB segments for mid-sized blocks, so the pools differ by the arena and not by segment rounding.
    pools = []
    for ckpt in (False, True, False):
        model, sync, opt = setup()
        model.bert.set_activation_checkpointing(ckpt)
        step = graphs.GraphedStep(model, sync, optimizer=opt)
        losses = [step(batches[0]).get("loss").detach().clone()]   # eager warm-up
        losses += [step(b)["loss"].detach().clone() for b in batches[1:]]   # capture + replay, replay
        torch.cuda.synchronize()
        assert len(step.graphs) == 1
        pool = tuple(next(iter(step.graphs.values())).graph.pool())
        pools.append(sum(seg["total_size"] for seg in torch.cuda.memory_snapshot() if tuple(seg["segment_pool_id"]) == pool))
        for a, b in zip(losses, ref_losses):
            assert torch.equal(a, b), ckpt
        for (n, p), q in zip(model.named_parameters(), ref.parameters()):
            assert torch.equal(p.detach(), q.detach()), (ckpt, n)
        if ckpt:
            model.bert.set_activation_checkpointing(False)   # a new signature: warm-up call, then a second capture
            step(batches[0])
            step(batches[1])
            assert len(step.graphs) == 2
        del step, model, sync, opt
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
    assert 0 < pools[1] < pools[2], pools
    torch.use_deterministic_algorithms(False)


# ---------------------------------------------------------------------------------------------------------------------------
# memory
# ---------------------------------------------------------------------------------------------------------------------------
def _encoder_peak(L, ckpt, B=32, S=164, H=768, A=12, I=3072):
    """Peak allocated above the pre-call baseline over one forward + backward of a training-mode BertEncoder (dropout on)."""
    from visualbert_b200 import BertConfig, synthetic
    from visualbert_b200.modeling import BertEncoder
    cfg = BertConfig.from_dict(synthetic.bert_config_dict(L, H, A, I, vocab=512))
    enc = BertEncoder(cfg).to(DEV).train(True)
    enc.activation_checkpointing = ckpt
    x = torch.randn(B, S, H, device=DEV, dtype=BF, requires_grad=True)
    mask = torch.zeros(B, S, device=DEV)

    def run():
        y = enc(x, mask, output_all_encoded_layers=False, seed=1)[-1]
        y.backward(torch.ones_like(y))
        del y

    run()   # weights, scratch and gradients allocated outside the measurement
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    run()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del enc, x
    torch.cuda.empty_cache()
    return peak


def test_checkpointed_memory_is_one_slot_plus_the_checkpoints():
    """8 layers, H = 768, B = 32, S = 164: the peak is at most (L - 1) checkpoint regions + one slot + the backward's fp32 gradient
    buffer (the parameters' .grad are not flat-buffer views here, so each layer's gradients are computed into a fresh buffer and
    handed to autograd) + its dy and dx + 64 MB; the backward scratch exists before the measurement. From 4 to 8 layers the peak
    grows by about one region and one layer's gradients per layer, where the arena path grows by a slot per layer."""
    from visualbert_b200 import _lib
    B, S, H, A, I = 32, 164, 768, 12, 3072
    stride = int(_lib.lib().vb_encoder_arena_layout(B, S, H, A, I, 1, None))
    cs = int(_lib.lib().vb_encoder_ckpt_layout(B, S, H, A, I, -1, None))
    act = B * S * H * 2
    grads = 4 * (4 * H * H + 2 * H * I + 9 * H + I)   # fp32 gradient bytes of one layer
    mb = 1 << 20
    peaks = {(L, c): _encoder_peak(L, c) for L in (4, 8) for c in (True, False)}
    info = {k: v // mb for k, v in peaks.items()}
    assert peaks[8, True] <= 7 * cs + stride + 8 * grads + 4 * act + 64 * mb, (info, cs // mb, stride // mb)
    assert abs((peaks[8, True] - peaks[4, True]) - 4 * (cs + grads)) <= 16 * mb, (info, cs // mb, grads // mb)
    assert peaks[8, False] - peaks[4, False] >= 4 * stride - 16 * mb, (info, stride // mb)
