"""Selective FFN recomputation on the GPU: vb_encoder_fwd_ffnrc / vb_encoder_bwd_ffnrc (and the _varlen forms) against
vb_encoder_fwd / vb_encoder_bwd on the same descriptors and inputs, bit for bit; their kernel lists against the arena calls'
(the backward adds exactly L - 1 FFN-up GEMMs); the model with set_ffn_recompute against the model without it (loss, every
output, every gradient and dx, attention maps, bypass_transformer, frozen patterns, unpadded batches, with full checkpointing
on at the same time, GraphedStep with BertAdam); and the memory the mode exists for.

Like test_zz_checkpointing_gpu.py, the file sorts after the tests that count kernel records through torch.profiler, so its
model steps and graph captures do not run ahead of them in one process."""
import collections
import ctypes
import itertools
import json
import time

import pytest
import torch

from test_zz_checkpointing_gpu import FROZEN, GOLDEN, Grads, GuardedBytes, _build, _layers, _same, _scratch, _st

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
DEV = "cuda:0"
PROFILE_PAD_S = 0.05


@pytest.fixture(autouse=True)
def _cublas(monkeypatch):
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    yield
    torch.use_deterministic_algorithms(False)


class _Calls:
    """One stack of L random layers with its inputs, run through the arena calls or the _ffnrc calls."""

    def __init__(self, B, S, A, L, p, lens=None, frozen=None, with_dx=True):
        from visualbert_b200 import _lib
        self.lib = lib = _lib.lib()
        torch.manual_seed(B * 1000 + S + L)
        self.B, self.S, self.A, self.L, self.lens, self.frozen, self.with_dx = B, S, A, L, lens, frozen, with_dx
        self.H, self.I = H, I = 64 * A, 256 * A
        self.vl = vl = lens is not None
        self.M = M = sum(lens) if vl else B * S
        drop = 1 if p > 0 else 0
        if vl:
            self.cu = torch.tensor([0] + list(itertools.accumulate(lens)), dtype=torch.int32, device=DEV)
            mbias = None
        else:
            valid = torch.arange(S, device=DEV)[None, :] < torch.randint(S // 2, S + 1, (B, 1), device=DEV)
            mbias = ((~valid).float() * -10000.0).contiguous()
        self.mbias = mbias
        self.descs, self.keep = _layers(L, B, S, A, p, p, mbias)
        self.x = torch.randn(M, H, device=DEV).to(BF)
        self.dy = torch.randn(M, H, device=DEV).to(BF)
        n = _lib.VB_ENCODER_ARENA_BUFFERS
        self.off, self.roff, fb = (ctypes.c_int64 * n)(), (ctypes.c_int64 * n)(), ctypes.c_int64()
        if vl:
            self.stride = int(lib.vb_encoder_arena_layout_varlen(B, S, M, H, A, I, drop, self.roff))
            self.fstride = int(lib.vb_encoder_arena_layout_ffnrc_varlen(B, S, M, H, A, I, drop, self.off, ctypes.byref(fb)))
        else:
            self.stride = int(lib.vb_encoder_arena_layout(B, S, H, A, I, drop, self.roff))
            self.fstride = int(lib.vb_encoder_arena_layout_ffnrc(B, S, H, A, I, drop, self.off, ctypes.byref(fb)))
        self.ffn_bytes = fb.value
        self.sc, self.sc_keep = _scratch(M, H, I, A)

    def buffers(self, ffnrc):
        """Fresh guarded arena (and shared FFN buffer), gradients and dx."""
        arena = GuardedBytes(self.L * (self.fstride if ffnrc else self.stride), fill=0xA5)
        ffn = GuardedBytes(self.ffn_bytes, fill=0xA5) if ffnrc else None
        return arena, ffn, Grads(self.L, self.H, self.I, self.frozen), GuardedBytes(self.M * self.H * 2) if self.with_dx else None

    def fwd(self, arena, ffn):
        from visualbert_b200 import _lib
        lib = self.lib
        if self.vl and ffn is None:
            rc = lib.vb_encoder_fwd_varlen(self.descs, self.L, self.cu.data_ptr(), self.M, self.x.data_ptr(), arena.ptr(), _st())
        elif self.vl:
            rc = lib.vb_encoder_fwd_ffnrc_varlen(self.descs, self.L, self.cu.data_ptr(), self.M, self.x.data_ptr(), arena.ptr(), ffn.ptr(),
                                                 _st())
        elif ffn is None:
            rc = lib.vb_encoder_fwd(self.descs, self.L, ctypes.c_void_p(self.x.data_ptr()), ctypes.c_void_p(arena.ptr()), _st())
        else:
            rc = lib.vb_encoder_fwd_ffnrc(self.descs, self.L, self.x.data_ptr(), arena.ptr(), ffn.ptr(), _st())
        _lib.check(rc, "forward")

    def bwd(self, arena, ffn, g, dx):
        from visualbert_b200 import _lib
        lib = self.lib
        dxp, sref = dx.ptr() if dx is not None else None, ctypes.byref(self.sc)
        if self.vl and ffn is None:
            rc = lib.vb_encoder_bwd_varlen(self.descs, self.L, self.cu.data_ptr(), self.M, self.x.data_ptr(), arena.ptr(), self.dy.data_ptr(),
                                           dxp, g.arr, sref, _st())
        elif self.vl:
            rc = lib.vb_encoder_bwd_ffnrc_varlen(self.descs, self.L, self.cu.data_ptr(), self.M, self.x.data_ptr(), arena.ptr(), ffn.ptr(),
                                                 self.dy.data_ptr(), dxp, g.arr, sref, _st())
        elif ffn is None:
            rc = lib.vb_encoder_bwd(self.descs, self.L, ctypes.c_void_p(self.x.data_ptr()), ctypes.c_void_p(arena.ptr()),
                                    ctypes.c_void_p(self.dy.data_ptr()), ctypes.c_void_p(dxp), g.arr, sref, _st())
        else:
            rc = lib.vb_encoder_bwd_ffnrc(self.descs, self.L, self.x.data_ptr(), arena.ptr(), ffn.ptr(), self.dy.data_ptr(), dxp, g.arr,
                                          sref, _st())
        _lib.check(rc, "backward")


class _Det:
    def __init__(self, c, on):
        self.c, self.on, self.ws = c, on, None

    def __enter__(self):
        if self.on:
            from visualbert_b200 import _lib
            lib = self.c.lib
            self.ws = torch.empty(max(int(lib.vb_deterministic_workspace_bytes(self.c.M, self.c.H, self.c.I, 0, 0)), 256), device=DEV,
                                  dtype=torch.uint8)
            _lib.check(lib.vb_set_deterministic(self.ws.data_ptr(), self.ws.numel()), "vb_set_deterministic")

    def __exit__(self, *exc):
        if self.on:
            self.c.lib.vb_set_deterministic(None, 0)


def _compare(B, S, A, L, p, lens=None, with_dx=True, frozen=None, det=True):
    """Arena calls and _ffnrc calls on the same descriptors, inputs and fresh gradient buffers."""
    from visualbert_b200 import _lib
    c = _Calls(B, S, A, L, p, lens, frozen, with_dx)
    what = f"B={B} S={S} A={A} L={L} p={p} lens={lens} dx={with_dx} frozen={frozen is not None} det={det}"
    n, st, fs, off, roff = c.M * c.H * 2, c.stride, c.fstride, c.off, c.roff
    mi, half, top = c.M * c.I * 2, c.ffn_bytes // 2, (c.L - 1) * c.stride
    with _Det(c, det):
        arena_r, _, g_r, dx_r = c.buffers(False)
        arena, ffn, g, dx = c.buffers(True)
        n0 = _lib.launch_count()
        c.fwd(arena_r, None)
        n1 = _lib.launch_count()
        c.fwd(arena, ffn)
        n2 = _lib.launch_count()
        torch.cuda.synchronize()
        assert n2 - n1 == n1 - n0, f"{what}: forward launches {n2 - n1} vs {n1 - n0}"
        for l in range(c.L):   # every slot buffer the arena call keeps, u and g apart, alignment gaps included
            for k in range(_lib.VB_ENCODER_ARENA_BUFFERS):
                if k in (7, 8):
                    continue
                size = n if k == 13 else off[k + 1] - off[k]
                assert torch.equal(arena.t[l * fs + off[k]: l * fs + off[k] + size], arena_r.t[l * st + roff[k]: l * st + roff[k] + size]), \
                    f"{what}: slot {l} buffer {_lib.ARENA_NAMES[k]}"
        # the shared buffer holds the top layer's gelu'(u) and g
        assert torch.equal(ffn.t[:mi], arena_r.t[top + roff[7]: top + roff[7] + mi]), f"{what}: top gelu'(u)"
        assert torch.equal(ffn.t[half: half + mi], arena_r.t[top + roff[8]: top + roff[8] + mi]), f"{what}: top g"
        u0, g0 = arena_r.t[roff[7]: roff[7] + mi].clone(), arena_r.t[roff[8]: roff[8] + mi].clone()
        n3 = _lib.launch_count()
        c.bwd(arena_r, None, g_r, dx_r)
        n4 = _lib.launch_count()
        c.bwd(arena, ffn, g, dx)
        n5 = _lib.launch_count()
        torch.cuda.synchronize()
    assert (n5 - n4) - (n4 - n3) == c.L - 1, f"{what}: backward launches {n5 - n4} vs {n4 - n3}"
    # after the backward the shared buffer holds layer 0's intermediates, rebuilt bit for bit
    assert torch.equal(ffn.t[:mi], u0), f"{what}: gelu'(u) of layer 0"
    assert torch.equal(ffn.t[half: half + mi], g0), f"{what}: g of layer 0"
    if with_dx:
        if det:
            assert torch.equal(dx.t, dx_r.t), f"{what}: dx"
        else:
            d, r = dx.t.view(BF).float(), dx_r.t.view(BF).float()
            assert (d - r).norm().item() <= 1e-2 * r.norm().item(), f"{what}: dx"
    got, want = g.values(), g_r.values()
    assert got.keys() == want.keys()
    for k in want:
        if det:
            assert torch.equal(got[k], want[k]), f"{what}: gradient {k}"
        else:   # fp32 red.add accumulation: the order of the partial sums is not fixed
            assert (got[k] - want[k]).norm().item() <= 1e-4 * want[k].norm().item() + 1e-6, f"{what}: gradient {k}"
    for buf, name in ((arena, "arena"), (ffn, "ffn"), (dx, "dx")):
        if buf is not None:
            buf.check_bands(f"{what} {name}")
    g.check_bands(what)


@pytest.mark.parametrize("S", [164, 200, 300])          # wgmma, whole-head and staged attention
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_ffnrc_calls_equal_the_arena_calls_dense(S, p):
    _compare(3, S, 2, 4, p)                              # M = 3 S: no tile-native gelu'


@pytest.mark.parametrize("L", [1, 2, 12])
def test_ffnrc_calls_with_1_2_and_12_layers(L):
    _compare(3, 164, 2, L, 0.1)


def test_ffnrc_calls_with_tile_native_gelu_prime_at_h768():
    """H = 768, I = 3072, M = 256: the training forward keeps gelu'(u) tile-native; the rebuild writes it the same way."""
    _compare(4, 64, 12, 12, 0.1)


def test_ffnrc_calls_without_dx_and_with_frozen_fields():
    _compare(3, 164, 2, 4, 0.1, with_dx=False, frozen=FROZEN)
    _compare(3, 300, 2, 4, 0.1, with_dx=True, frozen=FROZEN)


@pytest.mark.parametrize("lens", [[37, 0, 164, 5], [256, 256, 0, 256, 256]])   # the second: M = 1024, tile-native
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_ffnrc_calls_equal_the_arena_calls_varlen(lens, p):
    _compare(len(lens), max(lens), 2, 4, p, lens=lens)


def test_ffnrc_calls_varlen_without_dx_and_with_frozen_fields():
    _compare(4, 164, 2, 4, 0.1, lens=[37, 0, 164, 5], with_dx=False, frozen=FROZEN)


def test_ffnrc_calls_default_mode_within_reordering():
    _compare(3, 164, 2, 4, 0.1, det=False)


# ---------------------------------------------------------------------------------------------------------------------------
# the kernel lists
# ---------------------------------------------------------------------------------------------------------------------------
def _kernels(fn, path):
    """(name, grid) of every CUDA kernel fn launches, in launch order (copies and memsets left out), from a chrome trace.

    The profiler now and then loses kernel records, far more often late in a long process: a window whose record count is not
    the number of launches the library counted is profiled again, up to four times."""
    from torch.profiler import ProfilerActivity, profile
    from visualbert_b200 import _lib
    for _ in range(4):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            time.sleep(PROFILE_PAD_S)
            n0 = _lib.launch_count()
            fn()
            n = _lib.launch_count() - n0
            torch.cuda.synchronize()
            time.sleep(PROFILE_PAD_S)
        prof.export_chrome_trace(str(path))
        with open(path) as f:
            ev = json.load(f)["traceEvents"]
        ks = sorted((e for e in ev if e.get("cat") == "kernel"), key=lambda e: e["ts"])
        out = [(e["name"], tuple(e.get("args", {}).get("grid", ()))) for e in ks]
        if len(out) == n:
            return out
    raise AssertionError(f"the profiler recorded {len(out)} kernels of {n} launches in every window")


@pytest.mark.parametrize("case", [dict(B=3, S=164, A=2, L=4, p=0.1), dict(B=4, S=64, A=12, L=3, p=0.1),
                                  dict(B=4, S=164, A=2, L=3, p=0.1, lens=[37, 0, 164, 5])])
def test_ffnrc_kernel_lists(case, tmp_path):
    """The forward launches the arena forward's kernels with the same grids, in the same order; the backward launches the arena
    backward's kernels plus L - 1 instances of the forward's FFN-up GEMM (gemm_wgmma_kernel with the GELU training epilogue,
    one per layer of the forward)."""
    c = _Calls(case["B"], case["S"], case["A"], case["L"], case["p"], case.get("lens"))
    L = c.L
    with _Det(c, True):
        arena_r, _, g_r, dx_r = c.buffers(False)
        arena, ffn, g, dx = c.buffers(True)
        # warm-up: tensor maps and modules loaded outside the profiled windows
        c.fwd(arena_r, None); c.bwd(arena_r, None, g_r, dx_r); c.fwd(arena, ffn); c.bwd(arena, ffn, g, dx)
        f_ref = _kernels(lambda: c.fwd(arena_r, None), tmp_path / "f_ref.json")
        b_ref = _kernels(lambda: c.bwd(arena_r, None, g_r, dx_r), tmp_path / "b_ref.json")
        f = _kernels(lambda: c.fwd(arena, ffn), tmp_path / "f.json")
        b = _kernels(lambda: c.bwd(arena, ffn, g, dx), tmp_path / "b.json")
    assert f == f_ref
    extra = collections.Counter(b) - collections.Counter(b_ref)
    assert not (collections.Counter(b_ref) - collections.Counter(b)), "a kernel of the arena backward is missing"
    assert len(extra) == 1, extra
    (k, n), = extra.items()
    assert n == L - 1 and "gemm_wgmma_kernel" in k[0], extra
    assert collections.Counter(f)[k] == L, f"{k} is not the forward's FFN-up GEMM (once per layer)"


# ---------------------------------------------------------------------------------------------------------------------------
# the model
# ---------------------------------------------------------------------------------------------------------------------------
def _step(model, batch, state, ffn, ckpt=False, det=True):
    """One forward + backward from a given dropout state -> (every tensor output, encoder outputs, {name: grad})."""
    torch.use_deterministic_algorithms(det)
    try:
        model.bert.set_ffn_recompute(ffn)
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
        model.bert.set_ffn_recompute(False)
        model.bert.set_activation_checkpointing(False)


def _check_model(model, batch, what, ckpt=False, det=True):
    state = model.bert.dropout_state()
    want = _step(model, batch, state, False, ckpt, det)
    got = _step(model, batch, state, True, ckpt, det)
    _same(got[0], want[0], f"{what} outputs")
    _same(got[1], want[1], f"{what} encoder outputs")
    assert got[2].keys() == want[2].keys() and len(want[2]) > 0, what
    for k in want[2]:
        if det:
            assert torch.equal(got[2][k], want[2][k]), f"{what}: gradient of {k}"
        else:
            assert (got[2][k] - want[2][k]).norm().item() <= 1e-4 * want[2][k].norm().item() + 1e-6, f"{what}: gradient of {k}"
    return want


@pytest.mark.parametrize("name", GOLDEN)
def test_model_ffn_recompute_keeps_every_bit(name):
    """Every golden case's head in training mode with dropout: 1, 2 and 3 layers, H = 128 and 768, the attention-weights case
    (its maps compared as outputs) and bypass_transformer (the text encoder call)."""
    model, batch = _build(name)
    _check_model(model, batch, name)


@pytest.mark.parametrize("name", ["small_ragged_pretraining", "base3_ragged_pretraining"])
def test_model_ffn_recompute_unpadded(name):
    model, batch = _build(name, unpadded=True)
    _check_model(model, batch, f"{name} unpadded")


@pytest.mark.parametrize("name", ["small_attention_weights", "small_bypass_nlvr", "base3_ragged_pretraining"])
def test_model_with_checkpointing_on_too_is_the_checkpointed_path(name):
    model, batch = _build(name)
    _check_model(model, batch, f"{name} with checkpointing", ckpt=True)


@pytest.mark.parametrize("name", ["small_vqa", "base3_ragged_pretraining"])
def test_model_default_mode_outputs_equal_and_gradients_within_reordering(name):
    model, batch = _build(name)
    _check_model(model, batch, f"{name} default mode", det=False)


def _synthetic(L, H, A, I, head="pretraining", B=4, T=20, V=10):
    from visualbert_b200 import BertConfig, TrainVisualBERTObjective, synthetic
    cfg = synthetic.bert_config_dict(L, H, A, I, vocab=512)
    model = TrainVisualBERTObjective(BertConfig.from_dict(cfg), head, visual_embedding_dim=64)
    model.load_state_dict(synthetic.init_state_dict(cfg, head, 64, seed=0), strict=False)
    model.to(DEV).train(True)
    batch = synthetic.make_batch(B, T, V, 64, head=head, seed=1234, vocab=512, ragged=True)
    return model, {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in batch.items()}


def test_model_twelve_layers_h768_tile_native():
    """12 layers, H = 768, I = 3072, B = 8, S = 32: M = 256, so gelu'(u) is tile-native."""
    model, batch = _synthetic(12, 768, 12, 3072, B=8, T=20, V=12)
    _check_model(model, batch, "12 layers H 768")


@pytest.mark.parametrize("pattern", ["b", "c"])
def test_model_ffn_recompute_with_frozen_layers(pattern):
    """Patterns (b) and (c) of the frozen-parameter tests: the bottom layer frozen with the embeddings (the call covers the
    layers above it), and every layer frozen with the text embeddings (only the input gradient flows)."""
    model, batch = _synthetic(3, 256, 4, 1024)
    names = [n for n, _ in model.named_parameters()]
    emb = [n for n in names if n.startswith("bert.embeddings.")]
    text = [n for n in emb if any(t in n for t in ("word_embeddings", ".position_embeddings.", ".token_type_embeddings."))]
    layers = [n for n in names if n.startswith("bert.encoder.layer.")]
    frozen = emb + [n for n in layers if n.startswith("bert.encoder.layer.0.")] if pattern == "b" else text + layers
    for n, p in model.named_parameters():
        p.requires_grad_(n not in frozen)
    want = _check_model(model, batch, f"frozen ({pattern})")
    assert not (set(frozen) & want[2].keys())


def test_ffn_recompute_graphed_step_with_optimizer():
    """GraphedStep(optimizer=BertAdam) with the switch on gives the losses and parameters of the eager step without it after
    three steps; its graph's pool is smaller than the arena path's; changing the flag captures a new graph."""
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
        for m in model.modules():   # the heads' torch dropout draws from torch's generator, which replays do not advance
            if isinstance(m, torch.nn.Dropout):
                m.p = 0.0
        model.to(DEV).train(True)
        model.bert.set_dropout_state(state)
        sync = parallel.FlatGradSync(model)
        opt = BertAdam(list(model.parameters()), lr=1e-3, warmup=0.1, t_total=10, max_grad_norm=1.0)
        return model, sync, opt

    ref, ref_sync, ref_opt = setup()
    ref_losses, ref_grads = [], []
    for b in batches:
        ref_sync.zero()
        out = ref(**b)
        out["loss"].backward()
        ref_losses.append(out["loss"].detach().clone())
        ref_opt.step()
        ref_grads.append([p.grad.detach().clone() for p in ref.parameters()])

    # the first capture of a process allocates the capture stream's library workspaces inside its pool: the arena step is
    # captured once before the two captures whose pools are compared (B = 64, S = 40: the arena, 4 slots of 21 MB, is larger
    # than the allocator's 20 MB segments for mid-sized blocks, so the pools differ by the arena and not by segment rounding)
    pools = []
    for ffn in (False, True, False):
        model, sync, opt = setup()
        model.bert.set_ffn_recompute(ffn)
        step = graphs.GraphedStep(model, sync, optimizer=opt)
        losses = [step(batches[0]).get("loss").detach().clone()]   # eager warm-up
        for i, b in enumerate(batches[1:], 1):   # capture + replay, replay
            losses.append(step(b)["loss"].detach().clone())
            torch.cuda.synchronize()
            for p, q in zip(model.parameters(), ref_grads[i]):   # the gradients of the replayed step, as its optimizer left them
                assert torch.equal(p.grad, q), (ffn, i)
        torch.cuda.synchronize()
        assert len(step.graphs) == 1
        pool = tuple(next(iter(step.graphs.values())).graph.pool())
        pools.append(sum(seg["total_size"] for seg in torch.cuda.memory_snapshot() if tuple(seg["segment_pool_id"]) == pool))
        for a, b in zip(losses, ref_losses):
            assert torch.equal(a, b), ffn
        for (n, p), q in zip(model.named_parameters(), ref.parameters()):
            assert torch.equal(p.detach(), q.detach()), (ffn, n)
        if ffn:
            model.bert.set_ffn_recompute(False)   # a new signature: warm-up call, then a second capture
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
def _encoder(L, ffn, H=768, A=12, I=3072):
    from visualbert_b200 import BertConfig, synthetic
    from visualbert_b200.modeling import BertEncoder
    cfg = BertConfig.from_dict(synthetic.bert_config_dict(L, H, A, I, vocab=512))
    enc = BertEncoder(cfg).to(DEV).train(True)
    enc.ffn_recompute = ffn
    return enc


def test_arena_and_shared_buffer_are_the_layout():
    """The training call allocates L slots of the _ffnrc stride plus one shared buffer of the size the layout gives, dense and
    unpadded."""
    from visualbert_b200 import _lib, ops
    lib = _lib.lib()
    B, S, H, A, I, L = 4, 40, 256, 4, 1024, 3
    enc = _encoder(L, True, H, A, I)
    x = torch.randn(B, S, H, device=DEV, dtype=BF, requires_grad=True)
    y = enc(x, torch.zeros(B, S, device=DEV), output_all_encoded_layers=False, seed=1)[-1]
    fb = ctypes.c_int64()
    stride = int(lib.vb_encoder_arena_layout_ffnrc(B, S, H, A, I, 1, None, ctypes.byref(fb)))
    node = y.grad_fn
    assert node.arena.numel() == L * stride and node.ffn.numel() == fb.value == 2 * ((B * S * I * 2 + 255) // 256 * 256)
    y.backward(torch.ones_like(y))
    assert node.ffn is None and node.arena is None   # released by the backward
    valid = torch.arange(S, device=DEV)[None, :] < torch.tensor([[S], [7], [0], [S - 3]], device=DEV)
    plan = ops.unpad_plan(valid)
    xp = torch.randn(plan["total"], H, device=DEV, dtype=BF, requires_grad=True)
    y = enc(xp, None, output_all_encoded_layers=False, seed=1, varlen=plan)[-1]
    stride = int(lib.vb_encoder_arena_layout_ffnrc_varlen(B, plan["max_seq"], plan["total"], H, A, I, 1, None, ctypes.byref(fb)))
    assert y.grad_fn.arena.numel() == L * stride and y.grad_fn.ffn.numel() == fb.value
    y.backward(torch.ones_like(y))


def _encoder_peak(L, ffn, B=32, S=164):
    """Peak allocated above the pre-call baseline over one forward + backward of a training-mode BertEncoder (dropout on)."""
    enc = _encoder(L, ffn)
    x = torch.randn(B, S, 768, device=DEV, dtype=BF, requires_grad=True)
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


def test_peak_memory_drops_by_the_ffn_intermediates():
    """8 layers, H = 768, I = 3072, B = 32, S = 164: the peak drops by at least 90 % of (L - 1) * 2 * M * I * 2 bytes."""
    L, M, I = 8, 32 * 164, 3072
    saving = (L - 1) * 2 * M * I * 2
    arena, ffnrc = _encoder_peak(L, False), _encoder_peak(L, True)
    assert arena - ffnrc >= 0.9 * saving, (arena >> 20, ffnrc >> 20, saving >> 20)
