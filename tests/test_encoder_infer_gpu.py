"""The forward-only encoder route on the GPU: the VB_EPI_GELU_FWD epilogue against VB_EPI_GELU's aux_out and an fp64 reference,
vb_encoder_infer / vb_encoder_infer_varlen against vb_encoder_fwd / vb_encoder_fwd_varlen bit for bit on every attention route
with and without dropout, the model under torch.no_grad() against the same model with grad enabled, and the memory the route
exists for: outputs that own only their own bytes and a peak that does not grow with the depth."""
import ctypes
import itertools

import pytest
import torch

import golden_util
from gemm_ref_util import GELU_APPROX, GELU_LIP, check_close, gelu64, tile_n

pytestmark = pytest.mark.gpu

BF, F32 = torch.bfloat16, torch.float32
NAN16 = 0x7FA5     # bf16 NaN bit pattern of the guard bands
GUARD = 4096       # guard bytes on each side of a raw buffer (keeps the 256-byte alignment of the allocation)


def _dev():
    return torch.device("cuda:0")


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


class Guarded:
    """rows x cols bf16 output inside a [2 + rows + 3, cols + 16 g] allocation prefilled with a NaN bit pattern."""

    def __init__(self, rows, cols, g):
        self.ld = cols + 16 * g
        self.buf = torch.full((2 + rows + 3, self.ld), NAN16, dtype=torch.int16, device=_dev()).view(BF)
        self.t = self.buf[2:2 + rows, :cols]
        self.inside = torch.zeros(self.buf.shape, dtype=torch.bool, device=_dev())
        self.inside[2:2 + rows, :cols] = True

    def check_bands(self, what):
        n = int((self.buf.view(torch.int16)[~self.inside] != NAN16).sum())
        assert n == 0, f"{what}: {n} elements written outside the output"


class GuardedBytes:
    """n bytes between two GUARD-byte bands of 0xA5."""

    def __init__(self, n):
        self.n = n
        self.buf = torch.full((n + 2 * GUARD,), 0xA5, dtype=torch.uint8, device=_dev())
        self.t = self.buf[GUARD:GUARD + n]

    def ptr(self):
        return self.t.data_ptr()

    def check_bands(self, what):
        assert bool((self.buf[:GUARD] == 0xA5).all()) and bool((self.buf[GUARD + self.n:] == 0xA5).all()), f"{what}: guard band overwritten"


# ---------------------------------------------------------------------------------------------------------------------------
# the epilogue
# ---------------------------------------------------------------------------------------------------------------------------
TILE_EDGES = [(1, 16, 8), (64, 112, 48), (127, 128, 64), (128, 144, 72), (129, 240, 200), (255, 256, 768), (300, 272, 3072),
              (1000, 384, 72), (129, 768, 8), (64, 2304, 200), (127, 3072, 48), (1000, 2304, 768), (300, 16, 3072),
              (300, 2112, 200), (256, 512, 136)]   # the tile edges of test_gemm_reference_gpu.py, and one tile-native shape


def _gemm(**kw):
    from visualbert_b200 import _lib
    a = _lib.GemmArgs()
    for k, v in kw.items():
        setattr(a, k, v)
    _lib.check(_lib.lib().vb_gemm(ctypes.byref(a), _st()), "vb_gemm")


def test_gelu_fwd_epilogue_equals_the_gelu_epilogues_activation():
    """D of VB_EPI_GELU_FWD is aux_out of VB_EPI_GELU bit for bit (row-major and tile-native gelu'), within the fp64 bound of
    gemm_ref_util, written nowhere outside D; both tile widths, strided A, B and D; the kernels launched are the two
    EPI = 9 instantiations."""
    from torch.profiler import ProfilerActivity, profile
    from visualbert_b200 import _lib
    widths, worst = set(), 0.0
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for M, N, K in TILE_EDGES:
            torch.manual_seed(M + N + K)
            lda = ldb = (K + 7) // 8 * 8 + 8
            A = torch.randn(M, lda, device=_dev()).to(BF)[:, :K]
            B = (0.05 * torch.randn(N, ldb, device=_dev())).to(BF)[:, :K]
            bias = torch.randn(N, device=_dev())
            kw = dict(A=A.data_ptr(), lda=lda, B=B.data_ptr(), ldb=ldb, M=M, N=N, K=K, bias=bias.data_ptr())
            case = f"M={M} N={N} K={K}"
            tiled = bool(_lib.lib().vb_gemm_gp_tiled_ok(M, N))
            gp, g = Guarded(M, N, 0 if tiled else 1), Guarded(M, N, 1)
            _gemm(D=gp.t.data_ptr(), ldd=gp.ld, epilogue=_lib.VB_EPI_GELU, aux_out=g.t.data_ptr(), ld_aux=g.ld, gp_tiled=int(tiled), **kw)
            d = Guarded(M, N, 2)
            _gemm(D=d.t.data_ptr(), ldd=d.ld, epilogue=_lib.VB_EPI_GELU_FWD, **kw)
            torch.cuda.synchronize()
            d.check_bands(case)
            assert torch.isfinite(d.t).all(), f"{case}: D has elements the call did not write"
            assert torch.equal(d.t.contiguous().view(torch.int16), g.t.contiguous().view(torch.int16)), f"{case}: differs from VB_EPI_GELU's aux_out"
            a64, b64 = A.double(), B.double()
            acc, mag = a64 @ b64.t() + bias.double(), a64.abs() @ b64.abs().t() + bias.double().abs()
            worst = max(worst, check_close(d.t, gelu64(acc), GELU_LIP * mag, True, case, GELU_APPROX * (1.0 + acc.abs())))
            widths.add(tile_n(N))
    assert widths == {128, 256}
    names = {e.name for e in prof.events() if "gemm_wgmma_kernel" in e.name}
    if names:   # the profiler may record nothing on a machine without CUPTI access
        for bn in (128, 256):
            assert any(f"gemm_wgmma_kernel<false, false, {bn}, false, 9>" in n for n in names), sorted(names)
    print(f"\ngelu_fwd worst error / bound: {worst:.3g}")


# ---------------------------------------------------------------------------------------------------------------------------
# the encoder call through the C ABI
# ---------------------------------------------------------------------------------------------------------------------------
def _layers(L, B, S, A, p_h, p_a, mask_bias):
    """L random layers of hidden 64 A, intermediate 256 A: (descriptor array, the tensors it points to)."""
    from visualbert_b200 import _lib
    H, I, dev = 64 * A, 256 * A, _dev()
    rnd = lambda *s, sc=1.0: sc * torch.randn(*s, device=dev)
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


def _compare(B, S, A, L, p_h, p_a, lens=None, maps=False):
    from visualbert_b200 import _lib
    lib, dev = _lib.lib(), _dev()
    torch.manual_seed(B * 1000 + S)
    H, I = 64 * A, 256 * A
    vl = lens is not None
    M = sum(lens) if vl else B * S
    drop = 1 if p_a > 0 else 0
    if vl:
        cu = torch.tensor([0] + list(itertools.accumulate(lens)), dtype=torch.int32, device=dev)
        mbias = None
    else:
        valid = torch.arange(S, device=dev)[None, :] < torch.randint(S // 2, S + 1, (B, 1), device=dev)
        mbias = ((~valid).float() * -10000.0).contiguous()
    descs, keep = _layers(L, B, S, A, p_h, p_a, mbias)
    x = torch.randn(M, H, device=dev).to(BF)
    off = (ctypes.c_int64 * _lib.VB_ENCODER_ARENA_BUFFERS)()
    if vl:
        stride = int(lib.vb_encoder_arena_layout_varlen(B, S, M, H, A, I, drop, off))
    else:
        stride = int(lib.vb_encoder_arena_layout(B, S, H, A, I, drop, off))
    arena = torch.zeros(L * stride, device=dev, dtype=torch.uint8)
    n0 = _lib.launch_count()
    if vl:
        _lib.check(lib.vb_encoder_fwd_varlen(descs, L, cu.data_ptr(), M, x.data_ptr(), arena.data_ptr(), _st()), "vb_encoder_fwd_varlen")
    else:
        _lib.check(lib.vb_encoder_fwd(descs, L, ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(arena.data_ptr()), _st()), "vb_encoder_fwd")
    n_arena = _lib.launch_count() - n0
    want = [arena[l * stride + off[13]: l * stride + off[13] + M * H * 2].view(torch.int16).view(M, H) for l in range(L)]

    nbytes = int(lib.vb_encoder_infer_workspace(B, S, H, A, I, drop, M if vl else -1))
    assert 0 < nbytes <= stride
    ws, y_all, y_last = GuardedBytes(nbytes), GuardedBytes(L * M * H * 2), GuardedBytes(M * H * 2)

    def infer(yl, ya, probs=None):
        n = _lib.launch_count()
        if vl:
            _lib.check(lib.vb_encoder_infer_varlen(descs, L, cu.data_ptr(), M, x.data_ptr(), ws.ptr(), yl, ya, _st()), "vb_encoder_infer_varlen")
        else:
            _lib.check(lib.vb_encoder_infer(descs, L, x.data_ptr(), ws.ptr(), yl, ya, probs, _st()), "vb_encoder_infer")
        return _lib.launch_count() - n

    what = f"B={B} S={S} A={A} L={L} p_h={p_h} p_a={p_a} lens={lens}"
    assert infer(None, y_all.ptr()) <= n_arena, what
    assert infer(y_last.ptr(), None) <= n_arena, what
    torch.cuda.synchronize()
    got = y_all.t.view(torch.int16).view(L, M, H)
    for l in range(L):
        assert torch.equal(got[l], want[l]), f"{what}: layer {l} of y_all differs from the arena's"
    assert torch.equal(y_last.t.view(torch.int16).view(M, H), want[-1]), f"{what}: y_last differs"
    for b, name in ((ws, "workspace"), (y_all, "y_all"), (y_last, "y_last")):
        b.check_bands(f"{what} {name}")
    if maps:
        p_want = torch.empty(L, B, A, S, S, device=dev)
        p_got = torch.full_like(p_want, float("nan"))
        _lib.check(lib.vb_encoder_attention_probs(descs, L, arena.data_ptr(), p_want.data_ptr(), _st()), "vb_encoder_attention_probs")
        assert infer(None, y_all.ptr(), p_got.data_ptr()) == n_arena + L
        torch.cuda.synchronize()
        assert torch.equal(p_got, p_want), f"{what}: attention maps differ"
    del keep


@pytest.mark.parametrize("S", [164, 200, 300])          # wgmma, whole-head and staged attention
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_infer_equals_the_training_forward_dense(S, p):
    _compare(3, S, 2, 3, p, p, maps=p == 0.0)            # M = 3 S is no multiple of 128


def test_infer_equals_the_training_forward_with_tile_native_gelu_prime():
    """M and I multiples of 256: the training forward keeps gelu'(u) tile-native (another GEMM kernel); same activations.
    One layer and two layers: y_last straight from the only layer, and through one ping-pong buffer."""
    _compare(4, 64, 4, 1, 0.0, 0.0)
    _compare(4, 64, 4, 2, 0.1, 0.1)
    _compare(2, 128, 12, 4, 0.1, 0.0)


@pytest.mark.parametrize("lens", [[37, 0, 164, 5], [200, 0, 13], [300, 7, 0, 64]])
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_infer_equals_the_training_forward_varlen(lens, p):
    _compare(len(lens), max(lens), 2, 3, p, p, lens=lens)


# ---------------------------------------------------------------------------------------------------------------------------
# the model
# ---------------------------------------------------------------------------------------------------------------------------
def _build(name, train, unpadded=False):
    from visualbert_b200 import BertConfig, TrainVisualBERTObjective
    cfg, sd, batch, c, gold = golden_util.load(name)
    model = TrainVisualBERTObjective(BertConfig.from_dict(cfg), c["head"], visual_embedding_dim=c["Dv"], **c.get("flags", {}))
    model.load_state_dict(sd, strict=False)
    model.to(_dev()).train(train)
    if unpadded:
        model.bert.set_unpadded(True)
    batch = {k: (v.to(_dev()) if torch.is_tensor(v) else v) for k, v in batch.items()}
    return model, batch, c


def _forward(model, batch, grad, state, **kw):
    """One forward from a given dropout state (the library's and torch's own generator, which the PyTorch task heads draw
    from) -> every tensor of the output dict, plus what model.bert returned."""
    model.bert.set_dropout_state(state)
    torch.manual_seed(7)
    seen = {}
    hook = model.bert.register_forward_hook(lambda m, i, o: seen.__setitem__("bert", o))
    with torch.set_grad_enabled(grad):
        out = model(**batch, **kw)
        res = {k: out[k] for k in list(out.keys())}   # resolves the lazily built pretraining logits
    hook.remove()
    seq, pooled = seen["bert"][0], seen["bert"][1]
    res["bert.sequence_output"], res["bert.pooled_output"] = seq, pooled
    return res


def _same(a, b, what):
    if torch.is_tensor(a):
        assert torch.is_tensor(b) and a.shape == b.shape and a.dtype == b.dtype, what
        assert torch.equal(a.detach(), b.detach()), f"{what} differs"
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), what
        for i, (u, v) in enumerate(zip(a, b)):
            _same(u, v, f"{what}[{i}]")
    else:
        assert a == b, what


MODEL_CASES = [("cfg1_pretraining", False), ("small_vqa", False), ("small_nlvr", False), ("small_multichoice", False),
               ("small_flickr", False), ("small_bypass_nlvr", False), ("small_vcr_alignment", False),
               ("small_ragged_pretraining", True), ("base3_ragged_pretraining", True)]


@pytest.mark.parametrize("name, unpadded", MODEL_CASES)
@pytest.mark.parametrize("train", [False, True])
def test_no_grad_forward_equals_the_grad_enabled_forward(name, unpadded, train):
    model, batch, c = _build(name, train, unpadded)
    state = model.bert.dropout_state()
    want = _forward(model, batch, True, state)
    got = _forward(model, batch, False, state)
    assert set(got) == set(want) and "loss" in got
    for k in want:
        _same(got[k], want[k], f"{name} train={train} {k}")
    assert not got["bert.sequence_output"].requires_grad
    if c.get("flags", {}).get("bypass_transformer") or train:
        return
    # every layer's output (eval mode: with grad enabled this is the whole-encoder arena call too)
    want = _forward(model, batch, True, state, output_all_encoded_layers=True)
    got = _forward(model, batch, False, state, output_all_encoded_layers=True)
    assert len(got["sequence_output"]) == len(model.bert.encoder.layer)
    for k in want:
        _same(got[k], want[k], f"{name} all layers {k}")


@pytest.mark.parametrize("train", [False, True])
def test_no_grad_attention_maps_equal_the_arena_routes(train):
    model, batch, c = _build("small_attention_weights", train)
    state = model.bert.dropout_state()
    model.bert.set_dropout_state(state)
    want = model(**batch)["attention_weights"]
    model.bert.set_dropout_state(state)
    with torch.no_grad():
        got = model(**batch)["attention_weights"]
    assert len(got) == len(want) == 2
    _same(list(got), list(want), f"attention maps train={train}")


def test_backward_is_unchanged_by_no_grad_forwards_in_between():
    """The plan and its descriptor array are shared by both routes: a no_grad forward before a training step, and one (in eval
    mode, so with other dropout settings stamped into the descriptors) between a forward and its backward, change neither the
    loss nor the gradients."""
    model, batch, c = _build("base3_ragged_pretraining", True)
    state = model.bert.dropout_state()

    def step(before, between):
        model.zero_grad(set_to_none=True)
        if before:
            with torch.no_grad():
                model(**batch)
        model.bert.set_dropout_state(state)
        torch.manual_seed(7)
        out = model(**batch)
        if between:
            model.eval()
            with torch.no_grad():
                model(**batch)
            model.train()
        out["loss"].backward()
        return out["loss"].detach().clone(), {k: p.grad.detach().clone() for k, p in model.named_parameters() if p.grad is not None}

    loss0, g0 = step(False, False)
    for before, between in ((True, False), (False, True)):
        loss, g = step(before, between)
        assert torch.equal(loss, loss0)
        assert set(g) == set(g0)
        for k in g0:   # fp32 red.add accumulation: the order of the partial sums is not fixed
            assert (g[k] - g0[k]).norm().item() <= 1e-4 * g0[k].norm().item() + 1e-12, k


# ---------------------------------------------------------------------------------------------------------------------------
# memory
# ---------------------------------------------------------------------------------------------------------------------------
def _big_model(L):
    from visualbert_b200 import BertConfig, TrainVisualBERTObjective, synthetic
    cfg = synthetic.bert_config_dict(L, 768, 12, 3072, vocab=2048)
    sd = synthetic.init_state_dict(cfg, "pretraining", 2048, seed=0)
    model = TrainVisualBERTObjective(BertConfig.from_dict(cfg), "pretraining", visual_embedding_dim=2048)
    model.load_state_dict(sd, strict=False)
    model.to(_dev()).eval()
    batch = synthetic.make_batch(64, 128, 36, 2048, head="pretraining", seed=1234, vocab=2048, ragged=True)
    return model, {k: (v.to(_dev()) if torch.is_tensor(v) else v) for k, v in batch.items()}


def _peak(model, batch, grad):
    seen = {}
    hook = model.bert.register_forward_hook(lambda m, i, o: seen.__setitem__("nbytes", o[0].untyped_storage().nbytes()))
    with torch.set_grad_enabled(grad):
        model(**batch)   # weight bank and first-call set-up outside the measurement
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out = model(**batch)
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
    hook.remove()
    del out
    return peak, seen["nbytes"]


def test_no_grad_forward_memory_does_not_grow_with_depth():
    """H = 768, B = 64, S = 164, eval: the sequence output of a no_grad forward owns B S H bf16 and nothing else; the peak above
    the pre-call baseline is the same for 2 and 8 layers and below workspace + 256 MB, while the grad-enabled forward's grows
    by one arena slot per layer."""
    from visualbert_b200 import _lib
    B, S, H, A, I = 64, 164, 768, 12, 3072
    ws = int(_lib.lib().vb_encoder_infer_workspace(B, S, H, A, I, 0, -1))
    stride = int(_lib.lib().vb_encoder_arena_layout(B, S, H, A, I, 0, None))
    peaks = {}
    for L in (2, 8):
        model, batch = _big_model(L)
        peaks[L, False], nbytes = _peak(model, batch, False)
        assert nbytes == B * S * H * 2
        peaks[L, True], nbytes_arena = _peak(model, batch, True)
        assert nbytes_arena >= L * stride
        del model, batch
        torch.cuda.empty_cache()
    mb = 1 << 20
    assert abs(peaks[8, False] - peaks[2, False]) < 64 * mb, {k: v // mb for k, v in peaks.items()}
    assert peaks[8, False] < ws + 256 * mb, (peaks[8, False] // mb, ws // mb)
    assert peaks[8, True] - peaks[2, True] >= 6 * stride - 64 * mb, {k: v // mb for k, v in peaks.items()}
