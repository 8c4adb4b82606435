"""Deterministic reductions (vb_set_deterministic, torch.use_deterministic_algorithms) on the GPU.

- Op level: the split-K weight-gradient GEMM (shapes chosen from the SM count so that they really split), the LayerNorm backward
  column sums, vb_colsum_bf16 and the BertAdam norms: inside the fp64 bound (GEMM: tests/gemm_ref_util.py; column sums: a stated
  fp32 bound), identical bits on a second call, guard bands around the outputs and the workspace's unused tail intact, and the
  deterministic kernels seen in the profiler.
- Whole training steps with dropout on, run twice in deterministic mode: loss, every gradient, and the parameters and Adam moments
  after two BertAdam steps are torch.equal (pretraining and vqa heads, both dense attention routes, unpadded, two fresh processes).
- Deterministic vs default: the same forward bits and loss; gradients within fp32 reordering (relative 1e-5).
- The default path launches none of the new kernels, also after the mode was switched on and off again.
- A workspace that is too small is refused through vb_last_error, naming the bytes, before anything is launched.

torch's own deterministic mode needs CUBLAS_WORKSPACE_CONFIG for the cuBLAS matmuls of the heads: the fixture below sets it.
"""
import ctypes
import os
import subprocess
import sys
import time

import pytest
import torch

from gemm_ref_util import check_close, tiles, wgrad_splits

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_KERNELS = ("splitk_reduce_kernel", "partials_reduce_kernel", "ln_bwd_part_kernel", "colsum_part_kernel", "embed_keys_kernel",
               "embed_vis_copy_kernel", "embed_seg_kernel", "embed_seg_join_kernel", "adam_sumsq_part_kernel",
               "adam_update_ordered_kernel", "DeviceRadixSort", ", 10>")


@pytest.fixture(autouse=True)
def _cublas_and_mode(monkeypatch):
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    yield
    torch.use_deterministic_algorithms(False)
    from visualbert_b200 import _lib
    _lib.lib().vb_set_deterministic(None, 0)


def _lib():
    from visualbert_b200 import _lib as L
    return L


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# torch.profiler can lose the kernel records nearest the edges of its capture window (the first kernel of a short window,
# or the whole of one): each counted window starts after the device is idle and leaves host time at both ends
PROFILE_PAD_S = 0.05


def _kernels(fn):
    """The names of the CUDA kernels fn launches, in launch order (copies and memsets left out)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        time.sleep(PROFILE_PAD_S)
        fn()
        torch.cuda.synchronize()
        time.sleep(PROFILE_PAD_S)
    out = []
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and "memset" not in e.name.lower() and "memcpy" not in e.name.lower():
            out.append(e.name)
    return out


class _Ws:
    """A deterministic-mode workspace filled with 0xFF bytes (a NaN pattern) and switched on for the calling thread."""

    def __init__(self, nbytes):
        self.t = torch.full((nbytes,), 255, device="cuda:0", dtype=torch.uint8)
        assert _lib().lib().vb_set_deterministic(self.t.data_ptr(), nbytes) == 0

    def tail_intact(self, used):
        return bool((self.t[used:] == 255).all())


def _guarded(rows, cols, dtype=torch.float32, fill=0.0):
    """[rows, cols] view with one NaN guard row above and below."""
    full = torch.full((rows + 2, cols), float("nan"), device="cuda:0", dtype=dtype)
    full[1:-1] = fill
    return full, full[1:-1]


def _guards_ok(full):
    return bool(torch.isnan(full[0]).all() and torch.isnan(full[-1]).all())


# ---------------------------------------------------------------------------------------------------------------------------
# op level
# ---------------------------------------------------------------------------------------------------------------------------
def _wgrad_call(dY, X, D, bias):
    from visualbert_b200 import ops
    Mr, N = dY.shape
    K = X.shape[1]
    ops._gemm(dY.device, A=dY.data_ptr(), lda=N, a_mn_major=1, B=X.data_ptr(), ldb=K, b_mn_major=1, M=N, N=K, K=Mr,
              D=D.data_ptr(), ldd=K, d_fp32=1, bias=0 if bias is None else bias.data_ptr())


@pytest.mark.parametrize("N,K,rows", [(3072, 768, 2000), (2304, 768, 2056), (768, 3072, 2000), (256, 272, 1412),
                                      (3000, 768, 2000), (296, 144, 1412)])   # the last two: M off the 128-row tile edge
def test_split_k_weight_gradient(N, K, rows):
    """dW[N, K] += dY^T X + bias through slabs: inside the fp64 bound, two calls bit-identical, guards and workspace tail intact."""
    g = torch.Generator(device="cuda:0").manual_seed(N + K)
    dY = torch.randn(rows, N, device="cuda:0", generator=g).to(torch.bfloat16)
    X = torch.randn(rows, K, device="cuda:0", generator=g).to(torch.bfloat16)
    bias = torch.randn(K, device="cuda:0", generator=g)
    D0 = torch.randn(N, K, device="cuda:0", generator=g)
    splits = wgrad_splits(tiles(N, K), (rows + 63) // 64, _sms())
    assert splits > 1, "the shape must split"
    used = splits * N * K * 4
    ws = _Ws(used + 4096)
    outs = []
    for _ in range(2):
        full, D = _guarded(N, K)
        D.copy_(D0)
        names = _kernels(lambda: _wgrad_call(dY, X, D, bias))
        assert any(", 10>" in n for n in names) and any("splitk_reduce_kernel" in n for n in names), names
        assert _guards_ok(full) and ws.tail_intact(used)
        outs.append(D.clone())
    assert torch.equal(outs[0], outs[1])
    a, b = dY.double(), X.double()
    ref = D0.double() + bias.double() + a.t() @ b
    mag = D0.double().abs() + bias.double().abs() + a.abs().t() @ b.abs()
    check_close(outs[0], ref, mag, False, f"deterministic split-K {N}x{K}x{rows}")
    # the same call with the mode off (red.add of the splits) agrees to fp32 reordering
    _lib().lib().vb_set_deterministic(None, 0)
    D = D0.clone()
    _wgrad_call(dY, X, D, bias)
    assert ((D - outs[0]).abs().max() / outs[0].abs().max()).item() <= 1e-5


def test_split_k_lowers_to_what_fits():
    """A workspace smaller than the slabs lowers the split factor (down to 1, the default single-writer kernel), still deterministic."""
    rows, N, K = 2000, 3072, 768
    g = torch.Generator(device="cuda:0").manual_seed(7)
    dY = torch.randn(rows, N, device="cuda:0", generator=g).to(torch.bfloat16)
    X = torch.randn(rows, K, device="cuda:0", generator=g).to(torch.bfloat16)
    _Ws(N * K * 4 + 256)   # room for one slab only: one split
    D1 = torch.zeros(N, K, device="cuda:0")
    names = _kernels(lambda: _wgrad_call(dY, X, D1, None))
    assert not any("splitk_reduce_kernel" in n for n in names), names
    D2 = torch.zeros(N, K, device="cuda:0")
    _wgrad_call(dY, X, D2, None)
    assert torch.equal(D1, D2)
    ref = dY.double().t() @ X.double()
    check_close(D1, ref, dY.double().abs().t() @ X.double().abs(), False, "one split")


def _ln_bwd(dy, x, gamma, dgamma, dbeta, dbias, dx):
    rows, H = x.shape
    mean = x.float().mean(1)
    rstd = torch.rsqrt(x.float().var(1, unbiased=False) + 1e-12)
    L = _lib().lib()
    rc = L.vb_layernorm_bwd(ctypes.c_void_p(dy.data_ptr()), ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(mean.data_ptr()),
                            ctypes.c_void_p(rstd.data_ptr()), ctypes.c_void_p(gamma.data_ptr()), ctypes.c_void_p(dx.data_ptr()), None,
                            ctypes.c_void_p(dgamma.data_ptr()), ctypes.c_void_p(dbeta.data_ptr()), ctypes.c_void_p(dbias.data_ptr()),
                            rows, H, ctypes.c_float(0.0), ctypes.c_uint64(0), ctypes.c_uint32(0), ctypes.c_float(0.0),
                            ctypes.c_uint32(0), _stream())
    _lib().check(rc, "vb_layernorm_bwd")
    return mean, rstd


@pytest.mark.parametrize("rows,H", [(41984, 768), (3001, 1024), (77, 256)])
def test_layernorm_backward_column_sums(rows, H):
    """dgamma / dbeta / dbias from per-block partials added in block order: |err| <= 2^-16 * sum |terms| against fp64, bits repeat."""
    g = torch.Generator(device="cuda:0").manual_seed(rows)
    x = torch.randn(rows, H, device="cuda:0", generator=g).to(torch.bfloat16)
    dy = torch.randn(rows, H, device="cuda:0", generator=g).to(torch.bfloat16)
    gamma = torch.randn(H, device="cuda:0", generator=g)
    used = min(2 * _sms(), (rows + 7) // 8) * 3 * H * 4
    ws = _Ws(used + 4096)
    res = []
    for _ in range(2):
        fulls = [_guarded(1, H, fill=0.5) for _ in range(3)]
        dx = torch.empty(rows, H, device="cuda:0", dtype=torch.bfloat16)
        names = _kernels(lambda: res.append(_ln_bwd(dy, x, gamma, fulls[0][1], fulls[1][1], fulls[2][1], dx)))
        assert any("ln_bwd_part_kernel" in n for n in names) and any("partials_reduce_kernel" in n for n in names), names
        assert all(_guards_ok(f) for f, _ in fulls) and ws.tail_intact(used)
        res[-1] = (res[-1], [v.clone() for _, v in fulls], dx.clone())
    (mean, rstd), (dg, db, dbias), dx = res[0]
    assert all(torch.equal(a, b) for a, b in zip(res[0][1], res[1][1])) and torch.equal(dx, res[1][2])
    xh = (x.double() - mean.double()[:, None]) * rstd.double()[:, None]
    d = dy.double()
    for got, terms, what in ((dg, d * xh, "dgamma"), (db, d, "dbeta"), (dbias, dx.double(), "dbias")):
        ref = 0.5 + terms.sum(0)
        err = (got[0].double() - ref).abs()
        bound = 2.0 ** -16 * (0.5 + terms.abs().sum(0)) + (2.0 ** -8 * d.abs().sum(0) if what == "dbias" else 0)
        assert bool((err <= bound).all()), f"{what}: worst {float((err / bound).max()):.3g} of the bound"


@pytest.mark.parametrize("M,N", [(41984, 3072), (41984, 2304), (5000, 30528), (9, 16)])
def test_colsum(M, N):
    g = torch.Generator(device="cuda:0").manual_seed(M + N)
    x = torch.randn(M, N, device="cuda:0", generator=g).to(torch.bfloat16)
    gx = (N // 8 + 31) // 32
    gy = min(max(_sms() * 6 // gx, 1), (M + 7) // 8)
    used = gy * N * 4
    ws = _Ws(used + 4096)
    L = _lib().lib()
    outs = []
    for _ in range(2):
        full, out = _guarded(1, N, fill=1.0)
        names = _kernels(lambda: _lib().check(L.vb_colsum_bf16(ctypes.c_void_p(x.data_ptr()), ctypes.c_int64(N), ctypes.c_void_p(out.data_ptr()),
                                                               M, N, _stream()), "vb_colsum_bf16"))
        assert any("colsum_part_kernel" in n for n in names) and any("partials_reduce_kernel" in n for n in names), names
        assert _guards_ok(full) and ws.tail_intact(used)
        outs.append(out.clone())
    assert torch.equal(outs[0], outs[1])
    ref = 1.0 + x.double().sum(0)
    assert bool(((outs[0][0].double() - ref).abs() <= 2.0 ** -16 * (1.0 + x.double().abs().sum(0))).all())


def test_bert_adam_norms_and_update():
    """Per-tensor norms from one partial per chunk, summed in chunk order: two runs bit-identical; the default (atomic) step agrees
    to fp32 rounding; the clip is active (the norms matter)."""
    from visualbert_b200 import BertAdam
    g = torch.Generator(device="cuda:0").manual_seed(3)
    shapes = [(30522, 768), (768,), (3072, 768), (5,)]
    p0 = [torch.randn(s, device="cuda:0", generator=g) for s in shapes]
    g0 = [torch.randn(s, device="cuda:0", generator=g) * 3 for s in shapes]

    def run(det):
        torch.use_deterministic_algorithms(det)
        ps = [torch.nn.Parameter(p.clone()) for p in p0]
        for p, gg in zip(ps, g0):
            p.grad = gg.clone()
        opt = BertAdam(ps, lr=1e-3, warmup=0.1, t_total=10, max_grad_norm=1.0)
        names = []
        for _ in range(2):
            names += _kernels(opt.step)
        torch.use_deterministic_algorithms(False)
        st = [opt.state[p] for p in ps]
        return [p.detach().clone() for p in ps], [s["next_m"].clone() for s in st], [s["next_v"].clone() for s in st], names

    a, b, ref = run(True), run(True), run(False)
    assert any("adam_update_ordered_kernel" in n for n in a[3]) and any("adam_sumsq_part_kernel" in n for n in a[3])
    assert not any(k in n for n in ref[3] for k in NEW_KERNELS)
    for i in range(3):
        assert all(torch.equal(x, y) for x, y in zip(a[i], b[i]))
        for x, y in zip(a[i], ref[i]):
            assert ((x - y).abs().max() / y.abs().max()).item() <= 1e-5
    assert not torch.equal(a[0][0], p0[0])


def test_embedding_backward_tables():
    """vb_embed_bwd in deterministic mode at the benchmark's row count, every table against fp64 sums of the d_pre the call wrote.
    Runs that cross many 64-item windows: text type 0 (~20k items), padding id 0 (~12k), visual position 0 (9216); repeated ids
    (CLS, SEP), out-of-range ids and types (clamped), three token types, regions. Bound per table row: recursive fp32 summation
    through at most 64 + ceil(count / 64) + 3 additions, (64 + ceil(count / 64) + 3) * 2^-24 * (|prefill| + sum |terms|)."""
    from visualbert_b200 import _lib as L_
    L = L_.lib()
    dev = "cuda:0"
    B, T, V, H, Dv, vocab, max_pos, nt = 256, 128, 36, 768, 64, 1000, 160, 3
    S, M = T + V, B * (T + V)
    g = torch.Generator().manual_seed(11)
    lens = torch.randint(T // 4, T + 1, (B,), generator=g)
    pos = torch.arange(T)
    ids = torch.randint(0, vocab, (B, T), generator=g)
    ids[:, 0] = 101
    ids[torch.arange(B), lens - 1] = 102
    ids[pos[None, :] >= lens[:, None]] = 0                    # padding
    ids[0, 3], ids[1, 3], ids[2, 3] = vocab + 7, -3, vocab      # clamped to vocab - 1, 0, vocab - 1
    tt = (pos[None, :] >= (lens[:, None] // 2)).long()
    tt[pos[None, :] >= lens[:, None]] = 0
    tt[:, 7] = 2
    tt[3, 9] = 9                                               # clamped to nt - 1
    vt = torch.randint(0, nt, (B, V), generator=g)
    vt[0, 0] = 17
    ids, tt, vt = ids.to(dev), tt.to(dev), vt.to(dev)
    pre = torch.randn(M, H, generator=g).to(dev).to(torch.bfloat16)
    mean = pre.float().mean(1)
    rstd = torch.rsqrt(pre.float().var(1, unbiased=False) + 1e-12)
    gamma = torch.randn(H, generator=g).to(dev)
    dy = torch.randn(M, H, generator=g).to(dev).to(torch.bfloat16)
    feats = torch.randn(B * V, Dv, generator=g).to(dev).to(torch.bfloat16)
    wproj = torch.randn(H, Dv, generator=g).to(dev).to(torch.bfloat16)
    shapes = dict(word=vocab, pos=max_pos, type=nt, pos_vis=max_pos, type_vis=nt)
    prefill = {k: torch.randn(n, H, generator=g).to(dev) for k, n in shapes.items()}
    nbytes = L.vb_deterministic_workspace_bytes(M, H, Dv, 0, 0)
    ws = _Ws(nbytes + 4096)

    def call():
        tabs = {k: _guarded(n, H) for k, n in shapes.items()}
        for k, (_, t) in tabs.items():
            t.copy_(prefill[k])
        o = dict(dgamma=torch.zeros(H, device=dev), dbeta=torch.zeros(H, device=dev), db_proj=torch.zeros(H, device=dev),
                 dw_proj=torch.zeros(H, Dv, device=dev), d_pre=torch.empty(M, H, device=dev, dtype=torch.bfloat16),
                 d_vis=torch.empty(B * V, H, device=dev, dtype=torch.bfloat16))
        d = L_.EmbedDesc(batch=B, text_len=T, num_regions=V, hidden=H, visual_dim=Dv, vocab=vocab, max_pos=max_pos, n_types=nt,
                         eps=1e-12, dropout=0.0, seed=0, input_ids=ids.data_ptr(), token_type_ids=tt.data_ptr(), visual_type=vt.data_ptr(),
                         visual_feats=feats.data_ptr(), w_proj=wproj.data_ptr(), b_proj=0, word=0, pos=0, type=0, pos_vis=0,
                         type_vis=0, gamma=gamma.data_ptr(), beta=0, visual_addend=0)
        a = L_.EmbedActs(vis_proj=0, pre=pre.data_ptr(), mean=mean.data_ptr(), rstd=rstd.data_ptr())
        gr = L_.EmbedGrads(dword=tabs["word"][1].data_ptr(), dpos=tabs["pos"][1].data_ptr(), dtype=tabs["type"][1].data_ptr(),
                           dpos_vis=tabs["pos_vis"][1].data_ptr(), dtype_vis=tabs["type_vis"][1].data_ptr(), dw_proj=o["dw_proj"].data_ptr(),
                           db_proj=o["db_proj"].data_ptr(), dgamma=o["dgamma"].data_ptr(), dbeta=o["dbeta"].data_ptr(),
                           d_pre=o["d_pre"].data_ptr(), d_vis=o["d_vis"].data_ptr(), d_feats=0)
        names = _kernels(lambda: L_.check(L.vb_embed_bwd(ctypes.byref(d), ctypes.byref(a), ctypes.c_void_p(dy.data_ptr()),
                                                         ctypes.byref(gr), _stream()), "vb_embed_bwd"))
        for k in ("embed_seg_kernel", "embed_seg_join_kernel", "DeviceRadixSort", "embed_keys_kernel", "ln_bwd_part_kernel"):
            assert any(k in n for n in names), (k, names)
        assert all(_guards_ok(f) for f, _ in tabs.values()) and ws.tail_intact(nbytes)
        o.update({k: t.clone() for k, (_, t) in tabs.items()})
        return o

    r1, r2 = call(), call()
    for k in r1:
        assert torch.equal(r1[k], r2[k]), k
    de = r1["d_pre"].double().view(B, S, H)
    txt, vis = de[:, :T].reshape(-1, H), de[:, T:].reshape(-1, H)

    def scatter(n, index, rows):
        ref = torch.zeros(n, H, device=dev, dtype=torch.float64).index_add_(0, index, rows)
        mag = torch.zeros(n, H, device=dev, dtype=torch.float64).index_add_(0, index, rows.abs())
        cnt = torch.zeros(n, device=dev, dtype=torch.float64).index_add_(0, index, torch.ones(len(index), device=dev, dtype=torch.float64))
        return ref, mag, cnt

    vpos = torch.zeros(B * V, device=dev, dtype=torch.long)
    cases = dict(word=scatter(vocab, ids.reshape(-1).clamp(0, vocab - 1), txt),
                 pos=scatter(max_pos, pos.to(dev).repeat(B), txt),
                 type=scatter(nt, tt.reshape(-1).clamp(0, nt - 1), txt),
                 pos_vis=scatter(max_pos, vpos, vis),
                 type_vis=scatter(nt, vt.reshape(-1).clamp(0, nt - 1), vis))
    assert cases["type"][2][0] > 150 * 64 and cases["word"][2][0] > 100 * 64 and cases["pos_vis"][2][0] == B * V
    for k, (ref, mag, cnt) in cases.items():
        p0 = prefill[k].double()
        depth = 64 + torch.ceil(cnt / 64)[:, None] + 3
        err = (r1[k].double() - (p0 + ref)).abs()
        bound = depth * 2.0 ** -24 * (p0.abs() + mag)
        assert bool((err <= bound).all()), f"{k}: worst {float((err / bound).max()):.3g} of the bound"
        assert torch.equal(r1[k][cnt == 0], prefill[k][cnt == 0]), k   # rows no item maps to are untouched
    assert torch.equal(r1["d_vis"], r1["d_pre"].view(B, S, H)[:, T:].reshape(-1, H))
    dv = r1["d_vis"].double()
    assert bool(((r1["db_proj"].double() - dv.sum(0)).abs() <= 2.0 ** -16 * dv.abs().sum(0)).all())
    check_close(r1["dw_proj"], dv.t() @ feats.double(), dv.abs().t() @ feats.double().abs(), False, "dw_proj")


def test_too_small_workspace_fails_before_launching():
    L = _lib().lib()
    x = torch.randn(4096, 3072, device="cuda:0").to(torch.bfloat16)
    out = torch.zeros(3072, device="cuda:0")
    ws = _Ws(256)
    n0 = _lib().launch_count()
    rc = L.vb_colsum_bf16(ctypes.c_void_p(x.data_ptr()), ctypes.c_int64(3072), ctypes.c_void_p(out.data_ptr()), 4096, 3072, _stream())
    msg = L.vb_last_error().decode()
    assert rc != 0 and "needs" in msg and "bytes" in msg, msg
    need = int(msg.split("needs ")[1].split(" ")[0])
    assert need > 256
    torch.cuda.synchronize()
    assert _lib().launch_count() == n0 and bool((out == 0).all()) and ws.tail_intact(0)
    # the training path sizes its workspace by vb_deterministic_workspace_bytes: this call fits in it
    assert L.vb_deterministic_workspace_bytes(4096, 768, 3072, 0, 0) >= need


# ---------------------------------------------------------------------------------------------------------------------------
# whole training steps
# ---------------------------------------------------------------------------------------------------------------------------
def _model(layers, hidden, heads, inter, B, T, V, head="pretraining", Dv=64, ragged=True, unpadded=False):
    from visualbert_b200 import BertConfig, TrainVisualBERTObjective, synthetic
    cfg = synthetic.bert_config_dict(layers, hidden, heads, inter, vocab=512)
    sd = synthetic.init_state_dict(cfg, head, Dv, seed=0)
    batch = synthetic.make_batch(B, T, V, Dv, head=head, seed=1234, vocab=512, ragged=ragged)
    batch = {k: (v.to("cuda:0") if torch.is_tensor(v) else v) for k, v in batch.items()}
    model = TrainVisualBERTObjective(BertConfig.from_dict(cfg), head, visual_embedding_dim=Dv)
    model.load_state_dict(sd, strict=False)
    model = model.to("cuda:0").train(True)
    if unpadded:
        model.bert.set_unpadded(True)
    return model, batch


def _train_steps(model, batch, det, state, opt_steps=2):
    """Loss, gradients of the first step, then parameters and Adam moments after `opt_steps` BertAdam steps."""
    from visualbert_b200 import BertAdam
    torch.use_deterministic_algorithms(det)
    try:
        torch.manual_seed(1234)   # the vqa / nlvr classifiers' nn.Dropout draws from torch's generator
        model.bert.set_dropout_state(state)
        init = {k: p.detach().clone() for k, p in model.named_parameters()}
        opt = BertAdam(model.parameters(), lr=1e-3, warmup=0.1, t_total=10, max_grad_norm=1.0)
        loss = grads = None
        enc = []
        hook = model.bert.encoder.register_forward_hook(lambda m, i, o: enc.append(o[-1].detach().clone()))
        for i in range(opt_steps):
            model.zero_grad(set_to_none=True)
            out = model(**batch)
            out["loss"].backward()
            if i == 0:
                loss = out["loss"].detach().clone()
                grads = {k: p.grad.detach().clone() for k, p in model.named_parameters() if p.grad is not None}
            opt.step()
        hook.remove()
        torch.cuda.synchronize()
        after = {k: p.detach().clone() for k, p in model.named_parameters()}
        moments = {k: (opt.state[p]["next_m"].clone(), opt.state[p]["next_v"].clone()) for k, p in model.named_parameters()
                   if p in opt.state}
        with torch.no_grad():   # restore the parameters for the next run
            for k, p in model.named_parameters():
                p.copy_(init[k])
        return loss, grads, after, moments, enc[0]
    finally:
        torch.use_deterministic_algorithms(False)


CASES = {
    # dense, S = 30 (wgmma attention), pretraining: MLM with the tied decoder + NSP
    "pretraining_s30": dict(args=(2, 256, 4, 1024, 8, 20, 10), kw=dict(head="pretraining")),
    # dense, S = 210 (whole-head attention), vqa head
    "vqa_s210": dict(args=(2, 128, 2, 512, 4, 150, 60), kw=dict(head="vqa")),
    # unpadded ragged batch
    "pretraining_unpadded": dict(args=(2, 256, 4, 1024, 6, 40, 16), kw=dict(head="pretraining", unpadded=True)),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_training_step_is_bitwise_reproducible(case):
    c = CASES[case]
    model, batch = _model(*c["args"], **c["kw"])
    state = model.bert.dropout_state()
    names = _kernels(lambda: _train_steps(model, batch, True, state, opt_steps=1))
    assert any("splitk_reduce_kernel" in n for n in names) and any("embed_seg_kernel" in n for n in names), names
    r1 = _train_steps(model, batch, True, state)
    r2 = _train_steps(model, batch, True, state)
    assert torch.isfinite(r1[0]) and torch.equal(r1[0], r2[0])
    assert r1[1].keys() == r2[1].keys() and len(r1[1]) > 20
    for k in r1[1]:
        assert torch.equal(r1[1][k], r2[1][k]), k
    for k in r1[2]:
        assert torch.equal(r1[2][k], r2[2][k]), k
    for k in r1[3]:
        assert torch.equal(r1[3][k][0], r2[3][k][0]) and torch.equal(r1[3][k][1], r2[3][k][1]), k
    # default mode: the same forward and loss bits, gradients within fp32 reordering
    r0 = _train_steps(model, batch, False, state, opt_steps=1)
    assert torch.equal(r0[0], r1[0]) and torch.equal(r0[4], r1[4]) and torch.equal(r1[4], r2[4])
    for k, g in r1[1].items():
        scale = g.abs().max().item()
        if scale == 0:
            assert torch.equal(g, r0[1][k]), k
            continue
        assert (r0[1][k] - g).abs().max().item() <= 1e-5 * scale, k


def test_layer_by_layer_route_is_bitwise_reproducible():
    """output_all_encoded_layers=True in training runs every layer as its own encoder call."""
    model, batch = _model(2, 256, 4, 1024, 8, 20, 10, head="pretraining")
    state = model.bert.dropout_state()
    L = len(model.bert.encoder.layer)

    def run():
        torch.use_deterministic_algorithms(True)
        try:
            model.bert.set_dropout_state(state)
            model.zero_grad(set_to_none=True)
            out = model(**batch)
            out["loss"].backward()
            return {k: p.grad.detach().clone() for k, p in model.named_parameters() if p.grad is not None}
        finally:
            torch.use_deterministic_algorithms(False)

    from visualbert_b200 import modeling
    orig = modeling.BertEncoder.forward

    def all_layers(self, hidden_states, attention_mask, output_all_encoded_layers=True, *a, **kw):
        return orig(self, hidden_states, attention_mask, True, *a, **kw)

    modeling.BertEncoder.forward = all_layers
    try:
        g1, g2 = run(), run()
    finally:
        modeling.BertEncoder.forward = orig
    assert L == 2 and len(g1) > 20
    for k in g1:
        assert torch.equal(g1[k], g2[k]), k


def test_default_path_launches_no_new_kernel():
    model, batch = _model(2, 256, 4, 1024, 8, 20, 10, head="pretraining")
    state = model.bert.dropout_state()
    _train_steps(model, batch, False, state, opt_steps=1)   # first-call work (weight banks, plans) out of the comparison
    before = _kernels(lambda: _train_steps(model, batch, False, state, opt_steps=1))
    assert not [n for n in before if any(k in n for k in NEW_KERNELS)]
    _train_steps(model, batch, True, state, opt_steps=1)
    after = _kernels(lambda: _train_steps(model, batch, False, state, opt_steps=1))
    assert after == before


_SUBPROCESS = r"""
import hashlib, sys, torch
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[2])
import test_deterministic_gpu as t
torch.manual_seed(0)   # the parameters the state dict does not cover, and the library's dropout seed (torch.initial_seed)
model, batch = t._model(2, 256, 4, 1024, 8, 20, 10, head="pretraining")
loss, grads, after, moments, _ = t._train_steps(model, batch, True, model.bert.dropout_state())
h = hashlib.sha256(loss.cpu().numpy().tobytes())
for k in sorted(grads): h.update(grads[k].cpu().numpy().tobytes())
for k in sorted(after): h.update(after[k].cpu().numpy().tobytes())
print("DIGEST", h.hexdigest())
"""


def test_two_fresh_processes_give_the_same_bits():
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    digests = []
    for _ in range(2):
        out = subprocess.run([sys.executable, "-c", _SUBPROCESS, ROOT, os.path.dirname(os.path.abspath(__file__))], env=env,
                             capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stderr[-3000:]
        digests.append([l for l in out.stdout.splitlines() if l.startswith("DIGEST")][0])
    assert digests[0] == digests[1]


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two visible GPUs")
def test_two_devices_give_the_same_gradients():
    from visualbert_b200 import BertConfig, TrainVisualBERTObjective, synthetic
    cfg = synthetic.bert_config_dict(2, 256, 4, 1024, vocab=512)
    sd = synthetic.init_state_dict(cfg, "pretraining", 64, seed=0)
    cpu_batch = synthetic.make_batch(8, 20, 10, 64, head="pretraining", seed=1234, vocab=512, ragged=True)
    grads = []
    for dev in ("cuda:0", "cuda:1"):
        model = TrainVisualBERTObjective(BertConfig.from_dict(cfg), "pretraining", visual_embedding_dim=64)
        model.load_state_dict(sd, strict=False)
        model = model.to(dev).train(True)
        batch = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in cpu_batch.items()}
        torch.use_deterministic_algorithms(True)
        try:
            with torch.cuda.device(dev):
                model(**batch)["loss"].backward()
                torch.cuda.synchronize()
        finally:
            torch.use_deterministic_algorithms(False)
        grads.append({k: p.grad.detach().cpu() for k, p in model.named_parameters() if p.grad is not None})
    for k in grads[0]:
        assert torch.equal(grads[0][k], grads[1][k]), k
