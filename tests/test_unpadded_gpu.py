"""Unpadded ("variable-length") execution: vb_attention_fwd_varlen / _bwd_varlen on every attention route against an fp64
restatement and against the dense kernels on the same data, and BertVisualModel.set_unpadded against the goldens, the oracle
and the padded path.

The attention route is chosen from max_seq as the dense call chooses it from seq. Every output of a varlen call (ctx, lse, drow,
dQ, dK, dV) must lie within the per-element bound of attn_ref_util.py of its fp64 reference, with unit-normal and with peaked
(Q x 4) rows."""
import ctypes
import math
import re

import numpy as np
import pytest
import torch

import attn_ref_util as R
import golden_util
import vb_oracle

pytestmark = pytest.mark.gpu

GUARD_ROWS, GUARD_FLAT, SENTINEL = 64, 256, -12345.0
P_DROP = 0.1

# length mixes: the maximum selects the route (wgmma <= 192, whole-head <= 256, staged above); 0 and 1 are the empty and the
# one-row sequence, the others sit on tile edges and route cut-overs
MIXES = [[0, 1, 63, 64, 65], [127, 128, 129, 1], [176, 177, 0, 191, 192], [193, 64, 0], [255, 256, 1, 100],
         [257, 100, 0], [356, 0, 17, 200], [513, 64, 129]]
CASES = ([(tuple(m), A, 0.0) for m in MIXES for A in (1, 12)]
         + [(tuple(m), 12, P_DROP) for m in MIXES[:2]])
PEAKED_CASES = [(tuple(m), 2, p) for m in MIXES for p in (0.0, P_DROP)]


def _setup():
    from visualbert_b200 import _lib
    return _lib, _lib.lib(), torch.device("cuda:0"), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


class _Guarded:
    def __init__(self, n, dtype, guard, fill, dev):
        self.n, self.guard, self.fill = n, guard, fill
        self.buf = torch.full((n + 2 * guard,), fill, dtype=dtype, device=dev)
        self.t = self.buf[guard:guard + n]

    def intact(self):
        g = torch.cat([self.buf[:self.guard], self.buf[self.guard + self.n:]])
        if self.fill != self.fill:
            return bool(torch.isnan(g).all())
        return torch.equal(g, torch.full_like(g, self.fill))


def _cu(lens, dev):
    cu = [0]
    for n in lens:
        cu.append(cu[-1] + n)
    return torch.tensor(cu, dtype=torch.int32, device=dev)


def _run_varlen(lens, A, p, qkv, dctx, seed=99, stream=5, guarded=True):
    """One varlen forward + backward; inputs in NaN-guarded buffers, outputs NaN-filled views in sentinel-guarded ones."""
    _lib, L, dev, st = _setup()
    H, B, total, S = A * 64, len(lens), sum(lens), max(lens)
    nan = float("nan")
    gr, gf = (GUARD_ROWS, GUARD_FLAT) if guarded else (0, 0)
    T = {"qkv": _Guarded(total * 3 * H, torch.bfloat16, gr * 3 * H, nan, dev),
         "dctx": _Guarded(total * H, torch.bfloat16, gr * H, nan, dev),
         "ctx": _Guarded(total * H, torch.bfloat16, gr * H, SENTINEL, dev),
         "lse": _Guarded(A * total, torch.float32, gf, SENTINEL, dev),
         "dqkv": _Guarded(total * 3 * H, torch.bfloat16, gr * 3 * H, SENTINEL, dev),
         "drow": _Guarded(A * total, torch.float32, gf, SENTINEL, dev)}
    T["qkv"].t.copy_(qkv.reshape(-1)); T["dctx"].t.copy_(dctx.reshape(-1))
    for k in ("ctx", "lse", "dqkv", "drow"):
        T[k].t.fill_(nan)
    keep = None
    if p > 0:
        keep = torch.zeros(int(L.vb_attention_keep_bytes(B, S, A)), dtype=torch.uint8, device=dev)
        T["keep"] = keep
    cu = _cu(lens, dev)
    args = (p, seed, stream, st)
    kp = keep.data_ptr() if keep is not None else None
    _lib.check(L.vb_attention_fwd_varlen(T["qkv"].t.data_ptr(), cu.data_ptr(), T["ctx"].t.data_ptr(), T["lse"].t.data_ptr(), kp,
                                         B, S, total, A, H, *args), "attn_fwd_varlen")
    _lib.check(L.vb_attention_bwd_varlen(T["qkv"].t.data_ptr(), cu.data_ptr(), T["ctx"].t.data_ptr(), T["lse"].t.data_ptr(), kp,
                                         T["dctx"].t.data_ptr(), T["dqkv"].t.data_ptr(), T["drow"].t.data_ptr(), B, S, total, A, H,
                                         *args), "attn_bwd_varlen")
    return T


def _keep_bits(keep, B, S, A):
    nkb = (S + 63) // 64
    words = keep.view(torch.int64).view(2, B * A, nkb * 64, nkb)[0]
    bits = (words.unsqueeze(-1) >> torch.arange(64, device=keep.device)) & 1
    return bits.reshape(B * A, nkb * 64, nkb * 64)


def _err(out, ref, scale=0.0):
    out, ref = out.double(), ref.double()
    return ((out - ref).abs().max() / max(ref.abs().max().item(), scale, 1e-30)).item()


def _inputs(lens, A, seed, peaked=False):
    """qkv and dO unit normal; `peaked`: Q x 4 (scores of std ~4)."""
    g = torch.Generator(device="cuda:0")
    g.manual_seed(seed)
    total, H = sum(lens), A * 64
    qkv = torch.randn(total, 3 * H, device="cuda:0", generator=g)
    dctx = torch.randn(total, H, device="cuda:0", generator=g).bfloat16()
    if peaked:
        qkv[:, :H] *= 4.0
    return qkv.bfloat16(), dctx


def _check_reference(lens, A, p, qkv, dctx, T, where):
    """Every output of one varlen call within the bound of attn_ref_util.py, sequence by sequence (no key bias; the keep bits
    of sequence b are the [:n, :n] corner of its heads' blocks). Returns the worst error / bound per output."""
    H, B, S, total = A * 64, len(lens), max(lens), sum(lens)
    bits = _keep_bits(T["keep"], B, S, A) if p > 0 else None
    ctx, dqkv = T["ctx"].t.view(total, H), T["dqkv"].t.view(total, 3 * H)
    lse, drow = T["lse"].t.view(A, total), T["drow"].t.view(A, total)
    outs, refs, bounds, r = {}, {}, {}, 0
    for b, n in enumerate(lens):
        if n == 0:
            continue
        q, k, v = R.varlen_heads(qkv, r, n, A)
        dO, c = R.varlen_heads(dctx, r, n, A)[0], R.varlen_heads(ctx, r, n, A)[0]
        keep = bits[b * A:(b + 1) * A, :n, :n] if p > 0 else None
        ref = R.reference(q, k, v, None, keep, R.drop_scale(p), dO, c)
        dq, dk, dv = R.varlen_heads(dqkv, r, n, A)
        out = dict(ctx=c, lse=lse[:, r:r + n], drow=drow[:, r:r + n], dq=dq, dk=dk, dv=dv)
        for name, o in out.items():
            outs.setdefault(name, []).append(o)
            refs.setdefault(name, []).append(ref[name][0])
            bounds.setdefault(name, []).append(ref[name][1])
        r += n
    cat = lambda xs: torch.cat(xs, 1)
    worst = {name: R.check(cat(outs[name]), cat(refs[name]), cat(bounds[name]), f"{where}: {name}") for name in outs}
    print(f"{where}: worst error / bound " + ", ".join(f"{n} {w:.3f}" for n, w in worst.items()))
    return worst


def _check(lens, A, p, seed, peaked=False):
    where = f"lens={list(lens)} A={A} p={p}" + (" peaked" if peaked else "")
    qkv, dctx = _inputs(lens, A, seed, peaked)
    T = _run_varlen(lens, A, p, qkv, dctx)
    T2 = _run_varlen(lens, A, p, qkv, dctx, guarded=False)
    torch.cuda.synchronize()
    for k in ("ctx", "lse", "dqkv", "drow"):
        assert torch.isfinite(T[k].t).all(), f"{where}: {k} has unwritten (NaN) elements"
        assert torch.equal(T[k].t, T2[k].t), f"{where}: {k} differs between two identical calls"
    for k, gt in T.items():
        if k != "keep":
            assert gt.intact(), f"{where}: guard band of {k} changed"
    if sum(lens) == 0:
        return
    _check_reference(lens, A, p, qkv, dctx, T, where)


@pytest.mark.parametrize("lens,A,p", CASES)
def test_varlen_attention_matches_reference(lens, A, p):
    _check(lens, A, p, seed=sum(lens) * 7 + A)


@pytest.mark.parametrize("lens,A,p", PEAKED_CASES)
def test_varlen_attention_peaked(lens, A, p):
    """Scores of std ~4: the row maximum moves between key blocks, so the online-softmax rescales of the whole-head and staged
    kernels carry weight."""
    _check(lens, A, p, seed=sum(lens) * 11 + A, peaked=True)


def test_varlen_attention_many_heads():
    """B * A = 7 * 40 = 280 heads, more than twice the SM count: persistent whole-head CTAs walk several sequences."""
    g = torch.Generator().manual_seed(3)
    lens = [int(x) for x in torch.randint(0, 201, (40,), generator=g)]
    lens[0] = 200
    _check(tuple(lens), 7, 0.0, seed=11)


@pytest.mark.parametrize("lens", [(100, 37, 1, 64), (200, 150, 3), (356, 300, 17)])
def test_varlen_matches_dense_on_same_data(lens):
    """The dense kernels with a -10000 key mask on padded rows and the varlen kernels on the packed rows agree on every valid
    row (the masked keys get exactly zero probability in fp32)."""
    _lib, L, dev, st = _setup()
    A, B, S = 2, len(lens), max(lens)
    H = A * 64
    qkv, dctx = _inputs(lens, A, seed=5)
    T = _run_varlen(lens, A, 0.0, qkv, dctx, guarded=False)
    idx = torch.cat([torch.arange(n, device=dev) + b * S for b, n in enumerate(lens)])
    dq = torch.zeros(B * S, 3 * H, device=dev, dtype=torch.bfloat16).index_copy(0, idx, qkv)
    dd = torch.zeros(B * S, H, device=dev, dtype=torch.bfloat16).index_copy(0, idx, dctx)
    bias = torch.full((B, S), -10000.0, device=dev)
    for b, n in enumerate(lens):
        bias[b, :n] = 0.0
    ctx = torch.empty(B * S, H, device=dev, dtype=torch.bfloat16)
    lse = torch.empty(B, A, S, device=dev)
    dqkv = torch.empty(B * S, 3 * H, device=dev, dtype=torch.bfloat16)
    drow = torch.empty(B, A, S, device=dev)
    _lib.check(L.vb_attention_fwd(ctypes.c_void_p(dq.data_ptr()), ctypes.c_void_p(bias.data_ptr()), ctypes.c_void_p(ctx.data_ptr()),
                                  ctypes.c_void_p(lse.data_ptr()), None, B, S, A, H, ctypes.c_float(0.0), ctypes.c_uint64(1), 0, st), "fwd")
    _lib.check(L.vb_attention_bwd(ctypes.c_void_p(dq.data_ptr()), ctypes.c_void_p(bias.data_ptr()), ctypes.c_void_p(ctx.data_ptr()),
                                  ctypes.c_void_p(lse.data_ptr()), None, ctypes.c_void_p(dd.data_ptr()), ctypes.c_void_p(dqkv.data_ptr()),
                                  ctypes.c_void_p(drow.data_ptr()), B, S, A, H, ctypes.c_float(0.0), ctypes.c_uint64(1), 0, st), "bwd")
    torch.cuda.synchronize()
    total = sum(lens)
    vctx, vd = T["ctx"].t.view(total, H), T["dqkv"].t.view(total, 3 * H)
    e_ctx, e_d = _err(vctx, ctx[idx]), _err(vd, dqkv[idx])
    lse_d = torch.cat([lse[b, :, :n] for b, n in enumerate(lens)], 1)
    e_lse = (T["lse"].t.view(A, total) - lse_d).abs().max().item()
    print(f"lens={lens}: max rel diff ctx {e_ctx:.3g}, dqkv {e_d:.3g}, abs lse {e_lse:.3g}")
    # the two calls run the same kernels on the same rows; they differ only where the dense call's tiles hold padded keys
    assert e_ctx < 1e-2 and e_d < 2e-2 and e_lse < 2e-2


@pytest.mark.parametrize("S,want", [(100, "wgmma"), (200, "head"), (356, "staged")])
def test_varlen_routing(S, want):
    from torch.profiler import ProfilerActivity, profile
    lens, A = (S, S // 2, 0), 2
    qkv, dctx = _inputs(lens, A, seed=S)
    _run_varlen(lens, A, P_DROP, qkv, dctx)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        _run_varlen(lens, A, P_DROP, qkv, dctx)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    if not names:
        pytest.skip("torch.profiler recorded no device kernels")
    ran = {m.group(1) for n in names for m in [re.search(r"\b(attn_\w+_kernel)\b", n)] if m}
    fam = {"wgmma": {"attn_keep_mask_kernel", "attn_fwd_wgmma_kernel", "attn_delta_kernel", "attn_bwd_wgmma_kernel"},
           "head": {"attn_keep_mask_kernel", "attn_fwd_head_kernel", "attn_delta_kernel", "attn_bwd_head_kernel"},
           "staged": {"attn_fwd_kernel", "attn_bwd_dq_kernel", "attn_bwd_dkv_kernel"}}[want]
    assert ran == fam, f"S={S}: expected {sorted(fam)}, ran {sorted(ran)}"


# ------------------------------------------------------------------------------------------------------------------------
# model level
# ------------------------------------------------------------------------------------------------------------------------
MODEL_CASES = ["small_ragged_pretraining", "base3_ragged_pretraining", "small_vqa", "small_nlvr", "small_multichoice",
               "small_vcr_alignment"]
LOSS_RTOL, ACT_TOL, GRAD_COS, GRAD_NORM = 1e-2, 5e-2, 0.99, 0.06


def _model(cfg, c, sd, train=False):
    from visualbert_b200 import BertConfig, TrainVisualBERTObjective
    model = TrainVisualBERTObjective(BertConfig.from_dict(cfg), c["head"], visual_embedding_dim=c["Dv"], **c.get("flags", {}))
    model.load_state_dict(sd, strict=False)
    return model.to("cuda:0").train(train)


def _valid(batch):
    im = batch["input_mask"].reshape(-1, batch["input_mask"].shape[-1])
    vm = batch.get("image_mask")
    if vm is not None:
        im = torch.cat((im, vm.reshape(-1, vm.shape[-1])), 1)
    return im != 0


def _grads(model):
    return {k: p.grad.detach().float().clone() for k, p in model.named_parameters() if p.grad is not None}


def _run_model(model, batch):
    model.zero_grad(set_to_none=True)
    out = model(**batch)
    enc = model(**{**batch, "output_all_encoded_layers": True})
    out["loss"].backward()
    return out, enc, _grads(model)


@pytest.mark.parametrize("name", MODEL_CASES)
def test_unpadded_model_parity(name):
    cfg, sd, batch, c, gold = golden_util.load(name)
    dev = torch.device("cuda:0")
    batch = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in batch.items()}
    sd = {k: v.to(dev) for k, v in sd.items()}
    model = _model(cfg, c, sd)
    out_p, enc_p, g_p = _run_model(model, batch)
    model.bert.set_unpadded(True)
    out_u, enc_u, g_u = _run_model(model, batch)
    valid = _valid(batch)
    loss_u, loss_p = out_u["loss"].item(), out_p["loss"].item()
    # against the golden and the oracle (the tolerances of test_model_gpu.test_forward_backward_parity)
    assert abs(loss_u - float(gold["loss"])) <= LOSS_RTOL * abs(float(gold["loss"]))
    sdo = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    ref = vb_oracle.objective(sdo, cfg, c["head"], **{k: v for k, v in batch.items() if k != "position_embeddings_visual"})
    assert abs(loss_u - ref["loss"].item()) <= LOSS_RTOL * abs(ref["loss"].item())
    last_u, last_p = enc_u["sequence_output"][-1].float(), enc_p["sequence_output"][-1].float()
    ref_last = ref["sequence_output"].detach().float()
    assert ((last_u - ref_last)[valid].abs().max() / ref_last[valid].abs().max()).item() < ACT_TOL
    assert (last_u[~valid] == 0).all(), "masked rows must be zero"
    if valid[:, 0].all():
        pooled = enc_u["pooled_output"].float().detach().cpu().numpy()
        assert np.abs(pooled - gold["pooled"]).max() / max(np.abs(gold["pooled"]).max(), 1e-12) < ACT_TOL
    # the same arithmetic in torch bf16: the noise floor for ill-conditioned gradients (as in test_forward_backward_parity)
    sdb = {k: v.bfloat16().clone().requires_grad_(True) for k, v in sd.items()}
    kwb = {k: (v.bfloat16() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in batch.items()
           if k != "position_embeddings_visual"}
    refb = vb_oracle.objective(sdb, cfg, c["head"], **kwb)
    ref["loss"].backward()
    refb["loss"].float().backward()
    big = max(g.norm().item() for g in g_u.values())
    for k, a in g_u.items():
        if k == "cls.predictions.decoder.weight" or sdo.get(k) is None or sdo[k].grad is None:
            continue
        b = sdo[k].grad.float().reshape(-1)
        nb = b.norm().item()
        if nb < 1e-3 * big:
            continue
        a = a.reshape(-1)
        cos = torch.dot(a, b).item() / max(a.norm().item() * nb, 1e-30)
        err, err_bf16 = (a - b).norm().item(), (sdb[k].grad.float().reshape(-1) - b).norm().item()
        assert (cos >= GRAD_COS and abs(a.norm().item() / nb - 1) <= GRAD_NORM) or err <= err_bf16, f"{k}: cos {cos:.5f}"
    # against the padded path on the same model and batch
    assert abs(loss_u - loss_p) <= 1e-3 * abs(loss_p), (loss_u, loss_p)
    for lu, lp in zip(enc_u["sequence_output"], enc_p["sequence_output"]):
        lu, lp = lu.float(), lp.float()
        assert ((lu - lp)[valid].abs().max() / lp[valid].abs().max()).item() < 1e-2
    for k, a in g_u.items():
        b = g_p[k]
        if b.norm().item() < 1e-3 * big:
            continue
        cos = torch.dot(a.reshape(-1), b.reshape(-1)).item() / max(a.norm().item() * b.norm().item(), 1e-30)
        assert cos >= 0.999, f"{k}: unpadded vs padded gradient cosine {cos:.5f}"


def _synthetic_model(layers, hidden, heads, inter, B, T, V, Dv=64, head="pretraining", ragged=True, seed=1234, train=False):
    from visualbert_b200 import synthetic
    cfg = synthetic.bert_config_dict(layers, hidden, heads, inter, vocab=512)
    sd = synthetic.init_state_dict(cfg, head, Dv, seed=0)
    batch = synthetic.make_batch(B, T, V, Dv, head=head, seed=seed, vocab=512, ragged=ragged)
    batch = {k: (v.to("cuda:0") if torch.is_tensor(v) else v) for k, v in batch.items()}
    return _model(cfg, dict(head=head, Dv=Dv), sd, train), batch


def _compare_padded(model, batch, tol_loss=1e-3, tol_act=1e-2, tol_cos=0.999):
    model.bert.set_unpadded(False)
    out_p, enc_p, g_p = _run_model(model, batch)
    model.bert.set_unpadded(True)
    out_u, enc_u, g_u = _run_model(model, batch)
    valid = _valid(batch)
    assert abs(out_u["loss"].item() - out_p["loss"].item()) <= tol_loss * abs(out_p["loss"].item())
    lu, lp = enc_u["sequence_output"][-1].float(), enc_p["sequence_output"][-1].float()
    e_act = ((lu - lp)[valid].abs().max() / lp[valid].abs().max()).item()
    print(f"unpadded vs padded: loss {out_u['loss'].item():.6f} / {out_p['loss'].item():.6f}, last layer valid rows {e_act:.3g} of max")
    assert e_act < tol_act
    big = max(g.norm().item() for g in g_p.values())
    for k, a in g_u.items():
        b = g_p[k]
        if b.norm().item() < 1e-3 * big:
            continue
        cos = torch.dot(a.reshape(-1), b.reshape(-1)).item() / max(a.norm().item() * b.norm().item(), 1e-30)
        assert cos >= tol_cos, f"{k}: cosine {cos:.5f}"
    return out_u, enc_u, valid


def test_unpadded_full_depth():
    """12 layers, H = 768, S = 164 (128 text + 36 regions), ragged B = 16, eval mode. Both paths compute in bf16 and differ in
    accumulation order (packed region keys sit at other tile columns than padded ones), and the difference grows over 12 layers.
    The bounds are those of the smaller models (1e-2 of max for the last layer's valid rows, gradient cosine 0.999) or, where
    the two paths differ by more, the bf16 noise floor measured here: the unpadded-padded difference must not exceed the
    padded path's own error against the fp32 oracle on the same weights and batch."""
    from visualbert_b200 import synthetic
    model, batch = _synthetic_model(12, 768, 12, 3072, 16, 128, 36)
    cfg = synthetic.bert_config_dict(12, 768, 12, 3072, vocab=512)
    sd = {k: v.to("cuda:0").requires_grad_(True) for k, v in synthetic.init_state_dict(cfg, "pretraining", 64, seed=0).items()}
    model.bert.set_unpadded(False)
    out_p, enc_p, g_p = _run_model(model, batch)
    model.bert.set_unpadded(True)
    out_u, enc_u, g_u = _run_model(model, batch)
    ref = vb_oracle.objective(sd, cfg, "pretraining", **{k: v for k, v in batch.items() if k != "position_embeddings_visual"})
    ref["loss"].backward()
    valid = _valid(batch)
    lp, lu = out_p["loss"].item(), out_u["loss"].item()
    assert abs(lu - lp) <= 1e-3 * abs(lp), (lu, lp)
    hu, hp = enc_u["sequence_output"][-1].float(), enc_p["sequence_output"][-1].float()
    hr = ref["sequence_output"].detach().float()
    e_up = ((hu - hp)[valid].abs().max() / hp[valid].abs().max()).item()
    e_pr = ((hp - hr)[valid].abs().max() / hr[valid].abs().max()).item()
    print(f"full depth: loss {lu:.6f} / {lp:.6f} (oracle {ref['loss'].item():.6f}); last layer valid rows: unpadded-padded "
          f"{e_up:.3g}, padded-oracle {e_pr:.3g} of max")
    assert e_up <= max(1e-2, e_pr), (e_up, e_pr)
    big = max(g.norm().item() for g in g_p.values())
    worst = (1.0, "")
    for k, a in g_u.items():
        b = g_p[k]
        if k == "cls.predictions.decoder.weight" or b.norm().item() < 1e-3 * big:
            continue
        a, b = a.reshape(-1), b.reshape(-1)
        cos = torch.dot(a, b).item() / max(a.norm().item() * b.norm().item(), 1e-30)
        d_up = (a - b).norm().item()
        d_pr = (b - sd[k].grad.float().reshape(-1)).norm().item()
        worst = min(worst, (cos, f"{k}: cosine {cos:.5f}, |u - p| {d_up:.3g}, |p - oracle| {d_pr:.3g}"))
        assert cos >= 0.999 or d_up <= d_pr, f"{k}: unpadded-padded cosine {cos:.5f}, |u - p| {d_up:.3g} > |p - oracle| {d_pr:.3g}"
    print("full depth, lowest gradient cosine unpadded-padded:", worst[1])


def test_unpadded_edges():
    # an example with an all-zero mask: finite, zero rows, the other examples unchanged
    model, batch = _synthetic_model(2, 128, 2, 512, 4, 20, 6)
    out_u, enc_u, valid = _compare_padded(model, batch)
    b2 = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in batch.items()}
    b2["input_mask"][1] = 0
    b2["image_mask"][1] = 0
    with torch.no_grad():
        e2 = model(**{**b2, "output_all_encoded_layers": True})["sequence_output"][-1].float()
    assert torch.isfinite(e2).all() and (e2[1] == 0).all()
    last = enc_u["sequence_output"][-1].float()
    keep = valid.clone()
    keep[1] = False
    assert ((e2 - last)[keep].abs().max() / last[keep].abs().max()).item() < 1e-2
    # an example without regions, B = 1, and a batch without padding (which must match the padded path)
    model, batch = _synthetic_model(2, 128, 2, 512, 3, 20, 6)
    batch["image_mask"][0] = 0
    _compare_padded(model, batch)
    model, batch = _synthetic_model(2, 128, 2, 512, 1, 20, 6)
    _compare_padded(model, batch)
    model, batch = _synthetic_model(2, 128, 2, 512, 4, 20, 6, ragged=False)
    _compare_padded(model, batch)


def test_unpadded_forbidden_combinations_raise():
    from visualbert_b200 import BertConfig, TrainVisualBERTObjective, synthetic
    cfg = synthetic.bert_config_dict(1, 128, 2, 512, vocab=64)
    for flags in ({"bypass_transformer": True}, {"output_attention_weights": True}):
        m = TrainVisualBERTObjective(BertConfig.from_dict(cfg), "nlvr", visual_embedding_dim=64, **flags)
        with pytest.raises(ValueError):
            m.bert.set_unpadded(True)
    model, batch = _synthetic_model(1, 128, 2, 512, 2, 8, 3, train=True)
    model.bert.set_unpadded(True)
    with pytest.raises(ValueError):
        model(**{**batch, "output_all_encoded_layers": True})


def test_unpadded_train_mode_reproducible():
    """Dropout is active in the unpadded training step, the same seed and state reproduce the forward bit for bit, and
    everything stays finite. (Gradients are reproduced to rounding only: split-K weight gradients accumulate with fp32 atomics
    in either path.)"""
    model, batch = _synthetic_model(2, 256, 4, 1024, 6, 24, 8, train=True)
    model.bert.set_unpadded(True)
    state = model.bert.dropout_state()

    def step():
        model.zero_grad(set_to_none=True)
        out = model(**batch)
        out["loss"].backward()
        return out["loss"].detach().clone(), _grads(model)

    l1, g1 = step()
    l2, g2 = step()
    assert torch.isfinite(l1) and all(torch.isfinite(g).all() for g in g1.values())
    assert not torch.equal(l1, l2), "dropout masks did not change between steps"
    model.bert.set_dropout_state(state)
    l3, g3 = step()
    assert torch.equal(l1, l3)
    for k in g1:
        assert torch.allclose(g1[k], g3[k], rtol=1e-3, atol=1e-3 * g1[k].abs().max().item()), k
    model.eval()
    with torch.no_grad():
        e1 = model(**batch)["loss"]
    assert not torch.equal(e1, l1)


@pytest.mark.parametrize("lens,A,layer_index", [
    ((40, 0, 97, 63), 4, 0),        # total 200 < 256: D from attn_delta_kernel, row-major gelu'; wgmma attention
    ((190, 66, 0, 128), 4, 1),      # total 384: D from the EPI_DELTA epilogue (needs M, H >= 256); wgmma attention
    ((164, 120, 1, 227), 4, 3),     # total 512: EPI_DELTA, tile-native gelu' (M % 256 == 0); whole-head attention
    ((300, 17, 150, 0), 2, 11),     # total 467: staged attention (computes D itself), row-major gelu'
])
def test_varlen_layer_train_mode_matches_reference_math_with_the_same_masks(lens, A, layer_index):
    """One layer through vb_encoder_fwd_varlen / _bwd_varlen with hidden and attention dropout on, against the reference
    arithmetic (M.py:231-341) in fp32 with THE SAME masks: the hidden-state masks are regenerated with the hash restatement of
    dropout_util.py over the packed [total, H] tensors, the attention bits are read back from the arena's keep buffer,
    and attention runs per sequence. Checks the layer output, the input gradient and every parameter gradient."""
    from dropout_util import hidden_keep
    from visualbert_b200 import _lib
    L = _lib.lib()
    dev = torch.device("cuda:0")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    torch.manual_seed(29 + layer_index)
    B, S, total = len(lens), max(lens), sum(lens)
    H, I = A * 64, A * 256
    p_h, p_a, seed = 0.1, 0.1, 0x0FEDCBA987654321
    bf, f32 = torch.bfloat16, torch.float32
    rnd = lambda *s, sc=1.0: sc * torch.randn(*s, device=dev)
    x = rnd(total, H).to(bf)
    W = dict(qkv=rnd(3 * H, H, sc=0.05).to(bf), o=rnd(H, H, sc=0.05).to(bf), i=rnd(I, H, sc=0.05).to(bf), out=rnd(H, I, sc=0.05).to(bf))
    bvec = dict(qkv=rnd(3 * H, sc=0.1), o=rnd(H, sc=0.1), i=rnd(I, sc=0.1), out=rnd(H, sc=0.1))
    ln = dict(g1=1 + rnd(H, sc=0.1), b1=rnd(H, sc=0.1), g2=1 + rnd(H, sc=0.1), b2=rnd(H, sc=0.1))
    cu = _cu(lens, dev)

    # ---- the library: one-layer encoder, forward + backward ----
    off = (ctypes.c_int64 * _lib.VB_ENCODER_ARENA_BUFFERS)()
    stride = int(L.vb_encoder_arena_layout_varlen(B, S, total, H, A, I, 1, off))
    assert stride > 0
    arena = torch.empty(stride, device=dev, dtype=torch.uint8)
    d = (_lib.LayerDesc * 1)()
    d[0] = _lib.LayerDesc(batch=B, seq=S, hidden=H, heads=A, inter=I, hidden_dropout=p_h, attn_dropout=p_a, seed=seed,
                          layer_index=layer_index, w_qkv=W["qkv"].data_ptr(), w_attn_out=W["o"].data_ptr(),
                          w_inter=W["i"].data_ptr(), w_out=W["out"].data_ptr(), b_qkv=bvec["qkv"].data_ptr(),
                          b_attn_out=bvec["o"].data_ptr(), ln1_gamma=ln["g1"].data_ptr(), ln1_beta=ln["b1"].data_ptr(),
                          b_inter=bvec["i"].data_ptr(), b_out=bvec["out"].data_ptr(), ln2_gamma=ln["g2"].data_ptr(),
                          ln2_beta=ln["b2"].data_ptr(), mask_bias=0)
    _lib.check(L.vb_encoder_fwd_varlen(d, 1, cu.data_ptr(), total, x.data_ptr(), arena.data_ptr(), st), "fwd_varlen")
    y = arena[off[13]: off[13] + total * H * 2].view(bf).view(total, H)
    dy = rnd(total, H).to(bf)
    z = lambda *s: torch.zeros(*s, device=dev, dtype=f32)
    e = lambda *s, dt=bf: torch.empty(*s, device=dev, dtype=dt)
    G = dict(dw_qkv=z(3 * H, H), db_qkv=z(3 * H), dw_attn_out=z(H, H), db_attn_out=z(H), dln1_gamma=z(H), dln1_beta=z(H),
             dw_inter=z(I, H), db_inter=z(I), dw_out=z(H, I), db_out=z(H), dln2_gamma=z(H), dln2_beta=z(H))
    sc = dict(d_pre=e(total, H), d_pre_drop=e(total, H), d_big=e(total, max(I, 3 * H)), d_x1=e(total, H), d_ctx=e(total, H),
              drow=e(A, total, dt=f32))
    dx = e(total, H)
    g_ = (_lib.LayerGrads * 1)()
    g_[0] = _lib.LayerGrads(**{k: t.data_ptr() for k, t in G.items()})
    s_ = _lib.LayerScratch(**{k: t.data_ptr() for k, t in sc.items()})
    _lib.check(L.vb_encoder_bwd_varlen(d, 1, cu.data_ptr(), total, x.data_ptr(), arena.data_ptr(), dy.data_ptr(), dx.data_ptr(),
                                       g_, ctypes.addressof(s_), st), "bwd_varlen")
    torch.cuda.synchronize()

    # ---- the same masks ----
    nkb = (S + 63) // 64
    keep = arena[off[12]: off[12] + int(L.vb_attention_keep_bytes(B, S, A))]
    bits = _keep_bits(keep, B, S, A)
    n_a = int(p_a * 256.0 + 0.5)
    s_a = 256.0 / (256.0 - n_a)
    k1, s1 = hidden_keep(seed, layer_index * 8 + 1, total, H, p_h, dev)
    k2, s2 = hidden_keep(seed, layer_index * 8 + 2, total, H, p_h, dev)
    assert abs(k1.float().mean().item() - (1 - 26 / 256)) < 1e-2
    valid_bits = torch.cat([bits[b * A:(b + 1) * A, :n, :n].reshape(-1) for b, n in enumerate(lens) if n > 0]).float()
    assert abs(valid_bits.mean().item() - (1 - n_a / 256.0)) < 1e-2

    # ---- reference math, fp32, bf16-rounded weights, the library's masks, attention per sequence ----
    P = {k: v.float().requires_grad_(True) for k, v in W.items()}
    Bv = {k: v.clone().requires_grad_(True) for k, v in bvec.items()}
    Ln = {k: v.clone().requires_grad_(True) for k, v in ln.items()}
    xr = x.float().requires_grad_(True)

    def lnorm(t, g, b):
        u = t.mean(-1, keepdim=True)
        v = (t - u).pow(2).mean(-1, keepdim=True)
        return g * ((t - u) / torch.sqrt(v + 1e-12)) + b

    qkv = xr @ P["qkv"].t() + Bv["qkv"]
    parts, r = [], 0
    for b, n in enumerate(lens):
        q, k, v = qkv[r:r + n].view(n, 3, A, 64).permute(1, 2, 0, 3)
        probs = torch.softmax(q @ k.transpose(-1, -2) / 8.0, -1) * bits[b * A:(b + 1) * A, :n, :n].float() * s_a
        parts.append((probs @ v).permute(1, 0, 2).reshape(n, H))
        r += n
    ctx = torch.cat(parts)
    x1 = lnorm((ctx @ P["o"].t() + Bv["o"]) * k1.float() * s1 + xr, Ln["g1"], Ln["b1"])
    u = x1 @ P["i"].t() + Bv["i"]
    h = u * 0.5 * (1.0 + torch.erf(u / math.sqrt(2.0)))
    yr = lnorm((h @ P["out"].t() + Bv["out"]) * k2.float() * s2 + x1, Ln["g2"], Ln["b2"])
    yr.backward(dy.float())

    def rel(a_, b_):
        return ((a_.float() - b_.float()).abs().max() / b_.float().abs().max().clamp_min(1e-9)).item()

    def relnorm(a_, b_):
        return ((a_.float() - b_.float()).norm() / b_.float().norm().clamp_min(1e-12)).item()

    where = f"lens={lens}"
    assert torch.isfinite(y).all() and torch.isfinite(dx).all()
    assert rel(y, yr) < 2.5e-2, f"{where}: layer output {rel(y, yr)}"
    assert relnorm(dx, xr.grad) < 2.5e-2, f"{where}: dx {relnorm(dx, xr.grad)}"
    pairs = [("dw_qkv", P["qkv"]), ("db_qkv", Bv["qkv"]), ("dw_attn_out", P["o"]), ("db_attn_out", Bv["o"]),
             ("dln1_gamma", Ln["g1"]), ("dln1_beta", Ln["b1"]), ("dw_inter", P["i"]), ("db_inter", Bv["i"]),
             ("dw_out", P["out"]), ("db_out", Bv["out"]), ("dln2_gamma", Ln["g2"]), ("dln2_beta", Ln["b2"])]
    for name, ref in pairs:
        rr = relnorm(G[name], ref.grad)
        assert rr < 2.5e-2, f"{where}: {name} relative gradient error {rr}"
