"""The row kernels of the training step against an fp64 reference, element by element: LayerNorm forward and backward,
embedding forward and backward, the column sum, the cross-entropy and the casts.

Every call runs through the C ABI (ctypes) on the current stream with the library in its default mode (no deterministic workspace,
no dropout offset). The references and bounds are those of rowop_ref_util.py. Every output lives inside a larger allocation whose
bands (rows before and after, columns past the row's width) hold a NaN bit pattern that must survive the call; bf16 outputs are
prefilled with the same pattern, so an element the kernel skips shows up; accumulating fp32 outputs are prefilled with random values
and must come back as prefill + result. Dropout masks come from dropout_util.hidden_keep and are checked bit for bit: dropped
elements are exact +0. torch.profiler records the kernels each test launched, and they must be the instances each case was chosen
to reach (ln_fwd_kernel<1, 2, 3, 4, 8>, ln_bwd_kernel<1..4>, embed_fwd_kernel / embed_bwd_kernel<1, 4>, ...).

No call here passes a misaligned pointer or stride; those refusals are checked without a GPU in test_abi.py.
"""
import ctypes
import json
import re
import time

import numpy as np
import pytest
import torch

import rowop_ref_util as R
from dropout_util import hidden_keep
from gemm_ref_util import check_close

pytestmark = pytest.mark.gpu

BF, F32 = torch.bfloat16, torch.float32
NAN16, NAN32 = 0x7FA5, 0x7FBADBAD   # bf16 / fp32 NaN bit patterns of the guard bands
SEED_HI = 0xFEDCBA9876543210        # a dropout seed with the high bits set
WORST = {}                          # case family -> largest error / bound seen
KERNELS = re.compile(r"\b(ln_fwd_kernel|ln_bwd_kernel|embed_fwd_kernel|embed_bwd_kernel|colsum_kernel|ce_fwd_kernel|ce_bwd_kernel|"
                     r"cast_f32_bf16_kernel|cast_bf16_f32_kernel|mask_bias_kernel|cast_multi_kernel)(<\d+>)?")


def _dev():
    return torch.device("cuda:0")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _L():
    from visualbert_b200 import _lib
    return _lib


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _check(rc, what):
    _L().check(rc, what)


def _note(family, ratio):
    WORST[family] = max(WORST.get(family, 0.0), ratio)


def _report(families):
    print("\n" + "  ".join(f"{f}: {WORST[f]:.3g}" for f in families if f in WORST))


def _nc(H, cap=4):
    """register chunks per lane of the row kernels: ceil(H / 256); the LayerNorm forward serves every H > 1024 with NC = 8"""
    c = (H // 8 + 31) // 32
    return c if c <= 4 else cap


class Guarded:
    """rows x cols output inside a [lead + rows + tail, ld] allocation prefilled with a NaN bit pattern; `fill` (if given)
    replaces the pattern in range."""

    def __init__(self, rows, cols, dtype, ld=None, lead=2, tail=3, fill=None):
        self.ld = cols if ld is None else ld
        self.it, self.pat = (torch.int16, NAN16) if dtype == BF else (torch.int32, NAN32)
        self.buf = torch.full((lead + rows + tail, self.ld), self.pat, dtype=self.it, device=_dev()).view(dtype)
        self.t = self.buf[lead:lead + rows, :cols]
        if fill is not None:
            self.t.copy_(fill.reshape(rows, cols))
        self.inside = torch.zeros(self.buf.shape, dtype=torch.bool, device=_dev())
        self.inside[lead:lead + rows, :cols] = True

    def check_bands(self, what):
        n = int((self.buf.view(self.it)[~self.inside] != self.pat).sum())
        assert n == 0, f"{what}: {n} elements written outside the output"


def _vec(n, fill=None):
    """fp32 [n] output between guard rows (a [1, n] Guarded)."""
    return Guarded(1, n, F32, fill=fill)


# torch.profiler can lose the kernel records nearest the edges of its capture window (the first kernel of a short window,
# or the whole of one): each counted window starts after the device is idle and leaves host time at both ends
PROFILE_PAD_S = 0.05


class Launches:
    """Profiles a block of calls and checks, in launch order, every row kernel (KERNELS) against `expected`."""

    def __init__(self, tmp_path):
        self.expected = []
        self.trace = tmp_path / "rowop_trace.json"

    def want(self, case, *names):
        self.expected += [(case, n) for n in names]

    def __enter__(self):
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.synchronize()
        self.prof = profile(activities=[ProfilerActivity.CUDA])
        self.prof.__enter__()
        time.sleep(PROFILE_PAD_S)
        return self

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        time.sleep(PROFILE_PAD_S)
        self.prof.__exit__(*exc)
        if exc[0] is not None:
            return False
        self.prof.export_chrome_trace(str(self.trace))
        events = json.loads(self.trace.read_text())["traceEvents"]
        ks = sorted((e for e in events if e.get("cat") == "kernel"), key=lambda e: e["ts"])
        got = [m.group(1) + (m.group(2) or "") for m in (KERNELS.search(e.get("name", "")) for e in ks) if m]
        assert len(got) == len(self.expected), (f"{len(got)} row-kernel launches recorded for {len(self.expected)} expected; "
                                                f"{len(ks)} kernels in the trace: {[e.get('name', '')[:60] for e in ks[:8]]}")
        for g, (case, want) in zip(got, self.expected):
            assert g == want, f"{case}: launched {g}, expected {want}"
        return False


# ---- LayerNorm forward -------------------------------------------------------------------------------------------------------
def _ln_input(rows, H, ldx, seed):
    """bf16 [rows, H] view of a [rows, ldx] allocation: N(0.5, 2) rows, with a constant row (3), a zero row (6) and rows whose
    mean is far larger than their spread (5: 64 + N(0, 1); 8: -300 + N(0, 2)) where the row count allows."""
    g = torch.Generator(device=_dev()).manual_seed(seed)
    full = (torch.randn(rows, ldx, device=_dev(), generator=g) * 2 + 0.5).to(BF)
    x = full[:, :H]
    const = [r for r in (3, 6) if r < rows]
    if rows > 3:
        x[3] = 1.5
    if rows > 5:
        x[5] = (64 + torch.randn(H, device=_dev(), generator=g)).to(BF)
    if rows > 6:
        x[6] = 0.0
    if rows > 8:
        x[8] = (-300 + 2 * torch.randn(H, device=_dev(), generator=g)).to(BF)
    return x, const


def _ln_fwd_call(x, ldx, gamma, beta, y, mean, rstd):
    rows, H = x.shape
    _check(_L().lib().vb_layernorm_fwd(_p(x), ctypes.c_int64(ldx), _p(gamma), _p(beta), _p(y.t), ctypes.c_int64(y.ld),
                                       _p(mean), _p(rstd), rows, H, ctypes.c_float(R.LN_EPS), _st()), "vb_layernorm_fwd")


LN_FWD_H = [8, 128, 264, 768, 776, 1024, 1032, 1536, 2048]


def test_layernorm_forward(tmp_path):
    """Every H reaches NC = 1, 2, 3, 4 or 8 (264, 776, 1032: a partial last register chunk); rows 1, 7, 8, 9, 1000 (partial and
    whole 8-row blocks); unit strides with mean / rstd written, and wider strides with mean / rstd NULL. Constant rows give beta
    bit for bit (rstd = 1 / sqrt(eps)) and nothing non-finite."""
    dev = _dev()
    with Launches(tmp_path) as rec:
        for H in LN_FWD_H:
            g = torch.Generator(device=dev).manual_seed(H)
            gamma = 1 + 0.1 * torch.randn(H, device=dev, generator=g)
            beta = 0.1 * torch.randn(H, device=dev, generator=g)
            for rows in (1, 7, 8, 9, 1000):
                for ldx, ldy, stats in ((H, H, True), (H + 8, H + 24, False)):
                    case = f"ln_fwd H={H} rows={rows} ldx={ldx} ldy={ldy} stats={stats}"
                    x, const = _ln_input(rows, H, ldx, rows * H + ldx)
                    y = Guarded(rows, H, BF, ld=ldy)
                    mean, rstd = (_vec(rows), _vec(rows)) if stats else (None, None)
                    _ln_fwd_call(x, ldx, gamma, beta, y, mean and mean.t[0], rstd and rstd.t[0])
                    rec.want(case, f"ln_fwd_kernel<{_nc(H, 8)}>")
                    torch.cuda.synchronize()
                    y.check_bands(case + " y")
                    ref, mag, st = R.ln_fwd_ref(x, gamma, beta)
                    _note("ln_fwd y", R.check(y.t, ref, R.ln_fwd_bound(ref, mag), case))
                    for r in const:
                        R.check_bits(y.t[r], beta.to(BF), f"{case} constant row {r}")
                    if stats:
                        mean.check_bands(case + " mean")
                        rstd.check_bands(case + " rstd")
                        _note("ln_fwd stats", R.check_stats(mean.t[0], rstd.t[0], st, case))
    _report(["ln_fwd y", "ln_fwd stats"])


# ---- LayerNorm backward ------------------------------------------------------------------------------------------------------
def _ln_bwd_case(rec, family, rows, H, drop, in_drop, nulls, seed):
    dev = _dev()
    case = f"ln_bwd rows={rows} H={H} drop={drop} in_drop={in_drop} nulls={nulls}"
    g = torch.Generator(device=dev).manual_seed(seed)
    x = (torch.randn(rows, H, device=dev, generator=g) * 2 + 0.5).to(BF)
    dy = torch.randn(rows, H, device=dev, generator=g).to(BF)
    gamma = 1 + 0.1 * torch.randn(H, device=dev, generator=g)
    beta = torch.zeros(H, device=dev)
    yf, mean, rstd = Guarded(rows, H, BF), _vec(rows), _vec(rows)
    _ln_fwd_call(x, H, gamma, beta, yf, mean.t[0], rstd.t[0])   # mean / rstd as the forward wrote them
    rec.want(case, f"ln_fwd_kernel<{_nc(H, 8)}>")
    dx = Guarded(rows, H, BF)
    dx_drop = Guarded(rows, H, BF) if drop else None
    pre = {k: torch.randn(H, device=dev, generator=g) for k in ("dgamma", "dbeta", "dbias")}
    cols = {k: None if nulls else _vec(H, pre[k]) for k in pre}
    p, stream, in_p, in_stream = (0.1 if drop else 0.0), 7, (0.1 if in_drop else 0.0), R.EMBED_DROP_STREAM
    P = lambda o: None if o is None else _p(o.t)
    _check(_L().lib().vb_layernorm_bwd(_p(dy), _p(x), _p(mean.t), _p(rstd.t), _p(gamma), P(dx), P(dx_drop), P(cols["dgamma"]),
                                       P(cols["dbeta"]), P(cols["dbias"]), rows, H, ctypes.c_float(p), ctypes.c_uint64(SEED_HI),
                                       ctypes.c_uint32(stream), ctypes.c_float(in_p), ctypes.c_uint32(in_stream), _st()),
           "vb_layernorm_bwd")
    rec.want(case, f"ln_bwd_kernel<{_nc(H)}>")
    torch.cuda.synchronize()
    for name, o in [("dx", dx), ("dx_drop", dx_drop)] + list(cols.items()):
        if o is not None:
            o.check_bands(f"{case} {name}")
    in_keep, in_scale = hidden_keep(SEED_HI, in_stream, rows, H, in_p, dev) if in_drop else (None, 1.0)
    r = R.ln_bwd_ref(dy, x, mean.t[0], rstd.t[0], gamma, in_keep, in_scale)
    _note(family + " dx", R.check(dx.t, r["dx"], R.ln_bwd_bound(r["dx"], r["mag"]), case + " dx"))
    o_ref, o_mag = r["dx"], r["mag"]   # the gradient dbias sums: dx, or dx_drop before its bf16 rounding
    if drop:
        keep, scale = hidden_keep(SEED_HI, stream, rows, H, p, dev)
        _note(family + " dx_drop", R.check_dropout_rows(dx_drop.t, r["dx"], r["mag"], keep, scale, case + " dx_drop"))
        k = keep.double() * scale
        o_ref, o_mag = o_ref * k, o_mag * k
    if not nulls:
        sums = dict(dgamma=(r["dgamma"], r["dgamma_mag"], None), dbeta=(r["dbeta"], r["dbeta_mag"], None),
                    dbias=(o_ref, o_ref.abs(), R.C_LN * o_mag.sum(0)))
        for k, (terms, tmag, extra) in sums.items():
            want = pre[k].double() + terms.sum(0)
            _note(family + " sums", R.check(cols[k].t[0], want, R.colsum_bound(pre[k], tmag, extra), f"{case} {k}"))


def test_layernorm_backward(tmp_path):
    """H reaching NC = 1..4 (264: a partial last chunk); 1, 9 and 3 * 2 * SMs * 8 + 5 rows (the grid-stride loop wraps three times
    and the next-row prefetch runs past the end); hidden dropout (dx_drop, dbias summing it), the re-applied in_dropout mask and
    NULL column sums, alone and in every combination."""
    big = 3 * 2 * _sms() * 8 + 5
    with Launches(tmp_path) as rec:
        for H in (8, 264, 768, 1024):
            for rows in (1, 9, big):
                for combo in range(8):
                    drop, in_drop, nulls = bool(combo & 1), bool(combo & 2), bool(combo & 4)
                    _ln_bwd_case(rec, "ln_bwd", rows, H, drop, in_drop, nulls, seed=H + rows + combo)
    _report(["ln_bwd dx", "ln_bwd dx_drop", "ln_bwd sums"])


# ---- embedding ---------------------------------------------------------------------------------------------------------------
MAX_POS, VOCAB, DV = 40, 50, 64
EMBED_CASES = [  # B, T, V, H, n_types, visual_addend, dropout
    (1, 1, 0, 128, 1, False, False),
    (1, MAX_POS, 1, 784, 2, True, True),
    (33, MAX_POS, 36, 128, 3, False, True),
    (70, 1, 36, 784, 3, True, False),
    (70, MAX_POS, 0, 784, 2, False, True),
    (33, 1, 1, 128, 2, True, False),
    (70, MAX_POS, 36, 784, 1, False, False),
    (1, MAX_POS, 36, 128, 3, False, True),
]


def _embed_inputs(B, T, V, H, nt, seed):
    dev = _dev()
    g = torch.Generator(device=dev).manual_seed(seed)
    ids = torch.randint(0, VOCAB, (B, T), device=dev, generator=g)
    tt = torch.randint(0, nt, (B, T), device=dev, generator=g)
    vt = torch.randint(0, nt, (B, max(V, 1)), device=dev, generator=g)[:, :V].contiguous()
    # out of range: clamped to the first / last table row
    ids.view(-1)[0] = VOCAB + 3
    ids.view(-1)[-1] = -5
    if B * T > 2:
        ids.view(-1)[1] = VOCAB
    tt.view(-1)[-1] = nt + 4
    if B * T > 1:
        tt.view(-1)[0] = -1
    if V:
        vt.view(-1)[0] = -2
        vt.view(-1)[-1] = nt
    t = dict(word=torch.randn(VOCAB, H, device=dev, generator=g), pos=torch.randn(MAX_POS, H, device=dev, generator=g),
             type=torch.randn(nt, H, device=dev, generator=g), pos_vis=torch.randn(MAX_POS, H, device=dev, generator=g),
             type_vis=torch.randn(nt, H, device=dev, generator=g))
    feats = torch.randn(max(B * V, 1), DV, device=dev, generator=g).to(BF)[:B * V]
    w_proj = (0.1 * torch.randn(H, DV, device=dev, generator=g)).to(BF)
    b_proj = 0.1 * torch.randn(H, device=dev, generator=g)
    addend = torch.randn(max(B * V, 1), H, device=dev, generator=g).to(BF)[:B * V]
    gamma = 1 + 0.1 * torch.randn(H, device=dev, generator=g)
    beta = 0.1 * torch.randn(H, device=dev, generator=g)
    dy = torch.randn(B * (T + V), H, device=dev, generator=g).to(BF)
    return ids, tt, vt, t, feats, w_proj, b_proj, addend, gamma, beta, dy, g


def _embed_case(rec, B, T, V, H, nt, vis_add, drop, seed):
    L_, L = _L(), _L().lib()
    dev = _dev()
    S, M, BV = T + V, B * (T + V), B * V
    case = f"embed B={B} T={T} V={V} H={H} n_types={nt} addend={vis_add} drop={drop}"
    ids, tt, vt, tabs, feats, w_proj, b_proj, addend, gamma, beta, dy, g = _embed_inputs(B, T, V, H, nt, seed)
    p = 0.1 if drop else 0.0
    ptr = lambda t: 0 if t is None or t.numel() == 0 else t.data_ptr()
    d = L_.EmbedDesc(batch=B, text_len=T, num_regions=V, hidden=H, visual_dim=DV, vocab=VOCAB, max_pos=MAX_POS, n_types=nt,
                     eps=R.LN_EPS, dropout=p, seed=SEED_HI, input_ids=ids.data_ptr(), token_type_ids=tt.data_ptr(),
                     visual_type=ptr(vt), visual_feats=ptr(feats), w_proj=ptr(w_proj) if V else 0, b_proj=b_proj.data_ptr(),
                     word=tabs["word"].data_ptr(), pos=tabs["pos"].data_ptr(), type=tabs["type"].data_ptr(),
                     pos_vis=tabs["pos_vis"].data_ptr(), type_vis=tabs["type_vis"].data_ptr(), gamma=gamma.data_ptr(),
                     beta=beta.data_ptr(), visual_addend=ptr(addend) if vis_add else 0)
    y, pre, mean, rstd = Guarded(M, H, BF), Guarded(M, H, BF), _vec(M), _vec(M)
    vis_proj = Guarded(BV, H, BF) if V else None
    acts = L_.EmbedActs(vis_proj=vis_proj.t.data_ptr() if V else 0, pre=pre.t.data_ptr(), mean=mean.t.data_ptr(),
                        rstd=rstd.t.data_ptr())
    _check(L.vb_embed_fwd(ctypes.byref(d), _p(y.t), ctypes.byref(acts), _st()), "vb_embed_fwd")
    rec.want(case, f"embed_fwd_kernel<{_nc(H)}>")
    torch.cuda.synchronize()
    for name, o in (("y", y), ("pre", pre), ("mean", mean), ("rstd", rstd), ("vis_proj", vis_proj)):
        if o is not None:
            o.check_bands(f"{case} {name}")

    # forward: pre = bf16(fp64 sum) from the table rows the clamped ids pick and the stored projection; y = LN(pre) with the mask
    ic, tc = ids.clamp(0, VOCAB - 1).view(-1), tt.clamp(0, nt - 1).view(-1)
    T64 = {k: v.double() for k, v in tabs.items()}
    pos_rows = torch.arange(T, device=dev).repeat(B)
    txt_ref = T64["word"][ic] + T64["pos"][pos_rows] + T64["type"][tc]
    txt_mag = T64["word"][ic].abs() + T64["pos"][pos_rows].abs() + T64["type"][tc].abs()
    pre3 = pre.t.view(B, S, H)
    _note("embed pre", R.check(pre3[:, :T].reshape(-1, H), txt_ref, R.REL_BF16 * txt_ref.abs() + R.C_SUM * txt_mag, case + " pre text"))
    if V:
        f64, w64 = feats.double(), w_proj.double()
        acc, amag = f64 @ w64.t() + b_proj.double(), f64.abs() @ w64.abs().t() + b_proj.double().abs()
        if vis_add:
            acc, amag = acc + addend.double(), amag + addend.double().abs()
        _note("embed vis_proj", check_close(vis_proj.t, acc, amag, True, case + " vis_proj"))
        vc = vt.clamp(0, nt - 1).view(-1)
        vis_ref = vis_proj.t.double() + T64["pos_vis"][0] + T64["type_vis"][vc]
        vis_mag = vis_proj.t.double().abs() + T64["pos_vis"][0].abs() + T64["type_vis"][vc].abs()
        _note("embed pre", R.check(pre3[:, T:].reshape(-1, H), vis_ref, R.REL_BF16 * vis_ref.abs() + R.C_SUM * vis_mag,
                                   case + " pre visual"))
    ref, mag, st = R.ln_fwd_ref(pre.t, gamma, beta)
    _note("embed stats", R.check_stats(mean.t[0], rstd.t[0], st, case))
    if drop:
        keep, scale = hidden_keep(SEED_HI, R.EMBED_DROP_STREAM, M, H, p, dev)
        _note("embed y", R.check(y.t[keep], ref[keep] * scale, R.ln_fwd_bound(ref[keep] * scale, mag[keep] * scale), case + " y kept"))
        R.check_bits(y.t[~keep], torch.zeros_like(y.t[~keep]), case + " y dropped")
    else:
        keep, scale = None, 1.0
        _note("embed y", R.check(y.t, ref, R.ln_fwd_bound(ref, mag), case + " y"))

    # backward
    shapes = dict(word=VOCAB, pos=MAX_POS, type=nt, pos_vis=MAX_POS, type_vis=nt)
    prefill = {k: torch.randn(n, H, device=dev, generator=g) for k, n in shapes.items()}
    prefill.update(dgamma=torch.randn(H, device=dev, generator=g), dbeta=torch.randn(H, device=dev, generator=g),
                   db_proj=torch.randn(H, device=dev, generator=g), dw_proj=torch.randn(H, DV, device=dev, generator=g))
    out = {k: Guarded(v.shape[0] if v.dim() == 2 else 1, v.shape[-1], F32, fill=v) for k, v in prefill.items()}
    d_pre = Guarded(M, H, BF)
    d_vis = Guarded(BV, H, BF) if V else None
    d_feats = Guarded(BV, DV, BF) if V else None
    P = lambda k: out[k].t.data_ptr()
    gr = L_.EmbedGrads(dword=P("word"), dpos=P("pos"), dtype=P("type"), dpos_vis=P("pos_vis"), dtype_vis=P("type_vis"),
                       dw_proj=P("dw_proj"), db_proj=P("db_proj"), dgamma=P("dgamma"), dbeta=P("dbeta"), d_pre=d_pre.t.data_ptr(),
                       d_vis=d_vis.t.data_ptr() if V else 0, d_feats=d_feats.t.data_ptr() if V else 0)
    _check(L.vb_embed_bwd(ctypes.byref(d), ctypes.byref(acts), _p(dy), ctypes.byref(gr), _st()), "vb_embed_bwd")
    rec.want(case, f"ln_bwd_kernel<{_nc(H)}>", f"embed_bwd_kernel<{_nc(H)}>", *(["colsum_kernel"] if V else []))
    torch.cuda.synchronize()
    for name, o in list(out.items()) + [("d_pre", d_pre), ("d_vis", d_vis), ("d_feats", d_feats)]:
        if o is not None:
            o.check_bands(f"{case} {name}")
    r = R.ln_bwd_ref(dy, pre.t, mean.t[0], rstd.t[0], gamma, keep, scale)
    _note("embed d_pre", R.check(d_pre.t, r["dx"], R.ln_bwd_bound(r["dx"], r["mag"]), case + " d_pre"))
    for k in ("dgamma", "dbeta"):
        _note("embed sums", R.check(out[k].t[0], prefill[k].double() + r[k].sum(0), R.colsum_bound(prefill[k], r[k + "_mag"]),
                                    f"{case} {k}"))
    de = d_pre.t.double().view(B, S, H)
    txt, vis = de[:, :T].reshape(-1, H), de[:, T:].reshape(-1, H)
    idx = dict(word=(ic, txt), pos=(pos_rows, txt), type=(tc, txt))
    if V:
        idx.update(pos_vis=(torch.zeros(BV, dtype=torch.long, device=dev), vis), type_vis=(vt.clamp(0, nt - 1).view(-1), vis))
    for k, n in shapes.items():
        pre0 = prefill[k].double()
        if k not in idx:   # no regions: the visual tables are untouched
            R.check_bits(out[k].t, prefill[k], f"{case} {k}")
            continue
        index, rows = idx[k]
        ref_t = pre0.index_add(0, index, rows)
        mag_t = torch.zeros(n, H, device=dev, dtype=torch.float64).index_add_(0, index, rows.abs())
        _note("embed tables", R.check(out[k].t, ref_t, R.colsum_bound(prefill[k], mag_t[None]), f"{case} {k}"))
        cnt = torch.zeros(n, device=dev).index_add_(0, index, torch.ones(len(index), device=dev))
        R.check_bits(out[k].t[cnt == 0], prefill[k][cnt == 0], f"{case} {k} rows nothing maps to")
    if V:
        R.check_bits(d_vis.t, d_pre.t.view(B, S, H)[:, T:].reshape(-1, H), case + " d_vis")
        dv = d_vis.t.double()
        _note("embed sums", R.check(out["db_proj"].t[0], prefill["db_proj"].double() + dv.sum(0),
                                    R.colsum_bound(prefill["db_proj"], dv.abs()), case + " db_proj"))
        pw = prefill["dw_proj"].double()
        _note("embed proj grads", check_close(out["dw_proj"].t, pw + dv.t() @ feats.double(), pw.abs() + dv.abs().t() @ feats.double().abs(),
                                              False, case + " dw_proj"))
        _note("embed proj grads", check_close(d_feats.t, dv @ w_proj.double(), dv.abs() @ w_proj.double().abs(), True, case + " d_feats"))
    else:
        R.check_bits(out["db_proj"].t, prefill["db_proj"][None], case + " db_proj")
        R.check_bits(out["dw_proj"].t, prefill["dw_proj"], case + " dw_proj")


def test_embedding_forward_and_backward(tmp_path):
    """vb_embed_fwd + vb_embed_bwd in the default (atomic) mode, the descriptor built directly: B = 1, 33, 70 (the backward cuts
    batches over 32 into 32-example tasks); T = 1 and max_pos; no, one and 36 regions; H = 128 and 784 (NC = 1 and 4, 784 with a
    partial last chunk); one, two and three token types (types 0 and 1 sum in registers, type 2 through shared-memory atomics);
    ids and types out of range (clamped); the visual addend and dropout on and off; d_feats on."""
    with Launches(tmp_path) as rec:
        for i, c in enumerate(EMBED_CASES):
            _embed_case(rec, *c, seed=100 + i)
    _report(["embed pre", "embed vis_proj", "embed y", "embed stats", "embed d_pre", "embed sums", "embed tables", "embed proj grads"])


# ---- column sum --------------------------------------------------------------------------------------------------------------
def _colsum_gy(M, N):
    gx = (N // 8 + 31) // 32
    return min(max(_sms() * 6 // gx, 1), (M + 7) // 8)


def test_colsum(tmp_path):
    """vb_colsum_bf16 (default, atomic): M below one 8-row phase, around it, and just below and above one and two sweeps of the
    4-row unrolled loop (4 * gridDim.y * 8 rows); N from one chunk to the MLM decoder's 30528 columns; ld = N and ld > N."""
    dev = _dev()
    with Launches(tmp_path) as rec:
        for N in (8, 16, 264, 30528):
            sweep = 4 * _colsum_gy(1 << 30, N) * 8
            Ms = [1, 7, 8, 9, 31, 33, sweep - 1, sweep + 1, 2 * sweep - 1, 2 * sweep + 1]
            for M in Ms:
                for ld in (N, N + 8):
                    case = f"colsum M={M} N={N} ld={ld}"
                    g = torch.Generator(device=dev).manual_seed(M + N + ld)
                    x = torch.randn(M, ld, device=dev, generator=g).to(BF)[:, :N]
                    if M > 1:
                        x[M // 2] = 3.0   # a row far from the others
                    prefill = torch.randn(N, device=dev, generator=g)
                    out = _vec(N, prefill)
                    _check(_L().lib().vb_colsum_bf16(_p(x), ctypes.c_int64(ld), _p(out.t), M, N, _st()), "vb_colsum_bf16")
                    rec.want(case, "colsum_kernel")
                    torch.cuda.synchronize()
                    out.check_bands(case)
                    x64 = x.double()
                    _note("colsum", R.check(out.t[0], prefill.double() + x64.sum(0), R.colsum_bound(prefill, x64.abs()), case))
    _report(["colsum"])


# ---- cross-entropy -----------------------------------------------------------------------------------------------------------
def _ce_logits(rows, vocab, g):
    """rows of N(0, 3) logits; row 5 spread uniformly over +-80, rows 6 / 7 with one dominant logit (+40), row 8 all equal."""
    dev = _dev()
    z = 3 * torch.randn(rows, vocab, device=dev, generator=g)
    z[5] = (torch.rand(vocab, device=dev, generator=g) * 2 - 1) * 80
    dom = int(torch.randint(0, vocab, (1,), device=dev, generator=g))
    z[6, dom] = 40.0
    z[7, dom] = 40.0
    z[8] = 2.5
    return z.to(BF), dom


def test_cross_entropy(tmp_path):
    """vb_cross_entropy_fwd / _bwd for vocab 1..9, 2049 and 30522 (every vocab % 8 tail), padded = vocab rounded up to 8 and one
    chunk more, ld = padded and 16 columns more. Labels 0, vocab - 1, ignored (-1, -100, vocab), and on / off a dominant logit.
    Ignored rows: loss exactly 0 and a zero gradient row; columns [vocab, padded) come back as exact +0 and columns [padded, ld)
    untouched (they hold NaN patterns that the forward must not read either). rows = 0 launches nothing."""
    dev, L = _dev(), _L().lib()
    rows = 12
    with Launches(tmp_path) as rec:
        for vocab in (1, 7, 8, 9, 2049, 30522):
            p8 = (vocab + 7) // 8 * 8
            for padded, ld in ((p8, p8), (p8 + 8, p8 + 24)):
                case = f"ce vocab={vocab} padded={padded} ld={ld}"
                g = torch.Generator(device=dev).manual_seed(vocab + ld)
                z, dom = _ce_logits(rows, vocab, g)
                labels = torch.randint(0, vocab, (rows,), device=dev, generator=g)
                labels[0], labels[1], labels[2], labels[3], labels[4] = 0, vocab - 1, -1, -100, vocab
                labels[6], labels[7] = dom, (dom + 1) % vocab
                logits = Guarded(rows, padded, BF, ld=ld)
                logits.t[:, :vocab] = z
                lse, loss = _vec(rows), _vec(rows)
                _check(L.vb_cross_entropy_fwd(_p(logits.t), ctypes.c_int64(ld), _p(labels), rows, vocab, _p(lse.t), _p(loss.t),
                                              _st()), "vb_cross_entropy_fwd")
                scale = torch.tensor([0.37], device=dev)
                _check(L.vb_cross_entropy_bwd(_p(logits.t), ctypes.c_int64(ld), _p(labels), rows, vocab, padded, _p(lse.t),
                                              _p(scale), _st()), "vb_cross_entropy_bwd")
                rec.want(case, "ce_fwd_kernel", "ce_bwd_kernel")
                torch.cuda.synchronize()
                for name, o in (("logits", logits), ("lse", lse), ("loss", loss)):
                    o.check_bands(f"{case} {name}")
                lse_ref, loss_ref, prob, valid = R.ce_ref(z, labels, vocab)
                b = R.ce_lse_bound(lse_ref)
                _note("ce lse/loss", R.check(lse.t[0], lse_ref, b, case + " lse"))
                _note("ce lse/loss", R.check(loss.t[0][valid], loss_ref[valid], b[valid], case + " loss"))
                R.check_bits(loss.t[0][~valid], torch.zeros_like(loss.t[0][~valid]), case + " loss of ignored rows")
                gref = R.ce_grad_ref(prob, labels, valid, 0.37)
                _note("ce grad", R.check(logits.t[:, :vocab], gref, R.ce_grad_bound(gref, lse_ref, 0.37), case + " grad"))
                R.check_bits(logits.t[~valid], torch.zeros_like(logits.t[~valid]), case + " ignored rows")
                R.check_bits(logits.t[:, vocab:], torch.zeros_like(logits.t[:, vocab:]), case + " padding columns")
        # rows = 0: nothing launched, nothing written
        empty = Guarded(1, 16, BF)
        _check(L.vb_cross_entropy_fwd(_p(empty.t), ctypes.c_int64(16), None, 0, 9, None, None, _st()), "vb_cross_entropy_fwd")
        _check(L.vb_cross_entropy_bwd(_p(empty.t), ctypes.c_int64(16), None, 0, 9, 16, None, None, _st()), "vb_cross_entropy_bwd")
    empty.check_bands("ce rows=0")
    assert bool((empty.t.view(torch.int16) == NAN16).all()), "ce rows=0 wrote its logits"
    _report(["ce lse/loss", "ce grad"])


# ---- casts -------------------------------------------------------------------------------------------------------------------
def _f32_values(n, g):
    """fp32 values over the whole range: the cast edge values, then N(0, 1) times 2^k for k in [-140, 120] (subnormals, values
    that round up into the next exponent, overflow to Inf)."""
    dev = _dev()
    e = R.cast_edge_values().to(dev)
    k = torch.randint(-140, 121, (n,), device=dev, generator=g).double()
    v = (torch.randn(n, device=dev, generator=g, dtype=torch.float64) * torch.exp2(k)).float()
    v[:min(n, e.numel())] = e[:min(n, e.numel())]
    return v


def test_casts(tmp_path):
    """vb_cast_f32_to_bf16 and vb_cast_bf16_to_f32 at n = 8 and 2048 * 8 * SMs + 8 (the grid-stride loop wraps by one chunk),
    bit for bit: round to nearest even on the way down (NaN stays NaN), exact on the way up. vb_mask_bias with and without the
    image mask, bit for bit against the fp32 (1 - m) * -10000."""
    dev, L = _dev(), _L().lib()
    with Launches(tmp_path) as rec:
        for n in (8, 2048 * 8 * _sms() + 8):
            g = torch.Generator(device=dev).manual_seed(n)
            src = _f32_values(n, g)
            dst = Guarded(1, n, BF)
            _check(L.vb_cast_f32_to_bf16(_p(src), _p(dst.t), ctypes.c_int64(n), _st()), "vb_cast_f32_to_bf16")
            rec.want(f"cast down n={n}", "cast_f32_bf16_kernel")
            bits = torch.randint(-32768, 32768, (n,), device=dev, generator=g, dtype=torch.int32).to(torch.int16)
            src16 = bits.view(BF)
            up = Guarded(1, n, F32)
            _check(L.vb_cast_bf16_to_f32(_p(src16), _p(up.t), ctypes.c_int64(n), _st()), "vb_cast_bf16_to_f32")
            rec.want(f"cast up n={n}", "cast_bf16_f32_kernel")
            torch.cuda.synchronize()
            dst.check_bands(f"cast down n={n}")
            up.check_bands(f"cast up n={n}")
            R.check_cast_bf16(dst.t[0], src, f"cast down n={n}")
            want = (bits.to(torch.int32) << 16).view(F32)
            nan = torch.isnan(want)
            R.check_bits(up.t[0][~nan], want[~nan], f"cast up n={n}")
            assert bool(torch.isnan(up.t[0][nan]).all()), f"cast up n={n}: a NaN did not stay NaN"
        for B, T, V, with_image in ((5, 7, 3, True), (5, 7, 3, False), (300, 40, 36, True), (2, 9, 0, False)):
            case = f"mask_bias B={B} T={T} V={V} image={with_image}"
            g = torch.Generator(device=dev).manual_seed(B * T + V)
            im = torch.randint(0, 2, (B, T), device=dev, generator=g)
            im.view(-1)[0] = 3   # not a 0 / 1 mask: still (1 - m) * -10000
            vm = torch.randint(0, 2, (B, V), device=dev, generator=g) if with_image else None
            out = Guarded(B, T + V, F32)
            _check(L.vb_mask_bias(_p(im), _p(vm), _p(out.t), B, T, V, _st()), "vb_mask_bias")
            rec.want(case, "mask_bias_kernel")
            torch.cuda.synchronize()
            out.check_bands(case)
            m = torch.cat([im, vm if with_image else torch.ones(B, V, device=dev, dtype=torch.int64)], 1)
            R.check_bits(out.t, (1.0 - m.float()) * -10000.0, case)


def test_cast_multi(tmp_path):
    """vb_cast_multi over one table: bf16 items of 1, 7, 8192, 8193 and 3 * 8192 - 1 elements (chunk edges, the 8-wide vector
    path and its scalar tail), bf16 destinations and fp32 sources at odd element offsets (the scalar path), and fp32 items. Items
    sit in shared buffers separated by guard gaps; every element outside an item keeps its NaN pattern. Bit for bit."""
    L_, dev = _L(), _dev()
    C = L_.VB_CAST_CHUNK
    # (numel, src element offset, dst element offset, fp32 destination)
    items = [(1, 0, 0, False), (7, 0, 0, False), (C, 0, 0, False), (C + 1, 0, 0, False), (3 * C - 1, 0, 0, False),
             (C + 1, 0, 1, False), (3 * C - 1, 0, 3, False), (7, 0, 5, False), (C + 1, 1, 0, False),
             (C + 1, 0, 0, True), (1, 0, 0, True), (3 * C - 1, 1, 1, True)]
    gap = 24
    so = dof = fof = 0
    layout = []
    for n, s_off, d_off, f32 in items:
        s = so + s_off
        so = s + n + gap
        so = (so + 7) // 8 * 8
        if f32:
            d = fof + d_off
            fof = (d + n + gap + 7) // 8 * 8
        else:
            d = dof + d_off
            dof = (d + n + gap + 7) // 8 * 8
        layout.append((n, s, d, f32))
    g = torch.Generator(device=dev).manual_seed(9)
    src = _f32_values(so, g)
    edge = R.cast_edge_values().to(dev)
    for n, s, _, _ in layout:   # every item starts with the edge values (fp32 items copy their NaN payloads too)
        src[s:s + min(n, edge.numel())] = edge[:min(n, edge.numel())]
    # the profiler can miss the first kernel of a window: the guarded outputs are built, and checked, inside it as in the
    # other tests, so that cast_multi_kernel is neither the first nor the last activity of the trace
    with Launches(tmp_path) as rec:
        dbf = Guarded(1, dof, BF)
        df = Guarded(1, fof, F32)
        arr = (L_.CastItem * len(layout))()
        chunk = 0
        for i, (n, s, d, f32) in enumerate(layout):
            arr[i].src = src[s:].data_ptr()
            arr[i].dst = (df.t[0, d:] if f32 else dbf.t[0, d:]).data_ptr()
            arr[i].numel, arr[i].first_chunk, arr[i].dst_fp32 = n, chunk, int(f32)
            chunk += (n + C - 1) // C
        table = torch.from_numpy(np.frombuffer(bytes(arr), dtype=np.uint8).copy()).to(dev)
        _check(L_.lib().vb_cast_multi(_p(table), len(layout), chunk, _st()), "vb_cast_multi")
        rec.want("cast_multi", "cast_multi_kernel")
        torch.cuda.synchronize()
        inside = {False: torch.zeros(dof, dtype=torch.bool, device=dev), True: torch.zeros(fof, dtype=torch.bool, device=dev)}
        for n, s, d, f32 in layout:
            what = f"cast_multi numel={n} src+{s % 8} dst+{d % 8} fp32={f32}"
            if f32:
                R.check_bits(df.t[0, d:d + n], src[s:s + n], what)
            else:
                R.check_cast_bf16(dbf.t[0, d:d + n], src[s:s + n], what)
            inside[f32][d:d + n] = True
        dbf.check_bands("cast_multi bf16")
        df.check_bands("cast_multi fp32")
        assert bool((dbf.t[0].view(torch.int16)[~inside[False]] == NAN16).all()), "cast_multi wrote a bf16 gap"
        assert bool((df.t[0].view(torch.int32)[~inside[True]] == NAN32).all()), "cast_multi wrote an fp32 gap"
