"""Stage-by-stage fp64 check of one BertLayer call (vb_layer_fwd / vb_layer_bwd, or one layer of vb_encoder_fwd / vb_encoder_bwd
and their _varlen forms): every activation, every scratch buffer the backward leaves, every gradient and dx
(test_zz_layer_reference_gpu.py, test_layer_reference_cpu.py).

The kernels have their own reference tests; what this checks is the glue of csrc/vb_api.cu that chains them: which buffer is an
addend, which dropout stream each site draws (layer_index * 8 + site), whether d_pre or d_pre_drop enters a Linear, the layout
of drow, the tile-native gelu'(u), and the gradient carried between layers. Every stage's reference starts from the library's own
bf16 / fp32 inputs to that stage, so rounding does not compound across stages, and every bound is an existing one:
gemm_ref_util (GEMMs, GELU), attn_ref_util (attention), rowop_ref_util (LayerNorm, column sums).

Forward (x the layer input, s1 / s2 the survivors' scale of the hidden-dropout masks of streams 8 l + 1 and 8 l + 2):

    qkv        = x Wqkv^T + b                                 gemm bound
    ctx, lse   attn_ref_util.reference on qkv, the mask bias and the stored keep bits (unpadded: per sequence)
    pre1       = kept: (ctx Wo^T + bo) s1 + x, dropped: x bit for bit
    mean1, rstd1, x1 = LayerNorm(pre1)                        ln_fwd_bound / check_stats
    u (holds gelu'(u), tile-native when gp_tiled_ok(M, I)), g = gelu(u), u = x1 Wi^T + bi    GELU_LIP, GELU_APPROX
    pre2       = kept: (g Wout^T + bout) s2 + x1, dropped: x1 bit for bit
    mean2, rstd2, y = LayerNorm(pre2)

Backward. LN2's d_pre / d_pre_drop (rewritten by LN1) and d_u (rewritten by dqkv where the two share d_big) are recomputed in
fp64; their bounds are carried one stage forward as first-order terms, and every later stage starts again from a buffer that
survives the call:

    r2 = ln_bwd_ref(dy, pre2, mean2, rstd2, gamma2); dpm2 = r2.dx keep2 s2 within B2 = ln_bwd_bound(r2.dx, r2.mag, s2)
    dln2_gamma, dln2_beta, db_out  prefill + column sums                 colsum_bound (+ C_LN sum of dx_drop's magnitude)
    dw_out   = P + dpm2^T g                          C_ACC (|P| + |dpm2|^T |g|) + B2^T |g|
    d_u      = (dpm2 Wout) gelu'                     Bu = REL_BF16 |d_u| + C_ACC (|dpm2| |Wout|) |gelu'| + (B2 |Wout|) |gelu'|
               (gelu' is the stored bf16 acts.u; the rows of d_u past the first M 3H elements of d_big survive and are checked)
    db_inter = P + colsum(d_u)                       colsum_bound + sum Bu
    dw_inter = P + d_u^T x1                          C_ACC (|P| + |d_u|^T |x1|) + Bu^T |x1|
    d_x1     = d_u Wi + d_pre2                       REL_BF16 |ref| + C_ACC (|d_u| |Wi| + |d_pre2|) + Bu |Wi| + B(d_pre2)
    LN1 from the library's d_x1: d_pre, d_pre_drop (stream 8 l + 1), dln1_gamma, dln1_beta, db_attn_out as the row-op test
    dw_attn_out = P + dpm1^T ctx, d_ctx = dpm1 Wo    dpm1 the library's d_pre_drop (d_pre when p_h = 0): exact operands
    drow, dqkv  attn_ref_util.reference from the library's d_ctx and ctx; drow is [B, A, S] dense and [A, total] unpadded,
                whichever kernel wrote it; dqkv is the first M 3H elements of d_big, row stride 3H
    db_qkv = P + colsum(dqkv), dw_qkv = P + dqkv^T x, dx = dqkv Wqkv + d_pre (LN1's)   exact operands

The propagated terms are first order: the second-order products of two bounds are below 2^-16 of either and are not written.
Every check also requires its buffer to be finite over its whole extent (a NaN fill that the call did not overwrite fails).
"""
import torch

import attn_ref_util as AR
import gemm_ref_util as GR
import rowop_ref_util as RR
from dropout_util import hidden_keep

SITE_ATTN_OUT, SITE_FFN_OUT = 1, 2   # vb_api.cu kSiteAttnOut / kSiteFfnOut; kSiteAttnProbs = 0 draws the attention bits
PARAMS = ("w_qkv", "b_qkv", "w_attn_out", "b_attn_out", "ln1_gamma", "ln1_beta", "w_inter", "b_inter", "w_out", "b_out",
          "ln2_gamma", "ln2_beta")
GRADS = ("dw_qkv", "db_qkv", "dw_attn_out", "db_attn_out", "dln1_gamma", "dln1_beta", "dw_inter", "db_inter", "dw_out", "db_out",
         "dln2_gamma", "dln2_beta")


def drop_stream(layer_index, site):
    return layer_index * 8 + site


class _Checks:
    """Collects the worst error / bound per buffer; raise_if_bad() raises with the worst element of the worst buffer."""

    def __init__(self, what):
        self.what, self.worst, self.msgs = what, {}, {}

    def add(self, name, out, ref, bound, exact=None, want=None, where=""):
        """|out - ref| <= bound element by element; where `exact` is set, out must equal `want` bit for bit instead."""
        o = out.double()
        ratio = (o - ref).abs() / (bound + 1e-300)
        if exact is not None:
            same = out.reshape(-1).view(torch.int16) == want.reshape(-1).view(torch.int16)
            bad = torch.where(same.view(exact.shape), torch.zeros_like(ratio), torch.full_like(ratio, float("inf")))
            ratio = torch.where(exact, bad, ratio)
        ratio = torch.where(torch.isfinite(o), ratio, torch.full_like(ratio, float("inf")))
        w = float(ratio.max()) if ratio.numel() else 0.0
        if w > self.worst.get(name, -1.0):
            self.worst[name] = w
            if w > 1.0:
                idx = tuple(int(i) for i in torch.nonzero(ratio == ratio.max())[0])
                kind = ("dropped element not bit-exact" if exact is not None and bool(exact[idx])
                        else "non-finite" if not bool(torch.isfinite(o[idx])) else "outside the bound")
                self.msgs[name] = (f"{self.what}: {name}{where}: {int((ratio > 1).sum())} of {ratio.numel()} elements fail; worst at "
                                   f"{idx} ({kind}): out {float(o[idx]):.6g} ref {float(ref[idx]):.6g} bound {float(bound[idx]):.3g}")
        return w

    def raise_if_bad(self):
        bad = sorted((n for n, w in self.worst.items() if w > 1.0), key=lambda n: -self.worst[n])
        if bad:
            raise AssertionError(self.msgs[bad[0]] + "  |  failing: " + ", ".join(f"{n} {self.worst[n]:.3g}" for n in bad))


def _gemm(a, w, bias=None):
    """fp64 a w^T (+ bias) and its magnitude |a| |w|^T (+ |bias|)."""
    acc, mag = a @ w.t(), a.abs() @ w.abs().t()
    if bias is not None:
        acc, mag = acc + bias, mag + bias.abs()
    return acc, mag


def _dropout_resid(C, name, out, acc, mag, keep, scale, addend):
    """GEMM epilogue D = keep ? acc * scale + addend : addend (bf16); dropped elements equal the addend bit for bit."""
    add64 = addend.double()
    ref = acc * scale + add64
    C.add(name, out, ref, GR.bound(ref, mag * scale + add64.abs(), True), exact=~keep, want=addend)


def _ln_bwd_stage(C, tag, r, keep, scale, hd, d_pre, d_pre_drop, grads, prefill, names):
    """The LayerNorm backward's row outputs (when given) and its three column sums, as test_rowop_reference_gpu.py checks
    them. r: ln_bwd_ref. names: (dgamma, dbeta, dbias)."""
    if d_pre is not None:
        C.add(f"d_pre ({tag})", d_pre, r["dx"], RR.ln_bwd_bound(r["dx"], r["mag"]))
    if hd and d_pre_drop is not None:   # kept: dx * scale; dropped: exactly +0
        C.add(f"d_pre_drop ({tag})", d_pre_drop, r["dx"] * scale, RR.ln_bwd_bound(r["dx"], r["mag"], scale),
              exact=~keep, want=torch.zeros_like(d_pre_drop))
    kd = keep.double() * scale if hd else 1.0
    o_ref, o_mag = r["dx"] * kd, r["mag"] * kd
    sums = ((r["dgamma"], r["dgamma_mag"], None), (r["dbeta"], r["dbeta_mag"], None), (o_ref, o_ref.abs(), RR.C_LN * o_mag.sum(0)))
    for n, (terms, tmag, extra) in zip(names, sums):
        C.add(n, grads[n], prefill[n].double() + terms.sum(0), RR.colsum_bound(prefill[n], tmag, extra))


def _attention(C, cfg, qkv, ctx, lse, keep, d_ctx, drow, dqkv):
    """ctx, lse (forward) and drow, dqkv (backward) against attn_ref_util.reference, dense or per sequence."""
    B, S, A = cfg["B"], cfg["S"], cfg["A"]
    p_a, lens = cfg["p_a"], cfg.get("lens")
    scale = AR.drop_scale(p_a)
    bits = AR.keep_bits(keep, B * A, S) if p_a > 0 else None
    groups = []
    if lens is None:
        bias = cfg["mask_bias"].reshape(B, S).repeat_interleave(A, 0)
        q, k, v = AR.dense_heads(qkv, B, S, A)
        M = B * S
        groups.append(("", q, k, v, bias, bits, AR.dense_heads(d_ctx, B, S, A)[0], AR.dense_heads(ctx, B, S, A)[0],
                       lse.reshape(B * A, S), drow.reshape(B * A, S), AR.dense_heads(dqkv, B, S, A)))
    else:
        M = sum(lens)
        lse2, drow2 = lse.reshape(A, M), drow.reshape(A, M)
        r = 0
        for b, n in enumerate(lens):
            if n > 0:
                q, k, v = AR.varlen_heads(qkv, r, n, A)
                groups.append((f" (sequence {b}, rows {r}..{r + n})", q, k, v, None,
                               bits[b * A:(b + 1) * A, :n, :n] if bits is not None else None,
                               AR.varlen_heads(d_ctx, r, n, A)[0], AR.varlen_heads(ctx, r, n, A)[0],
                               lse2[:, r:r + n], drow2[:, r:r + n], AR.varlen_heads(dqkv, r, n, A)))
            r += n
        assert r == M, f"{C.what}: the sequences cover {r} of {M} rows"   # so lse and drow are checked over their whole extent
    for where, q, k, v, bias, kb, dO, c, ls, dr, dq3 in groups:
        ref = AR.reference(q, k, v, bias, kb, scale, dO, c)
        C.add("ctx", c, *ref["ctx"], where=where)
        C.add("lse", ls, *ref["lse"], where=where)
        C.add("drow", dr, *ref["drow"], where=where)
        for i, n in enumerate(("dq", "dk", "dv")):
            C.add("dqkv", dq3[i], *ref[n], where=f"{where} {n}")
        del ref


def check_layer(cfg, prm, x, dy, acts, scr, grads, prefill, dx=None, what="layer", strict=True):
    """Check everything one layer call read and wrote against fp64 references (module docstring).

    cfg: B, S (the longest sequence when unpadded), A, I, p_h, p_a, seed, layer_index, and mask_bias ([B, S] fp32, dense) or
         lens (the sequence lengths, unpadded).
    prm: the layer's parameters (PARAMS: bf16 weights, fp32 biases and LayerNorm gamma / beta).
    x, dy: the layer input and its output gradient (bf16, M rows); dx: the input gradient the call wrote, or None.
    acts: qkv, ctx, lse, pre1, mean1, rstd1, x1, u, g, pre2, mean2, rstd2, keep (uint8 keep buffer, or None) and y, as the
          activations / arena slot hold them (any shape of the right size; u as stored).
    scr: the scratch after the backward: d_pre, d_pre_drop (None when p_h = 0), d_big (M max(I, 3H) elements), d_x1, d_ctx, drow.
    grads, prefill: the 12 vb_layer_grads fields after the call and their values before it.
    Any device. Returns {buffer: worst error / bound}; raises AssertionError naming the worst element unless strict is False."""
    B, S, A, I = cfg["B"], cfg["S"], cfg["A"], cfg["I"]
    H = 64 * A
    lens = cfg.get("lens")
    M = sum(lens) if lens is not None else B * S
    p_h, seed, li = cfg["p_h"], cfg["seed"], cfg["layer_index"]
    hd = p_h > 0
    dev = x.device
    C = _Checks(what)
    W = {k: prm[k].double() for k in PARAMS}
    v2 = lambda t, n: t.reshape(M, n)
    x, dy, x1, g, ctx = v2(x, H), v2(dy, H), v2(acts["x1"], H), v2(acts["g"], I), v2(acts["ctx"], H)
    pre1, pre2, qkv = v2(acts["pre1"], H), v2(acts["pre2"], H), v2(acts["qkv"], 3 * H)
    mean1, rstd1, mean2, rstd2 = (acts[k].reshape(M) for k in ("mean1", "rstd1", "mean2", "rstd2"))
    keep1, s1 = hidden_keep(seed, drop_stream(li, SITE_ATTN_OUT), M, H, p_h, dev)
    keep2, s2 = hidden_keep(seed, drop_stream(li, SITE_FFN_OUT), M, H, p_h, dev)
    x64, x164, g64, ctx64 = x.double(), x1.double(), g.double(), ctx.double()

    # ---- forward ----
    acc, mag = _gemm(x64, W["w_qkv"], W["b_qkv"])
    C.add("qkv", qkv, acc, GR.bound(acc, mag, True))
    acc, mag = _gemm(ctx64, W["w_attn_out"], W["b_attn_out"])
    _dropout_resid(C, "pre1", pre1, acc, mag, keep1, s1, x)
    for tag, pre, mean, rstd, out, gam, bet in (("1", pre1, mean1, rstd1, x1, "ln1_gamma", "ln1_beta"),
                                                ("2", pre2, mean2, rstd2, v2(acts["y"], H), "ln2_gamma", "ln2_beta")):
        ref, lmag, stats = RR.ln_fwd_ref(pre, prm[gam], prm[bet])
        C.add("x1" if tag == "1" else "y", out, ref, RR.ln_fwd_bound(ref, lmag))
        mu, r, ax = stats
        C.add(f"mean{tag}", mean, mu, RR.C_LN * ax)
        C.add(f"rstd{tag}", rstd, r, RR.C_LN * r)
    acc, mag = _gemm(x164, W["w_inter"], W["b_inter"])
    gp = GR.untile(acts["u"], M, I) if GR.gp_tiled_ok(M, I) else acts["u"].reshape(M, I)
    approx = GR.GELU_APPROX * (1.0 + acc.abs())
    C.add("u (gelu')", gp, GR.gelu_prime64(acc), GR.bound(GR.gelu_prime64(acc), GR.GELU_LIP * mag, True, approx))
    C.add("g", g, GR.gelu64(acc), GR.bound(GR.gelu64(acc), GR.GELU_LIP * mag, True, approx))
    del acc, mag, approx
    acc, mag = _gemm(g64, W["w_out"], W["b_out"])
    _dropout_resid(C, "pre2", pre2, acc, mag, keep2, s2, x1)
    del acc, mag

    # ---- backward: LN2 and the FFN, from fp64 recomputations of the buffers LN1 and the attention backward rewrite ----
    r2 = RR.ln_bwd_ref(dy, pre2, mean2, rstd2, prm["ln2_gamma"])
    _ln_bwd_stage(C, "LN2", r2, keep2, s2, hd, None, None, grads, prefill, ("dln2_gamma", "dln2_beta", "db_out"))
    kd2 = keep2.double() * s2 if hd else torch.ones_like(r2["dx"])
    dpm2 = r2["dx"] * kd2
    B2 = RR.ln_bwd_bound(r2["dx"], r2["mag"], s2) * (kd2 != 0)          # dropped elements are exactly 0
    Bpre2 = RR.ln_bwd_bound(r2["dx"], r2["mag"])                          # LN2's d_pre, the residual addend of d_x1
    P = prefill["dw_out"].double()
    C.add("dw_out", grads["dw_out"], P + dpm2.t() @ g64, GR.C_ACC * (P.abs() + dpm2.abs().t() @ g64.abs()) + B2.t() @ g64.abs())
    gp64 = gp.double()
    dgl = dpm2 @ W["w_out"]
    d_u = dgl * gp64
    Bu = GR.REL_BF16 * d_u.abs() + (GR.C_ACC * (dpm2.abs() @ W["w_out"].abs()) + B2 @ W["w_out"].abs()) * gp64.abs()
    del dgl
    d_big = scr["d_big"].reshape(-1)
    if I > 3 * H:   # the rows of d_u the attention backward's dqkv does not overwrite
        C.add("d_u (d_big past dqkv)", d_big[M * 3 * H:M * I], d_u.reshape(-1)[M * 3 * H:], Bu.reshape(-1)[M * 3 * H:])
    P = prefill["db_inter"].double()
    C.add("db_inter", grads["db_inter"], P + d_u.sum(0), RR.colsum_bound(P, d_u.abs(), Bu.sum(0)))
    P = prefill["dw_inter"].double()
    C.add("dw_inter", grads["dw_inter"], P + d_u.t() @ x164,
          GR.C_ACC * (P.abs() + d_u.abs().t() @ x164.abs()) + Bu.t() @ x164.abs())
    ref = d_u @ W["w_inter"] + r2["dx"]
    C.add("d_x1", v2(scr["d_x1"], H), ref, GR.REL_BF16 * ref.abs() + GR.C_ACC * (d_u.abs() @ W["w_inter"].abs() + r2["dx"].abs())
          + Bu @ W["w_inter"].abs() + Bpre2)
    del d_u, Bu, r2, dpm2, B2, Bpre2, ref

    # ---- backward: LN1 and the attention, from the library's buffers ----
    d_pre = v2(scr["d_pre"], H)
    d_pre_drop = v2(scr["d_pre_drop"], H) if scr.get("d_pre_drop") is not None else None
    r1 = RR.ln_bwd_ref(v2(scr["d_x1"], H), pre1, mean1, rstd1, prm["ln1_gamma"])
    _ln_bwd_stage(C, "LN1", r1, keep1, s1, hd, d_pre, d_pre_drop, grads, prefill, ("dln1_gamma", "dln1_beta", "db_attn_out"))
    del r1
    dpm1 = (d_pre_drop if hd else d_pre).double()
    P = prefill["dw_attn_out"].double()
    C.add("dw_attn_out", grads["dw_attn_out"], P + dpm1.t() @ ctx64, GR.C_ACC * (P.abs() + dpm1.abs().t() @ ctx64.abs()))
    acc, mag = dpm1 @ W["w_attn_out"], dpm1.abs() @ W["w_attn_out"].abs()
    d_ctx = v2(scr["d_ctx"], H)
    C.add("d_ctx", d_ctx, acc, GR.bound(acc, mag, True))
    del dpm1, acc, mag
    dqkv = d_big[:M * 3 * H].view(M, 3 * H)
    _attention(C, cfg, qkv, ctx, acts["lse"], acts.get("keep"), d_ctx, scr["drow"], dqkv)
    dq64 = dqkv.double()
    P = prefill["db_qkv"].double()
    C.add("db_qkv", grads["db_qkv"], P + dq64.sum(0), RR.colsum_bound(P, dq64.abs()))
    P = prefill["dw_qkv"].double()
    C.add("dw_qkv", grads["dw_qkv"], P + dq64.t() @ x64, GR.C_ACC * (P.abs() + dq64.abs().t() @ x64.abs()))
    if dx is not None:
        dp64 = d_pre.double()
        ref = dq64 @ W["w_qkv"] + dp64
        C.add("dx", v2(dx, H), ref, GR.bound(ref, dq64.abs() @ W["w_qkv"].abs() + dp64.abs(), True))
    if strict:
        C.raise_if_bad()
    return C.worst
