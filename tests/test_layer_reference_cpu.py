"""The stage-by-stage layer check (layer_ref_util.py) is tight enough to catch the glue bugs it exists for.

A correct "library result" of one layer call is built on the host: fp32 arithmetic rounded to bf16 at every stage boundary, as
the kernels do, with the hidden-dropout masks of dropout_util and random attention keep bits packed into the keep buffer's
layout. Three shapes: a dense layer (B = 2, S = 70, A = 2, a partial last key block, ragged mask), one whose gelu'(u) is stored
tile-native (M = 256, I = 512) and an unpadded one with an empty sequence. The checker accepts each, with and without dropout.

Each glue bug below is then planted in one buffer of a correct result, and the checker must reject it. The smallest
error / bound among them is about 19: d_x1 without LN2's residual, whose bound carries the propagated bounds of the recomputed
d_u and d_pre. dw_out from d_pre instead of d_pre_drop reaches about 90, and every other bug 8000 or more. The swapped
dropout sites and the streams that ignore layer_index change dropped elements, which must match bit for bit, so they report
inf. The test asserts a margin of 10 for every bug.
"""
import math
import re

import pytest
import torch

import attn_ref_util as AR
import gemm_ref_util as GR
from dropout_util import hidden_keep
from layer_ref_util import GRADS, check_layer, drop_stream

BF = torch.bfloat16
SEED = 0x1234567890ABCDEF
MARGIN = 10.0


def tile_native(t, M, N):
    """row-major [M, N] -> the tile-native layout gemm_ref_util.untile decodes."""
    return t.reshape(M // 256, 2, 4, 32, N // 256, 2, 8, 16).permute(0, 4, 1, 5, 2, 6, 3, 7).reshape(M, N)


def _cfg(shape, p):
    if shape == "dense":
        cfg = dict(B=2, S=70, A=2, layer_index=3)
    elif shape == "tiled":
        cfg = dict(B=2, S=128, A=2, layer_index=5)
    else:
        cfg = dict(B=3, S=70, A=2, layer_index=11, lens=(70, 0, 33))
    cfg.update(I=256 * cfg["A"], p_h=p, p_a=p, seed=SEED)
    if shape != "unpadded":
        B, S = cfg["B"], cfg["S"]
        valid = torch.arange(S)[None, :] < torch.tensor([[S], [S - 23]])
        cfg["mask_bias"] = ((~valid).float() * -10000.0).contiguous()
    return cfg


def _params(H, I, g):
    r = lambda *s, sc=1.0: sc * torch.randn(*s, generator=g)
    return dict(w_qkv=r(3 * H, H, sc=0.05).to(BF), b_qkv=r(3 * H, sc=0.1), w_attn_out=r(H, H, sc=0.05).to(BF), b_attn_out=r(H, sc=0.1),
                ln1_gamma=1 + r(H, sc=0.1), ln1_beta=r(H, sc=0.1), w_inter=r(I, H, sc=0.05).to(BF), b_inter=r(I, sc=0.1),
                w_out=r(H, I, sc=0.05).to(BF), b_out=r(H, sc=0.1), ln2_gamma=1 + r(H, sc=0.1), ln2_beta=r(H, sc=0.1))


def _keep_buffer(BA, S, p, g):
    """A keep buffer holding random bits (keep probability 1 - round(256 p) / 256), rows = queries in half 0, the transpose in
    half 1, as attn_ref_util.keep_bits reads it."""
    nkb = (S + 63) // 64
    bits = (torch.randint(0, 256, (BA, nkb * 64, nkb * 64), generator=g) >= int(p * 256 + 0.5)).long()
    shifts = torch.arange(64)

    def pack(b):
        return (b.view(BA, nkb * 64, nkb, 64) << shifts).sum(-1)   # int64 wraps at bit 63 like the stored word

    return torch.stack([pack(bits), pack(bits.transpose(1, 2).contiguous())]).reshape(-1).view(torch.uint8)


def _ln32(x, gamma, beta):
    mean = x.mean(1)
    rstd = torch.rsqrt(((x - mean[:, None]) ** 2).mean(1) + 1e-12)
    return ((x - mean[:, None]) * rstd[:, None] * gamma + beta).to(BF), mean, rstd


def _ln_bwd32(dy, x, mean, rstd, gamma):
    xh = (x - mean[:, None]) * rstd[:, None]
    gg = dy * gamma
    return rstd[:, None] * (gg - gg.mean(1, keepdim=True) - xh * (gg * xh).mean(1, keepdim=True)), dy * xh


def _groups(cfg):
    """(sequence or None, first row, rows) of each attention problem: the dense batch, or one per non-empty sequence."""
    B, S, A = cfg["B"], cfg["S"], cfg["A"]
    if cfg.get("lens") is None:
        return [(None, 0, B * S)]
    out, r = [], 0
    for b, n in enumerate(cfg["lens"]):
        if n:
            out.append((b, r, n))
        r += n
    return out


def _heads(t, cfg, grp):
    B, S, A = cfg["B"], cfg["S"], cfg["A"]
    b, r, n = grp
    return AR.dense_heads(t, B, S, A) if b is None else AR.varlen_heads(t, r, n, A)


def _rows(h, cfg, grp):
    """[c, N, n, 64] heads -> [rows, c H], the inverse of _heads."""
    B, S, A = cfg["B"], cfg["S"], cfg["A"]
    b, r, n = grp
    c = h.shape[0]
    if b is None:
        return h.reshape(c, B, A, S, 64).permute(1, 3, 0, 2, 4).reshape(B * S, c * A * 64)
    return h.permute(2, 0, 1, 3).reshape(n, c * A * 64)


def simulate(cfg, prm, x, dy, prefill, keep_buf):
    """The layer call as the library computes it: fp32 stages, bf16 at every stage boundary. -> (acts, scratch, grads, dx,
    intermediates the planted bugs reuse)."""
    B, S, A, I = cfg["B"], cfg["S"], cfg["A"], cfg["I"]
    H, lens = 64 * A, cfg.get("lens")
    M = sum(lens) if lens is not None else B * S
    p_h, p_a, li = cfg["p_h"], cfg["p_a"], cfg["layer_index"]
    hd = p_h > 0
    W = {k: v.float() for k, v in prm.items()}
    xf = x.float()
    k1, s1 = hidden_keep(SEED, drop_stream(li, 1), M, H, p_h, "cpu")
    k2, s2 = hidden_keep(SEED, drop_stream(li, 2), M, H, p_h, "cpu")
    qkv = (xf @ W["w_qkv"].t() + W["b_qkv"]).to(BF)
    scale = AR.drop_scale(p_a)
    bits = AR.keep_bits(keep_buf, B * A, S) if p_a > 0 else None
    ctx, lse = torch.empty(M, H, dtype=BF), torch.empty(A * M)
    saved = []
    for grp in _groups(cfg):
        b, r, n = grp
        q, k, v = _heads(qkv, cfg, grp).float()
        if b is None:
            bias = cfg["mask_bias"].repeat_interleave(A, 0)[:, None, :]
            kb = bits.float() * scale if bits is not None else 1.0
        else:
            bias = 0.0
            kb = bits[b * A:(b + 1) * A, :n, :n].float() * scale if bits is not None else 1.0
        s = q @ k.transpose(-1, -2) / 8.0 + bias
        ls = torch.logsumexp(s, -1)
        P = torch.exp(s - ls[..., None])
        o = ((P * kb) @ v).to(BF)
        if b is None:
            ctx[:] = _rows(o[None], cfg, grp)
            lse[:] = ls.reshape(-1)
        else:
            ctx[r:r + n] = _rows(o[None], cfg, grp)
            lse.view(A, M)[:, r:r + n] = ls
        saved.append((grp, q, k, v, P, kb))
    pre1 = torch.where(k1, (ctx.float() @ W["w_attn_out"].t() + W["b_attn_out"]) * s1 + xf, xf).to(BF)
    x1, mean1, rstd1 = _ln32(pre1.float(), W["ln1_gamma"], W["ln1_beta"])
    u = x1.float() @ W["w_inter"].t() + W["b_inter"]
    gp = (0.5 * (1 + torch.erf(u / math.sqrt(2))) + u * torch.exp(-0.5 * u * u) / math.sqrt(2 * math.pi)).to(BF)
    g = (0.5 * u * (1 + torch.erf(u / math.sqrt(2)))).to(BF)
    acc2 = g.float() @ W["w_out"].t() + W["b_out"]
    pre2 = torch.where(k2, acc2 * s2 + x1.float(), x1.float()).to(BF)
    y, mean2, rstd2 = _ln32(pre2.float(), W["ln2_gamma"], W["ln2_beta"])
    acts = dict(qkv=qkv, ctx=ctx, lse=lse, pre1=pre1, mean1=mean1, rstd1=rstd1, x1=x1,
                u=tile_native(gp, M, I) if GR.gp_tiled_ok(M, I) else gp, g=g, pre2=pre2, mean2=mean2, rstd2=rstd2,
                keep=keep_buf if p_a > 0 else None, y=y)

    G = {k: v.clone() for k, v in prefill.items()}
    kd1, kd2 = (k1.float() * s1, k2.float() * s2) if hd else (1.0, 1.0)
    drop = lambda t, k, sc: torch.where(k, t * sc, torch.zeros_like(t))   # dropped elements are +0, not -0
    dp2, dg2 = _ln_bwd32(dy.float(), pre2.float(), mean2, rstd2, W["ln2_gamma"])
    G["dln2_gamma"] += dg2.sum(0); G["dln2_beta"] += dy.float().sum(0); G["db_out"] += (dp2 * kd2).sum(0)
    d_pre2 = dp2.to(BF)
    dpm2 = drop(dp2, k2, s2).to(BF) if hd else d_pre2
    G["dw_out"] += dpm2.float().t() @ g.float()
    dgl = dpm2.float() @ W["w_out"]
    d_u = (dgl * gp.float()).to(BF)
    G["db_inter"] += d_u.float().sum(0)
    G["dw_inter"] += d_u.float().t() @ x1.float()
    d_x1 = (d_u.float() @ W["w_inter"] + d_pre2.float()).to(BF)
    dp1, dg1 = _ln_bwd32(d_x1.float(), pre1.float(), mean1, rstd1, W["ln1_gamma"])
    G["dln1_gamma"] += dg1.sum(0); G["dln1_beta"] += d_x1.float().sum(0); G["db_attn_out"] += (dp1 * kd1).sum(0)
    d_pre = dp1.to(BF)
    d_pre_drop = drop(dp1, k1, s1).to(BF) if hd else None
    dpm1 = d_pre_drop if hd else d_pre
    G["dw_attn_out"] += dpm1.float().t() @ ctx.float()
    d_ctx = (dpm1.float() @ W["w_attn_out"]).to(BF)
    dqkv, drow = torch.empty(M, 3 * H, dtype=BF), torch.empty(A * M)
    for grp, q, k, v, P, kb in saved:
        b, r, n = grp
        dO, c = _heads(d_ctx, cfg, grp)[0].float(), _heads(ctx, cfg, grp)[0].float()
        D = (dO * c).sum(-1)
        dS = P * (kb * (dO @ v.transpose(-1, -2)) - D[..., None])
        h = torch.stack([dS @ k / 8.0, dS.transpose(-1, -2) @ q / 8.0, (P * kb).transpose(-1, -2) @ dO]).to(BF)
        if b is None:
            dqkv[:] = _rows(h, cfg, grp)
            drow[:] = D.reshape(-1)
        else:
            dqkv[r:r + n] = _rows(h, cfg, grp)
            drow.view(A, M)[:, r:r + n] = D
    d_big = torch.empty(M * max(I, 3 * H), dtype=BF)
    d_big[:M * I] = d_u.reshape(-1)
    d_big[:M * 3 * H] = dqkv.reshape(-1)
    G["db_qkv"] += dqkv.float().sum(0)
    G["dw_qkv"] += dqkv.float().t() @ xf
    dx = (dqkv.float() @ W["w_qkv"] + d_pre.float()).to(BF)
    scr = dict(d_pre=d_pre, d_pre_drop=d_pre_drop, d_big=d_big, d_x1=d_x1, d_ctx=d_ctx, drow=drow)
    inter = dict(d_pre2=d_pre2, dgl=dgl, d_u=d_u, dqkv=dqkv, acc2=acc2, M=M, H=H)
    return acts, scr, G, dx, inter


def _case(shape, p):
    cfg = _cfg(shape, p)
    g = torch.Generator().manual_seed(7)
    A, I = cfg["A"], cfg["I"]
    H = 64 * A
    M = sum(cfg["lens"]) if "lens" in cfg else cfg["B"] * cfg["S"]
    prm = _params(H, I, g)
    x, dy = torch.randn(M, H, generator=g).to(BF), torch.randn(M, H, generator=g).to(BF)
    sizes = dict(dw_qkv=(3 * H, H), db_qkv=(3 * H,), dw_attn_out=(H, H), db_attn_out=(H,), dln1_gamma=(H,), dln1_beta=(H,),
                 dw_inter=(I, H), db_inter=(I,), dw_out=(H, I), db_out=(H,), dln2_gamma=(H,), dln2_beta=(H,))
    prefill = {k: torch.randn(*sizes[k], generator=g) for k in GRADS}
    keep_buf = _keep_buffer(cfg["B"] * A, cfg["S"], cfg["p_a"], g)
    acts, scr, G, dx, inter = simulate(cfg, prm, x, dy, prefill, keep_buf)
    return cfg, prm, x, dy, prefill, keep_buf, acts, scr, G, dx, inter


@pytest.mark.parametrize("p", [0.1, 0.0])
@pytest.mark.parametrize("shape", ["dense", "tiled", "unpadded"])
def test_checker_accepts_the_correct_result(shape, p):
    cfg, prm, x, dy, prefill, _, acts, scr, G, dx, _ = _case(shape, p)
    worst = check_layer(cfg, prm, x, dy, acts, scr, G, prefill, dx, what=f"{shape} p={p}")
    print(f"\n{shape} p={p}: " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))
    assert set(worst) >= {"qkv", "ctx", "lse", "pre1", "x1", "u (gelu')", "g", "pre2", "y", "dw_out", "db_inter", "dw_inter",
                          "d_x1", "d_pre (LN1)", "dw_attn_out", "d_ctx", "drow", "dqkv", "db_qkv", "dw_qkv", "dx"} | set(GRADS)


def _bug_sites_swapped(c):
    cfg, prm, x, acts, inter = c["cfg"], c["prm"], c["x"], c["acts"], c["inter"]
    k, s = hidden_keep(SEED, drop_stream(cfg["layer_index"], 2), inter["M"], inter["H"], cfg["p_h"], "cpu")
    acc = acts["ctx"].float() @ prm["w_attn_out"].float().t() + prm["b_attn_out"]
    acts["pre1"] = torch.where(k, acc * s + x.float(), x.float()).to(BF)
    return "pre1"


def _bug_streams_ignore_layer(c):
    cfg, acts, inter = c["cfg"], c["acts"], c["inter"]
    k, s = hidden_keep(SEED, 2, inter["M"], inter["H"], cfg["p_h"], "cpu")
    acts["pre2"] = torch.where(k, inter["acc2"] * s + acts["x1"].float(), acts["x1"].float()).to(BF)
    return "pre2"


def _bug_dx_without_residual(c):
    c["dx"] = (c["inter"]["dqkv"].float() @ c["prm"]["w_qkv"].float()).to(BF)
    return "dx"


def _bug_d_x1_without_residual(c):
    c["scr"]["d_x1"] = (c["inter"]["d_u"].float() @ c["prm"]["w_inter"].float()).to(BF)
    return "d_x1"


def _bug_dw_out_from_d_pre(c):
    c["G"]["dw_out"] = c["prefill"]["dw_out"] + c["inter"]["d_pre2"].float().t() @ c["acts"]["g"].float()
    return "dw_out"


def _bug_db_qkv_row_stride_I(c):
    M, H, I = c["inter"]["M"], c["inter"]["H"], c["cfg"]["I"]
    c["G"]["db_qkv"] = c["prefill"]["db_qkv"] + c["scr"]["d_big"][:M * I].view(M, I)[:, :3 * H].float().sum(0)
    return "db_qkv"


def _bug_gelu_prime_read_row_major(c):
    """the backward's DGELU epilogue reads the tile-native gelu'(u) as if it were row-major: d_u, in d_big"""
    M, H, I = c["inter"]["M"], c["inter"]["H"], c["cfg"]["I"]
    d_u = (c["inter"]["dgl"] * c["acts"]["u"].reshape(M, I).float()).to(BF)
    c["scr"]["d_big"][M * 3 * H:M * I] = d_u.reshape(-1)[M * 3 * H:]
    return "d_u (d_big past dqkv)"


def _bug_drow_delta_seq(c):
    """unpadded EPI_DELTA with delta_seq = seq: row q of head h lands at h * seq + q of the [A, total] buffer"""
    cfg, inter = c["cfg"], c["inter"]
    A, S, M = cfg["A"], cfg["S"], inter["M"]
    D = c["scr"]["drow"].view(A, M).clone()
    bad = torch.zeros(A * M)
    for h in range(A):
        idx = h * S + torch.arange(M)
        ok = idx < A * M
        bad[idx[ok]] = D[h, ok]
    c["scr"]["drow"] = bad
    return "drow"


def _bug_ln2_stats_of_neighbour(c):
    """mean2 / rstd2 of the next layer (other weights, run on this layer's output)"""
    prm2 = _params(c["inter"]["H"], c["cfg"]["I"], torch.Generator().manual_seed(99))
    acts2 = simulate(c["cfg"], prm2, c["acts"]["y"], c["dy"], c["prefill"], c["keep_buf"])[0]
    c["acts"]["mean2"], c["acts"]["rstd2"] = acts2["mean2"], acts2["rstd2"]
    return "mean2"


def _bug_gradient_overwritten(c):
    c["G"]["dw_attn_out"] = c["G"]["dw_attn_out"] - c["prefill"]["dw_attn_out"]
    return "dw_attn_out"


BUGS = [("dense", _bug_sites_swapped), ("dense", _bug_streams_ignore_layer), ("dense", _bug_dx_without_residual),
        ("dense", _bug_d_x1_without_residual), ("dense", _bug_dw_out_from_d_pre), ("dense", _bug_db_qkv_row_stride_I),
        ("tiled", _bug_gelu_prime_read_row_major), ("unpadded", _bug_drow_delta_seq), ("dense", _bug_ln2_stats_of_neighbour),
        ("tiled", _bug_gradient_overwritten)]


@pytest.mark.parametrize("shape,bug", BUGS, ids=[b.__name__[5:] for _, b in BUGS])
def test_checker_rejects_a_planted_glue_bug(shape, bug):
    cfg, prm, x, dy, prefill, keep_buf, acts, scr, G, dx, inter = _case(shape, 0.1)
    c = dict(shape=shape, cfg=cfg, prm=prm, x=x, dy=dy, prefill=prefill, keep_buf=keep_buf, acts=acts, scr=scr, G=G, dx=dx,
             inter=inter)
    buf = bug(c)
    worst = check_layer(cfg, prm, x, dy, c["acts"], c["scr"], c["G"], prefill, c["dx"], strict=False)
    print(f"\n{bug.__name__[5:]}: {buf} error / bound {worst[buf]:.3g}")
    assert worst[buf] > MARGIN, f"{bug.__name__}: {buf} only {worst[buf]:.3g} x its bound"
    with pytest.raises(AssertionError, match=re.escape(buf)):
        check_layer(cfg, prm, x, dy, c["acts"], c["scr"], c["G"], prefill, c["dx"])
