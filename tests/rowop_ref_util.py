"""Reference arithmetic and error bounds of the row-kernel tests (test_rowop_reference_gpu.py, test_rowop_reference_cpu.py): the
LayerNorm forward and backward, the embedding, the column sum, the cross-entropy and the casts.

Every reference is fp64 and starts from the exact operands a kernel reads: the bf16 inputs, the fp32 mean / rstd the forward wrote
(for the backward), and the bf16 pre / d_pre / vis_proj the call itself wrote wherever an earlier stage's rounding is not what is
under test. An element passes when |out - ref| <= bound:

- LayerNorm forward, y = gamma xhat + beta:  REL_BF16 |ref| + C_LN (|gamma| (|xhat| + mean|x| rstd) + |beta|).
  REL_BF16 = 2^-8 is one rounding to bf16. C_LN covers the fp32 statistics and rsqrtf: an error of the fp32 mean is relative to
  the row's mean |x|, so it moves xhat by a multiple of mean|x| rstd (large for a row whose mean is much larger than its spread);
  the rstd error is relative, so it moves y by a multiple of |gamma| |xhat|. The same bound, with the row's fp32 mean and rstd
  against fp64: |mean - ref| <= C_LN mean|x|, |rstd - ref| <= C_LN rstd.
- LayerNorm backward, dx = rstd (g - mean(g) - xhat mean(g xhat)), g = dy' gamma (dy' = dy, or dy * keep * scale when the
  dropout that followed the LayerNorm is re-applied): REL_BF16 |ref| + C_LN rstd (|g| + mean|g| + |xhat| mean|g xhat|);
  dx_drop = dx * scale on kept elements with the bound times scale, exact +0 on dropped ones.
- Column sums (dgamma, dbeta, dbias, vb_colsum_bf16, the embedding tables, db_proj) are accumulated into a prefilled fp32 output
  and must come back as prefill + sum: C_SUM (|prefill| + sum |terms|), the recursive-summation bound (n - 1) 2^-24 of fp32
  additions with the depth n of the kernels' register / shared-memory / atomic sums folded into C_SUM; plus, where a term is
  itself an fp32 result (dgamma's dy xhat, dbias's dx), the sum of that term's own bound.
- Cross-entropy: |lse - ref| and |loss - ref| <= C_EXP (1 + |lse|) (ex2.approx.ftz, logf and the fp32 rounding of
  lse * log2 e, which is relative to |lse|); gradient (softmax - onehot) * scale: REL_BF16 |ref| + C_EXP |scale| (1 + |lse|).
- Exact: the casts (round to nearest even; NaN stays NaN), vb_mask_bias, the d_vis copy, and every dropped element.

Choosing the constants: from the fp32 outputs of test_rowop_reference_gpu.py on an H100 SXM (80 GB HBM3, 700 W power limit),
where no bf16 rounding hides them. The largest |mean - ref| / (mean|x|) and |rstd - ref| / rstd was about 2^-21.3 (C_LN = 2^-16:
~40x headroom); the largest column-sum error / (|prefill| + sum |terms|) about 2^-22.5 (C_SUM = 2^-17: ~45x); the largest
lse / loss error / (1 + |lse|) about 2^-23 (C_EXP = 2^-18: ~30x). In the bf16 outputs the one rounding dominates and their worst
ratio is close to 1 by construction. The planted bugs of test_rowop_reference_cpu.py exceed these bounds by orders of magnitude.
"""
import torch

REL_BF16 = 2.0 ** -8
C_LN = 2.0 ** -16
C_SUM = 2.0 ** -17
C_EXP = 2.0 ** -18
LN_EPS = 1e-12
EMBED_DROP_STREAM = 0xE0000001       # vb_api.cu kEmbedDropStream: the embeddings' dropout and the in_dropout of their backward


def _ratio(out, ref, bound, what):
    out = out.double()
    assert torch.isfinite(out).all(), f"{what}: {int((~torch.isfinite(out)).sum())} non-finite elements"
    err = (out - ref).abs()
    ratio = err / (bound + 1e-300)
    worst = float(ratio.max()) if ratio.numel() else 0.0
    if worst > 1.0:
        idx = tuple(int(i) for i in torch.nonzero(ratio == ratio.max())[0])
        n_bad = int((ratio > 1).sum())
        raise AssertionError(f"{what}: {n_bad} of {ratio.numel()} elements outside the bound; worst at {idx}: "
                             f"out {float(out[idx]):.6g} ref {float(ref[idx]):.6g} bound {float(bound[idx]):.3g}")
    return worst


def check(out, ref, bound, what):
    """Assert |out - ref| <= bound element by element (fp64 ref and bound of out's shape); returns the largest error / bound."""
    return _ratio(out, ref, bound, what)


def check_bits(out, want, what):
    """out and want bit for bit (same dtype)."""
    it = {2: torch.int16, 4: torch.int32, 8: torch.int64}[out.element_size()]
    n_bad = int((out.reshape(-1).view(it) != want.reshape(-1).view(it)).sum())
    assert n_bad == 0, f"{what}: {n_bad} of {out.numel()} elements differ bit for bit"


# ---- LayerNorm ---------------------------------------------------------------------------------------------------------------
def ln_stats(x):
    """fp64 mean, rstd (biased variance, eps inside the sqrt) and mean |x| of the rows of x."""
    x = x.double()
    mu = x.mean(-1)
    rstd = 1.0 / torch.sqrt(((x - mu[..., None]) ** 2).mean(-1) + LN_EPS)
    return mu, rstd, x.abs().mean(-1)


def ln_fwd_ref(x, gamma, beta):
    """-> ref y, its bound's magnitude term (C_LN multiplies it) and the fp64 stats (mean, rstd, mean|x|)."""
    mu, rstd, ax = ln_stats(x)
    xh = (x.double() - mu[:, None]) * rstd[:, None]
    g, b = gamma.double(), beta.double()
    ref = g * xh + b
    mag = g.abs() * (xh.abs() + (ax * rstd)[:, None]) + b.abs()
    return ref, mag, (mu, rstd, ax)


def ln_fwd_bound(ref, mag, scale=1.0):
    return REL_BF16 * ref.abs() + C_LN * scale * mag


def check_stats(mean, rstd, stats, what):
    mu, r, ax = stats
    return max(check(mean, mu, C_LN * ax, what + " mean"), check(rstd, r, C_LN * r, what + " rstd"))


def ln_bwd_ref(dy, x, mean, rstd, gamma, in_keep=None, in_scale=1.0):
    """fp64 LayerNorm backward from the kernel's operands (bf16 dy, x; the fp32 mean, rstd the forward wrote). in_keep: the keep
    mask of the dropout that followed the LayerNorm. -> dict of ref dx, its magnitude term, and the column-sum terms with their
    magnitudes (dgamma: dy' xhat, dbeta: dy')."""
    mu, rs = mean.double()[:, None], rstd.double()[:, None]
    xh = (x.double() - mu) * rs
    d = dy.double()
    if in_keep is not None:
        d = torch.where(in_keep, d * in_scale, torch.zeros_like(d))
    g = d * gamma.double()
    H = x.shape[1]
    c1, c2 = g.mean(1, keepdim=True), (g * xh).mean(1, keepdim=True)
    dx = rs * (g - c1 - xh * c2)
    mag = rs * (g.abs() + g.abs().mean(1, keepdim=True) + xh.abs() * (g * xh).abs().sum(1, keepdim=True) / H)
    # the kernel's xhat = fma(x, rstd, -mean * rstd) in fp32: off by ~2^-24 (|xhat| + |mean| rstd)
    return dict(dx=dx, mag=mag, dgamma=d * xh, dgamma_mag=d.abs() * (xh.abs() + mu.abs() * rs), dbeta=d, dbeta_mag=d.abs())


def ln_bwd_bound(ref, mag, scale=1.0):
    return REL_BF16 * ref.abs() * scale + C_LN * scale * mag


def colsum_bound(prefill, term_mag, extra=None):
    """bound of prefill + sum(terms, dim 0): C_SUM (|prefill| + sum |terms|) (+ extra, the summed bounds of fp32 terms)."""
    b = C_SUM * (prefill.double().abs() + term_mag.sum(0))
    return b if extra is None else b + extra


def check_dropout_rows(out, ref, mag, keep, scale, what):
    """out = keep ? bf16(ref * scale) : +0 — kept within ln_bwd_bound * scale, dropped exactly +0. Returns the worst kept ratio."""
    worst = check(out[keep], ref[keep] * scale, ln_bwd_bound(ref[keep], mag[keep], scale), what + " (kept)")
    check_bits(out[~keep], torch.zeros_like(out[~keep]), what + " (dropped)")
    return worst


# ---- cross-entropy -----------------------------------------------------------------------------------------------------------
def ce_ref(logits, labels, vocab):
    """logits bf16 [rows, >= vocab]; -> fp64 lse, loss (0 for labels outside [0, vocab)), softmax [rows, vocab], valid mask."""
    z = logits[:, :vocab].double()
    lse = torch.logsumexp(z, 1)
    valid = (labels >= 0) & (labels < vocab)
    lab = labels.clamp(0, vocab - 1)
    loss = torch.where(valid, lse - z.gather(1, lab[:, None])[:, 0], torch.zeros_like(lse))
    return lse, loss, torch.exp(z - lse[:, None]), valid


def ce_grad_ref(p, labels, valid, scale):
    """(softmax - onehot) * scale on valid rows, 0 on ignored ones (fp64 [rows, vocab])."""
    g = p.clone()
    rows = torch.nonzero(valid)[:, 0]
    g[rows, labels[rows]] -= 1.0
    g[~valid] = 0.0
    return g * scale


def ce_lse_bound(lse):
    return C_EXP * (1.0 + lse.abs())


def ce_grad_bound(ref, lse, scale):
    return REL_BF16 * ref.abs() + C_EXP * abs(scale) * (1.0 + lse.abs())[:, None]


# ---- casts -------------------------------------------------------------------------------------------------------------------
def bf16_bits_rne(x):
    """fp32 tensor -> int16 bit patterns of its round-to-nearest-even bf16 (NaN inputs give 0x7FC0; compare those as NaN)."""
    b = x.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    r = (b + 0x7FFF + ((b >> 16) & 1)) >> 16
    nan = torch.isnan(x)
    r = torch.where(nan, torch.full_like(r, 0x7FC0), r) & 0xFFFF
    return torch.where(r >= 0x8000, r - 0x10000, r).to(torch.int16)


def check_cast_bf16(out, src, what):
    """out (bf16) is the round-to-nearest-even bf16 of src (fp32) bit for bit; NaN inputs must give a NaN."""
    nan = torch.isnan(src)
    want = bf16_bits_rne(src)
    got = out.view(torch.int16)
    n_bad = int((got[~nan] != want[~nan]).sum())
    assert n_bad == 0, f"{what}: {n_bad} of {int((~nan).sum())} elements are not the round-to-nearest-even bf16"
    assert bool(torch.isnan(out[nan].float()).all()), f"{what}: a NaN input did not give a NaN"


def cast_edge_values():
    """fp32 values where a cast to bf16 goes wrong: ties to even both ways, a round-up into the next exponent (and to Inf),
    subnormals, signed zeros, +-Inf and NaNs."""
    bits = [0x3F808000, 0x3F818000, 0x3F80C000, 0x3F807FFF, 0x3FFFFFFF, 0x3FFF8000, 0x7F7FFFFF, 0x7F7F8000, 0xFF7FFFFF,
            0x00000001, 0x00008000, 0x00018000, 0x007FFFFF, 0x80000001, 0x807F8000, 0x00000000, 0x80000000,
            0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00001, 0x7F800001, 0x3F7FFFFF, 0xBF808001]
    t = torch.tensor(bits, dtype=torch.int64)
    return torch.where(t >= 2 ** 31, t - 2 ** 32, t).to(torch.int32).view(torch.float32)
