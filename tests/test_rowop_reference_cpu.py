"""The bounds of the row-kernel reference tests (rowop_ref_util.py) are tight enough to catch the bugs those tests exist for. Each
bad result is built on the host from a correct one: a LayerNorm row whose last partial 8-column chunk used a stale mean, one row
of dgamma contributions lost or added twice, one flipped keep bit in dx_drop and in the re-applied in_dropout mask, an embedding
row scattered into the neighbouring table row, a cross-entropy gradient without the onehot or with the scale applied twice, and a
padded column left non-zero. The correct results pass."""
import pytest
import torch

import rowop_ref_util as R
from dropout_util import hidden_keep

SEED_HI = 0xFEDCBA9876543210


def _ln_case(rows=6, H=264):
    g = torch.Generator().manual_seed(H)
    x = (torch.randn(rows, H, generator=g) * 2 + torch.arange(rows)[:, None] * 0.75).bfloat16()
    gamma = 1 + 0.1 * torch.randn(H, generator=g)
    beta = 0.1 * torch.randn(H, generator=g)
    return x, gamma, beta


def _ln_fwd_fp32(x, gamma, beta, mean=None):
    xf = x.float()
    mu = xf.mean(1, keepdim=True) if mean is None else mean
    rs = torch.rsqrt(((xf - xf.mean(1, keepdim=True)) ** 2).mean(1, keepdim=True) + R.LN_EPS)
    return (gamma * ((xf - mu) * rs) + beta).bfloat16(), mu[:, 0], rs[:, 0]


def test_layernorm_forward_bound_accepts_the_kernel_arithmetic():
    x, gamma, beta = _ln_case()
    y, mu, rs = _ln_fwd_fp32(x, gamma, beta)
    ref, mag, stats = R.ln_fwd_ref(x, gamma, beta)
    R.check(y, ref, R.ln_fwd_bound(ref, mag), "y")
    R.check_stats(mu, rs, stats, "stats")


def test_layernorm_forward_bound_rejects_a_stale_mean_in_the_last_partial_chunk():
    """H = 264: chunk 32 (columns 256..263) is the only one of the second register chunk; normalised with the previous row's
    mean it is rejected."""
    x, gamma, beta = _ln_case()
    y, _, _ = _ln_fwd_fp32(x, gamma, beta)
    ref, mag, _ = R.ln_fwd_ref(x, gamma, beta)
    for row in range(1, x.shape[0]):
        stale = x.float().mean(1, keepdim=True).roll(1, 0)
        bad_rows, _, _ = _ln_fwd_fp32(x, gamma, beta, mean=stale)
        bad = y.clone()
        bad[row, 256:] = bad_rows[row, 256:]
        with pytest.raises(AssertionError):
            R.check(bad, ref, R.ln_fwd_bound(ref, mag), f"row {row}")


def _ln_bwd_case(in_drop=False):
    x, gamma, _ = _ln_case(rows=40, H=136)
    g = torch.Generator().manual_seed(5)
    dy = torch.randn(x.shape, generator=g).bfloat16()
    xf = x.float()
    mean = xf.mean(1)
    rstd = torch.rsqrt(((xf - mean[:, None]) ** 2).mean(1) + R.LN_EPS)
    keep, scale = hidden_keep(SEED_HI, R.EMBED_DROP_STREAM, *x.shape, 0.1, "cpu") if in_drop else (None, 1.0)
    d = dy.float() if keep is None else torch.where(keep, dy.float() * scale, torch.zeros(x.shape))
    xh = (xf - mean[:, None]) * rstd[:, None]
    gg = d * gamma
    dx = rstd[:, None] * (gg - gg.mean(1, keepdim=True) - xh * (gg * xh).mean(1, keepdim=True))
    return x, gamma, dy, mean, rstd, keep, scale, d, xh, dx


@pytest.mark.parametrize("in_drop", [False, True])
def test_layernorm_backward_bounds_accept_the_kernel_arithmetic(in_drop):
    x, gamma, dy, mean, rstd, keep, scale, d, xh, dx = _ln_bwd_case(in_drop)
    r = R.ln_bwd_ref(dy, x, mean, rstd, gamma, keep, scale)
    R.check(dx.bfloat16(), r["dx"], R.ln_bwd_bound(r["dx"], r["mag"]), "dx")
    pre = torch.randn(x.shape[1], generator=torch.Generator().manual_seed(1))
    R.check(pre + (d * xh).sum(0), pre.double() + r["dgamma"].sum(0), R.colsum_bound(pre, r["dgamma_mag"]), "dgamma")
    R.check(pre + d.sum(0), pre.double() + r["dbeta"].sum(0), R.colsum_bound(pre, r["dbeta_mag"]), "dbeta")


@pytest.mark.parametrize("twice", [False, True])
def test_dgamma_bound_rejects_a_lost_or_doubled_row(twice):
    x, gamma, dy, mean, rstd, keep, scale, d, xh, dx = _ln_bwd_case()
    r = R.ln_bwd_ref(dy, x, mean, rstd, gamma)
    pre = torch.randn(x.shape[1], generator=torch.Generator().manual_seed(1))
    for row in (0, 17, x.shape[0] - 1):
        terms = d * xh
        bad = pre + terms.sum(0) + (terms[row] if twice else -terms[row])
        with pytest.raises(AssertionError):
            R.check(bad, pre.double() + r["dgamma"].sum(0), R.colsum_bound(pre, r["dgamma_mag"]), f"row {row}")


def test_dropout_checks_reject_one_flipped_keep_bit():
    """dx_drop: a flipped bit either zeroes a kept element or keeps a dropped one. in_dropout: a flipped bit changes dy' at one
    element, which moves dx of that element (and, through the row means, the whole row) outside the bound."""
    x, gamma, dy, mean, rstd, _, _, _, _, dx = _ln_bwd_case()
    r = R.ln_bwd_ref(dy, x, mean, rstd, gamma)
    keep, scale = hidden_keep(SEED_HI, 3, *x.shape, 0.1, "cpu")
    out = torch.where(keep, dx * scale, torch.zeros(x.shape)).bfloat16()
    R.check_dropout_rows(out, r["dx"], r["mag"], keep, scale, "correct mask")
    big = r["dx"].abs() > 0.05
    for was_kept in (True, False):
        i, j = (int(v) for v in torch.nonzero((keep == was_kept) & big)[0])
        flipped = keep.clone()
        flipped[i, j] = not was_kept
        with pytest.raises(AssertionError):
            R.check_dropout_rows(out, r["dx"], r["mag"], flipped, scale, f"dx_drop bit ({i}, {j})")

    x, gamma, dy, mean, rstd, keep, scale, _, _, dx = _ln_bwd_case(in_drop=True)
    r = R.ln_bwd_ref(dy, x, mean, rstd, gamma, keep, scale)
    R.check(dx.bfloat16(), r["dx"], R.ln_bwd_bound(r["dx"], r["mag"]), "correct in_dropout mask")
    for was_kept in (True, False):
        i, j = (int(v) for v in torch.nonzero((keep == was_kept) & (dy.float().abs() > 0.5))[0])
        flipped = keep.clone()
        flipped[i, j] = not was_kept
        rb = R.ln_bwd_ref(dy, x, mean, rstd, gamma, flipped, scale)
        with pytest.raises(AssertionError):
            R.check(dx.bfloat16(), rb["dx"], R.ln_bwd_bound(rb["dx"], rb["mag"]), f"in_dropout bit ({i}, {j})")


def test_table_bound_rejects_a_row_scattered_into_its_neighbour():
    g = torch.Generator().manual_seed(2)
    n_rows, H, vocab = 50, 16, 12
    de = torch.randn(n_rows, H, generator=g).bfloat16()
    ids = torch.randint(0, vocab, (n_rows,), generator=g)
    pre = torch.randn(vocab, H, generator=g)
    d64 = de.double()
    ref = pre.double().index_add(0, ids, d64)
    bound = R.colsum_bound(pre, torch.zeros(vocab, H, dtype=torch.float64).index_add(0, ids, d64.abs())[None])
    good = pre.index_add(0, ids, de.float())
    R.check(good, ref, bound, "correct scatter")
    for k in (0, 23, n_rows - 1):
        wrong = ids.clone()
        wrong[k] = (ids[k] + 1) % vocab
        bad = pre.index_add(0, wrong, de.float())
        with pytest.raises(AssertionError):
            R.check(bad, ref, bound, f"row {k} into table row {int(wrong[k])}")


def _ce_case(vocab=37, rows=9):
    g = torch.Generator().manual_seed(vocab)
    logits = (3 * torch.randn(rows, vocab, generator=g)).bfloat16()
    labels = torch.randint(0, vocab, (rows,), generator=g)
    labels[2] = -100
    return logits, labels, 0.37


def test_cross_entropy_bounds_accept_the_kernel_arithmetic():
    logits, labels, scale = _ce_case()
    lse, loss, p, valid = R.ce_ref(logits, labels, logits.shape[1])
    lf = torch.logsumexp(logits.float(), 1)
    R.check(lf, lse, R.ce_lse_bound(lse), "lse")
    ref = R.ce_grad_ref(p, labels, valid, scale)
    R.check(ref.float().bfloat16(), ref, R.ce_grad_bound(ref, lse, scale), "grad")


@pytest.mark.parametrize("bug", ["no onehot", "scale twice"])
def test_cross_entropy_gradient_bound_rejects(bug):
    logits, labels, scale = _ce_case()
    lse, _, p, valid = R.ce_ref(logits, labels, logits.shape[1])
    ref = R.ce_grad_ref(p, labels, valid, scale)
    bad = p * scale if bug == "no onehot" else ref * scale
    bad[~valid] = 0
    with pytest.raises(AssertionError):
        R.check(bad.float().bfloat16(), ref, R.ce_grad_bound(ref, lse, scale), bug)


def test_padded_column_check_rejects_a_non_zero():
    pad = torch.zeros(4, 7, dtype=torch.bfloat16)
    R.check_bits(pad, torch.zeros_like(pad), "zeros")
    for v in (1e-30, -0.0):   # a denormal-sized leftover, and -0 (not the +0 the kernel writes)
        bad = pad.clone()
        bad[3, 6] = v
        with pytest.raises(AssertionError):
            R.check_bits(bad, torch.zeros_like(pad), f"{v}")


def test_round_to_nearest_even_reference():
    """bf16_bits_rne agrees with torch's fp32 -> bf16 conversion on every value but NaN, including ties, the round-up into the
    next exponent and to Inf, and subnormals; and it is not truncation."""
    v = torch.cat([R.cast_edge_values(), torch.randn(4096) * 1e3, torch.randn(4096) * 1e-39])
    fin = ~torch.isnan(v)
    assert torch.equal(R.bf16_bits_rne(v)[fin], v[fin].bfloat16().view(torch.int16))
    R.check_cast_bf16(v.bfloat16(), v, "torch")
    trunc = (v.view(torch.int32) >> 16).to(torch.int16).view(torch.bfloat16)
    with pytest.raises(AssertionError):
        R.check_cast_bf16(trunc, v, "truncation")
