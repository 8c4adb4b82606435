"""The error bound of the GEMM reference tests (gemm_ref_util.py) is tight enough to catch the bugs those tests exist for:
built on the host from a correct result, a lost k-slab, a misplaced 16-column chunk, a bias added twice and a flipped dropout
bit are each rejected, while the correct bf16 and fp32 results pass."""
import pytest
import torch

from dropout_util import hidden_keep
from gemm_ref_util import check_close, check_dropout

M, N, K = 130, 96, 200   # a partial 128-row tile, six 16-column chunks, four 64-wide k-slabs (the last one partial)


def _operands():
    g = torch.Generator().manual_seed(0)
    A = torch.randn(M, K, generator=g).bfloat16()
    B = (0.05 * torch.randn(N, K, generator=g)).bfloat16()
    bias = torch.randn(N, generator=g)
    add = torch.randn(M, N, generator=g).bfloat16()
    C = torch.randn(M, N, generator=g)
    return A, B, bias, add, C


def _ref(A, B, skip_slab=None):
    a, b = A.double(), B.double()
    if skip_slab is not None:
        a = a.clone(); a[:, 64 * skip_slab:64 * (skip_slab + 1)] = 0
    return a @ b.t(), a.abs() @ b.abs().t()


def test_bound_accepts_the_correct_results():
    A, B, bias, add, C = _operands()
    acc, mag = _ref(A, B)
    out = (A.float() @ B.float().t() + bias + add.float()).bfloat16()
    check_close(out, acc + bias.double() + add.double(), mag + bias.double().abs() + add.double().abs(), True, "bf16")
    out32 = C + A.float() @ B.float().t() + bias
    check_close(out32, C.double() + acc + bias.double(), C.double().abs() + mag + bias.double().abs(), False, "fp32")


@pytest.mark.parametrize("bf16_out", [True, False])
def test_bound_rejects_a_missing_k_slab(bf16_out):
    A, B, bias, _, _ = _operands()
    out = A.float() @ B.float().t() + bias
    if bf16_out:
        out = out.bfloat16()
    for slab in range(4):
        acc, mag = _ref(A, B, skip_slab=slab)
        with pytest.raises(AssertionError):
            check_close(out, acc + bias.double(), mag + bias.double().abs(), bf16_out, f"slab {slab}")


def test_bound_rejects_a_chunk_from_the_neighbouring_columns():
    A, B, bias, add, _ = _operands()
    acc, mag = _ref(A, B)
    ref, m = acc + bias.double() + add.double(), mag + bias.double().abs() + add.double().abs()
    out = (A.float() @ B.float().t() + bias + add.float()).bfloat16()
    for row, c in ((0, 0), (127, 16), (129, 64)):
        bad = out.clone()
        bad[row, c:c + 16] = out[row, c + 16:c + 32]
        with pytest.raises(AssertionError):
            check_close(bad, ref, m, True, f"row {row} chunk {c // 16}")


@pytest.mark.parametrize("bf16_out", [True, False])
def test_bound_rejects_the_bias_added_twice(bf16_out):
    A, B, bias, _, C = _operands()
    acc, mag = _ref(A, B)
    base = torch.zeros(M, N) if bf16_out else C
    out = base + A.float() @ B.float().t() + 2 * bias
    if bf16_out:
        out = out.bfloat16()
    with pytest.raises(AssertionError):
        check_close(out, base.double() + acc + bias.double(), base.double().abs() + mag + bias.double().abs(), bf16_out, "bias")


@pytest.mark.parametrize("addend", [True, False])
def test_dropout_check_rejects_one_flipped_keep_bit(addend):
    A, B, bias, add, _ = _operands()
    add = add if addend else None
    acc, mag = _ref(A, B)
    acc, mag = acc + bias.double(), mag + bias.double().abs()
    keep, scale = hidden_keep(0xFEDCBA9876543210, 3, M, N, 0.1, "cpu")
    x = (A.float() @ B.float().t() + bias) * scale
    out = torch.where(keep, x + (add.float() if addend else 0.0), add.float() if addend else torch.zeros(M, N)).bfloat16()
    check_dropout(out, acc, mag, keep, scale, add, "correct mask")
    big = acc.abs() > 0.5
    for was_kept in (True, False):
        i = int(torch.nonzero((keep == was_kept) & big)[0, 0] * N + torch.nonzero((keep == was_kept) & big)[0, 1])
        flipped = keep.clone().view(-1)
        flipped[i] = not was_kept
        with pytest.raises(AssertionError):
            check_dropout(out, acc, mag, flipped.view(M, N), scale, add, f"bit {i} flipped")
