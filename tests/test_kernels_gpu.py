"""Op-level parity on the GPU: the MLM decoder with the fused cross-entropy, and the cross-entropy's ignore labels, through the
Python ops against a plain PyTorch fp32 restatement on identical bf16-rounded inputs. Tolerances are bf16 output rounding (2^-8
relative). The kernels themselves are checked element by element against fp64 references elsewhere: the GEMM in
test_gemm_reference_gpu.py; the LayerNorm, embedding, column-sum, cross-entropy and cast kernels in test_rowop_reference_gpu.py."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(out, ref):
    out, ref = out.float(), ref.float()
    assert torch.isfinite(out).all()
    return ((out - ref).abs().max() / ref.abs().max().clamp_min(1e-9)).item()


@pytest.mark.parametrize("n,V", [(300, 30522), (77, 1000), (5, 512)])
def test_mlm_decoder_and_fused_cross_entropy(n, V):
    """ops.mlm_decoder + ops.cross_entropy_rows against F.linear + F.cross_entropy (fp32) incl. gradients."""
    from visualbert_b200 import ops
    dev = torch.device("cuda:0")
    torch.manual_seed(11)
    H = 768
    E = (0.05 * torch.randn(V, H, device=dev)).requires_grad_(True)
    bias = (0.1 * torch.randn(V, device=dev)).requires_grad_(True)
    t0 = torch.randn(n, H, device=dev).bfloat16()
    labels = torch.randint(0, V, (n,), device=dev)
    t = t0.clone().requires_grad_(True)
    cache = ops.DecoderWeights()
    logits = ops.mlm_decoder(t, E, bias, cache)
    assert logits.shape == (n, (V + 15) // 16 * 16)
    loss = ops.cross_entropy_rows(logits, labels, V)
    (loss * 3.0).backward()
    tr = t0.float().requires_grad_(True); Er = E.detach().bfloat16().float().requires_grad_(True); br = bias.detach().clone().requires_grad_(True)
    lr = torch.nn.functional.cross_entropy(tr @ Er.t() + br, labels)
    (lr * 3.0).backward()
    assert abs(loss.item() - lr.item()) < 2e-3 * abs(lr.item())
    assert _rel(t.grad, tr.grad) < 2e-2
    assert _rel(E.grad, Er.grad) < 2e-2
    assert _rel(bias.grad, br.grad) < 2e-2


def test_cross_entropy_ignores_out_of_range_labels():
    """A label outside [0, V) (ignore indices such as -1 / -100, or >= V) contributes no loss and no gradient and is
    never used as an index (ADVICE r1: the kernels used to read logits[label] unchecked)."""
    from visualbert_b200 import ops
    dev = torch.device("cuda:0")
    torch.manual_seed(3)
    n, V = 12, 1000
    Vp = (V + 15) // 16 * 16
    base = torch.randn(n, Vp, device=dev).bfloat16()
    labels = torch.randint(0, V, (n,), device=dev)
    labels[1], labels[4], labels[7] = -100, V + 5, -1
    valid = (labels >= 0) & (labels < V)
    logits = base.clone().requires_grad_(True)
    loss = ops.cross_entropy_rows(logits, labels, V)
    loss.backward()
    grad = logits.grad.float()
    ref_in = base.float()[:, :V].requires_grad_(True)
    rows = torch.nn.functional.cross_entropy(ref_in[valid], labels[valid], reduction="sum") / n  # mean over ALL rows given
    rows.backward()
    assert abs(loss.item() - rows.item()) < 2e-3 * abs(rows.item())
    assert torch.all(grad[~valid] == 0)
    assert _rel(grad[valid][:, :V], ref_in.grad[valid]) < 2e-2
