"""Kernel-level parity on the GPU, through the C ABI (ctypes): the LayerNorm, MLM-decoder and cross-entropy kernels against a
plain PyTorch fp32 restatement of the same op on identical bf16-rounded inputs. Tolerances are bf16 output rounding (2^-8
relative). The GEMM is checked against an fp64 reference in test_gemm_reference_gpu.py."""
import ctypes
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

BF16_TOL = 1.0e-2  # relative to the reference tensor's max-abs


def _setup():
    from visualbert_b200 import _lib
    return _lib, _lib.lib(), torch.device("cuda:0"), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _rel(out, ref):
    out, ref = out.float(), ref.float()
    assert torch.isfinite(out).all()
    return ((out - ref).abs().max() / ref.abs().max().clamp_min(1e-9)).item()


@pytest.mark.parametrize("rows,H", [(1000, 768), (333, 1024), (77, 128), (64, 256)])
def test_layernorm_fwd_bwd(rows, H):
    _lib, L, dev, st = _setup()
    torch.manual_seed(4)
    x = (torch.randn(rows, H, device=dev) * 2 + 0.5).bfloat16()
    gamma = 1 + 0.1 * torch.randn(H, device=dev); beta = 0.1 * torch.randn(H, device=dev)
    y = torch.empty_like(x); mean = torch.empty(rows, device=dev); rstd = torch.empty(rows, device=dev)
    P = lambda t: ctypes.c_void_p(t.data_ptr())
    _lib.check(L.vb_layernorm_fwd(P(x), ctypes.c_int64(H), P(gamma), P(beta), P(y), ctypes.c_int64(H), P(mean), P(rstd),
                                  rows, H, ctypes.c_float(1e-12), st), "ln_fwd")
    xr = x.float().requires_grad_(True); gr = gamma.clone().requires_grad_(True); br = beta.clone().requires_grad_(True)
    u = xr.mean(-1, keepdim=True); s = (xr - u).pow(2).mean(-1, keepdim=True)
    yr = gr * ((xr - u) / torch.sqrt(s + 1e-12)) + br
    torch.cuda.synchronize()
    assert _rel(y, yr) < BF16_TOL
    dy = torch.randn(rows, H, device=dev).bfloat16()
    yr.backward(dy.float())
    dx = torch.empty_like(x); dg = torch.zeros(H, device=dev); db = torch.zeros(H, device=dev); dbias = torch.zeros(H, device=dev)
    _lib.check(L.vb_layernorm_bwd(P(dy), P(x), P(mean), P(rstd), P(gamma), P(dx), None, P(dg), P(db), P(dbias), rows, H,
                                  ctypes.c_float(0.0), ctypes.c_uint64(0), 0, ctypes.c_float(0.0), 0, st), "ln_bwd")
    torch.cuda.synchronize()
    assert _rel(dx, xr.grad) < BF16_TOL
    assert _rel(dg, gr.grad) < 2e-3
    assert _rel(db, br.grad) < 2e-3
    assert _rel(dbias, dx.float().sum(0)) < 2e-3


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
