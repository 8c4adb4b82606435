"""Kernel-level parity on the GPU, through the C ABI (ctypes): each CUDA kernel against a plain PyTorch fp32
restatement of the same op on identical bf16-rounded inputs. Tolerances are bf16 output rounding (2^-8 relative)."""
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


def _gemm(_lib, L, st, **kw):
    a = _lib.GemmArgs()
    for k, v in kw.items():
        setattr(a, k, v)
    _lib.check(L.vb_gemm(ctypes.byref(a), st), "vb_gemm")


@pytest.mark.parametrize("M,N,K", [(256, 512, 128), (300, 784, 200), (384, 384, 768), (512, 2112, 192), (41984 // 8, 2304, 768)])
def test_gemm_tn(M, N, K):
    _lib, L, dev, st = _setup()
    torch.manual_seed(0)
    A = torch.randn(M, K, device=dev).bfloat16(); B = (0.05 * torch.randn(N, K, device=dev)).bfloat16()
    bias = torch.randn(N, device=dev); R = torch.randn(M, N, device=dev).bfloat16()
    D = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
    _gemm(_lib, L, st, A=A.data_ptr(), lda=K, B=B.data_ptr(), ldb=K, M=M, N=N, K=K, D=D.data_ptr(), ldd=N,
          bias=bias.data_ptr(), addend=R.data_ptr(), ld_add=N)
    torch.cuda.synchronize()
    assert _rel(D, A.float() @ B.float().t() + bias + R.float()) < BF16_TOL


def test_gemm_gelu_and_dgelu():
    _lib, L, dev, st = _setup()
    torch.manual_seed(1)
    M, N, K = 512, 3072, 768
    A = torch.randn(M, K, device=dev).bfloat16(); B = (0.05 * torch.randn(N, K, device=dev)).bfloat16()
    bias = torch.randn(N, device=dev)
    U = torch.zeros(M, N, device=dev, dtype=torch.bfloat16); G = torch.zeros_like(U)
    _gemm(_lib, L, st, A=A.data_ptr(), lda=K, B=B.data_ptr(), ldb=K, M=M, N=N, K=K, D=U.data_ptr(), ldd=N,
          bias=bias.data_ptr(), epilogue=_lib.VB_EPI_GELU, aux_out=G.data_ptr(), ld_aux=N)
    torch.cuda.synchronize()
    u = (A.float() @ B.float().t() + bias).requires_grad_(True)
    g = torch.nn.functional.gelu(u)
    (gp,) = torch.autograd.grad(g.sum(), u)
    assert _rel(G, g) < BF16_TOL        # aux_out = gelu(u)
    assert _rel(U, gp) < BF16_TOL       # D = gelu'(u), saved for the backward
    D = torch.zeros_like(U)
    _gemm(_lib, L, st, A=A.data_ptr(), lda=K, B=B.data_ptr(), ldb=K, M=M, N=N, K=K, D=D.data_ptr(), ldd=N,
          epilogue=_lib.VB_EPI_DGELU, aux_in=U.data_ptr(), ld_aux=N)
    torch.cuda.synchronize()
    assert _rel(D, (A.float() @ B.float().t()) * U.float()) < BF16_TOL
    # gelu'(u) in the library's tile-native order (what vb_layer_fwd / _bwd use for acts.u): same values, permuted; the DGELU
    # epilogue of a GEMM with the same output shape consumes it
    if L.vb_gemm_gp_tiled_ok(M, N):
        Ut = torch.zeros_like(U); G2 = torch.zeros_like(U); D2 = torch.zeros_like(U)
        _gemm(_lib, L, st, A=A.data_ptr(), lda=K, B=B.data_ptr(), ldb=K, M=M, N=N, K=K, D=Ut.data_ptr(), ldd=N,
              bias=bias.data_ptr(), epilogue=_lib.VB_EPI_GELU, aux_out=G2.data_ptr(), ld_aux=N, gp_tiled=1)
        torch.cuda.synchronize()
        assert torch.equal(G2, G)
        # documented layout: [M/256][N/256][2 ranks][2 column halves][4 row quarters][8 chunks][32 lanes][16]
        t = Ut.view(M // 256, N // 256, 2, 2, 4, 8, 32, 16).permute(0, 2, 4, 6, 1, 3, 5, 7).reshape(M, N)
        assert torch.equal(t, U)
        Wd = (0.05 * torch.randn(K, N, device=dev)).bfloat16()   # dgrad form: D[M,N] = dY[M,K] W[K,N], B MN-major
        Dref = torch.zeros_like(U)
        _gemm(_lib, L, st, A=A.data_ptr(), lda=K, B=Wd.data_ptr(), ldb=N, b_mn_major=1, M=M, N=N, K=K, D=Dref.data_ptr(), ldd=N,
              epilogue=_lib.VB_EPI_DGELU, aux_in=U.data_ptr(), ld_aux=N)
        _gemm(_lib, L, st, A=A.data_ptr(), lda=K, B=Wd.data_ptr(), ldb=N, b_mn_major=1, M=M, N=N, K=K, D=D2.data_ptr(), ldd=N,
              epilogue=_lib.VB_EPI_DGELU, aux_in=Ut.data_ptr(), ld_aux=N, gp_tiled=1)
        torch.cuda.synchronize()
        assert torch.equal(D2, Dref)
        assert _rel(Dref, (A.float() @ Wd.float()) * U.float()) < BF16_TOL


def test_gemm_dgrad_and_wgrad():
    _lib, L, dev, st = _setup()
    torch.manual_seed(2)
    M, Nn, Kk = 1000, 3072, 768
    dY = torch.randn(M, Nn, device=dev).bfloat16(); W = (0.05 * torch.randn(Nn, Kk, device=dev)).bfloat16()
    X = torch.randn(M, Kk, device=dev).bfloat16()
    D = torch.zeros(M, Kk, device=dev, dtype=torch.bfloat16)
    _gemm(_lib, L, st, A=dY.data_ptr(), lda=Nn, B=W.data_ptr(), ldb=Kk, b_mn_major=1, M=M, N=Kk, K=Nn,
          D=D.data_ptr(), ldd=Kk)
    torch.cuda.synchronize()
    assert _rel(D, dY.float() @ W.float()) < BF16_TOL
    for splits in (1, 5):
        dW = torch.zeros(Nn, Kk, device=dev, dtype=torch.float32)
        _gemm(_lib, L, st, A=dY.data_ptr(), lda=Nn, a_mn_major=1, B=X.data_ptr(), ldb=Kk, b_mn_major=1, M=Nn, N=Kk,
              K=M, D=dW.data_ptr(), ldd=Kk, d_fp32=1, splits=splits)
        torch.cuda.synchronize()
        assert _rel(dW, dY.float().t() @ X.float()) < 1e-4


def test_gemm_dgrad_with_attention_delta_epilogue():
    """vb_gemm_args.delta_out: the input-gradient GEMM that produces dO also writes D[b, h, s] = sum_d dO * O (the rowsum the attention
    backward needs), from the bf16-rounded dO it stores — same numbers as a separate pass over dO and O."""
    _lib, L, dev, st = _setup()
    torch.manual_seed(5)
    B, S, A = 4, 164, 12
    M, N, K = B * S, A * 64, 768
    if not L.vb_gemm_delta_ok(M, N):
        pytest.skip("delta epilogue not available for this shape / build")
    dY = torch.randn(M, K, device=dev).bfloat16(); W = (0.05 * torch.randn(K, N, device=dev)).bfloat16()
    ctx = torch.randn(M, N, device=dev).bfloat16()
    D = torch.zeros(M, N, device=dev, dtype=torch.bfloat16); D0 = torch.zeros_like(D)
    delta = torch.full((B, A, S), float("nan"), device=dev)
    base = dict(A=dY.data_ptr(), lda=K, B=W.data_ptr(), ldb=N, b_mn_major=1, M=M, N=N, K=K, ldd=N)
    _gemm(_lib, L, st, D=D0.data_ptr(), **base)
    _gemm(_lib, L, st, D=D.data_ptr(), delta_ctx=ctx.data_ptr(), delta_out=delta.data_ptr(), delta_seq=S, **base)
    torch.cuda.synchronize()
    assert torch.equal(D, D0)                                   # the stored gradient is unchanged
    assert _rel(D, dY.float() @ W.float()) < BF16_TOL
    ref = (D.float() * ctx.float()).view(B, S, A, 64).sum(-1).permute(0, 2, 1)
    assert torch.isfinite(delta).all()
    assert (delta - ref).abs().max().item() < 2e-3 * ref.abs().max().item() + 1e-3


def test_gemm_dropout_statistics_and_determinism():
    _lib, L, dev, st = _setup()
    torch.manual_seed(3)
    M, N, K = 2048, 768, 256
    A = torch.randn(M, K, device=dev).bfloat16(); B = torch.randn(N, K, device=dev).bfloat16()
    base = dict(A=A.data_ptr(), lda=K, B=B.data_ptr(), ldb=K, M=M, N=N, K=K, ldd=N)
    D0 = torch.zeros(M, N, device=dev, dtype=torch.bfloat16); D1 = torch.zeros_like(D0); D2 = torch.zeros_like(D0); D3 = torch.zeros_like(D0)
    _gemm(_lib, L, st, D=D0.data_ptr(), **base)
    _gemm(_lib, L, st, D=D1.data_ptr(), dropout_p=0.1, dropout_seed=7, dropout_stream=3, **base)
    _gemm(_lib, L, st, D=D2.data_ptr(), dropout_p=0.1, dropout_seed=7, dropout_stream=3, **base)
    _gemm(_lib, L, st, D=D3.data_ptr(), dropout_p=0.1, dropout_seed=8, dropout_stream=3, **base)
    torch.cuda.synchronize()
    assert torch.equal(D1, D2)
    assert not torch.equal(D1, D3)
    dropped = (D1 == 0) & (D0 != 0)
    q = 26 / 256  # p = 0.1 quantised to n/256 (DESIGN.md §2); survivors are scaled by 1/(1-q) so the mean is preserved
    assert abs(dropped.float().mean().item() - q) < 3e-3
    kept = ~dropped
    assert _rel(D1[kept], D0.float()[kept] / (1 - q)) < BF16_TOL
    assert abs(D1.float().mean().item() - D0.float().mean().item()) < 0.02 * D0.float().abs().mean().item()


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
