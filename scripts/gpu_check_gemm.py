"""GPU bring-up check for vb_gemm. Each case runs in its own subprocess so a
trap/timeout in one variant does not hide the others. Usage: python scripts/gpu_check_gemm.py [case]"""
import ctypes
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = ["tn_small", "tn_tail", "tn_bias_add", "tn_gelu", "tn_dgelu", "tn_n128", "dgrad", "wgrad", "wgrad_split",
         "tn_dropout", "perf"]


def run_case(name):
    import torch
    from visualbert_b200 import _lib
    L = _lib.lib()
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    st = torch.cuda.current_stream().cuda_stream

    def call(**kw):
        a = _lib.GemmArgs()
        for k, v in kw.items():
            setattr(a, k, v)
        _lib.check(L.vb_gemm(ctypes.byref(a), ctypes.c_void_p(st)), "vb_gemm")

    def rnd(*shape, scale=1.0):
        return (torch.randn(*shape, device=dev) * scale).to(torch.bfloat16)

    def report(out, ref, tag):
        out = out.float(); ref = ref.float()
        err = (out - ref).abs().max().item()
        den = ref.abs().max().item()
        bad = (~torch.isfinite(out)).sum().item()
        print(f"  [{tag}] max_abs_err={err:.4e} ref_max={den:.4e} rel={err / max(den, 1e-9):.4e} nonfinite={bad}")
        return err / max(den, 1e-9)

    rel = None
    if name in ("tn_small", "tn_tail", "tn_n128"):
        M, N, K = {"tn_small": (256, 512, 128), "tn_tail": (300, 776, 200), "tn_n128": (384, 384, 768)}[name]
        A = rnd(M, K); B = rnd(N, K)
        D = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
        call(A=A.data_ptr(), lda=K, B=B.data_ptr(), ldb=K, M=M, N=N, K=K, D=D.data_ptr(), ldd=N)
        torch.cuda.synchronize()
        rel = report(D, A.float() @ B.float().t(), name)
    elif name == "tn_bias_add":
        M, N, K = 512, 768, 768
        A = rnd(M, K); B = rnd(N, K, scale=0.05); bias = torch.randn(N, device=dev); R = rnd(M, N)
        D = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
        call(A=A.data_ptr(), lda=K, B=B.data_ptr(), ldb=K, M=M, N=N, K=K, D=D.data_ptr(), ldd=N,
             bias=bias.data_ptr(), addend=R.data_ptr(), ld_add=N)
        torch.cuda.synchronize()
        rel = report(D, A.float() @ B.float().t() + bias + R.float(), name)
    elif name == "tn_gelu":
        M, N, K = 512, 3072, 768
        A = rnd(M, K); B = rnd(N, K, scale=0.05); bias = torch.randn(N, device=dev)
        U = torch.zeros(M, N, device=dev, dtype=torch.bfloat16); G = torch.zeros_like(U)
        call(A=A.data_ptr(), lda=K, B=B.data_ptr(), ldb=K, M=M, N=N, K=K, D=U.data_ptr(), ldd=N,
             bias=bias.data_ptr(), epilogue=_lib.VB_EPI_GELU, aux_out=G.data_ptr(), ld_aux=N)
        torch.cuda.synchronize()
        u = (A.float() @ B.float().t() + bias).requires_grad_(True)
        g = torch.nn.functional.gelu(u)
        (gp,) = torch.autograd.grad(g.sum(), u)
        r1 = report(U, gp, "gelu:gelu'(u)")
        r2 = report(G, g, "gelu:g")
        rel = max(r1, r2)
    elif name == "tn_dgelu":
        M, N, K = 512, 3072, 768
        A = rnd(M, K); B = rnd(N, K, scale=0.05); U = rnd(M, N)
        D = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
        call(A=A.data_ptr(), lda=K, B=B.data_ptr(), ldb=K, M=M, N=N, K=K, D=D.data_ptr(), ldd=N,
             epilogue=_lib.VB_EPI_DGELU, aux_in=U.data_ptr(), ld_aux=N)
        torch.cuda.synchronize()
        rel = report(D, (A.float() @ B.float().t()) * U.float(), name)
    elif name == "dgrad":
        # dX[M,K'] = dY[M,N'] @ W[N',K'] : A = dY (K-major over N'), B = W stored [N',K'] = [K_gemm, N_gemm]
        M, Nn, Kk = 640, 3072, 768  # gemm: M, N=Kk(768), K=Nn(3072)
        dY = rnd(M, Nn); W = rnd(Nn, Kk, scale=0.05); R = rnd(M, Kk)
        D = torch.zeros(M, Kk, device=dev, dtype=torch.bfloat16)
        call(A=dY.data_ptr(), lda=Nn, B=W.data_ptr(), ldb=Kk, b_mn_major=1, M=M, N=Kk, K=Nn, D=D.data_ptr(),
             ldd=Kk, addend=R.data_ptr(), ld_add=Kk)
        torch.cuda.synchronize()
        rel = report(D, dY.float() @ W.float() + R.float(), name)
    elif name in ("wgrad", "wgrad_split"):
        # dW[Nout,Kin] = dY[Mr,Nout]^T @ X[Mr,Kin] ; gemm M=Nout, N=Kin, K=Mr; both operands MN-major
        Mr, Nout, Kin = (1000, 768, 3072) if name == "wgrad" else (4096 + 72, 384, 768)
        dY = rnd(Mr, Nout); X = rnd(Mr, Kin)
        D = torch.zeros(Nout, Kin, device=dev, dtype=torch.float32)
        call(A=dY.data_ptr(), lda=Nout, a_mn_major=1, B=X.data_ptr(), ldb=Kin, b_mn_major=1, M=Nout, N=Kin, K=Mr,
             D=D.data_ptr(), ldd=Kin, d_fp32=1, splits=(1 if name == "wgrad" else 7))
        torch.cuda.synchronize()
        rel = report(D, dY.float().t() @ X.float(), name)
    elif name == "tn_dropout":
        M, N, K = 1024, 768, 768
        A = rnd(M, K); B = rnd(N, K, scale=0.05)
        D0 = torch.zeros(M, N, device=dev, dtype=torch.bfloat16); D1 = torch.zeros_like(D0); D2 = torch.zeros_like(D0)
        base = dict(A=A.data_ptr(), lda=K, B=B.data_ptr(), ldb=K, M=M, N=N, K=K, ldd=N)
        call(D=D0.data_ptr(), **base)
        call(D=D1.data_ptr(), dropout_p=0.1, dropout_seed=1234, dropout_stream=3, **base)
        call(D=D2.data_ptr(), dropout_p=0.1, dropout_seed=1234, dropout_stream=3, **base)
        torch.cuda.synchronize()
        same = torch.equal(D1, D2)
        dropped = (D1 == 0) & (D0 != 0)
        frac = dropped.float().mean().item()
        kept = ~dropped
        rel = report(D1[kept], (D0.float() / (1 - 26 / 256))[kept], "dropout:kept")
        print(f"  dropout deterministic={same} drop_frac={frac:.4f} (expect 0.1000)")
        if not same or abs(frac - 26 / 256) > 0.005:
            rel = 1.0
    elif name == "perf":
        res = {}
        for tag, (M, N, K, kw) in {
            "qkv_fwd": (41984, 2304, 768, {}),
            "ffn_up_gelu": (41984, 3072, 768, {"gelu": True}),
            "ffn_up_gelu_tiled": (41984, 3072, 768, {"gelu": True, "tiled": True}),
            "ffn_up_dual_nomath": (41984, 3072, 768, {"gelu": True, "epi": 3}),
            "ffn_up_plain": (41984, 3072, 768, {}),
            "attn_out_plain": (41984, 768, 768, {}),
            "attn_out_bias_add": (41984, 768, 768, {"add": True}),
            "attn_out_bias_add_drop": (41984, 768, 768, {"add": True, "drop": True}),
            "ffn_down_bias_add_drop": (41984, 768, 3072, {"add": True, "drop": True}),
            "qkv_bias": (41984, 2304, 768, {"bias": True}),
            "ffn_down": (41984, 768, 3072, {}),
            "dgrad_ffn_up": (41984, 768, 3072, {"dgrad": True}),
            "dgrad_ffn_down_dgelu": (41984, 3072, 768, {"dgrad": True, "dgelu": True}),
            "dgrad_ffn_down_dgelu_tiled": (41984, 3072, 768, {"dgrad": True, "dgelu": True, "tiled": True}),
            "dgrad_qkv_accum": (41984, 768, 2304, {"dgrad": True, "add": True}),
            "wgrad_ffn_up": (3072, 768, 41984, {"wgrad": True}),
            "wgrad_attn_out": (768, 768, 41984, {"wgrad": True}),
            "wgrad_ffn_down": (768, 3072, 41984, {"wgrad": True}),
        }.items():
            if kw.get("wgrad"):
                A = rnd(K, M); B = rnd(K, N)
                D = torch.zeros(M, N, device=dev, dtype=torch.float32)
                tiles = ((M + 127) // 128) * ((N + 255) // 256)
                splits = max(1, (torch.cuda.get_device_properties(dev).multi_processor_count * 2) // tiles)
                args = dict(A=A.data_ptr(), lda=M, a_mn_major=1, B=B.data_ptr(), ldb=N, b_mn_major=1, M=M, N=N, K=K,
                            D=D.data_ptr(), ldd=N, d_fp32=1, splits=splits)
            elif kw.get("dgrad"):
                A = rnd(M, K); B = rnd(K, N)
                D = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
                args = dict(A=A.data_ptr(), lda=K, B=B.data_ptr(), ldb=N, b_mn_major=1, M=M, N=N, K=K, D=D.data_ptr(), ldd=N)
                if kw.get("dgelu"):
                    U = rnd(M, N)
                    args.update(epilogue=_lib.VB_EPI_DGELU, aux_in=U.data_ptr(), ld_aux=N, gp_tiled=1 if kw.get("tiled") else 0)
                if kw.get("add"):
                    R = rnd(M, N)
                    args.update(addend=R.data_ptr(), ld_add=N)
            else:
                A = rnd(M, K); B = rnd(N, K)
                D = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
                args = dict(A=A.data_ptr(), lda=K, B=B.data_ptr(), ldb=K, M=M, N=N, K=K, D=D.data_ptr(), ldd=N)
                if kw.get("add") or kw.get("bias"):
                    bias = torch.randn(N, device=dev)
                    args.update(bias=bias.data_ptr())
                if kw.get("add"):
                    R = rnd(M, N)
                    args.update(addend=R.data_ptr(), ld_add=N)
                if kw.get("drop"):
                    args.update(dropout_p=0.1, dropout_seed=5, dropout_stream=1)
                if kw.get("gelu"):
                    G = torch.zeros_like(D)
                    bias = torch.randn(N, device=dev)
                    args.update(epilogue=kw.get("epi", _lib.VB_EPI_GELU), aux_out=G.data_ptr(), ld_aux=N, bias=bias.data_ptr(),
                                gp_tiled=1 if kw.get("tiled") else 0)
            for _ in range(3):
                call(**args)
            torch.cuda.synchronize()
            e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
            iters = 20
            e0.record()
            for _ in range(iters):
                call(**args)
            e1.record(); torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / iters
            tf = 2.0 * M * N * K / (ms * 1e-3) / 1e12
            # cuBLAS reference time for the same shape
            if kw.get("wgrad"):
                f = lambda: torch.matmul(A.t(), B)
            elif kw.get("dgrad"):
                f = lambda: torch.matmul(A, B)
            else:
                f = lambda: torch.matmul(A, B.t())
            for _ in range(3):
                f()
            torch.cuda.synchronize()
            e0.record()
            for _ in range(iters):
                f()
            e1.record(); torch.cuda.synchronize()
            ms_ref = e0.elapsed_time(e1) / iters
            tf_ref = 2.0 * M * N * K / (ms_ref * 1e-3) / 1e12
            print(f"  [perf:{tag}] M={M} N={N} K={K}: {ms:.3f} ms = {tf:.1f} TFLOP/s   (cuBLAS {ms_ref:.3f} ms = {tf_ref:.1f})")
            res[tag] = {"ms": ms, "tflops": tf, "cublas_ms": ms_ref, "cublas_tflops": tf_ref}
        print("PERF_JSON " + json.dumps(res))
        rel = 0.0
    ok = rel is not None and rel < 2e-2
    print(f"CASE {name}: {'OK' if ok else 'FAIL'} rel={rel}")
    return 0 if ok else 1


def main():
    if len(sys.argv) > 1 and sys.argv[1] != "all":
        sys.exit(run_case(sys.argv[1]))
    summary = {}
    for c in CASES:
        t0 = time.time()
        try:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), c], capture_output=True, text=True, timeout=240)
            out = r.stdout + r.stderr
            rc = r.returncode
        except subprocess.TimeoutExpired as e:
            out = (e.stdout or b"").decode() if isinstance(e.stdout, bytes) else (e.stdout or "")
            out += "\nTIMEOUT"
            rc = -9
        summary[c] = rc
        print(f"=== {c} rc={rc} ({time.time() - t0:.1f}s)")
        print("\n".join(out.strip().splitlines()[-14:]))
        sys.stdout.flush()
    print("SUMMARY", json.dumps(summary))



if __name__ == "__main__":
    main()
