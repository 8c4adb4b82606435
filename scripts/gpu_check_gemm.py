"""GPU timing of vb_gemm at the benchmark's shapes against cuBLAS (correctness: tests/test_gemm_reference_gpu.py).
Each case runs in its own subprocess so a trap/timeout in one variant does not hide the others. Usage: python scripts/gpu_check_gemm.py [case]"""
import ctypes
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = ["perf"]


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

    rel = None
    if name == "perf":
        res = {}
        for tag, (M, N, K, kw) in {
            "qkv_fwd": (41984, 2304, 768, {}),
            "ffn_up_gelu": (41984, 3072, 768, {"gelu": True}),
            "ffn_up_gelu_tiled": (41984, 3072, 768, {"gelu": True, "tiled": True}),
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
                    args.update(epilogue=_lib.VB_EPI_GELU, aux_out=G.data_ptr(), ld_aux=N, bias=bias.data_ptr(),
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
