"""Forward-only encoder route (torch.no_grad(): vb_encoder_infer, one layer-sized workspace) against the arena forward (eval
mode, grad enabled, trainable parameters: vb_encoder_fwd, one arena slot per layer) on the full TrainVisualBERTObjective. The
two are alternated in one process after warm-up of both; each forward is timed with CUDA events and ends in a synchronise.

    python scripts/bench_infer.py --out DIR [--reps 11] [--cfg5-batch 64]

Prints one JSON line per shape (and writes them to DIR/bench_infer.json): median ms per forward of both routes, the peak
allocation above the pre-call baseline of both, the bytes of the storage behind the returned sequence_output of both, and the
FFN-up GEMM alone with the VB_EPI_GELU and the VB_EPI_GELU_FWD epilogue (TFLOP/s from 2 M N K), with the card's name and
power limit. Needs a CUDA device."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from visualbert_b200 import BertConfig, TrainVisualBERTObjective, _lib, synthetic  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def build(layers, hidden, heads, inter, B, T, V, Dv=2048):
    dev = torch.device("cuda:0")
    cfg = synthetic.bert_config_dict(layers, hidden, heads, inter, vocab=30522)
    model = TrainVisualBERTObjective(BertConfig.from_dict(cfg), "pretraining", visual_embedding_dim=Dv)
    model.load_state_dict(synthetic.init_state_dict(cfg, "pretraining", Dv, seed=0), strict=False)
    model.to(dev).eval()
    batch = synthetic.make_batch(B, T, V, Dv, head="pretraining", seed=1, vocab=30522, ragged=True)
    return model, {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in batch.items()}


def timed(model, batch, grad):
    """-> (ms, peak bytes above the baseline, bytes of the storage behind sequence_output, loss)"""
    seen = {}
    hook = model.bert.register_forward_hook(lambda m, i, o: seen.__setitem__("nbytes", o[0].untyped_storage().nbytes()))
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.set_grad_enabled(grad):
        e0.record()
        out = model(**batch)
        e1.record()
        torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    loss = out["loss"].item()
    hook.remove()
    del out
    return e0.elapsed_time(e1), peak, seen["nbytes"], loss


def ffn_up(M, N, K, reps=50, rounds=3):
    """The FFN-up GEMM alone, both epilogues alternated in blocks of `reps` launches -> (TFLOP/s GELU, TFLOP/s GELU_FWD)"""
    dev = torch.device("cuda:0")
    A = torch.randn(M, K, device=dev).bfloat16()
    W = (0.05 * torch.randn(N, K, device=dev)).bfloat16()
    bias = torch.randn(N, device=dev)
    u, g = torch.empty(M, N, device=dev, dtype=torch.bfloat16), torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    base = dict(A=A.data_ptr(), lda=K, B=W.data_ptr(), ldb=K, M=M, N=N, K=K, bias=bias.data_ptr())
    tiled = int(_lib.lib().vb_gemm_gp_tiled_ok(M, N))   # as the training forward calls it
    args = {"gelu": _lib.GemmArgs(D=u.data_ptr(), ldd=N, epilogue=_lib.VB_EPI_GELU, aux_out=g.data_ptr(), ld_aux=N, gp_tiled=tiled, **base),
            "gelu_fwd": _lib.GemmArgs(D=g.data_ptr(), ldd=N, epilogue=_lib.VB_EPI_GELU_FWD, **base)}
    best = {}
    for r in range(rounds + 1):   # round 0 warms both up
        for k, a in args.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                _lib.check(_lib.lib().vb_gemm(ctypes.byref(a), st), "vb_gemm")
            e1.record()
            torch.cuda.synchronize()
            if r > 0:
                best.setdefault(k, []).append(e0.elapsed_time(e1) / reps)
    med = {k: sorted(v)[len(v) // 2] for k, v in best.items()}
    return {k: round(2.0 * M * N * K / (ms * 1e-3) / 1e12, 1) for k, ms in med.items()}, {k: round(ms, 4) for k, ms in med.items()}


def run(name, layers, hidden, heads, inter, B, T, V, reps):
    model, batch = build(layers, hidden, heads, inter, B, T, V)
    S = T + V
    for grad in (True, False):   # warm-up of both routes: module load, weight bank, allocator
        timed(model, batch, grad)
    t, peak, nbytes, loss = {True: [], False: []}, {}, {}, {}
    for _ in range(reps):
        for grad in (True, False):
            ms, peak[grad], nbytes[grad], loss[grad] = timed(model, batch, grad)
            t[grad].append(ms)
    assert loss[True] == loss[False], loss   # the two routes compute the same bits
    med = {k: sorted(v)[len(v) // 2] for k, v in t.items()}
    del model, batch
    torch.cuda.empty_cache()
    tf, ms = ffn_up(B * S, inter, hidden)
    ws = int(_lib.lib().vb_encoder_infer_workspace(B, S, hidden, heads, inter, 0, -1))
    stride = int(_lib.lib().vb_encoder_arena_layout(B, S, hidden, heads, inter, 0, None))
    return dict(shape=name, layers=layers, batch=B, seq=S, hidden=hidden, reps=reps,
                ms_arena=round(med[True], 2), ms_infer=round(med[False], 2),
                ms_arena_minmax=[round(min(t[True]), 2), round(max(t[True]), 2)],
                ms_infer_minmax=[round(min(t[False]), 2), round(max(t[False]), 2)],
                peak_gb_arena=round(peak[True] / 1e9, 3), peak_gb_infer=round(peak[False] / 1e9, 3),
                sequence_output_storage_mb_arena=round(nbytes[True] / 1e6, 1), sequence_output_storage_mb_infer=round(nbytes[False] / 1e6, 1),
                workspace_gb=round(ws / 1e9, 3), arena_gb=round(layers * stride / 1e9, 3),
                ffn_up_tflops_gelu=tf["gelu"], ffn_up_tflops_gelu_fwd=tf["gelu_fwd"], ffn_up_ms_gelu=ms["gelu"], ffn_up_ms_gelu_fwd=ms["gelu_fwd"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory that receives bench_infer.json")
    ap.add_argument("--reps", type=int, default=11)
    ap.add_argument("--cfg5-batch", type=int, default=64)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_infer: needs a CUDA device")
    gpu = card()
    res = []
    for shape in (("cfg2", 12, 768, 12, 3072, 256, 128, 36), ("cfg5-shaped", 24, 1024, 16, 4096, args.cfg5_batch, 256, 100)):
        r = run(*shape, reps=max(args.reps, 10))
        r["gpu"] = gpu
        print(json.dumps(r), flush=True)
        res.append(r)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "bench_infer.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
