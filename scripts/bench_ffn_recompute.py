"""Training-step time and activation memory of the three encoder memory settings in one process: the default arena, selective
FFN recomputation (set_ffn_recompute) and full activation checkpointing (set_activation_checkpointing).

    python scripts/bench_ffn_recompute.py --out DIR [--steps N] [--warmup W] [--configs cfg2,cfg5_b64] [--fit cfg5_b320]

Workloads: cfg2 pretraining (12 layers, H = 768, B = 256, S = 164) and the cfg5 shape (24 layers, H = 1024, S = 356) at B = 64
per GPU, where all three settings fit; after warm-up the three steps alternate step by step, each timed with CUDA events
(forward and backward, gradients into a parallel.FlatGradSync buffer, no optimizer). --fit: the cfg5 shape at B = 320, whose
arena (n_layers slots of vb_encoder_arena_layout) exceeds the card's memory, so only the FFN-recompute and checkpointed steps
alternate there. Reports the median ms per step and the peak allocated memory above the pre-step baseline (model and gradients
excluded), next to the activation bytes the layouts give. The card's name, power limit and clocks are read before and after
the timed steps. Writes DIR/bench_ffn_recompute.json and prints it.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = {
    "cfg2": dict(layers=12, hidden=768, heads=12, inter=3072, B=256, T=128, V=36, Dv=2048, head="pretraining"),
    "cfg5_b64": dict(layers=24, hidden=1024, heads=16, inter=4096, B=64, T=256, V=100, Dv=2048, head="pretraining"),
    "cfg5_b320": dict(layers=24, hidden=1024, heads=16, inter=4096, B=320, T=256, V=100, Dv=2048, head="pretraining"),
}
MODES = {"arena": (False, False), "ffn_recompute": (True, False), "checkpointed": (False, True)}   # (ffn, ckpt)


def _gpu_state():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,power.draw,clocks.sm,clocks.max.sm,temperature.gpu",
                        "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip()


def _setup(c):
    import torch
    from visualbert_b200 import BertConfig, TrainVisualBERTObjective, parallel, synthetic
    dev = torch.device("cuda:0")
    cfg = synthetic.bert_config_dict(c["layers"], c["hidden"], c["heads"], c["inter"])
    model = TrainVisualBERTObjective(BertConfig.from_dict(cfg), c["head"], visual_embedding_dim=c["Dv"])
    model.load_state_dict(synthetic.init_state_dict(cfg, c["head"], c["Dv"], seed=0), strict=False)
    model = model.to(dev).train(True)
    batch = synthetic.make_batch(c["B"], c["T"], c["V"], c["Dv"], head=c["head"], seed=1234)
    batch = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in batch.items()}
    return model, parallel.FlatGradSync(model), batch


def _timed_step(model, sync, batch, mode):
    """-> (ms, peak allocated bytes above the pre-step baseline)."""
    import torch
    ffn, ckpt = MODES[mode]
    model.bert.set_ffn_recompute(ffn)
    model.bert.set_activation_checkpointing(ckpt)
    sync.zero()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    model(**batch)["loss"].backward()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), torch.cuda.max_memory_allocated() - base


def _layouts(c):
    """Activation bytes of the encoder call in each setting, from the library's layout functions."""
    import ctypes
    from visualbert_b200 import _lib
    lib = _lib.lib()
    B, S, H, A, I, L = c["B"], c["T"] + c["V"], c["hidden"], c["heads"], c["inter"], c["layers"]
    stride = int(lib.vb_encoder_arena_layout(B, S, H, A, I, 1, None))
    fb = ctypes.c_int64()
    fstride = int(lib.vb_encoder_arena_layout_ffnrc(B, S, H, A, I, 1, None, ctypes.byref(fb)))
    cs = int(lib.vb_encoder_ckpt_layout(B, S, H, A, I, -1, None))
    return dict(S=S, arena_gb=round(L * stride / 1e9, 3), ffn_recompute_gb=round((L * fstride + fb.value) / 1e9, 3),
                shared_ffn_buffer_gb=round(fb.value / 1e9, 3), checkpointed_gb=round(((L - 1) * cs + stride) / 1e9, 3))


def bench(name, c, steps, warmup, modes):
    import torch
    model, sync, batch = _setup(c)
    for _ in range(warmup):
        for m in modes:
            _timed_step(model, sync, batch, m)
    state_before = _gpu_state()
    times, peak = {m: [] for m in modes}, {m: 0 for m in modes}
    for _ in range(steps):
        for m in modes:
            ms, p = _timed_step(model, sync, batch, m)
            times[m].append(ms)
            peak[m] = max(peak[m], p)
    med = {m: round(statistics.median(times[m]), 2) for m in modes}
    base = "arena" if "arena" in modes else "ffn_recompute"
    out = dict(config=name, B=c["B"], layers=c["layers"], hidden=c["hidden"], head=c["head"], steps=steps, ms=med,
               ms_all={m: [round(t, 2) for t in times[m]] for m in modes},
               vs_first={m: round(med[m] / med[base] - 1, 4) for m in modes},
               peak_above_baseline_gb={m: round(peak[m] / 1e9, 3) for m in modes}, layout=_layouts(c),
               card_memory_gb=round(torch.cuda.get_device_properties(0).total_memory / 1e9, 2),
               gpu_state_before=state_before, gpu_state_after=_gpu_state())
    del model, sync, batch
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--configs", default="cfg2,cfg5_b64")
    ap.add_argument("--fit", default="cfg5_b320", help="a workload whose arena does not fit the card ('' to skip)")
    a = ap.parse_args()
    sys.path.insert(0, ROOT)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_ffn_recompute: no CUDA device (the timings are GPU timings; there is no CPU fallback)")
    res = dict(gpu=torch.cuda.get_device_properties(0).name, nvidia_smi=_gpu_state(), results=[])
    for name in filter(None, a.configs.split(",")):
        res["results"].append(bench(name, SHAPES[name], a.steps, a.warmup, tuple(MODES)))
        print(json.dumps(res["results"][-1]), flush=True)
    if a.fit:
        c = SHAPES[a.fit]
        if _layouts(c)["arena_gb"] * 1e9 <= torch.cuda.get_device_properties(0).total_memory:
            raise SystemExit(f"bench_ffn_recompute: {a.fit}'s arena fits the card; pick a larger batch for --fit")
        res["fit"] = bench(a.fit, c, a.steps, a.warmup, ("ffn_recompute", "checkpointed"))
        print(json.dumps(res["fit"]), flush=True)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "bench_ffn_recompute.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
