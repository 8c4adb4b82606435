"""Training-step time and activation memory with and without activation checkpointing (set_activation_checkpointing), in one
process.

    python scripts/bench_checkpointing.py --out DIR [--steps N] [--warmup W] [--configs cfg2,cfg5_b64] [--fit cfg5_b320]

Workloads: cfg2 pretraining (12 layers, H = 768, B = 256, S = 164) and the cfg5 shape (24 layers, H = 1024, S = 356) at B = 64
per GPU. After warm-up the arena step and the checkpointed step alternate step by step, each timed with CUDA events (forward and
backward, gradients into a parallel.FlatGradSync buffer, no optimizer). Reports the median ms per step and the peak allocated
memory above the pre-step baseline (model, gradients and optimizer-free state excluded). --fit runs the checkpointed step alone
at a batch whose arena activations (n_layers arena slots, from vb_encoder_arena_layout) exceed the card's memory, and reports
its peak next to that arena size; the arena step is not attempted there. The card's name and power limit are read in the same
run. Writes DIR/bench_checkpointing.json and prints it.
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


def _timed_step(model, sync, batch, ckpt):
    """-> (ms, peak allocated bytes above the pre-step baseline)."""
    import torch
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
    from visualbert_b200 import _lib
    B, S, H, A, I = c["B"], c["T"] + c["V"], c["hidden"], c["heads"], c["inter"]
    stride = int(_lib.lib().vb_encoder_arena_layout(B, S, H, A, I, 1, None))
    cs = int(_lib.lib().vb_encoder_ckpt_layout(B, S, H, A, I, -1, None))
    L = c["layers"]
    return dict(S=S, arena_gb=round(L * stride / 1e9, 3), ckpt_region_mb=round(cs / 1e6, 2), slot_gb=round(stride / 1e9, 3),
                ckpt_activations_gb=round(((L - 1) * cs + stride) / 1e9, 3))


def bench(name, c, steps, warmup):
    import torch
    model, sync, batch = _setup(c)
    modes = (False, True)
    for _ in range(warmup):
        for m in modes:
            _timed_step(model, sync, batch, m)
    times, peak = {m: [] for m in modes}, {m: 0 for m in modes}
    for _ in range(steps):
        for m in modes:
            ms, p = _timed_step(model, sync, batch, m)
            times[m].append(ms)
            peak[m] = max(peak[m], p)
    key = {False: "arena", True: "checkpointed"}
    med = {key[m]: round(statistics.median(times[m]), 2) for m in modes}
    out = dict(config=name, B=c["B"], layers=c["layers"], hidden=c["hidden"], head=c["head"], steps=steps, ms=med,
               slowdown=round(med["checkpointed"] / med["arena"] - 1, 4),
               peak_above_baseline_gb={key[m]: round(peak[m] / 1e9, 3) for m in modes}, layout=_layouts(c))
    del model, sync, batch
    torch.cuda.empty_cache()
    return out


def fit(name, c, steps):
    """The checkpointed step alone at a batch whose arena would not fit the card."""
    import torch
    total = torch.cuda.get_device_properties(0).total_memory
    lay = _layouts(c)
    if lay["arena_gb"] * 1e9 <= total:
        raise SystemExit(f"bench_checkpointing: {name}'s arena ({lay['arena_gb']} GB) fits the card; pick a larger batch for --fit")
    model, sync, batch = _setup(c)
    _timed_step(model, sync, batch, True)
    runs = [_timed_step(model, sync, batch, True) for _ in range(steps)]
    out = dict(config=name, B=c["B"], layers=c["layers"], hidden=c["hidden"], card_memory_gb=round(total / 1e9, 2), layout=lay,
               checkpointed_ms=round(statistics.median(r[0] for r in runs), 2),
               checkpointed_peak_above_baseline_gb=round(max(r[1] for r in runs) / 1e9, 3),
               peak_allocated_gb=round(torch.cuda.max_memory_allocated() / 1e9, 3))
    del model, sync, batch
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--configs", default="cfg2,cfg5_b64")
    ap.add_argument("--fit", default="cfg5_b320", help="a workload only the checkpointed step fits ('' to skip)")
    a = ap.parse_args()
    sys.path.insert(0, ROOT)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_checkpointing: no CUDA device (the timings are GPU timings; there is no CPU fallback)")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    res = dict(gpu=torch.cuda.get_device_properties(0).name, nvidia_smi=q.stdout.strip(), results=[])
    for name in filter(None, a.configs.split(",")):
        res["results"].append(bench(name, SHAPES[name], a.steps, a.warmup))
        print(json.dumps(res["results"][-1]), flush=True)
    if a.fit:
        res["fit"] = fit(a.fit, SHAPES[a.fit], a.steps)
        print(json.dumps(res["fit"]), flush=True)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "bench_checkpointing.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
