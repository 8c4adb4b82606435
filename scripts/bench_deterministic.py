"""Training-step time with and without deterministic reductions (torch.use_deterministic_algorithms), in one process.

    python scripts/bench_deterministic.py --out DIR [--optimizer] [--steps N] [--warmup W] [--configs cfg2,cfg5]

cfg2 is the flagship shape (B = 256, S = 164, 12 layers, H = 768); cfg5 is its large-model shape at one GPU's share of the
batch (B = 64, S = 356, 24 layers, H = 1024). After warm-up in both modes the script alternates default and deterministic steps
(forward + backward, plus a BertAdam step with --optimizer), times each with CUDA events and reports the medians, their ratio,
and the size of the deterministic workspace. Writes DIR/bench_deterministic.json and prints it.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {
    "cfg2": dict(layers=12, hidden=768, heads=12, inter=3072, B=256, T=128, V=36, Dv=2048, head="pretraining"),
    "cfg5": dict(layers=24, hidden=1024, heads=16, inter=4096, B=64, T=256, V=100, Dv=2048, head="pretraining"),
}


def bench(name, c, steps, warmup, optimizer):
    import torch
    from visualbert_b200 import BertAdam, BertConfig, TrainVisualBERTObjective, ops, synthetic
    dev = torch.device("cuda:0")
    cfg = synthetic.bert_config_dict(c["layers"], c["hidden"], c["heads"], c["inter"])
    sd = synthetic.init_state_dict(cfg, c["head"], c["Dv"], seed=0)
    batch = synthetic.make_batch(c["B"], c["T"], c["V"], c["Dv"], head=c["head"], seed=1234)
    batch = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in batch.items()}
    model = TrainVisualBERTObjective(BertConfig.from_dict(cfg), c["head"], visual_embedding_dim=c["Dv"])
    model.load_state_dict(sd, strict=False)
    model = model.to(dev).train(True)
    opt = BertAdam(model.parameters(), lr=1e-5, warmup=0.1, t_total=1000) if optimizer else None

    def step(det):
        torch.use_deterministic_algorithms(det)
        try:
            model.zero_grad(set_to_none=True)
            model(**batch)["loss"].backward()
            if opt is not None:
                opt.step()
        finally:
            torch.use_deterministic_algorithms(False)

    for det in (False, True) * warmup:
        step(det)
    torch.cuda.synchronize()
    times = {False: [], True: []}
    for _ in range(steps):
        for det in (False, True):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            step(det)
            e1.record()
            torch.cuda.synchronize()
            times[det].append(e0.elapsed_time(e1))
    ws = max((t.numel() for t in ops._det_ws_cache.values()), default=0)
    d, n = statistics.median(times[False]), statistics.median(times[True])
    out = dict(config=name, optimizer=optimizer, steps=steps, default_ms=round(d, 3), deterministic_ms=round(n, 3),
               ratio=round(n / d, 4), workspace_bytes=int(ws), peak_allocated_bytes=int(torch.cuda.max_memory_allocated()))
    del model, opt, batch
    ops._det_ws_cache.clear()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--optimizer", action="store_true", help="include a BertAdam step in every timed step")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--configs", default="cfg2,cfg5")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_deterministic: no CUDA device (the timings are GPU timings; there is no CPU fallback)")
    os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")   # torch's deterministic mode requires it for the heads' matmuls
    props = torch.cuda.get_device_properties(0)
    res = dict(gpu=props.name, sms=props.multi_processor_count, results=[])
    for name in a.configs.split(","):
        res["results"].append(bench(name, SHAPES[name], a.steps, a.warmup, a.optimizer))
        print(json.dumps(res["results"][-1]), flush=True)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "bench_deterministic.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
