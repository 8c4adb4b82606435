"""Padded vs unpadded (BertVisualModel.set_unpadded) training steps at the cfg2 shape: 12 layers, H = 768, batch 256,
128 text positions + 36 regions, pretraining head, train mode.

Two batches: a ragged one (synthetic.make_batch(ragged=True): text lengths ~U[64, 128], region counts ~U[18, 36]) and a full
one (no padding, which shows what packing and unpacking cost). For each, padded and unpadded steps alternate in one process
after warm-up; every step (zero grads, forward, backward) is timed with CUDA events and the median is reported.

    python scripts/bench_unpadded.py --out DIR [--steps 10] [--warmup 3]

Writes DIR/bench_unpadded.json: per batch and mode the median / min step ms and pairs/s, the real-row fraction, the GPU name
and its power limit."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    from visualbert_b200 import BertConfig, TrainVisualBERTObjective, synthetic
    from visualbert_b200.parallel import BatchPrefetcher

    dev = torch.device("cuda:0")
    c = synthetic.CONFIGS["cfg2"]
    cfg = synthetic.bert_config_dict(c["layers"], c["hidden"], c["heads"], c["inter"])
    torch.manual_seed(0)
    model = TrainVisualBERTObjective(BertConfig.from_dict(cfg), c["head"], visual_embedding_dim=c["Dv"]).to(dev).train()
    pf = BatchPrefetcher(dev)
    B, S = c["B"], c["T"] + c["V"]
    result = dict(config="cfg2", batch=B, seq=S, layers=c["layers"], gpu=torch.cuda.get_device_name(dev),
                  power_limit_w=power_limit(), steps=args.steps, warmup=args.warmup, batches={})
    for kind, ragged in (("ragged", True), ("full", False)):
        host = synthetic.make_batch(B, c["T"], c["V"], c["Dv"], head=c["head"], seed=1234, ragged=ragged)
        valid = torch.cat((host["input_mask"], host["image_mask"]), 1) != 0
        batch = pf.take(pf.stage({k: (v.pin_memory() if torch.is_tensor(v) else v) for k, v in host.items()}))

        def step(unpadded):
            model.bert.set_unpadded(unpadded)
            model.zero_grad(set_to_none=True)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            model(**batch)["loss"].backward()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1)

        for _ in range(args.warmup):
            step(False)
            step(True)
        ms = {False: [], True: []}
        for _ in range(args.steps):
            for mode in (False, True):
                ms[mode].append(step(mode))
        entry = dict(real_row_fraction=valid.float().mean().item())
        for mode, name in ((False, "padded"), (True, "unpadded")):
            med = statistics.median(ms[mode])
            entry[name] = dict(step_ms_median=med, step_ms_min=min(ms[mode]), pairs_per_s=B / med * 1e3,
                               step_ms_all=ms[mode])
        entry["speedup"] = entry["padded"]["step_ms_median"] / entry["unpadded"]["step_ms_median"]
        result["batches"][kind] = entry
        print(f"{kind}: real rows {entry['real_row_fraction']:.3f}, padded {entry['padded']['step_ms_median']:.2f} ms, "
              f"unpadded {entry['unpadded']['step_ms_median']:.2f} ms, speedup {entry['speedup']:.3f}", flush=True)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "bench_unpadded.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps({k: v for k, v in result.items() if k != "batches"}))


if __name__ == "__main__":
    main()
