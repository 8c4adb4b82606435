"""Eager against CUDA-graphed training steps (graphs.GraphedStep) of VisualBERT-base (12 layers, H 768) at the per-GPU batches
of the reference's fine-tuning and pretraining configs, on one GPU, with FlatGradSync owning the gradients and no optimizer.

    python scripts/bench_graphs.py --out DIR [--steps 20] [--rounds 5]

Workloads: VQA head at S = 164 (128 text + 36 regions) with batches 8, 16, 64; NLVR head at S = 112 (76 + 36) with 8, 32;
pretraining at S = 164 with 12 (MLM targets as capacity-padded rows) and 256. Both kinds of step run on the same model, in
graph-capturable mode, alternated round by round after warm-up of both. A round times `steps` back-to-back steps with CUDA
events (so a host-bound step shows), and the host time to enqueue them; the table gives the median over rounds. The memory
held by the graph's private pool is the growth of torch's reserved memory over the capture. Before timing, the graphed and the
eager output are compared at the same dropout state (the heads' torch nn.Dropout is set to p = 0, since torch's own generator
is not replayed by the graph; the encoder's dropout stays on). Prints one JSON line per workload and writes them, with a
markdown table, to DIR. Needs a CUDA device."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from visualbert_b200 import BertConfig, TrainVisualBERTObjective, graphs, parallel, synthetic  # noqa: E402

WORKLOADS = [("vqa", 128, 8), ("vqa", 128, 16), ("vqa", 128, 64), ("nlvr", 76, 8), ("nlvr", 76, 32),
             ("pretraining", 128, 12), ("pretraining", 128, 256)]
V, DV = 36, 2048


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def build(head, T, B):
    dev = torch.device("cuda:0")
    cfg = synthetic.bert_config_dict(12, 768, 12, 3072, vocab=30522)
    model = TrainVisualBERTObjective(BertConfig.from_dict(cfg), head, visual_embedding_dim=DV)
    model.load_state_dict(synthetic.init_state_dict(cfg, head, DV, seed=0), strict=False)
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    model.to(dev).train(True)
    host = synthetic.make_batch(B, T, V, DV, head=head, seed=1, vocab=30522, ragged=True)
    if head == "pretraining":   # capacity: 15 % of the text positions plus slack, padded with -1
        host["masked_lm_rows"] = parallel.BatchPrefetcher.labelled_rows(host, capacity=int(0.2 * B * T) + 8)
    return model, {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in host.items()}


def run(model, sync, step, batch, graphed, n):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    start.record()
    for _ in range(n):
        if graphed:
            out = step(batch)
        else:
            sync.zero()
            out = model(**batch)
            out["loss"].backward()
    end.record()
    host = (time.perf_counter() - t0) * 1e3 / n
    torch.cuda.synchronize()
    return start.elapsed_time(end) / n, host, out


def bench(head, T, B, steps, rounds):
    model, batch = build(head, T, B)
    sync = parallel.FlatGradSync(model)
    step = graphs.GraphedStep(model, sync)
    run(model, sync, step, batch, False, 2)
    step(batch)                                    # eager warm-up of the graphed path
    torch.cuda.synchronize()
    torch.cuda.empty_cache()   # (capture empties the cache too: the pool is what the capture reserves beyond this)
    r0 = torch.cuda.memory_reserved()
    state = model.bert.dropout_state()
    graphed_loss = step(batch)["loss"].float().item()   # capture + first replay
    pool = torch.cuda.memory_reserved() - r0
    model.bert.set_dropout_state(state)
    sync.zero()
    eager_loss = model(**batch)["loss"].float().item()
    rel = abs(graphed_loss - eager_loss) / max(abs(eager_loss), 1e-30)
    e_ms, e_host, g_ms, g_host = [], [], [], []
    for _ in range(rounds):
        a, h, _ = run(model, sync, step, batch, False, steps)
        e_ms.append(a); e_host.append(h)
        a, h, _ = run(model, sync, step, batch, True, steps)
        g_ms.append(a); g_host.append(h)
    med = statistics.median
    r = dict(head=head, S=T + V, batch=B, eager_ms=med(e_ms), graphed_ms=med(g_ms), eager_host_ms=med(e_host),
             graphed_host_ms=med(g_host), speedup=med(e_ms) / med(g_ms), graph_pool_mib=pool / 2 ** 20,
             loss_rel_diff=rel, eager_loss=eager_loss, graphed_loss=graphed_loss, steps=steps, rounds=rounds)
    del step, model, sync, batch
    torch.cuda.empty_cache()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    gpu = card()
    rows = []
    for head, T, B in WORKLOADS:
        r = bench(head, T, B, a.steps, a.rounds)
        r["card"] = gpu
        print(json.dumps(r), flush=True)
        rows.append(r)
    with open(os.path.join(a.out, "bench_graphs.json"), "w") as f:
        f.write("\n".join(json.dumps(r) for r in rows) + "\n")
    lines = [f"card: {gpu}", "",
             "| head | S | batch | eager ms/step | graphed ms/step | speedup | eager host ms/step | graphed host ms/step | graph pool MiB | loss rel. diff |",
             "|---|---|---|---|---|---|---|---|---|---|"]
    for r in rows:
        lines.append(f"| {r['head']} | {r['S']} | {r['batch']} | {r['eager_ms']:.2f} | {r['graphed_ms']:.2f} | {r['speedup']:.2f} | "
                     f"{r['eager_host_ms']:.2f} | {r['graphed_host_ms']:.2f} | {r['graph_pool_mib']:.0f} | {r['loss_rel_diff']:.1e} |")
    with open(os.path.join(a.out, "bench_graphs.md"), "w") as f:
        f.write("\n".join(lines) + "\n")
    print("\n".join(lines))


if __name__ == "__main__":
    main()
