"""Training steps with the BertAdam step inside and outside the CUDA graph, for VisualBERT-base (12 layers, H 768) at the small
per-GPU batches of scripts/bench_graphs.py, on one GPU.

    python scripts/bench_graphs_optimizer.py --out DIR [--steps 20] [--rounds 5]

Workloads: VQA at S = 164 with batches 8, 16, 64; NLVR at S = 112 with 8, 32; pretraining at S = 164 with 12 (MLM targets as
capacity-padded rows). The optimizer is a BertAdam with warmup_linear, the two weight-decay groups of the reference's wrapper
and per-tensor clipping at 1.0. Four loops run on one model (in graph-capturable mode), each with its own optimizer:
  a  eager step, then the default BertAdam step
  b  graphs.GraphedStep, then the default BertAdam step (the recipe without the optimizer in the graph)
  c  graphs.GraphedStep(optimizer=...), the optimizer step inside the graph
  d  eager step, then the BertAdam step in graph-capturable mode (device-side schedule)
each without and with a loss.item() after every step (as a training loop that logs the loss does). After warm-up, a round times
`steps` back-to-back steps of every loop in turn with CUDA events, and the host time to enqueue them; the table gives the median
over rounds. The graph pool is the growth of torch's reserved memory over the capture. Before timing, the four loops run three
steps each from the same weights and dropout state under torch.use_deterministic_algorithms, and their parameters are compared
bit for bit. Prints one JSON line per workload and writes them, with a markdown table, to DIR. Needs a CUDA device."""
import argparse
import json
import os
import statistics
import sys
import time

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")   # the heads' cuBLAS calls under deterministic algorithms
import torch  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from bench_graphs import build, card  # noqa: E402
from visualbert_b200 import BertAdam, graphs, parallel  # noqa: E402

WORKLOADS = [("vqa", 128, 8), ("vqa", 128, 16), ("vqa", 128, 64), ("nlvr", 76, 8), ("nlvr", 76, 32), ("pretraining", 128, 12)]
LOOPS = ("a", "b", "c", "d")


def make_optimizer(model, capturable):
    named = [(n, p) for n, p in model.named_parameters() if "pooler" not in n]
    nd = ("bias", "LayerNorm.bias", "LayerNorm.weight")
    opt = BertAdam([{"params": [p for n, p in named if not any(x in n for x in nd)], "weight_decay": 0.01},
                    {"params": [p for n, p in named if any(x in n for x in nd)], "weight_decay": 0.0}],
                   lr=5e-5, warmup=0.1, t_total=10000, schedule="warmup_linear", max_grad_norm=1.0)
    return opt.set_graph_capturable(capturable)


class Loop:
    """One of the four ways to run a training step with its optimizer."""

    def __init__(self, kind, model, sync):
        self.kind, self.model, self.sync = kind, model, sync
        self.opt = make_optimizer(model, capturable=kind in ("c", "d"))
        self.step = None
        if kind == "b":
            self.step = graphs.GraphedStep(model, sync)
        elif kind == "c":
            self.step = graphs.GraphedStep(model, sync, optimizer=self.opt)

    def __call__(self, batch):
        if self.kind == "c":
            return self.step(batch)
        if self.kind == "b":
            out = self.step(batch)
        else:
            self.sync.zero()
            out = self.model(**batch)
            out["loss"].backward()
        self.opt.step()
        return out


def same_bits(model, sync, batch, n=3):
    """Each loop from the same weights and dropout state for n steps in deterministic mode: parameters bit-identical to (a)?"""
    params = list(model.parameters())
    start = [p.detach().clone() for p in params]
    state = model.bert.dropout_state()
    torch.use_deterministic_algorithms(True)
    try:
        finals = {}
        for kind in LOOPS:
            with torch.no_grad():
                for p, s in zip(params, start):
                    p.copy_(s)
            model.bert.set_dropout_state(state)
            loop = Loop(kind, model, sync)
            for _ in range(n):
                loop(batch)
            torch.cuda.synchronize()
            finals[kind] = [p.detach().clone() for p in params]
            del loop
        same = {k: all(torch.equal(x, y) for x, y in zip(finals["a"], finals[k])) for k in LOOPS}
    finally:
        torch.use_deterministic_algorithms(False)
        from visualbert_b200 import _lib
        _lib.lib().vb_set_deterministic(None, 0)
    with torch.no_grad():
        for p, s in zip(params, start):
            p.copy_(s)
    model.bert.set_dropout_state(state)
    torch.cuda.empty_cache()
    return same


def timed(loop, batch, n, item):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    start.record()
    for _ in range(n):
        out = loop(batch)
        if item:
            out["loss"].item()
    end.record()
    host = (time.perf_counter() - t0) * 1e3 / n
    torch.cuda.synchronize()
    return start.elapsed_time(end) / n, host


def bench(head, T, B, steps, rounds):
    model, batch = build(head, T, B)
    sync = parallel.FlatGradSync(model)
    model.bert.set_graph_capturable(True)
    same = same_bits(model, sync, batch)
    loops = {k: Loop(k, model, sync) for k in LOOPS}
    pool = {}
    for k, loop in loops.items():
        loop(batch)                       # eager warm-up (the graphed loops' first call)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        r0 = torch.cuda.memory_reserved()
        loop(batch)                       # capture + first replay for b and c
        torch.cuda.synchronize()
        pool[k] = (torch.cuda.memory_reserved() - r0) / 2 ** 20 if k in ("b", "c") else 0.0
    ms = {(k, item): [] for k in LOOPS for item in (False, True)}
    host = {key: [] for key in ms}
    for _ in range(rounds):
        for key in ms:
            a, h = timed(loops[key[0]], batch, steps, key[1])
            ms[key].append(a)
            host[key].append(h)
    med = statistics.median
    r = dict(head=head, S=T + 36, batch=B, steps=steps, rounds=rounds, bit_identical_to_a=same,
             graph_pool_mib={"b": pool["b"], "c": pool["c"]})
    for (k, item) in ms:
        tag = k + ("_item" if item else "")
        r[f"{tag}_ms"] = med(ms[(k, item)])
        r[f"{tag}_host_ms"] = med(host[(k, item)])
    del loops, model, sync, batch
    torch.cuda.empty_cache()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_graphs_optimizer.py needs a CUDA device")
    os.makedirs(a.out, exist_ok=True)
    gpu = card()
    rows = []
    for head, T, B in WORKLOADS:
        r = bench(head, T, B, a.steps, a.rounds)
        r["card"] = gpu
        print(json.dumps(r), flush=True)
        rows.append(r)
    with open(os.path.join(a.out, "bench_graphs_optimizer.json"), "w") as f:
        f.write("\n".join(json.dumps(r) for r in rows) + "\n")
    lines = [f"card (name, power limit): {gpu}", "",
             "a: eager + default BertAdam; b: GraphedStep + default BertAdam after it; c: GraphedStep(optimizer=...); "
             "d: eager + BertAdam in graph-capturable mode. ms/step from CUDA events (median of rounds); host = ms per step to "
             "enqueue; +item = with loss.item() after every step.", "",
             "| head | S | batch | a | b | c | d | a +item | b +item | c +item | d +item | host a | host b | host c | host d "
             "| pool b MiB | pool c MiB | b, c, d bit-identical to a |",
             "|---|---|---|---|---|---|---|---|---|---|---|---|---|---|---|---|---|---|"]
    for r in rows:
        cells = [f"{r[k + '_ms']:.2f}" for k in LOOPS] + [f"{r[k + '_item_ms']:.2f}" for k in LOOPS]
        cells += [f"{r[k + '_host_ms']:.2f}" for k in LOOPS]
        cells += [f"{r['graph_pool_mib']['b']:.0f}", f"{r['graph_pool_mib']['c']:.0f}",
                  " ".join(f"{k}:{'yes' if r['bit_identical_to_a'][k] else 'NO'}" for k in LOOPS[1:])]
        lines.append(f"| {r['head']} | {r['S']} | {r['batch']} | " + " | ".join(cells) + " |")
    with open(os.path.join(a.out, "bench_graphs_optimizer.md"), "w") as f:
        f.write("\n".join(lines) + "\n")
    print("\n".join(lines))


if __name__ == "__main__":
    main()
