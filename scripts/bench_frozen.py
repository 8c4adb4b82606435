"""Training-step time, peak memory and library launches with part of the model frozen (requires_grad=False), in one process.

    python scripts/bench_frozen.py --out DIR [--tree PATH] [--steps N] [--warmup W] [--configs cfg2,vqa64]

Patterns: every parameter trainable ("all"), (a) the word embeddings frozen, (b) the embeddings and encoder layers 0..5 frozen,
(c) the text embeddings and every encoder layer frozen while the visual projection, the visual tables and the heads train.
Each pattern has its own parallel.FlatGradSync built after its parameters were frozen, as a user would build it; the patterns
are alternated step by step after warm-up, each step timed with CUDA events. Reports the median ms per step (forward,
backward, no optimizer), the peak allocated memory over the pattern's steps and the library launches per step, next to the
card's name and power limit. --tree runs another checkout of the package (for example the parent commit's, built in place), so
two builds can be compared in one session. Writes DIR/bench_frozen[_<label>].json and prints it.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

SHAPES = {
    "cfg2": dict(layers=12, hidden=768, heads=12, inter=3072, B=256, T=128, V=36, Dv=2048, head="pretraining"),
    "vqa64": dict(layers=12, hidden=768, heads=12, inter=3072, B=64, T=128, V=36, Dv=2048, head="vqa"),
}
PATTERNS = ("all", "a", "b", "c")


def frozen_names(model, pattern, k=6):
    names = [n for n, _ in model.named_parameters()]
    emb = [n for n in names if n.startswith("bert.embeddings.")]
    text = [n for n in emb if any(t in n for t in ("word_embeddings", ".position_embeddings.", ".token_type_embeddings."))]
    layer = lambda i: [n for n in names if n.startswith(f"bert.encoder.layer.{i}.")]
    L = len(model.bert.encoder.layer)
    return set({"all": [], "a": ["bert.embeddings.word_embeddings.weight"], "b": emb + [n for i in range(k) for n in layer(i)],
                "c": text + [n for i in range(L) for n in layer(i)]}[pattern])


def bench(name, c, steps, warmup):
    import torch
    from visualbert_b200 import BertConfig, TrainVisualBERTObjective, _lib, parallel, synthetic
    dev = torch.device("cuda:0")
    cfg = synthetic.bert_config_dict(c["layers"], c["hidden"], c["heads"], c["inter"])
    sd = synthetic.init_state_dict(cfg, c["head"], c["Dv"], seed=0)
    batch = synthetic.make_batch(c["B"], c["T"], c["V"], c["Dv"], head=c["head"], seed=1234)
    batch = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in batch.items()}
    model = TrainVisualBERTObjective(BertConfig.from_dict(cfg), c["head"], visual_embedding_dim=c["Dv"])
    model.load_state_dict(sd, strict=False)
    model = model.to(dev).train(True)
    params = dict(model.named_parameters())
    syncs = {}
    for pat in PATTERNS:
        frozen = frozen_names(model, pat)
        for n, p in params.items():
            p.requires_grad_(n not in frozen)
            p.grad = None
            p.__dict__.pop("_vb_direct_grad", None)
        syncs[pat] = (frozen, parallel.FlatGradSync(model))

    def step(pat):
        frozen, sync = syncs[pat]
        for n, p in params.items():   # only this pattern's gradient views and flags are attached
            p.requires_grad_(n not in frozen)
            p.grad = None
            p.__dict__.pop("_vb_direct_grad", None)
        for p in sync.params:
            p._vb_direct_grad = True
        sync.zero()
        model(**batch)["loss"].backward()

    for _ in range(warmup):
        for pat in PATTERNS:
            step(pat)
    torch.cuda.synchronize()
    times = {p: [] for p in PATTERNS}
    peak = {p: 0 for p in PATTERNS}
    launches = {p: 0 for p in PATTERNS}
    for _ in range(steps):
        for pat in PATTERNS:
            torch.cuda.reset_peak_memory_stats()
            n0 = _lib.launch_count()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            step(pat)
            e1.record()
            torch.cuda.synchronize()
            times[pat].append(e0.elapsed_time(e1))
            launches[pat] = _lib.launch_count() - n0
            peak[pat] = max(peak[pat], torch.cuda.max_memory_allocated())
    out = dict(config=name, B=c["B"], head=c["head"], steps=steps,
               ms={p: round(statistics.median(times[p]), 3) for p in PATTERNS},
               peak_allocated_gb={p: round(peak[p] / 2 ** 30, 3) for p in PATTERNS}, launches_per_step=launches)
    del model, syncs, batch, params
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--tree", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                    help="checkout whose visualbert_b200 package is imported (default: this one)")
    ap.add_argument("--label", default="")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--configs", default="cfg2,vqa64")
    a = ap.parse_args()
    sys.path.insert(0, os.path.abspath(a.tree))
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_frozen: no CUDA device (the timings are GPU timings; there is no CPU fallback)")
    props = torch.cuda.get_device_properties(0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    res = dict(gpu=props.name, nvidia_smi=q.stdout.strip(), tree=os.path.abspath(a.tree), label=a.label, results=[])
    for name in a.configs.split(","):
        res["results"].append(bench(name, SHAPES[name], a.steps, a.warmup))
        print(json.dumps(res["results"][-1]), flush=True)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, f"bench_frozen{'_' + a.label if a.label else ''}.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
