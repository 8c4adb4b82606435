"""Analysis-mode forward (eval, no_grad, output_attention_weights=True): the whole-encoder call plus the attention-probability
kernel, against the method it replaced — the whole-encoder forward returning every layer, then per layer an fp32 torch
recompute of softmax(QK^T / 8 + mask) from that layer's input (fp32 Q / K projections from the master weights). The two are
alternated in one process after warm-up, timed with CUDA events; the maps kernel is also timed alone for its bandwidth.

    python scripts/bench_attention_maps.py [--reps 5] [--cfg5-batch 64] [--out results.json]

Prints one JSON line per shape: ms per forward and peak allocation of each method, the maps kernel's ms per forward and
GB/s (maps bytes = 4 L B A S^2) against the H100 SXM data sheet's 3.35 TB/s, and the card name and power limit."""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from visualbert_b200 import BertConfig, TrainVisualBERTObjective, ops, synthetic  # noqa: E402

HBM_PEAK = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def build(layers, hidden, heads, inter, B, T, V, Dv=2048):
    dev = torch.device("cuda:0")
    cfg = synthetic.bert_config_dict(layers, hidden, heads, inter, vocab=4096)
    model = TrainVisualBERTObjective(BertConfig.from_dict(cfg), "pretraining", visual_embedding_dim=Dv,
                                     output_attention_weights=True)
    model.load_state_dict(synthetic.init_state_dict(cfg, "pretraining", Dv, seed=0), strict=False)
    model.to(dev).eval()
    batch = synthetic.make_batch(B, T, V, Dv, head="pretraining", seed=1, vocab=4096, ragged=True)
    return model, {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in batch.items()}


def new_method(model, batch):
    return model(**batch)["attention_weights"]


def old_method(model, batch):
    """The deleted path, restated: all layer outputs from the whole-encoder call, then the fp32 recompute per layer."""
    bert = model.bert
    mask = torch.cat((batch["input_mask"], batch["image_mask"]), 1)
    bert.refresh_compute_weights()
    bias = ops.mask_bias(mask, None)
    x = bert.embeddings(batch["input_ids"], batch["token_type_ids"], visual_embeddings=batch["visual_embeddings"],
                        visual_embeddings_type=batch["visual_embeddings_type"])
    layers = bert.encoder(x, bias, output_all_encoded_layers=True, output_attention_weights=False)
    maps = []
    for layer, h in zip(bert.encoder.layer, [x] + layers[:-1]):
        a = layer.attention.self
        hf = h.float()
        B, S, H = hf.shape
        A = a.num_attention_heads

        def heads(lin):
            return F.linear(hf, lin.weight.float(), lin.bias.float()).view(B, S, A, H // A).permute(0, 2, 1, 3)
        scores = torch.matmul(heads(a.query), heads(a.key).transpose(-1, -2)) / 8.0
        maps.append(torch.softmax(scores + bias[:, None, None, :], dim=-1))
    return maps


def timed(fn, *args):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn(*args)
    e1.record()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del out
    return e0.elapsed_time(e1), peak


def kernel_ms(B, S, A, L, reps=20):
    """The maps kernel alone over L layers' worth of [B, A, S, S] maps, from random bf16 qkv."""
    dev = torch.device("cuda:0")
    qkv = torch.randn(B * S, 3 * A * 64, device=dev).bfloat16()
    bias = torch.zeros(B, S, device=dev)
    for _ in range(2):
        p = ops.attention_probs(qkv, bias, B, S, A)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        p = ops.attention_probs(qkv, bias, B, S, A)
    e1.record()
    torch.cuda.synchronize()
    del p
    return e0.elapsed_time(e1) / reps * L


def run(name, layers, hidden, heads, inter, B, T, V, reps):
    model, batch = build(layers, hidden, heads, inter, B, T, V)
    S = T + V
    with torch.no_grad():
        for fn in (new_method, old_method):   # warm-up: module load, weight bank, allocator
            timed(fn, model, batch)
        t = {"new": [], "old": []}
        peak = {}
        for _ in range(reps):
            for key, fn in (("new", new_method), ("old", old_method)):
                ms, pk = timed(fn, model, batch)
                t[key].append(ms)
                peak[key] = pk
        # the two methods' maps agree to the bf16 rounding of the layer inputs
        a, b = new_method(model, batch), old_method(model, batch)
        diff = max((x - y).abs().max().item() for x, y in zip(a, b))
        del a, b
        kms = kernel_ms(B, S, heads, layers)
    maps_bytes = 4 * layers * B * heads * S * S
    med = {k: sorted(v)[len(v) // 2] for k, v in t.items()}
    return dict(shape=name, layers=layers, batch=B, seq=S, hidden=hidden, heads=heads,
                ms_new=round(med["new"], 2), ms_old=round(med["old"], 2), ms_new_all=[round(x, 2) for x in t["new"]],
                ms_old_all=[round(x, 2) for x in t["old"]], speedup=round(med["old"] / med["new"], 2),
                peak_gb_new=round(peak["new"] / 1e9, 2), peak_gb_old=round(peak["old"] / 1e9, 2),
                maps_gb=round(maps_bytes / 1e9, 2), maps_kernel_ms=round(kms, 3),
                maps_kernel_gbps=round(maps_bytes / (kms * 1e-3) / 1e9, 1),
                maps_kernel_share_of_hbm_peak=round(maps_bytes / (kms * 1e-3) / HBM_PEAK, 3),
                max_abs_diff_new_vs_old=diff)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cfg5-batch", type=int, default=64)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_attention_maps: needs a CUDA device")
    gpu = card()
    res = []
    for shape in (("cfg2", 12, 768, 12, 3072, 256, 128, 36), ("cfg5", 24, 1024, 16, 4096, args.cfg5_batch, 256, 100)):
        r = run(*shape, reps=args.reps)
        r["gpu"] = gpu
        print(json.dumps(r), flush=True)
        res.append(r)
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
