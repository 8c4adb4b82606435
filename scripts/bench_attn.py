"""Attention kernels alone at the benchmark shape (cfg2: B=256, S=164, A=12) through the C ABI: parity against a torch fp32
restatement on a small slice, then CUDA-event timing of forward and backward (dropout on, like the training step).
Usage: python scripts/bench_attn.py [B] [S] [A] [iters]   (S picks the kernels: wgmma up to 192, whole-head up to 256, staged
beyond)"""
import ctypes, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from visualbert_b200 import _lib

B = int(sys.argv[1]) if len(sys.argv) > 1 else 256
S = int(sys.argv[2]) if len(sys.argv) > 2 else 164
A = int(sys.argv[3]) if len(sys.argv) > 3 else 12
iters = int(sys.argv[4]) if len(sys.argv) > 4 else 20
H = A * 64
L = _lib.lib()
dev = torch.device("cuda:0")
st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
P = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
torch.manual_seed(0)
qkv = torch.randn(B * S, 3 * H, device=dev).bfloat16()
lens = torch.randint(S // 2, S + 1, (B,), device=dev)
mask = (torch.arange(S, device=dev)[None, :] < lens[:, None]).float()
bias = ((1 - mask) * -10000.0).contiguous()
ctx = torch.empty(B * S, H, device=dev, dtype=torch.bfloat16)
lse = torch.empty(B, A, S, device=dev)
dctx = torch.randn(B * S, H, device=dev).bfloat16()
dqkv = torch.empty_like(qkv)
drow = torch.empty(B, A, S, device=dev)
L.vb_attention_keep_bytes.restype = ctypes.c_int64
keep = torch.zeros(int(L.vb_attention_keep_bytes(B, S, A)), device=dev, dtype=torch.uint8)


def fwd(p):
    _lib.check(L.vb_attention_fwd(P(qkv), P(bias), P(ctx), P(lse), P(keep) if p > 0 else None, B, S, A, H, ctypes.c_float(p),
                                  ctypes.c_uint64(7), 3, st), "attn_fwd")


def bwd(p):
    _lib.check(L.vb_attention_bwd(P(qkv), P(bias), P(ctx), P(lse), P(keep) if p > 0 else None, P(dctx), P(dqkv), P(drow), B, S, A, H,
                                  ctypes.c_float(p), ctypes.c_uint64(7), 3, st), "attn_bwd")


# parity on the first 2 batch items, no dropout
fwd(0.0); bwd(0.0); torch.cuda.synchronize()
nb = min(B, 2)
qr = qkv[: nb * S].float().requires_grad_(True)
q, k, v = qr.view(nb, S, 3, A, 64).permute(2, 0, 3, 1, 4)
sc = q @ k.transpose(-1, -2) / 8.0 + bias[:nb, None, None, :]
ref = (torch.softmax(sc, -1) @ v).permute(0, 2, 1, 3).reshape(nb * S, H)
ref.backward(dctx[: nb * S].float())
rel = lambda a, b: ((a.float() - b.float()).abs().max() / b.float().abs().max()).item()
print(f"parity: ctx {rel(ctx[:nb * S], ref):.2e}  lse {(lse[:nb] - torch.logsumexp(sc, -1)).abs().max().item():.2e}  "
      f"dqkv {rel(dqkv[:nb * S], qr.grad):.2e}")

for p in (0.0, 0.1):
    for name, fn in (("fwd", fwd), ("bwd", bwd)):
        for _ in range(3):
            fn(p)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(iters):
            fn(p)
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1000 / iters
        fl = (4.0 if name == "fwd" else 8.0) * B * A * S * S * 64
        print(f"{name} dropout={p}: {us:8.1f} us  ({fl / us * 1e-6:7.1f} TFLOP/s algorithmic)")
