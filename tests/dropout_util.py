"""Torch restatement of the library's hidden-state dropout mask (csrc/vb_common.cuh: mix32, dropout_key, dropout_keep8,
dropout_quantise), shared by the tests that check a kernel's mask bit for bit."""
import torch

M32 = 0xFFFFFFFF


def _mix32(x):
    x = x ^ (x >> 16); x = (x * 0x7feb352d) & M32
    x = x ^ (x >> 15); x = (x * 0x846ca68b) & M32
    return x ^ (x >> 16)


def _mix32_int(x):
    x &= M32
    x ^= x >> 16; x = (x * 0x7feb352d) & M32
    x ^= x >> 15; x = (x * 0x846ca68b) & M32
    return x ^ (x >> 16)


def hidden_keep(seed, stream, rows, cols, p, dev):
    """keep mask [rows, cols] (bool) and survivor scale of vb_common.cuh::dropout_keep8 for a [rows, cols] tensor."""
    n = int(p * 256.0 + 0.5)
    key = _mix32_int((seed & M32) ^ _mix32_int(((seed >> 32) + 0x9E3779B9 * (stream + 1)) & M32))
    idx = torch.arange(rows * cols, device=dev, dtype=torch.int64)
    e8, k = idx >> 3, idx & 7
    kk = key ^ (((e8 >> 31) * 0x27d4eb2f) & M32)
    h = _mix32((((e8 << 1) + (k >> 2)) & M32) ^ kk)
    byte = (h >> (8 * (k & 3))) & 0xFF
    return (byte >= n).view(rows, cols), 256.0 / (256.0 - n)
