"""BertAdam and its learning-rate schedules on the library's multi-tensor kernel (SURVEY.md §8f rank 2).

Mirror of the reference module `visualbert/pytorch_pretrained_bert/optimization.py` ("opt.py"): same class names,
constructor arguments, `state` layout (`step`, `next_m`, `next_v` — so optimizer checkpoints interchange) and update
rule; the per-tensor Python loop of `BertAdam.step` (opt.py:239-304, ~200 tensors x ~10 launches + a clip each) becomes
ONE call of `vb_bert_adam_step` (two launches) per distinct (b1, b2, e, max_grad_norm) — one in practice.

Differences, all deliberate: parameters must be fp32 CUDA tensors (no CPU path); `p.grad` is read but not rescaled in
place by the clip (the reference's `clip_grad_norm_` side effect; `zero_grad` follows anyway).
"""
import ctypes
import math

import numpy as np
import torch
from torch.optim import Optimizer
from torch.optim.optimizer import required

from . import _lib
from .ops import deterministic


class _LRSchedule:
    """Learning-rate multiplier as a function of training progress = step / t_total (opt.py:37-82)."""
    warn_t_total = False

    def __init__(self, warmup=0.002, t_total=-1, **kw):
        if not 0.0 <= warmup < 1.0 and not warmup == -1:
            raise ValueError("Invalid warmup: {} - should be in [0.0, 1.0[ or -1".format(warmup))
        self.warmup, self.t_total = float(max(warmup, 0.0)), float(t_total)

    def get_lr(self, step, nowarn=False):
        if self.t_total < 0:
            return 1.0
        return self.get_lr_(float(step) / self.t_total)

    def get_lr_(self, progress):
        return 1.0


class ConstantLR(_LRSchedule):
    pass


class WarmupConstantSchedule(_LRSchedule):
    """Linear ramp over the first `warmup` fraction, then 1 (opt.py:154-162)."""

    def get_lr_(self, progress):
        return progress / self.warmup if progress < self.warmup else 1.0


class WarmupLinearSchedule(_LRSchedule):
    """Linear ramp, then linear decay to 0 at progress 1 (opt.py:165-174)."""
    warn_t_total = True

    def get_lr_(self, progress):
        if progress < self.warmup:
            return progress / self.warmup
        return max((progress - 1.0) / (self.warmup - 1.0), 0.0)


class WarmupCosineSchedule(_LRSchedule):
    """Linear ramp, then cosine decay with `cycles` periods (opt.py:89-112)."""
    warn_t_total = True

    def __init__(self, warmup=0.002, t_total=-1, cycles=0.5, **kw):
        super().__init__(warmup=warmup, t_total=t_total, **kw)
        self.cycles = cycles

    def get_lr_(self, progress):
        if progress < self.warmup:
            return progress / self.warmup
        progress = (progress - self.warmup) / (1 - self.warmup)
        return 0.5 * (1.0 + math.cos(math.pi * self.cycles * 2 * progress))


SCHEDULES = {None: ConstantLR, "none": ConstantLR, "warmup_cosine": WarmupCosineSchedule,
             "warmup_constant": WarmupConstantSchedule, "warmup_linear": WarmupLinearSchedule}

_TABLE_DTYPE = np.dtype([("p", "<u8"), ("g", "<u8"), ("m", "<u8"), ("v", "<u8"), ("numel", "<i8"), ("lr", "<f4"),
                         ("weight_decay", "<f4"), ("first_chunk", "<i4"), ("reserved", "<i4")])
assert _TABLE_DTYPE.itemsize == ctypes.sizeof(_lib.AdamTensor)


class BertAdam(Optimizer):
    """Adam with the BERT weight-decay fix, no bias correction, per-parameter gradient clipping and a built-in
    warm-up schedule — constructor and semantics of the reference (opt.py:185-304)."""

    def __init__(self, params, lr=required, warmup=-1, t_total=-1, schedule="warmup_linear", b1=0.9, b2=0.999, e=1e-6,
                 weight_decay=0.01, max_grad_norm=1.0, **kwargs):
        if lr is not required and lr < 0.0:
            raise ValueError("Invalid learning rate: {} - should be >= 0.0".format(lr))
        if not isinstance(schedule, _LRSchedule) and schedule not in SCHEDULES:
            raise ValueError("Invalid schedule parameter: {}".format(schedule))
        if not 0.0 <= b1 < 1.0:
            raise ValueError("Invalid b1 parameter: {} - should be in [0.0, 1.0[".format(b1))
        if not 0.0 <= b2 < 1.0:
            raise ValueError("Invalid b2 parameter: {} - should be in [0.0, 1.0[".format(b2))
        if not e >= 0.0:
            raise ValueError("Invalid epsilon value: {} - should be >= 0.0".format(e))
        if not isinstance(schedule, _LRSchedule):
            schedule = SCHEDULES[schedule](warmup=warmup, t_total=t_total)
        defaults = dict(lr=lr, schedule=schedule, b1=b1, b2=b2, e=e, weight_decay=weight_decay, max_grad_norm=max_grad_norm)
        super().__init__(params, defaults)
        self._plans = {}  # (b1, b2, e, max_grad_norm) -> cached table for an unchanged set of tensors

    def get_lr(self):
        lr = []
        for group in self.param_groups:
            for p in group["params"]:
                state = self.state[p]
                if len(state) == 0:
                    return [0]
                lr.append(group["lr"] * group["schedule"].get_lr(state["step"]))
        return lr

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        buckets = {}
        for group in self.param_groups:
            key = (float(group["b1"]), float(group["b2"]), float(group["e"]), float(group["max_grad_norm"]))
            for p in group["params"]:
                if p.grad is None:
                    continue
                if p.grad.is_sparse:
                    raise RuntimeError("Adam does not support sparse gradients, please consider SparseAdam instead")
                if not (p.is_cuda and p.dtype == torch.float32 and p.is_contiguous() and p.grad.dtype == torch.float32
                        and p.grad.is_contiguous()):
                    raise _lib.VBertLibraryError("visualbert_b200.BertAdam needs contiguous fp32 CUDA parameters and "
                                                 "gradients (there is no CPU path)")
                state = self.state[p]
                if len(state) == 0:
                    state["step"] = 0
                    state["next_m"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                    state["next_v"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                lr = group["lr"] * group["schedule"].get_lr(state["step"])
                buckets.setdefault(key, []).append((p, state, lr, float(group["weight_decay"])))
        for key, items in buckets.items():
            self._launch(key, items)
        touched = [p for items in buckets.values() for p, _, _, _ in items]
        for items in buckets.values():
            for _, state, _, _ in items:
                state["step"] += 1
        if touched:
            # the kernel wrote through raw pointers: tell autograd / the bf16 weight caches that the values changed
            torch.autograd.graph.increment_version(touched)
        return loss

    def _launch(self, key, items):
        dev = items[0][0].device
        ident = tuple((p.data_ptr(), p.grad.data_ptr(), st["next_m"].data_ptr(), st["next_v"].data_ptr(), p.numel())
                      for p, st, _, _ in items)
        plan = self._plans.get(key)
        if plan is None or plan["ident"] != ident:
            tab = np.zeros(len(items), dtype=_TABLE_DTYPE)
            chunk = 0
            for i, (p, st, _, wd) in enumerate(items):
                tab[i] = (p.data_ptr(), p.grad.data_ptr(), st["next_m"].data_ptr(), st["next_v"].data_ptr(), p.numel(), 0.0, wd,
                          chunk, 0)
                chunk += (p.numel() + _lib.VB_ADAM_CHUNK - 1) // _lib.VB_ADAM_CHUNK
            plan = dict(ident=ident, tab=tab, n_chunks=chunk,
                        sumsq=torch.empty(len(items), device=dev, dtype=torch.float32),
                        dev_tab=torch.empty(tab.nbytes, device=dev, dtype=torch.uint8))
            self._plans[key] = plan
        tab = plan["tab"]
        tab["lr"] = np.asarray([lr for _, _, lr, _ in items], dtype=np.float32)
        tab["weight_decay"] = np.asarray([wd for _, _, _, wd in items], dtype=np.float32)
        # fresh pinned staging every step (torch's host allocator recycles it only after the async copy has run)
        host = torch.empty(tab.nbytes, dtype=torch.uint8, pin_memory=True)
        host.numpy()[:] = tab.view(np.uint8).reshape(-1)
        plan["dev_tab"].copy_(host, non_blocking=True)
        b1, b2, e, max_norm = key
        st = torch.cuda.current_stream(dev).cuda_stream
        with torch.cuda.device(dev), deterministic(dev, adam_chunks=plan["n_chunks"]):
            _lib.check(_lib.lib().vb_bert_adam_step(
                ctypes.c_void_p(plan["dev_tab"].data_ptr()), len(items), plan["n_chunks"], ctypes.c_void_p(plan["sumsq"].data_ptr()),
                ctypes.c_double(b1), ctypes.c_double(b2), ctypes.c_double(e), ctypes.c_double(max_norm), ctypes.c_void_p(st)),
                "vb_bert_adam_step")
