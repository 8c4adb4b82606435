"""BertAdam and its learning-rate schedules on the library's multi-tensor kernel (SURVEY.md §8f rank 2).

Mirror of the reference module `visualbert/pytorch_pretrained_bert/optimization.py` ("opt.py"): same class names,
constructor arguments, `state` layout (`step`, `next_m`, `next_v` — so optimizer checkpoints interchange) and update
rule; the per-tensor Python loop of `BertAdam.step` (opt.py:239-304, ~200 tensors x ~10 launches + a clip each) becomes
ONE call of `vb_bert_adam_step` (two launches) per distinct (b1, b2, e, max_grad_norm) — one in practice.

Differences, all deliberate: parameters must be fp32 CUDA tensors (no CPU path); `p.grad` is read but not rescaled in
place by the clip (the reference's `clip_grad_norm_` side effect; `zero_grad` follows anyway).

BertAdam.set_graph_capturable() moves the learning-rate schedule and the step counters onto the device
(vb_bert_adam_step_sched), so that a step can be captured in a CUDA graph and replayed (graphs.GraphedStep(optimizer=...)).
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
_GROUP_DTYPE = np.dtype([("lr", "<f8"), ("warmup", "<f8"), ("t_total", "<f8"), ("cycles", "<f8"), ("weight_decay", "<f4"),
                         ("schedule", "<i4")])
assert _GROUP_DTYPE.itemsize == ctypes.sizeof(_lib.AdamGroup)
# the schedules the update kernel evaluates (vb_adam_group.schedule); exact classes: a subclass may compute anything
_SCHEDULE_KINDS = {ConstantLR: _lib.VB_SCHED_CONSTANT, WarmupConstantSchedule: _lib.VB_SCHED_WARMUP_CONSTANT,
                   WarmupLinearSchedule: _lib.VB_SCHED_WARMUP_LINEAR, WarmupCosineSchedule: _lib.VB_SCHED_WARMUP_COSINE}


def _group_row(group):
    """The vb_adam_group of a parameter group; ValueError for a schedule the device cannot evaluate as the host would."""
    sched = group["schedule"]
    kind = _SCHEDULE_KINDS.get(type(sched))
    if kind is None:
        raise ValueError("BertAdam graph-capturable mode evaluates the schedule on the device, which knows only the classes of "
                         f"SCHEDULES ({', '.join(c.__name__ for c in _SCHEDULE_KINDS)}), not {type(sched).__name__}")
    if float(sched.t_total) == 0.0:
        raise ValueError("BertAdam graph-capturable mode: t_total = 0 (the schedule divides by it)")
    cycles = float(sched.cycles) if kind == _lib.VB_SCHED_WARMUP_COSINE else 0.0
    return (float(group["lr"]), float(sched.warmup), float(sched.t_total), cycles, float(group["weight_decay"]), kind)


def _capture_refusal(what):
    return ValueError(f"CUDA graph capture: BertAdam.step would {what} inside the graph (a zero-init there would reset the "
                      "moments on every replay); warm up first (run the step eagerly once)")


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
        self._capturable = False
        self._groups = None        # graph-capturable mode: the device group table and the rows it holds
        # bumped whenever a tensor table or the group table is reallocated: a graph captured against the old pointers is stale
        self.plan_generation = 0

    def set_graph_capturable(self, flag=True):
        """Opt-in CUDA-graph-capturable mode, off by default.

        When on, each parameter's state["step"] is a 0-d int64 tensor on its device (a view into the step array of the tensor
        table it is updated through), and step() launches vb_bert_adam_step_sched: the kernels evaluate the learning-rate
        schedule from those counters and advance them, and read each group's lr, weight decay and schedule from a device table.
        step() then reads nothing back and uploads nothing while the groups stay as they are, so it can be captured and replayed;
        a group table is uploaded again (outside any graph) when a group's lr, weight_decay or schedule parameters changed.
        The bits equal those of the default mode. Switching on moves the integer steps to the device, switching off brings them
        back as ints; state_dict() gives ints in either mode. ValueError for a schedule other than the four classes of
        SCHEDULES (a subclass included), and for a step() under stream capture that would have to create state, build a table or
        upload the group table."""
        flag = bool(flag)
        if flag:
            for group in self.param_groups:
                _group_row(group)
        if flag != self._capturable:
            self._capturable = flag
            self._convert_steps()
        return self

    def _convert_steps(self):
        """state["step"] as this mode keeps it (a device tensor or an int); the tables are built again at the next step."""
        for group in self.param_groups:
            for p in group["params"]:
                state = self.state.get(p)
                if not state or "step" not in state:
                    continue
                step = state["step"]
                if self._capturable:
                    step = step.detach().reshape(()) if torch.is_tensor(step) else torch.tensor(int(step))
                    state["step"] = step.to(device=p.device, dtype=torch.int64).clone()
                elif torch.is_tensor(step):
                    state["step"] = int(step.item())
        self._plans.clear()
        self._groups = None
        self.plan_generation += 1

    def state_dict(self):
        """As torch's, with every step a Python int, so that a checkpoint loads into either mode and into the reference."""
        sd = super().state_dict()
        sd["state"] = {k: (dict(v, step=int(v["step"].item())) if torch.is_tensor(v.get("step")) else v)
                       for k, v in sd["state"].items()}
        return sd

    def load_state_dict(self, state_dict):
        """Steps given as ints or tensors, in either mode."""
        super().load_state_dict(state_dict)
        self._convert_steps()

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
        if self._capturable:
            return self._step_sched(loss)
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

    def _step_sched(self, loss):
        """step() in graph-capturable mode: one vb_bert_adam_step_sched per (b1, b2, e, max_grad_norm), nothing read back. Every
        refusal under capture comes before anything is allocated or launched."""
        capturing = torch.cuda.is_available() and torch.cuda.is_current_stream_capturing()
        buckets = {}
        for gi, group in enumerate(self.param_groups):
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
                    if capturing:
                        raise _capture_refusal("allocate next_m / next_v")
                    state["step"] = torch.zeros((), dtype=torch.int64, device=p.device)
                    state["next_m"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                    state["next_v"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                buckets.setdefault(key, []).append((p, state, gi, float(group["weight_decay"])))
        if not buckets:
            return loss
        dev = next(iter(buckets.values()))[0][0].device
        self.sync_group_table(dev, capturing)
        plans = [(key, self._sched_plan(key, items, capturing)) for key, items in buckets.items()]
        groups = self._groups
        for key, plan in plans:
            b1, b2, e, max_norm = key
            st = torch.cuda.current_stream(dev).cuda_stream
            P = ctypes.c_void_p
            with torch.cuda.device(dev), deterministic(dev, adam_chunks=plan["n_chunks"]):
                _lib.check(_lib.lib().vb_bert_adam_step_sched(
                    P(plan["dev_tab"].data_ptr()), plan["n"], plan["n_chunks"], P(groups["dev"].data_ptr()), len(groups["rows"]),
                    P(plan["steps"].data_ptr()), P(plan["sumsq"].data_ptr()), P(plan["lr_out"].data_ptr()),
                    ctypes.c_double(b1), ctypes.c_double(b2), ctypes.c_double(e), ctypes.c_double(max_norm), P(st)),
                    "vb_bert_adam_step_sched")
        # the kernel wrote through raw pointers: tell autograd / the bf16 weight caches that the values changed
        torch.autograd.graph.increment_version([p for _, plan in plans for p in plan["params"]])
        return loss

    def sync_group_table(self, dev=None, capturing=False):
        """Upload the group table when a group's lr, weight_decay or schedule parameters changed (O(groups) to check). The copy
        is stream-ordered on the current stream. step() does this itself; a caller that replays a graph holding step() calls it
        before the replay (graphs.GraphedStep does)."""
        rows = [_group_row(g) for g in self.param_groups]
        g = self._groups
        if g is not None and g["rows"] == rows:
            return
        if capturing:
            raise _capture_refusal("upload its group table")
        dev = g["dev"].device if dev is None else dev
        host = np.array(rows, dtype=_GROUP_DTYPE)
        if g is None or g["dev"].numel() != host.nbytes or g["dev"].device != dev:
            buf = torch.empty(host.nbytes, device=dev, dtype=torch.uint8)
            self.plan_generation += 1
        else:
            buf = g["dev"]
        # fresh pinned staging (torch's host allocator recycles it only after the async copy has run)
        staging = torch.empty(host.nbytes, dtype=torch.uint8, pin_memory=True)
        staging.numpy()[:] = host.view(np.uint8)
        with torch.cuda.device(dev):
            buf.copy_(staging, non_blocking=True)
        self._groups = dict(rows=rows, host=host, dev=buf)

    def _sched_plan(self, key, items, capturing):
        """The device tensor table, step array and lr_out of one bucket, built again when its set of tensors changed."""
        ident = tuple((p.data_ptr(), p.grad.data_ptr(), st["next_m"].data_ptr(), st["next_v"].data_ptr(), p.numel(), gi)
                      for p, st, gi, _ in items)
        plan = self._plans.get(key)
        if plan is not None and plan["ident"] == ident:
            return plan
        if capturing:
            raise _capture_refusal("build its tensor table")
        dev = items[0][0].device
        tab = np.zeros(len(items), dtype=_TABLE_DTYPE)
        chunk = 0
        for i, (p, st, gi, wd) in enumerate(items):
            tab[i] = (p.data_ptr(), p.grad.data_ptr(), st["next_m"].data_ptr(), st["next_v"].data_ptr(), p.numel(), 0.0, wd,
                      chunk, gi)
            chunk += (p.numel() + _lib.VB_ADAM_CHUNK - 1) // _lib.VB_ADAM_CHUNK
        host_groups = self._groups["host"]
        _lib.check(_lib.lib().vb_bert_adam_sched_check(ctypes.c_void_p(tab.ctypes.data), len(items), chunk,
                                                       ctypes.c_void_p(host_groups.ctypes.data), len(host_groups)),
                   "vb_bert_adam_sched_check")
        steps = torch.stack([st["step"].to(device=dev, dtype=torch.int64).reshape(()) for _, st, _, _ in items])
        plan = dict(ident=ident, n=len(items), n_chunks=chunk, steps=steps, params=[p for p, _, _, _ in items],
                    sumsq=torch.empty(len(items), device=dev, dtype=torch.float32),
                    lr_out=torch.zeros(len(items), device=dev, dtype=torch.float32),
                    dev_tab=torch.from_numpy(tab.view(np.uint8).copy()).to(dev))
        for i, (_, st, _, _) in enumerate(items):
            st["step"] = steps[i]   # a view: the kernels advance it
        self._plans[key] = plan
        self.plan_generation += 1
        return plan

    def last_lr(self):
        """Graph-capturable mode: {parameter: lr its latest update used} as the kernels reported it (lr_out); reads the device."""
        return {p: float(lr) for plan in self._plans.values() for p, lr in zip(plan["params"], plan["lr_out"].tolist())}

    def _graph_signature(self):
        """What a captured step bakes in: the tables' addresses and the (b1, b2, e, max_grad_norm) kernel arguments."""
        return (self._capturable, self.plan_generation,
                tuple((float(g["b1"]), float(g["b2"]), float(g["e"]), float(g["max_grad_norm"]), len(g["params"]))
                      for g in self.param_groups))

    def _graph_params(self):
        return [p for plan in self._plans.values() for p in plan["params"]]

