"""CUDA-graph training steps: capture one whole training step (gradient zeroing, forward, backward and, with several ranks, the
gradient all-reduce) and replay it: the host enqueues one graph launch per step instead of hundreds of kernel launches from
Python. Whether that shortens a step depends on whether the step was host-bound (DESIGN.md §4, scripts/bench_graphs.py).

Dropout stays correct because the model runs in graph-capturable mode (BertVisualModel.set_graph_capturable): the step counter
is a device tensor that the graph itself increments, and the kernels read the dropout seed offset from device memory when they
run (vb_set_dropout_offset). Every replay therefore draws the masks an eager step would draw at the same dropout state.

The optimizer step can be part of the graph: GraphedStep(model, sync, optimizer=opt) with a visualbert_b200.BertAdam switches it
to graph-capturable mode (BertAdam.set_graph_capturable), where the kernels evaluate the learning-rate schedule from step
counters in device memory. Without `optimizer` it stays outside, as any other optimizer must: it updates the parameters in place
after the replay, and every replay re-casts the compute weights from them.
"""
import collections

import torch


def _signature(batch):
    sig = []
    for k in sorted(batch):
        v = batch[k]
        sig.append((k, tuple(v.shape), v.dtype, v.device) if torch.is_tensor(v) else (k, v))
    return tuple(sig)


class _Captured:
    def __init__(self, graph, inputs, outputs, opt_signature=None, opt_params=()):
        self.graph, self.inputs, self.outputs = graph, inputs, outputs
        self.opt_signature, self.opt_params = opt_signature, opt_params


class GraphedStep:
    """step = GraphedStep(model, sync); out = step(batch) runs one training step on `batch` and returns the model's output dict.

    model: a TrainVisualBERTObjective in training mode; its BertVisualModel is switched to graph-capturable mode. sync: the
    parallel.FlatGradSync that owns the gradients (they must live at a fixed address). loss_scale: factor applied to the loss
    before backward (default sync.loss_scale(), i.e. 1 / world size, with the all-reduce told the loss was prescaled).

    The first `warmup` calls at a new input-shape signature run eagerly on a side stream, as torch's capture recipe asks (they
    are real steps, and they size the library's lazily allocated workspaces); the next call captures the step and replays it.
    Each call advances the dropout state by exactly one step, whichever way it ran. Inputs are copied into the graph's static
    buffers; the returned outputs are the graph's and stay valid until the next call. Graphs are kept per signature in an LRU
    cache of `max_graphs` entries, each with its own memory pool (replays of different shapes interleave in any order, so pools
    are not shared); an evicted graph is freed. Raises ValueError for what cannot be captured (see set_graph_capturable, the
    vqa_advanced head, MLM rows that are not given); nothing is cached then. Pretraining batches give one shape when their
    masked_lm_rows have a fixed capacity (parallel.BatchPrefetcher(mlm_rows_capacity=N)).

    optimizer: None (the caller steps its optimizer after each call), or a visualbert_b200.BertAdam, which is switched to
    graph-capturable mode and stepped at the end of every step, after the all-reduce. Before each replay its group table is
    uploaded if a group's lr, weight decay or schedule changed; a graph whose optimizer tables were rebuilt since its capture
    (load_state_dict, a new set of tensors) or whose (b1, b2, e, max_grad_norm) changed is dropped and captured again. With
    gradient accumulation the optimizer must stay outside (it steps once per several calls).

    The set of trainable parameters (requires_grad) and the activation-checkpointing and FFN-recompute flags
    (set_activation_checkpointing, set_ffn_recompute) are part of the signature: after a parameter is frozen or unfrozen, or a
    flag changes, the next calls warm up and capture again, as for a new input shape."""

    def __init__(self, model, sync, loss_scale=None, warmup=1, max_graphs=4, optimizer=None):
        if not model.training:
            raise ValueError("GraphedStep: the model must be in training mode")
        if optimizer is not None:
            from .optimization import BertAdam
            if not isinstance(optimizer, BertAdam):
                raise ValueError("GraphedStep: only a visualbert_b200.BertAdam can be captured with the step (its schedule runs on "
                                 f"the device), not {type(optimizer).__name__}; step other optimizers after each call")
            optimizer.set_graph_capturable(True)
        self.model, self.sync, self.optimizer = model, sync, optimizer
        self.loss_scale = loss_scale
        self.warmup = int(warmup)
        self.max_graphs = int(max_graphs)
        self.graphs = collections.OrderedDict()
        self._eager_calls = collections.OrderedDict()   # signature -> eager calls, for signatures not captured yet (bounded)
        self._side = None
        model.bert.set_graph_capturable(True)

    def _step(self, batch):
        self.sync.zero()
        out = self.model(**batch)
        scale = self.sync.loss_scale() if self.loss_scale is None else self.loss_scale
        loss = out["loss"]
        (loss if scale == 1.0 else loss * scale).backward()
        if self.sync.world_size() > 1:
            self.sync.allreduce(prescaled=True)
        if self.optimizer is not None:
            self.optimizer.step()
        return out

    def _eager(self, batch):
        cur = torch.cuda.current_stream()
        if self._side is None or self._side.device != cur.device:
            self._side = torch.cuda.Stream(device=cur.device)
        self._side.wait_stream(cur)
        with torch.cuda.stream(self._side):
            out = self._step(batch)
        cur.wait_stream(self._side)
        return out

    def _capture(self, batch):
        opt = self.optimizer
        if opt is not None and not opt._capturable:
            raise ValueError("GraphedStep: the optimizer left graph-capturable mode (BertAdam.set_graph_capturable(False)); "
                             "every replay would apply the captured step's learning rates")
        inputs = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in batch.items()}
        graph = torch.cuda.CUDAGraph()
        torch.cuda.synchronize()
        with torch.cuda.graph(graph):   # a private memory pool per graph
            outputs = self._step(inputs)
        if opt is None:
            return _Captured(graph, inputs, outputs)
        return _Captured(graph, inputs, outputs, opt._graph_signature(), opt._graph_params())

    def __call__(self, batch):
        # which parameters train is part of the signature: a graph writes the gradients of the set it was captured with; so is
        # activation checkpointing and FFN recomputation, which change the calls (and the memory) of the step
        enc = self.model.bert.encoder
        sig = (_signature(batch), tuple(p.requires_grad for p in self.model.parameters()), enc.activation_checkpointing,
               enc.ffn_recompute)
        entry = self.graphs.get(sig)
        if entry is not None and self.optimizer is not None:
            if entry.opt_signature != self.optimizer._graph_signature():   # the graph holds stale pointers or arguments
                del self.graphs[sig]
                entry.graph.reset()
                entry = None
            else:
                self.optimizer.sync_group_table()   # a stream-ordered upload outside the graph, only on a change
        if entry is None:
            n = self._eager_calls.get(sig, 0)
            if n < self.warmup:
                self._eager_calls[sig] = n + 1
                self._eager_calls.move_to_end(sig)
                while len(self._eager_calls) > 4 * self.max_graphs:
                    self._eager_calls.popitem(last=False)
                return self._eager(batch)
            entry = self._capture(batch)   # an exception here leaves nothing cached
            self._eager_calls.pop(sig, None)
            self.graphs[sig] = entry
            while len(self.graphs) > self.max_graphs:
                _, old = self.graphs.popitem(last=False)
                old.graph.reset()
        else:
            self.graphs.move_to_end(sig)
            for k, v in entry.inputs.items():
                if torch.is_tensor(v):
                    v.copy_(batch[k])
        entry.graph.replay()
        if entry.opt_params:
            # the optimizer kernels wrote the parameters through raw pointers, as the eager step does
            torch.autograd.graph.increment_version(entry.opt_params)
        return entry.outputs
