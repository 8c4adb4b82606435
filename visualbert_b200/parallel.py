"""Data-parallel plumbing (SURVEY.md §8e): one process per GPU, replicated weights, and ONE all-reduce
per step over a flat fp32 gradient buffer — replacing the reference's single-process nn.DataParallel
(visualbert/models/model_wrapper.py:146: per-step parameter broadcast + gradient reduce to GPU 0).

`FlatGradSync` makes every `p.grad` a view into one contiguous buffer, so the collective needs no
packing copy; `allreduce()` issues a single `torch.distributed.all_reduce` (NCCL over NVLink on the
GPU machine, gloo in the CPU tests) and divides by the world size, i.e. the mean of per-rank mean losses —
the same semantics as the reference's `loss.mean()` over DataParallel replicas (model_wrapper.py:75).
"""
import torch
import torch.distributed as dist


class FlatGradSync:
    def __init__(self, module, process_group=None, reduce_dtype=torch.float32):
        """reduce_dtype: torch.float32 (default: exact sum of the ranks' fp32 gradients) or torch.bfloat16 (half the
        bytes on the wire; the sum is rounded to bf16 — an explicit opt-in, not reference semantics)."""
        self.reduce_dtype = reduce_dtype
        self._wire = None
        seen, self.params = set(), []

        def add(p):
            if p.requires_grad and id(p) not in seen:  # tied weights appear once
                seen.add(id(p))
                self.params.append(p)

        # modules may ask for groups of parameters to be adjacent (BertLayer: query|key|value weights, then
        # their biases, so the fused [3H, H] weight-gradient GEMM writes straight into this buffer)
        for m in module.modules():
            for group in getattr(m, "_vb_adjacent_param_groups", lambda: ())():
                for p in group:
                    add(p)
        for p in module.parameters():
            add(p)
        if not self.params:
            raise ValueError("FlatGradSync: module has no trainable parameters")
        dev = self.params[0].device
        # tensors inside an adjacency group stay back to back (the fused [3H, H] gradient needs that); every other
        # tensor starts on a 256-byte boundary so 16-byte vector accesses (red.add.v4, the optimizer) stay legal
        # whatever the sizes before it (decoder bias 30522, classifier bias 3129, ...)
        packed = set()
        for m in module.modules():
            for group in getattr(m, "_vb_adjacent_param_groups", lambda: ())():
                packed.update(id(p) for p in group[1:])
        offsets, off = [], 0
        for p in self.params:
            if id(p) not in packed:
                off = (off + 63) // 64 * 64
            offsets.append(off)
            off += p.numel()
        self.flat = torch.zeros(off, device=dev, dtype=torch.float32)
        self.group = process_group
        self.views = []
        for p, o in zip(self.params, offsets):
            v = self.flat[o: o + p.numel()].view_as(p)
            p.grad = v
            p._vb_direct_grad = True   # opt in: the backward kernels accumulate straight into this view (ops._grad_targets)
            self.views.append(v)

    def zero(self):
        """Replaces optimizer.zero_grad(): one memset; re-attaches views a caller may have dropped."""
        self.flat.zero_()
        for p, v in zip(self.params, self.views):
            if p.grad is not v:
                p.grad = v

    def world_size(self):
        return dist.get_world_size(self.group) if dist.is_available() and dist.is_initialized() else 1

    def loss_scale(self):
        """1 / world_size. Multiply the loss by it before backward() and call allreduce(prescaled=True): the mean over
        ranks (reference: `loss.mean()` over DataParallel replicas, model_wrapper.py:75) then costs no extra pass over
        the 440 MB buffer."""
        return 1.0 / self.world_size()

    def allreduce(self, prescaled=False):
        """The single collective of the step (sum over ranks; divided by the world size unless the loss was already
        scaled by loss_scale()). No-op for a lone process."""
        n = self.world_size()
        if n > 1:
            if self.reduce_dtype == torch.float32:
                dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=self.group)
            else:
                if self._wire is None:
                    self._wire = torch.empty(self.flat.numel(), device=self.flat.device, dtype=self.reduce_dtype)
                self._wire.copy_(self.flat)
                dist.all_reduce(self._wire, op=dist.ReduceOp.SUM, group=self.group)
                self.flat.copy_(self._wire)
            if not prescaled:
                self.flat.div_(n)
        return self.flat


def shard_batch(batch, rank, world_size):
    """Split every tensor of a reference-style batch dict on dim 0 (what DataParallel's scatter did,
    visualbert/models/train.py:146,179), keeping non-tensors."""
    out = {}
    for k, v in batch.items():
        if torch.is_tensor(v):
            n = v.shape[0]
            if n % world_size != 0:
                raise ValueError(f"batch dim {n} of '{k}' is not divisible by world size {world_size}")
            per = n // world_size
            out[k] = v[rank * per: (rank + 1) * per]
        else:
            out[k] = v
    return out


_TEXT_KEYS = {"input_ids": 0, "token_type_ids": 0, "input_mask": 0, "masked_lm_labels": -1}
_REGION_KEYS = {"image_mask": 0, "visual_embeddings_type": 0, "confidence": 0}          # region dim last
_REGION_ROW_KEYS = {"visual_embeddings": 0, "position_embeddings_visual": 0, "image_text_alignment": -1}  # region dim -2


def pad_batch(batch, text_len, regions, entities=None):
    """A reference batch dict padded to fixed shapes: text tensors to `text_len` positions, region tensors to `regions`
    (CUDA graphs replay one captured shape; AllenNLP pads each batch only to its longest example, so without this no shape
    would recur). Works for every head, 3-D VCR inputs included (the text / region dimension is found from the end).
    Padding: ids, token types and masks 0, masked_lm_labels -1, features 0, image_text_alignment -1; the flickr head's soft
    region targets (label [.., entities, regions]) get 0 and, with `entities`, flickr_position (-1) and label are padded to that
    many entities too (without it the entity count of a flickr batch varies, and such batches need bucketing by it).
    masked_lm_rows (flat indices b * (T + V) + t, -1 = capacity padding) are remapped to b * (text_len + regions) + t.
    Semantics: the padded positions are masked keys, whose key bias of
    -10000 gives them exactly zero probability in the fp32 softmax, so valid positions equal those of the unpadded batch to
    within rounding (row statistics of shorter batches are summed in another order); padded positions hold finite values
    nobody reads, and padded MLM rows carry no target."""
    def pad(t, dim, size, value):
        n = t.shape[dim]
        if n > size:
            raise ValueError(f"pad_batch: dimension {dim} of size {n} exceeds the padded size {size}")
        if n == size:
            return t
        shape = list(t.shape)
        shape[dim] = size - n
        return torch.cat((t, t.new_full(shape, value)), dim=dim)

    out = {}
    for k, v in batch.items():
        if not torch.is_tensor(v):
            out[k] = v
        elif k in _TEXT_KEYS:
            out[k] = pad(v, -1, text_len, _TEXT_KEYS[k])
        elif k in _REGION_KEYS:
            out[k] = pad(v, -1, regions, _REGION_KEYS[k])
        elif k in _REGION_ROW_KEYS:
            out[k] = pad(v, -2, regions, _REGION_ROW_KEYS[k])
        elif k == "label" and "flickr_position" in batch:
            out[k] = pad(v, -1, regions, 0)
            if entities is not None:
                out[k] = pad(out[k], -2, entities, 0)
        elif k == "flickr_position" and entities is not None:
            out[k] = pad(v, -1, entities, -1)
        elif k == "masked_lm_rows":
            ids = batch["input_ids"]
            T = ids.shape[-1]
            V = batch["visual_embeddings"].shape[-2] if torch.is_tensor(batch.get("visual_embeddings")) else 0
            b, t = torch.div(v, T + V, rounding_mode="floor"), v.remainder(T + V)
            if T + V != text_len + regions:
                out[k] = torch.where(v >= 0, b * (text_len + regions) + t, v)
            else:
                out[k] = v
        else:
            out[k] = v
    return out


class BatchPrefetcher:
    """Host→device staging of input batches on a copy stream, so the copy of batch i+1 overlaps the step on batch i.

    Replaces the `.cuda()` the reference's training loop does on the batch before every forward
    (`visualbert/models/model_wrapper.py:64-70`; DataParallel's scatter from host, `train.py:146`). Host tensors should
    be pinned. Usage:

        pf = BatchPrefetcher(device)
        staged = pf.stage(next(it))
        for ...:
            batch = pf.take(staged)            # compute stream waits for the copy, not the host
            staged = pf.stage(next(it))        # enqueue the next copy before launching this step
            loss = step(batch)
    """

    def __init__(self, device, mlm_rows=True, mlm_rows_capacity=None):
        """mlm_rows_capacity=N: `masked_lm_rows` always has N entries, the MLM targets followed by -1 ("no target"), so that every
        pretraining batch of one shape gives one tensor shape (what a CUDA graph replays; the model reads -1 entries as padding
        in graph-capturable mode, BertVisualModel.set_graph_capturable). A batch with more than N targets raises."""
        self.device = torch.device(device)
        self.stream = torch.cuda.Stream(device=self.device)
        self.mlm_rows = mlm_rows
        self.mlm_rows_capacity = mlm_rows_capacity

    @staticmethod
    def labelled_rows(host_batch, capacity=None):
        """Flat indices b * (T + V) + t of the MLM targets, from the HOST copy of the labels (what
        TrainVisualBERTObjective.forward accepts as `masked_lm_rows`): finding them on the device costs a host sync.
        Negative labels are "no target" (the reference's ignore index is -1); a label >= vocab contributes neither loss
        nor gradient in the cross-entropy kernels."""
        labels = host_batch.get("masked_lm_labels")
        if labels is None or labels.is_cuda:
            return None
        vis = host_batch.get("visual_embeddings")
        T = labels.shape[-1]
        V = 0 if vis is None else vis.shape[-2]
        flat = labels.reshape(-1, T)
        b, t = torch.nonzero(flat >= 0, as_tuple=True)
        rows = (b * (T + V) + t).to(torch.int64)
        if capacity is None:
            return rows
        if rows.numel() > capacity:
            raise ValueError(f"BatchPrefetcher: the batch has {rows.numel()} MLM targets, more than mlm_rows_capacity = {capacity}")
        return torch.cat((rows, torch.full((capacity - rows.numel(),), -1, dtype=torch.int64)))

    def stage(self, host_batch):
        if self.mlm_rows and "masked_lm_rows" not in host_batch:
            rows = self.labelled_rows(host_batch, self.mlm_rows_capacity)
            if rows is not None:
                host_batch = dict(host_batch, masked_lm_rows=rows.pin_memory())
        with torch.cuda.stream(self.stream):
            dev = {k: (v.to(self.device, non_blocking=True) if torch.is_tensor(v) else v) for k, v in host_batch.items()}
            ev = torch.cuda.Event()
            ev.record(self.stream)
        return dev, ev

    def take(self, staged):
        dev, ev = staged
        cur = torch.cuda.current_stream(self.device)
        cur.wait_event(ev)
        for v in dev.values():
            if torch.is_tensor(v):
                v.record_stream(cur)  # allocated on the copy stream, consumed on the compute stream
        return dev
