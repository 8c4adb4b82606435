"""torch.autograd bindings of the libvbert_b200 C ABI (include/vbert_b200.h).

PyTorch supplies device memory, the current stream and the autograd graph; every FLOP of the
encoder path runs in the sm_90a kernels. There is no fallback: on a machine without the library or
without a CUDA device these ops raise.

Activations are bf16; parameters are the model's fp32 master weights, cast to bf16 "compute weights"
in a WeightBank by one vb_cast_multi launch per refresh. Parameter gradients come back in fp32.
"""
import contextlib
import ctypes
import functools
import threading

import torch

from . import _lib

_BF16 = torch.bfloat16


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return 0 if t is None else t.data_ptr()


def _require_cuda(t, what):
    if not t.is_cuda:
        raise _lib.VBertLibraryError(
            f"{what}: tensor is on {t.device}; visualbert_b200 runs only on CUDA (sm_90a) — no CPU fallback")


# --------------------------------------------------------------------------------------------
# workspaces: backward scratch is shared by all layers of a step (same stream, sequential use)
# --------------------------------------------------------------------------------------------
_bwd_scratch_cache = {}


def _bwd_scratch(dev, M, H, I, A, need_drop):
    """Backward scratch of an encoder call over M rows (B * S dense, the packed total unpadded): views of the first M rows of
    buffers that are kept per device and only grow (by at least 1/4, in whole 256-row steps) when a call has more rows than
    any before. The row count of unpadded batches changes from step to step; a cache keyed on it would reallocate every
    backward."""
    key = (dev, H, I, A)
    c = _bwd_scratch_cache.get(key)
    if c is None or c["rows"] < M:
        rows = M if c is None else max(M, c["rows"] + c["rows"] // 4)
        rows = (rows + 255) // 256 * 256
        for k in [k for k in _bwd_scratch_cache if k[0] == dev]:   # free the smaller buffers before allocating
            del _bwd_scratch_cache[k]
        c = dict(rows=rows, d_pre=torch.empty(rows, H, device=dev, dtype=_BF16), d_pre_drop=None,
                 d_big=torch.empty(rows, max(I, 3 * H), device=dev, dtype=_BF16),
                 d_x1=torch.empty(rows, H, device=dev, dtype=_BF16), d_ctx=torch.empty(rows, H, device=dev, dtype=_BF16),
                 drow=torch.empty(A * rows, device=dev, dtype=torch.float32))
        _bwd_scratch_cache[key] = c
    if need_drop and c["d_pre_drop"] is None:
        c["d_pre_drop"] = torch.empty(c["rows"], H, device=dev, dtype=_BF16)
    w = {k: (c[k][:M] if c[k] is not None else None) for k in ("d_pre", "d_pre_drop", "d_big", "d_x1", "d_ctx")}
    w["drow"] = c["drow"][:A * M]   # [B, A, S] dense, [heads, total] unpadded
    return w


_det_ws_cache = {}
_det_current = threading.local()   # the (pointer, bytes) this thread last handed to vb_set_deterministic


@functools.lru_cache(maxsize=256)
def _det_workspace_bytes(sms, rows, H, I, vocab, adam_chunks):
    """vb_deterministic_workspace_bytes on the current device; the split factors it sizes come from the SM count, which is part
    of the cache key so that devices with different SM counts in one process each get their own size."""
    need = int(_lib.lib().vb_deterministic_workspace_bytes(rows, H, I, vocab, adam_chunks))
    if need < 0:
        _lib.check(1, "vb_deterministic_workspace_bytes")
    return need


def _det_workspace(dev, rows=0, H=0, I=0, vocab=0, adam_chunks=0):
    """The deterministic-mode workspace of a device (vb_deterministic_workspace_bytes): one buffer per device that only grows,
    like _bwd_scratch. Every library call uses it from its start, in stream order."""
    with torch.cuda.device(dev):
        need = _det_workspace_bytes(torch.cuda.get_device_properties(dev).multi_processor_count, rows, H, I, vocab, adam_chunks)
    ws = _det_ws_cache.get(dev)
    if ws is None or ws.numel() < need:
        _det_ws_cache.pop(dev, None)   # free the smaller buffer before allocating
        with _unfilled():
            ws = torch.empty(max(need, 256), device=dev, dtype=torch.uint8)
        _det_ws_cache[dev] = ws
    return ws


@contextlib.contextmanager
def _unfilled():
    """Allocations inside skip torch's fill of uninitialized memory, which torch.use_deterministic_algorithms turns on by default
    (torch.utils.deterministic.fill_uninitialized_memory): used only around buffers the library writes completely before anything
    reads them (the activation arena, backward scratch, embedding and decoder outputs), where the fill is pure HBM traffic — over
    12 GB per training step at the benchmark shape. Nothing is changed when torch's deterministic mode is off."""
    if not torch.are_deterministic_algorithms_enabled():
        yield
        return
    du = torch.utils.deterministic
    old = du.fill_uninitialized_memory
    du.fill_uninitialized_memory = False
    try:
        yield
    finally:
        du.fill_uninitialized_memory = old


@contextlib.contextmanager
def deterministic(dev, rows=0, H=0, I=0, vocab=0, adam_chunks=0):
    """Run the library calls inside in deterministic mode (vb_set_deterministic) when torch.use_deterministic_algorithms is on
    (warn_only included): every gradient reduction then adds in a fixed order, so the same inputs give the same bits. The mode is
    a thread-local flag of the library and the autograd engine runs backward on its own thread, so it is set around each call,
    not once per step; on exit the thread's previous setting comes back, so scopes may nest. Buffers allocated inside are
    _unfilled. With torch's flag off nothing is called and the default kernels run."""
    if not torch.are_deterministic_algorithms_enabled():
        yield
        return
    ws = _det_workspace(dev, rows, H, I, vocab, adam_chunks)
    prev = getattr(_det_current, "ws", (None, 0))
    _lib.check(_lib.lib().vb_set_deterministic(ws.data_ptr(), ws.numel()), "vb_set_deterministic")
    _det_current.ws = (ws.data_ptr(), ws.numel())
    try:
        with _unfilled():
            yield
    finally:
        _lib.lib().vb_set_deterministic(prev[0], prev[1])
        _det_current.ws = prev


def cast_to_bf16(src, out=None):
    """fp32 -> bf16 through vb_cast_f32_to_bf16 (numel must be a multiple of 8)."""
    _require_cuda(src, "cast_to_bf16")
    src = src.contiguous()
    if out is None:
        out = torch.empty(src.shape, device=src.device, dtype=_BF16)
    with torch.cuda.device(src.device):   # the library launches on the CURRENT device's stream: make it the tensor's
        _lib.check(_lib.lib().vb_cast_f32_to_bf16(ctypes.c_void_p(src.data_ptr()), ctypes.c_void_p(out.data_ptr()),
                                                  ctypes.c_int64(src.numel()), _stream()), "vb_cast_f32_to_bf16")
    return out


def mask_bias(input_mask, image_mask):
    """(1 - cat(input_mask, image_mask)) * -10000 as fp32 [B, T+V] (reference M.py:1417, 1286-1294)."""
    _require_cuda(input_mask, "mask_bias")
    B, T = input_mask.shape
    V = 0 if image_mask is None else image_mask.shape[1]
    im = input_mask.to(torch.int64).contiguous()
    vm = None if image_mask is None else image_mask.to(torch.int64).contiguous()
    out = torch.empty(B, T + V, device=input_mask.device, dtype=torch.float32)
    with torch.cuda.device(input_mask.device):
        _lib.check(_lib.lib().vb_mask_bias(ctypes.c_void_p(im.data_ptr()), ctypes.c_void_p(_ptr(vm)),
                                           ctypes.c_void_p(out.data_ptr()), B, T, V, _stream()), "vb_mask_bias")
    return out


def _grad_targets(params, adjacent_groups=()):
    """Direct-accumulate mode — OPT-IN: only parameters a gradient owner has flagged with `_vb_direct_grad = True`
    (parallel.FlatGradSync does, for the views of its flat buffer) get their gradients written straight into `.grad`
    by the kernels (all gradient outputs of the C ABI are `+=`), with autograd receiving None. Everyone else — plain
    optimizers, DDP with gradient_as_bucket_view, tensor / post-accumulate hooks, torch.autograd.grad — goes through
    AccumulateGrad as usual: the caller allocates fresh zero buffers and returns them to autograd.
    Additionally every `.grad` must be a contiguous fp32 tensor of the parameter's shape, and the parameters of each
    adjacent group must be laid out back to back."""
    for p in params:
        g = p.grad
        if (not getattr(p, "_vb_direct_grad", False) or g is None or g.dtype != torch.float32 or not g.is_contiguous()
                or g.device != p.device or g.shape != p.shape):
            return None
    for group in adjacent_groups:
        for a, b in zip(group[:-1], group[1:]):
            if a.grad.data_ptr() + a.grad.numel() * 4 != b.grad.data_ptr():
                return None
    return [p.grad for p in params]


class WeightBank:
    """Every bf16 compute copy the CUDA path reads (packed q|k|v, attention-output, FFN matrices of all layers, the visual
    projection, the tied MLM decoder table) plus the fp32 packed q|k|v biases, refreshed from the fp32 master
    parameters by ONE vb_cast_multi launch.

    `refresh(force=True)` is called at the start of every training-mode forward: the masters may have been changed by
    anything — the reference BertAdam updates through `p.data` (optimization.py:293), which does not bump
    `Tensor._version`, so version-keyed caching alone would silently train on stale bf16 weights. In eval mode the copy
    is redone only when a (data_ptr, _version) signature changed (load_state_dict, manual edits through autograd-visible
    ops)."""

    def __init__(self):
        self.sig = None
        self.items = []       # (src parameter, dst tensor, dst_is_fp32)
        self.table = None
        self.n_chunks = 0
        self.generation = 0

    def _signature(self, params):
        return tuple((p.data_ptr(), p._version) for p in params)

    def bind(self, items):
        """items: list of (src fp32 parameter, dst tensor [contiguous view], dst_is_fp32)."""
        import numpy as np
        self.items = items
        arr = (_lib.CastItem * len(items))()
        chunk = 0
        for i, (src, dst, f32) in enumerate(items):
            assert src.dtype == torch.float32 and src.is_contiguous() and dst.is_contiguous() and dst.numel() == src.numel()
            arr[i].src, arr[i].dst, arr[i].numel = src.data_ptr(), dst.data_ptr(), src.numel()
            arr[i].first_chunk, arr[i].dst_fp32 = chunk, 1 if f32 else 0
            chunk += (src.numel() + _lib.VB_CAST_CHUNK - 1) // _lib.VB_CAST_CHUNK
        self.n_chunks = chunk
        raw = np.frombuffer(bytes(arr), dtype=np.uint8).copy()
        self.table = torch.from_numpy(raw).to(items[0][0].device)
        self.ptrs = tuple(src.data_ptr() for src, _, _ in items)
        self.sig = None

    def bound_to(self, params):
        return self.table is not None and self.ptrs == tuple(p.data_ptr() for p in params)

    def refresh(self, force):
        srcs = [s_ for s_, _, _ in self.items]
        sig = self._signature(srcs)
        if not force and sig == self.sig:
            return
        with torch.cuda.device(self.table.device):
            _lib.check(_lib.lib().vb_cast_multi(ctypes.c_void_p(self.table.data_ptr()), len(self.items), self.n_chunks, _stream()),
                       "vb_cast_multi")
        self.sig = sig
        self.generation += 1


class _BankViews:
    """The compute weights of one module: views into a WeightBank. A model that owns the module lists `items()` in its own
    bank, sets `owner` and refreshes that bank once per forward. A module used on its own gets a private bank over its own
    masters at its first CUDA forward (again when the masters moved), refreshed on every get() by WeightBank.refresh's rule."""

    def __init__(self):
        self.buf = None
        self.owner = None     # the owning model's bank: refreshing is the model's job
        self.bank = None      # the private bank of a module without an owner

    def get(self, *masters, train=False):
        if self.owner is None:
            if self.bank is None or not self.bank.bound_to(masters):
                self.bank = WeightBank()
                self.bank.bind(self.items(*masters))
            self.bank.refresh(force=train)
        return self.buf


class LayerWeights(_BankViews):
    """One BertLayer: buf = (packed q|k|v [3H, H], attention output [H, H], intermediate [I, H], output [H, I]) in bf16 and
    the packed fp32 q|k|v bias [3H]."""

    def items(self, q, k, v, o, w1, w2, bq, bk, bv):
        H, I, dev = o.shape[0], w1.shape[0], q.device
        wqkv = torch.empty(3 * H, H, device=dev, dtype=_BF16)
        bqkv = torch.empty(3 * H, device=dev, dtype=torch.float32)
        self.buf = (wqkv, torch.empty(H, H, device=dev, dtype=_BF16), torch.empty(I, H, device=dev, dtype=_BF16),
                    torch.empty(H, I, device=dev, dtype=_BF16), bqkv)
        return [(q, wqkv[0:H], False), (k, wqkv[H:2 * H], False), (v, wqkv[2 * H:], False), (o, self.buf[1], False),
                (w1, self.buf[2], False), (w2, self.buf[3], False),
                (bq, bqkv[0:H], True), (bk, bqkv[H:2 * H], True), (bv, bqkv[2 * H:], True)]


class ProjectionWeights(_BankViews):
    """The visual projection matrix of the embeddings: buf = its bf16 copy."""

    def items(self, w):
        self.buf = torch.empty(w.shape, device=w.device, dtype=_BF16)
        return [(w, self.buf, False)]


class DecoderWeights(_BankViews):
    """The tied MLM decoder: buf = (bf16 copy of the word-embedding matrix with its rows padded to a multiple of 16, fp32
    bias padded likewise). The padding rows are zero (the GEMMs address all of them) and their bias is -30000, so the
    padding columns of the logits vanish in the softmax."""

    def items(self, E, bias):
        V = E.shape[0]
        Vp = (V + 15) // 16 * 16
        self.buf = (torch.zeros(Vp, E.shape[1], device=E.device, dtype=_BF16),
                    torch.full((Vp,), -30000.0, device=E.device, dtype=torch.float32))
        return [(E, self.buf[0][:V], False), (bias, self.buf[1][:V], True)]


def attention_probs(qkv, mbias, B, S, A):
    """Pre-dropout attention maps softmax(QK^T / 8 + mbias) as fp32 [B, A, S, S] from a layer's bf16 qkv [B*S, 3H]
    (vb_attention_probs)."""
    probs = torch.empty(B, A, S, S, device=qkv.device, dtype=torch.float32)
    with torch.cuda.device(qkv.device):
        _lib.check(_lib.lib().vb_attention_probs(qkv.data_ptr(), mbias.data_ptr(), probs.data_ptr(), B, S, A, qkv.shape[1] // 3,
                                                 _stream()), "vb_attention_probs")
    return probs


_GRAD_FIELDS = ("dw_qkv", "db_qkv", "dw_attn_out", "db_attn_out", "dln1_gamma", "dln1_beta",
                "dw_inter", "db_inter", "dw_out", "db_out", "dln2_gamma", "dln2_beta")   # vb_layer_grads


def _grad_sizes(H, I):
    return [3 * H * H, 3 * H, H * H, H, H, H, I * H, I, H * I, H, H, H]


def _layer_grads(params, L, H, I, dev):
    """The vb_layer_grads array of an L-layer backward and the buffer behind it: None when every pointer is a parameter's own
    `.grad` (_grad_targets; q|k|v are one packed output, so each layer's q, k, v weights and biases must be adjacent), else
    one zeroed flat fp32 buffer that _autograd_grads cuts up."""
    groups = []
    for l in range(L):
        qw, qb, kw, kb, vw, vb = params[16 * l: 16 * l + 6]
        groups += [(qw, kw, vw), (qb, kb, vb)]
    direct = _grad_targets(params, groups)
    grads = (_lib.LayerGrads * L)()
    if direct is not None:
        for l in range(L):
            t = direct[16 * l: 16 * l + 16]
            for name, g in zip(_GRAD_FIELDS, (t[0], t[1]) + tuple(t[6:16])):
                setattr(grads[l], name, g.data_ptr())
        return grads, None
    sizes = _grad_sizes(H, I)
    flat = torch.zeros(L * sum(sizes), device=dev, dtype=torch.float32)
    o = flat.data_ptr()
    for l in range(L):
        for name, sz in zip(_GRAD_FIELDS, sizes):
            setattr(grads[l], name, o)
            o += 4 * sz
    return grads, flat


def _autograd_grads(flat, L, H, I):
    """The 16 parameter gradients per layer, in bert_layer order, as views of _layer_grads' flat buffer."""
    out = []
    for part in flat.view(L, -1).unbind(0):
        dwqkv, dbqkv, dwo, dbo, dg1, db1, dwi, dbi, dwout, dbout, dg2, db2 = torch.split(part, _grad_sizes(H, I))
        dwq, dwk, dwv = dwqkv.view(3, H, H).unbind(0)
        dbq, dbk, dbv = dbqkv.view(3, H).unbind(0)
        out += [dwq, dbq, dwk, dbk, dwv, dbv, dwo.view(H, H), dbo, dg1, db1, dwi.view(I, H), dbi, dwout.view(H, I), dbout, dg2, db2]
    return tuple(out)


def _stamp(descs, L, meta, mbias):
    """The per-step fields of a descriptor array: dropout, seed (so a backward draws its forward's dropout streams), mask."""
    for l in range(L):
        d = descs[l]
        d.hidden_dropout, d.attn_dropout, d.seed = meta["hidden_dropout"], meta["attn_dropout"], meta["seed"]
        d.layer_index, d.mask_bias = meta["layer_index0"] + l, _ptr(mbias)


class EncoderPlan:
    """Host-side state of the encoder call (vb_encoder_fwd / vb_encoder_bwd): the ctypes descriptor array is built once per
    (shape, weights) and only its per-step fields (_stamp) are touched afterwards."""

    def __init__(self):
        self.key = None

    def prepare(self, caches, params, B, S, H, A, I, mbias, meta, dev, varlen=None):
        """-> (descs, weights, arena stride per layer, buffer offsets). varlen (unpadded calls): dict(cu_seqlens, max_seq,
        total); B is then the number of sequences, S = max_seq, and mbias is None.

        A forward keeps `descs` for its backward. So a new key gets a NEW array and the old one is never rewritten: a
        backward that runs after a forward of another shape or other weights still describes its own forward's arena."""
        L = len(caches)
        weights = [c.get(*[params[16 * l + i] for i in (0, 2, 4, 6, 10, 12, 1, 3, 5)], train=meta["train"]) for l, c in enumerate(caches)]
        key = (B, S, H, A, I, L, tuple(w[0].data_ptr() for w in weights), tuple(p.data_ptr() for p in params), dev)
        if key != self.key:
            self.descs = (_lib.LayerDesc * L)()
            for l in range(L):
                wqkv, wo, wi, wout, bqkv = weights[l]
                qw, qb, kw, kb, vw, vb, ow, ob, g1, b1, iw, ib, dw, db, g2, b2 = params[16 * l: 16 * l + 16]
                d = self.descs[l]
                d.batch, d.seq, d.hidden, d.heads, d.inter = B, S, H, A, I
                d.w_qkv, d.w_attn_out, d.w_inter, d.w_out = wqkv.data_ptr(), wo.data_ptr(), wi.data_ptr(), wout.data_ptr()
                d.b_qkv, d.b_attn_out, d.ln1_gamma, d.ln1_beta = bqkv.data_ptr(), ob.data_ptr(), g1.data_ptr(), b1.data_ptr()
                d.b_inter, d.b_out, d.ln2_gamma, d.ln2_beta = ib.data_ptr(), db.data_ptr(), g2.data_ptr(), b2.data_ptr()
            self.key = key
        _stamp(self.descs, L, meta, mbias)
        off = (ctypes.c_int64 * _lib.VB_ENCODER_ARENA_BUFFERS)()
        drop = 1 if meta["attn_dropout"] > 0 else 0
        if varlen is None:
            stride = int(_lib.lib().vb_encoder_arena_layout(B, S, H, A, I, drop, off))
        else:
            stride = int(_lib.lib().vb_encoder_arena_layout_varlen(B, S, varlen["total"], H, A, I, drop, off))
            if stride < 0:
                _lib.check(1, "vb_encoder_arena_layout_varlen")
        return self.descs, weights, stride, list(off)


class _EncoderFn(torch.autograd.Function):
    """BertEncoder (M.py:344-371): all layers in ONE vb_encoder_fwd / vb_encoder_bwd call over one activation arena.

    With meta["varlen"] = dict(cu_seqlens, batch, max_seq, total) the call is unpadded: x is [total, H], the packed valid rows
    (sequence b at rows cu_seqlens[b] .. cu_seqlens[b + 1]), mbias is None, and every output is [total, H]
    (vb_encoder_fwd_varlen / vb_encoder_bwd_varlen).

    With meta["attn_maps"] (dense calls only) the L layer outputs are followed by the L attention maps, fp32 [B, A, S, S] views
    of one [L, B, A, S, S] tensor written by vb_encoder_attention_probs right after the forward; they are not differentiable."""

    @staticmethod
    def _shape(x, meta):
        vl = meta.get("varlen")
        if vl is None:
            B, S, H = x.shape
            return B, S, H, B * S, (B, S, H)
        return vl["batch"], vl["max_seq"], x.shape[-1], vl["total"], (vl["total"], x.shape[-1])

    @staticmethod
    def forward(ctx, x, mbias, meta, *params):
        _require_cuda(x, "bert_encoder")
        B, S, H, M, oshape = _EncoderFn._shape(x, meta)
        vl = meta.get("varlen")
        L = len(params) // 16
        I = params[10].shape[0]
        A = meta["heads"]
        x = x.contiguous()
        with torch.cuda.device(x.device), deterministic(x.device, M, H, I):
            descs, weights, stride, off = meta["plan"].prepare(meta["caches"], params, B, S, H, A, I, mbias, meta, x.device, vl)
            arena = torch.empty(L * stride, device=x.device, dtype=torch.uint8)
            if vl is None:
                _lib.check(_lib.lib().vb_encoder_fwd(descs, L, ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(arena.data_ptr()),
                                                     _stream()), "vb_encoder_fwd")
            else:
                _lib.check(_lib.lib().vb_encoder_fwd_varlen(descs, L, vl["cu_seqlens"].data_ptr(), M, x.data_ptr(),
                                                            arena.data_ptr(), _stream()), "vb_encoder_fwd_varlen")
            maps = ()
            if meta.get("attn_maps"):
                if vl is not None:
                    raise ValueError("bert_encoder: attention maps need a dense (padded) call")
                probs = torch.empty(L, B, A, S, S, device=x.device, dtype=torch.float32)
                _lib.check(_lib.lib().vb_encoder_attention_probs(descs, L, arena.data_ptr(), probs.data_ptr(), _stream()),
                           "vb_encoder_attention_probs")
                maps = tuple(probs.unbind(0))
        n = M * H * 2
        outs = tuple(arena[l * stride + off[13]: l * stride + off[13] + n].view(_BF16).view(oshape) for l in range(L))
        ctx.meta, ctx.descs, ctx.arena, ctx.params, ctx.weights = meta, descs, arena, params, weights
        ctx.shape = (B, S, H, A, I, L, M, oshape)
        ctx.save_for_backward(x, mbias)
        ctx.mark_non_differentiable(*outs[:-1], *maps)
        ctx.set_materialize_grads(False)   # or autograd hands backward a 64 MB zero tensor for each of the L - 1 unused outputs
        return outs + maps

    @staticmethod
    def backward(ctx, *douts):
        x, mbias = ctx.saved_tensors
        meta, descs = ctx.meta, ctx.descs
        B, S, H, A, I, L, M, oshape = ctx.shape
        vl = meta.get("varlen")
        dev = x.device
        if douts[L - 1] is None:   # nothing downstream depends on the encoder output
            return (None,) * (3 + 16 * L)
        dy = douts[L - 1].to(_BF16).contiguous()
        grads, flat = _layer_grads(ctx.params, L, H, I, dev)
        with torch.cuda.device(dev), deterministic(dev, M, H, I):
            w = _bwd_scratch(dev, M, H, I, A, meta["hidden_dropout"] > 0)
            sc = _lib.LayerScratch(**{k: _ptr(t) for k, t in w.items()})
            dx = torch.empty(oshape, device=dev, dtype=_BF16)
            _stamp(descs, L, meta, mbias)   # a later forward with the same plan key has stamped its own step since
            if vl is None:
                _lib.check(_lib.lib().vb_encoder_bwd(descs, L, ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(ctx.arena.data_ptr()),
                                                     ctypes.c_void_p(dy.data_ptr()), ctypes.c_void_p(dx.data_ptr()), grads,
                                                     ctypes.byref(sc), _stream()), "vb_encoder_bwd")
            else:
                _lib.check(_lib.lib().vb_encoder_bwd_varlen(descs, L, vl["cu_seqlens"].data_ptr(), M, x.data_ptr(),
                                                            ctx.arena.data_ptr(), dy.data_ptr(), dx.data_ptr(), grads, ctypes.byref(sc),
                                                            _stream()), "vb_encoder_bwd_varlen")
        ctx.arena = None
        if flat is None:
            return (dx, None, None) + (None,) * (16 * L)
        return (dx, None, None) + _autograd_grads(flat, L, H, I)


def _encoder_infer(x, mbias, meta, params):
    """The forward of bert_encoder when no graph can be recorded (the reference evaluates under torch.no_grad(),
    train.py:292-325): vb_encoder_infer / vb_encoder_infer_varlen run every layer through one workspace that does not grow with
    the depth and store nothing a backward would read. The workspace lives for the call only — kept, it would sit in the
    allocator through the next training epoch — and the outputs are freshly allocated: one tensor when only the last layer is
    wanted, one [L, ...] tensor unbound into L views otherwise. Bit for bit the arena path's outputs, dropout included (same
    seed and layer indices in the descriptors)."""
    _require_cuda(x, "bert_encoder")
    B, S, H, M, oshape = _EncoderFn._shape(x, meta)
    vl = meta.get("varlen")
    L = len(params) // 16
    I = params[10].shape[0]
    A = meta["heads"]
    x = x.detach().contiguous()
    if meta.get("attn_maps") and vl is not None:
        raise ValueError("bert_encoder: attention maps need a dense (padded) call")
    with torch.cuda.device(x.device):
        descs = meta["plan"].prepare(meta["caches"], params, B, S, H, A, I, mbias, meta, x.device, vl)[0]
        nbytes = int(_lib.lib().vb_encoder_infer_workspace(B, S, H, A, I, 1 if meta["attn_dropout"] > 0 else 0, -1 if vl is None else M))
        if nbytes < 0:
            _lib.check(1, "vb_encoder_infer_workspace")
        ws = torch.empty(nbytes, device=x.device, dtype=torch.uint8)
        if meta.get("all_layers", True):
            y_all = torch.empty((L,) + tuple(oshape), device=x.device, dtype=_BF16)
            y_last, outs = None, tuple(y_all.unbind(0))
        else:
            y_last = torch.empty(oshape, device=x.device, dtype=_BF16)
            y_all, outs = None, (y_last,)
        probs = torch.empty(L, B, A, S, S, device=x.device, dtype=torch.float32) if meta.get("attn_maps") else None
        if vl is None:
            _lib.check(_lib.lib().vb_encoder_infer(descs, L, x.data_ptr(), ws.data_ptr(), _ptr(y_last), _ptr(y_all), _ptr(probs),
                                                   _stream()), "vb_encoder_infer")
        else:
            _lib.check(_lib.lib().vb_encoder_infer_varlen(descs, L, vl["cu_seqlens"].data_ptr(), M, x.data_ptr(), ws.data_ptr(),
                                                          _ptr(y_last), _ptr(y_all), _stream()), "vb_encoder_infer_varlen")
    return outs + (() if probs is None else tuple(probs.unbind(0)))


def bert_encoder(x, mbias, meta, params):
    """All layers at once. meta: dict(heads, layer_index0, hidden_dropout, attn_dropout, seed, train, caches=[LayerWeights],
    plan=EncoderPlan, optional varlen=unpad_plan(...), optional attn_maps=True, optional all_layers=False); params: 16 tensors
    per layer in bert_layer order. Returns the tuple of all layer outputs (only the last one is differentiable: a caller that
    needs gradients through intermediate outputs calls bert_layer once per layer) — with all_layers=False only the last
    layer's — followed, with attn_maps, by the L detached fp32 [B, A, S, S] attention maps.

    When no graph can be recorded (grad mode off, or neither x nor any parameter requires grad) the call takes the
    forward-only route (_encoder_infer); every other call keeps its activations in the arena of _EncoderFn."""
    if not (torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in params))):
        return _encoder_infer(x, mbias, meta, params)
    outs = _EncoderFn.apply(x, mbias, meta, *params)
    return outs if meta.get("all_layers", True) else outs[len(params) // 16 - 1:]


def unpad_plan(valid):
    """Row bookkeeping of an unpadded call from a [B, S] validity mask (any pattern, not only prefixes): the flat indices
    b * S + s of the valid positions in row-major order (each example keeps the order of its rows), cu_seqlens (int32
    [B + 1]: example b owns packed rows cu[b] .. cu[b + 1]), max_seq and total. One host synchronisation (max_seq and total);
    the index comes from a stable sort instead of nonzero, so it needs none."""
    B, S = valid.shape
    valid = valid.reshape(B, S).bool()
    lens = valid.sum(1, dtype=torch.int32)
    cu = torch.zeros(B + 1, device=valid.device, dtype=torch.int32)
    torch.cumsum(lens, 0, dtype=torch.int32, out=cu[1:])
    max_seq, total = (int(v) for v in torch.stack((lens.max(), cu[-1])).tolist())
    order = torch.sort((~valid).reshape(-1).to(torch.uint8), stable=True).indices
    return dict(index=order[:total], cu_seqlens=cu, batch=B, max_seq=max_seq, total=total)


def bert_layer(x, mbias, meta, params):
    """One layer: bert_encoder over a single layer, so its output is differentiable. meta as for bert_encoder, with one
    LayerWeights in caches, the layer's index as layer_index0 and a plan of the layer's own; params: the 16 tensors of one
    BertLayer in reference order (q.w, q.b, k.w, k.b, v.w, v.b, attention.output dense.w/.b, LayerNorm.w/.b,
    intermediate.dense.w/.b, output.dense.w/.b, LayerNorm.w/.b). With meta["attn_maps"] returns (output, detached fp32
    [B, A, S, S] attention maps)."""
    outs = bert_encoder(x, mbias, meta, params)
    return outs if meta.get("attn_maps") else outs[0]


class _EmbedFn(torch.autograd.Function):
    """BertEmbeddingsWithVisualEmbedding.forward (reference M.py:1198-1257) through vb_embed_fwd / vb_embed_bwd."""

    @staticmethod
    def forward(ctx, meta, input_ids, token_type_ids, visual_type, feats, word, pos, typ, typ_vis, pos_vis, pw, pb, gamma, beta,
                vis_extra=None):
        _require_cuda(word, "bert_embeddings")
        dev = word.device
        B, T = input_ids.shape
        V = 0 if feats is None else feats.shape[1]
        H = word.shape[1]
        M = B * (T + V)
        ids = input_ids.to(torch.int64).contiguous()
        tt = token_type_ids.to(torch.int64).contiguous()
        if V > 0:
            Dv = feats.shape[2]
            vt = visual_type.to(torch.int64).contiguous()
            f = feats.reshape(B * V, Dv)
            fb = cast_to_bf16(f) if f.dtype == torch.float32 else f.to(_BF16).contiguous()
            wp = meta["cache"].get(pw, train=meta.get("train", False))
            with _unfilled():
                vis_proj = torch.empty(B * V, H, device=dev, dtype=_BF16)
            xb = None if vis_extra is None else vis_extra.detach().reshape(B * V, H).to(_BF16).contiguous()
        else:
            Dv, vt, fb, wp, vis_proj, xb = 0, None, None, None, None, None
        with _unfilled():
            pre = torch.empty(M, H, device=dev, dtype=_BF16)
            mean = torch.empty(M, device=dev, dtype=torch.float32)
            rstd = torch.empty(M, device=dev, dtype=torch.float32)
            y = torch.empty(B, T + V, H, device=dev, dtype=_BF16)
        d = _lib.EmbedDesc(
            batch=B, text_len=T, num_regions=V, hidden=H, visual_dim=Dv, vocab=word.shape[0], max_pos=pos.shape[0],
            n_types=typ.shape[0], eps=1e-12, dropout=meta["dropout"], seed=meta["seed"],
            input_ids=ids.data_ptr(), token_type_ids=tt.data_ptr(), visual_type=_ptr(vt), visual_feats=_ptr(fb),
            w_proj=_ptr(wp), b_proj=_ptr(pb), word=word.data_ptr(), pos=pos.data_ptr(), type=typ.data_ptr(),
            pos_vis=pos_vis.data_ptr(), type_vis=typ_vis.data_ptr(), gamma=gamma.data_ptr(), beta=beta.data_ptr(),
            visual_addend=_ptr(xb))
        a = _lib.EmbedActs(vis_proj=_ptr(vis_proj), pre=pre.data_ptr(), mean=mean.data_ptr(), rstd=rstd.data_ptr())
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().vb_embed_fwd(ctypes.byref(d), ctypes.c_void_p(y.data_ptr()), ctypes.byref(a), _stream()),
                       "vb_embed_fwd")
        ctx.desc = d   # the backward's too: it does not read visual_addend
        ctx.shape = (B, T, V, H, Dv)
        ctx.feats_need_grad = feats is not None and feats.requires_grad
        ctx.feats_dtype = None if feats is None else feats.dtype
        ctx.feats_shape = None if feats is None else feats.shape
        ctx.extra = None if (vis_extra is None or not vis_extra.requires_grad) else (vis_extra.shape, vis_extra.dtype)
        ctx.params = (word, pos, typ, typ_vis, pos_vis, pw, pb, gamma, beta)
        ctx.save_for_backward(ids, tt, vt, fb, wp, pb, word, pos, typ, typ_vis, pos_vis, gamma, beta, pre, mean, rstd)
        return y

    @staticmethod
    def backward(ctx, dy):
        ids, tt, vt, fb, wp, pb, word, pos, typ, typ_vis, pos_vis, gamma, beta, pre, mean, rstd = ctx.saved_tensors
        B, T, V, H, Dv = ctx.shape
        dev = word.device
        M = B * (T + V)
        dy = dy.to(_BF16).contiguous()
        f32 = torch.float32
        direct = _grad_targets(ctx.params) if V > 0 else None
        if direct is not None:
            dword, dpos, dtyp, dtyp_vis, dpos_vis, dpw, dpb, dgamma, dbeta = direct
        else:
            dword = torch.zeros_like(word, dtype=f32)
            dpos = torch.zeros_like(pos, dtype=f32)
            dtyp = torch.zeros_like(typ, dtype=f32)
            dtyp_vis = torch.zeros_like(typ_vis, dtype=f32)
            dpos_vis = torch.zeros_like(pos_vis, dtype=f32)
            dgamma = torch.zeros_like(gamma, dtype=f32)
            dbeta = torch.zeros_like(beta, dtype=f32)
            dpw = torch.zeros(H, Dv, device=dev, dtype=f32) if V > 0 else None
            dpb = torch.zeros(H, device=dev, dtype=f32) if V > 0 else None
        with _unfilled():
            d_pre = torch.empty(M, H, device=dev, dtype=_BF16)
            if V > 0:
                d_vis = torch.empty(B * V, H, device=dev, dtype=_BF16)
                d_feats = torch.empty(B * V, Dv, device=dev, dtype=_BF16) if ctx.feats_need_grad else None
            else:
                d_vis = d_feats = None
        a = _lib.EmbedActs(vis_proj=0, pre=pre.data_ptr(), mean=mean.data_ptr(), rstd=rstd.data_ptr())
        g = _lib.EmbedGrads(
            dword=dword.data_ptr(), dpos=dpos.data_ptr(), dtype=dtyp.data_ptr(), dpos_vis=dpos_vis.data_ptr(),
            dtype_vis=dtyp_vis.data_ptr(), dw_proj=_ptr(dpw), db_proj=_ptr(dpb), dgamma=dgamma.data_ptr(),
            dbeta=dbeta.data_ptr(), d_pre=d_pre.data_ptr(), d_vis=_ptr(d_vis), d_feats=_ptr(d_feats))
        with torch.cuda.device(dev), deterministic(dev, M, H, Dv):
            _lib.check(_lib.lib().vb_embed_bwd(ctypes.byref(ctx.desc), ctypes.byref(a), ctypes.c_void_p(dy.data_ptr()),
                                               ctypes.byref(g), _stream()), "vb_embed_bwd")
        dfe = None
        if d_feats is not None:
            dfe = d_feats.view(ctx.feats_shape).to(ctx.feats_dtype)
        # the gradient of anything added to the projected region rows is d_vis itself
        dex = None if ctx.extra is None else d_vis.view(ctx.extra[0]).to(ctx.extra[1])
        if direct is not None:
            return (None, None, None, None, dfe) + (None,) * 9 + (dex,)
        return (None, None, None, None, dfe, dword, dpos, dtyp, dtyp_vis, dpos_vis, dpw, dpb, dgamma, dbeta, dex)


def bert_embeddings(meta, input_ids, token_type_ids, visual_type, feats, word, pos, typ, typ_vis, pos_vis, pw, pb, gamma, beta,
                    vis_extra=None):
    """vis_extra: optional [B, V, H] term added to the projected region rows before the LayerNorm (differentiable)."""
    return _EmbedFn.apply(meta, input_ids, token_type_ids, visual_type, feats, word, pos, typ, typ_vis, pos_vis, pw, pb,
                          gamma, beta, vis_extra)


# --------------------------------------------------------------------------------------------
# masked-LM head on the library's kernels (SURVEY.md §8f rank 1): decoder GEMMs on wgmma, fused cross-entropy
# --------------------------------------------------------------------------------------------
def _gemm(dev, **kw):
    a = _lib.GemmArgs()
    for k, v in kw.items():
        setattr(a, k, v)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().vb_gemm(ctypes.byref(a), _stream()), "vb_gemm")


class _MlmDecoderFn(torch.autograd.Function):
    """logits[n, Vp] = t[n, H] @ E[V, H]^T + bias (BertLMPredictionHead decoder, reference M.py:403-421) — forward,
    input-gradient and weight-gradient GEMMs all on gemm_wgmma_kernel; the weight gradient accumulates straight
    into the (tied) word-embedding gradient when that buffer exists."""

    @staticmethod
    def forward(ctx, t, E, bias, cache, train=False):
        _require_cuda(t, "mlm_decoder")
        n, H = t.shape
        V = E.shape[0]
        table, bias_p = cache.get(E, bias, train=train)
        Vp = table.shape[0]
        t = t.to(_BF16).contiguous()
        with _unfilled():
            logits = torch.empty(n, Vp, device=t.device, dtype=_BF16)
        _gemm(t.device, A=t.data_ptr(), lda=H, B=table.data_ptr(), ldb=H, M=n, N=Vp, K=H, D=logits.data_ptr(), ldd=Vp,
              bias=bias_p.data_ptr())
        ctx.save_for_backward(t, table)
        ctx.E, ctx.bias, ctx.V = E, bias, V
        return logits

    @staticmethod
    def backward(ctx, dlogits):
        t, table = ctx.saved_tensors
        E, bias, V = ctx.E, ctx.bias, ctx.V
        n, H = t.shape
        Vp = dlogits.shape[1]
        dlogits = dlogits.contiguous()
        with _unfilled():
            dt = torch.empty(n, H, device=t.device, dtype=_BF16)
        _gemm(t.device, A=dlogits.data_ptr(), lda=Vp, B=table.data_ptr(), ldb=H, b_mn_major=1, M=n, N=H, K=Vp, D=dt.data_ptr(), ldd=H)
        direct = _grad_targets((E, bias))
        if direct is not None:
            dE, db = direct
            db_pad = torch.zeros(Vp, device=t.device, dtype=torch.float32)
        else:
            dE = torch.zeros(V, H, device=t.device, dtype=torch.float32)
            db_pad = torch.zeros(Vp, device=t.device, dtype=torch.float32)
        with deterministic(t.device, n, H, 0, V):
            _gemm(t.device, A=dlogits.data_ptr(), lda=Vp, a_mn_major=1, B=t.data_ptr(), ldb=H, b_mn_major=1, M=V, N=H, K=n,
                  D=dE.data_ptr(), ldd=H, d_fp32=1, splits=1)
            with torch.cuda.device(t.device):
                _lib.check(_lib.lib().vb_colsum_bf16(ctypes.c_void_p(dlogits.data_ptr()), ctypes.c_int64(Vp),
                                                     ctypes.c_void_p(db_pad.data_ptr()), n, Vp, _stream()), "vb_colsum_bf16")
        if direct is not None:
            db.add_(db_pad[:V])
            return dt, None, None, None, None
        return dt, dE, db_pad[:V].clone(), None, None


def mlm_decoder(t, E, bias, cache, train=False):
    return _MlmDecoderFn.apply(t, E, bias, cache, train)


class _CrossEntropyFn(torch.autograd.Function):
    """mean over rows of (logsumexp(logits[:, :V]) - logits[row, label]); the backward overwrites the logits with
    their gradient in place (vb_cross_entropy_bwd)."""

    @staticmethod
    def forward(ctx, logits, labels, V):
        n, Vp = logits.shape
        labels = labels.to(torch.int64).contiguous()
        lse = torch.empty(n, device=logits.device, dtype=torch.float32)
        rows = torch.empty(n, device=logits.device, dtype=torch.float32)
        with torch.cuda.device(logits.device):
            _lib.check(_lib.lib().vb_cross_entropy_fwd(ctypes.c_void_p(logits.data_ptr()), ctypes.c_int64(Vp),
                                                       ctypes.c_void_p(labels.data_ptr()), n, V, ctypes.c_void_p(lse.data_ptr()),
                                                       ctypes.c_void_p(rows.data_ptr()), _stream()), "vb_cross_entropy_fwd")
        ctx.logits, ctx.labels, ctx.lse, ctx.V = logits, labels, lse, V
        return rows.mean()

    @staticmethod
    def backward(ctx, g):
        logits, labels, lse, V = ctx.logits, ctx.labels, ctx.lse, ctx.V
        n, Vp = logits.shape
        scale = (g.float() / n).reshape(1).contiguous()
        with torch.cuda.device(logits.device):
            _lib.check(_lib.lib().vb_cross_entropy_bwd(ctypes.c_void_p(logits.data_ptr()), ctypes.c_int64(Vp),
                                                       ctypes.c_void_p(labels.data_ptr()), n, V, Vp, ctypes.c_void_p(lse.data_ptr()),
                                                       ctypes.c_void_p(scale.data_ptr()), _stream()), "vb_cross_entropy_bwd")
        ctx.logits = None
        return logits, None, None


def cross_entropy_rows(logits, labels, V):
    return _CrossEntropyFn.apply(logits, labels, V)
