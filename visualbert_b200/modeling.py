"""VisualBERT model classes with the reference's public interface, running on libvbert_b200.

Drop-in boundary (SURVEY.md §8b): `TrainVisualBERTObjective` / `BertVisualModel` keep the constructor,
`from_pretrained`, forward signature, output dict and `state_dict` keys of
uclanlp/visualbert `visualbert/pytorch_pretrained_bert/modeling.py` (cited as M.py:line below), so the
repo's AllenNLP wrappers (`visualbert/models/model.py:213-288`) can import these classes instead.
What differs is underneath: embeddings + the BertLayer stack execute as hand-written sm_90a kernels
(bf16 activations, fp32 master weights and gradients); task heads, pooler and losses stay PyTorch.

Modules here are parameter containers with the reference's names; `forward` hands the parameters to
the fused ops in `visualbert_b200.ops`. There is no eager/CPU implementation of the encoder.
"""
import copy
import json
import logging
import math
import os
import tarfile
import tempfile

import torch
import torch.nn.functional as F
from torch import nn

from . import ops

logger = logging.getLogger(__name__)

CONFIG_NAME = "bert_config.json"
WEIGHTS_NAME = "pytorch_model.bin"


def gelu(x):
    """erf-form GELU (M.py:56-61: x * 0.5 * (1 + erf(x / sqrt(2)))); used only by the PyTorch task heads. F.gelu's default
    (approximate='none') is the same function as ONE kernel forward and one backward instead of four and seven."""
    return F.gelu(x)


ACT2FN = {"gelu": gelu, "relu": F.relu, "swish": lambda x: x * torch.sigmoid(x)}


class BertConfig(object):
    """Same fields / constructors / serialisation as the reference BertConfig (M.py:71-156)."""

    _FIELDS = dict(hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072,
                   hidden_act="gelu", hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1,
                   max_position_embeddings=512, type_vocab_size=2, initializer_range=0.02)

    def __init__(self, vocab_size_or_config_json_file, **kwargs):
        if isinstance(vocab_size_or_config_json_file, str):
            with open(vocab_size_or_config_json_file, "r", encoding="utf-8") as fh:
                self.__dict__.update(json.load(fh))
        elif isinstance(vocab_size_or_config_json_file, int):
            unknown = set(kwargs) - set(self._FIELDS)
            if unknown:
                raise TypeError(f"unexpected BertConfig arguments: {sorted(unknown)}")
            self.vocab_size = vocab_size_or_config_json_file
            for name, default in self._FIELDS.items():
                setattr(self, name, kwargs.get(name, default))
        else:
            raise ValueError("First argument must be either a vocabulary size (int)"
                             "or the path to a pretrained model config file (str)")

    @classmethod
    def from_dict(cls, json_object):
        cfg = cls(vocab_size_or_config_json_file=-1)
        cfg.__dict__.update(json_object)
        return cfg

    @classmethod
    def from_json_file(cls, json_file):
        with open(json_file, "r", encoding="utf-8") as fh:
            return cls.from_dict(json.load(fh))

    def to_dict(self):
        return copy.deepcopy(self.__dict__)

    def to_json_string(self):
        return json.dumps(self.to_dict(), indent=2, sort_keys=True) + "\n"

    def __repr__(self):
        return str(self.to_json_string())


class BertLayerNorm(nn.Module):
    """Parameter holder + PyTorch forward for the heads (TF-style LN, M.py:162-175). Inside the encoder the
    LayerNorms run in vb_layernorm kernels and only `.weight` / `.bias` of this module are used."""

    def __init__(self, hidden_size, eps=1e-12):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden_size))
        self.bias = nn.Parameter(torch.zeros(hidden_size))
        self.variance_epsilon = eps

    def forward(self, x):
        # biased variance, eps inside the square root, fp32 statistics (M.py:170-174) == F.layer_norm; one kernel each way
        # instead of the nine / fifteen elementwise launches of the literal formula
        return F.layer_norm(x.float(), (x.shape[-1],), self.weight, self.bias, self.variance_epsilon).to(x.dtype)


# ----------------------------------------------------------------------------------------------
# encoder (CUDA path)
# ----------------------------------------------------------------------------------------------
class BertSelfAttention(nn.Module):
    def __init__(self, config):
        super().__init__()
        if config.hidden_size % config.num_attention_heads != 0:
            raise ValueError("The hidden size (%d) is not a multiple of the number of attention heads (%d)"
                             % (config.hidden_size, config.num_attention_heads))
        if config.hidden_size // config.num_attention_heads != 64:
            raise ValueError("visualbert_b200 attention kernels require head size 64 (BERT-base / -large), got %d"
                             % (config.hidden_size // config.num_attention_heads))
        self.num_attention_heads = config.num_attention_heads
        self.query = nn.Linear(config.hidden_size, config.hidden_size)
        self.key = nn.Linear(config.hidden_size, config.hidden_size)
        self.value = nn.Linear(config.hidden_size, config.hidden_size)


class BertSelfOutput(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.dense = nn.Linear(config.hidden_size, config.hidden_size)
        self.LayerNorm = BertLayerNorm(config.hidden_size, eps=1e-12)


class BertAttention(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.self = BertSelfAttention(config)
        self.output = BertSelfOutput(config)


class BertIntermediate(nn.Module):
    def __init__(self, config):
        super().__init__()
        act = config.hidden_act if isinstance(config.hidden_act, str) else getattr(config.hidden_act, "__name__", "?")
        if act != "gelu":
            raise ValueError("visualbert_b200 fuses the erf-GELU of the reference into the FFN kernel; "
                             "hidden_act=%r is not supported" % (config.hidden_act,))
        self.dense = nn.Linear(config.hidden_size, config.intermediate_size)


class BertOutput(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.dense = nn.Linear(config.intermediate_size, config.hidden_size)
        self.LayerNorm = BertLayerNorm(config.hidden_size, eps=1e-12)


def _encoder_meta(owner, layers, seed, **more):
    """meta of one ops.bert_encoder / ops.bert_layer call over `layers`, for the module that makes the call. Each such
    module keeps its own ops.EncoderPlan: a plan shared between callers would be rebuilt at every call."""
    l0, train = layers[0], owner.training
    # full checkpointing keeps no FFN intermediate either, so it governs when both switches are on
    ckpt = bool(owner.__dict__.get("activation_checkpointing", False))
    plan = owner.__dict__.get("_plan")
    if plan is None:
        plan = owner.__dict__["_plan"] = ops.EncoderPlan()
    return dict(heads=l0.attention.self.num_attention_heads, layer_index0=l0.layer_index,
                hidden_dropout=l0.hidden_dropout_prob if train else 0.0,
                attn_dropout=l0.attention_probs_dropout_prob if train else 0.0, seed=int(seed), train=train,
                caches=[l._weights for l in layers], plan=plan, seed_offset=ops.current_seed_offset() if train else None,
                checkpoint=ckpt, ffn_recompute=bool(owner.__dict__.get("ffn_recompute", False)) and not ckpt, **more)


class BertLayer(nn.Module):
    """One transformer block (M.py:322-341) = a one-layer vb_encoder_fwd / vb_encoder_bwd call."""

    def __init__(self, config, layer_index=0):
        super().__init__()
        self.attention = BertAttention(config)
        self.intermediate = BertIntermediate(config)
        self.output = BertOutput(config)
        self.layer_index = layer_index
        self.hidden_dropout_prob = config.hidden_dropout_prob
        self.attention_probs_dropout_prob = config.attention_probs_dropout_prob
        self._weights = ops.LayerWeights()

    def _params(self):
        a, o = self.attention, self.output
        return (a.self.query.weight, a.self.query.bias, a.self.key.weight, a.self.key.bias,
                a.self.value.weight, a.self.value.bias, a.output.dense.weight, a.output.dense.bias,
                a.output.LayerNorm.weight, a.output.LayerNorm.bias, self.intermediate.dense.weight,
                self.intermediate.dense.bias, o.dense.weight, o.dense.bias, o.LayerNorm.weight, o.LayerNorm.bias)

    def _masters(self):
        """The fp32 parameters that have a compute copy, in the order of ops.LayerWeights.items."""
        a = self.attention
        return [a.self.query.weight, a.self.key.weight, a.self.value.weight, a.output.dense.weight, self.intermediate.dense.weight,
                self.output.dense.weight, a.self.query.bias, a.self.key.bias, a.self.value.bias]

    def _vb_adjacent_param_groups(self):
        a = self.attention.self
        return ((a.query.weight, a.key.weight, a.value.weight), (a.query.bias, a.key.bias, a.value.bias))

    def forward(self, hidden_states, attention_mask, seed=0, output_attention_probs=False):
        """hidden_states [B, S, H]; attention_mask: the fp32 additive key bias [B, S]
        ((1 - mask) * -10000), or the reference's extended mask [B, 1, 1, S]. With output_attention_probs returns
        (output, maps): maps = softmax(QK^T/sqrt(d) + mask) [B, A, S, S] in fp32 (M.py:241-247, 258-259), pre-dropout and
        detached, computed by vb_encoder_attention_probs from the same bf16 Q and K the layer's attention used."""
        if attention_mask.dim() == 4:
            attention_mask = attention_mask[:, 0, 0, :]
        meta = _encoder_meta(self, [self], seed, attn_maps=bool(output_attention_probs))
        return ops.bert_layer(hidden_states.to(torch.bfloat16), attention_mask.float().contiguous(), meta, self._params())


class BertEncoder(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.layer = nn.ModuleList([BertLayer(config, i) for i in range(config.num_hidden_layers)])
        self.output_attention_weights = getattr(config, "output_attention_weights", False)
        self.activation_checkpointing = False   # BertVisualModel.set_activation_checkpointing
        self.ffn_recompute = False              # BertVisualModel.set_ffn_recompute

    def forward(self, hidden_states, attention_mask, output_all_encoded_layers=True, seed=0, varlen=None,
                output_attention_weights=None):
        """varlen (ops.unpad_plan): unpadded call — hidden_states are the [total, H] packed valid rows, attention_mask is
        ignored, and every returned layer is [total, H]. It always runs the whole-encoder call (there is no per-layer
        varlen path), so it cannot serve attention weights or gradients through intermediate layers.

        output_attention_weights (default: the config's) returns (layers, maps), maps = one detached fp32 [B, A, S, S]
        pre-dropout attention map per layer, written by the attention-probability kernel from each layer's own qkv."""
        want_maps = self.output_attention_weights if output_attention_weights is None else output_attention_weights
        if varlen is not None:
            if want_maps or (output_all_encoded_layers and torch.is_grad_enabled() and self.training):
                raise ValueError("unpadded encoder: attention weights and gradients through intermediate layers need the "
                                 "padded per-layer path")
            if len(self.layer) == 0:
                return [hidden_states]
            meta = _encoder_meta(self, self.layer, seed, varlen=varlen, all_layers=bool(output_all_encoded_layers))
            return list(ops.bert_encoder(hidden_states.to(torch.bfloat16), None, meta, self._fused_params()))
        if attention_mask.dim() == 4:
            attention_mask = attention_mask[:, 0, 0, :]
        fused = (hidden_states.is_cuda and len(self.layer) > 0
                 and not (output_all_encoded_layers and torch.is_grad_enabled() and self.training))
        if fused:
            # one C call for the whole stack: vb_encoder_fwd / vb_encoder_bwd over one activation arena (with maps, one
            # vb_encoder_attention_probs call over the same arena), or vb_encoder_infer when no graph can be recorded
            meta = _encoder_meta(self, self.layer, seed, attn_maps=want_maps, all_layers=bool(output_all_encoded_layers))
            ys = ops.bert_encoder(hidden_states.to(torch.bfloat16), attention_mask.float().contiguous(), meta, self._fused_params())
            n = len(self.layer) if output_all_encoded_layers else 1
            return (list(ys[:n]), list(ys[n:])) if want_maps else list(ys)
        outs, attn = [], []
        for layer in self.layer:
            if want_maps:
                hidden_states, maps = layer(hidden_states, attention_mask, seed, output_attention_probs=True)
                attn.append(maps)
            else:
                hidden_states = layer(hidden_states, attention_mask, seed)
            if output_all_encoded_layers:
                outs.append(hidden_states)
        if not output_all_encoded_layers:
            outs.append(hidden_states)
        return (outs, attn) if want_maps else outs

    def _fused_params(self):
        return [p for l in self.layer for p in l._params()]


class BertPooler(nn.Module):
    """tanh(W h[CLS] + b) (M.py:374-386); tiny, stays PyTorch and fp32 (returns fp32 like the reference)."""

    def __init__(self, config):
        super().__init__()
        self.dense = nn.Linear(config.hidden_size, config.hidden_size)

    def forward(self, hidden_states):
        first = hidden_states[:, 0].float()  # [B, H]: negligible work, keep the reference's fp32 arithmetic
        return torch.tanh(F.linear(first, self.dense.weight.float(), self.dense.bias.float()))


class BertEmbeddingsWithVisualEmbedding(nn.Module):
    """Word/position/segment embeddings + projected region features (M.py:1169-1257) = vb_embed_fwd."""

    def __init__(self, config):
        super().__init__()
        H = config.hidden_size
        self.word_embeddings = nn.Embedding(config.vocab_size, H)
        self.position_embeddings = nn.Embedding(config.max_position_embeddings, H)
        self.token_type_embeddings = nn.Embedding(config.type_vocab_size, H)
        self.LayerNorm = BertLayerNorm(H, eps=1e-12)
        self.token_type_embeddings_visual = nn.Embedding(config.type_vocab_size, H)
        self.position_embeddings_visual = nn.Embedding(config.max_position_embeddings, H)
        self.projection = nn.Linear(config.visual_embedding_dim, H)
        self.hidden_dropout_prob = config.hidden_dropout_prob
        self._weights = ops.ProjectionWeights()

    def special_intialize(self, method_type=0):
        """Copy the text segment/position tables into the visual ones (M.py:1191-1196; name kept as in the reference)."""
        self.token_type_embeddings_visual.weight = nn.Parameter(self.token_type_embeddings.weight.data.clone(), requires_grad=True)
        self.position_embeddings_visual.weight = nn.Parameter(self.position_embeddings.weight.data.clone(), requires_grad=True)

    def forward(self, input_ids, token_type_ids=None, visual_embeddings=None, visual_embeddings_type=None,
                position_embeddings_visual=None, image_text_alignment=None, confidence=None, seed=0):
        vis_extra = None
        if image_text_alignment is not None and visual_embeddings is not None:
            # VCR branch (M.py:1223-1245): every region also gets the MEAN of the text position embeddings of the words
            # it is aligned to (-1 = padding; regions without any aligned word get 0). A gather over [B, V, A] indices —
            # done with torch ops (autograd reaches position_embeddings.weight) and handed to the CUDA path as an
            # additive term on the projected region rows.
            ali_mask = (image_text_alignment != -1)
            table = self.position_embeddings.weight
            gathered = table[(image_text_alignment * ali_mask.long())] * ali_mask.unsqueeze(-1).to(table.dtype)
            count = ali_mask.sum(2).clamp_(min=1).to(table.dtype)
            vis_extra = gathered.sum(2) / count.unsqueeze(-1)
            if vis_extra.size(1) != visual_embeddings.size(1):  # alignment padded longer than the regions (M.py:1241-1243)
                assert vis_extra.size(1) >= visual_embeddings.size(1)
                vis_extra = vis_extra[:, : visual_embeddings.size(1), :]
        if token_type_ids is None:
            token_type_ids = torch.zeros_like(input_ids)
        if visual_embeddings is not None and visual_embeddings_type is None:
            visual_embeddings_type = torch.zeros(visual_embeddings.shape[:-1], dtype=torch.long, device=input_ids.device)
        meta = dict(dropout=self.hidden_dropout_prob if self.training else 0.0, seed=int(seed), cache=self._weights,
                    train=self.training, seed_offset=ops.current_seed_offset() if self.training else None)
        return ops.bert_embeddings(
            meta, input_ids, token_type_ids, visual_embeddings_type, visual_embeddings,
            self.word_embeddings.weight, self.position_embeddings.weight, self.token_type_embeddings.weight,
            self.token_type_embeddings_visual.weight, self.position_embeddings_visual.weight,
            self.projection.weight, self.projection.bias, self.LayerNorm.weight, self.LayerNorm.bias, vis_extra)


# ----------------------------------------------------------------------------------------------
# heads (PyTorch; "task heads stay" — BASELINE.json north_star)
# ----------------------------------------------------------------------------------------------
def _lin(x, mod):
    return F.linear(x, mod.weight.to(x.dtype), None if mod.bias is None else mod.bias.to(x.dtype))


class BertPredictionHeadTransform(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.dense = nn.Linear(config.hidden_size, config.hidden_size)
        self.transform_act_fn = ACT2FN[config.hidden_act] if isinstance(config.hidden_act, str) else config.hidden_act
        self.LayerNorm = BertLayerNorm(config.hidden_size, eps=1e-12)

    def forward(self, hidden_states):
        return self.LayerNorm(self.transform_act_fn(_lin(hidden_states, self.dense).float()).to(hidden_states.dtype))


class BertLMPredictionHead(nn.Module):
    """Transform + decoder tied to the word-embedding matrix + output-only bias (M.py:403-421)."""

    def __init__(self, config, bert_model_embedding_weights):
        super().__init__()
        self.transform = BertPredictionHeadTransform(config)
        self.decoder = nn.Linear(bert_model_embedding_weights.size(1), bert_model_embedding_weights.size(0), bias=False)
        self.decoder.weight = bert_model_embedding_weights
        self.bias = nn.Parameter(torch.zeros(bert_model_embedding_weights.size(0)))

    def forward(self, hidden_states):
        t = self.transform(hidden_states)
        return F.linear(t, self.decoder.weight.to(t.dtype), self.bias.to(t.dtype))


class BertPreTrainingHeads(nn.Module):
    def __init__(self, config, bert_model_embedding_weights):
        super().__init__()
        self.predictions = BertLMPredictionHead(config, bert_model_embedding_weights)
        self.seq_relationship = nn.Linear(config.hidden_size, 2)

    def forward(self, sequence_output, pooled_output):
        return self.predictions(sequence_output), _lin(pooled_output, self.seq_relationship)


class FlickrAttention(nn.Module):
    """Single-head scaled dot-product scores between selected text positions and regions (M.py:1602-1646)."""

    def __init__(self, config):
        super().__init__()
        if config.hidden_size % config.num_attention_heads != 0:
            raise ValueError("The hidden size (%d) is not a multiple of the number of attention heads (%d)"
                             % (config.hidden_size, config.num_attention_heads))
        self.num_attention_heads = 1
        self.attention_head_size = config.hidden_size // config.num_attention_heads
        self.all_head_size = self.attention_head_size
        self.query = nn.Linear(config.hidden_size, self.all_head_size)
        self.key = nn.Linear(config.hidden_size, self.all_head_size)
        self.value = nn.Linear(config.hidden_size, self.all_head_size)
        self.dropout = nn.Dropout(config.attention_probs_dropout_prob)

    def forward(self, query, key, attention_mask):
        bias = (1.0 - attention_mask.to(query.dtype))[:, None, :] * -10000.0
        q, k = _lin(query, self.query), _lin(key, self.key)
        return torch.matmul(q, k.transpose(-1, -2)) / math.sqrt(self.attention_head_size) + bias


# ----------------------------------------------------------------------------------------------
# model shells
# ----------------------------------------------------------------------------------------------
class PreTrainedBertModel(nn.Module):
    """Weight init + `from_pretrained` with the reference's behaviour (M.py:458-596), local paths only."""

    def __init__(self, config, *inputs, **kwargs):
        super().__init__()
        if not isinstance(config, BertConfig) and not hasattr(config, "hidden_size"):
            raise ValueError("Parameter config in `{}(config)` should be an instance of class `BertConfig`."
                             .format(self.__class__.__name__))
        self.config = config

    def init_bert_weights(self, module):
        if isinstance(module, (nn.Linear, nn.Embedding)):
            module.weight.data.normal_(mean=0.0, std=self.config.initializer_range)
        elif isinstance(module, BertLayerNorm):
            module.bias.data.zero_()
            module.weight.data.fill_(1.0)
        if isinstance(module, nn.Linear) and module.bias is not None:
            module.bias.data.zero_()

    @classmethod
    def from_pretrained(cls, pretrained_model_name, state_dict=None, cache_dir=None, random_initialize=False,
                        *inputs, **kwargs):
        """`pretrained_model_name` is a directory holding bert_config.json (+ pytorch_model.bin) or a .tar.gz of one.
        The reference also resolves model names to S3 URLs (M.py:510-531); this build has no network access, so
        names that are not local paths raise."""
        path = pretrained_model_name
        if not os.path.exists(path) and cache_dir is not None and os.path.exists(os.path.join(cache_dir, path)):
            path = os.path.join(cache_dir, path)
        if not os.path.exists(path):
            raise EnvironmentError(
                "Model name '{}' is not a local path; visualbert_b200 does not download archives. Point it at a "
                "directory with {} and {}.".format(pretrained_model_name, CONFIG_NAME, WEIGHTS_NAME))
        tempdir = None
        if not os.path.isdir(path):
            tempdir = tempfile.mkdtemp()
            with tarfile.open(path, "r:gz") as archive:
                try:
                    archive.extractall(tempdir, filter="data")  # refuse absolute paths / links escaping the directory
                except TypeError:  # Python < 3.12
                    archive.extractall(tempdir)
            path = tempdir
        try:
            config = BertConfig.from_json_file(os.path.join(path, CONFIG_NAME))
            logger.info("Model config {}".format(config))
            model = cls(config, *inputs, **kwargs)
            if random_initialize:
                return model
            if state_dict is None:
                state_dict = torch.load(os.path.join(path, WEIGHTS_NAME), map_location="cpu")
        finally:
            if tempdir is not None:
                import shutil
                shutil.rmtree(tempdir, ignore_errors=True)
        # TF-era names (M.py:556-568)
        renamed = {}
        for k, v in state_dict.items():
            nk = k[:-5] + "weight" if k.endswith("gamma") else (k[:-4] + "bias" if k.endswith("beta") else k)
            renamed[nk] = v
        # prefix rule of the reference (M.py:585): a bare encoder (no `.bert` attribute) reads its weights from the
        # "bert."-prefixed entries of the checkpoint; a wrapper model takes the keys as they are (and, more lenient than
        # the reference, a checkpoint of the bare encoder is accepted for the wrapper's `.bert`)
        has_prefix = any(k.startswith("bert.") for k in renamed)
        if not hasattr(model, "bert"):
            target = model
            if has_prefix:
                renamed = {k[5:]: v for k, v in renamed.items() if k.startswith("bert.")}
        else:
            target = model if has_prefix else model.bert
        result = target.load_state_dict(renamed, strict=False)
        missing = [k for k in result.missing_keys if k != "cls.predictions.decoder.weight"]
        if missing:
            logger.info("Weights of {} not initialized from pretrained model: {}".format(model.__class__.__name__, missing))
        if result.unexpected_keys:
            logger.info("Weights from pretrained model not used in {}: {}".format(model.__class__.__name__, result.unexpected_keys))
        return model


class BertVisualModel(PreTrainedBertModel):
    """Embeddings -> encoder -> pooler (M.py:1260-1333)."""

    def __init__(self, config):
        super().__init__(config)
        self.embeddings = BertEmbeddingsWithVisualEmbedding(config)
        self.encoder = BertEncoder(config)
        self.pooler = BertPooler(config)
        self.bypass_transformer = getattr(config, "bypass_transformer", False)
        if self.bypass_transformer:  # M.py:1268-1269; its own dropout streams (layer index after the encoder's)
            self.additional_layer = BertLayer(config, config.num_hidden_layers)
        self.output_attention_weights = getattr(config, "output_attention_weights", False)
        self.apply(self.init_bert_weights)
        self._unpadded = False
        self._step = 0
        self._capturable = False
        self._seed_offset = None   # capturable mode: the step snapshot of the latest training forward (int64 [1])
        # base of the counter-hash dropout streams: follows torch.manual_seed (so runs are reproducible the torch way);
        # the data-parallel rank is mixed in per forward (next_seed) so replicas draw different masks
        self.dropout_seed = (0x5EED ^ torch.initial_seed()) & 0xFFFFFFFF

    def _bank_holders(self):
        """(ops weight holder, its fp32 masters) of everything the model's bank serves."""
        layers = list(self.encoder.layer) + ([self.additional_layer] if self.bypass_transformer else [])
        holders = [(l._weights, l._masters()) for l in layers]
        holders.append((self.embeddings._weights, [self.embeddings.projection.weight]))
        extra = self.__dict__.get("_bank_extra")
        if extra is not None:
            holders.append(extra)
        return holders

    def refresh_compute_weights(self):
        """bf16 compute copies of all matrices of the encoder path <- fp32 masters, ONE launch (ops.WeightBank). Always
        in training mode (any optimizer, including the reference BertAdam's `p.data` updates, is picked up), on a
        version change in eval mode. Called by forward(); public so callers that edit weights mid-eval can force it."""
        holders = self._bank_holders()
        srcs = [p for _, masters in holders for p in masters]
        if not srcs[0].is_cuda:
            return
        bank = self.__dict__.get("_bank")
        if bank is None or not bank.bound_to(srcs):
            bank = self.__dict__["_bank"] = ops.WeightBank()
            items = []
            for holder, masters in holders:
                items += holder.items(*masters)
                holder.owner = bank
            bank.bind(items)
        bank.refresh(force=self.training or self._capturable)

    def set_graph_capturable(self, flag=True):
        """Opt-in CUDA-graph-capturable mode, off by default.

        When on, the dropout step counter is an int64 tensor on the model's device (a non-persistent buffer: it moves with
        .to() and stays out of state_dict). Each training forward increments it and snapshots it into a tensor of its own; the
        descriptors carry the base seed K = (dropout_seed + c * rank) * golden and the kernels add the snapshot, read from device
        memory when they run (vb_set_dropout_offset). Every forward therefore draws exactly the seed next_seed() gives in the
        default mode, a backward uses its own forward's snapshot (gradient accumulation stays correct), and a captured graph
        draws fresh masks at every replay. The compute-weight cast is enqueued on every forward, eval mode included, so
        replays see parameter changes made between them. dropout_state() reads the counter back (one host synchronisation);
        set_dropout_state() writes it in place (a captured graph sees the new value). States carry over between the modes.
        Not available with the unpadded path (set_unpadded), which synchronises with the host."""
        flag = bool(flag)
        if flag and self._unpadded:
            raise ValueError("set_graph_capturable: not supported with set_unpadded (its row plan synchronises with the host)")
        if flag and not self._capturable:
            dev = next(self.parameters()).device
            self.register_buffer("_vb_step", torch.tensor([self._step], dtype=torch.int64, device=dev), persistent=False)
        elif not flag and self._capturable:
            self._step = int(self._vb_step.item())
            del self._vb_step
            self._seed_offset = None
        self._capturable = flag
        return self

    def set_activation_checkpointing(self, flag=True):
        """Opt-in activation checkpointing of the encoder, off by default.

        When on, a training forward of the whole-encoder call keeps ONE layer's activations (an arena slot) plus each lower
        layer's output and LayerNorm-2 statistics, instead of every layer's activations; the backward call recomputes each lower
        layer into the slot before running its backward (vb_encoder_fwd_ckpt / vb_encoder_bwd_ckpt). The recompute draws the
        same dropout masks, so the loss, the outputs and, in deterministic mode, every gradient are bit for bit those of the
        default path; a step costs about one more forward of the lower layers. Read at every forward; works with set_unpadded,
        set_graph_capturable (GraphedStep captures a new graph when the flag changes), deterministic mode, frozen parameters,
        output_attention_weights and bypass_transformer (its text encoder call). The padded per-layer route
        (output_all_encoded_layers=True in training mode under grad) keeps one single-layer arena per layer, as without the
        flag."""
        self.encoder.activation_checkpointing = bool(flag)
        return self

    def set_ffn_recompute(self, flag=True):
        """Opt-in selective recomputation of the encoder's FFN intermediates, off by default.

        When on, a training forward of the whole-encoder call keeps every layer's activations except gelu(u) and gelu'(u) of its
        FFN (2 * rows * intermediate_size bf16, half of a layer's activation memory): one buffer shared by all layers holds them
        for the layer being run, and the backward call rebuilds them for each layer below the top one with the FFN-up GEMM of
        its forward (vb_encoder_fwd_ffnrc / vb_encoder_bwd_ffnrc). That GEMM has the forward's weights, epilogue and tiling, so
        the loss, the outputs and, in deterministic mode, every gradient are bit for bit those of the default path; a step costs
        L - 1 more GEMMs. Read at every forward; works with set_unpadded, set_graph_capturable (GraphedStep captures a new graph
        when the flag changes), deterministic mode, frozen parameters, output_attention_weights and bypass_transformer (its
        text encoder call). With set_activation_checkpointing also on, full checkpointing governs. The padded per-layer route
        (output_all_encoded_layers=True in training mode under grad) and forward-only calls are not changed."""
        self.encoder.ffn_recompute = bool(flag)
        return self

    def set_unpadded(self, flag=True):
        """Opt-in unpadded ("variable-length") encoder execution, off by default.

        When on, forward packs the valid positions (attention_mask != 0 over cat(text mask, image mask); any pattern, the
        rows of an example keep their order) into [total, H] rows, runs the encoder on those rows only through the
        variable-length kernels (vb_encoder_fwd_varlen: no GEMM, LayerNorm or attention work on padding), and scatters every
        returned layer back to [B, S, H]. Semantics:
          - valid positions equal those of the padded path to within rounding: the padded path's key bias of -10000 gives
            those keys exactly zero probability in fp32 softmax, so the valid rows see the same keys either way;
          - masked positions are ZERO, where the padded path returns finite values (queries over the valid keys). This shows
            in output_all_encoded_layers outputs, in the lazily built pretraining `logits` at masked positions, in the pooled
            output of an example whose first position is masked, and for an example without any valid position, whose rows
            are all zero.
        One host synchronisation per forward (the longest sequence and the row count). Not available with
        bypass_transformer or output_attention_weights, nor, in training mode under grad, with output_all_encoded_layers=True
        (gradients through intermediate layers): those raise instead of running padded."""
        flag = bool(flag)
        if flag and self._capturable:
            raise ValueError("set_unpadded: not supported in graph-capturable mode (set_graph_capturable)")
        if flag and self.bypass_transformer:
            raise ValueError("set_unpadded: not supported with bypass_transformer")
        if flag and self.output_attention_weights:
            raise ValueError("set_unpadded: not supported with output_attention_weights")
        self._unpadded = flag
        return self

    def _encode_unpadded(self, x, attention_mask, output_all_encoded_layers, seed):
        if output_all_encoded_layers and torch.is_grad_enabled() and self.training:
            raise ValueError("unpadded forward: output_all_encoded_layers=True in training mode under grad needs gradients "
                             "through intermediate layers, which only the padded per-layer path provides")
        B, S, H = x.shape
        vl = ops.unpad_plan(attention_mask != 0)
        if vl["total"] == 0:   # no valid position anywhere: every row is zero
            z = x.to(torch.bfloat16) * 0
            return [z] * (len(self.encoder.layer) if output_all_encoded_layers else 1)
        idx = vl["index"]
        packed = x.reshape(B * S, H).index_select(0, idx)
        ys = self.encoder(packed, None, output_all_encoded_layers=output_all_encoded_layers, seed=seed, varlen=vl)
        zero = torch.zeros(B * S, H, device=x.device, dtype=torch.bfloat16)
        return [zero.index_copy(0, idx, y.to(torch.bfloat16)).view(B, S, H) for y in ys]

    def next_seed(self):
        """Per-forward dropout seed: forward and backward of one step share it; steps differ. In graph-capturable mode the
        step lives on the device: this returns the base K, and the seed the kernels use is K + the snapshot left in
        self._seed_offset (what the default mode returns, mod 2^64)."""
        rank = 0
        if torch.distributed.is_available() and torch.distributed.is_initialized():
            rank = torch.distributed.get_rank()
        base = ((self.dropout_seed + 0x632BE59B * rank) * 0x9E3779B97F4A7C15) & 0xFFFFFFFFFFFFFFFF
        if self._capturable:
            self._vb_step.add_(1)
            self._seed_offset = self._vb_step.clone()
            return base
        self._step += 1
        return (base + self._step) & 0xFFFFFFFFFFFFFFFF

    def dropout_state(self):
        """(base seed, forwards so far): save next to a checkpoint and hand back to set_dropout_state() to resume the
        exact dropout sequence (kept out of state_dict so reference checkpoints still load with strict=True). In
        graph-capturable mode this reads the device counter: one host synchronisation."""
        step = int(self._vb_step.item()) if self._capturable else int(self._step)
        return {"seed": int(self.dropout_seed), "step": step}

    def set_dropout_state(self, state):
        self.dropout_seed = int(state["seed"])
        self._step = int(state["step"])
        if self._capturable:
            self._vb_step.fill_(self._step)

    def forward(self, input_ids, token_type_ids, attention_mask, visual_embeddings, position_embeddings_visual,
                visual_embeddings_type, image_text_alignment, confidence, output_all_encoded_layers=True):
        if attention_mask is None:
            T = input_ids.size(1)
            V = 0 if visual_embeddings is None else visual_embeddings.size(1)
            attention_mask = torch.ones(input_ids.size(0), T + V, dtype=torch.long, device=input_ids.device)
        if token_type_ids is None:
            token_type_ids = torch.zeros_like(input_ids)
        capturing = input_ids.is_cuda and torch.cuda.is_current_stream_capturing()
        if capturing and not self._capturable:
            raise ValueError("CUDA graph capture of a forward needs graph-capturable mode: call set_graph_capturable() first "
                             "(otherwise every replay would reuse the captured step's dropout masks)")
        seed = self.next_seed() if self.training else 0
        with ops.forward_seed_offset(self._seed_offset if (self._capturable and self.training) else None):
            return self._forward(input_ids, token_type_ids, attention_mask, visual_embeddings, position_embeddings_visual,
                                 visual_embeddings_type, image_text_alignment, confidence, output_all_encoded_layers, seed)

    def _forward(self, input_ids, token_type_ids, attention_mask, visual_embeddings, position_embeddings_visual,
                 visual_embeddings_type, image_text_alignment, confidence, output_all_encoded_layers, seed):
        self.refresh_compute_weights()
        bias = None if self._unpadded else ops.mask_bias(attention_mask, None)
        x = self.embeddings(input_ids, token_type_ids, visual_embeddings=visual_embeddings,
                            visual_embeddings_type=visual_embeddings_type, position_embeddings_visual=position_embeddings_visual,
                            image_text_alignment=image_text_alignment, confidence=confidence, seed=seed)
        if self.bypass_transformer and visual_embeddings is not None:
            # M.py:1299-1314: the encoder runs over the text positions only (keys masked to the text part), the region
            # rows of the embedding output are appended afterwards and one more BertLayer sees the whole sequence
            assert not output_all_encoded_layers  # "Don't support this for the bypass model" (M.py:1300)
            T = input_ids.size(1)
            # the text encoder's attention maps are not part of the bypass model's outputs: they are not computed
            text = self.encoder(x[:, :T].contiguous(), bias[:, :T].contiguous(), output_all_encoded_layers=False, seed=seed,
                                output_attention_weights=False)[-1]
            final = self.additional_layer(torch.cat((text, x[:, T:]), dim=1), bias, seed)
            return final, self.pooler(final)
        if self._unpadded:
            if self.bypass_transformer or self.output_attention_weights:
                raise ValueError("unpadded forward: not supported with bypass_transformer or output_attention_weights")
            encoded_layers = self._encode_unpadded(x, attention_mask, output_all_encoded_layers, seed)
        elif self.output_attention_weights:
            encoded_layers, attn = self.encoder(x, bias, output_all_encoded_layers=output_all_encoded_layers, seed=seed)
        else:
            encoded_layers = self.encoder(x, bias, output_all_encoded_layers=output_all_encoded_layers, seed=seed)
        sequence_output = encoded_layers[-1]
        pooled_output = self.pooler(sequence_output)
        if not output_all_encoded_layers:
            encoded_layers = encoded_layers[-1]
        if self.output_attention_weights:
            return encoded_layers, pooled_output, attn
        return encoded_layers, pooled_output


class LazyOutputDict(dict):
    """Output dict whose expensive entries are computed on first access.

    The reference materialises MLM `logits` for all B*S positions ([B, S, vocab] — 5.1 GB in fp32 at the benchmark
    config) although the loss ignores every position whose label is -1 (all visual and ~85 % of text positions,
    M.py:1422, 1472) and its own training wrapper never reads `logits` in pretraining mode
    (visualbert/models/model.py:290-299). Here the loss is computed from the labelled rows only — the same value
    and gradients — and `logits` (full shape, reference semantics) is produced when somebody asks for it."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self._lazy = {}

    def set_lazy(self, key, thunk):
        self._lazy[key] = thunk
        super().__setitem__(key, None)

    def _resolve(self, key):
        if key in self._lazy:
            super().__setitem__(key, self._lazy.pop(key)())

    def __getitem__(self, key):
        self._resolve(key)
        return super().__getitem__(key)

    def get(self, key, default=None):
        if key in self:
            return self[key]
        return default

    def __setitem__(self, key, value):
        self._lazy.pop(key, None)
        super().__setitem__(key, value)

    def items(self):
        for k in list(self._lazy):
            self._resolve(k)
        return super().items()

    def values(self):
        for k in list(self._lazy):
            self._resolve(k)
        return super().values()


def transform_to_batch_sequence(tensor):
    if tensor is None or tensor.dim() == 2:
        return tensor
    assert tensor.dim() == 3
    return tensor.contiguous().view(-1, tensor.size(-1))


def transform_to_batch_sequence_dim(tensor):
    if tensor is None or tensor.dim() == 3:
        return tensor
    assert tensor.dim() == 4
    return tensor.contiguous().view(-1, tensor.size(-2), tensor.size(-1))


def masked_unk_softmax(x, dim, mask_idx):
    x1 = F.softmax(x, dim=dim)
    x1[:, mask_idx] = 0
    return x1 / torch.sum(x1, dim=1, keepdim=True)


def compute_score_with_logits(logits, labels):
    pred = torch.max(masked_unk_softmax(logits, 1, 0), 1)[1].data
    one_hots = torch.zeros_like(labels)
    one_hots.scatter_(1, pred.view(-1, 1), 1)
    return one_hots * labels


def compute_score_with_logits_flickr(logits, labels, recall=1):
    labels_mask = (labels != 0.0).float()
    upper_bound_labels = labels.sum(-1).view(-1).sum(-1)
    labels = torch.ones_like(labels) * labels_mask
    pred = torch.max(logits, -1)[1].data.unsqueeze(-1)
    scores = torch.gather(input=labels, dim=2, index=pred).view(-1).sum(-1)
    return scores, upper_bound_labels


def batched_index_select(t, dim, inds):
    dummy = inds.unsqueeze(2).expand(inds.size(0), inds.size(1), t.size(2))
    return t.gather(dim, dummy)


class TrainVisualBERTObjective(PreTrainedBertModel):
    """Reference objective/boundary class (M.py:1335-1598): same constructor, forward and output dict."""

    def __init__(self, config, training_head_type, visual_embedding_dim=512, hard_cap_seq_len=None, cut_first="text",
                 embedding_strategy="plain", bypass_transformer=False, output_attention_weights=False):
        super().__init__(config)
        config.visual_embedding_dim = visual_embedding_dim
        config.embedding_strategy = embedding_strategy
        config.bypass_transformer = bypass_transformer
        config.output_attention_weights = output_attention_weights
        self.output_attention_weights = output_attention_weights
        self.cut_first = cut_first
        self.hard_cap_seq_len = hard_cap_seq_len
        self.bert = BertVisualModel(config)
        self.training_head_type = training_head_type
        H = config.hidden_size
        if training_head_type in ("pretraining", "vqa_advanced"):
            self.cls = BertPreTrainingHeads(config, self.bert.embeddings.word_embeddings.weight)
        elif training_head_type == "multichoice":
            self.dropout = nn.Dropout(config.hidden_dropout_prob)
            self.classifier = nn.Linear(H, 1)
            self.num_choices = 4
        elif training_head_type == "vqa":
            self.dropout = nn.Dropout(config.hidden_dropout_prob)
            self.classifier = nn.Linear(H, 3129)
        elif training_head_type == "nlvr":
            self.dropout = nn.Dropout(config.hidden_dropout_prob)
            self.classifier = nn.Linear(H, 2)
        elif training_head_type == "flickr":
            self.dropout = nn.Dropout(config.hidden_dropout_prob)
            self.cls = BertPreTrainingHeads(config, self.bert.embeddings.word_embeddings.weight)
            self.flickr_attention = FlickrAttention(config)
        self.apply(self.init_bert_weights)

    @staticmethod
    def _labelled_rows(flat_labels, vocab=None):
        """Indices of the rows that carry an MLM target. `nonzero` synchronises with the device, so forward() calls this
        BEFORE the encoder is enqueued (the stream is empty then) instead of draining ~12 ms of queued work later.
        Labels outside [0, vocab) are treated like the reference's ignore index -1 (CrossEntropyLoss(ignore_index=-1))."""
        if flat_labels.is_cuda and torch.cuda.is_current_stream_capturing():
            raise ValueError("CUDA graph capture: finding the MLM target rows needs a host synchronisation (nonzero); pass "
                             "masked_lm_rows (parallel.BatchPrefetcher computes them on the host)")
        flat = flat_labels.contiguous().view(-1)
        keep = flat >= 0 if vocab is None else (flat >= 0) & (flat < vocab)
        return torch.nonzero(keep).squeeze(1)

    def _decoder_cache(self):
        """The tied decoder table rides the encoder's WeightBank (refreshed by the same launch, before the encoder runs)."""
        dw = self.__dict__.get("_decoder_weights")
        if dw is None:
            dw = ops.DecoderWeights()
            self.__dict__["_decoder_weights"] = dw
        return dw

    def _register_decoder_in_bank(self):
        if self.training_head_type != "pretraining" or not hasattr(self, "cls"):
            return
        head = self.cls.predictions
        self.bert.__dict__["_bank_extra"] = (self._decoder_cache(), [head.decoder.weight, head.bias])

    def _masked_lm_loss(self, sequence_output, flat_labels, rows=None):
        """CrossEntropyLoss(ignore_index=-1) of the MLM head (M.py:1471-1473) evaluated on the labelled rows only:
        ignored rows contribute neither to the sum nor to the count, so value and gradients are unchanged."""
        labels = flat_labels.contiguous().view(-1)
        if rows is None:
            rows = self._labelled_rows(flat_labels, self.cls.predictions.decoder.weight.size(0))
        head = self.cls.predictions
        if self.bert._capturable and sequence_output.is_cuda:
            # fixed-capacity rows (parallel.BatchPrefetcher(mlm_rows_capacity=N)): -1 entries are "no target". They read row 0
            # with label -1 (no loss, no gradient in the cross-entropy kernels); the loss is the sum over the valid rows divided by
            # their count, counted on the device, so neither the shapes nor the host depend on how many targets a batch has.
            valid = rows >= 0
            safe = rows.clamp(min=0)
            hidden = sequence_output.reshape(-1, sequence_output.size(-1)).index_select(0, safe)
            lab = torch.where(valid, labels.index_select(0, safe), torch.full_like(safe, -1))
            count = valid.sum(dtype=torch.float32).clamp(min=1.0).reshape(())
            scores = ops.mlm_decoder(head.transform(hidden), head.decoder.weight, head.bias, self._decoder_cache(), self.training)
            return ops.cross_entropy_rows(scores, lab, head.decoder.weight.size(0), count)
        hidden = sequence_output.reshape(-1, sequence_output.size(-1)).index_select(0, rows)
        if rows.numel() == 0 or not hidden.is_cuda:
            return F.cross_entropy(head(hidden).float(), labels.index_select(0, rows))
        # decoder + loss on the library's kernels: wgmma GEMMs (fwd / dgrad / wgrad into the tied word-embedding
        # gradient) and the fused cross-entropy; the small transform (dense + gelu + LayerNorm on ~12 % of the rows)
        # stays PyTorch
        scores = ops.mlm_decoder(head.transform(hidden), head.decoder.weight, head.bias, self._decoder_cache(), self.training)
        return ops.cross_entropy_rows(scores, labels.index_select(0, rows), head.decoder.weight.size(0))

    def forward(self, input_ids, token_type_ids, input_mask, visual_embeddings, position_embeddings_visual, image_mask,
                image_text_alignment=None, confidence=None, visual_embeddings_type=None, label=None,
                flickr_position=None, masked_lm_labels=None, image_lm_lables=None, is_random_next=None,
                output_all_encoded_layers=False, masked_lm_rows=None):
        """Reference signature (M.py:1373-1392) plus one optional extension: `masked_lm_rows`, the flat indices
        (b * (T + V) + t, int64, on the device) of the positions whose `masked_lm_labels` is not -1. When given (e.g. by
        `parallel.BatchPrefetcher`, which computes them on the host from the host copy of the labels) the forward pass
        contains no host synchronisation at all; when omitted they are found with one `nonzero` before the encoder."""
        if self.training_head_type == "vqa_advanced" and input_ids.is_cuda and torch.cuda.is_current_stream_capturing():
            raise ValueError("CUDA graph capture: the vqa_advanced head reads its accuracy with .item(); run it eagerly")
        if "_bank_extra" not in self.bert.__dict__:
            self._register_decoder_in_bank()
        flat_input_ids = transform_to_batch_sequence(input_ids)
        flat_token_type_ids = transform_to_batch_sequence(token_type_ids)
        flat_input_mask = transform_to_batch_sequence(input_mask)
        flat_image_mask = transform_to_batch_sequence(image_mask)
        flat_masked_lm_labels = transform_to_batch_sequence(masked_lm_labels)
        flat_position_embeddings_visual = transform_to_batch_sequence(position_embeddings_visual)
        flat_confidence = transform_to_batch_sequence(confidence)
        flat_image_text_alignment = transform_to_batch_sequence_dim(image_text_alignment)
        flat_visual_embeddings = transform_to_batch_sequence_dim(visual_embeddings)

        if visual_embeddings_type is not None:
            visual_embeddings_type = transform_to_batch_sequence(visual_embeddings_type)
        elif flat_image_mask is not None:
            visual_embeddings_type = torch.zeros_like(flat_image_mask, dtype=torch.long)

        if flat_image_mask is not None:
            flat_attention_mask = torch.cat((flat_input_mask, flat_image_mask), dim=-1)
            assert image_lm_lables is None  # not supported by the reference either (M.py:1419)
            if flat_masked_lm_labels is not None:
                assert flat_masked_lm_labels.size(-1) == flat_input_mask.size(-1)
                assert flat_masked_lm_labels.dim() == 2
                padded = torch.full_like(flat_attention_mask, -1)  # no MLM targets on visual positions
                padded[:, : flat_masked_lm_labels.size(1)] = flat_masked_lm_labels
                flat_masked_lm_labels = padded
        else:
            flat_attention_mask = flat_input_mask

        mlm_rows = masked_lm_rows
        if (mlm_rows is None and self.training_head_type == "pretraining" and flat_masked_lm_labels is not None
                and not output_all_encoded_layers):
            mlm_rows = self._labelled_rows(flat_masked_lm_labels, self.cls.predictions.decoder.weight.size(0))  # the only host sync of the step: do it up front
        if self.output_attention_weights:
            # analysis mode (M.py:1430-1444): nothing but the per-layer attention maps is returned
            attention_weights = self.bert(
                flat_input_ids, flat_token_type_ids, flat_attention_mask, visual_embeddings=flat_visual_embeddings,
                position_embeddings_visual=flat_position_embeddings_visual, visual_embeddings_type=visual_embeddings_type,
                image_text_alignment=flat_image_text_alignment, confidence=flat_confidence,
                output_all_encoded_layers=output_all_encoded_layers)[2]
            return {"attention_weights": attention_weights, "loss": None}
        sequence_output, pooled_output = self.bert(
            flat_input_ids, flat_token_type_ids, flat_attention_mask, visual_embeddings=flat_visual_embeddings,
            position_embeddings_visual=flat_position_embeddings_visual, visual_embeddings_type=visual_embeddings_type,
            image_text_alignment=flat_image_text_alignment, confidence=flat_confidence,
            output_all_encoded_layers=output_all_encoded_layers)

        output_dict = {}
        if output_all_encoded_layers:
            output_dict["sequence_output"] = sequence_output
            output_dict["pooled_output"] = pooled_output
            output_dict["loss"] = None
            return output_dict

        head = self.training_head_type
        if head == "pretraining":
            output_dict = LazyOutputDict()
            seq_relationship_score = _lin(pooled_output, self.cls.seq_relationship)
            output_dict.set_lazy("logits", lambda: self.cls.predictions(sequence_output))
            output_dict["seq_relationship_score"] = seq_relationship_score
            output_dict["loss"] = None
            if flat_masked_lm_labels is not None:
                masked_lm_loss = self._masked_lm_loss(sequence_output, flat_masked_lm_labels, mlm_rows)
                output_dict["masked_lm_loss"] = masked_lm_loss
                output_dict["loss"] = masked_lm_loss
                if is_random_next is not None:
                    next_sentence_loss = F.cross_entropy(seq_relationship_score.view(-1, 2).float(),
                                                         is_random_next.contiguous().view(-1), ignore_index=-1)
                    output_dict["next_sentence_loss"] = next_sentence_loss
                    output_dict["loss"] = masked_lm_loss + next_sentence_loss
            return output_dict

        if head == "multichoice":
            logits = _lin(self.dropout(pooled_output), self.classifier)
            reshaped_logits = logits.contiguous().view(-1, self.num_choices)
            output_dict["logits"] = reshaped_logits
            output_dict["loss"] = None
            if label is not None:
                output_dict["loss"] = F.cross_entropy(reshaped_logits.float(), label.contiguous())
            return output_dict

        if head == "vqa":
            index_to_gather = flat_input_mask.sum(1) - 2  # second-to-last valid text token (M.py:1504)
            gathered = torch.gather(sequence_output, 1, index_to_gather.view(-1, 1, 1).expand(-1, 1, sequence_output.size(-1))).float()
            logits = _lin(self.dropout(gathered), self.classifier)
            reshaped_logits = logits.contiguous().view(-1, 3129)
            output_dict["logits"] = logits
            output_dict["loss"] = None
            output_dict["accuracy"] = None
            if label is not None:
                log_probs = F.log_softmax(reshaped_logits.float(), dim=-1)
                output_dict["loss"] = F.kl_div(log_probs, label.contiguous(), reduction="batchmean")
                output_dict["accuracy"] = torch.sum(compute_score_with_logits(log_probs, label)) / label.size(0)
            return output_dict

        if head == "vqa_advanced":
            prediction_scores, seq_relationship_score = self.cls(sequence_output, pooled_output)
            output_dict["logits"] = prediction_scores
            output_dict["seq_relationship_score"] = seq_relationship_score
            masked_lm_loss = F.cross_entropy(prediction_scores.view(-1, self.config.vocab_size).float(),
                                             flat_masked_lm_labels.contiguous().view(-1), ignore_index=-1)
            output_dict["masked_lm_loss"] = masked_lm_loss
            output_dict["loss"] = masked_lm_loss
            pred = torch.max(prediction_scores, -1)[1].view(input_ids.size(0), -1)
            lab = flat_masked_lm_labels.view(input_ids.size(0), -1)
            all_right = ((lab == -1) | (pred == lab)).all(dim=1)  # same count as the reference's python loop (M.py:1538-1552)
            output_dict["accuracy"] = float(all_right.sum().item()) / pred.shape[0]
            return output_dict

        if head == "nlvr":
            logits = _lin(self.dropout(pooled_output), self.classifier)
            output_dict["logits"] = logits
            output_dict["loss"] = None
            if label is not None:
                output_dict["loss"] = F.cross_entropy(logits.contiguous().float(), label.contiguous())
            return output_dict

        if head == "flickr":
            if flickr_position is not None:
                entities_num = (flickr_position != -1).long().view(-1).sum(-1)
                flickr_position_mask = (flickr_position != -1).long()
                flickr_position = flickr_position * flickr_position_mask
                selected_positions = batched_index_select(sequence_output, 1, flickr_position)
                visual_features = sequence_output[:, flat_input_mask.size(1):, :]
                assert visual_features.size(1) == flat_image_mask.size(1)
                scores = self.flickr_attention(selected_positions, visual_features, flat_image_mask)
                scores = F.log_softmax(scores.float(), dim=-1)
                label = label.contiguous()
                output_dict["loss"] = F.kl_div(scores, label, reduction="batchmean")
                acc, upper_acc = compute_score_with_logits_flickr(scores, label)
                output_dict["accuracy"] = acc / entities_num
                output_dict["upperbound_accuracy"] = upper_acc / entities_num
                output_dict["entity_num"] = entities_num
            return output_dict
        raise ValueError("unknown training_head_type %r" % (head,))
