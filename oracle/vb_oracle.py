"""CPU oracle for the VisualBERT encoder hot path — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A plain functional restatement (torch tensor algebra, any float dtype, CPU or GPU) of the
reference algorithm in uclanlp/visualbert `visualbert/pytorch_pretrained_bert/modeling.py`
("M.py" below). Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / reference arm may
import this module, and only as the checker. The product path (visualbert_b200) never imports it.

Parity pinning: the reference repo holds NO tests, golden vectors or known-answer fixtures for this
path (SURVEY.md §4, §8c), so the oracle is pinned against outputs of the reference itself, generated
by oracle/make_golden.py (which imports the unmodified reference from a checkout named by
VB_REFERENCE) and committed under tests/golden/. tests/test_oracle_golden.py checks this module
against those fixtures on every CPU test run.

State is a dict name -> tensor using the reference's state_dict keys (SURVEY.md §8b), e.g.
`bert.encoder.layer.0.attention.self.query.weight`.
"""
import math

import torch
import torch.nn.functional as F


def gelu(x):
    """M.py:56-61 — exact erf form."""
    return x * 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0)))


def layer_norm(x, weight, bias, eps=1e-12):
    """M.py:171-175 — TF style: biased variance, eps inside the sqrt."""
    u = x.mean(-1, keepdim=True)
    s = (x - u).pow(2).mean(-1, keepdim=True)
    return weight * ((x - u) / torch.sqrt(s + eps)) + bias


def linear(x, sd, prefix):
    return F.linear(x, sd[prefix + ".weight"], sd[prefix + ".bias"])


def embeddings(sd, input_ids, token_type_ids, visual_embeddings, visual_embeddings_type,
               image_text_alignment=None, pfx="bert.embeddings."):
    """M.py:1198-1257 (dropout omitted: eval mode). Text first, then visual; every region uses
    visual position row 0 (M.py:1247); optional VCR alignment branch M.py:1223-1245."""
    T = input_ids.size(1)
    dt = sd[pfx + "word_embeddings.weight"].dtype
    pos = torch.arange(T, device=input_ids.device)
    e = (sd[pfx + "word_embeddings.weight"][input_ids]
         + sd[pfx + "position_embeddings.weight"][pos].unsqueeze(0)
         + sd[pfx + "token_type_embeddings.weight"][token_type_ids])
    if visual_embeddings is not None:
        v = F.linear(visual_embeddings.to(dt), sd[pfx + "projection.weight"], sd[pfx + "projection.bias"])
        tv = sd[pfx + "token_type_embeddings_visual.weight"][visual_embeddings_type]
        pv = sd[pfx + "position_embeddings_visual.weight"][0].view(1, 1, -1).expand_as(v)
        if image_text_alignment is not None:
            m = (image_text_alignment != -1).long()
            ali = m * image_text_alignment
            pa = sd[pfx + "position_embeddings.weight"][ali] * m.to(dt).unsqueeze(-1)
            pa = pa.sum(2)
            cnt = m.to(dt).sum(2)
            cnt[cnt == 0] = 1
            pa = pa / cnt.unsqueeze(-1)
            pa = pa[:, : v.size(1), :]
            pv = pa + pv
        e = torch.cat((e, v + pv + tv), dim=1)
    return layer_norm(e, sd[pfx + "LayerNorm.weight"], sd[pfx + "LayerNorm.bias"])


def self_attention(sd, pfx, x, ext_mask, num_heads, return_probs=False):
    """M.py:231-261: scale-then-mask, softmax, P·V, head merge."""
    B, S, H = x.shape
    d = H // num_heads

    def split(t):
        return t.view(B, S, num_heads, d).permute(0, 2, 1, 3)

    q = split(linear(x, sd, pfx + "query"))
    k = split(linear(x, sd, pfx + "key"))
    v = split(linear(x, sd, pfx + "value"))
    scores = torch.matmul(q, k.transpose(-1, -2)) / math.sqrt(d)
    scores = scores + ext_mask
    probs = torch.softmax(scores, dim=-1)
    ctx = torch.matmul(probs, v).permute(0, 2, 1, 3).contiguous().view(B, S, H)
    return (ctx, probs) if return_probs else ctx


def bert_layer(sd, pfx, x, ext_mask, num_heads, return_probs=False):
    """M.py:331-341 with 270-274, 302-305, 315-319; return_probs = the output_attention_weights branch (M.py:332-336)."""
    ctx = self_attention(sd, pfx + "attention.self.", x, ext_mask, num_heads, return_probs)
    if return_probs:
        ctx, probs = ctx
    a = layer_norm(linear(ctx, sd, pfx + "attention.output.dense") + x,
                   sd[pfx + "attention.output.LayerNorm.weight"], sd[pfx + "attention.output.LayerNorm.bias"])
    h = gelu(linear(a, sd, pfx + "intermediate.dense"))
    y = layer_norm(linear(h, sd, pfx + "output.dense") + a,
                   sd[pfx + "output.LayerNorm.weight"], sd[pfx + "output.LayerNorm.bias"])
    return (y, probs) if return_probs else y


def visual_model(sd, cfg, input_ids, token_type_ids, attention_mask, visual_embeddings,
                 visual_embeddings_type, image_text_alignment=None, pfx="bert.", bypass_transformer=False,
                 output_attention_weights=False):
    """BertVisualModel.forward, M.py:1275-1333. Returns (all layers, pooled[, attention probabilities per layer]).
    bypass_transformer (M.py:1299-1314): the encoder sees the TEXT positions only (mask sliced to the text keys), the
    visual rows of the embedding output are appended afterwards and one extra BertLayer runs over the full sequence."""
    dt = sd[pfx + "embeddings.word_embeddings.weight"].dtype
    ext = (1.0 - attention_mask[:, None, None, :].to(dt)) * -10000.0
    x = embeddings(sd, input_ids, token_type_ids, visual_embeddings, visual_embeddings_type,
                   image_text_alignment, pfx + "embeddings.")
    A = cfg["num_attention_heads"]
    if bypass_transformer and visual_embeddings is not None:
        T = input_ids.size(1)
        t, vis = x[:, :T], x[:, T:]
        for i in range(cfg["num_hidden_layers"]):
            t = bert_layer(sd, f"{pfx}encoder.layer.{i}.", t, ext[..., :T], A)
        y = bert_layer(sd, pfx + "additional_layer.", torch.cat((t, vis), dim=1), ext, A)
        return [y], torch.tanh(linear(y[:, 0], sd, pfx + "pooler.dense"))
    layers, probs = [], []
    for i in range(cfg["num_hidden_layers"]):
        x = bert_layer(sd, f"{pfx}encoder.layer.{i}.", x, ext, A, output_attention_weights)
        if output_attention_weights:
            x, pr = x
            probs.append(pr)
        layers.append(x)
    pooled = torch.tanh(linear(x[:, 0], sd, pfx + "pooler.dense"))  # M.py:380-386
    return (layers, pooled, probs) if output_attention_weights else (layers, pooled)


def _flat2(t):
    return None if t is None else (t if t.dim() == 2 else t.contiguous().view(-1, t.size(-1)))


def _flat3(t):
    return None if t is None else (t if t.dim() == 3 else t.contiguous().view(-1, t.size(-2), t.size(-1)))


def pretraining_heads(sd, seq, pooled):
    """BertPreTrainingHeads, M.py:389-452; decoder weight tied to the word embeddings (M.py:414)."""
    t = gelu(linear(seq, sd, "cls.predictions.transform.dense"))
    t = layer_norm(t, sd["cls.predictions.transform.LayerNorm.weight"], sd["cls.predictions.transform.LayerNorm.bias"])
    logits = F.linear(t, sd["bert.embeddings.word_embeddings.weight"]) + sd["cls.predictions.bias"]
    return logits, linear(pooled, sd, "cls.seq_relationship")


def objective(sd, cfg, head, input_ids, token_type_ids, input_mask, visual_embeddings, image_mask,
              visual_embeddings_type=None, label=None, masked_lm_labels=None, is_random_next=None,
              image_text_alignment=None, bypass_transformer=False, output_attention_weights=False, flickr_position=None):
    """TrainVisualBERTObjective.forward, M.py:1373-1598 for heads pretraining / vqa / nlvr /
    multichoice, eval mode (dropout off). Returns the reference's output dict."""
    ids, tt, im = _flat2(input_ids), _flat2(token_type_ids), _flat2(input_mask)
    vm, lab = _flat2(image_mask), _flat2(masked_lm_labels)
    ve, ali = _flat3(visual_embeddings), _flat3(image_text_alignment)
    vt = _flat2(visual_embeddings_type) if visual_embeddings_type is not None else torch.zeros_like(vm)
    am = torch.cat((im, vm), dim=-1)
    if lab is not None:
        full = torch.full_like(am, -1)
        full[:, : lab.size(1)] = lab
        lab = full
    res = visual_model(sd, cfg, ids, tt, am, ve, vt, ali, bypass_transformer=bypass_transformer,
                       output_attention_weights=output_attention_weights)
    layers, pooled = res[0], res[1]
    seq = layers[-1]
    out = {"sequence_output": seq, "pooled_output": pooled}
    if output_attention_weights:  # analysis mode: nothing but the attention maps is returned (M.py:1430-1444)
        return {"attention_weights": res[2], "loss": None}
    if head == "pretraining":
        logits, nsp = pretraining_heads(sd, seq, pooled)
        out["logits"], out["seq_relationship_score"], out["loss"] = logits, nsp, None
        if lab is not None:
            mlm = F.cross_entropy(logits.view(-1, logits.size(-1)), lab.view(-1), ignore_index=-1)
            out["masked_lm_loss"] = mlm
            out["loss"] = mlm
            if is_random_next is not None:
                nl = F.cross_entropy(nsp.view(-1, 2), is_random_next.view(-1), ignore_index=-1)
                out["next_sentence_loss"] = nl
                out["loss"] = mlm + nl
    elif head == "vqa":
        idx = im.sum(1) - 2  # M.py:1504
        g = seq[torch.arange(seq.size(0)), idx]
        logits = linear(g, sd, "classifier")
        out["logits"], out["loss"] = logits.unsqueeze(1), None
        if label is not None:
            out["loss"] = F.kl_div(torch.log_softmax(logits, -1), label, reduction="batchmean")
    elif head == "nlvr":
        logits = linear(pooled, sd, "classifier")
        out["logits"], out["loss"] = logits, None
        if label is not None:
            out["loss"] = F.cross_entropy(logits, label)
    elif head == "multichoice":
        logits = linear(pooled, sd, "classifier").view(-1, 4)
        out["logits"], out["loss"] = logits, None
        if label is not None:
            out["loss"] = F.cross_entropy(logits, label)
    elif head == "vqa_advanced":  # M.py:1527-1554: answer tokens predicted by the MLM head; accuracy = all labelled right
        logits, nsp = pretraining_heads(sd, seq, pooled)
        out["logits"], out["seq_relationship_score"] = logits, nsp
        mlm = F.cross_entropy(logits.view(-1, logits.size(-1)), lab.view(-1), ignore_index=-1)
        out["masked_lm_loss"] = out["loss"] = mlm
        pred = logits.argmax(-1)
        ok = ((lab == -1) | (pred == lab)).all(dim=1)
        out["accuracy"] = float(ok.sum().item()) / pred.size(0)
    elif head == "flickr":  # M.py:1568-1598 with FlickrAttention M.py:1602-1646
        out["loss"] = None
        if flickr_position is not None:
            pmask = (flickr_position != -1).long()
            entities = pmask.view(-1).sum(-1)
            pos = flickr_position * pmask
            sel = seq.gather(1, pos.unsqueeze(2).expand(pos.size(0), pos.size(1), seq.size(2)))   # M.py:1713-1716
            vis = seq[:, im.size(1):, :]
            d = sd["flickr_attention.query.weight"].size(0)
            q, k = linear(sel, sd, "flickr_attention.query"), linear(vis, sd, "flickr_attention.key")
            scores = torch.matmul(q, k.transpose(-1, -2)) / math.sqrt(d) + ((1.0 - vm.to(seq.dtype)) * -10000.0)[:, None, :]
            logp = torch.log_softmax(scores, dim=-1)
            out["loss"] = F.kl_div(logp, label, reduction="batchmean")
            lmask = (label != 0.0).to(seq.dtype)                                                  # M.py:1651-1653
            hit = lmask.gather(2, logp.argmax(-1, keepdim=True)).view(-1).sum(-1)                 # M.py:1671-1675
            out["accuracy"] = hit / entities
            out["upperbound_accuracy"] = label.sum(-1).view(-1).sum(-1) / entities
            out["entity_num"] = entities
    else:
        raise ValueError(head)
    return out


# ------------------------------------------------------------------------------------------------
# BertAdam (SURVEY.md §8f rank 2) — restatement of visualbert/pytorch_pretrained_bert/optimization.py ("opt.py")
# ------------------------------------------------------------------------------------------------
def lr_schedule(name, step, warmup, t_total, cycles=0.5):
    """Learning-rate multiplier of the `_LRSchedule` family (opt.py:37-182): `None`/'none' (ConstantLR, opt.py:84-86),
    'warmup_cosine' (opt.py:89-112), 'warmup_constant' (opt.py:154-162), 'warmup_linear' (opt.py:165-174)."""
    if t_total < 0:                                   # opt.py:61-62
        return 1.0
    warmup = max(float(warmup), 0.0)                  # opt.py:50
    progress = float(step) / float(t_total)           # opt.py:63
    if name in (None, "none"):
        return 1.0
    if name == "warmup_constant":
        return progress / warmup if progress < warmup else 1.0
    if name == "warmup_linear":
        return progress / warmup if progress < warmup else max((progress - 1.0) / (warmup - 1.0), 0.0)
    if name == "warmup_cosine":
        if progress < warmup:
            return progress / warmup
        progress = (progress - warmup) / (1 - warmup)
        return 0.5 * (1.0 + math.cos(math.pi * cycles * 2 * progress))
    raise ValueError(name)


def bert_adam_step(p, grad, m, v, step, lr, schedule="warmup_linear", warmup=-1, t_total=-1, b1=0.9, b2=0.999, e=1e-6,
                   weight_decay=0.01, max_grad_norm=1.0):
    """One BertAdam update of ONE parameter tensor (opt.py:253-297); returns (p, m, v, step+1, clipped grad).
    Adam without bias correction (opt.py:299-302), decoupled weight decay added to the update (opt.py:287-288),
    per-parameter gradient clipping (opt.py:272-273 -> torch clip_grad_norm_: coef = max_norm/(||g||+1e-6), applied
    when < 1), schedule evaluated at the parameter's own step counter (opt.py:290-291)."""
    g = grad.clone()
    if max_grad_norm > 0:
        norm = g.double().pow(2).sum().sqrt().to(g.dtype)
        coef = max_grad_norm / (norm + 1e-6)
        if coef < 1:
            g = g * coef
    m = m * b1 + (1 - b1) * g                          # opt.py:277
    v = v * b2 + (1 - b2) * g * g                      # opt.py:278
    update = m / (v.sqrt() + e)                        # opt.py:279
    if weight_decay > 0.0:
        update = update + weight_decay * p             # opt.py:287-288
    lr_scheduled = lr * lr_schedule(schedule, step, warmup, t_total)   # opt.py:290-291
    p = p - lr_scheduled * update                      # opt.py:293-294
    return p, m, v, step + 1, g
