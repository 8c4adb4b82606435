"""Deterministic synthetic weights and batches (SURVEY.md §8d) shared by tests, goldens and bench.

There is no network in the build/bench environment, so neither pretrained BERT weights nor the
COCO/VQA feature files exist: every measurement and parity check uses random-init weights of the
named architecture and synthetic region features of the reference's tensor-dict layout
(reference visualbert/dataloaders/coco_dataset.py:446-460 → keys of `model.forward`).
"""
import torch

# the BASELINE.json configs (index = cfg number - 1)
CONFIGS = {
    "cfg1": dict(layers=2, hidden=768, heads=12, inter=3072, B=4, V=36, T=20, Dv=2048, head="pretraining"),
    "cfg2": dict(layers=12, hidden=768, heads=12, inter=3072, B=256, V=36, T=128, Dv=2048, head="pretraining"),
    # configs[2..4] are quoted as GLOBAL batches over 8 data-parallel GPUs: `dp` = ranks the batch B is spread over
    "cfg3": dict(layers=12, hidden=768, heads=12, inter=3072, B=512, dp=8, V=36, T=128, Dv=2048, head="vqa"),
    "cfg4": dict(layers=12, hidden=768, heads=12, inter=3072, B=256, dp=8, V=72, T=40, Dv=2048, head="nlvr"),
    "cfg5": dict(layers=24, hidden=1024, heads=16, inter=4096, B=1024, dp=8, V=100, T=256, Dv=2048, head="pretraining"),
}


def bert_config_dict(layers, hidden, heads, inter, vocab=30522, max_pos=512, p_drop=0.1):
    return dict(vocab_size=vocab, hidden_size=hidden, num_hidden_layers=layers, num_attention_heads=heads,
                intermediate_size=inter, hidden_act="gelu", hidden_dropout_prob=p_drop,
                attention_probs_dropout_prob=p_drop, max_position_embeddings=max_pos, type_vocab_size=2,
                initializer_range=0.02)


def _layer_shapes(s, p, H, I):
    for n in ("query", "key", "value"):
        s[p + f"attention.self.{n}.weight"] = (H, H)
        s[p + f"attention.self.{n}.bias"] = (H,)
    s[p + "attention.output.dense.weight"] = (H, H)
    s[p + "attention.output.dense.bias"] = (H,)
    s[p + "attention.output.LayerNorm.weight"] = (H,)
    s[p + "attention.output.LayerNorm.bias"] = (H,)
    s[p + "intermediate.dense.weight"] = (I, H)
    s[p + "intermediate.dense.bias"] = (I,)
    s[p + "output.dense.weight"] = (H, I)
    s[p + "output.dense.bias"] = (H,)
    s[p + "output.LayerNorm.weight"] = (H,)
    s[p + "output.LayerNorm.bias"] = (H,)


def param_shapes(cfg, head, visual_dim, bypass_transformer=False):
    """Reference state_dict keys → shapes (SURVEY.md §8b). `bert.additional_layer.*` (bypass_transformer, M.py:1268-1269)
    is appended LAST so that the seeded draws of all other keys do not depend on the flag."""
    H, I, Vc = cfg["hidden_size"], cfg["intermediate_size"], cfg["vocab_size"]
    P, Tv = cfg["max_position_embeddings"], cfg["type_vocab_size"]
    s = {}
    e = "bert.embeddings."
    s[e + "word_embeddings.weight"] = (Vc, H)
    s[e + "position_embeddings.weight"] = (P, H)
    s[e + "token_type_embeddings.weight"] = (Tv, H)
    s[e + "LayerNorm.weight"] = (H,)
    s[e + "LayerNorm.bias"] = (H,)
    s[e + "token_type_embeddings_visual.weight"] = (Tv, H)
    s[e + "position_embeddings_visual.weight"] = (P, H)
    s[e + "projection.weight"] = (H, visual_dim)
    s[e + "projection.bias"] = (H,)
    for i in range(cfg["num_hidden_layers"]):
        _layer_shapes(s, f"bert.encoder.layer.{i}.", H, I)
    s["bert.pooler.dense.weight"] = (H, H)
    s["bert.pooler.dense.bias"] = (H,)
    if head in ("pretraining", "vqa_advanced", "flickr"):
        s["cls.predictions.bias"] = (Vc,)
        s["cls.predictions.transform.dense.weight"] = (H, H)
        s["cls.predictions.transform.dense.bias"] = (H,)
        s["cls.predictions.transform.LayerNorm.weight"] = (H,)
        s["cls.predictions.transform.LayerNorm.bias"] = (H,)
        s["cls.seq_relationship.weight"] = (2, H)
        s["cls.seq_relationship.bias"] = (2,)
    if head == "multichoice":
        s["classifier.weight"], s["classifier.bias"] = (1, H), (1,)
    elif head == "vqa":
        s["classifier.weight"], s["classifier.bias"] = (3129, H), (3129,)
    elif head == "nlvr":
        s["classifier.weight"], s["classifier.bias"] = (2, H), (2,)
    if head == "flickr":
        d = H // cfg["num_attention_heads"]
        for n in ("query", "key", "value"):
            s[f"flickr_attention.{n}.weight"], s[f"flickr_attention.{n}.bias"] = (d, H), (d,)
    if bypass_transformer:
        _layer_shapes(s, "bert.additional_layer.", H, I)
    return s


def init_state_dict(cfg, head, visual_dim, seed=0, dtype=torch.float32, bypass_transformer=False):
    """Seeded random init: matrices N(0, 0.02) (reference M.py:473-484); LayerNorm weights 1+N(0,0.1)
    and all biases N(0, 0.05) so that no parameter is trivially 0/1 in parity tests."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shp in param_shapes(cfg, head, visual_dim, bypass_transformer).items():
        if k.endswith("LayerNorm.weight"):
            t = 1.0 + 0.1 * torch.randn(shp, generator=g)
        elif k.endswith("bias"):
            t = 0.05 * torch.randn(shp, generator=g)
        else:
            t = 0.02 * torch.randn(shp, generator=g)
        sd[k] = t.to(dtype)
    return sd


def make_batch(B, T, V, Dv, head="pretraining", seed=1234, ragged=False, vocab=30522, nlvr_types=False,
               choices=None, alignment=None):
    """Reference tensor-dict for TrainVisualBERTObjective.forward (M.py:1373-1392).

    ragged=True draws text lengths ~U[T/2, T] and region counts ~U[V/2, V] (parity tests);
    choices=C produces VCR-style 3-D ids [B, C, T] / 4-D features [B, C, V, Dv];
    alignment=A adds VCR `image_text_alignment` [.., V, A]: text positions each region is tied to, -1 = padding
    (M.py:1223-1245), drawn AFTER everything else so the other tensors do not depend on it."""
    g = torch.Generator().manual_seed(seed)
    lead = (B,) if choices is None else (B, choices)
    n = B if choices is None else B * choices
    lo = 1000 if vocab > 2000 else 3
    ids = torch.randint(lo, min(30000, vocab), (n, T), generator=g)
    ids[:, 0] = 101 % vocab
    if ragged:
        tl = torch.randint(max(2, T // 2), T + 1, (n,), generator=g)
        vl = torch.randint(max(1, V // 2), V + 1, (n,), generator=g)
    else:
        tl = torch.full((n,), T)
        vl = torch.full((n,), V)
    ar = torch.arange(T).unsqueeze(0)
    input_mask = (ar < tl.unsqueeze(1)).long()
    ids[torch.arange(n), tl - 1] = 102 % vocab
    ids = ids * input_mask
    image_mask = (torch.arange(V).unsqueeze(0) < vl.unsqueeze(1)).long()
    feats = torch.randn(n, V, Dv, generator=g).clamp_(min=0)
    vtype = torch.zeros(n, V, dtype=torch.long)
    if nlvr_types:
        vtype[:, V // 2:] = 1
    batch = dict(
        input_ids=ids.view(*lead, T), token_type_ids=torch.zeros_like(ids).view(*lead, T),
        input_mask=input_mask.view(*lead, T), visual_embeddings=feats.view(*lead, V, Dv),
        position_embeddings_visual=None, image_mask=image_mask.view(*lead, V),
        visual_embeddings_type=vtype.view(*lead, V))
    if head == "pretraining":
        sel = (torch.rand(n, T, generator=g) < 0.15) & (input_mask == 1)
        sel[:, 1] = True  # at least one labelled token per row
        batch["masked_lm_labels"] = torch.where(sel, ids, torch.full_like(ids, -1)).view(*lead, T)
        batch["is_random_next"] = torch.randint(0, 2, (n,), generator=g)
    elif head == "vqa":
        r = torch.rand(n, 3129, generator=g)
        batch["label"] = r * (torch.rand(n, 3129, generator=g) < 0.003).float()
    elif head == "nlvr":
        batch["label"] = torch.randint(0, 2, (n,), generator=g)
    elif head == "multichoice":
        batch["label"] = torch.randint(0, choices or 4, (B,), generator=g)
    elif head == "vqa_advanced":  # answers as masked tokens (M.py:1527-1554): MLM labels only
        sel = (torch.rand(n, T, generator=g) < 0.15) & (input_mask == 1)
        sel[:, 1] = True
        batch["masked_lm_labels"] = torch.where(sel, ids, torch.full_like(ids, -1)).view(*lead, T)
    elif head == "flickr":  # phrase grounding (M.py:1568-1598): entity token positions and soft region targets
        E = 4
        pos = torch.stack([torch.randint(1, max(2, int(tl[i])), (E,), generator=g) for i in range(n)])
        n_ent = torch.randint(1, E + 1, (n,), generator=g)
        pos = torch.where(torch.arange(E).unsqueeze(0) < n_ent.unsqueeze(1), pos, torch.full_like(pos, -1))
        tgt = (torch.rand(n, E, V, generator=g) < 0.3).float() * image_mask.unsqueeze(1).float()
        tgt[:, :, 0] = 1.0  # every entity has at least one target region (region 0 is always valid)
        tgt = tgt * (pos != -1).unsqueeze(-1).float()
        batch["flickr_position"] = pos
        batch["label"] = tgt / tgt.sum(-1, keepdim=True).clamp(min=1.0)
    if alignment:
        ali = torch.randint(0, T, (n, V, alignment), generator=g)
        ali = torch.where(torch.rand(n, V, alignment, generator=g) < 0.4, torch.full_like(ali, -1), ali)
        ali[:, 0, :] = -1  # a region without any aligned word: the divide-by-zero guard of M.py:1236
        batch["image_text_alignment"] = ali.view(*lead, V, alignment)
    return batch
