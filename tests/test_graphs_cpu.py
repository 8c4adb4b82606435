"""CUDA-graph support without a GPU: parallel.pad_batch for every head (3-D VCR inputs included), the graph-capturable dropout
counter of BertVisualModel (same seed sequence as the default mode, across mode switches and saved states), and
vb_set_dropout_offset being set and cleared on the host."""
import ctypes

import pytest
import torch

from visualbert_b200 import BertConfig, TrainVisualBERTObjective, _lib, parallel, synthetic


@pytest.mark.parametrize("head,choices,alignment", [("pretraining", None, None), ("vqa", None, None), ("nlvr", None, None),
                                                    ("flickr", None, None), ("multichoice", 4, 3)])
def test_pad_batch_values_and_shapes(head, choices, alignment):
    b = synthetic.make_batch(2, 7, 5, 16, head=head, seed=3, vocab=512, ragged=True, choices=choices, alignment=alignment)
    p = parallel.pad_batch(b, 12, 9)
    lead = (2,) if choices is None else (2, choices)
    for k, fill in (("input_ids", 0), ("token_type_ids", 0), ("input_mask", 0), ("masked_lm_labels", -1)):
        if k in b:
            assert p[k].shape == lead + (12,)
            assert torch.equal(p[k][..., :7], b[k]) and bool((p[k][..., 7:] == fill).all())
    for k in ("image_mask", "visual_embeddings_type"):
        assert p[k].shape == lead + (9,)
        assert torch.equal(p[k][..., :5], b[k]) and bool((p[k][..., 5:] == 0).all())
    assert p["visual_embeddings"].shape == lead + (9, 16)
    assert torch.equal(p["visual_embeddings"][..., :5, :], b["visual_embeddings"])
    assert bool((p["visual_embeddings"][..., 5:, :] == 0).all())
    if alignment:
        assert p["image_text_alignment"].shape == lead + (9, alignment)
        assert torch.equal(p["image_text_alignment"][..., :5, :], b["image_text_alignment"])
        assert bool((p["image_text_alignment"][..., 5:, :] == -1).all())
    if head == "flickr":
        assert p["label"].shape[-1] == 9 and bool((p["label"][..., 5:] == 0).all())
        assert torch.equal(p["flickr_position"], b["flickr_position"])
    elif "label" in b:
        assert torch.equal(p["label"], b["label"])
    assert p["position_embeddings_visual"] is None
    with pytest.raises(ValueError, match="exceeds"):
        parallel.pad_batch(b, 6, 9)


def _bert():
    cfg = synthetic.bert_config_dict(1, 64, 1, 128, vocab=128)
    return TrainVisualBERTObjective(BertConfig.from_dict(cfg), "nlvr", visual_embedding_dim=16).bert


def _capturable_seed(m):
    k = m.next_seed()
    return (k + int(m._seed_offset.item())) & 0xFFFFFFFFFFFFFFFF


def test_capturable_counter_gives_the_default_sequence():
    a, b = _bert(), _bert()
    b.dropout_seed = a.dropout_seed
    ref = [a.next_seed() for _ in range(6)]
    got = [_capturable_seed(b.set_graph_capturable(True)) for _ in range(3)]
    assert b._vb_step.dtype == torch.int64 and "_vb_step" not in b.state_dict()
    assert b.dropout_state() == {"seed": a.dropout_seed, "step": 3}
    b.set_graph_capturable(False)        # the counter comes back to the host
    got += [b.next_seed()]
    b.set_graph_capturable(True)
    got += [_capturable_seed(b) for _ in range(2)]
    assert got == ref
    # a state saved in one mode restores in the other, both ways; steps that carry across bit 32 included
    st = {"seed": a.dropout_seed, "step": 2 ** 32 - 2}
    a.set_dropout_state(st)
    b.set_dropout_state(st)
    assert [_capturable_seed(b) for _ in range(2)] == [a.next_seed() for _ in range(2)]
    saved = b.dropout_state()
    assert saved["step"] == 2 ** 32
    b.set_graph_capturable(False)
    b.set_dropout_state(saved)
    a.set_dropout_state(saved)
    assert b.next_seed() == a.next_seed()


def test_capturable_mode_refuses_unpadded():
    m = _bert()
    m.set_graph_capturable(True)
    with pytest.raises(ValueError, match="graph-capturable"):
        m.set_unpadded(True)
    m.set_graph_capturable(False)
    m.set_unpadded(True)
    with pytest.raises(ValueError, match="set_unpadded"):
        m.set_graph_capturable(True)


def test_set_dropout_offset_without_a_device():
    L = _lib.lib()
    word = ctypes.c_uint64(5)   # any 8-byte-aligned address: the host never reads it
    assert L.vb_set_dropout_offset(ctypes.addressof(word)) == 0
    assert L.vb_set_dropout_offset(None) == 0
    assert L.vb_set_dropout_offset(ctypes.addressof(word) + 4) != 0
    assert b"8-byte aligned" in L.vb_last_error()
    assert L.vb_set_dropout_offset(None) == 0


def test_capacity_padded_rows_and_overflow():
    b = synthetic.make_batch(3, 9, 4, 16, head="pretraining", seed=11, vocab=512, ragged=True)
    plain = parallel.BatchPrefetcher.labelled_rows(b)
    n = plain.numel()
    rows = parallel.BatchPrefetcher.labelled_rows(b, capacity=n + 5)
    assert rows.shape == (n + 5,) and torch.equal(rows[:n], plain) and bool((rows[n:] == -1).all())
    assert torch.equal(parallel.BatchPrefetcher.labelled_rows(b, capacity=n), plain)
    with pytest.raises(ValueError, match="more than mlm_rows_capacity"):
        parallel.BatchPrefetcher.labelled_rows(b, capacity=n - 1)


@pytest.mark.parametrize("choices", [None, 2])
def test_pad_batch_remaps_masked_lm_rows(choices):
    b = synthetic.make_batch(3, 9, 4, 16, head="pretraining", seed=12, vocab=512, ragged=True, choices=choices)
    b["masked_lm_rows"] = parallel.BatchPrefetcher.labelled_rows(b, capacity=40)
    p = parallel.pad_batch(b, 13, 6)
    rows, labels = p["masked_lm_rows"], p["masked_lm_labels"].reshape(-1, 13)
    valid = rows >= 0
    assert int((rows == -1).sum()) == int((b["masked_lm_rows"] == -1).sum())
    ex, pos = rows[valid] // (13 + 6), rows[valid] % (13 + 6)
    assert bool((pos < 13).all())
    # every remapped row still points at a labelled text position, and they are exactly the labelled positions
    assert bool((labels[ex, pos] >= 0).all()) and int(valid.sum()) == int((labels >= 0).sum())


def test_pad_batch_flickr_entities():
    b = synthetic.make_batch(2, 7, 5, 16, head="flickr", seed=3, vocab=512)
    E = b["flickr_position"].shape[-1]
    p = parallel.pad_batch(b, 12, 9, entities=E + 2)
    assert p["flickr_position"].shape[-1] == E + 2 and bool((p["flickr_position"][..., E:] == -1).all())
    assert p["label"].shape[-2:] == (E + 2, 9) and bool((p["label"][..., E:, :] == 0).all())
    assert torch.equal(p["label"][..., :E, :5], b["label"])
