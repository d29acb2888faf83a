"""Calibration mask conventions on the CPU: the label ids / attention mask built per token batch, and the valid-token masks
derived from the label ids, against a literal per-row restatement of the reference's loops (calibration/llm.py:346-398)."""
from types import SimpleNamespace

import pytest
import torch

from auto_round_b200.autoround import label_ids_and_mask, repeated_tail
from auto_round_b200.quantizer import valid_token_masks

TOKENIZERS = [SimpleNamespace(pad_token_id=pid, pad_token=pt) for pid in (None, 1) for pt in (None, "<pad>")]


def _loop_labels(input_ids, pad_id):
    ids = input_ids.clone()
    if pad_id is not None:
        ids[ids == pad_id] = -100
    else:
        for b in range(ids.shape[0]):
            last = ids[b, -1].clone()
            j = ids.shape[1] - 2
            while j >= 0 and ids[b, j] == last:
                ids[b, j] = -100
                j -= 1
    ids[:, -1] = -100
    return ids


def _loop_mask(input_ids, pad_id, pad_token):
    if pad_id is not None and pad_token is not None:
        am = (input_ids != pad_id).to(torch.long)
    else:
        am = torch.ones_like(input_ids, dtype=torch.long)
        for b in range(input_ids.shape[0]):
            last = input_ids[b, -1]
            j = input_ids.shape[1] - 2
            rep = False
            while j >= 0 and input_ids[b, j] == last:
                rep = True
                am[b, j] = 0
                j -= 1
            if rep:
                am[b, -1] = 0
    am[:, -1] = 0
    return am


def _batches():
    g = torch.Generator().manual_seed(0)
    for seqlen in (1, 2, 3, 8, 33):
        for vocab in (2, 3, 50):
            ids = torch.randint(0, vocab, (6, seqlen), generator=g)
            ids[0] = ids[0, 0]                                          # one token throughout
            if seqlen > 2:
                ids[1, seqlen // 2:] = ids[1, -1]                       # repeated tail
                ids[2, 1:] = 1                                          # repeated tail of the pad id
            yield ids


@pytest.mark.parametrize("tok", TOKENIZERS, ids=lambda t: f"pad_id={t.pad_token_id},pad_token={t.pad_token}")
def test_labels_and_mask_match_the_row_loops(tok):
    for input_ids in _batches():
        before = input_ids.clone()
        ids, am = label_ids_and_mask(input_ids, tok)
        assert torch.equal(input_ids, before)                           # the model still reads the raw tokens
        assert torch.equal(ids, _loop_labels(input_ids, tok.pad_token_id)), input_ids
        assert torch.equal(am, _loop_mask(input_ids, tok.pad_token_id, tok.pad_token)), input_ids
        assert ids.dtype == input_ids.dtype and am.dtype == torch.long


def test_repeated_tail_stops_at_the_first_other_token():
    ids = torch.tensor([[5, 5, 5, 5], [1, 2, 2, 2], [2, 2, 1, 2], [1, 2, 3, 4]])
    want = torch.tensor([[1, 1, 1, 0], [0, 1, 1, 0], [0, 0, 0, 0], [0, 0, 0, 0]], dtype=torch.bool)
    assert torch.equal(repeated_tail(ids), want)


def _loop_token_masks(input_ids):
    masks = [(ids != -100).reshape(-1) for ids in input_ids]
    if all(bool(m.all()) for m in masks):
        return None, None
    return masks, torch.stack(masks).to(dtype=torch.uint8).contiguous()


def test_valid_token_masks_both_forms():
    assert valid_token_masks(None, "cpu") is None and valid_token_masks(None, "cpu", stacked=True) is None
    unmasked = [torch.arange(1, 9).reshape(1, 8) for _ in range(3)]
    assert valid_token_masks(unmasked, "cpu") is None and valid_token_masks(unmasked, "cpu", stacked=True) is None
    for tok in TOKENIZERS:
        for input_ids in _batches():
            ids_cache = list(torch.split(label_ids_and_mask(input_ids, tok)[0], 1, dim=0))
            want_rows, want_stacked = _loop_token_masks(ids_cache)
            rows = valid_token_masks(ids_cache, "cpu")
            stacked = valid_token_masks(ids_cache, "cpu", stacked=True)
            assert want_rows is not None                                # the last position is always masked
            assert len(rows) == len(want_rows) and all(torch.equal(a, b) for a, b in zip(rows, want_rows))
            assert rows[0].dtype == torch.bool
            assert stacked.dtype == torch.uint8 and stacked.is_contiguous() and torch.equal(stacked, want_stacked)
