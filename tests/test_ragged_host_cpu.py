"""CPU tests of the host side of batched generation over prompts of different lengths: the mask layout check, the
left-padded -> right-padded repacking in PrefillEngine.forward / generate(), the caller's layout of the results and the
eos / pad_token_id rule.  A stub stands in for the device forward and decode step."""
import pytest
import torch

from gpt4roi_b200.engine import (EngineConfig, KVCache, PrefillEngine, from_right_padded, right_pad_layout,
                                 to_right_padded)

V = 50


def test_right_pad_layout_accepts_right_and_left_padding_only():
    m = torch.tensor([[1, 1, 1, 0, 0], [0, 0, 1, 1, 1], [1, 1, 1, 1, 1], [0, 0, 0, 0, 1]])
    lens, shift = right_pad_layout(m)
    assert lens.tolist() == [3, 3, 5, 1] and shift.tolist() == [0, 2, 0, 4]
    for bad in ([[1, 0, 1, 0, 0]], [[0, 1, 1, 0, 0]], [[0, 0, 0, 0, 0]]):
        with pytest.raises(NotImplementedError):
            right_pad_layout(torch.tensor(bad))
    x = torch.arange(20).view(4, 5)
    r = to_right_padded(x, shift)
    assert r[1].tolist() == [7, 8, 9, 5, 6] and r[3].tolist() == [19, 15, 16, 17, 18]
    for b in range(4):
        assert r[b, :lens[b]].tolist() == x[b][m[b].bool()].tolist()     # the tokens first, in order
    assert torch.equal(from_right_padded(r, shift), x)
    y = torch.randn(4, 5, 3)
    assert torch.equal(from_right_padded(to_right_padded(y, shift), shift), y)


class _Stub:
    """Next-token rule: (last valid token + 1) % V.  forward_device records what it is given."""
    dev = torch.device('cpu')
    dt = torch.bfloat16

    def __init__(self):
        self.cfg = EngineConfig(hidden=64, n_heads=1, n_layers=1, mlp=128, vocab=V)   # head_dim 64: no CUDA graph
        self.seen = []

    def plan_boxes(self, bboxes):
        return None

    def forward_device(self, ids, images, plan, validate=True, last_only=False, seqlens=None, cache=None, **kw):
        self.seen.append((ids.clone(), None if seqlens is None else seqlens.clone()))
        B, L = ids.shape
        if cache is not None:
            cache.start(L, seqlens)
        if last_only:
            lens = torch.full((B,), L) if seqlens is None else seqlens.long()
            last = ids[torch.arange(B), lens - 1]
            return torch.nn.functional.one_hot((last + 1) % V, V).float()[:, None]
        return torch.nn.functional.one_hot((ids + 1) % V, V).float()

    def decode_step(self, ids, cache, pos_dev=None):
        cache.length += 1
        if cache.lens is not None:
            cache.lens.add_(1)
        return torch.nn.functional.one_hot((ids[:, 0] + 1) % V, V).float()[:, None]

    forward = PrefillEngine.forward
    generate = PrefillEngine.generate


def _batch():
    ids_r = torch.tensor([[3, 4, 5, 6], [7, 8, 0, 0], [9, 0, 0, 0]])
    mask_r = torch.tensor([[1, 1, 1, 1], [1, 1, 0, 0], [1, 0, 0, 0]])
    ids_l = torch.tensor([[3, 4, 5, 6], [0, 0, 7, 8], [0, 0, 0, 9]])
    mask_l = torch.tensor([[1, 1, 1, 1], [0, 0, 1, 1], [0, 0, 0, 1]])
    return ids_r, mask_r, ids_l, mask_l


def test_forward_repacks_left_padding_and_answers_in_the_callers_layout():
    ids_r, mask_r, ids_l, mask_l = _batch()
    eng = _Stub()
    out = eng.forward(ids_l, None, None, attention_mask=mask_l)
    ran, seqlens = eng.seen[-1]
    assert torch.equal(ran[mask_r.bool()], ids_r[mask_r.bool()]) and seqlens.tolist() == [4, 2, 1]
    assert torch.equal(out.argmax(-1), (ids_l + 1) % V)                       # logits in the caller's layout
    last = eng.forward(ids_l, None, None, attention_mask=mask_l, last_only=True)
    assert last[:, 0].argmax(-1).tolist() == [7, 9, 10]                        # each row's last valid token + 1
    cache = KVCache(eng.cfg, 3, 8, 'cpu')
    eng.forward(ids_r, None, None, attention_mask=mask_r, last_only=True, cache=cache)
    assert cache.length == 4 and cache.lens.tolist() == [4, 2, 1] and cache.lens.dtype == torch.int32


def test_generate_left_and_right_padding_give_the_same_tokens_and_keep_the_prompt():
    ids_r, mask_r, ids_l, mask_l = _batch()
    eng = _Stub()
    out_r = eng.generate(ids_r, torch.zeros(3, 3, 4, 4), None, max_new_tokens=3, attention_mask=mask_r)
    out_l = eng.generate(ids_l, torch.zeros(3, 3, 4, 4), None, max_new_tokens=3, attention_mask=mask_l)
    assert torch.equal(out_r[:, :4], ids_r) and torch.equal(out_l[:, :4], ids_l)
    assert out_r[:, 4:].tolist() == [[7, 8, 9], [9, 10, 11], [10, 11, 12]]
    assert torch.equal(out_l[:, 4:], out_r[:, 4:])
    assert eng.seen[-1][1].tolist() == [4, 2, 1]
    # an all-ones mask takes the uniform path (no per-sample lengths)
    eng.generate(ids_r, torch.zeros(3, 3, 4, 4), None, max_new_tokens=1, attention_mask=torch.ones_like(ids_r))
    assert eng.seen[-1][1] is None


def test_generate_pads_finished_rows_and_stops_when_all_are_done():
    ids_r, mask_r, _, _ = _batch()
    eng = _Stub()
    # row 1 emits 9 at step 0 (then pads); row 0 emits 9 at step 2; row 2 never does within the budget
    out = eng.generate(ids_r, torch.zeros(3, 3, 4, 4), None, max_new_tokens=4, attention_mask=mask_r, eos_token_id=9,
                       pad_token_id=0)
    assert out[:, 4:].tolist() == [[7, 8, 9, 0], [9, 0, 0, 0], [10, 11, 12, 13]]
    # every row finished -> the loop ends early
    out = eng.generate(ids_r[1:], torch.zeros(2, 3, 4, 4), None, max_new_tokens=6, attention_mask=mask_r[1:],
                       eos_token_id=11, pad_token_id=0)
    assert out[:, 4:].tolist() == [[9, 10, 11], [10, 11, 0]]
    # without pad_token_id the old rule holds: stop only when all rows emit eos at the same step
    out = eng.generate(ids_r, torch.zeros(3, 3, 4, 4), None, max_new_tokens=4, attention_mask=mask_r, eos_token_id=9)
    assert out.shape == (3, 8)
