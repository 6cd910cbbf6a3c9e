"""CPU tests of multi-turn reuse: KVCache.reusable's rules on host tensors, and the model seam handing a later turn on a
non-empty cache to the engine as one reuse-or-prefill call (a stub engine stands in for the CUDA one)."""
import torch

from gpt4roi_b200.engine import EngineConfig, KVCache
from tests.test_model_seam_cpu import _StubEngine, _tiny_model

CFG = EngineConfig(image_size=28, vit_hidden=32, vit_heads=2, vit_layers=2, vit_mlp=64, hidden=64, n_heads=2,
                   n_layers=1, mlp=128, vocab=140, bbox_token=132, im_patch_token=131, im_start_token=134,
                   im_end_token=135)
BB = CFG.bbox_token


def _cache(ids, images, boxes, max_len=32):
    B, L = ids.shape
    c = KVCache(CFG, B, max_len, 'cpu')
    c.start(L, None, ids)
    c.set_source(images, boxes)
    return c


def _row(*toks):
    return torch.tensor([list(toks)])


def test_kv_cache_is_zero_filled_and_grows_zero_filled():
    c = KVCache(CFG, 2, 8, 'cpu')
    assert all(bool((t == 0).all()) for t in c.k + c.v) and bool((c.ids == -1).all())
    c.k[0].fill_(1.0)
    c.start(3, None, torch.tensor([[5, 6, 7], [8, 9, 10]]))
    c.grow(20)
    assert c.max_len == 20 and c.k[0].shape[1] == 20
    assert bool((c.k[0][:, :8] == 1).all()) and bool((c.k[0][:, 8:] == 0).all()) and bool((c.v[0] == 0).all())
    assert c.ids[:, :3].tolist() == [[5, 6, 7], [8, 9, 10]] and bool((c.ids[:, 3:] == -1).all())


def test_reusable_prefix_rules():
    img = torch.randn(1, 3, 28, 28)
    box = [torch.tensor([[0.1, 0.1, 0.5, 0.5]])]
    c = _cache(_row(1, 2, BB, 4, 5, 6, 7), img, box)
    assert c.reusable(_row(1, 2, BB, 4, 5, 6, 7, 8, 9), img, box).tolist() == [7]        # all of it
    assert c.reusable(_row(1, 2, BB, 4, 5, 6, 7), img, box).tolist() == [6]              # len - 1 cap
    assert c.reusable(_row(1, 2, BB, 4, 9, 6, 7, 8), img, box).tolist() == [4]           # first id mismatch
    assert c.reusable(_row(1, 2, BB, 4, 5, 6, 7, 8), img + 1, box).tolist() == [0]       # another image
    assert c.reusable(_row(1, 2, BB, 4, 5, 6, 7, 8), None, box).tolist() == [0]
    other = [torch.tensor([[0.1, 0.1, 0.5, 0.6]])]
    assert c.reusable(_row(1, 2, BB, 4, 5, 6, 7, 8), img, other).tolist() == [2]         # stops at the changed box
    assert c.reusable(_row(1, 2, BB, 4, 5, 6, 7, 8), img, [None]).tolist() == [2]
    more = [torch.cat([box[0], torch.tensor([[0.2, 0.2, 0.3, 0.3]])])]
    assert c.reusable(_row(1, 2, BB, 4, 5, BB, 7, 8), img, more).tolist() == [5]         # new box in the tail
    e = _cache(_row(1, 2, 3, 4), img, [])                                                 # [] = no boxes, as plan_boxes
    assert e.boxes == [None] and e.reusable(_row(1, 2, 3, 4, 5), img, []).tolist() == [4]
    c.source_known = False                                                                 # unknown source
    assert c.reusable(_row(1, 2, BB, 4, 5, 6, 7, 8), img, box).tolist() == [0]


def test_reusable_pads_after_eos_and_left_padded_masks():
    img = torch.randn(2, 3, 28, 28)
    boxes = [None, None]
    ids = torch.tensor([[1, 2, 3, 4, 0, 0], [1, 5, 6, 7, 8, 9]])
    c = _cache(ids, img, boxes)
    # row 0 finished with eos 4 and was padded with 0 afterwards: its next turn continues after the eos
    nxt = torch.tensor([[1, 2, 3, 4, 11, 12, 13], [1, 5, 6, 7, 8, 9, 10]])
    assert c.reusable(nxt, img, boxes).tolist() == [4, 6]
    # the same prompts left-padded (row 0 one token shorter)
    left = torch.tensor([[0, 1, 2, 3, 4, 11, 12], [1, 5, 6, 7, 8, 9, 10]])
    mask = torch.tensor([[0, 1, 1, 1, 1, 1, 1], [1] * 7])
    assert c.reusable(left, img, boxes, attention_mask=mask).tolist() == [4, 6]
    # per-row lengths bound the match
    c.lens = torch.tensor([3, 6], dtype=torch.int32)
    assert c.reusable(nxt, img, boxes).tolist() == [3, 6]


class _ReuseStub(_StubEngine):
    def prefill_cached(self, cache, input_ids, images, bboxes, attention_mask=None, new_tokens=0):
        self.calls.append(('reuse', tuple(input_ids.shape), images is not None, bboxes))
        cache.length = input_ids.shape[1]
        return self._logits(input_ids[:, -1:])


def test_longer_input_on_a_filled_cache_reaches_the_engine_as_one_reuse_call():
    from transformers import DynamicCache
    m = _tiny_model().eval()
    stub = _ReuseStub(CFG)
    m._get_engine = lambda device: stub
    img = torch.zeros(1, 3, 28, 28)
    boxes = [torch.tensor([[0.1, 0.1, 0.5, 0.5]])]
    cache = DynamicCache()
    out1 = m.generate(torch.tensor([[1, 5, 9]]), images=img, bboxes=boxes, max_new_tokens=3, use_hf_loop=True,
                      pad_token_id=0, past_key_values=cache)
    assert out1.tolist() == [[1, 5, 9, 10, 11, 12]]
    assert cache._g4r_cache.kv.length == 5
    n = len(stub.calls)
    ids2 = torch.cat([out1, torch.tensor([[20, 21]])], 1)
    out2 = m.generate(ids2, images=img, bboxes=boxes, max_new_tokens=3, use_hf_loop=True, pad_token_id=0,
                      past_key_values=cache)
    assert out2.tolist() == [[1, 5, 9, 10, 11, 12, 20, 21, 22, 23, 24]]
    turn2 = stub.calls[n:]
    assert [c[0] for c in turn2] == ['reuse', 'decode', 'decode']
    assert turn2[0][1] == (1, 8) and turn2[0][2] is True and turn2[0][3] is boxes
    assert [c[2] for c in turn2[1:]] == [8, 9]
    # a prompt no longer than the cache plus one token (turn 1 regenerated on the same cache) is still a prompt
    n = len(stub.calls)
    out3 = m.generate(torch.tensor([[1, 5, 9]]), images=img, bboxes=boxes, max_new_tokens=3, use_hf_loop=True,
                      pad_token_id=0, past_key_values=cache)
    assert out3.tolist() == [[1, 5, 9, 10, 11, 12]]
    assert [c[0] for c in stub.calls[n:]] == ['reuse', 'decode', 'decode'] and stub.calls[n][1] == (1, 3)


def test_prepare_inputs_passes_a_later_turn_whole():
    from gpt4roi_b200.spi_llava import G4RCache
    m = _tiny_model()
    cache = G4RCache(KVCache(CFG, 1, 16, 'cpu'))
    cache.kv.length = 4
    ids = torch.tensor([[1, 2, 3, 4, 5, 6, 7]])
    mask = torch.ones_like(ids)
    got = m.prepare_inputs_for_generation(ids, past_key_values=cache, attention_mask=mask)
    assert got['input_ids'] is ids and got['attention_mask'] is mask
