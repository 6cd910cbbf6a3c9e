"""CPU tests of prefix reuse in continuous batching (ContinuousBatcher(prefix_reuse=True)): the row records, the choice
of row, the prefix copy, the reuse refusals, one chunk prefill per round, the failure fallback, Request.reused, the
unchanged default and the seam's flag -- on a stub engine whose prefill and chunk prefill write each token's id into its
K/V position, so that what every row holds can be read back.  The GPU tests run the same batcher on the real engine
(tests/test_serve_prefix_gpu.py)."""
import pytest
import torch

from gpt4roi_b200.engine import ContinuousBatcher, EngineConfig

V = 140
IMP, BOX, IMS, IME = 130, 131, 132, 133      # image patch, <bbox>, image start / end ids of the stub's config


def _cfg():
    return EngineConfig(image_size=28, vit_hidden=32, vit_heads=2, vit_layers=2, vit_mlp=64, hidden=256, n_heads=2,
                        n_layers=2, mlp=128, vocab=V, im_patch_token=IMP, bbox_token=BOX, im_start_token=IMS,
                        im_end_token=IME, dtype='fp16')


class _Stub:
    """Prefill (batch 1, forward_device), chunk prefill (extend) and decode step on the host: each writes token id t at its position
    p of every layer l as k[l][row, p, 0] = t, k[l][row, p, 1] = l + 1, v = -k; logits are one-hot((last id + 1) % V).
    `calls` records every prefill, chunk prefill (rows, starts, tails, boxes, and a copy of the K/V as the call found
    them) and decode step.  A chunk whose <bbox> count its boxes do not match raises, as the splice does (status 3)."""

    def __init__(self):
        self.cfg = _cfg()
        self.dev, self.dt, self.calls = torch.device('cpu'), self.cfg.torch_dtype, []

    def _logits(self, last):
        out = torch.zeros(last.shape[0], 1, V, dtype=self.dt)
        out[torch.arange(last.shape[0]), 0, (last + 1) % V] = 1.0
        return out

    def plan_boxes(self, bboxes):
        return bboxes

    def _write(self, k, v, row, pos, ids):
        for l in range(len(k)):
            k[l][row, pos, 0] = ids.to(self.dt)
            k[l][row, pos, 1] = l + 1
            v[l][row, pos] = -k[l][row, pos]

    def forward_device(self, input_ids, images, plan, validate=True, last_only=False, cache=None, **kw):
        assert last_only and cache is not None and cache.B == 1
        L = input_ids.shape[1]
        cache.start(L, None, input_ids)
        self._write(cache.k, cache.v, 0, slice(0, L), input_ids[0])
        self.calls.append(('prefill', input_ids[0].tolist(), images is not None, plan))
        return self._logits(input_ids[:, -1])

    def extend(self, cache, input_ids, images, bboxes, attention_mask=None, last_only=True):
        assert cache.rows is not None and attention_mask is not None
        rows, starts, lens = cache.rows.tolist(), cache.lens.tolist(), attention_mask.sum(1).tolist()
        tails = [input_ids[b, :n].tolist() for b, n in enumerate(lens)]
        self.calls.append(('extend', rows, starts, tails, images is not None,
                           [None if b is None else b.tolist() for b in bboxes],
                           ([t.clone() for t in cache.k], [t.clone() for t in cache.v])))
        for t, b in zip(tails, bboxes):
            if t.count(BOX) != (0 if b is None else b.shape[0]):
                raise RuntimeError('gpt4roi_b200 C-ABI error 3: <bbox> count')
        for i, (r, p, t) in enumerate(zip(rows, starts, tails)):
            assert p + len(t) <= cache.max_len
            self._write(cache.k, cache.v, r, slice(p, p + len(t)), torch.tensor(t))
        return self._logits(torch.tensor([t[-1] for t in tails]))

    def decode_step(self, ids, cache, pos_dev=None):
        """Writes every row's fed token at its length, idle rows too, as the graphed step does."""
        self.calls.append(('decode', cache.lens.tolist()))
        for r, p in enumerate(cache.lens.tolist()):
            self._write(cache.k, cache.v, r, slice(p, p + 1), ids[r])
        return self._logits(ids[:, 0])

    def kinds(self):
        return [c[0] for c in self.calls]


def _ids(*parts):
    return torch.tensor([sum((list(p) for p in parts), [])])


def _held(b, s):
    """The ids row s of the batcher's cache holds at positions 0.. (read from layer 0's K), as far as the record says."""
    n = b.row_record(s).shape[0]
    return b.cache.k[0][s, :n, 0].to(torch.int64).tolist()


IMG = [IMS] + [IMP] * 4 + [IME]
BOXES = [torch.tensor([[0.1, 0.1, 0.4, 0.4]]), torch.tensor([[0.2, 0.3, 0.6, 0.9]])]


def _image(seed):
    return torch.rand(1, 3, 28, 28, generator=torch.Generator().manual_seed(seed))


def test_row_record_after_admission_while_running_and_after_retirement():
    eng = _Stub()
    b = ContinuousBatcher(eng, slots=2, max_len=32, prefix_reuse=True)
    assert b.row_record(0).tolist() == [] and b.row_record(1).tolist() == []
    r = b.submit(_ids([1, 2, 3]), max_new_tokens=4)
    b.step()     # admitted (first token 4, K/V unwritten), then one decode step: token 4 written, 5 emitted
    assert r.tokens == [4, 5]
    assert b.row_record(0).tolist() == [1, 2, 3, 4] == _held(b, 0)
    b.run()
    assert r.tokens == [4, 5, 6, 7] and r.done
    assert b.row_record(0).tolist() == [1, 2, 3, 4, 5, 6] == _held(b, 0)     # the last token's K/V never written
    # a request done at admission: the record is its prompt
    one = b.submit(_ids([50, 51]), max_new_tokens=1)
    b.step()
    assert one.done and b.row_record(1).tolist() == [50, 51] == _held(b, 1)


def test_follow_up_turn_reuses_the_free_row_that_holds_the_conversation():
    eng = _Stub()
    b = ContinuousBatcher(eng, slots=3, max_len=40, prefix_reuse=True)
    img = _image(0)
    t1 = b.submit(_ids([1], IMG, [10, 11]), images=img, max_new_tokens=3)
    b.run()
    s1 = 0
    conv = b.row_record(s1).tolist()
    assert conv == [1] + IMG + [10, 11, 12, 13]
    eng.calls.clear()
    t2 = b.submit(_ids(conv, [14, 20, 21]), images=img.clone(), max_new_tokens=3)
    b.step()
    assert b.running[s1] is t2 and t2.reused == len(conv)
    ext = [c for c in eng.calls if c[0] == 'extend']
    assert eng.kinds()[0] == 'extend' and 'prefill' not in eng.kinds()
    assert ext[0][1:4] == ([s1], [len(conv)], [[14, 20, 21]])
    b.run()
    assert t2.sequences[0, -3:].tolist() == [22, 23, 24]
    assert t1.reused == 0 and _held(b, s1) == b.row_record(s1).tolist() == conv + [14, 20, 21, 22, 23]


def test_free_holder_wins_running_holder_copied_only_when_strictly_longer():
    eng = _Stub()
    b = ContinuousBatcher(eng, slots=3, max_len=40, prefix_reuse=True)
    img = _image(1)
    base = [1] + IMG + [10, 11, 12]
    a = b.submit(_ids(base, [40]), images=img, max_new_tokens=1)            # row 0, retires at admission
    run = b.submit(_ids(base, [50, 51]), images=img, max_new_tokens=20)      # row 1, keeps running
    b.step()
    assert a.done and b.running[1] is run
    # free row 0 holds base + [40], running row 1 holds base + [50, 51, ...]: both give len(base) -> the free row wins
    eng.calls.clear()
    c = b.submit(_ids(base, [60]), images=img, max_new_tokens=20)
    b.step()
    assert b.running[0] is c and c.reused == len(base)
    assert [x[1:3] for x in eng.calls if x[0] == 'extend'] == [([0], [len(base)])]
    # now the only free row (2) holds nothing; running row 1 holds base + [50, 51]: a strictly longer prefix -> copied
    eng.calls.clear()
    d = b.submit(_ids(base, [50, 51, 70]), images=img, max_new_tokens=3)
    b.step()
    assert b.running[2] is d and d.reused == len(base) + 2
    ext = [x for x in eng.calls if x[0] == 'extend']
    assert [x[1:4] for x in ext] == [([2], [len(base) + 2], [[70]])]


def test_copy_moves_exactly_the_prefix_of_every_layer():
    eng = _Stub()
    b = ContinuousBatcher(eng, slots=3, max_len=24, prefix_reuse=True)
    img = _image(2)
    donor = b.submit(_ids([1], IMG, [10, 11, 12, 13]), images=img, max_new_tokens=10)
    b.step()
    old = b.submit(_ids([7, 8, 9]), max_new_tokens=1)                          # row 1 holds something else
    b.step()
    assert old.done and b.running[0] is donor
    before = ([t.clone() for t in b.cache.k], [t.clone() for t in b.cache.v])
    # row 1 was retired later than row 2 was never used: the copy goes to row 2 (fresh rows first)
    p = 1 + len(IMG) + 3
    r = b.submit(_ids([1], IMG, [10, 11, 12, 99]), images=img, max_new_tokens=4)
    b.step()
    assert b.running[2] is r and r.reused == p
    seen = next(c for c in eng.calls if c[0] == 'extend')[6]     # the cache as the chunk prefill found it
    for before_l, seen_l in zip(before[0] + before[1], seen[0] + seen[1]):
        changed = (before_l != seen_l).any(-1)
        want = torch.zeros_like(changed)
        want[2, :p] = True
        assert torch.equal(changed, want)
        assert torch.equal(seen_l[2, :p], before_l[0, :p])


def test_reuse_refused_for_another_image_a_changed_box_and_an_uncovered_image_span():
    eng = _Stub()
    b = ContinuousBatcher(eng, slots=2, max_len=40, prefix_reuse=True)
    img = _image(3)
    first = _ids([1], IMG, [10, BOX, 11, 12])
    b.submit(first, images=img, bboxes=[BOXES[0]], max_new_tokens=1)
    b.run()
    eng.calls.clear()
    # another image: nothing reusable -> full prefill (into the never-used row 1)
    r = b.submit(_ids(first[0].tolist(), [13]), images=_image(4), bboxes=[BOXES[0]], max_new_tokens=1)
    b.run()
    assert r.reused == 0 and eng.kinds() == ['prefill']
    # a changed box: the prefix is cut at that <bbox>, which still covers the image span
    b = ContinuousBatcher(eng, slots=1, max_len=40, prefix_reuse=True)
    b.submit(first, images=img, bboxes=[BOXES[0]], max_new_tokens=1)
    b.run()
    r = b.submit(_ids(first[0].tolist(), [13]), images=img, bboxes=[BOXES[1]], max_new_tokens=1)
    b.run()
    cut = 1 + len(IMG) + 1
    assert r.reused == cut
    assert eng.calls[-1][0] == 'extend' and eng.calls[-1][3] == [[BOX, 11, 12, 13]]
    assert eng.calls[-1][5] == [BOXES[1].tolist()]
    # a prompt whose image span starts after the common prefix: reuse would need image tokens in the chunk
    b = ContinuousBatcher(eng, slots=1, max_len=40, prefix_reuse=True)
    b.submit(_ids([1, 2, 3, 4], IMG, [5]), images=img, max_new_tokens=1)
    b.run()
    eng.calls.clear()
    r = b.submit(_ids([1, 2, 3, 9], IMG, [5]), images=img, max_new_tokens=1)
    b.run()
    assert r.reused == 0 and eng.kinds() == ['prefill']


def test_empty_rows_first_then_least_recently_retired():
    eng = _Stub()
    b = ContinuousBatcher(eng, slots=3, max_len=16, prefix_reuse=True)
    order = []
    for first in (20, 30, 40):            # no prefix in common: each takes a row that never held anything, in order
        r = b.submit(_ids([first, first + 1]), max_new_tokens=1)
        b.step()
        order.append(b.row_record(0).tolist() == [first, first + 1])
    assert [b.row_record(s).tolist() for s in range(3)] == [[20, 21], [30, 31], [40, 41]]
    # rows retired in the order 0, 1, 2 -- the next unmatched request takes row 0, then 1
    long1 = b.submit(_ids([60, 61]), max_new_tokens=5)
    b.step()
    assert b.running[0] is long1
    long2 = b.submit(_ids([70, 71]), max_new_tokens=5)
    b.step()
    assert b.running[1] is long2
    # a request that matches row 2 (free, holding [40, 41]) goes there in place
    m = b.submit(_ids([40, 41, 42]), max_new_tokens=5)
    b.step()
    assert b.running[2] is m and m.reused == 2


def test_one_chunk_prefill_per_round_with_each_rows_start_and_tail():
    eng = _Stub()
    b = ContinuousBatcher(eng, slots=4, max_len=40, prefix_reuse=True)
    convs = [[1, 2, 3], [5, 6, 7, 8, 9], [11, 12], [15, 16, 17, 18]]
    for c in convs:
        b.submit(_ids(c), max_new_tokens=2)
    b.run()
    held = [b.row_record(s).tolist() for s in range(4)]
    assert held == [c + [c[-1] + 1] for c in convs]
    eng.calls.clear()
    tails = [[30], [40, 41, 42], [50, 51], [60]]
    order = [2, 0, 3]            # three follow-ups, submitted in this order, plus one fresh prompt
    reqs = [b.submit(_ids(held[s], tails[s]), max_new_tokens=3) for s in order]
    fresh = b.submit(_ids([90, 91, 92]), max_new_tokens=3)
    b.step()
    ext = [c for c in eng.calls if c[0] == 'extend']
    assert len(ext) == 1 and eng.kinds().index('prefill') < eng.kinds().index('extend')   # full prefills first
    assert ext[0][1:4] == (order, [len(held[s]) for s in order], [tails[s] for s in order])
    assert b.running[1] is fresh and [b.running[s] for s in order] == reqs
    assert [r.reused for r in reqs] == [len(held[s]) for s in order] and fresh.reused == 0
    b.run()
    for s, r in zip(order, reqs):
        t = tails[s][-1]
        assert r.sequences[0].tolist() == held[s] + tails[s] + [t + 1, t + 2, t + 3]
        assert _held(b, s) == held[s] + tails[s] + [t + 1, t + 2]


def test_a_donor_prefilled_earlier_in_the_same_round():
    eng = _Stub()
    b = ContinuousBatcher(eng, slots=2, max_len=40, prefix_reuse=True)
    img = _image(5)
    a = b.submit(_ids([1], IMG, [10, 11]), images=img, max_new_tokens=4)
    q = b.submit(_ids([1], IMG, [10, 12]), images=img, max_new_tokens=4)
    b.step()
    assert eng.kinds()[:2] == ['prefill', 'extend']
    ext = eng.calls[1]
    assert ext[1:4] == ([1], [1 + len(IMG) + 1], [[12]])
    assert b.running == [a, q] and q.reused == 1 + len(IMG) + 1


def test_a_bad_request_in_a_round_errs_alone_and_leaves_no_active_row():
    eng = _Stub()
    b = ContinuousBatcher(eng, slots=3, max_len=40, prefix_reuse=True)
    img = _image(6)
    for c in ([1], [2], [3]):          # each conversation holds one <bbox>
        b.submit(_ids(c, IMG, [BOX, 10]), images=img, bboxes=[BOXES[0]], max_new_tokens=1)
    b.run()
    eng.calls.clear()
    held = [b.row_record(s).tolist() for s in range(3)]
    good0 = b.submit(_ids(held[0], [20]), images=img, bboxes=[BOXES[0]], max_new_tokens=3)
    bad = b.submit(_ids(held[1], [BOX, 21]), images=img, bboxes=[BOXES[0]], max_new_tokens=3)   # no box for it
    good2 = b.submit(_ids(held[2], [22]), images=img, bboxes=[BOXES[0]], max_new_tokens=3)
    with pytest.raises(RuntimeError, match='<bbox> count'):
        b.step()
    ext = [c[1] for c in eng.calls if c[0] == 'extend']
    assert ext == [[0, 1, 2], [0], [1], [2]]          # the round, then each request alone
    assert bad.done and bad.error is not None and bad.tokens == []
    assert b.running[1] is None and b.active.tolist() == [1, 0, 1]
    assert b.row_record(1).tolist() == held[1]        # the row keeps the prefix it held
    b.run()
    assert good0.sequences[0].tolist() == held[0] + [20, 21, 22, 23] and good0.error is None
    assert good2.sequences[0].tolist() == held[2] + [22, 23, 24, 25] and good2.error is None
    assert b.active.tolist() == [0, 0, 0]


def _default_trace(**kw):
    """The engine calls, the rows' device state after every step, the answers and the cache of one traffic pattern."""
    eng = _Stub()
    b = ContinuousBatcher(eng, slots=2, max_len=32, **kw)
    reqs, state = [], []
    for p, n in (([1, 2], 3), ([1, 2, 3], 2), ([1, 2], 4), ([5], 1), ([1, 2, 3, 4], 2), ([1, 2, 3, 4, 6], 3)):
        reqs.append(b.submit(torch.tensor([p]), max_new_tokens=n))
        b.step()
        state.append([t.tolist() for t in (b.cache.lens, b.active, b.finished, b.step_count, b.ids)])
    while b.queue or any(r is not None for r in b.running):
        b.step()
        state.append([t.tolist() for t in (b.cache.lens, b.active, b.finished, b.step_count, b.ids)])
    calls = [[c[0], c[1]] + ([c[2]] if c[0] == 'prefill' else []) for c in eng.calls]
    return calls, state, [r.sequences.tolist() for r in reqs], b.cache.k[0][:, :, 0].tolist()


# _default_trace() as the batcher before prefix reuse existed (the parent of this change) gives it
_BEFORE = ([['prefill', [1, 2], False], ['decode', [2, 0]], ['prefill', [1, 2, 3], False], ['decode', [3, 3]],
            ['prefill', [1, 2], False], ['decode', [2, 4]], ['prefill', [5], False], ['decode', [3, 1]],
            ['prefill', [1, 2, 3, 4], False], ['decode', [4, 4]], ['prefill', [1, 2, 3, 4, 6], False], ['decode', [5, 5]],
            ['decode', [6, 5]]],
           [[[3, 0], [1, 0], [0, 0], [2, 0], [[4], [0]]], [[4, 4], [0, 0], [0, 0], [3, 2], [[5], [5]]],
            [[3, 4], [1, 0], [0, 0], [2, 2], [[4], [5]]], [[4, 1], [1, 0], [0, 0], [3, 1], [[5], [6]]],
            [[5, 5], [0, 0], [0, 0], [4, 2], [[6], [6]]], [[6, 5], [1, 0], [0, 0], [2, 2], [[8], [6]]],
            [[7, 5], [0, 0], [0, 0], [3, 2], [[9], [6]]]],
           [[[1, 2, 3, 4, 5]], [[1, 2, 3, 4, 5]], [[1, 2, 3, 4, 5, 6]], [[5, 6]], [[1, 2, 3, 4, 5, 6]],
            [[1, 2, 3, 4, 6, 7, 8, 9]]],
           [[1.0, 2.0, 3.0, 4.0, 6.0, 7.0, 8.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0,
             0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0],
            [1.0, 2.0, 3.0, 4.0, 5.0, 6.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0,
             0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0]])


def test_default_makes_exactly_the_calls_of_the_batcher_without_reuse():
    calls, state, seqs, k = _default_trace()
    assert (calls, state, seqs, k) == _BEFORE
    assert _default_trace(prefix_reuse=False) == _BEFORE
    assert 'extend' not in [c[0] for c in calls]
    assert _default_trace(prefix_reuse=True)[0] != calls      # the same traffic does reuse prefixes when asked


def test_reuse_needs_the_chunk_prefill():
    from tests.test_serve_cpu import _StubEngine
    with pytest.raises(NotImplementedError, match='head_dim 128'):
        ContinuousBatcher(_StubEngine(), slots=1, max_len=8, prefix_reuse=True)


def test_seam_passes_the_flag():
    from tests.test_model_seam_cpu import _tiny_model
    m = _tiny_model().eval()
    m._get_engine = lambda device: _Stub()
    assert m.continuous_batcher(slots=2, max_len=16).batcher.prefix_reuse is False
    sb = m.continuous_batcher(slots=2, max_len=16, prefix_reuse=True)
    assert sb.batcher.prefix_reuse is True
    r = sb.submit(torch.tensor([[1, 2]]), max_new_tokens=2)
    sb.run()
    r2 = sb.submit(torch.tensor([[1, 2, 3, 7]]), max_new_tokens=2)
    sb.run()
    assert r.reused == 0 and r2.reused == 3 and r2.sequences.tolist() == [[1, 2, 3, 7, 8, 9]]
