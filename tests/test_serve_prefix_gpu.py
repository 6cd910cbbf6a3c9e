"""GPU tests of prefix reuse in continuous batching: the cache-row-table kernels (kv_append / attention_cached with
cache_rows=) against the contiguous ones, and ContinuousBatcher(prefix_reuse=True) on the real engine -- without a match
it gives the tokens of the batcher without reuse; a follow-up turn and a question on a running request's image give what
generate(cache=) gives on the same conversation; its neighbours are untouched; a batched round gives each request's
alone-tokens; a bad request in a round errs alone; the model seam equals model.generate(past_key_values=)."""
import pytest
import torch

from gpt4roi_b200 import kernels
from gpt4roi_b200.engine import ContinuousBatcher, EngineConfig, KVCache, PrefillEngine, random_state_dicts
from tests.test_engine_gpu import make_inputs
from tests.test_serve_gpu import _request, _tokens

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
I32 = torch.int32
SLOTS, MAX_LEN = 4, 384     # the batcher equals generate() alone bitwise here (tests/test_serve_gpu.py)


# ---- the row-table kernels -------------------------------------------------------------------------------------------

@pytest.mark.parametrize('dt', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('D', [64, 128])
def test_row_table_kernels_equal_the_contiguous_ones(D, dt):
    """Chunk rows 0, 1, 2 continue cache rows 4, 1, 3 of a 5-row cache (permuted; the last one the cache's last row),
    two of them ending exactly at max_len, one with a 128-row tile wholly past its queries."""
    H = 32 if D == 128 else 16
    HD, S, lmax, Lc = H * D, 5, 400, 150
    torch.manual_seed(D)
    rows = torch.tensor([4, 1, 3], dtype=I32)
    qlen = torch.tensor([20, 150, 5], dtype=I32)
    start = torch.tensor([lmax - 20, 100, lmax - 5], dtype=I32)
    B = rows.shape[0]
    qkv = torch.randn(B * Lc, 3 * HD, device=DEV).to(dt)
    big_k = torch.randn(S, lmax, HD, device=DEV).to(dt)          # finite sentinels everywhere
    big_v = torch.randn(S, lmax, HD, device=DEV).to(dt)
    k0, v0 = big_k.clone(), big_v.clone()
    r, st, ql = rows.to(DEV), start.to(DEV), qlen.to(DEV)
    kernels.kv_append(qkv, big_k, big_v, B, Lc, 0, pos_rows=st, cache_rows=r, qlen=ql)
    changed = ((big_k != k0) | (big_v != v0)).any(-1).cpu()
    allowed = torch.zeros(S, lmax, dtype=torch.bool)
    for b in range(B):
        allowed[rows[b], start[b]:start[b] + qlen[b]] = True
    assert not bool((changed & ~allowed).any())
    for b in range(B):   # the valid rows hold the chunk's k / v
        s0, n = int(start[b]), int(qlen[b])
        assert torch.equal(big_k[rows[b], s0:s0 + n], qkv.view(B, Lc, -1)[b, :n, HD:2 * HD])
        assert torch.equal(big_v[rows[b], s0:s0 + n], qkv.view(B, Lc, -1)[b, :n, 2 * HD:])
    # the contiguous cache holding the same rows (room for the padding rows the contiguous append writes)
    ck = torch.zeros(B, lmax + Lc, HD, device=DEV, dtype=dt)
    cv = torch.zeros_like(ck)
    ck[:, :lmax], cv[:, :lmax] = k0[rows.long()], v0[rows.long()]
    kernels.kv_append(qkv, ck, cv, B, Lc, 0, pos_rows=st)
    for b in range(B):
        s0, n = int(start[b]), int(qlen[b])
        assert torch.equal(ck[b, :s0 + n], big_k[rows[b], :s0 + n])
    scale = D ** -0.5
    want = kernels.attention_cached(qkv, ck, cv, B, H, D, Lc, scale, st, ql)
    got = kernels.attention_cached(qkv, big_k, big_v, B, H, D, Lc, scale, st, ql, cache_rows=r)
    assert torch.equal(got, want)
    assert bool((got.view(B, Lc, -1)[2, 128:] == 0).all())     # row 2's second tile lies wholly past its 5 queries


# ---- the batcher -----------------------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def eng():
    cfg = EngineConfig(image_size=224, vit_layers=12, n_layers=2)
    sd, vit_sd = random_state_dicts(cfg, DEV, seed=61)
    return PrefillEngine(cfg, sd, vit_sd, DEV)


def _question(n, seed, box_at=None, cfg=None):
    q = torch.randint(3, 32000, (1, n), generator=torch.Generator().manual_seed(seed))
    if box_at is not None:
        q[0, box_at] = cfg.bbox_token
    return q


def _new_box(seed):
    return torch.tensor([[0.15, 0.2, 0.55, 0.7]]) + 0.01 * (seed % 5)


def _turn1(eng, seed, n=10, T=20, k=1):
    ids, images, boxes = make_inputs(eng.cfg, 1, [k], T, seed=seed)
    return dict(input_ids=ids, images=images.to(torch.bfloat16), bboxes=boxes, max_new_tokens=n)


def _gen(eng, spec, cache):
    out = eng.generate(spec['input_ids'].to(DEV), spec['images'], spec['bboxes'], max_new_tokens=spec['max_new_tokens'],
                       cache=cache)
    return out[0, spec['input_ids'].shape[1]:].cpu()


def _turn2(eng, spec1, seq1, case, seed):
    """The follow-up of a conversation whose turn 1 gave seq1 (prompt + answer, host [1, L])."""
    cfg = eng.cfg
    boxes = [b.clone() for b in spec1['bboxes']]
    seq = seq1.clone()
    if case == 'retokenized':          # the re-encoded answer differs two tokens before its end
        seq[0, -2] = (seq[0, -2] + 1) % 32000
    q = _question(48, seed, box_at=10 if case == 'box' else None, cfg=cfg)
    if case == 'box':
        boxes = [torch.cat([boxes[0], _new_box(seed)])]
    return dict(input_ids=torch.cat([seq, q], 1), images=spec1['images'], bboxes=boxes, max_new_tokens=10)


@pytest.mark.parametrize('case', ['text', 'box', 'retokenized'])
def test_follow_up_turn_equals_generate_with_the_conversation_cache(eng, case):
    spec1 = _turn1(eng, 300)
    b = ContinuousBatcher(eng, SLOTS, MAX_LEN, prefix_reuse=True)
    r1 = b.submit(**spec1)
    b.run()
    c = KVCache(eng.cfg, 1, MAX_LEN, DEV)
    assert torch.equal(_tokens(r1), _gen(eng, spec1, c))
    spec2 = _turn2(eng, spec1, r1.sequences, case, 301)
    reuse = int(c.reusable(spec2['input_ids'], spec2['images'], spec2['bboxes'])[0])
    r2 = b.submit(**spec2)
    b.run()
    assert r2.reused == reuse > eng.cfg.num_patches
    assert torch.equal(_tokens(r2), _gen(eng, spec2, c)), (case, _tokens(r2))


def test_no_match_gives_the_tokens_of_the_batcher_without_reuse(eng):
    specs = [_request(eng, i, 8 + 3 * i, i % 2 == 1) for i in range(6)]    # each its own image

    def run(reuse):
        b = ContinuousBatcher(eng, SLOTS, MAX_LEN, prefix_reuse=reuse)
        reqs = []
        for i, spec in enumerate(specs):
            if spec.get('do_sample'):
                torch.manual_seed(100 + i)
            reqs.append(b.submit(**spec))
            if i % 2:
                b.step()
        b.run()
        return reqs
    plain, reused = run(False), run(True)
    for p, r in zip(plain, reused):
        assert r.reused == 0 and torch.equal(_tokens(r), _tokens(p))


def test_question_on_a_running_requests_image_copies_its_prefix(eng):
    """A runs; B asks another question on A's image with A's system prompt: B takes a fresh row into which A's prefix
    is copied, and gives generate(B, cache=c) where c holds A's prompt."""
    a = _turn1(eng, 310, n=40)
    La = a['input_ids'].shape[1]
    keep = eng.cfg.num_patches + 3 + 4        # system token, image span, four more prompt tokens
    ids = torch.cat([a['input_ids'][:, :keep], _question(48, 311)], 1)
    box_kept = bool((ids == eng.cfg.bbox_token).any())
    bsp = dict(input_ids=ids, images=a['images'], bboxes=a['bboxes'] if box_kept else None, max_new_tokens=12)
    b = ContinuousBatcher(eng, SLOTS, MAX_LEN, prefix_reuse=True)
    ra = b.submit(**a)
    b.step()
    b.step()
    rb = b.submit(**bsp)
    b.step()
    assert b.running[0] is ra and b.running[1] is rb
    b.run()
    c = KVCache(eng.cfg, 1, MAX_LEN, DEV)
    _gen(eng, dict(a, max_new_tokens=1), c)     # c holds A's prompt
    reuse = int(c.reusable(bsp['input_ids'], bsp['images'], bsp['bboxes'])[0])
    assert rb.reused == reuse >= keep and La > keep
    assert torch.equal(_tokens(rb), _gen(eng, bsp, c))
    assert torch.equal(_tokens(ra), _gen(eng, a, KVCache(eng.cfg, 1, MAX_LEN, DEV)))


def test_neighbours_of_a_reuse_admission_keep_their_tokens(eng):
    spec1 = _turn1(eng, 320)
    others = [_request(eng, 1 + j, 30, j % 2 == 1) for j in range(2)]

    def run(with_reuse):
        b = ContinuousBatcher(eng, SLOTS, MAX_LEN, prefix_reuse=True)
        r1 = b.submit(**spec1)
        b.run()
        reqs = []
        for j, o in enumerate(others):
            if o.get('do_sample'):
                torch.manual_seed(200 + j)
            reqs.append(b.submit(**o))
        b.step()
        b.step()
        if with_reuse:
            r2 = b.submit(**_turn2(eng, spec1, r1.sequences, 'box', 321))
            b.step()
            assert r2.reused > 0
        b.run()
        return [_tokens(r) for r in reqs]
    for x, y in zip(run(False), run(True)):
        assert torch.equal(x, y)


def _conversations(eng, b, n):
    specs = [_turn1(eng, 330 + i, n=6 + i) for i in range(n)]
    reqs = [b.submit(**s) for s in specs]
    b.run()
    return specs, reqs


def test_batched_round_of_text_follow_ups_equals_each_alone(eng):
    """Three text-only follow-ups admitted in one step go through one chunk prefill at batch 3 (Lc = the longest tail):
    only LLaMA layers run on the tails, whose GEMM rows and attention rows are computed independently of the other rows
    of the batch, so each request gets the tokens it gets when admitted alone."""
    b = ContinuousBatcher(eng, SLOTS, MAX_LEN, prefix_reuse=True)
    specs, reqs = _conversations(eng, b, 3)
    follow = [_turn2(eng, s, r.sequences, 'text', 340 + i) for i, (s, r) in enumerate(zip(specs, reqs))]
    for i, f in enumerate(follow):                # tails of different lengths
        f['input_ids'] = f['input_ids'][:, :f['input_ids'].shape[1] - 7 * i]
    calls = []
    real = eng.extend
    eng.extend = lambda cache, ids, *a, **k: calls.append(tuple(ids.shape)) or real(cache, ids, *a, **k)
    try:
        got = [b.submit(**f) for f in follow]
        b.run()
    finally:
        eng.extend = real
    assert len(calls) == 1 and calls[0][0] == 3
    for s, f, r in zip(specs, follow, got):
        b1 = ContinuousBatcher(eng, SLOTS, MAX_LEN, prefix_reuse=True)
        first = b1.submit(**s)
        b1.run()
        alone = b1.submit(**f)
        b1.run()
        assert alone.reused == r.reused > 0
        assert torch.equal(_tokens(r), _tokens(alone))


def test_batched_round_with_new_boxes_equals_the_batch_extend_on_a_contiguous_cache(eng):
    """Tails with new boxes rerun ViT + fuse at batch k.  The fuse stack's GroupNorm statistics are summed per image
    (dense.gn_slots partial sums per (image, slot)), so batch size does not reorder them, but the conv and linear GEMMs
    of the ViT run other tile shapes at another M: the first-token logits are compared with PrefillEngine.extend at
    batch k on a contiguous cache holding the same rows, bitwise."""
    b = ContinuousBatcher(eng, SLOTS, MAX_LEN, prefix_reuse=True)
    specs, reqs = _conversations(eng, b, 2)
    follow = [_turn2(eng, s, r.sequences, 'box', 350 + i) for i, (s, r) in enumerate(zip(specs, reqs))]
    rows = [0, 1]                                  # the conversations' rows, free again
    snap = ([t[:2].clone() for t in b.cache.k], [t[:2].clone() for t in b.cache.v])
    seen = []
    real = eng.extend

    def record(cache, ids, images, bboxes, attention_mask=None, **k):
        out = real(cache, ids, images, bboxes, attention_mask=attention_mask, **k)
        seen.append((cache.rows.tolist(), ids.clone(), None if images is None else images.clone(),
                     [None if x is None else x.clone() for x in bboxes], attention_mask.clone(), out.clone()))
        return out
    eng.extend = record
    try:
        got = [b.submit(**f) for f in follow]
        b.step()
    finally:
        eng.extend = real
    assert len(seen) == 1 and seen[0][0] == rows
    _, ids, images, boxes, mask, logits = seen[0]
    c = KVCache(eng.cfg, 2, MAX_LEN, DEV, kv=([t.clone() for t in snap[0]], [t.clone() for t in snap[1]]))
    c.lens = torch.tensor([r.reused for r in got], dtype=I32, device=DEV)
    c.length = int(c.lens.max())
    c.source_known = True
    want = eng.extend(c, ids, images, boxes, attention_mask=mask)
    assert torch.equal(logits, want)


def test_bad_request_in_a_round_errs_alone(eng):
    b = ContinuousBatcher(eng, SLOTS, MAX_LEN, prefix_reuse=True)
    specs, reqs = _conversations(eng, b, 3)
    follow = [_turn2(eng, s, r.sequences, 'text', 360 + i) for i, (s, r) in enumerate(zip(specs, reqs))]
    follow[1]['input_ids'][0, -5] = eng.cfg.bbox_token        # a <bbox> without its box
    got = [b.submit(**f) for f in follow]
    with pytest.raises(ValueError, match='<bbox>'):
        b.step()
    assert got[1].done and got[1].error is not None and got[1].tokens == []
    assert b.running[1] is None and int(b.active[1]) == 0
    b.run()
    assert int(b.active.sum()) == 0
    for i in (0, 2):
        b1 = ContinuousBatcher(eng, SLOTS, MAX_LEN, prefix_reuse=True)
        b1.submit(**specs[i])
        b1.run()
        alone = b1.submit(**follow[i])
        b1.run()
        assert got[i].error is None and torch.equal(_tokens(got[i]), _tokens(alone))


def test_seam_two_turns_equal_model_generate_with_a_dynamic_cache():
    from transformers import DynamicCache
    from tests.test_model_seam_gpu import build_seam_model
    cfg = EngineConfig(image_size=224, vit_layers=24, n_layers=2)
    sd, vit_sd = random_state_dicts(cfg, DEV, seed=47)
    model = build_seam_model(cfg, sd, vit_sd, dtype=torch.float16).eval()
    ids1, images, boxes = make_inputs(cfg, 1, [2], 24, seed=9)
    img, bx = images.half().to(DEV), [x.half().to(DEV) for x in boxes]
    n1, n2 = 8, 8
    q = _question(48, 371)
    with torch.inference_mode():
        cache = DynamicCache()
        out1 = model.generate(ids1.to(DEV), images=img, bboxes=bx, max_new_tokens=n1, past_key_values=cache).cpu()
        ids2 = torch.cat([out1, q], 1)
        out2 = model.generate(ids2.to(DEV), images=img, bboxes=bx, max_new_tokens=n2, past_key_values=cache).cpu()
    # the decode attention splits its keys as generate()'s cache does: max_len within the same power-of-two band
    sb = model.continuous_batcher(slots=4, max_len=ids2.shape[1] + n2, prefix_reuse=True)
    r1 = sb.submit(ids1, images=img, bboxes=bx, max_new_tokens=n1)
    sb.run()
    assert torch.equal(r1.sequences, out1)
    r2 = sb.submit(ids2, images=img, bboxes=bx, max_new_tokens=n2)
    sb.run()
    assert r2.reused == out1.shape[1] - 1
    assert torch.equal(r2.sequences, out2)


def test_batched_round_past_the_rope_table_equals_each_alone(eng, monkeypatch):
    """max_len 1024, where max_len alone sizes a 1024-row RoPE table: a follow-up holding 1000 tokens with an 11-token
    tail shares its round with one whose tail has 49 tokens, so the chunk is 49 rows and the first row's padding rows sit
    at positions up to 1048.  The fused QKV-RoPE epilogue rotates those rows too: the table must cover every position it
    reads, and each request gets the tokens it gets when admitted alone."""
    from gpt4roi_b200 import dense
    max_len = 1024
    long1 = _turn1(eng, 380, n=8, T=735)            # 993 prompt tokens, then 8 new: the row holds 1000
    short1 = _turn1(eng, 381, n=8)

    def follow(spec1, seq, n, seed):
        return dict(input_ids=torch.cat([seq, _question(n, seed)], 1), images=spec1['images'], bboxes=spec1['bboxes'],
                    max_new_tokens=5)

    def turn2(specs, together):
        b = ContinuousBatcher(eng, SLOTS, max_len, prefix_reuse=True)
        first = [b.submit(**s) for s in specs]
        b.run()
        ups = [follow(s, r.sequences, n, 382 + i) for i, (s, r, n) in enumerate(zip(specs, first, (10, 48)))]
        if together:
            got = [b.submit(**u) for u in ups]
            b.run()
            return got
        got = []
        for u in ups:
            got.append(b.submit(**u))
            b.run()
        return got
    seen = []
    real = dense.qkv_rope

    def spy(h, w, cos, sin, L, *a, pos_rows=None, **k):
        if pos_rows is not None and h.shape[0] > pos_rows.shape[0]:     # a chunk, not a decode step
            seen.append((cos.shape[0], int(pos_rows.max()) + L))
        return real(h, w, cos, sin, L, *a, pos_rows=pos_rows, **k)
    monkeypatch.setattr(dense, 'qkv_rope', spy)
    together = turn2([long1, short1], True)
    assert together[0].reused == 1000 and together[1].reused > 0
    assert seen and max(n for _, n in seen) > 1024
    assert all(n <= rows for rows, n in seen), seen
    alone = turn2([long1, short1], False)
    for t, a in zip(together, alone):
        assert t.reused == a.reused and torch.equal(_tokens(t), _tokens(a))
