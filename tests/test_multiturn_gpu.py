"""Multi-turn generation: the chunk attention over the KV cache (kernels.attention_cached), the continuation splice,
PrefillEngine.extend / prefill_cached, generate(cache=) and past_key_values reuse through the model seam.  Every turn
must give what the no-cache path gives for the same full prompt."""
import pytest
import torch

from gpt4roi_b200 import kernels
from gpt4roi_b200.engine import EngineConfig, GraphedDecode, KVCache, PrefillEngine, random_state_dicts
from gpt4roi_b200.splice import splice_region_tokens
from tests.test_engine_gpu import make_inputs, rel

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
BF = torch.bfloat16
I32 = torch.int32

_STARTS = [0, 1, 63, 64, 65, 700, 2000]
_QLENS = [1, 17, 128, 129, 300]


def _cached_ref(qkv, kc, vc, start, qlen, B, Lc, H, D, scale):
    """Per-row fp32 causal attention of the chunk over cache rows 0..start+i, probabilities rounded to the storage
    type before P.V (as test_ragged_decode_gpu._attn_ref)."""
    HD = H * D
    out = []
    for b in range(B):
        s, n = int(start[b]), int(qlen[b])
        q = qkv.view(B, Lc, -1)[b, :n, :HD].float().view(n, H, D).permute(1, 0, 2)
        k = kc[b, :s + n].float().view(s + n, H, D).permute(1, 0, 2)
        v = vc[b, :s + n].float().view(s + n, H, D).permute(1, 0, 2)
        sc = q @ k.transpose(-1, -2) * scale
        mask = torch.arange(s + n, device=DEV)[None] > (s + torch.arange(n, device=DEV))[:, None]
        p = torch.softmax(sc.masked_fill(mask, float('-inf')), -1).to(qkv.dtype).float()
        out.append((p @ v).permute(1, 0, 2).reshape(n, HD))
    return out


def _chunk_case(B, D, H, seed, dtype=BF):
    torch.manual_seed(seed)
    start = torch.tensor([_STARTS[(b + seed) % len(_STARTS)] for b in range(B)], dtype=I32)
    qlen = torch.tensor([_QLENS[(3 * b + seed) % len(_QLENS)] for b in range(B)], dtype=I32)
    Lc = int(qlen.max())
    HD = H * D
    Lmax = int((start + Lc).max()) + 70
    qkv = torch.randn(B * Lc, 3 * HD, device=DEV).to(dtype)
    kc = torch.zeros(B, Lmax, HD, device=DEV, dtype=dtype)
    vc = torch.zeros_like(kc)
    for b in range(B):   # the cached prefix
        s = int(start[b])
        kc[b, :s] = torch.randn(s, HD, device=DEV).to(dtype)
        vc[b, :s] = torch.randn(s, HD, device=DEV).to(dtype)
    kernels.kv_append(qkv, kc, vc, B, Lc, 0, pos_rows=start.to(DEV))
    return qkv, kc, vc, start, qlen, Lc


@pytest.mark.parametrize('D', [64, 128])
@pytest.mark.parametrize('B', [1, 3, 8])
def test_attention_cached_matches_fp32_reference(B, D):
    H = 32 if D == 128 else 16
    for seed in ([0, 1, 2, 3, 4, 5, 6] if B == 1 else [B]):
        qkv, kc, vc, start, qlen, Lc = _chunk_case(B, D, H, seed)
        scale = D ** -0.5
        want = _cached_ref(qkv, kc, vc, start, qlen, B, Lc, H, D, scale)
        ql = None if bool((qlen == Lc).all()) else qlen.to(DEV)
        got = kernels.attention_cached(qkv, kc, vc, B, H, D, Lc, scale, start.to(DEV), ql).float().view(B, Lc, -1)
        for b in range(B):
            n = int(qlen[b])
            e = rel(got[b, :n], want[b])
            assert e < 4e-3, (seed, b, int(start[b]), n, e)


def _poison(shape, dtype=BF, n=8):
    """Leave n freed NaN-filled blocks of this shape in the caching allocator: the next allocations of that size
    (torch.empty) start out as NaN."""
    junk = [torch.full(shape, float('nan'), dtype=dtype, device=DEV) for _ in range(n)]
    del junk


def test_attention_cached_skipped_tiles_are_finite():
    """Rows past qlen[b] are fed on through wo into the next layer's K/V (read masked by later key blocks): a 128-row
    tile wholly past qlen[b] writes zeros, the other rows attend over the valid keys -- all finite whatever the
    allocator hands out."""
    B, H, D = 2, 32, 128
    Lc = 300
    start = torch.tensor([800, 37], dtype=I32)
    qlen = torch.tensor([100, 300], dtype=I32)
    qkv = torch.randn(B * Lc, 3 * H * D, device=DEV).to(BF)
    kc = torch.zeros(B, 1200, H * D, device=DEV, dtype=BF)
    vc = torch.zeros_like(kc)
    kc[:, :800] = torch.randn(B, 800, H * D, device=DEV).to(BF)
    vc[:, :800] = torch.randn(B, 800, H * D, device=DEV).to(BF)
    kernels.kv_append(qkv, kc, vc, B, Lc, 0, pos_rows=start.to(DEV))
    _poison((B * Lc, H * D))
    got = kernels.attention_cached(qkv, kc, vc, B, H, D, Lc, D ** -0.5, start.to(DEV), qlen.to(DEV)).view(B, Lc, -1)
    assert bool(torch.isfinite(got.float()).all())
    assert bool((got[0, 128:] == 0).all())           # row 0's tiles 1 and 2 lie wholly past its 100 queries
    want = _cached_ref(qkv, kc, vc, start, qlen, B, Lc, H, D, D ** -0.5)
    for b in range(B):
        assert rel(got[b, :int(qlen[b])].float(), want[b]) < 4e-3, b


def test_attention_cached_f16():
    B, H, D = 3, 32, 128
    qkv, kc, vc, start, qlen, Lc = _chunk_case(B, D, H, 11, dtype=torch.float16)
    want = _cached_ref(qkv, kc, vc, start, qlen, B, Lc, H, D, D ** -0.5)
    got = kernels.attention_cached(qkv, kc, vc, B, H, D, Lc, D ** -0.5, start.to(DEV), qlen.to(DEV)).float().view(B, Lc, -1)
    for b in range(B):
        assert rel(got[b, :int(qlen[b])], want[b]) < 4e-3, b


@pytest.mark.parametrize('D', [64, 128])
def test_attention_cached_from_empty_cache_equals_prefill_attention_bitwise(D):
    """start = 0: the chunk is the whole sequence; the result is bitwise the packed-QKV wgmma kernel's (causal), and
    with qlen = seqlens that kernel's seqlens path, on the valid rows."""
    B, L, H = 3, 300, 32 if D == 128 else 16
    torch.manual_seed(D)
    qkv = torch.randn(B * L, 3 * H * D, device=DEV).to(BF)
    kc = torch.zeros(B, L + 40, H * D, device=DEV, dtype=BF)
    vc = torch.zeros_like(kc)
    kernels.kv_append(qkv, kc, vc, B, L, 0)
    zero = torch.zeros(B, dtype=I32, device=DEV)
    want = kernels.attention(qkv, B, L, H, D, True, D ** -0.5, impl='tc')
    got = kernels.attention_cached(qkv, kc, vc, B, H, D, L, D ** -0.5, zero)
    assert torch.equal(got, want)
    seqlens = torch.tensor([300, 129, 64], dtype=I32, device=DEV)
    want = kernels.attention(qkv, B, L, H, D, True, D ** -0.5, seqlens=seqlens, impl='tc').view(B, L, -1)
    got = kernels.attention_cached(qkv, kc, vc, B, H, D, L, D ** -0.5, zero, seqlens).view(B, L, -1)
    for b in range(B):
        n = int(seqlens[b])
        assert torch.equal(got[b, :n], want[b, :n]), b


def test_continuation_splice_places_region_rows_and_rejects_image_tokens():
    cfg = EngineConfig()
    V, D = 1000, 64
    g = torch.Generator().manual_seed(5)
    embed = torch.randn(V, D, generator=g).to(DEV, BF)
    B, L = 3, 40
    ids = torch.randint(3, V, (B, L), generator=g)
    counts = [2, 0, 3]
    for b, k in enumerate(counts):
        ids[b, torch.randperm(L, generator=g)[:k]] = cfg.bbox_token
    K = sum(counts)
    rows = torch.randn(K, D, generator=g).to(DEV, BF)
    offs = torch.tensor([0, 2, 2, 5], dtype=I32, device=DEV)
    kw = dict(im_patch_token=cfg.im_patch_token, im_start_token=cfg.im_start_token, im_end_token=cfg.im_end_token,
              bbox_token=cfg.bbox_token)
    big = torch.randn(cfg.bbox_token + 8, D, generator=g).to(DEV, BF)    # ids up to the special tokens
    big[:V] = embed
    out = splice_region_tokens(ids.to(DEV), big, None, (rows, offs), 0, continuation=True, **kw)
    for b in range(B):
        ordn = 0
        for t in range(L):
            if int(ids[b, t]) == cfg.bbox_token:
                assert torch.equal(out[b, t], rows[int(offs[b]) + ordn]), (b, t)
                ordn += 1
            else:
                assert torch.equal(out[b, t], big[int(ids[b, t])]), (b, t)
    for tok in (cfg.im_patch_token, cfg.im_start_token, cfg.im_end_token):
        bad = ids.clone()
        bad[1, 5] = tok
        with pytest.raises(ValueError, match='Image tokens'):
            splice_region_tokens(bad.to(DEV), big, None, (rows, offs), 0, continuation=True, **kw)
    with pytest.raises(ValueError, match='<bbox>'):
        splice_region_tokens(ids.to(DEV), big, None, (rows, torch.tensor([0, 2, 3, 5], dtype=I32, device=DEV)), 0,
                             continuation=True, **kw)


# ---- engine --------------------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def eng224():
    cfg = EngineConfig(image_size=224, vit_layers=12, n_layers=2)
    sd, vit_sd = random_state_dicts(cfg, DEV, seed=41)
    return cfg, PrefillEngine(cfg, sd, vit_sd, DEV), sd, vit_sd


def _boxes(k, g, cfg):
    p = torch.rand(k, 2, 2, generator=g).sort(dim=1).values
    bx = torch.cat([p[:, 0, :], p[:, 1, :]], 1)
    bx[:, 2:] = torch.maximum(bx[:, 2:], bx[:, :2] + 2.0 / cfg.image_size).clamp(max=1.0)
    return bx


def conversation(cfg, B, T, splits, tail_boxes, seed):
    """B prompts of one length L (image span first, T text tokens): row b has one <bbox> before splits[b] and
    tail_boxes[b] <bbox> tokens at or after it; boxes in token order."""
    ids, images, _ = make_inputs(cfg, B, [0] * B, T, seed=seed)
    g = torch.Generator().manual_seed(seed + 7)
    P = cfg.num_patches
    L = ids.shape[1]
    boxes = []
    for b in range(B):
        s = splits[b]
        ids[b, P + 3 + int(torch.randint(0, s - P - 3, (1,), generator=g))] = cfg.bbox_token
        if tail_boxes[b]:
            ids[b, s + torch.randperm(L - s, generator=g)[:tail_boxes[b]]] = cfg.bbox_token
        boxes.append(_boxes(int((ids[b] == cfg.bbox_token).sum()), g, cfg))
    return ids, images.to(BF), boxes


def _prefix_then_extend(eng, cfg, ids, images, boxes, splits, last_only=False, extra=8, poison=False):
    B, L = ids.shape
    sp = torch.tensor(splits)
    pre_len = int(sp.max())
    pre = torch.zeros(B, pre_len, dtype=torch.int64)
    tl = L - sp
    Lc = int(tl.max())
    tail = torch.zeros(B, Lc, dtype=torch.int64)
    pre_boxes, tail_boxes = [], []
    for b in range(B):
        s = splits[b]
        pre[b, :s] = ids[b, :s]
        tail[b, :L - s] = ids[b, s:]
        n = int((ids[b, :s] == cfg.bbox_token).sum())
        pre_boxes.append(boxes[b][:n])
        tail_boxes.append(boxes[b][n:])
    cache = KVCache(cfg, B, L + extra, DEV)
    pmask = (torch.arange(pre_len)[None] < sp[:, None]).long()
    eng.forward(pre.to(DEV), images.to(DEV), pre_boxes, attention_mask=pmask, last_only=True, cache=cache)
    tmask = (torch.arange(Lc)[None] < tl[:, None]).long()
    if poison:   # chunk-sized activations (embeddings, attention outputs, ...) start out as NaN
        _poison((B * Lc, cfg.hidden))
    out = eng.extend(cache, tail.to(DEV), images.to(DEV), tail_boxes, attention_mask=tmask, last_only=last_only)
    assert cache.lens.tolist() == [L] * B
    assert torch.equal(cache.ids[:, :L].cpu(), ids)
    return out, cache


@pytest.mark.parametrize('tail,new_boxes', [(1, 0), (1, 1), (17, 0), (17, 2), (150, 0), (150, 3)])
def test_extend_matches_one_full_forward(eng224, tail, new_boxes):
    cfg, eng = eng224[:2]
    T = 180
    L = T + cfg.num_patches + 2
    ids, images, boxes = conversation(cfg, 1, T, [L - tail], [new_boxes], seed=tail + new_boxes)
    full = eng.forward(ids.to(DEV), images.to(DEV), boxes).float()
    got, _ = _prefix_then_extend(eng, cfg, ids, images, boxes, [L - tail])
    got = got.float()
    # a 1-row chunk runs the weight-streaming (skinny) GEMMs, which sum over K in another order than the full forward's
    # wgmma GEMMs: the decode step's tolerance (test_ragged_decode_gpu) applies to it
    assert rel(got[0, 0], full[0, L - tail]) < (5e-3 if tail > 1 else 1e-2)
    for i in range(tail):
        assert rel(got[0, i], full[0, L - tail + i]) < 1e-2, i


def test_extend_batch_with_different_reuse_per_row(eng224):
    cfg, eng = eng224[:2]
    T, B = 180, 4
    L = T + cfg.num_patches + 2
    splits = [L - 1, L - 17, L - 150, L - 60]
    ids, images, boxes = conversation(cfg, B, T, splits, [0, 1, 2, 1], seed=3)
    full = eng.forward(ids.to(DEV), images.to(DEV), boxes).float()
    got, _ = _prefix_then_extend(eng, cfg, ids, images, boxes, splits)
    got = got.float()
    for b in range(B):
        s = splits[b]
        assert rel(got[b, 0], full[b, s]) < 5e-3, b
        for i in range(L - s):
            assert rel(got[b, i], full[b, s + i]) < 1e-2, (b, i)


def test_extend_mixed_tails_with_skipped_tiles_stays_finite(eng224):
    """Tails of 100 and 200 tokens, starts 422 and 322 (not multiples of 64): row 0's second 128-row query tile is
    skipped, and row 0's last key block (keys up to 575) reaches the chunk rows 128..153 that tile fed into the cache of
    layer 2.  With the allocator full of NaN blocks the logits stay finite and match the full forward."""
    cfg, eng = eng224[:2]
    T = 264
    L = T + cfg.num_patches + 2
    splits = [L - 100, L - 200]
    assert [s % 64 for s in splits] == [38, 2]
    ids, images, boxes = conversation(cfg, 2, T, splits, [1, 2], seed=12)
    full = eng.forward(ids.to(DEV), images.to(DEV), boxes).float()
    got, cache = _prefix_then_extend(eng, cfg, ids, images, boxes, splits, poison=True)
    got = got.float()
    for b in range(2):
        s = splits[b]
        assert bool(torch.isfinite(got[b, :L - s]).all()), b
        assert rel(got[b, 0], full[b, s]) < 5e-3, b
        for i in range(L - s):
            assert rel(got[b, i], full[b, s + i]) < 1e-2, (b, i)
    assert all(bool(torch.isfinite(t.float()).all()) for t in cache.k + cache.v)


def test_extend_rejects_a_box_count_mismatch(eng224):
    """Boxes left over for a chunk without <bbox> tokens: ValueError, as the full prefill raises for that prompt."""
    cfg, eng = eng224[:2]
    T = 60
    L = T + cfg.num_patches + 2
    ids, images, boxes = conversation(cfg, 1, T, [L - 20], [0], seed=13)
    g = torch.Generator().manual_seed(14)
    extra = [torch.cat([boxes[0], _boxes(1, g, cfg)])]
    with pytest.raises(ValueError, match='<bbox>'):
        eng.forward(ids.to(DEV), images.to(DEV), extra)
    with pytest.raises(ValueError, match='<bbox>'):
        _prefix_then_extend(eng, cfg, ids, images, extra, [L - 20])


def test_graphed_decode_after_extend_equals_eager_bitwise(eng224):
    cfg, eng = eng224[:2]
    T, B, n = 120, 3, 6
    L = T + cfg.num_patches + 2
    splits = [L - 30, L - 5, L - 77]
    ids, images, boxes = conversation(cfg, B, T, splits, [1, 0, 2], seed=9)
    toks = torch.randint(3, 32000, (n, B, 1), generator=torch.Generator().manual_seed(1)).to(DEV)
    runs = []
    for graphed in (False, True):
        first, cache = _prefix_then_extend(eng, cfg, ids, images, boxes, splits, last_only=True, extra=n + 8)
        stepper = GraphedDecode(eng, cache) if graphed else None
        runs.append(torch.stack([(stepper.step(toks[t]) if graphed else eng.decode_step(toks[t], cache)).clone()
                                 for t in range(n)]))
        assert cache.lens.tolist() == [L + n] * B
    assert torch.equal(runs[0], runs[1])


def _near_tie_agrees(eng, ids, images, boxes, got, want, L):
    """got / want: [B, L + n] token ids of two runs on the same prompt.  Equal, or where a row first differs, the token
    `got` chose is within the near-tie margin of the no-cache logits at that position."""
    for b in range(ids.shape[0]):
        diff = (got[b, L:] != want[b, L:]).nonzero()
        if not len(diff):
            continue
        t = int(diff[0])
        seq = want[b:b + 1, :L + t].to(DEV)
        row = eng.forward(seq, images[b:b + 1].to(DEV), [boxes[b]], last_only=True).float()[0, 0]
        tok = int(got[b, L + t])
        margin = (row.max() - row[tok]).item()
        assert margin <= 3e-2 * row.std().item(), (b, t, tok, int(row.argmax()), margin)


@pytest.mark.parametrize('new_box', [False, True])
def test_two_turn_generate_with_cache_matches_no_cache(eng224, new_box):
    cfg, eng = eng224[:2]
    B, T, n1, n2 = 2, 60, 8, 6
    ids1, images, boxes = make_inputs(cfg, B, [1, 2], T, seed=21)
    images = images.to(BF)
    L1 = ids1.shape[1]
    cache = KVCache(cfg, B, L1 + n1, DEV)
    out1 = eng.generate(ids1.to(DEV), images, boxes, max_new_tokens=n1, cache=cache).cpu()
    assert torch.equal(out1, eng.generate(ids1.to(DEV), images, boxes, max_new_tokens=n1).cpu())
    g = torch.Generator().manual_seed(22)
    q = torch.randint(3, 32000, (B, 48), generator=g)
    boxes2 = [bx.clone() for bx in boxes]
    if new_box:
        q[:, 10] = cfg.bbox_token
        boxes2 = [torch.cat([bx, _boxes(1, g, cfg)]) for bx in boxes]
    ids2 = torch.cat([out1, q], 1)
    reuse = cache.reusable(ids2, images, boxes2)
    assert reuse.tolist() == [L1 + n1 - 1] * B        # everything but the last answer token
    got = eng.generate(ids2.to(DEV), images, boxes2, max_new_tokens=n2, cache=cache).cpu()
    want = eng.generate(ids2.to(DEV), images, boxes2, max_new_tokens=n2).cpu()
    assert cache.max_len >= ids2.shape[1] + n2
    _near_tie_agrees(eng, ids2, images, boxes2, got, want, ids2.shape[1])


def test_two_turn_generate_retokenized_answer_and_changed_image(eng224):
    """The re-encoded answer differs from the generated ids in the last token the cache holds: reuse stops there.
    A different image: nothing is reused (full prefill into the cache)."""
    cfg, eng = eng224[:2]
    B, T, n1, n2 = 2, 60, 8, 5
    ids1, images, boxes = make_inputs(cfg, B, [2, 1], T, seed=31)
    images = images.to(BF)
    L1 = ids1.shape[1]
    cache = KVCache(cfg, B, L1 + n1, DEV)
    out1 = eng.generate(ids1.to(DEV), images, boxes, max_new_tokens=n1, cache=cache).cpu()
    ids2 = torch.cat([out1, torch.randint(3, 32000, (B, 48), generator=torch.Generator().manual_seed(32))], 1)
    ids2[:, L1 + n1 - 2] = (ids2[:, L1 + n1 - 2] + 1) % 32000
    assert cache.reusable(ids2, images, boxes).tolist() == [L1 + n1 - 2] * B
    got = eng.generate(ids2.to(DEV), images, boxes, max_new_tokens=n2, cache=cache).cpu()
    want = eng.generate(ids2.to(DEV), images, boxes, max_new_tokens=n2).cpu()
    _near_tie_agrees(eng, ids2, images, boxes, got, want, ids2.shape[1])
    other = images.flip(0).contiguous()
    assert cache.reusable(ids2, other, boxes).tolist() == [0] * B
    got = eng.generate(ids2.to(DEV), other, boxes, max_new_tokens=n2, cache=cache).cpu()
    want = eng.generate(ids2.to(DEV), other, boxes, max_new_tokens=n2).cpu()
    _near_tie_agrees(eng, ids2, other, boxes, got, want, ids2.shape[1])


def test_two_turns_through_the_seam_with_dynamic_cache(eng224):
    from transformers import DynamicCache
    from tests.test_model_seam_gpu import build_seam_model
    cfg, _, sd, vit_sd = eng224
    model = build_seam_model(cfg, sd, vit_sd).eval()
    ids1, images, boxes = make_inputs(cfg, 1, [2], 40, seed=41)
    img = images.to(DEV)
    bx = [b.to(DEV) for b in boxes]
    n1, n2 = 7, 6
    outs = {}
    eng = model._get_engine(torch.device(DEV))
    chunks = []
    extend = eng.extend

    def counted(cache, input_ids, *a, **k):
        chunks.append(tuple(input_ids.shape))
        return extend(cache, input_ids, *a, **k)
    eng.extend = counted
    with torch.inference_mode():
        for hf in (False, True):
            cache = DynamicCache()
            out1 = model.generate(ids1.to(DEV), images=img, bboxes=bx, max_new_tokens=n1, past_key_values=cache,
                                  use_hf_loop=hf)
            q = torch.randint(3, 32000, (1, 48), generator=torch.Generator().manual_seed(43)).to(DEV)
            ids2 = torch.cat([out1, q], 1)
            # turn 2 reuses everything turn 1 left in the cache (all but the last answer token) and extends by the rest
            assert cache._g4r_cache.kv.reusable(ids2, img, bx).tolist() == [out1.shape[1] - 1]
            chunks.clear()
            out2 = model.generate(ids2, images=img, bboxes=bx, max_new_tokens=n2, past_key_values=cache, use_hf_loop=hf)
            assert chunks == [(1, 49)], (hf, chunks)
            assert cache._g4r_cache.kv.length >= ids2.shape[1]
            fresh = model.generate(ids2, images=img, bboxes=bx, max_new_tokens=n2, use_hf_loop=hf)
            outs[hf] = (out1.cpu(), ids2.cpu(), out2.cpu(), fresh.cpu())
    assert model._get_engine(torch.device(DEV)) is eng
    L1 = ids1.shape[1]
    # the two loops agree with each other (near-tie rule against the no-cache logits) ...
    _near_tie_agrees(eng, ids1, images, boxes, outs[True][0], outs[False][0], L1)
    if torch.equal(outs[True][1], outs[False][1]):
        _near_tie_agrees(eng, outs[False][1], images, boxes, outs[True][2], outs[False][2], outs[False][1].shape[1])
    # ... and each turn 2 on the reused cache with the same loop's no-cache run
    for hf in (False, True):
        ids2 = outs[hf][1]
        _near_tie_agrees(eng, ids2, images, boxes, outs[hf][2], outs[hf][3], ids2.shape[1])
