"""Decode over a batch of prompts of different lengths: per-sample positions (pos_rows, a device int32 [B]) in the
KV-cache append, the RoPE + KV epilogues of the decode GEMMs, the split-KV decode attention, the engine's decode step
and CUDA graph, and generate() through the model seam.  Shapes use H = 32, D = 128 unless stated."""
import pytest
import torch

import gpt4roi_b200.engine as E
from gpt4roi_b200 import dense, kernels
from gpt4roi_b200.engine import EngineConfig, GraphedDecode, KVCache, PrefillEngine, random_state_dicts
from tests.test_engine_gpu import make_inputs, rel

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
BF = torch.bfloat16
I32 = torch.int32


def _attn_ref(qkv, kc, vc, lens, H, D, scale):
    """Per-row fp32 softmax(q.K^T)V over the row's own keys, probabilities rounded to the storage type before P.V."""
    B, HD = qkv.shape[0], H * D
    out = []
    for b in range(B):
        n = int(lens[b])
        q = qkv[b, :HD].float().view(H, 1, D)
        k = kc[b, :n].float().view(n, H, D).permute(1, 0, 2)
        v = vc[b, :n].float().view(n, H, D).permute(1, 0, 2)
        p = torch.softmax(q @ k.transpose(-1, -2) * scale, -1).to(qkv.dtype).float()
        out.append((p @ v).reshape(HD))
    return torch.stack(out)


# 1 key; shorter than one split slice (2048 / 8 = 256); non-multiples of 64; 2048
_LENS = [1, 100, 2048, 777, 64, 193, 5, 1000]


@pytest.mark.parametrize('D', [64, 128])
@pytest.mark.parametrize('B', [1, 3, 8, 20])
def test_decode_attention_rows_matches_fp32_reference(B, D):
    H = 32
    torch.manual_seed(B * 10 + D)
    HD, Lmax = H * D, 2048 + 9
    lens = torch.tensor([_LENS[(b + B) % len(_LENS)] for b in range(B)], dtype=I32)
    qkv = torch.randn(B, 3 * HD, device=DEV).to(BF)
    kc = torch.randn(B, Lmax, HD, device=DEV).to(BF)
    vc = torch.randn(B, Lmax, HD, device=DEV).to(BF)
    scale = D ** -0.5
    want = _attn_ref(qkv, kc, vc, lens, H, D, scale)
    rows = (lens - 1).to(DEV)
    for bound in (int(lens.max()), Lmax):   # eager bound (longest row) and graph-style bound (Lmax)
        got = kernels.decode_attention(qkv, kc, vc, B, H, D, bound, scale, pos_rows=rows).float()
        for b in range(B):
            e = ((got[b] - want[b]).norm() / want[b].norm()).item()
            assert e < 4e-3, (bound, b, int(lens[b]), e)
    # all rows equal: bitwise the scalar entry (host length, and device length with the Lmax bound)
    for n in (1, 100, 777, 2048):
        same = torch.full((B,), n - 1, dtype=I32, device=DEV)
        a = kernels.decode_attention(qkv, kc, vc, B, H, D, n, scale)
        b_ = kernels.decode_attention(qkv, kc, vc, B, H, D, n, scale, pos_rows=same)
        assert torch.equal(a, b_), n
        pos_dev = torch.tensor([n - 1], dtype=I32, device=DEV)
        a = kernels.decode_attention(qkv, kc, vc, B, H, D, Lmax, scale, pos_dev=pos_dev)
        b_ = kernels.decode_attention(qkv, kc, vc, B, H, D, Lmax, scale, pos_rows=same)
        assert torch.equal(a, b_), n


def test_decode_attention_rows_f16():
    B, H, D = 5, 32, 128
    torch.manual_seed(3)
    HD, Lmax = H * D, 900
    lens = torch.tensor([1, 70, 899, 300, 129], dtype=I32)
    qkv = torch.randn(B, 3 * HD, device=DEV).half()
    kc = torch.randn(B, Lmax, HD, device=DEV).half()
    vc = torch.randn(B, Lmax, HD, device=DEV).half()
    want = _attn_ref(qkv, kc, vc, lens, H, D, D ** -0.5)
    got = kernels.decode_attention(qkv, kc, vc, B, H, D, Lmax, D ** -0.5, pos_rows=(lens - 1).to(DEV)).float()
    for b in range(B):
        assert ((got[b] - want[b]).norm() / want[b].norm()).item() < 4e-3, b


@pytest.mark.parametrize('Ln', [1, 3])
def test_kv_append_rows_places_each_sample_at_its_position(Ln):
    torch.manual_seed(Ln)
    B, HD, Lmax = 4, 256, 24
    pos = torch.tensor([0, 7, 20, 13], dtype=I32)
    qkv = torch.randn(B * Ln, 3 * HD, device=DEV).to(BF)
    sentinel = torch.tensor(-1234.0, dtype=BF)
    kc = torch.full((B, Lmax, HD), sentinel.item(), device=DEV, dtype=BF)
    vc = kc.clone()
    kernels.kv_append(qkv, kc, vc, B, Ln, 0, pos_rows=pos.to(DEV))
    want_k = torch.full_like(kc, sentinel.item())
    want_v = want_k.clone()
    for b in range(B):
        p = int(pos[b])
        want_k[b, p:p + Ln] = qkv.view(B, Ln, -1)[b, :, HD:2 * HD]
        want_v[b, p:p + Ln] = qkv.view(B, Ln, -1)[b, :, 2 * HD:]
    assert torch.equal(kc, want_k) and torch.equal(vc, want_v)


def _rope_tables(Lmax, D=128):
    inv = 1.0 / (10000.0 ** (torch.arange(0, D, 2).float() / D))
    emb = torch.cat([torch.arange(Lmax).float()[:, None] * inv[None]] * 2, -1)
    return emb.cos().to(DEV, BF).contiguous(), emb.sin().to(DEV, BF).contiguous()


def _qkv_weights(seed, hid=4096):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(3 * hid, hid, device=DEV, generator=g) * 0.02).to(BF)


@pytest.mark.parametrize('B', [8, 16])
def test_decode_gemm_rows_equals_scalar_launch_per_row(B):
    """RoPE + KV-append epilogue of the weight-streaming decode GEMM: output row b and cache row (b, pos_rows[b]) are
    bitwise those of the scalar launch at pos = pos_rows[b] (same M: rows are independent)."""
    hid, Lmax = 4096, 64
    torch.manual_seed(B)
    x = (torch.randn(B, hid, device=DEV) * 0.5).to(BF)
    w = _qkv_weights(B)
    cos, sin = _rope_tables(Lmax)
    pos = torch.randint(0, Lmax, (B,), dtype=I32)
    kc, vc = torch.zeros(B, Lmax, hid, device=DEV, dtype=BF), torch.zeros(B, Lmax, hid, device=DEV, dtype=BF)
    got = dense.decode_gemm(x, w, rope=(cos, sin, 2 * hid, 0, None), kv=(kc, vc), pos_rows=pos.to(DEV))
    for b in range(B):
        p = int(pos[b])
        kc1, vc1 = torch.zeros_like(kc), torch.zeros_like(vc)
        ref = dense.decode_gemm(x, w, rope=(cos, sin, 2 * hid, p, None), kv=(kc1, vc1))
        assert torch.equal(got[b], ref[b]), b
        assert torch.equal(kc[b, p], kc1[b, p]) and torch.equal(vc[b, p], vc1[b, p]), b
    # all rows equal: bitwise the scalar launch, output and caches
    p = 37
    kc2, vc2, kc3, vc3 = (torch.zeros_like(kc) for _ in range(4))
    a = dense.decode_gemm(x, w, rope=(cos, sin, 2 * hid, p, None), kv=(kc2, vc2))
    b_ = dense.decode_gemm(x, w, rope=(cos, sin, 2 * hid, 0, None), kv=(kc3, vc3),
                           pos_rows=torch.full((B,), p, dtype=I32, device=DEV))
    assert torch.equal(a, b_) and torch.equal(kc2, kc3) and torch.equal(vc2, vc3)


@pytest.mark.parametrize('B', [8, 20])
def test_qkv_rope_rows_equals_scalar_launch_per_row(B):
    """Fused QKV-RoPE GEMM with per-sample positions (B = 20: the wgmma epilogue; B = 8: the skinny kernel)."""
    hid, Lmax = 4096, 64
    torch.manual_seed(100 + B)
    x = (torch.randn(B, hid, device=DEV) * 0.5).to(BF)
    w = _qkv_weights(100 + B)
    cos, sin = _rope_tables(Lmax)
    pos = torch.randint(0, Lmax, (B,), dtype=I32)
    got = dense.qkv_rope(x, w, cos, sin, 1, 2 * hid, pos_rows=pos.to(DEV))
    for b in range(B):
        ref = dense.qkv_rope(x, w, cos, sin, 1, 2 * hid, pos0=int(pos[b]))
        assert torch.equal(got[b], ref[b]), b
    p = 41
    a = dense.qkv_rope(x, w, cos, sin, 1, 2 * hid, pos0=p)
    b_ = dense.qkv_rope(x, w, cos, sin, 1, 2 * hid, pos_rows=torch.full((B,), p, dtype=I32, device=DEV))
    assert torch.equal(a, b_)


# ---- engine ------------------------------------------------------------------------------------------------

def ragged_inputs(cfg, B, T, seed):
    """B prompts right-padded to one length L: row b keeps its first lens[b] tokens (pad id 0 after), and only the boxes
    of the <bbox> tokens inside them; box counts differ between rows."""
    ks = [1 + (b % 3) for b in range(B)]
    ids, images, boxes = make_inputs(cfg, B, ks, T, seed=seed)
    L = ids.shape[1]
    g = torch.Generator().manual_seed(seed + 1)
    lens = [L] + [L - int(torch.randint(1, T - 2, (1,), generator=g)) for _ in range(B - 1)]
    for b in range(B):
        ids[b, lens[b]:] = 0
        boxes[b] = boxes[b][:int((ids[b, :lens[b]] == cfg.bbox_token).sum())]
    return ids, images.to(BF), boxes, torch.tensor(lens)


def _teacher_forced(eng, cfg, B, T, seed, n_new=4, tol_first=5e-3):
    ids, images, boxes, lens = ragged_inputs(cfg, B, T, seed)
    L = ids.shape[1]
    toks = torch.randint(3, 32000, (n_new, B, 1), generator=torch.Generator().manual_seed(seed))
    mask = (torch.arange(L)[None] < lens[:, None]).long()
    cache = KVCache(cfg, B, L + n_new + 2, DEV)
    first = eng.forward(ids.to(DEV), images.to(DEV), boxes, attention_mask=mask, last_only=True, cache=cache).float()
    assert cache.lens is not None and cache.lens.tolist() == lens.tolist()
    steps = [eng.decode_step(toks[t].to(DEV), cache).float() for t in range(n_new)]
    assert cache.lens.tolist() == (lens + n_new).tolist() and cache.length == L + n_new
    for b in range(B):
        n = int(lens[b])
        seq = torch.cat([ids[b, :n], toks[:, b, 0]])[None]
        solo = eng.forward(seq.to(DEV), images[b:b + 1].to(DEV), [boxes[b]]).float()[0]
        e0 = rel(first[b, 0], solo[n - 1])
        assert e0 < tol_first, (b, e0)
        for t in range(n_new):
            e = rel(steps[t][b, 0], solo[n + t])
            assert e < 1e-2, (b, t, e)


@pytest.fixture(scope='module')
def eng224():
    cfg = EngineConfig(image_size=224, vit_layers=12, n_layers=2)
    sd, vit_sd = random_state_dicts(cfg, DEV, seed=41)
    return cfg, PrefillEngine(cfg, sd, vit_sd, DEV)


@pytest.mark.parametrize('fused', [0, 1])
def test_ragged_decode_matches_solo_prefill(eng224, fused):
    cfg, eng = eng224
    old = E._DECODE_FUSED
    E._DECODE_FUSED = fused
    try:
        _teacher_forced(eng, cfg, 4, 24, seed=50 + fused)
    finally:
        E._DECODE_FUSED = old


def test_ragged_decode_matches_solo_prefill_wgmma_route(eng224):
    cfg, eng = eng224
    # batch > 16: wgmma QKV-RoPE GEMM + kv_append rows.  The batch-20 prefill runs its GEMMs on other tile shapes than the
    # solo batch-1 runs, so bf16 roundings differ even for the full-length row (measured 5.2e-3 there): 1e-2 for step 0.
    _teacher_forced(eng, cfg, 20, 24, seed=60, n_new=3, tol_first=1e-2)


def test_ragged_graph_equals_eager_and_equal_lengths_equal_uniform(eng224):
    """GraphedDecode on a ragged cache == eager ragged decode, bitwise, at every step.  B = 4 and L >= 256: the eager
    bound (length + 1) and the graph bound (max_len) both give the split factor 4.  A ragged cache whose lengths are all
    equal == today's uniform cache, bitwise."""
    cfg, eng = eng224
    B, n_new = 4, 6
    ids, images, boxes, lens = ragged_inputs(cfg, B, 24, seed=70)
    L = ids.shape[1]
    assert L >= 256
    plan = eng.plan_boxes(boxes)
    toks = torch.randint(3, 32000, (n_new, B, 1), generator=torch.Generator().manual_seed(7)).to(DEV)
    seqlens = lens.to(DEV, I32)
    outs = []
    for graphed in (False, True):
        cache = KVCache(cfg, B, L + n_new + 2, DEV)
        eng.forward_device(ids.to(DEV), images.to(DEV), plan, last_only=True, seqlens=seqlens, cache=cache)
        stepper = GraphedDecode(eng, cache) if graphed else None
        seq = [(stepper.step(toks[t]) if graphed else eng.decode_step(toks[t], cache)).clone() for t in range(n_new)]
        assert cache.lens.tolist() == (lens + n_new).tolist()
        outs.append(torch.stack(seq))
    assert torch.equal(outs[0], outs[1])
    # all lengths equal (ragged machinery) vs no lengths (uniform path): first logits and every step
    ids_u, images_u, boxes_u = make_inputs(cfg, B, [1, 2, 1, 3], 24, seed=71)
    plan = eng.plan_boxes(boxes_u)
    Lu = ids_u.shape[1]
    res = []
    for ragged in (False, True):
        for graphed in (False, True):
            cache = KVCache(cfg, B, Lu + n_new + 2, DEV)
            sl = torch.full((B,), Lu, dtype=I32, device=DEV) if ragged else None
            first = eng.forward_device(ids_u.to(DEV), images_u.to(DEV, BF), plan, last_only=True, seqlens=sl,
                                       cache=cache).clone()
            assert (cache.lens is not None) == ragged
            stepper = GraphedDecode(eng, cache) if graphed else None
            seq = [(stepper.step(toks[t]) if graphed else eng.decode_step(toks[t], cache)).clone() for t in range(n_new)]
            res.append((first, torch.stack(seq)))
    for r in res[1:]:
        assert torch.equal(r[0], res[0][0]) and torch.equal(r[1], res[0][1])


def test_unfused_head_dim_route_refuses_ragged_cache():
    cfg = EngineConfig(image_size=224, vit_layers=1, n_layers=1, hidden=512, n_heads=8, mlp=256, vocab=1000)   # D = 64
    sd, vit_sd = random_state_dicts(cfg, DEV, seed=2)
    eng = PrefillEngine(cfg, sd, vit_sd, DEV, parts=('llm',))
    ids = torch.randint(3, 900, (2, 12))
    cache = KVCache(cfg, 2, 16, DEV)
    eng.forward_device(ids.to(DEV), None, None, last_only=True, seqlens=torch.tensor([12, 9], dtype=I32, device=DEV),
                       cache=cache)
    with pytest.raises(NotImplementedError):
        eng.decode_step(ids[:, :1].to(DEV), cache)


# ---- generate() through the model seam --------------------------------------------------------------------

def test_generate_ragged_batch_through_the_seam():
    from oracle import model_oracle
    from tests.test_model_seam_gpu import build_seam_model
    cfg = EngineConfig(image_size=224, vit_layers=24, n_layers=2)
    sd, vit_sd = random_state_dicts(cfg, DEV, seed=43)
    B, n_new = 3, 6
    ids, images, boxes, lens = ragged_inputs(cfg, B, 24, seed=80)
    L = ids.shape[1]
    model = build_seam_model(cfg, sd, vit_sd, dtype=torch.float16).eval()
    mask_r = (torch.arange(L)[None] < lens[:, None]).long()
    shift = L - lens
    ids_l = torch.stack([torch.roll(ids[b], int(shift[b])) for b in range(B)])
    mask_l = torch.stack([torch.roll(mask_r[b], int(shift[b])) for b in range(B)])
    img = images.half().to(DEV)
    bx = [b.half().to(DEV) for b in boxes]
    with torch.inference_mode():
        out_r = model.generate(ids.to(DEV), images=img, bboxes=bx, attention_mask=mask_r.to(DEV), max_new_tokens=n_new)
        out_l = model.generate(ids_l.to(DEV), images=img, bboxes=bx, attention_mask=mask_l.to(DEV), max_new_tokens=n_new)
        out_h = model.generate(ids.to(DEV), images=img, bboxes=bx, attention_mask=mask_r.to(DEV), max_new_tokens=n_new,
                               use_hf_loop=True, pad_token_id=0)
    assert out_r.shape == (B, L + n_new)
    assert torch.equal(out_r[:, :L].cpu(), ids) and torch.equal(out_l[:, :L].cpu(), ids_l)   # prompts as given
    new = out_r[:, L:]
    assert torch.equal(out_l[:, L:], new), (out_l[:, L:], new)
    assert torch.equal(out_h[:, L:], new), (out_h[:, L:], new)
    # teacher-forced oracle on each row's unpadded sequence: every token is the arg-max or within its near-tie margin
    for b in range(B):
        n = int(lens[b])
        seq = torch.cat([ids[b, :n], new[b, :-1].cpu()])[None]
        ref = model_oracle.forward(cfg, {k: v.half().float() for k, v in sd.items()},
                                   {k: v.half().float() for k, v in vit_sd.items()}, seq, images[b:b + 1].half().float(),
                                   [boxes[b].half().float()], DEV)
        for t in range(n_new):
            row = ref[0, n - 1 + t]
            tok = int(new[b, t])
            margin = (row.max() - row[tok]).item()
            assert margin <= 3e-2 * row.std().item(), (b, t, tok, int(row.argmax()), margin)
    # EOS: the token row 0 emits at step 2 ends row 0 there; it continues with pad_token_id, the others go on
    eos, pad = int(new[0, 2]), 0
    with torch.inference_mode():
        out_e = model.generate(ids.to(DEV), images=img, bboxes=bx, attention_mask=mask_r.to(DEV), max_new_tokens=n_new,
                               eos_token_id=eos, pad_token_id=pad)
    got = out_e[:, L:].cpu()
    want = new.cpu().clone()
    for b in range(B):
        hit = (want[b] == eos).nonzero()
        if len(hit):
            want[b, int(hit[0]) + 1:] = pad
    finished = [bool((want[b] == eos).any()) for b in range(B)]
    n_out = n_new if not all(finished) else max(int((want[b] == eos).nonzero()[0]) + 1 for b in range(B))
    assert torch.equal(got, want[:, :n_out]), (got, want)
    assert int(got[0, 2]) == eos and bool((got[0, 3:] == pad).all())
