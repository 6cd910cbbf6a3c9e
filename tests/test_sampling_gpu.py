"""GPU tests of next-token selection on the device (csrc/sample.cu via kernels.sample_tokens, engine.Sampler, the graphed
decode step with the sampler captured, and the model seam's sampling).  Draws are predicted exactly by the numpy
Philox4x32-10 and the float64 inverse CDF of tests/test_sampling_cpu.py; the distribution is checked against the
softmax of transformers' own processed scores."""
from functools import partial

import numpy as np
import pytest
import torch
from scipy import stats

from gpt4roi_b200 import kernels
from gpt4roi_b200.engine import EngineConfig, GraphedDecode, KVCache, PrefillEngine, Sampler, random_state_dicts
from tests.test_engine_gpu import make_inputs
from tests.test_sampling_cpu import hf_kept, kept_set, uniforms

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
V = 32006
SEED = 0x1234_5678_9ABC_DEF


@pytest.fixture(scope='module')
def eng2():
    cfg = EngineConfig(image_size=224, vit_layers=24, n_layers=2)
    sd, vit_sd = random_state_dicts(cfg, DEV, seed=41)
    return cfg, PrefillEngine(cfg, sd, vit_sd, DEV), sd, vit_sd


@pytest.fixture(scope='module')
def rows(eng2):
    """33 rows of logits: 30 real lm_head rows of the 2-layer config (a text-only prefill, every position), then
    adversarial rows -- 300 equal values just below the 10 largest (ties at the top-k threshold), one dominant logit,
    and a row with 5000 -inf entries and a repeated maximum."""
    cfg, eng = eng2[:2]
    g = torch.Generator().manual_seed(5)
    ids = torch.randint(3, 32000, (2, 15), generator=g)
    real = eng.forward(ids.to(DEV), None, None).reshape(30, V).float()
    real = real * (4.0 / real.std())        # random weights give flat rows: spread them to a trained model's range
    base = real[0].clone()
    top = base.topk(10).values
    ties = base.clone()
    ties[torch.randperm(V, generator=g)[:300].to(DEV)] = float(top[-1]) - 0.25
    dom = real[1].clone()
    dom[123] = dom.max() + 20
    ninf = real[2].clone()
    ninf[torch.randperm(V, generator=g)[:5000].to(DEV)] = float('-inf')
    ninf[[7, 900, 31000]] = ninf.max() + 1
    return torch.cat([real, ties[None], dom[None], ninf[None]], 0)


PARAMS = [(T, k, p) for T in (0.2, 0.7, 1.0) for k in (0, 1, 50, V) for p in (1.0, 0.9, 0.5)]


def _predict_row(x, order, T, top_k, top_p, u, tol=1e-5):
    """The token the kernel draws with uniform u: inverse CDF over the kept set in `order` (value descending, index
    ascending).  Returns (token, ambiguous, keep): ambiguous when u lies within tol of a CDF or top-p boundary."""
    keep, p, near = kept_set(x, T, top_k, top_p)
    o = order[keep[order]]
    cdf = np.cumsum(p[o])
    i = min(int(np.searchsorted(cdf, u, side='right')), len(o) - 1)
    return int(o[i]), near or bool(np.min(np.abs(cdf - u)) < tol), keep


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16], ids=['bf16', 'fp16'])
def test_kernel_draws_equal_the_restatement(rows, dtype):
    """Every parameter combination, B in {1, 8, 16, 33}: the kernel's token is the one the numpy Philox + float64
    inverse CDF predicts (draws within 1e-5 of a CDF or top-p boundary skipped and counted), lies in HF's kept set
    (or in the boundary group of equal values HF's sort splits), and greedy is torch.argmax, ties included."""
    lg = rows.to(dtype)
    xs = lg.double().cpu().numpy()
    orders = [np.lexsort((np.arange(V), -x)) for x in xs]
    step = 5
    u = uniforms(SEED, step, 33)
    rng_step = torch.tensor([step], dtype=torch.int64, device=DEV)
    skipped = checked = 0
    for B in (1, 8, 16, 33):
        out = torch.full((B, 1), -1, dtype=torch.int64, device=DEV)
        kernels.sample_tokens(lg[:B], out, True)
        assert torch.equal(out[:, 0], lg[:B].float().argmax(-1)), B
    for T, top_k, top_p in PARAMS:
        got = {}
        for B in (1, 8, 16, 33):
            out = torch.full((B, 1), -1, dtype=torch.int64, device=DEV)
            kernels.sample_tokens(lg[:B], out, False, T, top_k, top_p, SEED, rng_step)
            got[B] = out[:, 0].cpu()
        for B in (1, 8, 16):   # a row's draw does not depend on the batch around it
            assert torch.equal(got[B], got[33][:B]), (T, top_k, top_p, B)
        for r in range(33):
            tok = int(got[33][r])
            want, amb, keep = _predict_row(xs[r], orders[r], T, top_k, top_p, u[r])
            hf = hf_kept(xs[r], T, top_k, top_p)
            assert hf[tok] or (keep[tok] and (xs[r][hf] == xs[r][tok]).any()), (T, top_k, top_p, r, tok)
            if amb:
                skipped += 1
                continue
            checked += 1
            assert tok == want, (T, top_k, top_p, r, tok, want)
    print('%s: %d draws predicted exactly, %d skipped near a boundary' % (dtype, checked, skipped))
    assert skipped <= checked // 20


def test_distribution_matches_transformers_processed_softmax(rows):
    """T = 0.7, top_k = 50 on one row: 65 536 draws (1024 copies of the row x 64 steps) against the softmax of HF's
    processed scores -- chi-square at a fixed seed, and no draw outside the kept set."""
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopKLogitsWarper
    row = rows[3].to(torch.float16)
    B, steps = 1024, 64
    lg = row[None].repeat(B, 1).contiguous()
    rng_step = torch.zeros(1, dtype=torch.int64, device=DEV)
    out = torch.empty((B, 1), dtype=torch.int64, device=DEV)
    draws = []
    for _ in range(steps):
        kernels.sample_tokens(lg, out, False, 0.7, 50, 1.0, 99, rng_step)
        draws.append(out[:, 0].clone())
        rng_step.add_(1)
    draws = torch.cat(draws).cpu()
    s = row.float().cpu()[None]
    ids = torch.zeros((1, 1), dtype=torch.long)
    s = TopKLogitsWarper(50)(ids, TemperatureLogitsWarper(0.7)(ids, s))
    p = torch.softmax(s, -1)[0].double()
    kept = torch.isfinite(s[0])
    assert bool(kept[draws].all())
    support = kept.nonzero().flatten()
    obs = torch.bincount(draws, minlength=V)[support].double().numpy()
    exp = (p[support] * len(draws)).numpy()
    big = exp >= 5
    obs = np.append(obs[big], obs[~big].sum())
    exp = np.append(exp[big], exp[~big].sum())
    if exp[-1] == 0:
        obs, exp = obs[:-1], exp[:-1]
    chi = stats.chisquare(obs, exp * obs.sum() / exp.sum())
    print('chi-square over %d bins: stat %.1f, p = %.3f' % (len(obs), chi.statistic, chi.pvalue))
    assert chi.pvalue > 1e-3


def _gen(eng, ids, images, boxes, **kw):
    return eng.generate(ids.to(DEV), images, boxes, **kw).cpu()


def test_graphed_sampler_equals_eager_and_is_seeded(eng2):
    """generate with sampling: the CUDA-graph loop (sampler captured) and the eager loop give the same tokens at the
    same seed; a second run repeats them, another seed differs; the Philox counter advances once per replay."""
    cfg, eng = eng2[:2]
    ids, images, boxes = make_inputs(cfg, 2, [1, 2], 20, seed=3)
    images = images.to(torch.bfloat16)
    kw = dict(max_new_tokens=12, do_sample=True, temperature=0.7, top_k=50)
    a = _gen(eng, ids, images, boxes, generator=torch.Generator().manual_seed(1), **kw)
    b = _gen(eng, ids, images, boxes, generator=torch.Generator().manual_seed(1), use_graph=False, **kw)
    c = _gen(eng, ids, images, boxes, generator=torch.Generator().manual_seed(1), **kw)
    d = _gen(eng, ids, images, boxes, generator=torch.Generator().manual_seed(2), **kw)
    assert torch.equal(a, b) and torch.equal(a, c)
    assert not torch.equal(a, d)
    torch.manual_seed(7)
    e = _gen(eng, ids, images, boxes, **kw)
    torch.manual_seed(7)
    assert torch.equal(e, _gen(eng, ids, images, boxes, **kw))
    # the stepper on its own: each replay selects into its ids and advances the counter
    B, L = ids.shape
    cache = KVCache(cfg, B, L + 8, DEV)
    logits = eng.forward(ids.to(DEV), images.to(DEV), boxes, last_only=True, cache=cache)
    smp = Sampler(B, DEV, greedy=False, temperature=0.7, top_k=50, seed=11)
    st = GraphedDecode(eng, cache, sampler=smp)
    smp(logits, st.ids)
    smp.advance()
    seen = [st.ids.clone()]
    for n in range(3):
        st.step()
        assert int(smp.rng_step) == n + 2
        seen.append(st.ids.clone())
    # the same steps eagerly, with the same seed
    cache2 = KVCache(cfg, B, L + 8, DEV)
    logits = eng.forward(ids.to(DEV), images.to(DEV), boxes, last_only=True, cache=cache2)
    smp2 = Sampler(B, DEV, greedy=False, temperature=0.7, top_k=50, seed=11)
    tok = torch.empty((B, 1), dtype=torch.int64, device=DEV)
    eager = []
    for n in range(4):
        if n:
            logits = eng.decode_step(tok, cache2)
        smp2(logits, tok)
        smp2.advance()
        eager.append(tok.clone())
    assert torch.equal(torch.cat(seen, 1), torch.cat(eager, 1))


def test_eos_pad_rule_matches_the_host_rule(eng2):
    """Rows that emit eos at different steps: each gets pad afterwards and the loop ends when all have finished --
    the host rule the device rule replaces, applied to the same seeded run without eos."""
    cfg, eng = eng2[:2]
    ids, images, boxes = make_inputs(cfg, 4, [1, 0, 2, 1], 16, seed=9)
    images = images.to(torch.bfloat16)
    L = ids.shape[1]
    kw = dict(max_new_tokens=10, do_sample=True, temperature=1.0, top_k=3)
    free = _gen(eng, ids, images, boxes, generator=torch.Generator().manual_seed(4), **kw)[:, L:]
    best, eos = -1, None
    for t in free.unique().tolist():
        first = [(row == t).nonzero()[0].item() if (row == t).any() else 99 for row in free]
        score = len(set(first) - {99}) * 10 + sum(f < 99 for f in first)
        if score > best:
            best, eos = score, t
    pad = 0
    want, done = free.clone(), torch.zeros(4, dtype=torch.bool)
    stop = free.shape[1]
    for s in range(free.shape[1]):
        want[done, s] = pad
        done |= want[:, s] == eos
        if bool(done.all()):
            stop = s + 1
            break
    for graph in (True, False):
        got = _gen(eng, ids, images, boxes, generator=torch.Generator().manual_seed(4), eos_token_id=eos,
                   pad_token_id=pad, use_graph=graph, **kw)[:, L:]
        assert torch.equal(got, want[:, :stop]), (graph, eos, got, want)


def test_ragged_batch_and_cache_with_sampling(eng2):
    """Sampling on a right-padded batch of prompts of different lengths and on a two-turn cache= conversation:
    top_k = 1 reproduces the greedy tokens, and a full top-k draw runs and records its tokens in the cache."""
    cfg, eng = eng2[:2]
    ids, images, boxes = make_inputs(cfg, 2, [1, 0], 30, seed=13)
    images = images.to(torch.bfloat16)
    B, L = ids.shape
    mask = torch.ones(B, L, dtype=torch.long)
    mask[1, L - 9:] = 0
    g = dict(max_new_tokens=8, attention_mask=mask.to(DEV))
    greedy = _gen(eng, ids, images, boxes, **g)
    top1 = _gen(eng, ids, images, boxes, do_sample=True, temperature=0.7, top_k=1, **g)
    assert torch.equal(greedy, top1)
    samp = _gen(eng, ids, images, boxes, do_sample=True, temperature=0.7, top_k=50, **g)
    assert samp.shape == greedy.shape and torch.equal(samp[:, :L], ids)
    q = torch.randint(3, 32000, (B, 12), generator=torch.Generator().manual_seed(2))
    second = []
    for turn2 in (dict(), dict(do_sample=True, temperature=0.7, top_k=1)):
        cache = KVCache(cfg, B, L + 8, DEV)
        out1 = _gen(eng, ids, images, boxes, max_new_tokens=6, do_sample=True, temperature=0.7, top_k=50, cache=cache,
                    generator=torch.Generator().manual_seed(3))
        assert torch.equal(cache.ids[:, L:L + 5].cpu(), out1[:, L:L + 5])
        ids2 = torch.cat([out1, q], 1)
        second.append(_gen(eng, ids2, images, boxes, max_new_tokens=6, cache=cache, **turn2))
        assert torch.equal(second[-1][:, :ids2.shape[1]], ids2)
    assert torch.equal(second[0], second[1])


def test_seam_sampling_on_both_loops():
    """The demo's model (fp16, boxes bound with partial): do_sample=True, temperature=0.2, top_k=1 returns the greedy
    tokens on both loops; over many seeds the engine loop's first tokens follow the softmax of HF's processed scores
    for the demo call (T = 0.2, HF's default top_k = 50)."""
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopKLogitsWarper
    from tests.test_model_seam_gpu import build_seam_model
    cfg = EngineConfig(image_size=224, vit_layers=24, n_layers=2)
    sd, vit_sd = random_state_dicts(cfg, DEV, seed=37)       # test_demo_style_setup_and_generate_loops' model
    ids, images, boxes = make_inputs(cfg, 1, [2], 24, seed=5)
    model = build_seam_model(cfg, sd, vit_sd, dtype=torch.float16, app_style=True).eval()
    model.orig_forward = model.forward
    model.forward = partial(model.orig_forward, img_metas=[None], bboxes=[boxes[0].to(DEV).half()])
    img = images.half().to(DEV)
    with torch.inference_mode():
        greedy = model.generate(ids.to(DEV), images=img, do_sample=False, max_new_tokens=6)
        for hf in (False, True):
            top1 = model.generate(ids.to(DEV), images=img, do_sample=True, temperature=0.2, top_k=1, max_new_tokens=6,
                                  use_hf_loop=hf, pad_token_id=0)
            assert torch.equal(top1, greedy), hf
        logits = model.orig_forward(input_ids=ids.to(DEV), images=img, bboxes=[boxes[0].to(DEV).half()]).logits[:, -1]
        n = 400
        first = []
        for s in range(n):
            torch.manual_seed(1000 + s)
            first.append(int(model.generate(ids.to(DEV), images=img, do_sample=True, temperature=0.2,
                                            max_new_tokens=1)[0, -1]))
    model.forward = model.orig_forward
    x = torch.zeros((1, 1), dtype=torch.long)
    s = TopKLogitsWarper(50)(x, TemperatureLogitsWarper(0.2)(x, logits.float().cpu()))
    p = torch.softmax(s, -1)[0].double()
    first = torch.tensor(first)
    assert bool(torch.isfinite(s[0, first]).all())
    support = torch.isfinite(s[0]).nonzero().flatten()
    obs = torch.bincount(first, minlength=V)[support].double().numpy()
    exp = (p[support] * n).numpy()
    big = exp >= 5
    obs, exp = np.append(obs[big], obs[~big].sum()), np.append(exp[big], exp[~big].sum())
    if len(obs) > 1:
        chi = stats.chisquare(obs, exp * obs.sum() / exp.sum())
        print('seam first tokens: %d bins, p = %.3f' % (len(obs), chi.pvalue))
        assert chi.pvalue > 1e-3
