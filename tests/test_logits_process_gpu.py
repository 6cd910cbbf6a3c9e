"""GPU tests of transformers' history-dependent logits processors on the device (csrc/sample.cu:
g4r_sample_tokens_proc_*, kernels.sample_tokens_processed) and in the decode loop: greedy equal to torch.argmax of HF's
processed fp32 scores bit for bit, draws equal to the float64 restatement of tests/test_sampling_gpu.py on the
processed scores, the distribution against HF's processed softmax, the history append, and the engine loop against
transformers' own loop through the model seam."""
from functools import partial

import numpy as np
import pytest
import torch
from scipy import stats

from gpt4roi_b200 import kernels
from gpt4roi_b200.engine import EngineConfig, KVCache, random_state_dicts
from gpt4roi_b200.spi_llava import stop_strings_from_tokenizer
from tests.stop_tokenizer import seeded_tokenizer
from tests.test_engine_gpu import make_inputs
from tests.test_logits_process_cpu import hf_processors
from tests.test_ragged_decode_gpu import ragged_inputs
from tests.test_sampling_cpu import hf_kept, uniforms
from tests.test_sampling_gpu import _predict_row
from tests.test_stop_strings_cpu import clean_strings
from tests.test_stop_strings_gpu import expected, straddling_stop, unused_id

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
V = 32006
SEED = 0x0DDB_A11_5EED
EOS = [2, 31999]


def _rows(B, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, V, generator=g) * torch.tensor([0.5, 2.0, 4.0])[torch.arange(B) % 3][:, None]


def _history(B, n, seed):
    """B rows of n ids with heavy repetition: a short motif repeated, 20 % random ids, a few motif ids near the top
    logits."""
    g = torch.Generator().manual_seed(seed)
    h = torch.randint(0, 400, (B, 7), generator=g).repeat(1, n // 7 + 1)[:, :n].clone()
    noise = torch.rand(B, n, generator=g) < 0.2
    h[noise] = torch.randint(0, V, (int(noise.sum()),), generator=g)
    return h


def _processed(lg, hist, L, step, **proc):
    """HF's processors on the fp32-widened logits (CPU, as GenerationMixin._sample applies them)."""
    return hf_processors(L, eos=EOS, **proc)(hist[:, :L + step].cpu(), lg.float().cpu())


def _call(lg, hist, L, step, greedy, T=1.0, k=0, p=1.0, seed=SEED, append=True, **proc):
    out = torch.full((lg.shape[0], 1), -1, dtype=torch.int64, device=DEV)
    rng = torch.tensor([step], dtype=torch.int64, device=DEV)
    kernels.sample_tokens_processed(lg, out, greedy, T, k, p, seed, rng, history=hist, L=L,
                                    eos_ids=torch.tensor(EOS, dtype=torch.int32, device=DEV), append=append, **proc)
    return out[:, 0].cpu()


PROCS = [dict(repetition_penalty=1.3, no_repeat_ngram_size=3), dict(repetition_penalty=0.8, min_new_tokens=5),
         dict(no_repeat_ngram_size=1), dict(repetition_penalty=1.2, no_repeat_ngram_size=2, min_length=900)]


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16], ids=['bf16', 'fp16'])
@pytest.mark.parametrize('B', [1, 8])
def test_greedy_is_argmax_of_transformers_processed_scores(dtype, B):
    """Histories of 0 to 4000 ids (prompt lengths 0..800, steps 0..3200): the kernel's token is torch.argmax of HF's
    processed fp32 scores, bit for bit, and it lands in history[b, L + step]."""
    for case, (L, step) in enumerate([(0, 0), (1, 0), (700, 0), (706, 24), (800, 1200), (800, 3200)]):
        lg = _rows(B, case).to(dtype).to(DEV)
        for proc in PROCS:
            hist = _history(B, L + step + 1, seed=case).to(DEV)
            hist[:, L + step] = -5
            want = _processed(lg, hist, L, step, **proc).argmax(-1)
            got = _call(lg, hist, L, step, True, **proc)
            assert torch.equal(got, want), (L, step, proc, got, want)
            assert torch.equal(hist[:, L + step].cpu(), got)
            again = _call(lg, hist, L, step, True, append=False, **proc)
            assert torch.equal(again, got)


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16], ids=['bf16', 'fp16'])
def test_greedy_ties_and_bans_of_the_arg_max(dtype):
    """Crafted rows: a penalised value equal to an unpenalised one (the first index wins, whichever set it is in), a
    penalised value that would round onto its neighbour in the 16-bit type, and an n-gram ban of the arg-max."""
    lg = _rows(4, 9).to(dtype)
    lg[:, :] = lg.clamp(-3, 3)
    hist = torch.zeros((4, 12), dtype=torch.int64)
    # row 0: id 50 (penalised, 8.0 / 2 = 4.0) ties id 900 (4.0); 50 comes first
    lg[0, 50], lg[0, 900] = 8.0, 4.0
    hist[0, :4] = torch.tensor([50, 50, 7, 8])
    # row 1: the tie the other way round: id 30 (unpenalised 4.0) before id 40 (penalised 8.0 -> 4.0)
    lg[1, 30], lg[1, 40] = 4.0, 8.0
    hist[1, :4] = torch.tensor([40, 9, 40, 9])
    # row 2: 3.5 / 1.0625 = 3.294.. is not a 16-bit value; an unpenalised id holds its nearest 16-bit value
    lg[2, 11] = 3.5
    lg[2, 12] = torch.tensor(3.5 / 1.0625).to(dtype)
    hist[2, :4] = torch.tensor([11, 5, 6, 11])
    # row 3: n-gram (5, 6, 77) seen; the history ends in (5, 6); 77 is the arg-max and gets banned
    lg[3, 77] = 9.0
    hist[3, :6] = torch.tensor([5, 6, 77, 1, 5, 6])
    lg, hist = lg.to(DEV), hist.to(DEV)
    for L, proc in ((4, dict(repetition_penalty=2.0)), (4, dict(repetition_penalty=1.0625)),
                    (6, dict(no_repeat_ngram_size=3))):
        want = _processed(lg, hist, L, 0, **proc).argmax(-1)
        got = _call(lg, hist.clone(), L, 0, True, **proc)
        assert torch.equal(got, want), (proc, got, want)
    got = _call(lg, hist.clone(), 4, 0, True, repetition_penalty=2.0)
    assert got[0] == 50 and got[1] == 30
    got = _call(lg, hist.clone(), 6, 0, True, no_repeat_ngram_size=3)
    assert got[3] != 77 and _call(lg, hist.clone(), 6, 0, True)[3] == 77


SAMPLE = [(0.7, 0, 1.0), (0.7, 50, 1.0), (1.0, 0, 0.9), (0.2, 50, 0.5), (1.0, 1, 1.0), (0.7, V, 0.9)]


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16], ids=['bf16', 'fp16'])
def test_draws_equal_the_restatement_on_the_processed_scores(dtype):
    """B = 8 rows, histories of 706 to 1730 ids: every draw is the token the numpy Philox + float64 inverse CDF over
    HF's processed scores predicts (draws within 1e-5 of a boundary skipped and counted), it lies in HF's kept set (or
    the boundary group HF's sort splits), never on a banned id; B = 1 draws what row 0 of B = 8 draws; two runs are
    bitwise equal."""
    B = 8
    skipped = checked = 0
    for case, (L, step) in enumerate([(706, 0), (706, 1024), (200, 37)]):
        lg = _rows(B, 20 + case)
        # make penalised ids matter: the motif ids get values among the largest
        hist = _history(B, L + step + 1, seed=30 + case)
        for b in range(B):
            lg[b, hist[b, :20]] = lg[b].max() - torch.rand(20) * 0.5
        lg = lg.to(dtype).to(DEV)
        hist = hist.to(DEV)
        u = uniforms(SEED, step, B)
        for proc in PROCS:
            s = _processed(lg, hist, L, step, **proc).double().numpy()
            orders = [np.lexsort((np.arange(V), -x)) for x in s]
            for T, k, p in SAMPLE:
                got = _call(lg, hist.clone(), L, step, False, T, k, p, **proc)
                assert torch.equal(got, _call(lg, hist.clone(), L, step, False, T, k, p, **proc))
                assert got[0] == _call(lg[:1], hist[:1].clone(), L, step, False, T, k, p, **proc)[0]
                for r in range(B):
                    tok = int(got[r])
                    assert np.isfinite(s[r][tok]), (proc, T, k, p, r)
                    want, amb, keep = _predict_row(s[r], orders[r], T, k, p, u[r])
                    hf = hf_kept(s[r], T, k, p)
                    assert hf[tok] or (keep[tok] and (s[r][hf] == s[r][tok]).any()), (proc, T, k, p, r, tok)
                    if amb:
                        skipped += 1
                        continue
                    checked += 1
                    assert tok == want, (proc, T, k, p, r, tok, want)
    print('%s: %d draws predicted exactly, %d skipped near a boundary' % (dtype, checked, skipped))
    # the rows are built with many processed values close to the maximum, so more draws land near a boundary than on
    # plain rows (tests/test_sampling_gpu.py); the skipped ones still lie in HF's kept set (asserted above)
    assert skipped <= checked // 5


def test_distribution_matches_transformers_processed_softmax():
    """One row, 1024 copies x 64 seeds, repetition_penalty=1.5 and no_repeat_ngram_size=2 on a history whose ids hold
    the top logits: chi-square against the softmax of HF's processed scores (T = 0.7, top_k = 50)."""
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopKLogitsWarper
    row = _rows(1, 3)[0]
    hist1 = torch.randint(0, V, (300,), generator=torch.Generator().manual_seed(4))
    top = row.topk(30).indices
    hist1[::10] = top
    row = row.to(torch.float16)
    B, n = 1024, 64
    lg = row[None].repeat(B, 1).contiguous().to(DEV)
    hist = hist1[None].repeat(B, 1).contiguous().to(DEV)
    proc = dict(repetition_penalty=1.5, no_repeat_ngram_size=2)
    draws = torch.cat([_call(lg, hist, 300, 0, False, 0.7, 50, 1.0, seed=1000 + i, append=False, **proc)
                       for i in range(n)])
    s = _processed(row[None], hist1[None], 300, 0, **proc)
    ids = torch.zeros((1, 1), dtype=torch.long)
    s = TopKLogitsWarper(50)(ids, TemperatureLogitsWarper(0.7)(ids, s))
    p = torch.softmax(s, -1)[0].double()
    kept = torch.isfinite(s[0])
    assert bool(kept[draws].all())
    support = kept.nonzero().flatten()
    obs = torch.bincount(draws, minlength=V)[support].double().numpy()
    exp = (p[support] * len(draws)).numpy()
    big = exp >= 5
    obs, exp = np.append(obs[big], obs[~big].sum()), np.append(exp[big], exp[~big].sum())
    if exp[-1] == 0:
        obs, exp = obs[:-1], exp[:-1]
    chi = stats.chisquare(obs, exp * obs.sum() / exp.sum())
    print('chi-square over %d bins: stat %.1f, p = %.3f' % (len(obs), chi.statistic, chi.pvalue))
    assert chi.pvalue > 1e-3


def test_refusals():
    lg = torch.zeros((2, V), dtype=torch.bfloat16, device=DEV)
    out = torch.empty((2, 1), dtype=torch.int64, device=DEV)
    rng = torch.zeros(1, dtype=torch.int64, device=DEV)
    h = torch.zeros((2, 9000), dtype=torch.int64, device=DEV)
    with pytest.raises(RuntimeError, match='8192'):
        kernels.sample_tokens_processed(lg, out, False, 1.0, rng_step=rng, history=h, L=5, repetition_penalty=1.1)
    with pytest.raises(RuntimeError, match='history'):
        kernels.sample_tokens_processed(lg, out, True, rng_step=rng, history=h[:1], L=5)
    with pytest.raises(RuntimeError, match='rng_step'):
        kernels.sample_tokens_processed(lg, out, True, history=h, L=5)
    kernels.sample_tokens_processed(lg, out, True, rng_step=rng, history=h, L=5, repetition_penalty=1.1)   # greedy: any


# ---------------------------------------------------------------------------------------------------- the loops
LOOP = dict(repetition_penalty=1.3, no_repeat_ngram_size=3, min_new_tokens=8)


@pytest.fixture(scope='module')
def seam():
    from tests.test_model_seam_gpu import build_seam_model
    cfg = EngineConfig(image_size=224, vit_layers=24, n_layers=2)
    sd, vit_sd = random_state_dicts(cfg, DEV, seed=37)
    model = build_seam_model(cfg, sd, vit_sd, dtype=torch.float16, app_style=True).eval()
    return cfg, model


def _no_repeated_ngram(row, L, n):
    """No n-gram that ends in a new token (position >= L) occurs earlier in the row."""
    return all(tuple(row[i - n + 1:i + 1]) not in {tuple(row[j - n + 1:j + 1]) for j in range(n - 1, i)}
               for i in range(max(L, n - 1), len(row)))


def test_engine_loop_equals_hf_loop_single_prompt_and_left_padded_batch(seam):
    cfg, model = seam
    ids, images, boxes = make_inputs(cfg, 1, [2], 24, seed=5)
    L = ids.shape[1]
    img = images.half().to(DEV)
    bx = [b.half().to(DEV) for b in boxes]
    with torch.inference_mode():
        eos = int(model.generate(ids.to(DEV), images=img, bboxes=bx, max_new_tokens=1)[0, -1])
        kw = dict(images=img, bboxes=bx, max_new_tokens=24, eos_token_id=eos, pad_token_id=0, **LOOP)
        ours = model.generate(ids.to(DEV), **kw)
        hf = model.generate(ids.to(DEV), use_hf_loop=True, **kw)
        plain = model.generate(ids.to(DEV), images=img, bboxes=bx, max_new_tokens=24)
    assert torch.equal(ours, hf), (ours[:, L:], hf[:, L:])
    assert ours.shape[1] > L + 8 and int(ours[0, L]) != eos            # the first token would have been eos
    assert _no_repeated_ngram(ours[0].tolist(), L, 3) and not torch.equal(ours[:, :plain.shape[1]], plain)
    # min_length and min_new_tokens together: min_new_tokens takes precedence (HF's min_length = L + min_new_tokens)
    with torch.inference_mode():
        kw = dict(images=img, bboxes=bx, max_new_tokens=24, eos_token_id=eos, pad_token_id=0, min_length=L + 20,
                  min_new_tokens=2, repetition_penalty=1.3)
        ours = model.generate(ids.to(DEV), **kw)
        hf = model.generate(ids.to(DEV), use_hf_loop=True, **kw)
    assert torch.equal(ours, hf), (ours[:, L:], hf[:, L:])
    B = 3
    ids, images, boxes, lens = ragged_inputs(cfg, B, 24, seed=81)
    L = ids.shape[1]
    shift = L - lens
    mask = (torch.arange(L)[None] < lens[:, None]).long()
    ids_l = torch.stack([torch.roll(ids[b], int(shift[b])) for b in range(B)])
    mask_l = torch.stack([torch.roll(mask[b], int(shift[b])) for b in range(B)])
    img, bx = images.half().to(DEV), [b.half().to(DEV) for b in boxes]
    with torch.inference_mode():
        kw = dict(images=img, bboxes=bx, attention_mask=mask_l.to(DEV), max_new_tokens=16, pad_token_id=0, **LOOP)
        ours = model.generate(ids_l.to(DEV), **kw)
        hf = model.generate(ids_l.to(DEV), use_hf_loop=True, **kw)
    assert torch.equal(ours, hf), (ours[:, L:], hf[:, L:])


def test_graphed_equals_eager_and_neutral_is_the_current_loop(seam):
    cfg, model = seam
    eng = model._get_engine(torch.device(DEV))
    ids, images, boxes = make_inputs(cfg, 2, [1, 2], 24, seed=11)
    img = images.half().to(DEV)
    L = ids.shape[1]
    for kw in (dict(LOOP), dict(LOOP, do_sample=True, temperature=0.7, top_k=50),
               dict(do_sample=True, temperature=1.0, repetition_penalty=0.9, no_repeat_ngram_size=1)):
        a, b = (eng.generate(ids.to(DEV), img, boxes, max_new_tokens=20, use_graph=g, eos_token_id=2,
                             generator=torch.Generator().manual_seed(3), **kw) for g in (True, False))
        assert torch.equal(a, b), kw
        for r in a.tolist():
            assert _no_repeated_ngram(r, L, kw['no_repeat_ngram_size']), kw
    # neutral parameters: bitwise the loop without them, and the same kernels
    from torch.profiler import ProfilerActivity, profile

    def kernels_of(**kw):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = eng.generate(ids.to(DEV), img, boxes, max_new_tokens=6, use_graph=False, eos_token_id=2, **kw)
            torch.cuda.synchronize()
        return out, sorted(e.name for e in prof.events() if e.device_type.name == 'CUDA' and 'sample_tokens' in e.name)
    base, kb = kernels_of()
    same, ks = kernels_of(repetition_penalty=1.0, no_repeat_ngram_size=0, min_length=0, min_new_tokens=0)
    _, kp = kernels_of(repetition_penalty=1.2)
    assert torch.equal(base, same) and kb == ks and len(kb) == len(kp) > 0
    assert not any('<true>' in n for n in kb) and any('<true>' in n for n in kp)
    for gk in (dict(), dict(repetition_penalty=1.0, min_new_tokens=0)):
        g = eng.generate(ids.to(DEV), img, boxes, max_new_tokens=12, **gk)
        assert torch.equal(g, eng.generate(ids.to(DEV), img, boxes, max_new_tokens=12))


def test_several_answers_per_prompt_match_the_expanded_batch(seam):
    """num_return_sequences=4 with processors: the same seed's run on input_ids.repeat_interleave(4, 0) gives the same
    rows up to the attention's summation order -- here: identical first tokens (drawn from equal prefill logits) and
    most rows identical throughout -- and every row obeys its own no-repeat rule."""
    cfg, model = seam
    eng = model._get_engine(torch.device(DEV))
    ids, images, boxes = make_inputs(cfg, 1, [2], 24, seed=23)
    L = ids.shape[1]
    img = images.half().to(DEV)
    kw = dict(max_new_tokens=16, do_sample=True, temperature=0.7, top_k=50, repetition_penalty=1.3,
              no_repeat_ngram_size=2)
    grouped = eng.generate(ids.to(DEV), img, boxes, num_return_sequences=4, generator=torch.Generator().manual_seed(5),
                           **kw).cpu()
    expanded = eng.generate(ids.repeat_interleave(4, 0).to(DEV), img.repeat_interleave(4, 0),
                            [b for b in boxes for _ in range(4)], generator=torch.Generator().manual_seed(5), **kw).cpu()
    assert grouped.shape == expanded.shape == (4, L + 16)
    assert torch.equal(grouped[:, :L + 1], expanded[:, :L + 1])
    assert sum(torch.equal(g, e) for g, e in zip(grouped, expanded)) >= 2
    for r in grouped[:, L:].tolist():
        grams = [tuple(r[i:i + 2]) for i in range(len(r) - 1)]
        assert len(grams) == len(set(grams))


def test_stop_strings_cut_the_same_seed_run(seam):
    cfg, model = seam
    eng = model._get_engine(torch.device(DEV))
    tok = seeded_tokenizer(32000, seed=5)
    strings = clean_strings(tok)
    ids, images, boxes = make_inputs(cfg, 2, [1, 2], 24, seed=13)
    L = ids.shape[1]
    img = images.half().to(DEV)
    kw = dict(max_new_tokens=20, do_sample=True, temperature=1.0, top_k=50, **LOOP)
    base = eng.generate(ids.to(DEV), img, boxes, generator=torch.Generator().manual_seed(7), eos_token_id=2,
                        **kw)[:, L:].cpu()
    stop, at = straddling_stop(strings, base[0], first=4)
    want, steps = expected(strings, [stop], ids, torch.full((2,), L), base, 0)
    out = eng.generate(ids.to(DEV), img, boxes, generator=torch.Generator().manual_seed(7), eos_token_id=unused_id(base),
                       length_eos_ids=[2], pad_token_id=0, stop_strings=stop_strings_from_tokenizer(tok, [stop]),
                       **kw)[:, L:].cpu()
    # the pads of finished row 0 enter its own history only, so row 1 runs as without the stop string
    assert steps[0] == at and torch.equal(out[0, :at + 1], base[0, :at + 1]), (out, base)
    if steps[1] is None:
        assert torch.equal(out[1], base[1])
    assert torch.equal(out, want[:, :out.shape[1]])


def test_conversation_cache_history_is_the_whole_submitted_prompt(seam):
    """Turn 2 on a conversation cache with no_repeat_ngram_size=1: no new token repeats any id of the whole submitted
    prompt (turn 1 included) or another new token; graphed == eager on equal caches."""
    cfg, model = seam
    eng = model._get_engine(torch.device(DEV))
    ids1, images, boxes = make_inputs(cfg, 1, [2], 40, seed=17)
    L1 = ids1.shape[1]
    img = images.half().to(DEV)
    outs = []
    for graph in (True, False):
        cache = KVCache(eng.cfg, 1, L1 + 96, DEV)
        out1 = eng.generate(ids1.to(DEV), img, boxes, max_new_tokens=8, cache=cache, use_graph=graph, **LOOP).cpu()
        q = torch.randint(3, 32000, (1, 20), generator=torch.Generator().manual_seed(19))
        ids2 = torch.cat([out1, q], 1)
        out2 = eng.generate(ids2.to(DEV), img, boxes, max_new_tokens=12, cache=cache, use_graph=graph,
                            no_repeat_ngram_size=1).cpu()
        new = out2[0, ids2.shape[1]:].tolist()
        assert not set(new) & set(ids2[0].tolist()) and len(set(new)) == len(new)
        outs.append(out2)
    assert torch.equal(outs[0], outs[1])


def test_seam_both_loops_with_model_config_processors(seam):
    """The processors resolved from the model's generation config reach the engine loop: equal to the HF loop."""
    cfg, model = seam
    ids, images, boxes = make_inputs(cfg, 1, [2], 24, seed=29)
    img = images.half().to(DEV)
    fwd = model.forward
    model.forward = partial(fwd, img_metas=[None], bboxes=[boxes[0].to(DEV).half()])
    gc = model.generation_config
    gc.repetition_penalty, gc.no_repeat_ngram_size = 1.3, 3
    try:
        with torch.inference_mode():
            ours = model.generate(ids.to(DEV), images=img, max_new_tokens=16)
            hf = model.generate(ids.to(DEV), images=img, max_new_tokens=16, use_hf_loop=True)
    finally:
        gc.repetition_penalty, gc.no_repeat_ngram_size = 1.0, 0
        model.forward = fwd
    assert torch.equal(ours, hf), (ours, hf)
