"""GPU tests of generate()'s return_dict_in_generate outputs: the scores and logits the selection kernel
(csrc/sample.cu, g4r_sample_tokens_out_*) and the beam kernels (csrc/beam.cu, g4r_beam_step_out_*) write inside the
graphed step, against transformers' own processors and loops."""
import time

import numpy as np
import pytest
import torch

from gpt4roi_b200 import kernels
from gpt4roi_b200.engine import EngineConfig, random_state_dicts
from tests.test_beam_gpu import _hf_beams
from tests.test_engine_gpu import make_inputs
from tests.test_logits_process_cpu import hf_processors
from tests.test_logits_process_gpu import EOS, _history
from tests.test_ragged_decode_gpu import ragged_inputs
from tests.test_sampling_cpu import kept_set
from tests.test_sampling_gpu import eng2, rows   # noqa: F401  (fixtures)
from tests.stop_tokenizer import seeded_tokenizer
from tests.test_stop_strings_cpu import clean_strings
from tests.test_stop_strings_gpu import straddling_stop

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
V = 32006
SEED = 0x5C0_4E5
DTYPES = pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16], ids=['bf16', 'fp16'])
GRID = [(T, k, p) for T in (0.2, 0.7, 1.0) for k in (0, 1, 50, V) for p in (1.0, 0.9, 0.5)]
PROCS = [dict(), dict(repetition_penalty=1.3, no_repeat_ngram_size=3), dict(repetition_penalty=0.8, min_new_tokens=9),
         dict(no_repeat_ngram_size=1), dict(repetition_penalty=1.2, min_length=900)]


def _hf_scores(lg, hist, L, step, greedy, T, k, p, proc):
    """HF's next_token_scores on the CPU: the widened logits through the processors, then the warpers when sampling.
    -> (the scores before the warpers, the scores)."""
    from transformers.generation import logits_process as lp
    ids = hist[:, :L + step].cpu() if hist is not None else torch.zeros(lg.shape[0], 0, dtype=torch.int64)
    pre = hf_processors(L, eos=EOS, **proc)(ids, lg.float().cpu())
    procs = lp.LogitsProcessorList()
    if not greedy:
        if T != 1.0:
            procs.append(lp.TemperatureLogitsWarper(T))
        if k:
            procs.append(lp.TopKLogitsWarper(k))
        if p < 1.0:
            procs.append(lp.TopPLogitsWarper(p))
    return pre, procs(ids, pre.clone())


def _run(lg, greedy, T=1.0, k=0, p=1.0, hist=None, L=0, step=0, proc=None, outputs=True, seed=SEED):
    B = lg.shape[0]
    out = torch.full((B, 1), -1, dtype=torch.int64, device=DEV)
    fin = torch.zeros(B, dtype=torch.int32, device=DEV)
    rng = torch.tensor([step], dtype=torch.int64, device=DEV)
    sc = torch.full((step + 1, B, V), 7.0, device=DEV) if outputs else None
    raw = torch.full((step + 1, B, V), 7.0, device=DEV) if outputs else None
    h = None if hist is None else hist.clone()
    kw = {} if h is None else dict(history=h, L=L, eos_ids=torch.tensor(EOS, dtype=torch.int32, device=DEV), **proc)
    kernels.sample_tokens_out(lg, out, greedy, T, k, p, seed, rng, eos_id=EOS[0], pad_id=0, finished=fin,
                              scores=sc, raw_logits=raw, **kw)
    return out[:, 0].cpu(), fin.cpu(), None if h is None else h.cpu(), sc, raw


def _compare(ours, hf, pre, T, k, p, greedy):
    """Finite values bitwise equal, -inf sets equal; a row whose top-p boundary is within float rounding of a group
    (kept_set's `near`), or whose boundary group of equal values HF's sort splits, may differ in that group only."""
    bad = 0
    for r in range(ours.shape[0]):
        a, b = ours[r], hf[r]
        fa, fb = torch.isfinite(a), torch.isfinite(b)
        both = fa & fb
        assert torch.equal(a[both], b[both]), (r, (a[both] - b[both]).abs().max())
        diff = fa != fb
        if not diff.any():
            continue
        near = False
        if not greedy and p < 1.0:
            near = kept_set(pre[r].double().numpy(), T, k, p)[2]
        lowest = a[fa].min()
        whole_group = bool((fb[diff] == False).all() and (a[diff] == lowest).all())   # noqa: E712
        assert near or whole_group, (r, int(diff.sum()), T, k, p)
        bad += 1
    return bad


@DTYPES
def test_kernel_scores_equal_transformers_processors(rows, dtype):
    """Real and adversarial rows, the T / top_k / top_p grid and greedy, without and with each processor: the written
    scores are transformers' LogitsProcessorList on the CPU fp32 widened rows (finite values bitwise, -inf sets equal
    up to the top-p boundary group), the raw logits the widened logits exactly."""
    lg = rows.to(dtype)
    B, L, step = lg.shape[0], 40, 3
    hist = _history(B, L + 8, seed=9).to(DEV)
    split = 0
    for proc in PROCS:
        h = hist if proc else None
        for greedy, T, k, p in [(True, 1.0, 0, 1.0)] + [(False,) + g for g in GRID]:
            tok, _, _, sc, raw = _run(lg, greedy, T, k, p, h, L, step, proc)
            assert torch.equal(raw[step].cpu(), lg.float().cpu())
            assert (sc[:step] == 7.0).all() and (raw[:step] == 7.0).all()       # only slot *rng_step is written
            pre, want = _hf_scores(lg, h, L, step, greedy, T, k, p, proc)
            split += _compare(sc[step].cpu(), want, pre, T, k, p, greedy)
            if greedy:
                assert torch.equal(tok, want.argmax(-1)), proc
            else:   # the drawn token has a finite score
                assert torch.isfinite(sc[step].cpu().gather(1, tok[:, None])).all(), (proc, T, k, p)
    print('rows with a split top-p boundary group: %d' % split)


@DTYPES
def test_selection_unchanged_by_the_outputs(rows, dtype):
    """With outputs on or off, the same seed selects the same tokens and leaves the same finished flags and history;
    the call without outputs launches the selection-only kernel."""
    lg = rows.to(dtype)
    B, L = lg.shape[0], 40
    hist = _history(B, L + 8, seed=3).to(DEV)
    for proc in PROCS:
        h = hist if proc else None
        for greedy, T, k, p in [(True, 1.0, 0, 1.0), (False, 0.7, 50, 0.9), (False, 1.0, 0, 0.5), (False, 0.2, 0, 1.0)]:
            on = _run(lg, greedy, T, k, p, h, L, 2, proc)
            off = _run(lg, greedy, T, k, p, h, L, 2, proc, outputs=False)
            for a, b in zip(on[:3], off[:3]):
                assert (a is None and b is None) or torch.equal(a, b), (proc, greedy, T, k, p)


def test_no_output_launches_the_same_kernels(rows):
    from torch.profiler import ProfilerActivity, profile
    lg = rows[:4].to(torch.bfloat16)
    hist = _history(4, 48, seed=1).to(DEV)

    def names(fn):
        """The selection kernels fn launches.  Every fn here launches one, so an empty trace is the profiler's (it now
        and then returns one, sometimes several in a row): it is taken again, up to five times in all."""
        for attempt in range(5):
            time.sleep(0.05 * attempt)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(3):
                    fn()
                torch.cuda.synchronize()
            found = sorted({e.name for e in prof.events()
                            if e.device_type.name == 'CUDA' and 'sample_tokens' in e.name})
            if found:
                break
        return found
    out = torch.empty(4, 1, dtype=torch.int64, device=DEV)
    rng = torch.zeros(1, dtype=torch.int64, device=DEV)
    names(lambda: kernels.sample_tokens(lg, out, True))     # the profiler's first session starts its tracer
    for greedy in (True, False):
        plain = names(lambda: kernels.sample_tokens(lg, out, greedy, 0.7, 50, 0.9, 1, rng))
        none = names(lambda: kernels.sample_tokens_out(lg, out, greedy, 0.7, 50, 0.9, 1, rng))
        proc = names(lambda: kernels.sample_tokens_processed(lg, out, greedy, 0.7, 50, 0.9, 1, rng, history=hist,
                                                             L=40, repetition_penalty=1.2, append=False))
        proc_none = names(lambda: kernels.sample_tokens_out(lg, out, greedy, 0.7, 50, 0.9, 1, rng, history=hist, L=40,
                                                            repetition_penalty=1.2, append=False))
        buf = torch.empty(1, 4, V, device=DEV)
        withs = names(lambda: kernels.sample_tokens_out(lg, out, greedy, 0.7, 50, 0.9, 1, rng, scores=buf))
        assert plain == none and proc == proc_none and len(plain) == len(proc) == 1
        assert 'sample_tokens_out_kernel' not in plain[0] + proc[0] and 'sample_tokens_out_kernel' in withs[0]


def test_graphed_replays_fill_successive_slots_bitwise(rows):
    """A CUDA graph of the selection with outputs, replayed 64 times with new logits and the counter advanced, writes
    the same tokens, scores and logits as 64 eager calls."""
    lg = rows[:8].to(torch.bfloat16)
    B, n = 8, 64
    g = torch.Generator(device=DEV).manual_seed(2)
    steps = [(lg.float() + torch.randn(B, V, device=DEV, generator=g) * 0.5).to(torch.bfloat16) for _ in range(n)]
    hist0 = _history(B, 40 + n, seed=4).to(DEV)
    for greedy in (True, False):
        res = []
        for graphed in (False, True):
            src = torch.empty_like(lg)
            out = torch.empty(B, 1, dtype=torch.int64, device=DEV)
            rng = torch.zeros(1, dtype=torch.int64, device=DEV)
            sc = torch.zeros(n, B, V, device=DEV)
            raw = torch.zeros(n, B, V, device=DEV)
            hist = hist0.clone()

            def call():
                kernels.sample_tokens_out(src, out, greedy, 0.7, 50, 0.9, 11, rng, history=hist, L=40,
                                          repetition_penalty=1.2, no_repeat_ngram_size=2, scores=sc, raw_logits=raw)
            toks = []
            if graphed:
                src.copy_(steps[0])
                call()                     # warm-up: slot 0, rewritten by the first replay
                torch.cuda.synchronize()
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    call()
                hist.copy_(hist0)
            for s in range(n):
                src.copy_(steps[s])
                graph.replay() if graphed else call()
                toks.append(out.clone())
                rng.add_(1)
            torch.cuda.synchronize()
            res.append((torch.cat(toks, 1), sc, raw, hist))
        for a, b in zip(*res):
            assert torch.equal(a, b), greedy


# ---------------------------------------------------------------------------------------------------- the loops
@pytest.fixture(scope='module')
def seam():
    from tests.test_model_seam_gpu import build_seam_model
    cfg = EngineConfig(image_size=224, vit_layers=24, n_layers=2)
    sd, vit_sd = random_state_dicts(cfg, DEV, seed=37)
    model = build_seam_model(cfg, sd, vit_sd, dtype=torch.float16, app_style=True).eval()
    return cfg, model


def _close(ours, hf, L, what):
    """Same sequences, one entry per new token on each loop, and every entry close within the near-tie margin of the
    seam tests (3e-2 of the row's spread): the two loops run the same kernels, graphed and ungraphed."""
    assert torch.equal(ours.sequences, hf.sequences), (what, ours.sequences, hf.sequences)
    for name in ('scores', 'logits'):
        a, b = getattr(ours, name), getattr(hf, name)
        assert len(a) == len(b) == ours.sequences.shape[1] - L, (what, name, len(a), len(b))
        for s, (x, y) in enumerate(zip(a, b)):
            _close_entry(x, y, (what, name, s))


def test_engine_loop_equals_hf_loop(seam):
    """Greedy; sampled with processors; N = 3 answers; a left-padded batch; stop strings; a conversation cache: the
    engine loop's GenerateDecoderOnlyOutput against use_hf_loop=True's."""
    from transformers import DynamicCache
    from transformers.generation.utils import GenerateDecoderOnlyOutput
    cfg, model = seam
    ids, images, boxes = make_inputs(cfg, 1, [2], 24, seed=5)
    L = ids.shape[1]
    img = images.half().to(DEV)
    bx = [b.half().to(DEV) for b in boxes]
    out = dict(return_dict_in_generate=True, output_scores=True, output_logits=True)
    cases = [('greedy', dict()),
             ('sampled + processors', dict(do_sample=True, temperature=0.7, top_k=50, top_p=0.9,
                                           repetition_penalty=1.3, no_repeat_ngram_size=3)),
             ('N = 3', dict(do_sample=True, temperature=0.7, num_return_sequences=3))]
    with torch.inference_mode():
        for what, kw in cases:
            a = model.generate(ids.to(DEV), images=img, bboxes=bx, max_new_tokens=12,
                               generator=torch.Generator().manual_seed(1), **out, **kw)
            assert type(a) is GenerateDecoderOnlyOutput and len(a.scores) == a.sequences.shape[1] - L
            if kw.get('do_sample'):
                # HF draws with its own generator: its processors over the engine's tokens, teacher-forced, instead
                hf_scores = _teacher_forced_scores(model, a.sequences, L, img, bx, kw)
                assert len(hf_scores) == len(a.logits)
                for s, (x, y) in enumerate(zip(a.scores, hf_scores)):
                    _close_entry(x, y, (what, s))
                continue
            b = model.generate(ids.to(DEV), images=img, bboxes=bx, max_new_tokens=12, use_hf_loop=True, **out, **kw)
            _close(a, b, L, what)
        # a left-padded batch
        B = 3
        rids, rimages, rboxes, lens = ragged_inputs(cfg, B, 24, seed=81)
        Lr = rids.shape[1]
        shift = Lr - lens
        mask = (torch.arange(Lr)[None] < lens[:, None]).long()
        ids_l = torch.stack([torch.roll(rids[b], int(shift[b])) for b in range(B)])
        mask_l = torch.stack([torch.roll(mask[b], int(shift[b])) for b in range(B)])
        kw = dict(images=rimages.half().to(DEV), bboxes=[b.half().to(DEV) for b in rboxes],
                  attention_mask=mask_l.to(DEV), max_new_tokens=10, pad_token_id=0, **out)
        _close(model.generate(ids_l.to(DEV), **kw), model.generate(ids_l.to(DEV), use_hf_loop=True, **kw), Lr, 'ragged')
        # stop strings: one that straddles two of the greedy run's tokens
        tok = seeded_tokenizer(32000, seed=5)
        base = model.generate(ids.to(DEV), images=img, bboxes=bx, max_new_tokens=12)[0, L:].cpu()
        stop, at = straddling_stop(clean_strings(tok), base, first=2)
        kw = dict(images=img, bboxes=bx, max_new_tokens=12, stop_strings=[stop], tokenizer=tok, **out)
        a = model.generate(ids.to(DEV), **kw)
        _close(a, model.generate(ids.to(DEV), use_hf_loop=True, **kw), L, 'stop strings')
        assert a.sequences.shape[1] == L + at + 1
        # a conversation cache: the caller's cache comes back as past_key_values
        pkv = DynamicCache()
        a = model.generate(ids.to(DEV), images=img, bboxes=bx, max_new_tokens=8, past_key_values=pkv, **out)
        assert a.past_key_values is pkv and len(a.scores) == 8
        b = model.generate(ids.to(DEV), images=img, bboxes=bx, max_new_tokens=8, use_hf_loop=True, **out)
        _close(a, b, L, 'conversation cache')


def _teacher_forced_scores(model, seqs, L, img, bx, kw):
    """HF's next_token_scores for a given continuation: the seam's forward over each prefix, through the processors
    GenerationMixin builds for kw (the warpers included)."""
    from gpt4roi_b200.spi_llava import _generation_config
    gc = _generation_config(model, dict(kw, max_new_tokens=seqs.shape[1] - L))
    procs = model._get_logits_processor(gc, input_ids_seq_length=L, device='cpu', model_kwargs={})
    R = seqs.shape[0]
    n_img = R // img.shape[0]
    images = img.repeat_interleave(n_img, 0)
    boxes = [b for b in bx for _ in range(n_img)]
    res = []
    for s in range(seqs.shape[1] - L):
        logits = model(input_ids=seqs[:, :L + s], images=images, bboxes=boxes).logits[:, -1].float().cpu()
        res.append(procs(seqs[:, :L + s].cpu(), logits))
    return res


def _close_entry(x, y, what):
    x, y = x.float().cpu(), y.float().cpu()
    fx, fy = torch.isfinite(x), torch.isfinite(y)
    assert (fx != fy).float().mean() < 1e-3, what
    both = fx & fy
    assert ((x[both] - y[both]).abs() <= 3e-2 * y[both].std()).all(), (what, (x[both] - y[both]).abs().max())


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16], ids=['bf16', 'fp16_demo'])
def test_beam_outputs_equal_hf_loop(dtype):
    """Beam search: sequences and beam_indices equal to HF's, sequences_scores and every step's scores within 1e-5,
    and HF's identity compute_transition_scores(..., normalize_logits=False).sum(1) / len ** length_penalty ==
    sequences_scores within 1e-4; graphed == eager bitwise."""
    from transformers.generation.utils import GenerateBeamDecoderOnlyOutput
    from tests.test_model_seam_gpu import build_seam_model
    cfg = EngineConfig(image_size=224, vit_layers=24, n_layers=2)
    sd, vit_sd = random_state_dicts(cfg, DEV, seed=37)
    model = build_seam_model(cfg, sd, vit_sd, dtype=dtype, app_style=dtype == torch.float16).eval()
    ids, images, boxes = make_inputs(cfg, 2, [2, 1], 20, seed=5)
    B, L = ids.shape
    act = torch.float16 if dtype == torch.float16 else torch.float32
    img = images.to(DEV, act)
    bx = [b.to(DEV) for b in boxes]
    eng = model._get_engine(torch.device(DEV))
    free = eng.generate(ids.to(DEV), img, bx, max_new_tokens=8, num_beams=2, use_graph=False).cpu()
    eos = int(free[:, L + 1:].flatten().mode().values)
    with torch.inference_mode():
        for N, nrs, lp in ((2, 1, 1.0), (4, 4, 0.5), (3, 2, 1.5)):
            kw = dict(input_ids=ids.to(DEV), images=img, bboxes=bx, max_new_tokens=10, num_beams=N,
                      num_return_sequences=nrs, length_penalty=lp, eos_token_id=eos, pad_token_id=0, do_sample=False,
                      return_dict_in_generate=True, output_scores=True, output_logits=True)
            hf = _hf_beams(model, **kw)
            ours = model.generate(**kw)
            assert type(ours) is GenerateBeamDecoderOnlyOutput
            assert torch.equal(ours.sequences.cpu(), hf.sequences.cpu()), (N, nrs)
            assert torch.equal(ours.beam_indices.cpu(), hf.beam_indices.cpu().to(torch.int32)), (N, nrs)
            assert torch.allclose(ours.sequences_scores.cpu(), hf.sequences_scores.cpu(), atol=1e-5, rtol=0)
            assert len(ours.scores) == len(hf.scores) == len(ours.logits)
            for x, y in zip(ours.scores, hf.scores):
                assert torch.allclose(x.cpu(), y.cpu(), atol=1e-5, rtol=0)
            for x, y in zip(ours.logits, hf.logits):
                assert torch.allclose(x.cpu(), y.float().cpu(), atol=1e-5, rtol=0)
            ts = model.compute_transition_scores(ours.sequences, ours.scores, ours.beam_indices, normalize_logits=False)
            length = (ours.beam_indices >= 0).sum(1)
            assert torch.allclose(ts.sum(1).cpu() / length.cpu().float() ** lp, ours.sequences_scores.cpu(), atol=1e-4,
                                  rtol=0)
            kw2 = {k: v for k, v in kw.items() if k not in ('input_ids', 'images', 'bboxes', 'do_sample')}
            eager = eng.generate(ids.to(DEV), img, bx, use_graph=False, **kw2)
            graphed = eng.generate(ids.to(DEV), img, bx, use_graph=True, **kw2)
            for k in ('sequences', 'sequences_scores', 'beam_indices'):
                assert torch.equal(eager[k], graphed[k]), k
            for k in ('scores', 'logits'):
                assert all(torch.equal(a, b) for a, b in zip(eager[k], graphed[k])), k
