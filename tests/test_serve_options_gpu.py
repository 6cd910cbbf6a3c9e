"""GPU tests of per-request options in continuous batching: the per-row processed selection
(kernels.sample_tokens_rows_processed) against sample_tokens_processed / sample_tokens on each row alone, the per-row stop
lookup (kernels.stop_step_rows) against the host lookup, and ContinuousBatcher(request_options=True) on the real engine
-- each request equals generate() alone with the same options, whatever its neighbours, slot or earlier tenant; neutral
rows select as on a plain batcher; a follow-up turn under prefix reuse equals generate(cache=); the graph is captured
once; the model seam equals model.generate."""
import pytest
import torch

from gpt4roi_b200 import engine as E
from gpt4roi_b200 import kernels
from gpt4roi_b200.engine import ContinuousBatcher, EngineConfig, KVCache, StopStrings, _stop_lookup
from tests.test_serve_gpu import DEV, LD, V, _request, _rows_case, _tokens, eng  # noqa: F401  (eng: the fixture)
from tests.test_serve_prefix_gpu import _turn1, _turn2

pytestmark = pytest.mark.gpu
I32 = torch.int32
SLOTS, MAX_LEN = 4, 384     # the batcher equals generate() alone bitwise here (tests/test_serve_gpu.py)


# ---- the kernels ----------------------------------------------------------------------------------------------------

def _proc_case(S, seed, ld_h=256):
    """Per-row processors (about a third of the rows neutral), prompt lengths and histories over a small alphabet, so
    that the penalties, n-gram bans and suppressed eos ids all touch ids the logits rank high."""
    g = torch.Generator().manual_seed(seed)
    hist = torch.randint(0, 40, (S, ld_h), generator=g)
    plen = torch.randint(4, 160, (S,), generator=g).to(I32)
    pen = torch.tensor([1.0, 1.3, 0.7, 2.0])[torch.randint(0, 4, (S,), generator=g)]
    ngram = torch.tensor([0, 1, 2, 3])[torch.randint(0, 4, (S,), generator=g)].to(I32)
    minl = torch.randint(0, 300, (S,), generator=g).to(I32) * (torch.rand(S, generator=g) < 0.5)
    minn = torch.randint(0, 40, (S,), generator=g).to(I32) * (torch.rand(S, generator=g) < 0.5)
    eos = torch.randint(0, 40, (S, kernels.PROC_ROW_EOS), generator=g).to(I32)
    n_eos = torch.randint(0, kernels.PROC_ROW_EOS + 1, (S,), generator=g).to(I32)
    neutral = torch.rand(S, generator=g) < 0.33
    neutral[0] = False                 # row 0 (always active) runs the processed selection, row 1 the plain one
    neutral[1:2] = True
    pen[0] = 1.3
    pen[neutral], ngram[neutral], n_eos[neutral] = 1.0, 0, 0
    return hist, plen, pen, ngram, minl, minn, eos, n_eos


def _is_neutral(pen, ngram, minl, minn, n_eos):
    return pen == 1.0 and ngram == 0 and not ((minl or minn) and n_eos)


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('S', [1, 8, 16, 64])
def test_rows_processed_kernel_equals_each_row_alone(S, dtype):
    logits, p, active = _rows_case(S, dtype, seed=40 + S + (dtype == torch.float16))
    active[1:2] = 1
    hist, plen, pen, ngram, minl, minn, eos, n_eos = _proc_case(S, seed=S)
    ld_h = hist.shape[1]
    p['step'] = torch.stack([torch.randint(0, ld_h - int(plen[r]), (1,)) for r in range(S)])[:, 0]
    lg = logits[:, :V].to(DEV)
    want, neutral_rows = [], 0
    for r in range(S):
        if not active[r]:
            want.append(None)
            continue
        out = torch.empty(1, dtype=torch.int64, device=DEV)
        step = torch.tensor([int(p['step'][r])], dtype=torch.int64, device=DEV)
        rule = (bool(p['greedy'][r]), float(p['temperature'][r]), int(p['top_k'][r]), float(p['top_p'][r]),
                int(p['seed'][r]), step)
        if _is_neutral(float(pen[r]), int(ngram[r]), int(minl[r]), int(minn[r]), int(n_eos[r])):
            neutral_rows += 1
            kernels.sample_tokens(lg[r:r + 1], out, *rule)
        else:
            h = hist[r:r + 1].to(DEV)
            kernels.sample_tokens_processed(
                lg[r:r + 1], out, *rule, history=h, L=int(plen[r]), repetition_penalty=float(pen[r]),
                no_repeat_ngram_size=int(ngram[r]), min_length=int(minl[r]), min_new_tokens=int(minn[r]),
                eos_ids=eos[r, :int(n_eos[r])].to(DEV) if int(n_eos[r]) else None)
        want.append(int(out))
    assert neutral_rows >= (S > 1)
    eos_id = torch.tensor([w if (w is not None and r % 2 == 0) else -1 for r, w in enumerate(want)], dtype=I32)
    d = {k: v.to(DEV) for k, v in p.items()}
    out = torch.full((S, 1), -7, dtype=torch.int64, device=DEV)
    fin = torch.zeros(S, dtype=I32, device=DEV)
    lens0 = torch.randint(10, 300, (S,), dtype=I32)
    lens, h = lens0.to(DEV), hist.to(DEV)
    kernels.sample_tokens_rows_processed(lg, out, d['greedy'], d['temperature'], d['top_k'], d['top_p'], d['seed'],
                                         d['step'], eos_id.to(DEV), active.to(DEV), fin, lens, h, plen.to(DEV),
                                         pen.to(DEV), ngram.to(DEV), minl.to(DEV), minn.to(DEV), eos.to(DEV),
                                         n_eos.to(DEV))
    out, fin, step, lens, h = out.cpu()[:, 0], fin.cpu(), d['step'].cpu(), lens.cpu(), h.cpu()
    on = active.bool()
    for r in range(S):
        if on[r]:
            assert int(out[r]) == want[r], (r, int(out[r]), want[r])
            assert int(fin[r]) == int(int(eos_id[r]) == want[r]), r
            at = int(plen[r] + p['step'][r])
            neutral = _is_neutral(float(pen[r]), int(ngram[r]), int(minl[r]), int(minn[r]), int(n_eos[r]))
            expect = hist[r].clone()
            if not neutral:
                expect[at] = want[r]
            assert torch.equal(h[r], expect), r
        else:
            assert int(out[r]) == -7 and int(fin[r]) == 0 and torch.equal(h[r], hist[r]), r
    assert torch.equal(step, p['step'] + on.to(torch.int64))
    assert torch.equal(lens, lens0 + on.to(I32))


def test_stop_step_rows_equals_the_host_lookup_per_row():
    g = torch.Generator().manual_seed(3)
    B, V_tok = 64, 500
    tables = []
    for b in range(B):
        if b % 5 == 3:
            tables.append(None)
            continue
        n = int(torch.randint(1, 40, (1,), generator=g))
        t = torch.randint(0, n, (V_tok + 1, n), generator=g)
        t = t - 32768 * (torch.rand(V_tok + 1, n, generator=g) < 0.1).to(torch.int64)
        tables.append(t.to(torch.int16))
    dev_tables = [None if t is None else t.to(DEV) for t in tables]
    ptrs = torch.tensor([0 if t is None else t.data_ptr() for t in dev_tables], dtype=torch.int64, device=DEV)
    n_states = torch.tensor([1 if t is None else t.shape[1] for t in tables], dtype=I32)
    state0 = torch.tensor([int(torch.randint(0, int(n), (1,), generator=g)) for n in n_states], dtype=I32)
    ids = torch.randint(-3, V_tok + 20, (B,), generator=g)
    active = (torch.rand(B, generator=g) < 0.8).to(I32)
    fin0 = (torch.rand(B, generator=g) < 0.2).to(I32)
    state, fin = state0.to(DEV), fin0.to(DEV)
    kernels.stop_step_rows(ids.to(DEV), ptrs, n_states.to(DEV), V_tok, active.to(DEV), state, fin)
    state, fin = state.cpu(), fin.cpu()
    hits = 0
    for b in range(B):
        if active[b] and not fin0[b] and tables[b] is not None:
            new, hit = _stop_lookup(tables[b], ids[b:b + 1], state0[b:b + 1].to(torch.int64))
            assert (int(state[b]), int(fin[b])) == (int(new[0]), int(hit[0])), b
            hits += int(hit[0])
        else:
            assert (int(state[b]), int(fin[b])) == (int(state0[b]), int(fin0[b])), b
    assert hits > 0


# ---- the batcher on the engine --------------------------------------------------------------------------------------

def _tables(stops):
    """Stop tables over the seeded 32000-piece vocabulary, padded with ids it does not hold to the engine's 32006."""
    from tests.stop_tokenizer import seeded_tokenizer
    from tests.test_stop_strings_cpu import clean_strings
    strings = clean_strings(seeded_tokenizer(32000, seed=5))
    strings += [None] * (V - len(strings))
    return strings, (StopStrings(strings, stops) if stops is not None else None)


OPTS = [dict(repetition_penalty=1.3), dict(no_repeat_ngram_size=2), dict(repetition_penalty=0.8, min_new_tokens=4),
        dict(no_repeat_ngram_size=1, repetition_penalty=1.1), dict(), dict(min_new_tokens=6)]


def _spec(eng, i, n, sample):
    spec = _request(eng, i, n, sample)
    spec.update(OPTS[i % len(OPTS)])
    if 'min_new_tokens' in spec:
        spec['eos_token_id'] = int(torch.randint(0, 32000, (1,), generator=torch.Generator().manual_seed(i)))
    return spec


def _alone(eng, spec, i, **kw):
    if spec.get('do_sample'):
        torch.manual_seed(100 + i)
    args = {k: v for k, v in spec.items() if k not in ('input_ids', 'images', 'bboxes')}
    out = eng.generate(spec['input_ids'].to(DEV), spec['images'], spec['bboxes'],
                       cache=KVCache(eng.cfg, 1, MAX_LEN, DEV), **dict(args, **kw))
    return out[0, spec['input_ids'].shape[1]:].cpu()


def _submit(b, spec, i, **kw):
    if spec.get('do_sample'):
        torch.manual_seed(100 + i)
    return b.submit(**dict(spec, **kw))


def test_each_request_equals_generate_alone_with_its_options(eng):
    specs = [_spec(eng, i, 10 + 3 * i, i % 3 == 1) for i in range(8)]
    strings, _ = _tables(None)
    # request 5 stops on a string straddling two of its plain tokens, request 6 on one that never occurs
    from tests.test_stop_strings_gpu import straddling_stop
    stop, at = straddling_stop(strings, _alone(eng, specs[5], 5), first=2)
    stops = {5: _tables([stop])[1], 6: _tables(['ab#.xyab#.xy'])[1]}
    b = ContinuousBatcher(eng, SLOTS, MAX_LEN, request_options=True)
    reqs = []
    for i, spec in enumerate(specs):
        reqs.append(_submit(b, spec, i, stop_strings=stops.get(i)))
        if i % 2:
            b.step()
    b.run()
    differs = 0
    for i, (spec, r) in enumerate(zip(specs, reqs)):
        want = _alone(eng, spec, i, stop_strings=stops.get(i))
        assert torch.equal(_tokens(r), want), (i, _tokens(r), want)
        plain = {k: v for k, v in spec.items() if k not in ('repetition_penalty', 'no_repeat_ngram_size',
                                                               'min_new_tokens')}
        differs += not torch.equal(want, _alone(eng, plain, i))
    assert differs >= 3
    assert _tokens(reqs[5]).shape[0] == at + 1


@pytest.mark.parametrize('slots', [8, 16])
def test_greedy_requests_with_options_follow_generate_alone_up_to_a_near_tie(eng, slots):
    """The margin rule of tests/test_serve_gpu.py::test_greedy_requests_follow_generate_alone_up_to_a_near_tie, on the
    processed scores generate() selects from."""
    specs = [_spec(eng, i, 16 + 2 * i, False) for i in range(slots)]
    b = ContinuousBatcher(eng, slots, MAX_LEN, request_options=True)
    reqs = []
    for i, spec in enumerate(specs):
        reqs.append(b.submit(**spec))
        if i % 3 == 2:
            b.step()
    b.run()
    for i, (spec, r) in enumerate(zip(specs, reqs)):
        L = spec['input_ids'].shape[1]
        args = {k: v for k, v in spec.items() if k not in ('input_ids', 'images', 'bboxes')}
        res = eng.generate(spec['input_ids'].to(DEV), spec['images'], spec['bboxes'],
                           cache=KVCache(eng.cfg, 1, MAX_LEN, DEV), output_scores=True, return_dict_in_generate=True,
                           **args)
        want, got = res['sequences'][0, L:].cpu(), _tokens(r)
        n = min(got.shape[0], want.shape[0])
        diff = (got[:n] != want[:n]).nonzero()
        if len(diff):
            t = int(diff[0])
            assert t > 0, (i, got, want)
            row = res['scores'][t][0].float().cpu()
            finite = row[torch.isfinite(row)]
            margin = (row[want[t]] - row[got[t]]).item()
            assert 0 <= margin <= 3e-2 * finite.std().item(), (i, t, int(want[t]), int(got[t]), margin)
        else:
            assert got.shape == want.shape, (i, got.shape, want.shape)


def test_tokens_with_options_do_not_depend_on_neighbours_slot_or_earlier_tenant(eng):
    slots = 8
    for sample in (False, True):
        target = dict(_request(eng, 0, 24, sample), repetition_penalty=1.4, no_repeat_ngram_size=2)
        others = [_spec(eng, 1 + j, 6 + 5 * j, j % 2 == 1) for j in range(7)]
        b = ContinuousBatcher(eng, slots, MAX_LEN, request_options=True)
        alone = _submit(b, target, 0)
        b.run()
        want = _tokens(alone)
        b = ContinuousBatcher(eng, slots, MAX_LEN, request_options=True)
        for j in range(3):
            _submit(b, others[j], 1 + j)
        b.step()
        b.step()
        r = _submit(b, target, 0)
        b.step()
        assert b.running.index(r) == 3
        for j in range(3, 7):
            _submit(b, others[j], 1 + j)
            b.step()
        b.run()
        assert torch.equal(_tokens(r), want), (sample, _tokens(r), want)
        # in a slot a longer request with other options left
        b = ContinuousBatcher(eng, slots, MAX_LEN, request_options=True)
        _submit(b, dict(_request(eng, 9, 40, False), no_repeat_ngram_size=3, min_new_tokens=30, eos_token_id=5), 9)
        b.run()
        r = _submit(b, target, 0)
        b.step()
        assert b.running.index(r) == 0
        b.run()
        assert torch.equal(_tokens(r), want), (sample, _tokens(r), want)


def test_neutral_rows_give_the_tokens_of_a_plain_batcher(eng):
    specs = [_request(eng, i, 8 + 3 * i, i % 2 == 1) for i in range(10)]
    got = {}
    for opt in (False, True):
        b = ContinuousBatcher(eng, 8, MAX_LEN, request_options=opt)
        reqs = []
        for i, spec in enumerate(specs):
            reqs.append(_submit(b, spec, i, repetition_penalty=1.0, no_repeat_ngram_size=0))
            if i % 3 == 1:
                b.step()
        b.run()
        got[opt] = [_tokens(r) for r in reqs]
    for i, (a, c) in enumerate(zip(got[False], got[True])):
        assert torch.equal(a, c), (i, a, c)


def test_follow_up_turn_with_a_penalty_equals_generate_with_the_conversation_cache(eng):
    spec1 = dict(_turn1(eng, 310), repetition_penalty=1.2)
    b = ContinuousBatcher(eng, SLOTS, MAX_LEN, prefix_reuse=True, request_options=True)
    r1 = b.submit(**spec1)
    b.run()
    c = KVCache(eng.cfg, 1, MAX_LEN, DEV)
    args = dict(max_new_tokens=spec1['max_new_tokens'], repetition_penalty=1.2)
    out = eng.generate(spec1['input_ids'].to(DEV), spec1['images'], spec1['bboxes'], cache=c, **args)
    assert torch.equal(_tokens(r1), out[0, spec1['input_ids'].shape[1]:].cpu())
    spec2 = dict(_turn2(eng, spec1, r1.sequences, 'text', 311), repetition_penalty=1.2, no_repeat_ngram_size=2)
    r2 = b.submit(**spec2)
    b.run()
    assert r2.reused > eng.cfg.num_patches
    out = eng.generate(spec2['input_ids'].to(DEV), spec2['images'], spec2['bboxes'], cache=c,
                       max_new_tokens=spec2['max_new_tokens'], repetition_penalty=1.2, no_repeat_ngram_size=2)
    assert torch.equal(_tokens(r2), out[0, spec2['input_ids'].shape[1]:].cpu()), _tokens(r2)


def test_graph_is_captured_once_per_opted_in_batcher(eng, monkeypatch):
    calls = []
    real = E._capture

    def counting(*a, **k):
        calls.append(1)
        return real(*a, **k)
    monkeypatch.setattr(E, '_capture', counting)
    b = ContinuousBatcher(eng, 8, MAX_LEN, request_options=True)
    graph = b.graph
    assert len(calls) == 1
    _, stops = _tables(['ab'])
    for i in range(12):
        _submit(b, _spec(eng, i, 3 + i % 5, i % 3 == 0), i, stop_strings=stops if i % 4 == 0 else None)
        b.step()
    b.run()
    assert len(calls) == 1 and b.graph is graph


def test_seam_batcher_with_options_equals_model_generate():
    from tests.stop_tokenizer import seeded_tokenizer
    from tests.test_engine_gpu import make_inputs
    from tests.test_model_seam_gpu import build_seam_model
    from gpt4roi_b200.engine import random_state_dicts
    cfg = EngineConfig(image_size=224, vit_layers=24, n_layers=2)
    sd, vit_sd = random_state_dicts(cfg, DEV, seed=47)
    model = build_seam_model(cfg, sd, vit_sd, dtype=torch.float16).eval()
    tok = seeded_tokenizer(32000, seed=5)
    n = 12
    ids, images, boxes = make_inputs(cfg, 1, [2], 24, seed=9)
    L = ids.shape[1]
    img, bx = images.half().to(DEV), [b.half().to(DEV) for b in boxes]
    sb = model.continuous_batcher(slots=4, max_len=L + n, tokenizer=tok, request_options=True)
    base = model.generate(ids.to(DEV), images=img, bboxes=bx, max_new_tokens=n).cpu()[0, L:]
    strings, _ = _tables(None)
    from tests.test_stop_strings_gpu import straddling_stop
    stop, _ = straddling_stop(strings, base, first=4)
    cases = (dict(repetition_penalty=1.3), dict(do_sample=True, temperature=0.7, no_repeat_ngram_size=2),
             dict(min_new_tokens=3, eos_token_id=int(base[0])), dict(stop_strings=[stop], repetition_penalty=1.1),
             dict(do_sample=True, repetition_penalty=1.2, stop_strings=stop))
    for kw in cases:
        torch.manual_seed(5)
        want = model.generate(ids.to(DEV), images=img, bboxes=bx, max_new_tokens=n, tokenizer=tok, **kw).cpu()
        torch.manual_seed(5)
        r = sb.submit(ids, images=img, bboxes=bx, max_new_tokens=n, **kw)
        sb.run()
        assert torch.equal(r.sequences, want), (kw, r.sequences[:, L:], want[:, L:])
