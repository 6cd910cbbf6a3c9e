"""GPU tests of continuous batching: the per-row selection kernel (kernels.sample_tokens_rows) against sample_tokens on
each row alone, and engine.ContinuousBatcher on the real engine -- a request's tokens do not depend on its neighbours,
its slot or the slot's earlier tenant; they equal generate() on the request alone (greedy, sampled, stop strings); the
model seam equals model.generate; the decode graph is captured once per batcher."""
import pytest
import torch

from gpt4roi_b200 import engine as E
from gpt4roi_b200 import kernels
from gpt4roi_b200.engine import ContinuousBatcher, EngineConfig, KVCache, PrefillEngine, random_state_dicts
from tests.test_engine_gpu import make_inputs

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
V, LD = 32006, 32064


def _rows_case(S, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    logits = (torch.randn(S, LD, generator=g) * 3).to(dtype)
    logits[:, :64] = logits[:, 64:128]                       # duplicated values: ties inside a row
    p = dict(greedy=(torch.rand(S, generator=g) < 0.4).to(torch.int32),
             temperature=torch.empty(S).uniform_(0.5, 1.5, generator=g),
             top_k=torch.tensor([0, 1, 50, 400])[torch.randint(0, 4, (S,), generator=g)].to(torch.int32),
             top_p=torch.tensor([1.0, 0.95, 0.5, 0.0])[torch.randint(0, 4, (S,), generator=g)],
             seed=torch.randint(0, 2 ** 62, (S,), generator=g),
             step=torch.randint(0, 5000, (S,), generator=g))
    active = (torch.rand(S, generator=g) < 0.7).to(torch.int32)
    active[0] = 1
    return logits, p, active


def _alone(logits, p, r):
    out = torch.empty(1, dtype=torch.int64, device=DEV)
    kernels.sample_tokens(logits[r:r + 1, :V].to(DEV), out, bool(p['greedy'][r]), float(p['temperature'][r]),
                          int(p['top_k'][r]), float(p['top_p'][r]), int(p['seed'][r]),
                          torch.tensor([int(p['step'][r])], dtype=torch.int64, device=DEV))
    return int(out)


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('S', [1, 8, 16, 64])
def test_rows_kernel_equals_sample_tokens_on_each_row_alone(S, dtype):
    logits, p, active = _rows_case(S, dtype, seed=S + (dtype == torch.float16))
    want = [_alone(logits, p, r) if active[r] else None for r in range(S)]
    g = torch.Generator().manual_seed(7)
    # eos: half of the active rows have their own token as eos id, the rest another id or none
    eos = torch.tensor([w if (w is not None and r % 2 == 0) else int(torch.randint(-1, V, (1,), generator=g))
                        for r, w in enumerate(want)], dtype=torch.int32)
    finished0 = torch.zeros(S, dtype=torch.int32)
    finished0[~active.bool()] = torch.randint(0, 2, (int((active == 0).sum()),), generator=g, dtype=torch.int32)
    lens0 = torch.randint(10, 300, (S,), generator=g, dtype=torch.int32)
    for with_lens in (True, False):
        d = {k: v.to(DEV) for k, v in p.items()}
        out = torch.full((S, 1), -7, dtype=torch.int64, device=DEV)
        fin, lens = finished0.to(DEV), lens0.to(DEV)
        kernels.sample_tokens_rows(logits[:, :V].to(DEV), out, d['greedy'], d['temperature'], d['top_k'], d['top_p'],
                                   d['seed'], d['step'], eos.to(DEV), active.to(DEV), fin, lens if with_lens else None)
        out, fin, step, lens = out.cpu()[:, 0], fin.cpu(), d['step'].cpu(), lens.cpu()
        on = active.bool()
        for r in range(S):
            if on[r]:
                assert int(out[r]) == want[r], (r, int(out[r]), want[r])
                assert int(fin[r]) == int(int(eos[r]) == want[r]), r
            else:
                assert int(out[r]) == -7 and int(fin[r]) == int(finished0[r]), r
        assert torch.equal(step, p['step'] + on.to(torch.int64))
        assert torch.equal(lens, lens0 + (on.to(torch.int32) if with_lens else 0))


# ---- the batcher on the engine -------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def eng():
    cfg = EngineConfig(image_size=224, vit_layers=12, n_layers=2)
    sd, vit_sd = random_state_dicts(cfg, DEV, seed=61)
    return PrefillEngine(cfg, sd, vit_sd, DEV)


def _request(eng, i, n, sample):
    """Request i: a prompt of its own length and box count, n new tokens, greedy or sampled (seed 100 + i)."""
    ids, images, boxes = make_inputs(eng.cfg, 1, [1 + i % 3], 12 + 3 * i, seed=200 + i)
    kw = dict(do_sample=True, temperature=0.8, top_k=0 if i % 2 else 40, top_p=0.9 if i % 3 else 1.0) if sample else {}
    return dict(input_ids=ids, images=images.to(torch.bfloat16), bboxes=boxes, max_new_tokens=n, **kw)


def _submit(b, spec, i):
    gen = torch.Generator().manual_seed(100 + i) if spec.get('do_sample') else None
    return b.submit(generator=gen, **spec)


def _tokens(req):
    return req.sequences[0, req.input_ids.shape[1]:]


@pytest.mark.parametrize('slots', [8, 20])      # both sides of the fused decode step's batch limit (16)
@pytest.mark.parametrize('sample', [False, True])
def test_tokens_do_not_depend_on_neighbours_slot_or_earlier_tenant(eng, slots, sample):
    max_len = 384
    target = _request(eng, 0, 24, sample)
    others = [_request(eng, 1 + j, 6 + 5 * j, j % 2 == 1) for j in range(7)]
    # alone, in slot 0 of a fresh batcher
    b = ContinuousBatcher(eng, slots, max_len)
    alone = _submit(b, target, 0)
    b.run()
    want = _tokens(alone)
    assert want.shape[0] == 24
    # beside seven others admitted at different steps, in slot 3
    b = ContinuousBatcher(eng, slots, max_len)
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
    assert torch.equal(_tokens(r), want), (_tokens(r), want)
    # in a slot a longer request left: its prompt and answer lie past the target's prompt
    b = ContinuousBatcher(eng, slots, max_len)
    long_spec = _request(eng, 9, 40, False)
    assert long_spec['input_ids'].shape[1] > target['input_ids'].shape[1]
    _submit(b, long_spec, 9)
    b.run()
    r = _submit(b, target, 0)
    b.step()
    assert b.running.index(r) == 0
    b.run()
    assert torch.equal(_tokens(r), want), (_tokens(r), want)


def _generate_alone(eng, spec, i, max_len, **kw):
    if spec.get('do_sample'):
        torch.manual_seed(100 + i)
    args = {k: v for k, v in spec.items() if k not in ('input_ids', 'images', 'bboxes')}
    out = eng.generate(spec['input_ids'].to(DEV), spec['images'], spec['bboxes'],
                       cache=KVCache(eng.cfg, 1, max_len, DEV), **args, **kw)
    return out[0, spec['input_ids'].shape[1]:].cpu()


def test_each_request_equals_generate_alone_greedy_and_sampled(eng):
    """4 slots and max_len 384: the decode attention splits the keys four ways at batch 4 as at batch 1, and the decode
    GEMMs run the same tiles at M = 1 and M = 4, so every sum runs in generate()'s order and the tokens are identical."""
    max_len, slots = 384, 4
    specs = [_request(eng, i, 8 + 4 * i, i % 2 == 1) for i in range(6)]
    b = ContinuousBatcher(eng, slots, max_len)
    reqs = []
    for i, spec in enumerate(specs):
        if spec.get('do_sample'):
            torch.manual_seed(100 + i)      # the seed comes from torch's default generator, as in generate()
        reqs.append(b.submit(**spec))
        if i % 2:
            b.step()
    b.run()
    for i, (spec, r) in enumerate(zip(specs, reqs)):
        want = _generate_alone(eng, spec, i, max_len)
        assert torch.equal(_tokens(r), want), (i, _tokens(r), want)


@pytest.mark.parametrize('slots', [8, 16])
def test_greedy_requests_follow_generate_alone_up_to_a_near_tie(eng, slots):
    """At 8 and 16 slots the sums run in another order than generate()'s at batch 1.  The path that reorders them is the
    decode attention: its split-KV factor follows B * H against the SM count (csrc/decode.cu), so at max_len 384 it
    splits the keys 2 ways at 8 rows and 1 way at 16, where batch 1 splits them 4 ways; at 16 rows the decode GEMMs
    also run their 9..16-row tiles.  So each greedy request must give generate()'s tokens up to the first difference,
    if any, and there the two tokens must be a near tie of generate()'s own logits, within the margin of
    tests/test_model_seam_gpu.py.  The first token comes from the same batch-1 prefill and selection: always equal."""
    max_len = 384
    specs = [_request(eng, i, 16 + 2 * i, False) for i in range(slots)]
    b = ContinuousBatcher(eng, slots, max_len)
    reqs = []
    for i, spec in enumerate(specs):
        reqs.append(b.submit(**spec))
        if i % 3 == 2:
            b.step()
    b.run()
    for i, (spec, r) in enumerate(zip(specs, reqs)):
        L = spec['input_ids'].shape[1]
        res = eng.generate(spec['input_ids'].to(DEV), spec['images'], spec['bboxes'],
                           max_new_tokens=spec['max_new_tokens'], cache=KVCache(eng.cfg, 1, max_len, DEV),
                           output_logits=True, return_dict_in_generate=True)
        want, got = res['sequences'][0, L:].cpu(), _tokens(r)
        assert got.shape == want.shape, (i, got.shape, want.shape)
        diff = (got != want).nonzero()
        if len(diff):
            t = int(diff[0])
            assert t > 0, (i, got, want)
            row = res['logits'][t][0].float().cpu()
            margin = (row[want[t]] - row[got[t]]).item()
            assert 0 <= margin <= 3e-2 * row.std().item(), (i, t, int(want[t]), int(got[t]), margin)


def test_a_request_the_prefill_rejects_leaves_its_slot_idle(eng):
    """A request with a box more than its <bbox> tokens: the prefill raises ValueError (as forward() does), step()
    raises it, the request retires with the error, and the others -- one already running, one queued after it into the
    same slot -- give generate()'s tokens alone (4 slots: the split of test_each_request_equals_generate_alone...)."""
    max_len, slots = 384, 4
    a, c = _request(eng, 0, 20, False), _request(eng, 2, 12, False)
    bad = _request(eng, 1, 8, False)
    bad['bboxes'] = [torch.cat([bad['bboxes'][0], bad['bboxes'][0][:1]])]
    b = ContinuousBatcher(eng, slots, max_len)
    ra = b.submit(**a)
    b.step()
    rbad, rc = b.submit(**bad), b.submit(**c)
    with pytest.raises(ValueError, match='<bbox>'):
        b.step()
    assert rbad.done and isinstance(rbad.error, ValueError) and rbad.tokens == []
    assert b.active.tolist() == [1, 0, 0, 0] and b.running[1] is None
    b.run()
    assert b.running.count(None) == slots and int(b.active.sum()) == 0
    assert torch.equal(_tokens(ra), _generate_alone(eng, a, 0, max_len))
    assert torch.equal(_tokens(rc), _generate_alone(eng, c, 2, max_len))


def test_stop_strings_retire_one_request_while_its_neighbours_continue(eng):
    from gpt4roi_b200.spi_llava import stop_strings_from_tokenizer
    from tests.stop_tokenizer import seeded_tokenizer
    from tests.test_stop_strings_cpu import clean_strings
    from tests.test_stop_strings_gpu import straddling_stop
    tok = seeded_tokenizer(32000, seed=5)
    strings = clean_strings(tok)
    max_len, slots = 384, 4
    specs = [_request(eng, i, 20, False) for i in range(4)]
    base = _generate_alone(eng, specs[1], 1, max_len)
    stop, at = straddling_stop(strings, base, first=3)
    table = stop_strings_from_tokenizer(tok, [stop])
    b = ContinuousBatcher(eng, slots, max_len, stop_strings=table)
    reqs = [b.submit(**spec) for spec in specs]
    b.run()
    assert torch.equal(_tokens(reqs[1]), base[:at + 1])
    for i, (spec, r) in enumerate(zip(specs, reqs)):
        want = _generate_alone(eng, spec, i, max_len, stop_strings=table)
        assert torch.equal(_tokens(r), want), (i, _tokens(r), want)
    assert max(_tokens(r).shape[0] for r in reqs) > at + 1     # a neighbour ran on after request 1 retired


def test_graph_is_captured_once_per_batcher(eng, monkeypatch):
    calls = []
    real = E._capture

    def counting(*a, **k):
        calls.append(1)
        return real(*a, **k)
    monkeypatch.setattr(E, '_capture', counting)
    b = ContinuousBatcher(eng, 8, 384)
    graph = b.graph
    assert len(calls) == 1
    for i in range(12):
        _submit(b, _request(eng, i, 3 + i % 5, i % 3 == 0), i)
        b.step()
    b.run()
    assert len(calls) == 1 and b.graph is graph


def test_seam_batcher_equals_model_generate():
    from tests.test_model_seam_gpu import build_seam_model
    cfg = EngineConfig(image_size=224, vit_layers=24, n_layers=2)
    sd, vit_sd = random_state_dicts(cfg, DEV, seed=47)
    model = build_seam_model(cfg, sd, vit_sd, dtype=torch.float16).eval()
    n = 12
    ids, images, boxes = make_inputs(cfg, 1, [2], 24, seed=9)
    L = ids.shape[1]
    img, bx = images.half().to(DEV), [b.half().to(DEV) for b in boxes]
    # max_len = L + n: the decode attention is sized as generate()'s own cache sizes it
    sb = model.continuous_batcher(slots=4, max_len=L + n)
    for kw in (dict(), dict(do_sample=True, temperature=0.7), dict(do_sample=True)):
        torch.manual_seed(5)
        want = model.generate(ids.to(DEV), images=img, bboxes=bx, max_new_tokens=n, **kw).cpu()
        torch.manual_seed(5)
        r = sb.submit(ids, images=img, bboxes=bx, max_new_tokens=n, **kw)
        sb.run()
        assert torch.equal(r.sequences, want), (kw, r.sequences[:, L:], want[:, L:])
