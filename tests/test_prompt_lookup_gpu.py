"""Prompt-lookup decoding on the device (generate(prompt_lookup_num_tokens=k), csrc/lookup.cu, engine.LookupDecode):
the draft and acceptance kernel against transformers' rule, the verify step teacher-forced on the plain loop's tokens,
graph replays against eager steps, and generate() end to end against the plain engine loop and transformers' own
assisted decoding over the model seam (use_hf_loop=True), bf16 and fp16, on a 2-layer random engine.

The verify step runs the decode chain over k + 1 rows: its GEMMs take k + 1 rows and its attention splits the keys
otherwise than the 1-row step, so the contract is not bitwise equality with the plain loop: the tokens agree up to the
first near tie of the plain loop's logits (3e-2 of the row's spread, the margin of tests/test_model_seam_gpu.py)."""
import types

import pytest
import torch

from gpt4roi_b200 import kernels
from gpt4roi_b200.engine import (EngineConfig, KVCache, LookupDecode, PrefillEngine, lookup_accept, lookup_candidates,
                                 random_state_dicts)
from tests.test_engine_gpu import make_inputs

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _state(k, ngram, L, max_length, hist, eos):
    M = k + 1
    z = dict(device=DEV)
    return types.SimpleNamespace(
        k=k, max_ngram=ngram, prompt_len=L, max_length=max_length, hist=hist,
        eos=torch.tensor(eos, dtype=torch.int32, **z) if eos else None, ids=torch.zeros((M, 1), dtype=torch.int64, **z),
        state=torch.zeros(5, dtype=torch.int32, **z), base=torch.zeros(1, dtype=torch.int32, **z),
        pos=torch.zeros(M, dtype=torch.int32, **z), step=torch.zeros(M, dtype=torch.int64, **z),
        readback=torch.zeros(4 + M + k, dtype=torch.int64, **z))


def _histories():
    g = torch.Generator().manual_seed(3)
    out = []
    for i in range(60):
        n = int(torch.randint(2, 400 if i % 4 == 0 else 60, (1,), generator=g))
        V = int(torch.randint(2, 10, (1,), generator=g))
        out.append(torch.randint(0, V, (n,), generator=g).tolist())
    seg = torch.randint(100, 30000, (40,), generator=g).tolist()
    out += [seg + seg[:7], seg[:20] + [5, 6] + seg + seg[:1], [1, 2, 3, 1, 2], [9] * 300, [4, 5]]
    return out


def test_lookup_kernel_drafts_and_accepts_as_the_restated_rule():
    g = torch.Generator().manual_seed(11)
    for i, seq in enumerate(_histories()):
        n = len(seq)
        k = [1, 3, 8, 16, 31][i % 5]
        ngram = [1, 2, 3][i % 3]
        eos = [seq[int(torch.randint(0, n, (1,), generator=g))]] if i % 3 == 1 else []
        L = max(1, n - int(torch.randint(0, n, (1,), generator=g)))
        for max_length in (n + 2, n + k + 40):
            hist = torch.zeros(max_length + k, dtype=torch.int64, device=DEV)
            hist[:n] = torch.tensor(seq)
            st = _state(k, ngram, L, max_length, hist, eos)
            st.state.copy_(torch.tensor([n, 0, 0, 0, 0], dtype=torch.int32))
            kernels.lookup_step(st)
            draft = lookup_candidates(seq, k, ngram, max_length, eos)
            rb = st.readback.cpu()
            d = int(rb[3])
            assert d == len(draft) and rb[4 + k + 1:4 + k + 1 + d].tolist() == draft, (i, seq, draft, rb)
            ids = st.ids[:, 0].cpu().tolist()
            assert ids == [seq[-1]] + draft + [seq[-1]] * (k - d)
            assert st.pos.cpu().tolist() == list(range(n - 1, n + k)) and int(st.base) == n - 1
            assert st.step.cpu().tolist() == [n - L + j for j in range(k + 1)]
            # acceptance: a selection agreeing with the first few drafts, with the host's done flag either way
            sel = torch.tensor(draft + [7] * (k + 1 - d))
            cut = int(torch.randint(0, d + 1, (1,), generator=g))
            sel[cut] = 10 ** 6 + cut
            done = bool(i % 2)
            st.state[4] = int(done)
            kernels.lookup_step(st, sel.to(DEV))
            new, fin = lookup_accept(draft, sel.tolist(), n, max_length, done, eos)
            rb = st.readback.cpu()
            seq2 = seq + new
            assert int(rb[0]) == len(new) and rb[4:4 + len(new)].tolist() == new and int(rb[2]) == len(seq2)
            assert bool(rb[1]) == fin and hist[:len(seq2)].cpu().tolist() == seq2
            nxt = [] if fin or len(seq2) + 1 >= max_length else lookup_candidates(seq2, k, ngram, max_length, eos)
            assert int(rb[3]) == len(nxt) and rb[4 + k + 1:4 + k + 1 + len(nxt)].tolist() == nxt


@pytest.fixture(scope='module', params=['bf16', 'fp16'])
def eng(request):
    cfg = EngineConfig(image_size=224, vit_layers=12, n_layers=2, dtype=request.param)
    sd, vit_sd = random_state_dicts(cfg, DEV, seed=71)
    return PrefillEngine(cfg, sd, vit_sd, DEV)


def _repetitive(cfg, kind, seed):
    """A prompt built to repeat: the image prompt, then a random segment twice; or a conversation re-sent whole (the
    first question, an answer, then all of it again with a new question)."""
    ids, images, boxes = make_inputs(cfg, 1, [1], 16, seed=seed)
    g = torch.Generator().manual_seed(seed)
    seg = torch.randint(3, 30000, (24,), generator=g)
    if kind == 'segment':
        tail = torch.cat([seg, seg[:18]])
    else:
        text = ids[0, -15:]                          # the question's text tokens, without its <bbox>
        text = text[text != cfg.bbox_token]
        tail = torch.cat([seg, text, seg, torch.randint(3, 30000, (6,), generator=g)])
    return torch.cat([ids, tail[None]], 1), images.to(cfg.torch_dtype), boxes


def _near_tie_prefix(got, want, logits, what):
    """got must equal want up to the first difference, which must be a near tie of the plain loop's logits."""
    n = min(len(got), len(want))
    diff = [t for t in range(n) if got[t] != want[t]]
    if not diff:
        assert len(got) == len(want), (what, got, want)
        return n
    t = diff[0]
    row = logits[t][0].float().cpu()
    margin = (row[want[t]] - row[got[t]]).item()
    assert t > 0 and 0 <= margin <= 3e-2 * row.std().item(), (what, t, want[t], got[t], margin)
    return t


def test_teacher_forced_verify_matches_the_plain_loop(eng):
    """Feed the plain greedy continuation as the draft: each verify row's arg-max is the plain loop's next token up to
    the first near tie, and the K/V the verify step writes at base .. base + k are the plain loop's within rounding."""
    cfg = eng.cfg
    ids, images, boxes = _repetitive(cfg, 'segment', 5)
    L, T, k = ids.shape[1], 24, 8
    plain_kv = KVCache(cfg, 1, L + T + k, DEV)
    res = eng.generate(ids.to(DEV), images, boxes, max_new_tokens=T, cache=plain_kv, output_logits=True,
                       return_dict_in_generate=True)
    S = res['sequences'][0].cpu().tolist()
    assert len(S) == L + T
    for j0 in (1, 9):      # verify rows decide new tokens j0 .. j0 + k
        cache = KVCache(cfg, 1, L + T + k, DEV)
        eng.forward_device(ids.to(DEV), images.to(DEV), eng.plan_boxes(boxes), last_only=True, cache=cache)
        hist = torch.zeros((1, L + T + k), dtype=torch.int64, device=DEV)
        hist[0, :L + j0 - 1] = torch.tensor(S[:L + j0 - 1])
        st = LookupDecode(eng, cache, hist, L, T, k, use_graph=False)
        if j0 > 1:                       # bring the cache to L + j0 - 1 positions with the plain loop's K/V
            for kv, mine in ((plain_kv.k, cache.k), (plain_kv.v, cache.v)):
                for a, b in zip(kv, mine):
                    b[:, L:L + j0 - 1] = a[:, L:L + j0 - 1]
        base = L + j0 - 1
        row = S[base - 1:base + k]
        st.ids[:, 0] = torch.tensor(row, device=DEV)
        st.pos.copy_(torch.arange(base - 1, base - 1 + k + 1, dtype=torch.int32))
        st.base.fill_(base - 1)
        logits = eng.verify_step(st.ids, cache, st)
        got = logits[:, 0].float().argmax(-1).cpu().tolist()
        want = S[base:base + k + 1]
        _near_tie_prefix(got, want, res['logits'][j0 - 1:j0 + k], ('teacher-forced', cfg.dtype, j0))
        for li in range(cfg.n_layers):
            for a, b in ((plain_kv.k[li], cache.k[li]), (plain_kv.v[li], cache.v[li])):
                x, y = a[0, base - 1:base + k].float(), b[0, base - 1:base + k].float()
                assert ((x - y).norm() / x.norm()).item() < 2e-2, (cfg.dtype, j0, li)


@pytest.mark.parametrize('plant', ['drafts', 'none'])
def test_graph_replay_equals_eager_verify_steps(eng, plant):
    """Both captured steps -- the M-row verify step (a draft planted after the first token) and the one-row step of a
    step without a draft -- are bitwise the eager steps: history, readbacks and the K/V of every position the sequence
    holds (positions past it take rejected rows' and the capture warm-up's writes, which nothing reads)."""
    cfg = eng.cfg
    ids, images, boxes = _repetitive(cfg, 'segment', 6)
    L, T, k = ids.shape[1], 20, 5
    outs = []
    for use_graph in (False, True):
        cache = KVCache(cfg, 1, L + T + k, DEV)
        logits = eng.forward_device(ids.to(DEV), images.to(DEV), eng.plan_boxes(boxes), last_only=True, cache=cache)
        hist = torch.zeros((1, L + T + k), dtype=torch.int64, device=DEV)
        hist[0, :L] = ids[0]
        st = LookupDecode(eng, cache, hist, L, T, k, use_graph=use_graph)
        st.first(logits)
        d = k if plant == 'drafts' else 0
        st.ids[1:, 0] = ids[0, -k:].to(DEV)
        st.state[1] = d
        st.rb[3] = d
        rows, rbs = [], []
        for _ in range(4):
            rows.append(k + 1 if int(st.rb[3]) else 1)
            rbs.append(st.run().clone())
        assert rows[0] == (k + 1 if d else 1)
        held = int(rbs[-1][2]) - 1          # K/V are written for every token but the last
        outs.append((hist.clone(), rbs, [c[:, :held].clone() for c in cache.k + cache.v], rows))
    (h0, r0, k0, w0), (h1, r1, k1, w1) = outs
    assert w0 == w1 and torch.equal(h0, h1) and all(torch.equal(a, b) for a, b in zip(r0, r1))
    assert all(torch.equal(a, b) for a, b in zip(k0, k1))


def _plain_and_lookup(eng, ids, images, boxes, T, k, **kw):
    sampled = kw.get('do_sample')
    if sampled:
        torch.manual_seed(7)
    plain = eng.generate(ids.to(DEV), images, boxes, max_new_tokens=T, output_logits=True, return_dict_in_generate=True,
                         **kw)
    if sampled:
        torch.manual_seed(7)
    look = eng.generate(ids.to(DEV), images, boxes, max_new_tokens=T, prompt_lookup_num_tokens=k, **kw)
    L = ids.shape[1]
    return plain['sequences'][0, L:].cpu().tolist(), look[0, L:].cpu().tolist(), plain['logits'], \
        list(eng.lookup_accepted)


def test_generate_with_lookup_gives_the_plain_loops_tokens(eng):
    cfg = eng.cfg
    accepted_any = False
    for kind in ('segment', 'conversation'):
        ids, images, boxes = _repetitive(cfg, kind, 9)
        for kw in (dict(), dict(do_sample=True, temperature=0.7, top_k=50)):
            for k in (4, 10, 20):      # 20: more than 16 verify rows, the tiled GEMMs
                want, got, logits, acc = _plain_and_lookup(eng, ids, images, boxes, 64, k, **kw)
                what = (cfg.dtype, kind, kw, k)
                if kw:
                    # equal draws up to the first one that the two steps' slightly different logits flip: that token
                    # must still be one the plain loop's top-k could draw
                    t = next((i for i in range(min(len(got), len(want))) if got[i] != want[i]), None)
                    if t is None:
                        assert len(got) == len(want), (what, got, want)
                    else:
                        assert t > 0 and got[:t] == want[:t], (what, got, want)
                        assert got[t] in logits[t][0].float().topk(50).indices.tolist(), (what, t, got[t])
                else:
                    t = _near_tie_prefix(got, want, logits, what)
                    if t == len(want):
                        L = ids.shape[1]
                        seq = ids[0].tolist() + want + [-1] * (k + 1)
                        assert acc == _simulate(seq, L, 64, k, [])
                accepted_any = accepted_any or max(acc, default=0) > 1
                assert sum(acc) + 1 == len(got) <= 64
    assert accepted_any, 'no verify step accepted a draft'


def _simulate(seq, L, max_new, k, eos, start=1):
    """Appended counts per verify step on the greedy sequence seq (its tokens are every position's arg-max)."""
    ln, out, max_length = L + start, [], L + max_new
    while ln < max_length and seq[ln - 1] not in eos:
        draft = [] if ln + 1 >= max_length else lookup_candidates(seq[:ln], k, 2, max_length, eos)
        sel = seq[ln:ln + len(draft) + 1]
        if len(sel) < len(draft) + 1:
            break
        new, fin = lookup_accept(draft, sel, ln, max_length, False, eos)
        out.append(len(new))
        ln += len(new)
        if fin:
            break
    return out


def test_endings_match_the_plain_loop(eng):
    """max_new_tokens, an eos id (a token the plain loop emits, also in a list) and KeywordsStoppingCriteria-style
    host criteria end the lookup loop where they end the plain loop."""
    cfg = eng.cfg
    ids, images, boxes = _repetitive(cfg, 'segment', 12)
    L = ids.shape[1]
    free = eng.generate(ids.to(DEV), images, boxes, max_new_tokens=40)[0, L:].cpu().tolist()
    for T in (1, 2, 13):
        a = eng.generate(ids.to(DEV), images, boxes, max_new_tokens=T)
        b = eng.generate(ids.to(DEV), images, boxes, max_new_tokens=T, prompt_lookup_num_tokens=6)
        assert b.shape == a.shape == (1, L + T) and torch.equal(a[:, :L + 1], b[:, :L + 1]), (T, a, b)
    eos = free[17]
    a = eng.generate(ids.to(DEV), images, boxes, max_new_tokens=40, eos_token_id=eos)
    for e in (eos, [12345, eos]):
        b = eng.generate(ids.to(DEV), images, boxes, max_new_tokens=40, eos_token_id=e, prompt_lookup_num_tokens=6)
        n = min(a.shape[1], b.shape[1])
        assert torch.equal(a[:, :n], b[:, :n]) and b[0, -1].item() == eos, (e, a, b)
        assert a.shape == b.shape

    class _Stop:
        def __init__(self, tok):
            self.tok = tok

        def __call__(self, out, scores):
            return bool((out[0, L:] == self.tok).any())
    a = eng.generate(ids.to(DEV), images, boxes, max_new_tokens=40, stopping_criteria=[_Stop(free[11])])
    b = eng.generate(ids.to(DEV), images, boxes, max_new_tokens=40, stopping_criteria=[_Stop(free[11])],
                     prompt_lookup_num_tokens=6)
    assert torch.equal(a, b), (a, b)


@pytest.fixture(scope='module')
def seam():
    from tests.test_model_seam_gpu import build_seam_model
    cfg = EngineConfig(image_size=224, vit_layers=24, n_layers=2)
    sd, vit_sd = random_state_dicts(cfg, DEV, seed=37)
    model = build_seam_model(cfg, sd, vit_sd, dtype=torch.float16, app_style=True).eval()
    return cfg, model


class _Counts:
    """A streamer recording the size of every chunk it gets (HF's assisted loop puts each step's accepted tokens)."""

    def __init__(self):
        self.sizes = []

    def put(self, t):
        self.sizes.append(int(t.numel()))

    def end(self):
        pass


def test_hf_loop_assisted_decoding_runs_through_the_seam(seam):
    """transformers' own prompt-lookup decoding (use_hf_loop=True: crop, logits_to_keep > 1, the candidate tokens passed
    through) gives the engine loop's tokens where no near tie intervenes, and each of its steps appends the tokens
    the restated rule gives on that sequence (its first step verifies drafts from the prompt, the engine loop's first
    token comes from the prefill)."""
    cfg, model = seam
    eng = model._get_engine(torch.device(DEV))
    ids, images, boxes = _repetitive(cfg, 'segment', 15)
    L, T, k = ids.shape[1], 32, 6
    img = images.half().to(DEV)
    bx = [b.half().to(DEV) for b in boxes]
    with torch.inference_mode():
        plain = model.generate(ids.to(DEV), images=img, bboxes=bx, max_new_tokens=T, output_logits=True,
                               return_dict_in_generate=True)
        ours = model.generate(ids.to(DEV), images=img, bboxes=bx, max_new_tokens=T, prompt_lookup_num_tokens=k)
        counts = _Counts()
        hf = model.generate(ids.to(DEV), images=img, bboxes=bx, max_new_tokens=T, prompt_lookup_num_tokens=k,
                            use_hf_loop=True, streamer=counts)
    want = plain.sequences[0, L:].cpu().tolist()
    t1 = _near_tie_prefix(ours[0, L:].cpu().tolist(), want, plain.logits, 'engine loop')
    got_hf = hf[0, L:].cpu().tolist()
    t2 = _near_tie_prefix(got_hf[:T], want, plain.logits, 'hf loop')
    steps = counts.sizes[1:]                      # the first put is the prompt
    seq = hf[0].cpu().tolist()
    if t2 == len(want):
        sim = _simulate(seq + [-1] * (k + 1), L, len(seq) - L, k, [], start=0)
        assert steps[:len(sim) - 1] == sim[:len(sim) - 1], (steps, sim)
    if t1 == len(want):
        assert eng.lookup_accepted == _simulate(ids[0].tolist() + want + [-1] * (k + 1), L, T, k, [])
