"""CPU tests of prompt-lookup decoding (generate(prompt_lookup_num_tokens=k)): the host restatements of transformers'
draft rule (PromptLookupCandidateGenerator.get_candidates) and acceptance (_assisted_decoding), the lookup loop on a stub
engine whose next token follows a fixed rule, the stopping-criteria calls, the seam's resolution of the option, the
calls that keep today's loop, and KVCache / G4RCache.crop."""
import pytest
import torch

from gpt4roi_b200 import engine as E
from gpt4roi_b200.engine import EngineConfig, KVCache, LookupDecode, lookup_accept, lookup_candidates, lookup_loop

CFG = EngineConfig(image_size=28, vit_hidden=32, vit_heads=2, vit_layers=2, vit_mlp=64, hidden=64, n_heads=2,
                   n_layers=1, mlp=128, vocab=140, bbox_token=132, im_patch_token=131, im_start_token=134,
                   im_end_token=135)


def _hf_candidates(seq, k, ngram, max_length, eos):
    from transformers.generation.candidate_generator import PromptLookupCandidateGenerator
    gen = PromptLookupCandidateGenerator(eos_token_id=torch.tensor(eos, dtype=torch.long), num_output_tokens=k,
                                         max_matching_ngram_size=ngram, max_length=max_length)
    ids = torch.tensor([seq], dtype=torch.long)
    cand, _ = gen.get_candidates(ids)
    return cand[0, len(seq):].tolist()


@pytest.mark.parametrize('seed', range(40))
def test_draft_rule_equals_hf_on_seeded_histories(seed):
    g = torch.Generator().manual_seed(seed)
    n = int(torch.randint(2, 60, (1,), generator=g))
    V = int(torch.randint(3, 12, (1,), generator=g))      # a small vocabulary: matches are frequent
    seq = torch.randint(0, V, (n,), generator=g).tolist()
    k = int(torch.randint(1, 12, (1,), generator=g))
    ngram = int(torch.randint(1, 4, (1,), generator=g))
    eos = [int(torch.randint(0, V, (1,), generator=g))] if seed % 3 else []
    for max_length in (n + 1, n + 2, n + k, n + 50):
        assert lookup_candidates(seq, k, ngram, max_length, eos) == _hf_candidates(seq, k, ngram, max_length, eos), \
            (seq, k, ngram, max_length, eos)


def test_draft_rule_planted_cases():
    cases = [
        ([5, 6, 7, 8, 9, 5, 6], 3, 2, 50, []),          # bigram (5, 6) -> 7 8 9
        ([5, 6, 7, 8, 9, 4, 6], 3, 2, 50, []),          # bigram (4, 6) unseen: unigram 6 -> 7 8 9
        ([1, 2, 9, 1, 2, 8, 1, 2], 2, 2, 50, []),       # the leftmost occurrence wins: 9 1
        ([1, 2, 3, 4, 1, 2], 4, 2, 50, [3]),            # eos first: no draft, and no further search
        ([1, 2, 3, 7, 4, 1, 2], 4, 2, 50, [4]),         # cut before eos: 3 7
        ([1, 2, 3, 4, 5], 3, 2, 50, []),                # no match
        ([1, 2, 3, 1, 2], 3, 2, 6, []),                 # max_length == len + 1: no draft
        ([1, 2, 3, 4, 1, 2], 9, 2, 50, []),             # bounded by the sequence: 3 4 1 2
        ([3, 3, 3], 2, 3, 50, []),
        ([7], 3, 2, 50, []),
    ]
    want = [[7, 8, 9], [7, 8, 9], [9, 1], [], [3, 7], [], [], [3, 4, 1, 2], [3], []]
    for (seq, k, ng, ml, eos), w in zip(cases, want):
        assert lookup_candidates(seq, k, ng, ml, eos) == w == _hf_candidates(seq, k, ng, ml, eos), (seq, w)


def _hf_n_matches(drafts, selected, done):
    """_assisted_decoding's formula, transcribed on tensors."""
    cand = torch.tensor([drafts], dtype=torch.long)
    sel = torch.tensor([selected], dtype=torch.long)
    n = int(((~(cand == sel[:, :-1])).cumsum(dim=-1) < 1).sum())
    if done and n == len(drafts):
        n -= 1
    return n


@pytest.mark.parametrize('seed', range(30))
def test_acceptance_equals_hf_n_matches(seed):
    g = torch.Generator().manual_seed(100 + seed)
    d = int(torch.randint(1, 8, (1,), generator=g))
    drafts = torch.randint(0, 3, (d,), generator=g).tolist()
    selected = torch.randint(0, 3, (d + 1,), generator=g).tolist()
    for done in (False, True):
        n = _hf_n_matches(drafts, selected, done)
        new, fin = lookup_accept(drafts, selected, 10, 10 + 100, done, eos_ids=[2])
        assert new == selected[:n + 1] and fin == (2 in new)
    # the candidate reaching max_length counts as done (HF's MaxLengthCriteria on it); the budget caps the append
    n = _hf_n_matches(drafts, selected, True)
    new, _ = lookup_accept(drafts, selected, 10, 10 + d, False)
    assert new == selected[:min(n + 1, d)]


class _RuleEngine:
    """Stub engine: the token after position p is rule(token at p, p); verify_step runs the rule on every row."""

    def __init__(self, rule, vocab=CFG.vocab):
        self.rule, self.vocab, self.dev, self.cfg = rule, vocab, torch.device('cpu'), CFG
        self.dt = torch.float32
        self.verify_rows = []

    def logits_for(self, toks, pos):
        out = torch.zeros(len(toks), 1, self.vocab)
        for i, (t, p) in enumerate(zip(toks, pos)):
            out[i, 0, self.rule(int(t), int(p))] = 1.0
        return out

    def verify_step(self, ids, cache, st):
        self.verify_rows.append((ids.shape[0], int(st.state[1])))    # (rows, drafts)
        return self.logits_for(ids[:, 0].tolist(), st.pos.tolist())

    # the pieces of PrefillEngine the plain loop and _generate_lookup call
    def plan_boxes(self, bboxes):
        return None

    def forward_device(self, ids, images, plan, validate=True, last_only=True, seqlens=None, cache=None):
        if cache is not None:
            cache.start(ids.shape[1], seqlens, ids)
        L = ids.shape[1]
        return self.logits_for(ids[:, -1].tolist(), [L - 1] * ids.shape[0]).view(ids.shape[0], 1, -1)

    def decode_step(self, tok, cache, pos_dev=None):
        pos = cache.length
        cache.length += 1
        return self.logits_for(tok[:, 0].tolist(), [pos] * tok.shape[0])


def _greedy_sequence(rule, prompt, n):
    seq = list(prompt)
    for _ in range(n):
        seq.append(rule(seq[-1], len(seq) - 1))
    return seq


def _expected_steps(seq, L, max_new, k, ngram, eos):
    """Appended counts of each verify step after the first token, simulated with the restated rules on the greedy
    sequence (the tokens every position selects are those of `seq`, which runs k + 1 tokens past max_new)."""
    ln, steps = L + 1, []
    max_length = L + max_new
    while ln < max_length and seq[ln - 1] not in eos:
        draft = [] if ln + 1 >= max_length else lookup_candidates(seq[:ln], k, ngram, max_length, eos)
        sel = seq[ln:ln + len(draft) + 1]
        new, fin = lookup_accept(draft, sel, ln, max_length, False, eos)
        steps.append(len(new))
        ln += len(new)
        if fin:
            break
    return steps


def _run(rule, prompt, max_new, k, ngram=2, eos=(), criteria=None, streamer=None):
    eng = _RuleEngine(rule)
    L = len(prompt)
    cache = KVCache(CFG, 1, L + max_new + k, 'cpu')
    out = torch.zeros((1, L + max_new + k), dtype=torch.int64)
    out[0, :L] = torch.tensor(prompt)
    logits = eng.forward_device(out[:, :L], None, None, cache=cache)
    st = LookupDecode(eng, cache, out, L, max_new, k, ngram, eos, use_graph=False)
    n = lookup_loop(st, logits, max_new, criteria, streamer)
    return out[0, :L + n].tolist(), st, eng


def _cycle(t, p):
    return t % 5 + 1 if 1 <= t <= 5 else 1          # 1 2 3 4 5 1 2 ...


def _cycle_with_breaks(t, p):
    return 9 if p % 7 == 6 else _cycle(t, p)        # every 7th position breaks the cycle


@pytest.mark.parametrize('rule', [_cycle, _cycle_with_breaks])
@pytest.mark.parametrize('k', [1, 3, 8])
@pytest.mark.parametrize('max_new', [1, 2, 7, 30])
def test_loop_appends_hf_counts_and_never_passes_max_new_tokens(rule, k, max_new):
    prompt = [1, 2, 3, 4, 5, 1, 2, 3, 7, 9, 3]
    got, st, eng = _run(rule, prompt, max_new, k)
    want = _greedy_sequence(rule, prompt, max_new)
    assert got == want and len(got) - len(prompt) == max_new
    assert st.accepted == _expected_steps(_greedy_sequence(rule, prompt, max_new + k + 1), len(prompt), max_new, k, 2, [])
    assert all(r == (k + 1 if d else 1) for r, d in eng.verify_rows)   # a step without a draft runs one row
    if rule is _cycle and max_new >= 7:
        assert max(st.accepted) > 1              # drafts were accepted


def test_loop_stops_on_eos_inside_an_accepted_run():
    prompt = [1, 2, 3, 4, 5, 1, 2]
    for eos in ([4], [4, 77], [1]):
        got, st, _ = _run(_cycle, prompt, 30, 6, eos=eos)
        want = _greedy_sequence(_cycle, prompt, 30 + 7)
        cut = next(i for i in range(len(prompt), len(want)) if want[i] in eos)
        assert got == want[:cut + 1]
        assert st.accepted == _expected_steps(want, len(prompt), 30, 6, 2, eos)


class _Recorder:
    """A stopping criterion that records the sequences it is called with and stops when the sequence ends in `stop`."""

    def __init__(self, stop):
        self.stop, self.calls = stop, []

    def __call__(self, ids, scores):
        self.calls.append((ids[0].tolist(), scores))
        return ids[0, -len(self.stop):].tolist() == self.stop


def test_host_criteria_are_called_as_hf_calls_them():
    prompt = [1, 2, 3, 4, 5, 1, 2]
    crit = _Recorder([1, 2])
    got, st, _ = _run(_cycle, prompt, 30, 4, criteria=[crit])
    L = len(prompt)
    # first token 3 (after the prefill); then per step: the candidate (history + drafts), then the history after it
    hist = got
    calls = [c for c, _ in crit.calls]
    assert all(s is None for _, s in crit.calls)
    assert calls[0] == hist[:L + 1]
    cand = calls[1]
    draft = lookup_candidates(hist[:L + 1], 4, 2, L + 30, [])
    assert cand == hist[:L + 1] + draft
    # HF's is_done_candidate: the candidate ends in the stop sequence, so one draft fewer is accepted
    assert st.accepted[0] == len(draft)
    assert calls[2] == hist and hist[-2:] == [1, 2] and len(calls) == 3


class _Streamer:
    def __init__(self):
        self.chunks, self.ended = [], False

    def put(self, t):
        self.chunks.append(t.tolist())

    def end(self):
        self.ended = True


def test_streamer_gets_the_prompt_then_each_steps_tokens():
    """transformers' BaseStreamer contract as HF's generate drives it: the prompt ids [1, L] first, then the new tokens."""
    prompt = [1, 2, 3, 4, 5, 1, 2]
    s = _Streamer()
    got, st, _ = _run(_cycle, prompt, 20, 4, streamer=s)
    assert s.ended and s.chunks[0] == [prompt]
    assert [len(c) for c in s.chunks[1:]] == [1] + st.accepted
    assert sum(s.chunks[1:], []) == got[len(prompt):]


def test_text_streamer_skip_prompt_shows_every_new_token():
    from transformers import TextStreamer
    from tests.stop_tokenizer import seeded_tokenizer
    tok = seeded_tokenizer(CFG.vocab, seed=3)

    class _Collect(TextStreamer):
        text = ''

        def on_finalized_text(self, text, stream_end=False):
            self.text += text
    s = _Collect(tok, skip_prompt=True)
    prompt = [40, 41, 42, 43, 44, 40, 41]
    got, st, _ = _run(lambda t, p: 40 + (t - 39) % 5 if 40 <= t <= 44 else 40, prompt, 20, 4, streamer=s)
    assert max(st.accepted) > 1
    assert s.text == tok.decode(got[len(prompt):]), (s.text, tok.decode(got[len(prompt):]))


def test_a_step_without_a_draft_runs_one_row():
    prompt = [1, 2, 3, 4, 5, 6, 7]                  # no repeated n-gram: no draft while the answer does not repeat
    got, st, eng = _run(lambda t, p: p + 50, prompt, 12, 6)
    assert got == prompt + [p + 50 for p in range(len(prompt) - 1, len(prompt) + 11)]
    assert eng.verify_rows == [(1, 0)] * 11 and st.accepted == [1] * 11


CFG128 = EngineConfig(image_size=28, vit_hidden=32, vit_heads=2, vit_layers=2, vit_mlp=64, hidden=256, n_heads=2,
                      n_layers=1, mlp=128, vocab=140, bbox_token=132, im_patch_token=131, im_start_token=134,
                      im_end_token=135)   # head_dim 128: the verify step's fused-RoPE GEMM applies


def _rule_eng_for_generate(rule):
    eng = _RuleEngine(rule)
    eng.cfg = CFG128
    return eng


def test_generate_dispatch_in_and_out_of_scope(monkeypatch):
    """In-scope calls go to the lookup loop; batch > 1, a padded mask, processors, stop strings and outputs run the
    plain loop and its launches, whatever prompt_lookup_num_tokens says."""
    seen = []
    real = E._generate_lookup

    def spy(*a, **kw):
        seen.append('lookup')
        return real(*a, **kw)
    monkeypatch.setattr(E, '_generate_lookup', spy)
    eng = _rule_eng_for_generate(_cycle)
    ids = torch.tensor([[1, 2, 3, 4, 5, 1, 2]])
    img = torch.zeros(1, 3, 28, 28)
    plain = E._generate(eng, ids, img, None, max_new_tokens=12, use_graph=False)
    got = E._generate(eng, ids, img, None, max_new_tokens=12, use_graph=False, prompt_lookup_num_tokens=3)
    assert seen == ['lookup'] and torch.equal(got, plain) and max(eng.lookup_accepted) > 1
    for kw in (dict(repetition_penalty=1.2), dict(no_repeat_ngram_size=3), dict(output_scores=True),
               dict(return_dict_in_generate=True), dict(attention_mask=torch.tensor([[0, 1, 1, 1, 1, 1, 1]]))):
        seen.clear()
        E._generate(eng, ids, img, None, max_new_tokens=6, use_graph=False, prompt_lookup_num_tokens=3, **kw)
        assert seen == [], kw
    seen.clear()
    two = torch.cat([ids, ids])
    out = E._generate(eng, two, torch.zeros(2, 3, 28, 28), None, max_new_tokens=6, use_graph=False,
                      prompt_lookup_num_tokens=3)
    assert seen == [] and torch.equal(out, E._generate(eng, two, torch.zeros(2, 3, 28, 28), None, max_new_tokens=6,
                                                        use_graph=False))


def test_generate_lookup_leaves_the_conversation_cache_as_the_plain_loop_does(monkeypatch):
    eng = _rule_eng_for_generate(_cycle)
    ids = torch.tensor([[1, 2, 3, 4, 5, 1, 2]])
    L = ids.shape[1]
    cache = KVCache(CFG128, 1, 4, 'cpu')

    def prefill_cached(c, input_ids, images, bboxes, mask=None, new_tokens=0):
        c.grow(input_ids.shape[1] + new_tokens)
        return eng.forward_device(input_ids, None, None, cache=c)
    eng.prefill_cached = prefill_cached
    out = E._generate(eng, ids, torch.zeros(1, 3, 28, 28), None, max_new_tokens=10, use_graph=False, cache=cache,
                      prompt_lookup_num_tokens=4)
    n = out.shape[1] - L
    assert n == 10 and cache.length == L + n - 1 and cache.max_len >= L + 10 + 4
    assert cache.ids[0, :L + n - 1].tolist() == out[0, :L + n - 1].tolist()
    assert bool((cache.ids[0, L + n - 1:] == -1).all())


def test_kv_cache_crop():
    c = KVCache(CFG, 1, 16, 'cpu')
    c.start(6, None, torch.arange(6)[None])
    c.set_source(None, [None])
    c.k[0][:, :6] = 1.0
    c.crop(4)
    assert c.length == 4 and c.ids[0].tolist()[:6] == [0, 1, 2, 3, -1, -1] and bool((c.k[0][:, :6] == 1).all())
    assert c.reusable(torch.arange(8)[None], None, [None]).tolist() == [4]
    c.crop(10)                                   # never lengthens
    assert c.length == 4
    c.lens = torch.tensor([4], dtype=torch.int32)
    c.crop(2)
    assert c.length == 2 and c.lens.tolist() == [2]


def test_g4r_cache_crop_moves_the_captured_step():
    from gpt4roi_b200.spi_llava import G4RCache
    c = G4RCache(KVCache(CFG, 1, 16, 'cpu'))
    c.kv.start(9, None, torch.arange(9)[None])

    class _Step:
        pos = torch.tensor([9], dtype=torch.int32)
    c.stepper = _Step()
    c.crop(7)
    assert c.get_seq_length() == 7 and c.stepper.pos.tolist() == [7]


def test_seam_resolves_the_option_as_hf_does(monkeypatch):
    from transformers import GenerationConfig
    from tests.test_model_seam_cpu import _tiny_model
    m = _tiny_model().eval()
    got = []

    class _Eng:
        cfg = CFG
        dev = torch.device('cpu')

        def generate(self, *a, **kw):
            got.append(kw)
            return torch.zeros(1, 2, dtype=torch.long)
    m._get_engine = lambda device: _Eng()
    ids = torch.tensor([[1, 2, 3]])
    m.generate(ids, max_new_tokens=4)
    assert 'prompt_lookup_num_tokens' not in got[-1]
    m.generate(ids, max_new_tokens=4, prompt_lookup_num_tokens=5)
    assert got[-1]['prompt_lookup_num_tokens'] == 5 and got[-1]['max_matching_ngram_size'] == 2
    m.generate(ids, max_new_tokens=4, generation_config=GenerationConfig(prompt_lookup_num_tokens=3,
                                                                         max_matching_ngram_size=4))
    assert got[-1]['prompt_lookup_num_tokens'] == 3 and got[-1]['max_matching_ngram_size'] == 4
    m.generation_config.prompt_lookup_num_tokens = 6
    m.generate(ids, max_new_tokens=4)
    assert got[-1]['prompt_lookup_num_tokens'] == 6
    m.generate(ids, max_new_tokens=4, prompt_lookup_num_tokens=2)
    assert got[-1]['prompt_lookup_num_tokens'] == 2


def test_prepare_inputs_passes_the_uncached_tokens():
    from gpt4roi_b200.spi_llava import G4RCache
    from tests.test_model_seam_cpu import _tiny_model
    m = _tiny_model().eval()
    c = G4RCache(KVCache(CFG, 1, 32, 'cpu'))
    c.kv.start(6, None, torch.arange(6)[None])
    ids = torch.arange(10)[None]                 # 6 cached, then the last accepted token and 3 drafts
    mi = m.prepare_inputs_for_generation(ids[:, :7], past_key_values=c, is_first_iteration=False)
    assert mi['input_ids'].tolist() == [[6]] and mi['logits_to_keep'] == 1
    mi = m.prepare_inputs_for_generation(ids, past_key_values=c, is_first_iteration=False)
    assert mi['input_ids'].tolist() == [[6, 7, 8, 9]]
    mi = m.prepare_inputs_for_generation(ids[:, :7], past_key_values=c)           # no flag: one token longer
    assert mi['input_ids'].tolist() == [[6]]
