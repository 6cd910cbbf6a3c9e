"""CPU tests of stop strings in generate(): the lookup table of engine.StopStrings against transformers' own matcher
(StopStringCriteria) over seeded vocabularies, the builder's refusals and cache, the decode loop's stop / pad rule on a
CPU stand-in of the engine, and the model seam's resolution of stop_strings / tokenizer.  tests/test_stop_strings_gpu.py
runs the same table through the kernel and the real loops."""
import pytest
import torch

from gpt4roi_b200.engine import StopStrings
from tests.stop_tokenizer import FIXED, seeded_tokenizer
from tests.test_model_seam_cpu import _tiny_model
from tests.test_ragged_host_cpu import V, _batch, _Stub

EMPTY = FIXED.index('')
STOP_SETS = {'one_char': ['#'], 'hashes': ['###'], 'suffix_of_other': ['ab', 'bab'], 'shared_prefix': ['ab#', 'abx', 'ab'],
             'periodic': ['abab'], 'mixed': ['###', 'y.', 'abab']}


def clean_strings(tok):
    """The tokenizer's clean token strings as a list indexed by id (None: an id the vocabulary does not hold)."""
    from transformers.generation.stopping_criteria import StopStringCriteria
    strings, ids = StopStringCriteria.clean_tokenizer_vocab(tok)
    out = [None] * (max(ids) + 1)
    for s, i in zip(strings, ids):
        out[i] = s
    return out


def walk(stops, ids, lens, new):
    """ids [B, P + new]: right-padded prompts (lens valid tokens each) whose new tokens sit in the last `new` columns.
    -> hit bool [B, new]: the table walked from each row's prompt-derived state, one generated token at a time."""
    P = ids.shape[1] - new
    state = stops.initial_states(ids[:, :P], lens).to(torch.int64)
    hits = []
    for t in range(new):
        state, hit = stops.advance(ids[:, P + t], state)
        hits.append(hit)
    return torch.stack(hits, 1)


@pytest.mark.parametrize('name', sorted(STOP_SETS))
def test_table_equals_transformers_matcher_at_every_step(name):
    """2000 random id sequences per case (ids past the vocabulary included), prompts of four lengths, 10 generated
    tokens: at every step the table says exactly what StopStringCriteria says of the sequence so far -- the first hit
    and the steps without one.  With the empty-string token mapped away the comparison is with the stock matcher; with it
    in the generated part, with the matcher looking at the whole sequence instead of its last max(len(stop)) tokens (the
    one place the two differ, test_empty_string_tokens_are_transparent)."""
    from transformers.generation.stopping_criteria import StopStringCriteria
    stops = STOP_SETS[name]
    n_tok, new = 300, 10
    tok = seeded_tokenizer(n_tok, seed=3)
    table = StopStrings(clean_strings(tok), stops)
    assert table.table.shape == (n_tok + 1, table.S) and table.S <= 1 + sum(len(s) for s in stops)
    stock, whole = StopStringCriteria(tok, stops), StopStringCriteria(tok, stops)
    whole.maximum_token_len = 1 << 20
    g = torch.Generator().manual_seed(len(name))
    checked = found = 0
    for P in (1, 2, 4, 7):
        ids = torch.randint(0, n_tok + 4, (500, P + new), generator=g)
        ids[:, :P] = torch.where(ids[:, :P] == EMPTY, EMPTY + 1, ids[:, :P])
        for variant, crit in ((torch.where(ids == EMPTY, EMPTY + 1, ids), stock), (ids, whole)):
            lens = torch.full((500,), P)
            padded = torch.cat([variant[:, :P], torch.zeros(500, 3, dtype=torch.int64), variant[:, P:]], 1)   # right-padded
            ours = walk(table, padded, lens, new)
            for t in range(new):
                want = crit(variant[:, :P + t + 1], None)
                assert torch.equal(ours[:, t], want), (name, P, t, (ours[:, t] != want).nonzero().flatten()[:5])
            checked += ours.numel()
            found += int(ours.sum())
    print('%s: %d (sequence, step) pairs, %d hits' % (name, checked, found))
    assert found > 50


def test_empty_string_tokens_are_transparent():
    """A token whose string is empty neither advances nor breaks a match, as in transformers' matcher; an id outside the
    vocabulary breaks it.  transformers looks at the last max(len(stop)) tokens only, so a match that empty tokens
    stretch over more tokens than that is found by the table and missed there."""
    from transformers.generation.stopping_criteria import StopStringCriteria
    tok = seeded_tokenizer(40, seed=0)
    a, b, ab = FIXED.index('a'), FIXED.index('b'), FIXED.index('ab')
    for stop, seq, ours, hf in (('abab', [a, EMPTY, b, ab], True, True), ('abab', [a, 40, b, ab], False, False),
                                ('aba', [ab, EMPTY, a], True, True), ('aba', [a, b, EMPTY], False, False),
                                ('ab', [a, EMPTY, b], True, False), ('aba', [ab, EMPTY, EMPTY, a], True, False)):
        table = StopStrings(clean_strings(tok), [stop])
        ids = torch.tensor([seq])
        got = walk(table, ids, torch.tensor([1]), len(seq) - 1)[0, -1]
        assert bool(got) == ours and bool(StopStringCriteria(tok, [stop])(ids, None)[0]) == hf, (stop, seq)


def test_stop_token_ids_and_prompt_window():
    strings = ['', 'a', 'b', 'ab', 'c']
    table = StopStrings(strings, ['abc'], stop_token_ids=[2])
    state, hit = table.advance(torch.tensor([2, 1, 4]), torch.zeros(3, dtype=torch.int64))
    assert hit.tolist() == [True, False, False] and state.tolist() == [0, 1, 0]
    # the prompt's tail sets the state: 'ab' in the prompt, 'c' as the first new token
    ids = torch.tensor([[1, 2, 0, 0], [4, 3, 0, 0], [3, 0, 0, 0], [1, 4, 3, 1]])
    s0 = table.initial_states(ids, torch.tensor([2, 2, 1, 4]))
    assert s0.dtype == torch.int32 and s0.tolist() == [0, 2, 2, 1]   # row 0 ends on the stop token: state back at the root
    assert table.advance(torch.full((4,), 4), s0.to(torch.int64))[1].tolist() == [False, True, True, False]


def test_builder_refusals_and_cache():
    strings = ['', 'a', 'b', '#', None, 'ab']
    for bad in ([], [''], ['ab', ''], [3]):
        with pytest.raises(ValueError):
            StopStrings(strings, bad)
    with pytest.raises(ValueError, match='no token'):
        StopStrings(strings, ['zz'])
    with pytest.raises(ValueError, match='limit'):
        StopStrings(['a'] * 40000, ['a' * 1000])
    with pytest.raises(ValueError, match='outside the vocabulary'):
        StopStrings(strings, ['ab'], stop_token_ids=[6])
    one, two = StopStrings(strings, ['ab', '#']), StopStrings(list(strings), ('ab', '#'))
    assert one.table is two.table and one.table.dtype == torch.int16
    assert StopStrings(strings, 'ab').stop_strings == ('ab',)
    assert StopStrings(strings, ['ab']).table is not one.table
    # an id the vocabulary does not hold (4) and ids past it reset the state without a hit
    s, hit = one.advance(torch.tensor([4, 6, 99, -1]), torch.ones(4, dtype=torch.int64))
    assert s.tolist() == [0, 0, 0, 0] and not hit.any()


def _letters():
    """Token i's string is the i-th letter from 'A': the stub engine emits last + 1, so every row spells the alphabet."""
    return [chr(ord('A') + i) for i in range(V)]


def test_loop_stops_each_row_at_its_own_step_and_pads_like_transformers():
    ids, mask, _, _ = _batch()                     # rows end in G, I, J: they go on H I J K.., J K L M.., K L M N..
    images = torch.zeros(3, 3, 4, 4)
    stops = StopStrings(_letters(), ['HI', 'KLM'])
    out = _Stub().generate(ids, images, None, max_new_tokens=8, attention_mask=mask, eos_token_id=40, pad_token_id=0,
                           stop_strings=stops)
    assert out[:, :4].tolist() == ids.tolist()
    assert out[:, 4:].tolist() == [[7, 8, 0, 0], [9, 10, 11, 12], [10, 11, 12, 0]]
    # no eos / pad in force: transformers pads nothing, finished rows keep generating, the loop still ends with the last row
    out = _Stub().generate(ids, images, None, max_new_tokens=8, attention_mask=mask, stop_strings=stops)
    assert out[:, 4:].tolist() == [[7, 8, 9, 10], [9, 10, 11, 12], [10, 11, 12, 13]]
    out = _Stub().generate(ids, images, None, max_new_tokens=8, attention_mask=mask, pad_token_id=0, stop_strings=stops)
    assert out.shape == (3, 8)
    # eos and a stop string finish rows alike; a stop string may begin in the prompt (row 0: G | H)
    out = _Stub().generate(ids, images, None, max_new_tokens=8, attention_mask=mask, eos_token_id=11, pad_token_id=0,
                           stop_strings=StopStrings(_letters(), ['GH', 'LMN']))
    assert out[:, 4:].tolist() == [[7, 0, 0], [9, 10, 11], [10, 11, 0]]
    # max_new_tokens ends the loop when a row never matches
    out = _Stub().generate(ids, images, None, max_new_tokens=3, attention_mask=mask, eos_token_id=40, pad_token_id=0,
                           stop_strings=StopStrings(_letters(), ['HI']))
    assert out[:, 4:].tolist() == [[7, 8, 0], [9, 10, 11], [10, 11, 12]]
    # the same prompts left-padded give the same answer
    _, _, ids_l, mask_l = _batch()
    out_l = _Stub().generate(ids_l, images, None, max_new_tokens=8, attention_mask=mask_l, eos_token_id=40, pad_token_id=0,
                             stop_strings=stops)
    assert out_l[:, 4:].tolist() == [[7, 8, 0, 0], [9, 10, 11, 12], [10, 11, 12, 0]]


def test_host_stopping_criteria_still_fire_beside_stop_strings():
    ids, mask, _, _ = _batch()
    seen = []

    def after_two(out_ids, scores):
        seen.append(out_ids.shape[1])
        return out_ids.shape[1] >= 6
    out = _Stub().generate(ids, torch.zeros(3, 3, 4, 4), None, max_new_tokens=8, attention_mask=mask, eos_token_id=40,
                           pad_token_id=0, stopping_criteria=[after_two], stop_strings=StopStrings(_letters(), ['KLM']))
    assert seen == [5, 6] and out[:, 4:].tolist() == [[7, 8], [9, 10], [10, 11]]
    with pytest.raises(NotImplementedError, match='use_hf_loop=True'):
        _Stub().generate(ids, torch.zeros(3, 3, 4, 4), None, num_beams=2, stop_strings=StopStrings(_letters(), ['KLM']))


def test_seam_resolves_stop_strings_like_transformers():
    from transformers import GenerationConfig
    from gpt4roi_b200.spi_llava import resolve_generate, stop_strings_from_tokenizer
    m = _tiny_model()
    tok = seeded_tokenizer(120, seed=1)

    def stops(**kw):
        return resolve_generate(m, 3, None, **kw).stop_strings
    assert stops() is None
    assert stops(stop_strings='###') == ('###',)
    gc = GenerationConfig(stop_strings=['ab', '#'])
    assert stops(generation_config=gc) == ('ab', '#')
    assert stops(stop_strings=['y.'], generation_config=gc) == ('y.',)     # explicit kwarg first
    m.generation_config.stop_strings = ['abab']                           # then the model's config
    assert stops() == ('abab',)
    assert stops(generation_config=gc) == ('ab', '#')
    m._get_engine = lambda device: pytest.fail('no engine should be built')
    with pytest.raises(ValueError, match='could not locate a tokenizer'):
        m.generate(torch.tensor([[1, 5, 9]]), images=torch.zeros(1, 3, 28, 28), max_new_tokens=4)
    built = stop_strings_from_tokenizer(tok, ['###'])
    assert built is stop_strings_from_tokenizer(tok, '###') and built.V_tok == 120
    assert built.table is StopStrings(clean_strings(tok), ['###']).table


def test_seam_generate_hands_the_table_to_the_engine_and_refuses_beams():
    m = _tiny_model().eval()
    tok = seeded_tokenizer(120, seed=1)
    calls = []

    class _Engine:
        def generate(self, input_ids, images, bboxes, **kw):
            calls.append(kw)
            return input_ids
    m._get_engine = lambda device: _Engine()
    ids = torch.tensor([[1, 5, 9]])
    m.generate(ids, images=torch.zeros(1, 3, 28, 28), max_new_tokens=4, stop_strings=['###', 'ab'], tokenizer=tok,
               pad_token_id=0, eos_token_id=2)
    got = calls[-1]['stop_strings']
    assert isinstance(got, StopStrings) and got.stop_strings == ('###', 'ab') and calls[-1]['pad_token_id'] == 0
    m.generate(ids, images=torch.zeros(1, 3, 28, 28), max_new_tokens=4, tokenizer=tok)   # a tokenizer alone is not an error
    assert calls[-1]['stop_strings'] is None
    with pytest.raises(ValueError, match='could not locate a tokenizer'):
        m.generate(ids, images=torch.zeros(1, 3, 28, 28), max_new_tokens=4, stop_strings=['###'])
    with pytest.raises(NotImplementedError, match='stop_strings runs on the HF loop only'):
        m.generate(ids, images=torch.zeros(1, 3, 28, 28), max_new_tokens=4, num_beams=2, stop_strings=['###'],
                   tokenizer=tok)
