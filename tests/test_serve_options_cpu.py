"""CPU tests of per-request options in continuous batching (ContinuousBatcher(request_options=True)): the refusals of a
batcher built without the option, the history-dependent logits processors and stop strings of each request, the union
with the batcher's stop strings, the rows' history after every kind of admission, and the seam's resolution -- on the
stub engines of tests/test_serve_cpu.py and tests/test_serve_prefix_cpu.py, whose next token is (last id + 1) % vocab.
The GPU tests run the same batcher on the real engine (tests/test_serve_options_gpu.py)."""
import pytest
import torch

from gpt4roi_b200 import kernels
from gpt4roi_b200.engine import ContinuousBatcher, LogitsProcessors
from tests.test_serve_cpu import V, _seam, _StubEngine
from tests.test_serve_prefix_cpu import IMG, _ids, _image, _Stub

OPTIONS = [dict(repetition_penalty=1.3), dict(no_repeat_ngram_size=2), dict(min_length=6, eos_token_id=3),
           dict(min_new_tokens=2, eos_token_id=3), dict(min_new_tokens=2, length_eos_ids=[3, 9])]


def _tok():
    from tests.stop_tokenizer import seeded_tokenizer
    return seeded_tokenizer(V, seed=5)     # ids 3, 4, 5: '#', '##', '###'; id 1 '▁abcdef'


def _stops(strings):
    from gpt4roi_b200.spi_llava import stop_strings_from_tokenizer
    return stop_strings_from_tokenizer(_tok(), strings)


def _history(b, s, req):
    n = req.input_ids.shape[1] + len(req.tokens)
    return b.history[s, :n].tolist()


@pytest.mark.parametrize('kw', OPTIONS + [dict(stop_strings='###')])
def test_plain_batcher_refuses_each_option_and_an_opted_in_one_accepts_it(kw):
    kw = dict(kw, stop_strings=_stops(kw['stop_strings'])) if 'stop_strings' in kw else kw
    b = ContinuousBatcher(_StubEngine(), slots=1, max_len=16)
    with pytest.raises(NotImplementedError, match='model.generate.*request_options=True'):
        b.submit(torch.tensor([[1, 2]]), max_new_tokens=2, **kw)
    assert not b.queue
    b = ContinuousBatcher(_StubEngine(), slots=1, max_len=16, request_options=True)
    r = b.submit(torch.tensor([[1, 2]]), max_new_tokens=2, **kw)
    b.run()
    assert r.done and len(r.tokens) >= 1


def test_neutral_values_are_accepted_everywhere_and_change_nothing():
    for opt in (False, True):
        b = ContinuousBatcher(_StubEngine(), slots=1, max_len=16, request_options=opt)
        r = b.submit(torch.tensor([[1, 2]]), max_new_tokens=3, repetition_penalty=1.0, no_repeat_ngram_size=0,
                     min_length=0, min_new_tokens=0, eos_token_id=4)
        b.run()
        assert r.tokens == [3, 4] and r.processors is None


def test_opted_in_submit_checks_its_values():
    b = ContinuousBatcher(_StubEngine(), slots=1, max_len=16, request_options=True)
    with pytest.raises(NotImplementedError, match='at most 4 eos ids'):
        b.submit(torch.tensor([[1, 2]]), max_new_tokens=2, min_new_tokens=1, length_eos_ids=[1, 2, 3, 4, 5])
    with pytest.raises(ValueError, match='repetition_penalty must be > 0'):
        b.submit(torch.tensor([[1, 2]]), max_new_tokens=2, repetition_penalty=0.0)
    with pytest.raises(ValueError, match='token ids'):
        from gpt4roi_b200.engine import StopStrings
        b.submit(torch.tensor([[1, 2]]), max_new_tokens=2, stop_strings=StopStrings(['a', 'b', 'ab'], 'ab'))
    big = ContinuousBatcher(_StubEngine(), slots=1, max_len=kernels.PROC_LIST_MAX + 8, request_options=True)
    ids = torch.ones((1, kernels.PROC_LIST_MAX), dtype=torch.int64)
    with pytest.raises(NotImplementedError, match='at most %d prompt' % kernels.PROC_LIST_MAX):
        big.submit(ids, max_new_tokens=2, do_sample=True, repetition_penalty=1.2)
    big.submit(ids, max_new_tokens=2, repetition_penalty=1.2)            # greedy: no list, no limit
    assert not b.queue and len(big.queue) == 1


def test_min_new_tokens_suppresses_the_eos_the_stub_emits_first():
    b = ContinuousBatcher(_StubEngine(), slots=2, max_len=16, request_options=True)
    plain = b.submit(torch.tensor([[1, 2]]), max_new_tokens=6, eos_token_id=3)
    held = b.submit(torch.tensor([[1, 2]]), max_new_tokens=6, eos_token_id=3, min_new_tokens=2)
    b.run()
    assert plain.tokens == [3]
    # eos 3 is -inf for new tokens 0 and 1: the arg-max of the rest is id 0, then the stub counts up to eos again
    assert held.tokens == [0, 1, 2, 3]


def test_no_repeat_ngram_size_bans_the_repeat_the_stub_would_produce():
    b = ContinuousBatcher(_StubEngine(), slots=2, max_len=16, request_options=True)
    prompt = torch.tensor([[5, 6, 7, 5, 6]])
    plain = b.submit(prompt, max_new_tokens=3)
    banned = b.submit(prompt, max_new_tokens=3, no_repeat_ngram_size=3)
    b.run()
    assert plain.tokens == [7, 8, 9]
    assert banned.tokens[0] != 7 and banned.tokens == [0, 1, 2]


def test_repetition_penalty_rows_equal_logits_processors_on_their_own_history():
    eng = _StubEngine()
    b = ContinuousBatcher(eng, slots=2, max_len=16, request_options=True)
    r = b.submit(torch.tensor([[9, 4]]), max_new_tokens=4, repetition_penalty=2.0)
    b.run()
    # one-hot logits: the next id has 1, divided by 2 when it is in the history -- still the arg-max
    assert r.tokens == [5, 6, 7, 8]
    hist = torch.tensor([[9, 4] + r.tokens])
    lp = LogitsProcessors(hist, 2, repetition_penalty=2.0)
    assert float(lp.apply(eng._logits(torch.tensor([4]))[:, 0].float(), 0)[0, 5]) == 1.0


def test_a_request_stop_string_retires_only_its_own_request():
    b = ContinuousBatcher(_StubEngine(), slots=2, max_len=16, request_options=True)
    stopped = b.submit(torch.tensor([[1, 2]]), max_new_tokens=6, stop_strings=_stops('###'))
    free = b.submit(torch.tensor([[1, 2]]), max_new_tokens=6)
    b.run()
    assert stopped.tokens == [3, 4]          # '#' + '##' ends '###'
    assert free.tokens == [3, 4, 5, 6, 7, 8]
    # the batcher's own stop strings are every other row's default
    b = ContinuousBatcher(_StubEngine(), slots=2, max_len=16, stop_strings=_stops('###'), request_options=True)
    default = b.submit(torch.tensor([[1, 2]]), max_new_tokens=6)
    own = b.submit(torch.tensor([[1, 2]]), max_new_tokens=6, stop_strings=_stops('f#'))
    b.run()
    assert default.tokens == [3, 4] and own.tokens == [3]
    assert all(t is None for t in b.row_stops)     # retired rows drop their tables


def test_the_union_with_the_batchers_strings_stops_at_whichever_comes_first():
    m = _seam(_StubEngine())
    sb = m.continuous_batcher(slots=2, max_len=16, tokenizer=_tok(), stop_strings='###', request_options=True)
    early = sb.submit(torch.tensor([[1, 2]]), max_new_tokens=6, stop_strings=['f#'])     # 'abcdef' + '#': token 0
    late = sb.submit(torch.tensor([[1, 2]]), max_new_tokens=6, stop_strings=['#####'])   # '###' first, at token 1
    sb.run()
    assert early.tokens == [3] and late.tokens == [3, 4]
    assert early.stops.stop_strings == ('###', 'f#') and late.stops.stop_strings == ('###', '#####')


def test_history_holds_prompt_and_tokens_after_admission_and_after_a_row_changes_tenant():
    b = ContinuousBatcher(_StubEngine(), slots=1, max_len=16, request_options=True)
    a = b.submit(torch.tensor([[20, 21, 22, 23, 24, 25]]), max_new_tokens=4, repetition_penalty=1.5)
    b.step()
    assert _history(b, 0, a) == [20, 21, 22, 23, 24, 25, 26, 27]
    b.run()
    assert _history(b, 0, a) == [20, 21, 22, 23, 24, 25, 26, 27, 28, 29]
    c = b.submit(torch.tensor([[40, 41]]), max_new_tokens=3, no_repeat_ngram_size=2)     # a new tenant, shorter
    b.run()
    assert c.tokens == [42, 43, 44] and _history(b, 0, c) == [40, 41, 42, 43, 44]
    assert int(b.prompt_len[0]) == 2 and int(b.ngram[0]) == 2 and float(b.penalty[0]) == 1.0


def test_history_after_a_prefix_reuse_admission_is_the_whole_submitted_prompt():
    eng = _Stub()
    b = ContinuousBatcher(eng, slots=2, max_len=40, prefix_reuse=True, request_options=True)
    img = _image(0)
    t1 = b.submit(_ids([1], IMG, [10, 11]), images=img, max_new_tokens=3)
    b.run()
    conv = _ids([1], IMG, [10, 11], t1.tokens, [14])
    t2 = b.submit(conv, images=img, max_new_tokens=4, repetition_penalty=1.5)
    b.run()
    assert t2.reused > 0 and 'extend' in eng.kinds()
    s = next(s for s in range(2) if b.row_record(s).shape[0] >= conv.shape[1])
    assert _history(b, s, t2) == conv[0].tolist() + t2.tokens


# ---- the seam -------------------------------------------------------------------------------------------------------

def test_seam_resolves_stop_strings_from_the_kwarg_then_generation_config_then_the_model():
    from transformers import GenerationConfig
    m = _seam(_StubEngine())
    sb = m.continuous_batcher(slots=1, max_len=16, tokenizer=_tok(), request_options=True)
    ids = torch.tensor([[1, 2]])
    gc = GenerationConfig(stop_strings=['##'])
    r = sb.submit(ids, max_new_tokens=4, stop_strings=['###'], generation_config=gc)
    assert r.stops.stop_strings == ('###',)
    r = sb.submit(ids, max_new_tokens=4, generation_config=gc)
    assert r.stops.stop_strings == ('##',)
    m.generation_config.stop_strings = ['f#']
    try:
        r = sb.submit(ids, max_new_tokens=4)
    finally:
        m.generation_config.stop_strings = None
    assert r.stops.stop_strings == ('f#',)
    # a repeated stop set is one table: no new vocabulary pass
    assert sb.submit(ids, max_new_tokens=4, stop_strings=['###']).stops is sb.submit(
        ids, max_new_tokens=4, stop_strings=['###']).stops
    assert len(sb._vocab) == 1


def test_seam_min_new_tokens_sets_min_length_from_the_input_length():
    m = _seam(_StubEngine())
    sb = m.continuous_batcher(slots=1, max_len=16, request_options=True)
    r = sb.submit(torch.tensor([[1, 2, 3]]), max_new_tokens=4, min_new_tokens=2, eos_token_id=4)
    assert r.processors == dict(repetition_penalty=1.0, no_repeat_ngram_size=0, min_length=5, min_new_tokens=2,
                                eos_ids=[4])
    sb.run()
    assert r.tokens == [0, 1, 2, 3]      # eos 4 suppressed for the first two new tokens
    r = sb.submit(torch.tensor([[1, 2, 3]]), max_new_tokens=4, repetition_penalty=1.2, no_repeat_ngram_size=3)
    assert r.processors['repetition_penalty'] == pytest.approx(1.2) and r.processors['no_repeat_ngram_size'] == 3


def test_seam_stop_strings_need_a_tokenizer():
    from gpt4roi_b200.spi_llava import _STOP_STRINGS_NEED_TOKENIZER
    m = _seam(_StubEngine())
    sb = m.continuous_batcher(slots=1, max_len=16, request_options=True)
    with pytest.raises(ValueError, match='tokenizer') as e:
        sb.submit(torch.tensor([[1, 2]]), max_new_tokens=2, stop_strings=['###'])
    assert str(e.value) == _STOP_STRINGS_NEED_TOKENIZER
    r = sb.submit(torch.tensor([[1, 2]]), max_new_tokens=6, stop_strings=['###'], tokenizer=_tok())
    sb.run()
    assert r.tokens == [3, 4]


@pytest.mark.parametrize('kw', [dict(do_sample=True, min_p=0.1), dict(do_sample=True, typical_p=0.5),
                                dict(bad_words_ids=[[7]]), dict(num_beams=2),
                                dict(do_sample=True, num_return_sequences=2),
                                dict(return_dict_in_generate=True, output_scores=True),
                                dict(output_hidden_states=True), dict(past_key_values=object())])
def test_seam_with_options_still_refuses_what_only_generate_runs(kw):
    m = _seam(_StubEngine())
    sb = m.continuous_batcher(slots=1, max_len=16, request_options=True)
    with pytest.raises(NotImplementedError, match='model.generate'):
        sb.submit(torch.tensor([[1, 2]]), max_new_tokens=2, **kw)
    assert not sb.batcher.queue
