"""CPU tests of continuous batching (engine.ContinuousBatcher and model.continuous_batcher): the scheduling -- first in,
first out admission, slot reuse, per-request answer lengths, eos and stop-string retirement, the sequences' layout and
the streamer's calls -- on a stub engine whose next token is (last token + 1) % vocab, and the seam's resolution of
generate() keywords.  The GPU tests run the same batcher on the real engine (tests/test_serve_gpu.py)."""
import pytest
import torch

from gpt4roi_b200.engine import ContinuousBatcher, EngineConfig, StopStrings

V = 140


class _StubEngine:
    """The engine surface the batcher uses, on the host: prefill and decode give one-hot((last id + 1) % vocab) logits.
    The prefill writes its prompt ids into the K cache it is given; `calls` records every prefill and decode step."""

    def __init__(self):
        self.cfg = EngineConfig(image_size=28, vit_hidden=32, vit_heads=2, vit_layers=2, vit_mlp=64, hidden=64,
                                n_heads=2, n_layers=1, mlp=128, vocab=V)
        self.dev, self.dt, self.calls = torch.device('cpu'), self.cfg.torch_dtype, []
        self.fail_on = -1

    def _logits(self, last):
        out = torch.zeros(last.shape[0], 1, V, dtype=self.dt)
        out[torch.arange(last.shape[0]), 0, (last + 1) % V] = 1.0
        return out

    def plan_boxes(self, bboxes):
        return bboxes

    def forward_device(self, input_ids, images, plan, validate=True, last_only=False, cache=None, **kw):
        assert last_only and cache is not None and cache.B == 1
        if input_ids[0, -1] == self.fail_on:      # e.g. a <bbox> count its boxes do not match (splice status 3)
            raise RuntimeError('gpt4roi_b200 C-ABI error 3: bad prompt')
        L = input_ids.shape[1]
        cache.start(L, None, input_ids)
        cache.k[0][0, :L, 0] = input_ids[0].to(self.dt)
        self.calls.append(('prefill', input_ids[0].tolist(), images is not None, plan))
        return self._logits(input_ids[:, -1])

    def decode_step(self, ids, cache, pos_dev=None):
        assert pos_dev is not None, 'the batcher passes pos_dev, so that cache.lens has one writer'
        self.calls.append(('decode', cache.lens.tolist()))
        return self._logits(ids[:, 0])


class _Streamer:
    def __init__(self):
        self.events = []

    def put(self, value):
        self.events.append(('put', value.tolist()))

    def end(self):
        self.events.append(('end',))


def test_fifo_admission_slot_reuse_and_answer_lengths():
    eng = _StubEngine()
    b = ContinuousBatcher(eng, slots=2, max_len=32)
    prompts = [[3, 10], [4, 5, 20], [7, 30], [40], [8, 9, 50]]
    lengths = [2, 5, 1, 3, 2]
    reqs = [b.submit(torch.tensor([p]), max_new_tokens=n) for p, n in zip(prompts, lengths)]
    order = []
    for _ in range(20):
        order += b.step()
        if not b.queue and all(r is None for r in b.running):
            break
    assert [r.done for r in reqs] == [True] * 5
    # admitted in submission order: the prefills come first in, first out
    assert [c[1] for c in eng.calls if c[0] == 'prefill'] == prompts
    for p, n, r in zip(prompts, lengths, reqs):
        assert r.sequences.tolist() == [p + [(p[-1] + 1 + i) % V for i in range(n)]]
        assert r.sequences.dtype == torch.int64
    # request 0 (2 tokens) leaves slot 0 after one step; request 2 (1 token) takes it and is done at admission, so
    # request 3 takes it in the same step, and request 4 after it; request 1 keeps slot 1 for its 5 tokens
    assert order == [reqs[0], reqs[2], reqs[3], reqs[4], reqs[1]]
    # the decode steps see each row's own length: its prompt plus the tokens fed so far
    assert [c[1] for c in eng.calls if c[0] == 'decode'] == [[2, 3], [1, 4], [2, 5], [3, 6]]
    # the last prefill into slot 0 wrote its prompt over the earlier requests' rows; slot 1 kept request 1's
    assert b.cache.k[0][0, :3, 0].tolist() == [8.0, 9.0, 50.0]
    assert b.cache.k[0][1, :3, 0].tolist() == [4.0, 5.0, 20.0]


def test_eos_retires_a_row_while_its_neighbour_continues():
    eng = _StubEngine()
    b = ContinuousBatcher(eng, slots=2, max_len=32)
    early = b.submit(torch.tensor([[1, 10]]), max_new_tokens=8, eos_token_id=13)
    late = b.submit(torch.tensor([60]), max_new_tokens=6, eos_token_id=[99])
    done = b.run()
    assert early.sequences.tolist() == [[1, 10, 11, 12, 13]]      # eos is part of the output, as in generate()
    assert late.sequences.tolist() == [[60, 61, 62, 63, 64, 65, 66]]
    assert done == [early, late]
    eos_first = b.submit(torch.tensor([[4]]), max_new_tokens=5, eos_token_id=5)
    assert b.step() == [eos_first] and eos_first.sequences.tolist() == [[4, 5]]   # done at admission: no decode step


def test_failed_admission_leaves_its_slot_idle_and_the_others_running():
    """A request whose prefill raises: step() raises, the request is retired with the error, and its slot -- left at
    length 31 of max_len 32 by an earlier request -- stays idle instead of decoding on past max_len."""
    eng = _StubEngine()
    eng.fail_on = 99
    b = ContinuousBatcher(eng, slots=2, max_len=32)
    long = b.submit(torch.tensor([[1]]), max_new_tokens=20)
    b.submit(torch.arange(100, 130)[None], max_new_tokens=2)               # slot 1: prompt 30 + 1 fed token
    b.step()
    assert b.running[1] is None and b.cache.lens.tolist() == [2, 31]
    st = _Streamer()
    bad = b.submit(torch.tensor([[5, 99]]), max_new_tokens=4, streamer=st)
    good = b.submit(torch.tensor([[40]]), max_new_tokens=3)
    with pytest.raises(RuntimeError, match='bad prompt'):
        b.step()
    assert bad.done and isinstance(bad.error, RuntimeError) and bad.tokens == [] and st.events == [('end',)]
    assert b.active.tolist() == [1, 0] and b.running[1] is None
    b.step()                                                                 # the next request takes slot 1
    assert b.running[1] is good
    b.run()
    assert b.cache.lens.max() <= 32 and b.active.tolist() == [0, 0]
    assert long.sequences.tolist() == [[1] + list(range(2, 22))]
    assert good.sequences.tolist() == [[40, 41, 42, 43]] and good.error is None


def test_stop_string_retires_at_the_token_that_completes_it():
    strings = ['x'] * V
    strings[21], strings[22], strings[23] = 'a#', '##', 'b'
    stops = StopStrings(strings, ['###'])
    eng = _StubEngine()
    b = ContinuousBatcher(eng, slots=3, max_len=32, stop_strings=stops)
    hit = b.submit(torch.tensor([[5, 20]]), max_new_tokens=10)        # 21 'a#', 22 '##': '###' ends in the second
    other = b.submit(torch.tensor([[70]]), max_new_tokens=4)
    in_prompt = b.submit(torch.tensor([[3, 21]]), max_new_tokens=10)   # begins in the prompt, ends in the first token
    b.run()
    assert hit.sequences.tolist() == [[5, 20, 21, 22]]
    assert other.sequences.tolist() == [[70, 71, 72, 73, 74]]
    assert in_prompt.sequences.tolist() == [[3, 21, 22]]


def test_streamer_gets_prompt_then_each_token_then_end():
    eng = _StubEngine()
    b = ContinuousBatcher(eng, slots=1, max_len=16)
    st = [_Streamer(), _Streamer()]
    r0 = b.submit(torch.tensor([[2, 3]]), max_new_tokens=3, streamer=st[0])
    r1 = b.submit(torch.tensor([9]), max_new_tokens=2, eos_token_id=10, streamer=st[1])
    b.run()
    assert st[0].events == [('put', [[2, 3]]), ('put', [4]), ('put', [5]), ('put', [6]), ('end',)]
    assert st[1].events == [('put', [[9]]), ('put', [10]), ('end',)]
    assert r0.done and r1.done


def test_submit_refusals_and_images_reach_the_prefill():
    eng = _StubEngine()
    b = ContinuousBatcher(eng, slots=2, max_len=8)
    with pytest.raises(ValueError, match='max_len'):
        b.submit(torch.zeros(1, 5, dtype=torch.long), max_new_tokens=4)
    b.submit(torch.zeros(1, 5, dtype=torch.long), max_new_tokens=3)          # exactly max_len
    with pytest.raises(NotImplementedError, match='one eos id'):
        b.submit(torch.tensor([[1]]), max_new_tokens=2, eos_token_id=[2, 3])
    with pytest.raises(ValueError, match='one prompt'):
        b.submit(torch.zeros(2, 3, dtype=torch.long))
    with pytest.raises(ValueError, match='max_new_tokens'):
        b.submit(torch.tensor([[1]]), max_new_tokens=0)
    boxes = [torch.tensor([[0.1, 0.1, 0.4, 0.4]])]
    b.submit(torch.tensor([[1, 2]]), images=torch.zeros(1, 3, 28, 28), bboxes=boxes, max_new_tokens=2)
    b.run()
    pre = [c for c in eng.calls if c[0] == 'prefill']
    assert pre[0][2] is False and pre[1][2] is True and pre[1][3] is boxes
    # sampling exists on the device only: the host stand-in refuses a sampled row when it runs
    s = ContinuousBatcher(_StubEngine(), slots=1, max_len=8)
    s.submit(torch.tensor([[1]]), max_new_tokens=2, do_sample=True, temperature=0.7, top_k=5,
             generator=torch.Generator().manual_seed(0))
    with pytest.raises(RuntimeError, match='CUDA device only'):
        s.step()


def test_sampled_request_takes_its_seed_at_submission_as_generate_does():
    from gpt4roi_b200.engine import sampling_seed
    b = ContinuousBatcher(_StubEngine(), slots=1, max_len=8)
    r = b.submit(torch.tensor([[1]]), max_new_tokens=2, do_sample=True, generator=torch.Generator().manual_seed(3))
    assert r.seed == sampling_seed(torch.Generator().manual_seed(3)) and not r.greedy
    g = b.submit(torch.tensor([[1]]), max_new_tokens=2, do_sample=True, temperature=0.0)    # temperature 0: the arg-max, no seed drawn
    assert g.greedy and g.seed == 0


# ---- the model seam ---------------------------------------------------------------------------------------------

def _seam(stub):
    from tests.test_model_seam_cpu import _tiny_model
    m = _tiny_model().eval()
    m._get_engine = lambda device: stub
    return m


def test_seam_resolves_generate_keywords_like_the_engine_loop():
    from transformers import GenerationConfig
    m = _seam(_StubEngine())
    sb = m.continuous_batcher(slots=2, max_len=16)
    ids = torch.tensor([[1, 2]])
    r = sb.submit(ids, max_new_tokens=3, do_sample=True)                            # HF's defaults: top_k 50, T 1
    assert (r.greedy, r.temperature, r.top_k, r.top_p) == (False, 1.0, 50, 1.0)
    r = sb.submit(ids, max_new_tokens=3, generation_config=GenerationConfig(do_sample=True, temperature=0.5, top_p=0.9, top_k=0))
    assert (r.greedy, r.temperature, r.top_k, r.top_p) == (False, 0.5, 0, 0.9)
    m.generation_config.do_sample, m.generation_config.top_k = True, 7                # the model's own config counts
    try:
        r = sb.submit(ids, max_new_tokens=3, temperature=0.3)
    finally:
        m.generation_config.do_sample, m.generation_config.top_k = False, 50
    assert (r.greedy, r.temperature, r.top_k) == (False, 0.3, 7)
    r = sb.submit(ids, max_new_tokens=2, eos_token_id=4, pad_token_id=0)
    assert r.greedy and r.eos_id == 4


@pytest.mark.parametrize('kw', [dict(repetition_penalty=1.3), dict(num_beams=2), dict(do_sample=True, min_p=0.1),
                                dict(do_sample=True, num_return_sequences=2),
                                dict(return_dict_in_generate=True, output_scores=True),
                                dict(no_repeat_ngram_size=2), dict(stop_strings=['###']),
                                dict(generation_config='stop_strings')])
def test_seam_refuses_what_only_generate_runs(kw):
    from transformers import GenerationConfig
    if kw.get('generation_config') == 'stop_strings':
        kw = dict(generation_config=GenerationConfig(stop_strings=['###']))
    m = _seam(_StubEngine())
    sb = m.continuous_batcher(slots=1, max_len=16)
    with pytest.raises(NotImplementedError, match='model.generate'):
        sb.submit(torch.tensor([[1, 2]]), max_new_tokens=2, **kw)
    assert not sb.batcher.queue


def test_seam_runs_the_batcher_greedy_and_with_stop_strings_from_the_tokenizer():
    from tests.stop_tokenizer import seeded_tokenizer
    m = _seam(_StubEngine())
    sb = m.continuous_batcher(slots=2, max_len=16)
    r = sb.submit(torch.tensor([[1, 2]]), max_new_tokens=3, tokenizer=object())   # no stop strings: tokenizer unused
    assert sb.run() == [r] and r.sequences.tolist() == [[1, 2, 3, 4, 5]]
    from transformers import GenerationConfig                # only the rule is read from it, as on the engine loop
    r = sb.submit(torch.tensor([[1, 2]]), max_new_tokens=2, generation_config=GenerationConfig(max_new_tokens=9))
    assert sb.run() == [r] and r.sequences.tolist() == [[1, 2, 3, 4]]
    with pytest.raises(ValueError, match='tokenizer'):
        m.continuous_batcher(stop_strings=['###'])
    tok = seeded_tokenizer(V, seed=5)
    # ids 3, 4, 5 are '#', '##', '###' (tests/stop_tokenizer.py): from prompt token 2, '###' ends in the second new token
    sb = m.continuous_batcher(slots=2, max_len=16, tokenizer=tok, stop_strings='###')
    r = sb.submit(torch.tensor([[1, 2]]), max_new_tokens=6)
    sb.run()
    assert r.sequences.tolist() == [[1, 2, 3, 4]]
