"""CPU tests of several sampled answers per prompt (generate(do_sample=True, num_return_sequences=N)): the model seam's
resolution of num_return_sequences and its refusals, and the engine loop's row layout on a CPU stand-in of the engine
(tests/test_ragged_host_cpu.py), with a host draw that sends each row of a prompt down its own path.
tests/test_multisample_gpu.py runs the shared-prefix attention kernel and the real loops."""
import pytest
import torch

from gpt4roi_b200 import engine
from gpt4roi_b200.engine import SampleCache, StopStrings
from tests.test_model_seam_cpu import _tiny_model
from tests.test_ragged_host_cpu import V, _batch, _Stub
from tests.test_stop_strings_cpu import _letters

IMAGES = torch.zeros(3, 3, 4, 4)


class _RowSampler(engine.Sampler):
    """Host stand-in for the device draw: row r takes the arg-max shifted by r % N, so sample i of a prompt whose
    stub rule is last + 1 steps by 1 + i.  The eos -> pad rule and the stop strings run as in Sampler."""
    N = 1

    def _host(self, logits, out, update):
        x = logits.reshape(logits.shape[0], -1)
        x = torch.stack([torch.roll(x[r], r % self.N) for r in range(x.shape[0])])
        self.greedy = True
        return super()._host(x[:, None], out, update)


def _run(monkeypatch, N, ids, mask, **kw):
    monkeypatch.setattr(_RowSampler, 'N', N)
    monkeypatch.setattr(engine, 'Sampler', _RowSampler)
    stub = _Stub()
    seen = []
    step = stub.decode_step

    def decode_step(tok, cache, pos_dev=None):
        seen.append((tok.shape[0], type(cache).__name__, cache.lens.clone()))
        return step(tok, cache, pos_dev)
    stub.decode_step = decode_step
    out = stub.generate(ids, IMAGES, None, do_sample=True, temperature=0.7, num_return_sequences=N,
                        attention_mask=mask, **kw)
    return out, stub, seen


def _expected(lasts, N, n, eos=None, pad=None, stop=None):
    """Row b*N + i: last_b + k * (1 + i) for k = 1.., finished at eos or at the end of a stop string (letters), padded
    after when eos and pad are given; the loop ends when every row is finished or after n tokens."""
    rows, ends = [], []
    for last in lasts:
        for i in range(N):
            seq, done, text, end = [], False, '', n
            for k in range(1, n + 1):
                t = (last + k * (1 + i)) % V
                if done and eos is not None and pad is not None:
                    t = pad
                seq.append(t)
                if not done:
                    text += chr(ord('A') + t)
                    done = t == eos or (stop is not None and text.endswith(stop))
                    end = k if done else n
            rows.append(seq)
            ends.append(end)
    return [r[:max(ends)] for r in rows]


def test_rows_are_interleaved_per_prompt_and_continue_on_their_own(monkeypatch):
    ids, mask, ids_l, mask_l = _batch()            # last tokens 6, 8, 9
    out, stub, seen = _run(monkeypatch, 2, ids, mask, max_new_tokens=5)
    assert out.shape == (6, 9)
    assert torch.equal(out[:, :4], ids.repeat_interleave(2, 0))                       # the prompts as given, b*N + i
    assert out[:, 4:].tolist() == _expected([6, 8, 9], 2, 5)
    assert len(stub.seen) == 1 and tuple(stub.seen[0][0].shape) == (3, 4)          # one prefill, at batch B
    assert seen[0][:2] == (6, 'SampleCache') and seen[0][2].tolist() == [4, 4, 2, 2, 1, 1]
    out_l, _, _ = _run(monkeypatch, 2, ids_l, mask_l, max_new_tokens=5)             # left-padded: the same answers
    assert torch.equal(out_l[:, :4], ids_l.repeat_interleave(2, 0)) and torch.equal(out_l[:, 4:], out[:, 4:])
    out4, _, _ = _run(monkeypatch, 4, ids, mask, max_new_tokens=3)
    assert out4[:, 4:].tolist() == _expected([6, 8, 9], 4, 3)


def test_each_row_stops_on_its_own(monkeypatch):
    ids, mask, _, _ = _batch()
    # eos 12: rows stop at steps 6, 3, 4, 2, 3 and never (11, 13, 15, ..); finished rows get pad
    out, _, _ = _run(monkeypatch, 2, ids, mask, max_new_tokens=8, eos_token_id=12, pad_token_id=0)
    assert out[:, 4:].tolist() == _expected([6, 8, 9], 2, 8, eos=12, pad=0)
    # stop strings J, K, L end every row, at steps 3, 2, 1, 1, 1, 1: the loop ends with the last one
    out, _, _ = _run(monkeypatch, 2, ids, mask, max_new_tokens=8, eos_token_id=40, pad_token_id=0,
                     stop_strings=StopStrings(_letters(), ['J', 'K', 'L']))
    want = _expected([6, 8, 9], 2, 8, eos=40, pad=0, stop=('J', 'K', 'L'))
    assert out[:, 4:].tolist() == want and len(want[0]) == 3
    # stop strings, per row: 'KM' ends rows I K M and K M; the others run on
    out, _, _ = _run(monkeypatch, 2, ids, mask, max_new_tokens=6, eos_token_id=40, pad_token_id=0,
                     stop_strings=StopStrings(_letters(), ['KM']))
    assert out[:, 4:].tolist() == _expected([6, 8, 9], 2, 6, eos=40, pad=0, stop='KM')
    # host stopping_criteria see all B * N rows
    shapes = []

    def crit(out_ids, scores):
        shapes.append((tuple(out_ids.shape), tuple(scores.shape)))
        return False
    _run(monkeypatch, 2, ids, mask, max_new_tokens=3, stopping_criteria=[crit])
    assert shapes == [((6, 5), (6, V)), ((6, 6), (6, V)), ((6, 7), (6, V))]


def test_engine_refusals():
    eng = engine.PrefillEngine.__new__(engine.PrefillEngine)
    ids = torch.tensor([[1, 5, 9]])
    with pytest.raises(ValueError, match='num_return_sequences'):
        eng.generate(ids, None, None, num_return_sequences=2)                 # greedy
    with pytest.raises(NotImplementedError, match='use_hf_loop=True'):
        eng.generate(ids, None, None, do_sample=True, num_return_sequences=2, cache=object())
    cfg = engine.EngineConfig(hidden=64, n_heads=1, n_layers=1, mlp=128, vocab=V)
    with pytest.raises(ValueError, match='1..16'):
        SampleCache(cfg, 1, 17, 4, 4, 'cpu')
    c = SampleCache(cfg, 2, 3, 4, 5, 'cpu')
    assert c.full_k[0].shape[:2] == (2 + 6, 9) and c.k[0].shape[0] == 6 and c.prompt.k[0].shape[0] == 2
    c.start(torch.tensor([4, 2]))
    assert c.lens.tolist() == [4, 4, 4, 2, 2, 2] and c.prompt_lens.tolist() == [4, 2] and c.length == 4


def test_seam_resolves_num_return_sequences_like_transformers():
    from transformers import GenerationConfig
    from gpt4roi_b200.spi_llava import resolve_generate
    m = _tiny_model()

    def nrs(**kw):
        return resolve_generate(m, 5, None, **kw).num_return_sequences
    assert nrs() == 1
    assert nrs(do_sample=True, num_return_sequences=3) == 3
    gc = GenerationConfig(do_sample=True, num_return_sequences=4)
    assert nrs(generation_config=gc) == 4
    assert nrs(generation_config=gc, num_return_sequences=2) == 2     # explicit kwarg first
    m.generation_config.do_sample, m.generation_config.num_return_sequences = True, 5            # then the model's config
    assert nrs() == 5
    assert nrs(generation_config=gc) == 4
    m.generation_config.do_sample, m.generation_config.num_return_sequences = False, 1
    # sampling parameters resolve as before
    assert resolve_generate(m, 5, None, do_sample=True, temperature=0.7, num_return_sequences=3)[:4] == \
        (True, 0.7, 50, 1.0)
    # greedy with N > 1: HF's own ValueError, at the resolution and through generate
    with pytest.raises(ValueError, match='num_return_sequences'):
        nrs(do_sample=False, num_return_sequences=2)
    with pytest.raises(ValueError, match='num_return_sequences'):
        nrs(num_return_sequences=2)
    m._get_engine = lambda device: pytest.fail('no engine should be built')
    with pytest.raises(ValueError, match='num_return_sequences'):
        m.generate(torch.tensor([[1, 5, 9]]), images=torch.zeros(1, 3, 28, 28), num_return_sequences=2)


def test_seam_routes_samples_to_the_engine_and_beams_unchanged():
    from transformers import DynamicCache
    m = _tiny_model().eval()
    calls = []

    class _Engine:
        def generate(self, input_ids, images, bboxes, **kw):
            calls.append(kw)
            return input_ids
    m._get_engine = lambda device: _Engine()
    ids = torch.tensor([[1, 5, 9]])
    img = torch.zeros(1, 3, 28, 28)
    m.generate(ids, images=img, max_new_tokens=4, do_sample=True, temperature=0.7, num_return_sequences=5)
    assert calls[-1]['num_return_sequences'] == 5 and calls[-1]['do_sample'] is True
    assert calls[-1]['temperature'] == 0.7 and calls[-1]['top_k'] == 50 and calls[-1]['cache'] is None
    m.generate(ids, images=img, max_new_tokens=4, do_sample=True)
    assert calls[-1]['num_return_sequences'] == 1
    # num_beams > 1 still goes to beam search, its num_return_sequences from the beam resolution
    m.generate(ids, images=img, max_new_tokens=4, num_beams=3, num_return_sequences=2)
    assert calls[-1]['num_beams'] == 3 and calls[-1]['num_return_sequences'] == 2 and 'do_sample' not in calls[-1]
    n = len(calls)
    with pytest.raises(NotImplementedError, match='use_hf_loop=True'):
        m.generate(ids, images=img, max_new_tokens=4, do_sample=True, num_return_sequences=2,
                   past_key_values=DynamicCache())
    assert len(calls) == n
