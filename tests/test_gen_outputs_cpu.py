"""CPU tests of generate()'s return_dict_in_generate outputs (scores, logits, beam indices): the seam's resolution of the
flags as transformers resolves them, its refusals and return types, and the decode loop's output slots on a CPU
stand-in of the engine (Sampler._host fills the same slots the selection kernel fills on the device).
tests/test_gen_outputs_gpu.py checks the kernels and both loops on the H100."""
import pytest
import torch

from gpt4roi_b200.engine import StopStrings
from tests.test_model_seam_cpu import _tiny_model
from tests.test_ragged_host_cpu import V, _batch, _Stub

IMG = torch.zeros(3, 3, 4, 4)


def test_resolve_outputs_like_transformers():
    from transformers import GenerationConfig
    from gpt4roi_b200.spi_llava import resolve_generate
    m = _tiny_model()

    def outputs(**kw):
        return resolve_generate(m, 3, None, **kw).outputs
    off = dict(return_dict_in_generate=False, output_scores=False, output_logits=False)
    assert outputs() == off
    assert outputs(output_scores=True) == off                   # HF: scores only with return_dict_in_generate
    assert outputs(return_dict_in_generate=True) == dict(off, return_dict_in_generate=True)
    assert outputs(return_dict_in_generate=True, output_scores=True, output_logits=True) == \
        dict(return_dict_in_generate=True, output_scores=True, output_logits=True)
    gc = GenerationConfig(return_dict_in_generate=True, output_logits=True)
    assert outputs(generation_config=gc) == dict(off, return_dict_in_generate=True, output_logits=True)
    assert outputs(generation_config=gc, return_dict_in_generate=False) == off      # the kwarg first
    m.generation_config.return_dict_in_generate, m.generation_config.output_scores = True, True   # then the model's
    assert outputs() == dict(off, return_dict_in_generate=True, output_scores=True)
    assert not resolve_generate(m, 3, None).layer_outputs
    m._get_engine = lambda device: pytest.fail('no engine should be built')
    for bad in (dict(output_attentions=True), dict(output_hidden_states=True)):
        assert resolve_generate(m, 3, None, return_dict_in_generate=True, **bad).layer_outputs
        with pytest.raises(NotImplementedError, match='not materialised'):
            m.generate(torch.tensor([[1, 5, 9]]), images=IMG[:1], max_new_tokens=4, return_dict_in_generate=True, **bad)


def test_beam_search_outputs_resolve_at_generate_only():
    """generate() gets the same search whether the output flags come as kwargs, in generation_config= or in the
    model's config."""
    from transformers import GenerationConfig
    from gpt4roi_b200.spi_llava import resolve_generate
    m = _tiny_model().eval()
    m.generation_config.eos_token_id = 2
    base = resolve_generate(m, 3, 4, num_beams=2).beam
    calls = []

    class _Engine:
        def generate(self, input_ids, images, bboxes, **kw):
            calls.append(kw)
            return dict(sequences=input_ids, scores=None, logits=None, sequences_scores=torch.zeros(1),
                        beam_indices=torch.zeros(1, 1, dtype=torch.int32))
    m._get_engine = lambda device: _Engine()
    ids = torch.tensor([[1, 5, 9]])
    img = torch.zeros(1, 3, 28, 28)
    search = dict(num_beams=2, length_penalty=base['length_penalty'], early_stopping=base['early_stopping'],
                  num_return_sequences=1, eos_token_id=base['eos_token_id'], pad_token_id=base['pad_token_id'])
    for kw in (dict(num_beams=2, return_dict_in_generate=True, output_scores=True),
               dict(generation_config=GenerationConfig(num_beams=2, return_dict_in_generate=True, output_scores=True))):
        m.generate(ids, images=img, max_new_tokens=4, **kw)
        assert {k: calls[-1][k] for k in search} == search
        assert calls[-1]['return_dict_in_generate'] and calls[-1]['output_scores'] and not calls[-1]['output_logits']
    m.generation_config.return_dict_in_generate, m.generation_config.output_logits = True, True
    m.generate(ids, images=img, max_new_tokens=4, num_beams=2)
    assert calls[-1]['return_dict_in_generate'] and calls[-1]['output_logits'] and calls[-1]['num_beams'] == 2


def test_seam_returns_transformers_output_classes():
    from transformers import DynamicCache
    from transformers.generation.utils import GenerateBeamDecoderOnlyOutput, GenerateDecoderOnlyOutput
    m = _tiny_model().eval()
    calls = []

    class _Engine:
        cfg, dev = _Stub().cfg, torch.device('cpu')     # the seam builds a KVCache for past_key_values

        def generate(self, input_ids, images, bboxes, **kw):
            calls.append(kw)
            if not kw.get('return_dict_in_generate'):
                return input_ids
            sc = (torch.zeros(1, 140),) if kw['output_scores'] else None
            lg = (torch.ones(1, 140),) if kw['output_logits'] else None
            res = dict(sequences=input_ids, scores=sc, logits=lg)
            if kw.get('num_beams', 1) > 1:
                res.update(sequences_scores=torch.zeros(1), beam_indices=torch.zeros(1, 1, dtype=torch.int32))
            return res
    m._get_engine = lambda device: _Engine()
    ids = torch.tensor([[1, 5, 9]])
    img = torch.zeros(1, 3, 28, 28)
    out = m.generate(ids, images=img, max_new_tokens=4, output_scores=True)
    assert torch.is_tensor(out) and calls[-1]['output_scores'] is False       # no return_dict_in_generate: the ids
    out = m.generate(ids, images=img, max_new_tokens=4, return_dict_in_generate=True, output_scores=True)
    assert type(out) is GenerateDecoderOnlyOutput and out.scores[0].shape == (1, 140) and out.logits is None
    assert out.past_key_values is None and torch.equal(out.sequences, ids)
    pkv = DynamicCache()
    out = m.generate(ids, images=img, max_new_tokens=4, return_dict_in_generate=True, output_logits=True,
                     past_key_values=pkv)
    assert out.scores is None and out.logits[0].shape == (1, 140) and out.past_key_values is pkv
    out = m.generate(ids, images=img, max_new_tokens=4, num_beams=2, return_dict_in_generate=True)
    assert type(out) is GenerateBeamDecoderOnlyOutput and calls[-1]['num_beams'] == 2
    assert out.sequences_scores is None and out.beam_indices is not None and out.past_key_values is None
    out = m.generate(ids, images=img, max_new_tokens=4, num_beams=2, return_dict_in_generate=True, output_scores=True)
    assert out.sequences_scores is not None and out.scores is not None
    n = len(calls)
    for bad in (dict(output_attentions=True), dict(output_hidden_states=True)):
        with pytest.raises(NotImplementedError, match='not materialised'):
            m.generate(ids, images=img, max_new_tokens=4, return_dict_in_generate=True, **bad)
    assert len(calls) == n


def _check_slots(res, L, live_until=None):
    """One score and logit entry per new token, each a contiguous fp32 [R, V]; scores[s].argmax() is token s of every
    row still live at step s."""
    seq, scores, logits = res['sequences'], res['scores'], res['logits']
    n = seq.shape[1] - L
    assert len(scores) == len(logits) == n
    for s in range(n):
        for t in (scores[s], logits[s]):
            assert t.dtype == torch.float32 and t.shape == (seq.shape[0], V) and t.is_contiguous()
        live = torch.ones(seq.shape[0], dtype=torch.bool) if live_until is None else live_until > s
        assert torch.equal(scores[s].argmax(-1)[live], seq[live, L + s])


def test_stand_in_loop_fills_one_slot_per_token():
    ids_r, mask_r, _, _ = _batch()
    eng = _Stub()
    plain = eng.generate(ids_r, IMG, None, max_new_tokens=3, attention_mask=mask_r)
    res = eng.generate(ids_r, IMG, None, max_new_tokens=3, attention_mask=mask_r, output_scores=True,
                       output_logits=True)
    assert torch.equal(res['sequences'], plain)
    _check_slots(res, 4)
    for s in range(3):   # greedy with no processor: the scores are the widened logits
        assert torch.equal(res['scores'][s], res['logits'][s])
    assert eng.generate(ids_r, IMG, None, max_new_tokens=3, attention_mask=mask_r, output_logits=True)['scores'] is None
    only = eng.generate(ids_r, IMG, None, max_new_tokens=3, attention_mask=mask_r, return_dict_in_generate=True)
    assert only['scores'] is None and only['logits'] is None and torch.equal(only['sequences'], plain)


def test_stand_in_loop_stops_early_on_eos_with_pads():
    ids_r, mask_r, _, _ = _batch()
    eng = _Stub()
    # row 1 emits 9 at step 0 (then pads), row 0 at step 2, row 2 never: 5 tokens, 5 slots
    res = eng.generate(ids_r, IMG, None, max_new_tokens=5, attention_mask=mask_r, eos_token_id=9, pad_token_id=0,
                       output_scores=True, output_logits=True)
    assert res['sequences'][:, 4:].tolist() == [[7, 8, 9, 0, 0], [9, 0, 0, 0, 0], [10, 11, 12, 13, 14]]
    _check_slots(res, 4, live_until=torch.tensor([3, 1, 5]))
    assert res['scores'][1][1].argmax() == 10      # a finished row still gets its scores, as in HF
    # every row finished early: fewer slots than max_new_tokens
    res = eng.generate(ids_r[1:], IMG[1:], None, max_new_tokens=6, attention_mask=mask_r[1:], eos_token_id=11,
                       pad_token_id=0, output_scores=True, output_logits=True)
    assert res['sequences'][:, 4:].tolist() == [[9, 10, 11], [10, 11, 0]]
    _check_slots(res, 4, live_until=torch.tensor([3, 2]))


def test_stand_in_loop_with_stop_strings_and_processors():
    ids_r, mask_r, _, _ = _batch()
    eng = _Stub()
    stops = StopStrings([chr(65 + i) for i in range(V)], ['HI'])          # tokens 7 then 8
    res = eng.generate(ids_r, IMG, None, max_new_tokens=6, attention_mask=mask_r, stop_strings=stops,
                       eos_token_id=49, pad_token_id=0, output_scores=True, output_logits=True)
    assert res['sequences'][:, 4:].tolist() == [[7, 8, 0, 0, 0, 0], [9, 10, 11, 12, 13, 14], [10, 11, 12, 13, 14, 15]]
    _check_slots(res, 4, live_until=torch.tensor([2, 6, 6]))
    res = eng.generate(ids_r[:1], IMG[:1], None, max_new_tokens=6, stop_strings=stops, eos_token_id=49, pad_token_id=0,
                       output_scores=True, output_logits=True)
    assert res['sequences'][:, 4:].tolist() == [[7, 8]] and len(res['scores']) == len(res['logits']) == 2
    res = eng.generate(ids_r, IMG, None, max_new_tokens=6, attention_mask=mask_r, stop_strings=stops,
                       output_scores=True, output_logits=True)
    _check_slots(res, 4)
    # a processor changes the scores, not the raw logits: row 0's arg-max 7 is banned by min_new_tokens (eos 7)
    res = eng.generate(ids_r[:1], IMG[:1], None, max_new_tokens=3, eos_token_id=7, min_new_tokens=2,
                       repetition_penalty=2.0, output_scores=True, output_logits=True)
    assert res['scores'][0][0, 7] == float('-inf') and res['logits'][0][0, 7] == 1.0
    assert res['scores'][0][0, 3] == 0.0 and res['scores'][0][0, 0] == 0.0
    _check_slots(res, 4)
