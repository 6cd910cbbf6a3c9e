"""CPU tests of transformers' history-dependent logits processors on the engine loop (repetition_penalty,
no_repeat_ngram_size, min_length, min_new_tokens): the torch restatement the CPU stand-in path uses against HF's own
processor classes, the loop on a CPU stand-in engine against a reference loop built from HF's classes, and the model
seam's resolution and refusals.  tests/test_logits_process_gpu.py runs the kernel and the real loops."""
import pytest
import torch

from gpt4roi_b200 import engine
from gpt4roi_b200.engine import LogitsProcessors
from tests.test_model_seam_cpu import _tiny_model
from tests.test_ragged_host_cpu import _batch

V = 50
IMAGES = torch.zeros(3, 3, 4, 4)


def hf_processors(L, repetition_penalty=1.0, no_repeat_ngram_size=0, min_length=0, min_new_tokens=0, eos=()):
    """transformers' own processors, in the order GenerationMixin._get_logits_processor builds them."""
    from transformers.generation import logits_process as lp
    procs = lp.LogitsProcessorList()
    if repetition_penalty != 1.0:
        procs.append(lp.RepetitionPenaltyLogitsProcessor(repetition_penalty))
    if no_repeat_ngram_size > 0:
        procs.append(lp.NoRepeatNGramLogitsProcessor(no_repeat_ngram_size))
    if min_length > 0 and len(eos):
        procs.append(lp.MinLengthLogitsProcessor(min_length, list(eos)))
    if min_new_tokens > 0 and len(eos):
        procs.append(lp.MinNewTokensLengthLogitsProcessor(L, min_new_tokens, list(eos)))
    return procs


def _histories(R, n, seed, pad=0):
    """R rows of n ids with heavy repetition (a short random motif repeated, some ids random), pads on the left."""
    g = torch.Generator().manual_seed(seed)
    motif = torch.randint(1, 12, (R, 5), generator=g)
    h = motif.repeat(1, n // 5 + 1)[:, :n].clone()
    noise = torch.rand(R, n, generator=g) < 0.2
    h[noise] = torch.randint(1, V, (int(noise.sum()),), generator=g)
    for r in range(R):
        h[r, :int(torch.randint(0, 4, (1,), generator=g))] = pad
    return h


@pytest.mark.parametrize('n', [1, 2, 3])
@pytest.mark.parametrize('penalty', [0.7, 1.0, 1.3])
def test_restatement_equals_transformers(n, penalty):
    """LogitsProcessors.apply == HF's processor list, bitwise (-inf included), at every step of a history that grows
    across the prompt boundary, for min_length / min_new_tokens that end before, at and after it."""
    L, steps, R = 9, 8, 4
    hist = torch.zeros((R, L + steps), dtype=torch.int64)
    hist[:, :L + steps] = _histories(R, L + steps, seed=n)
    g = torch.Generator().manual_seed(7)
    for min_length, min_new in ((0, 0), (L + 3, 0), (0, 4), (L - 2, 2)):
        pr = LogitsProcessors(hist, L, penalty, n, min_length, min_new, eos_ids=[2, 7])
        hf = hf_processors(L, penalty, n, min_length, min_new, eos=[2, 7])
        for s in range(steps):
            x = (torch.randn(R, V, generator=g) * 3).to(torch.bfloat16).float()
            want = hf(hist[:, :L + s], x.clone())
            got = pr.apply(x.clone(), s)
            assert torch.equal(got, want), (n, penalty, min_length, min_new, s)


class _Stub:
    """Stand-in engine whose next-token logits depend on the row's last token through a fixed random table (heavy
    repetition without processors); forward_device answers the prompt's last valid token."""
    dev = torch.device('cpu')
    dt = torch.bfloat16

    def __init__(self, seed=0):
        self.cfg = engine.EngineConfig(hidden=64, n_heads=1, n_layers=1, mlp=128, vocab=V)   # head_dim 64: no graph
        g = torch.Generator().manual_seed(seed)
        self.table = (torch.randn(V, V, generator=g) * 2).to(torch.bfloat16)
        self.table[:, 3] = self.table.max() + 1       # id 3 is every row's favourite

    def plan_boxes(self, bboxes):
        return None

    def forward_device(self, ids, images, plan, validate=True, last_only=False, seqlens=None, cache=None, **kw):
        B, L = ids.shape
        if cache is not None:
            cache.start(L, seqlens)
        lens = torch.full((B,), L) if seqlens is None else seqlens.long()
        return self.table[ids[torch.arange(B), lens - 1]][:, None]

    def decode_step(self, ids, cache, pos_dev=None):
        cache.length += 1
        if cache.lens is not None:
            cache.lens.add_(1)
        return self.table[ids[:, 0]][:, None]

    generate = engine.PrefillEngine.generate


def _reference(stub, ids, max_new, shift=1, eos=None, pad=None, **proc):
    """The loop with HF's processor classes: history = the prompt as given, then the new tokens (pads included);
    row r's scores rolled by r % shift (the stand-in draw of N > 1)."""
    R, L = ids.shape
    hf = hf_processors(L, eos=[] if eos is None else [eos], **proc)
    h = ids.clone()
    done = torch.zeros(R, dtype=torch.bool)
    for s in range(max_new):
        x = stub.table[h[:, -1]].float()           # s = 0: the prompt's last token
        x = torch.stack([torch.roll(x[r], r % shift) for r in range(R)])
        tok = hf(h, x).argmax(-1)
        if eos is not None and pad is not None:
            tok = torch.where(done, torch.full_like(tok, pad), tok)
            done |= tok == eos
        h = torch.cat([h, tok[:, None]], 1)
        if eos is not None and pad is not None and bool(done.all()):
            break
    return h


PROC = dict(repetition_penalty=1.3, no_repeat_ngram_size=3, min_new_tokens=4)


def test_stand_in_loop_equals_the_transformers_loop():
    stub = _Stub()
    ids = torch.tensor([[5, 3, 9, 3, 4, 3]])
    plain = stub.generate(ids, IMAGES[:1], None, max_new_tokens=12)
    assert (plain[0, 6:] == 3).sum() > 6                          # without processors: the favourite, over and over
    for proc in (PROC, dict(repetition_penalty=0.8), dict(no_repeat_ngram_size=1), dict(no_repeat_ngram_size=2),
                 dict(min_length=10, repetition_penalty=1.5)):
        got = stub.generate(ids, IMAGES[:1], None, max_new_tokens=12, eos_token_id=3, **proc)
        want = _reference(stub, ids, 12, eos=3, **proc)
        assert torch.equal(got, want[:, :got.shape[1]]), proc
    # eos -> pad: the pads of a finished row are part of its history
    got = stub.generate(ids, IMAGES[:1], None, max_new_tokens=10, eos_token_id=3, pad_token_id=0, **PROC)
    assert torch.equal(got, _reference(stub, ids, 10, eos=3, pad=0, **PROC))


def test_stand_in_loop_left_padded_batch_keeps_the_pads_in_the_history():
    stub = _Stub(seed=1)
    _, _, ids_l, mask_l = _batch()          # pads (0) on the left of rows 1 and 2
    for proc in (PROC, dict(no_repeat_ngram_size=1, repetition_penalty=0.9)):
        got = stub.generate(ids_l, IMAGES, None, max_new_tokens=9, attention_mask=mask_l, eos_token_id=4,
                            pad_token_id=0, **proc)
        assert torch.equal(got, _reference(stub, ids_l, 9, eos=4, pad=0, **proc)), proc


class _RowSampler(engine.Sampler):
    """The stand-in draw of N > 1 (tests/test_multisample_cpu.py): row r's logits rolled by r % N, then the greedy
    host path, processors included."""
    N = 1

    def _host(self, logits, out, update):
        x = logits.reshape(logits.shape[0], -1)
        x = torch.stack([torch.roll(x[r], r % self.N) for r in range(x.shape[0])])
        self.greedy = True
        return super()._host(x[:, None], out, update)


def test_stand_in_loop_several_rows_per_prompt(monkeypatch):
    monkeypatch.setattr(_RowSampler, 'N', 3)
    monkeypatch.setattr(engine, 'Sampler', _RowSampler)
    stub = _Stub(seed=2)
    ids = torch.tensor([[5, 3, 9, 3], [7, 7, 3, 1]])
    got = stub.generate(ids, IMAGES[:2], None, max_new_tokens=8, do_sample=True, num_return_sequences=3, **PROC)
    assert got.shape == (6, 12)
    want = _reference(stub, ids.repeat_interleave(3, 0), 8, shift=3, **PROC)
    assert torch.equal(got, want)


def test_first_draw_reads_the_prompt_alone_and_warm_up_leaves_the_history(monkeypatch):
    seen = []
    apply = LogitsProcessors.apply

    def spy(self, scores, step):
        seen.append((step, self.L + step))
        return apply(self, scores, step)
    monkeypatch.setattr(LogitsProcessors, 'apply', spy)
    stub = _Stub()
    ids = torch.tensor([[5, 3, 9, 3, 4]])
    stub.generate(ids, IMAGES[:1], None, max_new_tokens=4, repetition_penalty=1.2)
    assert seen == [(0, 5), (1, 6), (2, 7), (3, 8)]
    # update=False selects but neither appends to the history nor advances `finished`
    h = torch.tensor([[5, 3, 9, 0, 0]])
    smp = engine.Sampler(1, 'cpu', eos_id=3, pad_id=0, processors=LogitsProcessors(h, 3, 1.2))
    out = torch.empty((1, 1), dtype=torch.int64)
    smp(stub.table[3][None, None], out, update=False)
    assert h.tolist() == [[5, 3, 9, 0, 0]] and int(smp.finished[0]) == 0
    smp(stub.table[3][None, None], out)
    assert h[0, 3] == out[0, 0] and h[0, 4] == 0


def test_neutral_parameters_build_no_processors(monkeypatch):
    made = []
    monkeypatch.setattr(engine, 'LogitsProcessors', type('P', (LogitsProcessors,), {
        '__init__': lambda self, *a, **k: made.append(a) or LogitsProcessors.__init__(self, *a, **k)}))
    stub = _Stub()
    ids = torch.tensor([[5, 3, 9]])
    stub.generate(ids, IMAGES[:1], None, max_new_tokens=3, repetition_penalty=1.0, no_repeat_ngram_size=0,
                  min_length=5, min_new_tokens=2)        # no eos id: HF builds no min-length processor either
    assert made == []
    stub.generate(ids, IMAGES[:1], None, max_new_tokens=3, min_new_tokens=2, eos_token_id=3)
    assert len(made) == 1


def test_engine_refusals():
    eng = engine.PrefillEngine.__new__(engine.PrefillEngine)
    ids = torch.tensor([[1, 5, 9]])
    for kw in (dict(repetition_penalty=1.2), dict(no_repeat_ngram_size=2), dict(min_new_tokens=2, eos_token_id=2)):
        with pytest.raises(NotImplementedError, match='use_hf_loop=True'):
            eng.generate(ids, None, None, num_beams=2, **kw)
    with pytest.raises(NotImplementedError, match='use_hf_loop=True'):
        eng.generate(ids, None, None, max_new_tokens=8190, do_sample=True, repetition_penalty=1.1)


def _hf_history_processors(m, L, **kw):
    """The history-dependent processors transformers' generate builds for an input of L tokens: the generation config
    after GenerationMixin._prepare_generated_length (which lets min_new_tokens override min_length), then
    _get_logits_processor.  A MinLengthLogitsProcessor whose min_length is at most L never suppresses anything and
    counts as absent."""
    from transformers.generation import logits_process as lp
    from gpt4roi_b200.spi_llava import _generation_config
    gc = _generation_config(m, {k: v for k, v in kw.items() if v is not None})
    gc = m._prepare_generated_length(gc, has_default_max_length=True, has_default_min_length='min_length' not in kw,
                                     model_input_name='input_ids', input_ids_length=L, inputs_tensor=None)
    procs = m._get_logits_processor(gc, input_ids_seq_length=L, device='cpu', model_kwargs={})
    got = dict(repetition_penalty=1.0, no_repeat_ngram_size=0, min_length=0, min_new_tokens=0, eos_ids=[])
    for p in procs:
        if isinstance(p, lp.RepetitionPenaltyLogitsProcessor):
            got['repetition_penalty'] = p.penalty
        elif isinstance(p, lp.NoRepeatNGramLogitsProcessor):
            got['no_repeat_ngram_size'] = p.ngram_size
        elif isinstance(p, lp.MinLengthLogitsProcessor) and p.min_length > L:
            got['min_length'], got['eos_ids'] = p.min_length, p.eos_token_id.tolist()
        elif isinstance(p, lp.MinNewTokensLengthLogitsProcessor):
            got['min_new_tokens'], got['eos_ids'] = p.min_new_tokens, p.eos_token_id.tolist()
    return got


def test_seam_resolves_the_processors_like_transformers():
    from transformers import GenerationConfig
    from gpt4roi_b200.spi_llava import resolve_generate
    m = _tiny_model()

    def resolved(**kw):
        return resolve_generate(m, 7, None, **kw)
    eos_model = m.generation_config.eos_token_id
    assert eos_model is not None
    cases = [dict(), dict(repetition_penalty=1.3), dict(no_repeat_ngram_size=3, min_new_tokens=8),
             dict(min_length=20), dict(min_length=20, eos_token_id=[5, 6]), dict(repetition_penalty=0.9, do_sample=True),
             dict(generation_config=GenerationConfig(repetition_penalty=1.1, no_repeat_ngram_size=2, min_length=4)),
             dict(generation_config=GenerationConfig(repetition_penalty=1.1), repetition_penalty=1.4)]
    for kw in cases:
        got = resolved(**kw).processors
        assert got == _hf_history_processors(m, 7, **kw), kw
    # min_new_tokens takes precedence over min_length, as in HF's generate: min_length = min_new_tokens + L
    both = resolved(min_length=30, min_new_tokens=3).processors
    assert both['min_length'] == 10 and both['min_new_tokens'] == 3
    assert both == _hf_history_processors(m, 7, min_length=30, min_new_tokens=3)
    # min_new_tokens=0 (HF: min_length = L) and min_length <= L suppress nothing: neutral, no processed kernel
    for kw in (dict(min_new_tokens=0), dict(min_length=7), dict(min_length=30, min_new_tokens=0)):
        got = resolved(**kw).processors
        assert got['min_length'] == 0 and got['min_new_tokens'] == 0 and got == _hf_history_processors(m, 7, **kw), kw
    # the eos list from the model's config when the caller gives none
    assert resolved(min_new_tokens=3).processors['eos_ids'] == [eos_model]
    assert resolved(min_new_tokens=3, eos_token_id=9).processors['eos_ids'] == [9]
    # then the model's generation config
    m.generation_config.repetition_penalty, m.generation_config.no_repeat_ngram_size = 1.2, 4
    got = resolved(do_sample=True, temperature=0.5)
    assert got[:4] == (True, 0.5, 50, 1.0) and got.processors['repetition_penalty'] == pytest.approx(1.2)
    assert got.processors['no_repeat_ngram_size'] == 4
    assert resolved(repetition_penalty=1.0).processors['repetition_penalty'] == 1.0


def test_seam_refusals():
    from transformers.generation.logits_process import LogitsProcessor, LogitsProcessorList
    from tests.test_serve_cpu import _seam, _StubEngine

    class Mine(LogitsProcessor):
        def __call__(self, input_ids, scores):
            return scores
    m = _seam(_StubEngine())
    sb = m.continuous_batcher(slots=1, max_len=16)
    m._get_engine = lambda device: pytest.fail('no engine should be built')
    ids = torch.tensor([[1, 2, 3, 4, 5]])
    for bad in (dict(min_p=0.1), dict(typical_p=0.5), dict(epsilon_cutoff=1e-3), dict(eta_cutoff=1e-3),
                dict(bad_words_ids=[[5]]), dict(suppress_tokens=[5]), dict(sequence_bias={(5,): 1.0}),
                dict(logits_processor=LogitsProcessorList([Mine()])), dict(num_beams=2)):
        with pytest.raises(NotImplementedError, match='use_hf_loop=True'):
            m.generate(ids, images=torch.zeros(1, 3, 28, 28), max_new_tokens=4, do_sample=True, temperature=0.7,
                       repetition_penalty=1.2, **bad)
    # the continuous batcher refuses the history-dependent ones too
    for bad in (dict(repetition_penalty=1.1), dict(no_repeat_ngram_size=3), dict(min_new_tokens=2)):
        with pytest.raises(NotImplementedError, match='use_hf_loop=True'):
            sb.submit(ids, max_new_tokens=2, do_sample=True, **bad)


def test_seam_routes_the_processors_to_the_engine_loop():
    m = _tiny_model().eval()
    calls = []

    class _Engine:
        def generate(self, input_ids, images, bboxes, **kw):
            calls.append(kw)
            return input_ids
    m._get_engine = lambda device: _Engine()
    ids = torch.tensor([[1, 5, 9]])
    img = torch.zeros(1, 3, 28, 28)
    m.generate(ids, images=img, max_new_tokens=4, repetition_penalty=1.3, no_repeat_ngram_size=3, min_new_tokens=8)
    kw = calls[-1]
    assert kw['repetition_penalty'] == pytest.approx(1.3) and kw['no_repeat_ngram_size'] == 3
    assert kw['min_new_tokens'] == 8 and kw['min_length'] == 3 + 8      # HF: min_length = min_new_tokens + L
    assert kw['length_eos_ids'] == [m.generation_config.eos_token_id] and kw['eos_token_id'] is None
    m.generate(ids, images=img, max_new_tokens=4, do_sample=True, temperature=0.7, repetition_penalty=1.1,
               eos_token_id=[7, 8], min_length=6)
    kw = calls[-1]
    assert kw['do_sample'] and kw['length_eos_ids'] == [7, 8] and kw['min_length'] == 6
    m.generate(ids, images=img, max_new_tokens=4, min_length=30, min_new_tokens=2)
    assert calls[-1]['min_length'] == 3 + 2 and calls[-1]['min_new_tokens'] == 2     # HF's min_new_tokens precedence
    m.generate(ids, images=img, max_new_tokens=4)
    assert calls[-1]['repetition_penalty'] == 1.0 and calls[-1]['length_eos_ids'] == []
    with pytest.raises(NotImplementedError, match='use_hf_loop=True'):
        m.generate(ids, images=img, max_new_tokens=4, num_beams=2, repetition_penalty=1.2)
