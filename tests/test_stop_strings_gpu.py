"""GPU tests of stop strings in generate(): the lookup kernel (csrc/stop.cu) against its torch restatement, and the
decode loop with stop strings -- engine loop against transformers' own loop through the model seam (single prompt,
left-padded batch, a stop string that begins in the prompt), eager against graphed step, sampling, and two turns on a
conversation cache.  The tokenizer is built in-process from a seeded vocabulary (tests/stop_tokenizer.py); stop strings
are cut out of the tokens a run without them produced, so that every match is certain."""
import pytest
import torch

from gpt4roi_b200 import kernels
from gpt4roi_b200.engine import EngineConfig, KVCache, StopStrings, random_state_dicts
from gpt4roi_b200.spi_llava import stop_strings_from_tokenizer
from tests.stop_tokenizer import seeded_tokenizer
from tests.test_engine_gpu import make_inputs
from tests.test_ragged_decode_gpu import ragged_inputs
from tests.test_stop_strings_cpu import clean_strings, walk

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
N_TOK = 32000          # the tokenizer's vocabulary; the model's has 32006 rows, so some ids have no string
PAD = 0


@pytest.mark.parametrize('B', [1, 8, 16, 64])
def test_stop_step_kernel_matches_torch_lookup(B):
    g = torch.Generator().manual_seed(B)
    V, S = 500, 37
    table = (torch.randint(0, S, (V + 1, S), generator=g) - 32768 * torch.randint(0, 2, (V + 1, S), generator=g)).to(torch.int16)
    table[V] = 0
    for rep in range(4):
        ids = torch.randint(0, V + 40, (B, 1), generator=g)          # some past the vocabulary
        if rep == 3:
            ids[0] = -1
        state = torch.randint(0, S, (B,), generator=g, dtype=torch.int32)
        finished = (torch.rand(B, generator=g) < 0.3).to(torch.int32)
        e = table[ids[:, 0].where((ids[:, 0] >= 0) & (ids[:, 0] < V), torch.tensor(V)), state.long()].long()
        live = finished == 0
        want_state = torch.where(live, (e & 0x7FFF).to(torch.int32), state)
        want_fin = finished | (live & (e < 0)).to(torch.int32)
        d_state, d_fin = state.to(DEV), finished.to(DEV)
        kernels.stop_step(ids.to(DEV), table.to(DEV), d_state, d_fin)
        assert torch.equal(d_state.cpu(), want_state) and torch.equal(d_fin.cpu(), want_fin)
    with pytest.raises(RuntimeError):
        kernels.stop_step(ids.to(DEV), table.to(DEV), d_state.long(), d_fin)
    with pytest.raises(RuntimeError):
        kernels.stop_step(ids.to(DEV), table.to(DEV).float(), d_state, d_fin)
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        kernels.stop_step(ids, table, state, finished)


@pytest.fixture(scope='module')
def seam():
    from tests.test_model_seam_gpu import build_seam_model
    cfg = EngineConfig(image_size=224, vit_layers=24, n_layers=2)
    sd, vit_sd = random_state_dicts(cfg, DEV, seed=47)
    model = build_seam_model(cfg, sd, vit_sd, dtype=torch.float16).eval()
    tok = seeded_tokenizer(N_TOK, seed=5)
    return cfg, model, tok, clean_strings(tok)


def straddling_stop(strings, new, first=1):
    """A stop string that begins inside new[i] and ends inside new[i + 1] (a character of overhang on either side), for
    the first i >= `first` whose two tokens have strings of two or more characters.  -> (stop string, i + 1)."""
    for i in range(first, len(new) - 1):
        a, b = (strings[t] if t < len(strings) else None for t in (int(new[i]), int(new[i + 1])))
        if a and b and len(a) >= 2 and len(b) >= 2:
            return a[1:] + b[:-1], i + 1
    raise AssertionError('no pair of neighbouring tokens with two or more characters each in %s' % new.tolist())


def expected(strings, stops, prompt, lens, new, pad):
    """What the loop must return for the new tokens `new` [B, n] of a run without stop strings: each row cut after the
    first token the CPU matcher (tests/test_stop_strings_cpu.py: equal to transformers') flags, filled with `pad`
    (None: left as generated), the width that of the last row to stop.  -> (tokens [B, n'], each row's stop step)."""
    hit = walk(StopStrings(strings, stops), torch.cat([prompt, new], 1), lens, new.shape[1])
    steps = [int(h.nonzero()[0]) if h.any() else None for h in hit]
    width = new.shape[1] if None in steps else max(steps) + 1
    want = new[:, :width].clone()
    if pad is not None:
        for b, s in enumerate(steps):
            if s is not None:
                want[b, s + 1:] = pad
    return want, steps


def unused_id(new):
    return next(t for t in range(5, 100) if not bool((new == t).any()))


def test_engine_loop_equals_hf_loop_single_prompt_and_prompt_straddle(seam):
    cfg, model, tok, strings = seam
    ids, images, boxes = make_inputs(cfg, 1, [2], 24, seed=9)
    L = ids.shape[1]
    img, bx = images.half().to(DEV), [b.half().to(DEV) for b in boxes]
    with torch.inference_mode():
        base = model.generate(ids.to(DEV), images=img, bboxes=bx, max_new_tokens=24)[:, L:].cpu()
        stop, at = straddling_stop(strings, base[0])
        eos = unused_id(base)
        want, steps = expected(strings, [stop], ids, torch.tensor([L]), base, PAD)
        assert steps == [at] and want.shape[1] == at + 1
        kw = dict(images=img, bboxes=bx, max_new_tokens=24, stop_strings=[stop], tokenizer=tok, pad_token_id=PAD,
                  eos_token_id=eos)
        ours = model.generate(ids.to(DEV), **kw)
        hf = model.generate(ids.to(DEV), use_hf_loop=True, **kw)
        assert torch.equal(ours[:, :L].cpu(), ids) and torch.equal(ours[:, L:].cpu(), want), (ours[:, L:], want)
        assert torch.equal(ours, hf), (ours[:, L:], hf[:, L:])
        # a stop string that begins with the prompt's last token and ends in the first new one: both stop at once
        stop0 = strings[int(ids[0, -1])] + strings[int(base[0, 0])][:1]
        kw['stop_strings'] = [stop0]
        ours = model.generate(ids.to(DEV), **kw)
        hf = model.generate(ids.to(DEV), use_hf_loop=True, **kw)
        assert ours.shape[1] == L + 1 and torch.equal(ours, hf) and int(ours[0, L]) == int(base[0, 0])
        # stop strings from the model's generation config, as transformers resolves them
        model.generation_config.stop_strings = [stop]
        try:
            cfg_run = model.generate(ids.to(DEV), images=img, bboxes=bx, max_new_tokens=24, tokenizer=tok, pad_token_id=PAD,
                                     eos_token_id=eos)
        finally:
            model.generation_config.stop_strings = None
        assert torch.equal(cfg_run[:, L:].cpu(), want)


def test_engine_loop_equals_hf_loop_left_padded_batch_rows_stop_at_different_steps(seam):
    cfg, model, tok, strings = seam
    B = 3
    ids, images, boxes, lens = ragged_inputs(cfg, B, 24, seed=81)
    L = ids.shape[1]
    shift = L - lens
    mask = (torch.arange(L)[None] < lens[:, None]).long()
    ids_l = torch.stack([torch.roll(ids[b], int(shift[b])) for b in range(B)])
    mask_l = torch.stack([torch.roll(mask[b], int(shift[b])) for b in range(B)])
    img, bx = images.half().to(DEV), [b.half().to(DEV) for b in boxes]
    with torch.inference_mode():
        kw = dict(images=img, bboxes=bx, attention_mask=mask_l.to(DEV), max_new_tokens=16)
        base = model.generate(ids_l.to(DEV), **kw)[:, L:].cpu()
        # row b's stop string begins with the row's own last prompt token, runs through its first b + 1 new tokens and
        # ends on the first character of the next: only that row can match it, whatever the other rows generate
        stops = [strings[int(ids[b, lens[b] - 1])] + ''.join(strings[int(t)] for t in base[b, :b + 1])
                 + strings[int(base[b, b + 1])][:1] for b in range(B)]
        eos = unused_id(base)
        want, steps = expected(strings, stops, ids, lens, base, PAD)
        assert steps == [1, 2, 3], (steps, stops)
        kw.update(stop_strings=stops, tokenizer=tok, pad_token_id=PAD, eos_token_id=eos)
        ours = model.generate(ids_l.to(DEV), **kw)
        hf = model.generate(ids_l.to(DEV), use_hf_loop=True, **kw)
    assert torch.equal(ours[:, :L].cpu(), ids_l) and torch.equal(ours[:, L:].cpu(), want), (ours[:, L:], want)
    assert torch.equal(ours, hf), (ours[:, L:], hf[:, L:])
    for b in range(B):
        assert bool((ours[b, L + steps[b] + 1:] == PAD).all())


def test_eager_step_equals_graphed_step_and_calls_do_not_leak_state(seam):
    cfg, model, tok, strings = seam
    eng = model._get_engine(torch.device(DEV))
    ids, images, boxes = make_inputs(cfg, 2, [1, 2], 24, seed=11)
    L = ids.shape[1]
    img = images.half().to(DEV)
    base = eng.generate(ids.to(DEV), img, boxes, max_new_tokens=16)[:, L:].cpu()
    s0, at0 = straddling_stop(strings, base[0], first=2)
    s1, at1 = straddling_stop(strings, base[1], first=6)
    eos = unused_id(base)
    lens = torch.full((2,), L)
    for stops in ([s0, s1], [s1], [s0, s1]):          # the second call's table differs from the first's
        table = stop_strings_from_tokenizer(tok, stops)
        want, _ = expected(strings, stops, ids, lens, base, PAD)
        outs = [eng.generate(ids.to(DEV), img, boxes, max_new_tokens=16, eos_token_id=eos, pad_token_id=PAD,
                             stop_strings=table, use_graph=graph)[:, L:].cpu() for graph in (False, True)]
        assert torch.equal(outs[0], outs[1]) and torch.equal(outs[1], want), (stops, outs, want)
    # no eos / pad in force: nothing is padded, the loop still ends when the last row has matched
    want, steps = expected(strings, [s0, s1], ids, lens, base, None)
    out = eng.generate(ids.to(DEV), img, boxes, max_new_tokens=16, stop_strings=stop_strings_from_tokenizer(tok, [s0, s1]))
    assert steps == [at0, at1] and torch.equal(out[:, L:].cpu(), want) and want.shape[1] == at1 + 1
    with pytest.raises(NotImplementedError, match='use_hf_loop=True'):
        eng.generate(ids.to(DEV), img, boxes, max_new_tokens=8, num_beams=2, stop_strings=table)


def test_sampled_run_with_stop_strings_is_a_prefix_of_the_same_seed_run(seam):
    """The extra kernel leaves the draws alone: with the same seed, the run with stop strings is the run without, row 0
    cut (and padded) where the CPU matcher says, row 1 -- which never matches -- token for token."""
    cfg, model, tok, strings = seam
    eng = model._get_engine(torch.device(DEV))
    ids, images, boxes = make_inputs(cfg, 2, [1, 2], 24, seed=13)
    L = ids.shape[1]
    img = images.half().to(DEV)
    kw = dict(max_new_tokens=20, do_sample=True, temperature=1.0, top_k=50)
    base = eng.generate(ids.to(DEV), img, boxes, generator=torch.Generator().manual_seed(7), **kw)[:, L:].cpu()
    again = eng.generate(ids.to(DEV), img, boxes, generator=torch.Generator().manual_seed(7), **kw)[:, L:].cpu()
    assert torch.equal(base, again)
    stop, at = straddling_stop(strings, base[0], first=4)
    want, steps = expected(strings, [stop], ids, torch.full((2,), L), base, PAD)
    assert steps == [at, None]
    out = eng.generate(ids.to(DEV), img, boxes, generator=torch.Generator().manual_seed(7), eos_token_id=unused_id(base),
                       pad_token_id=PAD, stop_strings=stop_strings_from_tokenizer(tok, [stop]), **kw)[:, L:].cpu()
    assert torch.equal(out, want), (out, want)
    assert torch.equal(out[1], base[1]) and bool((out[0, at + 1:] == PAD).all())


def test_two_turns_on_a_conversation_cache_with_stop_strings(seam):
    """generate(cache=, stop_strings=) twice: the stop string's first turn leaves the cache as reusable as a turn
    without stop strings does, and each turn stops where the CPU matcher (equal to transformers': test_stop_strings_cpu)
    says a run without stop strings on an equal cache would."""
    cfg, model, tok, strings = seam
    eng = model._get_engine(torch.device(DEV))
    ids1, images, boxes = make_inputs(cfg, 1, [2], 40, seed=17)
    L1 = ids1.shape[1]
    img = images.half().to(DEV)
    plain, stopped = KVCache(eng.cfg, 1, L1 + 96, DEV), KVCache(eng.cfg, 1, L1 + 96, DEV)
    base1 = eng.generate(ids1.to(DEV), img, boxes, max_new_tokens=12, cache=KVCache(eng.cfg, 1, L1 + 96, DEV))[:, L1:].cpu()
    stop1, at1 = straddling_stop(strings, base1[0])
    out1 = eng.generate(ids1.to(DEV), img, boxes, max_new_tokens=12, cache=stopped,
                        stop_strings=stop_strings_from_tokenizer(tok, [stop1])).cpu()
    assert torch.equal(out1[:, L1:], base1[:, :at1 + 1])
    ref1 = eng.generate(ids1.to(DEV), img, boxes, max_new_tokens=at1 + 1, cache=plain).cpu()
    assert torch.equal(ref1, out1)
    q = torch.randint(3, N_TOK, (1, 20), generator=torch.Generator().manual_seed(19))
    ids2 = torch.cat([out1, q], 1)
    L2 = ids2.shape[1]
    reuse = stopped.reusable(ids2, img, boxes).tolist()
    assert reuse == plain.reusable(ids2, img, boxes).tolist() and reuse[0] >= L1
    base2 = eng.generate(ids2.to(DEV), img, boxes, max_new_tokens=12, cache=plain)[:, L2:].cpu()
    stop2, at2 = straddling_stop(strings, base2[0])
    want, steps = expected(strings, [stop1, stop2], ids2, torch.tensor([L2]), base2, None)
    out2 = eng.generate(ids2.to(DEV), img, boxes, max_new_tokens=12, cache=stopped,
                        stop_strings=stop_strings_from_tokenizer(tok, [stop1, stop2])).cpu()
    assert steps[0] is not None and steps[0] <= at2
    assert torch.equal(out2[:, :L2], ids2) and torch.equal(out2[:, L2:], want), (out2[:, L2:], want)
