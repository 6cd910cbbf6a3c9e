"""Cost of per-request options in continuous batching (ContinuousBatcher(request_options=True)) on the 7B config (bf16,
the headline prompt: 706 tokens with 8 RoIs).  Measures:
  * the graphed batcher step at 8 and 16 slots with every slot running, in three setups -- plain (a batcher without
    the option), neutral (an opted-in batcher whose rows carry no option) and options (an opted-in batcher whose rows
    all sample at T 0.7 with repetition_penalty 1.2 and no_repeat_ngram_size 3) -- over histories of 706 ids (just
    admitted) and 1730 ids (each row's counters, lengths and history advanced by 1024 tokens); then the same with a
    per-request stop string that never matches;
  * the host time of the seam's stop table for a request: a new stop set (a pass over the vocabulary, a table build)
    and a repeated one (a lookup);
  * the traffic mix of tools/bench_serve.py (32 requests, answers of 16..256 tokens, all arriving at t = 0) with every
    request carrying those options and the stop string: model.generate per request against the batcher at 8 and 16
    slots, in generated tokens per second.
Every figure is the median of RUNS runs, the setups alternating within each run, with min and max.  CUDA events for the
step times; host clocks after a device synchronise for the rest.  Prints one JSON line per figure after a line with the
card's name, power limit and SM clocks, read in the same call.
usage: python tools/bench_serve_options.py"""
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import synthetic_inputs  # noqa: E402
from gpt4roi_b200.engine import ContinuousBatcher, EngineConfig, PrefillEngine, StopStrings, random_state_dicts  # noqa: E402
from tests.stop_tokenizer import seeded_tokenizer  # noqa: E402
from tools.bench_serve import DEV, MAX_NEW, MIN_NEW, N_REQ, card, timed  # noqa: E402

RUNS = 3
MAX_LEN = 2048
ADVANCE = 1024                          # 706 + 1024 = 1730 history ids
OPTIONS = dict(do_sample=True, temperature=0.7, repetition_penalty=1.2, no_repeat_ngram_size=3)
NEVER = 'x###y.###x###y'                # three given pieces in a row: random weights do not produce it


def spread(xs):
    return dict(median=statistics.median(xs), min=min(xs), max=max(xs), runs=len(xs))


def vocab(V):
    """The seeded vocabulary's clean strings (the seam's pass over a tokenizer), padded to the engine's V ids."""
    from gpt4roi_b200.spi_llava import _token_strings
    strings = _token_strings(seeded_tokenizer(32000, seed=5))
    return strings + [None] * (V - len(strings))


def step_setups(eng, req, slots):
    """{setup: batcher with every slot running}, built once; advance() moves every row 1024 tokens on."""
    ids, images, boxes = req
    out = {}
    for name, opt, kw in (('plain', False, {}), ('neutral', True, {}), ('options', True, OPTIONS)):
        b = ContinuousBatcher(eng, slots, MAX_LEN, request_options=opt)
        for _ in range(slots):
            b.submit(ids, images, boxes, max_new_tokens=MAX_NEW, **kw)
        b.step()
        out[name] = b
    return out


def set_stop(b, stops):
    """Give every row of an opted-in batcher the stop table `stops` (None: none), in place: the captured graph reads
    the tables through the row pointers, so the same graph times both."""
    table = None if stops is None else stops.on(DEV)
    b.row_stops = [table] * b.slots
    b.row_tables.fill_(0 if table is None else table.data_ptr())
    b.row_states.fill_(1 if table is None else stops.S)
    b.stop_state.zero_()


def advance(b, g):
    b.step_count += ADVANCE
    b.cache.lens += ADVANCE
    if b.request_options:
        L = int(b.prompt_len[0])
        b.history[:, L:L + ADVANCE] = torch.randint(0, 32000, (b.slots, ADVANCE), generator=g).to(DEV)


def traffic(eng, req, stops, lengths, way):
    ids, images, boxes = req
    t0 = time.perf_counter()
    if way == 'generate':
        for i, n in enumerate(lengths):
            eng.generate(ids, images, boxes, max_new_tokens=n, stop_strings=stops, **OPTIONS)
    else:
        b = ContinuousBatcher(eng, way, MAX_LEN, request_options=True)
        for n in lengths:
            b.submit(ids, images, boxes, max_new_tokens=n, stop_strings=stops, **OPTIONS)
        b.run()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    print(json.dumps(card()), flush=True)
    cfg = EngineConfig(image_size=336)
    sd, vit_sd = random_state_dicts(cfg, DEV, seed=0)
    eng = PrefillEngine(cfg, sd, vit_sd, DEV)
    del sd, vit_sd
    torch.cuda.empty_cache()
    ids, images, boxes = synthetic_inputs(cfg, 1, 8, 128)
    req = (ids.to(DEV), images.to(DEV, torch.bfloat16), boxes)
    L = ids.shape[1]
    strings = vocab(cfg.vocab)
    stops = StopStrings(strings, [NEVER])
    g = torch.Generator().manual_seed(0)

    # ---- the graphed step
    for slots in (8, 16):
        setups = step_setups(eng, req, slots)
        for hist in (L, L + ADVANCE):
            if hist > L:
                for b in setups.values():
                    advance(b, g)
            times = {}
            for _ in range(RUNS):
                for stop in (None, stops):
                    for k, b in setups.items():
                        if b.request_options:
                            set_stop(b, stop)
                        elif stop is not None:
                            continue
                        times.setdefault(k + ('_stop' if stop is not None else ''), []).append(
                            timed(b.graph.replay, 20))
            for k, t in times.items():
                print(json.dumps(dict(what='serve_options_step', slots=slots, setup=k, history=hist, prompt_len=L,
                                      step_ms=spread(t))), flush=True)
        del setups, b
        torch.cuda.empty_cache()

    # ---- the seam's stop table at submit
    from gpt4roi_b200.spi_llava import SeamBatcher
    tok = seeded_tokenizer(32000, seed=5)
    new, rep = [], []
    for i in range(RUNS):
        sb = SeamBatcher(None, ContinuousBatcher(eng, 1, 64, request_options=True), tokenizer=tok)
        t0 = time.perf_counter()
        sb._stop_table(tok, ('x###y.###', '#b%d' % i))
        new.append((time.perf_counter() - t0) * 1e3)
        t0 = time.perf_counter()
        sb._stop_table(tok, ('x###y.###', '#b%d' % i))
        rep.append((time.perf_counter() - t0) * 1e3)
    print(json.dumps(dict(what='serve_options_stop_table', new_set_ms=spread(new), repeated_set_ms=spread(rep))),
          flush=True)

    # ---- the traffic mix
    lengths = torch.randint(MIN_NEW, MAX_NEW + 1, (N_REQ,), generator=torch.Generator().manual_seed(0)).tolist()
    for way in ('generate', 8, 16):      # warm-up: every graph and shape the timed runs use
        traffic(eng, req, stops, [8, 8], way)
    ends = {w: [] for w in ('generate', 8, 16)}
    for _ in range(RUNS):
        for w in ends:
            ends[w].append(traffic(eng, req, stops, lengths, w))
            torch.cuda.empty_cache()
    for w, t in ends.items():
        print(json.dumps(dict(what='serve_options_7b_bf16', way='generate' if w == 'generate' else 'batcher%d' % w,
                              requests=N_REQ, prompt_len=L, new_tokens_max=sum(lengths),
                              tokens_per_s=spread([sum(lengths) / x for x in t]), makespan_s=spread(t))), flush=True)


if __name__ == '__main__':
    main()
