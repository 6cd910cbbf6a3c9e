"""Cost of stop strings in the decode loop (csrc/stop.cu, engine.StopStrings).  7B random weights in fp16 (the demo's
dtype), the headline prompt (706 tokens, 8 RoIs), a stop string that never matches, batch 1 and 8, one process, the
variants alternating, medians of 5.  Prints one JSON line per measurement after a line with the card's name, power limit
and SM clocks:
  * the graphed decode step with the sampler alone and with the sampler + stop_step (CUDA events over 200 replays);
  * eng.generate wall time per new token (host clock around a call that ends in a synchronise) at 256 and 1024 new
    tokens: no stop criterion, stop_strings=, and the reference's host callback (KeywordsStoppingCriteria, which decodes
    the whole continuation after every token).
The tokenizer is built in-process from a seeded vocabulary (tests/stop_tokenizer.py).
usage: python tools/bench_stop.py [--out FILE] [--reps N]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import synthetic_inputs  # noqa: E402
from gpt4roi_b200.engine import EngineConfig, GraphedDecode, KVCache, PrefillEngine, Sampler, random_state_dicts  # noqa: E402
from gpt4roi_b200.spi_llava import KeywordsStoppingCriteria, stop_strings_from_tokenizer  # noqa: E402
from tests.stop_tokenizer import seeded_tokenizer  # noqa: E402

DEV = 'cuda:0'
NEVER = '#.#y x.#.#y#.x#'      # two words, 15 characters: random tokens do not spell it
REPLAYS = 200


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return dict(device=torch.cuda.get_device_name(0), nvidia_smi=q[0] if q else None)


def emit(out, rec):
    line = json.dumps(rec)
    print(line, flush=True)
    if out is not None:
        out.write(line + '\n')
        out.flush()


def step_ms(eng, cfg, ids, images, boxes, stops):
    """One prefill, one capture, then REPLAYS replays of the graphed step between two CUDA events."""
    B, L = ids.shape
    cache = KVCache(cfg, B, L + REPLAYS + 32, DEV)
    logits = eng.forward_device(ids, images, eng.plan_boxes(boxes), last_only=True, cache=cache)
    state = None if stops is None else stops.initial_states(ids, torch.full((B,), L))
    smp = Sampler(B, DEV, greedy=True, stops=stops, stop_state=state)
    st = GraphedDecode(eng, cache, sampler=smp)
    smp(logits, st.ids)
    for _ in range(8):
        st.step()
    e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    torch.cuda.synchronize()
    e[0].record()
    for _ in range(REPLAYS):
        st.step()
    e[1].record()
    torch.cuda.synchronize()
    assert stops is None or not bool(smp.finished.any()), 'the stop string matched: the timed steps are not comparable'
    return e[0].elapsed_time(e[1]) / REPLAYS


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='also append the JSON lines to this file')
    ap.add_argument('--reps', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_stop: no CUDA device found; this measurement runs on the GPU only (there is no CPU path)')
    out = open(args.out, 'a') if args.out else None
    emit(out, card())
    tok = seeded_tokenizer(32000, seed=5)
    t0 = time.perf_counter()
    stops = stop_strings_from_tokenizer(tok, [NEVER])
    emit(out, dict(what='stop_table_build', stop_string=NEVER, states=stops.S, table_bytes=stops.table.numel() * 2,
                   host_ms_first=(time.perf_counter() - t0) * 1e3))
    t0 = time.perf_counter()
    stop_strings_from_tokenizer(tok, [NEVER])
    emit(out, dict(what='stop_table_cached', host_ms=(time.perf_counter() - t0) * 1e3))
    cfg = EngineConfig(image_size=336, dtype='fp16')
    sd, vit_sd = random_state_dicts(cfg, DEV, seed=0)
    eng = PrefillEngine(cfg, sd, vit_sd, DEV)
    del sd, vit_sd
    torch.cuda.empty_cache()
    for B in (1, 8):
        ids, images, boxes = synthetic_inputs(cfg, B, 8, 128)
        ids, images = ids.to(DEV), images.to(DEV, torch.float16)
        L = ids.shape[1]
        res = {False: [], True: []}
        for rep in range(args.reps):
            for with_stop in (False, True):
                res[with_stop].append(step_ms(eng, cfg, ids, images, boxes, stops if with_stop else None))
        a, b = statistics.median(res[False]), statistics.median(res[True])
        emit(out, dict(what='graphed_decode_step_7b_fp16', batch=B, prompt_len=L, replays=REPLAYS,
                       ms_sampler_only=res[False], ms_sampler_and_stop_step=res[True], median_sampler_only=a,
                       median_with_stop_step=b, added_pct=100 * (b - a) / a))
        variants = {
            'none': lambda: dict(),
            'stop_strings': lambda: dict(stop_strings=stops),
            'host_keywords_callback': lambda: dict(stopping_criteria=[KeywordsStoppingCriteria([NEVER], tok, ids)]),
        }
        eng.generate(ids, images, boxes, max_new_tokens=8)      # warm every shape of the call
        for n in (256, 1024):
            t = {k: [] for k in variants}
            for rep in range(args.reps):
                for name, kw in variants.items():
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    got = eng.generate(ids, images, boxes, max_new_tokens=n, **kw())
                    torch.cuda.synchronize()
                    dt = (time.perf_counter() - t0) * 1e3
                    assert got.shape[1] == L + n, 'the run stopped early (%d of %d tokens)' % (got.shape[1] - L, n)
                    t[name].append(dt / n)
            emit(out, dict(what='generate_wall_ms_per_new_token_7b_fp16', batch=B, prompt_len=L, new_tokens=n,
                           includes='prefill and graph capture, spread over the new tokens',
                           median={k: statistics.median(v) for k, v in t.items()}, all=t))


if __name__ == '__main__':
    main()
