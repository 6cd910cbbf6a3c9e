"""Cost of the history-dependent logits processors in the decode loop (csrc/sample.cu: g4r_sample_tokens_proc_*,
engine.LogitsProcessors).  7B random weights in fp16 (the demo's dtype) and bf16, the headline prompt (706 tokens,
8 RoIs), batch 1 and 8, sampling at T = 0.7, top_k = 50, repetition_penalty = 1.2 and no_repeat_ngram_size = 3, one
process, the variants alternating, medians of --reps.  Prints one JSON line per measurement after a line with the card's
name, power limit and SM clocks:
  * the graphed decode step with the sampler alone and with the processed sampler (CUDA events over 200 replays), at
    histories of L = 706 and 706 + 1024 ids (the processed sampler reads L + step ids; the KV cache is the same);
  * eng.generate wall time per new token (host clock around a call that ends in a synchronise), 256 new tokens, fp16;
  * where the added time goes: the selection kernel alone (CUDA events over 500 launches on the step's logits), plain
    vs processed with only the n-gram ban, only the penalty, both, and greedy with both.
The history beyond the prompt is filled with ids drawn from the vocabulary, as a long answer would add fresh ids: the
penalised list (and its sort) grows with it.
usage: python tools/bench_penalties.py [--out FILE] [--reps N]"""
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
from gpt4roi_b200 import kernels  # noqa: E402
from gpt4roi_b200.engine import (EngineConfig, GraphedDecode, KVCache, LogitsProcessors, PrefillEngine,  # noqa: E402
                                 Sampler, random_state_dicts)

DEV = 'cuda:0'
REPLAYS = 200
PROC = dict(repetition_penalty=1.2, no_repeat_ngram_size=3)
SAMPLE = dict(greedy=False, temperature=0.7, top_k=50, seed=1)


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


def history(ids, n):
    """The prompt, then n ids drawn from the vocabulary (seeded)."""
    g = torch.Generator().manual_seed(11)
    fresh = torch.randint(0, 32000, (ids.shape[0], n), generator=g).to(ids.device)
    return torch.cat([ids, fresh], 1).contiguous()


def kernel_us(logits, hist, L, step, greedy, launches=500, **proc):
    """The selection kernel alone on fixed logits: mean µs per launch, CUDA events around `launches` launches."""
    B = logits.shape[0]
    out = torch.empty((B, 1), dtype=torch.int64, device=DEV)
    rng = torch.tensor([step], dtype=torch.int64, device=DEV)
    s = dict(SAMPLE, greedy=greedy)

    def once():
        if proc:
            kernels.sample_tokens_processed(logits, out, s['greedy'], s['temperature'], s['top_k'], 1.0, s['seed'], rng,
                                            history=hist, L=L, append=False, **proc)
        else:
            kernels.sample_tokens(logits, out, s['greedy'], s['temperature'], s['top_k'], 1.0, s['seed'], rng)
    for _ in range(20):
        once()
    e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    torch.cuda.synchronize()
    e[0].record()
    for _ in range(launches):
        once()
    e[1].record()
    torch.cuda.synchronize()
    return 1e3 * e[0].elapsed_time(e[1]) / launches


def step_ms(eng, cfg, ids, images, boxes, processed, extra):
    """One prefill, one capture, then REPLAYS replays of the graphed step between two CUDA events.  extra: history ids
    beyond the prompt when the timing starts (the Philox counter starts there; the history holds the prompt, then
    ids drawn from the vocabulary)."""
    B, L = ids.shape
    cache = KVCache(cfg, B, L + REPLAYS + 32, DEV)
    logits = eng.forward_device(ids, images, eng.plan_boxes(boxes), last_only=True, cache=cache)
    hist = history(ids, extra + REPLAYS + 32)
    procs = LogitsProcessors(hist, L, **PROC) if processed else None
    smp = Sampler(B, DEV, processors=procs, **SAMPLE)
    smp.rng_step.fill_(extra)
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
    return e[0].elapsed_time(e[1]) / REPLAYS


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='also append the JSON lines to this file')
    ap.add_argument('--reps', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_penalties: no CUDA device found; this measurement runs on the GPU only (there is no CPU path)')
    out = open(args.out, 'a') if args.out else None
    emit(out, card())
    for dtype in ('fp16', 'bf16'):
        cfg = EngineConfig(image_size=336, dtype=dtype)
        sd, vit_sd = random_state_dicts(cfg, DEV, seed=0, dtype=cfg.torch_dtype)
        eng = PrefillEngine(cfg, sd, vit_sd, DEV)
        del sd, vit_sd
        torch.cuda.empty_cache()
        for B in (1, 8):
            ids, images, boxes = synthetic_inputs(cfg, B, 8, 128)
            ids, images = ids.to(DEV), images.to(DEV, cfg.torch_dtype)
            L = ids.shape[1]
            for extra in (0, 1024):
                res = {False: [], True: []}
                for rep in range(args.reps):
                    for processed in (False, True):
                        res[processed].append(step_ms(eng, cfg, ids, images, boxes, processed, extra))
                a, b = statistics.median(res[False]), statistics.median(res[True])
                emit(out, dict(what='graphed_decode_step_7b_' + dtype, batch=B, prompt_len=L, history_len=L + extra,
                               replays=REPLAYS, sampling=SAMPLE, processors=PROC, ms_sampler=res[False],
                               ms_processed_sampler=res[True], median_sampler=a, median_processed=b,
                               added_us=1e3 * (b - a), added_pct=100 * (b - a) / a))
                # the kernel alone, on this prompt's prefill logits
                logits = eng.forward_device(ids, images, eng.plan_boxes(boxes), last_only=True)[:, 0]
                hist = history(ids, extra + 8)
                distinct = [len(set(r[:L + extra].tolist())) for r in hist]
                variants = dict(plain={}, ngram_only=dict(no_repeat_ngram_size=3),
                                penalty_only=dict(repetition_penalty=1.2), both=PROC)
                t = {k: [] for k in variants}
                t['greedy_plain'], t['greedy_both'] = [], []
                for rep in range(args.reps):
                    for name, proc in variants.items():
                        t[name].append(kernel_us(logits, hist, L, extra, False, **proc))
                    t['greedy_plain'].append(kernel_us(logits, hist, L, extra, True))
                    t['greedy_both'].append(kernel_us(logits, hist, L, extra, True, **PROC))
                emit(out, dict(what='selection_kernel_us_' + dtype, batch=B, history_len=L + extra,
                               distinct_history_ids_per_row=distinct, sampling=SAMPLE,
                               median={k: statistics.median(v) for k, v in t.items()}, all=t))
            if dtype != 'fp16':
                continue
            kw = dict(do_sample=True, temperature=0.7, top_k=50)
            eng.generate(ids, images, boxes, max_new_tokens=8, **kw)      # warm every shape of the call
            eng.generate(ids, images, boxes, max_new_tokens=8, **kw, **PROC)
            n = 256
            t = {'sampler': [], 'processed': []}
            for rep in range(args.reps):
                for name in t:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    got = eng.generate(ids, images, boxes, max_new_tokens=n, **kw, **(PROC if name == 'processed' else {}))
                    torch.cuda.synchronize()
                    t[name].append((time.perf_counter() - t0) * 1e3 / n)
                    assert got.shape[1] == L + n
            emit(out, dict(what='generate_wall_ms_per_new_token_7b_fp16', batch=B, prompt_len=L, new_tokens=n,
                           includes='prefill and graph capture, spread over the new tokens',
                           median={k: statistics.median(v) for k, v in t.items()}, all=t))
        del eng
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
