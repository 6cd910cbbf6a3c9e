"""Cost of several sampled answers per prompt (generate(do_sample=True, num_return_sequences=N)) on the 7B config (bf16,
the headline prompt: 706 tokens with 8 RoIs), B in {1, 4}, N in {4, 8, 16}.  Prints one JSON line per (B, N), after a
line with the card's name, power limit and SM clocks:
  * step_ms: the graphed decode step over the B*N rows -- grouped: the prompts' K/V held once (SampleCache) and read
    once per step by the shared-prefix attention; expanded: the current loop on input_ids.repeat_interleave(N, 0), each
    row with its own copy of the prompt's K/V (the _rows attention, N x the prompt bytes).  Both at the first decode
    position, without the sampler (the same kernels on both sides);
  * ttft_ms: time to the first N tokens per prompt -- grouped: the prefill at batch B, the logits copy to B*N rows and
    the draw; expanded: the prefill of the B*N expanded rows and the draw;
  * floor_ms: the HBM byte floor of each step at the data sheet's 3.35 TB/s (the weights once, plus the K/V the
    attention must read: B prompts + B*N own rows grouped, B*N full rows expanded) -- a bound, not a measurement.
CUDA events (steps) / a host clock after a device synchronise (ttft); each figure the best of 2 runs.
usage: python tools/bench_multisample.py"""
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import synthetic_inputs  # noqa: E402
from gpt4roi_b200.engine import (EngineConfig, GraphedDecode, KVCache, PrefillEngine, SampleCache, Sampler,  # noqa: E402
                                 random_state_dicts)

DEV = 'cuda:0'
NEW = 32
HBM = 3.35e12


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return dict(device=torch.cuda.get_device_name(0), nvidia_smi=q[0] if q else None)


def timed(fn, iters, warmup=2):
    for _ in range(warmup):
        fn()
    e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    torch.cuda.synchronize()
    e[0].record()
    for _ in range(iters):
        fn()
    e[1].record()
    torch.cuda.synchronize()
    return e[0].elapsed_time(e[1]) / iters


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def weight_bytes(eng):
    n = sum(t.numel() for w in eng.layers for t in w.values()) + eng.lm_head.numel() + eng.norm_w.numel()
    return 2 * n


def main():
    print(json.dumps(card()), flush=True)
    cfg = EngineConfig(image_size=336)
    sd, vit_sd = random_state_dicts(cfg, DEV, seed=0)
    eng = PrefillEngine(cfg, sd, vit_sd, DEV)
    del sd, vit_sd
    torch.cuda.empty_cache()
    wb = weight_bytes(eng)
    row_kv = 2 * 2 * cfg.n_layers * cfg.hidden          # K and V bytes of one position, every layer
    for B in (1, 4):
        ids, images, boxes = synthetic_inputs(cfg, B, 8, 128)
        ids, images = ids.to(DEV), images.to(DEV, torch.bfloat16)
        L = ids.shape[1]
        plan = eng.plan_boxes(boxes)
        for N in (4, 8, 16):
            R = B * N
            res = {}
            for rep in range(2):
                # grouped: prefill once at batch B, N rows per prompt sharing its K/V
                c = SampleCache(cfg, B, N, L, NEW, DEV)
                smp = Sampler(R, DEV, greedy=False, temperature=0.7, top_k=50, seed=1)
                tok = torch.zeros((R, 1), dtype=torch.int64, device=DEV)

                def first_grouped():
                    lg = eng.forward_device(ids, images, plan, last_only=True, cache=c.prompt)
                    c.start(torch.full((B,), L, dtype=torch.int32, device=DEV))
                    smp(lg.repeat_interleave(N, 0), tok)
                res.setdefault('ttft_grouped_ms', []).append(wall(first_grouped))
                st = GraphedDecode(eng, c)
                res.setdefault('step_grouped_ms', []).append(timed(lambda: st.step(tok), 16))
                del st, c
                torch.cuda.empty_cache()
                # expanded: the current loop on the B*N repeated prompts
                xids, ximg = ids.repeat_interleave(N, 0), images.repeat_interleave(N, 0)
                xplan = eng.plan_boxes([b for b in boxes for _ in range(N)])
                kv = KVCache(cfg, R, L + NEW, DEV)
                res.setdefault('ttft_expanded_ms', []).append(
                    wall(lambda: smp(eng.forward_device(xids, ximg, xplan, last_only=True, cache=kv), tok)))
                kv.lens = torch.full((R,), L, dtype=torch.int32, device=DEV)   # the per-row positions generate() uses
                gd = GraphedDecode(eng, kv)
                res.setdefault('step_expanded_ms', []).append(timed(lambda: gd.step(tok), 16))
                del gd, kv, xids, ximg, xplan
                torch.cuda.empty_cache()
            best = {k: min(v) for k, v in res.items()}
            floor_g = (wb + (B * L + R * 16) * row_kv) / HBM * 1e3
            floor_x = (wb + R * (L + 16) * row_kv) / HBM * 1e3
            print(json.dumps(dict(what='multisample_7b_bf16', batch=B, num_return_sequences=N, prompt_len=L, best=best,
                                  floor_grouped_ms=floor_g, floor_expanded_ms=floor_x,
                                  step_speedup=best['step_expanded_ms'] / best['step_grouped_ms'], runs=res)),
                  flush=True)


if __name__ == '__main__':
    main()
