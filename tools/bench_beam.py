"""Cost of beam search on the 7B config (bf16, the headline prompt: 706 tokens with 8 RoIs), N = 4 beams, B in {1, 4},
64 new tokens with eos disabled.  Prints one JSON line per measurement, after a line with the card's name, power limit
and SM clock:
  * the engine loop (generate(num_beams=4)): time to first token (prefill at batch B + the first beam step) and ms per
    step of the graphed beam step;
  * the work transformers' loop does per step over this engine (use_hf_loop=True): the prefill of the B*N expanded rows,
    then per step a graphed decode step at B*N rows plus G4RCache.reorder_cache (a gather of every layer's K/V) --
    HF's Python overhead not included;
  * the graphed beam step against a greedy graphed decode step at the same B*N rows: the cost of the ancestry-table
    attention and the two beam kernels.
CUDA events / a host clock after a device synchronise.  usage: python tools/bench_beam.py"""
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import synthetic_inputs  # noqa: E402
from gpt4roi_b200.engine import (BeamCache, EngineConfig, GraphedBeamDecode, GraphedDecode, KVCache,  # noqa: E402
                                 PrefillEngine, random_state_dicts)
from gpt4roi_b200.spi_llava import G4RCache  # noqa: E402

DEV = 'cuda:0'
N, NEW = 4, 64


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return dict(device=torch.cuda.get_device_name(0), nvidia_smi=q[0] if q else None)


def timed(fn, iters, warmup=5):
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


def main():
    print(json.dumps(card()), flush=True)
    cfg = EngineConfig(image_size=336)
    sd, vit_sd = random_state_dicts(cfg, DEV, seed=0)
    eng = PrefillEngine(cfg, sd, vit_sd, DEV)
    del sd, vit_sd
    torch.cuda.empty_cache()
    for B in (1, 4):
        ids, images, boxes = synthetic_inputs(cfg, B, 8, 128)
        ids, images = ids.to(DEV), images.to(DEV, torch.bfloat16)
        L = ids.shape[1]
        plan = eng.plan_boxes(boxes)
        R = B * N
        res = {}
        for rep in range(2):
            # engine loop: prefill once at batch B, the first beam step, then the graphed beam step
            c = BeamCache(cfg, B, N, L, NEW, DEV)
            ttft = wall(lambda: (eng.forward_device(ids, images, plan, last_only=True, cache=c.prompt),
                                 c.start(torch.full((B,), L, dtype=torch.int32, device=DEV))))
            logits = eng.forward_device(ids, images, plan, last_only=True, cache=c.prompt)
            t1 = wall(lambda: c.step(logits, first=True))
            st = GraphedBeamDecode(eng, c)
            res.setdefault('engine_ttft_ms', []).append(ttft + t1)
            res.setdefault('beam_step_ms', []).append(timed(st.step, NEW - 2, warmup=1))
            del st, c
            # HF loop's work on this engine: B*N expanded rows prefilled, greedy graphed step + K/V gather per step
            xids = ids.repeat_interleave(N, 0)
            ximg = images.repeat_interleave(N, 0)
            xplan = eng.plan_boxes([b for b in boxes for _ in range(N)])
            kv = KVCache(cfg, R, L + NEW + 8, DEV)
            res.setdefault('hf_ttft_ms', []).append(
                wall(lambda: eng.forward_device(xids, ximg, xplan, last_only=True, cache=kv)))
            gd = GraphedDecode(eng, kv)
            tok = torch.zeros((R, 1), dtype=torch.int64, device=DEV)
            perm = torch.arange(R, device=DEV).flip(0)
            cache = G4RCache(kv)
            res.setdefault('greedy_step_ms', []).append(timed(lambda: gd.step(tok), 16, warmup=2))
            res.setdefault('hf_step_ms', []).append(timed(lambda: (gd.step(tok), cache.reorder_cache(perm)), 16,
                                                          warmup=2))
            del gd, kv, cache
            torch.cuda.empty_cache()
        best = {k: min(v) for k, v in res.items()}
        print(json.dumps(dict(what='beam_search_7b_bf16', batch=B, num_beams=N, prompt_len=L, new_tokens=NEW, runs=res,
                              beam_step_over_greedy_pct=100 * (best['beam_step_ms'] - best['greedy_step_ms'])
                              / best['greedy_step_ms'])), flush=True)


if __name__ == '__main__':
    main()
