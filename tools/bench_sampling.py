"""Cost of next-token selection on the device (csrc/sample.cu).  Prints one JSON line per measurement, after a line
with the card's name, power limit and SM clock:
  * the sampler kernel alone at B = 1, 8, 16 -- greedy, T = 0.2 with top-k 50 (the demo's call), and top-p 0.9 without
    top-k (the whole vocabulary) -- and, on the same logits, the torch restatement it replaces (transformers'
    TemperatureLogitsWarper / TopKLogitsWarper / TopPLogitsWarper, softmax, multinomial);
  * the 7B graphed decode step (fp16, the demo's dtype) at batch 1 and 8, with and without the sampler captured;
  * the engine loop's ms per token for the demo call (706-token prompt, 64 new tokens, T = 0.2, top-k 50).
CUDA events after warm-up.  usage: python tools/bench_sampling.py [--no-7b]"""
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import synthetic_inputs  # noqa: E402
from gpt4roi_b200 import kernels  # noqa: E402
from gpt4roi_b200.engine import (EngineConfig, GraphedDecode, KVCache, PrefillEngine, Sampler,  # noqa: E402
                                 random_state_dicts)

DEV = 'cuda:0'
V = 32006


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return dict(device=torch.cuda.get_device_name(0), nvidia_smi=q[0] if q else None)


def timed(fn, iters, warmup=10):
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


def torch_restatement(logits, T, top_k, top_p, greedy):
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper
    s = logits.float()
    if greedy:
        return s.argmax(-1, keepdim=True)
    ids = None
    s = TemperatureLogitsWarper(T)(ids, s)
    if top_k:
        s = TopKLogitsWarper(top_k)(ids, s)
    if top_p < 1:
        s = TopPLogitsWarper(top_p)(ids, s)
    return torch.multinomial(torch.softmax(s, -1), 1)


def kernel_alone():
    g = torch.Generator(device=DEV).manual_seed(0)
    modes = [('greedy', True, 1.0, 0, 1.0), ('T0.2_topk50', False, 0.2, 50, 1.0), ('topp0.9', False, 1.0, 0, 0.9)]
    for B in (1, 8, 16):
        lg = (torch.randn(B, V, device=DEV, generator=g) * 3).half()
        out = torch.empty((B, 1), dtype=torch.int64, device=DEV)
        step = torch.zeros(1, dtype=torch.int64, device=DEV)
        for name, greedy, T, k, p in modes:
            ms = timed(lambda: kernels.sample_tokens(lg, out, greedy, T, k, p, 1, step), 200)
            ref = timed(lambda: torch_restatement(lg, T, k, p, greedy), 50)
            print(json.dumps(dict(what='select', batch=B, mode=name, kernel_us=ms * 1e3, torch_restatement_us=ref * 1e3)),
                  flush=True)


def decode_7b():
    cfg = EngineConfig(image_size=336, dtype='fp16')
    sd, vit_sd = random_state_dicts(cfg, DEV, seed=0)
    eng = PrefillEngine(cfg, sd, vit_sd, DEV)
    del sd, vit_sd
    torch.cuda.empty_cache()
    steps = 64
    for B in (1, 8):
        ids, images, boxes = synthetic_inputs(cfg, B, 8, 128)
        ids, images = ids.to(DEV), images.to(DEV, torch.float16)
        L = ids.shape[1]
        res = {}
        for rep in range(2):   # alternate the two variants
            for with_sampler in (False, True):
                cache = KVCache(cfg, B, L + 2 * steps + 16, DEV)
                logits = eng.forward_device(ids, images, eng.plan_boxes(boxes), last_only=True, cache=cache)
                smp = Sampler(B, DEV, greedy=False, temperature=0.2, top_k=50, seed=5) if with_sampler else None
                st = GraphedDecode(eng, cache, sampler=smp)
                if smp is not None:
                    smp(logits, st.ids)
                    ms = timed(lambda: st.step(), steps, warmup=8)
                else:
                    nxt = logits[:, -1].argmax(-1, keepdim=True)
                    ms = timed(lambda: st.step(nxt), steps, warmup=8)
                res.setdefault(with_sampler, []).append(ms)
                del st, cache
        a, b = min(res[False]), min(res[True])
        print(json.dumps(dict(what='graphed_decode_step_7b_fp16', batch=B, prompt_len=L, ms_without_sampler=res[False],
                              ms_with_sampler=res[True], added_pct=100 * (b - a) / a)), flush=True)
    # the demo's call on the engine loop: 706-token prompt, 64 new tokens (capture included, as a caller sees it)
    ids, images, boxes = synthetic_inputs(cfg, 1, 8, 128)
    ids, images = ids.to(DEV), images.to(DEV, torch.float16)
    for name, kw in (('greedy', dict()), ('T0.2_topk50', dict(do_sample=True, temperature=0.2, top_k=50))):
        t = {}
        for n in (1, 64, 1, 64):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            eng.generate(ids, images, boxes, max_new_tokens=n, **kw)
            torch.cuda.synchronize()
            t.setdefault(n, []).append((time.perf_counter() - t0) * 1e3)
        print(json.dumps(dict(what='engine_loop_demo_call', mode=name, prompt_len=ids.shape[1], new_tokens=64,
                              total_ms=min(t[64]), first_token_ms=min(t[1]),
                              ms_per_token=(min(t[64]) - min(t[1])) / 63)), flush=True)


def main():
    print(json.dumps(card()), flush=True)
    kernel_alone()
    if '--no-7b' not in sys.argv:
        decode_7b()


if __name__ == '__main__':
    main()
