"""Prompt-lookup decoding (generate(prompt_lookup_num_tokens=k)), 7B, 336 px, bf16 and fp16, batch 1, graphed.
  1. the verify step (LookupDecode's graph: the decode chain over M = k + 1 rows, the per-row selection and the lookup
     kernel) for M = 1, 2, 4, 8, 11, 16 against the plain graphed decode step (GraphedDecode with its sampler), medians
     of alternating runs with the spread, on the headline prompt (8 RoIs, 128 text tokens, L = 706);
  2. from that curve, the tokens a step must append for lookup to break even: t_verify(M) / t_plain;
  2a. the one-row step lookup runs when no window matched (LookupDecode.graph1), and the plain step with its K/V write
     unfused (G4R_DECODE_FUSED=0: qkv_rope + kv_append, as the verify chain writes K/V) -- the cost of the unfused write
     on its own;
  3. end to end, ms per generated token for 256 new tokens, greedy, with and without lookup (k = 10), on two prompts
     built to repeat (the headline prompt with its text repeated; a conversation re-sent whole), and the tokens each
     verify step actually appended.
The weights are random (seeded): how often drafts are accepted on trained GPT4RoI weights is not measured here.
Prints one JSON line per measurement with the card's name, power limit and clocks.
usage: python tools/bench_prompt_lookup.py [reps]"""
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from bench import synthetic_inputs  # noqa: E402
from bench_ragged_decode import card  # noqa: E402
from gpt4roi_b200 import engine as E  # noqa: E402
from gpt4roi_b200.engine import (EngineConfig, GraphedDecode, KVCache, LookupDecode, PrefillEngine, Sampler,  # noqa: E402
                                 random_state_dicts)

MS = (1, 2, 4, 8, 11, 16)
NEW = 256


def _time(fn, n):
    e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    torch.cuda.synchronize()
    e[0].record()
    for _ in range(n):
        fn()
    e[1].record()
    torch.cuda.synchronize()
    return e[0].elapsed_time(e[1]) / n


def _stats(ts):
    ts = sorted(ts)
    return dict(median_ms=round(ts[len(ts) // 2], 4), min_ms=round(ts[0], 4), max_ms=round(ts[-1], 4))


def _prompts(cfg):
    ids, images, boxes = synthetic_inputs(cfg, 1, 8, 128, seed=0)
    text = ids[0, -127:]                                           # the text after the image, without <bbox>
    text = text[text != cfg.bbox_token][None]
    rep = torch.cat([ids, text[:, 10:74]], 1)                      # the question's text repeated
    conv = torch.cat([ids, text, text], 1)                         # a conversation re-sent: the text turn twice more
    return ids, images, boxes, dict(repeated_text=rep, conversation=conv)


def run(dtype, reps, info):
    dev = 'cuda:0'
    cfg = EngineConfig(image_size=336, dtype=dtype)
    sd, vit_sd = random_state_dicts(cfg, dev, seed=0)
    eng = PrefillEngine(cfg, sd, vit_sd, dev)
    del sd, vit_sd
    torch.cuda.empty_cache()
    ids, images, boxes, prompts = _prompts(cfg)
    ids, images = ids.to(dev), images.to(dev, cfg.torch_dtype)
    L = ids.shape[1]
    plan = eng.plan_boxes(boxes)

    def prefill(cache):
        return eng.forward_device(ids, images, plan, validate=True, last_only=True, cache=cache)
    # the plain graphed step
    cache = KVCache(cfg, 1, L + 4096, dev)
    logits = prefill(cache)
    sampler = Sampler(1, dev)
    plain = GraphedDecode(eng, cache, sampler=sampler)
    sampler(logits, plain.ids)
    # the same step with the K/V write unfused
    cache_u = KVCache(cfg, 1, L + 4096, dev)
    logits_u = prefill(cache_u)
    sampler_u = Sampler(1, dev)
    fused = E._DECODE_FUSED
    E._DECODE_FUSED = 0
    try:
        unfused = GraphedDecode(eng, cache_u, sampler=sampler_u)
    finally:
        E._DECODE_FUSED = fused
    sampler_u(logits_u, unfused.ids)
    steps = {}
    for M in MS[1:]:
        c = KVCache(cfg, 1, L + 4096, dev)
        lg = prefill(c)
        hist = torch.zeros((1, L + 4000 + M), dtype=torch.int64, device=dev)
        hist[0, :L] = ids[0]
        st = LookupDecode(eng, c, hist, L, 4000, M - 1)
        st.first(lg)
        steps[M] = st
    extra = {'plain step, K/V write unfused': unfused.step, 'lookup one-row step (no draft)': steps[2].graph1.replay}
    runs = {M: [] for M in list(MS) + list(extra)}
    n = 20
    for _ in range(reps):        # alternating: each round times every variant once
        for M in MS:
            runs[M].append(_time(plain.step if M == 1 else steps[M].graph.replay, n))
        for name, fn in extra.items():
            runs[name].append(_time(fn, n))
    base = _stats(runs[1])
    for name in extra:
        s = _stats(runs[name])
        print(json.dumps(dict(bench='prompt_lookup_verify_step', dtype=dtype, L=L, M=1, what=name, **s,
                              vs_plain_ms=round(s['median_ms'] - base['median_ms'], 4), weights='random (seeded)',
                              **info)), flush=True)
    for M in MS:
        s = _stats(runs[M])
        print(json.dumps(dict(bench='prompt_lookup_verify_step', dtype=dtype, L=L, M=M,
                              what='plain graphed decode step' if M == 1 else 'graphed verify step',
                              **s, breakeven_tokens_per_step=round(s['median_ms'] / base['median_ms'], 3),
                              weights='random (seeded)', **info)), flush=True)
    del steps, plain, cache, unfused, cache_u
    torch.cuda.empty_cache()
    for name, p in prompts.items():
        p = p.to(dev)
        for k in (None, 10):
            kw = {} if k is None else dict(prompt_lookup_num_tokens=k)
            eng.generate(p, images, boxes, max_new_tokens=16, **kw)            # warm
            ts, acc = [], []
            for _ in range(max(3, reps // 2)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                out = eng.generate(p, images, boxes, max_new_tokens=NEW, **kw)
                torch.cuda.synchronize()
                ts.append((time.perf_counter() - t0) * 1e3)
                if k is not None:
                    acc = list(eng.lookup_accepted)
            gen = out.shape[1] - p.shape[1]
            rec = dict(bench='prompt_lookup_generate', dtype=dtype, prompt=name, L=int(p.shape[1]), new_tokens=gen,
                       lookup_k=k, **_stats(ts), ms_per_token=round(sorted(ts)[len(ts) // 2] / gen, 4),
                       weights='random (seeded)', note='includes the prefill', **info)
            if k is not None:
                rec.update(verify_steps=len(acc), tokens_per_step=round(sum(acc) / max(len(acc), 1), 3),
                           max_appended=max(acc, default=0))
            print(json.dumps(rec), flush=True)
    del eng
    torch.cuda.empty_cache()


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 7
    info = card()
    for dtype in ('bf16', 'fp16'):
        run(dtype, reps, info)


if __name__ == '__main__':
    main()
