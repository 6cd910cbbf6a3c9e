"""Second turn of a conversation, 7B, bf16, 336 px: time to the first token with the KV cache of turn 1 reused
(PrefillEngine.prefill_cached -> extend of the new tokens only) against a full prefill of the whole conversation, and
the graphed decode step after extend.  gpt4roi/app.py re-submits the whole conversation every turn.
  turn 1: the headline prompt (8 RoIs, 128 text tokens, L = 706) + 64 greedy graphed tokens;
  turn 2: turn 1's output + a 48-token question, (a) without a new box, (b) with one new <bbox> (reruns ViT + fuse).
The cached-attention share of extend comes from CUDA events around every kernels.attention_cached call in a separate
(instrumented) run.  Prints one JSON line per (batch, variant) with the card's name, power limit and clocks.
usage: python tools/bench_multiturn.py [reps] [batch ...]"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from bench import synthetic_inputs  # noqa: E402
from bench_ragged_decode import card  # noqa: E402
from gpt4roi_b200 import kernels  # noqa: E402
from gpt4roi_b200.engine import EngineConfig, GraphedDecode, KVCache, PrefillEngine, random_state_dicts  # noqa: E402

N1, Q, STEPS = 64, 48, 32


def _median_ms(fn, reps):
    ts = []
    for _ in range(reps):
        e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        torch.cuda.synchronize()
        e[0].record()
        fn()
        e[1].record()
        torch.cuda.synchronize()
        ts.append(e[0].elapsed_time(e[1]))
    return sorted(ts)[len(ts) // 2], min(ts), max(ts)


def main():
    dev = 'cuda:0'
    args = [int(a) for a in sys.argv[1:]]
    reps = args[0] if args else 7
    batches = args[1:] or [1, 8]
    cfg = EngineConfig(image_size=336)
    sd, vit_sd = random_state_dicts(cfg, dev, seed=0)
    eng = PrefillEngine(cfg, sd, vit_sd, dev)
    del sd, vit_sd
    torch.cuda.empty_cache()
    info = card()
    for B in batches:
        ids1, images, boxes = synthetic_inputs(cfg, B, 8, 128)
        images = images.to(dev)
        cache = KVCache(cfg, B, ids1.shape[1] + N1 + Q + STEPS + 8, dev)
        out1 = eng.generate(ids1.to(dev), images, boxes, max_new_tokens=N1, cache=cache).cpu()
        g = torch.Generator().manual_seed(B)
        snap = (cache.lens.clone() if cache.lens is not None else None, cache.length, cache.ids.clone(),
                list(cache.boxes), cache.images)
        for variant in ('no_new_box', 'new_box'):
            q = torch.randint(3, 32000, (B, Q), generator=g)
            boxes2 = boxes
            if variant == 'new_box':
                q[:, Q // 2] = cfg.bbox_token
                boxes2 = [torch.cat([bx, torch.tensor([[0.2, 0.3, 0.6, 0.7]])]) for bx in boxes]
            ids2 = torch.cat([out1, q], 1)
            L2 = ids2.shape[1]

            def restore():
                cache.lens = None if snap[0] is None else snap[0].clone()
                cache.length = snap[1]
                cache.ids.copy_(snap[2])
                cache.boxes, cache.images, cache.source_known = list(snap[3]), snap[4], True

            def cached():
                restore()
                eng.prefill_cached(cache, ids2, images, boxes2, new_tokens=STEPS)[:, -1].float().argmax(-1)

            full_cache = KVCache(cfg, B, L2 + 8, dev)
            ids2_dev, plan2 = ids2.to(dev), eng.plan_boxes(boxes2)

            def full():
                eng.forward_device(ids2_dev, images, plan2, validate=True, last_only=True,
                                   cache=full_cache)[:, -1].float().argmax(-1)

            restore()
            reuse = cache.reusable(ids2, images, boxes2)
            for fn in (cached, full):   # warm-up
                fn()
                fn()
            # alternate the two paths so both see the same clocks
            t_cached, t_full = [], []
            for _ in range(reps):
                t_cached.append(_median_ms(cached, 1)[0])
                t_full.append(_median_ms(full, 1)[0])
            t_cached.sort()
            t_full.sort()
            # share of the cached attention in extend: events around each call in a separate instrumented run
            evs = []
            orig = kernels.attention_cached

            def timed(*a, **k):
                e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
                e[0].record()
                r = orig(*a, **k)
                e[1].record()
                evs.append(e)
                return r
            kernels.attention_cached = timed
            try:
                ext_ms = _median_ms(cached, 1)[0]
            finally:
                kernels.attention_cached = orig
            attn_ms = sum(e[0].elapsed_time(e[1]) for e in evs)
            # decode step after extend (graphed)
            restore()
            logits = eng.prefill_cached(cache, ids2, images, boxes2, new_tokens=STEPS)
            nxt = logits[:, -1].float().argmax(-1, keepdim=True)
            stepper = GraphedDecode(eng, cache)
            for _ in range(4):
                nxt = stepper.step(nxt)[:, -1].float().argmax(-1, keepdim=True)
            state = {'nxt': nxt}

            def steps():
                for _ in range(STEPS - 8):
                    state['nxt'] = stepper.step(state['nxt'])[:, -1].float().argmax(-1, keepdim=True)
            step_ms = _median_ms(steps, 1)[0] / (STEPS - 8)
            del stepper
            print(json.dumps(dict(
                batch=B, variant=variant, turn1_len=ids1.shape[1], turn2_len=L2, reused=int(reuse.min()),
                extend_tokens=int(L2 - reuse.min()), reps=reps,
                ttft_cached_ms=round(t_cached[len(t_cached) // 2], 3),
                ttft_cached_range_ms=[round(t_cached[0], 3), round(t_cached[-1], 3)],
                ttft_full_prefill_ms=round(t_full[len(t_full) // 2], 3),
                ttft_full_range_ms=[round(t_full[0], 3), round(t_full[-1], 3)],
                speedup=round(t_full[len(t_full) // 2] / t_cached[len(t_cached) // 2], 2),
                cached_attention_ms=round(attn_ms, 3), cached_attention_share=round(attn_ms / ext_ms, 4),
                decode_step_after_extend_ms=round(step_ms, 4), card=info)), flush=True)
            del full_cache
            torch.cuda.empty_cache()
        del cache
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
