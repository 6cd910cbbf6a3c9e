"""Decode-loop throughput (SURVEY.md 8(f1)): region-token prefill + KV-cache decode steps, 7B, bf16.
Prints one JSON line per batch size.  usage: python tools/bench_decode.py [new_tokens] [graph]"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import peaks, synthetic_inputs  # noqa: E402
from gpt4roi_b200.engine import EngineConfig, GraphedDecode, KVCache, PrefillEngine, random_state_dicts  # noqa: E402


def main():
    dev = 'cuda:0'
    n_new = int(sys.argv[1]) if len(sys.argv) > 1 else 64
    cfg = EngineConfig(image_size=336)
    sd, vit_sd = random_state_dicts(cfg, dev, seed=0)
    eng = PrefillEngine(cfg, sd, vit_sd, dev)
    del sd, vit_sd
    modes = (True,) if 'graph' in sys.argv[2:] else (False, True)
    for B, graphed in [(b, g) for b in (1, 8) for g in modes]:
        ids, images, boxes = synthetic_inputs(cfg, B, 8, 128)
        ids, images = ids.to(dev), images.to(dev)
        L = ids.shape[1]
        cache = KVCache(cfg, B, L + n_new + 4, dev)
        plan = eng.plan_boxes(boxes)
        e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        eng.forward_device(ids, images, plan, last_only=True, cache=cache)  # warm-up
        torch.cuda.synchronize()
        e[0].record()
        logits = eng.forward_device(ids, images, plan, validate=False, last_only=True, cache=cache)
        e[1].record()
        torch.cuda.synchronize()
        pre = e[0].elapsed_time(e[1])
        nxt = logits[:, -1].float().argmax(-1, keepdim=True)
        stepper = GraphedDecode(eng, cache) if graphed else None   # capture is outside the decode timing
        e[1].record()
        for _ in range(n_new):
            logits = stepper.step(nxt) if graphed else eng.decode_step(nxt, cache)
            nxt = logits[:, -1].float().argmax(-1, keepdim=True)
        e[2].record()
        torch.cuda.synchronize()
        dec = e[1].elapsed_time(e[2])
        print(json.dumps(dict(batch=B, prompt_len=L, new_tokens=n_new, prefill_ms=pre, decode_ms_per_token=dec / n_new,
                              decode_tokens_per_s=B * n_new / (dec / 1e3),
                              weight_stream_floor_ms=13.5e9 / (peaks()[0]['hbm_gbs'] * 1e9) * 1e3,
                              mode='cuda_graph' if graphed else 'eager_launches')), flush=True)


if __name__ == '__main__':
    main()
