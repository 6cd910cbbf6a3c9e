"""Graphed decode step over prompts of different lengths vs prompts of one length, 7B, bf16, after a 336-px
region-token prefill (L = 706: 576 image tokens + 128 text tokens + 2).  For each batch size two cases:
  ragged  -- prompt lengths spread evenly over [L/2, L] (the longest at L), per-sample positions in the KV cache;
  uniform -- every prompt at L (the scalar-position path).
Prints one JSON line per (batch, case) with the step time and the byte floor of the step: every weight once plus each
sample's own K/V rows, over the HBM peak (MEASURED_PEAKS.json or the H100 SXM data sheet, see bench.peaks), and the
card's name, power limit and clocks.  usage: python tools/bench_ragged_decode.py [steps] [batch ...]"""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import peaks, synthetic_inputs  # noqa: E402
from gpt4roi_b200.engine import EngineConfig, GraphedDecode, KVCache, PrefillEngine, random_state_dicts  # noqa: E402


def card():
    q = 'name,power.limit,clocks.sm,clocks.max.sm,clocks.mem'
    try:
        r = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=' + q, '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30)
        return dict(zip(q.split(','), [x.strip() for x in r.stdout.strip().split(',')]))
    except Exception:
        return dict(name=torch.cuda.get_device_name(0))


def main():
    dev = 'cuda:0'
    args = [int(a) for a in sys.argv[1:]]
    steps = args[0] if args else 64
    batches = args[1:] or [8, 16, 32]
    cfg = EngineConfig(image_size=336)
    sd, vit_sd = random_state_dicts(cfg, dev, seed=0)
    eng = PrefillEngine(cfg, sd, vit_sd, dev)
    del sd, vit_sd
    torch.cuda.empty_cache()
    w_bytes = sum(t.numel() * t.element_size() for w in eng.layers for t in w.values()) + \
        eng.lm_head.numel() * eng.lm_head.element_size()
    kv_row_bytes = 2 * cfg.n_layers * cfg.hidden * 2     # K and V, every layer, one position of one sample
    hbm = peaks()[0]['hbm_gbs'] * 1e9
    info = card()
    for B in batches:
        ids, images, boxes = synthetic_inputs(cfg, B, 8, 128)
        ids, images = ids.to(dev), images.to(dev)
        L = ids.shape[1]
        plan = eng.plan_boxes(boxes)
        spread = torch.linspace(L, L // 2, B).round().to(torch.int32) if B > 1 else torch.tensor([L], dtype=torch.int32)
        for case in ('ragged', 'uniform'):
            seqlens = spread.to(dev) if case == 'ragged' else None
            cache = KVCache(cfg, B, L + steps + 8, dev)
            logits = eng.forward_device(ids, images, plan, last_only=True, seqlens=seqlens, cache=cache)
            nxt = logits[:, -1].float().argmax(-1, keepdim=True)
            stepper = GraphedDecode(eng, cache)
            for _ in range(4):                                  # warm-up replays
                nxt = stepper.step(nxt)[:, -1].float().argmax(-1, keepdim=True)
            lens0 = (spread if case == 'ragged' else torch.full((B,), L, dtype=torch.int32)).long() + 4
            e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            torch.cuda.synchronize()
            e[0].record()
            for _ in range(steps):
                nxt = stepper.step(nxt)[:, -1].float().argmax(-1, keepdim=True)
            e[1].record()
            torch.cuda.synchronize()
            ms = e[0].elapsed_time(e[1]) / steps
            # keys read per step: each sample's own length + 1 (the new row), averaged over the timed window
            kv_bytes = kv_row_bytes * float((lens0 + 1).sum() + B * (steps - 1) / 2.0)
            floor_ms = (w_bytes + kv_bytes) / hbm * 1e3
            print(json.dumps(dict(batch=B, case=case, prompt_len=L, min_len=int(spread.min()) if case == 'ragged' else L,
                                  steps=steps, step_ms=round(ms, 4), tokens_per_s=round(B / (ms / 1e3), 1),
                                  weight_gb=round(w_bytes / 1e9, 3), kv_gb=round(kv_bytes / 1e9, 3),
                                  byte_floor_ms=round(floor_ms, 4), share_of_floor=round(floor_ms / ms, 3),
                                  hbm_peak_source=peaks()[1], card=info)), flush=True)
            del stepper, cache, logits
            torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
