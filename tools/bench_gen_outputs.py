"""Cost of generate()'s return_dict_in_generate outputs in the decode loop (csrc/sample.cu: g4r_sample_tokens_out_*,
which writes each row's fp32 scores and logits, 2 x 128 KB per row and token, into slot rng_step).  7B random weights in
bf16 and fp16, the headline prompt (706 tokens, 8 RoIs), batch 1 and 8, sampling at T = 0.7, top_k = 50, one process,
the variants alternating, medians of --reps.  Prints one JSON line per measurement after a line with the card's name,
power limit and SM clocks:
  * the graphed decode step with the sampler alone and with output_scores + output_logits (CUDA events over 200
    replays);
  * eng.generate wall time per new token (host clock around a call that ends in a synchronise), 256 new tokens, without
    and with the outputs.
usage: python tools/bench_gen_outputs.py [--out FILE] [--reps N]"""
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

DEV = 'cuda:0'
REPLAYS = 200
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


def step_ms(eng, cfg, ids, images, boxes, outputs):
    """One prefill, one capture, then REPLAYS replays of the graphed step between two CUDA events."""
    B, L = ids.shape
    n = REPLAYS + 32
    cache = KVCache(cfg, B, L + n, DEV)
    logits = eng.forward_device(ids, images, eng.plan_boxes(boxes), last_only=True, cache=cache)
    V = logits.shape[-1]
    bufs = [torch.empty((n, B, V), dtype=torch.float32, device=DEV) for _ in range(2)] if outputs else [None, None]
    smp = Sampler(B, DEV, scores=bufs[0], logits=bufs[1], **SAMPLE)
    st = GraphedDecode(eng, cache, sampler=smp)
    smp(logits, st.ids)
    smp.advance()
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
        sys.exit('bench_gen_outputs: no CUDA device found; this measurement runs on the GPU only (there is no CPU path)')
    out = open(args.out, 'a') if args.out else None
    emit(out, card())
    for dtype in ('bf16', 'fp16'):
        cfg = EngineConfig(image_size=336, dtype=dtype)
        sd, vit_sd = random_state_dicts(cfg, DEV, seed=0, dtype=cfg.torch_dtype)
        eng = PrefillEngine(cfg, sd, vit_sd, DEV)
        del sd, vit_sd
        torch.cuda.empty_cache()
        for B in (1, 8):
            ids, images, boxes = synthetic_inputs(cfg, B, 8, 128)
            ids, images = ids.to(DEV), images.to(DEV, cfg.torch_dtype)
            L = ids.shape[1]
            res = {False: [], True: []}
            for rep in range(args.reps):
                for outputs in (False, True):
                    res[outputs].append(step_ms(eng, cfg, ids, images, boxes, outputs))
            a, b = statistics.median(res[False]), statistics.median(res[True])
            emit(out, dict(what='graphed_decode_step_7b_' + dtype, batch=B, prompt_len=L, replays=REPLAYS,
                           sampling=SAMPLE, ms_plain=res[False], ms_outputs=res[True], median_plain=a,
                           median_outputs=b, added_us=1e3 * (b - a), added_pct=100 * (b - a) / a))
            kw = dict(do_sample=True, temperature=0.7, top_k=50)
            outs = dict(output_scores=True, output_logits=True)
            eng.generate(ids, images, boxes, max_new_tokens=8, **kw)      # warm every shape of the call
            eng.generate(ids, images, boxes, max_new_tokens=8, **kw, **outs)
            n = 256
            t = {'plain': [], 'outputs': []}
            for rep in range(args.reps):
                for name in t:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    got = eng.generate(ids, images, boxes, max_new_tokens=n, **kw, **(outs if name == 'outputs' else {}))
                    torch.cuda.synchronize()
                    t[name].append((time.perf_counter() - t0) * 1e3 / n)
                    seq = got['sequences'] if isinstance(got, dict) else got
                    assert seq.shape[1] == L + n
                    del got
            emit(out, dict(what='generate_wall_ms_per_new_token_7b_' + dtype, batch=B, prompt_len=L, new_tokens=n,
                           includes='prefill, graph capture and (outputs) the slot buffers, spread over the new tokens',
                           median={k: statistics.median(v) for k, v in t.items()}, all=t))
        del eng
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
