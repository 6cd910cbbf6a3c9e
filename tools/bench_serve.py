"""Serving throughput under request traffic on the 7B config (bf16, the headline prompt: 706 tokens with 8 RoIs): 32
greedy requests whose answer lengths are drawn (seeded) uniformly from 16..256 tokens, eos off so that the lengths hold,
arriving all at t = 0 or as a seeded Poisson stream (mean gap ARRIVAL_GAP_S).  Served four ways:
  * sequential: one eng.generate per request, in arrival order;
  * static8: batches of 8 requests in arrival order through eng.generate (a batch starts when its last request has
    arrived and the previous batch is done; every request of a batch waits for the batch's longest answer);
  * batcher8 / batcher16: engine.ContinuousBatcher with 8 / 16 slots, requests submitted as they arrive.
Per way: generated tokens per second over the whole run, time to first token and request latency (p50 / p90, from
each request's arrival).  Also the graphed decode step of the batcher with every slot running, and kernels.
sample_tokens_rows against kernels.sample_tokens at S = 8 and 16 (sampling, T 0.7, top-k 50).  Prints one JSON line per
figure after a line with the card's name, power limit and SM clocks.  Host clocks after a device synchronise (the
batcher's token readback synchronises every step; generate's first token is stamped from a stopping_criteria callback
that synchronises once); CUDA events for the step and kernel times.
usage: python tools/bench_serve.py"""
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
from gpt4roi_b200.engine import ContinuousBatcher, EngineConfig, PrefillEngine, random_state_dicts  # noqa: E402

DEV = 'cuda:0'
N_REQ, MIN_NEW, MAX_NEW = 32, 16, 256
ARRIVAL_GAP_S = 0.1
MAX_LEN = 1024


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return dict(device=torch.cuda.get_device_name(0), nvidia_smi=q[0] if q else None)


def timed(fn, iters, warmup=3):
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


def pct(xs, q):
    xs = sorted(xs)
    return xs[min(len(xs) - 1, int(round(q * (len(xs) - 1))))]


class _Stamp:
    """A streamer that records when the first token and the end reach the host."""

    def __init__(self):
        self.first = self.end_t = None
        self.n = -1

    def put(self, value):
        self.n += 1
        if self.n == 1:
            self.first = time.perf_counter()

    def end(self):
        self.end_t = time.perf_counter()


class _FirstToken:
    """A stopping_criteria callback of generate(): stamps the first token once it is on the device, never stops."""

    def __init__(self):
        self.t = None

    def __call__(self, ids, scores):
        if self.t is None:
            torch.cuda.synchronize()
            self.t = time.perf_counter()
        return False


def serve_generate(eng, req, arrive, batch):
    """Requests in arrival order, `batch` at a time, through eng.generate.  -> (ttft, latency) lists, end time."""
    ids, images, boxes = req
    t0 = time.perf_counter()
    ttft, lat, free = [None] * len(arrive), [None] * len(arrive), 0.0
    for s in range(0, len(arrive), batch):
        idx = list(range(s, min(s + batch, len(arrive))))
        start = max(free, max(arrive[i][0] for i in idx))
        while time.perf_counter() - t0 < start:
            time.sleep(1e-4)
        n = max(arrive[i][1] for i in idx)
        cb = _FirstToken()
        eng.generate(ids.repeat(len(idx), 1), images.repeat(len(idx), 1, 1, 1), boxes * len(idx),
                     max_new_tokens=n, stopping_criteria=[cb])
        torch.cuda.synchronize()
        free = time.perf_counter() - t0
        for i in idx:
            ttft[i] = cb.t - t0 - arrive[i][0]
            lat[i] = free - arrive[i][0]
    return ttft, lat, free


def serve_batcher(eng, req, arrive, slots):
    ids, images, boxes = req
    b = ContinuousBatcher(eng, slots, MAX_LEN)
    stamps = [_Stamp() for _ in arrive]
    t0 = time.perf_counter()
    nxt = 0
    while nxt < len(arrive) or b.queue or any(r is not None for r in b.running):
        now = time.perf_counter() - t0
        while nxt < len(arrive) and arrive[nxt][0] <= now:
            b.submit(ids, images, boxes, max_new_tokens=arrive[nxt][1], streamer=stamps[nxt])
            nxt += 1
        if b.queue or any(r is not None for r in b.running):
            b.step()
        else:
            time.sleep(1e-4)
    end = time.perf_counter() - t0
    ttft = [s.first - t0 - a[0] for s, a in zip(stamps, arrive)]
    lat = [s.end_t - t0 - a[0] for s, a in zip(stamps, arrive)]
    return ttft, lat, end, b


def step_time(eng, req, slots):
    ids, images, boxes = req
    b = ContinuousBatcher(eng, slots, MAX_LEN)
    for _ in range(slots):
        b.submit(ids, images, boxes, max_new_tokens=MAX_NEW)
    b.step()                                   # admits every slot
    return timed(b.graph.replay, 20)


def kernel_times(V):
    out = {}
    for S in (8, 16):
        lg = (torch.randn(S, V, device=DEV) * 3).to(torch.bfloat16)
        ids = torch.zeros(S, 1, dtype=torch.int64, device=DEV)
        step1 = torch.zeros(1, dtype=torch.int64, device=DEV)
        out['sample_tokens_S%d_ms' % S] = timed(
            lambda: kernels.sample_tokens(lg, ids, False, 0.7, 50, 1.0, 3, step1), 50)

        def vec(v, dt):
            return torch.full((S,), v, dtype=dt, device=DEV)
        rows = (vec(0, torch.int32), vec(0.7, torch.float32), vec(50, torch.int32), vec(1.0, torch.float32),
                vec(3, torch.int64), vec(0, torch.int64), vec(-1, torch.int32), vec(1, torch.int32), vec(0, torch.int32))
        out['sample_tokens_rows_S%d_ms' % S] = timed(lambda: kernels.sample_tokens_rows(lg, ids, *rows), 50)
    return out


def main():
    print(json.dumps(card()), flush=True)
    cfg = EngineConfig(image_size=336)
    sd, vit_sd = random_state_dicts(cfg, DEV, seed=0)
    eng = PrefillEngine(cfg, sd, vit_sd, DEV)
    del sd, vit_sd
    torch.cuda.empty_cache()
    ids, images, boxes = synthetic_inputs(cfg, 1, 8, 128)
    req = (ids.to(DEV), images.to(DEV, torch.bfloat16), boxes)
    L = ids.shape[1]
    print(json.dumps(dict(what='serve_kernels', **kernel_times(cfg.vocab))), flush=True)
    for slots in (8, 16):
        print(json.dumps(dict(what='serve_step', slots=slots, step_ms=step_time(eng, req, slots))), flush=True)
    g = torch.Generator().manual_seed(0)
    lengths = torch.randint(MIN_NEW, MAX_NEW + 1, (N_REQ,), generator=g).tolist()
    gaps = torch.empty(N_REQ).exponential_(1.0 / ARRIVAL_GAP_S, generator=g)
    poisson = (gaps.cumsum(0) - gaps[0]).tolist()
    # warm-up: every shape the timed runs use (generate at batch 1 and 8, the batcher's graphs)
    serve_generate(eng, req, [(0.0, 8)] * 8, 8)
    serve_generate(eng, req, [(0.0, 8)], 1)
    for slots in (8, 16):
        serve_batcher(eng, req, [(0.0, 8)] * 2, slots)
    for traffic, arrivals in (('all_at_t0', [0.0] * N_REQ), ('poisson', poisson)):
        arrive = list(zip(arrivals, lengths))
        for way, run in (('sequential', lambda: serve_generate(eng, req, arrive, 1)),
                         ('static8', lambda: serve_generate(eng, req, arrive, 8)),
                         ('batcher8', lambda: serve_batcher(eng, req, arrive, 8)[:3]),
                         ('batcher16', lambda: serve_batcher(eng, req, arrive, 16)[:3])):
            ttft, lat, end = run()
            print(json.dumps(dict(what='serve_7b_bf16', traffic=traffic, way=way, requests=N_REQ, prompt_len=L,
                                  new_tokens=sum(lengths), tokens_per_s=sum(lengths) / end, makespan_s=end,
                                  ttft_p50_s=pct(ttft, 0.5), ttft_p90_s=pct(ttft, 0.9),
                                  latency_p50_s=pct(lat, 0.5), latency_p90_s=pct(lat, 0.9))), flush=True)
            torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
