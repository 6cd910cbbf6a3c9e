"""Prefix reuse in the continuous batcher (ContinuousBatcher(prefix_reuse=True)) on the 7B config (bf16, 336 px, the
headline prompt: 706 tokens with 8 RoIs), greedy, eos off, answer lengths drawn (seeded) from 16..64 tokens.  Reuse off
against on, at 8 and 16 slots, on three kinds of traffic:
  * conversations: 16 users x 3 turns, each user with its own image.  Every turn sends the whole conversation again, as
    the demo and the gradio worker do: turn 2 = turn 1 + its answer + a 48-token question, turn 3 = turn 2 + its answer +
    a 48-token question holding one new <bbox> (and its box).  A user submits a turn when the previous one finishes.
  * shared images: 32 questions over 4 images, all at t = 0: each a 48-token question with 1-2 boxes after the image's
    common 600-token prompt (system text and image span).
  * no sharing: 32 headline prompts on 32 distinct images at t = 0 -- reuse finds nothing, so its matching is all it
    adds.
Per run: tokens per second over the run, time to first token p50 / p90 (per turn for the conversations, from each
request's submission) and the prompt tokens taken from the cache.  The runs alternate off / on, REPEATS times each; the
JSON lines give the median and the spread (min, max) of every figure.  Then the row-table chunk prefill
(PrefillEngine.extend on a row view of a 16-row cache, the batcher's path) at k = 1 / 4 / 8 requests against extend on a
contiguous k-row cache of the same contents: 48-token tails after 700 held tokens, host clock around each call after a
device synchronise, median of 5.  The first line gives the card's name, power limit and SM clocks.
usage: python tools/bench_serve_prefix.py"""
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from bench import synthetic_inputs  # noqa: E402
from bench_serve import _Stamp, card, pct  # noqa: E402
from gpt4roi_b200.engine import ContinuousBatcher, EngineConfig, KVCache, PrefillEngine, random_state_dicts  # noqa: E402

DEV = 'cuda:0'
MIN_NEW, MAX_NEW = 16, 64
MAX_LEN = 1024
USERS, TURNS = 16, 3
REPEATS = 3


def _lengths(n, seed):
    return torch.randint(MIN_NEW, MAX_NEW + 1, (n,), generator=torch.Generator().manual_seed(seed)).tolist()


def _question(seed, n_box=0, cfg=None):
    g = torch.Generator().manual_seed(seed)
    q = torch.randint(3, 32000, (1, 48), generator=g)
    boxes = []
    for k in range(n_box):
        q[0, 5 + 20 * k] = cfg.bbox_token
        p = torch.rand(2, 2, generator=g).sort(dim=0).values
        boxes.append(torch.tensor([[p[0, 0], p[0, 1], max(p[1, 0], p[0, 0] + 0.01), max(p[1, 1], p[0, 1] + 0.01)]]))
    return q, boxes


def _run(b, first, follow):
    """Serve: `first` (list of (spec, user)) submitted at t = 0; follow(user, finished request) -> the user's next spec or
    None.  -> (per-turn ttft lists, new tokens, seconds, reused tokens)."""
    t0 = time.perf_counter()
    live, ttft, tokens, reused = {}, {}, 0, 0

    def submit(spec, user, turn):
        st = _Stamp()
        r = b.submit(streamer=st, **spec)
        live[r] = (user, turn, st, time.perf_counter())

    for spec, user in first:
        submit(spec, user, 0)
    while b.queue or any(r is not None for r in b.running):
        for r in b.step():
            user, turn, st, sub = live.pop(r)
            ttft.setdefault(turn, []).append(st.first - sub)
            tokens += len(r.tokens)
            reused += r.reused
            nxt = follow(user, r)
            if nxt is not None:
                submit(nxt, user, turn + 1)
    torch.cuda.synchronize()
    return ttft, tokens, time.perf_counter() - t0, reused


def conversations(cfg, req_of):
    lengths = _lengths(USERS * TURNS, 1)
    first = [(dict(req_of(u), max_new_tokens=lengths[u * TURNS]), u) for u in range(USERS)]
    turn = {u: 0 for u in range(USERS)}

    def follow(u, r):
        turn[u] += 1
        if turn[u] >= TURNS:
            return None
        base = req_of(u)
        q, nb = _question(1000 * u + turn[u], n_box=1 if turn[u] == 2 else 0, cfg=cfg)
        prev_boxes = r.bboxes[0]
        seq = r.sequences.clone()
        # random weights may emit image / <bbox> ids, which a re-encoded answer would not hold: plain text instead
        ans = seq[:, r.input_ids.shape[1]:]
        ans[ans >= 32000] = 100
        return dict(input_ids=torch.cat([seq, q], 1), images=base['images'],
                    bboxes=[torch.cat([prev_boxes] + nb)], max_new_tokens=lengths[u * TURNS + turn[u]])
    return first, follow


def shared_images(cfg, images):
    lengths = _lengths(32, 2)
    first = []
    for i in range(32):
        ids, img = images[i % 4]
        q, nb = _question(2000 + i, n_box=1 + i % 2, cfg=cfg)
        first.append((dict(input_ids=torch.cat([ids, q], 1), images=img, bboxes=[torch.cat(nb)],
                           max_new_tokens=lengths[i]), i))
    return first, lambda u, r: None


def no_sharing(req_of):
    lengths = _lengths(32, 3)
    return [(dict(req_of(100 + i), max_new_tokens=lengths[i]), i) for i in range(32)], lambda u, r: None


def summary(runs):
    """runs: list of dicts of figures -> {figure: dict(median, min, max)}."""
    return {k: dict(median=statistics.median(r[k] for r in runs), min=min(r[k] for r in runs),
                    max=max(r[k] for r in runs)) for k in runs[0]}


def figures(ttft, tokens, secs, reused):
    out = dict(tokens_per_s=tokens / secs, seconds=secs, reused_tokens=reused)
    for t, xs in sorted(ttft.items()):
        out['turn%d_ttft_p50_ms' % (t + 1)] = 1e3 * pct(xs, 0.5)
        out['turn%d_ttft_p90_ms' % (t + 1)] = 1e3 * pct(xs, 0.9)
    return out


def chunk_prefill(eng, cfg):
    """The row-table chunk prefill against extend on a contiguous cache of the same contents (k rows, 48-token tails
    after 700 held tokens)."""
    S, start, Lc = 16, 700, 48
    big = KVCache(cfg, S, MAX_LEN, DEV)
    out = {}
    for k in (1, 4, 8):
        rows = list(range(0, 2 * k, 2))            # not adjacent
        ids = torch.randint(3, 32000, (k, Lc), generator=torch.Generator().manual_seed(k))
        cont = KVCache(cfg, k, MAX_LEN, DEV)
        for li in range(cfg.n_layers):
            cont.k[li].copy_(big.k[li][rows])
            cont.v[li].copy_(big.v[li][rows])
        view = KVCache(cfg, k, MAX_LEN, DEV, kv=(big.k, big.v), rows=torch.tensor(rows, dtype=torch.int32, device=DEV))
        res = {}
        for name, c in (('contiguous', cont), ('row_table', view)) * 6:
            times = res.setdefault(name, [])
            c.lens = torch.full((k,), start, dtype=torch.int32, device=DEV)
            c.length = start
            torch.cuda.synchronize()
            t = time.perf_counter()
            eng.extend(c, ids, None, None)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t)
        for name, times in res.items():
            times = times[1:]                      # the first call of each warms up
            out['k%d_%s_ms' % (k, name)] = 1e3 * statistics.median(times)
            out['k%d_%s_spread_ms' % (k, name)] = [1e3 * min(times), 1e3 * max(times)]
    return out


def main():
    print(json.dumps(card()), flush=True)
    cfg = EngineConfig(image_size=336)
    sd, vit_sd = random_state_dicts(cfg, DEV, seed=0)
    eng = PrefillEngine(cfg, sd, vit_sd, DEV)
    del sd, vit_sd
    torch.cuda.empty_cache()

    def req_of(seed):
        ids, images, boxes = synthetic_inputs(cfg, 1, 8, 128, seed=seed)
        return dict(input_ids=ids, images=images.to(DEV, torch.bfloat16), bboxes=boxes)
    common = []
    for i in range(4):                               # 600 shared tokens: system text and image span, no box
        ids, images, _ = synthetic_inputs(cfg, 1, 0, 128, seed=500 + i)
        common.append((ids[:, :600], images.to(DEV, torch.bfloat16)))
    print(json.dumps(dict(what='serve_prefix_chunk_prefill', **chunk_prefill(eng, cfg))), flush=True)
    workloads = (('conversations', lambda: conversations(cfg, req_of)),
                 ('shared_images', lambda: shared_images(cfg, common)),
                 ('no_sharing', lambda: no_sharing(req_of)))
    for slots in (8, 16):
        for name, make in workloads:
            for reuse in (False, True):             # warm-up: every shape of the timed runs
                first, _ = make()
                _run(ContinuousBatcher(eng, slots, MAX_LEN, prefix_reuse=reuse), first[:2], lambda u, r: None)
            runs = {False: [], True: []}
            for _ in range(REPEATS):
                for reuse in (False, True):
                    first, follow = make()
                    # a fresh batcher per run: rows start empty (its graph is captured outside the timed window)
                    b = ContinuousBatcher(eng, slots, MAX_LEN, prefix_reuse=reuse)
                    runs[reuse].append(figures(*_run(b, first, follow)))
                    del b
                    torch.cuda.empty_cache()
            for reuse in (False, True):
                print(json.dumps(dict(what='serve_prefix_7b_bf16', workload=name, slots=slots, prefix_reuse=reuse,
                                      repeats=REPEATS, **summary(runs[reuse]))), flush=True)


if __name__ == '__main__':
    main()
