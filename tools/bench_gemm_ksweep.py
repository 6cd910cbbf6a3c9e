"""Fixed cost per tile of the wgmma GEMM (csrc/gemm_wgmma.cu): each LLaMA / lm_head shape of the headline prefill
step and the 192 px 3x3 fuse conv (with GroupNorm statistics) timed at the same M and N over several K.

  python tools/bench_gemm_ksweep.py [--reps 5] [--min-ms 100] [--out FILE.json]

The persistent kernel runs ceil(tiles / SMs) rounds of 128 x 256 tiles (the width pick_block_n chooses for every
one of these shapes), so the time per round is close to slope x k-blocks + intercept: the slope is the mainloop
cost of one 64-deep k-block, the intercept what a tile costs besides its MMAs (the epilogue, the pipeline fill and the
launch).  A least-squares line through the per-K medians gives both; intercept x rounds x launches per step is the
time one headline step spends outside the mainloops of that shape.  The card's name, power limit and the SM clock
sampled during each shape's windows are printed with the numbers.  Needs a CUDA device; there is no CPU path."""
import argparse
import json
import math
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from bench import ClockSampler  # noqa: E402
from bench_gemm import gpu_info, time_window  # noqa: E402
from gpt4roi_b200 import dense  # noqa: E402

BF = torch.bfloat16
BN = 256


def shapes(dev):
    """(name, launches per headline step, m_tiles, n_tiles, [(k_blocks, fn)]) -- fn builds its inputs lazily."""
    g = torch.Generator(device=dev).manual_seed(0)

    def rn(*s, std=1.0):
        return (torch.randn(*s, device=dev, generator=g) * std).to(BF)
    B, L, hid, ffn, V = 8, 706, 4096, 11008, 32006
    M = B * L
    inv = 1.0 / (10000.0 ** (torch.arange(0, 128, 2, device=dev).float() / 128))
    emb = torch.cat([torch.arange(L, device=dev).float()[:, None] * inv[None]] * 2, -1)
    cos, sin = emb.cos().to(BF).contiguous(), emb.sin().to(BF).contiguous()
    res = rn(M, hid)
    buf = torch.empty(M, 32008, dtype=BF, device=dev)
    ks = (1024, 2048, 4096, 8192, 11008)

    def gemm(N, op):
        def make(K):
            x, w = rn(M, K), rn(N, K, std=0.02)
            return lambda: op(x, w)
        return make
    mt = math.ceil(M / 128)
    out = [('llama qkv+rope 5648x12288', 32, mt, 12288 // BN, ks,
            gemm(3 * hid, lambda x, w: dense.qkv_rope(x, w, cos, sin, L, 2 * hid))),
           ('llama o_proj 5648x4096 +residual', 32, mt, hid // BN, ks,
            gemm(hid, lambda x, w: dense.linear(x, w, residual=res))),
           ('llama gate/up swiglu 5648x22016', 32, mt, 2 * ffn // BN, ks,
            gemm(2 * ffn, lambda x, w: dense.linear(x, w, act='swiglu'))),
           ('llama down 5648x4096 +residual', 32, mt, hid // BN, ks,
            gemm(hid, lambda x, w: dense.linear(x, w, residual=res))),
           ('lm_head 5648x32006', 1, mt, math.ceil(V / BN), ks,
            gemm(V, lambda x, w: dense.linear(x, w, out=buf[:, :V])))]
    S, H = 1024, 192

    def conv(cin):
        xin, wf = rn(B, H, H, cin), rn(S, 3, 3, cin, std=0.01)
        st = torch.zeros(B, dense.gn_slots(H, H), 64, 2, device=dev)
        return lambda: dense.conv_nhwc(xin, wf, gn_stats=st)
    # conv K = 9 * Cin: Cin 128 .. 1024 gives 18 .. 144 k-blocks; 192 px tiles are 16 x 8 pixels
    out.append(('3x3 fuse conv 192px +GN stats', 5, B * (H // 16) * (H // 8), S // BN, (9 * 128, 9 * 256, 9 * 512, 9 * 1024),
                lambda K: conv(K // 9)))
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--min-ms', type=float, default=100.0)
    ap.add_argument('--out', default=None, help='also write the records as JSON to this file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_gemm_ksweep.py needs a CUDA device (an H100): there is no CPU measurement')
    dev = 'cuda:0'
    info = gpu_info()
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    print('# %s, power limit %s W, max SM clock %s MHz, %d SMs, tile 128x%d' % (
        info['name'], info['power_limit_w'], info['sm_max_mhz'], sms, BN))
    prev = os.environ.get('G4R_GEMM_BN')
    os.environ['G4R_GEMM_BN'] = str(BN)
    recs = []
    try:
        for name, per_step, m_tiles, n_tiles, ks, make in shapes(dev):
            rounds = math.ceil(m_tiles * n_tiles / sms)
            pts = []
            sampler = ClockSampler(0)
            sampler.start()
            for K in ks:
                fn = make(K)
                fn()
                torch.cuda.synchronize()
                ms = [time_window(fn, args.min_ms)[0] for _ in range(args.reps)]
                pts.append(dict(K=K, k_blocks=math.ceil(K / 64), ms=statistics.median(ms),
                                spread_ms=max(ms) - min(ms)))
                del fn
                torch.cuda.empty_cache()
            clk = sampler.stop()
            x = np.array([p['k_blocks'] for p in pts], float)
            y = np.array([p['ms'] for p in pts]) * 1e3 / rounds          # us per round
            slope, icpt = np.polyfit(x, y, 1)
            resid = y - (slope * x + icpt)
            rec = dict(shape=name, launches_per_step=per_step, rounds=rounds, sm_mhz=clk.get('sm_mhz'),
                       clock_reasons=clk.get('reasons'), points=pts, slope_us_per_kblock=round(float(slope), 4),
                       intercept_us=round(float(icpt), 3), fit_max_resid_us=round(float(np.abs(resid).max()), 3),
                       intercept_ms_per_step=round(float(icpt) * rounds * per_step / 1e3, 3))
            recs.append(rec)
            print('%-34s rounds %3d  slope %.3f us/k-block  intercept %6.2f us (fit resid <= %.2f)  '
                  'x rounds x %2d launches = %6.2f ms/step  (%s MHz)  per K: %s' % (
                      name, rounds, slope, icpt, rec['fit_max_resid_us'], per_step, rec['intercept_ms_per_step'],
                      rec['sm_mhz'], ' '.join('%d:%.3f' % (p['K'], p['ms']) for p in pts)), flush=True)
    finally:
        if prev is None:
            os.environ.pop('G4R_GEMM_BN', None)
        else:
            os.environ['G4R_GEMM_BN'] = prev
    llama = sum(r['intercept_ms_per_step'] for r in recs if not r['shape'].startswith('3x3'))
    print('# intercept per headline step: LLaMA + lm_head %.2f ms, all shapes %.2f ms' % (
        llama, sum(r['intercept_ms_per_step'] for r in recs)))
    summary = dict(gpu=info, sms=sms, block_n=BN, records=recs, llama_intercept_ms_per_step=round(llama, 3))
    print(json.dumps(summary))
    if args.out:
        with open(args.out, 'w') as fh:
            json.dump(summary, fh, indent=1)


if __name__ == '__main__':
    main()
