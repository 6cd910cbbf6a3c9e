"""Per-shape timing of the wgmma GEMM / implicit-GEMM conv (csrc/gemm_wgmma.cu) at every forward shape of the headline
prefill step (B=8, 336 px, 8 RoIs per image, L=706), at tile width 128, 256 and the automatic choice (G4R_GEMM_BN).

  python tools/bench_gemm.py [--reps 3] [--min-ms 200] [--out FILE.json]

Each (shape, width) window launches the same op back to back on one stream, timed with CUDA events, until it
exceeds --min-ms; the widths alternate inside every repetition and the median over repetitions is reported.
FLOP/s are algorithmic (2*M*N*K; conv: 2*pixels*Cout*taps*Cin*levels).  The share of peak is taken against the
dense bf16 data-sheet rate scaled to the SM clock sampled during that shape's windows: 989 TFLOP/s x clock / 1830
MHz (the H100 SXM boost clock the 989 figure is quoted at).  The card's name, power limit and maximum SM clock are
read in the same run.  Needs a CUDA device; there is no CPU path."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import ClockSampler  # noqa: E402
from gpt4roi_b200 import dense  # noqa: E402

BF = torch.bfloat16
PEAK_TFLOPS, PEAK_MHZ = 989.0, 1830.0
WIDTHS = ('128', '256', 'auto')


def gpu_info():
    q = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm',
                        '--format=csv,noheader,nounits'], capture_output=True, text=True)
    if q.returncode != 0:
        return dict(name=torch.cuda.get_device_name(0), power_limit_w=None, sm_max_mhz=None)
    name, pl, mx = [x.strip() for x in q.stdout.strip().split('\n')[0].split(',')]
    return dict(name=name, power_limit_w=float(pl), sm_max_mhz=int(float(mx)))


def shapes(dev):
    """(name, launches per headline step, flops per launch, fn) for every forward GEMM / conv shape of the step."""
    g = torch.Generator(device=dev).manual_seed(0)

    def rn(*s, std=1.0):
        return (torch.randn(*s, device=dev, generator=g) * std).to(BF)
    B, L, hid, ffn, V = 8, 706, 4096, 11008, 32006
    M = B * L
    out = []
    # ---- LLaMA-7B (32 layers) and lm_head, M = B*L = 5648
    x, res = rn(M, hid), rn(M, hid)
    inv = 1.0 / (10000.0 ** (torch.arange(0, 128, 2, device=dev).float() / 128))
    emb = torch.cat([torch.arange(L, device=dev).float()[:, None] * inv[None]] * 2, -1)
    cos, sin = emb.cos().to(BF).contiguous(), emb.sin().to(BF).contiguous()
    wqkv, wo, wgu, wdn = rn(3 * hid, hid, std=0.02), rn(hid, hid, std=0.02), rn(2 * ffn, hid, std=0.02), rn(hid, ffn, std=0.02)
    f = rn(M, ffn)
    lm = rn(V, hid, std=0.02)
    buf = torch.empty(M, 32008, dtype=BF, device=dev)
    out += [('llama qkv+rope 5648x12288x4096', 32, 2.0 * M * 3 * hid * hid,
             lambda: dense.qkv_rope(x, wqkv, cos, sin, L, 2 * hid)),
            ('llama o_proj 5648x4096x4096', 32, 2.0 * M * hid * hid, lambda: dense.linear(x, wo, residual=res)),
            ('llama gate/up swiglu 5648x22016x4096', 32, 2.0 * M * 2 * ffn * hid,
             lambda: dense.linear(x, wgu, act='swiglu')),
            ('llama down 5648x4096x11008', 32, 2.0 * M * hid * ffn, lambda: dense.linear(f, wdn, residual=res)),
            ('lm_head 5648x32006x4096', 1, 2.0 * M * V * hid, lambda: dense.linear(x, lm, out=buf[:, :V]))]
    # ---- CLIP ViT-L/14 (23 live layers), M = B*577 = 4616; fp32 residual stream
    Mv, C, Fv = B * 577, 1024, 4096
    xv, rv, fv = rn(Mv, C), torch.randn(Mv, C, device=dev, generator=g), rn(Mv, Fv)
    wq, bq, wov, bo = rn(3 * C, C, std=0.02), rn(3 * C), rn(C, C, std=0.02), rn(C)
    w1, b1, w2, b2 = rn(Fv, C, std=0.02), rn(Fv), rn(C, Fv, std=0.02), rn(C)
    f32 = dict(out_dtype=torch.float32, round_branch=True)
    out += [('vit qkv 4616x3072x1024', 23, 2.0 * Mv * 3 * C * C, lambda: dense.linear(xv, wq, bq)),
            ('vit out_proj 4616x1024x1024', 23, 2.0 * Mv * C * C, lambda: dense.linear(xv, wov, bo, residual=rv, **f32)),
            ('vit fc1 4616x4096x1024', 23, 2.0 * Mv * Fv * C, lambda: dense.linear(xv, w1, b1, act='quick_gelu')),
            ('vit fc2 4616x1024x4096', 23, 2.0 * Mv * C * Fv, lambda: dense.linear(fv, w2, b2, residual=rv, **f32))]
    # ---- SPI: 1x1 input convs (a GEMM over the padded 1088 channels), 3x3 fuse convs (5 rounds), 4-level pconv
    S, cpad, R, K = 1024, 1088, 14, B * 8
    win, bin_ = rn(S, cpad, std=0.02), rn(S)
    wf = rn(S, 3, 3, S, std=0.01)
    for H in (192, 96, 48, 24):
        up = rn(B * H * H, cpad)
        out.append(('1x1 input conv %dpx %dx1024x1088' % (H, B * H * H), 1, 2.0 * B * H * H * S * cpad,
                    lambda up=up: dense.linear(up, win, bin_)))
    for H in (192, 96, 48, 24):
        xin = rn(B, H, H, S)
        st = torch.zeros(B, dense.gn_slots(H, H), 64, 2, device=dev)
        out.append(('3x3 fuse conv %dpx (M=%d)' % (H, B * H * H), 5, 2.0 * B * H * H * S * 9 * S,
                    lambda xin=xin, st=st: dense.conv_nhwc(xin, wf, gn_stats=st)))
    feats = rn(4 * K, R, R, S)
    wp = rn(S, 4, 3, 3, S, std=0.01)
    bp = torch.zeros(S, device=dev)
    out.append(('pconv 4-level 3x3 (M=%d)' % (K * R * R), 1, 2.0 * K * R * R * S * 9 * S * 4,
                lambda: dense.conv_nhwc(feats, wp, bp, act='relu', levels=4)))
    return out


def time_window(fn, min_ms):
    """Back-to-back launches until the window exceeds min_ms; returns (ms per launch, launches)."""
    n = 1
    while True:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        e1.synchronize()
        ms = e0.elapsed_time(e1)
        if ms >= min_ms:
            return ms / n, n
        n = max(n + 1, int(n * min_ms * 1.2 / max(ms, 1e-3)))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--min-ms', type=float, default=200.0)
    ap.add_argument('--out', default=None, help='also write the records as JSON to this file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_gemm.py needs a CUDA device (an H100): there is no CPU measurement')
    dev = 'cuda:0'
    info = gpu_info()
    print('# %s, power limit %s W, max SM clock %s MHz' % (info['name'], info['power_limit_w'], info['sm_max_mhz']))
    prev = os.environ.get('G4R_GEMM_BN')
    recs = []
    try:
        for name, per_step, flops, fn in shapes(dev):
            for w in WIDTHS:                       # warm every width (module load, tensor-map encode, attributes)
                os.environ['G4R_GEMM_BN'] = w
                fn()
            torch.cuda.synchronize()
            ms = {w: [] for w in WIDTHS}
            sampler = ClockSampler(0)
            sampler.start()
            for _ in range(args.reps):
                for w in WIDTHS:
                    os.environ['G4R_GEMM_BN'] = w
                    ms[w].append(time_window(fn, args.min_ms)[0])
            clk = sampler.stop()
            mhz = clk.get('sm_mhz')
            peak = PEAK_TFLOPS * mhz / PEAK_MHZ if mhz else None
            rec = dict(shape=name, launches_per_step=per_step, gflop=flops / 1e9, sm_mhz=mhz,
                       clock_reasons=clk.get('reasons'))
            for w in WIDTHS:
                med = statistics.median(ms[w])
                tf = flops / 1e12 / (med / 1e3)
                rec[w] = dict(ms=round(med, 4), spread_ms=round(max(ms[w]) - min(ms[w]), 4), tflops=round(tf, 1),
                              frac_clock_peak=round(tf / peak, 3) if peak else None)
            recs.append(rec)
            print('%-40s  128: %7.3f ms %6.1f TF/s  256: %7.3f ms %6.1f TF/s  auto: %7.3f ms  (%s MHz)' % (
                name, rec['128']['ms'], rec['128']['tflops'], rec['256']['ms'], rec['256']['tflops'],
                rec['auto']['ms'], mhz), flush=True)
    finally:
        if prev is None:
            os.environ.pop('G4R_GEMM_BN', None)
        else:
            os.environ['G4R_GEMM_BN'] = prev
    step = {w: sum(r[w]['ms'] * r['launches_per_step'] for r in recs) for w in WIDTHS}
    print('# per headline step (launches x median ms): ' + ', '.join('%s %.1f ms' % (w, step[w]) for w in WIDTHS))
    summary = dict(gpu=info, records=recs, step_ms=step, peak='%g TFLOP/s x sm_mhz / %g MHz' % (PEAK_TFLOPS, PEAK_MHZ))
    print(json.dumps(summary))
    if args.out:
        with open(args.out, 'w') as fh:
            json.dump(summary, fh, indent=1)


if __name__ == '__main__':
    main()
