"""RoIAlign microbench (BASELINE config 5): N_maps x 100 RoIs, 4 levels x 1024 ch.
Prints one JSON object per variant; run on the GPU box:  python tools/bench_roialign.py [--maps 256]
Compares the sm_90a kernels with the reference CUDA kernel compiled unmodified for sm_90a
(oracle/_ref/_mmcv_ref_cuda_ext.so, 4 launches on NCHW fp32) and torchvision's CUDA roi_align."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import gpt4roi_b200 as g  # noqa: E402
from tests.helpers import PYRAMID, SCALES, make_rois  # noqa: E402


def peak_hbm():
    from bench import peaks   # MEASURED_PEAKS.json when present, else the H100 SXM data sheet
    p, how = peaks()
    return p['hbm_gbs'], how


def time_fn(fn, iters, flush=None):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        if flush is not None:
            flush.add_(1)  # > L2 sized write between iterations
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    return float(np.median(ts)), float(np.min(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--maps', type=int, default=256)
    ap.add_argument('--rois', type=int, default=100)
    ap.add_argument('--size', type=int, default=224)
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--variants', default='all', help="'all', 'nhwc' (skip the NCHW comparisons) or 'headline' (fp32 7x7 only)")
    a = ap.parse_args()
    dev = 'cuda:0'
    C = 1024
    rng = np.random.default_rng(0)
    rois = torch.from_numpy(make_rois(rng, a.maps, a.rois, a.size)).to(dev)
    K = rois.shape[0]
    peak, how = peak_hbm()
    flush = torch.zeros(256 * 1024 * 1024 // 4, device=dev)  # 256 MiB > 126 MB L2
    hs = PYRAMID[a.size]
    px = sum(h * h for h in hs)
    results = []

    def report(name, ms, in_b, out_b, note=''):
        alg = in_b + out_b + K * 20
        r = dict(variant=name, ms_median=ms[0], ms_min=ms[1], algorithmic_GB=alg / 1e9,
                 achieved_GBps=alg / 1e9 / (ms[0] / 1e3), peak_GBps=peak, peak_kind=how,
                 frac=alg / 1e9 / (ms[0] / 1e3) / peak, maps=a.maps, rois=K, size=a.size, note=note)
        results.append(r)
        print(json.dumps(r), flush=True)

    for dt, dname, esz in ((torch.float32, 'fp32', 4), (torch.bfloat16, 'bf16', 2)):
        if a.variants == 'headline' and dname != 'fp32':
            continue
        maps = [torch.randn(a.maps, h, h, C, device=dev, dtype=dt) for h in hs]
        in_b = a.maps * px * C * esz
        for ph in ((7,) if a.variants == 'headline' else (7, 14)):
            out_b = 4 * K * ph * ph * C * esz
            free = torch.cuda.mem_get_info()[0]
            if out_b > free * 0.9:
                print(json.dumps(dict(variant='b200_nhwc_mlvl_%s_p%d' % (dname, ph), skipped='out of memory budget')))
                continue
            out = torch.empty((4, K, ph, ph, C), device=dev, dtype=dt)
            fn = lambda: g.roi_align_mlvl(maps, rois, ph, SCALES, 2, out=out)
            report('b200_nhwc_mlvl_%s_p%d' % (dname, ph), time_fn(fn, a.iters, flush), in_b, out_b)
            del out
        del maps
        torch.cuda.empty_cache()

    if a.variants in ('nhwc', 'headline'):
        return
    # NCHW fp32 comparisons: drop-in kernel, reference CUDA kernel (sm_90a build), torchvision
    nm = min(a.maps, 64)  # NCHW copies; keep memory bounded
    sub = rois[rois[:, 0] < nm].contiguous()
    Ks = sub.shape[0]
    mapsn = [torch.randn(nm, C, h, h, device=dev) for h in hs]
    in_b = nm * px * C * 4
    out_b = 4 * Ks * 49 * C * 4
    outs = [torch.zeros(Ks, C, 7, 7, device=dev) for _ in hs]
    e0 = torch.zeros(0, device=dev)

    def scale_report(name, ms):
        alg = in_b + out_b + Ks * 20
        r = dict(variant=name, ms_median=ms[0], ms_min=ms[1], algorithmic_GB=alg / 1e9,
                 achieved_GBps=alg / 1e9 / (ms[0] / 1e3), peak_GBps=peak, peak_kind=how,
                 frac=alg / 1e9 / (ms[0] / 1e3) / peak, maps=nm, rois=Ks, size=a.size)
        print(json.dumps(r), flush=True)
        results.append(r)

    def ours():
        for l in range(4):
            g.roi_align_forward(mapsn[l], sub, outs[l], e0, e0, 7, 7, SCALES[l], 2, 1, True)
    scale_report('b200_nchw_dropin_fp32_p7', time_fn(ours, a.iters, flush))

    def ours_direct():   # the plane-gather kernel the fast path replaces (no workspace)
        from gpt4roi_b200 import lib as L
        for l in range(4):
            L.check(L.load().g4r_roi_align_forward(L.ptr(mapsn[l]), L.ptr(sub), L.ptr(outs[l]), None, None, nm, C, hs[l], hs[l],
                                                   Ks, 7, 7, SCALES[l], 2, 1, 1, L.F32, L.NCHW, L.stream_ptr(torch.device(dev))))
    scale_report('b200_nchw_direct_kernel_fp32_p7', time_fn(ours_direct, a.iters, flush))
    try:
        from oracle import build_ref
        ref = build_ref.load_cuda()
    except Exception as ex:
        ref = None
        print(json.dumps(dict(variant='reference_cuda_sm100a', skipped=str(ex))))
    if ref is not None:
        def reff():
            for l in range(4):
                ref.roi_align_forward(mapsn[l], sub, outs[l], e0, e0, aligned_height=7, aligned_width=7,
                                      spatial_scale=SCALES[l], sampling_ratio=2, pool_mode=1, aligned=True)
        scale_report('reference_cuda_kernel_sm100a_nchw_fp32_p7', time_fn(reff, a.iters, flush))
    try:
        import torchvision
        def tv():
            for l in range(4):
                torchvision.ops.roi_align(mapsn[l], sub, (7, 7), SCALES[l], 2, True)
        scale_report('torchvision_cuda_nchw_fp32_p7', time_fn(tv, a.iters, flush))
    except Exception as ex:
        print(json.dumps(dict(variant='torchvision', skipped=str(ex))))
    out_dir = os.path.join(ROOT, 'bench_out')
    os.makedirs(out_dir, exist_ok=True)
    json.dump(results, open(os.path.join(out_dir, 'roialign_microbench.json'), 'w'), indent=1)


if __name__ == '__main__':
    main()
