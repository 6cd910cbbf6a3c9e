"""CLIPImageProcessor image path (gpt4roi/app.py:118-136, gpt4roi/datasets/vcr.py:173-189): the reference's host path --
transformers' PIL CLIPImageProcessor(do_center_crop=False) + F.interpolate((224, 224), 'bilinear') per image on the CPU
-- against ClipPreprocessor (csrc/clip_preprocess.cu), on seeded 640x480 and 1920x1080 RGB images at batch 1 (a demo
request) and 16 (a training step).  GPU figures:
  kernels_ms   CUDA time of the two kernels per batch (torch.profiler, device sources)
  call_dev_ms  one ClipPreprocessor call on device uint8 sources (host tables + their copy + kernels), synchronised
  call_host_ms the same on host numpy sources (pinned staging and the host-to-device copy of the pixels included)
The card's name and power limit and the host CPU model are read in the same run.
usage: python tools/bench_clip_preprocess.py [--out FILE]   (prints one JSON line per workload, then a summary)"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gpt4roi_b200.input_pipeline import ClipPreprocessor  # noqa: E402

DEV = 'cuda:0'


def _cpu_model():
    try:
        for line in open('/proc/cpuinfo'):
            if line.startswith('model name'):
                return line.split(':', 1)[1].strip()
    except OSError:
        pass
    return 'not measured'


def _card():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30)
        name, power = [v.strip() for v in r.stdout.strip().split(',')[:2]]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), 'not measured'


def _reference_ms(imgs, reps):
    """Host ms per image of CLIPImageProcessorPil().preprocess(do_center_crop=False) + F.interpolate, or None."""
    try:
        from PIL import Image
        from transformers.models.clip.image_processing_pil_clip import CLIPImageProcessorPil
    except ImportError:
        return None
    proc = CLIPImageProcessorPil()

    def one(im):
        pv = proc.preprocess(Image.fromarray(im), do_center_crop=False, return_tensors='pt')['pixel_values'][0]
        return F.interpolate(pv.unsqueeze(0), size=(224, 224), mode='bilinear', align_corners=False).squeeze(0).half()

    for im in imgs[:3]:
        one(im)
    t0 = time.perf_counter()
    n = 0
    for _ in range(reps):
        for im in imgs:
            one(im)
            n += 1
    return (time.perf_counter() - t0) / n * 1e3


def _call_ms(pre, srcs, reps):
    for _ in range(3):
        pre(srcs)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        pre(srcs)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps * 1e3


def _kernels_ms(pre, srcs, reps):
    from torch.profiler import ProfilerActivity, profile
    pre(srcs)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            pre(srcs)
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if 'clip_resize_' in e.key)
    return us / reps / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--ref-reps', type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_clip_preprocess needs a CUDA device'
    card, power = _card()
    cpu = _cpu_model()
    rows = []
    for (h, w) in ((480, 640), (1080, 1920)):
        for B in (1, 16):
            rng = np.random.default_rng(h + B)
            imgs = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for _ in range(B)]
            pre = ClipPreprocessor(224, device=DEV, out_dtype=torch.float16)
            dev = [torch.from_numpy(im).to(DEV) for im in imgs]
            reps = 200 if B == 1 else 50
            ref = _reference_ms(imgs, max(1, args.ref_reps if B == 16 else 20 * args.ref_reps))
            row = dict(image='%dx%d' % (w, h), batch=B,
                       ref_host_ms_per_image=None if ref is None else round(ref, 3),
                       call_host_ms=round(_call_ms(pre, imgs, reps), 4),
                       call_dev_ms=round(_call_ms(pre, dev, reps), 4),
                       kernels_ms=round(_kernels_ms(pre, dev, reps), 4))
            row['call_host_ms_per_image'] = round(row['call_host_ms'] / B, 4)
            if ref is None:
                row['ref_host_ms_per_image'] = 'not measured'
            print(json.dumps(row), flush=True)
            rows.append(row)
    summary = dict(gpu=card, power_limit=power, cpu=cpu, cpu_threads=torch.get_num_threads(), rows=rows)
    print(json.dumps(summary))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(summary, f, indent=1)


if __name__ == '__main__':
    main()
