"""GPU comparison point (SURVEY.md 8(d) / BASELINE.md 3): the reference composition run with stock
PyTorch + transformers kernels (cuBLAS / cuDNN / eager attention, bf16 autocast) on the SAME GPU and
the SAME workload as bench.py (configs[1]: B=8, 336 px, 8 RoIs, L=706, 7B).  Test/measurement
infrastructure only (uses oracle/model_oracle.py); prints one JSON line.
"""
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import WORKLOAD, synthetic_inputs  # noqa: E402
from gpt4roi_b200.engine import EngineConfig, random_state_dicts  # noqa: E402
from oracle import model_oracle  # noqa: E402


def main():
    dev = 'cuda:0'
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    cfg = EngineConfig(image_size=WORKLOAD['image_size'])
    sd, vit_sd = random_state_dicts(cfg, dev, seed=0)
    vit = model_oracle.build_vit(cfg, vit_sd, dev, torch.bfloat16)
    llm = model_oracle.build_llm(cfg, sd, dev, torch.bfloat16)
    ids, images, boxes = synthetic_inputs(cfg, WORKLOAD['batch_per_gpu'], WORKLOAD['rois_per_image'], WORKLOAD['text_tokens'])
    ids, images = ids.to(dev), images.to(dev)
    for _ in range(2):
        model_oracle.forward(cfg, sd, vit_sd, ids, images, boxes, dev, autocast_bf16=True, vit=vit, llm=llm)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        model_oracle.forward(cfg, sd, vit_sd, ids, images, boxes, dev, autocast_bf16=True, vit=vit, llm=llm)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    print(json.dumps(dict(what='reference composition, PyTorch eager + transformers %s, bf16 autocast, same GPU' %
                          __import__('transformers').__version__, ms_per_step=ms,
                          samples_per_s=WORKLOAD['batch_per_gpu'] / (ms / 1e3), steps=steps,
                          workload='configs[1]: B=8, 336px, 8 RoIs, L=%d, 7B, full logits' % ids.shape[1])))


if __name__ == '__main__':
    main()
