"""Run the conv weight-gradient GEMM and one skinny decode GEMM at 7B / fuse-stack shapes -- meant to be wrapped by ncu:
  ncu --set full --clock-control none -k regex:"gemm_bf16_wgmma|gemm_skinny" -c 4 -o out python tools/profile_train_kernels.py"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gpt4roi_b200 import dense, train_ops  # noqa: E402

DEV = 'cuda:0'
BF = torch.bfloat16


def main():
    torch.manual_seed(0)
    # fuse-stack level 1 at 336 px, per-GPU batch 4: [4, 96, 96, 1024]
    x = (torch.randn(4, 96, 96, 1024, device=DEV) * 0.5).to(BF)
    dz = (torch.randn(4, 96, 96, 1024, device=DEV) * 0.1).to(BF)
    w = (torch.randn(1024, 3, 3, 1024, device=DEV) * 0.02).to(BF)
    for _ in range(2):
        train_ops.conv3x3_bwd(x, w, dz, need_dx=False)            # 1 wgmma GEMM launch each (b_mn == 2)
    # decode gate/up projection at batch 8
    h = (torch.randn(8, 4096, device=DEV) * 0.5).to(BF)
    wgu = (torch.randn(22016, 4096, device=DEV) * 0.02).to(BF)
    for _ in range(2):
        dense.linear(h, wgu, act='swiglu')
    torch.cuda.synchronize()


if __name__ == '__main__':
    main()
