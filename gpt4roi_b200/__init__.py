"""gpt4roi_b200 -- H100 (sm_90a) implementation of GPT4RoI's region-token forward path.

Host code is Python/PyTorch (device memory, streams, torch.distributed plumbing); the
compute is hand-written CUDA behind the C ABI in include/gpt4roi_b200.h
(libgpt4roi_b200.so, built in-tree by `python -m gpt4roi_b200.build`).
Importing this package does not load the library; the first call does, and raises if it
is missing -- there is no CPU / eager fallback.
"""
__version__ = '0.1.0'

from . import lib  # noqa: F401
from .roi_align import (RoIAlign, RoIAlignFunction, roi_align, roi_align_backward,  # noqa: F401
                        roi_align_forward, roi_align_mlvl, roi_align_mlvl_backward)
