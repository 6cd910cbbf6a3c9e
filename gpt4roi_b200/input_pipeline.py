"""GPU input pipeline (SURVEY.md 8(f2)): host-side mirror of the image / box transforms the reference runs per sample on
CPU dataloader workers (gpt4roi/datasets/coco_det.py:60-71,154), backed by ONE kernel for the whole batch's images
(`g4r_preprocess_images`, csrc/input_pipeline.cu).

    Resize((S,S), keep_ratio=False) -> RandomShift(0.5, 32) -> FilterAnnotations((2,2)) -> RandomFlip(0.5) ->
    Normalize(CLIP mean/std, to_rgb) -> Pad -> DefaultFormatBundle ;  boxes / S

The box side (a few boxes per image, float32) stays on the host exactly as the reference computes it -- it also decides
whether RandomShift applies at all (it leaves image AND boxes untouched when no box would survive,
mmdet/datasets/pipelines/transforms.py:541-544) -- the pixels (the 99.9 % of the work) run on the GPU, bit-identical to
cv2.resize + mmcv.imnormalize for fp32 output.  JPEG decoding is not part of this module (feed decoded uint8 BGR arrays,
what mmcv.imread returns; `torchvision.io.decode_jpeg(device='cuda')` gives them without leaving the GPU).
"""
import numpy as np
import torch

from . import lib as _L

CLIP_MEAN = (0.48145466 * 255, 0.4578275 * 255, 0.40821073 * 255)   # coco_det.py:56-58
CLIP_STD = (0.26862954 * 255, 0.26130258 * 255, 0.27577711 * 255)


def draw_augmentation(n, rng=None, shift_ratio=0.5, max_shift_px=32, flip_ratio=0.5):
    """Per-image (shift_x, shift_y) and flip decisions with the reference's distributions (RandomShift draws
    `random.random() < ratio` then two `numpy.random.randint(-max, max)` -- high exclusive -- x first;
    RandomFlip flips with probability flip_ratio).  rng: numpy Generator / RandomState-like with .random() / .integers()."""
    rng = rng or np.random.default_rng()
    shifts, flips = [], []
    for _ in range(n):
        if rng.random() < shift_ratio:
            shifts.append((int(rng.integers(-max_shift_px, max_shift_px)), int(rng.integers(-max_shift_px, max_shift_px))))
        else:
            shifts.append((0, 0))
        flips.append(bool(rng.random() < flip_ratio))
    return shifts, flips


def transform_boxes(boxes, src_h, src_w, S, shift=(0, 0), flip=False, shift_filter_px=1, min_wh=(2.0, 2.0)):
    """Box side of Resize (transforms.py:245-253) -> RandomShift (:527-551) -> FilterAnnotations (loading.py:578-596) ->
    RandomFlip (:388-420) -> / S (coco_det.py:154), float32 like the reference.  Returns (normalised boxes [K',4], indices of
    the kept input boxes, the shift actually applied)."""
    b = np.asarray(boxes, np.float32).reshape(-1, 4)
    idx = np.arange(len(b))
    b = b * np.array([S / src_w, S / src_h, S / src_w, S / src_h], dtype=np.float32)
    b[:, 0::2] = np.clip(b[:, 0::2], 0, S)
    b[:, 1::2] = np.clip(b[:, 1::2], 0, S)
    applied = (0, 0)
    if tuple(shift) != (0, 0):
        sb = b.copy()
        sb[:, 0::2] += shift[0]
        sb[:, 1::2] += shift[1]
        sb[:, 0::2] = np.clip(sb[:, 0::2], 0, S)
        sb[:, 1::2] = np.clip(sb[:, 1::2], 0, S)
        valid = ((sb[:, 2] - sb[:, 0]) > shift_filter_px) & ((sb[:, 3] - sb[:, 1]) > shift_filter_px)
        if valid.any():
            b, idx, applied = sb[valid], idx[valid], (int(shift[0]), int(shift[1]))
    if len(b):
        keep = ((b[:, 2] - b[:, 0]) > min_wh[0]) & ((b[:, 3] - b[:, 1]) > min_wh[1])
        b, idx = b[keep], idx[keep]
    if flip and len(b):
        f = b.copy()
        f[:, 0] = S - b[:, 2]
        f[:, 2] = S - b[:, 0]
        b = f
    return (b / np.float32(S)).astype(np.float32), idx, applied


class BatchPreprocessor:
    """Reusable pinned staging buffer + device buffers for batches of decoded images."""

    def __init__(self, S, device='cuda:0', out_dtype=torch.bfloat16, mean=CLIP_MEAN, std=CLIP_STD, to_rgb=True):
        if out_dtype not in (torch.float32, torch.bfloat16):
            raise TypeError('out_dtype must be float32 or bfloat16')
        self.S, self.dev, self.out_dtype, self.to_rgb = int(S), torch.device(device), out_dtype, bool(to_rgb)
        if self.dev.type != 'cuda':
            raise RuntimeError('gpt4roi_b200.input_pipeline: device %s -- implementation for device %s not found '
                               '(CUDA sm_90a only; no CPU fallback)' % (self.dev, self.dev.type))
        import ctypes
        self._mean = (ctypes.c_float * 3)(*[float(np.float32(m)) for m in mean])   # float32, as mmdet's Normalize stores them
        self._std = (ctypes.c_float * 3)(*[float(np.float32(s)) for s in std])
        self._pinned = None

    def __call__(self, images, boxes=None, shifts=None, flips=None):
        """images: list of uint8 HWC BGR arrays (numpy or CPU tensors) of any sizes; boxes: list of [K_i,4] xyxy in source
        pixels (or None); shifts / flips: per-image decisions (draw_augmentation) or None for the test pipeline.
        Returns (device tensor [B,3,S,S], list of normalised boxes (float32 CPU tensors), list of kept-box indices)."""
        B, S = len(images), self.S
        arrs = [np.ascontiguousarray(im.numpy() if isinstance(im, torch.Tensor) else im) for im in images]
        for a in arrs:
            if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3:
                raise TypeError('images must be uint8 HWC with 3 channels, got %s %s' % (a.dtype, a.shape))
        shifts = [(0, 0)] * B if shifts is None else [tuple(int(v) for v in s) for s in shifts]
        flips = [False] * B if flips is None else [bool(f) for f in flips]
        out_boxes, out_idx = [], []
        if boxes is not None:
            for i, a in enumerate(arrs):
                nb, idx, applied = transform_boxes(boxes[i], a.shape[0], a.shape[1], S, shifts[i], flips[i])
                shifts[i] = applied            # RandomShift is skipped for the image too when no box survives it
                out_boxes.append(torch.from_numpy(nb))
                out_idx.append(idx)
        sizes = [a.size for a in arrs]
        offs = np.zeros(B, np.int64)
        offs[1:] = np.cumsum([(n + 15) // 16 * 16 for n in sizes])[:-1]
        total = int(offs[-1] + (sizes[-1] + 15) // 16 * 16)
        if self._pinned is None or self._pinned.numel() < total:
            self._pinned = torch.empty(max(total, 1 << 20), dtype=torch.uint8).pin_memory()
        host = self._pinned.numpy()
        for a, o, n in zip(arrs, offs, sizes):
            host[o:o + n] = a.reshape(-1)
        meta = torch.tensor([[a.shape[0], a.shape[1], s[0], s[1], int(f)] for a, s, f in zip(arrs, shifts, flips)],
                            dtype=torch.int32)
        d_src = self._pinned[:total].to(self.dev, non_blocking=True)
        d_offs = torch.from_numpy(offs).to(self.dev, non_blocking=True)
        d_meta = meta.to(self.dev, non_blocking=True)
        d_hw, d_shift, d_flip = d_meta[:, 0:2].contiguous(), d_meta[:, 2:4].contiguous(), d_meta[:, 4].contiguous()
        out = torch.empty((B, 3, S, S), dtype=self.out_dtype, device=self.dev)
        with torch.cuda.device(self.dev):
            _L.check(_L.load().g4r_preprocess_images(
                _L.ptr(d_src), _L.ptr(d_offs), _L.ptr(d_hw), _L.ptr(d_shift), _L.ptr(d_flip), _L.ptr(out), B, S,
                self._mean, self._std, int(self.to_rgb), _L.dtype_code(out), _L.stream_ptr(self.dev)))
        return out, out_boxes, out_idx
