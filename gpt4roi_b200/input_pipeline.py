"""GPU input pipeline (SURVEY.md 8(f2)) for both ways the reference prepares images.

`BatchPreprocessor`: host-side mirror of the image / box transforms the reference runs per sample on CPU dataloader
workers for the mmdet datasets (gpt4roi/datasets/coco_det.py:60-71,154), backed by ONE kernel for the whole batch's
images (`g4r_preprocess_images`, csrc/input_pipeline.cu).

    Resize((S,S), keep_ratio=False) -> RandomShift(0.5, 32) -> FilterAnnotations((2,2)) -> RandomFlip(0.5) ->
    Normalize(CLIP mean/std, to_rgb) -> Pad -> DefaultFormatBundle ;  boxes / S

The box side (a few boxes per image, float32) stays on the host exactly as the reference computes it -- it also decides
whether RandomShift applies at all (it leaves image AND boxes untouched when no box would survive,
mmdet/datasets/pipelines/transforms.py:541-544) -- the pixels (the 99.9 % of the work) run on the GPU, bit-identical to
cv2.resize + mmcv.imnormalize for fp32 output.  JPEG decoding is not part of this module (feed decoded uint8 BGR arrays,
what mmcv.imread returns; `torchvision.io.decode_jpeg(device='cuda')` gives them without leaving the GPU).

`ClipPreprocessor`: the CLIPImageProcessor path of the demo and of the VCR / LLaVA-instruct datasets
(gpt4roi/app.py:118-136, gpt4roi/datasets/vcr.py:173-189, gpt4roi/datasets/det_llava.py:347-389),

    CLIPImageProcessor.preprocess(image, do_center_crop=False) -> F.interpolate((S, S), 'bilinear') ;  boxes / [w,h,w,h]

backed by two launches for the whole batch (`g4r_clip_preprocess`, csrc/clip_preprocess.cu), bit-identical to that path
for fp32 output.  The host computes each image's tap windows and weights (cached per image size); the pixels run on
the GPU.
"""
import ctypes
import functools
import math

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


CLIP_IMAGE_MEAN = (0.48145466, 0.4578275, 0.40821073)   # transformers OPENAI_CLIP_MEAN / OPENAI_CLIP_STD
CLIP_IMAGE_STD = (0.26862954, 0.26130258, 0.27577711)
_CLIP_BITS = 22          # fixed-point fraction bits of the resize weights
_CLIP_META = 13          # int64 fields per image, csrc/clip_preprocess.cu: M_SRC .. M_BX


def clip_resized_size(h, w, shortest_edge=224):
    """(H', W') of CLIPImageProcessor's shortest_edge resize: the short side becomes `shortest_edge`, the long side
    int(shortest_edge * long / short) in Python float (transformers get_resize_output_image_size)."""
    short, long = (w, h) if w <= h else (h, w)
    new_long = int(shortest_edge * long / short)
    return (new_long, shortest_edge) if w <= h else (shortest_edge, new_long)


def normalize_boxes(boxes, h, w):
    """xyxy boxes in source pixels -> boxes / [w, h, w, h] in float64, then float32 (gpt4roi/datasets/vcr.py:179,
    gpt4roi/app.py:121)."""
    b = np.asarray(boxes.cpu() if isinstance(boxes, torch.Tensor) else boxes, np.float64).reshape(-1, 4)
    return (b / np.array([w, h, w, h], np.float64)).astype(np.float32)


def _bicubic_taps(in_size, out_size, outs):
    """PIL's BICUBIC (a = -0.5) resample of one axis, for the output indices `outs` only: (first tap [n], tap count [n],
    22-bit fixed-point weights [n, ksize] int32).  The weights are computed in double in PIL's order -- window
    trunc(center -+ support + 0.5) clipped to the axis, cubic((i - center + 0.5) / filterscale), divided by their
    left-to-right sum -- then rounded half away from zero.  An unchanged axis is the identity, as PIL skips that pass."""
    if in_size == out_size:
        return outs, np.ones(len(outs), np.int64), np.full((len(outs), 1), 1 << _CLIP_BITS, np.int32)
    scale = float(in_size) / out_size
    fs = max(scale, 1.0)
    support = 2.0 * fs
    ksize = int(math.ceil(support)) * 2 + 1
    center = (outs.astype(np.float64) + 0.5) * scale
    lo = np.maximum(np.trunc(center - support + 0.5), 0).astype(np.int64)
    cnt = np.minimum(np.trunc(center + support + 0.5), in_size).astype(np.int64) - lo
    t = np.arange(ksize)
    x = np.abs(((lo[:, None] + t[None, :]) - center[:, None] + 0.5) * (1.0 / fs))
    w = np.where(x < 1.0, (1.5 * x - 2.5) * x * x + 1, np.where(x < 2.0, (((x - 5) * x + 8) * x - 4) * -0.5, 0.0))
    w = np.where(t[None, :] < cnt[:, None], w, 0.0)
    ww = np.zeros(len(outs))
    for j in range(ksize):
        ww = ww + w[:, j]
    w = np.where(ww[:, None] != 0.0, w / np.where(ww == 0.0, 1.0, ww)[:, None], w)
    f = w * float(1 << _CLIP_BITS)
    return lo, cnt, np.trunc(np.where(w < 0, f - 0.5, f + 0.5)).astype(np.int32)


def _bilinear_axis(in_size, out_size):
    """torch's CPU upsample_bilinear2d indices and float32 lambdas (align_corners=False, no scale factor): i0, i1, l0,
    l1.  The source coordinate is fma(float32(in) / out, o + 0.5, -0.5) as torch's vectorised builds compute it: the
    product is exact in double, and so is the sum whenever it is >= 0 (a negative one clamps to 0 either way), so one
    rounding to float32 is the FMA's."""
    o = np.arange(out_size)
    if in_size == out_size:
        return o, o, np.ones(out_size, np.float32), np.zeros(out_size, np.float32)
    scale = np.float64(np.float32(in_size) / np.float32(out_size))
    src = np.maximum((scale * (o + 0.5) - 0.5).astype(np.float32), np.float32(0))
    i0 = np.minimum(np.floor(src).astype(np.int64), in_size - 1)
    l1 = np.clip(src - i0.astype(np.float32), np.float32(0), np.float32(1)).astype(np.float32)
    return i0, i0 + (i0 < in_size - 1), (np.float32(1) - l1).astype(np.float32), l1


@functools.lru_cache(maxsize=256)
def _clip_plan(h, w, S, shortest_edge):
    """Per image size: the int32 tables csrc/clip_preprocess.cu reads (list | e1 | e2 | by | bx) and (vfirst, nr, nc,
    k1, k2, offsets of e1, e2, by, bx).  Only the resized rows / columns the bilinear reads get taps; the first pass
    resamples only the source rows (horizontal first) or columns (vertical first) their windows cover."""
    H, W = clip_resized_size(h, w, shortest_edge)
    y0, y1, ly0, ly1 = _bilinear_axis(H, S)
    x0, x1, lx0, lx1 = _bilinear_axis(W, S)
    ury, urx = np.unique(np.concatenate([y0, y1])), np.unique(np.concatenate([x0, x1]))
    vert, horz = _bicubic_taps(h, H, ury), _bicubic_taps(w, W, urx)
    vfirst = h > 100 * w and H < h         # PIL's Image.resize: vertical pass first for such tall images
    (lo1, cnt1, k1), (lo2, cnt2, k2), n_in = (vert, horz, w) if vfirst else (horz, vert, h)
    mark = np.zeros(n_in + 1, np.int64)
    np.add.at(mark, lo2, 1)
    np.add.at(mark, lo2 + cnt2, -1)
    lst = np.flatnonzero(np.cumsum(mark)[:n_in] > 0)   # source lines the second pass's windows cover
    e1 = np.concatenate([lo1[:, None], cnt1[:, None], k1], 1)
    e2 = np.concatenate([np.searchsorted(lst, lo2)[:, None], cnt2[:, None], k2], 1)
    nr, nc = (len(ury), len(lst)) if vfirst else (len(lst), len(urx))
    by = np.stack([np.searchsorted(ury, y0), np.searchsorted(ury, y1), ly0.view(np.int32), ly1.view(np.int32)], 1)
    bx = np.stack([np.searchsorted(urx, x0), np.searchsorted(urx, x1), lx0.view(np.int32), lx1.view(np.int32)], 1)
    parts = [lst, e1.ravel(), e2.ravel(), by.ravel(), bx.ravel()]
    offs = np.cumsum([0] + [len(p) for p in parts])
    tables = np.concatenate(parts).astype(np.int32)
    tables.flags.writeable = False
    return tables, (int(vfirst), nr, nc, k1.shape[1], k2.shape[1]) + tuple(int(v) for v in offs[1:5])


def _align16(n):
    return (n + 15) // 16 * 16


class ClipPreprocessor:
    """GPU replacement of the demo's and the VCR / LLaVA-instruct datasets' image preparation:
    `CLIPImageProcessor.preprocess(image, do_center_crop=False)` (the PIL processor: shortest_edge BICUBIC resize,
    rescale, normalise) followed by `F.interpolate(..., (S, S), mode='bilinear', align_corners=False)`, for a batch
    of images of any sizes in two launches.  fp32 output is bit-identical to that CPU path; bf16 / fp16 output is
    its `.to(dtype)`.  No CPU fallback."""

    def __init__(self, S=224, shortest_edge=224, device='cuda:0', out_dtype=torch.bfloat16, mean=CLIP_IMAGE_MEAN,
                 std=CLIP_IMAGE_STD):
        if out_dtype not in (torch.float32, torch.bfloat16, torch.float16):
            raise TypeError('out_dtype must be float32, bfloat16 or float16')
        self.S, self.shortest_edge, self.out_dtype = int(S), int(shortest_edge), out_dtype
        if not (0 < self.S <= 4096 and 0 < self.shortest_edge <= 4096):
            raise ValueError('S and shortest_edge must lie in 1..4096, got %d, %d' % (self.S, self.shortest_edge))
        self.dev = torch.device(device)
        if self.dev.type != 'cuda':
            raise RuntimeError('gpt4roi_b200.input_pipeline: device %s -- implementation for device %s not found '
                               '(CUDA sm_90a only; no CPU fallback)' % (self.dev, self.dev.type))
        if self.dev.index is None:
            self.dev = torch.device('cuda', torch.cuda.current_device())
        self._mean = (ctypes.c_float * 3)(*[float(np.float32(m)) for m in mean])   # float32, as the processor's
        self._std = (ctypes.c_float * 3)(*[float(np.float32(s)) for s in std])
        self._pinned = None
        self._staged = None      # event after the last copy out of the pinned buffer

    def _source(self, im):
        """uint8 HWC RGB image -> (numpy array, None) for host data or (None, contiguous device tensor)."""
        if isinstance(im, torch.Tensor):
            if im.is_cuda:
                if im.device != self.dev:
                    raise RuntimeError('image on %s, preprocessor on %s' % (im.device, self.dev))
                a, shape, dtype = None, tuple(im.shape), im.dtype
            else:
                a = im.numpy()
        elif hasattr(im, 'mode') and hasattr(im, 'size') and not isinstance(im, np.ndarray):
            if im.mode != 'RGB':
                raise TypeError('PIL images must be mode RGB, got %s' % im.mode)
            a = np.asarray(im)
        else:
            a = np.asarray(im)
        if a is not None:
            shape, dtype = a.shape, a.dtype
        if dtype not in (np.uint8, torch.uint8) or len(shape) != 3 or shape[2] != 3:
            raise TypeError('images must be uint8 HWC with 3 channels, got %s %s' % (dtype, tuple(shape)))
        if shape[0] < 1 or shape[1] < 1:
            raise ValueError('empty image %s' % (tuple(shape),))
        if a is None:
            return None, im.contiguous()
        return np.ascontiguousarray(a), None

    def __call__(self, images, boxes=None):
        """images: list of uint8 HWC RGB images of any sizes -- numpy arrays, CPU or CUDA uint8 tensors, PIL images;
        boxes: list of [K_i, 4] xyxy boxes in source pixels, or None.  Returns (device tensor [B, 3, S, S] of
        out_dtype, list of float32 CPU tensors boxes / [w, h, w, h] (empty when boxes is None))."""
        B, S = len(images), self.S
        if not 0 < B <= 65535:
            raise ValueError('need 1..65535 images, got %d' % B)
        if boxes is not None and len(boxes) != B:
            raise ValueError('%d box lists for %d images' % (len(boxes), B))
        srcs = [self._source(im) for im in images]
        hw = [(a if a is not None else t).shape[:2] for a, t in srcs]
        plans = [_clip_plan(int(h), int(w), S, self.shortest_edge) for h, w in hw]
        out_boxes = [] if boxes is None else [torch.from_numpy(normalize_boxes(bx, h, w)) for bx, (h, w) in zip(boxes, hw)]
        # one pinned staging area: host images | tables (int32) | meta (int64); one copy to the device
        img_off, n = [], 0
        for a, _ in srcs:
            img_off.append(n)
            n += _align16(a.size) if a is not None else 0
        tab_base, n = n, n + _align16(sum(p[0].nbytes for p in plans))
        meta_base, total = n, n + B * _CLIP_META * 8
        if self._staged is not None:
            self._staged.synchronize()       # the previous call's copy out of the pinned buffer has finished
        if self._pinned is None or self._pinned.numel() < total:
            self._pinned = torch.empty(max(total, 1 << 20), dtype=torch.uint8).pin_memory()
        host = self._pinned.numpy()
        d_buf = torch.empty(total, dtype=torch.uint8, device=self.dev)
        base = d_buf.data_ptr()
        meta = np.zeros((B, _CLIP_META), np.int64)
        tab = host[tab_base:meta_base].view(np.int32)
        t_at, tmp_at, max_work = 0, 0, 0
        for b, ((a, t), (h, w), (tables, (vf, nr, nc, k1, k2, o1, o2, oy, ox))) in enumerate(zip(srcs, hw, plans)):
            if a is not None:
                host[img_off[b]:img_off[b] + a.size] = a.reshape(-1)
            tab[t_at:t_at + len(tables)] = tables
            meta[b] = (base + img_off[b] if a is not None else t.data_ptr(), w, vf, tmp_at, nr, nc, t_at, t_at + o1,
                       k1, t_at + o2, k2, t_at + oy, t_at + ox)
            t_at += len(tables)
            tmp_at += _align16(nr * nc * 3)
            max_work = max(max_work, nr * nc)
        if max_work > 2 ** 31 - 256:
            raise ValueError('image too large for the resize pass: %d source pixels to resample' % max_work)
        host[meta_base:total] = meta.reshape(-1).view(np.uint8)
        d_buf.copy_(self._pinned[:total], non_blocking=True)
        self._staged = torch.cuda.Event()
        self._staged.record(torch.cuda.current_stream(self.dev))
        tmp = torch.empty(max(tmp_at, 16), dtype=torch.uint8, device=self.dev)
        out = torch.empty((B, 3, S, S), dtype=self.out_dtype, device=self.dev)
        with torch.cuda.device(self.dev):
            _L.check(_L.load().g4r_clip_preprocess(
                ctypes.c_void_p(base + meta_base), ctypes.c_void_p(base + tab_base), _L.ptr(tmp), _L.ptr(out), B, S,
                max_work, self._mean, self._std, _L.dtype_code(out), _L.stream_ptr(self.dev)), launches=2)
        return out, out_boxes
