"""oracle/clip_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

numpy restatement of the CLIPImageProcessor image path of the demo and of the VCR / LLaVA-instruct datasets
(gpt4roi/app.py:118-136, gpt4roi/datasets/vcr.py:173-189, gpt4roi/datasets/det_llava.py:347-389):

    CLIPImageProcessor.preprocess(image, do_center_crop=False)   (the PIL processor: transformers' CLIPImageProcessorPil)
      1. size    : short side -> shortest_edge, long side -> int(shortest_edge * long / short) (Python float)
      2. resize  : PIL Image.resize((W', H'), BICUBIC) -- separable, antialiased, fixed point
      3. rescale : float32(u8 * (1 / 255) in float64); normalise: (x - mean32) / std32 in float32
    F.interpolate(x[None], (S, S), mode='bilinear', align_corners=False)   (torch's CPU kernel, fp32)
    boxes / [w, h, w, h] in float64, then float32

Step 2, written from the algorithm (a separable convolution with a stretched cubic kernel, evaluated in double and
rounded to 22-bit fixed point):
    scale = in / out;  fs = max(scale, 1);  support = 2 * fs;  ksize = 2 * ceil(support) + 1
    per output index o: center = (o + 0.5) * scale;  lo = max(trunc(center - support + 0.5), 0);
                        hi = min(trunc(center + support + 0.5), in);  taps i = lo .. hi-1
                        w_i = cubic((i - center + 0.5) / fs) with a = -0.5, summed left to right into ww, w_i /= ww
                        fixed point k_i = trunc(w_i * 2^22 +- 0.5) (half away from zero)
    a pass: acc = 2^21 + sum_i u8[i] * k_i (int32), out = clamp(acc >> 22, 0, 255); horizontal pass first, into uint8,
    except that Image.resize runs the vertical pass first for an image taller than 100 x its width that shrinks in
    height; an axis whose size does not change is not resampled
Step 4, torch's upsample_bilinear2d on the CPU for a float32 NCHW tensor with C = 3 (the generic separable-index kernel):
    scale = float32(in) / out;  src = max(fma(scale, o + 0.5, -0.5), 0)   (float32; the vector builds contract the FMA)
    i0 = min(floor(src), in - 1); l1 = clamp(src - i0, 0, 1); l0 = 1 - l1; i1 = i0 + (i0 < in - 1)
    identity when in == out (l0 = 1, l1 = 0)
    t_r = fma(v[r, i0x], l0x, v[r, i1x] * l1x) per source row; out = fma(t_0, l0y, t_1 * l1y)
Pinned by tests/test_clip_preprocess_cpu.py to PIL, CLIPImageProcessorPil and F.interpolate themselves.
"""
import math

import numpy as np

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)    # OPENAI_CLIP_MEAN / _STD
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)
PRECISION_BITS = 22


def resized_size(h, w, shortest_edge=224):
    """(H', W') of the processor's shortest_edge rule (transformers get_resize_output_image_size, default_to_square=False)."""
    short, long = (w, h) if w <= h else (h, w)
    new_short, new_long = shortest_edge, int(shortest_edge * long / short)
    return (new_long, new_short) if w <= h else (new_short, new_long)


def _cubic(x):
    x = np.abs(x)
    a = -0.5
    near = ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    far = (((x - 5) * x + 8) * x - 4) * a
    return np.where(x < 1.0, near, np.where(x < 2.0, far, 0.0))


def bicubic_taps(in_size, out_size, outs=None):
    """Fixed-point tap windows of the output indices `outs` (default: all): (lo [n], count [n], k [n, ksize] int32)."""
    outs = np.arange(out_size) if outs is None else np.asarray(outs)
    scale = float(in_size) / out_size
    fs = max(scale, 1.0)
    support = 2.0 * fs
    ksize = int(math.ceil(support)) * 2 + 1
    center = (outs.astype(np.float64) + 0.5) * scale
    lo = np.maximum(np.trunc(center - support + 0.5), 0).astype(np.int64)
    hi = np.minimum(np.trunc(center + support + 0.5), in_size).astype(np.int64)
    cnt = hi - lo
    t = np.arange(ksize)
    live = t[None, :] < cnt[:, None]
    w = np.where(live, _cubic(((lo[:, None] + t[None, :]) - center[:, None] + 0.5) * (1.0 / fs)), 0.0)
    ww = np.zeros(len(outs))
    for j in range(ksize):                      # left to right, as the weights are summed
        ww = ww + w[:, j]
    w = np.where(ww[:, None] != 0.0, w / np.where(ww == 0.0, 1.0, ww)[:, None], w)
    f = w * float(1 << PRECISION_BITS)
    k = np.trunc(np.where(w < 0, f - 0.5, f + 0.5)).astype(np.int32)
    return lo, cnt, k


def _pass(x, in_size, out_size, axis):
    lo, cnt, k = bicubic_taps(in_size, out_size)
    x = np.moveaxis(x.astype(np.int64), axis, 0)
    acc = np.full((out_size,) + x.shape[1:], 1 << (PRECISION_BITS - 1), np.int64)
    for j in range(k.shape[1]):
        idx = np.minimum(lo + j, in_size - 1)
        kj = np.where(j < cnt, k[:, j], 0).reshape((-1,) + (1,) * (x.ndim - 1))
        acc += x[idx] * kj
    return np.moveaxis(np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8), 0, axis)


def vertical_first(h, w, H):
    """PIL's Image.resize runs the vertical pass first for images taller than 100 x their width that shrink in
    height; otherwise the horizontal pass goes first."""
    return h > 100 * w and H < h


def resize_bicubic_u8(img, H, W):
    """PIL Image.fromarray(img).resize((W, H), BICUBIC) for uint8 HWC RGB, integer-exact."""
    h, w = img.shape[:2]
    if vertical_first(h, w, H):
        x = _pass(img, h, H, 0)
        return _pass(x, w, W, 1) if W != w else x
    x = _pass(img, w, W, 1) if W != w else img
    return _pass(x, h, H, 0) if H != h else x


def rescale_normalize(u8, mean=CLIP_MEAN, std=CLIP_STD):
    """uint8 HWC -> float32 CHW: float32(u8 * (1 / 255) in float64), then (x - mean32) / std32 in float32."""
    x = (u8.astype(np.float64) * (1 / 255)).astype(np.float32).transpose(2, 0, 1)
    m = np.asarray(mean, np.float32)[:, None, None]
    s = np.asarray(std, np.float32)[:, None, None]
    return np.ascontiguousarray((x - m) / s)


def pixel_values(img, shortest_edge=224, mean=CLIP_MEAN, std=CLIP_STD):
    """CLIPImageProcessorPil().preprocess(img, do_center_crop=False)['pixel_values'][0]: float32 [3, H', W']."""
    H, W = resized_size(img.shape[0], img.shape[1], shortest_edge)
    return rescale_normalize(resize_bicubic_u8(img, H, W), mean, std)


def fma32(a, b, c):
    """float32 fused multiply-add, correctly rounded: a * b is exact in float64, the sum is rounded to odd in float64
    (an inexact sum keeps its error in the sticky last bit) and then once to float32."""
    a, b, c = (np.asarray(v, np.float32).astype(np.float64) for v in (a, b, c))
    p = a * b
    s = p + c
    bp = s - c
    err = (p - bp) + (c - (s - bp))           # two-sum: s + err == p + c exactly
    even = (s.view(np.int64) & 1) == 0
    fix = (err != 0) & even
    s = np.where(fix, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    return s.astype(np.float32)


def bilinear_axis(in_size, out_size):
    """torch's (i0, i1, l0, l1) for align_corners=False and no scale factor, float32."""
    o = np.arange(out_size)
    if in_size == out_size:
        return o, o, np.ones(out_size, np.float32), np.zeros(out_size, np.float32)
    scale = np.float32(in_size) / np.float32(out_size)
    src = fma32(scale, (o + np.float32(0.5)).astype(np.float32), np.float32(-0.5))
    src = np.maximum(src, np.float32(0))
    i0 = np.minimum(np.floor(src).astype(np.int64), in_size - 1)
    l1 = np.clip(src - i0.astype(np.float32), np.float32(0), np.float32(1)).astype(np.float32)
    l0 = (np.float32(1) - l1).astype(np.float32)
    i1 = i0 + (i0 < in_size - 1)
    return i0, i1, l0, l1


def bilinear_square(x, S):
    """F.interpolate(torch.from_numpy(x)[None], (S, S), mode='bilinear', align_corners=False)[0] on the CPU."""
    _, H, W = x.shape
    y0, y1, ly0, ly1 = bilinear_axis(H, S)
    x0, x1, lx0, lx1 = bilinear_axis(W, S)
    r0, r1 = x[:, y0], x[:, y1]
    t0 = fma32(r0[:, :, x0], lx0, (r0[:, :, x1] * lx1).astype(np.float32))
    t1 = fma32(r1[:, :, x0], lx0, (r1[:, :, x1] * lx1).astype(np.float32))
    return fma32(t0, ly0[:, None], (t1 * ly1[:, None]).astype(np.float32))


def clip_preprocess(img, S=224, shortest_edge=224, mean=CLIP_MEAN, std=CLIP_STD):
    """The whole image path: uint8 HWC RGB -> float32 [3, S, S]."""
    return bilinear_square(pixel_values(img, shortest_edge, mean, std), S)


def normalize_boxes(boxes, h, w):
    """vcr.py:179 / app.py:121: xyxy / [w, h, w, h] in float64, then float32."""
    return (np.asarray(boxes, np.float64).reshape(-1, 4) / np.array([w, h, w, h], np.float64)).astype(np.float32)
