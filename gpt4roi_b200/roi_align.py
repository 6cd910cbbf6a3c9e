"""Operator seam: `roi_align`, `RoIAlign`, `RoIAlignFunction` and the `mmcv._ext` entry points.

Host-side mirror of the reference operator API (same names, argument meaning and error
behaviour), backed by the sm_90a kernels behind the C ABI:

    mmcv-1.4.7/mmcv/ops/roi_align.py:14-128   RoIAlignFunction (autograd)
    mmcv-1.4.7/mmcv/ops/roi_align.py:131      roi_align
    mmcv-1.4.7/mmcv/ops/roi_align.py:134-224  RoIAlign (nn.Module)
    mmcv-1.4.7/mmcv/ops/csrc/pytorch/pybind.cpp:611-620  _ext.roi_align_forward/backward

plus the fused multi-level entry used by the SPI module (`roi_align_mlvl`).
"""
import torch
import torch.nn as nn
from torch.autograd import Function
from torch.autograd.function import once_differentiable
from torch.nn.modules.utils import _pair

from . import lib as _L


# ---------------------------------------------------------------------------------------
# mmcv._ext entry points (11 keyword-callable arguments each; write in place, return None)
# ---------------------------------------------------------------------------------------
def roi_align_forward(input, rois, output, argmax_y, argmax_x, aligned_height, aligned_width,
                      spatial_scale, sampling_ratio, pool_mode, aligned):
    """Drop-in for mmcv._ext.roi_align_forward (pybind.cpp:611-615). NCHW, in place."""
    dev = _L.require_cuda_same_device([('input', input), ('rois', rois), ('output', output),
                                       ('argmax_y', argmax_y), ('argmax_x', argmax_x)])
    _L.require_contiguous([('input', input), ('rois', rois), ('output', output)])
    if rois.dtype != input.dtype or output.dtype != input.dtype:
        # the reference reads rois.data_ptr<scalar_t>() with input's scalar_t (roi_align_cuda.cu:22)
        raise RuntimeError('expected rois/output of dtype %s (same as input), got %s/%s'
                           % (input.dtype, rois.dtype, output.dtype))
    if input.dim() != 4 or rois.dim() != 2 or rois.size(1) != 5:
        raise RuntimeError('input must be [N,C,H,W] and rois [K,5]')
    n, c, h, w = input.shape
    k = rois.size(0)
    if tuple(output.shape) != (k, c, int(aligned_height), int(aligned_width)):
        raise RuntimeError('output must be [K,C,PH,PW] = %s, got %s'
                           % ((k, c, aligned_height, aligned_width), tuple(output.shape)))
    pool_mode = int(pool_mode)
    if pool_mode == _L.POOL_MAX and (argmax_y.shape != output.shape or argmax_x.shape != output.shape):
        raise RuntimeError('max pooling needs argmax_y/argmax_x shaped like output')
    lib = _L.load()
    code = _L.dtype_code(input)
    # scratch for the transpose -> NHWC kernel -> transpose path (0 when the direct NCHW kernel is the better fit)
    need = int(lib.g4r_roi_align_forward_workspace(n, c, h, w, k, int(aligned_height), int(aligned_width),
                                                   int(sampling_ratio), pool_mode, code, _L.NCHW))
    ws = torch.empty(need, dtype=torch.uint8, device=dev) if need else None
    with torch.cuda.device(dev):
        _L.check(lib.g4r_roi_align_forward_ws(
            _L.ptr(input), _L.ptr(rois), _L.ptr(output),
            _L.ptr(argmax_y) if pool_mode == _L.POOL_MAX else None,
            _L.ptr(argmax_x) if pool_mode == _L.POOL_MAX else None,
            n, c, h, w, k, int(aligned_height), int(aligned_width), float(spatial_scale),
            int(sampling_ratio), pool_mode, int(bool(aligned)), code, _L.NCHW,
            _L.ptr(ws), need, _L.stream_ptr(dev)), launches=3 if need else 1)


def roi_align_backward(grad_output, rois, argmax_y, argmax_x, grad_input, aligned_height,
                       aligned_width, spatial_scale, sampling_ratio, pool_mode, aligned):
    """Drop-in for mmcv._ext.roi_align_backward (pybind.cpp:616-620). grad_input pre-zeroed."""
    dev = _L.require_cuda_same_device([('grad_output', grad_output), ('rois', rois),
                                       ('argmax_y', argmax_y), ('argmax_x', argmax_x),
                                       ('grad_input', grad_input)])
    _L.require_contiguous([('grad_output', grad_output), ('rois', rois), ('grad_input', grad_input)])
    if rois.dtype != grad_output.dtype or grad_input.dtype != grad_output.dtype:
        raise RuntimeError('expected rois/grad_input of dtype %s, got %s/%s'
                           % (grad_output.dtype, rois.dtype, grad_input.dtype))
    n, c, h, w = grad_input.shape
    k = rois.size(0)
    pool_mode = int(pool_mode)
    with torch.cuda.device(dev):
        _L.check(_L.load().g4r_roi_align_backward(
            _L.ptr(grad_output), _L.ptr(rois),
            _L.ptr(argmax_y) if pool_mode == _L.POOL_MAX else None,
            _L.ptr(argmax_x) if pool_mode == _L.POOL_MAX else None,
            _L.ptr(grad_input), n, c, h, w, k, int(aligned_height), int(aligned_width),
            float(spatial_scale), int(sampling_ratio), pool_mode, int(bool(aligned)),
            _L.dtype_code(grad_output), _L.NCHW, _L.stream_ptr(dev)))


# ---------------------------------------------------------------------------------------
# operator API (mirrors mmcv/ops/roi_align.py)
# ---------------------------------------------------------------------------------------
class RoIAlignFunction(Function):
    """mmcv/ops/roi_align.py:14-128 (ONNX `symbolic` is a deployment back-end: out of scope)."""

    @staticmethod
    def forward(ctx, input, rois, output_size, spatial_scale=1.0, sampling_ratio=0,
                pool_mode='avg', aligned=True):
        ctx.output_size = _pair(output_size)
        ctx.spatial_scale = spatial_scale
        ctx.sampling_ratio = sampling_ratio
        assert pool_mode in ('max', 'avg')
        ctx.pool_mode = 0 if pool_mode == 'max' else 1
        ctx.aligned = aligned
        ctx.input_shape = input.size()

        assert rois.size(1) == 5, 'RoI must be (idx, x1, y1, x2, y2)!'

        output_shape = (rois.size(0), input.size(1), ctx.output_size[0], ctx.output_size[1])
        output = input.new_zeros(output_shape)
        if ctx.pool_mode == 0:
            argmax_y = input.new_zeros(output_shape)
            argmax_x = input.new_zeros(output_shape)
        else:
            argmax_y = input.new_zeros(0)
            argmax_x = input.new_zeros(0)

        roi_align_forward(input, rois, output, argmax_y, argmax_x,
                          aligned_height=ctx.output_size[0], aligned_width=ctx.output_size[1],
                          spatial_scale=ctx.spatial_scale, sampling_ratio=ctx.sampling_ratio,
                          pool_mode=ctx.pool_mode, aligned=ctx.aligned)

        ctx.save_for_backward(rois, argmax_y, argmax_x)
        return output

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        rois, argmax_y, argmax_x = ctx.saved_tensors
        grad_input = grad_output.new_zeros(ctx.input_shape)
        # complex head architecture may cause grad_output uncontiguous (roi_align.py:114-115)
        grad_output = grad_output.contiguous()
        roi_align_backward(grad_output, rois, argmax_y, argmax_x, grad_input,
                           aligned_height=ctx.output_size[0], aligned_width=ctx.output_size[1],
                           spatial_scale=ctx.spatial_scale, sampling_ratio=ctx.sampling_ratio,
                           pool_mode=ctx.pool_mode, aligned=ctx.aligned)
        return grad_input, None, None, None, None, None, None


roi_align = RoIAlignFunction.apply


class RoIAlign(nn.Module):
    """RoI align pooling layer -- same constructor and forward as mmcv.ops.RoIAlign
    (mmcv/ops/roi_align.py:134-224), including the deprecated `out_size` / `sample_num`
    keyword aliases (:171-177).  `use_torchvision=True` is refused: this module is the
    sm_90a path and has no alternate back-end.
    """

    def __init__(self, output_size=None, spatial_scale=1.0, sampling_ratio=0, pool_mode='avg',
                 aligned=True, use_torchvision=False, **deprecated):
        super(RoIAlign, self).__init__()
        if 'out_size' in deprecated:
            output_size = deprecated.pop('out_size')
        if 'sample_num' in deprecated:
            sampling_ratio = deprecated.pop('sample_num')
        if deprecated:
            raise TypeError('unexpected arguments %s' % sorted(deprecated))
        if output_size is None:
            raise TypeError("missing required argument 'output_size'")
        if use_torchvision:
            raise NotImplementedError('gpt4roi_b200.RoIAlign has a single (sm_90a) back-end')
        self.output_size = _pair(output_size)
        self.spatial_scale = float(spatial_scale)
        self.sampling_ratio = int(sampling_ratio)
        self.pool_mode = pool_mode
        self.aligned = aligned
        self.use_torchvision = use_torchvision

    def forward(self, input, rois):
        """input: NCHW images; rois: Kx5 boxes (batch index, x1, y1, x2, y2)."""
        return roi_align(input, rois, self.output_size, self.spatial_scale, self.sampling_ratio,
                         self.pool_mode, self.aligned)

    def __repr__(self):
        s = self.__class__.__name__
        s += f'(output_size={self.output_size}, '
        s += f'spatial_scale={self.spatial_scale}, '
        s += f'sampling_ratio={self.sampling_ratio}, '
        s += f'pool_mode={self.pool_mode}, '
        s += f'aligned={self.aligned}, '
        s += f'use_torchvision={self.use_torchvision})'
        return s


# ---------------------------------------------------------------------------------------
# fused multi-level entry (NHWC) used by the SPI module
# ---------------------------------------------------------------------------------------
def roi_align_mlvl(maps, rois, output_size, spatial_scales, sampling_ratio=2, aligned=True,
                   out_dtype=None, gn_scale=None, gn_shift=None, out=None):
    """All levels + all RoIs in one launch (replaces gpt4roi/models/layers.py:307-313).

    maps: list (<=4) of NHWC tensors [N,H_l,W_l,C] (fp32 / fp16 / bf16, same dtype);
    rois: fp32 [K,5] (batch_idx, x1, y1, x2, y2) in input-pixel units;
    returns [n_levels,K,PH,PW,C] (NHWC) of `out_dtype` (default: maps dtype).
    gn_scale/gn_shift: optional lists of fp32 [N,C] -- per-tap affine+ReLU (fused GroupNorm).
    """
    n_levels = len(maps)
    if not 1 <= n_levels <= _L.MAX_LEVELS:
        raise ValueError('1..%d levels supported, got %d' % (_L.MAX_LEVELS, n_levels))
    named = [('maps[%d]' % i, m) for i, m in enumerate(maps)] + [('rois', rois)]
    if gn_scale is not None:
        named += [('gn_scale[%d]' % i, t) for i, t in enumerate(gn_scale)]
        named += [('gn_shift[%d]' % i, t) for i, t in enumerate(gn_shift)]
    dev = _L.require_cuda_same_device(named)
    _L.require_contiguous(named)
    if rois.dtype != torch.float32 or rois.dim() != 2 or rois.size(1) != 5:
        raise RuntimeError('rois must be fp32 [K,5]')
    n, _, _, c = maps[0].shape
    for m in maps:
        if m.dim() != 4 or m.shape[0] != n or m.shape[3] != c or m.dtype != maps[0].dtype:
            raise RuntimeError('all maps must be NHWC [N,H_l,W_l,C] with the same N, C and dtype')
    ph, pw = _pair(output_size)
    k = rois.size(0)
    out_dtype = out_dtype or maps[0].dtype
    if out is None:
        out = torch.empty((n_levels, k, ph, pw, c), dtype=out_dtype, device=dev)
    elif tuple(out.shape) != (n_levels, k, ph, pw, c) or out.dtype != out_dtype or not out.is_contiguous():
        raise RuntimeError('out has the wrong shape/dtype')
    if k == 0:
        return out
    gs = gb = None
    if gn_scale is not None:
        for t in list(gn_scale) + list(gn_shift):
            if t.dtype != torch.float32 or tuple(t.shape) != (n, c):
                raise RuntimeError('gn_scale/gn_shift must be fp32 [N,C]')
        gs, gb = _L.ptr_array(gn_scale), _L.ptr_array(gn_shift)
    with torch.cuda.device(dev):
        _L.check(_L.load().g4r_roi_align_mlvl_forward(
            _L.ptr_array(maps), _L.int_array([m.shape[1] for m in maps]),
            _L.int_array([m.shape[2] for m in maps]), _L.float_array(spatial_scales), n_levels,
            _L.ptr(rois), _L.ptr(out), n, c, k, ph, pw, int(sampling_ratio), int(bool(aligned)),
            _L.dtype_code(maps[0]), _L._DTYPE[out_dtype], gs, gb, _L.stream_ptr(dev)))
    return out


def roi_align_mlvl_backward(grad_output, rois, map_shapes, spatial_scales, sampling_ratio=2,
                            aligned=True):
    """Gradient of roi_align_mlvl w.r.t. the maps: list of fp32 NHWC [N,H_l,W_l,C]."""
    dev = _L.require_cuda_same_device([('grad_output', grad_output), ('rois', rois)])
    _L.require_contiguous([('grad_output', grad_output), ('rois', rois)])
    n_levels, k, ph, pw, c = grad_output.shape
    grads = [torch.zeros(tuple(s), dtype=torch.float32, device=dev) for s in map_shapes]
    if k == 0:
        return grads
    n = map_shapes[0][0]
    with torch.cuda.device(dev):
        _L.check(_L.load().g4r_roi_align_mlvl_backward(
            _L.ptr(grad_output), _L.int_array([s[1] for s in map_shapes]),
            _L.int_array([s[2] for s in map_shapes]), _L.float_array(spatial_scales), n_levels,
            _L.ptr(rois), _L.ptr_array(grads), n, c, k, ph, pw, int(sampling_ratio),
            int(bool(aligned)), _L.dtype_code(grad_output), _L.stream_ptr(dev)))
    return grads
