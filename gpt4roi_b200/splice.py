"""Region-token splice: host-side mirror of the per-sample loop in
gpt4roi/models/spi_llava.py:99-196 (+ the embed_tokens lookup at :44-45), backed by the
`g4r_splice_region_tokens` kernels (csrc/splice.cu).

The reference raises ValueError from inside its python loop (device->host syncs at
spi_llava.py:105,114-128); here the kernel writes a per-sample status word and
`splice_region_tokens(..., validate=True)` reads it back once per batch and raises the
same errors.  `validate=False` skips the read-back (used under CUDA-graph capture after the
batch layout has been validated once).
"""
import torch

from . import lib as _L

_MESSAGES = {
    1: 'The number of image start tokens and image end tokens should be the same.',
    2: 'The image end token should follow the image start token.',
    3: 'The number of <bbox> tokens does not match the number of boxes of the sample.',
    4: 'More than one <im_start> per sample is not supported.',
    5: '<im_patch> tokens present without <im_start>.',
    6: 'Token id out of range of the embedding table.',
    7: 'Image tokens in a continuation chunk (the image span must lie in the cached prefix).',
}


def splice_region_tokens(input_ids, embed_weight, image_features, region_features, num_patches,
                         im_patch_token, im_start_token, im_end_token, bbox_token,
                         out=None, validate=True, return_plan=False, continuation=False):
    """Build `inputs_embeds` [B,L,D].

    input_ids       int64 [B,L] (cuda)
    embed_weight    [V,D] bf16/fp16 -- `model.embed_tokens.weight`
    image_features  [B,P,D] projected patch rows (same dtype), or None when P == 0
    region_features list (len B) of [K_i,D] tensors / None entries, a packed
                    (rows [K,D], offsets int32 [B+1]) tuple, or None (bboxes=None)
    continuation    the rows continue a sequence held in the KV cache (multi-turn generation): no image tokens may
                    appear (ValueError), and every sample's <bbox> tokens take its region rows in order
                    (g4r_splice_continuation); image_features must be None
    """
    B, L = input_ids.shape
    V, D = embed_weight.shape
    dev = _L.require_cuda_same_device([('input_ids', input_ids), ('embed_weight', embed_weight),
                                       ('image_features', image_features)])
    if input_ids.dtype != torch.int64:
        raise TypeError('input_ids must be int64')
    if embed_weight.dtype not in (torch.bfloat16, torch.float16):
        raise TypeError('splice moves 16-bit rows; got %s' % embed_weight.dtype)
    P = int(num_patches)
    if image_features is not None:
        if image_features.dtype != embed_weight.dtype or tuple(image_features.shape) != (B, P, D):
            raise RuntimeError('image_features must be [B,P,D]=%s of %s' % ((B, P, D), embed_weight.dtype))
    rows = offs = None
    if region_features is not None:
        if isinstance(region_features, tuple):
            rows, offs = region_features
        else:
            if len(region_features) != B:
                raise RuntimeError('need one region-feature entry per sample')
            counts = [0 if r is None else int(r.shape[0]) for r in region_features]
            parts = [r.to(embed_weight.dtype) for r in region_features if r is not None and r.shape[0] > 0]
            rows = torch.cat(parts, 0) if parts else embed_weight.new_zeros((1, D))
            offs = torch.tensor([0] + list(torch.tensor(counts).cumsum(0).tolist()) if counts else [0],
                                dtype=torch.int32).to(dev, non_blocking=True)
        if rows.dtype != embed_weight.dtype or rows.shape[-1] != D:
            raise RuntimeError('region rows must be [K,D] of %s' % embed_weight.dtype)
        rows = rows.contiguous()
    _L.require_contiguous([('input_ids', input_ids), ('embed_weight', embed_weight),
                           ('image_features', image_features)])
    if out is None:
        out = torch.empty((B, L, D), dtype=embed_weight.dtype, device=dev)
    plan = torch.empty((B, L), dtype=torch.int32, device=dev)
    status = torch.empty((B,), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        if continuation:
            if image_features is not None:
                raise RuntimeError('a continuation chunk takes no image_features')
            _L.check(_L.load().g4r_splice_continuation(
                _L.ptr(input_ids), _L.ptr(embed_weight), _L.ptr(rows), _L.ptr(offs), _L.ptr(out), _L.ptr(plan),
                _L.ptr(status), B, L, D, V, int(im_patch_token), int(im_start_token), int(im_end_token),
                int(bbox_token), _L.stream_ptr(dev)), launches=2)
        else:
            _L.check(_L.load().g4r_splice_region_tokens(
                _L.ptr(input_ids), _L.ptr(embed_weight), _L.ptr(image_features), _L.ptr(rows), _L.ptr(offs),
                _L.ptr(out), _L.ptr(plan), _L.ptr(status), B, L, P, D, V, int(im_patch_token),
                int(im_start_token), int(im_end_token), int(bbox_token), _L.stream_ptr(dev)), launches=2)
    if validate:
        st = status.cpu()
        bad = torch.nonzero(st)
        if bad.numel():
            b = int(bad[0])
            raise ValueError('%s (sample %d)' % (_MESSAGES.get(int(st[b]), 'splice error %d' % int(st[b])), b))
    return (out, plan) if return_plan else out


_TAG_REGION = 0x20000000   # csrc/splice.cu: plan codes >= this are image / region rows


def splice_backward(plan, d_out, num_patches, n_regions, vocab, want_embed_grad=True):
    """Backward of splice_region_tokens: d_out [B,L,D] (bf16) -> (d_image [B,P,D], d_region [K,D],
    d_embed fp32 [V,D] dense or None).  The positions of every token id are grouped on the host side of the
    call (torch.sort on B*L indices -- index plumbing like plan_boxes); the sums run in the kernel."""
    B, L, D = d_out.shape
    dev = d_out.device
    P, K = int(num_patches), int(n_regions)
    d_out = d_out.contiguous()
    # zero-filled: the kernel writes only rows the plan tags as image / region rows -- a text-only sample
    # (spi_llava.py:104-111) leaves its d_image rows, a sample whose boxes are unused its d_region rows, untouched
    d_image = torch.zeros((B, P, D), dtype=d_out.dtype, device=dev) if P > 0 else None
    d_region = torch.zeros((K, D), dtype=d_out.dtype, device=dev) if K > 0 else None
    with torch.cuda.device(dev):
        _L.check(_L.load().g4r_splice_backward(_L.ptr(plan), _L.ptr(d_out), _L.ptr(d_image), _L.ptr(d_region),
                                               B, L, P, D, _L.stream_ptr(dev)))
    d_embed = None
    if want_embed_grad:
        codes = plan.reshape(-1)
        rows = torch.nonzero(codes < _TAG_REGION).squeeze(1)
        ids_sorted, perm = torch.sort(codes[rows], stable=True)
        order = rows[perm].to(torch.int32).contiguous()
        uniq, counts = torch.unique_consecutive(ids_sorted, return_counts=True)
        seg = torch.zeros(uniq.numel() + 1, dtype=torch.int32, device=dev)
        seg[1:] = counts.cumsum(0)
        d_embed = torch.zeros((vocab, D), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _L.check(_L.load().g4r_embed_grad_rows(_L.ptr(d_out), _L.ptr(order), _L.ptr(seg),
                                                   _L.ptr(uniq.to(torch.int32).contiguous()), int(uniq.numel()),
                                                   _L.ptr(d_embed), D, _L.stream_ptr(dev)))
    return d_image, d_region, d_embed
