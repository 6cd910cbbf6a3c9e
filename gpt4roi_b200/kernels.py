"""Torch-tensor front-ends of the elementwise / attention entry points of the C ABI
(csrc/elementwise.cu, csrc/attention.cu).  No computation happens in Python."""
import ctypes
import os

import torch

from . import lib as _L


def _call(fn_name, dev, *args, act=torch.bfloat16):
    """act: the 16-bit storage type of the call's tensors -- selects the bf16 entry point or its fp16 twin."""
    with torch.cuda.device(dev):
        _L.check(getattr(_L.load(), _L.sym(fn_name, act))(*args, _L.stream_ptr(dev)))


def _bf16(*ts):
    """All given tensors share one 16-bit storage type (bf16, or fp16 for the demo's dtype); returns it."""
    dt = None
    for t in ts:
        if t is None:
            continue
        if t.dtype not in (torch.bfloat16, torch.float16) or (dt is not None and t.dtype != dt):
            raise TypeError('bf16 (or all-fp16) tensors required, got %s' % ', '.join(str(u.dtype) for u in ts if u is not None))
        dt = t.dtype
    return dt


def layernorm(x, weight, bias, eps=1e-5, out=None):
    act = _bf16(x, weight, bias)
    D = x.shape[-1]
    x2 = x.reshape(-1, D)
    out = torch.empty_like(x2) if out is None else out
    _call('g4r_layernorm_bf16', x.device, _L.ptr(x2), x2.stride(0), _L.ptr(weight), _L.ptr(bias), _L.ptr(out),
          out.stride(0), x2.shape[0], D, float(eps), act=act)
    return out.view(x.shape) if out.is_contiguous() and out.numel() == x.numel() else out


def layernorm_ex(x, weight, bias, eps=1e-5, out_dtype=None):
    """LayerNorm with 16-bit/fp32 input rows and 16-bit/fp32 output rows (CLIP's fp32 residual stream); the 16-bit
    type is the weight's."""
    act = _bf16(weight, bias)
    out_dtype = act if out_dtype is None else out_dtype
    if x.dtype not in (act, torch.float32) or out_dtype not in (act, torch.float32):
        raise TypeError('layernorm_ex: rows must be %s or fp32, got %s -> %s' % (act, x.dtype, out_dtype))
    D = x.shape[-1]
    x2 = x.reshape(-1, D)
    out = torch.empty(x2.shape, dtype=out_dtype, device=x.device)
    _call('g4r_layernorm_ex', x.device, _L.ptr(x2), x2.stride(0), int(x.dtype == torch.float32), _L.ptr(weight),
          _L.ptr(bias), _L.ptr(out), out.stride(0), int(out_dtype == torch.float32), x2.shape[0], D, float(eps), act=act)
    return out.view(x.shape)


def cast_tokens_f32_bf16(hidden, skip_first=1, dtype=torch.bfloat16):
    """hidden fp32 [B,T,C] -> dense 16-bit [B*(T-skip_first), C] (drops the CLS row)."""
    B, T, C = hidden.shape
    out = torch.empty((B * (T - skip_first), C), dtype=dtype, device=hidden.device)
    src = ctypes.c_void_p(hidden.data_ptr() + skip_first * C * 4)
    _call('g4r_cast_f32_bf16', hidden.device, src, C, T * C, _L.ptr(out), B, T - skip_first, C, act=dtype)
    return out


def rmsnorm(x, weight, eps=1e-6, out=None):
    """x 16-bit (the weight's type) or fp32 rows (an fp32 residual stream); 16-bit output."""
    act = _bf16(weight)
    if x.dtype not in (act, torch.float32):
        raise TypeError('rmsnorm: %s or fp32 rows required, got %s' % (act, x.dtype))
    D = x.shape[-1]
    x2 = x.reshape(-1, D)
    out = torch.empty(x2.shape, dtype=act, device=x.device) if out is None else out
    _call('g4r_rmsnorm_ex', x.device, _L.ptr(x2), x2.stride(0), int(x.dtype == torch.float32), _L.ptr(weight),
          _L.ptr(out), out.stride(0), x2.shape[0], D, float(eps), act=act)
    return out.view(x.shape) if out.is_contiguous() and out.numel() == x.numel() else out


def rope_inplace(qkv, cos, sin, L, n_heads_qk, head_dim):
    """qkv [rows, width] packed; rotates the first n_heads_qk heads of every row in place."""
    act = _bf16(qkv, cos, sin)
    _call('g4r_rope_inplace_bf16', qkv.device, _L.ptr(qkv), qkv.stride(0), _L.ptr(cos), _L.ptr(sin),
          qkv.shape[0], int(L), int(n_heads_qk), int(head_dim), act=act)
    return qkv


ATTN_IMPL = os.environ.get('G4R_ATTN', 'tc')  # 'tc' = wgmma kernel, 'mma' = mma.sync kernel


def attention(qkv, B, L, n_heads, head_dim, causal, scale, out=None, seqlens=None, impl=None):
    """qkv: packed bf16 [B*L, 3*n_heads*head_dim] = (q | k | v); returns [B*L, n_heads*head_dim]."""
    act = _bf16(qkv)
    hd = n_heads * head_dim
    if out is None:
        out = torch.empty((B * L, hd), dtype=act, device=qkv.device)
    ld = qkv.stride(0)
    esz = 2
    base = qkv.data_ptr()
    q, k, v = (ctypes.c_void_p(base + i * hd * esz) for i in range(3))
    fn = 'g4r_attention_tc_bf16' if (impl or ATTN_IMPL) == 'tc' else 'g4r_attention_bf16'
    _call(fn, qkv.device, q, k, v, _L.ptr(out), ld, L * ld, out.stride(0), L * out.stride(0),
          B, n_heads, L, head_dim, int(bool(causal)), float(scale), _L.ptr(seqlens), act=act)
    return out


def attention_cached(qkv, kcache, vcache, B, n_heads, head_dim, Lc, scale, start, qlen=None, cache_rows=None):
    """Chunk attention over the KV cache: qkv packed [B*Lc, 3*HD] (RoPE-rotated at each row's positions), whose k|v were
    already appended to caches [B, Lmax, HD] at start[b]..; start / qlen device int32 [B] (qlen None: all Lc rows valid).
    Query i of row b attends over cache positions 0 .. start[b] + i.  Returns [B*Lc, HD]; rows >= qlen[b] hold finite
    filler (zeros for 128-row tiles wholly past qlen[b]).
    cache_rows: device int32 [B] -- the caches are [rows, Lmax, HD] (any number of rows) and chunk row b reads cache row
    cache_rows[b] (g4r_attention_cached_rows_bf16); qlen is then required."""
    act = _bf16(qkv, kcache, vcache)
    hd = n_heads * head_dim
    out = torch.empty((B * Lc, hd), dtype=act, device=qkv.device)
    if cache_rows is not None:
        _call('g4r_attention_cached_rows_bf16', qkv.device, _L.ptr(qkv), qkv.stride(0), _L.ptr(kcache), _L.ptr(vcache),
              kcache.shape[0], kcache.shape[1], _L.ptr(out), out.stride(0), B, n_heads, Lc, head_dim, float(scale),
              _L.ptr(_L.require_pos_rows(start, B)), _L.ptr(_L.require_pos_rows(qlen, B)),
              _L.ptr(_L.require_pos_rows(cache_rows, B)), act=act)
        return out
    _call('g4r_attention_cached_bf16', qkv.device, _L.ptr(qkv), qkv.stride(0), _L.ptr(kcache), _L.ptr(vcache),
          kcache.shape[1], _L.ptr(out), out.stride(0), B, n_heads, Lc, head_dim, float(scale),
          _L.ptr(_L.require_pos_rows(start, B)), None if qlen is None else _L.ptr(_L.require_pos_rows(qlen, B)), act=act)
    return out


def patchify(images, ps, kpad):
    act = _bf16(images)
    B, _, S, _ = images.shape
    G = S // ps
    out = torch.empty((B * G * G, kpad), dtype=act, device=images.device)
    _call('g4r_patchify_bf16', images.device, _L.ptr(images.contiguous()), _L.ptr(out), B, S, ps, kpad, act=act)
    return out


def vit_embed(patch, cls, pos, B, P):
    act = _bf16(patch, cls, pos)
    D = patch.shape[-1]
    out = torch.empty((B, P + 1, D), dtype=act, device=patch.device)
    _call('g4r_vit_embed_bf16', patch.device, _L.ptr(patch), _L.ptr(cls), _L.ptr(pos), _L.ptr(out), B, P, D, act=act)
    return out


def upsample_tokens_coords(hidden, G, Ho, cpad, has_cls=True, dtype=None):
    """hidden: [B, 1+G*G, C] ViT hidden state, 16-bit or fp32 (CLS first; has_cls=False: [B, G*G, C]);
    returns 16-bit NHWC [B,Ho,Ho,cpad] (`dtype`: the 16-bit type for fp32 tokens, default bf16)."""
    B, T, C = hidden.shape
    skip = 1 if has_cls else 0
    if T != G * G + skip or not hidden.is_contiguous() or hidden.dtype not in (torch.float32, torch.bfloat16, torch.float16):
        raise RuntimeError('upsample_tokens_coords: contiguous bf16/fp16/fp32 [B,%d,C] tokens required, got %s %s'
                           % (G * G + skip, tuple(hidden.shape), hidden.dtype))
    act = hidden.dtype if hidden.dtype != torch.float32 else (dtype or torch.bfloat16)
    out = torch.empty((B, Ho, Ho, cpad), dtype=act, device=hidden.device)
    f32 = hidden.dtype == torch.float32
    tok = ctypes.c_void_p(hidden.data_ptr() + skip * C * (4 if f32 else 2))  # skip CLS
    _call('g4r_upsample_tokens_coords_f32' if f32 else 'g4r_upsample_tokens_coords_bf16', hidden.device, tok, C,
          T * C, _L.ptr(out), B, G, Ho, C, cpad, act=act)
    return out


def fuse_gather(own, top, down, own_ss=None, top_ss=None, down_ss=None, out=None):
    """own/top/down: NHWC bf16 [B,H,H,C]; *_ss: optional (scale, shift) fp32 [B,C] pairs."""
    act = _bf16(own, top, down)
    B, H, _, C = own.shape
    out = torch.empty_like(own) if out is None else out

    def ss(p):
        return (None, None) if p is None else (_L.ptr(p[0]), _L.ptr(p[1]))
    a, b, c = ss(own_ss), ss(top_ss), ss(down_ss)
    _call('g4r_fuse_gather_bf16', own.device, _L.ptr(own), a[0], a[1], H, _L.ptr(top), b[0], b[1], top.shape[1],
          _L.ptr(down), c[0], c[1], down.shape[1], _L.ptr(out), B, C, act=act)
    return out


def gn_finalize(stats, gamma, beta, count, eps=1e-5):
    """stats: fp32 [B, slots, groups, 2] partial sums from dense.conv_nhwc(gn_stats=...)."""
    B, slots, groups, _ = stats.shape
    C = gamma.shape[0]
    scale = torch.empty((B, C), dtype=torch.float32, device=stats.device)
    shift = torch.empty_like(scale)
    _call('g4r_gn_finalize', stats.device, _L.ptr(stats), _L.ptr(gamma), _L.ptr(beta), _L.ptr(scale),
          _L.ptr(shift), B, C, groups, slots, float(count), float(eps), act=_bf16(gamma, beta))
    return scale, shift


def affine_relu_nhwc(z, scale, shift):
    """z bf16 NHWC [B,H,W,C], scale/shift fp32 [B,C] (gn_finalize) -> relu(z*scale+shift) bf16 NHWC."""
    act = _bf16(z)
    B, H, W, C = z.shape
    out = torch.empty_like(z)
    _call('g4r_affine_relu_nhwc_bf16', z.device, _L.ptr(z), _L.ptr(scale), _L.ptr(shift), _L.ptr(out), B, H * W, C, act=act)
    return out


def pos_embed_mlp(boxes, w0, b0, g2, be2, w3, b3, g5, be5, eps=1e-5):
    K = boxes.shape[0]
    out = torch.empty((K, 1024), dtype=torch.float32, device=boxes.device)
    if K:
        _call('g4r_pos_embed_mlp', boxes.device, _L.ptr(boxes), _L.ptr(w0), _L.ptr(b0), _L.ptr(g2), _L.ptr(be2),
              _L.ptr(w3), _L.ptr(b3), _L.ptr(g5), _L.ptr(be5), _L.ptr(out), K, float(eps),
              act=_bf16(w0, b0, g2, be2, w3, b3, g5, be5))
    return out


def add_bias_pos_cast(acc, bias, pos):
    """acc: fp32 [splits, K, D] (split-K slabs) or [K, D]."""
    if acc.dim() == 2:
        acc = acc[None]
    splits, K, D = acc.shape
    act = _bf16(bias)
    out = torch.empty((K, D), dtype=act, device=acc.device)
    if K:
        _call('g4r_add_bias_pos_cast', acc.device, _L.ptr(acc), splits, _L.ptr(bias), _L.ptr(pos), _L.ptr(out), K, D, act=act)
    return out


def _logit_rows(name, logits):
    """16-bit logits [rows, V] or [rows, 1, V] -> ([rows, V] with unit column stride, their 16-bit type)."""
    rows = logits.reshape(logits.shape[0], logits.shape[-1]) if logits.dim() == 3 else logits
    if rows.stride(1) != 1:
        raise RuntimeError('%s: logits rows must have unit column stride' % name)
    return rows, _bf16(rows)


def sample_tokens(logits, out, greedy, temperature=1.0, top_k=0, top_p=1.0, seed=0, rng_step=None, eos_id=-1,
                  pad_id=-1, finished=None):
    """Next token of every row of 16-bit logits [B, V] (or [B, 1, V]; unit column stride) into out (int64, B contiguous
    elements, e.g. the [B, 1] ids buffer of a decode step): the arg-max (greedy), or a draw from the temperature /
    top-k / top-p processed softmax with Philox key `seed` and counter (*rng_step, row) -- rng_step: device int64 [1].
    top_k 0 / top_p 1 switch that filter off.  finished (device int32 [B]) with eos_id, pad_id >= 0: transformers'
    eos -> pad rule, updated in place."""
    rows, act = _logit_rows('sample_tokens', logits)
    B, V = rows.shape
    if out.dtype != torch.int64 or out.numel() != B or not out.is_contiguous():
        raise RuntimeError('sample_tokens: out must be a contiguous int64 tensor of %d elements' % B)
    if rng_step is not None and (rng_step.dtype != torch.int64 or rng_step.numel() != 1):
        raise RuntimeError('sample_tokens: rng_step must be a device int64 [1] counter')
    if finished is not None and (finished.dtype != torch.int32 or finished.numel() != B or not finished.is_contiguous()):
        raise RuntimeError('sample_tokens: finished must be a contiguous device int32 [%d] vector' % B)
    _L.require_cuda_same_device([('logits', rows), ('out', out), ('rng_step', rng_step), ('finished', finished)])
    _call('g4r_sample_tokens_bf16', rows.device, _L.ptr(rows), rows.stride(0), B, V, float(temperature), int(top_k),
          float(top_p), int(bool(greedy)), int(seed) & 0xFFFFFFFFFFFFFFFF, _L.ptr(rng_step), int(eos_id), int(pad_id),
          _L.ptr(finished), _L.ptr(out), act=act)
    return out


def sample_tokens_rows(logits, out, greedy, temperature, top_k, top_p, seed, step, eos_id, active, finished, lens=None):
    """Next token of every active row of 16-bit logits [S, V] (or [S, 1, V]; unit column stride) into out (int64, S
    contiguous elements), each row with its own rule (include/gpt4roi_b200.h: g4r_sample_tokens_rows_bf16): row r selects
    as sample_tokens on that row alone with rng_step = step[r].  Per-row contiguous device vectors of S entries: greedy,
    top_k, eos_id (-1: none), active (int32); temperature, top_p (fp32); seed (int64, read as uint64); step (int64).
    An active row sets finished[r] when its token is eos_id[r], advances step[r] and, when given, lens[r] (int32 [S]);
    an inactive row is left alone.  A sampled row needs temperature > 0 and top_p >= 0: the caller checks, the rule is
    device data."""
    rows, act = _logit_rows('sample_tokens_rows', logits)
    S, V = rows.shape
    if out.dtype != torch.int64 or out.numel() != S or not out.is_contiguous():
        raise RuntimeError('sample_tokens_rows: out must be a contiguous int64 tensor of %d elements' % S)
    named = [('greedy', greedy, torch.int32), ('temperature', temperature, torch.float32),
             ('top_k', top_k, torch.int32), ('top_p', top_p, torch.float32), ('seed', seed, torch.int64),
             ('step', step, torch.int64), ('eos_id', eos_id, torch.int32), ('active', active, torch.int32),
             ('finished', finished, torch.int32), ('lens', lens, torch.int32)]
    for name, t, dt in named:
        if t is None and name == 'lens':
            continue
        if t is None or t.dtype != dt or t.numel() != S or not t.is_contiguous():
            raise RuntimeError('sample_tokens_rows: %s must be a contiguous device %s [%d] vector' % (name, dt, S))
    _L.require_cuda_same_device([('logits', rows), ('out', out)] + [(n, t) for n, t, _ in named])
    _call('g4r_sample_tokens_rows_bf16', rows.device, _L.ptr(rows), rows.stride(0), S, V,
          *[_L.ptr(t) for _, t, _ in named[:8]], _L.ptr(finished), _L.ptr(out), _L.ptr(lens), act=act)
    return out


PROC_LIST_MAX = 8192   # history ids per row that sampling with a repetition penalty holds (csrc/sample.cu)
PROC_ROW_EOS = 4       # ids a row's minimum lengths suppress in sample_tokens_rows_processed (csrc/sample.cu)


def sample_tokens_rows_processed(logits, out, greedy, temperature, top_k, top_p, seed, step, eos_id, active, finished,
                                 lens, history, prompt_len, repetition_penalty, no_repeat_ngram_size, min_length,
                                 min_new_tokens, eos_ids, n_eos):
    """sample_tokens_rows with transformers' history-dependent logits processors per row (include/gpt4roi_b200.h:
    g4r_sample_tokens_rows_proc_bf16): an active row whose four processors are neutral selects as sample_tokens_rows
    does; any other selects as sample_tokens_processed on that row alone with L = prompt_len[r] and rng_step = step[r],
    and writes its token to history[r, prompt_len[r] + step[r]].  The arguments of sample_tokens_rows (lens may be
    None), then: history, a contiguous device int64 [S, ld_h] tensor; per-row contiguous device vectors of S entries:
    prompt_len, no_repeat_ngram_size, min_length, min_new_tokens, n_eos (int32), repetition_penalty (fp32); eos_ids, a
    contiguous device int32 [S, 4] tensor whose row r holds the n_eos[r] ids row r's minimum lengths suppress.  The
    values are device data: the caller checks them (penalty > 0, lengths >= 0, n_eos <= 4, and a sampled row with a
    penalty holding at most min(ld_h, PROC_LIST_MAX) history ids)."""
    rows, act = _logit_rows('sample_tokens_rows_processed', logits)
    S, V = rows.shape
    if out.dtype != torch.int64 or out.numel() != S or not out.is_contiguous():
        raise RuntimeError('sample_tokens_rows_processed: out must be a contiguous int64 tensor of %d elements' % S)
    named = [('greedy', greedy, torch.int32), ('temperature', temperature, torch.float32),
             ('top_k', top_k, torch.int32), ('top_p', top_p, torch.float32), ('seed', seed, torch.int64),
             ('step', step, torch.int64), ('eos_id', eos_id, torch.int32), ('active', active, torch.int32),
             ('finished', finished, torch.int32), ('lens', lens, torch.int32)]
    procs = [('prompt_len', prompt_len, torch.int32), ('repetition_penalty', repetition_penalty, torch.float32),
             ('no_repeat_ngram_size', no_repeat_ngram_size, torch.int32), ('min_length', min_length, torch.int32),
             ('min_new_tokens', min_new_tokens, torch.int32), ('n_eos', n_eos, torch.int32)]
    for name, t, dt in named + procs:
        if t is None and name == 'lens':
            continue
        if t is None or t.dtype != dt or t.numel() != S or not t.is_contiguous():
            raise RuntimeError('sample_tokens_rows_processed: %s must be a contiguous device %s [%d] vector'
                               % (name, dt, S))
    if history is None or history.dtype != torch.int64 or history.dim() != 2 or history.shape[0] != S \
            or history.shape[1] < 1 or not history.is_contiguous():
        raise RuntimeError('sample_tokens_rows_processed: history must be a contiguous int64 [%d, ld_h] tensor' % S)
    if eos_ids is None or eos_ids.dtype != torch.int32 or tuple(eos_ids.shape) != (S, PROC_ROW_EOS) \
            or not eos_ids.is_contiguous():
        raise RuntimeError('sample_tokens_rows_processed: eos_ids must be a contiguous int32 [%d, %d] tensor'
                           % (S, PROC_ROW_EOS))
    _L.require_cuda_same_device([('logits', rows), ('out', out), ('history', history), ('eos_ids', eos_ids)]
                                + [(n, t) for n, t, _ in named + procs])
    p = [_L.ptr(t) for _, t, _ in procs]
    _call('g4r_sample_tokens_rows_proc_bf16', rows.device, _L.ptr(rows), rows.stride(0), S, V,
          *[_L.ptr(t) for _, t, _ in named[:8]], _L.ptr(finished), _L.ptr(out), _L.ptr(lens), _L.ptr(history),
          history.shape[1], *p[:5], _L.ptr(eos_ids), p[5], act=act)
    return out


def sample_tokens_processed(logits, out, greedy, temperature=1.0, top_k=0, top_p=1.0, seed=0, rng_step=None, eos_id=-1,
                            pad_id=-1, finished=None, history=None, L=0, repetition_penalty=1.0, no_repeat_ngram_size=0,
                            min_length=0, min_new_tokens=0, eos_ids=None, append=True):
    """sample_tokens on the scores transformers' history-dependent processors leave (include/gpt4roi_b200.h:
    g4r_sample_tokens_proc_bf16): RepetitionPenaltyLogitsProcessor, NoRepeatNGramLogitsProcessor, MinLengthLogitsProcessor
    and MinNewTokensLengthLogitsProcessor, applied on the device to row b's history history[b, :L + rng_step].
    history: contiguous device int64 [B, ld_h] (ld_h >= L); rng_step (device int64 [1]) is required, also for greedy;
    eos_ids: device int32 [n] (None: none), the ids min_length / min_new_tokens suppress.  append: write the selected
    id to history[b, L + rng_step] (after the eos -> pad rule)."""
    rows, act = _logit_rows('sample_tokens_processed', logits)
    B, V = rows.shape
    if out.dtype != torch.int64 or out.numel() != B or not out.is_contiguous():
        raise RuntimeError('sample_tokens_processed: out must be a contiguous int64 tensor of %d elements' % B)
    if rng_step is None or rng_step.dtype != torch.int64 or rng_step.numel() != 1:
        raise RuntimeError('sample_tokens_processed: rng_step must be a device int64 [1] counter')
    if finished is not None and (finished.dtype != torch.int32 or finished.numel() != B or not finished.is_contiguous()):
        raise RuntimeError('sample_tokens_processed: finished must be a contiguous device int32 [%d] vector' % B)
    if history is None or history.dtype != torch.int64 or history.dim() != 2 or history.shape[0] != B \
            or not history.is_contiguous():
        raise RuntimeError('sample_tokens_processed: history must be a contiguous int64 [%d, ld_h] tensor' % B)
    ld_h = history.shape[1]
    if not 0 <= int(L) <= ld_h:
        raise RuntimeError('sample_tokens_processed: the prompt length L=%d must lie in [0, %d]' % (L, ld_h))
    if not repetition_penalty > 0 or int(no_repeat_ngram_size) < 0 or int(min_length) < 0 or int(min_new_tokens) < 0:
        raise RuntimeError('sample_tokens_processed: repetition_penalty must be > 0 and the lengths >= 0 (got %r, %r, %r, '
                           '%r)' % (repetition_penalty, no_repeat_ngram_size, min_length, min_new_tokens))
    if not greedy and repetition_penalty != 1.0 and ld_h > PROC_LIST_MAX:
        raise RuntimeError('sample_tokens_processed: sampling with a repetition penalty holds at most %d history ids per '
                           'row (ld_h=%d)' % (PROC_LIST_MAX, ld_h))
    if eos_ids is not None and (eos_ids.dtype != torch.int32 or eos_ids.dim() != 1 or not eos_ids.is_contiguous()):
        raise RuntimeError('sample_tokens_processed: eos_ids must be a contiguous device int32 vector')
    n_eos = 0 if eos_ids is None else eos_ids.numel()
    _L.require_cuda_same_device([('logits', rows), ('out', out), ('rng_step', rng_step), ('finished', finished),
                                 ('history', history), ('eos_ids', eos_ids)])
    _call('g4r_sample_tokens_proc_bf16', rows.device, _L.ptr(rows), rows.stride(0), B, V, float(temperature),
          int(top_k), float(top_p), int(bool(greedy)), int(seed) & 0xFFFFFFFFFFFFFFFF, _L.ptr(rng_step), int(eos_id),
          int(pad_id), _L.ptr(finished), _L.ptr(out), _L.ptr(history), ld_h, int(L), float(repetition_penalty),
          int(no_repeat_ngram_size), int(min_length), int(min_new_tokens), _L.ptr(eos_ids) if n_eos else None, n_eos,
          int(bool(append)), act=act)
    return out


def _slot_buffer(name, t, rows, V):
    """An output slot buffer: None, or a contiguous device fp32 [n_slots, rows, V] tensor; returns n_slots (0: None)."""
    if t is None:
        return 0
    if t.dtype != torch.float32 or t.dim() != 3 or tuple(t.shape[1:]) != (rows, V) or not t.is_contiguous() \
            or t.shape[0] < 1:
        raise RuntimeError('%s must be a contiguous fp32 [n_slots, %d, %d] tensor, got %s %s'
                           % (name, rows, V, t.dtype, tuple(t.shape)))
    return t.shape[0]


def sample_tokens_out(logits, out, greedy, temperature=1.0, top_k=0, top_p=1.0, seed=0, rng_step=None, eos_id=-1,
                      pad_id=-1, finished=None, history=None, L=0, repetition_penalty=1.0, no_repeat_ngram_size=0,
                      min_length=0, min_new_tokens=0, eos_ids=None, append=True, scores=None, raw_logits=None):
    """sample_tokens (history None) or sample_tokens_processed, writing transformers' generate() outputs into slot
    *rng_step of scores / raw_logits (contiguous device fp32 [n_slots, B, V], either may be None; include/gpt4roi_b200.h:
    g4r_sample_tokens_out_bf16): scores gets HF's next_token_scores (the processors, then when sampling / temperature
    and -inf below the top-k / top-p thresholds), raw_logits the widened logits.  With both None it launches what
    sample_tokens / sample_tokens_processed launch."""
    rows, act = _logit_rows('sample_tokens_out', logits)
    B, V = rows.shape
    if scores is None and raw_logits is None:
        if history is None:
            return sample_tokens(logits, out, greedy, temperature, top_k, top_p, seed, rng_step, eos_id, pad_id, finished)
        return sample_tokens_processed(logits, out, greedy, temperature, top_k, top_p, seed, rng_step, eos_id, pad_id,
                                       finished, history, L, repetition_penalty, no_repeat_ngram_size, min_length,
                                       min_new_tokens, eos_ids, append)
    n_slots = max(_slot_buffer('sample_tokens_out: scores', scores, B, V),
                  _slot_buffer('sample_tokens_out: raw_logits', raw_logits, B, V))
    if scores is not None and raw_logits is not None and scores.shape[0] != raw_logits.shape[0]:
        raise RuntimeError('sample_tokens_out: scores and raw_logits must hold the same number of slots')
    if out.dtype != torch.int64 or out.numel() != B or not out.is_contiguous():
        raise RuntimeError('sample_tokens_out: out must be a contiguous int64 tensor of %d elements' % B)
    if rng_step is None or rng_step.dtype != torch.int64 or rng_step.numel() != 1:
        raise RuntimeError('sample_tokens_out: rng_step (the output slot) must be a device int64 [1] counter')
    if finished is not None and (finished.dtype != torch.int32 or finished.numel() != B or not finished.is_contiguous()):
        raise RuntimeError('sample_tokens_out: finished must be a contiguous device int32 [%d] vector' % B)
    ld_h = 0
    if history is not None:
        if history.dtype != torch.int64 or history.dim() != 2 or history.shape[0] != B or not history.is_contiguous():
            raise RuntimeError('sample_tokens_out: history must be a contiguous int64 [%d, ld_h] tensor' % B)
        ld_h = history.shape[1]
        if not 0 <= int(L) <= ld_h:
            raise RuntimeError('sample_tokens_out: the prompt length L=%d must lie in [0, %d]' % (L, ld_h))
        if not greedy and repetition_penalty != 1.0 and ld_h > PROC_LIST_MAX:
            raise RuntimeError('sample_tokens_out: sampling with a repetition penalty holds at most %d history ids per '
                               'row (ld_h=%d)' % (PROC_LIST_MAX, ld_h))
    if not repetition_penalty > 0 or int(no_repeat_ngram_size) < 0 or int(min_length) < 0 or int(min_new_tokens) < 0:
        raise RuntimeError('sample_tokens_out: repetition_penalty must be > 0 and the lengths >= 0 (got %r, %r, %r, %r)'
                           % (repetition_penalty, no_repeat_ngram_size, min_length, min_new_tokens))
    if eos_ids is not None and (eos_ids.dtype != torch.int32 or eos_ids.dim() != 1 or not eos_ids.is_contiguous()):
        raise RuntimeError('sample_tokens_out: eos_ids must be a contiguous device int32 vector')
    n_eos = 0 if eos_ids is None else eos_ids.numel()
    _L.require_cuda_same_device([('logits', rows), ('out', out), ('rng_step', rng_step), ('finished', finished),
                                 ('history', history), ('eos_ids', eos_ids), ('scores', scores),
                                 ('raw_logits', raw_logits)])
    _call('g4r_sample_tokens_out_bf16', rows.device, _L.ptr(rows), rows.stride(0), B, V, float(temperature),
          int(top_k), float(top_p), int(bool(greedy)), int(seed) & 0xFFFFFFFFFFFFFFFF, _L.ptr(rng_step), int(eos_id),
          int(pad_id), _L.ptr(finished), _L.ptr(out), _L.ptr(history), ld_h, int(L), float(repetition_penalty),
          int(no_repeat_ngram_size), int(min_length), int(min_new_tokens), _L.ptr(eos_ids) if n_eos else None, n_eos,
          int(bool(append)), _L.ptr(scores), _L.ptr(raw_logits), n_slots, act=act)
    return out


def stop_step(ids, table, state, finished):
    """Stop strings, one step: every row b with finished[b] == 0 advances its matcher state by the token ids[b] through
    table (int16 [V_tok + 1, S], engine.StopStrings) and sets finished[b] when an occurrence of a stop string ended in
    that token.  ids: int64, B contiguous elements (the decode step's ids buffer, after sample_tokens); state, finished:
    contiguous device int32 [B], updated in place."""
    B = ids.numel()
    if ids.dtype != torch.int64 or not ids.is_contiguous():
        raise RuntimeError('stop_step: ids must be a contiguous int64 tensor')
    if table.dtype != torch.int16 or table.dim() != 2 or table.stride(1) != 1 or table.shape[0] < 2:
        raise RuntimeError('stop_step: table must be an int16 [V_tok + 1, S] tensor with unit column stride')
    for name, t in (('state', state), ('finished', finished)):
        if t.dtype != torch.int32 or t.numel() != B or not t.is_contiguous():
            raise RuntimeError('stop_step: %s must be a contiguous device int32 [%d] vector' % (name, B))
    _L.require_cuda_same_device([('ids', ids), ('table', table), ('state', state), ('finished', finished)])
    _call('g4r_stop_step', ids.device, _L.ptr(ids), _L.ptr(table), table.stride(0), table.shape[0] - 1, table.shape[1],
          B, _L.ptr(state), _L.ptr(finished))
    return finished


def stop_step_rows(ids, tables, n_states, V_tok, active, state, finished):
    """stop_step with a table per row (include/gpt4roi_b200.h: g4r_stop_step_rows): every row b with active[b] != 0,
    finished[b] == 0 and a table advances its matcher state by the token ids[b] through its table and sets finished[b]
    on a hit.  tables: a contiguous device int64 [B] vector of table addresses (0: the row has no stop strings), row b's
    an int16 [V_tok + 1, n_states[b]] contiguous tensor (engine.StopStrings) the caller keeps alive; V_tok is shared.
    ids: int64, B contiguous elements; n_states, active, state, finished: contiguous device int32 [B]."""
    B = ids.numel()
    if ids.dtype != torch.int64 or not ids.is_contiguous():
        raise RuntimeError('stop_step_rows: ids must be a contiguous int64 tensor')
    if int(V_tok) < 1:
        raise RuntimeError('stop_step_rows: V_tok must be >= 1, got %d' % V_tok)
    named = [('tables', tables, torch.int64), ('n_states', n_states, torch.int32), ('active', active, torch.int32),
             ('state', state, torch.int32), ('finished', finished, torch.int32)]
    for name, t, dt in named:
        if t is None or t.dtype != dt or t.numel() != B or not t.is_contiguous():
            raise RuntimeError('stop_step_rows: %s must be a contiguous device %s [%d] vector' % (name, dt, B))
    _L.require_cuda_same_device([('ids', ids)] + [(n, t) for n, t, _ in named])
    _call('g4r_stop_step_rows', ids.device, _L.ptr(ids), _L.ptr(tables), _L.ptr(n_states), int(V_tok), B,
          _L.ptr(active), _L.ptr(state), _L.ptr(finished))
    return finished


def lookup_step(st, sel=None):
    """Prompt-lookup decoding, one launch (csrc/lookup.cu): with sel (the verify step's selected tokens, int64 [M]) the
    acceptance of transformers' _assisted_decoding and then the next draft (g4r_lookup_step); without, the draft alone
    (g4r_lookup_draft, after the prefill's first token).  st: an engine.LookupDecode -- its device buffers ids, hist,
    state, base, pos, step, eos, readback and its k, max_ngram, prompt_len, max_length."""
    M = st.k + 1
    named = [('ids', st.ids, torch.int64, M), ('state', st.state, torch.int32, 5), ('base', st.base, torch.int32, 1),
             ('pos', st.pos, torch.int32, M), ('step', st.step, torch.int64, M),
             ('readback', st.readback, torch.int64, 4 + M + st.k)]
    if sel is not None:
        named.append(('sel', sel, torch.int64, M))
    for name, t, dt, n in named:
        if t.dtype != dt or t.numel() != n or not t.is_contiguous():
            raise RuntimeError('lookup_step: %s must be a contiguous device %s tensor of %d elements' % (name, dt, n))
    h = st.hist
    if h.dtype != torch.int64 or not h.is_contiguous() or h.numel() < st.max_length:
        raise RuntimeError('lookup_step: hist must be a contiguous int64 tensor of >= %d elements' % st.max_length)
    n_eos = 0 if st.eos is None else st.eos.numel()
    _L.require_cuda_same_device([('hist', h), ('eos', st.eos)] + [(n, t) for n, t, _, _ in named])
    tail = (_L.ptr(st.eos), n_eos, _L.ptr(st.state), _L.ptr(st.base), _L.ptr(st.pos), _L.ptr(st.step),
            _L.ptr(st.readback))
    if sel is None:
        _call('g4r_lookup_draft', h.device, _L.ptr(st.ids), _L.ptr(h), h.numel(), st.k, st.max_ngram, st.prompt_len,
              st.max_length, *tail)
    else:
        _call('g4r_lookup_step', h.device, _L.ptr(sel), _L.ptr(st.ids), _L.ptr(h), h.numel(), st.k, st.max_ngram,
              st.prompt_len, st.max_length, *tail)


def kv_append(qkv, kcache, vcache, B, Ln, pos0, pos_dev=None, pos_rows=None, cache_rows=None, qlen=None):
    """Copy the k|v parts of packed qkv rows [B*Ln, 3*HD] into caches [B, Lmax, HD] at pos0..pos0+Ln-1.
    pos_rows: device int32 [B] -- sample b's rows go to pos_rows[b]..pos_rows[b]+Ln-1 instead (pos0 / pos_dev unused).
    cache_rows (with pos_rows and qlen, device int32 [B]): the caches are [rows, Lmax, HD] (any number of rows) and only
    sample b's first qlen[b] rows are written, to cache row cache_rows[b] at pos_rows[b].. (g4r_kv_append_rows_at_bf16)."""
    HD = kcache.shape[-1]
    act = _bf16(qkv, kcache, vcache)
    if cache_rows is not None:
        if pos_rows is None or qlen is None:
            raise ValueError('kv_append: cache_rows needs pos_rows and qlen')
        _call('g4r_kv_append_rows_at_bf16', qkv.device, _L.ptr(qkv), qkv.stride(0), _L.ptr(kcache), _L.ptr(vcache), B,
              Ln, _L.ptr(_L.require_pos_rows(pos_rows, B)), _L.ptr(_L.require_pos_rows(cache_rows, B)),
              _L.ptr(_L.require_pos_rows(qlen, B)), kcache.shape[1], HD, act=act)
        return
    if pos_rows is not None:
        _call('g4r_kv_append_rows_bf16', qkv.device, _L.ptr(qkv), qkv.stride(0), _L.ptr(kcache), _L.ptr(vcache), B, Ln,
              _L.ptr(_L.require_pos_rows(pos_rows, B)), kcache.shape[1], HD, act=act)
        return
    _call('g4r_kv_append_bf16', qkv.device, _L.ptr(qkv), qkv.stride(0), _L.ptr(kcache), _L.ptr(vcache), B, Ln,
          int(pos0), _L.ptr(pos_dev), kcache.shape[1], HD, act=act)


def decode_attention(qkv, kcache, vcache, B, n_heads, head_dim, kv_len, scale, pos_dev=None, pos_rows=None):
    """qkv [B, 3*HD] (one new token per sample); caches [B, Lmax, HD]; returns [B, HD].
    pos_rows: device int32 [B] -- sample b attends over its first pos_rows[b] + 1 keys; kv_len is then only the bound
    (>= every row's length) that sizes the split and the score buffer."""
    act = _bf16(qkv, kcache, vcache)
    out = torch.empty((B, n_heads * head_dim), dtype=act, device=qkv.device)
    if pos_rows is not None:
        _call('g4r_decode_attention_rows_bf16', qkv.device, _L.ptr(qkv), qkv.stride(0), _L.ptr(kcache), _L.ptr(vcache),
              _L.ptr(out), out.stride(0), B, n_heads, head_dim, int(kv_len), _L.ptr(_L.require_pos_rows(pos_rows, B)),
              kcache.shape[1], float(scale), act=act)
        return out
    _call('g4r_decode_attention_bf16', qkv.device, _L.ptr(qkv), qkv.stride(0), _L.ptr(kcache), _L.ptr(vcache),
          _L.ptr(out), out.stride(0), B, n_heads, head_dim, int(kv_len), _L.ptr(pos_dev), kcache.shape[1], float(scale),
          act=act)
    return out


def decode_attention_beam(qkv, kcache, vcache, R, n_heads, head_dim, kv_bound, scale, pos_rows, anc):
    """Beam-search decode attention: qkv [R, 3*HD] (one new token per beam row); caches [rows, Lmax, HD] shared by all
    R rows; row r attends over positions 0..pos_rows[r], reading position p from cache row anc[r, p] (anc: device int32
    [R, Lmax]).  kv_bound (>= every pos_rows[r] + 1) sizes the split and the score buffer.  Returns [R, HD]."""
    act = _bf16(qkv, kcache, vcache)
    Lmax = kcache.shape[1]
    if anc.dtype != torch.int32 or tuple(anc.shape) != (R, Lmax) or not anc.is_contiguous():
        raise RuntimeError('decode_attention_beam: anc must be a contiguous device int32 [%d, %d] table' % (R, Lmax))
    out = torch.empty((R, n_heads * head_dim), dtype=act, device=qkv.device)
    _call('g4r_decode_attention_beam_bf16', qkv.device, _L.ptr(qkv), qkv.stride(0), _L.ptr(kcache), _L.ptr(vcache),
          _L.ptr(out), out.stride(0), R, n_heads, head_dim, int(kv_bound), _L.ptr(_L.require_pos_rows(pos_rows, R)),
          _L.ptr(anc), Lmax, float(scale), act=act)
    return out


GROUP_MAX_N = 16   # rows per prompt the shared-prefix decode attention supports (csrc/decode.cu)


def decode_attention_group(qkv, kcache, vcache, B, N, n_heads, head_dim, prompt_bound, gen_bound, scale, prompt_lens,
                           pos_rows):
    """Decode attention for N sampled rows per prompt sharing the prompt's keys: qkv [B*N, 3*HD] (row r = b*N + i);
    caches [B + B*N, Lmax, HD] -- rows 0..B-1 the prompts, row B + r row r's own generated positions.  Row r attends
    over positions 0..prompt_lens[b]-1 of cache row b and prompt_lens[b]..pos_rows[r] of cache row B + r (prompt_lens:
    device int32 [B], pos_rows: device int32 [B*N]).  prompt_bound / gen_bound (>= every prompt length / every row's
    count of own keys) size the split and the score buffer.  1 <= N <= 16 and head_dim 128.  Returns [B*N, HD]."""
    if not 1 <= N <= GROUP_MAX_N:
        raise ValueError('decode_attention_group: %d rows per prompt; the kernel supports 1..%d' % (N, GROUP_MAX_N))
    act = _bf16(qkv, kcache, vcache)
    if kcache.shape[0] != B + B * N or tuple(vcache.shape) != tuple(kcache.shape):
        raise RuntimeError('decode_attention_group: caches must hold %d rows (B prompts + B*N sample rows)' % (B + B * N))
    out = torch.empty((B * N, n_heads * head_dim), dtype=act, device=qkv.device)
    _call('g4r_decode_attention_group_bf16', qkv.device, _L.ptr(qkv), qkv.stride(0), _L.ptr(kcache), _L.ptr(vcache),
          _L.ptr(out), out.stride(0), int(B), int(N), n_heads, head_dim, int(prompt_bound), int(gen_bound),
          _L.ptr(_L.require_pos_rows(prompt_lens, B)), _L.ptr(_L.require_pos_rows(pos_rows, B * N)), kcache.shape[1],
          float(scale), act=act)
    return out


def beam_step(logits, row_div, st):
    """One beam-search step (csrc/beam.cu) on 16-bit logits [rows, V] (or [rows, 1, V]; unit column stride) with the
    device state of st (engine.BeamCache): B*N rows, or B with row_div = N (the first step, from the prefill).  When st
    holds output buffers (out_scores / out_logits: fp32 [n_slots, B*N, V]; bidx: int32 [2 (running, finished), 2, B, N,
    G] beam-index columns), the step also writes them (g4r_beam_step_out_bf16)."""
    rows, act = _logit_rows('beam_step', logits)
    V = rows.shape[1]
    B, N = st.n_samples, st.N
    if rows.shape[0] * row_div != B * N:
        raise RuntimeError('beam_step: logits must be [%d, V] rows' % (B * N // row_div))
    _L.require_cuda_same_device([('logits', rows), ('state', st.state), ('anc', st.anc)])
    scores, raw, bidx = st.out_scores, st.out_logits, st.bidx
    if scores is not None or raw is not None or bidx is not None:
        n_slots = max(_slot_buffer('beam_step: scores', scores, B * N, V),
                      _slot_buffer('beam_step: raw_logits', raw, B * N, V))
        if scores is not None and raw is not None and scores.shape[0] != raw.shape[0]:
            raise RuntimeError('beam_step: scores and raw_logits must hold the same number of slots')
        shape = (2, 2, B, N, st.G)
        if bidx is not None and (bidx.dtype != torch.int32 or tuple(bidx.shape) != shape or not bidx.is_contiguous()):
            raise RuntimeError('beam_step: the beam indices must be a contiguous int32 %s tensor' % (shape,))
        _L.require_cuda_same_device([('logits', rows), ('scores', scores), ('raw_logits', raw), ('beam_indices', bidx)])
        _call('g4r_beam_step_out_bf16', rows.device, _L.ptr(rows), rows.stride(0), int(row_div), B, N, V, st.K,
              _L.ptr(st.eos), st.n_eos, st.prompt_len, st.max_length, float(st.length_penalty), st.early, st.G, st.Lmax,
              _L.ptr(st.prompt_lens), _L.ptr(st.state), _L.ptr(st.run_score), _L.ptr(st.cand_score),
              _L.ptr(st.cand_tok), _L.ptr(st.run_seq), _L.ptr(st.fin_seq), _L.ptr(st.fin_score), _L.ptr(st.fin_state),
              _L.ptr(st.ids), _L.ptr(st.pos_rows), _L.ptr(st.anc), _L.ptr(scores), _L.ptr(raw), n_slots,
              None if bidx is None else _L.ptr(bidx[0]), None if bidx is None else _L.ptr(bidx[1]), act=act)
        return
    _call('g4r_beam_step_bf16', rows.device, _L.ptr(rows), rows.stride(0), int(row_div), B, N, V, st.K,
          _L.ptr(st.eos), st.n_eos, st.prompt_len, st.max_length, float(st.length_penalty), st.early, st.G, st.Lmax,
          _L.ptr(st.prompt_lens), _L.ptr(st.state), _L.ptr(st.run_score), _L.ptr(st.cand_score), _L.ptr(st.cand_tok),
          _L.ptr(st.run_seq), _L.ptr(st.fin_seq), _L.ptr(st.fin_score), _L.ptr(st.fin_state), _L.ptr(st.ids),
          _L.ptr(st.pos_rows), _L.ptr(st.anc), act=act)
