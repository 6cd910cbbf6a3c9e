"""Each attention kernel and its fp16 twin (csrc/act_type.cuh) against an fp64 restatement of the same operation on
the same 16-bit inputs, rounded where the kernel rounds: the wgmma (tc) and mma.sync prefill kernels, their training
forward with lse, the chunk attention over the KV cache, the split-KV decode kernels (scalar, device position,
per-row positions, beam ancestry, shared-prompt group) and the KV-cache append.

Notation as in test_infer_kernels_gpu.py: u = 2^-24 is the fp32 unit roundoff, u16 the storage type's; rd() rounds
to the storage type.  A kernel whose fp32 result lies within e32 of the fp64 `ref` and is rounded once returns a value
between rd(ref - e32) and rd(ref + e32) (`_check_rounded`).  The reference does not compute softmax(QK^T)V; it
replays where each kernel rounds P, so that e32 stays near fp32 size (_flash_ref, _decode_ref) and resolves a single
key admitted or dropped even on flat random inputs.

Planted inputs.  Every head gets a direction u of +-1 entries (one per sample, so a sample's bait cannot pass for its
neighbour's keys); the queries carry A_PL * u and chosen keys carry A_PL * u too, which puts their scaled scores
A_PL^2 sqrt(D) (4.5 at D = 64, 6.4 at D = 128) above the rest.  A kernel that admits or drops one such key moves an
output by O(|v|), far outside the bound.  Each planted case proves its own power: it recomputes the reference with
the edge moved by one key each way and asserts that the bound rejects that result (`_assert_rejects`).

Every output is filled with NaN before the call (`out=` of kernels.attention, or the entry point called through
`lib` with an output of our own), so an element the kernel never writes fails, and every launch is run twice and
must repeat bit for bit."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from gpt4roi_b200 import kernels
from gpt4roi_b200 import lib as _L

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
BF, H16, F32, F64 = torch.bfloat16, torch.float16, torch.float32, torch.float64
DTS = [pytest.param(BF, id='bf16'), pytest.param(H16, id='fp16')]
U = 2.0 ** -24
KBN = 64                      # key block of both flash kernels (kFaBN, kBN), aligned to key 0
A_PL = 0.75                   # planted query / key height along u
EDGE_L = [1, 63, 64, 65, 127, 128, 129, 257, 577, 706]
SEQLENS = [1, 64, 65, 137]    # plus L itself
INF = float('inf')


def bits(t):
    t = t.contiguous()
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def nan(shape, dt):
    return torch.full(shape, float('nan'), dtype=dt, device=DEV)


def ptr(t, offset_elems=0):
    return ctypes.c_void_p(t.data_ptr() + offset_elems * t.element_size())


def raw(name, dt, *args):
    """The entry point `name` (its fp16 twin for dt = fp16) called directly through the C ABI."""
    with torch.cuda.device(DEV):
        _L.check(getattr(_L.load(), _L.sym(name, dt))(*args, _L.stream_ptr(DEV)))


def sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def f32(x):
    """The fp32 value the kernels receive for a Python float argument."""
    return torch.tensor(x, dtype=F32).item()


def _check_rounded(got, ref, e32, dt, what=''):
    """rd(ref - e32) <= got <= rd(ref + e32); NaN (an unwritten sentinel) fails."""
    lo = (ref - e32).to(dt).double()
    hi = (ref + e32).to(dt).double()
    g = got.double()
    ok = (g >= lo) & (g <= hi)
    if not bool(ok.all()):
        i = tuple((~ok).nonzero()[0].tolist())
        raise AssertionError('%s: %d of %d outside [rd(ref - e32), rd(ref + e32)]; first at %s: got %r, want %r..%r'
                             % (what, int((~ok).sum()), ok.numel(), i, g[i].item(), lo[i].item(), hi[i].item()))


def _assert_rejects(mut, ref, e32, dt, what):
    """The planted case tells the kernel from a mutant: rd(mut), the output a kernel computing the mutant exactly would
    return, lies outside [rd(ref - e32), rd(ref + e32)] somewhere (or is NaN, as a row with no key is)."""
    m = mut.to(dt).double()
    inside = (m >= (ref - e32).to(dt).double()) & (m <= (ref + e32).to(dt).double())   # NaN: a row left keyless
    assert not bool(inside.all()), 'the bound cannot tell the kernel from its mutant: %s' % what


# ---------------------------------------------------------------------------------------------------------------
# References
# ---------------------------------------------------------------------------------------------------------------
def _tc_sum(n):
    """Relative error of a tensor-core fp32 sum of n exact products, per unit of sum|term|.  Each k16 step of
    mma.sync / wgmma adds 16 products to the accumulator after aligning all 17 addends to the largest exponent; NVIDIA
    documents no rounding for that alignment, so it may truncate: each addend loses < 2^-23 of the largest, together
    < 17 * 2u * max <= 34u * sum|addends|.  Over ceil(n / 16) steps: 34u ceil(n / 16) sum|term|."""
    return 34 * U * -(-n // 16)


def _flash_ref(q, k, v, mask, scale, dt, bound=True):
    """fp64 restatement of the flash kernels (attention_wgmma.cu, attention.cu): q [H, M, D], k / v [H, N, D] 16-bit,
    mask [M, N] (True: the query sees the key).  Keys go in 64-key blocks from key 0; after block t the running max
    is m_t (exact scores s = q.k); P is rounded relative to it and rescaled by the alphas:
        p_j = exp(scale (s_j - m_t(j))),  A_j = exp(scale (m_t(j) - m_final)),  l = sum_j p_j A_j  (unrounded p),
        O = sum_j rd(p_j) A_j v_j / l,  rounded once.
    Returns (O, e32) [H, M, D], e32 the kernel's fp32 error before that rounding:
      * score: s'_j within d_j = _tc_sum(D) sum_d |q_d k_jd|; the running max m' within max_j d_j;
      * p' = exp2f(fmaf(s', c, -rd(m' c))), c = rd(scale * rd(log2 e)) (2u): the argument is within
        scale (d_j + max d) + 8u scale max|s| (c's 2u on |s - m|, rd(m c), the fma), exp2f 2 ulp (4u):
        eps_j = scale (d_j + max d) + 8u scale max|s| + 4u relative;
      * rounding flips: rd(p'_j) lies between rd(p_j (1 - eps_j)) and rd(p_j (1 + eps_j)) (rounding is monotone), so
        the numerator's P error is at most sum_j (rd(p_j (1 + eps_j)) - rd(p_j (1 - eps_j))) A_j |v_j| / l, one extra
        matmul; with fp16 a P below 2^-14 is subnormal, whose step is an absolute 2^-24: 2^-25 sum_j A_j |v_j| / l
        more;
      * the alphas: each exp2f 4u and the o *= alpha product u per block, their arguments as p's: eps_A = 2 scale
        max d + 8u scale max|s| + 5u nblk;
      * l: the p' (max eps), the alphas, and an fp32 chain of at most N + 2 nblk + 2 adds (each thread sums its 16
        keys of a block into l_run, l_run *= alpha, two quad shuffles);
      * P V: _tc_sum(64) per block plus the accumulator's carry, (136 + 1) u nblk with the alpha product; 1 / l and
        o * inv: 2u.  Together eta = max eps + 2 eps_A + (N + 2 nblk + 2)u + 137u nblk + 2u on sum rd(p) A |v| / l.
    All these relative errors are below 2^-8, so their products, left out above, add less than 2^-8 of the sum:
    e32 carries a factor 1 + 2^-8."""
    H, M, D = q.shape
    N = k.shape[1]
    nb = -(-N // KBN)
    qd, kd, vd = q.double(), k.double(), v.double()
    s = (qd @ kd.mT).masked_fill(~mask, -INF)
    mt = F.pad(s, (0, nb * KBN - N), value=-INF).view(H, M, nb, KBN).amax(-1).cummax(-1).values
    mj = torch.where(mask, mt.repeat_interleave(KBN, -1)[..., :N], 0.0)
    p = torch.where(mask, torch.exp(scale * (s - mj)), 0.0)
    A = torch.where(mask, torch.exp(scale * (mj - mt[..., -1:])), 0.0)
    l = (p * A).sum(-1, keepdim=True)
    pr = p.to(dt).double()
    ref = ((pr * A) @ vd) / l
    if not bound:
        return ref, None
    d = _tc_sum(D) * (qd.abs() @ kd.abs().mT).masked_fill(~mask, 0.0)
    dmax = d.amax(-1, keepdim=True)
    smax = s.abs().masked_fill(~mask, 0.0).amax(-1, keepdim=True)
    eps = (scale * (d + dmax) + 8 * U * scale * smax + 4 * U).masked_fill(~mask, 0.0)
    eps_a = 2 * scale * dmax + 8 * U * scale * smax + 5 * U * nb
    eta = eps.amax(-1, keepdim=True) + 2 * eps_a + (N + 2 * nb + 2) * U + 137 * U * nb + 2 * U
    assert float(eta.max()) < 2 ** -8
    flip = (p * (1 + eps)).to(dt).double() - (p * (1 - eps)).to(dt).double()
    av = vd.abs()
    e = flip * A @ av + eta * ((pr * A) @ av)
    if dt == H16:
        e = e + 2.0 ** -25 * (A @ av)
    return ref, e * (1 + 2.0 ** -8) / l


def _flash_ref_heads(q, k, v, mask, scale, dt, bound=True, chunk=8):
    """_flash_ref in chunks of heads, so the [H, M, N] fp64 temporaries stay a few hundred MB."""
    outs = [_flash_ref(q[h:h + chunk], k[h:h + chunk], v[h:h + chunk], mask, scale, dt, bound)
            for h in range(0, q.shape[0], chunk)]
    return torch.cat([o[0] for o in outs]), (torch.cat([o[1] for o in outs]) if bound else None)


def _decode_ref(q, k, v, scale, dt, bound=True):
    """fp64 restatement of the decode kernels (decode.cu) for one query row: q [H, D], k / v [H, N, D], the row's keys
    in order.  They round P after normalising it, as HF's eager attention does: O = sum_j rd(P_j) v_j, P = softmax
    of the exact scaled scores, rounded once.  e32:
      * score: q is scaled and rounded to fp32 first (u), then each lane sums 8 products of its 16-byte slice (at most
        3 roundings per pair: 12) and 4 shuffle levels: d_j = 17u scale sum_d |q_d k_jd|;
      * p' = __expf(s' - gmax'): the subtraction u|x| and __expf's 2 + 1.16|x| ulp (ulp <= 2u), |x| <= 2 max|s|:
        (4 + 7 max|s|)u; P_j = p_j / sum p moves by d_j + max d through the scores;
      * the sum over the row's keys: per-thread partials, 5 shuffle levels, 8 warps, S <= 8 ranks: (N + 21)u;
        1 / sum and the product: 2u;  eps = d_j + max d + (4 + 7 max|s|)u + (N + 23)u;
      * rounding flips as in _flash_ref: sum_j (rd(P_j (1 + eps)) - rd(P_j (1 - eps))) |v_j|, and for fp16 the
        subnormal half-step 2^-25 sum_j |v_j|;
      * P V on the CUDA cores: per-lane-group partials, the group partials (16 or 32) and the ranks (<= 8):
        (N + 40)u on sum rd(P) |v|.
    Factor 1 + 2^-8 for the products of these first-order terms, as in _flash_ref."""
    qd, kd, vd = q.double(), k.double(), v.double()
    N = kd.shape[1]
    s = scale * (kd @ qd[..., None])[..., 0]
    P = torch.softmax(s, -1)
    Pr = P.to(dt).double()
    ref = (Pr[:, None, :] @ vd)[:, 0]
    if not bound:
        return ref, None
    d = 17 * U * scale * (kd.abs() @ qd.abs()[..., None])[..., 0]
    smax = s.abs().amax(-1, keepdim=True)
    eps = d + d.amax(-1, keepdim=True) + (4 + 7 * smax) * U + (N + 23) * U
    assert float(eps.max()) < 2 ** -8
    flip = (P * (1 + eps)).to(dt).double() - (P * (1 - eps)).to(dt).double()
    av = vd.abs()
    e = (flip[:, None, :] @ av)[:, 0] + (N + 40) * U * (Pr[:, None, :] @ av)[:, 0]
    if dt == H16:
        e = e + 2.0 ** -25 * av.sum(1)
    return ref, e * (1 + 2.0 ** -8)


def _causal_mask(M, N, Lk, causal, qoff=0, shift=0):
    """[M, N]: query i (at position qoff + i) sees key j < Lk, and j <= qoff + i + shift when causal."""
    i = torch.arange(M, device=DEV)[:, None]
    j = torch.arange(N, device=DEV)[None, :]
    m = j < Lk
    return m & (j <= qoff + i + shift) if causal else m.expand(M, N)


def _dirs(n, H, D, g):
    """n x H directions of +-1 entries."""
    return (torch.randint(0, 2, (n, H, D), generator=g, device=DEV) * 2 - 1).float()


# ---------------------------------------------------------------------------------------------------------------
# Prefill: tc and mma, training forward
# ---------------------------------------------------------------------------------------------------------------
def _prefill_inputs(B, L, H, D, dt, seed, profile, lens, causal):
    """Packed qkv [B*L, 3*H*D] and the planted key set of each sample.
    planted:    the keys the mask edges of sample b turn on: its last valid key lens[b] - 1, the first masked one
                lens[b] (if < L), keys at 64-key tile edges (causal: each is the diagonal of its own row and the key
                just above the diagonal of the row before); and keys 0..63 of sample b + 1 along sample b's
                direction, which the flash kernels' tail tile of sample b reads.
    ascending:  key height rises along the keys (every block raises the running max, alpha != 1 each time);
    descending: falls (the first block holds the max);  random: no direction (scores of sigma ~ 0.5)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    u = _dirs(B + 1, H, D, g)
    a = 0.0 if profile == 'random' else A_PL
    q = torch.randn(B, L, H, D, generator=g, device=DEV) * 0.7 + a * u[:B, None]
    k = torch.randn(B, L, H, D, generator=g, device=DEV) * 0.7
    v = torch.randn(B, L, H, D, generator=g, device=DEV)
    hs = torch.zeros(B, L, device=DEV)
    planted = []
    if profile == 'planted':
        for b in range(B):
            Lk = lens[b]
            J = {Lk - 1} | ({Lk} if Lk < L else set())
            if causal:
                J |= {j for j in (0, 1, 62, 63, 64, 65, 127, 128, 129, 256, 257, 575, 576, 704, 705) if j < L}
            planted.append(sorted(J))
            hs[b, sorted(J)] = A_PL
            if b + 1 < B:   # bait for sample b in sample b + 1's first tile
                k[b + 1, :KBN] += A_PL * u[b][None]
    elif profile in ('ascending', 'descending'):
        ramp = torch.arange(L, device=DEV) / max(L - 1, 1)
        hs[:] = (ramp if profile == 'ascending' else 1 - ramp) * 8 / (A_PL * D ** 0.5)
    k += hs[:, :, None, None] * u[:B, None]
    qkv = torch.cat([t.reshape(B * L, H * D) for t in (q, k, v)], 1).to(dt).contiguous()
    return qkv, planted


def _heads(t, B, L, H, D, part):
    """Sample-major [B, H, L, D] view of part 0 / 1 / 2 (q / k / v) of packed rows, or of an output (part None)."""
    x = t if part is None else t[:, part * H * D:(part + 1) * H * D]
    return x.reshape(B, L, H, D).permute(0, 2, 1, 3)


def _run_prefill(launch, B, L, H, D, causal, dt, seed, profile, lens=None, what=''):
    """launch(qkv, out, seqlens) on NaN-filled outputs twice (bitwise repeatable), then every sample against
    _flash_ref; rows >= lens[b] only finite.  Planted profiles assert the discrimination of each mask edge."""
    scale = f32(D ** -0.5)
    ragged = lens is not None
    lens = lens if ragged else [L] * B
    qkv, planted = _prefill_inputs(B, L, H, D, dt, seed, profile, lens, causal)
    seq = torch.tensor(lens, dtype=torch.int32, device=DEV) if ragged else None
    out = nan((B * L, H * D), dt)
    launch(qkv, out, seq)
    again = nan((B * L, H * D), dt)
    launch(qkv, again, seq)
    assert torch.equal(bits(out), bits(again)), '%s: two runs differ' % what
    Q, K, V = (_heads(qkv, B, L, H, D, i) for i in (0, 1, 2))
    O = _heads(out, B, L, H, D, None)
    for b in range(B):
        Lk = lens[b]
        M = Lk if ragged else L
        w = '%s %s b=%d Lk=%d' % (what, profile, b, Lk)
        assert torch.isfinite(O[b]).all(), '%s: non-finite output' % w
        mask = _causal_mask(M, L, Lk, causal)
        ref, e32 = _flash_ref_heads(Q[b, :, :M], K[b], V[b], mask, scale, dt)
        _check_rounded(O[b, :, :M], ref, e32, dt, w)
        if profile != 'planted':
            continue

        def mut(mask_m, k=K[b], v=V[b]):
            return _flash_ref_heads(Q[b, :, :M], k, v, mask_m, scale, dt, bound=False)[0]
        _assert_rejects(mut(_causal_mask(M, L, Lk - 1, causal)), ref, e32, dt, w + ': last key dropped')
        if causal:
            pass   # a key past the bound lies above the diagonal of every checked row: the causal mask hides it
        elif Lk < L:
            _assert_rejects(mut(_causal_mask(M, L, Lk + 1, causal)), ref, e32, dt, w + ': key Lk admitted')
        else:
            # one key past the sample: the next sample's key 0 (the tc kernel's TMA tile) or a second copy of key
            # L - 1 (the mma kernel clamps its tail loads)
            ext = _causal_mask(M, L + 1, L + 1, False)
            if b + 1 < B:
                _assert_rejects(mut(ext, torch.cat([K[b], K[b + 1, :, :1]], 1), torch.cat([V[b], V[b + 1, :, :1]], 1)),
                                ref, e32, dt, w + ': next sample key 0 admitted')
            if Lk > 1:   # a second copy of a row's only key leaves its softmax unchanged
                _assert_rejects(mut(ext, torch.cat([K[b], K[b, :, -1:]], 1), torch.cat([V[b], V[b, :, -1:]], 1)),
                                ref, e32, dt, w + ': duplicate of key L-1 admitted')
        if causal and M > 1:
            for sh, name in ((-1, 'diagonal dropped'), (1, 'key above the diagonal admitted')):
                _assert_rejects(mut(_causal_mask(M, L, Lk, True, shift=sh)), ref, e32, dt, w + ': ' + name)


def _attn(impl, B, L, H, D, causal):
    def launch(qkv, out, seq):
        kernels.attention(qkv, B, L, H, D, causal, f32(D ** -0.5), out=out, seqlens=seq, impl=impl)
    return launch


def _attn_lse(impl, B, L, H, D, causal):
    """The training forward (bf16 only) through the C ABI, with a NaN-filled lse that must come back finite."""
    name = 'g4r_attention_tc_lse_bf16' if impl == 'tc' else 'g4r_attention_fwd_lse_bf16'

    def launch(qkv, out, seq):
        assert seq is None
        hd = H * D
        lse = nan((B, H, L), F32)
        raw(name, BF, ptr(qkv), ptr(qkv, hd), ptr(qkv, 2 * hd), ptr(out), qkv.stride(0), L * qkv.stride(0), hd,
            L * hd, B, H, L, D, int(causal), f32(D ** -0.5), ptr(lse))
        assert torch.isfinite(lse).all()
    return launch


@pytest.mark.parametrize('dt', DTS)
@pytest.mark.parametrize('causal', [False, True], ids=['full', 'causal'])
@pytest.mark.parametrize('D', [64, 128])
@pytest.mark.parametrize('L', EDGE_L)
@pytest.mark.parametrize('impl', ['tc', 'mma'])
def test_prefill_attention_edges(impl, L, D, causal, dt):
    """Every tile edge of both prefill kernels, H = 2: planted keys at the key bound and the causal diagonal, B = 3
    (samples 0 and 1 have their neighbour's first tile baited); seqlens {1, 64, 65, 137, L} (clipped to L) in one
    ragged batch; ascending and descending score ramps."""
    H = 2
    what = '%s L=%d D=%d causal=%d' % (impl, L, D, causal)
    _run_prefill(_attn(impl, 3, L, H, D, causal), 3, L, H, D, causal, dt, L + D, 'planted', what=what)
    lens = [min(s, L) for s in SEQLENS + [L]]
    _run_prefill(_attn(impl, 5, L, H, D, causal), 5, L, H, D, causal, dt, L + D + 1, 'planted', lens, what)
    for prof in ('ascending', 'descending'):
        _run_prefill(_attn(impl, 2, L, H, D, causal), 2, L, H, D, causal, dt, L + D + 2, prof, what=what)


@pytest.mark.parametrize('dt', DTS)
@pytest.mark.parametrize('impl', ['tc', 'mma'])
@pytest.mark.parametrize('shape', ['vit257', 'vit577', 'llama706'])
def test_prefill_attention_engine_shapes(shape, impl, dt):
    """The engine's shapes on random inputs and planted ones: ViT (B 8, T 257 / 577, H 16, D 64, full) and the LLaMA
    prefill (B 2, L 706, H 32, D 128, causal), the latter also ragged (seqlens 706 and 451)."""
    B, L, H, D, causal = {'vit257': (8, 257, 16, 64, False), 'vit577': (8, 577, 16, 64, False),
                          'llama706': (2, 706, 32, 128, True)}[shape]
    for prof in ('random', 'planted'):
        _run_prefill(_attn(impl, B, L, H, D, causal), B, L, H, D, causal, dt, L, prof, what=shape)
    if causal:
        _run_prefill(_attn(impl, B, L, H, D, causal), B, L, H, D, causal, dt, L + 1, 'planted', [706, 451], shape)


@pytest.mark.parametrize('impl', ['tc', 'mma'])
@pytest.mark.parametrize('L', EDGE_L + ['trainer'])
def test_training_forward_output(L, impl):
    """The O of the training forward (attention_fwd_lse on either kernel, bf16), which the backward's delta is computed
    from and the training tests never check: the trainer shape (B 4, L 706, H 32, D 128, causal), random and
    planted, and the tile-edge L values planted at H 2, B 3."""
    if L == 'trainer':
        B, L, H = 4, 706, 32
        profiles = ('random', 'planted')
    else:
        B, H = 3, 2
        profiles = ('planted',)
    for prof in profiles:
        _run_prefill(_attn_lse(impl, B, L, H, 128, True), B, L, H, 128, True, BF, L + 7, prof,
                     what='%s lse L=%d' % (impl, L))


# ---------------------------------------------------------------------------------------------------------------
# Chunk attention over the KV cache
# ---------------------------------------------------------------------------------------------------------------
STARTS = [0, 1, 63, 64, 65, 700, 2000]


@pytest.mark.parametrize('dt', DTS)
@pytest.mark.parametrize('D', [64, 128])
@pytest.mark.parametrize('Lc', [1, 17, 128, 129, 300])
def test_attention_cached_edges(Lc, D, dt):
    """g4r_attention_cached: one row per start in {0, 1, 63, 64, 65, 700, 2000}, H 2, qlen Lc on even rows and
    1 / 17 / 129 (clipped to Lc) on odd ones.  Query i of row b sits at position start + i and sees keys
    0 .. start + i, in 64-key blocks aligned to position 0 (_flash_ref with the causal mask offset by start).
    Planted keys: start - 1, start, start + 1, the 64-aligned block edges around start, start + i and start + i + 1
    for i at the chunk's tile edges, and start + qlen, which no valid query sees.  The rest of the cache holds
    finite random keys.  Rows >= qlen are finite; 128-row tiles wholly past qlen are +0 bit for bit."""
    B, H = len(STARTS), 2
    HD = H * D
    Lmax = 2368
    scale = f32(D ** -0.5)
    qlens = [Lc if b % 2 == 0 else min(Lc, (1, 17, 129)[b // 2 % 3]) for b in range(B)]
    g = torch.Generator(device=DEV).manual_seed(Lc * 3 + D)
    u = _dirs(B, H, D, g)
    q = torch.randn(B, Lc, H, D, generator=g, device=DEV) * 0.7 + A_PL * u[:, None]
    kc = torch.randn(B, Lmax, H, D, generator=g, device=DEV) * 0.7
    vc = torch.randn(B, Lmax, H, D, generator=g, device=DEV)
    for b, st in enumerate(STARTS):
        a0 = st // KBN * KBN
        J = {st - 1, st, st + 1, a0 - 1, a0, a0 + KBN - 1, a0 + KBN, st + qlens[b]}
        J |= {st + i + e for i in (0, 16, 63, 64, 127, 128, 255, 256, Lc - 1) for e in (0, 1)}
        J = sorted(j for j in J if 0 <= j < Lmax)
        kc[b, J] += A_PL * u[b][None]
    qkv = torch.cat([q.reshape(B * Lc, HD), torch.zeros(B * Lc, 2 * HD, device=DEV)], 1).to(dt).contiguous()
    kc, vc = kc.reshape(B, Lmax, HD).to(dt).contiguous(), vc.reshape(B, Lmax, HD).to(dt).contiguous()
    start = torch.tensor(STARTS, dtype=torch.int32, device=DEV)
    qlen = torch.tensor(qlens, dtype=torch.int32, device=DEV)

    def launch():
        out = nan((B * Lc, HD), dt)
        raw('g4r_attention_cached_bf16', dt, ptr(qkv), qkv.stride(0), ptr(kc), ptr(vc), Lmax, ptr(out), out.stride(0),
            B, H, Lc, D, scale, ptr(start), ptr(qlen))
        return out
    out = launch()
    assert torch.equal(bits(out), bits(launch()))
    O = out.view(B, Lc, H, D).permute(0, 2, 1, 3)
    for b, st in enumerate(STARTS):
        ql = qlens[b]
        w = 'cached Lc=%d D=%d start=%d qlen=%d' % (Lc, D, st, ql)
        assert torch.isfinite(O[b]).all(), w
        for t0 in range(0, Lc, 128):
            if t0 >= ql:
                assert bool((bits(O[b, :, t0:t0 + 128]) == 0).all()), w + ': tile %d past qlen not zero' % t0
        N = min(Lmax, st + ql + 1)
        Qb = q[b, :ql].permute(1, 0, 2).to(dt)
        Kb = kc[b, :N].view(N, H, D).permute(1, 0, 2)
        Vb = vc[b, :N].view(N, H, D).permute(1, 0, 2)
        ref, e32 = _flash_ref_heads(Qb, Kb, Vb, _causal_mask(ql, N, N, True, st), scale, dt)
        _check_rounded(O[b, :, :ql], ref, e32, dt, w)
        for sh, name in ((-1, 'key start + i dropped'), (1, 'key start + i + 1 admitted')):
            mut = _flash_ref_heads(Qb, Kb, Vb, _causal_mask(ql, N, N, True, st, sh), scale, dt, bound=False)[0]
            _assert_rejects(mut, ref, e32, dt, '%s: %s' % (w, name))


# ---------------------------------------------------------------------------------------------------------------
# Decode attention: split-KV clusters
# ---------------------------------------------------------------------------------------------------------------
def _split(H, B, bound):
    """Cluster size S of the decode launchers (launch_decode_attention, g4r_decode_attention_group_bf16)."""
    S = 1
    while S < 8 and H * B * S < 2 * sms() and bound // (2 * S) >= 64:
        S *= 2
    return S


def _slice_edges(n, S):
    """First and last key of every non-empty rank slice of a row with n keys split S ways (per = ceil(n / S))."""
    per = -(-n // S)
    return sorted({j for r in range(S) if r * per < n for j in (r * per, min(n, (r + 1) * per) - 1)})


def _slice_drop(n, S, first):
    """Key indices of a row of n keys without the first (or last) key of every slice: the mutant whose slices start
    one late (end one early)."""
    drop = set()
    per = -(-n // S)
    for r in range(S):
        if r * per < n:
            drop.add(r * per if first else min(n, (r + 1) * per) - 1)
    return [j for j in range(n) if j not in drop]


def _row_kv(cache, kl, H, D):
    """[H, n, D] keys (or values) of one query row from its (cache row, position) list."""
    return cache[[c for c, _ in kl], [p for _, p in kl]].view(-1, H, D).permute(1, 0, 2)


def _decode_rows(q, kc, vc, H, D, keys, dt, scale, bound=True):
    """Reference (and bound) of each query row r of packed q rows over its key list keys[r]; a row with no key is
    NaN, as the kernels' 0 * (1 / 0) would make it."""
    refs, es = [], []
    for r, kl in enumerate(keys):
        if not kl:
            refs.append(torch.full((H * D,), float('nan'), dtype=F64, device=DEV))
            continue
        ref, e = _decode_ref(q[r, :H * D].view(H, D), _row_kv(kc, kl, H, D), _row_kv(vc, kl, H, D), scale, dt, bound)
        refs.append(ref.reshape(-1))
        es.append(e.reshape(-1) if bound else None)
    return torch.stack(refs), (torch.stack(es) if bound else None)


def _decode_mutants(q, kc, vc, H, D, keys, dt, scale, ref, e32, muts, what):
    """muts: (name, f(r, keys of row r) -> the keys a mutant kernel would read); each must be rejected."""
    for name, mk in muts:
        mk_keys = [mk(r, kl) for r, kl in enumerate(keys)]
        if mk_keys == keys:   # e.g. own-key mutants where no row owns a key
            continue
        mut = _decode_rows(q, kc, vc, H, D, mk_keys, dt, scale, bound=False)[0]
        _assert_rejects(mut, ref, e32, dt, '%s: %s' % (what, name))


def _decode_cache(Bc, Lmax, H, D, dt, g):
    kc = torch.randn(Bc, Lmax, H, D, generator=g, device=DEV) * 0.7
    vc = torch.randn(Bc, Lmax, H, D, generator=g, device=DEV)
    return kc, vc


DECODE_LENS = [100, 200, 300, 1000]   # S = 1, 2, 4, 8 at H * B * 8 < 2 * num_sms


@pytest.mark.parametrize('dt', DTS)
@pytest.mark.parametrize('D', [64, 128])
@pytest.mark.parametrize('mode', ['host', 'pos_dev', 'rows'])
def test_decode_attention_split_edges(mode, D, dt):
    """g4r_decode_attention (host kv_len), with pos_dev (device position, host bound 1000) and _rows (per-row
    lengths 1, 5, 300, 1000 under the bound 1000), H 4.  S comes from the launcher's rule; the host cases reach
    S = 1, 2, 4, 8, the bound-1000 cases slice short rows so that ranks own no key.  Planted: the first and last key
    of every rank slice of each row, and its own (newest) key; the key after it is bait.  Mutants: the own key
    dropped, the bait admitted, every slice one key short at either end."""
    H, Lmax = 4, 1088
    HD = H * D
    scale = f32(D ** -0.5)
    g = torch.Generator(device=DEV).manual_seed(D + len(mode))
    if mode == 'host':
        cases = [(2, n, [n, n]) for n in DECODE_LENS]
    elif mode == 'pos_dev':
        cases = [(2, 1000, [n, n]) for n in (1, 5, 300, 1000)]
    else:
        cases = [(4, 1000, [1, 5, 300, 1000])]
    seen, empty = set(), False
    for B, bound, lens in cases:
        S = _split(H, B, bound)
        seen.add(S)
        empty |= any(r * -(-n // S) >= n for n in lens for r in range(S))
        u = _dirs(1, H, D, g)[0]
        kc, vc = _decode_cache(B, Lmax, H, D, dt, g)
        for b, n in enumerate(lens):
            kc[b, _slice_edges(n, S) + [n]] += A_PL * u[None]
        qkv = torch.cat([(torch.randn(B, H, D, generator=g, device=DEV) * 0.7 + A_PL * u).reshape(B, HD),
                         torch.zeros(B, 2 * HD, device=DEV)], 1).to(dt).contiguous()
        kc, vc = kc.reshape(B, Lmax, HD).to(dt).contiguous(), vc.reshape(B, Lmax, HD).to(dt).contiguous()
        pos_dev = torch.tensor([lens[0] - 1], dtype=torch.int32, device=DEV)
        rows = torch.tensor([n - 1 for n in lens], dtype=torch.int32, device=DEV)

        def launch():
            out = nan((B, HD), dt)
            if mode == 'rows':
                raw('g4r_decode_attention_rows_bf16', dt, ptr(qkv), qkv.stride(0), ptr(kc), ptr(vc), ptr(out),
                    out.stride(0), B, H, D, bound, ptr(rows), Lmax, scale)
            else:
                raw('g4r_decode_attention_bf16', dt, ptr(qkv), qkv.stride(0), ptr(kc), ptr(vc), ptr(out),
                    out.stride(0), B, H, D, bound, ptr(pos_dev) if mode == 'pos_dev' else None, Lmax, scale)
            return out
        out = launch()
        assert torch.equal(bits(out), bits(launch()))
        keys = [[(b, j) for j in range(n)] for b, n in enumerate(lens)]
        ref, e32 = _decode_rows(qkv, kc, vc, H, D, keys, dt, scale)
        w = 'decode %s D=%d S=%d lens=%s' % (mode, D, S, lens)
        _check_rounded(out, ref, e32, dt, w)
        muts = [('own key dropped', lambda r, kl: kl[:-1]),
                ('key after the own key admitted', lambda r, kl: kl + [(r, len(kl))]),
                ('slices end one key early', lambda r, kl: [kl[j] for j in _slice_drop(len(kl), S, False)]),
                ('slices start one key late', lambda r, kl: [kl[j] for j in _slice_drop(len(kl), S, True)])]
        _decode_mutants(qkv, kc, vc, H, D, keys, dt, scale, ref, e32, muts, w)
    if mode == 'host':
        assert seen == {1, 2, 4, 8}, seen
    else:
        assert empty


@pytest.mark.parametrize('dt', DTS)
@pytest.mark.parametrize('D', [64, 128])
def test_decode_attention_beam_ancestry(D, dt):
    """g4r_decode_attention_beam: R 4 beam rows over 8 shared cache rows, random ancestry anc[r, p] in 0..7, lengths
    7, 150, 400, 1000 under the bound 1000 (S 8).  Row r's planted keys sit at (anc[r, p], p) for its slice edges and
    its newest position, with anc[r, p] >= R there, so they are reachable only through the table: reading cache row
    r instead (an ignored ancestry) sees flat keys and is rejected."""
    R, Rc, H, Lmax, bound = 4, 8, 4, 1024, 1000
    HD = H * D
    scale = f32(D ** -0.5)
    lens = [7, 150, 400, 1000]
    g = torch.Generator(device=DEV).manual_seed(D + 11)
    S = _split(H, R, bound)
    u = _dirs(1, H, D, g)[0]
    kc, vc = _decode_cache(Rc, Lmax, H, D, dt, g)
    anc = torch.randint(0, Rc, (R, Lmax), generator=g, device=DEV, dtype=torch.int32)
    for r, n in enumerate(lens):
        J = torch.tensor(_slice_edges(n, S) + [n - 1], device=DEV)
        anc[r, J] = torch.randint(R, Rc, (len(J),), generator=g, device=DEV, dtype=torch.int32)
        kc[anc[r, J].long(), J] += A_PL * u[None]
    qkv = torch.cat([(torch.randn(R, H, D, generator=g, device=DEV) * 0.7 + A_PL * u).reshape(R, HD),
                     torch.zeros(R, 2 * HD, device=DEV)], 1).to(dt).contiguous()
    kc, vc = kc.reshape(Rc, Lmax, HD).to(dt).contiguous(), vc.reshape(Rc, Lmax, HD).to(dt).contiguous()
    rows = torch.tensor([n - 1 for n in lens], dtype=torch.int32, device=DEV)

    def launch():
        out = nan((R, HD), dt)
        raw('g4r_decode_attention_beam_bf16', dt, ptr(qkv), qkv.stride(0), ptr(kc), ptr(vc), ptr(out), out.stride(0),
            R, H, D, bound, ptr(rows), ptr(anc), Lmax, scale)
        return out
    out = launch()
    assert torch.equal(bits(out), bits(launch()))
    ac = anc.tolist()
    keys = [[(ac[r][p], p) for p in range(n)] for r, n in enumerate(lens)]
    ref, e32 = _decode_rows(qkv, kc, vc, H, D, keys, dt, scale)
    w = 'beam D=%d' % D
    _check_rounded(out, ref, e32, dt, w)
    muts = [('ancestry ignored', lambda r, kl: [(r, p) for _, p in kl]),
            ('slices end one key early', lambda r, kl: [kl[j] for j in _slice_drop(len(kl), S, False)])]
    _decode_mutants(qkv, kc, vc, H, D, keys, dt, scale, ref, e32, muts, w)


@pytest.mark.parametrize('dt', DTS)
@pytest.mark.parametrize('N', [1, 2, 3, 5, 7, 8, 16])
def test_decode_attention_group_edges(N, dt):
    """g4r_decode_attention_group, D 128, H 2, B 3 prompts of 5 (shorter than S = 8), 64 and 700 keys under the
    prompt bound 700; row i of a prompt owns (1, 0, 2, 9, 40)[i % 5] generated keys.  N = 3, 5, 7 leave lane groups
    without a query.  Planted: prompt key P - 1 and own key P (the prompt / own boundary); baits at prompt row
    position P, own row position P - 1 and own position pos + 1, which no valid read reaches.  Mutants: the prompt
    one key short or long, the own keys read one position early, one own key short or long."""
    B, H, D, Lmax = 3, 2, 128, 768
    HD = H * D
    scale = f32(D ** -0.5)
    plens = [5, 64, 700]
    own = [(1, 0, 2, 9, 40)[i % 5] for i in range(N)]
    gen_bound = max(own)
    g = torch.Generator(device=DEV).manual_seed(N)
    S = _split(H, B, 700)
    assert S == 8 and min(plens) < S
    u = _dirs(1, H, D, g)[0]
    kc, vc = _decode_cache(B + B * N, Lmax, H, D, dt, g)
    keys = []
    for b, P in enumerate(plens):
        kc[b, [P - 1, P]] += A_PL * u[None]
        for i in range(N):
            r = b * N + i
            n = own[i]
            kc[B + r, P - 1] += A_PL * u
            kc[B + r, P + n] += A_PL * u
            if n:
                kc[B + r, P] += A_PL * u
            keys.append([(b, j) for j in range(P)] + [(B + r, j) for j in range(P, P + n)])
    qkv = torch.cat([(torch.randn(B * N, H, D, generator=g, device=DEV) * 0.7 + A_PL * u).reshape(B * N, HD),
                     torch.zeros(B * N, 2 * HD, device=DEV)], 1).to(dt).contiguous()
    kc, vc = kc.reshape(-1, Lmax, HD).to(dt).contiguous(), vc.reshape(-1, Lmax, HD).to(dt).contiguous()
    pl = torch.tensor(plens, dtype=torch.int32, device=DEV)
    pos = torch.tensor([plens[r // N] - 1 + own[r % N] for r in range(B * N)], dtype=torch.int32, device=DEV)

    def launch():
        out = nan((B * N, HD), dt)
        raw('g4r_decode_attention_group_bf16', dt, ptr(qkv), qkv.stride(0), ptr(kc), ptr(vc), ptr(out), out.stride(0),
            B, N, H, D, 700, gen_bound, ptr(pl), ptr(pos), Lmax, scale)
        return out
    out = launch()
    assert torch.equal(bits(out), bits(launch()))
    ref, e32 = _decode_rows(qkv, kc, vc, H, D, keys, dt, scale)
    w = 'group N=%d' % N
    _check_rounded(out, ref, e32, dt, w)

    def split(r, kl):
        P = plens[r // N]
        return [x for x in kl if x[0] < B], [x for x in kl if x[0] >= B], P
    muts = [('prompt one key short', lambda r, kl: (lambda p, o, P: p[:-1] + o)(*split(r, kl))),
            ('prompt one key long', lambda r, kl: (lambda p, o, P: p + [(r // N, P)] + o)(*split(r, kl))),
            ('own keys one position early', lambda r, kl: (lambda p, o, P: p + [(B + r, j - 1) for _, j in o])(*split(r, kl))),
            ('one own key short', lambda r, kl: (lambda p, o, P: p + o[:-1])(*split(r, kl))),
            ('one own key long', lambda r, kl: (lambda p, o, P: p + o + [(B + r, P + len(o))])(*split(r, kl)))]
    _decode_mutants(qkv, kc, vc, H, D, keys, dt, scale, ref, e32, muts, w)


# ---------------------------------------------------------------------------------------------------------------
# KV-cache append
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dt', DTS)
@pytest.mark.parametrize('B,Ln,HD,Lmax', [(3, 1, 256, 64), (3, 5, 1024, 96), (8, 706, 4096, 1024)])
@pytest.mark.parametrize('mode', ['host', 'pos_dev', 'rows'])
def test_kv_append_places_rows_bitwise(mode, B, Ln, HD, Lmax, dt):
    """g4r_kv_append (host pos0 or device position) and _rows into NaN-filled caches: rows pos .. pos + Ln - 1 of
    each sample equal the k | v slices of its packed rows bit for bit, every other row keeps its NaN sentinel; the
    positions include 0 and the last legal one, Lmax - Ln.  B 8 x 706 rows of 4096 take several passes of the
    grid-stride loop."""
    g = torch.Generator(device=DEV).manual_seed(B * Ln + HD)
    qkv = torch.randn(B * Ln, 3 * HD + 64, generator=g, device=DEV).to(dt)[:, :3 * HD]
    last = Lmax - Ln
    if mode == 'rows':
        cases = [[(0, last, min(7, last))[b % 3] for b in range(B)]]
    else:
        cases = [[0] * B, [last] * B]
    for starts in cases:
        p0 = starts[0]
        kc, vc = nan((B, Lmax, HD), dt), nan((B, Lmax, HD), dt)
        if mode == 'rows':
            rows = torch.tensor(starts, dtype=torch.int32, device=DEV)
            raw('g4r_kv_append_rows_bf16', dt, ptr(qkv), qkv.stride(0), ptr(kc), ptr(vc), B, Ln, ptr(rows), Lmax, HD)
        elif mode == 'pos_dev':
            pd = torch.tensor([p0], dtype=torch.int32, device=DEV)
            raw('g4r_kv_append_bf16', dt, ptr(qkv), qkv.stride(0), ptr(kc), ptr(vc), B, Ln, 0, ptr(pd), Lmax, HD)
        else:
            raw('g4r_kv_append_bf16', dt, ptr(qkv), qkv.stride(0), ptr(kc), ptr(vc), B, Ln, p0, None, Lmax, HD)
        wk, wv = nan((B, Lmax, HD), dt), nan((B, Lmax, HD), dt)
        rows_ = qkv.view(B, Ln, 3 * HD)
        for b, s in enumerate(starts):
            wk[b, s:s + Ln] = rows_[b, :, HD:2 * HD]
            wv[b, s:s + Ln] = rows_[b, :, 2 * HD:]
        assert torch.equal(bits(kc), bits(wk)), 'k cache, starts %s' % starts
        assert torch.equal(bits(vc), bits(wv)), 'v cache, starts %s' % starts
