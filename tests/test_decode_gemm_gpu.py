"""The weight-streaming decode GEMM (csrc/gemm_skinny.cu) and its fp16 twin against an fp64 restatement of the same
operation on the same 16-bit inputs: every template instance `gemm_skinny()` selects, the decode step's five GEMMs at
every M = 1..16, the edge shapes of each instance, the fused RoPE + KV-cache epilogue and the host-side refusals.

Instances.  `gemm_skinny()` picks one of seven `gemm_skinny_bf16<MT, MB, WARPS, ROPE, DEPTH>` instances per dtype from
M, N and the SM count (`instance` restates the rule, with `wide_prefers_8_warps`).  `test_instances` launches every
case of the file at every row count it uses, through the same entry, in one CUDA profiler session per dtype, taken in
a child process: each launch must have run the instance the rule predicts, and together they must have launched all
seven.

Error bound.  Notation as in test_attention_kernels_gpu.py: u = 2^-24, rd() rounds to the storage type, and a kernel
whose fp32 result lies within e32 of the fp64 `ref` and is rounded once returns a value in [rd(ref - e32),
rd(ref + e32)] (`_check_rounded`).  For output (m, n) let y = sum_k x[m, k] W[n, k] and S = sum_k |x[m, k] W[n, k]|
(both in fp64).  The products of two 16-bit values are exact in fp32.
  * K chain: each warp accumulates its k-blocks with mma.sync m16n8k16, at most ceil(K / 16) steps:
    _tc_sum(K) S (the truncating-alignment bound of test_attention_kernels_gpu._tc_sum).
  * The WARPS partials are added in fixed order starting from 0: WARPS - 1 fp32 adds, each within u of its running
    sum, itself below S (1 + _tc_sum(K)): (WARPS - 1) u S.
    Together e_acc = (_tc_sum(K) + (WARPS - 1) u) S.
  * bias (16-bit or fp32, exact in fp32) and residual add: z = y + t is one fp32 add: e' = e + u (|z| + e).
  * relu: 1-Lipschitz and exact: e unchanged.
  * quick_gelu g(v) = v / (1 + __expf(-c v)), c = fp32(1.702): g(v) = silu(c v) / c, so |g'| <= max|silu'| < 1.1 and
    the input error costs 1.1 e.  __expf is within 2 + floor(1.173 |t|) ulp (2u each) of exp(t) (CUDA C Programming
    Guide, intrinsic functions); t = -c v is rounded once, which moves exp(t) by |t| u; 1 + E, the IEEE division:
    u each.  Relative error of the evaluation eps = (2 + 1.173 |t|) 2u + |t| u + 2u, on |g(v')| <= |g(z)| + 1.1 e:
    e' = 1.1 e + (|g(z)| + 1.1 e) eps.
  * SwiGLU out_j = silu(a) b with a = gate row 2j, b = up row 2j + 1 (each with its own e_a, e_b):
    gt / (1 + __expf(-gt)) * up: eps = (2 + 1.173 |a|) 2u + 3u (exp, 1 + E, division, product), so
    e' = 1.1 e_a (|b| + e_b) + |silu(a)| e_b + (|silu(a)| + 1.1 e_a)(|b| + e_b) eps.
All relative errors above are below 2^-10, so the products of two of them, left out, are below 2^-10 of the total:
e32 carries a factor 1 + 2^-8.

Layouts.  Outputs are written through `Canvas` (a view with padded row stride inside a NaN-filled buffer) in the
vector / odd / offset layouts of test_gemm_tiles_gpu._layouts, residuals are stored in the same layout inside NaN,
the activations have a row stride lda = K + 64 and the weights ldw = K + 32, both with the padding NaN-filled.  An
output row >= M or column >= N, an element never written, or a read past K or past a residual row shows as a
stored-outside-the-output failure, a NaN, or a value off the bound.

RoPE / KV cache.  The rotated q|k columns are checked bitwise against HF's rotate-half formula with the kernel's
rounding points, applied in torch to the kernel's own unrotated output: the plain launch of the instance with the same
WARPS and DEPTH (<2, MB, 4, false, 1>, whose own output meets the fp64 bound).  That launch reduces every output
element over the same k order and warp split as the RoPE instance, so its 16-bit output is bitwise the RoPE
epilogue's input; test_instances checks that premise.  The KV caches start NaN-filled: cache row (m, pos_m) must equal
the k / v output slices bitwise and every other element must be unchanged."""
import json
import os
import re
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from gpt4roi_b200 import dense, kernels
from gpt4roi_b200 import lib as _L
from tests.test_attention_kernels_gpu import U, _check_rounded, _tc_sum
from tests.test_gemm_tiles_gpu import Canvas, _layouts, rope_tables

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
BF, H16, F32, F64 = torch.bfloat16, torch.float16, torch.float32, torch.float64
DTS = [pytest.param(BF, id='bf16'), pytest.param(H16, id='fp16')]
SLACK = 1 + 2.0 ** -8
NAN_BITS = {BF: 0x7fc1, H16: 0x7e01}


def bits(t):
    return t.contiguous().view(torch.int16)


def nan(shape, dt):
    t = torch.empty(shape, dtype=dt, device=DEV)
    t.view(torch.int16).fill_(NAN_BITS[dt])
    return t


def raw(name, dt, *args):
    """The entry point `name` (its fp16 twin for dt = fp16) called directly through the C ABI."""
    with torch.cuda.device(DEV):
        _L.check(getattr(_L.load(), _L.sym(name, dt))(*args, _L.stream_ptr(torch.device(DEV))))


def sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


# ---- the selection rule and the profiler ----------------------------------------------------------------------

def prefers_8_warps(tiles, n_sms):
    """wide_prefers_8_warps: the CTA size (4 warps: 4 CTAs per SM, 8 warps: 2) whose last wave is the fuller."""
    w4, w8 = tiles / (4.0 * n_sms), tiles / (2.0 * n_sms)
    waste = lambda w: float(int(w + 0.999999)) / w
    return waste(w8) < 0.95 * waste(w4)


def instance(M, N, rope, n_sms):
    """gemm_skinny(): the (MT, MB, WARPS, ROPE, DEPTH) template arguments of the launch for M rows, N weight rows."""
    if rope:
        return (2, 1 if M <= 8 else 2, 4, True, 1)
    tiles = -(-N // 32)
    if tiles >= 2 * n_sms:    # 32-row tiles once they still give >= 2 CTAs per SM
        if M > 8:
            return (2, 2, 4, False, 1)
        return (2, 1, 8, False, 1) if prefers_8_warps(tiles, n_sms) else (2, 1, 4, False, 1)
    return (1, 1, 8, False, 2) if M <= 8 else (1, 2, 16, False, 1)


ALL_INSTANCES = {(2, 1, 4, True, 1), (2, 2, 4, True, 1), (1, 1, 8, False, 2), (1, 2, 16, False, 1),
                 (2, 1, 8, False, 1), (2, 1, 4, False, 1), (2, 2, 4, False, 1)}
_KERNEL = re.compile(r'\b(g4r|g4r_h)::gemm_skinny_bf16<(\d+), (\d+), (\d+), (true|false), (\d+)>')


def traced_instances(launches, dt):
    """Runs launches (a list of functions that each launch one GEMM and nothing else) in one CUDA profiler session
    and returns the (MT, MB, WARPS, ROPE, DEPTH) of the gemm_skinny_bf16 kernels of the trace in start order (namespace
    g4r: bf16, g4r_h: fp16; demangled as `void g4r::gemm_skinny_bf16<1, 1, 8, false, 2>(g4r::SkinnyParams)`).
    The profiler now and then returns an empty trace, or one a few records short, so a trace with fewer kernels than
    launches is taken again, up to three times in all."""
    ns = 'g4r' if dt == BF else 'g4r_h'
    for _ in range(3):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for go in launches:
                go()
            torch.cuda.synchronize()
        found = {}
        for e in prof.events():
            if 'gemm_skinny_bf16' in e.name:
                m = _KERNEL.search(e.name)
                assert m and m[1] == ns, 'cannot read the template arguments of kernel %r' % e.name
                found[e.time_range.start] = (int(m[2]), int(m[3]), int(m[4]), m[5] == 'true', int(m[6]))
        if len(found) == len(launches):
            break
    return [found[t] for t in sorted(found)]


def wide_tiles(n_sms, eight):
    """The smallest count of 32-row tiles that takes the wide path with 8 warps (eight) or 4 warps (not eight) at
    M <= 8."""
    t = 2 * n_sms
    while prefers_8_warps(t, n_sms) != eight:
        t += 1
    return t


# ---- operands and references ----------------------------------------------------------------------------------

class Operands:
    """Seeded operands of one (N, K) case for up to 16 rows, with the fp64 products y and sums S of all 16 rows.
    x is a [16, K] view with row stride K + 64 and W a [N, K] view with row stride K + 32, both padded with NaN."""

    def __init__(self, N, K, dt, seed, ref=True):
        g = torch.Generator(device=DEV).manual_seed(seed)
        self.N, self.K, self.dt = N, K, dt
        xb = nan((16, K + 64), dt)
        xb[:, :K] = torch.randn(16, K, generator=g, device=DEV).to(dt)
        self.x = xb[:, :K]
        wb = nan((N, K + 32), dt)
        wb[:, :K] = (torch.randn(N, K, generator=g, device=DEV) * K ** -0.5).to(dt)
        self.w = wb[:, :K]
        self.bias = (torch.randn(N, generator=g, device=DEV) * 0.5).to(dt)
        self.bias32 = torch.randn(N, generator=g, device=DEV) * 0.5
        self.res = torch.randn(16, N, generator=g, device=DEV).to(dt)
        if not ref:
            return
        xd = self.x.double()
        wd = self.w.double()
        self.y = xd @ wd.t()
        self.S = xd.abs() @ wd.abs().t()
        del wd


def _add(z, e, t):
    """One fp32 add of an exact addend t (bias or residual)."""
    s = z + t.double()
    return s, e + U * (s.abs() + e)


def _quick_gelu(z, e):
    c = torch.tensor(1.702, dtype=F32).item()
    g = z * torch.sigmoid(c * z)
    t = c * (z.abs() + e)
    eps = (2 + 1.173 * t) * 2 * U + t * U + 2 * U
    return g, 1.1 * e + (g.abs() + 1.1 * e) * eps


def _swiglu(a, ea, b, eb):
    sa = F.silu(a)
    eps = (2 + 1.173 * (a.abs() + ea)) * 2 * U + 3 * U
    bb = b.abs() + eb
    return sa * b, 1.1 * ea * bb + sa.abs() * eb + (sa.abs() + 1.1 * ea) * bb * eps


# epilogue -> (entry, bias, act, residual): 'decode' is g4r_decode_gemm_*, 'linear' dense.linear (gemm_impl), the
# entries the engine's decode step calls
EPILOGUES = {
    'none': ('decode', None, None, False),
    'residual': ('decode', None, None, True),
    'swiglu': ('decode', None, 'swiglu', False),
    'lin_none': ('linear', None, None, False),
    'lin_residual': ('linear', None, None, True),
    'lin_bias_relu': ('linear', 'bf16', 'relu', False),
    'lin_bias32_quick_gelu': ('linear', 'f32', 'quick_gelu', False),
    'lin_bias32_swiglu': ('linear', 'f32', 'swiglu', False),
    'lin_bias_residual': ('linear', 'bf16', None, True),
}
EDGE_EPILOGUES = ('none', 'residual', 'swiglu', 'lin_bias_relu', 'lin_bias32_quick_gelu', 'lin_bias32_swiglu',
                  'lin_bias_residual')


def reference(ep, o, M, warps):
    """(fp64 reference, e32) of epilogue ep for the first M rows, on `warps` warps per CTA."""
    _, bias, act, residual = EPILOGUES[ep]
    y, S = o.y[:M], o.S[:M]
    e = (_tc_sum(o.K) + (warps - 1) * U) * S
    z = y
    if bias is not None:
        z, e = _add(z, e, o.bias if bias == 'bf16' else o.bias32)
    if act == 'relu':
        z = torch.relu(z)
    elif act == 'quick_gelu':
        z, e = _quick_gelu(z, e)
    elif act == 'swiglu':
        z, e = _swiglu(z[:, 0::2], e[:, 0::2], z[:, 1::2], e[:, 1::2])
    if residual:
        z, e = _add(z, e, o.res[:M])
    return z, e * SLACK


def prepare(ep, o, M, layout):
    """A fresh canvas of the given layout (and the residual in the same layout, inside NaN) for epilogue ep on the
    first M rows, and the function that launches into it: (canvas, go).  go() only launches, so that a traced session
    holds nothing but the GEMM kernels."""
    entry, bias, act, residual = EPILOGUES[ep]
    N, K, dt = o.N, o.K, o.dt
    n_out = N // 2 if act == 'swiglu' else N
    _, ld, col0 = layout
    cv = Canvas(M, n_out, dt, ld, col0)
    res = None
    if residual:
        rc = Canvas(M, n_out, dt, ld, col0)
        rc.out.copy_(o.res[:M])
        res = rc.out
    x = o.x[:M]

    def go():
        if entry == 'decode':
            raw('g4r_decode_gemm_bf16', dt, _L.ptr(x), x.stride(0), _L.ptr(o.w), o.w.stride(0), _L.ptr(cv.out), ld, M, N,
                K, dense.ACT[act], _L.ptr(res), ld if res is not None else 0, None, None, 0, 0, None, None, None, 0, 0)
        else:
            b = None if bias is None else (o.bias if bias == 'bf16' else o.bias32)
            dense.linear(x, o.w, bias=b, act=act, residual=res, out=cv.out)
        return cv
    return cv, go


def run(ep, o, M, layout):
    """One launch of epilogue ep on the first M rows into a fresh canvas (prepare)."""
    return prepare(ep, o, M, layout)[1]()


def check_epilogues(eps, o, Ms, extra_layout=None, what=''):
    """For every M: each epilogue in each layout (_layouts of its output width, plus extra_layout) inside its canvas,
    bitwise equal across layouts and to a repeated launch, and within the fp64 bound of the instance the rule predicts
    (test_instances traces the same launches)."""
    n_sms = sms()
    layouts = {ep: _layouts(o.N // 2 if EPILOGUES[ep][2] == 'swiglu' else o.N) + ([extra_layout] if extra_layout else [])
               for ep in eps}
    runs = {M: {ep: [run(ep, o, M, lay) for lay in layouts[ep] + layouts[ep][:1]] for ep in eps} for M in Ms}
    for M in Ms:
        want = instance(M, o.N, False, n_sms)
        for ep in eps:
            got = runs[M][ep][0].out
            for (name, ld, col0), cv in zip(layouts[ep], runs[M][ep]):
                w = '%s %s M=%d, %s output (ldd=%d, column %d)' % (what, ep, M, name, ld, col0)
                cv.check(w)
                assert torch.equal(bits(cv.out), bits(got)), w + ': differs from the %s output' % layouts[ep][0][0]
            assert torch.equal(bits(runs[M][ep][-1].out), bits(got)), '%s %s M=%d: a repeated launch differs' % (
                what, ep, M)
            ref, e32 = reference(ep, o, M, want[2])
            _check_rounded(got, ref, e32, o.dt, '%s %s M=%d %s' % (what, ep, M, want))


# ---- the engine's decode GEMMs at every M ---------------------------------------------------------------------

# (name, N, K, epilogue, extra layout): o_proj and down add the residual stream, gate/up is the fused SwiGLU
# (g4r_decode_gemm), lm_head writes into the vocab_pad buffer (row stride 32064).  q|k|v is test_rope_kv's.
ENGINE = [('o_proj', 4096, 4096, 'lin_residual', None), ('gate_up', 22016, 4096, 'swiglu', None),
          ('down', 4096, 11008, 'lin_residual', None), ('lm_head', 32006, 4096, 'lin_none', ('vocab_pad', 32064, 0))]


@pytest.mark.parametrize('dt', DTS)
@pytest.mark.parametrize('name,N,K,ep,extra', ENGINE, ids=[e[0] for e in ENGINE])
def test_engine_gemm(name, N, K, ep, extra, dt):
    o = Operands(N, K, dt, seed=N + K)
    check_epilogues([ep], o, range(1, 17), extra, name)


# ---- edge shapes of every instance ----------------------------------------------------------------------------

# Each class of N takes one instance at M <= 8 and one at M 9..16: 'narrow' (16-row tiles) <1,1,8,false,2> and
# <1,2,16,false,1>; 'wide8' / 'wide4' (32-row tiles) <2,1,8,false,1> / <2,1,4,false,1> and <2,2,4,false,1>.
# K: 32 (one sub-block: one active warp); 544 / 1056 / 2080, one 32-block past a whole warp stride (128 k per warp) of
# 4 / 8 / 16 warps; 3072, three k-blocks per warp at 8 warps, an odd count for DEPTH = 2 (its `break` path, and a
# refill of the first slot); 11008 (down_proj).
# N: the class's base; 'narrow' also N = 8 (below one 16-row tile) and 1000 (ends inside a tile); 'wide' N ending
# inside the first (32006-like: 6 rows) and inside the second (20 rows) 16-row half of the last 32-row tile.
EDGE_K = (32, 544, 1056, 2080, 3072, 11008)
EDGE_CASES = [(cls, 'base', K) for cls in ('narrow', 'wide8', 'wide4') for K in EDGE_K]
EDGE_CASES += [('narrow', 8, 1056), ('narrow', 1000, 1056)]
EDGE_CASES += [(cls, n, 1056) for cls in ('wide8', 'wide4') for n in ('first16', 'second16')]
EDGE_M = (1, 3, 8, 9, 16)


def edge_n(cls, n, n_sms):
    if cls == 'narrow':
        return 4096 if n == 'base' else n
    t = wide_tiles(n_sms, cls == 'wide8')
    return {'base': 32 * t, 'first16': 32 * t - 26, 'second16': 32 * t - 12}[n]


@pytest.mark.parametrize('dt', DTS)
@pytest.mark.parametrize('cls,n,K', EDGE_CASES, ids=['%s-N%s-K%d' % c for c in EDGE_CASES])
def test_edge_shapes(cls, n, K, dt):
    n_sms = sms()
    N = edge_n(cls, n, n_sms)
    # the case's class is the one the rule gives its N
    want_small = {'narrow': (1, 1, 8, False, 2), 'wide8': (2, 1, 8, False, 1), 'wide4': (2, 1, 4, False, 1)}[cls]
    assert instance(8, N, False, n_sms) == want_small
    o = Operands(N, K, dt, seed=N * 3 + K)
    check_epilogues(EDGE_EPILOGUES, o, EDGE_M, what='%s N=%d K=%d' % (cls, N, K))


# ---- fused RoPE + KV-cache append -----------------------------------------------------------------------------

LMAX = 160   # cache length and RoPE table rows: the last position is LMAX - 1


def rope_positions(mode, M):
    """Sequence position of each of the M rows."""
    if mode == 'pos0':
        return [LMAX - 1] * M
    if mode == 'pos_dev':
        return [61] * M
    if mode == 'pos_rows':
        return [(LMAX - 1 - 13 * m) % LMAX for m in range(M)]   # distinct, the first at LMAX - 1
    return [LMAX - M + m for m in range(M)]                     # verify: one sample of M rows from LMAX - M


def plain_rows(N, n_sms):
    """Weight rows of a plain launch that runs <2, MB, 4, false, 1> at M <= 8 too: N padded to a wide 4-warp count."""
    t = max(-(-N // 32), 2 * n_sms)
    while prefers_8_warps(t, n_sms):
        t += 1
    return 32 * t


def rope_launcher(mode, x, w, cos, sin, hd, out, kc, vc):
    """The function that launches q|k|v + RoPE (+ the KV append, except in the verify step) of the M rows of x into
    out, through the entry the engine uses for the mode: g4r_decode_gemm (host pos0 or device pos_dev),
    g4r_decode_gemm_rows (per-row pos_rows), or g4r_gemm_qkv_rope_rows with rope_L = M and a one-entry pos_rows (the
    prompt-lookup verify step)."""
    M, K = x.shape
    N, dt = w.shape[0], x.dtype
    pos = rope_positions(mode, M)
    # the returned function holds the tensors themselves and takes their addresses when it launches, so nothing it
    # writes or reads can be freed before it runs
    common = lambda: (_L.ptr(x), x.stride(0), _L.ptr(w), w.stride(0), _L.ptr(out), out.stride(0), M, N, K)
    if mode == 'verify':
        base = torch.tensor([pos[0]], dtype=torch.int32, device=DEV)
        return lambda: raw('g4r_gemm_qkv_rope_rows_bf16', dt, *common(), _L.ptr(cos), _L.ptr(sin), 2 * hd, M,
                           _L.ptr(base))
    if mode == 'pos_rows':
        rows = torch.tensor(pos, dtype=torch.int32, device=DEV)
        return lambda: raw('g4r_decode_gemm_rows_bf16', dt, *common(), 0, None, 0, _L.ptr(cos), _L.ptr(sin), 2 * hd,
                           _L.ptr(rows), _L.ptr(kc), _L.ptr(vc), LMAX, hd)
    pd = torch.tensor([pos[0]], dtype=torch.int32, device=DEV) if mode == 'pos_dev' else None
    return lambda: raw('g4r_decode_gemm_bf16', dt, *common(), 0, None, 0, _L.ptr(cos), _L.ptr(sin), 2 * hd,
                       pos[0] if mode == 'pos0' else 0, _L.ptr(pd), _L.ptr(kc), _L.ptr(vc), LMAX, hd)


def rotate_half_rounded(plain, cos, sin, pos, n_rot):
    """HF's q * cos + rotate_half(q) * sin on the first n_rot columns (128-dim heads) of the 16-bit plain output, with
    the kernel's rounding points: each product rounded to 16 bits, their fp32 sum rounded once."""
    M, dt = plain.shape[0], plain.dtype
    q = plain[:, :n_rot].float().view(M, n_rot // 128, 128)
    p = torch.tensor(pos, device=DEV)
    c, s = cos[p].float()[:, None], sin[p].float()[:, None]
    r = lambda t: t.to(dt).float()
    x1, x2 = q[..., :64], q[..., 64:]
    o1 = (r(x1 * c[..., :64]) + r(-x2 * s[..., :64])).to(dt)
    o2 = (r(x2 * c[..., 64:]) + r(x1 * s[..., 64:])).to(dt)
    return torch.cat([o1, o2], -1).view(M, n_rot)


# (name, heads, K): hd = 128 * heads columns each of q, k and v; the engine's 7B q|k|v is 32 heads over K = 4096
ROPE_SHAPES = [('h2-K32', 2, 32), ('h2-K544', 2, 544), ('h2-K11008', 2, 11008), ('engine', 32, 4096)]
ROPE_MODES = ('pos0', 'pos_dev', 'pos_rows', 'verify')


@pytest.mark.parametrize('dt', DTS)
@pytest.mark.parametrize('mode', ROPE_MODES)
@pytest.mark.parametrize('shape', ROPE_SHAPES, ids=[s[0] for s in ROPE_SHAPES])
def test_rope_kv(shape, mode, dt):
    name, heads, K = shape
    n_sms = sms()
    hd = 128 * heads
    N = 3 * hd
    o = Operands(plain_rows(N, n_sms), K, dt, seed=N + K + 7)
    o.w[N:].zero_()                       # padding rows of the plain launch
    o.y[:, N:] = 0
    o.S[:, N:] = 0
    w = o.w[:N]
    cos, sin = rope_tables(LMAX, dt)
    Ms = range(1, 17) if name == 'engine' and mode == 'pos_rows' else (1, 3, 8, 9, 16)
    layouts = _layouts(N)[:1] if mode == 'verify' else _layouts(N)   # qkv_rope takes 16-byte row pitches only

    def prepare_rope(M):
        """Fresh canvases and NaN-filled caches [M + 1, LMAX, hd] for each layout, and the function that launches into
        them."""
        runs, gos = [], []
        for _, ld, col0 in layouts:
            cv = Canvas(M, N, dt, ld, col0)
            kc, vc = nan((M + 1, LMAX, hd), dt), nan((M + 1, LMAX, hd), dt)
            gos.append(rope_launcher(mode, o.x[:M], w, cos, sin, hd, cv.out, kc, vc))
            runs.append((cv, kc, vc))

        def go():
            for g in gos:
                g()
            return runs
        return go

    def launch(M):
        return prepare_rope(M)()

    # the unrotated output, from the plain launch with the RoPE instance's WARPS / DEPTH (test_instances traces it)
    for M in Ms:
        assert instance(M, o.N, False, n_sms) == (2, 1 if M <= 8 else 2, 4, False, 1)
    plains = {M: run('none', o, M, _layouts(o.N)[0]) for M in Ms}
    ropes = {M: launch(M) for M in Ms}
    again = {M: launch(M) for M in Ms}
    for M in Ms:
        what = '%s %s M=%d' % (name, mode, M)
        ref, e32 = reference('none', o, M, 4)
        _check_rounded(plains[M].out, ref, e32, dt, what + ' plain')
        plain = plains[M].out[:, :N]
        pos = rope_positions(mode, M)
        runs = ropes[M]
        got = runs[0][0].out
        for (lname, ld, col0), (cv, kc, vc) in zip(layouts, runs):
            cv.check('%s, %s output' % (what, lname))
            assert torch.equal(bits(cv.out), bits(got)), '%s: the %s output differs' % (what, lname)
        assert torch.equal(bits(got[:, :2 * hd]), bits(rotate_half_rounded(plain, cos, sin, pos, 2 * hd))), \
            what + ': q|k columns differ from rotate-half of the unrotated output'
        assert torch.equal(bits(got[:, 2 * hd:]), bits(plain[:, 2 * hd:])), what + ': v columns are not the plain output'
        kc, vc = runs[0][1], runs[0][2]
        if mode == 'verify':
            assert bool((bits(kc) == NAN_BITS[dt]).all() and (bits(vc) == NAN_BITS[dt]).all()), \
                what + ': the verify step has no KV write'
        else:
            for cache, cols, kind in ((kc, slice(hd, 2 * hd), 'K'), (vc, slice(2 * hd, 3 * hd), 'V')):
                want = nan(cache.shape, dt)
                for m in range(M):
                    want[m, pos[m]] = got[m, cols]
                assert torch.equal(bits(cache), bits(want)), \
                    '%s: %s cache differs from the output slices at rows (m, pos_m) or was written elsewhere' % (what, kind)
        for (cv, kc, vc), (cv2, kc2, vc2) in zip(runs, again[M]):
            assert torch.equal(bits(cv2.out), bits(cv.out)) and torch.equal(bits(kc2), bits(kc)) and \
                torch.equal(bits(vc2), bits(vc)), what + ': a repeated launch differs'


@pytest.mark.parametrize('dt', DTS)
@pytest.mark.parametrize('M', [5, 12])
def test_position_sources_agree(M, dt):
    """Host pos0, a device pos_dev and an all-equal pos_rows name the same position: same output and caches, bit for
    bit, through dense.decode_gemm."""
    torch.manual_seed(M)
    hd, K, P = 256, 544, LMAX - 1
    x = torch.randn(M, K, device=DEV).to(dt)
    w = (torch.randn(3 * hd, K, device=DEV) * K ** -0.5).to(dt)
    cos, sin = rope_tables(LMAX, dt)
    results = []
    for src in ('pos0', 'pos_dev', 'pos_rows'):
        kc, vc = nan((M, LMAX, hd), dt), nan((M, LMAX, hd), dt)
        pos_dev = torch.tensor([P], dtype=torch.int32, device=DEV) if src == 'pos_dev' else None
        rows = torch.full((M,), P, dtype=torch.int32, device=DEV) if src == 'pos_rows' else None
        out = dense.decode_gemm(x, w, rope=(cos, sin, 2 * hd, P if src == 'pos0' else 0, pos_dev), kv=(kc, vc),
                                pos_rows=rows)
        results.append((src, out, kc, vc))
    for src, out, kc, vc in results[1:]:
        for a, b in zip((out, kc, vc), results[0][1:]):
            assert torch.equal(bits(a), bits(b)), '%s differs from host pos0' % src
    assert bool(torch.isfinite(results[0][1].float()).all())


# ---- programmatic dependent launch ----------------------------------------------------------------------------

@pytest.mark.parametrize('dt', DTS)
def test_pdl_chain(dt):
    """rmsnorm -> decode_gemm with programmatic dependent launch on and off: the GEMM issues its first weight block
    before griddepcontrol.wait and must read its activations only after it.  The rmsnorm output starts NaN-filled
    each time, so activations read early show as NaN; on and off must agree bit for bit."""
    n_sms = sms()
    torch.manual_seed(3)
    K, hd = 4096, 256
    cos, sin = rope_tables(LMAX, dt)
    ln = (1 + 0.1 * torch.randn(K, device=DEV)).to(dt)
    weights = {'narrow': (torch.randn(4096, K, device=DEV) * K ** -0.5).to(dt),
               'wide8': (torch.randn(32 * wide_tiles(n_sms, True), K, device=DEV) * K ** -0.5).to(dt),
               'wide4': (torch.randn(32 * wide_tiles(n_sms, False), K, device=DEV) * K ** -0.5).to(dt),
               'rope': (torch.randn(3 * hd, K, device=DEV) * K ** -0.5).to(dt)}
    for M in (4, 12):
        xs = torch.randn(M, K, device=DEV).to(dt)
        for name, w in weights.items():
            def chain(pdl):
                prev = _L.set_pdl(pdl)
                try:
                    h = nan((M, K), dt)
                    kernels.rmsnorm(xs, ln, 1e-6, out=h)
                    if name == 'rope':
                        kc, vc = nan((M, LMAX, hd), dt), nan((M, LMAX, hd), dt)
                        out = dense.decode_gemm(h, w, rope=(cos, sin, 2 * hd, 0, None), kv=(kc, vc),
                                                pos_rows=torch.arange(M, dtype=torch.int32, device=DEV))
                        out = (out, kc, vc)
                    else:
                        out = (dense.decode_gemm(h, w, act='swiglu' if name == 'wide8' else None),)
                    torch.cuda.synchronize()
                    return out
                finally:
                    _L.set_pdl(prev)
            on, off = chain(True), chain(False)
            assert bool(torch.isfinite(on[0].float()).all()), '%s M=%d: NaN activations read under PDL' % (name, M)
            for a, b in zip(on, off):
                assert torch.equal(bits(a), bits(b)), '%s M=%d: PDL on and off differ' % (name, M)


# ---- host-side refusals ---------------------------------------------------------------------------------------

def _decode_args(dt, M=4, K=256, hd=128):
    x = torch.randn(M, K, device=DEV).to(dt)
    w = (torch.randn(3 * hd, K, device=DEV) * K ** -0.5).to(dt)
    cos, sin = rope_tables(LMAX, dt)
    kc, vc = torch.zeros(M, LMAX, hd, dtype=dt, device=DEV), torch.zeros(M, LMAX, hd, dtype=dt, device=DEV)
    return x, w, cos, sin, kc, vc


@pytest.mark.parametrize('dt', DTS)
def test_refuses_dropped_epilogues(dt):
    """The RoPE epilogue ends without the residual or activation, and SwiGLU without the residual: refused."""
    x, w, cos, sin, kc, vc = _decode_args(dt)
    M, hd = x.shape[0], kc.shape[2]
    rope = (cos, sin, 2 * hd, 0, None)
    res = torch.zeros(M, w.shape[0], dtype=dt, device=DEV)
    with pytest.raises(_L.G4RError, match='residual cannot be combined with RoPE'):
        dense.decode_gemm(x, w, residual=res, rope=rope)
    with pytest.raises(_L.G4RError, match='residual cannot be combined with SwiGLU'):
        dense.decode_gemm(x, w, act='swiglu', residual=res[:, :w.shape[0] // 2])
    with pytest.raises(_L.G4RError, match='activation cannot be combined with RoPE'):
        dense.decode_gemm(x, w, act='swiglu', rope=rope, kv=(kc, vc))


@pytest.mark.parametrize('dt', DTS)
def test_refuses_operand_layout(dt):
    """x / W not 16-byte aligned, or a row stride below K: refused before any launch (the kernel reads both with
    16-byte vector loads over K elements per row)."""
    x, w, *_ = _decode_args(dt)
    M, K = x.shape
    N = w.shape[0]
    xb = torch.zeros(M, K + 8, dtype=dt, device=DEV)
    wb = torch.zeros(N, K + 8, dtype=dt, device=DEV)
    out = torch.empty(M, N, dtype=dt, device=DEV)
    with pytest.raises(_L.G4RError, match='16-byte aligned'):
        dense.decode_gemm(xb[:, 4:K + 4], w)
    with pytest.raises(_L.G4RError, match='16-byte aligned'):
        dense.decode_gemm(x, wb[:, 4:K + 4])
    for ldx, ldw in ((K - 8, K), (K, K - 8)):
        with pytest.raises(_L.G4RError, match='must be >= K'):
            raw('g4r_decode_gemm_bf16', dt, _L.ptr(xb), ldx, _L.ptr(wb), ldw, _L.ptr(out), N, M, N, K, 0, None, 0,
                None, None, 0, 0, None, None, None, 0, 0)


@pytest.mark.parametrize('dt', DTS)
def test_refuses_bad_cache_and_positions(dt):
    """dense.decode_gemm checks every tensor's device, the caches' dtype, contiguity and shape, and a host pos0."""
    x, w, cos, sin, kc, vc = _decode_args(dt)
    M, hd = x.shape[0], kc.shape[2]
    rope = (cos, sin, 2 * hd, 0, None)
    other = H16 if dt == BF else BF
    bad_kv = {
        'dtype': (kc.to(other), vc.to(other)),
        'fp32': (kc.float(), vc.float()),
        'non-contiguous': (torch.zeros(M, hd, LMAX, dtype=dt, device=DEV).transpose(1, 2), vc),
        'too few rows': (kc[:M - 1], vc[:M - 1]),
        'head width': (kc[..., :hd // 2].contiguous(), vc[..., :hd // 2].contiguous()),
        'unequal shapes': (kc, torch.zeros(M, LMAX - 1, hd, dtype=dt, device=DEV)),
        'on the host': (kc.cpu(), vc.cpu()),
    }
    for what, kv in bad_kv.items():
        with pytest.raises(RuntimeError):
            dense.decode_gemm(x, w, rope=rope, kv=kv)
            pytest.fail('accepted caches: %s' % what)
    for what, r in {'cos on the host': (cos.cpu(), sin, 2 * hd, 0, None),
                    'pos_dev on the host': (cos, sin, 2 * hd, 0, torch.zeros(1, dtype=torch.int32))}.items():
        with pytest.raises(RuntimeError):
            dense.decode_gemm(x, w, rope=r, kv=(kc, vc))
            pytest.fail('accepted %s' % what)
    with pytest.raises(RuntimeError):
        dense.decode_gemm(x, w, rope=rope, kv=(kc, vc), pos_rows=torch.zeros(M, dtype=torch.int32))
    # host pos0: a row of the caches and of the tables
    for pos0, tables in ((LMAX, (cos, sin)), (-1, (cos, sin)), (LMAX - 1, (cos[:LMAX - 1], sin[:LMAX - 1]))):
        with pytest.raises(RuntimeError, match='pos0'):
            dense.decode_gemm(x, w, rope=(*tables, 2 * hd, pos0, None), kv=(kc, vc))
    with pytest.raises(RuntimeError, match='pos0'):
        dense.decode_gemm(x, w, rope=(cos[:8], sin[:8], 2 * hd, 8, None))


# ---- the selection rule and instance coverage -----------------------------------------------------------------

def test_selection_rule_on_h100():
    """The rule restated above gives the instances the kernel's comments name for the engine's shapes on 132 SMs."""
    table = [(1, 12288, True, (2, 1, 4, True, 1)), (9, 12288, True, (2, 2, 4, True, 1)),
             (8, 4096, False, (1, 1, 8, False, 2)), (16, 4096, False, (1, 2, 16, False, 1)),
             (8, 22016, False, (2, 1, 8, False, 1)), (8, 32006, False, (2, 1, 4, False, 1)),
             (16, 22016, False, (2, 2, 4, False, 1)), (16, 32006, False, (2, 2, 4, False, 1))]
    for M, N, rope, want in table:
        assert instance(M, N, rope, 132) == want, (M, N, rope)


def trace_cases(dt):
    """One launch of every case of this file at every row count it uses, through the same entry, traced in one
    profiler session (for the RoPE cases also the plain launch whose output is the rotation's input).  Returns
    [(case, predicted instance)] and the instances the trace shows, in launch order."""
    n_sms = sms()
    cases = []   # (what, predicted instance, launch)

    def add(what, o, ep, Ms, rope=None):
        for M in Ms:
            if rope is None:
                _, go = prepare(ep, o, M, _layouts(o.N // 2 if EPILOGUES[ep][2] == 'swiglu' else o.N)[0])
                cases.append(('%s M=%d' % (what, M), instance(M, o.N, False, n_sms), go))
                continue
            mode, N, hd, cos, sin = rope
            _, go = prepare('none', o, M, _layouts(o.N)[0])
            cases.append(('%s plain M=%d' % (what, M), (2, 1 if M <= 8 else 2, 4, False, 1), go))
            cv = Canvas(M, N, dt, *_layouts(N)[0][1:])
            kc, vc = nan((M + 1, LMAX, hd), dt), nan((M + 1, LMAX, hd), dt)
            cases.append(('%s M=%d' % (what, M), instance(M, N, True, n_sms),
                          rope_launcher(mode, o.x[:M], o.w[:N], cos, sin, hd, cv.out, kc, vc)))

    for name, N, K, ep, _ in ENGINE:
        add(name, Operands(N, K, dt, seed=N + K, ref=False), ep, range(1, 17))
    for cls, n, K in EDGE_CASES:
        N = edge_n(cls, n, n_sms)
        o = Operands(N, K, dt, seed=N * 3 + K, ref=False)
        for ep in ('none', 'lin_bias32_swiglu'):   # one epilogue of each entry
            add('%s N=%d K=%d %s' % (cls, N, K, ep), o, ep, EDGE_M)
    cos, sin = rope_tables(LMAX, dt)
    for name, heads, K in ROPE_SHAPES:
        hd = 128 * heads
        o = Operands(plain_rows(3 * hd, n_sms), K, dt, seed=3 * hd + K + 7, ref=False)
        for mode in ROPE_MODES:
            Ms = range(1, 17) if name == 'engine' and mode == 'pos_rows' else (1, 3, 8, 9, 16)
            add('%s %s' % (name, mode), o, 'none', Ms, rope=(mode, 3 * hd, hd, cos, sin))
    got = traced_instances([go for _, _, go in cases], dt)
    return [(what, want) for what, want, _ in cases], got


_TRACE_MARK = 'decode-gemm-trace: '
_TRACE_CHILD = """
import json, sys
sys.path.insert(0, sys.argv[1])
import torch
from tests import test_decode_gemm_gpu as T
cases, got = T.trace_cases({'bf16': torch.bfloat16, 'fp16': torch.float16}[sys.argv[2]])
print(T._TRACE_MARK + json.dumps({'cases': cases, 'got': got}))
"""


@pytest.mark.parametrize('dt', DTS)
def test_instances(dt):
    """Every case ran the instance the rule predicts, and together they launched all seven instances.  The trace is
    taken in a child process: once a process has used the CUDA profiler, later sessions in it come back empty after
    enough other GPU work, so tracing here would break the profiler-based tests of files that run after this one."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    flags = [f for f, on in (('-E', sys.flags.ignore_environment), ('-s', sys.flags.no_user_site),
                             ('-I', sys.flags.isolated)) if on]
    r = subprocess.run([sys.executable, *flags, '-c', _TRACE_CHILD, root, 'bf16' if dt == BF else 'fp16'],
                       capture_output=True, text=True, cwd=root, timeout=600)
    lines = [l for l in r.stdout.splitlines() if l.startswith(_TRACE_MARK)]
    assert r.returncode == 0 and lines, 'the tracing process failed (rc %d):\n%s' % (r.returncode, r.stderr[-4000:])
    res = json.loads(lines[-1][len(_TRACE_MARK):])
    cases, got = res['cases'], [tuple(g) for g in res['got']]
    assert len(got) == len(cases), 'the trace holds %d of the %d launches' % (len(got), len(cases))
    wrong = ['%s: ran %s, the rule predicts %s' % (what, g, tuple(want)) for (what, want), g in zip(cases, got)
             if g != tuple(want)]
    assert not wrong, '%d launches on another instance; first: %s' % (len(wrong), wrong[0])
    assert set(got) == ALL_INSTANCES, 'not launched: %s' % sorted(ALL_INSTANCES - set(got))
