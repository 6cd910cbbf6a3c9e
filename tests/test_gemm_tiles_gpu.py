"""The wgmma GEMM / implicit-GEMM conv (csrc/gemm_wgmma.cu) at both tile widths and on a 2-CTA persistent grid.

`pick_block_n` picks the tile width (BN = 128 or 256) per launch from the shape and the SM count, so tests that leave
it alone check whichever kernel the rule picks for their shape.  Here the `width` fixture forces each width through
G4R_GEMM_BN, and every case checks from the profiler that the forced width is the kernel that ran.  `small_grid` caps
the persistent grid at 2 CTAs, so each CTA loops over many tiles and carries its ring stage and phase from one tile to
the next.  Each case checks
  * the fp32 torch reference of the same op on the same 16-bit inputs, with the rounding points the kernel documents;
    where the epilogue is exactly reproducible in torch (adds, relu, 16-bit rounding), also bitwise against that
    epilogue applied in torch to the kernel's own fp32 accumulators;
  * bitwise equality between the default grid and the 2-CTA grid, and between the 256 and the 128 kernel;
  * outputs written through `Canvas`: a view with padded row stride inside a NaN-filled buffer, so a store outside
    the output or an output element never stored shows.  GEMM outputs (and their residuals) take three layouts: a
    row pitch that allows 16-byte vector accesses, an odd one, and a 16-byte pitch whose base is not 16-byte aligned
    (the last two must take the scalar path)."""
import contextlib
import re
import time

import pytest
import torch
import torch.nn.functional as F

from gpt4roi_b200 import dense, kernels, lib
from tests.test_dense_gpu import _close as _close_bf16
from tests.test_fp16_gpu import _close as _close_f16

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
BF, H, F32 = torch.bfloat16, torch.float16, torch.float32


# ---- fixtures and helpers -------------------------------------------------------------------------------------

@pytest.fixture(params=['128', '256'])
def width(request, monkeypatch):
    """Forces the tile width of every forward GEMM / conv launch (pick_block_n reads G4R_GEMM_BN at each launch)."""
    monkeypatch.setenv('G4R_GEMM_BN', request.param)
    return int(request.param)


def _at_128(monkeypatch, fn):
    """fn() on the 128-wide kernel, then back to 256."""
    monkeypatch.setenv('G4R_GEMM_BN', '128')
    try:
        return fn()
    finally:
        monkeypatch.setenv('G4R_GEMM_BN', '256')


_KERNEL = re.compile(r'g4r(?:_h)?::gemm_bf16_wgmma<(false|true), (\d), (\d), (\d+)>')


def launched_widths(fn):
    """fn() under the CUDA profiler: returns its result and the set of (CONV, TA, TB, BN) template arguments of the
    gemm_bf16_wgmma kernels it launched (bf16 namespace g4r, fp16 g4r_h).  fn must be repeatable: a trace that
    comes back without any GEMM kernel is taken again, up to five times in all, because the profiler now and then
    returns an empty one, sometimes several in a row."""
    for attempt in range(5):
        time.sleep(0.05 * attempt)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        seen = set()
        for e in prof.events():
            if 'gemm_bf16_wgmma' in e.name:
                m = _KERNEL.search(e.name)
                assert m, 'cannot read the template arguments of kernel %r' % e.name
                seen.add((m[1] == 'true', int(m[2]), int(m[3]), int(m[4])))
        if seen:
            break
    return out, seen


def _num_sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


@contextlib.contextmanager
def sm_budget(n):
    """The persistent GEMM grids use n CTAs (the SM reserve is global to the process: restored on exit)."""
    prev = lib.set_sm_reserve(_num_sms() - n)
    try:
        yield
    finally:
        lib.set_sm_reserve(prev)


def small_grid():
    """Two CTAs: each loops over many tiles."""
    return sm_budget(2)


_NAN_BITS = {BF: (torch.int16, 0x7fc1), H: (torch.int16, 0x7e01), F32: (torch.int32, 0x7fc00001)}


class Canvas:
    """Output buffer `out` [rows, cols] with row stride ld starting at column col0, inside a NaN-filled [rows + 2, ld]
    buffer (one guard row above and one below, ld - cols spare columns)."""

    def __init__(self, rows, cols, dtype, ld, col0=0):
        self.itype, self.bits = _NAN_BITS[dtype]
        self.buf = torch.empty(rows + 2, ld, dtype=dtype, device=DEV)
        self.buf.view(self.itype).fill_(self.bits)
        self.out = self.buf[1:rows + 1, col0:col0 + cols]
        self.col0 = col0

    def check(self, what):
        """Every element outside `out` is bitwise unchanged and every element inside it is finite."""
        rows, cols = self.out.shape
        outside = torch.ones(self.buf.shape, dtype=torch.bool, device=DEV)
        outside[1:rows + 1, self.col0:self.col0 + cols] = False
        assert bool((self.buf.view(self.itype)[outside] == self.bits).all()), '%s: stored outside the output' % what
        assert bool(torch.isfinite(self.out.float()).all()), '%s: output elements not stored' % what


def _layouts(n):
    """(name, row stride, first column) of the outputs a GEMM case writes: a padded stride that keeps 16-byte vector
    stores (a multiple of 8 elements, e.g. lm_head's 32008), an odd stride (the scalar path), and the padded stride
    with the output starting one element in (16-byte pitch, base not 16-byte aligned: the scalar path too)."""
    vec = (n // 8 + 1) * 8
    return [('vector', vec, 0), ('odd', n + 1 if n % 2 == 0 else n + 2, 0), ('offset', vec, 1)]


def _randn(gen, *shape, scale=1.0):
    return torch.randn(*shape, generator=gen, device=DEV) * scale


# ---- GEMM epilogues -------------------------------------------------------------------------------------------

# (M, N, K) cover: N below one tile (72); N ending inside the first (32006) or the second (200, 1000) 128-column half
# of the last 256 tile, or on the boundary (640); K below one k-block (8) and not a multiple of 64 (72, 136); 1, 2, 3,
# 8, 16 and 64 k-blocks against ring depths of 4 (BN = 128) and 3 (BN = 256); more tiles than the grid (4616 rows,
# 706 x 32006 with the lm_head's padded ldd); 1- and 5-row tiles on the wgmma kernel (outputs the skinny kernel does
# not take).
GEMM_SHAPES = [(17, 72, 8), (128, 128, 64), (129, 200, 136), (300, 640, 512), (257, 1000, 72), (4616, 1024, 1024),
               (706, 32006, 4096), (1, 1000, 72), (5, 640, 512)]
EPILOGUES = ('none', 'bias_relu', 'bias32_quick_gelu', 'residual', 'stream_out32', 'stream_out16', 'out32', 'swiglu',
             'splitk2', 'splitk3')
# what the M <= 16 skinny kernel does not take, so M = 1 / 5 run it on the wgmma kernel
_WGMMA_AT_SMALL_M = ('stream_out32', 'stream_out16', 'out32', 'splitk2', 'splitk3')


def _applies(M, K, ep):
    if M <= 16 and ep not in _WGMMA_AT_SMALL_M:
        return False
    if ep.startswith('splitk'):
        return -(-K // 64) % int(ep[-1]) == 0
    return True


GEMM_CASES = [(s, ep, BF) for s in GEMM_SHAPES for ep in EPILOGUES if _applies(s[0], s[2], ep)]
GEMM_CASES += [((300, 640, 512), ep, H) for ep in EPILOGUES if _applies(300, 512, ep)]   # fp16 twin


def _gemm_id(case):
    (M, N, K), ep, dt = case
    return '%dx%dx%d-%s-%s' % (M, N, K, ep, 'bf16' if dt == BF else 'fp16')


class GemmOperands:
    """Seeded operands of one GEMM case; residuals are stored in the layout of the output they go with."""

    def __init__(self, M, N, K, dt):
        g = torch.Generator(device=DEV).manual_seed(M * 7 + N + K)
        self.M, self.N, self.K, self.dt = M, N, K, dt
        self.a = _randn(g, M, K).to(dt)
        self.b = _randn(g, N, K, scale=K ** -0.5).to(dt)
        self.bias = _randn(g, N, scale=0.5).to(dt)
        self.bias32 = _randn(g, N, scale=0.5)
        self.res = _randn(g, M, N).to(dt)
        self.res32 = _randn(g, M, N)

    def strided(self, t, ld, col0):
        buf = torch.zeros(self.M, ld, dtype=t.dtype, device=DEV)
        buf[:, col0:col0 + self.N] = t
        return buf[:, col0:col0 + self.N]


def run_epilogue(ep, o, layout):
    """One launch of epilogue `ep` into a fresh canvas of the given layout (the residual has the same layout)."""
    M, N, K, dt = o.M, o.N, o.K, o.dt
    _, ld, col0 = layout
    if ep.startswith('splitk'):
        # split-K slabs [k][M][ldd]: dense.linear allocates them itself, so the C entry point takes the canvas
        k = int(ep[-1])
        cv = Canvas(k * M, N, F32, ld, col0)
        with torch.cuda.device(DEV):
            lib.check(getattr(lib.load(), lib.sym('g4r_gemm_bf16', dt))(
                lib.ptr(o.a), K, lib.ptr(o.b), K, lib.ptr(cv.out), ld, M, N, K, None, 0, None, 0, 0, 1, k,
                lib.stream_ptr(torch.device(DEV))))
        return cv
    n_out = N // 2 if ep == 'swiglu' else N
    out_dtype = F32 if ep in ('out32', 'stream_out32') else dt
    kw = {}
    if ep == 'swiglu':
        kw = dict(act='swiglu')
    elif ep == 'bias_relu':
        kw = dict(bias=o.bias, act='relu')
    elif ep == 'bias32_quick_gelu':
        kw = dict(bias=o.bias32, act='quick_gelu')
    elif ep == 'residual':
        kw = dict(residual=o.strided(o.res, ld, col0))
    elif ep.startswith('stream'):
        kw = dict(bias=o.bias, residual=o.strided(o.res32, ld, col0), round_branch=True)
    cv = Canvas(M, n_out, out_dtype, ld, col0)
    dense.linear(o.a, o.b, out=cv.out, out_dtype=out_dtype, **kw)
    return cv


def gemm_references(ep, o, acc32):
    """(fp32 reference of the op, or None; torch result that must match bitwise, or None).  acc32 is the kernel's
    own fp32 output at the same width."""
    base = o.a.float() @ o.b.float().t()
    dt = o.dt
    if ep == 'none':
        return base, acc32.to(dt)
    if ep == 'out32':
        return base, acc32
    if ep == 'bias_relu':
        return torch.relu(base + o.bias.float()), torch.relu(acc32 + o.bias.float()).to(dt)
    if ep == 'bias32_quick_gelu':
        z = base + o.bias32
        return z * torch.sigmoid(1.702 * z), None
    if ep == 'residual':
        return base + o.res.float(), (acc32 + o.res.float()).to(dt)
    if ep.startswith('stream'):
        # the branch act(x W^T + b) is rounded to 16 bits before the fp32 residual add (CLIP under autocast)
        want = (base + o.bias.float()).to(dt).float() + o.res32
        exact = (acc32 + o.bias.float()).to(dt).float() + o.res32
        return (want, exact) if ep == 'stream_out32' else (want, exact.to(dt))
    if ep == 'swiglu':
        # interleaved rows: output column j = silu(gate row 2j) * (up row 2j + 1)
        return F.silu(base[:, 0::2]) * base[:, 1::2], None
    # split-K: slab s holds the k-blocks [s * kb / k, (s + 1) * kb / k), i.e. the fp32 GEMM of that slice of K
    k = int(ep[-1])
    kc = -(-o.K // 64) // k * 64
    slabs = [dense.linear(o.a[:, s * kc:(s + 1) * kc], o.b[:, s * kc:(s + 1) * kc], out_dtype=F32) for s in range(k)]
    return None, torch.cat(slabs)


@pytest.mark.parametrize('case', GEMM_CASES, ids=_gemm_id)
def test_gemm_epilogue(width, monkeypatch, case):
    (M, N, K), ep, dt = case
    close = _close_bf16 if dt == BF else _close_f16
    o = GemmOperands(M, N, K, dt)
    acc32 = dense.linear(o.a, o.b, out_dtype=F32)
    want, exact = gemm_references(ep, o, acc32)
    layouts = _layouts(N // 2 if ep == 'swiglu' else N)

    def launch():
        runs = {('default grid', lay): run_epilogue(ep, o, lay) for lay in layouts}
        with small_grid():
            runs.update({('2-CTA grid', lay): run_epilogue(ep, o, lay) for lay in layouts})
        return runs

    runs, seen = launched_widths(launch)
    assert seen == {(False, 0, 0, width)}, seen
    got = runs['default grid', layouts[0]].out
    for (grid, (name, ld, col0)), cv in runs.items():
        what = '%s, BN=%d, %s, %s output (ldd=%d, column %d)' % (ep, width, grid, name, ld, col0)
        cv.check(what)
        assert torch.equal(cv.out, got), what + ': differs from the vector output on the default grid'
    if ep.startswith('splitk'):
        close(got.reshape(int(ep[-1]), M, N).sum(0), o.a.float() @ o.b.float().t(), rtol=1e-4, atol=1e-3)
    elif ep == 'out32':
        close(got, want, rtol=1e-4, atol=1e-3)
    else:
        close(got, want)
    if exact is not None:
        assert torch.equal(got, exact), '%s, BN=%d: differs from the epilogue applied to the fp32 accumulators' % (ep, width)
    if width == 256:
        assert torch.equal(_at_128(monkeypatch, lambda: run_epilogue(ep, o, layouts[0])).out, got), \
            '%s: the 256 and 128 kernels differ' % ep


# ---- fused QKV projection + rotary embedding ------------------------------------------------------------------

POS0, POS_DEV, POS_ROWS = 37, 61, (0, 37, 300, 5)
QKV_CASES = [
    (2, 77, 4, 'pos0', BF), (2, 77, 4, 'pos_dev', BF),      # N = 1536: whole 256 tiles
    (3, 50, 3, 'pos0', BF), (3, 50, 3, 'pos_dev', BF),      # N = 1152: the last 256 tile's second half lies past N
    (3, 17, 3, 'pos_rows', BF), (4, 150, 4, 'pos_rows', BF),  # PrefillEngine.extend: samples end inside 128-row tiles
    (4, 150, 4, 'pos_rows', H),
]


def rope_tables(n, dt):
    """cos / sin [n, 128] at positions 0..n-1, LLaMA's frequencies.  The two halves of each row differ (HF's are
    equal), so an epilogue that reads the wrong half shows."""
    inv = 1.0 / (10000.0 ** (torch.arange(0, 128, 2).float() / 128))
    fr = torch.arange(n).float()[:, None] * inv[None]
    emb = torch.cat([fr, 1.3 * fr + 0.7], -1)
    return emb.cos().to(DEV, dt).contiguous(), emb.sin().to(DEV, dt).contiguous()


@pytest.mark.parametrize('B,L,nh,mode,dt', QKV_CASES,
                         ids=['B%d-L%d-H%d-%s-%s' % (c[:4] + ('bf16' if c[4] == BF else 'fp16',)) for c in QKV_CASES])
def test_qkv_rope(width, monkeypatch, B, L, nh, mode, dt):
    torch.manual_seed(B * L + nh)
    M, K, rope_cols = B * L, nh * 128, 2 * nh * 128
    x = (torch.randn(M, K, device=DEV) * 0.5).to(dt)
    w = (torch.randn(3 * K, K, device=DEV) * K ** -0.5).to(dt)
    cos, sin = rope_tables(512, dt)
    starts = {'pos0': [POS0] * B, 'pos_dev': [POS_DEV] * B, 'pos_rows': list(POS_ROWS[:B])}[mode]

    def run():
        if mode == 'pos0':
            return dense.qkv_rope(x, w, cos, sin, L, rope_cols, pos0=POS0)
        if mode == 'pos_dev':
            return dense.qkv_rope(x, w, cos, sin, L, rope_cols, pos_dev=torch.tensor([POS_DEV], dtype=torch.int32, device=DEV))
        return dense.qkv_rope(x, w, cos, sin, L, rope_cols, pos_rows=torch.tensor(starts, dtype=torch.int32, device=DEV))

    def launch():
        out = run()
        with small_grid():
            return out, run()

    (got, got_small), seen = launched_widths(launch)
    assert seen == {(False, 0, 0, width)}, seen
    assert torch.isfinite(got.float()).all()
    assert torch.equal(got, got_small), 'BN=%d: the 2-CTA grid differs' % width
    # unfused: the plain GEMM, then the rope kernel on each sample's rows with its own slice of the tables
    unfused = dense.linear(x, w)
    for b, s in enumerate(starts):
        kernels.rope_inplace(unfused[b * L:(b + 1) * L], cos[s:s + L].contiguous(), sin[s:s + L].contiguous(), L,
                             2 * nh, 128)
    assert torch.equal(got, unfused), 'BN=%d: fused RoPE differs from GEMM + rope kernel' % width
    # fp32 HF formula: q * cos + rotate_half(q) * sin
    base = x.float() @ w.float().t()
    pos = torch.tensor([starts[r // L] + r % L for r in range(M)], device=DEV)
    c, s = cos.float()[pos][:, None], sin.float()[pos][:, None]
    qk = base[:, :rope_cols].reshape(M, 2 * nh, 128)
    want = base.clone()
    want[:, :rope_cols] = (qk * c + torch.cat([-qk[..., 64:], qk[..., :64]], -1) * s).reshape(M, rope_cols)
    (_close_bf16 if dt == BF else _close_f16)(got, want)
    if width == 256:
        assert torch.equal(_at_128(monkeypatch, run), got), 'the 256 and 128 kernels differ'


# ---- implicit-GEMM conv, each branch of conv_tiling -----------------------------------------------------------

CONV_CASES = [  # n, H, W, Cin, Cout, k, levels, bias, act, dtype
    (2, 16, 16, 64, 128, 3, 1, 'bf16', 'relu', BF),      # 16-wide tile
    (2, 24, 24, 128, 256, 3, 1, None, None, BF),         # 8-wide tile
    (2, 12, 12, 64, 48, 3, 1, 'bf16', None, BF),         # partial x tile; GroupNorm over 3 groups
    (2, 7, 7, 64, 64, 3, 1, 'f32', 'relu', BF),          # W < 8: 49-row tile
    (1, 6, 6, 64, 16, 1, 1, None, 'relu', BF),           # GroupNorm over 1 group
    (3, 14, 14, 1024, 1024, 3, 4, 'f32', 'relu', BF),    # the RoI pconv: 126-row tile, sum over 4 pyramid levels
    (2, 12, 12, 64, 48, 3, 1, 'bf16', None, H),
]


def _conv_id(c):
    n, Hh, W, cin, cout, k, lv, bias, act, dt = c
    return 'n%d-%dx%d-%dto%d-k%d-lv%d-%s-%s' % (n, Hh, W, cin, cout, k, lv, act or 'none', 'bf16' if dt == BF else 'fp16')


def conv_reference(x, w, bias, act, n, levels):
    """Sum over levels of F.conv2d on each level's images with that level's weight slice, in fp32 (no TF32)."""
    k = w.shape[-2]
    xs = x.float().permute(0, 3, 1, 2)
    ws = w.float() if levels > 1 else w.float()[:, None]
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        y = sum(F.conv2d(xs[l * n:(l + 1) * n], ws[:, l].permute(0, 3, 1, 2), padding=k // 2) for l in range(levels))
    if bias is not None:
        y = y + bias.float()[None, :, None, None]
    if act == 'relu':
        y = torch.relu(y)
    return y.permute(0, 2, 3, 1)


@pytest.mark.parametrize('n,Hh,W,cin,cout,k,levels,bias_kind,act,dt', CONV_CASES, ids=[_conv_id(c) for c in CONV_CASES])
def test_conv(width, monkeypatch, n, Hh, W, cin, cout, k, levels, bias_kind, act, dt):
    torch.manual_seed(Hh * W + cout + levels)
    x = torch.randn(levels * n, Hh, W, cin, device=DEV).to(dt)
    wshape = (cout, levels, k, k, cin) if levels > 1 else (cout, k, k, cin)
    w = (torch.randn(wshape, device=DEV) * (levels * k * k * cin) ** -0.5).to(dt)
    bias = None if bias_kind is None else (torch.randn(cout, device=DEV) * 0.5).to(F32 if bias_kind == 'f32' else dt)
    groups, slots = cout // 16, dense.gn_slots(Hh, W)

    def run(fill=float('nan')):
        cv = Canvas(n * Hh * W, cout, dt, cout)
        st = torch.full((n, slots, groups, 2), fill, device=DEV)
        dense.conv_nhwc(x, w, bias, act=act, gn_stats=st, out=cv.out.view(n, Hh, W, cout), levels=levels)
        return cv, st

    def launch():
        out = run()
        with small_grid():
            return out, run()

    ((cv, st), (cv_s, st_s)), seen = launched_widths(launch)
    assert seen == {(True, 0, 0, width)}, seen
    cv.check('conv BN=%d' % width)
    cv_s.check('conv BN=%d, 2-CTA grid' % width)
    # every (tile, warp) slot of every group is stored: none is left NaN, and a zero-filled buffer ends up equal
    _, st0 = run(0.0)
    for s, grid in ((st, 'default grid'), (st_s, '2-CTA grid')):
        missing = torch.isnan(s).any(-1).any(1)   # [image, group]
        assert not bool(missing.any()), 'BN=%d, %s: GroupNorm slots not stored for (image, group) %s' % (
            width, grid, missing.nonzero().tolist())
    assert torch.equal(st, st0), 'BN=%d: GroupNorm statistics depend on the prefill' % width
    got = cv.out.view(n, Hh, W, cout)
    assert torch.equal(cv_s.out, cv.out) and torch.equal(st_s, st), 'BN=%d: the 2-CTA grid differs' % width
    (_close_bf16 if dt == BF else _close_f16)(got, conv_reference(x, w, bias, act, n, levels))
    # the statistics are those of the stored 16-bit output
    g = got.double().reshape(n, Hh * W, groups, 16)
    tot = st.double().sum(1)
    for i, ref in enumerate((g.sum((1, 3)), (g * g).sum((1, 3)))):
        bound = 1e-5 * (g.abs() if i == 0 else g * g).sum((1, 3)) + 1e-6
        assert bool(((tot[..., i] - ref).abs() <= bound).all()), ('sum', 'sum of squares')[i]
    if width == 256:
        cv128, st128 = _at_128(monkeypatch, run)
        assert torch.equal(cv128.out, cv.out) and torch.equal(st128, st), 'the 256 and 128 kernels differ'


# ---- MN-major operands (the training step's backward GEMMs, 128-wide tiles only) ------------------------------

@pytest.mark.parametrize('out_dtype', [BF, F32], ids=['bf16', 'fp32'])
@pytest.mark.parametrize('a_mn,b_mn', [(False, True), (True, True), (True, False)], ids=['NT', 'TT', 'TN'])
@pytest.mark.parametrize('M,N,K', [(296, 648, 520), (1024, 1000, 264)])
def test_matmul_t_small_grid(M, N, K, a_mn, b_mn, out_dtype):
    torch.manual_seed(M + N + K)
    a = (torch.randn(M, K, device=DEV) * 0.5).bfloat16()
    b = (torch.randn(N, K, device=DEV) * K ** -0.5).bfloat16()
    a_st = a.t().contiguous() if a_mn else a
    b_st = b.t().contiguous() if b_mn else b

    layouts = _layouts(N)

    def run(layout):
        cv = Canvas(M, N, out_dtype, layout[1], layout[2])
        dense.matmul_t(a_st, b_st, a_mn, b_mn, out_dtype=out_dtype, out=cv.out)
        return cv

    def launch():
        runs = {('default grid', lay): run(lay) for lay in layouts}
        with small_grid():
            runs.update({('2-CTA grid', lay): run(lay) for lay in layouts})
        return runs

    runs, seen = launched_widths(launch)
    assert seen == {(False, int(a_mn), int(b_mn), 128)}, seen
    got = runs['default grid', layouts[0]].out
    for (grid, (name, ld, col0)), cv in runs.items():
        what = 'matmul_t, %s, %s output (ldd=%d, column %d)' % (grid, name, ld, col0)
        cv.check(what)
        assert torch.equal(cv.out, got), what + ': differs from the vector output on the default grid'
    want = a.float() @ b.float().t()
    if out_dtype == F32:
        _close_bf16(got, want, rtol=1e-4, atol=1e-3)
    else:
        _close_bf16(got, want)


# ---- the width rule -------------------------------------------------------------------------------------------

def _rule(m_tiles, n, grid):
    """pick_block_n: the width with fewer rounds x tile cost, a 128 x 256 tile costing 1.6 128 x 128 tiles."""
    rounds = lambda bn: -(-(m_tiles * -(-n // bn)) // grid)
    return 256 if rounds(256) * 160 < rounds(128) * 100 else 128


# (name, M, N, width on 132 SMs) from the comment above pick_block_n; K does not enter the rule.
RULE_GEMMS = [('LLaMA q|k|v', 5648, 12288, 256), ('LLaMA o_proj', 5648, 4096, 256),
              ('LLaMA gate|up', 5648, 22016, 256), ('ViT out_proj', 4616, 1024, 128)]


def test_width_rule(monkeypatch):
    monkeypatch.delenv('G4R_GEMM_BN', raising=False)
    sms = _num_sms()
    for name, M, N, on_h100 in RULE_GEMMS:
        a = torch.randn(M, 64, device=DEV).bfloat16()
        b = torch.randn(N, 64, device=DEV).bfloat16()
        m_tiles = -(-M // 128)
        if sms == 132:
            assert _rule(m_tiles, N, sms) == on_h100, name
        for grid in (sms, 2):
            with sm_budget(grid):
                _, seen = launched_widths(lambda: dense.linear(a, b))
            assert seen == {(False, 0, 0, _rule(m_tiles, N, grid))}, (name, grid, seen)
    # the conv applies the same rule to its spatial tiles: 2 x 24 x 24 -> 256 channels is 12 tiles of 128 pixels
    x = torch.randn(2, 24, 24, 64, device=DEV).bfloat16()
    w = torch.randn(256, 1, 1, 64, device=DEV).bfloat16()
    m_tiles = 2 * dense.gn_slots(24, 24) // 4
    for grid in (sms, 2):
        with sm_budget(grid):
            _, seen = launched_widths(lambda: dense.conv_nhwc(x, w))
        assert seen == {(True, 0, 0, _rule(m_tiles, 256, grid))}, ('conv', grid, seen)
