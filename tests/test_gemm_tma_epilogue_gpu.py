"""The register epilogue of the wgmma GEMM (csrc/gemm_wgmma.cu, epilogue_regs): 16-bit outputs whose rows allow
16-byte vector accesses are finished from the accumulators and written with TMA stores, the residual loaded by TMA
into the same staging boxes.  Outputs whose base is not 16-byte aligned take the staged epilogue, so each case here
runs the same op both ways and requires bitwise equality, on a 2-CTA grid where every CTA runs many consecutive
tiles of the kind (the staging boxes are reused from one tile to the next), with
  * a 16-row last row tile (M = 3 * 128 + 16) and N = 1040 (SwiGLU: 520 output columns), which ends inside a
    64-column box, in a padded row; every element outside the output stays bitwise unchanged;
  * the output written in place over its own residual (out=residual);
  * RoPE at per-sample positions, samples ending inside row tiles, against the GEMM followed by the rope kernel."""
import pytest
import torch

from gpt4roi_b200 import dense, kernels, lib
from tests.test_gemm_tiles_gpu import Canvas, rope_tables, small_grid, width  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
BF, H, F32 = torch.bfloat16, torch.float16, torch.float32
M, N, K = 3 * 128 + 16, 1040, 192
LD = 1048   # a 16-byte row pitch: column 0 takes the register epilogue, column 1 the staged one
KINDS = ('none', 'bias_relu', 'bias32_quick_gelu', 'residual', 'swiglu')


def _operands(dt):
    g = torch.Generator(device=DEV).manual_seed(11)
    rn = lambda *s, scale=1.0: torch.randn(*s, generator=g, device=DEV) * scale  # noqa: E731
    return dict(a=rn(M, K).to(dt), b=rn(N, K, scale=K ** -0.5).to(dt), bias=rn(N, scale=0.5).to(dt),
                bias32=rn(N, scale=0.5), res=rn(M, N).to(dt))


def _run(kind, o, dt, col0, in_place=False):
    n_out = N // 2 if kind == 'swiglu' else N
    cv = Canvas(M, n_out, dt, LD, col0)
    kw = {'none': {}, 'bias_relu': dict(bias=o['bias'], act='relu'),
          'bias32_quick_gelu': dict(bias=o['bias32'], act='quick_gelu'), 'swiglu': dict(act='swiglu')}.get(kind)
    if kind == 'residual':
        if in_place:
            cv.out.copy_(o['res'])
            kw = dict(residual=cv.out)
        else:
            res = torch.zeros(M, LD, dtype=dt, device=DEV)[:, col0:col0 + N]
            res.copy_(o['res'])
            kw = dict(residual=res)
    dense.linear(o['a'], o['b'], out=cv.out, **kw)
    return cv


@pytest.mark.parametrize('dt', [BF, H], ids=['bf16', 'fp16'])
@pytest.mark.parametrize('kind', KINDS)
def test_register_epilogue_matches_staged(width, kind, dt):
    o = _operands(dt)
    with small_grid():
        got = _run(kind, o, dt, 0)
        staged = _run(kind, o, dt, 1)
        again = _run(kind, o, dt, 0)
    for cv, what in ((got, 'register'), (staged, 'staged')):
        cv.check('%s, BN=%d, %s epilogue' % (kind, width, what))
    assert torch.equal(got.out, staged.out), '%s, BN=%d: register and staged epilogues differ' % (kind, width)
    assert torch.equal(got.out, again.out), '%s, BN=%d: not reproducible' % (kind, width)
    assert torch.equal(_run(kind, o, dt, 0).out, got.out), '%s, BN=%d: the full grid differs' % (kind, width)


@pytest.mark.parametrize('dt', [BF, H], ids=['bf16', 'fp16'])
def test_residual_in_place(width, dt):
    o = _operands(dt)
    want = _run('residual', o, dt, 0)
    with small_grid():
        got = _run('residual', o, dt, 0, in_place=True)
    got.check('in-place residual, BN=%d' % width)
    assert torch.equal(got.out, want.out), 'BN=%d: out=residual differs from a separate output' % width


@pytest.mark.parametrize('dt', [BF, H], ids=['bf16', 'fp16'])
def test_rope_per_row_positions(width, dt):
    B, L, nh = 4, 100, 2            # M = 400: samples end inside row tiles, a 16-row last tile
    Mr, Kr, rope_cols = B * L, nh * 128, 2 * nh * 128
    g = torch.Generator(device=DEV).manual_seed(5)
    x = (torch.randn(Mr, Kr, generator=g, device=DEV) * 0.5).to(dt)
    w = (torch.randn(3 * Kr, Kr, generator=g, device=DEV) * Kr ** -0.5).to(dt)
    cos, sin = rope_tables(512, dt)
    pos_rows = torch.tensor([0, 37, 300, 5], dtype=torch.int32, device=DEV)
    fn = getattr(lib.load(), lib.sym('g4r_gemm_qkv_rope_rows_bf16', dt))

    # the fused RoPE epilogue needs a 16-byte aligned output, so the reference is the unfused one: the plain GEMM,
    # then the rope kernel on each sample's rows with its own slice of the tables
    cv = Canvas(Mr, 3 * Kr, dt, 3 * Kr + 8)
    with small_grid(), torch.cuda.device(DEV):
        lib.check(fn(lib.ptr(x), Kr, lib.ptr(w), Kr, lib.ptr(cv.out), 3 * Kr + 8, Mr, 3 * Kr, Kr, lib.ptr(cos),
                     lib.ptr(sin), rope_cols, L, lib.ptr(pos_rows), lib.stream_ptr(torch.device(DEV))))
    cv.check('RoPE, BN=%d' % width)
    unfused = dense.linear(x, w)
    for b, s in enumerate(pos_rows.tolist()):
        kernels.rope_inplace(unfused[b * L:(b + 1) * L], cos[s:s + L].contiguous(), sin[s:s + L].contiguous(), L,
                             2 * nh, 128)
    assert torch.equal(cv.out, unfused), 'RoPE, BN=%d: fused RoPE differs from GEMM + rope kernel' % width
    assert torch.equal(dense.qkv_rope(x, w, cos, sin, L, rope_cols, pos_rows=pos_rows), cv.out)
