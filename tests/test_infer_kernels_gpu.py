"""Each inference elementwise kernel of csrc/elementwise.cu on its own, bf16 and its fp16 twin (csrc/act_type.cuh),
through the `kernels` wrappers PrefillEngine calls, at the shapes the engine runs (EngineConfig at 224 and 336 px),
against plain torch of the same operation in float64 on the device, run on the same 16-bit inputs.  Where a kernel
rounds in the middle the reference rounds at the same point.  Copies, casts and layout kernels must match bit for bit.

Notation used in the docstrings: u = 2^-24 is the fp32 unit roundoff; u16 is the storage type's, 2^-8 for bf16 and
2^-11 for fp16.  A kernel that computes y in fp32 to within e32 of the exact y and rounds it once to the storage type
returns a value between rd(y - e32) and rd(y + e32), because rounding is monotone: `_check_rounded` asserts exactly
that interval.  Where y +- e32 round to the same value the output is that value, bit for bit.

Every output buffer is filled with NaN before the call (through the wrapper's `out=`, or by calling the entry point
through `lib` with an output of our own), so an element a kernel fails to write is caught rather than read back from
the caching allocator's block of an earlier identical call.  The grid-stride kernels are launched on at most
num_sms * 16 blocks of 256 threads (fuse_gather: num_sms * 32 blocks); each test asserts from the device's SM count
that at least one of its cases needs more than one pass of the loop."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from gpt4roi_b200 import dense, kernels
from gpt4roi_b200 import lib as _L

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
BF, H16, F32, F64 = torch.bfloat16, torch.float16, torch.float32, torch.float64
DTS = [pytest.param(BF, id='bf16'), pytest.param(H16, id='fp16')]
U = 2.0 ** -24
U16 = {BF: 2.0 ** -8, H16: 2.0 ** -11}
PYR = {336: (192, 96, 48, 24), 224: (128, 64, 32, 16)}


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


def passes(total, per_block=256, cap_per_sm=16):
    """Passes of a grid-stride loop over `total` items, `per_block` per block, on min(blocks needed, num_sms *
    cap_per_sm) blocks -- grid_for in csrc/elementwise.cu (and the affine_relu / fuse_gather launchers)."""
    blocks = min(-(-total // per_block), sms() * cap_per_sm)
    return -(-total // (blocks * per_block))


def _check_rounded(got, ref, e32, dt, what=''):
    """got: the kernel's storage-type output of a value it computed in fp32 within e32 of the fp64 `ref` and rounded
    once.  Rounding is monotone, so rd(ref - e32) <= got <= rd(ref + e32).  NaN (an unwritten sentinel) fails."""
    lo = (ref - e32).to(dt).double()
    hi = (ref + e32).to(dt).double()
    g = got.double()
    ok = (g >= lo) & (g <= hi)
    if not bool(ok.all()):
        i = tuple((~ok).nonzero()[0].tolist())
        raise AssertionError('%s: %d of %d outside [rd(ref - e32), rd(ref + e32)]; first at %s: got %r, want %r..%r'
                             % (what, int((~ok).sum()), ok.numel(), i, g[i].item(), lo[i].item(), hi[i].item()))


def _check_within(got, ref, bound, what=''):
    err = (got.double() - ref).abs()
    ok = err <= bound
    assert bool(ok.all()), '%s: %d of %d over the bound; worst excess %.3e' % (
        what, int((~ok).sum()), ok.numel(), (err - bound).max().item())


# ---------------------------------------------------------------------------------------------------------------
# ViT front: patchify, embeddings
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dt', DTS)
@pytest.mark.parametrize('S', [224, 336])
def test_patchify_is_unfold(S, dt):
    """A pure layout kernel: rows [B*P, 592] equal F.unfold(stride = patch) bit for bit, including -0, +-inf and the
    storage type's smallest subnormal, and the 4 pad columns are +0.  One element per thread: 8 images at 336 px are
    2.7M elements, several passes of the loop."""
    B, ps, kpad = 8, 14, 592
    G = S // ps
    torch.manual_seed(S)
    img = torch.randn(B, 3, S, S, device=DEV).to(dt)
    flat = img.view(-1)
    tiny = torch.finfo(dt).tiny * torch.finfo(dt).eps
    for j, v in zip((0, 12345, flat.numel() // 2 + 7, flat.numel() - 1), (-0.0, float('inf'), -float('inf'), tiny)):
        flat[j] = v
    assert passes(B * G * G * kpad) > 1
    out = nan((B * G * G, kpad), dt)
    raw('g4r_patchify_bf16', dt, ptr(img), ptr(out), B, S, ps, kpad)
    want = torch.zeros(B * G * G, kpad, dtype=dt, device=DEV)
    want[:, :3 * ps * ps] = F.unfold(img.float(), ps, stride=ps).transpose(1, 2).reshape(-1, 3 * ps * ps).to(dt)
    assert torch.equal(bits(out), bits(want))
    assert torch.equal(bits(kernels.patchify(img, ps, kpad)), bits(out))


@pytest.mark.parametrize('dt', DTS)
def test_vit_embed_is_one_rounding(dt):
    """x[b, 0] = cls + pos[0], x[b, 1 + p] = patch[b, p] + pos[1 + p]: one fp32 add of two 16-bit values and one
    rounding, the same operations as (x.float() + pos.float()).to(dt), so bit for bit.  B = 8, P = 576, D = 1024 is
    590 848 vectors: two passes on a 132-SM H100."""
    B, P, D = 8, 576, 1024
    torch.manual_seed(1)
    patch = (torch.randn(B * P, D, device=DEV) * 0.5).to(dt)
    cls = torch.randn(D, device=DEV).to(dt)
    pos = (torch.randn(P + 1, D, device=DEV) * 0.1).to(dt)
    assert passes(B * (P + 1) * D // 8) > 1
    out = nan((B, P + 1, D), dt)
    raw('g4r_vit_embed_bf16', dt, ptr(patch), ptr(cls), ptr(pos), ptr(out), B, P, D)
    x = torch.cat([cls.expand(B, 1, D), patch.view(B, P, D)], 1)
    want = (x.float() + pos.float()[None]).to(dt)
    assert torch.equal(bits(out), bits(want))
    assert torch.equal(bits(kernels.vit_embed(patch, cls, pos, B, P)), bits(out))


# ---------------------------------------------------------------------------------------------------------------
# Row norms
# ---------------------------------------------------------------------------------------------------------------
def _chain(D):
    """Longest fp32 addition chain of a row statistic: the warp-per-row kernel sums 8 * ceil(D / 256) values per lane
    and 5 shuffle levels; the CTA-per-row kernel 8 * ceil(D / 2048) per thread, 5 levels and 8 warp partials."""
    return 8 * -(-D // 256) + 13


def _ln_ref(x, w, b, eps):
    """fp64 LayerNorm of the (exact) input rows and the fp32 error budget of the kernel's output before any final
    rounding.  The mean carries (n + 1)u mean|x|; the two-pass variance (n + 4)u relative plus the mean's error
    squared; rsqrtf 2 ulp (4u), so rstd is within e_v / 2 + 4u relative; (x - mean) * rstd * w + b adds <= 4 roundings."""
    xd = x.double()
    D = xd.shape[-1]
    n = _chain(D)
    mean = xd.mean(-1, keepdim=True)
    var = (xd - mean).pow(2).mean(-1, keepdim=True)
    rstd = (var + eps).rsqrt()
    xh = (xd - mean) * rstd
    wd, bd = w.double(), b.double()
    ref = xh * wd + bd
    e_mean = (n + 1) * U * xd.abs().mean(-1, keepdim=True)
    r_rstd = ((n + 4) * U * var + e_mean ** 2) / (var + eps) / 2 + 4 * U
    e32 = wd.abs() * (xh.abs() * (r_rstd + 2 * U) + e_mean * rstd) + 2 * U * ((wd * xh).abs() + bd.abs())
    return ref, e32


def _rows(M, D, dt, seed, ld=None):
    """M rows of width D with per-row offsets from -4 to 4 (|mean| up to ~2 sigma); a view of a wider buffer for
    ld > D."""
    torch.manual_seed(seed)
    ld = D if ld is None else ld
    buf = torch.randn(M, ld, device=DEV) * 2 + torch.linspace(-4, 4, M, device=DEV)[:, None]
    return buf.to(dt)[:, :D]


@pytest.mark.parametrize('dt', DTS)
@pytest.mark.parametrize('x32,o32', [(False, False), (False, True), (True, False), (True, True)],
                         ids=['16to16', '16to32', '32to16', '32to32'])
def test_layernorm_ex_matches_fp64(x32, o32, dt):
    """CLIP's norms on the fp32 residual stream (vit_pre_ln: 16-bit -> fp32; ln1 / ln2: fp32 -> 16-bit) and the other
    two combinations, D = 1024, against fp64 LayerNorm of the same rows.  fp32 outputs are within e32 (_ln_ref);
    16-bit ones between rd(ref -+ e32).  Rows M = 577 and 8 * 577 (the engine's B = 1 and 8), M = 1..17 (partial
    8-row CTAs) and M = 577 read from a buffer with row stride 1088."""
    D, eps = 1024, 1e-5
    torch.manual_seed(7)
    w = (torch.rand(D, device=DEV) + 0.5).to(dt)
    b = (torch.randn(D, device=DEV) * 0.5).to(dt)
    xt = F32 if x32 else dt
    ot = F32 if o32 else dt
    cases = [(577, None), (8 * 577, None), (577, D + 64)] + [(m, None) for m in range(1, 18)]
    for M, ld in cases:
        x = _rows(M, D, xt, M, ld)
        out = nan((M, D), ot)
        raw('g4r_layernorm_ex', dt, ptr(x), x.stride(0), int(x32), ptr(w), ptr(b), ptr(out), out.stride(0), int(o32),
            M, D, eps)
        ref, e32 = _ln_ref(x, w, b, eps)
        what = 'M=%d ld=%s' % (M, ld)
        if o32:
            _check_within(out, ref, e32, what)
        else:
            _check_rounded(out, ref, e32, dt, what)
        assert torch.equal(bits(kernels.layernorm_ex(x, w, b, eps, out_dtype=ot)), bits(out))


def _rms_ref(x, eps):
    """z = x * rsqrt(mean(x^2) + eps) in fp64 and the kernel's fp32 error on it: the sum of squares carries (n + 1)u
    relative, / D and + eps 2u more, rsqrtf 4u: rstd within (n + 3)u / 2 + 4u; the product one more u."""
    xd = x.double()
    n = _chain(xd.shape[-1])
    rstd = (xd.pow(2).mean(-1, keepdim=True) + eps).rsqrt()
    z = xd * rstd
    return z, z.abs() * ((n + 3) * U / 2 + 5 * U)


@pytest.mark.parametrize('dt', DTS)
@pytest.mark.parametrize('D', [1024, 4096, 8192, 520])
@pytest.mark.parametrize('M', [1, 8, 64, 65, 5648])
def test_norm_16bit_rows_both_paths(M, D, dt):
    """layernorm / rmsnorm on 16-bit rows: M <= 64 takes the CTA-per-row kernel (decode step), M = 65 and 5648 (B = 8
    x L = 706) the warp-per-row kernel.  LayerNorm: between rd(ref -+ e32) (_ln_ref).  RMSNorm is LlamaRMSNorm:
    w * rd(x * rstd), so the reference rounds z = x * rstd to the storage type before the weight.  The kernel's z is
    within e_z of the exact one (_rms_ref), so its rounded z lies between rd(z - e_z) and rd(z + e_z); w times a
    16-bit value is exact in fp32, so the output lies between rd(w * rd(z - e_z)) and rd(w * rd(z + e_z))."""
    torch.manual_seed(M + D)
    x = _rows(M, D, dt, M * 7 + D)
    w = (torch.rand(D, device=DEV) + 0.5).to(dt)
    w[::7] *= -1
    b = (torch.randn(D, device=DEV) * 0.5).to(dt)
    out = nan((M, D), dt)
    kernels.layernorm(x, w, b, 1e-5, out=out)
    ref, e32 = _ln_ref(x, w, b, 1e-5)
    _check_rounded(out, ref, e32, dt, 'layernorm')

    out = nan((M, D), dt)
    kernels.rmsnorm(x, w, 1e-6, out=out)
    z, ez = _rms_ref(x, 1e-6)
    wd = w.double()
    a = (wd * (z - ez).to(dt).double()).to(dt).double()
    c = (wd * (z + ez).to(dt).double()).to(dt).double()
    g = out.double()
    ok = (g >= torch.minimum(a, c)) & (g <= torch.maximum(a, c))
    assert bool(ok.all()), 'rmsnorm: %d of %d outside' % (int((~ok).sum()), ok.numel())


@pytest.mark.parametrize('dt', DTS)
@pytest.mark.parametrize('M', [1, 65, 5648])
def test_rmsnorm_fp32_rows_matches_fp64(M, dt):
    """rmsnorm on an fp32 residual stream (llama_stream='fp32'), D = 4096, rows read with stride 4160: LlamaRMSNorm
    does not round x * rstd for fp32 input, so out = rd(w * z) with the kernel's w * z within |w z| (e_z + u) of the
    fp64 value (_rms_ref)."""
    D = 4096
    x = _rows(M, D, F32, M, D + 64)
    torch.manual_seed(M)
    w = (torch.rand(D, device=DEV) + 0.5).to(dt)
    out = nan((M, D), dt)
    kernels.rmsnorm(x, w, 1e-6, out=out)
    z, ez = _rms_ref(x, 1e-6)
    wd = w.double()
    _check_rounded(out, wd * z, wd.abs() * (ez + U * z.abs()), dt)


# ---------------------------------------------------------------------------------------------------------------
# RoPE, token cast
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dt', DTS)
def test_rope_is_hf_formula_bit_for_bit(dt):
    """q * cos + rotate_half(q) * sin on the q and k heads of the packed [B*L, q|k|v] rows (B = 8, L = 706: 5648 rows,
    32 heads each, head_dim 128), with the cos / sin tables built as LlamaRotaryEmbedding builds them.  Run in torch in
    the storage type, each op rounds once; the kernel rounds at the same three points, so bit for bit.  v stays
    untouched.  2.9M vectors: several passes."""
    B, L, nh, D = 8, 706, 32, 128
    torch.manual_seed(5)
    qkv = torch.randn(B * L, 3 * nh * D, device=DEV).to(dt)
    inv = 1.0 / (10000.0 ** (torch.arange(0, D, 2, dtype=torch.int64).float() / D))
    fr = torch.arange(L, dtype=torch.float32)[:, None] * inv[None, :]
    emb = torch.cat((fr, fr), -1)
    cos, sin = emb.cos().to(DEV, dt).contiguous(), emb.sin().to(DEV, dt).contiguous()
    assert passes(B * L * 2 * nh * D // 16) > 1
    ref = qkv.clone().view(B, L, 3 * nh, D)
    got = kernels.rope_inplace(qkv, cos, sin, L, 2 * nh, D).view(B, L, 3 * nh, D)
    qk = ref[:, :, :2 * nh]
    rot = torch.cat((-qk[..., D // 2:], qk[..., :D // 2]), -1)
    want = qk * cos[None, :, None, :] + rot * sin[None, :, None, :]
    assert torch.equal(bits(got[:, :, :2 * nh]), bits(want))
    assert torch.equal(bits(got[:, :, 2 * nh:]), bits(ref[:, :, 2 * nh:]))


def _i32(patterns):
    return torch.tensor([p - (1 << 32) if p >= 1 << 31 else p for p in patterns], dtype=torch.int32, device=DEV)


# fp32 bit patterns where a cast to bf16 or fp16 goes wrong first
CAST_PATTERNS = [
    0x3F808000, 0x3F818000, 0xBF808000, 0x3F808001, 0x3F807FFF,          # bf16 ties, just off ties
    0x3F801000, 0x3F803000, 0xBF801000, 0x3F801001,                      # fp16 ties, just off a tie
    0x00000001, 0x007FFFFF, 0x80000001, 0x00008000,                      # fp32 subnormals
    0x33000000, 0x33400000, 0x33800000, 0xB3000000, 0x3727C5AC,          # fp16 subnormal range: 2^-25, 3*2^-26, 2^-24
    0x477FE000, 0x477FEFFF, 0x477FF000, 0x47C35000, 0xC7C35000,          # fp16 max, just below / at overflow, +-1e5
    0x7F7F7FFF, 0x7F7F8000, 0x7F7FFFFF, 0xFF7F8000,                      # near / above bf16 max
    0x00000000, 0x80000000, 0x7F800000, 0xFF800000,                      # zeros, infinities
    0x7FC00000, 0x7F800001, 0xFFC00001,                                  # NaNs
]


@pytest.mark.parametrize('dt', DTS)
def test_cast_tokens_matches_torch_bit_for_bit(dt):
    """The mm_projector input: hidden[:, 1:] of the fp32 ViT stream [B = 8, T = 577, C = 1024] to dense 16-bit rows,
    equal to torch's .to(dt) (on the host) bit for bit: ties both ways, subnormals, +-0, +-inf, values that overflow
    fp16 or bf16; NaN in -> NaN out.  The patterns sit in the dropped CLS rows too, in the middle of a vector and in
    the last row of the last image.  589 824 vectors: two passes on a 132-SM H100."""
    B, T, C = 8, 577, 1024
    torch.manual_seed(2)
    hid = torch.randn(B, T, C, device=DEV) * 3
    n = len(CAST_PATTERNS)
    iv = hid.view(B, T * C).view(torch.int32)
    for b in range(B):
        for start in (0, C + 5 * b, (T - 1) * C + 3):
            iv[b, start:start + n] = _i32(CAST_PATTERNS)
    assert passes(B * (T - 1) * C // 8) > 1
    out = nan((B * (T - 1), C), dt)
    raw('g4r_cast_f32_bf16', dt, ptr(hid, C), C, T * C, ptr(out), B, T - 1, C)
    src = hid[:, 1:].reshape(-1, C)
    isn = torch.isnan(src)
    assert torch.isnan(out[isn]).all()
    want = src.cpu().to(dt).to(DEV)
    assert torch.equal(bits(out)[~isn], bits(want)[~isn])
    again = kernels.cast_tokens_f32_bf16(hid, dtype=dt)
    assert torch.equal(bits(again)[~isn], bits(out)[~isn])


# ---------------------------------------------------------------------------------------------------------------
# SPI: token upsampling + coordinates, fuse gather, GroupNorm, affine + ReLU
# ---------------------------------------------------------------------------------------------------------------
def _lerp_e32(Hs, M):
    """fp32 error of an align_corners bilinear resample from Hs pixels, taps at most M in magnitude.  The kernel's
    source position scale * dst (scale = (Hs - 1) / (Ho - 1) rounded, then the product rounded) is within 2u(Hs - 1)
    of the exact one; the interpolant moves by at most 2M per unit of position along each of the two axes: 8u(Hs - 1)M.
    1 - l1 rounds (u per axis) and the two lerp levels round 3 times each: 8uM more."""
    return (8 * (Hs - 1) + 8) * U * M


@pytest.mark.parametrize('dt', DTS)
@pytest.mark.parametrize('tok', ['f32', '16bit'])
@pytest.mark.parametrize('B', [1, 4])
@pytest.mark.parametrize('S,has_cls', [(336, True), (224, True), (336, False)], ids=['336', '224', '336-nocls'])
def test_upsample_tokens_coords_matches_fp64(S, has_cls, B, tok, dt):
    """ViT tokens (G x G, C = 1024; fp32 as the engine's taps, or 16-bit) to every pyramid level (Ho = G, 2G, 4G, 8G;
    Ho = G is the identity), Cpad = 1088.  Feature channels vs fp64 F.interpolate(align_corners=True): between
    rd(ref -+ e32), e32 from _lerp_e32 with M = max|tap| (0 for the identity, where the weights are exactly 1 and 0).
    Channel C is x = linspace(-1, 1, Ho)[xo], C + 1 is y, both equal torch.linspace on the device cast to the storage
    type bit for bit; channels C + 2.. are +0.  The 8G levels take several passes."""
    G, C, cpad = S // 14, 1024, 1088
    skip = 1 if has_cls else 0
    T = G * G + skip
    torch.manual_seed(G + B)
    hid = torch.randn(B, T, C, device=DEV) * 1.5
    if tok != 'f32':
        hid = hid.to(dt)
    name = 'g4r_upsample_tokens_coords_f32' if tok == 'f32' else 'g4r_upsample_tokens_coords_bf16'
    taps = hid[:, skip:].double().view(B, G, G, C).permute(0, 3, 1, 2)
    M = taps.abs().max().item()
    assert passes(B * (8 * G) ** 2 * cpad // 8) > 1
    for Ho in (G, 2 * G, 4 * G, 8 * G):
        out = nan((B, Ho, Ho, cpad), dt)
        raw(name, dt, ptr(hid, skip * C), C, T * C, ptr(out), B, G, Ho, C, cpad)
        ref = F.interpolate(taps, size=(Ho, Ho), mode='bilinear', align_corners=True).permute(0, 2, 3, 1)
        _check_rounded(out[..., :C], ref, 0.0 if Ho == G else _lerp_e32(G, M), dt, 'Ho=%d' % Ho)
        lin = bits(torch.linspace(-1, 1, Ho, device=DEV).to(dt))
        assert torch.equal(bits(out[..., C]), lin[None, None, :].expand(B, Ho, Ho)), 'x coordinate, Ho=%d' % Ho
        assert torch.equal(bits(out[..., C + 1]), lin[None, :, None].expand(B, Ho, Ho)), 'y coordinate, Ho=%d' % Ho
        assert bool((bits(out[..., C + 2:]) == 0).all())
        again = kernels.upsample_tokens_coords(hid, G, Ho, cpad, has_cls=has_cls, dtype=dt)
        assert torch.equal(bits(again), bits(out))


def _fuse_launch(B, H, C):
    """(passes, pixel stride) of fuse_gather's grid-stride loop: whole pixels of C / 8 threads per block (2 at
    C = 1024), at most num_sms * 32 blocks."""
    nvec = C // 8
    threads = nvec if nvec >= 256 else (256 // nvec) * nvec
    ppb = threads // nvec
    npix = B * H * H
    blocks = min(-(-npix // ppb), sms() * 32)
    return -(-npix // (blocks * ppb)), blocks * ppb


@pytest.mark.parametrize('dt', DTS)
@pytest.mark.parametrize('affine', [True, False], ids=['gn', 'plain'])
@pytest.mark.parametrize('B', [1, 3])
@pytest.mark.parametrize('sizes', [PYR[336], PYR[224], (200, 100, 50, 25)], ids=['336', '224', 'odd'])
def test_fuse_gather_matches_fp64(sizes, B, affine, dt):
    """One MLVLFuseModule._single_shuffle level for all four levels of the pyramid (l = 0 and 3 take own as down /
    top), C = 1024: [own[:, :C/2] | resize(top[:, 3C/4:]) | resize(down[:, C/2:3C/4])], with the previous round's
    GroupNorm + ReLU relu(v * scale + shift) applied to every tap when `affine`; scale and shift differ per image, so
    a thread that crosses into another image and keeps the old ones is caught.  Reference: the same restatement in
    fp64.  Taps: the affine adds <= 2u(|v scale| + |shift|); resampled blocks add _lerp_e32 of the source size.
    On a 132-SM H100 the pixel stride (8448) is a multiple of every engine pyramid size, so there the x coordinate
    never wraps; the 200/100/50/25 pyramid makes it wrap (asserted), which the engine sizes leave untested."""
    C = 1024
    q = C // 4
    torch.manual_seed(sizes[0] + B + affine)
    maps = [torch.randn(B, h, h, C, device=DEV).to(dt) for h in sizes]
    ss = [(torch.rand(B, C, device=DEV) * 1.5 + 0.25, torch.randn(B, C, device=DEV) * 0.5) if affine else None
          for _ in sizes]
    n_pass, step = _fuse_launch(B, sizes[0], C)
    assert n_pass > 1
    if sizes[0] == 200:
        assert step % 200 != 0

    acts, e_aff = [], []   # fp64 activated taps (NCHW) and the affine's fp32 error bound, per level
    for m, p in zip(maps, ss):
        x = m.double()
        if p is None:
            acts.append(x.permute(0, 3, 1, 2))
            e_aff.append(0.0)
            continue
        sc, sh = p[0].double()[:, None, None, :], p[1].double()[:, None, None, :]
        acts.append(torch.relu(x * sc + sh).permute(0, 3, 1, 2))
        e_aff.append(2 * U * (x.abs() * sc.abs() + sh.abs()).max().item())
    tap_max = [a.abs().max().item() for a in acts]

    for l, Hl in enumerate(sizes):
        top, down = min(l + 1, 3), max(l - 1, 0)
        out = nan((B, Hl, Hl, C), dt)
        kernels.fuse_gather(maps[l], maps[top], maps[down], ss[l], ss[top], ss[down], out=out)

        def rs(x):
            return F.interpolate(x, size=(Hl, Hl), mode='bilinear', align_corners=True)

        def e_src(i):
            return e_aff[i] + (0.0 if sizes[i] == Hl else _lerp_e32(sizes[i], tap_max[i]))
        ref = torch.cat([acts[l][:, :2 * q], rs(acts[top][:, 3 * q:]), rs(acts[down][:, 2 * q:3 * q])], 1)
        e32 = torch.cat([torch.full((2 * q,), e_aff[l], dtype=F64, device=DEV),
                         torch.full((q,), e_src(top), dtype=F64, device=DEV),
                         torch.full((q,), e_src(down), dtype=F64, device=DEV)])
        _check_rounded(out, ref.permute(0, 2, 3, 1), e32, dt, 'level %d' % l)


def _gn_bound(n, m, v, eps):
    """Relative error of gn_finalize's scale = gamma * rsqrt(var + eps) from fp32 slot sums whose addition chain is
    n long, for a group of mean m and variance v.  |s' - s| <= n u sum|y| and |ss' - ss| <= (n + 1)u ss, so the
    one-pass var' = ss/count - mean^2 is within dv = (3n + 5)u (v + m^2) (using mean|y| <= sqrt(v + m^2)); rsqrtf
    adds 2 ulp and gamma * rstd one rounding:  e_a = dv / (2(v + eps)) + 6u  <=  ((3n + 5)/2 (1 + m^2/v) + 6)u.
    The mean itself is within (n + 1)u mean|y| <= (n + 1)u sqrt(v + m^2)."""
    dv = (3 * n + 5) * U * (v + m * m)
    return dv / (2 * (v + eps)) + 6 * U, (n + 1) * U * (v + m * m).sqrt()


def _check_gn(y, stats, gamma, beta, n_chain, dt, eps=1e-5):
    """Call gn_finalize on `stats` of the 16-bit map y [B, HW, C] (64 groups of 16) and check scale / shift against
    fp64 F.group_norm's statistics of y (_gn_bound), and the GN output y * scale + shift against fp64 group_norm:
    within half a storage ulp at the output's scale, u16 (|gn| + |gamma|), so that one rounding of it lands on a
    neighbour of the exact value."""
    B, HW, C = y.shape
    groups = stats.shape[2]
    sc, sh = nan((B, C), F32), nan((B, C), F32)
    raw('g4r_gn_finalize', dt, ptr(stats), ptr(gamma), ptr(beta), ptr(sc), ptr(sh), B, C, groups, stats.shape[1],
        float(HW * (C // groups)), eps)
    yd = y.double().view(B, HW, groups, C // groups)
    m = yd.mean((1, 3))
    v = (yd - m[:, None, :, None]).pow(2).mean((1, 3))
    e_a, e_m = _gn_bound(n_chain, m, v, eps)
    rep = C // groups
    m, v, e_a, e_m = (t.repeat_interleave(rep, 1) for t in (m, v, e_a, e_m))
    gd, bd = gamma.double()[None], beta.double()[None]
    a64 = gd * (v + eps).rsqrt()
    s64 = bd - m * a64
    _check_within(sc, a64, e_a * a64.abs(), 'scale')
    _check_within(sh, s64, a64.abs() * e_m + (m * a64).abs() * (e_a + U) + U * (bd.abs() + (m * a64).abs()), 'shift')
    gn64 = F.group_norm(y.double().permute(0, 2, 1), groups, gamma.double(), beta.double(), eps).permute(0, 2, 1)
    gn = y.double() * sc.double()[:, None, :] + sh.double()[:, None, :]
    _check_within(gn, gn64, U16[dt] * (gn64.abs() + gamma.double().abs()), 'GN output')
    return sc, sh


@pytest.mark.parametrize('dt', DTS)
@pytest.mark.parametrize('Hl', [192, 96])
def test_gn_finalize_on_conv_stats_matches_fp64(Hl, dt):
    """GroupNorm statistics as the engine makes them: a 3x3 conv_nhwc (C = 1024 -> 1024, B = 2) writes fp32 partial
    (sum, sumsq) per (tile, warp) slot of its 16-bit output, 64 groups, the real slot count dense.gn_slots(H, H);
    gn_finalize combines them.  Chain (_gn_bound): each slot is 16 values per lane + 5 shuffle levels; gn_finalize
    sums ceil(slots / 32) slots per lane + 5 levels.  Reference: fp64 group_norm of the same 16-bit conv output."""
    B, C, G = 2, 1024, 64
    torch.manual_seed(Hl)
    x = torch.relu(torch.randn(B, Hl, Hl, C, device=DEV)).to(dt)
    w = (torch.randn(C, 3, 3, C, device=DEV) * (9 * C) ** -0.5).to(dt)
    slots = dense.gn_slots(Hl, Hl)
    stats = torch.zeros(B, slots, G, 2, dtype=F32, device=DEV)
    y = dense.conv_nhwc(x, w, gn_stats=stats)
    gamma = (torch.rand(C, device=DEV) + 0.5).to(dt)
    beta = (torch.randn(C, device=DEV) * 0.5).to(dt)
    sc, sh = _check_gn(y.view(B, Hl * Hl, C), stats, gamma, beta, 21 + -(-slots // 32) + 5, dt)
    again = kernels.gn_finalize(stats, gamma, beta, Hl * Hl * (C // G))
    assert torch.equal(again[0], sc) and torch.equal(again[1], sh)


@pytest.mark.parametrize('dt', DTS)
def test_gn_finalize_one_pass_variance_edges(dt):
    """Synthetic stats at the finest 336 px level (192^2 pixels, the real slot count, count 589 824 per group):
    groups with mean +-4 sigma (mean^2 / var = 16, the one-pass cancellation the bound in _gn_bound grows with), a
    constant group of 0.75 (every partial sum exact, so var is exactly 0 and rstd = rsqrtf(eps)), and a constant
    group of rd(0.1), whose one-pass var is a rounding residue clamped at >= 0 (no NaN).  The slot sums are fp64 sums
    stored to fp32 (chain 1 + ceil(slots / 32) + 5)."""
    B, Hl, C, G = 2, 192, 1024, 64
    HW = Hl * Hl
    slots = dense.gn_slots(Hl, Hl)
    torch.manual_seed(11)
    y = torch.randn(B, HW, G, 16, device=DEV)
    y[:, :, 0] = y[:, :, 0] * 0.5 + 2.0
    y[:, :, 1] = y[:, :, 1] * 0.25 - 1.0
    y[:, :, 2] = 0.75
    y[:, :, 3] = 0.1
    y[:, :, 4] = y[:, :, 4] * 2.0 + 8.0
    y = y.view(B, HW, C).to(dt)
    slot_of = torch.arange(HW, device=DEV) * slots // HW
    per = y.double().view(B, HW, G, 16)
    st = torch.zeros(B, slots, G, 2, dtype=F64, device=DEV)
    st[..., 0].index_add_(1, slot_of, per.sum(-1))
    st[..., 1].index_add_(1, slot_of, per.pow(2).sum(-1))
    stats = st.float().contiguous()
    gamma = (torch.rand(C, device=DEV) + 0.5).to(dt)
    beta = (torch.randn(C, device=DEV) * 0.5).to(dt)
    sc, sh = _check_gn(y, stats, gamma, beta, 1 + -(-slots // 32) + 5, dt)
    rs = torch.tensor(1e-5, dtype=F32).double().rsqrt().item()
    g2 = gamma[32:48].double()
    _check_within(sc[:, 32:48], (g2 * rs)[None].expand(B, 16), 6 * U * (g2 * rs).abs()[None], 'constant group scale')
    assert torch.isfinite(sc).all() and torch.isfinite(sh).all()


@pytest.mark.parametrize('dt', DTS)
def test_affine_relu_nhwc_matches_fp64(dt):
    """relu(z * scale[b, c] + shift[b, c]) on a 192^2 x 1024 map, B = 2, per-image scale / shift with both signs.
    One fmaf (within u|pre| of the fp64 pre-activation), ReLU, one rounding: between rd(relu(pre -+ u|pre|)); where
    the fp64 pre-activation is below -u|pre| the output is +0 exactly.  9.4M vectors: many passes."""
    B, Hl, C = 2, 192, 1024
    torch.manual_seed(12)
    z = torch.randn(B, Hl, Hl, C, device=DEV).to(dt)
    scale = torch.rand(B, C, device=DEV) * 2 - 0.5
    shift = torch.randn(B, C, device=DEV) * 0.5
    assert passes(B * Hl * Hl * C // 8) > 1
    out = nan((B, Hl, Hl, C), dt)
    raw('g4r_affine_relu_nhwc_bf16', dt, ptr(z), ptr(scale), ptr(shift), ptr(out), B, Hl * Hl, C)
    pre = z.double() * scale.double()[:, None, None, :] + shift.double()[:, None, None, :]
    e = U * pre.abs()
    lo, hi = torch.relu(pre - e).to(dt).double(), torch.relu(pre + e).to(dt).double()
    g = out.double()
    assert bool(((g >= lo) & (g <= hi)).all())
    neg = pre + e < 0
    assert int(neg.sum()) > 0 and bool((bits(out)[neg] == 0).all())
    assert torch.equal(bits(kernels.affine_relu_nhwc(z, scale, shift)), bits(out))


# ---------------------------------------------------------------------------------------------------------------
# Region-token head: pos_embedd MLP, split-K sum + bias + pos + cast
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dt', DTS)
@pytest.mark.parametrize('K', [1, 5, 64])
def test_pos_embed_mlp_matches_fp64(K, dt):
    """Linear(4,256) ReLU LN(256) Linear(256,1024) ReLU LN(1024) on the boxes, in fp64 with the kernel's (autocast's)
    rounding points to the storage type: the boxes, the first Linear's output, the LN(256) output (the second Linear's
    input) and the second Linear's output.  The fp32 arithmetic differs from the fp64 one by about sqrt(256)u = 16u
    relative (sums of 256 products with random signs; the LN statistics less), so a value rounds to the other
    neighbour than in the reference only that close to a rounding boundary: a fraction of about 16u / u16 <= 2^-9 of
    them, each moving one element by at most one ulp (2 u16).  Through the final LayerNorm that keeps rel-L2 <=
    sqrt(2^-8) * 2 u16 = u16 / 8.  A rounding point left out (or added) costs ~0.4 u16, the RMS of a rounding."""
    torch.manual_seed(K)

    def r(*shape, sc=1.0, off=0.0):
        return (torch.randn(*shape, device=DEV) * sc + off).to(dt)
    w0, b0, g2, be2 = r(256, 4, sc=0.5), r(256, sc=0.1), r(256, sc=0.1, off=1.0), r(256, sc=0.1)
    w3, b3, g5, be5 = r(1024, 256, sc=0.0625), r(1024, sc=0.1), r(1024, sc=0.1, off=1.0), r(1024, sc=0.1)
    boxes = torch.rand(K, 4, device=DEV)
    out = nan((K, 1024), F32)
    raw('g4r_pos_embed_mlp', dt, ptr(boxes), ptr(w0), ptr(b0), ptr(g2), ptr(be2), ptr(w3), ptr(b3), ptr(g5),
        ptr(be5), ptr(out), K, 1e-5)

    def rd(x):
        return x.to(dt).double()
    P = [t.double() for t in (w0, b0, g2, be2, w3, b3, g5, be5)]
    u1 = rd(rd(boxes) @ P[0].T + P[1])
    h1 = rd(F.layer_norm(F.relu(u1), (256,), P[2], P[3], 1e-5))
    u2 = rd(h1 @ P[4].T + P[5])
    want = F.layer_norm(F.relu(u2), (1024,), P[6], P[7], 1e-5)
    err = ((out.double() - want).norm() / want.norm()).item()
    assert err <= U16[dt] / 8, err
    assert torch.equal(kernels.pos_embed_mlp(boxes, w0, b0, g2, be2, w3, b3, g5, be5), out)


@pytest.mark.parametrize('dt', DTS)
@pytest.mark.parametrize('K', [1, 5, 64])
@pytest.mark.parametrize('splits', [1, 7, 16])
def test_add_bias_pos_cast_is_torch_restatement(splits, K, dt):
    """t = rd(rd(sum_s acc[s] + bias) + pos): the split-K slabs of flatten_linear summed in order s = 0, 1, ... in
    fp32 (the engine uses 16 splits at C R R = 200704), the bias added and the sum rounded to the storage type
    (flatten_linear's output), the fp32 pos_embedd added and rounded again (updims' input).  The same fp32 operations
    in torch: bit for bit."""
    D = 1024
    torch.manual_seed(splits * 100 + K)
    acc = torch.randn(splits, K, D, device=DEV) * 4
    bias = torch.randn(D, device=DEV).to(dt)
    pos = torch.randn(K, D, device=DEV)
    out = nan((K, D), dt)
    raw('g4r_add_bias_pos_cast', dt, ptr(acc), splits, ptr(bias), ptr(pos), ptr(out), K, D)
    a = torch.zeros(K, D, device=DEV)
    for s in range(splits):
        a = a + acc[s]
    want = ((a + bias.float()).to(dt).float() + pos).to(dt)
    assert torch.equal(bits(out), bits(want))
    assert torch.equal(bits(kernels.add_bias_pos_cast(acc, bias, pos)), bits(out))
