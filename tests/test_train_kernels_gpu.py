"""Each training-step kernel on its own, through the train_ops / splice wrappers the trainer calls, at the shapes,
strides and edges the trainer produces, against plain torch of the same operation in float64 on the device, run on
the same bf16 inputs.  Where a kernel rounds in the middle the reference rounds at the same point (straight-through:
x + (bf16(x) - x).detach()).  Every tolerance is derived from the rounding in its docstring; u = 2^-24 is the fp32
unit roundoff.  Copies and casts must be exact.

The whole-step tests (test_train_gpu.py) bound these kernels only to the error of bf16 autocast itself; a dropped
slab, a wrong tail or a swapped gradient slot fits inside those bounds and is caught here instead."""
import math

import pytest
import torch
import torch.nn.functional as F

from gpt4roi_b200 import kernels, train_ops
from gpt4roi_b200 import lib as _L

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
BF = torch.bfloat16
F64 = torch.float64
U = 2.0 ** -24
# Rounding to bf16 (8 significant bits) moves a value by at most 2^-8 of itself; over many values spread across
# binades the RMS of that relative error is 2^-8 / sqrt(3) * E[1/m^2]^0.5 (m the significand in [1, 2)) ~= 1.7e-3,
# which is what a rel-L2 of a bf16 output against an unrounded reference measures.
BF16_RMS = 1.7e-3


def rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def st(x):
    """bf16 rounding in the forward, identity in the backward."""
    return x + (x.to(BF).to(x.dtype) - x).detach()


def bits(t):
    return t.contiguous().view(torch.int16)


def _i16(patterns):
    return torch.tensor([p - (1 << 16) if p >= 1 << 15 else p for p in patterns], dtype=torch.int16, device=DEV)


def _i32(patterns):
    return torch.tensor([p - (1 << 32) if p >= 1 << 31 else p for p in patterns], dtype=torch.int32, device=DEV)


# ---------------------------------------------------------------------------------------------------------------
# colsum (every bias gradient)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('N', [8, 1024, 2056, 4096])
@pytest.mark.parametrize('M', [1, 5, 63, 64, 65, 1412, 5648])
def test_colsum_matches_fp64(M, N):
    """fp32 column sums of a bf16 matrix vs fp64.  Each column is summed in fp32 as up to 64 row-strided slabs that
    are then added in order: a recursive sum of M terms, so |err| <= M*u*sum|x| per column (exact for M = 1).
    N = 2056 leaves a partial 2048-column CTA; the strided input is x[:, :N] of a wider buffer.  Same bits twice."""
    torch.manual_seed(M * 31 + N)
    wide = torch.randn(M, N + 24, device=DEV).to(BF)
    for x in (wide[:, :N].contiguous(), wide[:, :N]):
        got = train_ops.colsum(x)
        xd = x.double()
        err = (got.double() - xd.sum(0)).abs()
        bound = M * U * xd.abs().sum(0)
        assert torch.all(err <= bound), (x.stride(), (err - bound).max().item())
        assert torch.equal(got, train_ops.colsum(x))


# ---------------------------------------------------------------------------------------------------------------
# global gradient norm, clip coefficient, AdamW with the device coefficient
# ---------------------------------------------------------------------------------------------------------------
def _sumsq_chain(t):
    """Longest chain of fp32 additions in sumsq_partial for t (all terms >= 0, so the relative error of the sum is at
    most chain * u): a 16-byte-aligned tensor is read as vectors by kSumsqSlabs x 256 threads plus a short serial
    tail in block 0; a misaligned one entirely by block 0's 256 threads.  +16 for the block reduction tree."""
    n, V = t.numel(), 16 // t.element_size()
    if t.data_ptr() % 16 == 0:
        return V * -(-n // (_L.load().g4r_sumsq_slabs() * 256 * V)) + 1 + 16
    return -(-n // 256) + 16


def _grad_list():
    """The mix the trainer feeds grad_sumsq: bf16 and fp32, sizes 1 / 7 / 8 / 100003, views at an element offset of 1
    (not 16-byte aligned: block 0's serial loop reads them), and an lm_head-sized bf16 gradient."""
    torch.manual_seed(7)
    bf_base = torch.randn(100004, device=DEV).to(BF)
    f32_base = torch.randn(1001, device=DEV)
    return [torch.randn(1, device=DEV).to(BF) * 3, torch.randn(7, device=DEV), torch.randn(8, device=DEV).to(BF),
            torch.randn(100003, device=DEV) * 0.1, bf_base[1:], f32_base[1:],
            (torch.randn(32006, 4096, device=DEV) * 2e-3).to(BF)]


def _torch_clip(ts, max_norm, pre_scale):
    """torch.nn.utils.clip_grad_norm_ in fp64 on grad * pre_scale -> (total norm, the coefficient it applied)."""
    ps = []
    for t in ts:
        p = torch.zeros(t.shape, dtype=F64, device=DEV, requires_grad=True)
        p.grad = t.double() * pre_scale
        ps.append(p)
    g0 = ps[2].grad.clone()
    norm = torch.nn.utils.clip_grad_norm_(ps, max_norm).item()
    return norm, ((ps[2].grad * g0).sum() / (g0 * g0).sum()).item()


@pytest.mark.parametrize('world', [1, 8])
@pytest.mark.parametrize('ratio', [0.25, 4.0])
def test_grad_norm_and_clip_coef_match_clip_grad_norm(ratio, world):
    """grad_sumsq + clip_coef vs clip_grad_norm_ (fp64) with max_norm = ratio * norm (clipping / no clipping) and
    pre_scale = 1/world.  Each tensor's slab row sums to its fp64 sum of squares within chain*u (_sumsq_chain); the
    total adds 7 x kSumsqSlabs partials over 256 threads (+ 30 adds), so the norm is within (max chain + 30)/2*u + 2u
    relative and the coefficient within that + 2u."""
    ts = _grad_list()
    slabs = train_ops.grad_sumsq(ts)
    for i, t in enumerate(ts):
        want = t.double().pow(2).sum().item()
        got = slabs[i].double().sum().item()
        assert abs(got - want) <= _sumsq_chain(t) * U * want, (i, got, want)
    pre = 1.0 / world
    norm_true = math.sqrt(sum(t.double().pow(2).sum().item() for t in ts)) * pre
    max_norm = ratio * norm_true
    out = train_ops.clip_coef(slabs, max_norm, pre_scale=pre)
    norm_ref, coef_ref = _torch_clip(ts, max_norm, pre)
    tol = (max(_sumsq_chain(t) for t in ts) + 30) / 2 * U + 2 * U
    assert abs(out[0].item() - norm_ref) <= tol * norm_ref, (out[0].item(), norm_ref)
    assert abs(out[1].item() - coef_ref) <= (tol + 2 * U) * coef_ref, (out[1].item(), coef_ref)
    if ratio > 1:
        assert out[1].item() == 1.0
    assert torch.equal(slabs, train_ops.grad_sumsq(ts))                    # fixed summation order


def test_clip_coef_edge_rules():
    """max_norm <= 0 means no clipping: the coefficient is exactly 1 (clip_grad_norm_ would scale by max_norm/norm,
    i.e. zero or flip the gradients); the norm is still reported.  All-zero gradients: norm 0, coefficient 1."""
    ts = _grad_list()[:6]
    slabs = train_ops.grad_sumsq(ts)
    norm_ref = math.sqrt(sum(t.double().pow(2).sum().item() for t in ts))
    for max_norm in (0.0, -1.0):
        out = train_ops.clip_coef(slabs, max_norm)
        assert out[1].item() == 1.0
        assert abs(out[0].item() - norm_ref) <= 1e-4 * norm_ref
    zeros = [torch.zeros_like(t) for t in ts]
    out = train_ops.clip_coef(train_ops.grad_sumsq(zeros), 1.0, pre_scale=0.125)
    assert out[0].item() == 0.0 and out[1].item() == 1.0


@pytest.mark.parametrize('ratio', [0.3, 3.0])
@pytest.mark.parametrize('wd', [0.0, 0.1])
@pytest.mark.parametrize('g_dtype', [BF, torch.float32])
@pytest.mark.parametrize('n', [1, 3, 5, 100003])
def test_adamw_with_device_clip_coef_matches_torch(n, g_dtype, wd, ratio):
    """The production optimizer path: clip_coef(grad_sumsq([g]), max_norm, 1/world) fed to adamw_step as scale_dev,
    vs clip_grad_norm_ + torch.optim.AdamW in fp64 at step 1000 (state['step'] = 999 with nonzero moments, so the
    bias corrections are far from 1).  n = 1, 3, 5 run the scalar tail of the last CTA.  Error budget: a handful of
    fp32 roundings (4u per moment term, 8u on p, 16u on the update), the coefficient's own error c (test above), and
    the fp32 betas: beta stored in fp32 makes 1 - beta off by up to u*beta/(1 - beta) (999u for 0.999) and
    1 - beta^step off by up to (step + 2)u*beta^step/(1 - beta^step).  m and v are checked against their terms, p
    against |p| and the size of the Adam step.  The bf16 copy p16 equals bf16(p) exactly."""
    torch.manual_seed(n + int(wd * 10) + (g_dtype == BF))
    lr, betas, eps, pre = 2e-3, (0.9, 0.999), 1e-8, 0.5
    p0 = torch.randn(n, device=DEV)
    m0 = torch.randn(n, device=DEV) * 1e-2
    v0 = torch.rand(n, device=DEV) * 1e-4 + 1e-6
    grad = (torch.randn(n, device=DEV) * 0.5).to(g_dtype)
    max_norm = ratio * grad.double().norm().item() * pre
    slabs = train_ops.grad_sumsq([grad])
    coef = train_ops.clip_coef(slabs, max_norm, pre_scale=pre)
    p, m, v = p0.clone(), m0.clone(), v0.clone()
    p16 = torch.full((n,), float('nan'), device=DEV, dtype=BF)
    train_ops.adamw_step(p, grad, m, v, p16, lr, betas, eps, wd, 1000, grad_scale=pre, scale_dev=coef[1:])

    ref = p0.double().requires_grad_()
    ref.grad = grad.double() * pre
    torch.nn.utils.clip_grad_norm_([ref], max_norm)
    g_eff = ref.grad.clone()
    opt = torch.optim.AdamW([ref], lr=lr, betas=betas, eps=eps, weight_decay=wd)
    opt.state[ref] = {'step': torch.tensor(999.0), 'exp_avg': m0.double(), 'exp_avg_sq': v0.double()}
    opt.step()
    pr = ref.detach()
    c = (_sumsq_chain(grad) + 30) * U

    def e_beta(b):
        return U * b / (1 - b)

    def e_bias(b, step=1000):
        return (step + 2) * U * b ** step / (1 - b ** step)
    e_m = 4 * U + c + e_beta(betas[0])
    e_v = 4 * U + 2 * c + e_beta(betas[1])
    e_upd = e_m + (e_v + e_bias(betas[1])) / 2 + e_bias(betas[0]) + 16 * U
    upd = (pr - p0.double() * (1 - lr * wd)).abs()
    assert torch.all((p.double() - pr).abs() <= 8 * U * pr.abs() + e_upd * upd + 1e-12)
    mr, vr = opt.state[ref]['exp_avg'], opt.state[ref]['exp_avg_sq']
    assert torch.all((m.double() - mr).abs() <= e_m * (0.9 * m0.double().abs() + 0.1 * g_eff.abs()) + 1e-30)
    assert torch.all((v.double() - vr).abs() <= e_v * (0.999 * v0.double() + 1e-3 * g_eff.pow(2)) + 1e-30)
    assert torch.equal(bits(p16), bits(p.to(BF)))


# ---------------------------------------------------------------------------------------------------------------
# pos_embedd backward
# ---------------------------------------------------------------------------------------------------------------
_POS_NAMES = ('0.weight', '0.bias', '2.weight', '2.bias', '3.weight', '3.bias', '5.weight', '5.bias')


@pytest.mark.parametrize('K', [1, 3, 64])
def test_pos_embed_mlp_bwd_matches_fp64_autograd(K):
    """All 8 pos_embedd gradients vs fp64 autograd of the forward Linear(4,256) ReLU LN(256) Linear(256,1024) ReLU
    LN(1024) with the kernel's rounding points (boxes, both Linear outputs, the second Linear's input) bf16 in the
    forward and straight-through in the backward, as the kernel treats them.  Residual error: fp32 sums of <= 1024
    terms (<= 6e-5) and the few values whose fp32 and fp64 pre-images round to neighbouring bf16 values (one bf16
    ulp, 2^-8, on ~2^-15 of the values): rel-L2 <= 2e-3 per tensor."""
    torch.manual_seed(K)

    def r(*shape, sc=1.0, off=0.0):
        return (torch.randn(*shape, device=DEV) * sc + off).to(BF)
    params = (r(256, 4, sc=0.5), r(256, sc=0.1), r(256, sc=0.1, off=1.0), r(256, sc=0.1),
              r(1024, 256, sc=0.0625), r(1024, sc=0.1), r(1024, sc=0.1, off=1.0), r(1024, sc=0.1))
    boxes = torch.rand(K, 4, device=DEV)
    dout = torch.randn(K, 1024, device=DEV).to(BF)
    got = train_ops.pos_embed_mlp_bwd(boxes, params, dout)

    P = [t.double().requires_grad_() for t in params]
    w0, b0, g2, be2, w3, b3, g5, be5 = P
    bx = boxes.to(BF).double()
    u1 = st(bx @ w0.T + b0)
    h1 = st(F.layer_norm(F.relu(u1), (256,), g2, be2, 1e-5))
    u2 = st(h1 @ w3.T + b3)
    out = F.layer_norm(F.relu(u2), (1024,), g5, be5, 1e-5)
    # the reference forward is the forward kernel's arithmetic
    assert rel(kernels.pos_embed_mlp(boxes, *params), out) < 1e-3
    (out * dout.double()).sum().backward()
    errs = {nm: rel(got[nm], t.grad) for nm, t in zip(_POS_NAMES, P)}
    assert all(e <= 2e-3 for e in errs.values()), errs


# ---------------------------------------------------------------------------------------------------------------
# exact elementwise kernels
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('shape', [(1, 8), (37, 4096)])
def test_relu_bwd_is_exact(shape):
    """out = where(y > 0, dy, 0) bit for bit, with y = +0, -0, bf16 subnormals of both signs and dy = -0 present."""
    torch.manual_seed(shape[0])
    y = torch.randn(shape, device=DEV).to(BF)
    dy = torch.randn(shape, device=DEV).to(BF)
    flat = y.view(-1)
    flat.view(torch.int16)[:8] = _i16([0x0000, 0x8000, 0x0001, 0x8001, 0x007F, 0x3F80, 0xBF80, 0x0080])
    dy.view(-1)[1] = -0.0
    got = train_ops.relu_bwd(dy, y)
    want = torch.where(y > 0, dy, torch.zeros_like(dy))
    assert torch.equal(bits(got), bits(want))


@pytest.mark.parametrize('n,H,W,C', [(1, 5, 7, 256), (3, 12, 9, 1024)])
def test_pad_nhwc_is_exact(n, H, W, C):
    """Padded conv-dW operand: W + 3 zero guard rows, then each image zero-ringed (F.pad by one pixel), then the
    guard again; bit for bit, over a buffer that held NaNs just before."""
    torch.manual_seed(H * W)
    x = torch.randn(n, H, W, C, device=DEV).to(BF)
    guard = W + 3
    rows = 2 * guard + n * (H + 2) * (W + 2)
    del_me = torch.full((rows, C), float('nan'), device=DEV, dtype=BF)   # leave NaNs in the allocator's block
    del del_me
    out, g = train_ops.pad_nhwc(x)
    assert g == guard
    z = torch.zeros(guard, C, device=DEV, dtype=BF)
    want = torch.cat([z, F.pad(x, (0, 0, 1, 1, 1, 1)).reshape(-1, C), z])
    assert torch.equal(bits(out), bits(want))


def test_cast_f32_bf16_matches_torch_bit_for_bit():
    """Round to nearest even like torch's .to(bfloat16) (computed on the host): ties both ways, fp32 subnormals
    (including the largest, which rounds up to the smallest normal), +-0, +-inf, values above the largest finite
    bf16 (to it or to inf), and NaN in -> NaN out (payload free)."""
    torch.manual_seed(3)
    N, D = 33, 520
    x = torch.randn(N, D, device=DEV) * 100
    pat = [0x3F808000, 0x3F818000, 0xBF808000, 0xBF818000, 0x3F808001, 0x3F807FFF,          # ties / just off ties
           0x00000001, 0x00008000, 0x00018000, 0x007FFFFF, 0x80000001, 0x807FFFFF,          # subnormals
           0x00000000, 0x80000000, 0x7F800000, 0xFF800000,                                  # zeros, infinities
           0x7F7F7FFF, 0x7F7F8000, 0x7F7FFFFF, 0xFF7F8000, 0x7F7F0000,                      # near / above bf16 max
           0x7FC00000, 0x7F800001, 0xFFC00001]                                              # NaNs
    x.view(-1).view(torch.int32)[:len(pat)] = _i32(pat)
    x.view(-1).view(torch.int32)[D + 5:D + 5 + len(pat)] = _i32(pat)           # again, inside a row and a vector
    got = train_ops.cast_f32_bf16(x)
    nan = torch.isnan(x)
    assert torch.isnan(got[nan]).all()
    want = x.cpu().to(BF).to(DEV)
    assert torch.equal(bits(got)[~nan], bits(want)[~nan])


# ---------------------------------------------------------------------------------------------------------------
# splice backward + embed_tokens gradient
# ---------------------------------------------------------------------------------------------------------------
TAG_IMAGE, TAG_REGION = 0x40000000, 0x20000000


def _splice_batch():
    """4 samples, LLaVA vocabulary (32006 rows, special tokens 32001 patch / 32002 bbox / 32004 start / 32005 end):
    0 text-only, with 300 pads, a <bbox>, 32003 and <im_end> (all embedding rows) and one box it does not use;
    1 image, zero boxes, 240 pads;  2 image + 3 boxes + 32003;  3 image + 2 boxes, id 13 repeated 300 times."""
    V, P, B, L = 32006, 16, 4, 640
    PATCH, BBOX, START, END = 32001, 32002, 32004, 32005
    g = torch.Generator().manual_seed(0)
    ids = torch.randint(1, 32000, (B, L), generator=g)
    ids[0, :300] = 0
    ids[0, 400:403] = torch.tensor([BBOX, 32003, END])

    def image(b, s, boxes_at):
        ids[b, s] = START
        ids[b, s + 1:s + 1 + P] = PATCH
        ids[b, s + 1 + P] = END
        for t in boxes_at:
            ids[b, t] = BBOX
    image(1, 1, [])
    ids[1, 400:] = 0
    image(2, 10, [100, 200, 300])
    ids[2, 500] = 32003
    image(3, 0, [50, 600])
    ids[3, 100:400] = 13
    counts = [1, 0, 3, 2]
    offs = [0, 1, 1, 4, 6]
    codes = ids.clone()
    for b in range(B):                                   # the plan, restated from spi_llava.py's splice rules
        row = ids[b].tolist()
        if PATCH not in row:
            continue
        s = row.index(START)
        codes[b, s + 1:s + 1 + P] = TAG_IMAGE | torch.arange(P)
        k = offs[b]
        for t, v in enumerate(row):
            if v == BBOX:
                codes[b, t] = TAG_REGION | k
                k += 1
    return ids, codes, counts, (V, P, PATCH, BBOX, START, END)


def test_splice_backward_matches_index_reference():
    """d_image / d_region are row copies: exact, and rows no position names (sample 0's image rows, its unused box)
    stay zero.  d_embed = fp64 segment sums of the d_out rows of each token id: an fp32 sum of n rows is within
    n*u*sum|terms| of it; ids that never occur have exactly zero rows.  D = 4104 runs a partial last 2048-column
    pass.  Same bits twice; want_embed_grad=False gives the same row moves and no d_embed."""
    from gpt4roi_b200.splice import splice_backward, splice_region_tokens
    ids, codes, counts, (V, P, PATCH, BBOX, START, END) = _splice_batch()
    B, L = ids.shape
    D = 4104
    torch.manual_seed(1)
    emb = torch.randn(V, D, device=DEV).to(BF)
    img = torch.randn(B, P, D, device=DEV).to(BF)
    regions = [torch.randn(c, D, device=DEV).to(BF) if c else None for c in counts]
    K = sum(counts)
    _, plan = splice_region_tokens(ids.to(DEV), emb, img, regions, P, PATCH, START, END, BBOX, return_plan=True)
    assert torch.equal(plan.cpu().long(), codes)
    d_out = torch.randn(B, L, D, device=DEV).to(BF)
    d_image, d_region, d_embed = splice_backward(plan, d_out, P, K, V)

    c = codes.reshape(-1).to(DEV)
    rows = d_out.reshape(-1, D)
    is_img, is_reg = (c & TAG_IMAGE) != 0, (c & TAG_REGION) != 0
    is_emb = ~(is_img | is_reg)
    want_img = torch.zeros(B, P, D, device=DEV, dtype=BF)
    b_of = torch.arange(B * L, device=DEV) // L
    want_img[b_of[is_img], c[is_img] & ~TAG_IMAGE] = rows[is_img]
    want_reg = torch.zeros(K, D, device=DEV, dtype=BF)
    want_reg[c[is_reg] & ~TAG_REGION] = rows[is_reg]
    assert torch.equal(bits(d_image), bits(want_img))
    assert torch.equal(bits(d_region), bits(want_reg))
    assert torch.all(d_region[0] == 0) and torch.all(d_image[0] == 0)

    e = c[is_emb]
    assert int(e.max()) == V - 1 and int(e.min()) == 0
    ref = torch.zeros(V, D, dtype=F64, device=DEV).index_add_(0, e, rows[is_emb].double())
    absum = torch.zeros(V, D, dtype=F64, device=DEV).index_add_(0, e, rows[is_emb].double().abs())
    n = torch.bincount(e, minlength=V).double()
    assert int(n[0]) == 540 and int(n[13]) >= 300
    err = (d_embed.double() - ref).abs()
    assert torch.all(err <= n[:, None] * U * absum), (err - n[:, None] * U * absum).max().item()
    assert torch.all(d_embed[n == 0] == 0)
    again = splice_backward(plan, d_out, P, K, V)
    assert torch.equal(d_embed, again[2]) and torch.equal(d_image, again[0]) and torch.equal(d_region, again[1])
    di, dr, de = splice_backward(plan, d_out, P, K, V, want_embed_grad=False)
    assert de is None and torch.equal(di, d_image) and torch.equal(dr, d_region)


# ---------------------------------------------------------------------------------------------------------------
# cross entropy on the trainer's padded logits layout
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('M', [1, 255, 257, 1412])
def test_cross_entropy_on_padded_logits_matches_fp64(M):
    """Logits as the trainer allocates them: empty((M, 32064))[:, :32006], so the 16-byte vector loop covers 32000
    columns and the scalar loop the last 6.  Rows: plain, peaked (one entry 40 above the rest, often the target),
    and bf16 values near +3e4 and -3e4; targets include 0, V-1 and -100; grad_scale 0.25.
    loss: each row's lse = max + log(sum of 32006 exps) carries <= 2u|lse| + 1e-5 (fp32 sum over 125-term chains,
    __expf / logf), the mean adds (M/256 + 20)u relative.  dlogits: p = exp(x - lse) with relative error
    e = 4u|lse| + 2e-5, then (p - onehot) * k rounded to bf16 (8 significant bits: within 2^-8 relative):
    |err| <= (2^-8 + 2e) |ref| + 2e k.  Ignored rows are
    exactly 0; want_grad=False returns the same loss bits."""
    V, LD = 32006, 32064
    torch.manual_seed(M)
    vals = torch.randn(M, V, device=DEV) * 2
    r = torch.arange(M, device=DEV)
    peak = torch.randint(0, V, (M,), device=DEV)
    peak[1 % M] = V - 1
    peaked = (r % 5 == 1)
    vals[r[peaked], peak[peaked]] += 40
    big = r % 5 == 2
    vals[big] = 3e4 + torch.randn(int(big.sum()), V, device=DEV) * 400
    neg = r % 5 == 3
    vals[neg] = -3e4 + torch.randn(int(neg.sum()), V, device=DEV) * 400
    logits = torch.empty((M, LD), device=DEV, dtype=BF)[:, :V]
    logits.copy_(vals.to(BF))
    tg = torch.randint(0, V, (M,), device=DEV)
    tg[peaked & (r % 10 == 1)] = peak[peaked & (r % 10 == 1)]
    tg[torch.rand(M, device=DEV) < 0.2] = -100
    tg[0] = V - 1 if M == 1 else 0
    if M > 2:
        tg[1], tg[2] = V - 1, -100
    k_scale = 0.25
    loss, cnt, dl = train_ops.cross_entropy(logits, tg, grad_scale=k_scale)
    assert dl.stride(0) == LD

    lf = logits.double().requires_grad_()
    want = F.cross_entropy(lf, tg, ignore_index=-100)
    (want * k_scale).backward()
    valid = tg >= 0
    nval = int(valid.sum())
    lse = torch.logsumexp(lf.detach(), -1)
    assert int(cnt.item()) == nval
    row_loss = (lse - lf.detach().gather(1, tg.clamp_min(0)[:, None])[:, 0])[valid]
    tol = (1e-5 + 2 * U * lse[valid].abs().max().item() + 2 * U * row_loss.abs().max().item()
           + (M / 256 + 20) * U * abs(want.item()))
    assert abs(loss.item() - want.item()) <= tol, (loss.item(), want.item())
    k = k_scale / nval
    e = (4 * U * lse.abs() + 2e-5)[:, None]
    ref = lf.grad
    err = (dl.double() - ref).abs()
    bound = (2.0 ** -8 + 2 * e) * ref.abs() + 2 * e * k + 1e-37
    worst = int(torch.argmax(err - bound))
    wr, wc = divmod(worst, V)
    assert torch.all(err <= bound), ('row', wr, 'col', wc, 'target', int(tg[wr]), 'got', dl[wr, wc].item(),
                                     'want', ref[wr, wc].item(), 'k', k)
    assert torch.all(dl[~valid] == 0)
    loss2, cnt2, dl2 = train_ops.cross_entropy(logits, tg, grad_scale=k_scale, want_grad=False)
    assert dl2 is None and torch.equal(loss, loss2) and torch.equal(cnt, cnt2)


# ---------------------------------------------------------------------------------------------------------------
# RMSNorm backward: the 8192-wide variant and strided gradients
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('M,D', [(1, 8192), (37, 8192), (129, 5120), (1, 4096)])
def test_rmsnorm_bwd_wide_rows_and_strided_grads(M, D):
    """LlamaRMSNorm backward vs fp64 autograd of w * bf16(x * rsqrt(mean(x^2) + eps)) (straight-through), dy and dres
    rows strided wider than D.  D = 8192 and 5120 take the 4-vectors-per-thread variant (5120 leaves part of it
    idle).  dx is rounded to bf16 (BF16_RMS) after fp32 row reductions over D (<= 5e-4): rel-L2 <= 2.5e-3.  dw is an
    fp32 sum of M
    products with bf16(x_hat) (a few x_hat round to the neighbouring bf16 in fp32): rel-L2 <= 5e-4."""
    torch.manual_seed(M + D)
    x = (torch.randn(M, D, device=DEV) * 2).to(BF)
    w = (torch.rand(D, device=DEV) + 0.5).to(BF)
    dy = torch.empty(M, D + 64, device=DEV, dtype=BF)[:, :D]
    dy.copy_(torch.randn(M, D, device=DEV))
    dres = torch.empty(M, D + 128, device=DEV, dtype=BF)[:, :D]
    dres.copy_(torch.randn(M, D, device=DEV))
    xd, wd = x.double().requires_grad_(), w.double().requires_grad_()
    y = wd * st(xd * torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + 1e-6))
    (y * dy.double()).sum().backward()
    for r in (None, dres):
        dx, dw = train_ops.rmsnorm_bwd(x, w, dy, 1e-6, dres=r)
        want = xd.grad + (r.double() if r is not None else 0)
        assert rel(dx, want) <= 2.5e-3
        assert rel(dw, wd.grad) <= 5e-4


# ---------------------------------------------------------------------------------------------------------------
# GroupNorm + ReLU backward at the fuse-stack shapes
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('B,H', [(2, 6), (3, 16), (3, 32)])
def test_gn_relu_bwd_trainer_shapes(B, H):
    """GroupNorm(64) + ReLU backward on a conv output with the forward's own statistics, C = 1024, vs fp64 autograd of
    group_norm(z) masked where the forward's ReLU was off (z*scale + shift <= 0 with the fp32 scale / shift the
    forward applied; the fp64 value has the sign of the kernel's single-rounding fma).  6x6 gives one slab per pixel.
    Channel 5 is dead on the whole map: its dgamma / dbeta are exactly 0.  Residual error: the forward's fp32
    statistics (E[z^2] - mean^2 over <= 16384 values) and fp32 sums: dz (bf16, BF16_RMS) rel-L2 <= 3e-3, dgamma / dbeta
    (fp32) <= 5e-4.  accumulate=True adds the same bits again (exactly twice the value)."""
    from gpt4roi_b200 import dense
    torch.manual_seed(B * H)
    C, G, dead = 1024, 64, 5
    x = (torch.randn(B, H, H, C, device=DEV) * 0.5).to(BF)
    w = (torch.randn(C, 3, 3, C, device=DEV) * 0.02).to(BF)
    gamma = (torch.rand(C, device=DEV) + 0.5).to(BF)
    beta = (torch.randn(C, device=DEV) * 0.2).to(BF)
    gamma[dead], beta[dead] = 0.25, -64.0
    stats = torch.zeros((B, dense.gn_slots(H, H), G, 2), dtype=torch.float32, device=DEV)
    z = dense.conv_nhwc(x, w, gn_stats=stats)
    count = H * H * (C // G)
    scale, shift = kernels.gn_finalize(stats, gamma, beta, count=count)
    on = (z.double() * scale.double()[:, None, None, :] + shift.double()[:, None, None, :]) > 0
    assert not on[..., dead].any()
    for dt in (torch.float32, BF):
        dA = torch.randn(B, H, H, C, device=DEV).to(dt)
        zd = z.double().permute(0, 3, 1, 2).requires_grad_()
        gd, bd = gamma.double().requires_grad_(), beta.double().requires_grad_()
        a = F.group_norm(zd, G, gd, bd, 1e-5) * on.permute(0, 3, 1, 2)
        (a * dA.double().permute(0, 3, 1, 2)).sum().backward()
        dg = torch.full((C,), float('nan'), device=DEV)
        db = torch.full((C,), float('nan'), device=DEV)
        dz = train_ops.gn_relu_bwd(z, dA, scale, shift, stats, count, gamma, dg, db, accumulate=False)
        assert rel(dz, zd.grad.permute(0, 2, 3, 1)) <= 3e-3
        assert rel(dg, gd.grad) <= 5e-4 and rel(db, bd.grad) <= 5e-4
        assert dg[dead].item() == 0.0 and db[dead].item() == 0.0
        dg2, db2 = dg.clone(), db.clone()
        train_ops.gn_relu_bwd(z, dA, scale, shift, stats, count, gamma, dg2, db2, accumulate=True)
        assert torch.equal(dg2, 2 * dg) and torch.equal(db2, 2 * db)


# ---------------------------------------------------------------------------------------------------------------
# attention forward (lse) + backward
# ---------------------------------------------------------------------------------------------------------------
def _attn_ref(qkv, out, dout, B, L, H, D, scale, rounded=True):
    """fp64 attention backward as the kernel defines it: delta = rowsum(dO * O) from the O it is given, P from the
    exact lse; with `rounded`, P is rounded to bf16 before P^T dO and dS before dS K / dS^T Q, as the kernel does.
    -> (lse [B,H,L], dqkv [B*L, 3*H*D], floor [B*L, 3*H*D]).  floor bounds what fp32 cancellation in dP - delta
    (two sums of D exact bf16 products, each within (D + 2)u * sum|terms|) adds to dQ and dK: it is what is left
    where dS itself cancels to ~0 (L = 1: a single key, dS = 0 exactly)."""
    hid = H * D

    def heads(t):
        return t.double().reshape(B, L, H, D).permute(0, 2, 1, 3)
    q, k, v = (heads(t) for t in qkv.split(hid, 1))
    o, do = heads(out), heads(dout)
    s = (q @ k.transpose(-1, -2)) * scale
    s = s.masked_fill(torch.ones(L, L, device=qkv.device, dtype=torch.bool).triu(1), float('-inf'))
    lse = torch.logsumexp(s, -1)
    p = torch.exp(s - lse[..., None])
    rnd = (lambda t: t.to(BF).double()) if rounded else (lambda t: t)
    dv = rnd(p).transpose(-1, -2) @ do
    ds = p * (do @ v.transpose(-1, -2) - (do * o).sum(-1, keepdim=True))
    dq = rnd(ds) @ k * scale
    dk = rnd(ds).transpose(-1, -2) @ q * scale
    e_ds = p * (D + 2) * U * (do.abs() @ v.abs().transpose(-1, -2) + (do * o).abs().sum(-1, keepdim=True))
    floor = (e_ds @ k.abs() * scale, e_ds.transpose(-1, -2) @ q.abs() * scale, torch.zeros_like(dv))

    def flat(ts):
        return torch.cat([t.permute(0, 2, 1, 3).reshape(B * L, hid) for t in ts], 1)
    return lse, flat((dq, dk, dv)), flat(floor)


def _attn_inputs(B, L, H, D, peaked):
    hid = H * D
    qkv = torch.randn(B * L, 3 * hid, device=DEV)
    if peaked:
        # scores spread x9, and a sink: key 0 of every sample lies along a direction u that every query shares
        qkv *= 3
        u = torch.randint(0, 2, (H, D), device=DEV).float() * 2 - 1
        qkv[:, :hid] += u.reshape(1, hid)
        qkv.view(B, L, 3 * hid)[:, 0, hid:2 * hid] = 4 * u.reshape(1, hid)
    return qkv.to(BF), torch.randn(B * L, hid, device=DEV).to(BF)


@pytest.mark.parametrize('peaked', [False, True])
@pytest.mark.parametrize('impl', ['tc', 'mma'])
@pytest.mark.parametrize('D', [64, 128])
@pytest.mark.parametrize('L', [1, 17, 63, 65, 128, 129])
def test_attention_lse_and_bwd_at_tile_edges(monkeypatch, L, D, impl, peaked):
    """Causal attention, B = 3, H = 2, L across the 64-row tile edges, both training forwards (wgmma 'tc' and
    mma.sync 'mma').  lse vs fp64 logsumexp: each score is an fp32 sum of D exact bf16 products (<= D*u*A with
    A = scale*sum|q_d k_d|), plus the online rescaling over <= L keys and the fp32 exp2 / log: |err| <=
    (D + 8)u*max A + (L + 32)u + 2u|lse|.  dQ, dK, dV vs the fp64 backward with the kernel's rounding points
    (_attn_ref; it equals fp64 autograd when nothing is rounded, checked here): bf16 outputs (BF16_RMS), fp32 sums over
    <= 129 keys / 128 dims, the lse error above and P / dS values that round to a neighbouring bf16: error L2 norm
    <= 4e-3 of the reference's plus the norm of _attn_ref's cancellation floor.  Peaked scores (a sink key dominating
    every row) make delta = rowsum(dO*O) cancel against dP; the reference takes delta from the same bf16 O, as the
    kernel does.  Same bits twice."""
    monkeypatch.setattr(kernels, 'ATTN_IMPL', impl)
    torch.manual_seed(L * 7 + D + peaked)
    B, H = 3, 2
    hid = H * D
    scale = D ** -0.5
    qkv, dout = _attn_inputs(B, L, H, D, peaked)
    out, lse = train_ops.attention_fwd_lse(qkv, B, L, H, D, True, scale)
    want_lse, want, floor = _attn_ref(qkv, out, dout, B, L, H, D, scale)

    q, k = (t.double().abs().reshape(B, L, H, D).permute(0, 2, 1, 3) for t in qkv[:, :2 * hid].split(hid, 1))
    A = ((q @ k.transpose(-1, -2)) * scale).tril().amax(-1)
    tol = (D + 8) * U * A + (L + 32) * U + 2 * U * want_lse.abs()
    assert torch.all((lse.double() - want_lse).abs() <= tol), ((lse.double() - want_lse).abs() - tol).max().item()

    dqkv = train_ops.attention_bwd(qkv, out, dout, lse, B, L, H, D, True, scale)
    for i, nm in enumerate('qkv'):
        sl = slice(i * hid, (i + 1) * hid)
        err = (dqkv[:, sl].double() - want[:, sl]).norm().item()
        assert err <= 4e-3 * want[:, sl].norm().item() + floor[:, sl].norm().item(), (nm, err, want[:, sl].norm().item())
    out2, lse2 = train_ops.attention_fwd_lse(qkv, B, L, H, D, True, scale)
    assert torch.equal(out, out2) and torch.equal(lse, lse2)
    assert torch.equal(dqkv, train_ops.attention_bwd(qkv, out, dout, lse, B, L, H, D, True, scale))

    # the reference, unrounded and with its own exact O, is fp64 autograd of softmax(QK^T*scale + causal) V
    qf = qkv.double().requires_grad_()
    qq, kk, vv = (t.reshape(B, L, H, D).permute(0, 2, 1, 3) for t in qf.split(hid, 1))
    s = (qq @ kk.transpose(-1, -2) * scale).masked_fill(
        torch.ones(L, L, device=DEV, dtype=torch.bool).triu(1), float('-inf'))
    o = (torch.softmax(s, -1) @ vv).permute(0, 2, 1, 3).reshape(B * L, hid)
    (o * dout.double()).sum().backward()
    _, exact, _ = _attn_ref(qkv, o.detach(), dout, B, L, H, D, scale, rounded=False)
    assert rel(exact, qf.grad) < 1e-10
