"""GPU numerics tests for the wgmma GEMM / implicit-GEMM conv (floating point: tolerance
tests against a plain PyTorch fp32 reference of the same op on the same bf16 inputs)."""
import pytest
import torch
import torch.nn.functional as F

from gpt4roi_b200 import dense

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _close(got, want, rtol=1.6e-2, atol=None):
    want = want.float()
    got = got.float()
    atol = atol if atol is not None else 1e-2 * want.abs().max().item()
    torch.testing.assert_close(got, want, rtol=rtol, atol=atol)
    # bf16 output of an fp32 accumulation: mean error must be far below one bf16 ulp
    rel = (got - want).abs().mean() / want.abs().mean().clamp_min(1e-6)
    assert rel < 4e-3, rel


@pytest.mark.parametrize('M,N,K', [(128, 128, 64), (128, 256, 128), (256, 512, 4096), (200, 384, 320),
                                   (64, 1024, 1024), (5648, 4096, 4096), (706, 32006, 4096), (577, 3072, 1024),
                                   (100, 72, 136)])
def test_gemm_plain(M, N, K):
    torch.manual_seed(M + N + K)
    a = (torch.randn(M, K, device=DEV) * 0.5).bfloat16()
    b = (torch.randn(N, K, device=DEV) * 0.5).bfloat16()
    got = dense.linear(a, b)
    want = a.float() @ b.float().t()
    _close(got, want)


def test_gemm_epilogues():
    torch.manual_seed(0)
    M, N, K = 300, 640, 512
    a = (torch.randn(M, K, device=DEV) * 0.3).bfloat16()
    b = (torch.randn(N, K, device=DEV) * 0.3).bfloat16()
    bias = torch.randn(N, device=DEV).bfloat16()
    res = torch.randn(M, N, device=DEV).bfloat16()
    base = a.float() @ b.float().t()
    _close(dense.linear(a, b, bias), base + bias.float())
    _close(dense.linear(a, b, bias.float()), base + bias.float())
    _close(dense.linear(a, b, bias, act='relu'), torch.relu(base + bias.float()))
    z = base + bias.float()
    _close(dense.linear(a, b, bias, act='quick_gelu'), z * torch.sigmoid(1.702 * z))
    _close(dense.linear(a, b, bias, residual=res), base + bias.float() + res.float())
    _close(dense.linear(a, b, out_dtype=torch.float32), base, rtol=1e-4, atol=1e-3)
    # SwiGLU with interleaved gate/up rows
    g, u = base[:, 0::2], base[:, 1::2]
    _close(dense.linear(a, b, act='swiglu'), F.silu(g) * u)
    # deterministic split-K: per-split fp32 slabs, summed by the caller
    slabs = dense.linear(a, b, out_dtype=torch.float32, k_splits=4)
    assert slabs.shape == (4, M, N)
    _close(slabs.sum(0), base, rtol=1e-4, atol=1e-3)
    assert torch.equal(slabs, dense.linear(a, b, out_dtype=torch.float32, k_splits=4))  # reproducible


def test_gemm_strided_rows_and_3d_input():
    torch.manual_seed(1)
    x = (torch.randn(2, 50, 256, device=DEV)).bfloat16()
    w = (torch.randn(384, 256, device=DEV) * 0.1).bfloat16()
    got = dense.linear(x, w)
    assert got.shape == (2, 50, 384)
    _close(got, x.float() @ w.float().t())
    big = torch.zeros(100, 512, device=DEV, dtype=torch.bfloat16)
    dense.linear(x.reshape(100, 256), w, out=big[:, :384])  # padded row stride (lm_head style)
    _close(big[:, :384], (x.float() @ w.float().t()).reshape(100, 384))


@pytest.mark.parametrize('H,W,Cin,Cout,k', [(16, 16, 64, 128, 3), (24, 24, 128, 256, 3), (48, 48, 64, 64, 3),
                                            (14, 14, 128, 128, 3), (32, 32, 1088, 1024, 1), (96, 96, 1024, 1024, 3)])
def test_conv_nhwc(H, W, Cin, Cout, k):
    torch.manual_seed(H + Cin)
    n = 2
    x = (torch.randn(n, H, W, Cin, device=DEV) * 0.5).bfloat16()
    w = (torch.randn(Cout, Cin, k, k, device=DEV) * (1.0 / (Cin * k * k) ** 0.5)).bfloat16()
    bias = torch.randn(Cout, device=DEV).bfloat16()
    stats = torch.zeros(n, dense.gn_slots(H, W), Cout // 16, 2, device=DEV)
    got = dense.conv_nhwc(x, w.permute(0, 2, 3, 1).contiguous(), bias, act='relu', gn_stats=stats)
    want = torch.relu(F.conv2d(x.permute(0, 3, 1, 2).float(), w.float(), bias.float(), padding=k // 2))
    want = want.permute(0, 2, 3, 1)
    _close(got, want)
    # fused GroupNorm statistics of the bf16 output
    g = got.float().reshape(n, H * W, Cout // 16, 16)
    torch.testing.assert_close(stats.sum(1)[..., 0], g.sum((1, 3)), rtol=1e-3, atol=1e-1)
    torch.testing.assert_close(stats.sum(1)[..., 1], (g * g).sum((1, 3)), rtol=1e-3, atol=1e-1)
    stats2 = torch.zeros_like(stats)
    dense.conv_nhwc(x, w.permute(0, 2, 3, 1).contiguous(), bias, act='relu', gn_stats=stats2)
    assert torch.equal(stats, stats2)  # plain stores into fixed slots: bitwise reproducible


def test_qkv_rope_fused_equals_unfused():
    """RoPE fused into the QKV GEMM epilogue == GEMM followed by the stand-alone rope kernel, bitwise."""
    from gpt4roi_b200 import kernels
    torch.manual_seed(3)
    B, L, H, D = 2, 77, 4, 128
    hid = H * D
    x = (torch.randn(B * L, hid, device=DEV) * 0.5).bfloat16()
    w = (torch.randn(3 * hid, hid, device=DEV) * 0.05).bfloat16()
    inv = 1.0 / (10000.0 ** (torch.arange(0, D, 2).float() / D))
    emb = torch.cat([torch.arange(L).float()[:, None] * inv[None]] * 2, -1)
    cos, sin = emb.cos().to(DEV, torch.bfloat16).contiguous(), emb.sin().to(DEV, torch.bfloat16).contiguous()
    fused = dense.qkv_rope(x, w, cos, sin, L, 2 * hid)
    ref = dense.linear(x, w)
    kernels.rope_inplace(ref, cos, sin, L, 2 * H, D)
    assert torch.equal(fused, ref)


# ---- M <= 16 weight-streaming path (gemm_skinny.cu: the decode step) ---------------------------------

@pytest.mark.parametrize('M', [1, 3, 8, 9, 16])
@pytest.mark.parametrize('N,K', [(4096, 4096), (4096, 11008), (32006, 4096), (200, 96), (16, 32)])
def test_skinny_gemm_plain_matches_fp32_and_tile_path(M, N, K):
    torch.manual_seed(M * 7 + N + K)
    a = (torch.randn(M, K, device=DEV) * 0.5).bfloat16()
    b = (torch.randn(N, K, device=DEV) * 0.5).bfloat16()
    got = dense.linear(a, b)
    _close(got, a.float() @ b.float().t())
    # against the 128-row wgmma tile kernel on a padded copy (M=17 rows disables the skinny route)
    a17 = torch.cat([a, torch.zeros(17 - M, K, device=DEV, dtype=torch.bfloat16)])
    tile = dense.linear(a17, b)[:M]
    assert (got.float() - tile.float()).abs().max() <= 2e-2 * tile.float().abs().max()
    assert torch.equal(got, dense.linear(a, b))  # reproducible (fixed-order k-slice reduction)


def test_skinny_gemm_epilogues():
    torch.manual_seed(1)
    M, N, K = 5, 1312, 640
    a = (torch.randn(M, K, device=DEV) * 0.3).bfloat16()
    b = (torch.randn(N, K, device=DEV) * 0.3).bfloat16()
    bias = torch.randn(N, device=DEV).bfloat16()
    res = torch.randn(M, N, device=DEV).bfloat16()
    base = a.float() @ b.float().t()
    z = base + bias.float()
    _close(dense.linear(a, b, bias), z)
    _close(dense.linear(a, b, bias.float()), z)
    _close(dense.linear(a, b, bias, act='relu'), torch.relu(z))
    _close(dense.linear(a, b, bias, act='quick_gelu'), z * torch.sigmoid(1.702 * z))
    _close(dense.linear(a, b, bias, residual=res), z + res.float())
    _close(dense.linear(a, b, act='swiglu'), F.silu(base[:, 0::2]) * base[:, 1::2])
    # wide-N variant (32-row tiles) with SwiGLU, as the LLaMA gate/up projection at batch 8
    M, N, K = 8, 22016, 4096
    a = (torch.randn(M, K, device=DEV) * 0.3).bfloat16()
    b = (torch.randn(N, K, device=DEV) * 0.05).bfloat16()
    base = a.float() @ b.float().t()
    _close(dense.linear(a, b, act='swiglu'), F.silu(base[:, 0::2]) * base[:, 1::2])
    # strided activation rows (lda > K); fp32 output falls through to the tile kernel and stays correct
    big = (torch.randn(M, 2 * K, device=DEV) * 0.3).bfloat16()
    _close(dense.linear(big[:, :K], b), big[:, :K].float() @ b.float().t())
    _close(dense.linear(a, b, out_dtype=torch.float32), base, rtol=1e-4, atol=1e-3)


@pytest.mark.parametrize('B,L', [(1, 1), (8, 1), (2, 5), (16, 1)])
def test_skinny_qkv_rope_equals_unfused(B, L):
    """Fused-RoPE skinny QKV GEMM (host pos0 and device-side position) == plain GEMM + rope kernel, bitwise."""
    from gpt4roi_b200 import kernels
    torch.manual_seed(5 + B)
    H, D, pos0, Lmax = 4, 128, 37, 64
    hid = H * D
    x = (torch.randn(B * L, hid, device=DEV) * 0.5).bfloat16()
    w = (torch.randn(3 * hid, hid, device=DEV) * 0.05).bfloat16()
    inv = 1.0 / (10000.0 ** (torch.arange(0, D, 2).float() / D))
    emb = torch.cat([torch.arange(Lmax).float()[:, None] * inv[None]] * 2, -1)
    cos, sin = emb.cos().to(DEV, torch.bfloat16).contiguous(), emb.sin().to(DEV, torch.bfloat16).contiguous()
    ref = dense.linear(x, w)
    kernels.rope_inplace(ref, cos[pos0:pos0 + L].contiguous(), sin[pos0:pos0 + L].contiguous(), L, 2 * H, D)
    fused = dense.qkv_rope(x, w, cos, sin, L, 2 * hid, pos0=pos0)
    assert torch.equal(fused, ref)
    pos_dev = torch.tensor([pos0], dtype=torch.int32, device=DEV)
    fused_dev = dense.qkv_rope(x, w, cos, sin, L, 2 * hid, pos0=0, pos_dev=pos_dev)
    assert torch.equal(fused_dev, ref)


# ---- backward-pass GEMMs: operand transposes in the UMMA descriptors (SURVEY 8(a)14) ---------------------

@pytest.mark.parametrize('M,N,K', [(128, 128, 64), (300, 640, 512), (706, 4096, 4096), (4096, 1024, 706),
                                   (200, 72, 136), (5648, 4096, 11008)])
@pytest.mark.parametrize('a_mn,b_mn', [(False, True), (True, True), (True, False)])
def test_gemm_transposed_operands(M, N, K, a_mn, b_mn):
    torch.manual_seed(M + N + K)
    a = (torch.randn(M, K, device=DEV) * 0.5).bfloat16()
    b = (torch.randn(N, K, device=DEV) * 0.5).bfloat16()
    want = a.float() @ b.float().t()
    a_st = a.t().contiguous() if a_mn else a      # stored [K, M]
    b_st = b.t().contiguous() if b_mn else b      # stored [K, N]
    if (M % 8 if a_mn else K % 8) or (N % 8 if b_mn else K % 8):   # 16-byte row strides (TMA)
        with pytest.raises(RuntimeError):
            dense.matmul_t(a_st, b_st, a_mn, b_mn)
        return
    _close(dense.matmul_t(a_st, b_st, a_mn, b_mn), want)
    _close(dense.matmul_t(a_st, b_st, a_mn, b_mn, out_dtype=torch.float32), want, rtol=1e-4, atol=1e-3)


def test_linear_backward_matches_autograd():
    """grad_x = grad_y.W and grad_W = grad_y^T.x through matmul_t == torch autograd of F.linear (fp32 reference)."""
    torch.manual_seed(2)
    M, N, K = 1412, 4096, 1024
    x = (torch.randn(M, K, device=DEV) * 0.5).bfloat16()
    w = (torch.randn(N, K, device=DEV) * 0.05).bfloat16()
    gy = (torch.randn(M, N, device=DEV) * 0.1).bfloat16()
    xf, wf = x.float().requires_grad_(), w.float().requires_grad_()
    (F.linear(xf, wf) * gy.float()).sum().backward()
    _close(dense.matmul_t(gy, w, b_mn=True), xf.grad)
    _close(dense.matmul_t(gy, x, a_mn=True, b_mn=True), wf.grad)
