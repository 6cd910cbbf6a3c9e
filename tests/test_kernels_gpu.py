"""GPU numerics tests of the elementwise / attention kernels against plain PyTorch fp32 references
of the same op (floating point: tolerance stated per test)."""
import math

import pytest
import torch
import torch.nn.functional as F

from gpt4roi_b200 import kernels

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
BF = torch.bfloat16


def close(got, want, rtol=1.6e-2, atol=1.6e-2):
    torch.testing.assert_close(got.float(), want.float(), rtol=rtol, atol=atol)


@pytest.mark.parametrize('D', [256, 1024, 4096])
def test_layernorm_rmsnorm(D):
    torch.manual_seed(D)
    x = (torch.randn(77, D, device=DEV) * 2 + 0.5).to(BF)
    w = (torch.rand(D, device=DEV) + 0.5).to(BF)
    b = torch.randn(D, device=DEV).to(BF)
    close(kernels.layernorm(x, w, b, 1e-5), F.layer_norm(x.float(), (D,), w.float(), b.float(), 1e-5))
    xf = x.float()
    want = w.float() * (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-6)).to(BF).float()
    close(kernels.rmsnorm(x, w, 1e-6), want, rtol=8e-3, atol=8e-3)


@pytest.mark.parametrize('M', [1, 8, 64])
@pytest.mark.parametrize('D', [1024, 4096, 8192, 520])
def test_norm_few_rows_cta_per_row_variant(M, D):
    """M <= 64 takes the CTA-per-row kernel (decode step); same reference as the warp-per-row one."""
    torch.manual_seed(D + M)
    x = (torch.randn(M, D, device=DEV) * 2 + 0.5).to(BF)
    w = (torch.rand(D, device=DEV) + 0.5).to(BF)
    b = torch.randn(D, device=DEV).to(BF)
    close(kernels.layernorm(x, w, b, 1e-5), F.layer_norm(x.float(), (D,), w.float(), b.float(), 1e-5))
    xf = x.float()
    want = w.float() * (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-6)).to(BF).float()
    close(kernels.rmsnorm(x, w, 1e-6), want, rtol=8e-3, atol=8e-3)


def test_rope_matches_hf_formula():
    """The kernel rounds where HF's bf16 ops round (bf16(bf16(x cos) + bf16(rot sin))): bit for bit."""
    torch.manual_seed(0)
    B, L, H, D = 2, 37, 4, 128
    qkv = torch.randn(B * L, 3 * H * D, device=DEV).to(BF)
    inv = 1.0 / (10000.0 ** (torch.arange(0, D, 2).float() / D))
    emb = torch.cat([torch.arange(L).float()[:, None] * inv[None]] * 2, -1)
    cos, sin = emb.cos().to(DEV, BF), emb.sin().to(DEV, BF)
    ref = qkv.clone().view(B, L, 3 * H, D)

    def rot(x):
        return torch.cat((-x[..., D // 2:], x[..., :D // 2]), -1)
    qk = ref[:, :, :2 * H]
    want = qk * cos[None, :, None, :] + rot(qk) * sin[None, :, None, :]   # bf16 ops, like HF
    got = kernels.rope_inplace(qkv.clone(), cos, sin, L, 2 * H, D).view(B, L, 3 * H, D)
    assert torch.equal(got[:, :, 2 * H:], ref[:, :, 2 * H:])                # v untouched
    assert torch.equal(got[:, :, :2 * H].view(torch.int16), want.view(torch.int16))


@pytest.mark.parametrize('impl', ['tc', 'mma'])
@pytest.mark.parametrize('L,H,D,causal', [(577, 16, 64, False), (706, 32, 128, True), (64, 2, 128, True),
                                          (130, 3, 64, True), (50, 2, 128, False), (300, 2, 128, True)])
def test_attention(L, H, D, causal, impl):
    torch.manual_seed(L)
    B = 2
    qkv = (torch.randn(B * L, 3 * H * D, device=DEV) * 0.7).to(BF)
    out = kernels.attention(qkv, B, L, H, D, causal, D ** -0.5, impl=impl).view(B, L, H, D)
    q, k, v = (t.permute(0, 2, 1, 3).float() for t in qkv.view(B, L, 3, H, D).unbind(2))
    s = (q @ k.transpose(-1, -2)) * D ** -0.5
    if causal:
        s = s.masked_fill(torch.ones(L, L, device=DEV, dtype=torch.bool).triu(1), float('-inf'))
    want = (s.softmax(-1) @ v).permute(0, 2, 1, 3)
    close(out, want, rtol=2e-2, atol=2e-2)
    assert (out.float() - want).abs().mean() < 2e-3


def test_patchify_and_embed():
    torch.manual_seed(1)
    B, S, ps, C = 2, 56, 14, 64
    img = torch.randn(B, 3, S, S, device=DEV).to(BF)
    kpad = 592
    pat = kernels.patchify(img, ps, kpad)
    want = F.unfold(img.float(), ps, stride=ps).transpose(1, 2).reshape(-1, 3 * ps * ps)
    assert torch.equal(pat[:, :588].float(), want) and pat[:, 588:].abs().sum() == 0
    P = (S // ps) ** 2
    pe = torch.randn(B * P, C, device=DEV).to(BF)
    cls, pos = torch.randn(C, device=DEV).to(BF), torch.randn(P + 1, C, device=DEV).to(BF)
    got = kernels.vit_embed(pe, cls, pos, B, P)
    want = torch.cat([cls.float().expand(B, 1, C), pe.float().view(B, P, C)], 1) + pos.float()[None]
    close(got, want, rtol=1e-2, atol=1e-2)


def test_upsample_tokens_coords():
    torch.manual_seed(2)
    B, G, C = 2, 6, 64
    hid = torch.randn(B, G * G + 1, C, device=DEV).to(BF)
    for Ho in (6, 12, 48):
        out = kernels.upsample_tokens_coords(hid, G, Ho, 128)
        x = hid[:, 1:].float().view(B, G, G, C).permute(0, 3, 1, 2)
        want = F.interpolate(x, size=(Ho, Ho), mode='bilinear', align_corners=True).permute(0, 2, 3, 1)
        close(out[..., :C], want, rtol=1e-2, atol=1e-2)
        lin = torch.linspace(-1, 1, Ho, device=DEV)
        close(out[..., C], lin[None, None, :].expand(B, Ho, Ho), rtol=1e-2, atol=4e-3)
        close(out[..., C + 1], lin[None, :, None].expand(B, Ho, Ho), rtol=1e-2, atol=4e-3)
        assert out[..., C + 2:].abs().sum() == 0


def test_fuse_gather_matches_single_shuffle():
    """gpt4roi/models/layers.py:152-180 with the previous round's GN+ReLU fused into the taps."""
    torch.manual_seed(3)
    B, C = 2, 64
    q = C // 4
    sizes = [24, 12, 6]
    raw = [torch.randn(B, h, h, C, device=DEV).to(BF) for h in sizes]
    ss = [(torch.rand(B, C, device=DEV) + 0.5, torch.randn(B, C, device=DEV) * 0.2) for _ in sizes]
    act = [torch.relu(r.float() * s[:, None, None, :] + t[:, None, None, :]).permute(0, 3, 1, 2) for r, (s, t) in zip(raw, ss)]
    for l in range(3):
        top, down = min(l + 1, 2), max(l - 1, 0)
        got = kernels.fuse_gather(raw[l], raw[top], raw[down], ss[l], ss[top], ss[down])
        tar = act[l]
        ft = F.interpolate(act[top][:, 2 * q:][:, q:], size=tar.shape[-2:], mode='bilinear', align_corners=True)
        fd = F.interpolate(act[down][:, 2 * q:][:, :q], size=tar.shape[-2:], mode='bilinear', align_corners=True)
        want = torch.cat([tar[:, :2 * q], ft, fd], 1).permute(0, 2, 3, 1)
        close(got, want, rtol=1e-2, atol=1e-2)
    # without GN (first round): plain values
    got = kernels.fuse_gather(raw[1], raw[2], raw[0])
    x = [r.float().permute(0, 3, 1, 2) for r in raw]
    want = torch.cat([x[1][:, :2 * q], F.interpolate(x[2][:, 3 * q:], size=(12, 12), mode='bilinear', align_corners=True),
                      F.interpolate(x[0][:, 2 * q:3 * q], size=(12, 12), mode='bilinear', align_corners=True)], 1)
    close(got, want.permute(0, 2, 3, 1), rtol=1e-2, atol=1e-2)


def test_gn_finalize_and_pos_mlp():
    torch.manual_seed(4)
    B, H, C, G = 2, 12, 1024, 64
    y = (torch.randn(B, H, H, C, device=DEV) * 1.5 + 0.3).to(BF)
    g = y.float().view(B, H * H, G, C // G)
    full = torch.stack([g.sum((1, 3)), (g * g).sum((1, 3))], -1)
    stats = torch.stack([full * 0.25, full * 0.5, full * 0.25], 1).contiguous()  # 3 partial slots
    gamma, beta = (torch.rand(C, device=DEV) + 0.5).to(BF), torch.randn(C, device=DEV).to(BF)
    sc, sh = kernels.gn_finalize(stats, gamma, beta, H * H * (C // G))
    want = F.group_norm(y.float().permute(0, 3, 1, 2), G, gamma.float(), beta.float(), 1e-5).permute(0, 2, 3, 1)
    got = y.float() * sc[:, None, None, :] + sh[:, None, None, :]
    torch.testing.assert_close(got, want, rtol=1e-3, atol=1e-3)
    # pos_embedd MLP
    K = 5
    boxes = torch.rand(K, 4, device=DEV)
    w0, b0 = (torch.randn(256, 4, device=DEV) * 0.5).to(BF), (torch.randn(256, device=DEV) * 0.1).to(BF)
    g2, be2 = torch.ones(256, device=DEV).to(BF), torch.zeros(256, device=DEV).to(BF)
    w3, b3 = (torch.randn(1024, 256, device=DEV) * 0.06).to(BF), (torch.randn(1024, device=DEV) * 0.06).to(BF)
    g5, be5 = (torch.rand(1024, device=DEV) + 0.5).to(BF), torch.randn(1024, device=DEV).to(BF)
    got = kernels.pos_embed_mlp(boxes, w0, b0, g2, be2, w3, b3, g5, be5)
    x = F.relu(F.linear(boxes, w0.float(), b0.float()))
    x = F.layer_norm(x, (256,), g2.float(), be2.float())
    x = F.relu(F.linear(x, w3.float(), b3.float()))
    want = F.layer_norm(x, (1024,), g5.float(), be5.float())
    torch.testing.assert_close(got, want, rtol=3e-2, atol=3e-2)
    acc, pos = torch.randn(K, 1024, device=DEV), torch.randn(K, 1024, device=DEV)
    bias = torch.randn(1024, device=DEV).to(BF)
    got = kernels.add_bias_pos_cast(acc, bias, pos)
    close(got, (acc + bias.float()).to(BF).float() + pos, rtol=1e-2, atol=1e-2)


@pytest.mark.parametrize('impl', ['tc', 'mma'])
def test_attention_seqlens(impl):
    """Right-padded batch: keys >= seqlens[b] are masked; valid rows equal the unpadded computation."""
    torch.manual_seed(5)
    B, L, H, D = 3, 200, 2, 128
    lens = torch.tensor([200, 137, 64], dtype=torch.int32, device=DEV)
    qkv = (torch.randn(B * L, 3 * H * D, device=DEV) * 0.7).to(BF)
    out = kernels.attention(qkv, B, L, H, D, True, D ** -0.5, seqlens=lens, impl=impl).view(B, L, H, D)
    for b in range(B):
        n = int(lens[b])
        solo = qkv.view(B, L, -1)[b, :n].contiguous()
        ref = kernels.attention(solo, 1, n, H, D, True, D ** -0.5, impl=impl).view(n, H, D)
        torch.testing.assert_close(out[b, :n].float(), ref.float(), rtol=1e-2, atol=1e-2)


# ---- decode step kernels (SURVEY 8(f1)) ----------------------------------------------------------------

@pytest.mark.parametrize('B,H,D', [(1, 32, 128), (8, 32, 128), (3, 4, 64), (2, 5, 128)])
@pytest.mark.parametrize('kv_len', [1, 5, 63, 64, 129, 706, 1300])
def test_decode_attention_matches_fp32_reference(B, H, D, kv_len):
    """Cluster split-KV single-query attention vs a plain fp32 softmax(q.K^T)V with the reference's
    rounding point (probabilities cast to bf16 before P.V).  Tolerance: bf16 output, rel-L2 <= 4e-3."""
    torch.manual_seed(B * 1000 + H + kv_len)
    HD, Lmax = H * D, kv_len + 7
    qkv = (torch.randn(B, 3 * HD, device=DEV)).bfloat16()
    kc = torch.randn(B, Lmax, HD, device=DEV).bfloat16()
    vc = torch.randn(B, Lmax, HD, device=DEV).bfloat16()
    scale = D ** -0.5
    got = kernels.decode_attention(qkv, kc, vc, B, H, D, kv_len, scale).float()
    q = qkv[:, :HD].float().view(B, H, 1, D)
    k = kc[:, :kv_len].float().view(B, kv_len, H, D).permute(0, 2, 1, 3)
    v = vc[:, :kv_len].float().view(B, kv_len, H, D).permute(0, 2, 1, 3)
    p = torch.softmax(q @ k.transpose(-1, -2) * scale, -1).bfloat16().float()
    want = (p @ v).permute(0, 2, 1, 3).reshape(B, HD)
    rel = ((got - want).norm() / want.norm()).item()
    assert rel < 4e-3, rel
    # device-side length (CUDA-graph replay): kv_len argument only sizes the score buffer
    pos_dev = torch.tensor([kv_len - 1], dtype=torch.int32, device=DEV)
    got_dev = kernels.decode_attention(qkv, kc, vc, B, H, D, Lmax, scale, pos_dev=pos_dev).float()
    rel = ((got_dev - want).norm() / want.norm()).item()
    assert rel < 4e-3, rel
    assert torch.equal(kernels.decode_attention(qkv, kc, vc, B, H, D, kv_len, scale).float(), got)  # reproducible


def test_kv_append_places_rows():
    torch.manual_seed(0)
    B, Ln, HD, Lmax, pos0 = 3, 4, 256, 20, 9
    qkv = torch.randn(B * Ln, 3 * HD, device=DEV).bfloat16()
    kc = torch.zeros(B, Lmax, HD, device=DEV, dtype=torch.bfloat16)
    vc = torch.zeros_like(kc)
    kernels.kv_append(qkv, kc, vc, B, Ln, pos0)
    want_k = torch.zeros_like(kc)
    want_v = torch.zeros_like(kc)
    want_k[:, pos0:pos0 + Ln] = qkv[:, HD:2 * HD].view(B, Ln, HD)
    want_v[:, pos0:pos0 + Ln] = qkv[:, 2 * HD:].view(B, Ln, HD)
    assert torch.equal(kc, want_k) and torch.equal(vc, want_v)
    kc2, vc2 = torch.zeros_like(kc), torch.zeros_like(kc)
    kernels.kv_append(qkv, kc2, vc2, B, Ln, 0, pos_dev=torch.tensor([pos0], dtype=torch.int32, device=DEV))
    assert torch.equal(kc2, want_k) and torch.equal(vc2, want_v)
    with pytest.raises(RuntimeError):
        kernels.kv_append(qkv, kc, vc, B, Ln, Lmax - 1)
