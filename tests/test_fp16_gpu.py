"""fp16 mode of the inference path (VERDICT r1 #7, SURVEY.md 8(f1)): the demo builds the model with `.half()` and
passes `images.half()` / `bboxes.half()` (gpt4roi/app.py:74-98,271,296).  Every inference kernel has an fp16 twin
(`*_f16` entry points, csrc/act_type.cuh: same sources, fp16 storage and tensor-core operand format, fp32
accumulation, the same rounding points).  Checked here through the C ABI:

  * kernel level -- GEMM (+ epilogues), conv, norms, wgmma attention, the decode GEMM / attention -- against fp32
    torch references on fp16-representable inputs; tolerances are the bf16 tests' divided by 4 (fp16 carries three more
    mantissa bits), stated inline;
  * engine level -- region-token prefill vs the fp32 oracle on fp16-representable weights: closer than the bf16 engine
    on the same inputs; decode loop (CUDA graph + eager) vs the prefill of the grown sequence;
  * seam level -- `SPILlavaMPTForCausalLM(...).half()` selects the fp16 engine and returns fp16 logits."""
import pytest
import torch
import torch.nn.functional as F

from gpt4roi_b200 import dense, kernels
from gpt4roi_b200.engine import EngineConfig, PrefillEngine, random_state_dicts
from oracle import model_oracle
from tests.test_engine_gpu import make_inputs, rel

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
H = torch.float16


def _close(got, want, rtol=4e-3, atol=4e-3):
    got, want = got.float(), want.float()
    err = (got - want).abs()
    bound = atol + rtol * want.abs()
    assert bool((err <= bound).all()), 'max err %.3e (bound %.3e)' % (err.max().item(), bound.flatten()[err.argmax()].item())


@pytest.mark.parametrize('M,N,K', [(128, 128, 64), (200, 384, 320), (706, 4096, 4096), (5648, 1024, 1024), (8, 4096, 4096)])
def test_gemm_f16_plain_and_epilogues(M, N, K):
    """D = act(A W^T + bias) + residual on the wgmma tile kernel and, for M <= 16, the skinny
    kernel: fp16 operands, fp32 accumulate, one rounding to fp16."""
    torch.manual_seed(M + N + K)
    a = (torch.randn(M, K, device=DEV) * 0.5).to(H)
    w = (torch.randn(N, K, device=DEV) * 0.05).to(H)
    b = (torch.randn(N, device=DEV) * 0.1).to(H)
    r = torch.randn(M, N, device=DEV).to(H)
    want = a.float() @ w.float().t()
    _close(dense.linear(a, w), want)
    _close(dense.linear(a, w, b, act='relu', residual=r), F.relu(want + b.float()) + r.float())
    qg = want + b.float()
    _close(dense.linear(a, w, b, act='quick_gelu'), qg * torch.sigmoid(1.702 * qg))
    if M > 16:
        _close(dense.linear(a, w, out_dtype=torch.float32), want, rtol=1e-4, atol=1e-3)
        r32 = torch.randn(M, N, device=DEV)
        got = dense.linear(a, w, b, residual=r32, out_dtype=torch.float32, round_branch=True)
        _close(got, (want + b.float()).to(H).float() + r32, rtol=1e-3, atol=2e-3)
    with pytest.raises(TypeError):
        dense.linear(a, w.bfloat16())                      # mixed 16-bit types are rejected, not converted


def test_swiglu_and_qkv_rope_f16():
    torch.manual_seed(1)
    M, K, I = 412, 1024, 2048
    x = (torch.randn(M, K, device=DEV) * 0.5).to(H)
    wg, wu = (torch.randn(I, K, device=DEV) * 0.04).to(H), (torch.randn(I, K, device=DEV) * 0.04).to(H)
    wgu = torch.stack([wg, wu], 1).reshape(2 * I, K).contiguous()
    g, u = x.float() @ wg.float().t(), x.float() @ wu.float().t()
    _close(dense.linear(x, wgu, act='swiglu'), F.silu(g) * u)
    # fused q|k|v projection + rotary embedding == unfused GEMM followed by the rope kernel (same rounding points)
    L, nh, hd = 103, 8, 128
    xs = (torch.randn(4 * L, K, device=DEV) * 0.5).to(H)
    wqkv = (torch.randn(3 * nh * hd, K, device=DEV) * 0.03).to(H)
    inv = 1.0 / (10000.0 ** (torch.arange(0, hd, 2).float() / hd))
    fr = torch.arange(L).float()[:, None] * inv[None]
    emb = torch.cat([fr, fr], -1)
    cos, sin = emb.cos().to(DEV, H).contiguous(), emb.sin().to(DEV, H).contiguous()
    fused = dense.qkv_rope(xs, wqkv, cos, sin, L, 2 * nh * hd)
    plain = dense.linear(xs, wqkv)
    kernels.rope_inplace(plain, cos, sin, L, 2 * nh, hd)
    assert torch.equal(fused, plain)


def test_conv_and_groupnorm_stats_f16():
    torch.manual_seed(2)
    n, Hh, cin, cout = 2, 24, 128, 256
    x = torch.randn(n, Hh, Hh, cin, device=DEV).to(H)
    w = (torch.randn(cout, 3, 3, cin, device=DEV) * 0.03).to(H)
    st = torch.zeros((n, dense.gn_slots(Hh, Hh), cout // 16, 2), dtype=torch.float32, device=DEV)
    got = dense.conv_nhwc(x, w, gn_stats=st)
    want = F.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), padding=1).permute(0, 2, 3, 1)
    _close(got, want)
    # the epilogue's GroupNorm partial sums are those of the fp16 output it stored
    g16 = got.float().view(n, Hh * Hh, cout // 16, 16)
    s = st.sum(1)
    assert rel(s[..., 0], g16.sum((1, 3))) < 1e-4 and rel(s[..., 1], (g16 * g16).sum((1, 3))) < 1e-4
    gamma, beta = torch.randn(cout, device=DEV).to(H), torch.randn(cout, device=DEV).to(H)
    sc, sh = kernels.gn_finalize(st, gamma, beta, count=Hh * Hh * 16)
    y = kernels.affine_relu_nhwc(got, sc, sh)
    ref = F.relu(F.group_norm(got.float().permute(0, 3, 1, 2), cout // 16, gamma.float(), beta.float())).permute(0, 2, 3, 1)
    _close(y, ref, rtol=5e-3, atol=5e-3)


@pytest.mark.parametrize('M,D', [(5, 4096), (300, 4096), (77, 1024)])
def test_norms_f16(M, D):
    torch.manual_seed(M)
    x = torch.randn(M, D, device=DEV).to(H)
    w, b = (1 + 0.1 * torch.randn(D, device=DEV)).to(H), (0.1 * torch.randn(D, device=DEV)).to(H)
    _close(kernels.layernorm(x, w, b, 1e-5), F.layer_norm(x.float(), (D,), w.float(), b.float(), 1e-5))
    xf = x.float()
    want = w.float() * (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-6)).to(H).float()   # LlamaRMSNorm in fp16
    _close(kernels.rmsnorm(x, w, 1e-6), want, rtol=2e-3, atol=2e-3)
    x32 = torch.randn(M, D, device=DEV)
    got = kernels.layernorm_ex(x32, w, b, 1e-5)
    assert got.dtype == H
    _close(got, F.layer_norm(x32, (D,), w.float(), b.float(), 1e-5))


@pytest.mark.parametrize('B,L,nh,hd,causal', [(2, 577, 16, 64, False), (2, 706, 8, 128, True), (1, 130, 4, 128, True)])
def test_attention_tcgen05_f16(B, L, nh, hd, causal):
    torch.manual_seed(L)
    qkv = (torch.randn(B * L, 3 * nh * hd, device=DEV) * 0.7).to(H)
    got = kernels.attention(qkv, B, L, nh, hd, causal, hd ** -0.5)
    q, k, v = (t.view(B, L, nh, hd).transpose(1, 2).float() for t in qkv.split(nh * hd, 1))
    want = F.scaled_dot_product_attention(q, k, v, is_causal=causal).transpose(1, 2).reshape(B * L, nh * hd)
    _close(got, want, rtol=5e-3, atol=3e-3)
    legacy = kernels.attention(qkv, B, L, nh, hd, causal, hd ** -0.5, impl='mma')
    _close(legacy, want, rtol=5e-3, atol=3e-3)


def test_decode_kernels_f16():
    """Skinny GEMM with the RoPE + KV-append epilogue and the single-query attention, fp16."""
    torch.manual_seed(5)
    B, nh, hd, Lmax, pos = 3, 32, 128, 64, 17
    HD = nh * hd
    x = (torch.randn(B, HD, device=DEV) * 0.5).to(H)
    wqkv = (torch.randn(3 * HD, HD, device=DEV) * 0.02).to(H)
    inv = 1.0 / (10000.0 ** (torch.arange(0, hd, 2).float() / hd))
    fr = torch.arange(Lmax).float()[:, None] * inv[None]
    emb = torch.cat([fr, fr], -1)
    cos, sin = emb.cos().to(DEV, H).contiguous(), emb.sin().to(DEV, H).contiguous()
    kc = (torch.randn(B, Lmax, HD, device=DEV) * 0.5).to(H)
    vc = (torch.randn(B, Lmax, HD, device=DEV) * 0.5).to(H)
    qkv = dense.decode_gemm(x, wqkv, rope=(cos, sin, 2 * HD, pos, None), kv=(kc, vc))
    ref = dense.qkv_rope(x, wqkv, cos, sin, 1, 2 * HD, pos0=pos)          # M <= 16: also the skinny kernel, no cache write
    assert torch.equal(qkv, ref)
    assert torch.equal(kc[:, pos], qkv[:, HD:2 * HD]) and torch.equal(vc[:, pos], qkv[:, 2 * HD:])
    out = kernels.decode_attention(qkv, kc, vc, B, nh, hd, pos + 1, hd ** -0.5)
    q = qkv[:, :HD].view(B, nh, 1, hd).float()
    k = kc[:, :pos + 1].view(B, pos + 1, nh, hd).transpose(1, 2).float()
    v = vc[:, :pos + 1].view(B, pos + 1, nh, hd).transpose(1, 2).float()
    want = F.scaled_dot_product_attention(q, k, v).reshape(B, HD)
    _close(out, want, rtol=5e-3, atol=3e-3)


def _fp16_weights(cfg, seed):
    sd, vit_sd = random_state_dicts(cfg, DEV, seed=seed, dtype=torch.float32)
    return {k: v.half().float() for k, v in sd.items()}, {k: v.half().float() for k, v in vit_sd.items()}


def test_engine_f16_vs_fp32_oracle_and_vs_bf16_engine():
    """Region-token prefill in fp16 vs the fp32 oracle on the same fp16-representable weights and inputs: per-stage and
    logits rel-L2 below 6e-3 (bf16 engine, same test in tests/test_engine_gpu.py: 2e-2), and closer than the bf16
    engine run on the same inputs."""
    cfg = EngineConfig(image_size=224, vit_layers=24, n_layers=2, dtype='fp16')
    sd, vit_sd = _fp16_weights(cfg, 7)
    ids, images, boxes = make_inputs(cfg, 2, [3, 1], 24)
    images = images.half()
    eng = PrefillEngine(cfg, sd, vit_sd, DEV)
    assert eng.dt == H and eng.layers[0]['wqkv'].dtype == H
    st = {}
    got = eng.forward(ids.to(DEV), images.to(DEV), boxes, stage_taps=st)
    assert got.dtype == H and torch.isfinite(got.float()).all()
    ref32, inter = model_oracle.forward(cfg, sd, vit_sd, ids, images.float(), boxes, DEV, autocast_bf16=False,
                                        return_intermediates=True)
    e16 = rel(got, ref32)
    cfg_b = EngineConfig(image_size=224, vit_layers=24, n_layers=2)
    e_b = rel(PrefillEngine(cfg_b, sd, vit_sd, DEV).forward(ids.to(DEV), images.to(DEV, torch.bfloat16), boxes), ref32)
    e_reg = rel(st['region'], torch.cat(inter['region']))
    e_vit = max(rel(t, r) for t, r in zip(st['vit_taps'], inter['vit_taps']))
    print('fp16 engine vs fp32 oracle: logits %.3e (bf16 engine %.3e), region tokens %.3e, ViT taps %.3e' % (e16, e_b, e_reg, e_vit))
    assert e16 < 6e-3 and e_reg < 6e-3 and e_vit < 6e-3
    assert e16 < e_b
    agree = (got.float().argmax(-1) == ref32.argmax(-1)).float().mean().item()
    assert agree > 0.97, agree


def test_decode_loop_f16_matches_prefill():
    """generate() in fp16: the CUDA-graph decode loop and the eager loop produce the same tokens, and the logits of the
    last decode step equal the prefill of the grown sequence within 1e-2 rel-L2 (the bf16 test's bound)."""
    cfg = EngineConfig(image_size=224, vit_layers=12, n_layers=2, dtype='fp16')
    sd, vit_sd = _fp16_weights(cfg, 11)
    eng = PrefillEngine(cfg, sd, vit_sd, DEV)
    ids, images, boxes = make_inputs(cfg, 2, [2, 1], 20, seed=2)
    n_new = 7
    out_g = eng.generate(ids, images.half(), boxes, max_new_tokens=n_new, use_graph=True)
    out_e = eng.generate(ids, images.half(), boxes, max_new_tokens=n_new, use_graph=False)
    assert torch.equal(out_g, out_e)
    assert out_g.shape == (2, ids.shape[1] + n_new)
    full = eng.forward(out_g[:, :-1], images.half(), boxes)                # teacher-forced prefill over the grown sequence
    nxt = full[:, ids.shape[1] - 1:].float().argmax(-1)
    assert (nxt == out_g[:, ids.shape[1]:].to(nxt.device)).float().mean().item() >= 0.85   # near-ties may flip a token


def test_seam_half_model_selects_fp16_engine():
    from tests.test_model_seam_gpu import build_seam_model
    cfg = EngineConfig(image_size=224, vit_layers=12, n_layers=1)
    sd, vit_sd = _fp16_weights(cfg, 13)
    ids, images, boxes = make_inputs(cfg, 1, [2], 12, seed=4)
    model = build_seam_model(cfg, sd, vit_sd, dtype=torch.float16).eval()
    with torch.no_grad():
        out = model(input_ids=ids.to(DEV), images=images.half().to(DEV), bboxes=[b.half().to(DEV) for b in boxes])
    eng = model._get_engine(torch.device(DEV))
    assert eng.dt == H and out.logits.dtype == H
    ref = model_oracle.forward(cfg, sd, vit_sd, ids, images.half().float(), [b.half().float() for b in boxes], DEV)
    e = rel(out.logits, ref)
    print('seam .half(): logits rel-L2 vs fp32 oracle %.3e' % e)
    assert e < 6e-3
    model = model.bfloat16()                                              # re-cast -> the bf16 engine is rebuilt
    with torch.no_grad():
        out_b = model(input_ids=ids.to(DEV), images=images.to(DEV), bboxes=boxes)
    assert model._get_engine(torch.device(DEV)).dt == torch.bfloat16 and out_b.logits.dtype == torch.bfloat16
