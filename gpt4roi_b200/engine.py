"""Region-token prefill engine: CLIP-ViT-L/14 -> MLVL fuse -> multi-level RoIAlign -> region
projector -> splice -> LLaMA prefill -> lm_head, every op a hand-written sm_90a kernel behind
the C ABI.  PyTorch supplies device memory, streams and CUDA-graph capture only.

Reference call stack reproduced (SURVEY.md 3.3):
  gpt4roi/models/spi_llava.py:23-205   SPILlavaLlamaModel.forward
  gpt4roi/models/layers.py:182-195     MLVLFuseModule.forward
  gpt4roi/models/layers.py:218-236     MLVLROIQueryModule.forward
  gpt4roi/models/layers.py:280-335     MlvlRoIExtractor.forward
  llava/model/llava.py:203-261         LlavaLlamaForCausalLM.forward (lm_head)
  transformers CLIPVisionModel / LlamaModel (third party, pyproject.toml:19)

Weights come in with the reference's parameter names (SURVEY.md App. C) and are re-laid-out
ONCE at load time (fused QKV, interleaved gate/up, NHWC conv filters, flatten_linear permuted
from (c,ph,pw) to (ph,pw,c)).  Numerics: bf16 storage, fp32 accumulation, rounding points of the
reference under bf16 autocast.
"""
import collections
import math
import os

import torch

from . import dense, kernels, lib
from .roi_align import roi_align_mlvl
from .splice import splice_region_tokens

BF16 = torch.bfloat16


class EngineConfig:
    def __init__(self, image_size=336, patch_size=14, vit_hidden=1024, vit_heads=16, vit_layers=24,
                 vit_mlp=4096, vit_eps=1e-5, select_layer=-2, num_levels=4,
                 hidden=4096, n_heads=32, n_layers=32, mlp=11008, vocab=32006, rms_eps=1e-6,
                 rope_theta=10000.0, roi_out=14, roi_sampling=2, spi_dim=1024, gn_groups=64,
                 im_patch_token=32001, bbox_token=32002, im_start_token=32004, im_end_token=32005,
                 llama_stream=None, dtype='bf16'):
        """dtype: the 16-bit storage type of weights and activations -- 'bf16' (training scripts, BASELINE "7B bf16
        prefill") or 'fp16' (the demo: gpt4roi/app.py:74-98,271 builds the model with .half()); fp16 runs the `_f16`
        twins of every kernel (csrc/act_type.cuh), same fp32 accumulation and rounding points.
        llama_stream: dtype of the LLaMA residual stream in the prefill -- 'bf16' (default: what the reference has
        when the model was cast to bf16, the BASELINE "7B bf16 prefill" mode) or 'fp32' (what the reference has
        whenever its parameters are fp32 under autocast; closer to the fp32 anchor at 32 layers, somewhat slower:
        tests/test_parity_7b_gpu.py).  Env G4R_LLAMA_STREAM overrides the default."""
        if llama_stream is None:
            llama_stream = os.environ.get('G4R_LLAMA_STREAM', 'bf16')
        if llama_stream not in ('fp32', 'bf16'):
            raise ValueError('llama_stream must be fp32 or bf16 (bf16 = the 16-bit storage type)')
        if dtype in (torch.bfloat16, torch.float16):
            dtype = 'bf16' if dtype == torch.bfloat16 else 'fp16'
        if dtype not in ('bf16', 'fp16'):
            raise ValueError("dtype must be 'bf16' or 'fp16'")
        self.__dict__.update(locals())
        del self.__dict__['self']
        self.torch_dtype = torch.bfloat16 if dtype == 'bf16' else torch.float16
        self.grid = image_size // patch_size
        self.num_patches = self.grid ** 2
        self.head_dim = hidden // n_heads
        self.vit_head_dim = vit_hidden // vit_heads
        self.strides = [patch_size / 8, patch_size / 4, patch_size / 2, patch_size][-num_levels:] \
            if num_levels <= 4 else None
        self.level_sizes = [self.grid * 2 ** (num_levels - 1 - l) for l in range(num_levels)]
        # spi_llava.py:68-82: hidden_states[select::-3][::-1][-num_levels:]
        sel = select_layer if select_layer >= 0 else vit_layers + 1 + select_layer
        lv = list(range(sel, -1, -3))[::-1][-num_levels:]
        self.select_index = sel
        self.level_layers = lv


def _b(t, dev, dt=BF16):
    return t.detach().to(device=dev, dtype=dt).contiguous()


class PrefillEngine:
    """Holds re-laid-out weights on one GPU and runs the fused forward."""

    def __init__(self, cfg, llm_sd, vit_sd, device, parts=('vit', 'spi', 'llm')):
        """parts: which weight groups to prepare -- ('spi',) builds an SPI-module-only engine (the model-seam
        mirrors of MLVLROIQueryModule / MLVLFuseModule / MlvlRoIExtractor run on it)."""
        self.cfg = cfg
        self.dev = torch.device(device)
        self.dt = cfg.torch_dtype          # bf16, or fp16 for the demo's dtype
        self.parts = tuple(parts)
        if 'vit' in self.parts:
            self._prepare_vit(vit_sd)
        if 'spi' in self.parts:
            self._prepare_spi(llm_sd)
        if 'llm' in self.parts:
            self._prepare_llm(llm_sd)
        self._rope_cache = {}

    # ------------------------------------------------------------------ weight preparation
    def _prepare_vit(self, sd):
        c, dev = self.cfg, self.dev
        p = 'vision_model.'
        kreal = 3 * c.patch_size ** 2
        self.vit_kpad = (kreal + 7) // 8 * 8
        w = sd[p + 'embeddings.patch_embedding.weight'].reshape(c.vit_hidden, kreal)
        wp = torch.zeros(c.vit_hidden, self.vit_kpad, dtype=self.dt, device=dev)
        wp[:, :kreal] = w.to(dev, self.dt)
        self.vit_patch_w = wp
        self.vit_cls = _b(sd[p + 'embeddings.class_embedding'], dev, self.dt)
        self.vit_pos = _b(sd[p + 'embeddings.position_embedding.weight'], dev, self.dt)
        self.vit_pre_ln = (_b(sd[p + 'pre_layrnorm.weight'], dev, self.dt), _b(sd[p + 'pre_layrnorm.bias'], dev, self.dt))
        self.vit_layers = []
        for i in range(c.select_index):  # layers beyond the selected hidden state are dead work
            q = p + 'encoder.layers.%d.' % i
            wqkv = torch.cat([sd[q + 'self_attn.%s_proj.weight' % n] for n in 'qkv'], 0)
            bqkv = torch.cat([sd[q + 'self_attn.%s_proj.bias' % n] for n in 'qkv'], 0)
            self.vit_layers.append(dict(
                ln1=(_b(sd[q + 'layer_norm1.weight'], dev, self.dt), _b(sd[q + 'layer_norm1.bias'], dev, self.dt)),
                wqkv=_b(wqkv, dev, self.dt), bqkv=_b(bqkv, dev, self.dt),
                wo=_b(sd[q + 'self_attn.out_proj.weight'], dev, self.dt), bo=_b(sd[q + 'self_attn.out_proj.bias'], dev, self.dt),
                ln2=(_b(sd[q + 'layer_norm2.weight'], dev, self.dt), _b(sd[q + 'layer_norm2.bias'], dev, self.dt)),
                w1=_b(sd[q + 'mlp.fc1.weight'], dev, self.dt), b1=_b(sd[q + 'mlp.fc1.bias'], dev, self.dt),
                w2=_b(sd[q + 'mlp.fc2.weight'], dev, self.dt), b2=_b(sd[q + 'mlp.fc2.bias'], dev, self.dt)))

    def _prepare_spi(self, sd):
        """SPI-module weights in engine layout.  The two halves are independent (a stand-alone MLVLFuseModule or
        MlvlRoIExtractor mirror owns only one of them): whatever keys are present are prepared."""
        c, dev = self.cfg, self.dev
        p = 'model.spi_module.'
        C = c.spi_dim
        self.spi_cpad = (C + 2 + 63) // 64 * 64  # 1026 -> 1088
        if p + 'mlvl_fuse.input_conv.0.weight' in sd:
            self.in_w, self.in_b = [], []
            for l in range(c.num_levels):
                w = sd[p + 'mlvl_fuse.input_conv.%d.weight' % l].reshape(C, C + 2)
                wp = torch.zeros(C, self.spi_cpad, dtype=self.dt, device=dev)
                wp[:, :C + 2] = w.to(dev, self.dt)
                self.in_w.append(wp)
                self.in_b.append(_b(sd[p + 'mlvl_fuse.input_conv.%d.bias' % l], dev, self.dt))
            self.fuse = []
            for r in range(5):
                q = p + 'mlvl_fuse.fuse_convs.%d.' % r
                w = sd[q + 'conv.weight'].to(dev, self.dt).permute(0, 2, 3, 1).contiguous()  # [Cout,kh,kw,Cin]
                self.fuse.append(dict(w=w, gamma=_b(sd[q + 'gn.weight'], dev, self.dt), beta=_b(sd[q + 'gn.bias'], dev, self.dt)))
        q = p + 'roi_align.'
        if q + 'flatten_linear.weight' in sd:
            pw = torch.stack([sd[q + 'pconvs.%d.weight' % l].to(dev, self.dt).permute(0, 2, 3, 1)
                              for l in range(c.num_levels)], 1).contiguous()  # [Cout, L, kh, kw, Cin]
            self.pconv_w = pw
            self.pconv_b = sum(sd[q + 'pconvs.%d.bias' % l].to(dev, torch.float32) for l in range(c.num_levels)).contiguous()
            R = c.roi_out
            fw = sd[q + 'flatten_linear.weight']  # [1024, C*R*R] in (c, ph, pw) order (layers.py:326)
            self.flat_w = fw.to(dev, self.dt).reshape(-1, C, R, R).permute(0, 2, 3, 1).reshape(fw.shape[0], -1).contiguous()
            self.flat_b = _b(sd[q + 'flatten_linear.bias'], dev, self.dt)
            self.pos = [_b(sd[q + 'pos_embedd.%s' % n], dev, self.dt) for n in
                        ('0.weight', '0.bias', '2.weight', '2.bias', '3.weight', '3.bias', '5.weight', '5.bias')]
            self.up_w, self.up_b = _b(sd[q + 'updims.weight'], dev, self.dt), _b(sd[q + 'updims.bias'], dev, self.dt)
            kb = self.flat_w.shape[1] // 64
            self.flat_splits = next(s for s in (16, 14, 8, 7, 4, 2, 1) if kb % s == 0)
        if 'model.mm_projector.weight' in sd:
            self.proj_w, self.proj_b = _b(sd['model.mm_projector.weight'], dev, self.dt), _b(sd['model.mm_projector.bias'], dev, self.dt)

    def _prepare_llm(self, sd):
        c, dev = self.cfg, self.dev
        self.embed = _b(sd['model.embed_tokens.weight'], dev, self.dt)
        self.layers = []
        for i in range(c.n_layers):
            q = 'model.layers.%d.' % i
            wqkv = torch.cat([sd[q + 'self_attn.%s_proj.weight' % n].to(dev, self.dt) for n in 'qkv'], 0).contiguous()
            g, u = sd[q + 'mlp.gate_proj.weight'].to(dev, self.dt), sd[q + 'mlp.up_proj.weight'].to(dev, self.dt)
            wgu = torch.stack([g, u], 1).reshape(2 * g.shape[0], g.shape[1]).contiguous()  # rows: g0,u0,g1,u1,...
            self.layers.append(dict(
                ln_in=_b(sd[q + 'input_layernorm.weight'], dev, self.dt), wqkv=wqkv,
                wo=_b(sd[q + 'self_attn.o_proj.weight'], dev, self.dt),
                ln_post=_b(sd[q + 'post_attention_layernorm.weight'], dev, self.dt), wgu=wgu,
                wdown=_b(sd[q + 'mlp.down_proj.weight'], dev, self.dt)))
            del g, u
        self.norm_w = _b(sd['model.norm.weight'], dev, self.dt)
        self.lm_head = _b(sd['lm_head.weight'], dev, self.dt) if 'lm_head.weight' in sd else None   # LlamaModel-only seam
        self.vocab_pad = (c.vocab + 63) // 64 * 64

    def _rope(self, L):
        """cos/sin tables exactly as LlamaRotaryEmbedding (modeling_llama.py:118-135): fp32 then bf16."""
        if L not in self._rope_cache:
            c = self.cfg
            inv = 1.0 / (c.rope_theta ** (torch.arange(0, c.head_dim, 2, dtype=torch.int64).float() / c.head_dim))
            freqs = torch.arange(L, dtype=torch.float32)[:, None] * inv[None, :]
            emb = torch.cat((freqs, freqs), -1)
            self._rope_cache[L] = (emb.cos().to(self.dev, self.dt).contiguous(), emb.sin().to(self.dev, self.dt).contiguous())
        return self._rope_cache[L]

    def _rope_span(self, n):
        """cos/sin tables covering positions 0..n-1, for kernels that index them by position (decode steps, chunks
        continuing a cache).  Sized to a power of two >= 1024, so a cache that grows every turn adds a table only when it
        doubles."""
        return self._rope(max(1024, 1 << (int(n) - 1).bit_length()))

    # ------------------------------------------------------------------ stages
    def vit(self, images):
        """images bf16 [B,3,S,S] -> dict{layer index: hidden state [B,P+1,C]} for the consumed layers."""
        c = self.cfg
        B = images.shape[0]
        P, T = c.num_patches, c.num_patches + 1
        patches = kernels.patchify(images, c.patch_size, self.vit_kpad)
        pe = dense.linear(patches, self.vit_patch_w)
        x = kernels.vit_embed(pe, self.vit_cls, self.vit_pos, B, P)
        # Residual stream in fp32, as the reference has it under autocast: nn.LayerNorm returns fp32
        # (pre_layrnorm turns the bf16 embeddings into an fp32 stream) and `residual + bf16_branch`
        # stays fp32; the Linears see bf16 inputs (autocast cast) and produce bf16 outputs.
        F32 = torch.float32
        x = kernels.layernorm_ex(x, *self.vit_pre_ln, eps=c.vit_eps, out_dtype=F32).view(B * T, c.vit_hidden)
        taps = {}
        scale = c.vit_head_dim ** -0.5
        for i, w in enumerate(self.vit_layers):
            h = kernels.layernorm_ex(x, *w['ln1'], eps=c.vit_eps)
            qkv = dense.linear(h, w['wqkv'], w['bqkv'])
            a = kernels.attention(qkv, B, T, c.vit_heads, c.vit_head_dim, False, scale)
            x = dense.linear(a, w['wo'], w['bo'], residual=x, out_dtype=F32, round_branch=True)
            h = kernels.layernorm_ex(x, *w['ln2'], eps=c.vit_eps)
            f = dense.linear(h, w['w1'], w['b1'], act='quick_gelu')
            x = dense.linear(f, w['w2'], w['b2'], residual=x, out_dtype=F32, round_branch=True)
            if (i + 1) in c.level_layers:
                taps[i + 1] = x.view(B, T, c.vit_hidden)
        return taps

    def fuse_maps(self, taps, has_cls=True, pre_upsampled=False):
        """MLVLROIQueryModule upsampling + MLVLFuseModule: returns the last round's raw conv outputs
        (bf16 NHWC) and the per-(image,channel) GroupNorm scale/shift still to be applied.
        taps: {layer: [B, 1+P, C]} ViT hidden states (CLS first), or with has_cls=False a list / dict of
        [B, P, C] token maps in level order (what MLVLROIQueryModule.forward receives, layers.py:218-224).
        pre_upsampled: the level-l entry already has the pyramid size [B, H_l*H_l, C] (MLVLFuseModule.forward's
        input, layers.py:182): the resampling step degenerates to the identity and only appends the coordinates."""
        c = self.cfg
        C = c.spi_dim
        if isinstance(taps, (list, tuple)):
            taps = {layer: t for layer, t in zip(c.level_layers, taps)}
        B = next(iter(taps.values())).shape[0]
        maps = []
        for l, layer in enumerate(c.level_layers):
            H = c.level_sizes[l]
            up = kernels.upsample_tokens_coords(taps[layer], H if pre_upsampled else c.grid, H, self.spi_cpad,
                                                has_cls=has_cls, dtype=self.dt)
            m = dense.linear(up.view(-1, self.spi_cpad), self.in_w[l], self.in_b[l]).view(B, H, H, C)
            maps.append(m)
        ss = [None] * c.num_levels
        n = c.num_levels
        for r in range(5):
            new, stats = [], []
            for l in range(n):
                top, down = min(l + 1, n - 1), max(l - 1, 0)
                x_in = kernels.fuse_gather(maps[l], maps[top], maps[down], ss[l], ss[top], ss[down])
                st = torch.zeros((B, dense.gn_slots(c.level_sizes[l], c.level_sizes[l]), c.gn_groups, 2),
                                 dtype=torch.float32, device=self.dev)
                new.append(dense.conv_nhwc(x_in, self.fuse[r]['w'], gn_stats=st))
                stats.append(st)
            maps = new
            ss = [kernels.gn_finalize(stats[l], self.fuse[r]['gamma'], self.fuse[r]['beta'],
                                      count=c.level_sizes[l] ** 2 * (C // c.gn_groups)) for l in range(n)]
        return maps, ss

    def region_tokens(self, maps, ss, boxes, batch_idx):
        """MlvlRoIExtractor.forward: boxes fp32 [K,4] normalised xyxy, batch_idx fp32 [K] -> [K,hidden]."""
        c = self.cfg
        K = boxes.shape[0]
        rois = torch.cat([batch_idx[:, None], boxes * float(c.image_size)], 1).contiguous()  # layers.py:294-302
        scales = [float(torch.tensor(1.0 / s, dtype=torch.float32)) for s in c.strides]
        # ss=None: the maps are already activated (MlvlRoIExtractor.forward called on its own)
        feats = roi_align_mlvl(maps, rois, c.roi_out, scales, c.roi_sampling, True, out_dtype=self.dt,
                               gn_scale=None if ss is None else [s for s, _ in ss],
                               gn_shift=None if ss is None else [b for _, b in ss])
        R = c.roi_out
        pc = dense.conv_nhwc(feats.view(c.num_levels * K, R, R, c.spi_dim), self.pconv_w, self.pconv_b,
                             act='relu', levels=c.num_levels)
        acc = dense.linear(pc.view(K, -1), self.flat_w, out_dtype=torch.float32, k_splits=self.flat_splits) \
            if self.flat_splits > 1 else dense.linear(pc.view(K, -1), self.flat_w, out_dtype=torch.float32)
        pos = kernels.pos_embed_mlp(boxes.contiguous(), *self.pos)
        t = kernels.add_bias_pos_cast(acc, self.flat_b, pos)
        return dense.linear(t, self.up_w, self.up_b)

    def llama(self, embeds, B, L, last_only=False, seqlens=None, cache=None, hidden_taps=None, want='logits',
              start=None):
        """hidden_taps: optional dict {n: None}; filled with a copy of the residual stream after decoder layer n
        (1-based; the parity tests record error growth with depth).  want='hidden' returns the final-norm
        hidden states [B, L, hidden] instead of logits (LlamaModel.forward's last_hidden_state).
        start: device int32 [B] -- the L rows of each sample continue the sequence held in `cache`: they sit at
        positions start[b].. (seqlens: each sample's valid rows), are appended there and attend over the cached prefix
        too (kernels.attention_cached; head_dim 128).  On a row view (cache.rows) the rows are those of the larger cache
        the table names, and only each sample's valid rows are appended."""
        c = self.cfg
        x = embeds.view(B * L, c.hidden)
        if start is None:
            cos, sin = self._rope(L)
        else:
            # the fused QKV-RoPE epilogue rotates every chunk row, padding included, at start[b] + t (t < L): a cache that
            # grows covers those positions; a row view never grows, so its table is sized by the last position touched
            n = cache.max_len if cache.rows is None else max(cache.max_len, int(start.max()) + L)
            cos, sin = self._rope_span(n)
        scale = c.head_dim ** -0.5
        # fp32 residual stream: the first o_proj epilogue widens it (bf16 residual in, fp32 out); every branch output
        # is rounded to bf16 before the fp32 add, as a bf16 nn.Linear output added to an fp32 stream under autocast
        f32 = dict(out_dtype=torch.float32, round_branch=True) if c.llama_stream == 'fp32' else {}
        rows = cache.rows if start is not None else None
        if rows is not None:   # a row view of a larger cache: only each row's valid chunk rows are appended
            qlen = seqlens if seqlens is not None else torch.full((B,), L, dtype=torch.int32, device=self.dev)
        for li, w in enumerate(self.layers):
            h = kernels.rmsnorm(x, w['ln_in'], c.rms_eps)
            if rows is not None:
                qkv = dense.qkv_rope(h, w['wqkv'], cos, sin, L, 2 * c.hidden, pos_rows=start)
                kernels.kv_append(qkv, cache.k[li], cache.v[li], B, L, 0, pos_rows=start, cache_rows=rows, qlen=qlen)
                a = kernels.attention_cached(qkv, cache.k[li], cache.v[li], B, c.n_heads, c.head_dim, L, scale, start,
                                             qlen, cache_rows=rows)
            elif start is not None:
                qkv = dense.qkv_rope(h, w['wqkv'], cos, sin, L, 2 * c.hidden, pos_rows=start)
                kernels.kv_append(qkv, cache.k[li], cache.v[li], B, L, 0, pos_rows=start)
                a = kernels.attention_cached(qkv, cache.k[li], cache.v[li], B, c.n_heads, c.head_dim, L, scale, start,
                                             seqlens)
            elif c.head_dim == 128 and (2 * c.hidden) % 256 == 0:
                qkv = dense.qkv_rope(h, w['wqkv'], cos, sin, L, 2 * c.hidden)   # RoPE fused into the GEMM epilogue
            else:
                qkv = dense.linear(h, w['wqkv'])
                kernels.rope_inplace(qkv, cos, sin, L, 2 * c.n_heads, c.head_dim)
            if start is None:
                if cache is not None:  # keep post-RoPE K and V for the decode loop
                    kernels.kv_append(qkv, cache.k[li], cache.v[li], B, L, 0)
                a = kernels.attention(qkv, B, L, c.n_heads, c.head_dim, True, scale, seqlens=seqlens)
            x = dense.linear(a, w['wo'], residual=x, **f32)
            h = kernels.rmsnorm(x, w['ln_post'], c.rms_eps)
            f = dense.linear(h, w['wgu'], act='swiglu')
            x = dense.linear(f, w['wdown'], residual=x, **f32)
            if hidden_taps is not None and (li + 1) in hidden_taps:
                hidden_taps[li + 1] = x.view(B, L, c.hidden).clone()
        if last_only and seqlens is not None:   # each row's last valid position (right-padded rows)
            x = x.view(B * L, c.hidden).index_select(0, torch.arange(B, device=x.device) * L + seqlens.long() - 1)
        elif last_only:
            x = x.view(B, L, c.hidden)[:, -1].contiguous()
        x = kernels.rmsnorm(x, self.norm_w, c.rms_eps)
        if want == 'hidden':
            return x.view(B, -1, c.hidden)
        if self.lm_head is None:
            raise RuntimeError('this engine was built without lm_head.weight (LlamaModel seam): use want="hidden"')
        rows = x.shape[0]
        # padded row stride keeps the epilogue's 128-bit stores aligned (vocab 32006 is not a multiple of 8)
        buf = torch.empty((rows, self.vocab_pad), dtype=self.dt, device=self.dev)
        dense.linear(x, self.lm_head, out=buf[:, :c.vocab])
        return buf.view(B, rows // B, self.vocab_pad)[:, :, :c.vocab]

    # ------------------------------------------------------------------ whole path
    def plan_boxes(self, bboxes):
        """Host-side packing of the per-sample box lists (the reference does this with torch.cat and
        python loops at layers.py:283-302): returns device tensors so that `forward_device` contains no
        host->device traffic and can be captured in a CUDA graph."""
        if bboxes is None or len(bboxes) == 0:
            return None
        counts = [0 if b is None else int(b.shape[0]) for b in bboxes]
        K = sum(counts)
        offs = torch.tensor([0] + list(torch.tensor(counts).cumsum(0).tolist()), dtype=torch.int32).to(self.dev)
        if K > 0:
            boxes = torch.cat([b.to(self.dev, torch.float32) for b in bboxes if b is not None and b.shape[0]], 0).contiguous()
            bidx = torch.cat([torch.full((n,), float(i)) for i, n in enumerate(counts)]).to(self.dev)
        else:
            boxes = torch.zeros((0, 4), dtype=torch.float32, device=self.dev)
            bidx = torch.zeros((0,), dtype=torch.float32, device=self.dev)
        return dict(K=K, boxes=boxes, bidx=bidx, offs=offs)

    def _region(self, plan, taps):
        """The splice's region argument for a box plan: (region-token rows, per-sample offsets), or None without a plan.
        taps: the ViT hidden states the rows are computed from; None, or a plan without boxes: one zero row."""
        if plan is None:
            return None
        if plan['K'] > 0 and taps is not None:
            maps, ss = self.fuse_maps(taps)
            rows = self.region_tokens(maps, ss, plan['boxes'], plan['bidx'])
        else:
            rows = torch.zeros((1, self.cfg.hidden), dtype=self.dt, device=self.dev)
        return rows, plan['offs']

    def forward_device(self, input_ids, images, plan, validate=True, last_only=False, seqlens=None, cache=None,
                       hidden_taps=None, want='logits', stage_taps=None):
        """Device-only forward (capturable): input_ids int64 [B,L], images bf16 [B,3,S,S] on the GPU.
        images=None: text-only forward (spi_llava.py:47-48 skips the vision branch when no image is given).
        stage_taps: optional dict filled with 'vit_taps', 'region', 'embeds' (parity tests)."""
        c = self.cfg
        B, L = input_ids.shape
        vision = images is not None
        img_rows = region = None
        if vision:
            taps = self.vit(images)
            feat = kernels.cast_tokens_f32_bf16(taps[c.select_index], dtype=self.dt)  # spi_llava.py:68-73 (+ autocast cast, CLS dropped)
            img_rows = dense.linear(feat, self.proj_w, self.proj_b).view(B, c.num_patches, c.hidden)
            region = self._region(plan, taps)
        embeds = splice_region_tokens(input_ids, self.embed, img_rows, region, c.num_patches if vision else 0,
                                      c.im_patch_token, c.im_start_token, c.im_end_token, c.bbox_token,
                                      validate=validate and vision)
        if stage_taps is not None and vision:
            stage_taps['vit_taps'] = [taps[l][:, 1:] for l in c.level_layers]
            stage_taps['region'] = region[0] if (region is not None and plan['K'] > 0) else None
            stage_taps['embeds'] = embeds
        if cache is not None:
            cache.start(L, seqlens, input_ids)
        return self.llama(embeds, B, L, last_only=last_only, seqlens=seqlens, cache=cache, hidden_taps=hidden_taps,
                          want=want)

    def forward(self, input_ids, images, bboxes, validate=True, last_only=False, attention_mask=None,
                hidden_taps=None, want='logits', stage_taps=None, cache=None):
        """Public entry: input_ids int64 [B,L]; images [B,3,S,S]; bboxes list (len B) of [K_i,4]
        normalised xyxy or None (host or device tensors).  Returns logits [B,L,V] (bf16) -- [B,1,V]
        with last_only, taken at each row's last valid position.  attention_mask: None / all-ones, or a 0/1 mask [B,L]
        whose rows are right-padded (the collator's pad_sequence layout, data_modules.py:33-44) or left-padded (HF's
        layout for decoder-only generation).  Left-padded rows are rotated to the right-padded layout for the run and
        the logits rotated back, so they come in the caller's layout; logits at padded positions are don't-care.
        hidden_taps / stage_taps / the cache hold the right-padded layout; the cache also records the token ids, images
        and boxes it was computed from (a later turn reuses it: generate(cache=))."""
        plan = self.plan_boxes(bboxes)
        input_ids, lens, shift = _right_padded(input_ids.to(self.dev, non_blocking=True), attention_mask)
        # a mask, even an all-ones one, gives the cache per-row lengths
        seqlens = None if attention_mask is None else lens.to(torch.int32)
        images = None if images is None else images.to(self.dev, self.dt, non_blocking=True).contiguous()
        out = self.forward_device(input_ids, images, plan, validate, last_only, seqlens, cache=cache,
                                  hidden_taps=hidden_taps, want=want, stage_taps=stage_taps)
        if cache is not None:
            cache.set_source(images, bboxes)
        if shift is not None and not last_only:
            out = from_right_padded(out, shift)
        return out


    # ------------------------------------------------------------------ multi-turn generation
    def extend(self, cache, input_ids, images, bboxes, attention_mask=None, last_only=True):
        """Prefill a chunk that continues the sequences `cache` holds (a later turn of a conversation): input_ids int64
        [B, Lc], right-padded (attention_mask: 0/1 [B, Lc], None: every row has Lc tokens); row b's tokens go to
        positions cache.row_lens()[b] onwards and attend over the cached prefix.  The chunk may hold <bbox> tokens but
        no image tokens; bboxes: per row, the boxes of the chunk's <bbox> tokens (those beyond the boxes already
        cached), whose region tokens come from a ViT + fuse rerun on `images` (only when the chunk holds any).
        Returns logits [B, 1, V] at each row's last chunk token (last_only=False: [B, Lc, V] at every chunk position);
        the cache then holds prefix + chunk and records them.  It grows (zero-filled) when a row's start plus Lc exceeds
        its length, so a CUDA graph captured on it must be rebuilt afterwards.  A row view (cache.rows: rows of a larger
        cache, the continuous batcher's) never grows: each row appends only its valid tokens, which must fit in max_len."""
        c = self.cfg
        if c.head_dim != 128:
            raise NotImplementedError('continuing a cached sequence needs the fused-RoPE QKV GEMM (head_dim 128)')
        ids, lens, shift = _right_padded(input_ids.to(self.dev), attention_mask)
        if shift is not None:
            raise NotImplementedError('extend takes right-padded chunks')
        B, Lc = ids.shape
        valid = lens.to(torch.int32)
        qlen = _seqlens(lens, Lc)
        start = cache.row_lens().clone()
        start_h = start.cpu()
        if cache.rows is None:
            cache.grow(int(start_h.max()) + Lc)   # every row appends all Lc chunk rows, its padding included
        elif bool((start_h + lens.cpu() > cache.max_len).any()):
            raise ValueError('extend: a row view of a larger cache cannot grow: start + chunk length %s exceed max_len %d'
                             % ((start_h + lens.cpu()).tolist(), cache.max_len))
        plan = self.plan_boxes(bboxes)
        taps = None
        if plan is not None and plan['K'] > 0 and bool((ids == c.bbox_token).any()):
            images = images.to(self.dev, self.dt).contiguous()
            taps = self.vit(images)
        region = self._region(plan, taps)   # the splice checks each row's <bbox> count against its boxes (status 3)
        embeds = splice_region_tokens(ids, self.embed, None, region, 0, c.im_patch_token, c.im_start_token,
                                      c.im_end_token, c.bbox_token, validate=True, continuation=True)
        logits = self.llama(embeds, B, Lc, last_only=last_only, seqlens=qlen, cache=cache, start=start)
        # what the cache now holds: the kept boxes of the prefix, then the chunk's
        rec = cache.ids.cpu()
        boxes = []
        for b in range(B):
            n_old = int((rec[b, :int(start_h[b])] == c.bbox_token).sum())
            old = cache.boxes[b] if cache.boxes is not None and cache.boxes[b] is not None else torch.zeros(0, 4)
            new = _row_boxes(bboxes, b, host=True)
            new = torch.zeros(0, 4) if new is None else new
            boxes.append(torch.cat([old[:n_old], new], 0))
        if cache.rows is None:
            cache.record_ids(ids, start)
        else:   # the padding was not appended, and may reach past max_len
            for b, n in enumerate(lens.tolist()):
                cache.ids[b, int(start_h[b]):int(start_h[b]) + n] = ids[b, :n]
        cache.lens = (start + valid).to(torch.int32)
        cache.length = int(cache.lens.max())
        if images is not None:
            cache.images = images.to(self.dev, self.dt).clone()
        cache.boxes = boxes
        cache.source_known = True
        return logits

    def prefill_cached(self, cache, input_ids, images, bboxes, attention_mask=None, new_tokens=0):
        """Prefill a prompt into an existing cache that may hold an earlier turn of the conversation: the prefix it
        already holds (KVCache.reusable) is kept and only the rest is computed (extend) when every row's reusable prefix
        covers its image span; otherwise a full prefill overwrites the cache.  The cache first grows (zero-filled) to
        hold the prompt plus `new_tokens`.  input_ids [B, L] (attention_mask: rows right- or left-padded).
        Returns logits [B, 1, V] at each row's last token."""
        c = self.cfg
        B, L = input_ids.shape
        if B != cache.B:
            raise ValueError('the cache holds %d rows, the prompt has %d' % (cache.B, B))
        ids, lens, _ = _right_padded(input_ids.to(self.dev), attention_mask)
        cache.grow(L + new_tokens)
        reuse = cache.reusable(input_ids, images, bboxes, attention_mask)
        ids_h, lens_h = ids.cpu(), lens.cpu()
        covered = c.head_dim == 128
        for b in range(B):
            covered = covered and covers_image_span(c, ids_h[b, :int(lens_h[b])], int(reuse[b]))
        if not covered:
            images = None if images is None else images.to(self.dev, self.dt).contiguous()
            logits = self.forward_device(ids, images, self.plan_boxes(bboxes), validate=True, last_only=True,
                                         seqlens=_seqlens(lens, L), cache=cache)
            cache.set_source(images, bboxes)
            return logits
        tl = lens_h - reuse
        Lc = int(tl.max())
        tail = torch.zeros((B, Lc), dtype=torch.int64)
        tail_boxes = []
        for b in range(B):
            r = int(reuse[b])
            tail[b, :int(tl[b])] = ids_h[b, r:int(lens_h[b])]
            n_old = int((ids_h[b, :r] == c.bbox_token).sum())
            row = _row_boxes(bboxes, b)
            tail_boxes.append(None if row is None else row[n_old:])
        mask = (torch.arange(Lc)[None] < tl[:, None]).long()
        cache.lens = reuse.to(self.dev, torch.int32)
        cache.length = int(reuse.max())
        return self.extend(cache, tail, images, tail_boxes, attention_mask=mask)


def covers_image_span(cfg, ids, p):
    """Whether a kept prefix of p tokens of the prompt `ids` (host int64 [L]) holds all its image tokens: a later chunk
    (extend) takes no image tokens, so a prefix is reusable only when this holds."""
    span = ((ids == cfg.im_patch_token) | (ids == cfg.im_start_token) | (ids == cfg.im_end_token)).nonzero()
    return len(span) == 0 or int(span.max()) < p


def same_image(held, image):
    """Whether K/V computed from the image `held` ([3, S, S], None: text-only) can serve a prompt on `image` (the same
    image, compared in held's device and dtype; or both None)."""
    if held is None or image is None:
        return held is None and image is None
    return torch.equal(held, image.to(held.device, held.dtype))


def reusable_prefix(cfg, row, rec, held, old_boxes, new_boxes):
    """KVCache.reusable's rule for one row: how many leading tokens of `row` (host int64 [n], the new prompt) a cache row
    holding the ids `rec` (host int64, at least `held` entries) at its first `held` positions, computed with the boxes
    old_boxes (host fp32 [K, 4] or None) for its <bbox> tokens, can keep for a prompt whose boxes are new_boxes: the
    longest common prefix, cut at the first <bbox> whose box differs, and at most n - 1 (the image is checked by the
    caller)."""
    n = row.shape[0]
    m = min(n - 1, int(held))
    diff = (row[:m] != rec[:m]).nonzero()
    p = int(diff[0]) if len(diff) else m
    for k, t in enumerate((row[:p] == cfg.bbox_token).nonzero().flatten().tolist()):
        if old_boxes is None or new_boxes is None or k >= old_boxes.shape[0] or k >= new_boxes.shape[0] \
                or not torch.equal(old_boxes[k], new_boxes[k]):
            p = t
            break
    return max(p, 0)


def _row_boxes(bboxes, b, host=False):
    """Row b's boxes of a per-row box list, or None (bboxes None or empty, as plan_boxes takes them: no boxes).
    host: as a host fp32 tensor of its own."""
    row = None if bboxes is None or len(bboxes) == 0 else bboxes[b]
    return row.detach().to('cpu', torch.float32, copy=True) if host and row is not None else row


def right_pad_layout(attention_mask):
    """0/1 mask [B, L] whose rows are each right- or left-padded -> (lens, shift), int64 [B] on the mask's device:
    row b's tokens are columns shift[b] .. shift[b] + lens[b] - 1 (shift 0: right-padded, L - lens[b]: left-padded).
    Any other layout (holes, padding on both sides, an empty row) raises NotImplementedError."""
    m = attention_mask.to(torch.int64)
    B, L = m.shape
    lens = m.sum(1)
    shift = m.argmax(1)                      # first 1 of the row
    col = torch.arange(L, device=m.device)[None]
    want = (col >= shift[:, None]) & (col < (shift + lens)[:, None])
    ok = (m == want.to(torch.int64)).all(1) & (lens > 0) & ((shift == 0) | (shift + lens == L))
    if not bool(ok.all()):
        raise NotImplementedError('attention_mask rows must be right- or left-padded runs of ones (rows %s are not)'
                                  % (~ok).nonzero().flatten().tolist())
    return lens, shift


def _right_padded(x, attention_mask):
    """x [B, L, ...] with its 0/1 attention_mask [B, L] (None: every row has L entries) -> (x in the right-padded
    layout the engine runs on, on x's device and contiguous; lens int64 [B]; shift as right_pad_layout gives it, None
    when no row is left-padded and x is as given)."""
    B, L = x.shape[:2]
    if attention_mask is None:
        return x.contiguous(), torch.full((B,), L, dtype=torch.int64, device=x.device), None
    lens, shift = right_pad_layout(attention_mask.to(x.device))
    if not bool(shift.any()):
        return x.contiguous(), lens, None
    return to_right_padded(x, shift), lens, shift


def _seqlens(lens, L):
    """lens int64 [B] -> the int32 seqlens of a prefill, None when every row has all L entries."""
    return None if bool((lens == L).all()) else lens.to(torch.int32)


def _rotate(x, shift):
    B, L = x.shape[:2]
    idx = (torch.arange(L, device=x.device)[None] + shift.to(x.device)[:, None]) % L
    return x.gather(1, idx.view(B, L, *([1] * (x.dim() - 2))).expand(x.shape))


def to_right_padded(x, shift):
    """[B, L, ...] in the caller's layout -> right-padded layout: row b rotated left by shift[b] (right_pad_layout)."""
    return _rotate(x, shift)


def from_right_padded(x, shift):
    """Inverse of to_right_padded."""
    return _rotate(x, (x.shape[1] - shift) % x.shape[1])


_DECODE_FUSED = int(os.environ.get('G4R_DECODE_FUSED', '1'))


class KVCache:
    """Per-layer K/V cache [B, Lmax, n_heads*head_dim] (the engine's 16-bit type, post-RoPE keys) for the decode loop.
    length: columns in use (padded prompt length + decode steps).  lens: None when every sample uses all `length`
    columns, else a device int32 [B] with each sample's own length (a right-padded batch of prompts of different
    lengths): sample b's next token sits at position lens[b] and attends over columns 0..lens[b].

    For multi-turn generation the cache also records what its K/V were computed from, so that a later turn can reuse
    them (reusable, generate(cache=)): `ids` (int64 [B, Lmax], on the cache's device) holds the token id at every
    position whose K/V the same write filled, -1 elsewhere; `images` the rows' images (None: text-only) and `boxes`
    each row's boxes (host fp32 [K, 4] or None) for its <bbox> tokens.  Until a writer records the images and boxes
    (`source_known`), nothing is reusable.
    The K/V tensors are zero-filled, and grow() zero-fills the new space: the chunk attention (kernels.attention_cached)
    reads cache rows past each row's valid length, up to the next multiple of 64, and needs them finite.
    A row view (`rows`) is a cache whose B rows are rows rows[b] of larger K/V tensors (the continuous batcher's): the
    chunk prefill (PrefillEngine.extend) reads and appends through that table, and the view cannot grow."""

    def __init__(self, cfg, B, max_len, device, kv=None, rows=None):
        """kv: optional (k, v) lists of per-layer [B, max_len, HD] tensors to use instead of allocating (BeamCache's
        prompt rows).  rows: with kv, a device int32 [B] table -- the kv tensors are [R, max_len, HD] with any R, and
        row b of this cache is row rows[b] of theirs."""
        hd = cfg.n_heads * cfg.head_dim
        dt = cfg.torch_dtype
        self.cfg = cfg
        if kv is not None:
            self.k, self.v = list(kv[0]), list(kv[1])
        else:
            self.k = [torch.zeros((B, max_len, hd), dtype=dt, device=device) for _ in range(cfg.n_layers)]
            self.v = [torch.zeros((B, max_len, hd), dtype=dt, device=device) for _ in range(cfg.n_layers)]
        if rows is not None and (kv is None or rows.dtype != torch.int32 or tuple(rows.shape) != (B,)):
            raise ValueError('KVCache: rows must be a device int32 [%d] table over given kv tensors' % B)
        self.rows = rows
        self.ids = torch.full((B, max_len), -1, dtype=torch.int64, device=device)
        self.B, self.max_len, self.length = B, max_len, 0
        self.lens = None
        self.images, self.boxes, self.source_known = None, None, False

    def start(self, L, seqlens=None, ids=None):
        """A prefill of L columns fills the cache; seqlens (device int32 [B]): the valid length of each row; ids (int64
        [B, L], right-padded layout): the token ids it was computed from (None: unknown, e.g. a prefill from embeddings).
        The images and boxes are unknown until set_source."""
        self.length = L
        self.lens = None if seqlens is None else seqlens.to(torch.int32).clone()
        self.ids.fill_(-1)
        if ids is not None:
            self.ids[:, :L] = ids
        self.source_known = False

    def set_source(self, images, bboxes):
        """Record the images [B, 3, S, S] (None: text-only) and per-row box lists the cached K/V were computed from."""
        self.images = None if images is None else images.detach().clone()
        self.boxes = [_row_boxes(bboxes, b, host=True) for b in range(self.B)]
        self.source_known = True

    def row_lens(self):
        """Each row's valid length, device int32 [B]."""
        if self.lens is not None:
            return self.lens
        return torch.full((self.B,), self.length, dtype=torch.int32, device=self.ids.device)

    def record_ids(self, tokens, pos):
        """tokens int64 [B, n] whose K/V were written at positions pos[b] .. pos[b] + n - 1 (pos: int32 [B])."""
        idx = pos.to(self.ids.device, torch.int64)[:, None] + torch.arange(tokens.shape[1], device=self.ids.device)[None]
        self.ids.scatter_(1, idx, tokens.to(self.ids.device, torch.int64))

    def grow(self, max_len):
        """Enlarge to max_len positions, keeping the contents; the new space is zero-filled (ids: -1).  The K/V tensors
        are replaced, so a CUDA graph captured on the old ones must be rebuilt."""
        if max_len <= self.max_len:
            return
        if self.rows is not None:
            raise ValueError('a row view of a larger cache cannot grow (max_len %d, %d asked)' % (self.max_len, max_len))

        def big(t, fill):
            n = torch.full((t.shape[0], max_len) + tuple(t.shape[2:]), fill, dtype=t.dtype, device=t.device)
            n[:, :self.max_len] = t
            return n
        for kv in (self.k, self.v):
            for i in range(len(kv)):
                kv[i] = big(kv[i], 0)
        self.ids = big(self.ids, -1)
        self.max_len = max_len

    def crop(self, n):
        """Keep the first n positions (transformers' DynamicCache.crop, which assisted decoding calls after every verify
        step): lengths only -- the K/V past n stay in memory but become unreachable, later writes overwrite them, and
        their recorded ids are cleared so that reusable() stops at n.  The tensors are not replaced, so a CUDA graph
        captured on the cache stays valid."""
        n = max(int(n), 0)
        if n >= self.length and self.lens is None:
            return
        self.length = min(self.length, n)
        if self.lens is not None:
            self.lens.clamp_(max=n)
        self.ids[:, n:] = -1

    def _same_image(self, b, images):
        return same_image(None if self.images is None else self.images[b], None if images is None else images[b])

    def reusable(self, input_ids, images, bboxes, attention_mask=None):
        """How many leading tokens of each row of a new prompt the cache already holds, as a host int64 [B]: the longest
        prefix of the row's tokens (unpadded: attention_mask rows right- or left-padded) equal to the recorded ids,
        cut at the first <bbox> whose box differs from the recorded one, 0 when the row's image differs, and at most
        len - 1 so that at least the last token is computed and gives logits."""
        B = input_ids.shape[0]
        out = torch.zeros(B, dtype=torch.int64)
        if B != self.B or not self.source_known:
            return out
        ids, lens, _ = _right_padded(input_ids.cpu(), attention_mask)
        held = self.row_lens().cpu()
        rec = self.ids.cpu()
        for b in range(B):
            if not self._same_image(b, images):
                continue
            out[b] = reusable_prefix(self.cfg, ids[b, :int(lens[b])], rec[b], held[b], self.boxes[b],
                                     _row_boxes(bboxes, b, host=True))
        return out


def _decode_step(self, token_ids, cache, pos_dev=None):
    """One decode step (SURVEY.md 8(f1)): token_ids int64 [B,1] -> logits [B,1,V]; the vision / SPI branch
    is skipped exactly as the reference does for input_ids.shape[1] == 1 (spi_llava.py:47-48).
    pos_dev: optional device int32 holding the current length (CUDA-graph replay: the kernels read the
    position from memory instead of from a launch argument).
    On a cache with per-sample lengths (cache.lens) every kernel takes sample b's position from cache.lens[b], which
    the step advances on the device -- except under graph capture (pos_dev given), where GraphedDecode.step does."""
    if cache.length + 1 > cache.max_len:
        raise RuntimeError('KV cache is full (%d)' % cache.max_len)
    # every kernel of the step only READS weights: let each one start in its predecessor's tail and fetch its first
    # weight block before it waits for the predecessor (programmatic dependent launch, csrc/common.cuh)
    prev = lib.set_pdl(True)
    try:
        return _decode_step_chain(self, token_ids, cache, pos_dev)
    finally:
        lib.set_pdl(prev)


def _decode_step_chain(self, token_ids, cache, pos_dev):
    c = self.cfg
    B = token_ids.shape[0]
    pos = cache.length
    kv_len = cache.max_len if pos_dev is not None else pos + 1   # sizes the score buffer when device-driven
    rows = cache.lens        # per-sample positions (<= pos): these override pos / pos_dev in every kernel
    anc = getattr(cache, 'anc', None)   # a BeamCache: attention through its ancestry table, positions set by beam_step
    x = splice_region_tokens(token_ids, self.embed, None, None, 0, c.im_patch_token, c.im_start_token,
                             c.im_end_token, c.bbox_token, validate=False).view(B, c.hidden)
    cos, sin = self._rope_span(cache.max_len)
    scale = c.head_dim ** -0.5
    fused = c.head_dim == 128 and (2 * c.hidden) % 256 == 0
    # KV-cache append folded into the q|k|v GEMM's RoPE epilogue (7 launches per layer instead of 8).
    # G4R_DECODE_FUSED=0: the unfused sequence, which B > 16 and head_dim != 128 run anyway.
    fuse_step = fused and B <= 16 and c.hidden % 256 == 0 and _DECODE_FUSED > 0
    swiglu_gemm = dense.decode_gemm if fuse_step else dense.linear
    for li, w in enumerate(self.layers):
        h = kernels.rmsnorm(x, w['ln_in'], c.rms_eps)
        if fuse_step:
            qkv = dense.decode_gemm(h, w['wqkv'], rope=(cos, sin, 2 * c.hidden, pos, pos_dev), kv=(cache.k[li], cache.v[li]),
                                    pos_rows=rows)
        elif fused:
            qkv = dense.qkv_rope(h, w['wqkv'], cos, sin, 1, 2 * c.hidden, pos0=pos, pos_dev=pos_dev, pos_rows=rows)
        else:
            if pos_dev is not None:
                raise NotImplementedError('graph decode needs the fused-RoPE QKV GEMM (head_dim 128)')
            if rows is not None:
                raise NotImplementedError('prompts of different lengths need the fused-RoPE QKV GEMM (head_dim 128)')
            qkv = dense.linear(h, w['wqkv'])
            kernels.rope_inplace(qkv, cos[pos:pos + 1].contiguous(), sin[pos:pos + 1].contiguous(), 1, 2 * c.n_heads, c.head_dim)
        if not fuse_step:
            kernels.kv_append(qkv, cache.k[li], cache.v[li], B, 1, pos, pos_dev, pos_rows=rows)
        a = _decode_attention(cache, li, qkv, kv_len, scale, pos_dev, rows, anc)
        x = dense.linear(a, w['wo'], residual=x)
        h = kernels.rmsnorm(x, w['ln_post'], c.rms_eps)
        f = swiglu_gemm(h, w['wgu'], act='swiglu')
        x = dense.linear(f, w['wdown'], residual=x)
    cache.length = pos + 1
    if rows is not None and pos_dev is None and anc is None:
        rows.add_(1)
    x = kernels.rmsnorm(x, self.norm_w, c.rms_eps)
    buf = torch.empty((B, self.vocab_pad), dtype=self.dt, device=self.dev)
    dense.linear(x, self.lm_head, out=buf[:, :c.vocab])
    return buf[:, None, :c.vocab]


def _verify_step(self, token_ids, cache, st):
    """The verify step of prompt-lookup decoding: the decode chain over the M <= st.k + 1 rows token_ids (int64 [M, 1])
    of one sequence held in cache row 0, row i at position st.pos[i] (device int32, consecutive from st.base[0]).
    Each row's K/V is written at its position (qkv_rope with the per-sample base, then kv_append: the rows are one
    sample of M rows), and row i attends over positions 0..st.pos[i] (decode_attention_beam with the all-zero ancestry
    table st.anc[:M] (int32 [>= M, max_len]): a causal M-query attention over cache row 0).  Returns logits [M, 1, V].  M <= 16 runs
    the weight-streaming decode GEMMs, a larger M the tiled ones.  Every position is read from device memory, so the
    step can be captured (LookupDecode)."""
    prev = lib.set_pdl(True)
    try:
        c = self.cfg
        M = token_ids.shape[0]
        x = splice_region_tokens(token_ids, self.embed, None, None, 0, c.im_patch_token, c.im_start_token,
                                 c.im_end_token, c.bbox_token, validate=False).view(M, c.hidden)
        cos, sin = self._rope_span(cache.max_len)
        scale = c.head_dim ** -0.5
        swiglu_gemm = dense.decode_gemm if M <= 16 and c.hidden % 256 == 0 else dense.linear
        for li, w in enumerate(self.layers):
            h = kernels.rmsnorm(x, w['ln_in'], c.rms_eps)
            qkv = dense.qkv_rope(h, w['wqkv'], cos, sin, M, 2 * c.hidden, pos_rows=st.base)
            kernels.kv_append(qkv, cache.k[li], cache.v[li], 1, M, 0, pos_rows=st.base)
            a = kernels.decode_attention_beam(qkv, cache.k[li], cache.v[li], M, c.n_heads, c.head_dim, cache.max_len,
                                              scale, st.pos[:M], st.anc[:M])
            x = dense.linear(a, w['wo'], residual=x)
            h = kernels.rmsnorm(x, w['ln_post'], c.rms_eps)
            f = swiglu_gemm(h, w['wgu'], act='swiglu')
            x = dense.linear(f, w['wdown'], residual=x)
        x = kernels.rmsnorm(x, self.norm_w, c.rms_eps)
        buf = torch.empty((M, self.vocab_pad), dtype=self.dt, device=self.dev)
        dense.linear(x, self.lm_head, out=buf[:, :c.vocab])
        return buf[:, None, :c.vocab]
    finally:
        lib.set_pdl(prev)


def _decode_attention(cache, li, qkv, kv_len, scale, pos_dev, rows, anc):
    c = cache.cfg
    if isinstance(cache, SampleCache):   # N rows per prompt: the prompt's keys read once for all of them
        return kernels.decode_attention_group(qkv, cache.full_k[li], cache.full_v[li], cache.n_samples, cache.N,
                                              c.n_heads, c.head_dim, cache.prompt_len, cache.G, scale,
                                              cache.prompt_lens, rows)
    if anc is None:
        return kernels.decode_attention(qkv, cache.k[li], cache.v[li], qkv.shape[0], c.n_heads, c.head_dim, kv_len, scale,
                                        pos_dev, pos_rows=rows)
    return kernels.decode_attention_beam(qkv, cache.full_k[li], cache.full_v[li], qkv.shape[0], c.n_heads, c.head_dim,
                                         kv_len, scale, rows, anc)


STOP_TABLE_MAX_BYTES = 64 << 20
_STOP_TABLES = collections.OrderedDict()   # (token strings, stop strings, stop token ids) -> host table; the last 8 used


def _stop_lookup(table, tokens, state):
    """kernels.stop_step's lookup with torch indexing: tokens, state int64 [n] -> (new state int64 [n], hit bool [n])."""
    V = table.shape[0] - 1
    e = table[torch.where((tokens < 0) | (tokens > V), V, tokens), state].to(torch.int64)
    return e & 0x7FFF, e < 0


class StopStrings:
    """The stop strings of a generate call as a lookup table (transformers' StopStringCriteria as a state machine): a
    row stops at the first generated token in which an occurrence of a stop string ends, in the concatenation of the
    tokens' strings -- the occurrence may begin in earlier tokens and the last token may run past its end.

    token_strings: the string every token id stands for (StopStringCriteria.clean_tokenizer_vocab), a list indexed by
    id, None for ids the vocabulary does not hold.  stop_token_ids: ids that stop a row by themselves
    (KeywordsStoppingCriteria.keyword_ids).

    The matcher is the Aho-Corasick automaton of the stop strings over their own characters plus one class for every
    other character: states = trie nodes (S <= 1 + sum of the lengths), failure links and output sets folded into a
    dense transition table.  `table` (host int16 [V_tok + 1, S]) composes it with the tokens: entry (t, s) is the
    state after token t's string is fed from state s, bit 15 set when an accepting state was entered on the way.  An id
    the vocabulary does not hold, and the last row (where ids >= V_tok go), sends every state to the root without a hit,
    as HF's matcher breaks a match there.  An empty string leaves the state as it is, as HF's does -- with one
    difference: HF looks at the last max(len(stop)) tokens only, so a match that empty-string tokens stretch over more
    tokens than that is found here and missed there.
    kernels.stop_step walks the table on the device (Sampler); initial_states() gives each row's state after its
    prompt."""

    def __init__(self, token_strings, stop_strings, stop_token_ids=()):
        stops = (stop_strings,) if isinstance(stop_strings, str) else tuple(stop_strings)
        if not stops:
            raise ValueError('stop_strings: no stop string given')
        if not all(isinstance(s, str) and s for s in stops):
            raise ValueError('stop_strings: every stop string must be a non-empty str, got %r' % (stops,))
        self.stop_strings = stops
        self.max_len = max(len(s) for s in stops)
        self.V_tok = len(token_strings)
        key = (tuple(token_strings), stops, tuple(int(t) for t in stop_token_ids))
        if key in _STOP_TABLES:
            _STOP_TABLES.move_to_end(key)
        else:
            _STOP_TABLES[key] = self._build(*key)
            if len(_STOP_TABLES) > 8:
                _STOP_TABLES.popitem(last=False)
        self.table = _STOP_TABLES[key]
        self.S = self.table.shape[1]
        self._device = {}

    @staticmethod
    def _automaton(stops):
        """-> (delta int64 [S, A], accept bool [S], code: character -> column of delta; column 0: any other character)."""
        code = {ch: i + 1 for i, ch in enumerate(sorted(set(''.join(stops))))}
        goto, accept = [{}], [False]
        for s in stops:
            n = 0
            for ch in s:
                if code[ch] not in goto[n]:
                    goto[n][code[ch]] = len(goto)
                    goto.append({})
                    accept.append(False)
                n = goto[n][code[ch]]
            accept[n] = True
        S, A = len(goto), len(code) + 1
        delta = torch.zeros((S, A), dtype=torch.int64)
        fail = [0] * S
        order = [0]
        for n in order:                          # breadth first: a node's failure state is finished before the node
            accept[n] = accept[n] or accept[fail[n]]
            delta[n] = delta[fail[n]] if n else 0
            for c, m in goto[n].items():
                fail[m] = int(delta[fail[n], c]) if n else 0
                delta[n, c] = m
                order.append(m)
        return delta, torch.tensor(accept), code

    @classmethod
    def _build(cls, token_strings, stops, stop_token_ids):
        V = len(token_strings)
        delta, accept, code = cls._automaton(stops)
        S = delta.shape[0]
        if V == 0 or S > 32767 or S * (V + 1) * 2 > STOP_TABLE_MAX_BYTES:
            raise ValueError('stop_strings: %d matcher states x %d tokens need a %d-byte table; the limit is %d bytes '
                             'and 32767 states' % (S, V, S * (V + 1) * 2, STOP_TABLE_MAX_BYTES))
        known = torch.tensor([t is not None for t in token_strings])
        lens = torch.tensor([len(t or '') for t in token_strings])
        chars = torch.zeros((V, max(int(lens.max()), 1)), dtype=torch.int64)
        for i, t in enumerate(token_strings):
            if t and any(ch in code for ch in t):
                chars[i, :len(t)] = torch.tensor([code.get(ch, 0) for ch in t])
        cur = torch.arange(S).repeat(V, 1)
        hit = torch.zeros((V, S), dtype=torch.bool)
        for p in range(chars.shape[1]):          # all (token, state) pairs at once, one character position per pass
            live = (lens > p)[:, None]
            nxt = delta[cur, chars[:, p, None]]
            cur = torch.where(live, nxt, cur)
            hit |= live & accept[nxt]
        if not bool(hit.any()):                  # StopStringCriteria refuses the same
            raise ValueError('stop_strings: no token of the vocabulary can end any of %r (characters the vocabulary '
                             'does not hold?)' % (stops,))
        cur[~known] = 0
        for t in stop_token_ids:
            if not 0 <= t < V:
                raise ValueError('stop_token_ids: %d is outside the vocabulary (%d tokens)' % (t, V))
            cur[t], hit[t] = 0, True
        table = torch.zeros((V + 1, S), dtype=torch.int16)
        table[:V] = (cur - 32768 * hit.to(torch.int64)).to(torch.int16)
        return table

    def on(self, device):
        """The table on `device` (copied once per device)."""
        device = torch.device(device)
        if device.type == 'cpu':
            return self.table
        if device not in self._device:
            self._device[device] = self.table.to(device)
        return self._device[device]

    def advance(self, tokens, state):
        """One lookup on the host: tokens, state int64 [n] -> (new state int64 [n], hit bool [n])."""
        return _stop_lookup(self.table, tokens, state)

    def initial_states(self, ids, lens):
        """Each row's state after its prompt, int32 [B] on the host: the table walked (hits ignored) over the last
        max(len(stop)) of the row's lens[b] tokens, ids[b, :lens[b]] -- which is what lets a stop string begin in the
        prompt and end in the answer."""
        ids, lens = ids.cpu(), lens.cpu().to(torch.int64)
        state = torch.zeros(ids.shape[0], dtype=torch.int64)
        for k in range(self.max_len, 0, -1):
            col = lens - k
            new, _ = self.advance(ids.gather(1, col.clamp(min=0)[:, None])[:, 0], state)
            state = torch.where(col >= 0, new, state)
        return state.to(torch.int32)


class LogitsProcessors:
    """transformers' history-dependent logits processors for one decode loop, in HF's order: RepetitionPenalty-
    (repetition_penalty != 1), NoRepeatNGram- (no_repeat_ngram_size > 0), MinLength- and MinNewTokensLengthLogitsProcessor
    (min_length / min_new_tokens > 0, suppressing `eos_ids`).  history: int64 [R, ld_h] -- row r's prompt as given (pads
    included), then the tokens selected so far; the selection of new token s reads history[r, :L + s] and writes the
    token it selects to history[r, L + s] (kernels.sample_tokens_processed), so the loop's output buffer serves."""

    def __init__(self, history, L, repetition_penalty=1.0, no_repeat_ngram_size=0, min_length=0, min_new_tokens=0,
                 eos_ids=()):
        self.history, self.L = history, int(L)
        self.repetition_penalty = 1.0 if repetition_penalty is None else float(repetition_penalty)
        self.no_repeat_ngram_size = int(no_repeat_ngram_size or 0)
        self.min_length, self.min_new_tokens = int(min_length or 0), int(min_new_tokens or 0)
        self.eos_list = [int(e) for e in eos_ids]
        self.eos_ids = (torch.tensor(self.eos_list, dtype=torch.int32, device=history.device) if self.eos_list
                        else None)

    @staticmethod
    def neutral(repetition_penalty=1.0, no_repeat_ngram_size=0, min_length=0, min_new_tokens=0, eos_ids=()):
        """True when none of the four would change a score (HF then builds none of them)."""
        return ((repetition_penalty is None or float(repetition_penalty) == 1.0) and not no_repeat_ngram_size
                and not ((min_length or min_new_tokens) and len(eos_ids)))

    def apply(self, scores, step):
        """The four processors restated with torch on fp32 scores [R, V] at new token `step` (the host stand-in path)."""
        h = self.history[:, :self.L + step].to(scores.device)
        Lh = h.shape[1]
        p = self.repetition_penalty
        if p != 1.0 and Lh:
            x = scores.gather(1, h)
            scores = scores.scatter(1, h, torch.where(x < 0, x * p, x / p))
        n = self.no_repeat_ngram_size
        if n > 0 and Lh + 1 >= n:
            scores = scores.clone()
            for r, row in enumerate(h.tolist()):
                tail = row[Lh - n + 1:]
                banned = sorted({row[j + n - 1] for j in range(Lh - n + 1) if row[j:j + n - 1] == tail})
                scores[r, banned] = float('-inf')
        if self.eos_list and (Lh < self.min_length or step < self.min_new_tokens):
            scores = scores.clone()
            scores[:, self.eos_list] = float('-inf')
        return scores

    def append(self, tok, step):
        if self.L + step < self.history.shape[1]:
            self.history[:, self.L + step] = tok.view(-1).to(self.history.device)


class Sampler:
    """Next-token selection of the decode loop (kernels.sample_tokens): arg-max, or a draw from the temperature /
    top-k / top-p processed softmax, with transformers' eos -> pad rule when eos_id and pad_id are both given.
    Its per-step state lives on the device, so a CUDA graph can capture the call: `rng_step` (int64 [1], the Philox
    counter, advanced once per selected token) and `finished` (int32 [B], the rows that have emitted eos_id).
    stops (a StopStrings, with stop_state: each row's state after its prompt, int32 [B]): every call then ends with
    kernels.stop_step on the tokens just selected, which keeps the rows' matcher states in `stop_state` and sets
    `finished` for a row whose token ends a stop string.
    processors (a LogitsProcessors): the selection runs on the scores its processors leave, reading each row's history
    at length L + rng_step and appending the selected token to it (kernels.sample_tokens_processed).
    scores / logits (fp32 [n_slots, B, V], either may be None): every call also writes transformers'
    next_token_scores / next_token_logits of its rows into slot rng_step (kernels.sample_tokens_out); without them it
    launches exactly what it launches otherwise."""

    def __init__(self, B, device, greedy=True, temperature=1.0, top_k=None, top_p=None, seed=0, eos_id=None,
                 pad_id=None, stops=None, stop_state=None, processors=None, scores=None, logits=None):
        self.greedy = bool(greedy)
        self.temperature = float(temperature)
        self.top_k = 0 if top_k is None else int(top_k)
        self.top_p = 1.0 if top_p is None else float(top_p)
        self.seed = int(seed)
        rule = eos_id is not None and pad_id is not None
        self.eos_id, self.pad_id = (int(eos_id), int(pad_id)) if rule else (-1, -1)
        self.rng_step = torch.zeros(1, dtype=torch.int64, device=device)
        self.finished = torch.zeros(B, dtype=torch.int32, device=device)
        self.stop_table = None if stops is None else stops.on(device)
        if stops is not None:
            self.stop_state = torch.zeros_like(self.finished) if stop_state is None else stop_state.to(device, torch.int32)
        self.processors = processors
        self.out_scores, self.out_logits = scores, logits

    def __call__(self, logits, out, update=True):
        """Select from logits [B, 1, V] into out (int64 [B, 1]).  update=False leaves `finished`, `stop_state` and the
        processors' history alone (warm-up: the stop-string lookup then runs on copies, so that a graph capture is not
        its first launch)."""
        if not logits.is_cuda:
            return self._host(logits, out, update)
        pr = self.processors
        if self.out_scores is not None or self.out_logits is not None:
            proc = {} if pr is None else dict(
                history=pr.history, L=pr.L, repetition_penalty=pr.repetition_penalty,
                no_repeat_ngram_size=pr.no_repeat_ngram_size, min_length=pr.min_length,
                min_new_tokens=pr.min_new_tokens, eos_ids=pr.eos_ids, append=update)
            kernels.sample_tokens_out(logits, out, self.greedy, self.temperature, self.top_k, self.top_p, self.seed,
                                      self.rng_step, self.eos_id, self.pad_id, self.finished if update else None,
                                      scores=self.out_scores, raw_logits=self.out_logits, **proc)
        elif pr is None:
            kernels.sample_tokens(logits, out, self.greedy, self.temperature, self.top_k, self.top_p, self.seed,
                                  self.rng_step, self.eos_id, self.pad_id, self.finished if update else None)
        else:
            kernels.sample_tokens_processed(
                logits, out, self.greedy, self.temperature, self.top_k, self.top_p, self.seed, self.rng_step,
                self.eos_id, self.pad_id, self.finished if update else None, history=pr.history, L=pr.L,
                repetition_penalty=pr.repetition_penalty, no_repeat_ngram_size=pr.no_repeat_ngram_size,
                min_length=pr.min_length, min_new_tokens=pr.min_new_tokens, eos_ids=pr.eos_ids, append=update)
        if self.stop_table is not None:
            state, finished = (self.stop_state, self.finished) if update else (self.stop_state.clone(), self.finished.clone())
            kernels.stop_step(out, self.stop_table, state, finished)
        return out

    def _host(self, logits, out, update):
        """Host tensors come only from CPU stand-ins of the engine (the loop's host-side tests): the arg-max (of the
        processed fp32 scores with processors), the output slots, the eos -> pad rule and the history append, restated.
        Sampling exists on the device only."""
        if not self.greedy:
            raise RuntimeError('token sampling runs on the CUDA device only (csrc/sample.cu): logits are on %s'
                               % logits.device)
        scores = logits.reshape(logits.shape[0], -1)
        if self.processors is not None:
            scores = self.processors.apply(scores.float(), int(self.rng_step))
        slot = int(self.rng_step)
        for buf, val in ((self.out_scores, scores), (self.out_logits, logits)):
            if buf is not None and slot < buf.shape[0]:
                buf[slot].copy_(val.reshape(buf.shape[1:]))
        tok = scores.argmax(-1)
        if update and self.eos_id >= 0:
            tok = torch.where(self.finished.bool(), torch.full_like(tok, self.pad_id), tok)
            self.finished |= (tok == self.eos_id).to(torch.int32)
        if update and self.stop_table is not None:
            live = self.finished == 0
            state, hit = _stop_lookup(self.stop_table, tok, self.stop_state.to(torch.int64))
            self.stop_state = torch.where(live, state.to(torch.int32), self.stop_state)
            self.finished |= (live & hit).to(torch.int32)
        if update and self.processors is not None:
            self.processors.append(tok, int(self.rng_step))
        out.copy_(tok.view(out.shape))
        return out

    def advance(self):
        self.rng_step.add_(1)


def sampling_seed(generator=None):
    """The Philox key of one generate call, drawn from `generator` (default: torch's default CPU generator), so that
    torch.manual_seed makes sampling reproducible."""
    dev = generator.device if generator is not None else 'cpu'
    return int(torch.randint(0, 2 ** 62, (1,), generator=generator, device=dev).item())


@torch.no_grad()
def _generate(self, input_ids, images, bboxes, max_new_tokens=32, do_sample=False, temperature=1.0,
              stopping_criteria=None, eos_token_id=None, generator=None, use_graph=True, attention_mask=None,
              pad_token_id=None, cache=None, top_k=None, top_p=None, num_beams=1, length_penalty=1.0,
              early_stopping=False, num_return_sequences=1, stop_strings=None, repetition_penalty=1.0,
              no_repeat_ngram_size=0, min_length=0, min_new_tokens=0, length_eos_ids=None, output_scores=False,
              output_logits=False, return_dict_in_generate=False, prompt_lookup_num_tokens=None,
              max_matching_ngram_size=None, streamer=None):
    """Prefill + greedy / sampled decode (gpt4roi/app.py:286-300 calls
    model.generate(input_ids, images=..., do_sample=True, temperature=0.2, max_new_tokens=1024,
    stopping_criteria=[...]) with the boxes bound to forward).  Returns ids [B, L + new]: the prompt as given,
    then the new tokens (HF's layout).
    do_sample with temperature > 0: every token is drawn on the device (Sampler) from softmax(logits / temperature),
    restricted to the top_k largest values (None / 0: all) and then to the top_p nucleus (None / 1: all), as
    transformers' TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper; the draws are keyed by a seed taken
    from `generator` (default: torch's default generator).  Otherwise the arg-max.
    attention_mask: 0/1 [B, L] for a batch of prompts of different lengths, each row right- or left-padded; the
    prefill runs on the right-padded layout and every sample continues from its own last token.
    pad_token_id (with eos_token_id): a sample that has emitted eos_token_id gets pad_token_id from then on and the
    loop ends once every sample has (transformers' GenerationMixin rule); without it the loop ends when all samples
    emit eos_token_id at the same step.
    cache: a KVCache to generate into -- a conversation's earlier turns (gpt4roi/app.py re-submits the whole
    conversation every turn): the prefix it already holds is reused and only the rest is prefilled (prefill_cached);
    afterwards it holds the conversation including this turn's answer (the last new token excepted), ready for the next.
    Rows that finished with pad_token_id keep those pads in the recorded ids, so the next turn's reuse stops there.
    stop_strings: a StopStrings -- transformers' generate(stop_strings=...), matched on the device per row: a row is
    finished at the first new token in which a stop string ends (it may begin in the row's prompt), that token is part
    of the output, and the loop ends once every row is finished.  As in HF, finished rows are filled with pad_token_id
    only when eos_token_id and pad_token_id are both given; otherwise they keep generating until the last row stops.
    Host stopping_criteria callbacks may be given as well.
    num_beams > 1: deterministic beam search (transformers' GenerationMixin._beam_search, do_sample=False) with
    length_penalty, early_stopping (True, False or "never") and num_return_sequences <= num_beams; eos_token_id may be
    a list.  The prompt is prefilled once per sample and the beams share its KV cache (BeamCache).  Returns
    [B * num_return_sequences, L + n] as HF crops it.
    num_return_sequences = N > 1 with sampling (num_beams 1): N independent answers per prompt, as HF's _sample
    returns them after expanding the inputs -- [B * N, L + n], row b*N + i is sample i of prompt b, each row with its
    own tokens, eos -> pad rule, stop-string state and finished flag; host stopping_criteria see all B * N rows.  Row r
    draws with Philox counter (step, r), so the result is that of this loop on input_ids.repeat_interleave(N, 0) with
    the same seed, up to the attention's summation order.  The prompts are prefilled once, at batch B, and the N rows
    of a prompt share its KV cache (SampleCache), whose keys the decode attention reads once per step for all N.
    Greedy selection with N > 1 raises ValueError, as HF does; a conversation cache (cache=) with N > 1 raises
    NotImplementedError.
    repetition_penalty, no_repeat_ngram_size, min_length, min_new_tokens: transformers' RepetitionPenalty-,
    NoRepeatNGram-, MinLength- and MinNewTokensLengthLogitsProcessor, applied on the device before the selection, greedy
    or sampled (LogitsProcessors; kernels.sample_tokens_processed), to each row's history: its prompt as given (pads
    of a left-padded batch included; on a conversation cache the whole submitted prompt), then its new tokens (pads of
    finished rows included).  length_eos_ids: the ids min_length / min_new_tokens suppress (HF's resolved eos list;
    None: [eos_token_id] when one is given); they do not change when the loop stops or pads.  With all four neutral the
    loop launches the kernels it launches without them.  Sampling with a repetition penalty holds at most
    kernels.PROC_LIST_MAX history ids per row; beyond that, and with beam search, they raise NotImplementedError.
    output_scores / output_logits / return_dict_in_generate (transformers' generate outputs): with any of them the call
    returns a dict -- sequences (the ids above), scores and logits (None unless asked for: one fp32 [R, V] tensor per
    new token, R = B * num_return_sequences; scores are HF's next_token_scores, the fp32 logits through the processors
    and, when sampling, the temperature / top-k / top-p warpers, -inf where HF masks; logits the widened logits; entry 0
    comes from the prefill).  The selection kernel writes them inside the (graphed) step into slot s of fp32 buffers
    [max_new_tokens, R, V], allocated up front: 4 * V bytes (128 KB at V = 32 000) per row, token and output, where HF
    grows its tuples as it goes -- the same peak at full length.  Beam search adds sequences_scores (the returned
    beams' final scores) and beam_indices (int32 [B * num_return_sequences, n], b * num_beams + beam, -1 past a beam's
    end); its scores are each beam row's log_softmax before the running score is added, as HF stores them.
    prompt_lookup_num_tokens = k (with max_matching_ngram_size, default 2): prompt-lookup decoding, transformers'
    PromptLookupCandidateGenerator and _assisted_decoding -- each step drafts up to k ids by copying what followed the
    leftmost earlier occurrence of the sequence's last n-gram, and verifies them in one decode chain over k + 1 rows
    (LookupDecode, one CUDA graph); a step without a draft runs over one row.  It runs for batch 1 with greedy or
    temperature / top-k / top-p selection, eos_token_id an id or a list, a conversation cache and host stopping_criteria
    (called on the candidate sequence before each step and on the sequence after it, as HF calls them; streamer:
    transformers' BaseStreamer contract -- the prompt, then the first token, then each step's accepted tokens); token j
    is drawn with Philox counter j, so with equal logits the tokens are those of the plain loop with the same seed.
    Stated deviations from HF's assisted loop: where HF's acceptance would run past max_new_tokens the loop stops
    there; when sampling, HF's PromptLookupCandidateGenerator also cuts a draft at the first id its warpers mask on
    constant logits (top_k, top_p < 1: a fixed set of ids), which the draft rule here does not -- the tokens' distribution
    is the plain loop's either way, but drafts and accept counts can differ from use_hf_loop=True's.  After the call,
    self.lookup_accepted (a diagnostic, overwritten by the next lookup call) lists the tokens each verify step appended.
    Every other call (batch > 1, a padded mask, logits processors, stop_strings, outputs, beams,
    num_return_sequences > 1) ignores the option and runs the plain loop."""
    if length_eos_ids is None:
        length_eos_ids = [] if eos_token_id is None else (
            list(eos_token_id) if isinstance(eos_token_id, (list, tuple)) else [eos_token_id])
    neutral = LogitsProcessors.neutral(repetition_penalty, no_repeat_ngram_size, min_length, min_new_tokens,
                                       length_eos_ids)
    if num_beams > 1:
        if not neutral:
            raise NotImplementedError('beam search with repetition_penalty / no_repeat_ngram_size / min_length / '
                                      'min_new_tokens runs on the HF loop only: pass use_hf_loop=True')
        if do_sample:
            raise NotImplementedError('beam search with do_sample runs on the HF loop only: pass use_hf_loop=True')
        if stopping_criteria is not None:
            raise NotImplementedError('beam search with stopping_criteria runs on the HF loop only: pass use_hf_loop=True')
        if stop_strings is not None:
            raise NotImplementedError('beam search with stop_strings runs on the HF loop only: pass use_hf_loop=True')
        if cache is not None:
            raise NotImplementedError('beam search on a conversation cache (cache=) runs on the HF loop only: pass '
                                      'use_hf_loop=True')
        return _generate_beams(self, input_ids, images, bboxes, max_new_tokens, num_beams, eos_token_id, pad_token_id,
                               attention_mask, length_penalty, early_stopping, num_return_sequences, use_graph,
                               output_scores, output_logits, return_dict_in_generate)
    B, L = input_ids.shape
    N = int(num_return_sequences)
    greedy = not (do_sample and temperature > 0)
    if prompt_lookup_num_tokens and B == 1 and N == 1 and neutral and stop_strings is None \
            and not (output_scores or output_logits or return_dict_in_generate) and self.cfg.head_dim == 128 \
            and max_new_tokens >= 1 and (attention_mask is None or bool(attention_mask.bool().all())):
        eos = [] if eos_token_id is None else [int(e) for e in (
            eos_token_id if isinstance(eos_token_id, (list, tuple)) else [eos_token_id])]
        return _generate_lookup(self, input_ids, images, bboxes, max_new_tokens, int(prompt_lookup_num_tokens),
                                int(max_matching_ngram_size or 2), greedy, temperature, top_k, top_p, generator, eos,
                                stopping_criteria, cache, use_graph, streamer)
    if N != 1:
        if N < 1:
            raise ValueError('num_return_sequences must be >= 1, got %d' % N)
        if greedy:
            raise ValueError('Greedy methods without beam search do not support `num_return_sequences` different than 1 '
                             '(got %d).' % N)
        if cache is not None:
            raise NotImplementedError('several sampled answers per prompt (num_return_sequences=%d) on a conversation '
                                      'cache (cache=) run on the HF loop only: pass use_hf_loop=True' % N)
    if not greedy and repetition_penalty is not None and float(repetition_penalty) != 1.0 \
            and L + max_new_tokens > kernels.PROC_LIST_MAX:
        raise NotImplementedError('sampling with repetition_penalty holds at most %d prompt + new tokens per row on the '
                                  'engine loop (%d asked): pass use_hf_loop=True'
                                  % (kernels.PROC_LIST_MAX, L + max_new_tokens))
    ids = input_ids.to(self.dev)
    if cache is not None:
        logits = self.prefill_cached(cache, input_ids, images, bboxes, attention_mask, new_tokens=max_new_tokens)
        pos0 = cache.row_lens().clone()
    elif N > 1:   # the B prompts prefilled once; each prompt's N rows share its K/V
        cache = SampleCache(self.cfg, B, N, L, max_new_tokens, self.dev)
        run_ids, lens, _ = _right_padded(ids, attention_mask)
        logits = self.forward_device(run_ids, None if images is None else images.to(self.dev, self.dt),
                                     self.plan_boxes(bboxes), validate=True, last_only=True, seqlens=_seqlens(lens, L),
                                     cache=cache.prompt)
        cache.start(lens)
        logits = logits.repeat_interleave(N, 0)   # every row's first token is drawn from its prompt's logits
        pos0 = None
    else:
        cache = KVCache(self.cfg, B, L + max_new_tokens, self.dev)
        run_ids, lens, _ = _right_padded(ids, attention_mask)
        logits = self.forward_device(run_ids, images.to(self.dev, self.dt), self.plan_boxes(bboxes), validate=True,
                                     last_only=True, seqlens=_seqlens(lens, L), cache=cache)
        pos0 = None
    R = B * N
    rule = pad_token_id is not None and eos_token_id is not None
    stop_state = None
    if stop_strings is not None:     # the submitted prompt's tokens, also on a conversation cache
        stop_state = stop_strings.initial_states(*_right_padded(input_ids.cpu(), attention_mask)[:2])
        if N > 1:
            stop_state = stop_state.repeat_interleave(N)
    out = torch.empty((R, L + max_new_tokens), dtype=torch.int64, device=self.dev)
    out[:, :L] = ids if N == 1 else ids.repeat_interleave(N, 0)
    procs = None if neutral else LogitsProcessors(out, L, repetition_penalty, no_repeat_ngram_size, min_length,
                                                  min_new_tokens, length_eos_ids)   # `out` is the rows' history
    slots = [torch.empty((max(max_new_tokens, 1), R, logits.shape[-1]), dtype=torch.float32, device=self.dev)
             if want else None for want in (output_scores, output_logits)]
    sampler = Sampler(R, self.dev, greedy, temperature, top_k, top_p, seed=0 if greedy else sampling_seed(generator),
                      eos_id=eos_token_id, pad_id=pad_token_id, stops=stop_strings, stop_state=stop_state,
                      processors=procs, scores=slots[0], logits=slots[1])
    stepper = None
    if use_graph and max_new_tokens > 4 and self.cfg.head_dim == 128:
        stepper = GraphedDecode(self, cache, sampler=sampler)   # each replay also selects the next token into its ids
    tok = stepper.ids if stepper is not None else torch.empty((R, 1), dtype=torch.int64, device=self.dev)
    sampler(logits, tok)              # the first new token, from the prefill logits
    sampler.advance()
    n = 0
    for step in range(max_new_tokens):
        out[:, L + step:L + step + 1].copy_(tok)
        n = step + 1
        if (rule or stop_strings is not None) and bool(sampler.finished.all()):
            break
        if not rule and eos_token_id is not None and bool((tok == eos_token_id).all()):
            break
        if stopping_criteria is not None and any(bool(torch.as_tensor(sc(out[:, :L + n], logits[:, -1].float())).all())
                                                 for sc in stopping_criteria):
            break
        if step + 1 < max_new_tokens:
            if stepper is not None:
                logits = stepper.step()
            else:
                logits = self.decode_step(tok, cache)
                sampler(logits, tok)
                sampler.advance()
    out = out[:, :L + n]
    if pos0 is not None and n > 1:   # outside the decode step, so its (graphed) launch sequence is unchanged
        cache.record_ids(out[:, L:L + n - 1], pos0)
    if not (output_scores or output_logits or return_dict_in_generate):
        return out
    scores, raw = (None if t is None else tuple(t[:n].unbind(0)) for t in slots)
    return dict(sequences=out, scores=scores, logits=raw)


def _capture(dev, warm, body):
    """Run warm() on a side stream, wait for the device, then capture body() into a CUDA graph on the current stream.
    Returns (graph, what body returned: the graph's static outputs)."""
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        warm()
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize(dev)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = body()
    return graph, out


class GraphedDecode:
    """CUDA-graph replay of one decode step: ~260 launches become one.  The current length lives in a
    device int32 that the QKV-RoPE epilogue, kv_append and decode_attention read; `step` bumps it (and the
    per-sample lengths cache.lens of a batch of prompts of different lengths, which those kernels then read instead).
    sampler (a Sampler): the captured step ends with it selecting the next token from the step's logits into `ids`,
    the graph's own input, so the host copies no token in: write the first token into `ids`, then call step() with no
    argument, once per token; step() also advances the sampler's Philox counter."""

    def __init__(self, engine, cache, sampler=None):
        self.eng, self.cache, self.sampler = engine, cache, sampler
        dev = engine.dev
        self.ids = torch.zeros((cache.B, 1), dtype=torch.int64, device=dev)
        self.pos = torch.tensor([cache.length], dtype=torch.int32, device=dev)
        start = cache.length

        def warm():
            for _ in range(2):  # writes slot `start`, overwritten by the first real step
                logits = engine.decode_step(self.ids, cache, self.pos)
                cache.length = start
            if sampler is not None:   # into a scratch buffer, `finished` untouched
                sampler(logits, torch.empty_like(self.ids), update=False)

        def body():
            logits = engine.decode_step(self.ids, cache, self.pos)
            if sampler is not None:
                sampler(logits, self.ids)
            return logits
        self.graph, self.logits = _capture(dev, warm, body)
        cache.length = start

    def step(self, token_ids=None):
        """token_ids: int64 [B, 1], the tokens to feed (without a sampler); with one, None: the graph feeds itself."""
        if self.cache.length + 1 > self.cache.max_len:
            raise RuntimeError('KV cache is full (%d)' % self.cache.max_len)
        if token_ids is not None:
            self.ids.copy_(token_ids, non_blocking=True)
        self.graph.replay()
        self.pos.add_(1)
        if self.cache.lens is not None:   # per-sample positions: the graph reads this very tensor
            self.cache.lens.add_(1)
        self.cache.length += 1
        if self.sampler is not None:
            self.sampler.advance()
        return self.logits


def lookup_candidates(seq, num_output_tokens, max_ngram=2, max_length=None, eos_ids=()):
    """transformers' PromptLookupCandidateGenerator.get_candidates restated on a host list of ids (one sequence; no
    logits processors): the draft ids for the next verify step, [] for none.  For n-gram sizes min(max_ngram,
    len - 1) down to 1, the leftmost window equal to the sequence's last n-gram whose continuation is not empty wins;
    the draft is up to num_output_tokens ids after it (bounded by the sequence's length and max_length), cut before its
    first eos id.  No draft when max_length == len + 1.  csrc/lookup.cu computes the same on the device."""
    seq = [int(t) for t in seq]
    n = len(seq)
    max_length = n + num_output_tokens + 1 if max_length is None else int(max_length)
    if max_length == n + 1:
        return []
    eos = {int(e) for e in eos_ids}
    for g in range(min(max_ngram, n - 1), 0, -1):
        tail = seq[n - g:]
        for idx in range(n - g + 1):
            if seq[idx:idx + g] != tail:
                continue
            start = idx + g
            end = min(start + num_output_tokens, n, max_length)
            if start < end:
                draft = seq[start:end]
                cut = next((i for i, t in enumerate(draft) if t in eos), len(draft))
                return draft[:cut]      # an eos first: no draft, and the search ends there, as HF's does
    return []


def lookup_accept(drafts, selected, length, max_length, done_candidate=False, eos_ids=()):
    """The acceptance of transformers' _assisted_decoding (its branch without candidate logits), restated: drafts (d ids)
    were verified after a sequence of `length` ids and `selected` (d + 1 ids) are the tokens chosen at the d + 1
    positions.  n = the count of leading drafts equal to the selected tokens; when the candidate sequence is done
    (done_candidate: the stopping criteria on it, or length + d >= max_length) and all d matched, n -= 1.  Returns (the
    appended tokens -- the first n + 1 selected, at most max_length - length of them --, whether one is an eos id)."""
    d = len(drafts)
    n = 0
    while n < d and int(drafts[n]) == int(selected[n]):
        n += 1
    if (done_candidate or length + d >= max_length) and d > 0 and n == d:
        n -= 1
    new = [int(t) for t in selected[:min(n + 1, max_length - length)]]
    eos = {int(e) for e in eos_ids}
    return new, any(t in eos for t in new)


class LookupDecode:
    """Prompt-lookup decoding of one sequence (transformers' generate(prompt_lookup_num_tokens=k), batch 1): each step
    verifies the last accepted token and up to k drafted ids in one decode chain over M = k + 1 rows
    (PrefillEngine.verify_step), selects a token per row (kernels.sample_tokens_rows, row i with Philox counter j0 + i
    where j0 is the index of the first new token it decides, so new token j is always drawn with counter j as the plain
    batch-1 loop draws it), then accepts and drafts the next step on the device (kernels.lookup_step).  A step with no
    draft (no window matched) runs the same over the one row of the last token, a plain one-token step: the host knows
    the draft count from the previous readback.  On CUDA each of the two is one graph, captured once (`graph`, M rows;
    `graph1`, one row); the host replays one per step and reads `readback` once per step.
    hist: int64 [1, >= prompt_len + max_new_tokens], the prompt then the accepted tokens (the loop's output buffer).
    The cache must hold prompt_len + max_new_tokens + k positions: rows past the accepted length write K/V there, which
    nothing reads and later steps overwrite.  On CPU tensors (the loop's host tests) the engine's verify_step is a
    stand-in and the selection (greedy only), acceptance and draft run as their host restatements."""

    def __init__(self, engine, cache, hist, prompt_len, max_new_tokens, k, max_ngram=2, eos_ids=(), greedy=True,
                 temperature=1.0, top_k=None, top_p=None, seed=0, use_graph=True):
        if int(k) < 1 or int(max_ngram) < 1:
            raise ValueError('prompt lookup needs prompt_lookup_num_tokens >= 1 and max_matching_ngram_size >= 1 (got '
                             '%r, %r)' % (k, max_ngram))
        self.eng, self.cache = engine, cache
        self.k, self.max_ngram = int(k), int(max_ngram)
        self.prompt_len, self.max_length = int(prompt_len), int(prompt_len) + int(max_new_tokens)
        self.hist = hist.view(-1)
        dev = self.hist.device
        M = self.k + 1
        self.eos_list = [int(e) for e in eos_ids]
        self.eos = torch.tensor(self.eos_list, dtype=torch.int32, device=dev) if self.eos_list else None
        z = dict(device=dev)
        self.ids = torch.zeros((M, 1), dtype=torch.int64, **z)        # the verify step's input
        self.sel = torch.zeros(M, dtype=torch.int64, **z)             # its selected tokens
        self.state = torch.zeros(5, dtype=torch.int32, **z)           # len, d, finished, appended, host_done
        self.base = torch.zeros(1, dtype=torch.int32, **z)
        self.pos = torch.zeros(M, dtype=torch.int32, **z)
        self.step = torch.zeros(M, dtype=torch.int64, **z)
        self.readback = torch.zeros(4 + M + self.k, dtype=torch.int64, **z)
        self.greedy = bool(greedy)
        self.rule = [torch.full((M,), v, dtype=dt, **z) for v, dt in (
            (int(self.greedy), torch.int32), (float(temperature), torch.float32), (int(top_k or 0), torch.int32),
            (1.0 if top_p is None else float(top_p), torch.float32), (int(seed), torch.int64))]
        self.no_eos = torch.full((M,), -1, dtype=torch.int32, **z)    # eos is the lookup kernel's business
        self.active = torch.ones(M, dtype=torch.int32, **z)
        self.finished = torch.zeros(M, dtype=torch.int32, **z)        # scratch of the selection
        self.anc = torch.zeros((M, cache.max_len), dtype=torch.int32, **z) if dev.type == 'cuda' else None
        self.accepted = []                                            # tokens appended by each verify step
        self.use_graph = bool(use_graph) and dev.type == 'cuda'
        self.graph = self.graph1 = None
        self.rb = None                                                # the last readback, on the host

    def _capture(self, rows):
        """Capture the verify step over `rows` rows once the first draft is in place: the warm-up runs it at the first
        step's positions (whose K/V that step rewrites), and its other writes are undone."""
        mutable = [self.ids, self.sel, self.state, self.base, self.pos, self.step, self.readback, self.finished,
                   self.hist]
        saved = [t.clone() for t in mutable]
        graph, _ = _capture(self.hist.device, lambda: [self._body(rows) for _ in range(2)], lambda: self._body(rows))
        for t, s in zip(mutable, saved):
            t.copy_(s)
        return graph

    def _select(self, logits, rows):
        """Select rows [0, rows) of logits [rows, 1, V] into self.sel[:rows]."""
        if logits.is_cuda:
            g, t, k, p, s = (v[:rows] for v in self.rule)
            kernels.sample_tokens_rows(logits, self.sel[:rows], g, t, k, p, s, self.step[:rows], self.no_eos[:rows],
                                       self.active[:rows], self.finished[:rows])
            return
        if not self.greedy:
            raise RuntimeError('token sampling runs on the CUDA device only (csrc/sample.cu): logits are on %s'
                               % logits.device)
        self.sel[:rows] = logits.reshape(rows, -1).argmax(-1)

    def _body(self, rows):
        logits = self.eng.verify_step(self.ids[:rows], self.cache, self)
        self._select(logits, rows)
        if logits.is_cuda:
            kernels.lookup_step(self, self.sel)
        else:
            self._host_accept()
        return logits

    # host restatement of csrc/lookup.cu (CPU tensors)
    def _host_accept(self):
        ln, d, done = int(self.state[0]), int(self.state[1]), bool(self.state[4])
        new, fin = lookup_accept(self.ids[1:1 + d, 0].tolist(), self.sel.tolist(), ln, self.max_length, done,
                                 self.eos_list)
        self.hist[ln:ln + len(new)] = torch.tensor(new, dtype=torch.int64)
        self.readback[4:4 + len(new)] = torch.tensor(new, dtype=torch.int64)
        self.readback[0] = len(new)
        self.state[0], self.state[3] = ln + len(new), len(new)
        self.state[2] = int(bool(self.state[2]) or fin)
        self._host_draft()

    def _host_draft(self):
        ln, fin = int(self.state[0]), bool(self.state[2])
        draft = [] if fin or ln + 1 >= self.max_length else lookup_candidates(
            self.hist[:ln].tolist(), self.k, self.max_ngram, self.max_length, self.eos_list)
        d = len(draft)
        M = self.k + 1
        last = int(self.hist[ln - 1])
        row = [last] + draft + [last] * (self.k - d)
        self.ids[:, 0] = torch.tensor(row, dtype=torch.int64)
        self.pos.copy_(torch.arange(M, dtype=torch.int32) + ln - 1)
        self.base[0] = ln - 1
        self.step.copy_(torch.arange(M, dtype=torch.int64) + ln - self.prompt_len)
        self.state[1] = d
        self.readback[1:4] = torch.tensor([int(fin), ln, d])
        self.readback[4 + M:] = torch.tensor(draft + [-1] * (self.k - d), dtype=torch.int64)

    def first(self, logits):
        """The first new token, selected from the prefill's logits [1, 1, V] (Philox counter 0), appended to the history;
        then the first draft.  Returns (the token, whether it is an eos id)."""
        L = self.prompt_len
        self.step[0] = 0
        self._select(logits.reshape(1, 1, -1), 1)
        tok = int(self.sel[0])
        fin = tok in self.eos_list
        self.hist[L] = tok
        self.state.copy_(torch.tensor([L + 1, 0, int(fin), 1, 0], dtype=torch.int32))
        if self.hist.is_cuda:
            kernels.lookup_step(self)
        else:
            self._host_draft()
        if self.use_graph and not fin:
            self.graph, self.graph1 = self._capture(self.k + 1), self._capture(1)
        self.rb = self.readback.cpu()
        return tok, fin

    def run(self, host_done=None):
        """One verify step: host_done (the host's stopping criteria on the candidate sequence; None without criteria) is
        written before it.  M rows when the step has drafts, else the one-row step.  Returns the readback on the host
        (also kept as `rb`): int64 [appended, finished, len, d, the appended tokens (M slots), the next drafts (k
        slots)]."""
        if host_done is not None:
            self.state[4] = int(bool(host_done))
        rows = self.k + 1 if int(self.rb[3]) else 1
        graph = self.graph if rows > 1 else self.graph1
        if graph is not None:
            graph.replay()
        else:
            self._body(rows)
        self.rb = rb = self.readback.cpu()
        self.accepted.append(int(rb[0]))
        return rb


def lookup_loop(st, logits, max_new_tokens, stopping_criteria=None, streamer=None):
    """The host side of prompt-lookup decoding on a LookupDecode `st` from the prefill's logits: the first token, then
    verify steps until max_new_tokens, an eos id or a stopping criterion.  Host stopping_criteria are called as
    transformers' _assisted_decoding calls them -- on the candidate sequence (the history plus the drafts) before
    each verify step, whose acceptance then keeps one draft fewer when all match, and on the history after the
    accepted tokens are appended -- each with scores None.  The streamer follows transformers' BaseStreamer contract
    as HF's generate drives it: put(the prompt ids [1, L]) first, then the first token, then each step's accepted
    tokens, then end().  Returns the count of new tokens in st.hist."""
    L = st.prompt_len
    out = st.hist.view(1, -1)
    if streamer is not None:
        streamer.put(out[:, :L].cpu())
    tok, fin = st.first(logits)
    n = 1
    if streamer is not None:
        streamer.put(torch.tensor([tok]))

    def stop(seq):
        return any(bool(torch.as_tensor(sc(seq, None)).all()) for sc in stopping_criteria)
    while not fin and n < max_new_tokens:
        if stopping_criteria is not None and stop(out[:, :L + n]):
            break
        rb = st.rb
        done = None
        if stopping_criteria is not None:
            d = int(rb[3])
            drafts = rb[4 + st.k + 1:4 + st.k + 1 + d].to(out.device)
            done = stop(torch.cat([out[:, :L + n], drafts[None]], 1))
        rb = st.run(done)
        acc = int(rb[0])
        n += acc
        fin = bool(rb[1])
        if streamer is not None:
            streamer.put(rb[4:4 + acc].clone())
    if streamer is not None:
        streamer.end()
    return n


@torch.no_grad()
def _generate_lookup(self, input_ids, images, bboxes, max_new_tokens, k, max_ngram, greedy, temperature, top_k, top_p,
                     generator, eos_ids, stopping_criteria, cache, use_graph, streamer):
    """generate()'s prompt-lookup path (batch 1): the prefill as the plain loop runs it, into a cache with room for k
    more positions, then lookup_loop on a LookupDecode."""
    L = input_ids.shape[1]
    ids = input_ids.to(self.dev)
    if cache is not None:
        logits = self.prefill_cached(cache, input_ids, images, bboxes, None, new_tokens=max_new_tokens + k)
    else:
        cache = KVCache(self.cfg, 1, L + max_new_tokens + k, self.dev)
        logits = self.forward_device(ids, None if images is None else images.to(self.dev, self.dt),
                                     self.plan_boxes(bboxes), validate=True, last_only=True, cache=cache)
    out = torch.zeros((1, L + max_new_tokens + k), dtype=torch.int64, device=self.dev)
    out[:, :L] = ids
    st = LookupDecode(self, cache, out, L, max_new_tokens, k, max_ngram, eos_ids, greedy, temperature, top_k, top_p,
                      seed=0 if greedy else sampling_seed(generator), use_graph=use_graph)
    n = lookup_loop(st, logits, max_new_tokens, stopping_criteria, streamer)
    # the cache holds the prompt and every new token but the last, as after the plain loop
    cache.length = L + n - 1
    if cache.lens is not None:
        cache.lens.fill_(L + n - 1)
    cache.ids[:, L:] = -1
    if n > 1:
        cache.record_ids(out[:, L:L + n - 1], torch.full((1,), L, dtype=torch.int32, device=self.dev))
    self.lookup_accepted = st.accepted   # diagnostic: tokens appended by each verify step of the engine's last lookup call
    return out[:, :L + n]


class Request:
    """A request of a ContinuousBatcher: `sequences` (host int64 [1, L + n]: the prompt as given, then the n new tokens,
    HF's layout) grows by one token per step while it runs; `done` turns True when it retires -- it emitted its eos id,
    ended a stop string, or has max_new_tokens new tokens -- or when its admission failed: `error` is then the exception,
    which ContinuousBatcher.step() raised, and the request has no new tokens.  `reused`: how many prompt tokens its
    admission took from K/V a batcher row already held (ContinuousBatcher(prefix_reuse=True)); 0 for a full prefill.
    `processors` (ContinuousBatcher(request_options=True)): the request's repetition_penalty, no_repeat_ngram_size,
    min_length, min_new_tokens and length_eos_ids, None when all are neutral; `stops`: its own StopStrings or None."""

    def __init__(self, input_ids, images, bboxes, max_new_tokens, greedy, temperature, top_k, top_p, seed, eos_id,
                 streamer, processors=None, stops=None):
        self.input_ids, self.images, self.bboxes = input_ids, images, bboxes
        self.max_new_tokens = max_new_tokens
        self.greedy, self.temperature, self.top_k, self.top_p, self.seed = greedy, temperature, top_k, top_p, seed
        self.eos_id, self.streamer = eos_id, streamer
        self.processors, self.stops = processors, stops
        self.tokens = []
        self.done = False
        self.error = None
        self.reused = 0

    @property
    def sequences(self):
        return torch.cat([self.input_ids.cpu(), torch.tensor(self.tokens, dtype=torch.int64)[None]], 1)


def _image_sig(image):
    """A few hundred strided samples of an image, on the host (None without an image): images whose samples differ differ,
    so a batcher admission compares each row's image on the device only when the samples agree."""
    return None if image is None else image.reshape(-1)[::2039].float().cpu()


def _held_ids(rec):
    """The token ids a ContinuousBatcher row record stands for: its ids, then its request's new tokens but the last."""
    if rec is None:
        return torch.zeros(0, dtype=torch.int64)
    if rec['req'] is None:
        return rec['ids']
    return torch.cat([rec['ids'], torch.tensor(rec['req'].tokens[:-1], dtype=torch.int64)])


class ContinuousBatcher:
    """Continuous (in-flight) batching of generate requests on one engine: `slots` decode rows, each holding one request
    with its own prompt length, sampling rule, seed, eos id and answer length.  A queued request joins a free row
    between two decode steps -- prefilled at batch 1 straight into its row of the batcher's KV cache -- while the others
    keep decoding, and leaves it as soon as it finishes, so the weights streamed by each step serve every running request.

    Row r's token is the one generate() selects for the request alone: the first from its prefill logits, then one per
    decode step, drawn by kernels.sample_tokens_rows with Philox key = its seed and counter (its token count, 0), as a
    batch-1 generate() draws.  The decode step runs on a KVCache(cfg, slots, max_len) with per-row lengths, allocated
    up front and never grown; on CUDA it is one graph (decode step, selection, stop strings), captured once, whose
    device-side state -- the per-row rule arrays, `active`, `finished`, the lengths -- admissions rewrite in place.
    stop_strings: a StopStrings for every request (transformers' stop_strings).  On CPU tensors (the engine's host
    stand-ins) the steps run eagerly with a greedy host selection.

    prefix_reuse=True: a request prefills only what no row already holds -- a follow-up turn of a conversation that is
    sent again whole, or another question on the same image.  The batcher keeps a host record of each row (row_record:
    the token ids whose K/V it holds, its image and boxes; a row keeps it after its request retires) and admits a
    request, FIFO as always, where KVCache.reusable's rules find the longest prefix that covers the prompt's image span:
    in place when a free row holds it; else, when a running row (or one prefilled earlier in the same step) holds a
    strictly longer one, in a free row into which that prefix's K/V are copied; else by a full prefill.  Free rows are
    taken never-used first, then least recently retired, so held conversations live as long as they can.  The requests
    of a step that reuse a prefix are prefilled together by one chunk prefill (PrefillEngine.extend on a row view of
    the cache).  A reused request's tokens are those of that chunk prefill -- generate(cache=) on the conversation --
    not those of a full prefill, and may depend on what the row held: the caller opts into that.

    request_options=True: each request may also carry transformers' history-dependent logits processors
    (repetition_penalty, no_repeat_ngram_size, min_length, min_new_tokens) and its own stop strings, as generate() runs
    them for a batch of one.  The graph then ends with kernels.sample_tokens_rows_processed, reading each row's
    processors and its history -- int64 [slots, max_len], row s the whole submitted prompt (under prefix reuse too,
    the part taken from the cache included), then the request's new tokens -- and kernels.stop_step_rows, reading each
    row's own stop table.  A request's StopStrings replaces the batcher's for its row; every table must have the
    batcher's V_tok (that of `stop_strings`, else the engine's vocabulary).  A row whose processors are all neutral
    selects exactly as on a batcher without the option.  The choice is made once, here: one graph per batcher."""

    def __init__(self, engine, slots, max_len, stop_strings=None, prefix_reuse=False, request_options=False):
        if slots < 1 or max_len < 2:
            raise ValueError('ContinuousBatcher needs slots >= 1 and max_len >= 2 (got %d, %d)' % (slots, max_len))
        if prefix_reuse and engine.cfg.head_dim != 128:
            raise NotImplementedError('prefix_reuse needs the chunk prefill, which needs head_dim 128 (got %d)'
                                      % engine.cfg.head_dim)
        self.prefix_reuse = bool(prefix_reuse)
        # per row (prefix_reuse): what its K/V were computed from -- dict(ids: the held prefix, host int64, req: the
        # request whose prompt and tokens follow it or None, images, boxes) or None (never held anything)
        self.records = [None] * int(slots)
        self.retired = [0] * int(slots)   # when each row's request retired (a counter): the least recent is taken first
        self.clock = 0
        self.eng, self.slots, self.max_len = engine, int(slots), int(max_len)
        dev = engine.dev
        S = self.slots
        self.cache = KVCache(engine.cfg, S, self.max_len, dev)
        self.cache.lens = torch.zeros(S, dtype=torch.int32, device=dev)

        def vec(fill, dt):
            return torch.full((S,), fill, dtype=dt, device=dev)
        # the per-row rule and state that kernels.sample_tokens_rows reads, in its argument order
        self.greedy, self.temperature = vec(1, torch.int32), vec(1.0, torch.float32)
        self.top_k, self.top_p = vec(0, torch.int32), vec(1.0, torch.float32)
        self.seed, self.step_count = vec(0, torch.int64), vec(0, torch.int64)
        self.eos_id, self.active, self.finished = vec(-1, torch.int32), vec(0, torch.int32), vec(0, torch.int32)
        self.stops = stop_strings
        self.stop_table = None if stop_strings is None else stop_strings.on(dev)
        self.stop_state = vec(0, torch.int32)
        self.request_options = bool(request_options)
        if self.request_options:
            # the per-row processors and stop tables that kernels.sample_tokens_rows_processed / stop_step_rows read
            self.history = torch.zeros((S, self.max_len), dtype=torch.int64, device=dev)
            self.prompt_len, self.penalty = vec(0, torch.int32), vec(1.0, torch.float32)
            self.ngram, self.min_length, self.min_new_tokens = (vec(0, torch.int32) for _ in range(3))
            self.length_eos = torch.zeros((S, kernels.PROC_ROW_EOS), dtype=torch.int32, device=dev)
            self.n_length_eos = vec(0, torch.int32)
            self.V_tok = engine.cfg.vocab if stop_strings is None else stop_strings.V_tok
            self.row_tables, self.row_states = vec(0, torch.int64), vec(1, torch.int32)
            self.row_stops = [None] * S     # each running row's table: the graph reads it through row_tables
            self.row_procs = [None] * S     # each running row's processors (the host stand-in restates them)
        self.ids = torch.zeros((S, 1), dtype=torch.int64, device=dev)     # the decode step's input: each row's last token
        self.pos = torch.zeros(1, dtype=torch.int32, device=dev)          # pos_dev: positions come from cache.lens
        self.readback = torch.zeros((S, 2), dtype=torch.int64, device=dev)   # (token, finished) per row: one copy out
        self.queue = collections.deque()
        self.running = [None] * S
        self.graph = None
        if engine.dev.type == 'cuda':
            self.graph, _ = _capture(dev, self._decode, self._decode)   # every row is idle: the warm-up selects nothing

    def _select(self, logits, rows, lens):
        """The selection of rows `rows` (a slice) from logits [n, 1, V] into self.ids[rows], then the stop strings."""
        ids, fin = self.ids[rows], self.finished[rows]
        if logits.is_cuda and self.request_options:
            kernels.sample_tokens_rows_processed(
                logits, ids, self.greedy[rows], self.temperature[rows], self.top_k[rows], self.top_p[rows],
                self.seed[rows], self.step_count[rows], self.eos_id[rows], self.active[rows], fin, lens,
                self.history[rows], self.prompt_len[rows], self.penalty[rows], self.ngram[rows], self.min_length[rows],
                self.min_new_tokens[rows], self.length_eos[rows], self.n_length_eos[rows])
            kernels.stop_step_rows(ids, self.row_tables[rows], self.row_states[rows], self.V_tok, self.active[rows],
                                   self.stop_state[rows], fin)
            return
        if logits.is_cuda:
            kernels.sample_tokens_rows(logits, ids, self.greedy[rows], self.temperature[rows], self.top_k[rows],
                                       self.top_p[rows], self.seed[rows], self.step_count[rows], self.eos_id[rows],
                                       self.active[rows], fin, lens)
            if self.stop_table is not None:
                kernels.stop_step(ids, self.stop_table, self.stop_state[rows], fin)
            return
        # host stand-in (Sampler._host's counterpart): greedy rows only, same state updates as the kernels
        live = self.active[rows].bool()
        if bool((live & (self.greedy[rows] == 0)).any()):
            raise RuntimeError('token sampling runs on the CUDA device only (csrc/sample.cu): logits are on %s'
                               % logits.device)
        scores = logits.reshape(live.shape[0], -1)
        if self.request_options:
            scores = scores.float().clone()
            for i, s in enumerate(range(self.slots)[rows]):
                if live[i] and self.row_procs[s] is not None:
                    scores[i:i + 1] = LogitsProcessors(self.history[s:s + 1], int(self.prompt_len[s]),
                                                       **self.row_procs[s]).apply(scores[i:i + 1],
                                                                                  int(self.step_count[s]))
        tok = torch.where(live, scores.argmax(-1), ids[:, 0])
        ids[:, 0] = tok
        eos = self.eos_id[rows]
        fin |= (live & (eos >= 0) & (tok == eos)).to(torch.int32)
        if self.request_options:
            for i, s in enumerate(range(self.slots)[rows]):
                at = int(self.prompt_len[s] + self.step_count[s])
                if live[i] and at < self.max_len:
                    self.history[s, at] = tok[i]
        self.step_count[rows] += live.to(torch.int64)
        if lens is not None:
            lens += live.to(torch.int32)
        if self.request_options:
            for i, s in enumerate(range(self.slots)[rows]):
                if live[i] and not fin[i] and self.row_stops[s] is not None:
                    new, hit = _stop_lookup(self.row_stops[s], tok[i:i + 1], self.stop_state[s:s + 1].to(torch.int64))
                    self.stop_state[s] = int(new[0])
                    fin[i] |= int(hit[0])
        elif self.stop_table is not None:
            state = self.stop_state[rows]
            new, hit = _stop_lookup(self.stop_table, tok, state.to(torch.int64))
            open_ = fin == 0
            state.copy_(torch.where(open_, new.to(torch.int32), state))
            fin |= (open_ & hit).to(torch.int32)

    def _decode(self):
        """One decode step over every row (the captured graph's body): forward, selection, stop strings, readback."""
        self.cache.length = 0     # positions come from cache.lens; pos_dev sizes the attention by max_len
        logits = self.eng.decode_step(self.ids, self.cache, self.pos)
        self.cache.length = 0
        self._select(logits, slice(None), self.cache.lens)
        self.readback[:, 0:1].copy_(self.ids)
        self.readback[:, 1].copy_(self.finished)
        return logits

    def submit(self, input_ids, images=None, bboxes=None, max_new_tokens=32, do_sample=False, temperature=1.0,
               top_k=None, top_p=None, generator=None, eos_token_id=None, streamer=None, repetition_penalty=1.0,
               no_repeat_ngram_size=0, min_length=0, min_new_tokens=0, length_eos_ids=None, stop_strings=None):
        """Queue one request and return its Request.  input_ids: int64 [1, L] or [L]; images [1, 3, S, S] or None;
        bboxes: a list of one [K, 4] box tensor, or None.  Sampling as generate(): do_sample with temperature > 0 draws
        from the temperature / top_k / top_p processed softmax with a seed taken from `generator` (default: torch's
        default generator) now, at submission; otherwise the arg-max.  eos_token_id: an id, or a list of one.
        streamer: transformers' BaseStreamer contract -- put(prompt ids) at admission, put(token) per new token, end().
        repetition_penalty, no_repeat_ngram_size, min_length, min_new_tokens, length_eos_ids (1..4 ids; None:
        [eos_token_id] when one is given) as generate() takes them, and stop_strings (a StopStrings, which replaces the
        batcher's for this request) need a batcher built with request_options=True; otherwise a value that would
        change a token raises NotImplementedError.  The request's stop table is built here, before any decode step
        needs it."""
        ids = torch.as_tensor(input_ids)
        if ids.dim() == 1:
            ids = ids[None]
        if ids.dim() != 2 or ids.shape[0] != 1 or ids.shape[1] < 1:
            raise ValueError('submit takes one prompt: input_ids [1, L] or [L], got %s' % (tuple(ids.shape),))
        L, n = ids.shape[1], int(max_new_tokens)
        if n < 1:
            raise ValueError('max_new_tokens must be >= 1, got %d' % n)
        if L + n > self.max_len:
            raise ValueError('prompt (%d) + max_new_tokens (%d) exceed the batcher\'s max_len %d'
                             % (L, n, self.max_len))
        if length_eos_ids is None:
            length_eos_ids = [] if eos_token_id is None else (
                list(eos_token_id) if isinstance(eos_token_id, (list, tuple)) else [eos_token_id])
        neutral = LogitsProcessors.neutral(repetition_penalty, no_repeat_ngram_size, min_length, min_new_tokens,
                                           length_eos_ids)
        if not self.request_options and (not neutral or stop_strings is not None):
            raise NotImplementedError('%s per request: run it with model.generate, or build the batcher with '
                                      '`request_options=True`' % ('stop_strings' if neutral else
                                                                  'a logits processor (repetition_penalty, '
                                                                  'no_repeat_ngram_size, min_length, min_new_tokens)'))
        if isinstance(eos_token_id, (list, tuple)):
            if len(eos_token_id) > 1:
                raise NotImplementedError('the continuous batcher stops a request on one eos id, got %r: run it with '
                                          'model.generate' % (list(eos_token_id),))
            eos_token_id = eos_token_id[0] if eos_token_id else None
        greedy = not (do_sample and temperature > 0)
        if not greedy and top_p is not None and top_p < 0:
            raise ValueError('top_p must be >= 0, got %r' % (top_p,))
        procs = None
        if not neutral:
            procs = dict(repetition_penalty=1.0 if repetition_penalty is None else float(repetition_penalty),
                         no_repeat_ngram_size=int(no_repeat_ngram_size or 0), min_length=int(min_length or 0),
                         min_new_tokens=int(min_new_tokens or 0), eos_ids=[int(e) for e in length_eos_ids])
            if not procs['repetition_penalty'] > 0 or min(procs['no_repeat_ngram_size'], procs['min_length'],
                                                           procs['min_new_tokens']) < 0:
                raise ValueError('repetition_penalty must be > 0 and no_repeat_ngram_size, min_length, min_new_tokens '
                                 '>= 0 (got %r)' % (procs,))
            if (procs['min_length'] or procs['min_new_tokens']) and len(procs['eos_ids']) > kernels.PROC_ROW_EOS:
                raise NotImplementedError('the continuous batcher suppresses at most %d eos ids below a minimum length, '
                                          'got %r: run it with model.generate' % (kernels.PROC_ROW_EOS,
                                                                                  procs['eos_ids']))
            if not greedy and procs['repetition_penalty'] != 1.0 and L + n > kernels.PROC_LIST_MAX:
                raise NotImplementedError('sampling with repetition_penalty holds at most %d prompt + new tokens per '
                                          'row (%d asked): run it with model.generate and use_hf_loop=True'
                                          % (kernels.PROC_LIST_MAX, L + n))
        if stop_strings is not None:
            if stop_strings.V_tok != self.V_tok:
                raise ValueError('stop_strings: the table covers %d token ids, the batcher\'s %d (one tokenizer per '
                                 'batcher)' % (stop_strings.V_tok, self.V_tok))
            stop_strings.on(self.eng.dev)
        req = Request(ids.to(torch.int64), images, bboxes, n, greedy, float(temperature), int(top_k or 0),
                      1.0 if top_p is None else float(top_p), 0 if greedy else sampling_seed(generator),
                      -1 if eos_token_id is None else int(eos_token_id), streamer, procs, stop_strings)
        self.queue.append(req)
        return req

    def _emit(self, s, tok, finished):
        """Give slot s's request its new token; retire it when it is done.  Returns it when it retired."""
        req = self.running[s]
        req.tokens.append(int(tok))
        if req.streamer is not None:
            req.streamer.put(torch.tensor([int(tok)]))
        if not (finished or len(req.tokens) >= req.max_new_tokens):
            return None
        req.done = True
        self.running[s] = None
        self.active[s] = 0
        if self.request_options:          # inactive now: the graph no longer reads its table
            self.row_stops[s] = self.row_procs[s] = None
        self.clock += 1
        self.retired[s] = self.clock
        if req.streamer is not None:
            req.streamer.end()
        return req

    def _set_row(self, req, s):
        """Write slot s's device state for `req`: its rule, counters and flags, its stop state and, with
        request_options, its history (the whole submitted prompt), processors and stop table."""
        dev, row = self.eng.dev, slice(s, s + 1)
        L = req.input_ids.shape[1]
        for t, v in ((self.greedy, int(req.greedy)), (self.temperature, req.temperature), (self.top_k, req.top_k),
                     (self.top_p, req.top_p), (self.seed, req.seed), (self.step_count, 0),
                     (self.eos_id, req.eos_id), (self.finished, 0), (self.active, 1)):
            t[row] = v
        if not self.request_options:
            if self.stops is not None:
                self.stop_state[row] = self.stops.initial_states(req.input_ids, torch.tensor([L])).to(dev)
            return
        self.history[s, :L] = req.input_ids[0].to(dev)
        self.prompt_len[row] = L
        pr = req.processors or dict(repetition_penalty=1.0, no_repeat_ngram_size=0, min_length=0, min_new_tokens=0,
                                    eos_ids=[])
        eos = pr['eos_ids'] if pr['min_length'] or pr['min_new_tokens'] else []
        for t, v in ((self.penalty, pr['repetition_penalty']), (self.ngram, pr['no_repeat_ngram_size']),
                     (self.min_length, pr['min_length']), (self.min_new_tokens, pr['min_new_tokens']),
                     (self.n_length_eos, len(eos))):
            t[row] = v
        if eos:
            self.length_eos[s, :len(eos)] = torch.tensor(eos, dtype=torch.int32).to(dev)
        self.row_procs[s] = req.processors
        stops = req.stops if req.stops is not None else self.stops
        self.row_stops[s] = None if stops is None else stops.on(dev)
        if stops is not None:
            self.stop_state[row] = stops.initial_states(req.input_ids, torch.tensor([L])).to(dev)
            self.row_states[row] = stops.S
        self.row_tables[row] = 0 if stops is None else self.row_stops[s].data_ptr()

    def _admit(self, req, s):
        """Prefill `req` into slot s (batch 1, straight into the slot's rows of the cache) and select its first token.
        The slot's device state is written only once the prefill has succeeded, and a failure after that makes the slot
        idle again: a request that cannot run (say, a <bbox> count its boxes do not match) leaves no active row behind."""
        eng, cfg = self.eng, self.eng.cfg
        dev = eng.dev
        ids = req.input_ids.to(dev)
        L = ids.shape[1]
        row = slice(s, s + 1)
        one = KVCache(cfg, 1, self.max_len, dev, kv=([k[row] for k in self.cache.k], [v[row] for v in self.cache.v]))
        images = None if req.images is None else req.images.to(dev, eng.dt)
        logits = eng.forward_device(ids, images, eng.plan_boxes(req.bboxes), validate=True, last_only=True, cache=one)
        try:
            self._set_row(req, s)
            self._select(logits, row, None)
            self.cache.lens[row] = L
            tok, fin = torch.stack([self.ids[s, 0], self.finished[s].to(torch.int64)]).tolist()
        except BaseException:
            self.active[row] = 0
            raise
        if req.streamer is not None:
            req.streamer.put(req.input_ids.cpu())
        self.running[s] = req
        return self._emit(s, tok, fin)

    def step(self):
        """Admit queued requests into free slots (first in, first out), run one decode step over every slot, hand each
        running request its token and retire the finished ones.  Returns the requests that finished.  When a request's
        admission fails, it is retired with `error` set and the exception propagates; its slot stays idle and the next
        step() carries on with the other requests."""
        done = []
        if self.prefix_reuse:
            while self.queue and None in self.running:
                done += self._admit_round()
        for s in range(self.slots):
            while self.running[s] is None and self.queue:
                req = self.queue.popleft()
                try:
                    r = self._admit(req, s)
                except Exception as e:   # the request retires unanswered; the others keep their rows
                    req.error, req.done = e, True
                    if req.streamer is not None:
                        req.streamer.end()
                    raise
                if r is not None:
                    done.append(r)
        if not any(r is not None for r in self.running):
            return done
        if self.graph is not None:
            self.graph.replay()
        else:
            self._decode()
        rb = self.readback.cpu()
        for s in range(self.slots):
            if self.running[s] is not None:
                r = self._emit(s, rb[s, 0], bool(rb[s, 1]))
                if r is not None:
                    done.append(r)
        return done

    # ---------------------------------------------------------------- prefix reuse
    def row_record(self, s):
        """The token ids (host int64) whose K/V row s holds: after an admission the prompt, then, while the request runs
        and after it retires, also every new token but the last (whose K/V are never written)."""
        return _held_ids(self.records[s])

    def _set_record(self, s, ids, req, images, boxes, sig=None):
        self.records[s] = dict(ids=ids, req=req, images=images, boxes=boxes,
                               sig=_image_sig(images) if sig is None else sig)

    def _match(self, rec, ids, images, boxes, sig):
        """How many leading tokens of the prompt `ids` (host int64 [L]) a row record can give (0: none usable).
        sig: _image_sig(images), which settles most image mismatches on the host."""
        if rec is None:
            return 0
        held = _held_ids(rec)
        p = reusable_prefix(self.eng.cfg, ids, held, held.shape[0], rec['boxes'], boxes)
        # the image last: comparing it waits for the device, and only a usable token prefix needs it
        if p == 0 or not covers_image_span(self.eng.cfg, ids, p):
            return 0
        if sig is not None and rec['sig'] is not None and not torch.equal(sig, rec['sig']):
            return 0
        if not same_image(rec['images'], images):
            return 0
        return p

    def _free_row(self, free):
        """The free row a request without an in-place match takes: one that never held anything, else the least
        recently retired."""
        fresh = [s for s in free if self.records[s] is None]
        return fresh[0] if fresh else min(free, key=lambda s: self.retired[s])

    def _plan_round(self):
        """Pop queued requests while rows are free and plan each against the rows as they will be after the round's full
        prefills: -> [(req, row, p, donor)] -- p = 0: full prefill; donor None: the row holds the prefix itself."""
        dev, dt = self.eng.dev, self.eng.dt
        free = [s for s in range(self.slots) if self.running[s] is None]
        virtual = list(self.records)
        plan = []
        while self.queue and free:
            req = self.queue.popleft()
            ids = req.input_ids[0].cpu()
            images = None if req.images is None else req.images.to(dev, dt)[0]
            sig = _image_sig(images)
            boxes = _row_boxes(req.bboxes, 0, host=True)
            p = {s: self._match(virtual[s], ids, images, boxes, sig) for s in range(self.slots)}
            pf = max((p[s] for s in free), default=0)
            pr = max((p[s] for s in range(self.slots) if s not in free), default=0)
            if pf > 0 and pf >= pr:
                s = min((s for s in free if p[s] == pf), key=lambda s: self.retired[s])
                plan.append((req, s, pf, None))
                n = pf
            elif pr > pf:
                donor = next(s for s in range(self.slots) if s not in free and p[s] == pr)
                s = self._free_row(free)
                plan.append((req, s, pr, donor))
                n = pr
            else:
                s = self._free_row(free)
                plan.append((req, s, 0, None))
                n = ids.shape[0]
            free.remove(s)
            # what the row holds once the round's prefills and copies ran: the prompt after a full prefill, the kept
            # prefix otherwise (the chunk prefill runs last)
            virtual[s] = dict(ids=ids[:n], req=None, images=images, boxes=boxes, sig=sig)
        return plan

    def _admit_round(self):
        """Admit the requests of one round: full prefills (batch 1, as _admit), then the prefix copies, then one chunk
        prefill over every row that reuses a prefix.  Returns the requests that finished at admission."""
        plan = self._plan_round()
        done, error = [], None
        for i, (req, s, p, donor) in enumerate(plan):
            if p:
                continue
            self.records[s] = None            # the prefill overwrites the row
            try:
                r = self._admit(req, s)
            except Exception as e:
                req.error, req.done = e, True
                if req.streamer is not None:
                    req.streamer.end()
                # the round's other requests not admitted yet go back to the head of the queue, in order
                for j in reversed(range(len(plan))):
                    if j > i or (j < i and plan[j][2]):
                        self.queue.appendleft(plan[j][0])
                raise
            self._set_record(s, req.input_ids[0].cpu(), req, None if req.images is None else
                             req.images.to(self.eng.dev, self.eng.dt)[0], _row_boxes(req.bboxes, 0, host=True))
            if r is not None:
                done.append(r)
        reuse = [(req, s, p, donor) for req, s, p, donor in plan if p]
        for req, s, p, donor in reuse:       # truncate each record to its kept prefix, copying it in from the donor
            src = self.records[s if donor is None else donor]
            held = self.row_record(s if donor is None else donor)[:p]
            if donor is not None:
                for kv in (self.cache.k, self.cache.v):
                    for t in kv:
                        t[s, :p].copy_(t[donor, :p])
            self._set_record(s, held, None, src['images'], src['boxes'], src['sig'])
        if len(reuse) > 1:
            try:
                done += self._extend(reuse)
                reuse = []
            except Exception:
                pass                          # one bad request fails the batch: each one alone, below
        for one in reuse:
            try:
                done += self._extend([one])
            except Exception as e:
                req = one[0]
                req.error, req.done = e, True
                if req.streamer is not None:
                    req.streamer.end()
                error = error or e
        if error is not None:
            raise error
        return done

    def _extend(self, group):
        """One chunk prefill of the prompts' tails over their rows' held prefixes, then each request's first token."""
        eng, cfg = self.eng, self.eng.cfg
        dev = eng.dev
        k = len(group)
        slots = [s for _, s, _, _ in group]
        starts = [p for _, _, p, _ in group]
        tails = [req.input_ids[0].cpu()[p:] for req, _, p, _ in group]
        Lc = max(t.shape[0] for t in tails)
        ids = torch.zeros((k, Lc), dtype=torch.int64)
        mask = torch.zeros((k, Lc), dtype=torch.int64)
        tail_boxes, new_box = [], False
        for i, ((req, s, p, _), t) in enumerate(zip(group, tails)):
            ids[i, :t.shape[0]], mask[i, :t.shape[0]] = t, 1
            boxes = _row_boxes(req.bboxes, 0)
            n_old = int((req.input_ids[0, :p] == cfg.bbox_token).sum())
            tail_boxes.append(None if boxes is None else boxes[n_old:])
            new_box = new_box or bool((t == cfg.bbox_token).any())
        images = None
        if new_box:   # the tails' region tokens come from a ViT + fuse rerun on the requests' images
            images = torch.stack([torch.zeros((3, cfg.image_size, cfg.image_size), dtype=eng.dt, device=dev)
                                  if req.images is None else req.images.to(dev, eng.dt)[0] for req, _, _, _ in group])
        view = KVCache(cfg, k, self.max_len, dev, kv=(self.cache.k, self.cache.v),
                       rows=torch.tensor(slots, dtype=torch.int32, device=dev))
        view.lens = torch.tensor(starts, dtype=torch.int32, device=dev)
        view.length = max(starts)
        for (req, s, p, _) in group:          # the rows' device state, as _admit writes it
            self.cache.lens[s:s + 1] = p
            self._set_row(req, s)
        try:
            logits = eng.extend(view, ids, images, tail_boxes, attention_mask=mask)
            first = []
            for i, (req, s, p, _) in enumerate(group):
                row = slice(s, s + 1)
                self._select(logits[i:i + 1], row, None)
                self.cache.lens[row] = req.input_ids.shape[1]
                first.append(torch.stack([self.ids[s, 0], self.finished[s].to(torch.int64)]))
            first = torch.stack(first).tolist()
        except BaseException:
            for s in slots:
                self.active[s] = 0
            raise
        done = []
        for (req, s, p, _), (tok, fin) in zip(group, first):
            req.reused = p
            rec = self.records[s]
            self._set_record(s, req.input_ids[0].cpu(), req, rec['images'], _row_boxes(req.bboxes, 0, host=True),
                             rec['sig'])
            if req.streamer is not None:
                req.streamer.put(req.input_ids.cpu())
            self.running[s] = req
            r = self._emit(s, tok, fin)
            if r is not None:
                done.append(r)
        return done

    def run(self):
        """Step until nothing is queued or running; returns every request that finished, in the order they did."""
        done = []
        while self.queue or any(r is not None for r in self.running):
            done += self.step()
        return done


class _SharedPromptCache:
    """KV layout of N decode rows per prompt that share the prompt's K/V (beam search, several sampled answers).  Per
    layer one [B + B*N, Lmax, HD] tensor (full_k / full_v): rows 0..B-1 hold the B prompts (n_samples; the B-row
    prefill writes them through `prompt`, a KVCache whose k / v are the views [:B]), row B + r the positions decode row
    r generates (the decode step writes row r's new K/V at pos_rows[r] = lens[r] through the views k / v = [B:]).
    prompt_lens: each prompt's length, device int32 [B]."""

    def __init__(self, cfg, B, N, prompt_len, max_new_tokens, device):
        hd = cfg.n_heads * cfg.head_dim
        dt = cfg.torch_dtype
        dev = torch.device(device)
        R = B * N
        Lmax = prompt_len + max_new_tokens
        self.cfg, self.B, self.N, self.prompt_len = cfg, R, N, prompt_len
        self.n_samples = B
        self.full_k = [torch.zeros((B + R, Lmax, hd), dtype=dt, device=dev) for _ in range(cfg.n_layers)]
        self.full_v = [torch.zeros((B + R, Lmax, hd), dtype=dt, device=dev) for _ in range(cfg.n_layers)]
        self.prompt = KVCache(cfg, B, Lmax, dev, kv=([t[:B] for t in self.full_k], [t[:B] for t in self.full_v]))
        self.k = [t[B:] for t in self.full_k]
        self.v = [t[B:] for t in self.full_v]
        self.max_len = self.Lmax = Lmax
        self.length = 0
        self.G = max_new_tokens
        self.lens = torch.zeros(R, dtype=torch.int32, device=dev)          # pos_rows of the decode step
        self.prompt_lens = torch.full((B,), prompt_len, dtype=torch.int32, device=dev)


class SampleCache(_SharedPromptCache):
    """KV cache of N sampled answers per prompt (generate(num_return_sequences=N, do_sample=True)): the shared-prompt
    layout with sample row r = b*N + i in cache row B + r.  Rows never reorder, so there is no ancestry table: position p
    of row r lies in prompt row b below prompt_lens[b], else in row B + r.  The decode attention
    (kernels.decode_attention_group) reads each prompt's keys once per step for all N of its rows."""

    def __init__(self, cfg, B, N, prompt_len, max_new_tokens, device):
        if not 1 <= N <= kernels.GROUP_MAX_N:
            raise ValueError('num_return_sequences=%d: the engine loop samples 1..%d answers per prompt; pass '
                             'use_hf_loop=True for more' % (N, kernels.GROUP_MAX_N))
        super().__init__(cfg, B, N, prompt_len, max_new_tokens, device)

    def start(self, lens):
        """After the prefill: lens (int64 or int32 [B]) each prompt's length; every sample row's first new token goes
        to its prompt's length."""
        self.prompt_lens.copy_(lens.to(torch.int32))
        self.lens.copy_(self.prompt_lens.repeat_interleave(self.N))
        self.length = self.prompt_len


class BeamCache(_SharedPromptCache):
    """KV cache and device state of beam search over B samples of N beams, in the shared-prompt layout (beam row r in
    cache row B + r).  A cell is written once and never moved: `anc` (int32 [B*N, Lmax]) names the cache row
    that holds position p of beam row r -- its sample's prompt row below lens[b], else the beam row that wrote it --
    and the beam step permutes its generated columns when the beams are reordered.  The rest is the state of
    transformers' _beam_search that kernels.beam_step keeps on the device (see g4r_beam_step_bf16)."""

    def __init__(self, cfg, B, N, prompt_len, max_new_tokens, device, eos=(), length_penalty=1.0, early_stopping=False,
                 fill=-1):
        super().__init__(cfg, B, N, prompt_len, max_new_tokens, device)
        dev = torch.device(device)
        R = B * N
        Lmax = self.Lmax
        self.max_length = prompt_len + max_new_tokens
        eos = [int(e) for e in eos]
        self.n_eos = len(eos)
        self.K = max(2, 1 + len(eos)) * N            # beams_to_keep
        self.eos = torch.tensor(eos, dtype=torch.int32, device=dev) if eos else None
        self.length_penalty = float(length_penalty)
        if early_stopping not in (True, False, 'never'):
            raise ValueError('early_stopping must be True, False or "never", got %r' % (early_stopping,))
        self.early = 2 if early_stopping == 'never' else int(bool(early_stopping))
        self.fill = int(fill)
        self.pos_rows = self.lens
        self.anc = torch.zeros((R, Lmax), dtype=torch.int32, device=dev)
        self.ids = torch.zeros((R, 1), dtype=torch.int64, device=dev)     # the graph's own input
        self.state = torch.zeros(4 * B + 2, dtype=torch.int32, device=dev)
        self.state[1:4 * B:4] = 1                                           # early-stop heuristic unsatisfied
        self.run_score = torch.zeros((B, N), dtype=torch.float32, device=dev)
        self.run_score[:, 1:] = -1e9
        self.run_score = self.run_score.view(R)
        self.cand_score = torch.empty(R * self.K, dtype=torch.float32, device=dev)
        self.cand_tok = torch.empty(R * self.K, dtype=torch.int32, device=dev)
        self.run_seq = torch.full((2, B, N, self.G), self.fill, dtype=torch.int64, device=dev)
        self.fin_seq = torch.full((2, B, N, self.G), self.fill, dtype=torch.int64, device=dev)
        self.fin_score = torch.full((B, N), -1e9, dtype=torch.float32, device=dev)
        self.fin_state = torch.zeros((B, N, 2), dtype=torch.int32, device=dev)
        self.out_scores = self.out_logits = self.bidx = None

    def keep_outputs(self, V, scores=False, logits=False, indices=False):
        """Have every beam step also write transformers' generate outputs (kernels.beam_step): scores / logits into
        slot g (the step's count of generated tokens) of fp32 [max_new_tokens, B*N, V] buffers, and the beam indices
        (int32 [running / finished, 2, B, N, G], -1 where nothing was generated) beside the sequences."""
        dev = self.anc.device
        shape = (self.G, self.B, V)
        self.out_scores = torch.empty(shape, dtype=torch.float32, device=dev) if scores else None
        self.out_logits = torch.empty(shape, dtype=torch.float32, device=dev) if logits else None
        self.bidx = torch.full((2, 2, self.n_samples, self.N, self.G), -1, dtype=torch.int32, device=dev) \
            if indices else None

    def start(self, lens):
        """After the prefill: lens (device int32 [B]) each sample's prompt length; every beam row's prompt positions
        point at its sample's prompt row."""
        B = self.n_samples
        self.prompt_lens = lens.to(torch.int32).contiguous()
        self.anc.copy_(torch.arange(B, dtype=torch.int32, device=self.anc.device).repeat_interleave(self.N)[:, None]
                       .expand(self.anc.shape))
        self.length = self.prompt_len

    def step(self, logits, first=False):
        """The beam step on this step's logits (first: the prefill's [B, V] rows, shared by each sample's beams)."""
        kernels.beam_step(logits, self.N if first else 1, self)

    def done(self):
        """Whether the search has ended (transformers' _beam_search_has_unfinished_sequences is False): one word."""
        return bool(self.state[4 * self.n_samples + 1])

    def result(self, num_return_sequences, prompt_ids):
        """[B * num_return_sequences, L + n]: each sample's best finished beams after the prompt as given, cropped to the
        longest returned one (HF's "prepare outputs")."""
        B, N = self.n_samples, self.N
        g = int(self.state[0])
        seqs = self.fin_seq[g & 1][:, :num_return_sequences].reshape(B * num_return_sequences, self.G)
        n = int(self.fin_state[:, :num_return_sequences, 1].max())
        prompt = prompt_ids.to(seqs.device).repeat_interleave(num_return_sequences, 0)
        return torch.cat([prompt, seqs[:, :n]], 1)

    def outputs(self, num_return_sequences, prompt_ids):
        """result() with the outputs keep_outputs asked for, as a dict: sequences, scores / logits (a tuple of one
        [B*N, V] tensor per step, or None), sequences_scores (fp32 [B * num_return_sequences]: the returned beams' final
        scores) and beam_indices (int32 [B * num_return_sequences, n], or None), HF's _beam_search outputs."""
        seqs = self.result(num_return_sequences, prompt_ids)
        g = int(self.state[0])
        n = seqs.shape[1] - prompt_ids.shape[1]
        nrs = num_return_sequences
        scores, raw = (None if t is None else tuple(t[:g].unbind(0)) for t in (self.out_scores, self.out_logits))
        bidx = None if self.bidx is None else \
            self.bidx[1, g & 1, :, :nrs].reshape(self.n_samples * nrs, self.G)[:, :n]
        return dict(sequences=seqs, scores=scores, logits=raw, beam_indices=bidx,
                    sequences_scores=self.fin_score[:, :nrs].reshape(-1).clone())


class GraphedBeamDecode:
    """CUDA-graph replay of one beam-search step: the decode step over the B*N beam rows of a BeamCache (attention
    through its ancestry table) followed by the beam step, which writes the next ids into cache.ids -- the graph's own
    input -- and the beam rows' positions and ancestry, so step() takes nothing from the host.  Build it after the
    first beam step (from the prefill logits) has run."""

    def __init__(self, engine, cache):
        self.eng, self.cache = engine, cache
        dev = engine.dev
        self.pos = torch.tensor([cache.length], dtype=torch.int32, device=dev)   # sizes the step by max_len
        start = cache.length

        def warm():
            for _ in range(2):  # writes each beam row's current position, rewritten by the first real step
                engine.decode_step(cache.ids, cache, self.pos)
                cache.length = start

        def body():
            logits = engine.decode_step(cache.ids, cache, self.pos)
            cache.step(logits)
            return logits
        self.graph, self.logits = _capture(dev, warm, body)
        cache.length = start

    def step(self):
        if self.cache.length + 1 > self.cache.max_len:
            raise RuntimeError('KV cache is full (%d)' % self.cache.max_len)
        self.graph.replay()
        self.cache.length += 1
        return self.logits


@torch.no_grad()
def _generate_beams(self, input_ids, images, bboxes, max_new_tokens, num_beams, eos_token_id, pad_token_id,
                    attention_mask, length_penalty, early_stopping, num_return_sequences, use_graph,
                    output_scores=False, output_logits=False, return_dict_in_generate=False):
    B, L = input_ids.shape
    N = int(num_beams)
    if not 1 <= num_return_sequences <= N:
        raise ValueError('num_return_sequences (%d) must be between 1 and num_beams (%d)' % (num_return_sequences, N))
    if max_new_tokens < 1:
        raise ValueError('max_new_tokens must be >= 1')
    eos = [] if eos_token_id is None else [int(e) for e in (eos_token_id if isinstance(eos_token_id, (list, tuple))
                                                               else [eos_token_id])]
    fill = (pad_token_id or eos[0]) if eos else -1        # HF's output_fill_value
    ids = input_ids.to(self.dev)
    cache = BeamCache(self.cfg, B, N, L, max_new_tokens, self.dev, eos, length_penalty, early_stopping, fill)
    run_ids, lens, _ = _right_padded(ids, attention_mask)
    logits = self.forward_device(run_ids, None if images is None else images.to(self.dev, self.dt),
                                 self.plan_boxes(bboxes), validate=True, last_only=True, seqlens=_seqlens(lens, L),
                                 cache=cache.prompt)
    cache.start(lens)
    want = output_scores or output_logits or return_dict_in_generate
    if want:
        cache.keep_outputs(logits.shape[-1], output_scores, output_logits, indices=True)
    cache.step(logits, first=True)
    stepper = None
    if use_graph and max_new_tokens > 4 and self.cfg.head_dim == 128:
        stepper = GraphedBeamDecode(self, cache)
    for _ in range(max_new_tokens):      # the max-length criterion ends the search by then
        if cache.done():
            break
        if stepper is not None:
            stepper.step()
        else:
            cache.step(self.decode_step(cache.ids, cache))
    if want:
        return cache.outputs(num_return_sequences, ids)
    return cache.result(num_return_sequences, ids)


PrefillEngine.decode_step = _decode_step
PrefillEngine.verify_step = _verify_step
PrefillEngine.generate = _generate


class GraphedPrefill:
    """CUDA-graph replay of PrefillEngine.forward_device for a fixed (B, L, box counts) shape:
    the ~1500 kernel launches of one prefill become one graph launch.  Inputs are staged through
    static device buffers; `run` accepts (pinned) host tensors."""

    def __init__(self, engine, input_ids, images, bboxes, last_only=True):
        self.eng = engine
        dev = engine.dev
        self.ids = input_ids.to(dev).clone()
        self.images = images.to(dev, engine.dt).clone()
        self.plan = engine.plan_boxes(bboxes)
        self.counts = None if bboxes is None else [0 if b is None else int(b.shape[0]) for b in bboxes]

        def body(validate=False):
            return engine.forward_device(self.ids, self.images, self.plan, validate=validate, last_only=last_only)

        def warm():
            body(validate=True)   # validation runs here only: it reads a status word back, which a capture cannot
            body()
        self.graph, self.out = _capture(dev, warm, body)

    def run(self, input_ids, images, bboxes):
        self.ids.copy_(input_ids, non_blocking=True)
        self.images.copy_(images, non_blocking=True)
        if self.plan is not None and self.plan['K'] > 0:
            counts = [0 if b is None else int(b.shape[0]) for b in bboxes]
            if counts != self.counts:
                raise ValueError('box counts differ from the captured shape')
            off = 0
            for b in bboxes:
                if b is not None and b.shape[0]:
                    self.plan['boxes'][off:off + b.shape[0]].copy_(b, non_blocking=True)
                    off += b.shape[0]
        self.graph.replay()
        return self.out


def random_state_dicts(cfg, device, seed=0, dtype=BF16):
    """Seeded random-init weights with the reference's parameter names and init scales
    (conv normal(0,0.01): layers.py:146-150,275-278; GN (1,0); HF defaults elsewhere).
    Used by bench.py / tests: no checkpoints are available offline."""
    g = torch.Generator(device=device)
    g.manual_seed(seed)

    def rn(*shape, std=0.02):
        return (torch.randn(*shape, generator=g, device=device, dtype=torch.float32) * std).to(dtype)

    C, D = cfg.vit_hidden, cfg.hidden
    vit = {'vision_model.embeddings.class_embedding': rn(C),
           'vision_model.embeddings.patch_embedding.weight': rn(C, 3, cfg.patch_size, cfg.patch_size),
           'vision_model.embeddings.position_embedding.weight': rn(cfg.num_patches + 1, C),
           'vision_model.pre_layrnorm.weight': torch.ones(C, device=device, dtype=dtype),
           'vision_model.pre_layrnorm.bias': torch.zeros(C, device=device, dtype=dtype)}
    for i in range(cfg.vit_layers):
        q = 'vision_model.encoder.layers.%d.' % i
        for n in ('q', 'k', 'v', 'out'):
            vit[q + 'self_attn.%s_proj.weight' % n] = rn(C, C)
            vit[q + 'self_attn.%s_proj.bias' % n] = rn(C)
        for n in ('layer_norm1', 'layer_norm2'):
            vit[q + n + '.weight'] = torch.ones(C, device=device, dtype=dtype)
            vit[q + n + '.bias'] = torch.zeros(C, device=device, dtype=dtype)
        vit[q + 'mlp.fc1.weight'], vit[q + 'mlp.fc1.bias'] = rn(cfg.vit_mlp, C), rn(cfg.vit_mlp)
        vit[q + 'mlp.fc2.weight'], vit[q + 'mlp.fc2.bias'] = rn(C, cfg.vit_mlp), rn(C)
    sd = {'model.embed_tokens.weight': rn(cfg.vocab, D), 'lm_head.weight': rn(cfg.vocab, D),
          'model.norm.weight': torch.ones(D, device=device, dtype=dtype),
          'model.mm_projector.weight': rn(D, C), 'model.mm_projector.bias': rn(D)}
    for i in range(cfg.n_layers):
        q = 'model.layers.%d.' % i
        for n in ('q', 'k', 'v', 'o'):
            sd[q + 'self_attn.%s_proj.weight' % n] = rn(D, D)
        sd[q + 'mlp.gate_proj.weight'], sd[q + 'mlp.up_proj.weight'] = rn(cfg.mlp, D), rn(cfg.mlp, D)
        sd[q + 'mlp.down_proj.weight'] = rn(D, cfg.mlp)
        sd[q + 'input_layernorm.weight'] = torch.ones(D, device=device, dtype=dtype)
        sd[q + 'post_attention_layernorm.weight'] = torch.ones(D, device=device, dtype=dtype)
    S = cfg.spi_dim
    p = 'model.spi_module.'
    for l in range(cfg.num_levels):
        sd[p + 'mlvl_fuse.input_conv.%d.weight' % l] = rn(S, S + 2, 1, 1, std=0.01)
        sd[p + 'mlvl_fuse.input_conv.%d.bias' % l] = torch.zeros(S, device=device, dtype=dtype)
        sd[p + 'roi_align.pconvs.%d.weight' % l] = rn(S, S, 3, 3, std=0.01)
        sd[p + 'roi_align.pconvs.%d.bias' % l] = torch.zeros(S, device=device, dtype=dtype)
    for r in range(5):
        sd[p + 'mlvl_fuse.fuse_convs.%d.conv.weight' % r] = rn(S, S, 3, 3, std=0.01)
        sd[p + 'mlvl_fuse.fuse_convs.%d.gn.weight' % r] = torch.ones(S, device=device, dtype=dtype)
        sd[p + 'mlvl_fuse.fuse_convs.%d.gn.bias' % r] = torch.zeros(S, device=device, dtype=dtype)
    q = p + 'roi_align.'
    sd[q + 'pos_embedd.0.weight'], sd[q + 'pos_embedd.0.bias'] = rn(256, 4, std=0.5), rn(256, std=0.1)
    sd[q + 'pos_embedd.2.weight'] = torch.ones(256, device=device, dtype=dtype)
    sd[q + 'pos_embedd.2.bias'] = torch.zeros(256, device=device, dtype=dtype)
    sd[q + 'pos_embedd.3.weight'], sd[q + 'pos_embedd.3.bias'] = rn(1024, 256, std=0.06), rn(1024, std=0.06)
    sd[q + 'pos_embedd.5.weight'] = torch.ones(1024, device=device, dtype=dtype)
    sd[q + 'pos_embedd.5.bias'] = torch.zeros(1024, device=device, dtype=dtype)
    sd[q + 'updims.weight'], sd[q + 'updims.bias'] = rn(D, 1024, std=0.03), rn(D, std=0.03)
    R = cfg.roi_out
    sd[q + 'flatten_linear.weight'] = rn(1024, S * R * R, std=0.002)
    sd[q + 'flatten_linear.bias'] = rn(1024, std=0.002)
    return sd, vit
