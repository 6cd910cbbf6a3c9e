"""Training step of the LLaMA stack (SURVEY.md 8(a) row 14 -- first slice).

The reference's stage-2 step (gpt4roi/train/train.py:698-712: HF Trainer over SPILlavaMPTForCausalLM under
bf16 autocast, DDP gradient all-reduce, AdamW with the parameter groups of llava_trainer.py:59-144) spends
6.48 B of its 7.04 B trainable parameters in the 32 LLaMA decoder layers.  This module is that part, built on
the sm_90a kernels only:

    inputs_embeds (from the region-token prefill front end: engine.PrefillEngine splice)
      -> 32 x [RMSNorm -> fused QKV GEMM + RoPE -> causal attention (saves LSE) -> o_proj + residual
               -> RMSNorm -> gate/up GEMM -> SwiGLU -> down_proj + residual]
      -> RMSNorm -> lm_head -> shifted cross entropy (llava/model/llava.py:238-249)
    backward: cross-entropy gradient -> lm_head -> ... every Linear through g4r_gemm_bf16_t
              (grad_x = grad_y.W, grad_W = grad_y^T.x, transposes in the UMMA descriptors), flash-attention
              backward, RoPE^T (= RoPE with -sin), SwiGLU / RMSNorm backward
    step: gradient all-reduce over NCCL (bucket = one decoder layer, overlapped with the rest of the
          backward on a side stream) + fused AdamW on fp32 master weights, bf16 copies for the next forward.

Returned beside the loss: the gradient w.r.t. inputs_embeds, which is what the not-yet-built backward of the
splice / projector / SPI module (RoIAlign backward kernels exist) will consume.

Precision: fp32 master weights and optimizer moments, bf16 weights/activations/gradients, fp32 accumulation
in every GEMM and reduction.  The reference keeps the residual stream in fp32 under autocast (fp32 embeddings,
`residual + bf16_branch` promotes); this first slice keeps it in bf16 like the inference path -- a stated
deviation, covered by the tolerance of the parity test (tests/test_train_gpu.py).
No PyTorch autograd, no torch.nn ops on the compute path: torch supplies device memory, streams and NCCL.
"""
import torch

from . import dense, kernels, train_ops

BF16 = torch.bfloat16
F32 = torch.float32

LAYER_KEYS = ('ln_in', 'wqkv', 'wo', 'ln_post', 'wgu', 'wdown')


def fuse_llama_layer(state_dict, i, device=None, dtype=F32):
    """HF LLaMA layer i -> the engine's fused layout: wqkv = [q; k; v], wgu = rows (gate_0, up_0, gate_1, up_1, ...)."""
    q = 'model.layers.%d.' % i
    cvt = lambda t: t.detach().to(device=device if device is not None else t.device, dtype=dtype).contiguous()
    wqkv = torch.cat([cvt(state_dict[q + 'self_attn.%s_proj.weight' % n]) for n in 'qkv'], 0).contiguous()
    g, u = cvt(state_dict[q + 'mlp.gate_proj.weight']), cvt(state_dict[q + 'mlp.up_proj.weight'])
    wgu = torch.stack([g, u], 1).reshape(2 * g.shape[0], g.shape[1]).contiguous()
    return dict(ln_in=cvt(state_dict[q + 'input_layernorm.weight']), wqkv=wqkv,
                wo=cvt(state_dict[q + 'self_attn.o_proj.weight']),
                ln_post=cvt(state_dict[q + 'post_attention_layernorm.weight']), wgu=wgu,
                wdown=cvt(state_dict[q + 'mlp.down_proj.weight']))


def unfuse_llama_layer(layer, i):
    """Inverse of fuse_llama_layer: fused layer dict -> HF / reference parameter names (views, no copies)."""
    q = 'model.layers.%d.' % i
    H = layer['wqkv'].shape[0] // 3
    return {q + 'self_attn.q_proj.weight': layer['wqkv'][:H], q + 'self_attn.k_proj.weight': layer['wqkv'][H:2 * H],
            q + 'self_attn.v_proj.weight': layer['wqkv'][2 * H:], q + 'self_attn.o_proj.weight': layer['wo'],
            q + 'mlp.gate_proj.weight': layer['wgu'][0::2], q + 'mlp.up_proj.weight': layer['wgu'][1::2],
            q + 'mlp.down_proj.weight': layer['wdown'], q + 'input_layernorm.weight': layer['ln_in'],
            q + 'post_attention_layernorm.weight': layer['ln_post']}


def save_checkpoint(state_dict, out_dir, max_shard_bytes=10 * 1024 ** 3, dtype=None, config=None, rank=None):
    """Write `state_dict` (reference parameter names) the way the reference's trainer does
    (train.py:88-98 -> Trainer._save -> save_pretrained): `pytorch_model-XXXXX-of-YYYYY.bin` shards,
    `pytorch_model.bin.index.json` and -- when `config` (a transformers config or a dict) is given -- `config.json`,
    so that SPILlavaMPTForCausalLM.from_pretrained(out_dir) loads it.  Only rank 0 writes (`rank` defaults to
    torch.distributed's rank, or 0); other ranks return [].  Resume needs the fp32 weights: pass dtype=None.
    Returns the shard file names."""
    import json
    import os
    if rank is None:
        import torch.distributed as dist
        rank = dist.get_rank() if (dist.is_available() and dist.is_initialized()) else 0
    if rank != 0:
        return []
    os.makedirs(out_dir, exist_ok=True)
    shards, cur, cur_bytes = [], {}, 0
    for k, v in state_dict.items():
        t = v.detach().to('cpu', dtype if dtype is not None else v.dtype).contiguous()
        if t.untyped_storage().nbytes() != t.numel() * t.element_size():
            t = t.clone()                 # a view of a larger (fused) storage: torch.save would write all of it
        nbytes = t.numel() * t.element_size()
        if cur and cur_bytes + nbytes > max_shard_bytes:
            shards.append(cur)
            cur, cur_bytes = {}, 0
        cur[k] = t
        cur_bytes += nbytes
    if cur:
        shards.append(cur)
    names = ['pytorch_model-%05d-of-%05d.bin' % (i + 1, len(shards)) for i in range(len(shards))]
    weight_map, total = {}, 0
    for name, shard in zip(names, shards):
        torch.save(shard, os.path.join(out_dir, name))
        for k, t in shard.items():
            weight_map[k] = name
            total += t.numel() * t.element_size()
    with open(os.path.join(out_dir, 'pytorch_model.bin.index.json'), 'w') as f:
        json.dump({'metadata': {'total_size': total}, 'weight_map': weight_map}, f, indent=2, sort_keys=True)
    if config is not None:
        if hasattr(config, 'save_pretrained'):
            config.save_pretrained(out_dir)
        else:
            with open(os.path.join(out_dir, 'config.json'), 'w') as f:
                json.dump(dict(config), f, indent=2, sort_keys=True)
    return names


def load_checkpoint(ckpt_dir):
    """Read a sharded HF checkpoint directory written by save_checkpoint / save_pretrained into one state dict."""
    import json
    import os
    with open(os.path.join(ckpt_dir, 'pytorch_model.bin.index.json')) as f:
        index = json.load(f)
    out = {}
    for name in sorted(set(index['weight_map'].values())):
        out.update(torch.load(os.path.join(ckpt_dir, name), map_location='cpu'))
    return out


def lr_lambda(step, total_steps, warmup_steps, kind='cosine'):
    """Multiplier of the base learning rate at optimizer step `step` (0-based), exactly transformers'
    get_cosine_schedule_with_warmup / get_linear_schedule_with_warmup / constant (the reference runs
    `--lr_scheduler_type cosine --warmup_ratio 0.003 [--warmup_steps 3000]`, train_stage1.sh:31-32,
    train_stage2.sh:47-53; HF: warmup_steps wins over warmup_ratio when > 0)."""
    import math
    if kind == 'constant' or total_steps is None:
        return 1.0
    if step < warmup_steps:
        return float(step) / float(max(1, warmup_steps))
    prog = float(step - warmup_steps) / float(max(1, total_steps - warmup_steps))
    if kind == 'linear':
        return max(0.0, 1.0 - prog)
    return max(0.0, 0.5 * (1.0 + math.cos(math.pi * prog)))


def warmup_steps_for(total_steps, warmup_steps=0, warmup_ratio=0.0):
    """transformers.TrainingArguments.get_warmup_steps."""
    import math
    return warmup_steps if warmup_steps > 0 else math.ceil(total_steps * warmup_ratio)


MATRIX_KEYS = ('wqkv', 'wo', 'wgu', 'wdown')      # bf16 gradients: one flat bucket per layer, in this order
NORM_KEYS = ('ln_in', 'ln_post')                  # fp32 gradients [hidden]: one [n_layers, 2, hidden] buffer


def layer_views(flat, cfg):
    """The four matrices of one decoder layer (engine layout: wqkv | wo | wgu | wdown) as views of one flat buffer."""
    H, F = cfg.hidden, cfg.mlp
    shapes = dict(wqkv=(3 * H, H), wo=(H, H), wgu=(2 * F, H), wdown=(H, F))
    out, o = {}, 0
    for k in MATRIX_KEYS:
        n = shapes[k][0] * shapes[k][1]
        out[k] = flat[o:o + n].view(shapes[k])
        o += n
    return out


def layer_numel(cfg):
    H, F = cfg.hidden, cfg.mlp
    return 3 * H * H + H * H + 2 * F * H + H * F


class LlamaTrainStack:
    """LLaMA decoder stack with explicit forward / backward / AdamW on the sm_90a kernels.

    Storage: per decoder layer ONE flat bf16 weight buffer (the four matrices are views of it) and, where this object
    owns the optimizer, flat fp32 master / moment buffers -- the whole vector, or this rank's 1/world slice of it
    (`shard=True`, the FSDP-equivalent of train_stage2.sh:51-52: gradients are reduce-scattered, AdamW runs on the
    slice, the updated bf16 slice is all-gathered back into the flat weight buffer).  lm_head is one more such
    buffer; norm weights (fp32 gradients, 4096 floats each) stay replicated.

    own_optimizer=False: no fp32 masters / moments are allocated -- the bf16 weights are refreshed from an external
    state dict (`load_weights`, the model-seam path where torch.optim owns the parameters).
    train_layers / train_head=False (stage 1, ONLY_SPI=1, train.py:685-696): the backward computes only the
    activation gradients (no weight-gradient GEMMs) and the optimizer skips those tensors."""

    def __init__(self, cfg, state_dict, device, lr=2e-5, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0,
                 own_optimizer=True, train_layers=True, train_head=True, shard=False, world=1, rank=0):
        """cfg: engine.EngineConfig; state_dict: HF names (model.layers.N..., model.norm.weight, lm_head.weight).
        weight_decay follows llava_trainer.py:59-144: decay on matrices, none on norm weights."""
        self.cfg, self.dev = cfg, torch.device(device)
        self.lr, self.betas, self.eps, self.wd = lr, betas, eps, weight_decay
        self.train_layers, self.train_head = train_layers, train_head
        self.step_count = 0
        if cfg.head_dim != 128:
            raise ValueError('LlamaTrainStack: head_dim 128 required (fused-RoPE QKV GEMM)')
        self.own_layers = own_optimizer and train_layers
        self.own_head = own_optimizer and train_head
        self.shard = bool(shard) and world > 1
        self.world, self.rank = (world, rank) if self.shard else (1, 0)
        n = layer_numel(cfg)
        nh = cfg.vocab * cfg.hidden
        if n % (self.world * 8) or nh % (self.world * 8):
            raise ValueError('sharded optimizer: the flat layer size must divide by 8 x world')
        self.slice = slice(self.rank * (n // self.world), (self.rank + 1) * (n // self.world))
        self.slice_head = slice(self.rank * (nh // self.world), (self.rank + 1) * (nh // self.world))
        self.wflat, self.w = [], []
        self.mflat, self.m1flat, self.m2flat = [], [], []
        self.master_ln, self.m1_ln, self.m2_ln = [], [], []
        for i in range(cfg.n_layers):
            fused = fuse_llama_layer(state_dict, i, self.dev, F32 if self.own_layers else BF16)
            flat = torch.empty(n, dtype=BF16, device=self.dev)
            views = layer_views(flat, cfg)
            for k in MATRIX_KEYS:
                views[k].copy_(fused[k])
            views['ln_in'], views['ln_post'] = fused['ln_in'].to(BF16), fused['ln_post'].to(BF16)
            self.wflat.append(flat)
            self.w.append(views)
            if self.own_layers:
                full = torch.cat([fused[k].reshape(-1) for k in MATRIX_KEYS]) if self.world == 1 else None
                if full is None:   # only this rank's slice is kept in fp32
                    full = torch.cat([fused[k].reshape(-1) for k in MATRIX_KEYS])[self.slice].clone()
                self.mflat.append(full)
                self.m1flat.append(torch.zeros_like(full))
                self.m2flat.append(torch.zeros_like(full))
                ln = dict(ln_in=fused['ln_in'].float().clone(), ln_post=fused['ln_post'].float().clone())
                self.master_ln.append(ln)
                self.m1_ln.append({k: torch.zeros_like(v) for k, v in ln.items()})
                self.m2_ln.append({k: torch.zeros_like(v) for k, v in ln.items()})
            del fused
        head = state_dict['lm_head.weight'].detach().to(self.dev)
        self.w_top = dict(norm=state_dict['model.norm.weight'].detach().to(self.dev, BF16).contiguous(),
                          lm_head=head.to(BF16).contiguous())
        if self.own_head:
            hf = head.to(F32).reshape(-1)
            self.mflat_head = hf[self.slice_head].clone() if self.world > 1 else hf.clone()
            self.m1_head, self.m2_head = torch.zeros_like(self.mflat_head), torch.zeros_like(self.mflat_head)
            self.master_norm = state_dict['model.norm.weight'].detach().to(self.dev, F32).contiguous().clone()
            self.m1_norm, self.m2_norm = torch.zeros_like(self.master_norm), torch.zeros_like(self.master_norm)
        del head
        self.pending = {}          # layer index (or 'head') -> all-gather work handle of its refreshed bf16 weights
        # AdamW runs on a side stream, one launch per layer in FORWARD order, each followed by an event: the next step's
        # forward waits per layer (layer 0's update is ready long before layer 31's), so the optimizer's HBM-bound 197 GB
        # of traffic hides behind the compute-bound GEMMs of the next forward instead of standing between two steps
        self.opt_stream = torch.cuda.Stream(device=self.dev) if (self.dev.type == 'cuda' and own_optimizer) else None
        self.opt_events = {}
        if self.opt_stream is not None:
            # these buffers are written by kernels queued on the side stream: tell the caching allocator, so that freeing
            # this object (end of a test, `del trainer` in bench.py) cannot hand their memory to a main-stream allocation
            # while the last update is still in flight
            persistent = list(self.wflat) + list(self.mflat) + list(self.m1flat) + list(self.m2flat)
            for d in list(self.master_ln) + list(self.m1_ln) + list(self.m2_ln):
                persistent += list(d.values())
            for w in self.w:
                persistent += [w['ln_in'], w['ln_post']]
            persistent += [self.w_top['norm'], self.w_top['lm_head']]
            if self.own_head:
                persistent += [self.mflat_head, self.m1_head, self.m2_head, self.master_norm, self.m1_norm, self.m2_norm]
            for t_ in persistent:
                if t_.is_cuda:
                    t_.record_stream(self.opt_stream)
        self._rope_cache = {}
        self.saved = None
        self.grads = None

    def load_weights(self, state_dict):
        """Refresh the bf16 compute weights in place from a reference-named state dict (any float dtype)."""
        H = self.cfg.hidden
        for i, w in enumerate(self.w):
            q = 'model.layers.%d.' % i
            for j, n in enumerate('qkv'):
                w['wqkv'][j * H:(j + 1) * H].copy_(state_dict[q + 'self_attn.%s_proj.weight' % n])
            w['wo'].copy_(state_dict[q + 'self_attn.o_proj.weight'])
            w['wgu'][0::2].copy_(state_dict[q + 'mlp.gate_proj.weight'])
            w['wgu'][1::2].copy_(state_dict[q + 'mlp.up_proj.weight'])
            w['wdown'].copy_(state_dict[q + 'mlp.down_proj.weight'])
            w['ln_in'].copy_(state_dict[q + 'input_layernorm.weight'])
            w['ln_post'].copy_(state_dict[q + 'post_attention_layernorm.weight'])
        self.w_top['norm'].copy_(state_dict['model.norm.weight'])
        self.w_top['lm_head'].copy_(state_dict['lm_head.weight'])

    def _full(self, shard_t, group=None):
        """fp32 slice -> the whole vector (all-gather over the data-parallel group when sharded)."""
        if self.world == 1:
            return shard_t
        import torch.distributed as dist
        out = torch.empty(shard_t.numel() * self.world, dtype=shard_t.dtype, device=shard_t.device)
        dist.all_gather_into_tensor(out, shard_t.contiguous(), group=group)
        return out

    def _named(self, flats, lns, head, norm):
        out = {}
        for i in range(len(self.w)):
            d = dict(layer_views(self._full(flats[i]), self.cfg))
            d['ln_in'], d['ln_post'] = lns[i]['ln_in'], lns[i]['ln_post']
            out.update(unfuse_llama_layer(d, i))
        if head is not None:
            out['lm_head.weight'] = self._full(head).view(self.cfg.vocab, self.cfg.hidden)
            out['model.norm.weight'] = norm
        return out

    def state_dict(self):
        """Weights under the reference's parameter names: the fp32 masters where this object owns the optimizer
        (gathered from the ranks' slices when sharded -- a collective call: every rank must make it), else the bf16
        compute copies."""
        self.sync_optimizer()
        if self.own_layers:
            out = self._named(self.mflat, self.master_ln, None, None)
        else:
            out = {}
            for i, w in enumerate(self.w):
                out.update(unfuse_llama_layer(w, i))
        if self.own_head:
            out['lm_head.weight'] = self._full(self.mflat_head).view(self.cfg.vocab, self.cfg.hidden)
            out['model.norm.weight'] = self.master_norm
        else:
            out['model.norm.weight'], out['lm_head.weight'] = self.w_top['norm'], self.w_top['lm_head']
        return out

    def moments(self):
        """(exp_avg, exp_avg_sq) under reference names for the tensors this object optimises (collective if sharded)."""
        self.sync_optimizer()
        m1, m2 = {}, {}
        if self.own_layers:
            m1.update(self._named(self.m1flat, self.m1_ln, None, None))
            m2.update(self._named(self.m2flat, self.m2_ln, None, None))
        if self.own_head:
            for d, h, nrm in ((m1, self.m1_head, self.m1_norm), (m2, self.m2_head, self.m2_norm)):
                d['lm_head.weight'] = self._full(h).view(self.cfg.vocab, self.cfg.hidden)
                d['model.norm.weight'] = nrm
        return m1, m2

    def load_moments(self, exp_avg, exp_avg_sq):
        for src, flats, lns, head, nrm in ((exp_avg, self.m1flat, self.m1_ln, 'm1_head', 'm1_norm'),
                                           (exp_avg_sq, self.m2flat, self.m2_ln, 'm2_head', 'm2_norm')):
            if self.own_layers:
                for i in range(len(self.w)):
                    fused = fuse_llama_layer(src, i, self.dev)
                    full = torch.cat([fused[k].reshape(-1) for k in MATRIX_KEYS])
                    flats[i].copy_(full[self.slice] if self.world > 1 else full)
                    lns[i]['ln_in'].copy_(fused['ln_in'])
                    lns[i]['ln_post'].copy_(fused['ln_post'])
            if self.own_head:
                hf = src['lm_head.weight'].to(self.dev, F32).reshape(-1)
                getattr(self, head).copy_(hf[self.slice_head] if self.world > 1 else hf)
                getattr(self, nrm).copy_(src['model.norm.weight'])

    # ------------------------------------------------------------------ helpers
    def _rope(self, L):
        if L not in self._rope_cache:
            c = self.cfg
            inv = 1.0 / (c.rope_theta ** (torch.arange(0, c.head_dim, 2, dtype=torch.int64).float() / c.head_dim))
            emb = torch.cat([torch.arange(L, dtype=F32)[:, None] * inv[None, :]] * 2, -1)
            cos, sin = emb.cos().to(self.dev, BF16).contiguous(), emb.sin().to(self.dev, BF16).contiguous()
            self._rope_cache[L] = (cos, sin, (-sin).contiguous())
        return self._rope_cache[L]

    def _wait_weights(self, key):
        """Sharded optimizer: the all-gather that refreshes this layer's bf16 weights was launched by the last
        optimizer step on the side stream; the forward waits for it only here, right before the first use."""
        h = self.pending.pop(key, None)
        if h is not None:
            h.wait()
        ev = self.opt_events.pop(key, None)
        if ev is not None:
            torch.cuda.current_stream(self.dev).wait_event(ev)

    def sync_optimizer(self):
        """Make the current stream wait for every optimizer update still in flight on the side stream."""
        if self.opt_stream is not None:
            torch.cuda.current_stream(self.dev).wait_stream(self.opt_stream)
        self.opt_events.clear()

    # ------------------------------------------------------------------ forward
    def forward(self, inputs_embeds, targets, seqlens=None):
        """inputs_embeds [B, L, hidden] bf16; targets int64 [B, L]: labels shifted left by one
        (targets[:, t] = labels[:, t+1], targets[:, -1] = -100).  Returns the mean loss (0-d fp32 tensor)."""
        c = self.cfg
        B, L, Hd = inputs_embeds.shape
        M = B * L
        cos, sin, _ = self._rope(L)
        scale = c.head_dim ** -0.5
        x = inputs_embeds.reshape(M, Hd).contiguous()
        saved = []
        for li, w in enumerate(self.w):
            self._wait_weights(li)
            h1 = kernels.rmsnorm(x, w['ln_in'], c.rms_eps)
            qkv = dense.qkv_rope(h1, w['wqkv'], cos, sin, L, 2 * c.hidden)
            a, lse = train_ops.attention_fwd_lse(qkv, B, L, c.n_heads, c.head_dim, True, scale)
            x_mid = dense.linear(a, w['wo'], residual=x)
            h2 = kernels.rmsnorm(x_mid, w['ln_post'], c.rms_eps)
            gu = dense.linear(h2, w['wgu'])
            f = train_ops.swiglu_fwd(gu)
            x_out = dense.linear(f, w['wdown'], residual=x_mid)
            saved.append(dict(x_in=x, h1=h1, qkv=qkv, a=a, lse=lse, x_mid=x_mid, h2=h2, gu=gu, f=f))
            x = x_out
        self._wait_weights('head')
        hn = kernels.rmsnorm(x, self.w_top['norm'], c.rms_eps)
        vpad = (c.vocab + 63) // 64 * 64                       # 16-byte-aligned logits rows
        logits = torch.empty((M, vpad), dtype=BF16, device=self.dev)[:, :c.vocab]
        dense.linear(hn, self.w_top['lm_head'], out=logits)
        self.saved = dict(layers=saved, x_last=x, hn=hn, logits=logits, targets=targets.reshape(M).contiguous(), B=B, L=L)
        loss, count, _ = train_ops.cross_entropy(logits, self.saved['targets'], want_grad=False)
        return loss

    # ------------------------------------------------------------------ backward
    def backward(self, loss_scale=1.0, on_layer_grads=None, on_top_grads=None):
        """Gradients of loss_scale * loss.  Fills self.grads and returns the gradient w.r.t. inputs_embeds
        [B, L, hidden] (bf16).  Per decoder layer the four matrix gradients (bf16) are views of ONE flat buffer
        (`g['flat']`, the DDP bucket: one collective per layer) and the two norm-weight gradients rows of one
        fp32 [n_layers, 2, hidden] buffer.  on_top_grads(g_top) fires as soon as the lm_head / final-norm
        gradients exist (start of the backward), on_layer_grads(i, g) when decoder layer i's are complete."""
        c, s = self.cfg, self.saved
        B, L = s['B'], s['L']
        _, _, nsin = self._rope(L)
        cos = self._rope(L)[0]
        scale = c.head_dim ** -0.5
        _, _, dlogits = train_ops.cross_entropy(s['logits'], s['targets'], grad_scale=loss_scale, want_grad=True)
        g_top = {}
        if self.train_head:
            g_top['lm_head'] = dense.matmul_t(dlogits, s['hn'], a_mn=True, b_mn=True)           # dW = dY^T X
            g_top['flat'] = g_top['lm_head'].view(-1)
        dhn = dense.matmul_t(dlogits, self.w_top['lm_head'], b_mn=True)                          # dX = dY W
        del dlogits
        dx, gn = train_ops.rmsnorm_bwd(s['x_last'], self.w_top['norm'], dhn, c.rms_eps)
        if self.train_head:
            g_top['norm'] = gn
            if on_top_grads is not None:
                on_top_grads(g_top)
        nl = len(self.w)
        grads = [None] * nl
        norm_g = torch.empty((nl, 2, c.hidden), dtype=F32, device=self.dev) if self.train_layers else None
        tl = self.train_layers
        for i in range(nl - 1, -1, -1):
            w, a = self.w[i], s['layers'][i]
            g = {}
            if tl:
                shapes = [w[k].shape for k in MATRIX_KEYS]
                flat = torch.empty(sum(sh.numel() for sh in shapes), dtype=BF16, device=self.dev)
                o = 0
                for k, sh in zip(MATRIX_KEYS, shapes):
                    g[k] = flat[o:o + sh.numel()].view(sh)
                    o += sh.numel()
                g['flat'] = flat
            # x_out = x_mid + down(f)
            if tl:
                dense.matmul_t(dx, a['f'], a_mn=True, b_mn=True, out=g['wdown'])
            df = dense.matmul_t(dx, w['wdown'], b_mn=True)
            dgu = train_ops.swiglu_bwd(a['gu'], df)
            if tl:
                dense.matmul_t(dgu, a['h2'], a_mn=True, b_mn=True, out=g['wgu'])
            dh2 = dense.matmul_t(dgu, w['wgu'], b_mn=True)
            dx_mid, gln = train_ops.rmsnorm_bwd(a['x_mid'], w['ln_post'], dh2, c.rms_eps, dres=dx)
            if tl:
                norm_g[i, 1].copy_(gln)
                g['ln_post'] = norm_g[i, 1]
            # x_mid = x_in + o_proj(attn)
            if tl:
                dense.matmul_t(dx_mid, a['a'], a_mn=True, b_mn=True, out=g['wo'])
            da = dense.matmul_t(dx_mid, w['wo'], b_mn=True)
            dqkv = train_ops.attention_bwd(a['qkv'], a['a'], da, a['lse'], B, L, c.n_heads, c.head_dim, True, scale)
            kernels.rope_inplace(dqkv, cos, nsin, L, 2 * c.n_heads, c.head_dim)             # RoPE^T = RoPE(-theta)
            if tl:
                dense.matmul_t(dqkv, a['h1'], a_mn=True, b_mn=True, out=g['wqkv'])
            dh1 = dense.matmul_t(dqkv, w['wqkv'], b_mn=True)
            dx, gln = train_ops.rmsnorm_bwd(a['x_in'], w['ln_in'], dh1, c.rms_eps, dres=dx_mid)
            if tl:
                norm_g[i, 0].copy_(gln)
                g['ln_in'] = norm_g[i, 0]
            grads[i] = g
            s['layers'][i] = None                                                            # free activations
            if tl and on_layer_grads is not None:
                on_layer_grads(i, g)
        self.grads = dict(layers=grads, top=g_top, norms=norm_g)
        self.saved = None
        return dx.view(B, L, c.hidden)

    def grad_tensors(self):
        """(sharded, replicated) contiguous gradient tensors of this stack for the global norm.  Sharded mode: the
        reduce-scattered slices (each rank holds a different 1/world of the summed gradient); replicated tensors are
        identical on every rank after their all-reduce."""
        sharded, repl = [], []
        if self.train_layers:
            (sharded if self.shard else repl).extend(g['rs'] if self.shard else g['flat'] for g in self.grads['layers'])
            repl.append(self.grads['norms'])
        if self.train_head:
            (sharded if self.shard else repl).append(self.grads['top']['rs'] if self.shard else self.grads['top']['flat'])
            repl.append(self.grads['top']['norm'])
        return sharded, repl

    def grads_state_dict(self):
        """Gradients under the reference's parameter names (views; model-seam path, unsharded)."""
        out = {}
        if self.train_layers:
            for i, g in enumerate(self.grads['layers']):
                out.update(unfuse_llama_layer(g, i))
        if self.train_head:
            out['model.norm.weight'], out['lm_head.weight'] = self.grads['top']['norm'], self.grads['top']['lm_head']
        return out

    # ------------------------------------------------------------------ optimizer
    def optimizer_step(self, grad_scale=1.0, lr=None, scale_dev=None, reducer=None):
        """Fused AdamW on every trained tensor: ONE launch per decoder layer over the flat fp32 master / moments (or
        this rank's slice of them), writing the refreshed bf16 weights straight into the flat weight buffer; sharded
        mode then all-gathers each layer's bf16 slice (async on the reducer's stream; the next forward waits per layer)."""
        self.step_count += 1
        t = self.step_count
        lr = self.lr if lr is None else lr

        def upd(master, m1, m2, w16, grad, decay):
            train_ops.adamw_step(master.view(-1), grad.reshape(-1), m1.view(-1), m2.view(-1), w16.reshape(-1), lr,
                                 self.betas, self.eps, self.wd if decay else 0.0, t, grad_scale, scale_dev)
        side = self.opt_stream if (self.opt_stream is not None and not self.shard) else None
        if side is not None:
            side.wait_stream(torch.cuda.current_stream(self.dev))     # gradients, clip coefficient
            ctx = torch.cuda.stream(side)
        else:
            import contextlib
            ctx = contextlib.nullcontext()
        with ctx:
            if self.own_layers:
                if side is not None:
                    self.grads['norms'].record_stream(side)
                for i, g in enumerate(self.grads['layers']):
                    w16 = self.wflat[i][self.slice] if self.shard else self.wflat[i]
                    gflat = g['rs'] if self.shard else g['flat']
                    upd(self.mflat[i], self.m1flat[i], self.m2flat[i], w16, gflat, True)
                    if self.shard:
                        self.pending[i] = reducer.all_gather(self.wflat[i], w16)
                    for k in NORM_KEYS:
                        upd(self.master_ln[i][k], self.m1_ln[i][k], self.m2_ln[i][k], self.w[i][k], g[k], False)
                    if side is not None:
                        gflat.record_stream(side)       # the allocator may reuse the buffer only after this update ran
                        ev = torch.cuda.Event()
                        ev.record(side)
                        self.opt_events[i] = ev
            if self.own_head:
                hflat = self.w_top['lm_head'].view(-1)
                w16 = hflat[self.slice_head] if self.shard else hflat
                gtop = self.grads['top']['rs'] if self.shard else self.grads['top']['flat']
                upd(self.mflat_head, self.m1_head, self.m2_head, w16, gtop, True)
                if self.shard:
                    self.pending['head'] = reducer.all_gather(hflat, w16)
                upd(self.master_norm, self.m1_norm, self.m2_norm, self.w_top['norm'], self.grads['top']['norm'], False)
                if side is not None:
                    gtop.record_stream(side)
                    self.grads['top']['norm'].record_stream(side)
                    ev = torch.cuda.Event()
                    ev.record(side)
                    self.opt_events['head'] = ev
        if side is not None and scale_dev is not None:
            scale_dev.record_stream(side)
        self.grads = None


class LayerBucketAllReduce:
    """DDP gradient all-reduce (NCCL over NVLink; gloo in the CPU tests): ONE collective per decoder layer -- the
    layer's flat bf16 gradient buffer -- launched from the backward hook on a side stream so that the collective of
    layer i overlaps the backward of layers < i; the lm_head / final-norm gradients go out at the start of the
    backward, the small fp32 tensors (norm weights, front end) as one flat buffer at the end.
    Sums in place; the 1/world average is folded into AdamW's grad_scale.
    reduce_fp32=True all-reduces an fp32 copy of each bucket (the reference's DDP/FSDP reduce fp32 gradients)."""

    def __init__(self, group=None, reduce_fp32=False, shard_grads=False):
        """shard_grads=True: the per-layer buckets are reduce-scattered instead of all-reduced (each rank receives
        1/world of the summed gradient) -- used with the sharded optimizer of LlamaTrainStack(shard=True)."""
        import torch.distributed as dist
        self.dist, self.group = dist, group
        self.handles = []
        self.reduce_fp32 = reduce_fp32
        self.shard_grads = shard_grads
        self.calls = 0
        self.stream = torch.cuda.Stream() if torch.cuda.is_available() else None

    def active(self):
        return self.dist.is_available() and self.dist.is_initialized() and self.dist.get_world_size(self.group) > 1

    def _issue(self, tensors):
        for t in tensors:
            self.calls += 1
            if self.reduce_fp32 and t.dtype != F32:
                t32 = t.float()
                h = self.dist.all_reduce(t32, group=self.group, async_op=True)
                self.handles.append((h, t, t32))
            else:
                self.handles.append((self.dist.all_reduce(t, group=self.group, async_op=True), None, None))

    def reduce_now(self, tensors):
        if not self.active():
            return
        tensors = [t for t in tensors if t is not None]
        if self.stream is not None and tensors and tensors[0].is_cuda:
            self.stream.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(self.stream):
                self._issue(tensors)
        else:
            self._issue(tensors)

    def hook(self, i, grads):
        if self.shard_grads and 'flat' in grads:
            grads['rs'] = self.reduce_scatter(grads['flat'])
            return
        self.reduce_now([grads['flat']] if 'flat' in grads else [grads[k] for k in LAYER_KEYS])

    def top_hook(self, g_top):
        if self.shard_grads and 'flat' in g_top:
            g_top['rs'] = self.reduce_scatter(g_top['flat'])
            return
        self.reduce_now([g_top.get('lm_head')])

    def reduce_scatter(self, flat):
        """Sum `flat` over the ranks, this rank keeping slice [rank*n/world, (rank+1)*n/world) (bf16 in, bf16 out):
        the gradient half of the FSDP-equivalent step.  Async on the side stream; returns the output slice tensor
        (valid after wait())."""
        world = self.dist.get_world_size(self.group)
        out = torch.empty(flat.numel() // world, dtype=flat.dtype, device=flat.device)
        self.calls += 1
        if self.stream is not None and flat.is_cuda:
            self.stream.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(self.stream):
                h = self.dist.reduce_scatter_tensor(out, flat, group=self.group, async_op=True)
        else:
            h = self.dist.reduce_scatter_tensor(out, flat, group=self.group, async_op=True)
        self.handles.append((h, None, None))
        return out

    def all_gather(self, full, mine):
        """In-place all-gather of every rank's slice into `full` (`mine` is this rank's slice OF `full`): the weight
        half of the FSDP-equivalent step.  Async on the side stream; returns the work handle (wait() before use)."""
        self.calls += 1
        if self.stream is not None and full.is_cuda:
            self.stream.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(self.stream):
                return self.dist.all_gather_into_tensor(full, mine, group=self.group, async_op=True)
        return self.dist.all_gather_into_tensor(full, mine, group=self.group, async_op=True)

    def wait(self):
        for h, dst, src in self.handles:
            h.wait()                       # the current stream waits for the collective
            if dst is not None:
                dst.copy_(src)
        self.handles = []
        if self.stream is not None:
            torch.cuda.current_stream().wait_stream(self.stream)


def train_step(stack, inputs_embeds, targets, reducer=None, world_size=1):
    """One optimisation step of the LLaMA stack: forward, backward (+ overlapped gradient all-reduce), AdamW.
    Returns (loss tensor, d_inputs_embeds)."""
    loss = stack.forward(inputs_embeds, targets)
    d_in = stack.backward(on_layer_grads=reducer.hook if reducer is not None else None,
                          on_top_grads=reducer.top_hook if reducer is not None else None)
    if reducer is not None:
        reducer.reduce_now([stack.grads['norms'], stack.grads['top']['norm']])
        reducer.wait()
    stack.optimizer_step(grad_scale=1.0 / world_size)
    return loss, d_in


def bootstrap_stage2(stage1_dir, stage2_dir):
    """train_stage2.sh:10-24: when the stage-2 work dir has no checkpoint yet, create `checkpoint-0` in it and soft-link
    every stage-1 file EXCEPT the optimizer / scheduler / trainer state (`scheduler.pt`, `training_args.bin`,
    `optimizer.pt`, `trainer_state.json`, and this package's optimizer file), so that stage 2 starts from the stage-1
    weights with a fresh optimizer.  Returns the checkpoint directory to load (the newest `checkpoint-*` when one exists:
    "WORKDIR is not empty, resume training")."""
    import os
    existing = sorted((d for d in os.listdir(stage2_dir) if os.path.isdir(os.path.join(stage2_dir, d))),
                      key=lambda d: (int(d.split('-')[-1]) if d.split('-')[-1].isdigit() else -1)) if os.path.isdir(stage2_dir) else []
    if existing:
        return os.path.join(stage2_dir, existing[-1])
    if not os.path.isdir(stage1_dir):
        raise FileNotFoundError('Stage1 work directory %s does not exist.' % stage1_dir)
    ck = os.path.join(stage2_dir, 'checkpoint-0')
    os.makedirs(ck, exist_ok=True)
    skip = {'scheduler.pt', 'training_args.bin', 'optimizer.pt', 'trainer_state.json', 'g4r_optimizer.pt'}
    for name in sorted(os.listdir(stage1_dir)):
        src = os.path.join(stage1_dir, name)
        if os.path.isfile(src) and name not in skip:
            dst = os.path.join(ck, name)
            if not os.path.lexists(dst):
                os.symlink(os.path.abspath(src), dst)
    return ck


def apply_delta(base_state_dict, delta_state_dict):
    """scripts/apply_delta.py:15-43 on state dicts: GPT4RoI's released weights are a DELTA over LLaMA-7B.
    target[name] = delta[name] + base[name]; `mm_projector.*` / `spi_module.*` exist only in the delta and are kept;
    `embed_tokens` / `lm_head` have 6 more rows than the base (the added special tokens): the base is added to the
    leading block.  Any other name missing from the base raises NameError, like the script.  Modifies and returns delta."""
    for name, param in delta_state_dict.items():
        if name not in base_state_dict:
            if name in ('model.mm_projector.weight', 'model.mm_projector.bias') or 'spi_module' in name:
                continue
            raise NameError(name)
        bparam = base_state_dict[name].to(device=param.device, dtype=param.dtype)
        if param.shape == bparam.shape:
            param += bparam
        else:
            assert name in ('model.embed_tokens.weight', 'lm_head.weight'), \
                '%s dimension mismatch: %s vs %s' % (name, tuple(param.shape), tuple(bparam.shape))
            param[:bparam.shape[0], :bparam.shape[1]] += bparam
    return delta_state_dict


class FrontEndTrain:
    """Training-mode front end: the region-token forward up to `inputs_embeds` with the tensors its backward needs,
    and the backward of everything in front of the LLaMA stack that stage 2 trains: splice
    (`spi_llava.py:99-196`), `embed_tokens`, `mm_projector` and the whole SPI module (`SpiTrain`).  The CLIP tower
    is frozen in both stages (train.py:604-612) and is not differentiated.
    head_only=True stops at the pconv output / position-MLP input and returns those hand-over gradients
    (`d_pconv_out`, `d_pos`) instead of running SpiTrain (kept for the slice-level test)."""

    def __init__(self, engine, head_only=False):
        self.eng = engine
        self.head_only = head_only
        self.spi = SpiTrain(engine)
        self.saved = None

    def forward(self, input_ids, images, bboxes):
        from .roi_align import roi_align_mlvl
        from .splice import splice_region_tokens
        eng, c = self.eng, self.eng.cfg
        dev = eng.dev
        input_ids = input_ids.to(dev)
        images = images.to(dev, BF16)
        B, L = input_ids.shape
        plan_b = eng.plan_boxes(bboxes)
        taps = eng.vit(images)
        feat = kernels.cast_tokens_f32_bf16(taps[c.select_index])
        img_rows = dense.linear(feat, eng.proj_w, eng.proj_b).view(B, c.num_patches, c.hidden)
        K = plan_b['K'] if plan_b is not None else 0
        region, pc, t = None, None, None
        if K > 0 and not self.head_only:
            region = (self.spi.forward(taps, plan_b), plan_b['offs'])
        elif K > 0:
            maps, ss = eng.fuse_maps(taps)
            boxes, bidx = plan_b['boxes'], plan_b['bidx']
            rois = torch.cat([bidx[:, None], boxes * float(c.image_size)], 1).contiguous()
            scales = [float(torch.tensor(1.0 / s, dtype=F32)) for s in c.strides]
            feats = roi_align_mlvl(maps, rois, c.roi_out, scales, c.roi_sampling, True, out_dtype=BF16,
                                   gn_scale=[s for s, _ in ss], gn_shift=[b for _, b in ss])
            R = c.roi_out
            pc = dense.conv_nhwc(feats.view(c.num_levels * K, R, R, c.spi_dim), eng.pconv_w, eng.pconv_b,
                                 act='relu', levels=c.num_levels).view(K, -1)
            acc = dense.linear(pc, eng.flat_w, out_dtype=F32)
            pos = kernels.pos_embed_mlp(boxes.contiguous(), *eng.pos)
            t = kernels.add_bias_pos_cast(acc, eng.flat_b, pos)
            region = (dense.linear(t, eng.up_w, eng.up_b), plan_b['offs'])
        elif plan_b is not None:
            region = (torch.zeros((1, c.hidden), dtype=BF16, device=dev), plan_b['offs'])
        embeds, plan = splice_region_tokens(input_ids, eng.embed, img_rows, region, c.num_patches, c.im_patch_token,
                                            c.im_start_token, c.im_end_token, c.bbox_token, return_plan=True)
        self.saved = dict(feat=feat, plan=plan, pc=pc, t=t, K=K, B=B)
        return embeds

    def backward(self, d_embeds, want_embed=True, want_proj=True, want_spi=True):
        """d_embeds [B,L,hidden] bf16 -> dict of gradients under the reference's parameter names.
        want_*: skip the gradients of frozen groups (stage 1 trains the SPI module only, train.py:685-696)."""
        from .splice import splice_backward
        eng, c, s = self.eng, self.eng.cfg, self.saved
        d_image, d_region, d_embed = splice_backward(s['plan'], d_embeds, c.num_patches, s['K'], c.vocab,
                                                     want_embed_grad=want_embed)
        out = {}
        if want_embed:
            out['model.embed_tokens.weight'] = d_embed
        if want_proj:
            _, gw, gb = train_ops.linear_bwd(s['feat'], eng.proj_w, d_image.view(-1, c.hidden), need_dx=False)
            out['model.mm_projector.weight'], out['model.mm_projector.bias'] = gw, gb
        if s['K'] > 0 and not self.head_only and want_spi:
            out.update(self.spi.backward(d_region))
        elif s['K'] > 0 and not self.head_only:
            pass
        elif s['K'] > 0:
            q = 'model.spi_module.roi_align.'
            dt, out[q + 'updims.weight'], out[q + 'updims.bias'] = train_ops.linear_bwd(s['t'], eng.up_w, d_region)
            out[q + 'flatten_linear.bias'] = train_ops.colsum(dt)
            d_pc, gfw, _ = train_ops.linear_bwd(s['pc'], eng.flat_w, dt, has_bias=False)
            # engine layout of flatten_linear.weight is [out, (ph, pw, c)]; the reference's is [out, (c, ph, pw)]
            R, C = c.roi_out, c.spi_dim
            out[q + 'flatten_linear.weight'] = gfw.view(-1, R, R, C).permute(0, 3, 1, 2).reshape(gfw.shape[0], -1)
            out['d_pos'] = dt
            out['d_pconv_out'] = d_pc
        self.saved = None
        return out


class SpiTrain:
    """Forward (with saved activations) and complete backward of the SPI module -- MLVLROIQueryModule
    (gpt4roi/models/layers.py:198-236): pyramid upsampling, MLVLFuseModule (4 input 1x1 convs + 5 shared
    ConvModule(3x3, GN(64), ReLU) rounds with the channel shuffle between levels), MlvlRoIExtractor (4 RoIAligns,
    4 pconvs, flatten_linear, box position MLP, updims) -- on the sm_90a kernels, no autograd.
    Inputs: the CLIP hidden states (frozen tower) and the boxes; output: one region token per box.
    `backward(d_region)` returns gradients under the reference's parameter names and layouts (fp32 or bf16)."""

    def __init__(self, engine):
        self.eng = engine
        self.saved = None

    def forward(self, taps, plan_b, has_cls=True):
        """taps: {layer: [B,1+P,C]} ViT hidden states, or (has_cls=False) a list of [B,P,C] token maps in level order."""
        from .roi_align import roi_align_mlvl
        eng, c = self.eng, self.eng.cfg
        C, n = c.spi_dim, c.num_levels
        if isinstance(taps, (list, tuple)):
            taps = {layer: t for layer, t in zip(c.level_layers, taps)}
        B = next(iter(taps.values())).shape[0]
        ups, maps = [], []
        for l, layer in enumerate(c.level_layers):
            H = c.level_sizes[l]
            up = kernels.upsample_tokens_coords(taps[layer], c.grid, H, eng.spi_cpad, has_cls=has_cls)
            ups.append(up)
            maps.append(dense.linear(up.view(-1, eng.spi_cpad), eng.in_w[l], eng.in_b[l]).view(B, H, H, C))
        zs, sts, sss = [maps], [None], [[None] * n]
        for r in range(5):
            new, stats = [], []
            prev, ss = zs[-1], sss[-1]
            for l in range(n):
                top, down = min(l + 1, n - 1), max(l - 1, 0)
                x_in = kernels.fuse_gather(prev[l], prev[top], prev[down], ss[l], ss[top], ss[down])
                st = torch.zeros((B, dense.gn_slots(c.level_sizes[l], c.level_sizes[l]), c.gn_groups, 2), dtype=F32, device=eng.dev)
                new.append(dense.conv_nhwc(x_in, eng.fuse[r]['w'], gn_stats=st))
                stats.append(st)
            zs.append(new)
            sts.append(stats)
            sss.append([kernels.gn_finalize(stats[l], eng.fuse[r]['gamma'], eng.fuse[r]['beta'],
                                            count=c.level_sizes[l] ** 2 * (C // c.gn_groups)) for l in range(n)])
        boxes, bidx = plan_b['boxes'], plan_b['bidx']
        K = boxes.shape[0]
        rois = torch.cat([bidx[:, None], boxes * float(c.image_size)], 1).contiguous()
        scales = [float(torch.tensor(1.0 / s, dtype=F32)) for s in c.strides]
        ss = sss[-1]
        feats = roi_align_mlvl(zs[-1], rois, c.roi_out, scales, c.roi_sampling, True, out_dtype=BF16,
                               gn_scale=[s for s, _ in ss], gn_shift=[b for _, b in ss])
        R = c.roi_out
        pc = dense.conv_nhwc(feats.view(n * K, R, R, C), eng.pconv_w, eng.pconv_b, act='relu', levels=n)
        acc = dense.linear(pc.view(K, -1), eng.flat_w, out_dtype=F32)
        pos = kernels.pos_embed_mlp(boxes.contiguous(), *eng.pos)
        t = kernels.add_bias_pos_cast(acc, eng.flat_b, pos)
        region = dense.linear(t, eng.up_w, eng.up_b)
        self.saved = dict(ups=ups, zs=zs, sts=sts, sss=sss, rois=rois, scales=scales, feats=feats, pc=pc, t=t,
                          boxes=boxes.contiguous(), K=K, B=B)
        return region

    def backward(self, d_region):
        from .roi_align import roi_align_mlvl_backward
        eng, c, s = self.eng, self.eng.cfg, self.saved
        C, n, R, K, B = c.spi_dim, c.num_levels, c.roi_out, s['K'], s['B']
        p = 'model.spi_module.'
        q = p + 'roi_align.'
        g = {}
        # ---- head: updims, + pos, flatten_linear (layers.py:326-335)
        dt, g[q + 'updims.weight'], g[q + 'updims.bias'] = train_ops.linear_bwd(s['t'], eng.up_w, d_region)
        g[q + 'flatten_linear.bias'] = train_ops.colsum(dt)
        for name, v in train_ops.pos_embed_mlp_bwd(s['boxes'], eng.pos, dt).items():
            g[q + 'pos_embedd.' + name] = v
        pcf = s['pc'].view(K, -1)
        d_pc, gfw, _ = train_ops.linear_bwd(pcf, eng.flat_w, dt, has_bias=False)
        g[q + 'flatten_linear.weight'] = gfw.view(-1, R, R, C).permute(0, 3, 1, 2).reshape(gfw.shape[0], -1)
        # ---- relu(sum_l pconv_l(roi_feats_l))  (layers.py:318-325)
        dZ = train_ops.relu_bwd(d_pc, pcf).view(K, R, R, C)
        gb = train_ops.colsum(dZ.view(-1, C))
        feats = s['feats'].view(n, K, R, R, C)
        d_feats = torch.empty_like(feats)
        for l in range(n):
            wl = eng.pconv_w[:, l]                                       # [Cout, 3, 3, Cin], rows n*9*Cin apart
            dx, dW = train_ops.conv3x3_bwd(feats[l], wl, dZ)
            d_feats[l] = dx
            g[q + 'pconvs.%d.weight' % l] = dW.permute(0, 3, 1, 2)
            g[q + 'pconvs.%d.bias' % l] = gb
        # ---- 4 x RoIAlign (the forward fused the last GroupNorm+ReLU into its taps)
        shapes = [tuple(z.shape) for z in s['zs'][-1]]
        dA = roi_align_mlvl_backward(d_feats, s['rois'], shapes, s['scales'], c.roi_sampling, True)
        # ---- MLVLFuseModule, rounds 4 .. 0 (layers.py:152-195)
        for r in range(4, -1, -1):
            gamma = eng.fuse[r]['gamma']
            dg, db = torch.empty(C, dtype=F32, device=eng.dev), torch.empty(C, dtype=F32, device=eng.dev)
            zr, st, ss = s['zs'][r + 1], s['sts'][r + 1], s['sss'][r + 1]
            dz = [train_ops.gn_relu_bwd(zr[l], dA[l], ss[l][0], ss[l][1], st[l], c.level_sizes[l] ** 2 * (C // c.gn_groups),
                                        gamma, dg, db, accumulate=l > 0) for l in range(n)]
            prev, pss = s['zs'][r], s['sss'][r]
            wf = train_ops.conv_weight_flip_t(eng.fuse[r]['w'])
            dW, d_in = None, []
            for l in range(n):
                top, down = min(l + 1, n - 1), max(l - 1, 0)
                x_in = kernels.fuse_gather(prev[l], prev[top], prev[down], pss[l], pss[top], pss[down])
                dx, dW = train_ops.conv3x3_bwd(x_in, eng.fuse[r]['w'], dz[l], dw_acc=dW, wf=wf)
                d_in.append(dx)
            g[p + 'mlvl_fuse.fuse_convs.%d.conv.weight' % r] = dW.permute(0, 3, 1, 2)
            g[p + 'mlvl_fuse.fuse_convs.%d.gn.weight' % r] = dg
            g[p + 'mlvl_fuse.fuse_convs.%d.gn.bias' % r] = db
            dA = [train_ops.fuse_gather_bwd(d_in, m) for m in range(n)]
            s['zs'][r + 1] = None
        # ---- input 1x1 convs on [tokens | coords] (layers.py:185-191); the CLIP tower is frozen: no grad_x
        for l in range(n):
            dm = train_ops.cast_f32_bf16(dA[l].view(-1, C))
            up = s['ups'][l].view(-1, eng.spi_cpad)
            gw = dense.matmul_t(dm, up, a_mn=True, b_mn=True)            # [C, cpad]
            g[p + 'mlvl_fuse.input_conv.%d.weight' % l] = gw[:, :C + 2].reshape(C, C + 2, 1, 1)
            g[p + 'mlvl_fuse.input_conv.%d.bias' % l] = train_ops.colsum(dm)
        self.saved = None
        return g


FRONT_GROUPS = (('embed', ('model.embed_tokens.weight',)), ('proj', ('model.mm_projector.',)), ('spi', ('model.spi_module.',)))
ALL_GROUPS = ('embed', 'proj', 'spi', 'llama', 'head')


def trainable_from_env(environ=None):
    """The reference's trainable-set switches (gpt4roi/train/train.py:685-696): ONLY_SPI=1 trains the SPI module
    only (stage 1, train_stage1.sh:8), PROJ=1 additionally un-freezes mm_projector; otherwise stage 2 trains
    everything except the CLIP tower.  Returns (groups, spi_decay): llava_trainer.py:68-90 gives the SPI group
    weight_decay 0.01 on every tensor when ONLY_SPI is set without PROJ, else 0."""
    import os
    env = os.environ if environ is None else environ
    if env.get('ONLY_SPI'):
        if env.get('PROJ'):
            return ('spi', 'proj'), 0.0
        return ('spi',), 0.01
    return ALL_GROUPS, None


class Stage2Trainer:
    """One optimisation step of GPT4RoI training (scripts train_stage{1,2}.sh -> gpt4roi/train/train.py:698-712 ->
    HF Trainer.training_step): forward, backward, DDP gradient all-reduce, global grad-norm clip
    (max_grad_norm 1.0, the HF default the scripts do not override), warm-up + cosine learning rate
    (train_stage2.sh:47-53) and torch.optim.AdamW semantics -- all on the sm_90a kernels; no autograd.
    Stage 2 trains every parameter except the frozen CLIP tower (embed_tokens, mm_projector, the SPI module, the
    32 LLaMA layers, final norm, lm_head); `trainable` selects the reference's other sets
    (ONLY_SPI / PROJ, `trainable_from_env`).  Loss: llava/model/llava.py:238-249.

        front = FrontEndTrain(PrefillEngine without LLaMA layers)   ViT (frozen) -> projector / SPI -> splice
        stack = LlamaTrainStack                                     decoder stack -> lm_head -> cross entropy
    """

    def __init__(self, cfg, state_dict, vit_state_dict, device, lr=2e-5, betas=(0.9, 0.999), eps=1e-8,
                 weight_decay=0.0, reducer=None, world_size=1, trainable=ALL_GROUPS, max_grad_norm=1.0,
                 schedule=None, spi_decay_all=None, own_optimizer=True, sm_reserve=None, shard_optimizer=False):
        """schedule: None (constant lr) or dict(total_steps=N, warmup_steps=0, warmup_ratio=0.003, kind='cosine').
        spi_decay_all: weight decay applied to EVERY SPI tensor (the ONLY_SPI group of llava_trainer.py:68-78);
        None = the default rule (decay `weight_decay` on matrices, none on biases / norm weights).
        shard_optimizer: FSDP-equivalent of train_stage2.sh:51-52 (`--fsdp "full_shard auto_wrap"` over
        LlamaDecoderLayer): per decoder layer (and lm_head) the gradient bucket is reduce-scattered, each rank keeps
        fp32 masters + AdamW moments for its 1/world slice only, and the refreshed bf16 slice is all-gathered into
        the flat weight buffer, overlapped with the next forward.  The bf16 compute weights stay replicated (14 GB)."""
        import copy
        from .engine import PrefillEngine
        if getattr(cfg, 'dtype', 'bf16') != 'bf16':
            raise NotImplementedError('the training step is bf16 only (train_stage*.sh --bf16 True); the fp16 kernels are '
                                      'the inference twins for the demo')
        self.cfg, self.dev = cfg, torch.device(device)
        self.lr, self.betas, self.eps, self.wd = lr, betas, eps, weight_decay
        self.reducer, self.world = reducer, world_size
        self.shard = bool(shard_optimizer) and world_size > 1 and own_optimizer
        self.rank = 0
        if self.shard:
            import torch.distributed as dist
            if reducer is None or not reducer.active():
                raise ValueError('shard_optimizer=True needs an initialised process group and a reducer')
            self.rank = dist.get_rank(reducer.group)
            reducer.shard_grads = True
        self.trainable = tuple(trainable)
        bad = set(self.trainable) - set(ALL_GROUPS)
        if bad:
            raise ValueError('unknown trainable groups %s (choose from %s)' % (sorted(bad), ALL_GROUPS))
        self.max_grad_norm = max_grad_norm
        self.schedule = dict(schedule) if schedule else None
        if self.schedule is not None:
            self.schedule.setdefault('kind', 'cosine')
            self.schedule['warmup_steps'] = warmup_steps_for(self.schedule['total_steps'], self.schedule.get('warmup_steps', 0),
                                                             self.schedule.get('warmup_ratio', 0.0))
        self.spi_decay_all = spi_decay_all
        self.own_optimizer = own_optimizer
        # SMs kept free of the persistent GEMM kernels while a gradient collective runs beside the backward
        # (lib.set_sm_reserve); pair it with NCCL_MAX_CTAS=<same> set before the process group is created
        import os
        # the default is 0: whether reserving SMs shortens the step depends on the interconnect; measure before setting it
        self.sm_reserve = int(os.environ.get('G4R_DDP_SM_RESERVE', '0')) if sm_reserve is None else int(sm_reserve)
        fcfg = copy.copy(cfg)
        fcfg.n_layers = 0                                   # the front-end engine holds no decoder layers
        self.eng = PrefillEngine(fcfg, state_dict, vit_state_dict, device)
        self.front = FrontEndTrain(self.eng)
        self.stack = LlamaTrainStack(cfg, state_dict, device, lr, betas, eps, weight_decay, own_optimizer=own_optimizer,
                                     train_layers='llama' in self.trainable, train_head='head' in self.trainable,
                                     shard=self.shard, world=world_size, rank=self.rank)
        front_all = [k for k in state_dict if k.startswith('model.spi_module.') or k.startswith('model.mm_projector.')
                     or k == 'model.embed_tokens.weight']
        self.w16 = {k: state_dict[k].detach().to(self.dev, BF16).contiguous() for k in front_all}
        names = [k for k in front_all if any(grp in self.trainable and k.startswith(pre)
                                             for grp, pres in FRONT_GROUPS for pre in pres)]
        self.front_names = names
        self.front_shapes = {k: tuple(state_dict[k].shape) for k in names}
        self.front_offsets, o = {}, 0
        for k in names:
            self.front_offsets[k] = o
            o += (state_dict[k].numel() + 3) // 4 * 4          # 16-byte aligned slices of the flat fp32 bucket
        self.front_numel = o
        if own_optimizer:
            self.master = {k: state_dict[k].detach().to(self.dev, F32).contiguous() for k in names}
            self.m1 = {k: torch.zeros_like(v) for k, v in self.master.items()}
            self.m2 = {k: torch.zeros_like(v) for k, v in self.master.items()}
        else:
            self.master, self.m1, self.m2 = {}, {}, {}
        self.front_flat = None
        self.clip = None          # device fp32 [2]: (gradient norm, clip coefficient) of the last step
        self.last_lr = lr

    @staticmethod
    def shift_labels(labels):
        """labels [B,L] (-100 = ignored) -> targets with targets[:, t] = labels[:, t+1] (llava.py:241-242)."""
        t = torch.full_like(labels, -100)
        t[:, :-1] = labels[:, 1:]
        return t

    def _front_slice(self, k):
        o = self.front_offsets[k]
        n = 1
        for d in self.front_shapes[k]:
            n *= d
        return self.front_flat[o:o + n].view(self.front_shapes[k])

    def load_weights(self, state_dict):
        """Model-seam path (own_optimizer=False): refresh every bf16 compute weight from the reference-named
        parameters that torch.optim just updated."""
        for k in self.w16:
            self.w16[k].copy_(state_dict[k])
        self.eng._prepare_spi(self.w16)
        self.eng.embed = self.w16['model.embed_tokens.weight']
        self.stack.load_weights(state_dict)

    def forward_loss(self, input_ids, images, bboxes, labels):
        embeds = self.front.forward(input_ids, images, bboxes)
        return self.stack.forward(embeds, self.shift_labels(labels.to(self.dev)))

    def backward(self, loss_scale=1.0):
        """Backward of the last forward_loss; gradients are left in self.stack.grads and self.front_flat (already
        all-reduced over the data-parallel group when a reducer is attached)."""
        red = self.reducer if (self.reducer is not None and self.reducer.active()) else None
        from . import lib as _lib
        if red is not None and self.sm_reserve > 0:
            _lib.set_sm_reserve(self.sm_reserve)
        d_embeds = self.stack.backward(loss_scale=loss_scale, on_layer_grads=red.hook if red is not None else None,
                                       on_top_grads=red.top_hook if red is not None else None)
        tr = self.trainable
        fg = self.front.backward(d_embeds, want_embed='embed' in tr, want_proj='proj' in tr, want_spi='spi' in tr)
        # one flat fp32 bucket for every front-end gradient: a rank whose micro-batch has no boxes (no SPI
        # gradients) contributes zeros, so every rank hands the same buffer to the collective
        self.front_flat = torch.zeros(max(self.front_numel, 4), dtype=F32, device=self.dev)
        for k in self.front_names:
            if k in fg and fg[k] is not None:
                self._front_slice(k).copy_(fg[k].reshape(self.front_shapes[k]))
        if red is not None:
            small = [self.front_flat]
            if self.stack.train_layers:
                small.append(self.stack.grads['norms'])
            if self.stack.train_head:
                small.append(self.stack.grads['top']['norm'])
            red.reduce_now(small)
            red.wait()
            if self.sm_reserve > 0:
                _lib.set_sm_reserve(0)

    def forward_backward(self, input_ids, images, bboxes, labels):
        """Returns the loss; see backward()."""
        loss = self.forward_loss(input_ids, images, bboxes, labels)
        self.backward()
        return loss

    def _clip_coef(self, scale):
        """Global gradient norm over every trained tensor (torch clip_grad_norm_ semantics) -> device (norm, coef).
        Sharded mode: each rank sums the squares of its reduce-scattered slices, rank 0 adds the replicated tensors,
        one 4-byte all-reduce joins them."""
        sharded, repl = self.stack.grad_tensors()
        if self.front_numel:
            repl = repl + [self.front_flat]
        if self.shard:
            mine = sharded + (repl if self.rank == 0 else [])
            tot = train_ops.grad_sumsq(mine).sum().reshape(1) if mine else torch.zeros(1, dtype=F32, device=self.dev)
            self.reducer.dist.all_reduce(tot, group=self.reducer.group)
            return train_ops.clip_coef(tot, self.max_grad_norm, pre_scale=scale)
        return train_ops.clip_coef(train_ops.grad_sumsq(sharded + repl), self.max_grad_norm, pre_scale=scale)

    def current_lr(self):
        if self.schedule is None:
            return self.lr
        return self.lr * lr_lambda(self.stack.step_count, self.schedule['total_steps'], self.schedule['warmup_steps'],
                                   self.schedule['kind'])

    def _front_decay(self, k):
        if k.startswith('model.spi_module.') and self.spi_decay_all is not None:
            return self.spi_decay_all
        no_decay = k.endswith('.bias') or '.gn.' in k or 'pos_embedd.2.' in k or 'pos_embedd.5.' in k
        return 0.0 if no_decay else self.wd

    def optimizer_step(self):
        """clip_grad_norm_(max_grad_norm) -> AdamW at the scheduled learning rate (HF Trainer order)."""
        if not self.own_optimizer:
            raise RuntimeError('this trainer was built with own_optimizer=False (torch.optim owns the parameters)')
        scale = 1.0 / self.world
        scale_dev = None
        if self.max_grad_norm is not None and self.max_grad_norm > 0:
            self.clip = self._clip_coef(scale)
            scale_dev = self.clip[1:]
        lr = self.last_lr = self.current_lr()
        self.stack.optimizer_step(grad_scale=scale, lr=lr, scale_dev=scale_dev, reducer=self.reducer)
        t = self.stack.step_count
        for k in self.front_names:
            train_ops.adamw_step(self.master[k].view(-1), self._front_slice(k).reshape(-1), self.m1[k].view(-1),
                                 self.m2[k].view(-1), self.w16[k].view(-1), lr, self.betas, self.eps,
                                 self._front_decay(k), t, scale, scale_dev)
        self.front_flat = None
        if self.front_names:
            # refresh the engine's bf16 tensors (its own layouts: padded 1x1 weights, KHWC convs, stacked pconvs ...)
            self.eng._prepare_spi(self.w16)
            self.eng.embed = self.w16['model.embed_tokens.weight']

    def step(self, input_ids, images, bboxes, labels):
        loss = self.forward_backward(input_ids, images, bboxes, labels)
        self.optimizer_step()
        return loss

    @property
    def front_grads(self):
        """Front-end gradients (fp32 views of the flat bucket) under the reference's parameter names."""
        return None if self.front_flat is None else {k: self._front_slice(k) for k in self.front_names}

    def grads_state_dict(self):
        """Every gradient of the last backward under the reference's parameter names (model-seam path)."""
        if self.shard:
            raise RuntimeError('sharded optimizer: full gradients are never materialised (each rank holds 1/world slices)')
        out = {k: self._front_slice(k) for k in self.front_names}
        out.update(self.stack.grads_state_dict())
        return out

    # ------------------------------------------------------------------ checkpoint / resume
    def state_dict(self):
        """All parameters of the model's state dict under reference names and layouts -- what the reference's
        trainer saves (train.py:88-98): fp32 masters for the trained tensors, bf16 for frozen ones; the CLIP tower
        is not part of the model's state dict (llava.py:47-48)."""
        out = dict(self.w16)
        out.update(self.master)
        out.update(self.stack.state_dict())
        return out

    def save_pretrained(self, out_dir, dtype=None, max_shard_bytes=10 * 1024 ** 3, config=None, rank=None):
        return save_checkpoint(self.state_dict(), out_dir, max_shard_bytes, dtype, config=config, rank=rank)

    def optimizer_state(self):
        """AdamW step count (= scheduler position) and moments under reference names (resume: pass the saved fp32
        weights to __init__, then load_optimizer_state).  Sharded mode: a collective call (slices are gathered)."""
        m1, m2 = dict(self.m1), dict(self.m2)
        s1, s2 = self.stack.moments()
        m1.update(s1)
        m2.update(s2)
        return dict(step=self.stack.step_count, exp_avg=m1, exp_avg_sq=m2, schedule=self.schedule, lr=self.lr)

    def load_optimizer_state(self, state):
        self.stack.step_count = int(state['step'])
        if state.get('schedule') is not None:
            self.schedule = dict(state['schedule'])
        for src, dst in ((state['exp_avg'], self.m1), (state['exp_avg_sq'], self.m2)):
            for k in dst:
                dst[k].copy_(src[k])
        self.stack.load_moments(state['exp_avg'], state['exp_avg_sq'])

    def save_optimizer(self, path):
        """optimizer.pt + scheduler position in one file (HF Trainer writes optimizer.pt / scheduler.pt beside the
        weights; train_stage2.sh:21 excludes them when bootstrapping stage 2 from stage 1)."""
        st = self.optimizer_state()
        st['exp_avg'] = {k: v.detach().cpu().clone() for k, v in st['exp_avg'].items()}
        st['exp_avg_sq'] = {k: v.detach().cpu().clone() for k, v in st['exp_avg_sq'].items()}
        torch.save(st, path)

    def load_optimizer(self, path):
        self.load_optimizer_state(torch.load(path, map_location='cpu'))
