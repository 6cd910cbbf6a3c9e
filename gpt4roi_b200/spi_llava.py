"""Model seam: drop-in mirrors of the reference's model classes, running on the sm_90a engine.

Same class names, constructor arguments, forward keyword arguments, attributes and -- above all --
parameter names/shapes as the reference, so its checkpoints load unchanged and its train / serve
scripts can import these classes instead:

    gpt4roi/models/layers.py:96-195     MLVLFuseModule          forward(inputs)
    gpt4roi/models/layers.py:198-236    MLVLROIQueryModule      forward(mlvl_feats, bboxes)
    gpt4roi/models/layers.py:239-335    MlvlRoIExtractor        forward(feats, rois)
    gpt4roi/models/spi_llava.py:15-205  SPILlavaLlamaModel      forward(...) -> BaseModelOutputWithPast
    gpt4roi/models/spi_llava.py:215-306 SPILlavaMPTForCausalLM  forward / generate / prepare_inputs_for_generation
    llava/model/llava.py:36-40          LlavaConfig
    llava/model/utils.py:26-46          KeywordsStoppingCriteria

The modules are PARAMETER CONTAINERS with the reference's state-dict layout (SURVEY.md Appendix C; mmcv's
ConvModule names `.conv` / `.gn` included).  Their `forward` runs no PyTorch op on the compute path: it hands
the weights to `engine.PrefillEngine` (re-laid-out once, rebuilt when a parameter's version counter or a token
id changes) which launches the hand-written kernels.

  * inference: prefill `forward` (from `input_ids` or `inputs_embeds`), `generate()` (own KV-cache decode loop,
    or HF's GenerationMixin loop through `prepare_inputs_for_generation` / `past_key_values`);
  * training: with grad enabled, `forward(labels=...)` runs the explicit forward of `train.Stage2Trainer` inside
    ONE `torch.autograd.Function` whose backward returns the gradient of every `requires_grad` parameter, so
    `loss.backward()`, DDP hooks, `clip_grad_norm_` and `torch.optim` of HF Trainer work unchanged
    (gpt4roi/train/train.py:698-712).  The trainable set follows the parameters' `requires_grad` flags
    (ONLY_SPI / PROJ: train.py:685-696).

Anything outside this (output_attentions, left padding, list-of-images) raises instead of falling back.
"""
import collections
import weakref
from typing import List, NamedTuple, Optional

import torch
import torch.nn as nn
from transformers import LlamaConfig, LlamaForCausalLM, LlamaModel
from transformers.modeling_outputs import BaseModelOutputWithPast, CausalLMOutputWithPast

from .engine import (BF16, ContinuousBatcher, EngineConfig, KVCache, PrefillEngine, StopStrings, _right_padded,
                     from_right_padded, right_pad_layout)
from .roi_align import RoIAlign

DEFAULT_IMAGE_PATCH_TOKEN = '<im_patch>'
DEFAULT_IM_START_TOKEN = '<im_start>'
DEFAULT_IM_END_TOKEN = '<im_end>'
SPI_PREFIX = 'model.spi_module.'


class LlavaConfig(LlamaConfig):
    model_type = 'llava'  # llava/model/llava.py:37 (the reference's checkpoints carry "model_type": "llava")


def _param_version(module):
    """Changes whenever a parameter is updated in place (optimizer step, load_state_dict, .data.copy_), replaced, or
    cast (`.half()` / `.bfloat16()` swap `.data` without bumping the version counter)."""
    return tuple((id(p), p._version, p.dtype) for p in module.parameters())


def _engine_dtype(module):
    """fp16 parameters (the demo: gpt4roi/app.py:74-98 `.half()`) -> the fp16 kernels; anything else -> bf16 (the
    training scripts' --bf16, and fp32 masters under autocast)."""
    p = next(module.parameters(), None)
    return 'fp16' if p is not None and p.dtype == torch.float16 else 'bf16'


# =========================================================================================
# SPI module mirrors
# =========================================================================================
class _ConvModule(nn.Module):
    """Parameter layout of mmcv.cnn.ConvModule(conv -> GN -> ReLU): `.conv.weight`, `.gn.{weight,bias}`
    (mmcv-1.4.7/mmcv/cnn/bricks/conv_module.py:70-208; conv has no bias when a norm follows)."""

    def __init__(self, cin, cout, groups=64):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, 3, stride=1, padding=1, bias=False)
        self.gn = nn.GroupNorm(groups, cout)


def _spi_engine(module, prefix, sd_extra, grid, device):
    """SPI-only PrefillEngine over `module`'s own parameters (keys re-prefixed to the reference's full names),
    cached on the module until a parameter changes."""
    key = (str(device), int(grid), _param_version(module))
    cache = module.__dict__.setdefault('_g4r_engine', {})
    if cache.get('key') != key:
        sd = {SPI_PREFIX + prefix + k: v for k, v in module.state_dict().items()}
        sd.update(sd_extra)
        cfg = EngineConfig(image_size=int(grid) * 14, n_layers=0, dtype=_engine_dtype(module))
        cache['eng'] = PrefillEngine(cfg, sd, None, device, parts=('spi',))
        cache['key'] = key
    return cache['eng']


def _to_tokens(feats, dt=BF16):
    """list of [B,P,C] token maps or [B,C,G,G] NCHW maps (layers.py:219-224) -> (list of contiguous [B,P,C], G);
    dt: the engine's 16-bit type (fp32 maps pass through: the resampling kernel reads them directly)."""
    out = []
    for f in feats:
        if f.dim() == 4:
            f = f.permute(0, 2, 3, 1).reshape(f.shape[0], -1, f.shape[1])
        if f.dtype not in (torch.float32, dt):
            f = f.to(dt)
        out.append(f.contiguous())
    G = int(round(out[0].shape[1] ** 0.5))
    if G * G != out[0].shape[1]:
        raise ValueError('token maps must be square (got %d tokens)' % out[0].shape[1])
    return out, G


class MLVLFuseModule(nn.Module):
    def __init__(self, input_dims=1024, embed_dims=1024, num_levels=3, num_fuse=4):
        super().__init__()
        self.embed_dims, self.num_levels, self.num_fuse, self.input_dims = embed_dims, num_levels, num_fuse, input_dims
        self.shuffle_channles = embed_dims // 4
        self.remain_chs = embed_dims - 2 * self.shuffle_channles
        self.fuse_lvl_list = [(l, min(l + 1, num_levels - 1), max(l - 1, 0)) for l in range(num_levels)]
        self.input_conv = nn.ModuleList([nn.Conv2d(input_dims + 2, embed_dims, 1) for _ in range(num_levels)])
        self.fuse_convs = nn.ModuleList([_ConvModule(embed_dims, embed_dims) for _ in range(num_fuse)])
        self.init_weights()

    def init_weights(self):  # layers.py:146-150
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.normal_(m.weight, 0, 0.01)
                if m.bias is not None:
                    nn.init.constant_(m.bias, 0)

    @torch.no_grad()
    def forward(self, inputs):
        """layers.py:182-195: list of NCHW maps [B,1024,H_l,H_l] (already at the pyramid sizes) -> list of fused,
        activated NCHW maps.  Inference only; gradients flow through MLVLROIQueryModule.forward."""
        from . import kernels
        if self.num_levels != 4 or self.num_fuse != 5 or self.embed_dims != 1024:
            raise NotImplementedError('the sm_90a SPI kernels are built for the GPT4RoI configuration (4 levels, 5 rounds, 1024 ch)')
        dev = inputs[0].device
        G = inputs[-1].shape[-1]
        eng = _spi_engine(self, 'mlvl_fuse.', {}, G, dev)
        if [m.shape[-1] for m in inputs] != eng.cfg.level_sizes:
            raise ValueError('expected pyramid sizes %s, got %s' % (eng.cfg.level_sizes, [m.shape[-1] for m in inputs]))
        maps, ss = eng.fuse_maps(_to_tokens(inputs, eng.dt)[0], has_cls=False, pre_upsampled=True)
        outs = [kernels.affine_relu_nhwc(m, s[0], s[1]) for m, s in zip(maps, ss)]
        return [o.permute(0, 3, 1, 2).to(inputs[0].dtype) for o in outs]


class MlvlRoIExtractor(nn.Module):
    def __init__(self, roi_layer, out_channels, featmap_strides, embed_dims=1024, stride=1, norm_init=True,
                 fuse_level=3, finest_scale=56, init_cfg=None):
        super().__init__()
        cfg = dict(roi_layer)
        assert cfg.pop('type') == 'RoIAlign'
        # mmdet BaseRoIExtractor.build_roi_layers (base_roi_extractor.py:37-60): one layer per stride
        self.roi_layers = nn.ModuleList([RoIAlign(spatial_scale=1 / s, **cfg) for s in featmap_strides])
        self.out_channels, self.featmap_strides = out_channels, featmap_strides
        self.embed_dims, self.finest_scale, self.fuse_level, self.norm_init = embed_dims, finest_scale, fuse_level, norm_init
        self.pconvs = nn.ModuleList(nn.Conv2d(embed_dims, embed_dims, 3, stride=1, padding=1) for _ in range(fuse_level))
        self.pos_embedd = nn.Sequential(nn.Linear(4, 256), nn.ReLU(inplace=True), nn.LayerNorm(256),
                                        nn.Linear(256, 1024), nn.ReLU(inplace=True), nn.LayerNorm(1024))
        self.updims = nn.Linear(1024, 4096)
        self.flatten_linear = nn.Linear(embed_dims * self.roi_layers[0].output_size[0] ** 2, 1024)
        for m in self.modules():  # layers.py:275-278
            if isinstance(m, nn.Conv2d):
                nn.init.normal_(m.weight, 0, 0.01)
                nn.init.constant_(m.bias, 0)

    @property
    def num_inputs(self):
        return len(self.featmap_strides)

    @torch.no_grad()
    def forward(self, feats, rois, roi_scale_factor=None):
        """layers.py:280-335: feats = list of fused NCHW maps [B,1024,H_l,H_l]; rois = list (len B) of [K_i,4]
        normalised xyxy boxes -> list of [K_i,4096] region tokens.  The reference's `* 224` (layers.py:297) is the
        image side = 14 x the coarsest map side here (SURVEY.md 8(c), 336-px lift).  Inference only."""
        dev = feats[0].device
        G = feats[-1].shape[-1]
        eng = _spi_engine(self, 'roi_align.', {}, G, dev)
        maps = [f.permute(0, 2, 3, 1).to(eng.dt).contiguous() for f in feats]
        plan = eng.plan_boxes(rois)
        if plan is None or plan['K'] == 0:
            return [feats[0].new_zeros((0, self.updims.out_features)) for _ in rois]
        rows = eng.region_tokens(maps, None, plan['boxes'], plan['bidx'])
        offs = plan['offs'].tolist()
        return [rows[offs[i]:offs[i + 1]] for i in range(len(rois))]


class _SpiQueryFn(torch.autograd.Function):
    """MLVLROIQueryModule.forward with an explicit backward (train.SpiTrain): the gradient of every SPI parameter,
    none for the token maps (the CLIP tower is frozen in both training stages, train.py:604-612)."""

    @staticmethod
    def forward(ctx, module, eng, tokens, plan, names, *params):
        from .train import SpiTrain
        spi = SpiTrain(eng)
        rows = spi.forward(tokens, plan, has_cls=False)
        ctx.spi, ctx.names, ctx.n_in = spi, names, len(params)
        return rows

    @staticmethod
    def backward(ctx, d_rows):
        g = ctx.spi.backward(d_rows.to(BF16).contiguous())
        return (None,) * 5 + tuple(g.get(SPI_PREFIX + n) for n in ctx.names)


class MLVLROIQueryModule(nn.Module):
    def __init__(self, embed_dims=1024, out_dims=4096, num_levels=3):
        super().__init__()
        self.mlvl_fuse = MLVLFuseModule(input_dims=embed_dims, embed_dims=embed_dims, num_levels=num_levels, num_fuse=5)
        strids = [14 / 8, 14 / 4, 14 / 2, 14]
        assert len(strids) == num_levels
        self.roi_align = MlvlRoIExtractor(roi_layer=dict(type='RoIAlign', output_size=14, sampling_ratio=2),
                                          out_channels=embed_dims, embed_dims=embed_dims, fuse_level=num_levels,
                                          featmap_strides=strids)

    def forward(self, mlvl_feats, bboxes):
        """layers.py:218-236: mlvl_feats = list[4] of [B,P,1024] token maps (CLS dropped) or [B,1024,G,G];
        bboxes = list[B] of [K_i,4] normalised xyxy -> list[B] of [K_i,4096].  One fused pipeline: pyramid
        up-sampling + coordinate channels, 1x1 input convs, 5 fuse rounds, multi-level RoIAlign, pconvs,
        flatten_linear, box position MLP, updims.  With grad enabled the SPI parameters receive gradients
        (explicit backward on the same kernels)."""
        dt = torch.float16 if _engine_dtype(self) == 'fp16' else BF16
        tokens, G = _to_tokens(list(mlvl_feats), dt)
        dev = tokens[0].device
        eng = _spi_engine(self, '', {}, G, dev)
        plan = eng.plan_boxes(bboxes)
        out_dims = self.roi_align.updims.out_features
        if plan is None or plan['K'] == 0:
            return [tokens[0].new_zeros((0, out_dims), dtype=dt) for _ in bboxes]
        named = [(n, p) for n, p in self.named_parameters() if p.requires_grad]
        if torch.is_grad_enabled() and named:
            if dt != BF16:
                raise NotImplementedError('fp16 parameters with grad enabled: the training kernels are bf16 (the reference '
                                          'trains with --bf16 True); call under torch.no_grad() or cast the module')
            if any(t.requires_grad for t in tokens):
                raise NotImplementedError('gradients w.r.t. the CLIP features are not provided (the tower is frozen)')
            rows = _SpiQueryFn.apply(self, eng, tokens, plan, tuple(n for n, _ in named), *[p for _, p in named])
        else:
            maps, ss = eng.fuse_maps(tokens, has_cls=False)
            rows = eng.region_tokens(maps, ss, plan['boxes'], plan['bidx'])
        offs = plan['offs'].tolist()
        return [rows[offs[i]:offs[i + 1]] for i in range(len(bboxes))]


# =========================================================================================
# LLaVA / LLaMA mirrors
# =========================================================================================
class G4RCache:
    """`past_key_values` of this seam: the engine's KV cache (bf16, post-RoPE keys, [B, Lmax, H*D] per layer) plus
    the CUDA-graph stepper of the decode loop.  Opaque to callers, like HF's Cache objects."""

    def __init__(self, kv):
        self.kv = kv
        self.stepper = None

    def get_seq_length(self, layer_idx=0):
        return self.kv.length

    def __len__(self):
        return self.kv.length

    def __bool__(self):
        return True

    def crop(self, n):
        """Keep the first n positions (transformers' assisted decoding crops the cache to the accepted length after
        every verify step): KVCache.crop, and the captured decode step, if any, continues from n."""
        self.kv.crop(n)
        if self.stepper is not None:
            self.stepper.pos.fill_(self.kv.length)

    def reorder_cache(self, beam_idx):
        """transformers' beam search (GenerationMixin._beam_search) after every step: row i of the cache becomes row
        beam_idx[i] -- every layer's K/V, the recorded ids, lengths, images and boxes.  In place, so a CUDA graph
        captured on the cache (the stepper) stays valid."""
        kv = self.kv
        idx = beam_idx.to(kv.ids.device, torch.long)
        for t in kv.k + kv.v:
            t.copy_(t.index_select(0, idx.to(t.device)))
        kv.ids.copy_(kv.ids.index_select(0, idx))
        if kv.lens is not None:
            kv.lens.copy_(kv.lens.index_select(0, idx.to(kv.lens.device)))
        if kv.images is not None:
            kv.images.copy_(kv.images.index_select(0, idx.to(kv.images.device)))
        if kv.boxes is not None:
            kv.boxes = [kv.boxes[i] for i in idx.tolist()]


def _find_cache(past_key_values):
    """Our cache, whether handed back directly or riding on the (otherwise unused) HF Cache object that
    GenerationMixin.generate() creates and threads through its loop."""
    if past_key_values is None:
        return None
    if isinstance(past_key_values, G4RCache):
        return past_key_values
    return getattr(past_key_values, '_g4r_cache', None)


class _EngineHost:
    """Engine construction shared by SPILlavaLlamaModel (no lm_head) and SPILlavaMPTForCausalLM."""

    def _engine_modules(self):
        raise NotImplementedError

    def _token_ids(self, vc):
        bbox = getattr(vc, 'bbox_token', None)
        if bbox is None:
            # the serving path (gpt4roi/app.py:100-104,283) sets only im_patch/im_start/im_end on the vision
            # config and `model.model.tokenizer`; the reference resolves <bbox> through the tokenizer at
            # spi_llava.py:150-152
            tok = None
            for m in self._engine_modules():
                tok = getattr(m, 'tokenizer', None) or tok
            if tok is not None:
                bbox = tok.convert_tokens_to_ids(['<bbox>'])[0]
        return dict(im_patch_token=getattr(vc, 'im_patch_token', -1), bbox_token=-2 if bbox is None else int(bbox),
                    im_start_token=getattr(vc, 'im_start_token', -3), im_end_token=getattr(vc, 'im_end_token', -4))

    def _engine_config(self, config, vt):
        vc = vt.config
        return EngineConfig(image_size=vc.image_size, patch_size=vc.patch_size, vit_hidden=vc.hidden_size,
                            vit_heads=vc.num_attention_heads, vit_layers=vc.num_hidden_layers,
                            vit_mlp=vc.intermediate_size, vit_eps=vc.layer_norm_eps,
                            select_layer=getattr(config, 'mm_vision_select_layer', -1),
                            hidden=config.hidden_size, n_heads=config.num_attention_heads,
                            n_layers=config.num_hidden_layers, mlp=config.intermediate_size,
                            vocab=config.vocab_size, rms_eps=config.rms_norm_eps,
                            rope_theta=_rope_theta(config), dtype=_engine_dtype(self), **self._token_ids(vc))


def _rope_theta(config):
    rp = getattr(config, 'rope_parameters', None)
    if isinstance(rp, dict) and 'rope_theta' in rp:
        return float(rp['rope_theta'])
    return float(getattr(config, 'rope_theta', 10000.0))


class SPILlavaLlamaModel(LlamaModel, _EngineHost):
    config_class = LlavaConfig

    def __init__(self, config):
        super().__init__(config)
        if hasattr(config, 'mm_vision_tower') and getattr(config, 'mm_vision_tower_instance', None) is not None:
            self.vision_tower = [config.mm_vision_tower_instance]  # python list: HACK for FSDP (llava.py:47-48)
        if getattr(config, 'use_mm_proj', True):
            self.mm_projector = nn.Linear(getattr(config, 'mm_hidden_size', 1024), config.hidden_size)
        self.num_level_spi_features = 4
        self.spi_module = MLVLROIQueryModule(embed_dims=1024, out_dims=4096, num_levels=4)
        self.__dict__['_g4r_owner'] = None   # weakref to the CausalLM wrapper (shares its engine)

    def _engine_modules(self):
        return [self]

    def _get_engine(self, device):
        owner = self.__dict__.get('_g4r_owner')
        owner = owner() if owner is not None else None
        if owner is not None:
            return owner._get_engine(device)
        vt = getattr(self, 'vision_tower', None)
        if vt is None:
            raise RuntimeError('vision tower not attached (model.vision_tower is a list of one CLIPVisionModel)')
        vt = vt[0]
        key = (str(device), id(vt), tuple(sorted(self._token_ids(vt.config).items())), _param_version(self))
        st = self.__dict__.setdefault('_g4r_engine', {})
        if st.get('key') != key:
            sd = {'model.' + k: v for k, v in self.state_dict().items()}
            st['eng'] = PrefillEngine(self._engine_config(self.config, vt), sd, vt.state_dict(), device)
            st['key'] = key
        return st['eng']

    def forward(self, input_ids: torch.LongTensor = None, attention_mask: Optional[torch.Tensor] = None,
                img_metas=None, bboxes=None, past_key_values=None, inputs_embeds: Optional[torch.FloatTensor] = None,
                use_cache: Optional[bool] = None, output_attentions: Optional[bool] = None,
                output_hidden_states: Optional[bool] = None, images: Optional[torch.FloatTensor] = None,
                return_dict: Optional[bool] = None, **kwargs):
        """spi_llava.py:23-205 -> LlamaModel.forward: returns the final-norm hidden states [B,L,hidden]
        (BaseModelOutputWithPast.last_hidden_state).  Inference only at this level."""
        if output_attentions or output_hidden_states:
            raise NotImplementedError('attention maps / per-layer hidden states are not materialised by the fused engine')
        dev = (input_ids if input_ids is not None else inputs_embeds).device
        eng = self._get_engine(dev)
        hidden, cache = _run_engine(eng, input_ids, images, bboxes, attention_mask, past_key_values, inputs_embeds,
                                    use_cache, want='hidden', training=self.training)
        if return_dict is False:
            return (hidden, cache)
        return BaseModelOutputWithPast(last_hidden_state=hidden, past_key_values=cache)


def _seqlens(eng, attention_mask, L):
    if attention_mask is None:
        return None
    m = attention_mask.to(eng.dev).to(torch.int32)
    if m.shape[1] != L:
        return None          # a grown decode-time mask (HF generate appends ones): positions come from the cache
    if bool((m == 1).all()):
        return None
    lens, _ = right_pad_layout(m)   # right-padded (data_modules.py:33-44) or left-padded (HF generate) rows
    return lens.to(torch.int32).contiguous()


def _stack_images(images):
    """`images` as a python list of [3,S,S] tensors (the LLaVA base's variable-length branch, spi_llava.py:52-64 /
    train.py:440-464 `image_aspect_ratio`): the reference pushes each through the CLIP tower on its own and then leaves
    `mlvl_spi_features` undefined, so region tokens cannot be used with it there.  CLIP's fixed position embedding
    makes every admissible image S x S anyway, so the list is one batch: it is stacked and takes the fused path
    (region features included).  Mixed sizes have no defined result in the reference and raise here."""
    if type(images) is not list:
        return images
    if len(images) == 0:
        return None
    shapes = {tuple(im.shape[-3:]) for im in images}
    if len(shapes) != 1:
        raise NotImplementedError('images of different sizes in one batch: the CLIP tower has one position-embedding '
                                  'grid (got %s)' % sorted(shapes))
    return torch.stack([im.reshape(im.shape[-3:]) for im in images], 0)


@torch.no_grad()
def _run_engine(eng, input_ids, images, bboxes, attention_mask, past_key_values, inputs_embeds, use_cache, want,
                training=False, max_cache=None, last_only=False, new_prompt=False, logits_to_keep=0):
    """Inference dispatch shared by both model classes: prefill (ids or embeds, with or without the vision
    branch) or one decode step on our cache.  Mirrors spi_llava.py:44-48: the vision branch runs when images are
    given and (the input is longer than one token or the module is in training mode).
    On a non-empty cache, an input one token longer than what the cache holds is a decode step of its last token; a
    longer one, or any input marked as a generate call's prompt (new_prompt: HF's first iteration), is a later turn of
    the conversation (HF's documented past_key_values reuse): the prefix the cache holds is reused and the rest
    prefilled (PrefillEngine.prefill_cached).  A multi-token input with logits_to_keep > 1 that is not a new prompt
    continues the cached sequence (transformers' assisted decoding feeds the last token and its drafts so): its tokens
    are prefilled as one chunk after what the cache holds (PrefillEngine.extend) and the last logits_to_keep logits
    are returned."""
    c = eng.cfg
    cache = _find_cache(past_key_values)
    if cache is not None and cache.kv.length > 0:
        if inputs_embeds is not None:
            raise NotImplementedError('decode steps take input_ids')
        if want == 'hidden':
            raise NotImplementedError('decode steps return logits (use the CausalLM wrapper)')
        if new_prompt or input_ids.shape[1] > cache.kv.length + 1:
            cache.stepper = None          # the cache is extended or grown: a captured step would be stale
            budget = max_cache - input_ids.shape[1] if max_cache is not None else int(getattr(eng, 'decode_budget', 1024))
            out = eng.prefill_cached(cache.kv, input_ids, _stack_images(images), bboxes, attention_mask,
                                     new_tokens=max(budget, 1))
            return out, cache
        if input_ids.shape[1] > 1 and logits_to_keep > 1:
            out = eng.extend(cache.kv, input_ids.to(eng.dev), None, None, last_only=False)
            cache.stepper = None          # the chunk moved the lengths (and may have grown the cache)
            return out[:, -int(logits_to_keep):], cache
        if input_ids.shape[1] != 1:
            input_ids = input_ids[:, -1:]
        ids = input_ids.to(eng.dev).contiguous()
        if cache.stepper is None and c.head_dim == 128 and cache.kv.length + 4 < cache.kv.max_len:
            from .engine import GraphedDecode
            cache.stepper = GraphedDecode(eng, cache.kv)
        cache.kv.record_ids(ids, cache.kv.row_lens())   # outside the (graphed) step: its launches stay unchanged
        out = cache.stepper.step(ids) if cache.stepper is not None else eng.decode_step(ids, cache.kv)
        return out, cache
    new_cache = None
    if use_cache:
        B, L = (input_ids if input_ids is not None else inputs_embeds).shape[:2]
        cap = max_cache if max_cache is not None else L + int(getattr(eng, 'decode_budget', 1024))
        new_cache = G4RCache(KVCache(c, B, cap, eng.dev))
        if past_key_values is not None and not isinstance(past_key_values, G4RCache):
            try:
                past_key_values._g4r_cache = new_cache      # ride on HF's Cache object
            except Exception:
                pass
    kv = new_cache.kv if new_cache is not None else None
    if inputs_embeds is not None:
        B, L = inputs_embeds.shape[:2]
        x = inputs_embeds.to(eng.dev, eng.dt)
        seqlens = _seqlens(eng, attention_mask, L)
        x, _, shift = _right_padded(x, attention_mask if seqlens is not None else None)
        if kv is not None:
            kv.start(L, seqlens)
        out = eng.llama(x, B, L, seqlens=seqlens, cache=kv, want=want, last_only=last_only)
        if shift is not None and not last_only:
            out = from_right_padded(out, shift)
        return out, new_cache
    B, L = input_ids.shape
    run_vision = images is not None and (L != 1 or training)
    images = _stack_images(images)
    mask = attention_mask if _seqlens(eng, attention_mask, L) is not None else None
    out = eng.forward(input_ids, images if run_vision else None, bboxes if run_vision else None,
                      attention_mask=mask, want=want, cache=kv, last_only=last_only)
    return out, new_cache


class _TrainStepFn(torch.autograd.Function):
    """The whole training forward (frozen CLIP -> projector / SPI -> splice -> LLaMA -> lm_head -> shifted CE,
    llava.py:203-261) as one autograd node over the model's trainable parameters."""

    @staticmethod
    def forward(ctx, runner, input_ids, images, bboxes, labels, names, *params):
        loss = runner.forward_loss(input_ids, images, bboxes, labels)
        ctx.runner, ctx.names = runner, names
        return loss.clone()

    @staticmethod
    def backward(ctx, g):
        r = ctx.runner
        r.backward(loss_scale=float(g))
        grads = r.grads_state_dict()
        out = tuple(grads.get(n) for n in ctx.names)
        r.stack.grads = None
        return (None,) * 6 + out


def _generation_config(model, given):
    """The generation config of a generate call as transformers resolves it (GenerationMixin._prepare_generation_config:
    the explicit kwargs `given`, then its `generation_config` entry, then model.generation_config, then HF's defaults),
    special tokens prepared."""
    from transformers.utils import logging as hf_logging
    given = dict(given)
    verbosity = hf_logging.get_verbosity()
    hf_logging.set_verbosity_error()     # HF's notes on flags and pad tokens belong to its own loop
    try:
        gc, _ = model._prepare_generation_config(given.pop('generation_config', None), **given)
        model._prepare_special_tokens(gc, True, 'cpu')
    finally:
        hf_logging.set_verbosity(verbosity)
    return gc


class ResolvedGenerate(NamedTuple):
    """A generate call's configuration, as resolve_generate reads it off transformers' resolution."""
    do_sample: bool
    temperature: float
    top_k: int              # 0: off
    top_p: float            # 1: off
    processors: dict        # repetition_penalty, no_repeat_ngram_size, min_length, min_new_tokens, eos_ids
    names: tuple            # every processor beyond the three warpers HF would build, in HF's order
    other: tuple            # those of `names` the engine loop does not run
    num_return_sequences: int
    beam: Optional[dict]    # None when num_beams is 1
    outputs: dict           # return_dict_in_generate, output_scores, output_logits
    layer_outputs: bool     # output_attentions / output_hidden_states asked for
    lookup: tuple           # (prompt_lookup_num_tokens or None, max_matching_ngram_size)
    stop_strings: Optional[tuple]


_LAYER_OUTPUTS = ('output_attentions / output_hidden_states: attention maps and per-layer hidden states are not '
                  'materialised by the fused engine')
_STOP_STRINGS_NEED_TOKENIZER = (
    "There are one or more stop strings, either in the arguments to `generate` or in the model's generation config, "
    "but we could not locate a tokenizer. When generating with stop strings, you must pass the model's tokenizer to "
    "the `tokenizer` argument of `generate`.")


def resolve_generate(model, input_len, max_new_tokens, do_sample=None, temperature=None, eos_token_id=None,
                     **kwargs):
    """A generate call's configuration, resolved once as transformers resolves it (GenerationMixin.
    _prepare_generation_config: explicit kwargs, then `generation_config=`, then model.generation_config, then HF's
    defaults; `do_sample=True` alone therefore samples with top_k=50), for an input of `input_len` tokens.  Values
    HF's config validation or its processors refuse raise HF's ValueError here (greedy with num_return_sequences > 1,
    num_return_sequences > num_beams, max_new_tokens < 1, ...); what the engine loop or the batcher does not run is
    left to their callers to refuse.

    The selection rule is (False, 1.0, 0, 1.0) for greedy.  The processors are read off HF's own _get_logits_processor:
    without beam search after HF's length preparation (GenerationMixin._prepare_generated_length: a given
    min_new_tokens sets min_length to min_new_tokens + input_len); `processors` holds the history-dependent ones with
    neutral values for those HF does not build or that can never suppress anything (min_length at most input_len,
    min_new_tokens 0), and eos_ids, the resolved eos list (generation_config._eos_token_tensor: the eos_token_id kwarg,
    else the model's) that the minimum lengths suppress.  `other` lists the rest (min_p, typical_p, epsilon / eta
    cutoffs, bad_words_ids, suppress_tokens, sequence_bias, a caller's logits_processor, ...).  With num_beams > 1 the
    list is built as HF builds it for beam search, and `names` and `other` both hold every processor in it, the
    neutral ones included: the engine loop runs none with beams.  `beam` is a dict of num_beams, length_penalty,
    early_stopping, num_return_sequences, eos_token_id (a list), pad_token_id and max_length.  output_scores and
    output_logits count only with return_dict_in_generate, as in HF.  The n-gram size of prompt lookup defaults to 2,
    as HF's PromptLookupCandidateGenerator takes it."""
    from transformers.generation import logits_process as lp
    given = dict(kwargs, do_sample=do_sample, temperature=temperature, eos_token_id=eos_token_id,
                 max_new_tokens=max_new_tokens)
    gc = _generation_config(model, {k: v for k, v in given.items() if v is not None})
    beam = None
    if (gc.num_beams or 1) > 1:
        eos, pad = gc._eos_token_tensor, gc._pad_token_tensor
        beam = dict(num_beams=int(gc.num_beams),
                    length_penalty=float(gc.length_penalty if gc.length_penalty is not None else 1.0),
                    early_stopping=gc.early_stopping if gc.early_stopping is not None else False,
                    num_return_sequences=int(gc.num_return_sequences or 1),
                    eos_token_id=None if eos is None else eos.flatten().tolist(),
                    pad_token_id=None if pad is None else int(pad),
                    max_length=int(input_len + gc.max_new_tokens if gc.max_new_tokens is not None else gc.max_length))
    elif gc.min_new_tokens is not None:
        gc.min_length = gc.min_new_tokens + input_len
    procs = model._get_logits_processor(gc, input_ids_seq_length=input_len, device='cpu', model_kwargs={},
                                        logits_processor=kwargs.get('logits_processor'))
    found = dict(repetition_penalty=1.0, no_repeat_ngram_size=0, min_length=0, min_new_tokens=0, eos_ids=[])
    names, other = [], []
    for p in procs:
        if beam is not None:
            other.append(type(p).__name__)
        elif isinstance(p, (lp.TemperatureLogitsWarper, lp.TopKLogitsWarper, lp.TopPLogitsWarper)):
            continue
        elif type(p) is lp.RepetitionPenaltyLogitsProcessor and not p.prompt_ignore_length:
            found['repetition_penalty'] = float(p.penalty)
        elif type(p) is lp.NoRepeatNGramLogitsProcessor:
            found['no_repeat_ngram_size'] = int(p.ngram_size)
        elif type(p) is lp.MinLengthLogitsProcessor:
            if p.min_length <= input_len:     # at most the prompt's length: it never suppresses anything
                continue
            found['min_length'] = int(p.min_length)
            found['eos_ids'] = p.eos_token_id.flatten().tolist()
        elif type(p) is lp.MinNewTokensLengthLogitsProcessor and p.prompt_length_to_skip == input_len:
            found['min_new_tokens'] = int(p.min_new_tokens)
            found['eos_ids'] = p.eos_token_id.flatten().tolist()
        else:
            other.append(type(p).__name__)
        names.append(type(p).__name__)
    if not gc.do_sample:
        rule = (False, 1.0, 0, 1.0)
    else:
        rule = (True, float(gc.temperature if gc.temperature is not None else 1.0), int(gc.top_k or 0),
                float(gc.top_p if gc.top_p is not None else 1.0))
    rd = bool(gc.return_dict_in_generate)
    stops = gc.stop_strings
    return ResolvedGenerate(
        *rule, processors=found, names=tuple(names), other=tuple(other),
        num_return_sequences=int(gc.num_return_sequences or 1), beam=beam,
        outputs=dict(return_dict_in_generate=rd, output_scores=rd and bool(gc.output_scores),
                     output_logits=rd and bool(gc.output_logits)),
        layer_outputs=bool(gc.output_attentions or gc.output_hidden_states),
        lookup=(int(gc.prompt_lookup_num_tokens) if gc.prompt_lookup_num_tokens else None,
                int(gc.max_matching_ngram_size or 2)),
        stop_strings=None if stops is None else (stops,) if isinstance(stops, str) else tuple(stops))


def _generate_output(res, outs, past_key_values):
    """The engine loop's result as transformers' own generate output class (GenerateDecoderOnlyOutput, or
    GenerateBeamDecoderOnlyOutput for beam search).  past_key_values: the caller's cache, else None (the engine's own
    cache is not a transformers Cache)."""
    from transformers.generation.utils import GenerateBeamDecoderOnlyOutput, GenerateDecoderOnlyOutput
    if 'beam_indices' in res:
        return GenerateBeamDecoderOnlyOutput(
            sequences=res['sequences'], sequences_scores=res['sequences_scores'] if outs['output_scores'] else None,
            scores=res['scores'], logits=res['logits'], beam_indices=res['beam_indices'], past_key_values=past_key_values)
    return GenerateDecoderOnlyOutput(sequences=res['sequences'], scores=res['scores'], logits=res['logits'],
                                     past_key_values=past_key_values)


_STOP_STRINGS = collections.OrderedDict()   # (vocabulary, stop strings) -> StopStrings; the last 8 used


def _token_strings(tokenizer):
    """The string of every token id as transformers' matcher sees it (StopStringCriteria.clean_tokenizer_vocab), a list
    indexed by id, None for ids the vocabulary does not hold."""
    from transformers.generation.stopping_criteria import StopStringCriteria
    strings, ids = StopStringCriteria.clean_tokenizer_vocab(tokenizer)
    by_id = [None] * (max(ids) + 1)
    for s, i in zip(strings, ids):
        by_id[i] = s
    return by_id


def stop_strings_from_tokenizer(tokenizer, stop_strings):
    """The engine's StopStrings table for `tokenizer`: its token strings are what transformers' matcher uses
    (StopStringCriteria.clean_tokenizer_vocab).  Kept per (vocabulary, stop strings), as HF keeps its own tables."""
    stops = (stop_strings,) if isinstance(stop_strings, str) else tuple(stop_strings)
    key = (tuple(sorted(tokenizer.get_vocab().items())), stops)     # sorted: a fast tokenizer lists it in no fixed order
    if key not in _STOP_STRINGS:
        _STOP_STRINGS[key] = StopStrings(_token_strings(tokenizer), stops)
        if len(_STOP_STRINGS) > 8:
            _STOP_STRINGS.popitem(last=False)
    _STOP_STRINGS.move_to_end(key)
    return _STOP_STRINGS[key]


class SPILlavaMPTForCausalLM(LlamaForCausalLM, _EngineHost):
    """Drop-in for gpt4roi.models.spi_llava.SPILlavaMPTForCausalLM (spi_llava.py:215-306)."""
    config_class = LlavaConfig

    def __init__(self, config):
        super(LlamaForCausalLM, self).__init__(config)
        self.model = SPILlavaLlamaModel(config)
        self.lm_head = nn.Linear(config.hidden_size, config.vocab_size, bias=False)
        self.post_init()
        self.model.__dict__['_g4r_owner'] = weakref.ref(self)
        self.__dict__['_g4r_engine'] = {}
        self.__dict__['_g4r_runner'] = {}

    def get_model(self):
        return self.model

    def _engine_modules(self):
        return [self, self.model]

    # ---- engine plumbing ---------------------------------------------------------------
    def set_vision_tower(self, clip_vision_model, image_size=None):
        """Attach the frozen CLIP tower (the reference keeps it in a python list outside the state dict)."""
        self.model.vision_tower = [clip_vision_model]
        self.invalidate_engine()

    def invalidate_engine(self):
        """Drop the cached engine / training runner (they are also rebuilt automatically when a parameter's
        version counter, the vision tower or a special-token id changes)."""
        self.__dict__['_g4r_engine'] = {}
        self.__dict__['_g4r_runner'] = {}

    def _vision_tower(self):
        vt = getattr(self.model, 'vision_tower', None)
        if vt is None:
            raise RuntimeError('vision tower not attached (model.model.vision_tower is a list of one CLIPVisionModel)')
        return vt[0]

    def _check_branches(self, vt):
        if not getattr(vt.config, 'use_im_start_end', True):
            raise NotImplementedError('use_im_start_end=False (spi_llava.py:163-194) never injects region tokens in the '
                                      'reference (its <bbox> scatter lives in the use_im_start_end branch only) and no '
                                      'GPT4RoI script uses it (--mm_use_im_start_end True in train_stage{1,2}.sh)')

    def _get_engine(self, device):
        vt = self._vision_tower()
        self._check_branches(vt)
        key = (str(device), id(vt), tuple(sorted(self._token_ids(vt.config).items())), _param_version(self))
        st = self.__dict__['_g4r_engine']
        if st.get('key') != key:
            st.clear()
            st['eng'] = PrefillEngine(self._engine_config(self.config, vt), self.state_dict(), vt.state_dict(), device)
            st['key'] = key
        return st['eng']

    def _trainable_groups(self):
        groups = set()
        for n, p in self.named_parameters():
            if not p.requires_grad:
                continue
            if n == 'model.embed_tokens.weight':
                groups.add('embed')
            elif n.startswith('model.mm_projector.'):
                groups.add('proj')
            elif n.startswith(SPI_PREFIX):
                groups.add('spi')
            elif n.startswith('model.layers.'):
                groups.add('llama')
            else:
                groups.add('head')
        return tuple(sorted(groups))

    def _get_runner(self, device):
        from .train import Stage2Trainer
        vt = self._vision_tower()
        self._check_branches(vt)
        groups = self._trainable_groups()
        key = (str(device), id(vt), tuple(sorted(self._token_ids(vt.config).items())), groups)
        st = self.__dict__['_g4r_runner']
        ver = _param_version(self)
        if st.get('key') != key:
            st.clear()
            self.__dict__['_g4r_engine'].clear()       # the inference engine's copy would double the footprint
            st['runner'] = Stage2Trainer(self._engine_config(self.config, vt), self.state_dict(), vt.state_dict(), device,
                                         trainable=groups, own_optimizer=False, max_grad_norm=None)
            st['key'], st['ver'] = key, ver
        elif st.get('ver') != ver:
            st['runner'].load_weights(self.state_dict())
            st['ver'] = ver
        return st['runner']

    # ---- reference-facing forward (spi_llava.py:226-240 + llava.py:203-261) -------------
    def forward(self, input_ids: torch.LongTensor = None, attention_mask: Optional[torch.Tensor] = None,
                past_key_values: Optional[List[torch.FloatTensor]] = None,
                inputs_embeds: Optional[torch.FloatTensor] = None, labels: Optional[torch.LongTensor] = None,
                use_cache: Optional[bool] = None, output_attentions: Optional[bool] = None,
                output_hidden_states: Optional[bool] = None, images: Optional[torch.FloatTensor] = None,
                return_dict: Optional[bool] = None, img_metas=None, bboxes=None, logits_to_keep: int = 0, **kwargs):
        """logits_to_keep=1 (HF's convention; our prepare_inputs_for_generation sets it): the prefill computes the
        final norm + lm_head for the last position only and returns logits [B,1,V]."""
        if output_attentions or output_hidden_states:
            raise NotImplementedError('attention maps / per-layer hidden states are not materialised by the fused engine')
        return_dict = return_dict if return_dict is not None else getattr(self.config, 'use_return_dict', True)
        dev = (input_ids if input_ids is not None else inputs_embeds).device
        named = [(n, p) for n, p in self.named_parameters() if p.requires_grad]
        train_path = self.training and torch.is_grad_enabled() and labels is not None and bool(named)
        if train_path:
            if inputs_embeds is not None or past_key_values is not None:
                raise NotImplementedError('the training forward takes input_ids (HF Trainer passes the collator keys, data_modules.py:41-54)')
            images = _stack_images(images)
            if images is None:
                raise NotImplementedError('training batches carry one image per sample (data_modules.py:46-52)')
            runner = self._get_runner(dev)
            loss = _TrainStepFn.apply(runner, input_ids, images, bboxes, labels, tuple(n for n, _ in named),
                                      *[p for _, p in named])
            B, L = input_ids.shape
            logits = runner.stack.saved['logits'].view(B, L, -1).detach()
            if not return_dict:
                return (loss, logits)
            return CausalLMOutputWithPast(loss=loss, logits=logits, past_key_values=None, hidden_states=None, attentions=None)
        if self.training and torch.is_grad_enabled() and bool(named) and labels is None:
            raise NotImplementedError('a differentiable forward needs `labels` (the loss is part of the fused training node)')
        eng = self._get_engine(dev)
        logits, cache = _run_engine(eng, input_ids, images, bboxes, attention_mask, past_key_values, inputs_embeds,
                                    use_cache, want='logits', training=self.training,
                                    last_only=(logits_to_keep == 1 and labels is None),
                                    new_prompt=bool(kwargs.get('is_first_iteration')), logits_to_keep=logits_to_keep)
        loss = None
        if labels is not None:  # llava.py:238-249
            shift_logits = logits[..., :-1, :].float().reshape(-1, self.config.vocab_size)
            shift_labels = labels[..., 1:].reshape(-1).to(shift_logits.device)
            loss = nn.functional.cross_entropy(shift_logits, shift_labels)
        if not return_dict:
            return (loss, logits, cache) if loss is not None else (logits, cache)
        return CausalLMOutputWithPast(loss=loss, logits=logits, past_key_values=cache, hidden_states=None, attentions=None)

    def prepare_inputs_for_generation(self, input_ids, past_key_values=None, attention_mask=None, inputs_embeds=None,
                                      **kwargs):
        """llava/model/llava.py:263-283: after the first step only the last token is fed; `images` ride along (the
        forward skips the vision branch for one-token inputs, spi_llava.py:47-48).  A generate call's prompt on a
        non-empty cache (a later turn of a conversation, a regenerated or a shorter one) is passed whole, with its mask:
        the forward reuses the prefix the cache holds and prefills the rest.  The prompt is HF's first iteration
        (`is_first_iteration`); without that flag, an input longer than the cache plus one token is taken as one.
        After the first iteration the tokens the cache does not hold yet are passed: the last one, or with assisted
        decoding (prompt_lookup_num_tokens) the last one and the candidate tokens, whose logits the forward keeps as
        HF's logits_to_keep asks."""
        cache = _find_cache(past_key_values)
        first = kwargs.get('is_first_iteration')
        if cache is not None and cache.kv.length > 0:
            decode = (input_ids.shape[1] == cache.kv.length + 1) if first is None else not first
            if decode:
                input_ids = input_ids[:, min(cache.kv.length, input_ids.shape[1] - 1):]
        if inputs_embeds is not None and (cache is None or cache.kv.length == 0):
            model_inputs = {'inputs_embeds': inputs_embeds}
        else:
            model_inputs = {'input_ids': input_ids}
        model_inputs.update({'past_key_values': past_key_values, 'use_cache': kwargs.get('use_cache'),
                             'attention_mask': attention_mask, 'images': kwargs.get('images', None),
                             'logits_to_keep': 1})
        if 'bboxes' in kwargs:
            model_inputs['bboxes'] = kwargs['bboxes']
        if first:
            model_inputs['is_first_iteration'] = True
        return model_inputs

    @staticmethod
    def _expand_inputs_for_generation(expand_size=1, is_encoder_decoder=False, input_ids=None, **model_kwargs):
        """HF's expansion (beam search, num_return_sequences) repeats tensors only; the per-sample python lists of
        `bboxes` and `images` are repeated the same way (row i -> rows i*expand_size ..), so every expanded row keeps
        its own boxes."""
        input_ids, model_kwargs = LlamaForCausalLM._expand_inputs_for_generation(
            expand_size=expand_size, is_encoder_decoder=is_encoder_decoder, input_ids=input_ids, **model_kwargs)
        if expand_size > 1:
            for key in ('bboxes', 'images'):
                v = model_kwargs.get(key)
                if isinstance(v, (list, tuple)):
                    model_kwargs[key] = [x for x in v for _ in range(expand_size)]
        return input_ids, model_kwargs

    @torch.no_grad()
    def generate(self, input_ids=None, images=None, bboxes=None, max_new_tokens=32, do_sample=None,
                 temperature=None, stopping_criteria=None, eos_token_id=None, use_hf_loop=False, **kwargs):
        """Region-token prefill + KV-cache decode on the sm_90a engine.  Accepts the arguments the demo
        passes (gpt4roi/app.py:293-300); boxes may be given here or bound the way app.py does
        (`self.forward = partial(self.forward, bboxes=...)`, :286-291).  Returns ids [B, L+new] like HF.
        use_hf_loop=True runs transformers' own GenerationMixin.generate over this model's forward /
        prepare_inputs_for_generation / past_key_values instead of the engine's loop.
        attention_mask (right- or left-padded) and pad_token_id reach either loop: prompts of different lengths in one
        batch each continue from their own last token, and finished rows are filled with pad_token_id.
        The engine loop resolves the call's keywords, generation_config= and the model's generation config once, as
        transformers resolves them (resolve_generate), and refuses what it does not run before it builds an engine.
        Sampling there follows HF's resolution of do_sample / temperature / top_k / top_p (the demo's call samples
        from the top 50 at T = 0.2, as on the HF loop); the draws are keyed by torch's default generator (or
        `generator=`), so torch.manual_seed makes them reproducible.  repetition_penalty, no_repeat_ngram_size,
        min_length and min_new_tokens (with HF's resolved eos list) run there too, on the device inside the decode
        step, greedy or sampled; other logits processors raise NotImplementedError there.
        stop_strings (with tokenizer=, as transformers' generate takes them) are matched on the device, per row,
        inside the decode step (engine.StopStrings): a row that has produced a stop string is finished
        and, when eos_token_id and pad_token_id are given, filled with pad_token_id, as on the HF loop.  Host
        stopping_criteria (KeywordsStoppingCriteria) keep running as callbacks after every token.
        num_beams > 1 (do_sample false) runs beam search on the engine loop (length_penalty, early_stopping,
        num_return_sequences, eos / max length as HF resolves them): the prompt is prefilled once per sample and the
        beams share its KV cache; beam sampling, logits processors, stopping_criteria, stop_strings and
        past_key_values raise NotImplementedError there, and run with use_hf_loop=True.
        do_sample with num_return_sequences = N > 1 returns N independent samples per prompt, [B * N, L + new] with row
        b*N + i sample i of prompt b, as HF does; the engine loop prefills each prompt once and its N rows share the
        prompt's KV cache.  With past_key_values it raises NotImplementedError (run it with use_hf_loop=True).
        return_dict_in_generate with output_scores / output_logits returns, on the engine loop too, transformers'
        GenerateDecoderOnlyOutput (GenerateBeamDecoderOnlyOutput with beam search: sequences_scores,
        beam_indices) with HF's scores / logits, written by the selection and beam kernels inside the graphed step;
        model.compute_transition_scores takes them.  Its past_key_values is the caller's cache when one was passed,
        else None.  output_attentions / output_hidden_states raise NotImplementedError on both loops.
        prompt_lookup_num_tokens = k (max_matching_ngram_size, default 2), transformers' prompt lookup decoding: on
        the engine loop each step drafts up to k tokens by copying what followed the earliest earlier occurrence of
        the sequence's last n-gram in the prompt or the answer, and verifies them in one graphed
        decode step over k + 1 rows (engine.LookupDecode), so a repetitive answer takes fewer weight passes.  It runs
        for batch 1 with greedy or temperature / top_k / top_p selection, one eos id or a list, past_key_values and
        host stopping_criteria (called as HF's assisted decoding calls them); the tokens are the plain loop's, up to the
        attention's summation order, and a streamer= gets the prompt, then each step's accepted tokens (transformers'
        BaseStreamer contract, as HF's generate drives it).  When sampling with top_k / top_p, HF's own assisted loop
        also drops draft ids its warpers mask on constant logits; the engine's draft rule does not, so drafts and accept
        counts (not the tokens' distribution) can differ from use_hf_loop=True's.  Any other call (batch > 1,
        logits processors, stop_strings, outputs, beams, num_return_sequences > 1) ignores the option and runs the plain
        loop.  With use_hf_loop=True transformers' own assisted decoding runs over this model's cache (G4RCache.crop)."""
        if bboxes is None:
            bboxes = getattr(getattr(self, 'forward', None), 'keywords', {}).get('bboxes')
        if use_hf_loop:
            eng = self._get_engine(input_ids.device)
            eng.decode_budget = int(max_new_tokens) + 8
            kw = dict(kwargs)
            if stopping_criteria is not None:
                kw['stopping_criteria'] = stopping_criteria
            if eos_token_id is not None:
                kw['eos_token_id'] = eos_token_id
            if do_sample and temperature is not None:
                kw['temperature'] = temperature
            return super().generate(input_ids, images=images, bboxes=bboxes, max_new_tokens=max_new_tokens,
                                    do_sample=bool(do_sample), use_cache=True, **kw)
        L = input_ids.shape[1]
        gen = {k: v for k, v in kwargs.items()
               if k not in ('attention_mask', 'past_key_values', 'generator', 'tokenizer')}
        r = resolve_generate(self, L, max_new_tokens, do_sample, temperature, eos_token_id, **gen)
        pkv = kwargs.get('past_key_values')
        # refusals, in the order a caller meets them, before an engine is built
        hf = 'runs on the HF loop only: pass use_hf_loop=True'
        if r.layer_outputs:
            raise NotImplementedError(_LAYER_OUTPUTS)
        if r.stop_strings is not None and kwargs.get('tokenizer') is None:
            raise ValueError(_STOP_STRINGS_NEED_TOKENIZER)
        if r.beam is not None:
            if r.do_sample:
                raise NotImplementedError('beam search with do_sample (beam sampling) ' + hf)
            if r.names:
                raise NotImplementedError('the engine loop applies no logits processor to beam search; %s %s'
                                          % (', '.join(r.names), hf))
            if stopping_criteria is not None:
                raise NotImplementedError('beam search with stopping_criteria ' + hf)
            if r.stop_strings is not None:
                raise NotImplementedError('beam search with stop_strings ' + hf)
            if pkv is not None:
                raise NotImplementedError('beam search on a conversation cache (past_key_values) ' + hf)
        elif r.other:
            raise NotImplementedError('the engine loop applies temperature, top_k, top_p, repetition_penalty, '
                                      'no_repeat_ngram_size, min_length and min_new_tokens only; %s run on the HF '
                                      'loop: pass use_hf_loop=True' % ', '.join(r.other))
        elif r.num_return_sequences > 1 and pkv is not None:
            raise NotImplementedError('several sampled answers per prompt (num_return_sequences=%d) on a conversation '
                                      'cache (past_key_values) run on the HF loop only: pass use_hf_loop=True'
                                      % r.num_return_sequences)
        outs = r.outputs
        eng = self._get_engine(input_ids.device)
        if r.beam is not None:
            beam = dict(r.beam)
            res = eng.generate(input_ids, images, bboxes, max_new_tokens=beam.pop('max_length') - L,
                               attention_mask=kwargs.get('attention_mask'), **beam, **outs)
            return _generate_output(res, outs, None) if outs['return_dict_in_generate'] else res
        lookup, ngram = r.lookup
        lk = {} if lookup is None else dict(prompt_lookup_num_tokens=lookup, max_matching_ngram_size=ngram,
                                            streamer=kwargs.get('streamer'))
        kv = None
        if pkv is not None:   # a conversation's cache: reused and left holding this turn too
            cache = _find_cache(pkv)
            if cache is None:
                cache = G4RCache(KVCache(eng.cfg, input_ids.shape[0], L + max_new_tokens, eng.dev))
                pkv._g4r_cache = cache      # ride on HF's Cache object, as the HF loop's prefill does
            cache.stepper = None
            kv = cache.kv
        procs = r.processors
        res = eng.generate(input_ids, images, bboxes, max_new_tokens=max_new_tokens, do_sample=r.do_sample,
                           temperature=r.temperature, top_k=r.top_k, top_p=r.top_p, stopping_criteria=stopping_criteria,
                           eos_token_id=eos_token_id, attention_mask=kwargs.get('attention_mask'),
                           pad_token_id=kwargs.get('pad_token_id'), cache=kv, generator=kwargs.get('generator'),
                           stop_strings=None if r.stop_strings is None else
                           stop_strings_from_tokenizer(kwargs['tokenizer'], r.stop_strings),
                           num_return_sequences=r.num_return_sequences, repetition_penalty=procs['repetition_penalty'],
                           no_repeat_ngram_size=procs['no_repeat_ngram_size'], min_length=procs['min_length'],
                           min_new_tokens=procs['min_new_tokens'], length_eos_ids=procs['eos_ids'], **outs, **lk)
        return _generate_output(res, outs, pkv) if outs['return_dict_in_generate'] else res

    def continuous_batcher(self, slots=8, max_len=2048, tokenizer=None, stop_strings=None, prefix_reuse=False,
                           request_options=False):
        """A ContinuousBatcher (engine.ContinuousBatcher: requests join and leave the graphed decode step one row at a
        time) on this model's engine, with `slots` rows of up to max_len tokens each.  stop_strings (with tokenizer=;
        the model's generation config counts, as in generate()) apply to every request.  Its submit(input_ids,
        images=, bboxes=, max_new_tokens=, **generate_kwargs) resolves each request's sampling rule as the engine loop
        of generate() does.  prefix_reuse=True: a request prefills only what no row already holds (a conversation sent
        again whole each turn, several questions on one image); its tokens are then those of
        generate(past_key_values=) on the conversation (engine.ContinuousBatcher).  request_options=True: each
        request may also carry repetition_penalty, no_repeat_ngram_size, min_length, min_new_tokens and its own stop
        strings, which end it alongside the batcher's (SeamBatcher.submit)."""
        stops = resolve_generate(self, 0, None, stop_strings=stop_strings).stop_strings
        if stops is not None and tokenizer is None:
            raise ValueError(_STOP_STRINGS_NEED_TOKENIZER)
        eng = self._get_engine(self.device)
        return SeamBatcher(self, ContinuousBatcher(eng, slots, max_len, None if stops is None else
                                                   stop_strings_from_tokenizer(tokenizer, stops),
                                                   prefix_reuse=prefix_reuse, request_options=request_options),
                           tokenizer, stops)

    def initialize_vision_tokenizer(self, mm_use_im_start_end, tokenizer, device, tune_mm_mlp_adapter=False,
                                    pretrain_mm_mlp_adapter=None):
        """spi_llava.py:242-306: token bookkeeping, embedding resize and the optional copy of the pretrained
        <im_start>/<im_end> embedding rows (plain tensor ops on parameters, as in the reference)."""
        vision_config = self.get_model().vision_tower[0].config
        vision_config.use_im_start_end = mm_use_im_start_end
        tokenizer.add_tokens([DEFAULT_IMAGE_PATCH_TOKEN], special_tokens=True)
        self.resize_token_embeddings(len(tokenizer))
        num_spi_tokens = tokenizer.add_tokens(['<bbox>', '<point>'], special_tokens=True)
        if mm_use_im_start_end:
            num_new_tokens = tokenizer.add_tokens([DEFAULT_IM_START_TOKEN, DEFAULT_IM_END_TOKEN], special_tokens=True)
            self.resize_token_embeddings(len(tokenizer))
            vision_config.im_start_token, vision_config.im_end_token = tokenizer.convert_tokens_to_ids(
                [DEFAULT_IM_START_TOKEN, DEFAULT_IM_END_TOKEN])
            num_new_tokens = num_new_tokens + num_spi_tokens
            inp = self.get_input_embeddings().weight.data
            out = self.get_output_embeddings().weight.data
            if num_new_tokens > 0:
                inp[-num_new_tokens:] = inp[:-num_new_tokens].mean(dim=0, keepdim=True)
                out[-num_new_tokens:] = out[:-num_new_tokens].mean(dim=0, keepdim=True)
            if tune_mm_mlp_adapter:   # spi_llava.py:274-281
                self.get_model().orig_embeds_params = [self.get_input_embeddings().weight.data.clone().to(device=device)]
                for p in self.get_input_embeddings().parameters():
                    p.requires_grad = True
                for p in self.get_output_embeddings().parameters():
                    p.requires_grad = False
            if pretrain_mm_mlp_adapter:   # spi_llava.py:283-296
                weights = torch.load(pretrain_mm_mlp_adapter, map_location='cpu')
                embed_tokens_weight = weights['model.embed_tokens.weight']
                n_im = num_new_tokens - num_spi_tokens
                if inp.shape == embed_tokens_weight.shape:
                    inp[-n_im:] = embed_tokens_weight[-n_im:]
                elif embed_tokens_weight.shape[0] == n_im:
                    inp[-n_im:] = embed_tokens_weight
                else:
                    raise ValueError('Unexpected embed_tokens_weight shape. Pretrained: %s. Current: %s. Numer of new tokens: %d.'
                                     % (tuple(embed_tokens_weight.shape), tuple(inp.shape), n_im))
        vision_config.im_patch_token = tokenizer.convert_tokens_to_ids([DEFAULT_IMAGE_PATCH_TOKEN])[0]
        vision_config.bbox_token = tokenizer.convert_tokens_to_ids(['<bbox>'])[0]
        vision_config.point_token = tokenizer.convert_tokens_to_ids(['<point>'])[0]
        for m in self.modules():
            m.tokenizer = tokenizer
        self.invalidate_engine()


class SeamBatcher:
    """model.continuous_batcher(): the engine's ContinuousBatcher (`batcher`) with generate()'s keyword resolution.
    tokenizer, stop_strings: the batcher's own (continuous_batcher(tokenizer=, stop_strings=)), which a batcher built
    with request_options=True unites with each request's stop strings."""

    def __init__(self, model, batcher, tokenizer=None, stop_strings=None):
        self.model, self.batcher = model, batcher
        self.tokenizer, self.stop_strings = tokenizer, tuple(stop_strings or ())
        self._vocab = {}                            # id(tokenizer) -> (tokenizer, token strings): cleaned once
        self._tables = collections.OrderedDict()    # (id(tokenizer), stop strings) -> (tokenizer, StopStrings)

    def _stop_table(self, tokenizer, stops):
        """The StopStrings of `stops` over `tokenizer`'s vocabulary, padded with ids it does not hold to the
        batcher's V_tok.  The vocabulary is cleaned once per tokenizer and a table built once per stop set, so a
        repeated set costs a dictionary lookup."""
        key = (id(tokenizer), stops)
        if key in self._tables:
            self._tables.move_to_end(key)
            return self._tables[key][1]
        if id(tokenizer) not in self._vocab:
            strings = _token_strings(tokenizer)
            strings += [None] * (self.batcher.V_tok - len(strings))
            self._vocab[id(tokenizer)] = (tokenizer, strings)
        self._tables[key] = (tokenizer, StopStrings(self._vocab[id(tokenizer)][1], stops))
        if len(self._tables) > 64:
            self._tables.popitem(last=False)
        return self._tables[key][1]

    def submit(self, input_ids, images=None, bboxes=None, max_new_tokens=32, do_sample=None, temperature=None,
               eos_token_id=None, generator=None, streamer=None, **generate_kwargs):
        """Queue one request ([1, L] or [L] ids) and return its engine.Request.  do_sample / temperature / top_k /
        top_p / generation_config resolve as on generate()'s engine loop (resolve_generate: `do_sample=True` alone
        samples from the top 50); eos_token_id stops the request as it stops that loop.  As on that loop, only the
        sampling rule (and what is refused below) is read from generation_config: max_new_tokens and eos_token_id are
        this call's arguments.  What the batcher does not run -- logits processors, beam search, several answers per
        prompt, generate outputs, stop strings per request (stop_strings=, or in generation_config) -- raises
        NotImplementedError naming model.generate.  tokenizer= is accepted and unused: the batcher's stop strings, if
        any, were resolved with its own tokenizer.
        On a batcher built with request_options=True, repetition_penalty, no_repeat_ngram_size, min_length and
        min_new_tokens resolve and run as on generate()'s engine loop, and stop strings (stop_strings=, else
        generation_config's, else the model's) are matched with the batcher's own: the request ends at the first
        string of either set.  They are matched over tokenizer=, else the batcher's tokenizer; with neither, HF's
        ValueError.  Other logits processors, beam search, several answers per prompt, generate outputs and
        past_key_values still raise NotImplementedError naming model.generate."""
        if self.batcher.request_options:
            return self._submit_options(input_ids, images, bboxes, max_new_tokens, do_sample, temperature,
                                        eos_token_id, generator, streamer, generate_kwargs)
        gen = {k: v for k, v in generate_kwargs.items() if k not in ('pad_token_id', 'attention_mask', 'tokenizer')}
        gc = gen.get('generation_config')
        for k, v in (('stop_strings', gen.pop('stop_strings', None)), ('past_key_values', gen.pop('past_key_values', None)),
                     ('generation_config.stop_strings', getattr(gc, 'stop_strings', None))):
            if v is not None:
                raise NotImplementedError('%s per request: the batcher takes stop strings once '
                                          '(continuous_batcher(tokenizer=, stop_strings=)) and has no conversation '
                                          'cache; run the request with model.generate' % k)
        mask = generate_kwargs.get('attention_mask')
        if mask is not None and not bool(torch.as_tensor(mask).bool().all()):
            raise NotImplementedError('a padded prompt: submit its tokens alone, or run it with model.generate')
        r = resolve_generate(self.model, torch.as_tensor(input_ids).shape[-1], None, do_sample, temperature,
                             eos_token_id, **gen)
        if r.num_return_sequences > 1:
            why = 'num_return_sequences > 1'
        elif r.layer_outputs:
            why = _LAYER_OUTPUTS
        elif r.outputs['return_dict_in_generate']:
            why = 'return_dict_in_generate / output_scores / output_logits'
        elif r.beam is not None:
            why = 'beam search (num_beams=%d) runs on the HF loop only: pass use_hf_loop=True' % r.beam['num_beams']
        elif r.names:
            why = ('the engine loop applies temperature, top_k and top_p only; %s run on the HF loop: pass '
                   'use_hf_loop=True' % ', '.join(r.names))
        else:
            why = None
        if why is not None:
            raise NotImplementedError('the continuous batcher selects with temperature, top_k and top_p only (%s): run '
                                      'this request with model.generate' % why)
        return self.batcher.submit(input_ids, images, bboxes, max_new_tokens, r.do_sample, r.temperature, r.top_k,
                                   r.top_p, generator, eos_token_id, streamer)

    def _submit_options(self, input_ids, images, bboxes, max_new_tokens, do_sample, temperature, eos_token_id,
                        generator, streamer, generate_kwargs):
        gen = {k: v for k, v in generate_kwargs.items() if k not in ('pad_token_id', 'attention_mask', 'tokenizer')}
        if gen.pop('past_key_values', None) is not None:
            raise NotImplementedError('past_key_values per request: the batcher has no conversation cache (build it '
                                      'with prefix_reuse=True and send the whole conversation); run the request with '
                                      'model.generate')
        mask = generate_kwargs.get('attention_mask')
        if mask is not None and not bool(torch.as_tensor(mask).bool().all()):
            raise NotImplementedError('a padded prompt: submit its tokens alone, or run it with model.generate')
        r = resolve_generate(self.model, torch.as_tensor(input_ids).shape[-1], None, do_sample, temperature,
                             eos_token_id, **gen)
        if r.num_return_sequences > 1:
            why = 'num_return_sequences > 1'
        elif r.layer_outputs:
            why = _LAYER_OUTPUTS
        elif r.outputs['return_dict_in_generate']:
            why = 'return_dict_in_generate / output_scores / output_logits'
        elif r.beam is not None:
            why = 'beam search (num_beams=%d) runs on the HF loop only: pass use_hf_loop=True' % r.beam['num_beams']
        elif r.other:
            why = '%s run on the HF loop: pass use_hf_loop=True' % ', '.join(r.other)
        else:
            why = None
        if why is not None:
            raise NotImplementedError('the continuous batcher selects with temperature, top_k, top_p, '
                                      'repetition_penalty, no_repeat_ngram_size, min_length and min_new_tokens only '
                                      '(%s): run this request with model.generate' % why)
        stops = None
        if r.stop_strings is not None:
            tok = generate_kwargs.get('tokenizer') or self.tokenizer
            if tok is None:
                raise ValueError(_STOP_STRINGS_NEED_TOKENIZER)
            union = tuple(dict.fromkeys(self.stop_strings + r.stop_strings))
            stops = self._stop_table(tok, union)
        procs = r.processors
        return self.batcher.submit(input_ids, images, bboxes, max_new_tokens, r.do_sample, r.temperature, r.top_k,
                                   r.top_p, generator, eos_token_id, streamer,
                                   repetition_penalty=procs['repetition_penalty'],
                                   no_repeat_ngram_size=procs['no_repeat_ngram_size'], min_length=procs['min_length'],
                                   min_new_tokens=procs['min_new_tokens'], length_eos_ids=procs['eos_ids'],
                                   stop_strings=stops)

    def step(self):
        return self.batcher.step()

    def run(self):
        return self.batcher.run()


class KeywordsStoppingCriteria:
    """llava/model/utils.py:26-46 (the demo's stop criterion, gpt4roi/app.py:280-282): stop when the last token
    is a one-token keyword or a keyword appears in the decoded continuation.  Works with both generate loops."""

    def __init__(self, keywords, tokenizer, input_ids):
        self.keywords = keywords
        ids = [tokenizer(k).input_ids for k in keywords]
        self.keyword_ids = [i[0] for i in ids if type(i) is list and len(i) == 1]
        self.tokenizer = tokenizer
        self.start_len = None
        self.input_ids = input_ids

    def __call__(self, output_ids, scores, **kwargs):
        if self.start_len is None:
            self.start_len = self.input_ids.shape[1]
            return False
        for kid in self.keyword_ids:
            if output_ids[0, -1] == kid:
                return True
        outputs = self.tokenizer.batch_decode(output_ids[:, self.start_len:], skip_special_tokens=True)[0]
        return any(k in outputs for k in self.keywords)
