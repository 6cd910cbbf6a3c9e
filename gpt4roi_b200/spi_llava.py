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
import weakref
from typing import List, Optional

import torch
import torch.nn as nn
from transformers import LlamaConfig, LlamaForCausalLM, LlamaModel
from transformers.modeling_outputs import BaseModelOutputWithPast, CausalLMOutputWithPast

from .engine import BF16, EngineConfig, KVCache, PrefillEngine
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
    lens = m.sum(1)
    if bool((lens == L).all()):
        return None
    if not bool((m == (torch.arange(L, device=eng.dev)[None] < lens[:, None])).all()):
        raise NotImplementedError('only right-padded attention masks are supported (data_modules.py:33-44 pads right)')
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
                training=False, max_cache=None, last_only=False):
    """Inference dispatch shared by both model classes: prefill (ids or embeds, with or without the vision
    branch) or one decode step on our cache.  Mirrors spi_llava.py:44-48: the vision branch runs when images are
    given and (the input is longer than one token or the module is in training mode)."""
    c = eng.cfg
    cache = _find_cache(past_key_values)
    if cache is not None and cache.kv.length > 0:
        if inputs_embeds is not None:
            raise NotImplementedError('decode steps take input_ids')
        if input_ids.shape[1] != 1:
            input_ids = input_ids[:, -1:]
        ids = input_ids.to(eng.dev).contiguous()
        if cache.stepper is None and c.head_dim == 128 and cache.kv.length + 4 < cache.kv.max_len:
            from .engine import GraphedDecode
            cache.stepper = GraphedDecode(eng, cache.kv)
        out = cache.stepper.step(ids) if cache.stepper is not None else eng.decode_step(ids, cache.kv)
        if want == 'hidden':
            raise NotImplementedError('decode steps return logits (use the CausalLM wrapper)')
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
        x = inputs_embeds.to(eng.dev, eng.dt).contiguous()
        if kv is not None:
            kv.length = L
        out = eng.llama(x, B, L, seqlens=_seqlens(eng, attention_mask, L), cache=kv, want=want, last_only=last_only)
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
                                    last_only=(logits_to_keep == 1 and labels is None))
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
        forward skips the vision branch for one-token inputs, spi_llava.py:47-48)."""
        cache = _find_cache(past_key_values)
        if cache is not None and cache.kv.length > 0:
            input_ids = input_ids[:, -1:]
        if inputs_embeds is not None and (cache is None or cache.kv.length == 0):
            model_inputs = {'inputs_embeds': inputs_embeds}
        else:
            model_inputs = {'input_ids': input_ids}
        model_inputs.update({'past_key_values': past_key_values, 'use_cache': kwargs.get('use_cache'),
                             'attention_mask': attention_mask, 'images': kwargs.get('images', None),
                             'logits_to_keep': 1})
        if 'bboxes' in kwargs:
            model_inputs['bboxes'] = kwargs['bboxes']
        return model_inputs

    @torch.no_grad()
    def generate(self, input_ids=None, images=None, bboxes=None, max_new_tokens=32, do_sample=False,
                 temperature=1.0, stopping_criteria=None, eos_token_id=None, use_hf_loop=False, **kwargs):
        """Region-token prefill + KV-cache decode on the sm_90a engine.  Accepts the arguments the demo
        passes (gpt4roi/app.py:293-300); boxes may be given here or bound the way app.py does
        (`self.forward = partial(self.forward, bboxes=...)`, :286-291).  Returns ids [B, L+new] like HF.
        use_hf_loop=True runs transformers' own GenerationMixin.generate over this model's forward /
        prepare_inputs_for_generation / past_key_values instead of the engine's loop."""
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
            if do_sample:
                kw['temperature'] = temperature
            return super().generate(input_ids, images=images, bboxes=bboxes, max_new_tokens=max_new_tokens,
                                    do_sample=do_sample, use_cache=True, **kw)
        eng = self._get_engine(input_ids.device)
        return eng.generate(input_ids, images, bboxes, max_new_tokens=max_new_tokens, do_sample=do_sample,
                            temperature=temperature, stopping_criteria=stopping_criteria, eos_token_id=eos_token_id)

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
