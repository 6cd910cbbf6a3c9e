"""CPU test: the model-seam mirror exposes exactly the reference's SPI parameter names/shapes
(SURVEY.md Appendix C, probed from the reference's own MLVLROIQueryModule)."""
import torch

APPENDIX_C = {
    **{'mlvl_fuse.input_conv.%d.weight' % i: (1024, 1026, 1, 1) for i in range(4)},
    **{'mlvl_fuse.input_conv.%d.bias' % i: (1024,) for i in range(4)},
    **{'mlvl_fuse.fuse_convs.%d.conv.weight' % i: (1024, 1024, 3, 3) for i in range(5)},
    **{'mlvl_fuse.fuse_convs.%d.gn.weight' % i: (1024,) for i in range(5)},
    **{'mlvl_fuse.fuse_convs.%d.gn.bias' % i: (1024,) for i in range(5)},
    **{'roi_align.pconvs.%d.weight' % i: (1024, 1024, 3, 3) for i in range(4)},
    **{'roi_align.pconvs.%d.bias' % i: (1024,) for i in range(4)},
    'roi_align.pos_embedd.0.weight': (256, 4), 'roi_align.pos_embedd.0.bias': (256,),
    'roi_align.pos_embedd.2.weight': (256,), 'roi_align.pos_embedd.2.bias': (256,),
    'roi_align.pos_embedd.3.weight': (1024, 256), 'roi_align.pos_embedd.3.bias': (1024,),
    'roi_align.pos_embedd.5.weight': (1024,), 'roi_align.pos_embedd.5.bias': (1024,),
    'roi_align.updims.weight': (4096, 1024), 'roi_align.updims.bias': (4096,),
    'roi_align.flatten_linear.weight': (1024, 200704), 'roi_align.flatten_linear.bias': (1024,),
}


def test_spi_module_state_dict_matches_reference_layout():
    from gpt4roi_b200.spi_llava import MLVLROIQueryModule
    with torch.device('meta'):
        m = MLVLROIQueryModule(embed_dims=1024, out_dims=4096, num_levels=4)
    got = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert got == APPENDIX_C
    assert len(got) == 43
    r = repr(m.roi_align.roi_layers[0])
    assert r == ('RoIAlign(output_size=(14, 14), spatial_scale=%s, sampling_ratio=2, pool_mode=avg, '
                 'aligned=True, use_torchvision=False)' % (1 / (14 / 8)))


def test_random_state_dict_uses_reference_names():
    from gpt4roi_b200.engine import EngineConfig, random_state_dicts
    cfg = EngineConfig(n_layers=0, vit_layers=0)
    with torch.device('meta'):
        pass
    sd, _ = random_state_dicts(cfg, 'cpu', dtype=torch.bfloat16)
    spi = {k[len('model.spi_module.'):]: tuple(v.shape) for k, v in sd.items() if k.startswith('model.spi_module.')}
    assert spi == APPENDIX_C


# ---------------------------------------------------------------------------------------------
# Model seam plumbing on CPU: a stub engine stands in for the CUDA engine so that the reference-facing
# control flow (forward / prepare_inputs_for_generation / past_key_values / HF generate / requires_grad
# groups / token-id resolution) is exercised without a GPU.  The GPU tests run the same entry points
# on the real engine (tests/test_model_seam_gpu.py).
# ---------------------------------------------------------------------------------------------
def _tiny_model(n_layers=1):
    from transformers import CLIPVisionConfig, CLIPVisionModel
    from gpt4roi_b200.spi_llava import LlavaConfig, SPILlavaMPTForCausalLM
    cfg = LlavaConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=n_layers, num_attention_heads=2,
                      num_key_value_heads=2, vocab_size=140, mm_vision_select_layer=-2, use_mm_proj=True,
                      mm_hidden_size=1024, tie_word_embeddings=False)
    with torch.device('meta'):
        m = SPILlavaMPTForCausalLM(cfg)
        vt = CLIPVisionModel(CLIPVisionConfig(hidden_size=32, intermediate_size=64, num_hidden_layers=2,
                                              num_attention_heads=2, image_size=28, patch_size=14))
    m.model.vision_tower = [vt]
    vc = vt.config
    vc.im_patch_token, vc.im_start_token, vc.im_end_token, vc.use_im_start_end = 131, 134, 135, True
    return m


class _StubEngine:
    """next-token rule: logits = one-hot((last_id + 1) % vocab); records the calls it receives."""

    def __init__(self, cfg):
        self.cfg, self.dev, self.calls = cfg, torch.device('cpu'), []

    def _logits(self, ids):
        out = torch.zeros(ids.shape[0], ids.shape[1], self.cfg.vocab)
        out.scatter_(2, ((ids + 1) % self.cfg.vocab)[..., None], 1.0)
        return out

    def forward(self, input_ids, images, bboxes, attention_mask=None, want='logits', cache=None, **kw):
        self.calls.append(('prefill', tuple(input_ids.shape), images is not None, bboxes))
        if cache is not None:
            cache.length = input_ids.shape[1]
        return self._logits(input_ids)

    def decode_step(self, ids, cache, pos_dev=None):
        self.calls.append(('decode', tuple(ids.shape), cache.length))
        cache.length += 1
        return self._logits(ids)


def test_full_model_state_dict_and_config_type():
    m = _tiny_model()
    keys = set(m.state_dict().keys())
    assert 'lm_head.weight' in keys and 'model.embed_tokens.weight' in keys and 'model.mm_projector.weight' in keys
    assert {k[len('model.spi_module.'):] for k in keys if k.startswith('model.spi_module.')} == set(APPENDIX_C)
    assert not any('vision_tower' in k for k in keys)          # python list: outside the state dict (llava.py:47-48)
    assert m.config.model_type == 'llava'                       # llava/model/llava.py:37


def test_hf_generate_loop_drives_the_seam_with_our_cache():
    """transformers' GenerationMixin.generate over forward / prepare_inputs_for_generation / past_key_values:
    one prefill with the images and boxes, then one-token decode steps on our cache."""
    from gpt4roi_b200.engine import EngineConfig
    m = _tiny_model().eval()
    ecfg = EngineConfig(image_size=28, vit_hidden=32, vit_heads=2, vit_layers=2, vit_mlp=64, hidden=64, n_heads=2,
                        n_layers=1, mlp=128, vocab=140)
    stub = _StubEngine(ecfg)
    m._get_engine = lambda device: stub
    ids = torch.tensor([[1, 5, 9]])
    boxes = [torch.tensor([[0.1, 0.1, 0.5, 0.5]])]
    out = m.generate(ids, images=torch.zeros(1, 3, 28, 28), bboxes=boxes, max_new_tokens=4, do_sample=False,
                     use_hf_loop=True, pad_token_id=0)
    assert out.tolist() == [[1, 5, 9, 10, 11, 12, 13]]
    kinds = [c[0] for c in stub.calls]
    assert kinds == ['prefill', 'decode', 'decode', 'decode']
    assert stub.calls[0][1] == (1, 3) and stub.calls[0][2] is True and stub.calls[0][3] is boxes
    assert [c[2] for c in stub.calls[1:]] == [3, 4, 5]           # cache length seen by each decode step


def test_engine_loop_resolves_each_call_once():
    """The engine loop's generate() and the batcher's submit() resolve a call's generation config once and build HF's
    processor list at most once, whatever the call asks for."""
    from tests.stop_tokenizer import seeded_tokenizer
    from tests.test_serve_cpu import _seam, _StubEngine as _ServeStub
    m = _seam(_ServeStub())
    sb = m.continuous_batcher(slots=1, max_len=16)
    calls = []

    class _Engine:
        def generate(self, input_ids, images, bboxes, **kw):
            calls.append(kw)
            res = dict(sequences=input_ids, scores=None, logits=None, sequences_scores=None,
                       beam_indices=torch.zeros(1, 1, dtype=torch.int32))
            return res if kw['return_dict_in_generate'] else input_ids
    m._get_engine = lambda device: _Engine()
    counts = dict(config=0, processors=0)

    def counted(name, key):
        orig = getattr(m, name)

        def f(*a, **kw):
            counts[key] += 1
            return orig(*a, **kw)
        setattr(m, name, f)
    counted('_prepare_generation_config', 'config')
    counted('_get_logits_processor', 'processors')
    ids = torch.tensor([[1, 5, 9]])
    tok = seeded_tokenizer(140, seed=1)
    for kw in (dict(), dict(do_sample=True, temperature=0.7), dict(num_beams=2), dict(prompt_lookup_num_tokens=3),
               dict(stop_strings='###', tokenizer=tok), dict(return_dict_in_generate=True, output_scores=True)):
        counts.update(config=0, processors=0)
        m.generate(ids, images=torch.zeros(1, 3, 28, 28), max_new_tokens=4, **kw)
        assert counts['config'] == 1 and counts['processors'] <= 1, (kw, counts)
    assert len(calls) == 6
    for kw in (dict(), dict(do_sample=True, top_k=5)):
        counts.update(config=0, processors=0)
        sb.submit(ids, max_new_tokens=2, **kw)
        assert counts['config'] == 1 and counts['processors'] <= 1, (kw, counts)


def test_prepare_inputs_for_generation_follows_reference():
    from gpt4roi_b200.engine import EngineConfig, KVCache
    from gpt4roi_b200.spi_llava import G4RCache
    m = _tiny_model()
    ids = torch.tensor([[1, 2, 3, 4]])
    img = torch.zeros(1, 3, 28, 28)
    first = m.prepare_inputs_for_generation(ids, past_key_values=None, attention_mask=None, images=img, use_cache=True)
    assert first['input_ids'].shape == (1, 4) and first['images'] is img and first['use_cache'] is True
    ecfg = EngineConfig(image_size=28, hidden=64, n_heads=2, n_layers=1, mlp=128, vocab=140)
    cache = G4RCache(KVCache(ecfg, 1, 16, 'cpu'))
    cache.kv.length = 4
    nxt = m.prepare_inputs_for_generation(torch.tensor([[1, 2, 3, 4, 5]]), past_key_values=cache, images=img)
    assert nxt['input_ids'].tolist() == [[5]] and nxt['past_key_values'] is cache          # llava.py:266-267
    emb = torch.zeros(1, 4, 64)
    assert 'inputs_embeds' in m.prepare_inputs_for_generation(ids, inputs_embeds=emb)       # llava.py:270-271


def test_trainable_groups_follow_requires_grad_flags():
    """ONLY_SPI / PROJ (gpt4roi/train/train.py:685-696) are expressed through requires_grad on the seam."""
    from gpt4roi_b200.train import trainable_from_env
    m = _tiny_model()
    assert m._trainable_groups() == ('embed', 'head', 'llama', 'proj', 'spi')
    for n, p in m.named_parameters():
        p.requires_grad = 'spi_module' in n
    assert m._trainable_groups() == ('spi',)
    for n, p in m.named_parameters():
        if 'mm_projector' in n:
            p.requires_grad = True
    assert m._trainable_groups() == ('proj', 'spi')
    assert trainable_from_env({'ONLY_SPI': '1'}) == (('spi',), 0.01)
    assert trainable_from_env({'ONLY_SPI': '1', 'PROJ': '1'}) == (('spi', 'proj'), 0.0)
    assert set(trainable_from_env({})[0]) == {'embed', 'proj', 'spi', 'llama', 'head'}


def test_bbox_token_resolves_through_tokenizer_like_the_reference():
    """app.py sets only im_patch/im_start/im_end on the vision config and model.model.tokenizer; the reference
    looks <bbox> up through the tokenizer (spi_llava.py:150-152)."""
    m = _tiny_model()

    class Tok:
        def convert_tokens_to_ids(self, toks):
            return [132 if t == '<bbox>' else 0 for t in toks]
    vc = m.model.vision_tower[0].config
    assert m._token_ids(vc)['bbox_token'] == -2
    m.model.tokenizer = Tok()
    ids = m._token_ids(vc)
    assert ids == dict(im_patch_token=131, bbox_token=132, im_start_token=134, im_end_token=135)
    vc.bbox_token = 133                                         # initialize_vision_tokenizer's attribute wins
    assert m._token_ids(vc)['bbox_token'] == 133


def test_keywords_stopping_criteria():
    from gpt4roi_b200.spi_llava import KeywordsStoppingCriteria

    class Tok:
        def __call__(self, s):
            return type('E', (), {'input_ids': [7] if s == '###' else [1, 2]})()

        def batch_decode(self, ids, skip_special_tokens=True):
            return [' '.join(str(int(i)) for i in row) for row in ids]
    ids = torch.tensor([[1, 2, 3]])
    sc = KeywordsStoppingCriteria(['###', '4 5'], Tok(), ids)
    assert sc(torch.tensor([[1, 2, 3, 9]]), None) is False      # first call only latches the prompt length
    assert sc(torch.tensor([[1, 2, 3, 9, 7]]), None) is True    # one-token keyword id
    assert sc(torch.tensor([[1, 2, 3, 4, 5]]), None) is True    # keyword in the decoded continuation
    assert sc(torch.tensor([[1, 2, 3, 8, 8]]), None) is False


def test_lr_schedule_matches_transformers():
    import torch.optim
    from transformers import get_cosine_schedule_with_warmup
    from gpt4roi_b200.train import lr_lambda, warmup_steps_for
    total = 200
    warm = warmup_steps_for(total, 0, 0.03)
    assert warm == 6 and warmup_steps_for(total, 3000, 0.003) == 3000     # warmup_steps wins (train_stage2.sh:49-50)
    p = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.AdamW([p], lr=2e-5)
    sch = get_cosine_schedule_with_warmup(opt, warm, total)
    for step in range(total):
        want = opt.param_groups[0]['lr']
        assert abs(2e-5 * lr_lambda(step, total, warm) - want) < 1e-12, step
        opt.step()
        sch.step()
