"""Import shims that let the reference's OWN python modules run unmodified in the build
container (SURVEY.md Appendix A, variant 6b).  TEST INFRASTRUCTURE: used only by
tests/golden/make_golden.py and the optional live-reference tests, where the reference
tree is available ($GPT4ROI_REFERENCE).

  * leaf stubs for third-party packages that are not installed (addict, yapf, terminaltables,
    pycocotools, matplotlib) -- none of them is touched on the hot path;
  * `mmcv._ext` := proxy module whose only real entries are roi_align_forward/backward, backed by
    EITHER the reference's CPU kernel compiled unmodified (oracle/_ref, default) or the
    gpt4roi_b200 drop-in (use_b200=True) -- every other op raises when called;
  * AutoConfig / AutoModelForCausalLM.register no-op'ed (llava/model/llava.py:329 collides with
    the `llava` model type that newer transformers ship).
"""
import importlib
import os
import sys
import types

REF = os.environ.get('GPT4ROI_REFERENCE', '')
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _stub(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


class _AttrDict(dict):
    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)

    def __setattr__(self, k, v):
        self[k] = v


def install(use_b200=False):
    if not os.path.isdir(REF):
        raise RuntimeError('reference tree %s not present' % REF)
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    _stub('addict', Dict=_AttrDict)
    _stub('yapf')
    _stub('yapf.yapflib')
    _stub('yapf.yapflib.yapf_api', FormatCode=lambda s, **k: (s, False))
    _stub('terminaltables', AsciiTable=object)
    for n in ('pycocotools', 'pycocotools.coco', 'pycocotools.cocoeval', 'pycocotools.mask'):
        _stub(n, COCO=object, COCOeval=object)
    for n in ('matplotlib', 'matplotlib.pyplot', 'matplotlib.collections', 'matplotlib.patches'):
        if n not in sys.modules:
            try:
                importlib.import_module(n)
            except Exception:
                _stub(n, PatchCollection=object, Polygon=object)
    if REF not in sys.path:
        sys.path.insert(0, REF)
    if use_b200:
        from gpt4roi_b200 import mmcv_ext
        mmcv_ext.install()
    else:
        from oracle import build_ref
        ext = build_ref.load()
        from gpt4roi_b200 import mmcv_ext
        m = mmcv_ext._ExtModule('mmcv._ext')
        m.roi_align_forward = ext.roi_align_forward
        m.roi_align_backward = ext.roi_align_backward
        sys.modules['mmcv._ext'] = m
    import transformers
    transformers.AutoConfig.register = staticmethod(lambda *a, **k: None)
    transformers.AutoModelForCausalLM.register = classmethod(lambda cls, *a, **k: None)
    # llava/__init__ and llava/model/__init__ pull in MPT; register them as bare packages
    for name, path in (('llava', 'llava'), ('llava.model', 'llava/model')):
        if name not in sys.modules:
            pkg = types.ModuleType(name)
            pkg.__path__ = [os.path.join(REF, path)]
            sys.modules[name] = pkg


def load_layers(image_size=224):
    """gpt4roi/models/layers.py, unmodified for 224; for other sizes the three literals named in
    SURVEY.md 8(c) are lifted (asserts at :221-222,:290-291 and `* 224` at :297)."""
    install()
    if image_size == 224:
        return importlib.import_module('gpt4roi.models.layers')
    src = open(os.path.join(REF, 'gpt4roi', 'models', 'layers.py')).read()
    assert src.count('assert h == 16') == 2 and src.count('assert w == 16') == 2 and src.count('* 224') == 1
    src = src.replace('assert h == 16', 'pass').replace('assert w == 16', 'pass').replace('* 224', '* %d' % image_size)
    mod = types.ModuleType('gpt4roi_models_layers_%d' % image_size)
    exec(compile(src, 'layers_lifted_%d.py' % image_size, 'exec'), mod.__dict__)
    return mod


def build_roi_query_module(image_size=224):
    """The reference's own MLVLROIQueryModule(embed_dims=1024, out_dims=4096, num_levels=4) (gpt4roi/models/
    layers.py:198-236) on CPU -- used by bench.py's CPU arm in this container to time the reference's code path."""
    layers = load_layers(image_size)
    return layers.MLVLROIQueryModule(embed_dims=1024, out_dims=4096, num_levels=4)
