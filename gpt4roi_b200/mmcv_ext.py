"""`mmcv._ext` drop-in: lets the reference's own `mmcv.ops.roi_align` / `RoIAlign`
(mmcv-1.4.7/mmcv/ops/roi_align.py) run UNCHANGED on the sm_90a kernels.

`mmcv/utils/ext_loader.py:12-16` only does `importlib.import_module('mmcv._ext')` and
`assert hasattr(ext, fun)`.  The reference tree is read-only and mmcv is not pip
installed, so the replacement cannot be copied to `mmcv/_ext*.so`; instead `install()`
registers a module object under `sys.modules['mmcv._ext']` BEFORE `mmcv.ops` is first
imported.  `roi_align_forward` / `roi_align_backward` are the real entry points
(keyword-callable with the 11 argument names of pybind.cpp:611-620); every other symbol
that `mmcv/ops/__init__.py` asserts on (~150 names of ops GPT4RoI never calls) resolves to
a stub that raises NotImplementedError when CALLED, so `import mmcv.ops` succeeds and
nothing silently falls back.
"""
import importlib
import sys
import types

# the package re-exports the *function* `roi_align`, which shadows the submodule attribute
_ra = importlib.import_module(__package__ + '.roi_align')


class _ExtModule(types.ModuleType):
    def __getattr__(self, name):
        if name.startswith('__'):
            raise AttributeError(name)

        def _unavailable(*args, **kwargs):
            raise NotImplementedError(
                'mmcv._ext.%s is not part of the GPT4RoI region-token path; gpt4roi_b200 '
                'provides only roi_align_forward/roi_align_backward' % name)
        _unavailable.__name__ = name
        return _unavailable


def make_module():
    m = _ExtModule('mmcv._ext')
    m.__doc__ = 'gpt4roi_b200 drop-in for mmcv._ext (sm_90a RoIAlign)'
    m.roi_align_forward = _ra.roi_align_forward
    m.roi_align_backward = _ra.roi_align_backward
    m.__gpt4roi_b200__ = True
    return m


def install(force=False):
    """Register the drop-in as `mmcv._ext`.  Call before `import mmcv.ops`."""
    cur = sys.modules.get('mmcv._ext')
    if cur is not None and not force:
        if getattr(cur, '__gpt4roi_b200__', False):
            return cur
        raise RuntimeError('mmcv._ext is already imported (%r); install() must run before '
                           'mmcv.ops is imported, or pass force=True' % (cur,))
    if 'mmcv.ops.roi_align' in sys.modules and not force:
        raise RuntimeError('mmcv.ops.roi_align was imported before gpt4roi_b200.mmcv_ext.install()')
    m = make_module()
    sys.modules['mmcv._ext'] = m
    pkg = sys.modules.get('mmcv')
    if pkg is not None:
        setattr(pkg, '_ext', m)
    return m
