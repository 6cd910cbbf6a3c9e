"""CPU tests of the CLIPImageProcessor image path (gpt4roi/app.py:118-136, gpt4roi/datasets/vcr.py:173-189): the oracle
(oracle/clip_oracle.py) pinned to PIL's BICUBIC resize, to transformers' PIL CLIP processor and to torch's CPU
F.interpolate; the host tables of gpt4roi_b200.input_pipeline.ClipPreprocessor replayed in numpy exactly as
csrc/clip_preprocess.cu reads them; box normalisation; refusal of malformed input."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import clip_oracle as O
from gpt4roi_b200 import input_pipeline as IP

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (h, w): downscales of the short side from 1.01x to 10.3x, upscales (short side < 224), short side exactly 224,
# 1 x 1 and 1 x N, extreme aspects; (23000, 226) takes PIL's vertical-first order (taller than 100 x its width and
# shrinking in height)
SHAPES = [(226, 300), (230, 229), (250, 251), (300, 400), (333, 500), (480, 640), (640, 480), (448, 449), (600, 900),
          (720, 1280), (1080, 1920), (1000, 1003), (1500, 2000), (2300, 2400), (2400, 2310),
          (224, 224), (224, 300), (400, 224), (224, 225), (225, 224),
          (1, 1), (1, 7), (7, 1), (1, 2), (2, 2), (3, 5), (13, 17), (50, 60), (100, 150), (150, 100), (199, 223),
          (223, 500), (3000, 40), (40, 3000), (2000, 7), (5, 900), (41, 3001), (23000, 226)]


def _seeded_shapes(n=8):
    rng = np.random.default_rng(7)
    return [(int(rng.integers(1, 1200)), int(rng.integers(1, 1200))) for _ in range(n)]


ALL_SHAPES = SHAPES + _seeded_shapes()


def _image(h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


def _vector_isa():
    return torch.backends.cpu.get_cpu_capability() in ('AVX2', 'AVX512')


class _threads:
    """torch's CPU bilinear takes a channels-last kernel when it runs on one thread; pin the thread count."""

    def __init__(self, n):
        self.n = n

    def __enter__(self):
        self.old = torch.get_num_threads()
        torch.set_num_threads(self.n)

    def __exit__(self, *exc):
        torch.set_num_threads(self.old)


def _interpolate(pv, S):
    return F.interpolate(torch.from_numpy(pv)[None], (S, S), mode='bilinear', align_corners=False)[0].numpy()


def test_resized_size_matches_transformers():
    pytest.importorskip('transformers')
    from transformers.image_transforms import get_resize_output_image_size
    from transformers.image_utils import ChannelDimension
    for h, w in ALL_SHAPES + [(480, 640), (3000, 40), (7, 3)]:
        for se in (224, 336):
            want = get_resize_output_image_size(np.zeros((h, w, 1)), se, default_to_square=False,
                                                input_data_format=ChannelDimension.LAST)
            assert O.resized_size(h, w, se) == tuple(want) == IP.clip_resized_size(h, w, se), (h, w, se)
    assert O.resized_size(480, 640) == (224, 298) and O.resized_size(3000, 40) == (16800, 224)


def test_resize_matches_pil_bitwise():
    Image = pytest.importorskip('PIL.Image')
    assert len(ALL_SHAPES) >= 40
    for i, (h, w) in enumerate(ALL_SHAPES):
        img = _image(h, w, i)
        H, W = O.resized_size(h, w)
        want = np.asarray(Image.fromarray(img).resize((W, H), Image.BICUBIC))
        assert np.array_equal(O.resize_bicubic_u8(img, H, W), want), (h, w)


def test_resize_matches_pil_other_targets():
    """Downscales and upscales to targets that are not the short-side rule's, both axes changing."""
    Image = pytest.importorskip('PIL.Image')
    for i, (h, w, H, W) in enumerate([(300, 400, 37, 501), (17, 900, 64, 90), (2000, 3, 199, 41), (5, 5, 1, 1),
                                               (2000, 3, 2100, 41)]):
        img = _image(h, w, 100 + i)
        want = np.asarray(Image.fromarray(img).resize((W, H), Image.BICUBIC))
        assert np.array_equal(O.resize_bicubic_u8(img, H, W), want), (h, w, H, W)


def _processor():
    pytest.importorskip('PIL.Image')
    pytest.importorskip('transformers')
    try:
        from transformers.models.clip.image_processing_pil_clip import CLIPImageProcessorPil
    except ImportError:
        pytest.skip('transformers has no PIL CLIP image processor (CLIPImageProcessorPil)')
    return CLIPImageProcessorPil()


PV_SHAPES = [(480, 640), (640, 480), (226, 300), (1080, 1920), (224, 300), (400, 224), (1, 1), (1, 7), (13, 17),
             (100, 150), (3000, 40), (40, 3000), (223, 500), (2300, 2400), (23000, 226)]


def test_pixel_values_match_clip_processor_bitwise():
    from PIL import Image
    proc = _processor()
    for i, (h, w) in enumerate(PV_SHAPES):
        img = _image(h, w, 200 + i)
        want = proc.preprocess(Image.fromarray(img), do_center_crop=False, return_tensors='np')['pixel_values'][0]
        got = O.pixel_values(img)
        assert got.dtype == want.dtype == np.float32 and np.array_equal(got, want), (h, w)


def test_square_resample_matches_interpolate():
    """Bitwise where torch runs its generic separable kernel (more than one thread) built for AVX2 / AVX512, which
    contract the source-coordinate and lerp arithmetic into FMAs as the oracle does.  torch's baseline build rounds
    them separately: test_square_resample_baseline_isa_bound."""
    with _threads(max(2, torch.get_num_threads())):
        for i, (h, w) in enumerate(PV_SHAPES):
            pv = O.pixel_values(_image(h, w, 300 + i))
            for S in (224, 336):
                want, got = _interpolate(pv, S), O.bilinear_square(pv, S)
                if _vector_isa():
                    assert np.array_equal(got, want), (h, w, S)
                else:
                    assert np.abs(got - want).max() <= 2e-4, (h, w, S)


def test_square_resample_one_thread_bound():
    """On one thread torch takes its channels-last kernel for C = 3, which sums the four weighted pixels with
    precomputed products of the row and column lambdas: a few ulp from the two-lerp order (values are within +-3,
    ulp 2.4e-7)."""
    with _threads(1):
        for i, (h, w) in enumerate(PV_SHAPES[:6]):
            pv = O.pixel_values(_image(h, w, 400 + i))
            for S in (224, 336):
                assert np.abs(O.bilinear_square(pv, S) - _interpolate(pv, S)).max() <= 1.5e-6, (h, w, S)


def test_square_resample_baseline_isa_bound():
    """torch's non-vector (DEFAULT) CPU build rounds scale * (o + 0.5) before subtracting 0.5, which can move a
    source coordinate by one float32 ulp (3e-5 at 500) and so a lambda; with values within +-3 the output moves by at
    most ~1e-4."""
    code = ('import numpy as np, torch, torch.nn.functional as F\n'
            'from oracle import clip_oracle as O\n'
            'assert torch.backends.cpu.get_cpu_capability() == "DEFAULT"\n'
            'torch.set_num_threads(2)\n'
            'm = 0.0\n'
            'for i, (h, w) in enumerate([(223, 500), (1080, 1920), (3000, 40)]):\n'
            '    pv = O.pixel_values(np.random.default_rng(i).integers(0, 256, (h, w, 3), dtype=np.uint8))\n'
            '    for S in (224, 336):\n'
            '        t = F.interpolate(torch.from_numpy(pv)[None], (S, S), mode="bilinear", align_corners=False)[0]\n'
            '        m = max(m, float(np.abs(O.bilinear_square(pv, S) - t.numpy()).max()))\n'
            'print(m)\n')
    env = dict(os.environ, ATEN_CPU_CAPABILITY='default', PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    assert float(r.stdout.split()[-1]) <= 2e-4


def test_whole_path_matches_reference_path():
    """Oracle end to end == CLIPImageProcessorPil + F.interpolate, as the demo calls them."""
    from PIL import Image
    proc = _processor()
    with _threads(max(2, torch.get_num_threads())):
        for i, (h, w) in enumerate([(480, 640), (3000, 40), (1, 1), (226, 300)]):
            img = _image(h, w, 500 + i)
            pv = proc.preprocess(Image.fromarray(img), do_center_crop=False, return_tensors='pt')['pixel_values'][0]
            want = F.interpolate(pv.unsqueeze(0), size=(224, 224), mode='bilinear', align_corners=False).squeeze(0)
            got = O.clip_preprocess(img, 224)
            if _vector_isa():
                assert np.array_equal(got, want.numpy()), (h, w)
            else:
                assert np.abs(got - want.numpy()).max() <= 2e-4, (h, w)


def _replay_tables(img, S, se=224, mean=IP.CLIP_IMAGE_MEAN, std=IP.CLIP_IMAGE_STD):
    """csrc/clip_preprocess.cu's two passes in numpy, reading _clip_plan's tables exactly as the kernels do."""
    h, w = img.shape[:2]
    tab, (vf, nr, nc, k1, k2, o1, o2, oy, ox) = IP._clip_plan(h, w, S, se)
    lst = tab[:o1]
    e1 = tab[o1:o2].reshape(-1, 2 + k1)
    e2 = tab[o2:oy].reshape(-1, 2 + k2)
    by, bx = tab[oy:ox].reshape(S, 4), tab[ox:].reshape(S, 4)
    nrr, ncr = (nr, len(e2)) if vf else (len(e2), nc)                     # needed resized rows / columns
    assert (nr, nc) == ((len(e1), len(lst)) if vf else (len(lst), len(e1)))
    assert nrr <= 2 * S and ncr <= 2 * S and len(lst) <= (w if vf else h)
    src = img.astype(np.int64)
    if vf:
        src = src.transpose(1, 0, 2)                                        # a vertical pass is a horizontal one on
    tmp = np.full((len(lst), len(e1), 3), 1 << 21, np.int64)                # the transposed image
    for t in range(k1):
        live = t < e1[:, 1]
        tmp += src[lst][:, np.where(live, e1[:, 0] + t, 0)] * np.where(live, e1[:, 2 + t], 0)[None, :, None]
    tmp = np.clip(tmp >> 22, 0, 255)
    res = np.full((len(e2), tmp.shape[1], 3), 1 << 21, np.int64)
    for t in range(k2):
        live = t < e2[:, 1]
        res += tmp[np.where(live, e2[:, 0] + t, 0)] * np.where(live, e2[:, 2 + t], 0)[:, None, None]
    res = np.clip(res >> 22, 0, 255).astype(np.uint8)
    if vf:
        res = res.transpose(1, 0, 2)
    assert res.shape == (nrr, ncr, 3)
    x = O.rescale_normalize(res, mean, std)                                     # [3, nrr, ncr]
    ly0, ly1 = by[:, 2].view(np.float32), by[:, 3].view(np.float32)
    lx0, lx1 = bx[:, 2].view(np.float32), bx[:, 3].view(np.float32)
    r0, r1 = x[:, by[:, 0]], x[:, by[:, 1]]
    t0 = O.fma32(r0[:, :, bx[:, 0]], lx0, (r0[:, :, bx[:, 1]] * lx1).astype(np.float32))
    t1 = O.fma32(r1[:, :, bx[:, 0]], lx0, (r1[:, :, bx[:, 1]] * lx1).astype(np.float32))
    return O.fma32(t0, ly0[:, None], (t1 * ly1[:, None]).astype(np.float32))


def test_host_tables_replay_equals_oracle():
    """The tap windows, fixed-point weights, row selection and bilinear tables the kernel reads give the oracle's
    output bit for bit, including the work bound: at most 2S resized rows and columns per image."""
    assert IP._clip_plan(23000, 226, 224, 224)[1][0] == 1 and IP._clip_plan(3000, 40, 224, 224)[1][0] == 0
    for i, (h, w) in enumerate(SHAPES[::2] + [(23000, 226), (2000, 7)] + _seeded_shapes(3)):
        img = _image(h, w, 600 + i)
        for S, se in ((224, 224), (336, 224), (336, 336)):
            assert np.array_equal(_replay_tables(img, S, se), O.clip_preprocess(img, S, se)), (h, w, S, se)


def test_bilinear_tables_equal_oracle():
    for n in (1, 16, 223, 224, 225, 298, 336, 500, 16800):
        for S in (224, 336):
            a, b = IP._bilinear_axis(n, S), O.bilinear_axis(n, S)
            for x, y in zip(a, b):
                assert x.dtype.kind == y.dtype.kind and np.array_equal(x, y), (n, S)


def test_box_normalisation_is_vcr_arithmetic():
    rng = np.random.default_rng(9)
    for h, w in [(480, 640), (3000, 40), (1, 1), (333, 517)]:
        boxes = rng.uniform(0, max(h, w), (5, 4))
        want = (boxes[:, :4] / np.array([w, h, w, h])[None]).astype(np.float32)     # vcr.py:179, then float32
        for b in (boxes, torch.from_numpy(boxes), boxes.tolist()):
            got = IP.normalize_boxes(b, h, w)
            assert got.dtype == np.float32 and np.array_equal(got, want)
        assert np.array_equal(O.normalize_boxes(boxes, h, w), want)


def test_clip_preprocessor_refuses_cpu_and_bad_input():
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        IP.ClipPreprocessor(device='cpu')
    with pytest.raises(TypeError, match='float32, bfloat16 or float16'):
        IP.ClipPreprocessor(device='cuda:0', out_dtype=torch.float64)
    pre = IP.ClipPreprocessor(device='cuda:0')          # no CUDA call before a launch: the checks come first
    ok = np.zeros((4, 4, 3), np.uint8)
    with pytest.raises(TypeError, match='uint8 HWC with 3 channels'):
        pre([ok, np.zeros((4, 4, 3), np.float32)])
    with pytest.raises(TypeError, match='uint8 HWC with 3 channels'):
        pre([np.zeros((4, 4, 4), np.uint8)])
    with pytest.raises(TypeError, match='uint8 HWC with 3 channels'):
        pre([np.zeros((4, 4), np.uint8)])
    with pytest.raises(TypeError, match='uint8 HWC with 3 channels'):
        pre([torch.zeros(3, 4, 4, dtype=torch.uint8)])
    with pytest.raises(ValueError, match='empty image'):
        pre([np.zeros((0, 4, 3), np.uint8)])
    with pytest.raises(ValueError, match='1..65535 images'):
        pre([])
    with pytest.raises(ValueError, match='box lists'):
        pre([ok, ok], boxes=[np.zeros((1, 4))])
    Image = pytest.importorskip('PIL.Image')
    with pytest.raises(TypeError, match='mode RGB'):
        pre([Image.fromarray(np.zeros((4, 4), np.uint8))])
