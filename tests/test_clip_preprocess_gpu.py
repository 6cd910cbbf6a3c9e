"""GPU tests of ClipPreprocessor (csrc/clip_preprocess.cu): the CLIPImageProcessor + F.interpolate image path of the
demo and the VCR / LLaVA-instruct datasets, bit for bit against the oracle (oracle/clip_oracle.py, itself pinned to
PIL, transformers and torch by tests/test_clip_preprocess_cpu.py) on ragged batches of host and device images; bf16 /
fp16 output as torch's .to() of the fp32 result; generate() on the kernel's images against the reference path's."""
import numpy as np
import pytest
import torch

from gpt4roi_b200.input_pipeline import ClipPreprocessor
from oracle import clip_oracle as O

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'

# downscales 1.01x .. 10x, upscales, short side exactly 224, 1 x 1, 1 x N, extreme aspects, PIL's vertical-first order
EDGE = [(226, 300), (480, 640), (640, 480), (1080, 1920), (2300, 2400), (224, 300), (400, 224), (224, 224), (1, 1),
        (1, 7), (7, 1), (13, 17), (100, 150), (3000, 40), (40, 3000), (223, 500), (23000, 226)]
_ORACLE = {}


def _image(h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


def _want(h, w, seed, S):
    key = (h, w, seed, S)
    if key not in _ORACLE:
        _ORACLE[key] = O.clip_preprocess(_image(h, w, seed), S)
    return _ORACLE[key]


def _batch(B, seed):
    rng = np.random.default_rng(seed)
    shapes = [EDGE[i % len(EDGE)] for i in range(seed, seed + B)] if B > 1 else [EDGE[seed % len(EDGE)]]
    shapes = [s if rng.random() < 0.6 else (int(rng.integers(1, 700)), int(rng.integers(1, 700))) for s in shapes]
    return [(h, w, 1000 * seed + i) for i, (h, w) in enumerate(shapes)]


def _inputs(spec, kinds):
    out = []
    for (h, w, sd), kind in zip(spec, kinds):
        img = _image(h, w, sd)
        if kind == 'numpy':
            out.append(img)
        elif kind == 'cpu':
            out.append(torch.from_numpy(img))
        else:
            out.append(torch.from_numpy(img).to(DEV))
    return out


@pytest.mark.parametrize('B,seed', [(1, 0), (1, 3), (7, 1), (32, 2)])
@pytest.mark.parametrize('S', [224, 336])
def test_fp32_bitwise_ragged(B, seed, S):
    spec = _batch(B, seed + S)
    kinds = [('numpy', 'cpu', 'cuda')[(i + seed) % 3] for i in range(B)]
    pre = ClipPreprocessor(S=S, device=DEV, out_dtype=torch.float32)
    got, boxes = pre(_inputs(spec, kinds))
    assert got.shape == (B, 3, S, S) and got.dtype == torch.float32 and boxes == []
    got = got.cpu().numpy()
    for b, (h, w, sd) in enumerate(spec):
        want = _want(h, w, sd, S)
        assert np.array_equal(got[b], want), (b, h, w, kinds[b], float(np.abs(got[b] - want).max()))


def test_every_edge_shape_from_host_and_device():
    """Each edge shape alone and all of them in one batch, from host and from device memory; a second call on the
    same preprocessor reuses its pinned buffer."""
    spec = [(h, w, 77 + i) for i, (h, w) in enumerate(EDGE)]
    want = np.stack([_want(h, w, sd, 224) for h, w, sd in spec])
    pre = ClipPreprocessor(device=DEV, out_dtype=torch.float32)
    for kind in ('numpy', 'cuda'):
        got = pre(_inputs(spec, [kind] * len(spec)))[0].cpu().numpy()
        assert np.array_equal(got, want), kind
    for i, s in enumerate(spec):
        assert np.array_equal(pre(_inputs([s], ['cpu']))[0][0].cpu().numpy(), want[i]), s


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
def test_half_outputs_are_rounded_fp32(dtype):
    spec = _batch(7, 5)
    want = torch.from_numpy(np.stack([_want(h, w, sd, 224) for h, w, sd in spec])).to(dtype)
    got, _ = ClipPreprocessor(device=DEV, out_dtype=dtype)(_inputs(spec, ['numpy', 'cuda'] * 4))
    assert got.dtype == dtype
    assert torch.equal(got.cpu().view(torch.int16), want.view(torch.int16))


def test_pil_input_and_boxes():
    Image = pytest.importorskip('PIL.Image')
    img = _image(333, 517, 9)
    boxes = [np.array([[10.5, 20, 300, 330], [0, 0, 517, 333]]), torch.tensor([[1.0, 2.0, 3.0, 4.0]])]
    got, nb = ClipPreprocessor(device=DEV, out_dtype=torch.float32)([Image.fromarray(img), img], boxes)
    want = O.clip_preprocess(img, 224)
    assert np.array_equal(got[0].cpu().numpy(), want) and np.array_equal(got[1].cpu().numpy(), want)
    for b, n in zip(boxes, nb):
        assert n.dtype == torch.float32 and np.array_equal(n.numpy(), O.normalize_boxes(np.asarray(b), 333, 517))


def test_generate_on_kernel_images_equals_reference_path():
    """The demo's path (gpt4roi/app.py:118-136): CLIPImageProcessorPil + F.interpolate + .half(), boxes / [w, h, w, h];
    generate() on the kernel's fp16 images and boxes gives the same tokens."""
    pytest.importorskip('PIL.Image')
    pytest.importorskip('transformers')
    from PIL import Image
    import torch.nn.functional as F
    from transformers.models.clip.image_processing_pil_clip import CLIPImageProcessorPil
    from gpt4roi_b200.engine import EngineConfig, PrefillEngine, random_state_dicts
    from tests.test_engine_gpu import make_inputs
    cfg = EngineConfig(image_size=224, vit_layers=12, n_layers=2, dtype='fp16')
    sd, vit_sd = random_state_dicts(cfg, DEV, seed=5, dtype=torch.float32)
    eng = PrefillEngine(cfg, sd, vit_sd, DEV)
    ids, _, _ = make_inputs(cfg, 2, [2, 1], 20, seed=4)
    srcs = [_image(480, 640, 1), _image(1080, 1920, 2)]
    pix_boxes = [np.array([[30.0, 40, 300, 420], [100, 10, 630, 200]]), np.array([[500.0, 300, 1700, 1000]])]
    proc = CLIPImageProcessorPil()
    th = torch.get_num_threads()
    torch.set_num_threads(max(2, th))
    try:
        ref = []
        for im in srcs:
            pv = proc.preprocess(Image.fromarray(im), do_center_crop=False, return_tensors='pt')['pixel_values'][0]
            ref.append(F.interpolate(pv.unsqueeze(0), size=(224, 224), mode='bilinear', align_corners=False)[0])
    finally:
        torch.set_num_threads(th)
    ref_images = torch.stack(ref).half()
    ref_boxes = [torch.tensor(b / np.array([w, h, w, h])[None], dtype=torch.float32)
                 for b, (h, w) in zip(pix_boxes, [s.shape[:2] for s in srcs])]
    images, boxes = ClipPreprocessor(device=DEV, out_dtype=torch.float16)(srcs, pix_boxes)
    if torch.backends.cpu.get_cpu_capability() in ('AVX2', 'AVX512'):
        assert torch.equal(images.cpu().view(torch.int16), ref_images.view(torch.int16))
    assert all(torch.equal(a, b) for a, b in zip(boxes, ref_boxes))
    out_k = eng.generate(ids, images, boxes, max_new_tokens=6)
    out_r = eng.generate(ids, ref_images.to(DEV), ref_boxes, max_new_tokens=6)
    assert torch.equal(out_k.cpu(), out_r.cpu())

