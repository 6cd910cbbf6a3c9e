"""Shared test helpers: golden loaders and synthetic inputs (SURVEY.md 8(d))."""
import json
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def load_kat():
    with open(os.path.join(GOLDEN, 'mmcv_roi_align_kat.json')) as f:
        return json.load(f)


REF_CASES_SEED = 20260923


def load_ref_cases():
    """The reference RoIAlign cases of make_golden.py: its outputs, argmaxes and input gradients are stored
    (roi_align_ref_cases*.npz); the inputs and output gradients are replayed from the same seeded generator, in the
    order make_golden.py drew them."""
    z = {}
    for fn in ('roi_align_ref_cases.npz', 'roi_align_ref_cases_grad.npz'):
        with np.load(os.path.join(GOLDEN, fn)) as f:
            z.update({k: f[k] for k in f.files})
    meta = json.loads(bytes(z['meta']).decode())
    rng = np.random.default_rng(REF_CASES_SEED)
    for m in meta:
        n = m['name']
        z[n + '.input'] = rng.standard_normal((m['N'], m['C'], m['H'], m['W'])).astype(np.float32)
        rng.uniform(0, 1, (12, 2, 2))            # the 12 random boxes (stored in .rois)
        rng.integers(0, m['N'], (m['K'], 1))     # their image indices (stored in .rois)
        z[n + '.grad_output'] = rng.standard_normal((m['K'], m['C'], m['PH'], m['PW'])).astype(np.float32)
    return z, meta


def random_boxes(rng, k, size, min_wh=2.0):
    """k xyxy boxes in pixel units of a size x size image; x1<x2, y1<y2, >= min_wh wide/high."""
    p = np.sort(rng.uniform(0, 1, (k, 2, 2)), axis=1)
    b = np.concatenate([p[:, 0, :], p[:, 1, :]], 1) * size
    b[:, 2] = np.maximum(b[:, 2], b[:, 0] + min_wh)
    b[:, 3] = np.maximum(b[:, 3], b[:, 1] + min_wh)
    return np.minimum(b, size).astype(np.float32)


def adversarial_boxes(S):
    e = 1.0
    return np.array([
        [0, 0, S, S], [10.5, 20.25, 10.5, 20.25], [5, 5, 5, 60], [-e, -e, S + e, S + e],
        [S - 0.4, S - 0.4, S, S], [0, 0, 0.3, 0.3], [S * 0.5, -e, S + e, S * 0.5],
        [3.999, 7.001, 100.5, 50.499], [S, S, S, S], [0, 0, 2, 2],
        [S * 0.25, S * 0.25, S * 0.25 + 1e-3, S * 0.75],
    ], dtype=np.float32)


def make_rois(rng, n_img, k_per_img, size, adversarial=False):
    rows = []
    for i in range(n_img):
        b = random_boxes(rng, k_per_img, size)
        if adversarial:
            b = np.concatenate([b, adversarial_boxes(size)], 0)
        rows.append(np.concatenate([np.full((len(b), 1), i, np.float32), b], 1))
    return np.concatenate(rows, 0).astype(np.float32)


PYRAMID = {224: (128, 64, 32, 16), 336: (192, 96, 48, 24)}
STRIDES = (14 / 8, 14 / 4, 14 / 2, 14)
SCALES = tuple(float(np.float32(1.0 / s)) for s in STRIDES)


def golden_stream_mismatch():
    """The golden fixtures hold the reference's OUTPUTS; their inputs and weights (hundreds of MB) are regenerated
    from seeded CPU generators and verified by checksum.  A different RNG stream (another torch build) would make
    every pin to the reference disappear silently if the tests merely skipped -- so this FAILS unless
    G4R_ALLOW_GOLDEN_SKIP=1 is set (then it skips, loudly)."""
    import pytest
    import torch
    msg = ('seeded CPU RNG stream differs from the one the golden fixtures were generated with (torch %s); regenerate them '
           'with tests/golden/make_golden.py where the reference tree is available' % torch.__version__)
    if os.environ.get('G4R_ALLOW_GOLDEN_SKIP') == '1':
        pytest.skip(msg)
    pytest.fail(msg)
