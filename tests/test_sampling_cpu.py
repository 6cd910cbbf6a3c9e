"""CPU tests of the device sampler's specification (csrc/sample.cu, include/gpt4roi_b200.h: g4r_sample_tokens_bf16):
a numpy Philox4x32-10 that reproduces the Random123 known-answer vectors, a float64 restatement of the kept set that
equals transformers' own TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper, and the model seam's
resolution of the sampling parameters.  tests/test_sampling_gpu.py predicts the kernel's draws with these
restatements."""
import numpy as np
import pytest
import torch

from tests.test_model_seam_cpu import _tiny_model

V = 32006
_MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """Philox4x32-10 (Salmon et al., SC'11): ctr uint32 [..., 4], key uint32 [..., 2] -> uint32 [..., 4]."""
    ctr, key = np.asarray(ctr, np.uint64), np.asarray(key, np.uint64)
    c = [ctr[..., i] for i in range(4)]
    k0, k1 = key[..., 0], key[..., 1]
    for r in range(10):
        if r:
            k0 = (k0 + np.uint64(0x9E3779B9)) & _MASK
            k1 = (k1 + np.uint64(0xBB67AE85)) & _MASK
        p0 = np.uint64(0xD2511F53) * c[0]
        p1 = np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & _MASK, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & _MASK]
    return np.stack(c, -1).astype(np.uint32)


def uniforms(seed, step, rows):
    """The kernel's uniform for each of `rows` rows at Philox counter (step, row, 0), key seed: (word0 >> 8) * 2^-24."""
    rows = np.arange(rows, dtype=np.uint64)
    ctr = np.stack([np.full_like(rows, step & 0xFFFFFFFF), np.full_like(rows, step >> 32), rows,
                    np.zeros_like(rows)], -1)
    key = np.broadcast_to(np.array([seed & 0xFFFFFFFF, seed >> 32], np.uint64), (len(rows), 2))
    return (philox4x32_10(ctr, key)[:, 0] >> 8).astype(np.float64) * 2.0 ** -24


def kept_set(x, T, top_k, top_p, tol=1e-5):
    """float64 restatement of the kept set of one row x (the 16-bit values, as float64): s = x / T; top-k keeps
    s >= the k-th largest s (0 < top_k < V); top-p (top_p < 1) keeps each value whose strictly larger survivors hold
    less than top_p of the survivors' softmax mass (a group of equal values is kept or dropped whole).
    Returns (keep, p, near): keep bool [V]; p the float64 probabilities over the kept set; near: the row has a value
    whose larger-mass share lies within `tol` of top_p (float32 arithmetic may decide it either way)."""
    s = x / T
    n = len(s)
    keep = np.ones(n, bool)
    if 0 < top_k < n:
        keep = s >= np.sort(s)[::-1][top_k - 1]
    near = False
    if top_p < 1:
        e = np.where(keep, np.exp(s - s[keep].max()), 0.0)
        larger = _larger_mass(s, e)
        z = e.sum()
        near = bool(np.any(keep & (np.abs(larger / z - top_p) < tol)))
        top = s == s[keep].max()
        keep = keep & ((larger < top_p * z) | top)
    e = np.where(keep, np.exp(s - s[keep].max()), 0.0)
    return keep, e / e.sum(), near


def _larger_mass(s, e):
    """For every token: the total of e over the tokens with a strictly larger s."""
    vals, inv = np.unique(-s, return_inverse=True)         # groups of equal s, largest first
    gm = np.bincount(inv, weights=e, minlength=len(vals))
    return (np.cumsum(gm) - gm)[inv]


def hf_kept(x, T, top_k, top_p):
    """transformers' own processors on the fp32-widened row (GenerationMixin._sample: scores.float())."""
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper
    s = torch.tensor(x, dtype=torch.float32)[None]
    ids = torch.zeros((1, 1), dtype=torch.long)
    if T != 1.0:
        s = TemperatureLogitsWarper(T)(ids, s)
    if top_k:
        s = TopKLogitsWarper(top_k)(ids, s)
    if top_p < 1.0:
        s = TopPLogitsWarper(top_p)(ids, s)
    return torch.isfinite(s[0]).numpy()


def random_rows(dtype, n, seed):
    g = torch.Generator().manual_seed(seed)
    scale = torch.tensor([0.5, 2.0, 4.0])[torch.arange(n) % 3][:, None]
    return (torch.randn(n, V, generator=g) * scale).to(dtype).double().numpy()


def test_philox_matches_random123_known_answers():
    z = philox4x32_10(np.zeros((1, 4), np.uint32), np.zeros((1, 2), np.uint32))[0]
    assert [int(w) for w in z] == [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]
    f = philox4x32_10(np.full((1, 4), 0xFFFFFFFF, np.uint32), np.full((1, 2), 0xFFFFFFFF, np.uint32))[0]
    assert [int(w) for w in f] == [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]
    u = uniforms(123, 7, 1000)
    assert u.min() >= 0 and u.max() < 1 and abs(u.mean() - 0.5) < 0.05


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16], ids=['bf16', 'fp16'])
def test_kept_set_restatement_equals_transformers(dtype):
    """Equal to HF's processors on every token, except: tokens of a row whose top-p boundary lies within 1e-5 of a
    cumulative mass (counted), and the boundary group of equal values that HF's sort splits (the kernel keeps it
    whole; counted, and HF's kept set is then a subset of ours)."""
    rows = random_rows(dtype, 3, seed=11)
    # a row with many equal values at every level (ties at the top-k / top-p boundaries)
    rows = np.concatenate([rows, np.round(rows[:1] * 2) / 2], 0)
    near_rows = split_groups = checked = 0
    for x in rows:
        for T in (0.2, 0.7, 1.0):
            for top_k in (0, 1, 50, V):
                for top_p in (1.0, 0.9, 0.5):
                    ours, _, near = kept_set(x, T, top_k, top_p)
                    hf = hf_kept(x, T, top_k, top_p)
                    checked += 1
                    if near:
                        near_rows += 1
                        continue
                    diff = ours != hf
                    if diff.any():
                        assert top_p < 1 and not (hf & ~ours).any(), (T, top_k, top_p)
                        assert len(np.unique(x[diff])) == 1 and (x[ours] >= x[diff][0]).all(), (T, top_k, top_p)
                        assert ((x == x[diff][0]) & hf).any(), 'only a group that HF split may differ'
                        split_groups += 1
    print('kept sets: %d cases, %d skipped (top-p boundary within 1e-5), %d boundary groups split by HF'
          % (checked, near_rows, split_groups))
    assert near_rows <= checked // 10


def test_seam_resolves_sampling_like_transformers():
    from transformers import GenerationConfig
    from gpt4roi_b200.spi_llava import resolve_generate
    from tests.test_serve_cpu import _seam, _StubEngine
    m = _seam(_StubEngine())

    def rule(**kw):
        return resolve_generate(m, 5, kw.pop('max_new_tokens', None), **kw)[:4]
    # gpt4roi/app.py:293-300: do_sample=True, temperature=0.2 and no top_k -> HF's global default top_k=50
    assert rule(do_sample=True, temperature=0.2, max_new_tokens=1024) == (True, 0.2, 50, 1.0)
    assert rule(do_sample=True, temperature=0.2, top_k=0, top_p=0.9) == (True, 0.2, 0, 0.9)
    gc = GenerationConfig(do_sample=True, temperature=0.7, top_k=20, top_p=0.8)
    assert rule(generation_config=gc) == (True, 0.7, 20, 0.8)
    assert rule(generation_config=gc, top_k=5) == (True, 0.7, 5, 0.8)     # explicit kwargs first
    m.generation_config.top_p = 0.95                                        # then the model's config
    assert rule(do_sample=True) == (True, 1.0, 50, 0.95)
    assert rule(generation_config=gc) == (True, 0.7, 20, 0.8)
    assert rule(do_sample=False, temperature=0.2, top_k=3) == (False, 1.0, 0, 1.0)
    assert rule() == (False, 1.0, 0, 1.0)
    # the batcher runs the three warpers only
    sb = m.continuous_batcher(slots=1, max_len=16)
    ids = torch.tensor([[1, 2, 3, 4, 5]])
    for bad in (dict(repetition_penalty=1.1), dict(min_p=0.1), dict(num_beams=2), dict(typical_p=0.5),
                dict(no_repeat_ngram_size=3)):
        with pytest.raises(NotImplementedError, match='use_hf_loop=True'):
            sb.submit(ids, max_new_tokens=2, do_sample=True, temperature=0.2, **bad)
    with pytest.raises(NotImplementedError, match='use_hf_loop=True'):
        sb.submit(ids, max_new_tokens=2, do_sample=False, repetition_penalty=1.1)
