"""GPU tests of several sampled answers per prompt (generate(do_sample=True, num_return_sequences=N)): the shared-prefix
decode attention (decode.cu, g4r_decode_attention_group_*) against an fp64 reference and against the beam kernel given
the equivalent static ancestry table, and the engine loop against the current loop run on the explicitly expanded batch
(input_ids.repeat_interleave(N, 0), the same seed), per-row stopping, graphed against eager, one prefill per prompt
and the model seam on both loops."""
import numpy as np
import pytest
import torch

from gpt4roi_b200 import kernels, lib
from gpt4roi_b200.engine import EngineConfig, PrefillEngine, StopStrings, random_state_dicts
from tests.test_engine_gpu import make_inputs
from tests.test_sampling_gpu import _predict_row

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
TOL = {torch.bfloat16: 8e-3, torch.float16: 2e-3}     # test_beam_gpu.py's tolerances for the beam kernel


# ---------------------------------------------------------------------------------------------- attention
def _group_ref(q, kc, vc, B, N, plens, pos, H, D, scale):
    R = B * N
    out = torch.empty(R, H * D, dtype=torch.float64, device=q.device)
    for r in range(R):
        b = r // N
        P, n = int(plens[b]), int(pos[r]) + 1
        k = torch.cat([kc[b, :P], kc[B + r, P:n]]).double().view(-1, H, D)
        v = torch.cat([vc[b, :P], vc[B + r, P:n]]).double().view(-1, H, D)
        s = torch.einsum('hd,nhd->hn', q[r, :H * D].double().view(H, D), k) * scale
        out[r] = torch.einsum('hn,nhd->hd', torch.softmax(s, -1), v).reshape(-1)
    return out


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16], ids=['bf16', 'fp16'])
@pytest.mark.parametrize('B', [1, 3])
@pytest.mark.parametrize('N', [1, 2, 4, 8, 16])
def test_group_attention_vs_fp64_and_beam_kernel(dtype, B, N):
    """Equal and ragged prompt lengths (a 5-key prompt is shorter than one split slice, so some CTAs own no prompt key),
    0, 1 and many generated keys per row, D = 128: within the beam kernel's tolerance of an fp64 reference and of
    g4r_decode_attention_beam with the static table (prompt row below the prompt's length, the row's own row above);
    two runs bitwise equal."""
    H, D, L, G = 32, 128, 300, 40
    R, Lmax = B * N, L + G
    g = torch.Generator(device=DEV).manual_seed(10 * N + B)
    kc = torch.randn(B + R, Lmax, H * D, generator=g, device=DEV).to(dtype)
    vc = torch.randn(B + R, Lmax, H * D, generator=g, device=DEV).to(dtype)
    q = torch.randn(R, 3 * H * D, generator=g, device=DEV).to(dtype)
    scale = D ** -0.5
    samp = torch.arange(R, device=DEV) // N
    for ragged in (False, True):
        plens = torch.tensor([5, L, 137][:B] if ragged else [L] * B, dtype=torch.int32, device=DEV)
        own = torch.randint(2, G, (R,), generator=g, device=DEV)
        own = torch.where(torch.arange(R, device=DEV) % 3 == 0, 0, torch.where(torch.arange(R, device=DEV) % 3 == 1, 1, own))
        pos = (plens[samp] - 1 + own).to(torch.int32)
        got = kernels.decode_attention_group(q, kc, vc, B, N, H, D, L, G, scale, plens, pos)
        assert torch.equal(got, kernels.decode_attention_group(q, kc, vc, B, N, H, D, L, G, scale, plens, pos))
        err = _rel(got, _group_ref(q, kc, vc, B, N, plens, pos, H, D, scale))
        assert err < TOL[dtype], (ragged, err)
        col = torch.arange(Lmax, device=DEV)[None]
        anc = torch.where(col < plens[samp][:, None], samp[:, None], B + torch.arange(R, device=DEV)[:, None])
        beam = kernels.decode_attention_beam(q, kc, vc, R, H, D, Lmax, scale, pos, anc.to(torch.int32).contiguous())
        assert _rel(got, beam) < TOL[dtype], ragged


def test_group_attention_refuses_unsupported_shapes():
    H, D = 32, 128
    kc = torch.zeros(1 + 17, 64, H * D, dtype=torch.bfloat16, device=DEV)
    q = torch.zeros(17, 3 * H * D, dtype=torch.bfloat16, device=DEV)
    pl = torch.full((1,), 8, dtype=torch.int32, device=DEV)
    pos = torch.full((17,), 8, dtype=torch.int32, device=DEV)
    with pytest.raises(ValueError, match='1..16'):
        kernels.decode_attention_group(q, kc, kc, 1, 17, H, D, 32, 8, 1.0, pl, pos)
    out = torch.empty(17, H * D, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(lib.G4RError, match='supports 1..16'):      # the C entry point refuses it too
        kernels._call('g4r_decode_attention_group_bf16', q.device, lib.ptr(q), q.stride(0), lib.ptr(kc), lib.ptr(kc),
                      lib.ptr(out), out.stride(0), 1, 17, H, D, 32, 8, lib.ptr(pl), lib.ptr(pos), 64, 1.0)
    with pytest.raises(lib.G4RError, match='head_dim'):
        kernels._call('g4r_decode_attention_group_bf16', q.device, lib.ptr(q), q.stride(0), lib.ptr(kc), lib.ptr(kc),
                      lib.ptr(out), out.stride(0), 1, 2, 2 * H, 64, 32, 8, lib.ptr(pl), lib.ptr(pos), 64, 1.0)


# ---------------------------------------------------------------------------------------------- loops
@pytest.fixture(scope='module', params=['bf16', 'fp16'])
def eng2(request):
    cfg = EngineConfig(image_size=224, vit_layers=24, n_layers=2, dtype=request.param)
    sd, vit_sd = random_state_dicts(cfg, DEV, seed=45)
    return cfg, PrefillEngine(cfg, sd, vit_sd, DEV)


def _ragged(cfg):
    """Two prompts, the second left-padded by 5."""
    ids, images, boxes = make_inputs(cfg, 2, [2, 1], 20, seed=5)
    short, _, short_boxes = make_inputs(cfg, 1, [1], 15, seed=6)
    ids[1] = torch.cat([torch.zeros(5, dtype=torch.long), short[0]])
    boxes[1] = short_boxes[0]
    mask = torch.ones(ids.shape, dtype=torch.long)
    mask[1, :5] = 0
    return ids.to(DEV), images.to(DEV, cfg.torch_dtype), [b.to(DEV) for b in boxes], mask.to(DEV)


def _traced(eng, ids, images, boxes, **kw):
    """eng.generate, eager, recording the prefill's last-position logits and every decode step's logits (fp32)."""
    prefill, steps = [], []

    def fwd(*a, **k):
        out = PrefillEngine.forward_device(eng, *a, **k)
        prefill.append(out[:, -1].float().clone())
        return out

    def dec(tok, cache, pos_dev=None):
        out = PrefillEngine.decode_step(eng, tok, cache, pos_dev)
        steps.append(out[:, 0].float().clone())
        return out
    eng.forward_device, eng.decode_step = fwd, dec
    try:
        out = eng.generate(ids, images, boxes, use_graph=False, **kw)
    finally:
        del eng.forward_device, eng.decode_step
    return out.cpu(), prefill, steps


def _explained(xs, toks, u):
    """Each run's token is the one the numpy Philox + float64 inverse CDF of tests/test_sampling_gpu.py gives for its
    own logits (T 0.7, top-k 50) with the row's uniform u, or u lies within 1e-5 of a boundary there."""
    for x, t in zip(xs, toks):
        x = x.double().cpu().numpy()
        want, amb, _ = _predict_row(x, np.lexsort((np.arange(len(x)), -x)), 0.7, 50, 1.0, u)
        if not (amb or want == t):
            return False
    return True


def test_engine_loop_equals_the_expanded_batch(eng2):
    """N in {2, 4}, ragged left-padded prompts: the grouped loop against the current loop on repeat_interleave(N)
    inputs with the same seed.  The prefill logits and every decode step's logits of the rows whose inputs agree are
    within the attention tolerance.  Tokens are equal except at near-ties: where a row's tokens first differ, each
    run's token must be the one its own logits give with that draw's uniform (the logits' last-bit differences moved a
    CDF boundary across it); such draws are counted and are at most one in ten of the draws compared."""
    from gpt4roi_b200.engine import sampling_seed
    from tests.test_sampling_cpu import uniforms
    cfg, eng = eng2
    ids, images, boxes, mask = _ragged(cfg)
    B, L = ids.shape
    tol = TOL[cfg.torch_dtype]
    draws = diverged = 0
    for N in (2, 4):
        kw = dict(max_new_tokens=8, do_sample=True, temperature=0.7, top_k=50)
        got, gp, gs = _traced(eng, ids, images, boxes, num_return_sequences=N, attention_mask=mask,
                              generator=torch.Generator().manual_seed(N), **kw)
        want, wp, ws = _traced(eng, ids.repeat_interleave(N, 0), images.repeat_interleave(N, 0),
                               [b for b in boxes for _ in range(N)], attention_mask=mask.repeat_interleave(N, 0),
                               generator=torch.Generator().manual_seed(N), **kw)
        assert got.shape == want.shape == (B * N, L + 8)
        assert torch.equal(got[:, :L], want[:, :L])
        assert len(gp) == 1 and gp[0].shape[0] == B
        assert _rel(gp[0].repeat_interleave(N, 0), wp[0]) < tol
        same = torch.ones(B * N, dtype=torch.bool)
        for s in range(len(gs)):
            same &= got[:, L + s] == want[:, L + s]      # the token this step consumed
            if same.any():
                assert _rel(gs[s][same.to(DEV)], ws[s][same.to(DEV)]) < tol, (N, s)
        seed = sampling_seed(torch.Generator().manual_seed(N))
        for r in range(B * N):
            d = (got[r, L:] != want[r, L:]).nonzero()
            if len(d) == 0:
                draws += got.shape[1] - L
                continue
            c = int(d[0])                               # token c: Philox step c, from the prefill (c = 0) or step c - 1
            xs = (gp[0][r // N], wp[0][r]) if c == 0 else (gs[c - 1][r], ws[c - 1][r])
            assert _explained(xs, (int(got[r, L + c]), int(want[r, L + c])), uniforms(seed, c, B * N)[r]), (N, r, c)
            draws += c + 1
            diverged += 1
    print('%s: %d of %d draws compared took the other side of a moved CDF boundary' % (cfg.dtype, diverged, draws))
    assert diverged <= draws // 10


def test_graphed_equals_eager_and_one_prefill(eng2):
    """The graphed loop is bitwise the eager one; the vision branch and the prefill run once, at batch B."""
    cfg, eng = eng2
    ids, images, boxes, mask = _ragged(cfg)
    kw = dict(max_new_tokens=10, do_sample=True, temperature=0.7, top_k=50, num_return_sequences=4, attention_mask=mask)
    calls = []
    orig = eng.forward_device

    def counting(input_ids, *a, **k):
        calls.append(tuple(input_ids.shape))
        return orig(input_ids, *a, **k)
    eng.forward_device = counting
    try:
        graphed = eng.generate(ids, images, boxes, generator=torch.Generator().manual_seed(7), **kw).cpu()
    finally:
        del eng.forward_device
    assert calls == [tuple(ids.shape)]
    eager = eng.generate(ids, images, boxes, generator=torch.Generator().manual_seed(7), use_graph=False, **kw).cpu()
    assert torch.equal(graphed, eager)
    again = eng.generate(ids, images, boxes, generator=torch.Generator().manual_seed(7), **kw).cpu()
    assert torch.equal(graphed, again)
    assert graphed.shape == (8, ids.shape[1] + 10)
    assert not all(torch.equal(graphed[0], graphed[i]) for i in (1, 2, 3))          # the samples differ


def _first_hits(new, hit):
    """new [R, n] tokens, hit(token) -> bool: each row's first step that finishes it (n when none)."""
    n = new.shape[1]
    return [next((s for s in range(n) if hit(int(t[s]))), n) for t in new]


def test_rows_of_one_prompt_stop_on_their_own(eng2):
    """eos -> pad and stop strings with N = 4: rows of one prompt stop at different steps, finished rows get pad, the
    loop ends when the last one stops -- the free run cut by the host rule; graphed and eager alike."""
    cfg, eng = eng2
    ids, images, boxes, mask = _ragged(cfg)
    L = ids.shape[1]
    kw = dict(max_new_tokens=10, do_sample=True, temperature=1.0, top_k=3, num_return_sequences=4, attention_mask=mask)
    free = eng.generate(ids, images, boxes, generator=torch.Generator().manual_seed(4), **kw).cpu()[:, L:]
    pad = 0

    def cut(first):
        want = free.clone()
        for r, f in enumerate(first):
            want[r, f + 1:] = pad
        return want[:, :min(max(first) + 1, free.shape[1])]

    # eos: the token whose first occurrences spread over the most steps
    eos = max(free.unique().tolist(), key=lambda t: len(set(_first_hits(free, lambda x: x == t)) - {free.shape[1]}))
    first = _first_hits(free, lambda x: x == eos)
    assert len(set(first)) > 1
    # stop strings: every token is one letter (id % 26); the letter whose first occurrences spread the most
    strings = [chr(97 + i % 26) for i in range(32000)]
    letter = max('abcdefghijklmnopqrstuvwxyz',
                 key=lambda c: len(set(_first_hits(free, lambda x: x < 32000 and strings[x] == c))))
    sfirst = _first_hits(free, lambda x: x < 32000 and strings[x] == letter)
    stops = StopStrings(strings, [letter])
    never = 32005                      # an eos id the run does not produce: the pad rule is in force
    assert not bool((free == never).any())
    for graph in (True, False):
        got = eng.generate(ids, images, boxes, generator=torch.Generator().manual_seed(4), eos_token_id=eos,
                           pad_token_id=pad, use_graph=graph, **kw).cpu()[:, L:]
        assert torch.equal(got, cut(first)), (graph, eos)
        got = eng.generate(ids, images, boxes, generator=torch.Generator().manual_seed(4), eos_token_id=never,
                           pad_token_id=pad, stop_strings=stops, use_graph=graph, **kw).cpu()[:, L:]
        assert torch.equal(got, cut(sfirst)), (graph, letter)


def test_seam_on_both_loops():
    """model.generate(do_sample=True, num_return_sequences=N) returns [B*N, L+n] equal to the engine call; the HF loop
    (use_hf_loop=True) returns the same shape with each row starting with its prompt."""
    from tests.test_model_seam_gpu import build_seam_model
    cfg = EngineConfig(image_size=224, vit_layers=24, n_layers=2)
    sd, vit_sd = random_state_dicts(cfg, DEV, seed=37)
    model = build_seam_model(cfg, sd, vit_sd).eval()
    ids, images, boxes, mask = _ragged(cfg)
    img = images.float()
    B, L = ids.shape
    eng = model._get_engine(torch.device(DEV))
    with torch.inference_mode():
        for N in (2, 3):
            kw = dict(bboxes=boxes, attention_mask=mask, max_new_tokens=6, pad_token_id=0)
            ours = model.generate(ids, images=img, do_sample=True, temperature=0.7, num_return_sequences=N,
                                  generator=torch.Generator().manual_seed(N), **kw).cpu()
            direct = eng.generate(ids, img, boxes, max_new_tokens=6, do_sample=True, temperature=0.7, top_k=50,
                                  num_return_sequences=N, attention_mask=mask, pad_token_id=0,
                                  generator=torch.Generator().manual_seed(N)).cpu()
            assert ours.shape == (B * N, L + 6) and torch.equal(ours, direct)
            hf = model.generate(ids, images=img, do_sample=True, temperature=0.7, num_return_sequences=N,
                                use_hf_loop=True, **kw).cpu()
            assert hf.shape == ours.shape and torch.equal(hf[:, :L], ids.cpu().repeat_interleave(N, 0))
