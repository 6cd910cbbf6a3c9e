"""GPU tests of beam search: the ancestry-table decode attention (decode.cu, BEAM), the beam step kernels (beam.cu)
against the torch restatement of tests/test_beam_cpu.py, and the engine loop against transformers' own beam search run
over the model seam (use_hf_loop=True)."""
import pytest
import torch

from gpt4roi_b200 import kernels
from gpt4roi_b200.engine import BeamCache, EngineConfig, PrefillEngine, random_state_dicts
from tests.test_beam_cpu import ref_accumulate, ref_select
from tests.test_engine_gpu import make_inputs

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
V = 32006


@pytest.fixture(scope='module')
def eng2():
    cfg = EngineConfig(image_size=224, vit_layers=24, n_layers=2)
    sd, vit_sd = random_state_dicts(cfg, DEV, seed=43)
    return cfg, PrefillEngine(cfg, sd, vit_sd, DEV), sd, vit_sd


# ---------------------------------------------------------------------------------------------- attention
def _attn_ref(q, kc, vc, anc, pos, H, D, scale):
    R = q.shape[0]
    out = torch.empty(R, H * D, dtype=torch.float32, device=q.device)
    for r in range(R):
        n = int(pos[r]) + 1
        rows = anc[r, :n].long()
        k = kc[rows, torch.arange(n, device=q.device)].float().view(n, H, D)
        v = vc[rows, torch.arange(n, device=q.device)].float().view(n, H, D)
        s = torch.einsum('hd,nhd->hn', q[r, :H * D].float().view(H, D), k) * scale
        out[r] = torch.einsum('hn,nhd->hd', torch.softmax(s, -1), v).reshape(-1)
    return out


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16], ids=['bf16', 'fp16'])
@pytest.mark.parametrize('R', [2, 8, 16, 32])
def test_beam_attention_vs_fp32_and_identity(dtype, R):
    """Random ancestry tables mixing prompt rows and beam rows over ragged lengths: the kernel against an fp32
    reference; with an identity table it is bitwise g4r_decode_attention_rows."""
    H, D, Lmax = 32, 128, 300
    B = max(1, R // 4)
    g = torch.Generator(device=DEV).manual_seed(R)
    kc = torch.randn(B + R, Lmax, H * D, generator=g, device=DEV).to(dtype)
    vc = torch.randn(B + R, Lmax, H * D, generator=g, device=DEV).to(dtype)
    q = torch.randn(R, 3 * H * D, generator=g, device=DEV).to(dtype)
    lens = torch.randint(20, 200, (B,), generator=g, device=DEV)
    gen = 60
    samp = torch.arange(R, device=DEV) * B // R
    pos = (lens[samp] + torch.randint(0, gen, (R,), generator=g, device=DEV)).to(torch.int32)
    col = torch.arange(Lmax, device=DEV)[None]
    beam_rows = B + samp[:, None] * 0 + torch.randint(0, R, (R, Lmax), generator=g, device=DEV)
    anc = torch.where(col < lens[samp][:, None], samp[:, None].expand(R, Lmax), beam_rows).to(torch.int32).contiguous()
    scale = D ** -0.5
    got = kernels.decode_attention_beam(q, kc, vc, R, H, D, Lmax, scale, pos, anc)
    want = _attn_ref(q, kc, vc, anc, pos, H, D, scale)
    err = ((got.float() - want).norm() / want.norm()).item()
    assert err < (8e-3 if dtype == torch.bfloat16 else 2e-3), err
    # identity table over the beam rows only: rows kernel on the [B:] view
    ident = (B + torch.arange(R, device=DEV, dtype=torch.int32))[:, None].expand(R, Lmax).contiguous()
    a = kernels.decode_attention_beam(q, kc, vc, R, H, D, Lmax, scale, pos, ident)
    b = kernels.decode_attention(q, kc[B:], vc[B:], R, H, D, Lmax, scale, pos_rows=pos)
    assert torch.equal(a, b)


# ---------------------------------------------------------------------------------------------- beam step
@pytest.fixture(scope='module')
def pool(eng2):
    """Real lm_head rows of the 2-layer config (text-only prefill), spread to a trained model's range."""
    cfg, eng = eng2[:2]
    ids = torch.randint(3, 32000, (4, 16), generator=torch.Generator().manual_seed(6))
    real = eng.forward(ids.to(DEV), None, None).reshape(64, V).float()
    return real * (4.0 / real.std())


def _host_state(c):
    g = int(c.state[0])
    return dict(run_score=c.run_score.cpu().clone(), fin_score=c.fin_score.cpu().clone(),
                fin_state=c.fin_state.cpu().clone(), state=c.state.cpu().clone(), run_seq=c.run_seq[g & 1].cpu().clone(),
                fin_seq=c.fin_seq[g & 1].cpu().clone(), ids=c.ids.view(-1).cpu().clone(), pos_rows=c.pos_rows.cpu().clone(),
                anc=c.anc.cpu().clone())


def _near_tie(acc64, N, K, tol=1e-5):
    """A sample whose top K + 1 candidate scores hold two different values within tol (float64): the kernel's fp32 sum
    order may rank them differently from the restatement."""
    R = acc64.shape[0]
    for b in range(R // N):
        top = acc64[b * N:(b + 1) * N].reshape(-1).topk(K + 1).values
        d = (top[:-1] - top[1:]).abs()
        if bool(((d > 0) & (d < tol)).any()):
            return True
    return False


def _step_logits(pool, R, step, adversarial, eos, g):
    rows = pool[torch.randint(0, pool.shape[0], (R,), generator=g)].clone()
    if adversarial:
        rows[0] = rows[1 % R]                                   # equal rows: exact ties across beams
        rows[:, 100:140] = rows.max(-1, keepdim=True).values    # exact ties within a row, at the top
        rows[:, eos[0]] = rows.max(-1).values + 0.5             # eos in the top
        rows[:, 2000:7000:3] = float('-inf')
    return rows


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16], ids=['bf16', 'fp16'])
def test_beam_step_vs_restatement(pool, dtype):
    """N in {2, 4, 8}, B in {1, 3}, real and adversarial rows, every early_stopping mode: parents, tokens, flags,
    sequences and the ancestry table identical to the restatement, scores within 1e-6 (relative, or absolute near
    0); steps whose top candidates hold two different float64 scores within 1e-5 are counted and skipped; two runs are
    bitwise equal."""
    cfg0 = EngineConfig(n_layers=0, vit_layers=0)
    checked = skipped = 0
    for N in (2, 4, 8):
        for B in (1, 3):
            for adv, early, lp in ((False, False, 1.0), (True, True, 2.0), (True, 'never', -0.5)):
                eos = [7]
                L, G = 9, 6
                runs = []
                for rep in range(2):
                    g = torch.Generator().manual_seed(100 * N + 10 * B + adv)
                    c = BeamCache(cfg0, B, N, L, G, DEV, eos, lp, early, fill=0)
                    lens = torch.tensor([L - (b % 3) for b in range(B)], dtype=torch.int32, device=DEV)
                    c.start(lens)
                    trace = []
                    for step in range(G):
                        first = step == 0
                        rows = _step_logits(pool, B if first else B * N, step, adv, eos, g).to(dtype)
                        before = _host_state(c)
                        c.step(rows, first=first)
                        trace.append(_host_state(c))
                        if rep:
                            continue
                        acc = ref_accumulate(rows.cpu(), N if first else 1, before['run_score'])
                        acc64 = rows.cpu().double().repeat_interleave(N if first else 1, 0)
                        acc64 = before['run_score'].double()[:, None] + torch.log_softmax(acc64, -1)
                        if _near_tie(acc64, N, c.K):
                            skipped += 1
                            break
                        want = ref_select(acc, before, N, eos, L, L + G, lp, early, lens=lens.cpu())
                        got = trace[-1]
                        for k in ('fin_state', 'state', 'run_seq', 'fin_seq', 'ids', 'pos_rows', 'anc'):
                            assert torch.equal(got[k], want[k]), (N, B, adv, step, k)
                        for k in ('run_score', 'fin_score'):
                            # atol: the fp32 rounding of log sum exp over 32k terms, for scores near 0
                            assert torch.allclose(got[k], want[k], rtol=1e-6, atol=1e-6), (N, B, adv, step, k)
                        checked += 1
                        if int(got['state'][4 * B + 1]):
                            break
                    runs.append(trace)
                for a, b in zip(*runs):
                    for k in a:
                        assert torch.equal(a[k], b[k]), k
    print('%s: %d steps equal to the restatement, %d skipped at a near tie' % (dtype, checked, skipped))
    assert skipped <= checked // 10


# ---------------------------------------------------------------------------------------------- loops
def _stable_topk(orig):
    def topk(x, k, dim=-1, largest=True, sorted=True, **kw):
        v, i = torch.sort(x, dim=dim, descending=largest, stable=True)
        return torch.return_types.topk((v.narrow(dim, 0, k), i.narrow(dim, 0, k)))
    return topk


def _hf_beams(model, **kw):
    """transformers' beam search over the seam, with torch.topk swapped for a stable sort (the kernels' tie rule)."""
    orig = torch.topk
    torch.topk = _stable_topk(orig)
    try:
        return model.generate(use_hf_loop=True, **kw)
    finally:
        torch.topk = orig


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16], ids=['bf16', 'fp16_demo'])
def test_engine_loop_equals_hf_loop(dtype):
    """2-layer config: N in {2, 4}, num_return_sequences in {1, N}, early_stopping True / False, an eos that fires,
    left-padded ragged prompts; token for token equal to HF's beam search over the seam; graphed = eager."""
    from tests.test_model_seam_gpu import build_seam_model
    cfg = EngineConfig(image_size=224, vit_layers=24, n_layers=2)
    sd, vit_sd = random_state_dicts(cfg, DEV, seed=37)
    model = build_seam_model(cfg, sd, vit_sd, dtype=dtype, app_style=dtype == torch.float16).eval()
    ids, images, boxes = make_inputs(cfg, 2, [2, 1], 20, seed=5)
    short, _, short_boxes = make_inputs(cfg, 1, [1], 15, seed=6)
    B, L = ids.shape
    ids[1] = torch.cat([torch.zeros(5, dtype=torch.long), short[0]])   # left-padded second prompt
    boxes[1] = short_boxes[0]
    mask = torch.ones(B, L, dtype=torch.long)
    mask[1, :5] = 0
    act = torch.float16 if dtype == torch.float16 else torch.bfloat16
    img = images.to(DEV, act if dtype == torch.float16 else torch.float32)
    bx = [b.to(DEV) for b in boxes]
    eng = model._get_engine(torch.device(DEV))
    # an eos that fires: the most frequent token of a free run
    free = eng.generate(ids.to(DEV), img, bx, max_new_tokens=8, num_beams=2, attention_mask=mask.to(DEV),
                        use_graph=False).cpu()
    eos = int(free[:, L + 1:].flatten().mode().values)
    n_diff = 0
    with torch.inference_mode():
        for N, nrs, early in ((2, 1, False), (2, 2, True), (4, 1, True), (4, 4, False)):
            kw = dict(input_ids=ids.to(DEV), images=img, bboxes=bx, attention_mask=mask.to(DEV), max_new_tokens=10,
                      num_beams=N, num_return_sequences=nrs, early_stopping=early, eos_token_id=eos, pad_token_id=0,
                      do_sample=False)
            hf = _hf_beams(model, **kw).cpu()
            ours = model.generate(**kw).cpu()
            kw2 = {k: v for k, v in kw.items() if k not in ('input_ids', 'images', 'bboxes', 'do_sample')}
            eager = eng.generate(ids.to(DEV), img, bx, use_graph=False, **kw2).cpu()
            assert torch.equal(ours, eager), (N, nrs, early)
            if not torch.equal(ours, hf):
                n_diff += 1
                print('engine vs HF differ (N=%d nrs=%d early=%s):\n%s\n%s' % (N, nrs, early, ours, hf))
            assert ours.shape[0] == B * nrs
    print('engine loop vs HF loop: %d of 4 cases differ' % n_diff)
    assert n_diff == 0


def test_prefill_runs_once_per_sample(eng2):
    """The engine loop runs the vision branch and the prefill once, at batch B, whatever N."""
    cfg, eng = eng2[:2]
    ids, images, boxes = make_inputs(cfg, 2, [1, 2], 16, seed=8)
    calls = []
    orig = eng.forward_device

    def counting(input_ids, *a, **k):
        calls.append(tuple(input_ids.shape))
        return orig(input_ids, *a, **k)
    eng.forward_device = counting
    try:
        out = eng.generate(ids.to(DEV), images.to(torch.bfloat16), boxes, max_new_tokens=6, num_beams=4,
                           num_return_sequences=2)
    finally:
        del eng.forward_device
    assert calls == [tuple(ids.shape)]
    assert out.shape[0] == 4 and torch.equal(out[::2, :ids.shape[1]].cpu(), ids)
