"""CPU tests of beam search: a torch restatement of one device beam step (csrc/beam.cu) against transformers' own
_beam_search helpers, the model seam's resolution and refusals, and the HF loop over the seam with num_beams
(G4RCache.reorder_cache, the expansion of per-sample box lists).  tests/test_beam_gpu.py checks the kernels against
the restatement."""
import pytest
import torch
from transformers.generation.utils import GenerationMixin

from tests.test_model_seam_cpu import _StubEngine, _tiny_model

NEG = -1.0e9


def new_state(B, N, prompt_len, G, fill=-1, Lmax=None):
    """The beam state of engine.BeamCache, on the host (G: generated columns; Lmax: ancestry table width)."""
    Lmax = prompt_len + G if Lmax is None else Lmax
    run = torch.zeros(B, N)
    run[:, 1:] = NEG
    anc = torch.arange(B, dtype=torch.int32).repeat_interleave(N)[:, None].expand(B * N, Lmax).contiguous()
    state = torch.zeros(4 * B + 2, dtype=torch.int32)
    state[1:4 * B:4] = 1
    return dict(run_score=run.reshape(B * N), fin_score=torch.full((B, N), NEG),
                fin_state=torch.zeros(B, N, 2, dtype=torch.int32), state=state,
                run_seq=torch.full((B, N, G), fill, dtype=torch.int64), fin_seq=torch.full((B, N, G), fill, dtype=torch.int64),
                ids=torch.zeros(B * N, dtype=torch.int64), pos_rows=torch.zeros(B * N, dtype=torch.int32), anc=anc)


def ref_accumulate(logits, row_div, run_score):
    """Kernel A's scores: running_score[r] + ((x - max) - log sum exp(x - max)), fp32, for every token of every beam
    row ([rows, V] 16-bit logits; row_div = N: each sample's single prefill row, shared by its beams)."""
    x = logits.float().repeat_interleave(row_div, 0)
    mx = x.max(-1, keepdim=True).values
    logz = torch.exp(x - mx).double().sum(-1, keepdim=True).float().log()
    return run_score[:, None] + ((x - mx) - logz)


def ref_select(acc, st, N, eos, prompt_len, max_length, length_penalty, early, lens=None):
    """Kernel B on accumulated scores acc [B*N, V] (fp32): the restated step of transformers' _beam_search with the
    tie rule (score descending, flat index beam * V + token ascending).  Returns a new state dict; early is True,
    False or 'never'."""
    R, V = acc.shape
    B = R // N
    K = max(2, 1 + len(eos)) * N
    st = {k: v.clone() for k, v in st.items()}
    Lmax = st['anc'].shape[1]
    lens = torch.full((B,), prompt_len, dtype=torch.int32) if lens is None else lens
    f32 = lambda v: torch.tensor(v, dtype=torch.float32)
    flags = []
    for b in range(B):
        g = int(st['state'][4 * b])
        flat = acc[b * N:(b + 1) * N].reshape(-1)
        order = torch.sort(flat, descending=True, stable=True).indices[:K]
        lp, par, tok = flat[order], order // V, order % V
        hit = torch.isin(tok, torch.tensor(eos, dtype=torch.long)) | (prompt_len + g + 1 >= max_length)
        rs = lp + torch.where(hit, f32(NEG), f32(-0.0))
        run_k = torch.sort(rs, descending=True, stable=True).indices[:N]
        unsat = bool(st['state'][4 * b + 1])
        full = bool(st['fin_state'][b, :, 0].all()) and early is True
        x = lp / f32((g + 1) ** length_penalty)
        x = x + (f32(NEG) if full else f32(-0.0))
        x = x + (f32(-0.0) if unsat else f32(NEG))
        did = hit & (torch.arange(K) < N)
        x = x + torch.where(did, f32(-0.0), f32(NEG))
        merged = torch.cat([st['fin_score'][b], x])
        sel = torch.sort(merged, descending=True, stable=True).indices[:N]
        # sequences
        run_old, fin_old = st['run_seq'][b].clone(), st['fin_seq'][b].clone()
        cand_seq = run_old[par]
        cand_seq[:, g] = tok
        st['run_seq'][b] = cand_seq[run_k]
        new_fin = torch.cat([fin_old, cand_seq])[sel]
        st['fin_seq'][b] = new_fin
        fin_flag = torch.cat([st['fin_state'][b, :, 0].bool(), did])[sel]
        fin_len = torch.cat([st['fin_state'][b, :, 1], torch.full((K,), g + 1, dtype=torch.int32)])[sel]
        st['fin_score'][b] = merged[sel]
        st['fin_state'][b, :, 0] = fin_flag.to(torch.int32)
        st['fin_state'][b, :, 1] = fin_len
        st['run_score'][b * N:(b + 1) * N] = rs[run_k]
        # ancestry, ids, positions
        lb = int(lens[b])
        old = st['anc'][b * N:(b + 1) * N, lb:lb + g].clone()
        for j in range(N):
            k = int(run_k[j])
            r = b * N + j
            st['anc'][r, lb:lb + g] = old[int(par[k])]
            st['anc'][r, lb + g] = B + r
            st['ids'][r] = tok[k]
            st['pos_rows'][r] = lb + g
        # early-stop heuristic at cur_len + 1
        best_len = max_length - prompt_len if (early == 'never' and length_penalty > 0) else g + 1
        best = rs[run_k[0]] / f32(best_len ** length_penalty)
        worst = torch.where(fin_flag, st['fin_score'][b].min(), f32(NEG))
        st['state'][4 * b] = g + 1
        st['state'][4 * b + 1] = int(unsat and bool((best > worst).any()))
        st['state'][4 * b + 2] = (1 if bool(fin_flag.all()) else 0) | (2 if bool(hit.all()) else 0)
        flags.append((bool(st['state'][4 * b + 1]), bool(fin_flag.all()), bool(hit.all())))
    any_unsat = any(f[0] for f in flags)
    all_fin = all(f[1] for f in flags)
    all_hit = all(f[2] for f in flags)
    st['state'][4 * B + 1] = int(not (any_unsat and not (all_fin and early is True) and not all_hit))
    return st


def hf_step(acc, hs, N, eos, cur_len, prompt_len, max_length, length_penalty, early):
    """One iteration of transformers' _beam_search (steps c-g) with its own helpers, on accumulated scores [B*N, V]."""
    h = GenerationMixin
    self = type('H', (GenerationMixin,), {})
    self = self.__new__(self)
    B, V = acc.shape[0] // N, acc.shape[1]
    K = max(2, 1 + len(eos)) * N
    mask = torch.cat([torch.ones(N, dtype=torch.bool), torch.zeros(K - N, dtype=torch.bool)])
    lp, seqs, bidx = self._get_top_k_continuations(acc.reshape(B, N * V), hs['running_sequences'],
                                                   hs['running_beam_indices'], cur_len, prompt_len, False, K, N, V, B)
    hit = torch.isin(seqs[:, :, cur_len], torch.tensor(eos, dtype=torch.long)) | (cur_len + 1 >= max_length)
    rseq, rscore, rbidx = self._get_running_beams_for_next_iteration(lp, seqs, bidx, hit, N)
    fseq, fscore, fbidx, fin = self._update_finished_beams(
        hs['sequences'], seqs, hs['beam_scores'], lp, hs['beam_indices'], bidx, hs['unsat'], hs['is_sent_finished'], hit,
        mask, N, cur_len, prompt_len, length_penalty, early)
    unsat = h._check_early_stop_heuristic(hs['unsat'], rscore, fscore, fin, cur_len + 1, max_length, prompt_len, early,
                                          length_penalty)
    more = h._beam_search_has_unfinished_sequences(unsat, fin, hit, early)
    return dict(running_sequences=rseq, running_beam_scores=rscore, running_beam_indices=rbidx, sequences=fseq,
                beam_scores=fscore, beam_indices=fbidx, is_sent_finished=fin, unsat=unsat), bool(more)


def hf_state(B, N, prompt, max_length, fill):
    L = prompt.shape[1]
    rs = torch.full((B, N, max_length), fill, dtype=torch.int64)
    rs[:, :, :L] = prompt[:, None]
    run = torch.zeros(B, N)
    run[:, 1:] = NEG
    bi = torch.full((B, N, max_length - L), -1, dtype=torch.int32)
    return dict(running_sequences=rs, running_beam_scores=run, running_beam_indices=bi, sequences=rs.clone(),
                beam_scores=torch.full((B, N), NEG), beam_indices=bi.clone(),
                is_sent_finished=torch.zeros(B, N, dtype=torch.bool), unsat=torch.ones(B, 1, dtype=torch.bool))


def hf_output(hs, N, nrs, prompt_len):
    """HF's "# 5. prepare outputs" crop."""
    seq = hs['sequences'][:, :nrs].reshape(-1, hs['sequences'].shape[-1])
    bi = hs['beam_indices'][:, :nrs].reshape(-1, hs['beam_indices'].shape[-1])
    n = int((bi + 1).bool().sum(1).max())
    return seq[:, :prompt_len + n]


def run_both(B, N, V, eos, length_penalty, early, steps, seed, nrs=1):
    """Drive HF's helpers and the restatement over the same tie-free random log-prob rows for up to `steps` steps
    (max_length = prompt + steps, so the last step is the max-length step); compare the states after every step."""
    g = torch.Generator().manual_seed(seed)
    L = 5
    prompt = torch.randint(0, V, (B, L), generator=g)
    max_length = L + steps
    fill = 0
    hs = hf_state(B, N, prompt, max_length, fill)
    st = new_state(B, N, L, steps, fill)
    for step in range(steps):
        # distinct log-probs; eos made likely so that beams finish
        logp = torch.log_softmax(torch.randn(B * N, V, generator=g) * 3, -1)
        for e in eos:
            logp[:, e] = logp.max(-1).values - torch.rand(B * N, generator=g) * 0.5
        logp = torch.log_softmax(logp, -1)
        acc_hf = (logp.reshape(B, N, V) + hs['running_beam_scores'][:, :, None]).reshape(B * N, V)
        acc = st['run_score'][:, None] + logp
        assert torch.equal(acc, acc_hf)
        hs, more = hf_step(acc_hf, hs, N, eos, L + step, L, max_length, length_penalty, early)
        st = ref_select(acc, st, N, eos, L, max_length, length_penalty, early)
        assert torch.equal(st['run_score'].view(B, N), hs['running_beam_scores'])
        live = hs['running_beam_scores'] > NEG / 2      # masked running beams tie at -1e9 (HF's topk order)
        assert torch.equal(st['run_seq'][live], hs['running_sequences'][:, :, L:][live])
        # a slot that holds no finished sequence keeps a -1e9 score; which of the equal -1e9 entries fills it is HF's
        # topk tie order, so only finished slots are compared entry by entry
        fin = hs['is_sent_finished']
        assert torch.equal(st['fin_state'][..., 0].bool(), fin)
        assert torch.equal(st['fin_score'], hs['beam_scores'])
        assert torch.equal(st['fin_seq'][fin], hs['sequences'][:, :, L:][fin])
        assert torch.equal(st['fin_state'][..., 1][fin], (hs['beam_indices'] + 1).bool().sum(-1).to(torch.int32)[fin])
        assert torch.equal(st['state'][1:4 * B:4].bool(), hs['unsat'][:, 0])
        assert bool(st['state'][4 * B + 1]) == (not more)
        if not more:
            break
    assert bool(hs['is_sent_finished'][:, :nrs].all())
    out = hf_output(hs, N, nrs, L)
    n = int(st['fin_state'][:, :nrs, 1].max())
    mine = torch.cat([prompt.repeat_interleave(nrs, 0), st['fin_seq'][:, :nrs].reshape(B * nrs, -1)[:, :n]], 1)
    assert torch.equal(mine, out)
    return step + 1


@pytest.mark.parametrize('early', [True, False, 'never'])
@pytest.mark.parametrize('length_penalty', [1.0, 0.0, -0.5, 2.0])
@pytest.mark.parametrize('eos', [[7], [7, 11]], ids=['eos1', 'eos2'])
def test_restatement_equals_transformers_helpers(early, length_penalty, eos):
    """Random tie-free steps, B = 2, N in {2, 3}: running / finished sequences, scores, flags, the early-stop state, the
    done flag and the final crop equal HF's; with 40 steps the search ends by eos, with 6 by the max-length step."""
    for N, steps, seed in ((2, 6, 1), (3, 40, 2), (3, 6, 3)):
        ran = run_both(2, N, 50, eos, length_penalty, early, steps, seed, nrs=N if seed == 2 else 1)
        assert ran <= steps


def test_max_length_step_finishes_every_top_beam():
    """One step before max_length: every candidate hits, the top N are finished and the search is done."""
    B, N, V, L = 1, 2, 30, 4
    st = new_state(B, N, L, 1)
    g = torch.Generator().manual_seed(0)
    acc = st['run_score'][:, None] + torch.log_softmax(torch.randn(B * N, V, generator=g), -1)
    out = ref_select(acc, st, N, [], L, L + 1, 1.0, False)
    assert out['fin_state'][0, :, 0].tolist() == [1, 1] and out['fin_state'][0, :, 1].tolist() == [1, 1]
    assert int(out['state'][4 * B + 1]) == 1
    top2 = torch.sort(acc[0], descending=True, stable=True).indices[:2]
    assert out['fin_seq'][0, :, 0].tolist() == top2.tolist()


def test_tie_rule_prefers_lower_flat_index():
    """Equal scores across and within beams: the lower beam * V + token wins, for the running and the finished picks."""
    B, N, V = 1, 2, 8
    st = new_state(B, N, 3, 4)
    st['run_score'][:] = 0.0
    acc = torch.full((2, V), -5.0)
    acc[1, 2] = acc[0, 6] = acc[0, 3] = -1.0
    out = ref_select(acc, st, N, [], 3, 7, 1.0, False)
    assert out['ids'].tolist() == [3, 6]          # flat 3 and 6 beat flat 8 + 2 = 10
    assert out['anc'][:, 3].tolist() == [1, 2]    # B + r


# ---------------------------------------------------------------------------------------------
# seam
# ---------------------------------------------------------------------------------------------
def test_resolve_beam_search_and_refusals():
    from transformers import GenerationConfig
    from gpt4roi_b200.spi_llava import resolve_generate
    from tests.test_serve_cpu import _seam, _StubEngine
    m = _seam(_StubEngine())
    m.generation_config.eos_token_id = 2
    assert resolve_generate(m, 10, 8).beam is None
    r = resolve_generate(m, 10, 8, num_beams=4).beam
    assert r == dict(num_beams=4, length_penalty=1.0, early_stopping=False, num_return_sequences=1, eos_token_id=[2],
                     pad_token_id=2, max_length=18)
    r = resolve_generate(m, 10, 8, num_beams=3, length_penalty=-0.5, early_stopping='never', num_return_sequences=3,
                         eos_token_id=[5, 6], pad_token_id=0).beam
    assert (r['length_penalty'], r['early_stopping'], r['num_return_sequences'], r['eos_token_id'], r['pad_token_id']) \
        == (-0.5, 'never', 3, [5, 6], 0)
    r = resolve_generate(m, 10, 8, generation_config=GenerationConfig(num_beams=2, early_stopping=True)).beam
    assert r['num_beams'] == 2 and r['early_stopping'] is True
    # the search does not depend on the output flags
    assert resolve_generate(m, 10, 8, num_beams=2, output_scores=True, return_dict_in_generate=True).beam == \
        resolve_generate(m, 10, 8, num_beams=2).beam
    with pytest.raises(ValueError):
        resolve_generate(m, 10, 8, num_beams=2, num_return_sequences=3)
    ids = torch.arange(1, 11)[None]
    m._get_engine = lambda device: pytest.fail('no engine should be built')
    for bad in (dict(do_sample=True), dict(repetition_penalty=1.3), dict(no_repeat_ngram_size=2)):
        with pytest.raises(NotImplementedError, match='use_hf_loop'):
            m.generate(ids, images=torch.zeros(1, 3, 28, 28), max_new_tokens=8, num_beams=2, **bad)
    # any processor, even a min_length at most the prompt's length
    with pytest.raises(NotImplementedError, match='MinLengthLogitsProcessor'):
        m.generate(ids, images=torch.zeros(1, 3, 28, 28), max_new_tokens=8, num_beams=2, min_length=5)
    m._get_engine = lambda device: _StubEngine()
    with pytest.raises(NotImplementedError, match='num_beams=2'):
        m.continuous_batcher(slots=1, max_len=32).submit(ids, max_new_tokens=2, num_beams=2)


def test_engine_loop_refusals():
    """stopping_criteria and past_key_values with beams are refused by the seam, do_sample / cache= by the engine."""
    from transformers import DynamicCache
    from gpt4roi_b200.engine import PrefillEngine
    m = _tiny_model()
    m._get_engine = lambda device: pytest.fail('no engine should be built')
    ids = torch.tensor([[1, 5, 9]])
    with pytest.raises(NotImplementedError, match='stopping_criteria'):
        m.generate(ids, images=torch.zeros(1, 3, 28, 28), num_beams=2, stopping_criteria=[lambda *a: False])
    with pytest.raises(NotImplementedError, match='past_key_values'):
        m.generate(ids, images=torch.zeros(1, 3, 28, 28), num_beams=2, past_key_values=DynamicCache())
    eng = PrefillEngine.__new__(PrefillEngine)
    with pytest.raises(NotImplementedError, match='use_hf_loop'):
        eng.generate(ids, None, None, num_beams=2, do_sample=True)
    with pytest.raises(NotImplementedError, match='use_hf_loop'):
        eng.generate(ids, None, None, num_beams=2, cache=object())
    with pytest.raises(NotImplementedError, match='use_hf_loop'):
        eng.generate(ids, None, None, num_beams=2, stopping_criteria=[lambda *a: False])


class _BeamStub(_StubEngine):
    """Stub with a beam-dependent next-token rule: logits favour (last + 1) and, a little less, (last + 2) and
    (last + 3), so that beams branch and reorder."""

    def _logits(self, ids):
        V = self.cfg.vocab
        out = torch.full((ids.shape[0], ids.shape[1], V), -10.0)
        for d, v in ((1, 3.0), (2, 2.6), (3, 2.0)):
            out.scatter_(2, ((ids + d) % V)[..., None], v)
        return out


def test_hf_loop_beam_search_through_the_seam():
    """use_hf_loop=True, num_beams=2 on the stub engine: HF's result (its beam search driven directly through a plain
    function of the same rule), the prefill sees 2 rows and 2 box entries, and the cache is reordered."""
    from gpt4roi_b200.engine import EngineConfig
    m = _tiny_model().eval()
    ecfg = EngineConfig(image_size=28, vit_hidden=32, vit_heads=2, vit_layers=2, vit_mlp=64, hidden=64, n_heads=2,
                        n_layers=1, mlp=128, vocab=140)
    stub = _BeamStub(ecfg)
    m._get_engine = lambda device: stub
    ids = torch.tensor([[1, 5, 9]])
    boxes = [torch.tensor([[0.1, 0.1, 0.5, 0.5]])]
    out = m.generate(ids, images=torch.zeros(1, 3, 28, 28), bboxes=boxes, max_new_tokens=4, do_sample=False,
                     num_beams=2, use_hf_loop=True, pad_token_id=0)
    pre = stub.calls[0]
    assert pre[0] == 'prefill' and pre[1] == (2, 3) and len(pre[3]) == 2 and pre[3][0] is boxes[0] \
        and pre[3][1] is boxes[0]
    # the same search by the restatement on the stub's rule
    V = ecfg.vocab
    N, L = 2, 3
    st = new_state(1, N, L, 4, fill=0)
    last = torch.tensor([9, 9])
    for step in range(4):
        x = stub._logits(last[:, None])[:, 0]
        st = ref_select(st['run_score'][:, None] + torch.log_softmax(x, -1), st, N, [], L, L + 4, 1.0, False)
        last = st['ids'].clone()
        if int(st['state'][-1]):
            break
    n = int(st['fin_state'][0, :1, 1].max())
    assert out.tolist() == torch.cat([ids, st['fin_seq'][0, :1, :n]], 1).tolist()


def test_reorder_cache_permutes_rows():
    from gpt4roi_b200.engine import EngineConfig, KVCache
    from gpt4roi_b200.spi_llava import G4RCache
    cfg = EngineConfig(image_size=28, hidden=64, n_heads=2, n_layers=2, mlp=128, vocab=140)
    kv = KVCache(cfg, 3, 6, 'cpu')
    for t in kv.k + kv.v:
        t.copy_(torch.randn(t.shape).to(t.dtype))
    kv.ids.copy_(torch.arange(18).view(3, 6))
    kv.lens = torch.tensor([4, 5, 6], dtype=torch.int32)
    kv.boxes = ['a', 'b', 'c']
    before = [t.clone() for t in kv.k + kv.v]
    ptrs = [t.data_ptr() for t in kv.k + kv.v]
    idx = torch.tensor([2, 0, 0])
    G4RCache(kv).reorder_cache(idx)
    for t, b, p in zip(kv.k + kv.v, before, ptrs):
        assert torch.equal(t, b[idx]) and t.data_ptr() == p
    assert torch.equal(kv.ids, torch.arange(18).view(3, 6)[idx])
    assert kv.lens.tolist() == [6, 4, 4] and kv.boxes == ['c', 'a', 'a']


def test_expand_inputs_repeats_box_lists():
    from gpt4roi_b200.spi_llava import SPILlavaMPTForCausalLM
    a, b = torch.zeros(1, 4), torch.ones(2, 4)
    ids, kw = SPILlavaMPTForCausalLM._expand_inputs_for_generation(
        expand_size=3, input_ids=torch.tensor([[1, 2], [3, 4]]), bboxes=[a, b], images=torch.zeros(2, 3, 4, 4),
        attention_mask=torch.ones(2, 2))
    assert ids.tolist() == [[1, 2]] * 3 + [[3, 4]] * 3
    assert [x is a for x in kw['bboxes']] == [True] * 3 + [False] * 3 and kw['bboxes'][3] is b
    assert kw['images'].shape[0] == 6 and kw['attention_mask'].shape[0] == 6
