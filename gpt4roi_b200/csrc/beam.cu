// beam.cu -- one step of deterministic beam search on the device (transformers' GenerationMixin._beam_search with
// do_sample=False): the last two kernels of the graphed beam decode step.  They read the lm_head logits of the B*N beam
// rows and write the next ids straight into the graph's input, the beam rows' positions and the ancestry table the
// decode attention reads (decode.cu, BEAM), so a replay needs nothing from the host.
//
// Kernel A (beam_topk_kernel), one CTA per beam row: the row's fp32 max and sum of exp(x - max) in a fixed order, then
// the row's top K = beams_to_keep tokens by (value descending, index ascending), emitted with the accumulated score
// running_score[r] + ((x - max) - log sum), the operation order of torch's log_softmax followed by HF's addition.
// Kernel B (beam_select_kernel), one CTA per sample: the N*K candidates are merged by (score descending, flat index
// beam*V + token ascending) -- the only stated deviation from HF, whose CUDA topk order among equal scores is
// unspecified -- and then HF's helpers run in order on the sample's top K: _get_top_k_continuations,
// _get_running_beams_for_next_iteration, _update_finished_beams, _check_early_stop_heuristic and the sample's part of
// _beam_search_has_unfinished_sequences.  The last CTA to finish (an integer ticket) folds the samples' flags into the
// batch's done word.  No float atomics and every float sum has a fixed order, so a replay is bitwise repeatable.
//
// Outputs (g4r_beam_step_out_*, transformers' return_dict_in_generate): kernel A writes every id's log-softmax value
// (x - max) - log sum -- HF's scores entry, before the running score is added -- and the widened logit into slot g (the
// sample's generated-token count, read from the device state, so graph replays fill successive slots) of fp32 buffers
// [n_slots, B*N, V]; kernel B keeps a beam-index column beside the sequences (HF's beam_indices: b*N + parent beam at
// column g, -1 where nothing was generated), double-buffered and gathered exactly as the sequences are.
//
// Beam KV layout (engine.BeamCache): cache rows 0..B-1 hold the prompts, rows B..B+B*N-1 the beams.  A cell is written
// once and never moved; anc[r, p] names the cache row that holds position p of beam row r.  Reordering the beams
// permutes the generated columns of anc (staged in shared memory) instead of copying K/V.
#include "common.cuh"
#include "act_type.cuh"   // bf16 as written; fp16 twin with -DG4R_ACT_HALF

namespace G4R_NS {
namespace {

constexpr int TOPK_THREADS = 512;
constexpr int SEL_THREADS = 256;
constexpr int BEAM_MAX_KEEP = 64;   // beams_to_keep = max(2, 1 + n_eos) * N
constexpr int BEAM_MAX_N = 32;
constexpr int BEAM_MAX_CAND = 1024; // N * beams_to_keep
constexpr float NEG_BIG = -1.0e9f;  // HF's mask value; exact in fp32

#ifdef G4R_ACT_HALF
__device__ __forceinline__ float bits_value(unsigned b) { return __half2float(__ushort_as_half((unsigned short)b)); }
constexpr unsigned ACT_INF_BITS = 0x7C00u;
#else
__device__ __forceinline__ float bits_value(unsigned b) { return __uint_as_float(b << 16); }
constexpr unsigned ACT_INF_BITS = 0x7F80u;
#endif

// Order key of a 16-bit float (as in sample.cu): keys ascend with the value, -0 folds onto +0, NaN onto the top key.
__device__ __forceinline__ unsigned order_key(unsigned bits) {
  if ((bits & 0x7FFFu) > ACT_INF_BITS) return 0xFFFFu;
  if (bits == 0x8000u) bits = 0;
  return (bits & 0x8000u) ? (~bits & 0xFFFFu) : (bits | 0x8000u);
}
__device__ __forceinline__ float key_value(unsigned key) {
  return bits_value((key & 0x8000u) ? (key & 0x7FFFu) : (~key & 0xFFFFu));
}

}  // namespace

__global__ void __launch_bounds__(TOPK_THREADS)
beam_topk_kernel(const unsigned short* __restrict__ logits, long long ld, int row_div, int V, int K,
                 const float* __restrict__ run_score, float* __restrict__ cand_score, int* __restrict__ cand_tok,
                 const int* __restrict__ state, int N, float* __restrict__ out_scores, float* __restrict__ out_logits,
                 int n_slots) {
  extern __shared__ unsigned short keys[];   // [V] order keys of the row
  constexpr int W = TOPK_THREADS / 32;
  __shared__ unsigned long long s_best[W];
  __shared__ float s_sum[W];
  __shared__ unsigned s_max[W];
  const int r = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // step 0: the N beams of a sample read its one prefill row (row_div = N)
  const unsigned short* row = logits + (long long)(r / row_div) * ld;
  unsigned mk = 0;
  for (int i = tid; i < V; i += TOPK_THREADS) {
    const unsigned k = order_key(row[i]);
    keys[i] = (unsigned short)k;
    mk = max(mk, k);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mk = max(mk, __shfl_xor_sync(0xffffffffu, mk, o));
  if (lane == 0) s_max[warp] = mk;
  __syncthreads();
  mk = s_max[0];
#pragma unroll
  for (int w = 1; w < W; w++) mk = max(mk, s_max[w]);
  const float mx = key_value(mk);
  float s = 0.f;
  for (int i = tid; i < V; i += TOPK_THREADS) s += expf(__fsub_rn(key_value(keys[i]), mx));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) s_sum[warp] = s;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int w = 0; w < W; w++) tot += s_sum[w];
  const float logz = logf(tot);
  const float base = run_score[r];
  if (out_scores || out_logits) {
    const int slot = state[4 * (r / N)];
    if (slot < n_slots) {
      const long long o = ((long long)slot * gridDim.x + r) * V;
      for (int i = tid; i < V; i += TOPK_THREADS) {
        const float x = bits_value(row[i]);
        if (out_scores) out_scores[o + i] = __fsub_rn(__fsub_rn(x, mx), logz);
        if (out_logits) out_logits[o + i] = x;
      }
    }
  }
  // top K by (value descending, index ascending): packed = key << 32 | ~index is unique per element, so the k-th pick
  // is the largest packed value below the (k-1)-th
  unsigned long long prev = ~0ULL;
  for (int k = 0; k < K; k++) {
    unsigned long long best = 0;
    for (int i = tid; i < V; i += TOPK_THREADS) {
      const unsigned long long p = ((unsigned long long)keys[i] << 32) | (0xFFFFFFFFu - (unsigned)i);
      if (p < prev && p > best) best = p;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long n = __shfl_xor_sync(0xffffffffu, best, o);
      best = n > best ? n : best;
    }
    if (lane == 0) s_best[warp] = best;
    __syncthreads();
    best = s_best[0];
#pragma unroll
    for (int w = 1; w < W; w++) best = s_best[w] > best ? s_best[w] : best;
    __syncthreads();   // s_best is rewritten by the next pick
    prev = best;
    if (tid == 0) {
      const float x = key_value((unsigned)(best >> 32));
      cand_score[(long long)r * K + k] = __fadd_rn(base, __fsub_rn(__fsub_rn(x, mx), logz));
      cand_tok[(long long)r * K + k] = (int)(0xFFFFFFFFu - (unsigned)best);
    }
  }
}

// state (int32): per sample b, state[4b + 0] = generated tokens so far (g), [4b + 1] = HF's
// is_early_stop_heuristic_unsatisfied, [4b + 2] = flags (1: every finished slot filled, 2: every top-K candidate hit a
// stopping criterion); state[4B] = ticket, state[4B + 1] = done (the whole batch).  fin_state (int32 [B, N, 2]): the
// finished slot's is_sent_finished and generated length.  run_seq / fin_seq: int64 [2, B, N, G] generated columns,
// double-buffered by the parity of g (read g & 1, write the other); run_bidx / fin_bidx: int32 [2, B, N, G] beam-index
// columns beside them, the same way (null: not kept).
__global__ void __launch_bounds__(SEL_THREADS)
beam_select_kernel(const float* __restrict__ cand_score, const int* __restrict__ cand_tok, int N, int K, int V,
                   const int* __restrict__ eos_ids, int n_eos, int prompt_len, int max_length, double length_penalty,
                   int early, int G, int Lmax, const int* __restrict__ lens, int* state, float* __restrict__ run_score,
                   long long* __restrict__ run_seq, long long* __restrict__ fin_seq, float* __restrict__ fin_score,
                   int* __restrict__ fin_state, long long* __restrict__ ids, int* __restrict__ pos_rows,
                   int* __restrict__ anc, int* __restrict__ run_bidx, int* __restrict__ fin_bidx) {
  extern __shared__ int stage[];   // [N][g] generated columns of anc
  __shared__ float s_cs[BEAM_MAX_CAND];
  __shared__ int s_ct[BEAM_MAX_CAND];
  __shared__ float s_lp[BEAM_MAX_KEEP];
  __shared__ int s_par[BEAM_MAX_KEEP], s_tok[BEAM_MAX_KEEP];
  __shared__ int s_run[BEAM_MAX_N], s_sel[BEAM_MAX_N];   // running pick (index into top K), finished pick (merged index)
  const int b = blockIdx.x, B = gridDim.x, tid = threadIdx.x;
  const int g = state[4 * b];
  const int M = N * K;
  for (int c = tid; c < M; c += SEL_THREADS) {
    s_cs[c] = cand_score[(long long)b * M + c];
    s_ct[c] = cand_tok[(long long)b * M + c];
  }
  __syncthreads();
  // ---- _get_top_k_continuations: the sample's top K of N*V by (score descending, flat index ascending)
  for (int c = tid; c < M; c += SEL_THREADS) {
    const float s = s_cs[c];
    const long long fi = (long long)(c / K) * V + s_ct[c];
    int rank = 0;
    for (int d = 0; d < M; d++) {
      const float t = s_cs[d];
      rank += (t > s) || (t == s && (long long)(d / K) * V + s_ct[d] < fi);
    }
    if (rank < K) {
      s_lp[rank] = s;
      s_par[rank] = c / K;
      s_tok[rank] = s_ct[c];
    }
  }
  const int lb = lens[b];
  for (int i = tid; i < N * g; i += SEL_THREADS)
    stage[i] = anc[(long long)(b * N + i / g) * Lmax + lb + i % g];
  __syncthreads();
  if (tid == 0) {
    const int cur = prompt_len + g;
    const bool max_hit = cur + 1 >= max_length;       // MaxLengthCriteria on topk_running_sequences[:, :, :cur + 1]
    bool hit[BEAM_MAX_KEEP];
    bool all_hit = true;
    for (int k = 0; k < K; k++) {
      bool e = max_hit;
      for (int q = 0; q < n_eos; q++) e = e || s_tok[k] == eos_ids[q];   // EosTokenCriteria
      hit[k] = e;
      all_hit = all_hit && e;
    }
    // ---- _get_running_beams_for_next_iteration: top N of topk_log_probs + hit * -1e9
    float rs[BEAM_MAX_KEEP];
    for (int k = 0; k < K; k++) rs[k] = __fadd_rn(s_lp[k], hit[k] ? NEG_BIG : -0.f);
    for (int k = 0; k < K; k++) {
      int rank = 0;
      for (int d = 0; d < K; d++) rank += (rs[d] > rs[k]) || (rs[d] == rs[k] && d < k);
      if (rank < N) s_run[rank] = k;
    }
    // ---- _update_finished_beams
    const int unsat_old = state[4 * b + 1];
    bool all_fin_old = true;
    for (int j = 0; j < N; j++) all_fin_old = all_fin_old && fin_state[(b * N + j) * 2] != 0;
    const bool full = all_fin_old && early == 1;
    const float denom = (float)pow((double)(g + 1), length_penalty);   // (cur_len + 1 - prompt_len) ** length_penalty
    float ms[BEAM_MAX_N + BEAM_MAX_KEEP];
    for (int j = 0; j < N; j++) ms[j] = fin_score[b * N + j];
    for (int k = 0; k < K; k++) {
      float x = __fdiv_rn(s_lp[k], denom);
      x = __fadd_rn(x, full ? NEG_BIG : -0.f);
      x = __fadd_rn(x, unsat_old ? -0.f : NEG_BIG);
      x = __fadd_rn(x, (hit[k] && k < N) ? -0.f : NEG_BIG);
      ms[N + k] = x;
    }
    for (int m = 0; m < N + K; m++) {
      int rank = 0;
      for (int d = 0; d < N + K; d++) rank += (ms[d] > ms[m]) || (ms[d] == ms[m] && d < m);
      if (rank < N) s_sel[rank] = m;
    }
    // new finished scores / flags (the sequences are copied below, from the old buffers)
    float fs[BEAM_MAX_N];
    int ff[BEAM_MAX_N], fl[BEAM_MAX_N];
    for (int j = 0; j < N; j++) {
      const int m = s_sel[j];
      fs[j] = ms[m];
      if (m < N) {
        ff[j] = fin_state[(b * N + m) * 2];
        fl[j] = fin_state[(b * N + m) * 2 + 1];
      } else {
        ff[j] = hit[m - N] && (m - N) < N;
        fl[j] = g + 1;
      }
    }
    bool all_fin = true;
    float worst = fs[0];
    for (int j = 0; j < N; j++) {
      fin_score[b * N + j] = fs[j];
      fin_state[(b * N + j) * 2] = ff[j];
      fin_state[(b * N + j) * 2 + 1] = fl[j];
      all_fin = all_fin && ff[j];
      worst = fminf(worst, fs[j]);
      run_score[b * N + j] = rs[s_run[j]];
    }
    // ---- _check_early_stop_heuristic at cur_len + 1
    const int best_len = (early == 2 && length_penalty > 0.0) ? max_length - prompt_len : g + 1;
    const float best = __fdiv_rn(rs[s_run[0]], (float)pow((double)best_len, length_penalty));
    bool improve = false;
    for (int j = 0; j < N; j++) improve = improve || best > (ff[j] ? worst : NEG_BIG);
    state[4 * b + 1] = unsat_old && improve;
    state[4 * b + 2] = (all_fin ? 1 : 0) | (all_hit ? 2 : 0);
  }
  __syncthreads();
  // ---- the new running beams: ids, positions, ancestry, sequences
  const int p = g & 1;
  const long long* rsrc = run_seq + ((long long)p * B + b) * N * G;
  long long* rdst = run_seq + ((long long)(p ^ 1) * B + b) * N * G;
  const long long* fsrc = fin_seq + ((long long)p * B + b) * N * G;
  long long* fdst = fin_seq + ((long long)(p ^ 1) * B + b) * N * G;
  for (int j = 0; j < N; j++) {
    const int k = s_run[j], par = s_par[k];
    int* arow = anc + (long long)(b * N + j) * Lmax + lb;
    for (int i = tid; i < g; i += SEL_THREADS) arow[i] = stage[par * g + i];
    for (int i = tid; i < G; i += SEL_THREADS) rdst[(long long)j * G + i] = i == g ? s_tok[k] : rsrc[(long long)par * G + i];
    const int m = s_sel[j];
    if (m < N) {
      for (int i = tid; i < G; i += SEL_THREADS) fdst[(long long)j * G + i] = fsrc[(long long)m * G + i];
    } else {
      const int fk = m - N, fpar = s_par[fk];
      for (int i = tid; i < G; i += SEL_THREADS)
        fdst[(long long)j * G + i] = i == g ? s_tok[fk] : rsrc[(long long)fpar * G + i];
    }
    if (run_bidx) {   // the beam indices, gathered as the sequences above
      const int* rbs = run_bidx + ((long long)p * B + b) * N * G;
      int* rbd = run_bidx + ((long long)(p ^ 1) * B + b) * N * G;
      const int* fbs = fin_bidx + ((long long)p * B + b) * N * G;
      int* fbd = fin_bidx + ((long long)(p ^ 1) * B + b) * N * G;
      for (int i = tid; i < G; i += SEL_THREADS) rbd[(long long)j * G + i] = i == g ? b * N + par : rbs[(long long)par * G + i];
      if (m < N) {
        for (int i = tid; i < G; i += SEL_THREADS) fbd[(long long)j * G + i] = fbs[(long long)m * G + i];
      } else {
        const int fpar = s_par[m - N];
        for (int i = tid; i < G; i += SEL_THREADS)
          fbd[(long long)j * G + i] = i == g ? b * N + fpar : rbs[(long long)fpar * G + i];
      }
    }
    if (tid == 0) {
      arow[g] = B + b * N + j;   // cache row of beam row b*N+j (the B prompt rows come first): it writes position lens[b] + g
      ids[b * N + j] = s_tok[k];
      pos_rows[b * N + j] = lb + g;
    }
  }
  // ---- _beam_search_has_unfinished_sequences over the batch: the last CTA folds every sample's flags
  if (tid == 0) {
    state[4 * b] = g + 1;
    __threadfence();
    const int t = atomicAdd(&state[4 * B], 1);
    if (t == B - 1) {
      __threadfence();
      const volatile int* vs = state;
      bool any_unsat = false, all_fin = true, all_hit = true;
      for (int s = 0; s < B; s++) {
        any_unsat = any_unsat || vs[4 * s + 1];
        all_fin = all_fin && (vs[4 * s + 2] & 1);
        all_hit = all_hit && (vs[4 * s + 2] & 2);
      }
      state[4 * B + 1] = !(any_unsat && !(all_fin && early == 1) && !all_hit);
      state[4 * B] = 0;
    }
  }
}

}  // namespace G4R_NS

using namespace G4R_NS;

static int beam_step(const void* logits, long long ld, int row_div, int B, int N, int V, int K, const int* eos_ids,
                     int n_eos, int prompt_len, int max_length, double length_penalty, int early_stopping, int G,
                     int Lmax, const int* lens, int* state, float* run_score, float* cand_score, int* cand_tok,
                     long long* run_seq, long long* fin_seq, float* fin_score, int* fin_state, long long* ids,
                     int* pos_rows, int* anc, float* scores, float* raw_logits, int n_slots, int* run_bidx,
                     int* fin_bidx, void* stream) {
  G4R_REQUIRE(logits && lens && state && run_score && cand_score && cand_tok && run_seq && fin_seq && fin_score &&
              fin_state && ids && pos_rows && anc && (n_eos == 0 || eos_ids),
              "beam_step: NULL argument");
  G4R_REQUIRE(B > 0 && N > 1 && N <= BEAM_MAX_N && K >= N && K <= BEAM_MAX_KEEP && N * K <= BEAM_MAX_CAND && V >= K &&
              ld >= V && (row_div == 1 || row_div == N) && G > 0 && early_stopping >= 0 && early_stopping <= 2,
              "beam_step: bad arguments (B=%d N=%d K=%d V=%d row_div=%d G=%d)", B, N, K, V, row_div, G);
  G4R_REQUIRE((!scores && !raw_logits) || n_slots > 0, "beam_step: outputs need n_slots > 0 (n_slots=%d)", n_slots);
  G4R_REQUIRE(!run_bidx == !fin_bidx, "beam_step: run_bidx and fin_bidx go together");
  const size_t smem_a = (size_t)V * sizeof(unsigned short);
  const size_t smem_b = (size_t)N * G * sizeof(int);
  G4R_REQUIRE(smem_a <= 200 * 1024 && smem_b <= 200 * 1024,
              "beam_step: V=%d or N*max_new_tokens=%d too large for shared memory", V, N * G);
  cudaStream_t st = (cudaStream_t)stream;
  static bool set = false;
  if (!set) {
    G4R_CUDA(cudaFuncSetAttribute(beam_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    G4R_CUDA(cudaFuncSetAttribute(beam_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    set = true;
  }
  beam_topk_kernel<<<B * N, TOPK_THREADS, smem_a, st>>>((const unsigned short*)logits, ld, row_div, V, K, run_score,
                                                         cand_score, cand_tok, state, N, scores, raw_logits, n_slots);
  G4R_LAUNCH_CHECK("beam_topk");
  beam_select_kernel<<<B, SEL_THREADS, smem_b, st>>>(cand_score, cand_tok, N, K, V, eos_ids, n_eos, prompt_len,
                                                     max_length, length_penalty, early_stopping, G, Lmax, lens, state,
                                                     run_score, run_seq, fin_seq, fin_score, fin_state, ids, pos_rows,
                                                     anc, run_bidx, fin_bidx);
  G4R_LAUNCH_CHECK("beam_select");
  return G4R_OK;
}

extern "C" int g4r_beam_step_bf16(const void* logits, long long ld, int row_div, int B, int N, int V, int K,
                                  const int* eos_ids, int n_eos, int prompt_len, int max_length, double length_penalty,
                                  int early_stopping, int G, int Lmax, const int* lens, int* state, float* run_score,
                                  float* cand_score, int* cand_tok, long long* run_seq, long long* fin_seq,
                                  float* fin_score, int* fin_state, long long* ids, int* pos_rows, int* anc,
                                  void* stream) {
  return beam_step(logits, ld, row_div, B, N, V, K, eos_ids, n_eos, prompt_len, max_length, length_penalty,
                   early_stopping, G, Lmax, lens, state, run_score, cand_score, cand_tok, run_seq, fin_seq, fin_score,
                   fin_state, ids, pos_rows, anc, nullptr, nullptr, 0, nullptr, nullptr, stream);
}

extern "C" int g4r_beam_step_out_bf16(const void* logits, long long ld, int row_div, int B, int N, int V, int K,
                                      const int* eos_ids, int n_eos, int prompt_len, int max_length,
                                      double length_penalty, int early_stopping, int G, int Lmax, const int* lens,
                                      int* state, float* run_score, float* cand_score, int* cand_tok,
                                      long long* run_seq, long long* fin_seq, float* fin_score, int* fin_state,
                                      long long* ids, int* pos_rows, int* anc, float* scores, float* raw_logits,
                                      int n_slots, int* run_bidx, int* fin_bidx, void* stream) {
  return beam_step(logits, ld, row_div, B, N, V, K, eos_ids, n_eos, prompt_len, max_length, length_penalty,
                   early_stopping, G, Lmax, lens, state, run_score, cand_score, cand_tok, run_seq, fin_seq, fin_score,
                   fin_state, ids, pos_rows, anc, scores, raw_logits, n_slots, run_bidx, fin_bidx, stream);
}
