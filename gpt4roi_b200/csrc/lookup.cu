// lookup.cu -- prompt-lookup decoding of generate() on the device (transformers' prompt_lookup_num_tokens: the
// PromptLookupCandidateGenerator draft rule and the acceptance of _assisted_decoding), batch 1.  The verify step runs the
// decode chain over M = k + 1 rows of one sequence -- the last accepted token, then the k drafts -- and selects a token
// per row (g4r_sample_tokens_rows).  This kernel, the verify step's last launch, then
//   1. accepts: n = the count of leading drafts equal to the selected tokens; when the candidate sequence was already
//      done (its length reaches max_length, or the host's stopping criteria said so) and every draft matched, n -= 1;
//      the n + 1 selected tokens are appended to the history, at most up to max_length;
//   2. sets `finished` when an appended token is an eos id;
//   3. drafts the next step from the updated history: for n-gram sizes min(max_ngram, len - 1) .. 1, the leftmost
//      window equal to the history's last n-gram that has a continuation wins (one CTA scans the windows in parallel,
//      min-index reduction per size); the draft is up to k ids after it, cut at the first eos id;
//   4. writes the next step's inputs (ids, positions, Philox counters) and a readback for the host.
// g4r_lookup_draft runs steps 3-4 alone (after the prefill's first token).  Integer only, so there is no fp16 twin.
#include "common.cuh"

namespace g4r {

constexpr int kLookupThreads = 256;

__device__ __forceinline__ bool lookup_is_eos(long long t, const int* eos, int n_eos) {
  for (int e = 0; e < n_eos; e++)
    if (t == (long long)eos[e]) return true;
  return false;
}

// state: int32 [5] = {len (history length), d (drafts in ids[1..d]), finished, appended last step, host "candidate
// done" flag}.  readback: int64 [4 + M + k] = {appended, finished, len, d, appended tokens [M], next drafts [k]}.
__global__ void __launch_bounds__(kLookupThreads)
lookup_kernel(int accept, const long long* __restrict__ sel, long long* __restrict__ ids, long long* __restrict__ hist,
              int k, int max_ngram, int prompt_len, int max_length, const int* __restrict__ eos, int n_eos,
              int* __restrict__ state, int* __restrict__ base, int* __restrict__ pos, long long* __restrict__ step,
              long long* __restrict__ readback) {
  __shared__ int s_len, s_fin, s_best, s_d, s_start;
  const int M = k + 1;
  if (threadIdx.x == 0) {
    int len = state[0], fin = state[2], acc = 0;
    if (accept) {
      const int d = state[1];
      int n = 0;
      while (n < d && ids[1 + n] == sel[n]) n++;
      const bool done_cand = len + d >= max_length || state[4] != 0;
      if (done_cand && d > 0 && n == d) n--;
      acc = min(n + 1, max_length - len);
      for (int t = 0; t < acc; t++) {
        hist[len + t] = sel[t];
        readback[4 + t] = sel[t];
        if (lookup_is_eos(sel[t], eos, n_eos)) fin = 1;
      }
      len += acc;
      state[3] = acc;
    }
    s_len = len;
    s_fin = fin;
    s_d = 0;
    readback[0] = acc;
  }
  __syncthreads();
  const int len = s_len;
  // HF drafts nothing when one token is left (max_length == len + 1); a finished or full sequence is not run again
  if (!s_fin && len + 1 < max_length) {
    const int limit = min(len, max_length);   // a window at idx has a continuation iff idx + g < limit
    for (int g = min(max_ngram, len - 1); g >= 1; g--) {
      if (threadIdx.x == 0) s_best = INT_MAX;
      __syncthreads();
      const long long* tail = hist + len - g;
      for (int idx = threadIdx.x; idx + g < limit; idx += blockDim.x) {
        bool eq = true;
        for (int j = 0; j < g && eq; j++) eq = hist[idx + j] == tail[j];
        if (eq) atomicMin(&s_best, idx);
      }
      __syncthreads();
      const int best = s_best;
      if (best != INT_MAX) {
        if (threadIdx.x == 0) {
          const int start = best + g, end = min(start + k, limit);
          int d = 0;
          while (start + d < end && !lookup_is_eos(hist[start + d], eos, n_eos)) d++;
          s_d = d;
          s_start = start;
        }
        break;   // uniform: every thread read the same s_best
      }
    }
  }
  __syncthreads();
  const int d = s_d;
  const long long last = hist[len - 1];
  for (int i = threadIdx.x; i < M; i += blockDim.x) {
    const long long t = (i >= 1 && i <= d) ? hist[s_start + i - 1] : last;   // rows past the draft repeat the last token
    ids[i] = t;
    pos[i] = len - 1 + i;
    step[i] = (long long)(len - prompt_len) + i;
    if (i >= 1) readback[4 + M + i - 1] = (i <= d) ? t : -1;
  }
  if (threadIdx.x == 0) {
    base[0] = len - 1;
    state[0] = len;
    state[1] = d;
    state[2] = s_fin;
    readback[1] = s_fin;
    readback[2] = len;
    readback[3] = d;
  }
}

}  // namespace g4r

using namespace g4r;

static int lookup_launch(int accept, const long long* sel, long long* ids, long long* hist, long long ld_h, int k,
                         int max_ngram, int prompt_len, int max_length, const int* eos, int n_eos, int* state, int* base,
                         int* pos, long long* step, long long* readback, void* stream) {
  G4R_REQUIRE(ids && hist && state && base && pos && step && readback && (sel || !accept), "lookup: null pointer");
  G4R_REQUIRE(k >= 1 && max_ngram >= 1 && prompt_len >= 1 && max_length > prompt_len && max_length <= ld_h &&
                  (n_eos == 0 || eos != nullptr) && n_eos >= 0,
              "lookup: bad arguments (k=%d max_ngram=%d prompt_len=%d max_length=%d ld_h=%lld n_eos=%d)", k, max_ngram,
              prompt_len, max_length, ld_h, n_eos);
  lookup_kernel<<<1, kLookupThreads, 0, (cudaStream_t)stream>>>(accept, sel, ids, hist, k, max_ngram, prompt_len,
                                                                max_length, eos, n_eos, state, base, pos, step,
                                                                readback);
  G4R_LAUNCH_CHECK("lookup");
  return G4R_OK;
}

extern "C" int g4r_lookup_step(const long long* sel, long long* ids, long long* hist, long long ld_h, int k,
                               int max_ngram, int prompt_len, int max_length, const int* eos, int n_eos, int* state,
                               int* base, int* pos, long long* step, long long* readback, void* stream) {
  return lookup_launch(1, sel, ids, hist, ld_h, k, max_ngram, prompt_len, max_length, eos, n_eos, state, base, pos, step,
                       readback, stream);
}

extern "C" int g4r_lookup_draft(long long* ids, long long* hist, long long ld_h, int k, int max_ngram, int prompt_len,
                                int max_length, const int* eos, int n_eos, int* state, int* base, int* pos,
                                long long* step, long long* readback, void* stream) {
  return lookup_launch(0, nullptr, ids, hist, ld_h, k, max_ngram, prompt_len, max_length, eos, n_eos, state, base, pos,
                       step, readback, stream);
}
