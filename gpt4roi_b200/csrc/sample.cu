// sample.cu -- next-token selection on the device for the decode loop behind generate(): arg-max, or a draw from the
// temperature / top-k / top-p processed softmax (transformers' GenerationMixin._sample with TemperatureLogitsWarper,
// TopKLogitsWarper and TopPLogitsWarper), plus the eos -> pad rule for finished rows.  It is the last kernel of the
// graphed decode step: it reads the lm_head logits [B, V] and writes the next ids straight into the graph's input.
//
// One CTA (1024 threads) per row.  Sampling needs no sort: every distinct 16-bit logit value has one probability, so
// the row is reduced to a histogram over the 65 536 bit patterns (packed 16-bit counts in 132 KB of shared memory,
// integer atomics, so the counts do not depend on the order of the updates).  The bins are walked in value order --
// thread t owns the 64 consecutive order keys [64t, 64t + 64) -- and block-wide suffix scans of the per-thread counts
// and masses (count * exp(v / T - max / T)) give the top-k threshold, the top-p threshold and the bin the inverse CDF
// lands in.  Every float sum has a fixed order (per-thread walk from the top key down, then a fixed shuffle tree), so
// the same logits, seed and step give the same token on every run.  Within the chosen value the j-th occurrence in
// index order is the token: the CDF runs over (value descending, index ascending).
//
// Draws: Philox4x32-10 (Salmon et al., SC'11, the Random123 generator), key = seed, counter = (step, row, 0); the
// uniform is (word0 >> 8) * 2^-24.  `step` is read from device memory, so successive replays of one captured graph draw
// fresh numbers once the host advances it.
#include "common.cuh"
#include "act_type.cuh"   // bf16 as written; fp16 twin with -DG4R_ACT_HALF

namespace G4R_NS {

constexpr int SAMPLE_THREADS = 1024;
constexpr int SAMPLE_KEYS = SAMPLE_THREADS * 64;             // one bin per 16-bit pattern
constexpr int SAMPLE_WORDS = SAMPLE_KEYS / 2;                // two 16-bit counts per word
// thread t's 32 words sit at [33t, 33t + 32): the pad word makes word j of the 32 lanes of a warp hit 32 different
// banks, so the per-thread walks over the bins are conflict-free
constexpr int SAMPLE_SMEM_WORDS = SAMPLE_THREADS * 33;
constexpr size_t SAMPLE_SMEM = (size_t)SAMPLE_SMEM_WORDS * sizeof(unsigned);

#ifdef G4R_ACT_HALF
__device__ __forceinline__ float bits_value(unsigned b) { return __half2float(__ushort_as_half((unsigned short)b)); }
constexpr unsigned ACT_INF_BITS = 0x7C00u;
#else
__device__ __forceinline__ float bits_value(unsigned b) { return __uint_as_float(b << 16); }
constexpr unsigned ACT_INF_BITS = 0x7F80u;
#endif

// Order key of a 16-bit float: keys ascend with the value.  -0 is folded onto +0 and every NaN onto the top key, so
// equal values share one bin and the arg-max takes a NaN as torch.argmax does.
__device__ __forceinline__ unsigned order_key(unsigned bits) {
  if ((bits & 0x7FFFu) > ACT_INF_BITS) return 0xFFFFu;
  if (bits == 0x8000u) bits = 0;
  return (bits & 0x8000u) ? (~bits & 0xFFFFu) : (bits | 0x8000u);
}
__device__ __forceinline__ float key_value(unsigned key) {
  return bits_value((key & 0x8000u) ? (key & 0x7FFFu) : (~key & 0xFFFFu));
}
__device__ __forceinline__ int hist_word(unsigned key) { return (int)(key >> 6) * 33 + (int)((key >> 1) & 31); }
__device__ __forceinline__ unsigned bin_count(const unsigned* hist, unsigned key) {
  return (hist[hist_word(key)] >> ((key & 1) * 16)) & 0xFFFFu;
}

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; r++) {
    if (r) {
      k.x += 0x9E3779B9u;
      k.y += 0xBB67AE85u;
    }
    const unsigned hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const unsigned hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
  }
  return c;
}

// Inclusive and exclusive suffix sums over the threads of the block (thread t: sum over threads >= t / > t).  A fixed
// shuffle tree, so the float sums are reproducible.  `tot` is [32] shared scratch.
template <typename T>
__device__ __forceinline__ void suffix_scan(T v, T* tot, T& incl, T& excl) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T n = __shfl_down_sync(0xffffffffu, v, o);
    if (lane + o < 32) v += n;
  }
  T nxt = __shfl_down_sync(0xffffffffu, v, 1);
  if (lane == 31) nxt = T(0);
  if (lane == 0) tot[warp] = v;
  __syncthreads();
  if (warp == 0) {
    T x = tot[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const T n = __shfl_down_sync(0xffffffffu, x, o);
      if (lane + o < 32) x += n;
    }
    tot[lane] = x;
  }
  __syncthreads();
  const T above = warp + 1 < 32 ? tot[warp + 1] : T(0);
  incl = v + above;
  excl = nxt + above;
  __syncthreads();   // tot is reused by the next scan
}

// ---- the processed variant (g4r_sample_tokens_proc_*): transformers' history-dependent logits processors first
// (RepetitionPenaltyLogitsProcessor, NoRepeatNGramLogitsProcessor, MinLengthLogitsProcessor,
// MinNewTokensLengthLogitsProcessor), then the selection above on the processed fp32 scores.  The row's history
// h[0, L + *rng_step) becomes two bitmaps in shared memory: `pres` (ids present: the penalised ones) and `ban` (ids
// set to -inf: the n-gram matches, and the eos ids while a minimum length is in force).  Greedy compares fp32 order
// keys of the processed values.  Sampling keeps the 16-bit histogram for the untouched ids; the penalised ids are not
// 16-bit values, so they form a list (fp32 order key << 32 | ~index) sorted descending, which every per-thread walk
// merges into its bins: thread t owns the list entries whose value rounds down to one of its 64 keys, an entry strictly
// above its bin comes before the bin, one equal to it joins the bin's group.  Thresholds are fp32 order keys, so equal
// processed values form one group whichever set they come from.
constexpr int PROC_LIST_MAX = 8192;   // penalised ids a sampled row may hold: 64 KB of shared memory

struct SampleProc {
  long long* hist;        // int64 [B, ld_h]: row b's history, L + *rng_step ids long
  long long ld_h;
  int L;
  float penalty;          // 1: off
  int ngram;              // 0: off
  int min_length, min_new_tokens;
  const int* eos_ids;     // the ids min_length / min_new_tokens suppress
  int n_eos;
  int append;             // write the selected token to h[b, L + *rng_step]
};

// The output pass (g4r_sample_tokens_out_*): transformers' return_dict_in_generate scores.  Slot *rng_step of two fp32
// buffers [n_slots, B, V] gets, for every id, the processed score the selection used (the history-dependent processors,
// then, when sampling, / temperature and -inf below the top-k / top-p thresholds: HF's next_token_scores) and the
// widened logit (HF's next_token_logits).  Either pointer may be null; a slot past n_slots is not written.
struct SampleOut {
  float* scores;
  float* logits;
  long long n_slots;
};

template <typename F>
__device__ __forceinline__ void write_outputs(const SampleOut& o, const unsigned short* __restrict__ row, int V,
                                              long long slot, F&& score) {
  if (slot < 0 || slot >= o.n_slots) return;
  const long long base = (slot * gridDim.x + blockIdx.x) * V;
  for (int i = threadIdx.x; i < V; i += SAMPLE_THREADS) {
    if (o.scores) o.scores[base + i] = score(i);
    if (o.logits) o.logits[base + i] = bits_value(row[i]);
  }
}

// Order key of an fp32 value: ascends with the value; -0 folded onto +0, every NaN onto the top key (torch.argmax).
__device__ __forceinline__ unsigned f32_key(float y) {
  if (y != y) return 0xFFFFFFFFu;
  const unsigned u = __float_as_uint(y == 0.f ? 0.f : y);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float f32_of_key(unsigned k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}
// The largest 16-bit value <= y, as bits (rounding toward -inf).
#ifdef G4R_ACT_HALF
__device__ __forceinline__ unsigned bits_rd(float y) { return __half_as_ushort(__float2half_rd(y)); }
#else
__device__ __forceinline__ unsigned bits_rd(float y) {
  const unsigned u = __float_as_uint(y);
  return (u >> 16) + (((u & 0xFFFFu) && (u >> 31)) ? 1u : 0u);
}
#endif
__device__ __forceinline__ bool bit_of(const unsigned* bm, int i) { return (bm[i >> 5] >> (i & 31)) & 1u; }

// The processed units (distinct values, with counts) of thread `key0 >> 6`, from its top key down: f(order key,
// value, count) returns false to stop.  list[n0, n1) is the thread's part of the sorted penalised list.
template <typename F>
__device__ __forceinline__ void walk_units(const unsigned* hist, const unsigned long long* list, int n0, int n1,
                                           unsigned key0, F&& f) {
  int n = n0;
  for (int j = 63; j >= 0; j--) {
    const unsigned key = key0 + j;
    int c = (int)bin_count(hist, key);
    if (n >= n1 && !c) continue;   // no list entry left and an empty bin: as cheap as the plain kernel's walk
    while (n < n1) {   // penalised values strictly between this bin's value and the next bin's
      const unsigned yk = (unsigned)(list[n] >> 32);
      const float y = f32_of_key(yk);
      const unsigned bits = bits_rd(y);
      if (order_key(bits) != key || bits_value(bits) == y) break;
      int cy = 1;
      for (n++; n < n1 && (unsigned)(list[n] >> 32) == yk; n++) cy++;
      if (!f(yk, y, cy)) return;
    }
    const float v = key_value(key);
    const unsigned vk = f32_key(v);
    for (; n < n1 && (unsigned)(list[n] >> 32) == vk; n++) c++;   // penalised values equal to this bin's
    if (c && !f(vk, v, c)) return;
  }
}

// Which thread's keys a list entry's value rounds down to.
__device__ __forceinline__ int list_owner(unsigned long long e) {
  return (int)(order_key(bits_rd(f32_of_key((unsigned)(e >> 32)))) >> 6);
}

template <bool OUT>
__device__ void select_processed(const unsigned short* __restrict__ row, int V, float temperature, int top_k,
                                 float top_p, int greedy, unsigned long long seed, const long long* __restrict__ rng_step,
                                 const SampleProc& pr, const SampleOut& out, unsigned* smem, int& s_tok,
                                 unsigned rng_row) {
  __shared__ unsigned long long s_best[32];
  __shared__ int s_int[32];
  __shared__ float s_flt[32];
  __shared__ int s_P, s_find, s_low, s_j;
  __shared__ unsigned s_maxk, s_kthr, s_pthr, s_sel;
  __shared__ float s_zk;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int W = (V + 31) >> 5;
  unsigned* hist = smem;
  unsigned* pres = smem + (greedy ? 0 : SAMPLE_SMEM_WORDS);
  unsigned* ban = pres + W;
  unsigned long long* list = (unsigned long long*)(ban + W);
  const long long step = *rng_step;
  const long long* h = pr.hist + (long long)b * pr.ld_h;
  const int Lh = (int)min((long long)pr.L + step, pr.ld_h);
  const bool pen = pr.penalty != 1.f;
  const float p = pr.penalty;

  // ---- the bitmaps of the history
  for (int i = tid; i < 2 * W; i += SAMPLE_THREADS) pres[i] = 0u;
  if (tid == 0) s_tok = 0;
  __syncthreads();
  if (pen)
    for (int j = tid; j < Lh; j += SAMPLE_THREADS) {
      const long long t = h[j];
      if (t >= 0 && t < V) atomicOr(&pres[t >> 5], 1u << (t & 31));
    }
  const int n = pr.ngram;
  if (n > 0 && Lh + 1 >= n) {   // ban t when h[j, j + n) == (the last n - 1 ids of h, t)
    const long long* tail = h + Lh - (n - 1);
    for (int j = tid; j + n <= Lh; j += SAMPLE_THREADS) {
      bool m = true;
      for (int q = 0; q < n - 1 && m; q++) m = h[j + q] == tail[q];
      const long long t = h[j + n - 1];
      if (m && t >= 0 && t < V) atomicOr(&ban[t >> 5], 1u << (t & 31));
    }
  }
  if (Lh < pr.min_length || step < pr.min_new_tokens)
    for (int e = tid; e < pr.n_eos; e += SAMPLE_THREADS) {
      const int t = pr.eos_ids[e];
      if (t >= 0 && t < V) atomicOr(&ban[t >> 5], 1u << (t & 31));
    }
  __syncthreads();
  // processed value of id i (false: banned, -inf)
  auto value = [&](int i, float& y) -> bool {
    if (bit_of(ban, i)) return false;
    y = bits_value(row[i]);
    if (pen && bit_of(pres, i)) y = y < 0.f ? __fmul_rn(y, p) : __fdiv_rn(y, p);
    return true;
  };

  if (greedy) {
    // arg-max of the processed fp32 scores, first index among equals
    unsigned long long best = 0;
    for (int i = tid; i < V; i += SAMPLE_THREADS) {
      float y;
      const unsigned k = value(i, y) ? f32_key(y) : f32_key(-INFINITY);
      const unsigned long long q = ((unsigned long long)k << 32) | (0xFFFFFFFFu - (unsigned)i);
      best = q > best ? q : best;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long x = __shfl_xor_sync(0xffffffffu, best, o);
      best = x > best ? x : best;
    }
    if (lane == 0) s_best[warp] = best;
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < 32; w++) best = s_best[w] > best ? s_best[w] : best;
      s_tok = (int)(0xFFFFFFFFu - (unsigned)best);
    }
    if constexpr (OUT)
      write_outputs(out, row, V, step, [&](int i) {
        float y;
        return value(i, y) ? y : -INFINITY;
      });
    return;
  }

  // ---- histogram of the untouched ids; the penalised ids listed in index order
  for (int i = tid; i < SAMPLE_SMEM_WORDS; i += SAMPLE_THREADS) hist[i] = 0u;
  if (tid == 0) {
    s_P = 0;
    s_maxk = 0u;
    s_kthr = 0u;
    s_find = -1;
  }
  __syncthreads();
  for (int i = tid; i < V; i += SAMPLE_THREADS) {
    if (bit_of(ban, i) || (pen && bit_of(pres, i))) continue;
    const unsigned key = order_key(row[i]);
    atomicAdd(&hist[hist_word(key)], 1u << ((key & 1) * 16));
  }
  __syncthreads();   // the counts land in other threads' bins: complete before any walk reads them
  if (pen) {
    for (int base = 0; base < W; base += SAMPLE_THREADS) {
      const int w = base + SAMPLE_THREADS - 1 - tid;   // reversed, so the suffix scan gives index-order offsets
      unsigned m = w < W ? pres[w] & ~ban[w] : 0u;
      int c_incl, c_excl;
      suffix_scan(__popc(m), s_int, c_incl, c_excl);
      int at = s_P + c_excl;
      for (; m; m &= m - 1) {
        const int i = w * 32 + __ffs(m) - 1;
        float y;
        value(i, y);
        if (at < PROC_LIST_MAX) list[at] = ((unsigned long long)f32_key(y) << 32) | (0xFFFFFFFFu - (unsigned)i);
        at++;
      }
      __syncthreads();
      if (tid == 0) s_P += c_incl;   // thread 0 holds the chunk total
      __syncthreads();
    }
  }
  const int P = min(s_P, PROC_LIST_MAX);
  // ---- bitonic sort of the list, descending: (value desc, index asc); zero keys pad it to a power of two
  int Pp = 1;
  while (Pp < P) Pp <<= 1;
  if (P > 1) {
    for (int i = P + tid; i < Pp; i += SAMPLE_THREADS) list[i] = 0ull;
    __syncthreads();
    for (int size = 2; size <= Pp; size <<= 1)
      for (int stride = size >> 1; stride > 0; stride >>= 1) {
        for (int i = tid; i < (Pp >> 1); i += SAMPLE_THREADS) {
          const int lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
          const unsigned long long x = list[lo], y = list[hi];
          if ((x < y) == ((lo & size) == 0)) {
            list[lo] = y;
            list[hi] = x;
          }
        }
        __syncthreads();
      }
  }
  // ---- this thread's part of the list: the entries whose values round down to its keys
  int n0 = 0, n1 = 0;
  {
    int lo = 0, hi = P;   // first entry owned by a thread <= tid
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (list_owner(list[mid]) <= tid) hi = mid; else lo = mid + 1;
    }
    n0 = lo;
    hi = P;               // first entry owned by a thread < tid
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (list_owner(list[mid]) < tid) hi = mid; else lo = mid + 1;
    }
    n1 = lo;
  }
  const unsigned key0 = (unsigned)tid * 64;
  // ---- counts; the top value
  int cnt = 0, top_c = 0;
  unsigned top_k32 = 0u;
  walk_units(hist, list, n0, n1, key0, [&](unsigned k, float, int c) {
    if (!top_c) {
      top_k32 = k;
      top_c = c;
    }
    cnt += c;
    return true;
  });
  if (top_c) atomicMax(&s_maxk, top_k32);
  int c_incl, c_excl;
  suffix_scan(cnt, s_int, c_incl, c_excl);   // its barriers publish s_maxk
  const unsigned maxk = s_maxk;
  // ---- top-k: the k-th largest processed value, counting duplicates
  if (top_k > 0 && top_k < V) {
    if (c_incl >= top_k) atomicMax(&s_find, tid);
    __syncthreads();
    if (tid == s_find) {
      int c0 = c_excl;
      walk_units(hist, list, n0, n1, key0, [&](unsigned k, float, int c) {
        c0 += c;
        if (c0 >= top_k) s_kthr = k;
        return c0 < top_k;
      });
    }
    __syncthreads();
  }
  const unsigned kthr = s_kthr;
  // ---- masses of the top-k survivors
  const float smax = __fdiv_rn(f32_of_key(maxk), temperature);
  float mass = 0.f;
  walk_units(hist, list, n0, n1, key0, [&](unsigned k, float y, int c) {
    if (k < kthr) return false;
    mass += (float)c * expf(__fdiv_rn(y, temperature) - smax);
    return true;
  });
  float m_incl, m_excl;
  suffix_scan(mass, s_flt, m_incl, m_excl);
  const float z = s_flt[0];
  // ---- top-p over the processed groups
  unsigned thr = kthr;
  if (tid == 0) s_zk = z;
  if (top_p < 1.f) {
    const float pz = top_p * z;
    __syncthreads();
    if (tid == 0) {
      s_find = SAMPLE_THREADS;
      s_pthr = maxk;   // top_p <= 0: the top value alone
    }
    if (top_c && top_k32 == maxk) s_zk = (float)top_c * expf(__fdiv_rn(f32_of_key(maxk), temperature) - smax);
    __syncthreads();
    if (top_p > 0.f && m_excl < pz) atomicMin(&s_find, tid);
    __syncthreads();
    if (tid == s_find) {
      float cum = m_excl;
      walk_units(hist, list, n0, n1, key0, [&](unsigned k, float y, int c) {
        if (k < kthr || !(cum < pz)) return false;
        cum += (float)c * expf(__fdiv_rn(y, temperature) - smax);
        s_pthr = k;
        s_zk = cum;
        return true;
      });
    }
    __syncthreads();
    thr = max(thr, s_pthr);
  }
  __syncthreads();
  // ---- inverse CDF over the kept groups, from the top; a thread with kept groups takes it when rounding leaves the
  // target past every thread's inclusive mass
  const uint4 r = philox4x32_10(make_uint4((unsigned)step, (unsigned)((unsigned long long)step >> 32), rng_row, 0u),
                                make_uint2((unsigned)seed, (unsigned)(seed >> 32)));
  const float target = (float)(r.x >> 8) * 0x1p-24f * s_zk;
  if (tid == 0) {
    s_find = -1;
    s_low = SAMPLE_THREADS;
    s_sel = 0u;   // no group at all (every id banned): no id matches, token 0
    s_j = 0;
  }
  __syncthreads();
  if (m_incl > target) atomicMax(&s_find, tid);
  if (top_c && top_k32 >= thr) atomicMin(&s_low, tid);
  __syncthreads();
  if (tid == (s_find >= 0 ? s_find : s_low)) {
    float cum = m_excl;
    unsigned last = 0u;
    int last_c = 0;
    bool hit = false;
    walk_units(hist, list, n0, n1, key0, [&](unsigned k, float y, int c) {
      if (k < thr) return false;
      const float e = expf(__fdiv_rn(y, temperature) - smax);
      const float m = (float)c * e;
      if (cum + m > target) {
        const int jj = (int)((target - cum) / e);
        s_sel = k;
        s_j = min(max(jj, 0), c - 1);
        hit = true;
        return false;
      }
      cum += m;
      last = k;
      last_c = c;
      return true;
    });
    if (!hit && last_c) {   // rounding left the target past this thread's last kept group: its last occurrence
      s_sel = last;
      s_j = last_c - 1;
    }
  }
  __syncthreads();
  // ---- the s_j-th id, in index order, whose processed value is the chosen one
  const unsigned sel = s_sel;
  const int jsel = s_j;
  int seen = 0;
  for (int base = 0; base < V; base += SAMPLE_THREADS) {
    const int i = base + tid;
    float y;
    const bool hit = i < V && value(i, y) && f32_key(y) == sel;
    const int nh = __syncthreads_count(hit);
    if (seen + nh > jsel) {
      const unsigned ball = __ballot_sync(0xffffffffu, hit);
      if (lane == 0) s_int[warp] = __popc(ball);
      __syncthreads();
      if (hit) {
        int rank = seen + __popc(ball & ((1u << lane) - 1u));
        for (int w = 0; w < warp; w++) rank += s_int[w];
        if (rank == jsel) s_tok = i;
      }
      break;
    }
    seen += nh;
  }
  if constexpr (OUT)
    write_outputs(out, row, V, step, [&](int i) {
      float y;
      return value(i, y) && f32_key(y) >= thr ? __fdiv_rn(y, temperature) : -INFINITY;
    });
}

// rng_row: the row word of the Philox counter -- blockIdx.x for a batch, 0 for the per-row kernels, whose rows each
// draw as a batch of one would.
template <bool PROC, bool OUT>
__device__ __forceinline__ void sample_row(const unsigned short* __restrict__ logits, long long ld, int V,
                                           float temperature, int top_k, float top_p, int greedy,
                                           unsigned long long seed, const long long* __restrict__ rng_step, int eos_id,
                                           int pad_id, int* __restrict__ finished, long long* __restrict__ out_ids,
                                           const SampleProc& proc, const SampleOut& out, unsigned rng_row) {
  extern __shared__ unsigned hist[];
  __shared__ unsigned long long s_best[32];
  __shared__ int s_int[32];
  __shared__ float s_flt[32];
  __shared__ int s_find, s_kthr, s_pthr, s_sel, s_j, s_tok, s_maxkey;
  __shared__ float s_zk;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned short* row = logits + (long long)b * ld;

  if constexpr (PROC) {
    select_processed<OUT>(row, V, temperature, top_k, top_p, greedy, seed, rng_step, proc, out, hist, s_tok, rng_row);
  } else if (greedy) {
    // arg-max, first index among equals (torch.argmax)
    unsigned long long best = 0;
    for (int i = tid; i < V; i += SAMPLE_THREADS) {
      const unsigned long long p = ((unsigned long long)order_key(row[i]) << 32) | (0xFFFFFFFFu - (unsigned)i);
      best = p > best ? p : best;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long n = __shfl_xor_sync(0xffffffffu, best, o);
      best = n > best ? n : best;
    }
    if (lane == 0) s_best[warp] = best;
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < 32; w++) best = s_best[w] > best ? s_best[w] : best;
      s_tok = (int)(0xFFFFFFFFu - (unsigned)best);
    }
    if constexpr (OUT) write_outputs(out, row, V, *rng_step, [&](int i) { return bits_value(row[i]); });
  } else {
    // ---- histogram of the row's bit patterns
    for (int i = tid; i < SAMPLE_SMEM_WORDS; i += SAMPLE_THREADS) hist[i] = 0u;
    if (tid == 0) {
      s_maxkey = 0;
      s_find = -1;
      s_kthr = 0;
      s_tok = 0;
    }
    __syncthreads();
    for (int i = tid; i < V; i += SAMPLE_THREADS) {
      const unsigned key = order_key(row[i]);
      atomicAdd(&hist[hist_word(key)], 1u << ((key & 1) * 16));
    }
    __syncthreads();
    const unsigned* mine = hist + tid * 33;
    const unsigned key0 = (unsigned)tid * 64;
    // ---- counts; the top key
    int cnt = 0, top = -1;
    for (int j = 31; j >= 0; j--) {
      const unsigned w = mine[j];
      if (top < 0 && w) top = (int)(key0 + 2 * j + ((w >> 16) ? 1 : 0));
      cnt += (int)(w & 0xFFFFu) + (int)(w >> 16);
    }
    if (top >= 0) atomicMax(&s_maxkey, top);
    int c_incl, c_excl;
    suffix_scan(cnt, s_int, c_incl, c_excl);   // its barriers publish s_maxkey
    const unsigned maxkey = (unsigned)s_maxkey;
    // ---- top-k: the k-th largest value, counting duplicates (TopKLogitsWarper keeps s >= it)
    if (top_k > 0 && top_k < V) {
      if (c_incl >= top_k) atomicMax(&s_find, tid);
      __syncthreads();
      if (tid == s_find) {
        int c = c_excl;
        for (int j = 63; j >= 0; j--) {
          c += (int)bin_count(hist, key0 + j);
          if (c >= top_k) {
            s_kthr = (int)(key0 + j);
            break;
          }
        }
      }
      __syncthreads();
    }
    const unsigned kthr = (unsigned)s_kthr;
    // ---- masses of the top-k survivors: count * exp(v / T - max / T), in fp32 as HF's .float() scores
    const float smax = __fdiv_rn(key_value(maxkey), temperature);
    float mass = 0.f;
    for (int j = 63; j >= 0; j--) {
      const unsigned key = key0 + j;
      const unsigned c = bin_count(hist, key);
      if (c && key >= kthr) mass += (float)c * expf(__fdiv_rn(key_value(key), temperature) - smax);
    }
    float m_incl, m_excl;
    suffix_scan(mass, s_flt, m_incl, m_excl);
    const float z = s_flt[0];   // the scan left the block total there
    // ---- top-p: keep the values whose strictly larger survivors hold less than top_p of the mass
    unsigned thr = kthr;
    if (tid == 0) s_zk = z;
    if (top_p < 1.f) {
      const float pz = top_p * z;
      if (tid == 0) {
        s_find = SAMPLE_THREADS;
        s_pthr = (int)maxkey;      // top_p <= 0: the top value alone (min_tokens_to_keep = 1)
        s_zk = (float)bin_count(hist, maxkey) * expf(__fdiv_rn(key_value(maxkey), temperature) - smax);
      }
      __syncthreads();
      if (top_p > 0.f && m_excl < pz) atomicMin(&s_find, tid);
      __syncthreads();
      if (tid == s_find) {
        float cum = m_excl;
        for (int j = 63; j >= 0; j--) {
          const unsigned key = key0 + j;
          const unsigned c = bin_count(hist, key);
          if (!c || key < kthr) continue;
          if (!(cum < pz)) break;
          cum += (float)c * expf(__fdiv_rn(key_value(key), temperature) - smax);
          s_pthr = (int)key;
          s_zk = cum;
        }
      }
      __syncthreads();
      thr = max(thr, (unsigned)s_pthr);
    }
    __syncthreads();
    // ---- inverse CDF over the kept values, from the top
    const long long step = *rng_step;
    const uint4 r = philox4x32_10(make_uint4((unsigned)step, (unsigned)((unsigned long long)step >> 32), rng_row, 0u),
                                  make_uint2((unsigned)seed, (unsigned)(seed >> 32)));
    const float target = (float)(r.x >> 8) * 0x1p-24f * s_zk;
    if (tid == 0) {
      s_find = -1;
      s_sel = (int)thr;
      s_j = (int)bin_count(hist, thr) - 1;
    }
    __syncthreads();
    if (m_incl > target) atomicMax(&s_find, tid);
    __syncthreads();
    if (tid == s_find) {
      float cum = m_excl;
      int last = -1;
      for (int j = 63; j >= 0; j--) {
        const unsigned key = key0 + j;
        const unsigned c = bin_count(hist, key);
        if (!c || key < thr) continue;
        const float e = expf(__fdiv_rn(key_value(key), temperature) - smax);
        const float m = (float)c * e;
        if (cum + m > target) {
          const int jj = (int)((target - cum) / e);
          s_sel = (int)key;
          s_j = min(max(jj, 0), (int)c - 1);
          last = -2;
          break;
        }
        cum += m;
        last = (int)key;
      }
      if (last >= 0) {   // rounding left the target past this thread's last kept value: take its last occurrence
        s_sel = last;
        s_j = (int)bin_count(hist, (unsigned)last) - 1;
      }
    }
    __syncthreads();
    // ---- the s_j-th occurrence of the chosen value, in index order
    const unsigned sel = (unsigned)s_sel;
    const int jsel = s_j;
    int seen = 0;
    for (int base = 0; base < V; base += SAMPLE_THREADS) {
      const int i = base + tid;
      const bool hit = i < V && order_key(row[i]) == sel;
      const int n = __syncthreads_count(hit);
      if (seen + n > jsel) {
        const unsigned ball = __ballot_sync(0xffffffffu, hit);
        if (lane == 0) s_int[warp] = __popc(ball);
        __syncthreads();
        if (hit) {
          int rank = seen + __popc(ball & ((1u << lane) - 1u));
          for (int w = 0; w < warp; w++) rank += s_int[w];
          if (rank == jsel) s_tok = i;
        }
        break;
      }
      seen += n;
    }
    if constexpr (OUT)
      write_outputs(out, row, V, step, [&](int i) {
        return order_key(row[i]) >= thr ? __fdiv_rn(bits_value(row[i]), temperature) : -INFINITY;
      });
  }
  __syncthreads();
  if (tid == 0) {
    long long tok = s_tok;
    if (finished && eos_id >= 0 && pad_id >= 0) {   // transformers' eos -> pad rule (GenerationMixin._sample)
      if (finished[b]) tok = pad_id;
      else if (tok == eos_id) finished[b] = 1;
    }
    out_ids[b] = tok;
    if constexpr (PROC) {   // the history the next step reads: h[b, L + step] = the token selected now
      const long long at = (long long)proc.L + *rng_step;
      if (proc.append && at < proc.ld_h) proc.hist[(long long)b * proc.ld_h + at] = tok;
    }
  }
}

template <bool PROC>
__global__ void __launch_bounds__(SAMPLE_THREADS, 1)
sample_tokens_kernel(const unsigned short* __restrict__ logits, long long ld, int V, float temperature, int top_k,
                     float top_p, int greedy, unsigned long long seed, const long long* __restrict__ rng_step,
                     int eos_id, int pad_id, int* __restrict__ finished, long long* __restrict__ out_ids,
                     SampleProc proc) {
  sample_row<PROC, false>(logits, ld, V, temperature, top_k, top_p, greedy, seed, rng_step, eos_id, pad_id, finished,
                          out_ids, proc, SampleOut{}, blockIdx.x);
}

// The same selection followed by the output pass; a separate kernel, so the selection-only kernels stay as they are.
template <bool PROC>
__global__ void __launch_bounds__(SAMPLE_THREADS, 1)
sample_tokens_out_kernel(const unsigned short* __restrict__ logits, long long ld, int V, float temperature, int top_k,
                         float top_p, int greedy, unsigned long long seed, const long long* __restrict__ rng_step,
                         int eos_id, int pad_id, int* __restrict__ finished, long long* __restrict__ out_ids,
                         SampleProc proc, SampleOut out) {
  sample_row<PROC, true>(logits, ld, V, temperature, top_k, top_p, greedy, seed, rng_step, eos_id, pad_id, finished,
                         out_ids, proc, out, blockIdx.x);
}

// The per-row processors of g4r_sample_tokens_rows_proc_*: row r's SampleProc comes from entry r of each array.
struct SampleProcRows {
  long long* hist;              // int64 [S, ld_h]: row r's submitted prompt, then its new tokens
  long long ld_h;
  const int* prompt_len;        // [S]
  const float* penalty;         // [S], 1: off
  const int* ngram;             // [S], 0: off
  const int* min_length;        // [S]
  const int* min_new_tokens;    // [S]
  const int* eos_ids;           // [S, PROC_ROW_EOS]: the ids min_length / min_new_tokens suppress
  const int* n_eos;             // [S]
};
constexpr int PROC_ROW_EOS = 4;

// The per-row kernel (g4r_sample_tokens_rows_*): the decode step of a continuous batch, whose rows are independent
// requests.  Row r runs the plain selection on its own rule, seed and counter step[r]; an inactive row returns before
// any work.  `lens` is the step's last write: the decode kernels of the same step have read it already.
// PROC (g4r_sample_tokens_rows_proc_*): a row whose processors are not all neutral runs the processed selection on its
// history h[r, 0 .. prompt_len[r] + step[r]) and appends its token there; a neutral row runs the plain body, so it
// selects bitwise as the PROC = false instance does.
template <bool PROC>
__global__ void __launch_bounds__(SAMPLE_THREADS, 1)
sample_tokens_rows_kernel(const unsigned short* __restrict__ logits, long long ld, int V, const int* __restrict__ greedy,
                          const float* __restrict__ temperature, const int* __restrict__ top_k,
                          const float* __restrict__ top_p, const unsigned long long* __restrict__ seed,
                          long long* __restrict__ step, const int* __restrict__ eos_id, const int* __restrict__ active,
                          int* __restrict__ finished, long long* __restrict__ out_ids, int* __restrict__ lens,
                          SampleProcRows rp) {
  const int r = blockIdx.x;
  if (!active[r]) return;   // uniform over the CTA
  if constexpr (PROC) {
    const SampleProc pr{rp.hist, rp.ld_h, rp.prompt_len[r], rp.penalty[r], rp.ngram[r], rp.min_length[r],
                        rp.min_new_tokens[r], rp.eos_ids + (long long)r * PROC_ROW_EOS, rp.n_eos[r], 1};
    const bool neutral = pr.penalty == 1.f && pr.ngram == 0 && !((pr.min_length || pr.min_new_tokens) && pr.n_eos);
    if (neutral)   // uniform over the CTA
      sample_row<false, false>(logits, ld, V, temperature[r], top_k[r], top_p[r], greedy[r], seed[r], step + r, -1, -1,
                               nullptr, out_ids, SampleProc{}, SampleOut{}, 0u);
    else
      sample_row<true, false>(logits, ld, V, temperature[r], top_k[r], top_p[r], greedy[r], seed[r], step + r, -1, -1,
                              nullptr, out_ids, pr, SampleOut{}, 0u);
  } else {
    sample_row<false, false>(logits, ld, V, temperature[r], top_k[r], top_p[r], greedy[r], seed[r], step + r, -1, -1,
                             nullptr, out_ids, SampleProc{}, SampleOut{}, 0u);
  }
  if (threadIdx.x == 0) {   // the thread that wrote out_ids[r] (and appended it to the history)
    const long long tok = out_ids[r];
    if (eos_id[r] >= 0 && tok == eos_id[r]) finished[r] = 1;
    step[r] += 1;
    if (lens) lens[r] += 1;
  }
}

}  // namespace G4R_NS

using namespace G4R_NS;

// The selection-only kernels (OUT false) or their output-pass instances (OUT true).
template <bool OUT>
static int launch_plain(const void* logits, long long ld, int B, int V, float temperature, int top_k, float top_p,
                        int greedy, unsigned long long seed, const long long* rng_step, int eos_id, int pad_id,
                        int* finished, long long* out_ids, SampleOut out, void* stream) {
  G4R_REQUIRE(logits && out_ids && B > 0 && V > 0 && ld >= V, "sample_tokens: bad arguments (B=%d V=%d ld=%lld)", B, V, ld);
  G4R_REQUIRE(greedy || (V < 65536 && rng_step && temperature > 0.f && top_p >= 0.f),
              "sample_tokens: sampling needs V < 65536 (16-bit bin counts), rng_step, temperature > 0 and top_p >= 0 "
              "(V=%d T=%g top_p=%g)", V, (double)temperature, (double)top_p);
  cudaStream_t st = (cudaStream_t)stream;
  static bool set = false;
  if (!set) {
    if constexpr (OUT)
      G4R_CUDA(cudaFuncSetAttribute(sample_tokens_out_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)SAMPLE_SMEM));
    else
      G4R_CUDA(cudaFuncSetAttribute(sample_tokens_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)SAMPLE_SMEM));
    set = true;
  }
  if constexpr (OUT)
    sample_tokens_out_kernel<false><<<B, SAMPLE_THREADS, greedy ? 0 : SAMPLE_SMEM, st>>>(
        (const unsigned short*)logits, ld, V, temperature, top_k, top_p, greedy, seed, rng_step, eos_id, pad_id,
        finished, out_ids, SampleProc{}, out);
  else
    sample_tokens_kernel<false><<<B, SAMPLE_THREADS, greedy ? 0 : SAMPLE_SMEM, st>>>(
        (const unsigned short*)logits, ld, V, temperature, top_k, top_p, greedy, seed, rng_step, eos_id, pad_id,
        finished, out_ids, SampleProc{});
  G4R_LAUNCH_CHECK("sample_tokens");
  return G4R_OK;
}

template <bool OUT>
static int launch_proc(const void* logits, long long ld, int B, int V, float temperature, int top_k, float top_p,
                       int greedy, unsigned long long seed, const long long* rng_step, int eos_id, int pad_id,
                       int* finished, long long* out_ids, long long* history, long long ld_h, int L,
                       float repetition_penalty, int no_repeat_ngram_size, int min_length, int min_new_tokens,
                       const int* eos_ids, int n_eos, int append, SampleOut out, void* stream) {
  G4R_REQUIRE(logits && out_ids && B > 0 && V > 0 && V < 65536 && ld >= V,
              "sample_tokens_proc: bad arguments (B=%d V=%d ld=%lld; V < 65536)", B, V, ld);
  G4R_REQUIRE(greedy || (temperature > 0.f && top_p >= 0.f),
              "sample_tokens_proc: sampling needs temperature > 0 and top_p >= 0 (T=%g top_p=%g)", (double)temperature,
              (double)top_p);
  G4R_REQUIRE(history && rng_step && L >= 0 && ld_h >= L && repetition_penalty > 0.f && no_repeat_ngram_size >= 0 &&
                  n_eos >= 0 && (n_eos == 0 || eos_ids),
              "sample_tokens_proc: bad processor arguments (L=%d ld_h=%lld penalty=%g n=%d n_eos=%d; the history and "
              "rng_step are required, penalty > 0)", L, ld_h, (double)repetition_penalty, no_repeat_ngram_size, n_eos);
  const bool listed = !greedy && repetition_penalty != 1.f;
  G4R_REQUIRE(!listed || ld_h <= PROC_LIST_MAX,
              "sample_tokens_proc: sampling with a repetition penalty holds at most %d history ids per row (ld_h=%lld)",
              PROC_LIST_MAX, ld_h);
  int list_n = 1;
  while (listed && list_n < ld_h) list_n <<= 1;
  const size_t smem = (greedy ? 0 : SAMPLE_SMEM) + 2 * sizeof(unsigned) * ((V + 31) / 32) +
                      (listed ? list_n * sizeof(unsigned long long) : 0);
  cudaStream_t st = (cudaStream_t)stream;
  static bool set = false;
  if (!set) {
    const size_t most = SAMPLE_SMEM + 2 * sizeof(unsigned) * 2048 + PROC_LIST_MAX * sizeof(unsigned long long);
    if constexpr (OUT)
      G4R_CUDA(cudaFuncSetAttribute(sample_tokens_out_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)most));
    else
      G4R_CUDA(cudaFuncSetAttribute(sample_tokens_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)most));
    set = true;
  }
  SampleProc pr{history, ld_h, L, repetition_penalty, no_repeat_ngram_size, min_length, min_new_tokens, eos_ids, n_eos,
                append};
  if constexpr (OUT)
    sample_tokens_out_kernel<true><<<B, SAMPLE_THREADS, smem, st>>>(
        (const unsigned short*)logits, ld, V, temperature, top_k, top_p, greedy, seed, rng_step, eos_id, pad_id,
        finished, out_ids, pr, out);
  else
    sample_tokens_kernel<true><<<B, SAMPLE_THREADS, smem, st>>>(
        (const unsigned short*)logits, ld, V, temperature, top_k, top_p, greedy, seed, rng_step, eos_id, pad_id,
        finished, out_ids, pr);
  G4R_LAUNCH_CHECK("sample_tokens_proc");
  return G4R_OK;
}

extern "C" int g4r_sample_tokens_bf16(const void* logits, long long ld, int B, int V, float temperature, int top_k,
                                      float top_p, int greedy, unsigned long long seed, const long long* rng_step,
                                      int eos_id, int pad_id, int* finished, long long* out_ids, void* stream) {
  return launch_plain<false>(logits, ld, B, V, temperature, top_k, top_p, greedy, seed, rng_step, eos_id, pad_id,
                             finished, out_ids, SampleOut{}, stream);
}

extern "C" int g4r_sample_tokens_rows_bf16(const void* logits, long long ld, int S, int V, const int* greedy,
                                           const float* temperature, const int* top_k, const float* top_p,
                                           const unsigned long long* seed, long long* step, const int* eos_id,
                                           const int* active, int* finished, long long* out_ids, int* lens,
                                           void* stream) {
  G4R_REQUIRE(logits && out_ids && S > 0 && V > 0 && V < 65536 && ld >= V,
              "sample_tokens_rows: bad arguments (S=%d V=%d ld=%lld; V < 65536)", S, V, ld);
  G4R_REQUIRE(greedy && temperature && top_k && top_p && seed && step && eos_id && active && finished,
              "sample_tokens_rows: every per-row array but lens is required");
  cudaStream_t st = (cudaStream_t)stream;
  static bool set = false;
  if (!set) {
    G4R_CUDA(cudaFuncSetAttribute(sample_tokens_rows_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)SAMPLE_SMEM));
    set = true;
  }
  // the sampling amount always: which rows sample is device data, and a captured launch serves every later admission
  sample_tokens_rows_kernel<false><<<S, SAMPLE_THREADS, SAMPLE_SMEM, st>>>(
      (const unsigned short*)logits, ld, V, greedy, temperature, top_k, top_p, seed, step, eos_id, active, finished,
      out_ids, lens, SampleProcRows{});
  G4R_LAUNCH_CHECK("sample_tokens_rows");
  return G4R_OK;
}

extern "C" int g4r_sample_tokens_rows_proc_bf16(const void* logits, long long ld, int S, int V, const int* greedy,
                                                const float* temperature, const int* top_k, const float* top_p,
                                                const unsigned long long* seed, long long* step, const int* eos_id,
                                                const int* active, int* finished, long long* out_ids, int* lens,
                                                long long* history, long long ld_h, const int* prompt_len,
                                                const float* repetition_penalty, const int* no_repeat_ngram_size,
                                                const int* min_length, const int* min_new_tokens, const int* eos_ids,
                                                const int* n_eos, void* stream) {
  G4R_REQUIRE(logits && out_ids && S > 0 && V > 0 && V < 65536 && ld >= V,
              "sample_tokens_rows_proc: bad arguments (S=%d V=%d ld=%lld; V < 65536)", S, V, ld);
  G4R_REQUIRE(greedy && temperature && top_k && top_p && seed && step && eos_id && active && finished,
              "sample_tokens_rows_proc: every per-row array but lens is required");
  G4R_REQUIRE(history && ld_h >= 1 && prompt_len && repetition_penalty && no_repeat_ngram_size && min_length &&
                  min_new_tokens && eos_ids && n_eos,
              "sample_tokens_rows_proc: the history (ld_h=%lld >= 1) and every per-row processor array are required",
              ld_h);
  const long long listed = ld_h < PROC_LIST_MAX ? ld_h : PROC_LIST_MAX;
  long long list_n = 1;
  while (list_n < listed) list_n <<= 1;
  // the largest amount always: which rows sample, and which carry a penalty, is device data
  const size_t smem = SAMPLE_SMEM + 2 * sizeof(unsigned) * ((V + 31) / 32) + list_n * sizeof(unsigned long long);
  cudaStream_t st = (cudaStream_t)stream;
  static bool set = false;
  if (!set) {
    const size_t most = SAMPLE_SMEM + 2 * sizeof(unsigned) * 2048 + PROC_LIST_MAX * sizeof(unsigned long long);
    G4R_CUDA(cudaFuncSetAttribute(sample_tokens_rows_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)most));
    set = true;
  }
  const SampleProcRows rp{history, ld_h, prompt_len, repetition_penalty, no_repeat_ngram_size, min_length,
                          min_new_tokens, eos_ids, n_eos};
  sample_tokens_rows_kernel<true><<<S, SAMPLE_THREADS, smem, st>>>(
      (const unsigned short*)logits, ld, V, greedy, temperature, top_k, top_p, seed, step, eos_id, active, finished,
      out_ids, lens, rp);
  G4R_LAUNCH_CHECK("sample_tokens_rows_proc");
  return G4R_OK;
}

extern "C" int g4r_sample_tokens_proc_bf16(const void* logits, long long ld, int B, int V, float temperature, int top_k,
                                           float top_p, int greedy, unsigned long long seed, const long long* rng_step,
                                           int eos_id, int pad_id, int* finished, long long* out_ids,
                                           long long* history, long long ld_h, int L, float repetition_penalty,
                                           int no_repeat_ngram_size, int min_length, int min_new_tokens,
                                           const int* eos_ids, int n_eos, int append, void* stream) {
  return launch_proc<false>(logits, ld, B, V, temperature, top_k, top_p, greedy, seed, rng_step, eos_id, pad_id,
                            finished, out_ids, history, ld_h, L, repetition_penalty, no_repeat_ngram_size, min_length,
                            min_new_tokens, eos_ids, n_eos, append, SampleOut{}, stream);
}

extern "C" int g4r_sample_tokens_out_bf16(const void* logits, long long ld, int B, int V, float temperature, int top_k,
                                          float top_p, int greedy, unsigned long long seed, const long long* rng_step,
                                          int eos_id, int pad_id, int* finished, long long* out_ids,
                                          long long* history, long long ld_h, int L, float repetition_penalty,
                                          int no_repeat_ngram_size, int min_length, int min_new_tokens,
                                          const int* eos_ids, int n_eos, int append, float* scores, float* raw_logits,
                                          long long n_slots, void* stream) {
  G4R_REQUIRE(history || (repetition_penalty == 1.f && no_repeat_ngram_size == 0 && n_eos == 0),
              "sample_tokens_out: the logits processors need the history (penalty=%g n=%d n_eos=%d)",
              (double)repetition_penalty, no_repeat_ngram_size, n_eos);
  const SampleOut out{scores, raw_logits, n_slots};
  if (!scores && !raw_logits)   // nothing to write: exactly the selection-only launch
    return history ? launch_proc<false>(logits, ld, B, V, temperature, top_k, top_p, greedy, seed, rng_step, eos_id,
                                        pad_id, finished, out_ids, history, ld_h, L, repetition_penalty,
                                        no_repeat_ngram_size, min_length, min_new_tokens, eos_ids, n_eos, append, out,
                                        stream)
                   : launch_plain<false>(logits, ld, B, V, temperature, top_k, top_p, greedy, seed, rng_step, eos_id,
                                         pad_id, finished, out_ids, out, stream);
  G4R_REQUIRE(rng_step && n_slots > 0, "sample_tokens_out: the output slot is *rng_step: rng_step and n_slots > 0 are "
              "required (n_slots=%lld)", n_slots);
  return history ? launch_proc<true>(logits, ld, B, V, temperature, top_k, top_p, greedy, seed, rng_step, eos_id, pad_id,
                                     finished, out_ids, history, ld_h, L, repetition_penalty, no_repeat_ngram_size,
                                     min_length, min_new_tokens, eos_ids, n_eos, append, out, stream)
                 : launch_plain<true>(logits, ld, B, V, temperature, top_k, top_p, greedy, seed, rng_step, eos_id,
                                      pad_id, finished, out_ids, out, stream);
}
