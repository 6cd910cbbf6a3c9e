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

__global__ void __launch_bounds__(SAMPLE_THREADS, 1)
sample_tokens_kernel(const unsigned short* __restrict__ logits, long long ld, int V, float temperature, int top_k,
                     float top_p, int greedy, unsigned long long seed, const long long* __restrict__ rng_step,
                     int eos_id, int pad_id, int* __restrict__ finished, long long* __restrict__ out_ids) {
  extern __shared__ unsigned hist[];
  __shared__ unsigned long long s_best[32];
  __shared__ int s_int[32];
  __shared__ float s_flt[32];
  __shared__ int s_find, s_kthr, s_pthr, s_sel, s_j, s_tok, s_maxkey;
  __shared__ float s_zk;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned short* row = logits + (long long)b * ld;

  if (greedy) {
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
    const uint4 r = philox4x32_10(make_uint4((unsigned)step, (unsigned)((unsigned long long)step >> 32), (unsigned)b, 0u),
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
  }
  __syncthreads();
  if (tid == 0) {
    long long tok = s_tok;
    if (finished && eos_id >= 0 && pad_id >= 0) {   // transformers' eos -> pad rule (GenerationMixin._sample)
      if (finished[b]) tok = pad_id;
      else if (tok == eos_id) finished[b] = 1;
    }
    out_ids[b] = tok;
  }
}

}  // namespace G4R_NS

using namespace G4R_NS;

extern "C" int g4r_sample_tokens_bf16(const void* logits, long long ld, int B, int V, float temperature, int top_k,
                                      float top_p, int greedy, unsigned long long seed, const long long* rng_step,
                                      int eos_id, int pad_id, int* finished, long long* out_ids, void* stream) {
  G4R_REQUIRE(logits && out_ids && B > 0 && V > 0 && ld >= V, "sample_tokens: bad arguments (B=%d V=%d ld=%lld)", B, V, ld);
  G4R_REQUIRE(greedy || (V < 65536 && rng_step && temperature > 0.f && top_p >= 0.f),
              "sample_tokens: sampling needs V < 65536 (16-bit bin counts), rng_step, temperature > 0 and top_p >= 0 "
              "(V=%d T=%g top_p=%g)", V, (double)temperature, (double)top_p);
  cudaStream_t st = (cudaStream_t)stream;
  static bool set = false;
  if (!set) {
    G4R_CUDA(cudaFuncSetAttribute(sample_tokens_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SAMPLE_SMEM));
    set = true;
  }
  sample_tokens_kernel<<<B, SAMPLE_THREADS, greedy ? 0 : SAMPLE_SMEM, st>>>(
      (const unsigned short*)logits, ld, V, temperature, top_k, top_p, greedy, seed, rng_step, eos_id, pad_id, finished,
      out_ids);
  G4R_LAUNCH_CHECK("sample_tokens");
  return G4R_OK;
}
