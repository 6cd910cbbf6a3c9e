// attention_wgmma.cu -- fused attention forward on the Hopper tensor cores (sm_90a, wgmma):
//   O = softmax(Q K^T * scale [+ causal / length mask]) V,   one CTA = 128 queries of one (batch, head)
//
// Replaces transformers' eager attention (modeling_llama.py:199-222, modeling_clip.py) that the
// reference calls for every LLaMA / CLIP layer, without materialising the [B,H,L,L] scores.
//
//   warpgroup 0, one thread  TMA producer: Q tile once, then K_j / V_j tiles (64 keys) into 2-stage rings
//                            (cp.async.bulk.tensor, 128-byte swizzle, [rows x 64 cols] atoms)
//   warpgroups 1, 2          64 query rows each:  S_j = Q K_j^T  (wgmma, both operands in smem, fp32 in registers)
//                            online softmax on the register fragment (a row lives in one quad of threads),
//                            O += P_j V_j  (wgmma with P as the register A operand, bf16; V consumed as an
//                            MN-major B operand straight from its [keys][d] layout -- no transpose pass)
// Scores stay fp32 through the softmax (see attention.cu header).
//
// CACHED mode (g4r_attention_cached_bf16): the queries are a chunk of Lc new tokens per row that continues a sequence
// held in the KV cache [B, Lmax, H*D]; its own K/V were appended to the cache before the launch, so every key comes
// from the cache.  Row b's chunk starts at position start[b] (the number of cached tokens before it) and has qlen[b]
// valid queries; query i attends over cache positions 0 .. start[b] + i.  Key blocks stay aligned to position 0.
// Output rows >= qlen[b] stay finite: rows inside a computed tile attend over the valid keys, and 128-row tiles
// wholly past qlen[b] are written as zeros.
// The last key block reads cache rows past start[b] + qlen[b], up to the next multiple of 64: those rows must hold
// finite values (masked scores give p = 0, but 0 * NaN in P.V would still poison the row), so the cache is allocated
// zero-filled.
// Through a cache-row table (fa_cached_rows_wgmma, g4r_attention_cached_rows_bf16) chunk row b reads cache row
// cache_rows[b] of a cache with any number of rows: the K/V tensor maps span all of them, and reads past the last row
// come back as zeros from the TMA unit.
#include <stdlib.h>

#include "common.cuh"
#include "ptx.cuh"
#include "act_type.cuh"   // bf16 as written; fp16 twin with -DG4R_ACT_HALF

namespace G4R_NS {

constexpr int kFaBM = 128;
constexpr int kFaBN = 64;
constexpr int kFaThreads = 384;
constexpr int kAtomBytes = 128 * 128;  // [128 rows][64 bf16] swizzle-128B atom (Q)

struct FaParams {
  __nv_bfloat16* out;
  long long ldo, bso;
  int L, H;
  float scale;
  const int* seqlens;
  float* lse;   // optional [B, H, L]: natural-log sum-exp of the scaled scores (training forward; attention_bwd reads it)
  // CACHED mode only
  int kv_L;            // Lmax: rows per batch entry in the K/V tensor maps
  const int* start;    // [B] first position of each row's chunk
  const int* qlen;     // [B] valid queries of each row's chunk, or NULL (all L)
};

__device__ __forceinline__ uint32_t pack_act2(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

template <int D>
__device__ __forceinline__ void wgmma_pv(float (&o)[D / 2], const uint32_t (&a)[4], uint64_t db) {
  if constexpr (D == 128) ptx::wgmma_m64n128_rs<1>(o, a, db, 1);
  else ptx::wgmma_m64n64_rs<1>(o, a, db, 1);
}

// The kernel body, shared by fa_fwd_wgmma and fa_cached_rows_wgmma.  ROWS (CACHED only): chunk row b reads cache row
// cache_rows[b] of K/V tensor maps that span every row of the cache, instead of row b.
template <int D, bool CAUSAL, bool CACHED, bool ROWS>
__device__ __forceinline__ void fa_fwd_body(const CUtensorMap& tm_q, const CUtensorMap& tm_k, const CUtensorMap& tm_v,
                                            const FaParams& p, const int* cache_rows) {
  constexpr int ATOMS = D / 64;
  constexpr int Q_BYTES = ATOMS * kAtomBytes;     // Q tile: 128 rows x D
  constexpr int KV_ATOM = kFaBN * 128;            // [BN keys][64 bf16]
  constexpr int TILE_BYTES = ATOMS * KV_ATOM;     // K / V tile: BN rows x D
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + Q_BYTES;          // 2 stages
  uint8_t* sV = sK + 2 * TILE_BYTES;   // 2 stages
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + 2 * TILE_BYTES);
  uint64_t* q_full = bars;           // 1
  uint64_t* k_full = bars + 1;       // 2
  uint64_t* k_empty = bars + 3;      // 2
  uint64_t* v_full = bars + 5;       // 2
  uint64_t* v_empty = bars + 7;      // 2

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // heaviest query blocks first (causal: block i attends to i+1 key blocks): the long CTAs start early and the
  // short ones fill the tail of the last wave (LPT order)
  const int qb = CAUSAL ? (int)(gridDim.x - 1 - blockIdx.x) : (int)blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int q0 = qb * kFaBM;
  const int row_base = b * p.L;
  int kv_base = row_base, koff = 0, Lk, nblk;
  if constexpr (CACHED) {
    // causal in cache coordinates: query i of the chunk sits at position koff + i
    const int ql = p.qlen ? min(max(p.qlen[b], 1), p.L) : p.L;
    if (q0 >= ql) {
      // whole tile past the valid rows: no work, but its outputs are zeroed -- the engine feeds them on through wo
      // into the next layer's K/V, which later chunks read masked (p = 0) and need finite
      const int rows = min(kFaBM, p.L - q0);
      for (int i = threadIdx.x; i < rows * (D / 8); i += kFaThreads)
        *reinterpret_cast<uint4*>(p.out + (long long)b * p.bso + (long long)(q0 + i / (D / 8)) * p.ldo +
                                  (long long)h * D + (i % (D / 8)) * 8) = make_uint4(0, 0, 0, 0);
      return;
    }
    kv_base = (ROWS ? cache_rows[b] : b) * p.kv_L;
    koff = p.start[b];
    Lk = koff + min(q0 + kFaBM, ql);
    nblk = (Lk + kFaBN - 1) / kFaBN;
  } else {
    Lk = p.seqlens ? min(max(p.seqlens[b], 1), p.L) : p.L;
    nblk = CAUSAL ? min((Lk + kFaBN - 1) / kFaBN, (q0 + kFaBM + kFaBN - 1) / kFaBN) : (Lk + kFaBN - 1) / kFaBN;
  }

  if (threadIdx.x == 0) {
    ptx::prefetch_tensormap(&tm_q);
    ptx::prefetch_tensormap(&tm_k);
    ptx::prefetch_tensormap(&tm_v);
    ptx::mbar_init(q_full, 1);
    for (int i = 0; i < 2; i++) {
      ptx::mbar_init(&k_full[i], 1);
      ptx::mbar_init(&k_empty[i], 2);  // one arrival per consumer warpgroup
      ptx::mbar_init(&v_full[i], 1);
      ptx::mbar_init(&v_empty[i], 2);
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  if (warp == 0) {
    // ============================ TMA producer ============================
    if (lane == 0) {
      ptx::mbar_arrive_expect_tx(q_full, Q_BYTES);
      for (int a = 0; a < ATOMS; a++)
        ptx::tma_load_2d(sQ + a * kAtomBytes, &tm_q, q_full, h * D + a * 64, row_base + q0);
      for (int j = 0; j < nblk; j++) {
        const int st = j & 1;
        const uint32_t ph = (j >> 1) & 1;
        ptx::mbar_wait(&k_empty[st], ph ^ 1);
        ptx::mbar_arrive_expect_tx(&k_full[st], TILE_BYTES);
        for (int a = 0; a < ATOMS; a++)
          ptx::tma_load_2d(sK + st * TILE_BYTES + a * KV_ATOM, &tm_k, &k_full[st], h * D + a * 64,
                           kv_base + j * kFaBN);
        ptx::mbar_wait(&v_empty[st], ph ^ 1);
        ptx::mbar_arrive_expect_tx(&v_full[st], TILE_BYTES);
        for (int a = 0; a < ATOMS; a++)
          ptx::tma_load_2d(sV + st * TILE_BYTES + a * KV_ATOM, &tm_v, &v_full[st], h * D + a * 64,
                           kv_base + j * kFaBN);
      }
    }
    return;
  }
  if (threadIdx.x < kFaThreads - 256) return;  // rest of the producer warpgroup

  // ============================ consumers ============================
  const int ct = threadIdx.x - (kFaThreads - 256);
  const int wg = ct >> 7, wt = ct & 127;
  const int quad = lane & 3;
  // this thread's two query rows (accumulator fragment rows r and r + 8 of the warpgroup's 64)
  const int qrow0 = q0 + wg * 64 + (wt >> 5) * 16 + (lane >> 2), qrow1 = qrow0 + 8;
  const int wg_q0 = q0 + wg * 64;
  const float c = p.scale * 1.4426950408889634f;
  float o[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; i++) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  ptx::mbar_wait(q_full, 0);
  for (int j = 0; j < nblk; j++) {
    const int st = j & 1;
    const uint32_t ph = (j >> 1) & 1;
    // ---- S = Q K_j^T  (64 x 64 per warpgroup)
    float s[kFaBN / 2];
    ptx::mbar_wait(&k_full[st], ph);
    ptx::wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < D / 16; kk++) {
      const uint64_t da = ptx::gmma_desc_sw128(ptx::smem_u32(sQ + (kk >> 2) * kAtomBytes + wg * 8192)) + 2 * (kk & 3);
      const uint64_t db = ptx::gmma_desc_sw128(ptx::smem_u32(sK + st * TILE_BYTES + (kk >> 2) * KV_ATOM)) + 2 * (kk & 3);
      ptx::wgmma_m64n64_ss<0, 0>(s, da, db, kk != 0);
    }
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();
    ptx::fence_regs(s);
    if (wt == 0) ptx::mbar_arrive(&k_empty[st]);
    // ---- mask, row max (a row's 64 scores are spread over the 4 threads of a quad)
    const int key0 = j * kFaBN;
    const bool need_mask = (key0 + kFaBN > Lk) || (CAUSAL && key0 + kFaBN - 1 > koff + wg_q0);
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < kFaBN / 2; i++) {
      const int hr = (i >> 1) & 1;
      if (need_mask) {
        const int key = key0 + (i >> 2) * 8 + 2 * quad + (i & 1);
        if (key >= Lk || (CAUSAL && key > koff + (hr ? qrow1 : qrow0))) s[i] = -INFINITY;
      }
      mx[hr] = fmaxf(mx[hr], s[i]);
    }
    float alpha[2], mc[2];
#pragma unroll
    for (int hr = 0; hr < 2; hr++) {
      mx[hr] = fmaxf(mx[hr], __shfl_xor_sync(0xffffffffu, mx[hr], 1));
      mx[hr] = fmaxf(mx[hr], __shfl_xor_sync(0xffffffffu, mx[hr], 2));
      const float m_new = fmaxf(m_run[hr], mx[hr]);
      alpha[hr] = m_new == -INFINITY ? 1.f : exp2f((m_run[hr] - m_new) * c);  // m_run = -inf -> 0
      m_run[hr] = m_new;
      mc[hr] = (m_new == -INFINITY ? 0.f : m_new) * c;
    }
    // ---- exponentials: fp32 row sums, 16-bit P in the register A-operand layout of the PV product
    uint32_t pa[kFaBN / 16][4];
    float lsum[2] = {0.f, 0.f};
#pragma unroll
    for (int kc = 0; kc < kFaBN / 16; kc++) {
#pragma unroll
      for (int t = 0; t < 4; t++) {   // t: (n8 block 2kc + t/2, row half t%2)
        const int i = kc * 8 + (t >> 1) * 4 + (t & 1) * 2;
        const float p0 = exp2f(fmaf(s[i], c, -mc[t & 1]));
        const float p1 = exp2f(fmaf(s[i + 1], c, -mc[t & 1]));
        lsum[t & 1] += p0 + p1;
        pa[kc][t] = pack_act2(p0, p1);
      }
    }
    l_run[0] = l_run[0] * alpha[0] + lsum[0];
    l_run[1] = l_run[1] * alpha[1] + lsum[1];
#pragma unroll
    for (int i = 0; i < D / 2; i++) o[i] *= alpha[(i >> 1) & 1];
    // ---- O += P V_j
    ptx::mbar_wait(&v_full[st], ph);
    ptx::wgmma_fence();
#pragma unroll
    for (int kc = 0; kc < kFaBN / 16; kc++)
      wgmma_pv<D>(o, pa[kc], ptx::gmma_desc_sw128(ptx::smem_u32(sV + st * TILE_BYTES + kc * 2048), KV_ATOM));
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();
    ptx::fence_regs(o);
    if (wt == 0) ptx::mbar_arrive(&v_empty[st]);
  }
  // ---- epilogue: O / l -> bf16 -> global
#pragma unroll
  for (int hr = 0; hr < 2; hr++) {
    l_run[hr] += __shfl_xor_sync(0xffffffffu, l_run[hr], 1);
    l_run[hr] += __shfl_xor_sync(0xffffffffu, l_run[hr], 2);
  }
#pragma unroll
  for (int hr = 0; hr < 2; hr++) {
    const int qrow = hr ? qrow1 : qrow0;
    if (qrow >= p.L) continue;
    const float inv = 1.f / l_run[hr];
    // p = 2^((s - m) c) = e^(scale (s - m))  =>  lse = scale m + ln l
    if (p.lse != nullptr && quad == 0)
      p.lse[((long long)b * p.H + h) * p.L + qrow] = (m_run[hr] == -INFINITY ? 0.f : m_run[hr]) * p.scale + logf(l_run[hr]);
    __nv_bfloat16* orow = p.out + (long long)b * p.bso + (long long)qrow * p.ldo + (long long)h * D;
#pragma unroll
    for (int jd = 0; jd < D / 8; jd++)
      *reinterpret_cast<uint32_t*>(orow + jd * 8 + 2 * quad) = pack_act2(o[4 * jd + 2 * hr] * inv, o[4 * jd + 2 * hr + 1] * inv);
  }
}

template <int D, bool CAUSAL, bool CACHED = false>
__global__ void __launch_bounds__(kFaThreads, 1)
fa_fwd_wgmma(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
             const __grid_constant__ CUtensorMap tm_v, const __grid_constant__ FaParams p) {
  fa_fwd_body<D, CAUSAL, CACHED, false>(tm_q, tm_k, tm_v, p, nullptr);
}

// CACHED mode through a cache-row table (g4r_attention_cached_rows_bf16): chunk row b continues the sequence held in
// cache row cache_rows[b] (device int32 [B]) of a [rows, kv_L, H*D] cache.
template <int D>
__global__ void __launch_bounds__(kFaThreads, 1)
fa_cached_rows_wgmma(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                     const __grid_constant__ CUtensorMap tm_v, const __grid_constant__ FaParams p,
                     const int* __restrict__ cache_rows) {
  fa_fwd_body<D, true, true, true>(tm_q, tm_k, tm_v, p, cache_rows);
}

typedef CUresult (*EncodeTiledFn2)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                   CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                   CUtensorMapFloatOOBfill);

static int make_tmap_rows(CUtensorMap* m, const void* base, long long cols, long long rows, long long ld,
                          int box_rows) {
  static EncodeTiledFn2 enc = nullptr;
  if (!enc) {
    void* fp = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess) {
      set_error("cuTensorMapEncodeTiled unavailable");
      return G4R_ECUDA;
    }
    enc = reinterpret_cast<EncodeTiledFn2>(fp);
  }
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t str[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, str, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("attention: cuTensorMapEncodeTiled failed (CUresult %d)", (int)r);
    return G4R_ECUDA;
  }
  return G4R_OK;
}

template <int D>
constexpr int fa_smem_bytes() { return (D / 64) * kAtomBytes + 4 * (D / 64) * kFaBN * 128 + 128 + 1024; }  // +1024 alignment slack

template <int D, bool CAUSAL, bool CACHED = false>
static int launch_fa(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const FaParams& p, int B,
                     cudaStream_t st) {
  constexpr int smem = fa_smem_bytes<D>();
  static bool set = false;
  auto kern = fa_fwd_wgmma<D, CAUSAL, CACHED>;
  if (!set) {
    G4R_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    set = true;
  }
  dim3 grid((p.L + kFaBM - 1) / kFaBM, p.H, B);
  kern<<<grid, kFaThreads, smem, st>>>(tq, tk, tv, p);
  G4R_LAUNCH_CHECK("fa_fwd_wgmma");
  return G4R_OK;
}

template <int D>
static int launch_fa_rows(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const FaParams& p,
                          const int* cache_rows, int B, cudaStream_t st) {
  constexpr int smem = fa_smem_bytes<D>();
  static bool set = false;
  auto kern = fa_cached_rows_wgmma<D>;
  if (!set) {
    G4R_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    set = true;
  }
  dim3 grid((p.L + kFaBM - 1) / kFaBM, p.H, B);
  kern<<<grid, kFaThreads, smem, st>>>(tq, tk, tv, p, cache_rows);
  G4R_LAUNCH_CHECK("fa_cached_rows_wgmma");
  return G4R_OK;
}

}  // namespace g4r

using namespace G4R_NS;

// Same contract as g4r_attention_bf16 (attention.cu), with the restriction that q/k/v are contiguous in
// the batch dimension (bs == L*ld: the packed [B*L, width] QKV buffer), which the TMA descriptors need.
static int attention_tc_impl(const void* q, const void* k, const void* v, void* out, long long ld,
                             long long bs, long long ldo, long long bso, int B, int H, int L,
                             int head_dim, int causal, float scale, const int* seqlens, float* lse, void* stream) {
  G4R_REQUIRE(q && k && v && out && B > 0 && H > 0 && L > 0, "attention_tc: bad arguments");
  G4R_REQUIRE(head_dim == 64 || head_dim == 128, "attention_tc: head_dim %d (64 or 128)", head_dim);
  G4R_REQUIRE(bs == (long long)L * ld, "attention_tc: q/k/v must be one packed [B*L, width] buffer (bs == L*ld)");
  G4R_REQUIRE(ld % 8 == 0 && ldo % 8 == 0 && bso % 8 == 0, "attention_tc: strides must keep 16-byte alignment");
  G4R_REQUIRE((((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)out) & 15) == 0, "attention_tc: misaligned pointers");
  CUtensorMap tq, tk, tv;
  const long long cols = (long long)H * head_dim, rows = (long long)B * L;
  int rc;
  if ((rc = make_tmap_rows(&tq, q, cols, rows, ld, kFaBM))) return rc;
  if ((rc = make_tmap_rows(&tk, k, cols, rows, ld, kFaBN))) return rc;
  if ((rc = make_tmap_rows(&tv, v, cols, rows, ld, kFaBN))) return rc;
  FaParams p{(__nv_bfloat16*)out, ldo, bso, L, H, scale, seqlens, lse, 0, nullptr, nullptr};
  cudaStream_t st = (cudaStream_t)stream;
#define G4R_FA(DD) (causal ? launch_fa<DD, true>(tq, tk, tv, p, B, st) : launch_fa<DD, false>(tq, tk, tv, p, B, st))
  if (head_dim == 64) return G4R_FA(64);
  return G4R_FA(128);
#undef G4R_FA
}

extern "C" int g4r_attention_tc_bf16(const void* q, const void* k, const void* v, void* out, long long ld,
                                     long long bs, long long ldo, long long bso, int B, int H, int L,
                                     int head_dim, int causal, float scale, const int* seqlens, void* stream) {
  return attention_tc_impl(q, k, v, out, ld, bs, ldo, bso, B, H, L, head_dim, causal, scale, seqlens, nullptr, stream);
}

// Training forward on the wgmma kernel: additionally writes lse[B, H, L] (fp32, natural log) for g4r_attention_bwd_bf16.
#if G4R_BF16_ONLY   // training-step only: no fp16 twin
extern "C" int g4r_attention_tc_lse_bf16(const void* q, const void* k, const void* v, void* out, long long ld,
                                         long long bs, long long ldo, long long bso, int B, int H, int L,
                                         int head_dim, int causal, float scale, float* lse, void* stream) {
  G4R_REQUIRE(lse, "attention_tc_lse: lse is NULL");
  return attention_tc_impl(q, k, v, out, ld, bs, ldo, bso, B, H, L, head_dim, causal, scale, nullptr, lse, stream);
}
#endif

// Chunk attention over the KV cache (multi-turn generation): q is the chunk's packed, RoPE-rotated [B*Lc, >= H*D] rows
// (row stride ldq), kcache / vcache the [B, lmax, H*D] caches the chunk's own K/V were already appended to, start /
// qlen device int32 [B] (qlen may be NULL: every row has Lc valid queries).  See the CACHED note at the top.
extern "C" int g4r_attention_cached_bf16(const void* q, long long ldq, const void* kcache, const void* vcache, int lmax,
                                         void* out, long long ldo, int B, int H, int Lc, int head_dim, float scale,
                                         const int* start, const int* qlen, void* stream) {
  G4R_REQUIRE(q && kcache && vcache && out && start && B > 0 && H > 0 && Lc > 0 && lmax > 0,
              "attention_cached: bad arguments");
  G4R_REQUIRE(head_dim == 64 || head_dim == 128, "attention_cached: head_dim %d (64 or 128)", head_dim);
  G4R_REQUIRE(ldq % 8 == 0 && ldo % 8 == 0, "attention_cached: strides must keep 16-byte alignment");
  G4R_REQUIRE((((uintptr_t)q | (uintptr_t)kcache | (uintptr_t)vcache | (uintptr_t)out) & 15) == 0,
              "attention_cached: misaligned pointers");
  CUtensorMap tq, tk, tv;
  const long long cols = (long long)H * head_dim;
  int rc;
  if ((rc = make_tmap_rows(&tq, q, cols, (long long)B * Lc, ldq, kFaBM))) return rc;
  if ((rc = make_tmap_rows(&tk, kcache, cols, (long long)B * lmax, cols, kFaBN))) return rc;
  if ((rc = make_tmap_rows(&tv, vcache, cols, (long long)B * lmax, cols, kFaBN))) return rc;
  FaParams p{(__nv_bfloat16*)out, ldo, (long long)Lc * ldo, Lc, H, scale, nullptr, nullptr, lmax, start, qlen};
  cudaStream_t st = (cudaStream_t)stream;
  if (head_dim == 64) return launch_fa<64, true, true>(tq, tk, tv, p, B, st);
  return launch_fa<128, true, true>(tq, tk, tv, p, B, st);
}

// g4r_attention_cached_bf16 through a cache-row table (continuous batching: several chunks continue sequences held in
// rows of the batcher's cache that need not be adjacent): kcache / vcache are [rows, lmax, H*D]; chunk row b's keys and
// values come from cache row cache_rows[b] (device int32 [B], each < rows).  Same CACHED rules otherwise.
extern "C" int g4r_attention_cached_rows_bf16(const void* q, long long ldq, const void* kcache, const void* vcache,
                                              int rows, int lmax, void* out, long long ldo, int B, int H, int Lc,
                                              int head_dim, float scale, const int* start, const int* qlen,
                                              const int* cache_rows, void* stream) {
  G4R_REQUIRE(q && kcache && vcache && out && start && cache_rows && B > 0 && H > 0 && Lc > 0 && lmax > 0 && rows > 0,
              "attention_cached_rows: bad arguments");
  G4R_REQUIRE(head_dim == 64 || head_dim == 128, "attention_cached_rows: head_dim %d (64 or 128)", head_dim);
  G4R_REQUIRE(ldq % 8 == 0 && ldo % 8 == 0, "attention_cached_rows: strides must keep 16-byte alignment");
  G4R_REQUIRE((((uintptr_t)q | (uintptr_t)kcache | (uintptr_t)vcache | (uintptr_t)out) & 15) == 0,
              "attention_cached_rows: misaligned pointers");
  CUtensorMap tq, tk, tv;
  const long long cols = (long long)H * head_dim;
  int rc;
  if ((rc = make_tmap_rows(&tq, q, cols, (long long)B * Lc, ldq, kFaBM))) return rc;
  if ((rc = make_tmap_rows(&tk, kcache, cols, (long long)rows * lmax, cols, kFaBN))) return rc;
  if ((rc = make_tmap_rows(&tv, vcache, cols, (long long)rows * lmax, cols, kFaBN))) return rc;
  FaParams p{(__nv_bfloat16*)out, ldo, (long long)Lc * ldo, Lc, H, scale, nullptr, nullptr, lmax, start, qlen};
  cudaStream_t st = (cudaStream_t)stream;
  if (head_dim == 64) return launch_fa_rows<64>(tq, tk, tv, p, cache_rows, B, st);
  return launch_fa_rows<128>(tq, tk, tv, p, cache_rows, B, st);
}
