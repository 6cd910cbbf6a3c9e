// decode.cu -- KV-cache append and single-query attention for the decode loop behind generate()
// (SURVEY.md 8(f1)): after the region-token prefill, every further step is plain LLaMA with one new
// token per sample (the vision/SPI branch is skipped, gpt4roi/models/spi_llava.py:47-48;
// llava/model/llava.py:263-283 prepare_inputs_for_generation; gpt4roi/app.py:293-300).
// Both kernels are HBM-bound: the step streams the whole KV cache of the batch once.  Both take either one position
// for the whole batch (launch argument or device scalar) or one per sample (pos_rows, device int32 [B]: a batch of
// prompts of different lengths, right-padded, each continuing from its own length).
#include "common.cuh"
#include <cooperative_groups.h>
#include "act_type.cuh"   // bf16 as written; fp16 twin with -DG4R_ACT_HALF

namespace G4R_NS {

// rows [B*Ln, 3*HD] packed (q|k|v) -> caches [B, Lmax, HD] at positions pos0 .. pos0+Ln-1, or with pos_rows (a batch
// of prompts of different lengths) sample b's rows at pos_rows[b] .. pos_rows[b]+Ln-1
__global__ void __launch_bounds__(256)
kv_append_bf16(const __nv_bfloat16* __restrict__ qkv, long long ld, __nv_bfloat16* __restrict__ kc,
               __nv_bfloat16* __restrict__ vc, int B, int Ln, int pos0, const int* __restrict__ pos_dev,
               const int* __restrict__ pos_rows, int Lmax, int HD) {
  if (pos_dev) pos0 = *pos_dev;
  const int nvec = HD >> 3;
  const long long total = (long long)B * Ln * nvec * 2;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % nvec);
    const int which = (int)((i / nvec) & 1);  // 0 = k, 1 = v
    const long long r = i / (2LL * nvec);     // row in [0, B*Ln)
    const int t = (int)(r % Ln), b = (int)(r / Ln);
    const int p0 = pos_rows ? pos_rows[b] : pos0;
    const uint4 val = *reinterpret_cast<const uint4*>(qkv + r * ld + (long long)(1 + which) * HD + v * 8);
    __nv_bfloat16* dst = (which ? vc : kc) + ((long long)b * Lmax + p0 + t) * HD + v * 8;
    *reinterpret_cast<uint4*>(dst) = val;
  }
}

// rows [B*Ln, 3*HD] packed (q|k|v) -> caches [rows, Lmax, HD] through a cache-row table: chunk row b's first qlen[b]
// rows go to cache row cache_rows[b] at positions pos_rows[b] .. pos_rows[b]+qlen[b]-1; its padding rows are not
// written, and no write leaves the row (positions >= Lmax are dropped; the caller checks pos_rows[b] + qlen[b] <= Lmax)
__global__ void __launch_bounds__(256)
kv_append_rows_at_bf16(const __nv_bfloat16* __restrict__ qkv, long long ld, __nv_bfloat16* __restrict__ kc,
                       __nv_bfloat16* __restrict__ vc, int B, int Ln, const int* __restrict__ pos_rows,
                       const int* __restrict__ cache_rows, const int* __restrict__ qlen, int Lmax, int HD) {
  const int nvec = HD >> 3;
  const long long total = (long long)B * Ln * nvec * 2;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % nvec);
    const int which = (int)((i / nvec) & 1);  // 0 = k, 1 = v
    const long long r = i / (2LL * nvec);     // row in [0, B*Ln)
    const int t = (int)(r % Ln), b = (int)(r / Ln);
    const int pos = pos_rows[b] + t;
    if (t >= qlen[b] || pos >= Lmax) continue;
    const uint4 val = *reinterpret_cast<const uint4*>(qkv + r * ld + (long long)(1 + which) * HD + v * 8);
    __nv_bfloat16* dst = (which ? vc : kc) + ((long long)cache_rows[b] * Lmax + pos) * HD + v * 8;
    *reinterpret_cast<uint4*>(dst) = val;
  }
}

// Single-query attention over the KV cache: out = softmax(q . K^T * scale) V for the first kv_len
// cached positions.  Grid (H, B, S) with a thread-block cluster of S CTAs along z: each CTA of the
// cluster owns a contiguous slice of the keys (split-KV), and the softmax statistics and the partial
// outputs are combined through distributed shared memory -- no workspace, no atomics, and a fixed
// summation order (bitwise reproducible).  S is chosen so that even batch 1 (32 heads) fills the GPU.
// 256 threads; a half-warp owns one key/value row (16 lanes x 16 bytes = the 256-byte row, coalesced).
// Rounding as the reference's eager attention: fp32 softmax, probabilities cast to bf16 before P.V.
// pos_rows (prompts of different lengths): sample b attends over its own pos_rows[b] + 1 keys.  S and the score buffer
// still come from the host's bound kv_len (>= every row's length); each row slices its own keys into S parts, so a CTA
// of a short row may own no key at all -- it still joins every cluster barrier and contributes -inf to the max and 0 to
// the sum and to the output.  All rows equal: the slicing, and so the result, is the scalar kernel's.
// BEAM (beam search, pos_rows given): the caches are shared by every row, and key / value p of row b is read from cache
// row anc[b, p] (anc: int32 [rows, Lmax]) instead of row b.  A half-warp still loads one 256-byte row per key; the
// 16 lanes read the same anc entry.  Without BEAM `anc` is unused and the code is the non-beam kernel's.
template <int D, bool BEAM = false>
__global__ void __launch_bounds__(256)
decode_attention_bf16(const __nv_bfloat16* q, long long ldq, const __nv_bfloat16* kc, const __nv_bfloat16* vc,
                      __nv_bfloat16* out, long long ldo, int H, int kv_len, const int* __restrict__ pos_dev,
                      const int* __restrict__ pos_rows, int Lmax, float scale, int per_max,
                      const int* __restrict__ anc) {
  // Programmatic dependent launch (common.cuh): q and the newest K/V row come from the q|k|v GEMM that precedes this
  // kernel in the decode step, so there is nothing to fetch ahead; the launch itself and the prologue overlap its tail.
  // q / kc / vc carry no __restrict__: their loads must stay on the coherent path.
  pdl_sync();
  static_assert(D == 128 || D == 64, "head_dim");
  constexpr int LPR = D / 8;          // lanes per row (16 or 8)
  constexpr int RPW = 32 / LPR;       // rows per warp instruction (2 or 4)
  constexpr int GROUPS = 8 * RPW;     // row groups per CTA (16 or 32)
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  const int S = (int)cluster.num_blocks(), rank = (int)cluster.block_rank();
  if (pos_rows) kv_len = pos_rows[blockIdx.y] + 1;
  else if (pos_dev) kv_len = *pos_dev + 1;
  extern __shared__ float sm[];
  float* sc = sm;                       // [per_max] scores / probabilities of this CTA's slice
  float* part = sm + per_max;           // [GROUPS][D] partial outputs, then [D] CTA total in part[0..D)
  __shared__ float red[8];
  __shared__ float cl_max, cl_sum;      // this CTA's slice statistics, read by the cluster peers
  const int h = blockIdx.x, b = blockIdx.y;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int sub = lane % LPR, grp = warp * RPW + lane / LPR;
  const int HD = H * D;
  const int per = (kv_len + S - 1) / S;
  const int k0 = rank * per;
  const int n_loc = max(0, min(kv_len, k0 + per) - k0);

  float qf[8];
  {
    const uint4 raw = *reinterpret_cast<const uint4*>(q + (long long)b * ldq + (long long)h * D + sub * 8);
    const __nv_bfloat162* hh = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const float2 f = __bfloat1622float2(hh[j]);
      qf[2 * j] = f.x * scale;
      qf[2 * j + 1] = f.y * scale;
    }
  }
  // ---- phase 1: scores of the slice
  // row offset of local key `key` (BEAM: the cache row its ancestry table names)
  const long long kv0 = BEAM ? (long long)k0 * HD : ((long long)b * Lmax + k0) * HD;
  const int* arow = BEAM ? anc + (long long)b * Lmax + k0 : nullptr;
  auto key_off = [&](int key) -> long long {
    if constexpr (BEAM) return ((long long)arow[key] * Lmax + key) * HD;
    else return (long long)key * HD;
  };
  const __nv_bfloat16* kb = kc + kv0 + (long long)h * D + sub * 8;
  float mx = -INFINITY;
  for (int base = 0; base < n_loc; base += GROUPS * 4) {
    uint4 raw[4];
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const int key = base + u * GROUPS + grp;
      raw[u] = key < n_loc ? *reinterpret_cast<const uint4*>(kb + key_off(key)) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const __nv_bfloat162* hh = reinterpret_cast<const __nv_bfloat162*>(&raw[u]);
      float acc = 0.f;
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const float2 f = __bfloat1622float2(hh[j]);
        acc += f.x * qf[2 * j] + f.y * qf[2 * j + 1];
      }
#pragma unroll
      for (int o = LPR / 2; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      const int key = base + u * GROUPS + grp;
      if (key < n_loc) {
        if (sub == 0) sc[key] = acc;
        mx = fmaxf(mx, acc);
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if (lane == 0) red[warp] = mx;
  __syncthreads();
  if (tid == 0) {
    float m = red[0];
#pragma unroll
    for (int w = 1; w < 8; w++) m = fmaxf(m, red[w]);
    cl_max = m;
  }
  cluster.sync();
  float gmax = -INFINITY;
  for (int r = 0; r < S; r++) gmax = fmaxf(gmax, *cluster.map_shared_rank(&cl_max, r));
  float sum = 0.f;
  for (int key = tid; key < n_loc; key += 256) {
    const float p = __expf(sc[key] - gmax);
    sc[key] = p;
    sum += p;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if (lane == 0) red[warp] = sum;
  __syncthreads();
  if (tid == 0) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; w++) t += red[w];
    cl_sum = t;
  }
  cluster.sync();
  float gsum = 0.f;
  for (int r = 0; r < S; r++) gsum += *cluster.map_shared_rank(&cl_sum, r);
  const float inv = 1.f / gsum;
  // ---- phase 2: partial P.V of the slice (probabilities rounded to bf16 like P.to(q.dtype))
  const __nv_bfloat16* vb = vc + kv0 + (long long)h * D + sub * 8;
  float o8[8];
#pragma unroll
  for (int j = 0; j < 8; j++) o8[j] = 0.f;
  for (int base = 0; base < n_loc; base += GROUPS * 4) {
    uint4 raw[4];
    float pk[4];
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const int key = base + u * GROUPS + grp;
      const bool ok = key < n_loc;
      raw[u] = ok ? *reinterpret_cast<const uint4*>(vb + key_off(key)) : make_uint4(0, 0, 0, 0);
      pk[u] = ok ? __bfloat162float(__float2bfloat16_rn(sc[key] * inv)) : 0.f;
    }
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const __nv_bfloat162* hh = reinterpret_cast<const __nv_bfloat162*>(&raw[u]);
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const float2 f = __bfloat1622float2(hh[j]);
        o8[2 * j] += pk[u] * f.x;
        o8[2 * j + 1] += pk[u] * f.y;
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; j++) part[grp * D + sub * 8 + j] = o8[j];
  __syncthreads();
  float tot = 0.f;
  if (tid < D) {
#pragma unroll 4
    for (int g2 = 0; g2 < GROUPS; g2++) tot += part[g2 * D + tid];
  }
  __syncthreads();
  if (tid < D) part[tid] = tot;   // CTA total, visible to rank 0 after the cluster barrier
  cluster.sync();
  if (rank == 0 && tid < D) {
    float v = 0.f;
    for (int r = 0; r < S; r++) v += cluster.map_shared_rank(part, r)[tid];
    out[(long long)b * ldo + (long long)h * D + tid] = __float2bfloat16_rn(v);
  }
  cluster.sync();   // keep every CTA's shared memory alive until rank 0 has read it
}

// Shared-prefix ("cascade") decode attention for several sampled answers per prompt (generate(num_return_sequences=N,
// do_sample=True), engine.SampleCache).  Cache layout [B + B*N, Lmax, HD]: rows 0..B-1 hold the prompts, row B + r the
// generated positions of query row r = b*N + i.  Row r attends over positions 0..prompt_lens[b]-1 of prompt row b and
// prompt_lens[b]..pos_rows[r] of its own row.  Grid (H, B, S), a cluster of S CTAs along z as in decode_attention_bf16:
// CTA (h, b, rank) owns slice `rank` of prompt b's keys and slice `rank` of each of the N rows' own keys, so every
// prompt key / value row is fetched from HBM by one CTA and used there by all N queries (the N reads hit L1 / L2).
// 16 lane groups of 16 lanes (a lane holds 8 of the 128 features, as above); lane group g serves query g / KS and
// every KS-th key of that query's local keys (KS = 16 / N): QK^T and P.V on the CUDA cores, q and the partial output
// in registers.  One max and one sum per query over all its keys; the statistics and partial outputs combine across
// the cluster through distributed shared memory in rank order.  No atomics: bitwise repeatable.
// An empty slice (a prompt shorter than S keys, a row with no generated key yet) still joins every barrier.
constexpr int GROUP_MAX_N = 16;

__global__ void __launch_bounds__(256)
decode_attention_group_bf16(const __nv_bfloat16* q, long long ldq, const __nv_bfloat16* kc, const __nv_bfloat16* vc,
                            __nv_bfloat16* out, long long ldo, int H, int N, const int* __restrict__ prompt_lens,
                            const int* __restrict__ pos_rows, int Lmax, float scale, int per_max, int gper_max) {
  pdl_sync();
  constexpr int D = 128, LPR = 16, GROUPS = 16;
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  const int S = (int)cluster.num_blocks(), rank = (int)cluster.block_rank();
  const int h = blockIdx.x, b = blockIdx.y, B = gridDim.y;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int sub = lane % LPR, grp = warp * 2 + lane / LPR;
  const int HD = H * D;
  const int KS = GROUPS / N;                 // lane groups per query
  const int qi = grp / KS, part = grp % KS;  // this group's query and its share of the query's keys
  const bool active = qi < N;
  const int r = b * N + (active ? qi : 0);
  const int P = prompt_lens[b];
  const int per = (P + S - 1) / S;
  const int k0 = rank * per;
  const int n_loc = max(0, min(P, k0 + per) - k0);            // prompt keys of this CTA, shared by the N queries
  const int g = active ? max(0, pos_rows[r] + 1 - P) : 0;     // the row's own keys
  const int gper = (g + S - 1) / S;
  const int g0 = rank * gper;
  const int n_gen = max(0, min(g, g0 + gper) - g0);
  const int n_all = active ? n_loc + n_gen : 0;               // local keys of the query: prompt slice, then own slice
  // both lane groups of a warp run the same trip count (the reductions shuffle across the whole warp)
  const int n_warp = max(n_all, __shfl_xor_sync(0xffffffffu, n_all, 16));
  const int ld_sc = per_max + gper_max;
  extern __shared__ float sm[];
  float* sc = sm;                              // [N][ld_sc] scores / probabilities of the local keys
  float* part_o = sm + N * ld_sc;              // [GROUPS][D] partial outputs of the lane groups
  float* tot = part_o + GROUPS * D;            // [N][D] CTA totals, read by rank 0
  __shared__ float red[GROUPS];
  __shared__ float cl_max[GROUP_MAX_N], cl_sum[GROUP_MAX_N];

  float qf[8];
  {
    uint4 raw = make_uint4(0, 0, 0, 0);
    if (active) raw = *reinterpret_cast<const uint4*>(q + (long long)r * ldq + (long long)h * D + sub * 8);
    const __nv_bfloat162* hh = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const float2 f = __bfloat1622float2(hh[j]);
      qf[2 * j] = f.x * scale;
      qf[2 * j + 1] = f.y * scale;
    }
  }
  // local key j of the query: prompt row b at k0 + j, or its own row B + r at P + g0 + (j - n_loc)
  const long long prompt_off = ((long long)b * Lmax + k0) * HD + (long long)h * D + sub * 8;
  const long long own_off = ((long long)(B + r) * Lmax + P + g0 - n_loc) * HD + (long long)h * D + sub * 8;
  auto off = [&](int j) -> long long { return (j < n_loc ? prompt_off : own_off) + (long long)j * HD; };
  float* srow = sc + (active ? qi : 0) * ld_sc;
  const int step = 4 * KS;
  // ---- phase 1: scores of the local keys
  float mx = -INFINITY;
  for (int base = part; base - part < n_warp; base += step) {
    uint4 raw[4];
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const int j = base + u * KS;
      raw[u] = j < n_all ? *reinterpret_cast<const uint4*>(kc + off(j)) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const __nv_bfloat162* hh = reinterpret_cast<const __nv_bfloat162*>(&raw[u]);
      float acc = 0.f;
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const float2 f = __bfloat1622float2(hh[j]);
        acc += f.x * qf[2 * j] + f.y * qf[2 * j + 1];
      }
#pragma unroll
      for (int o = LPR / 2; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      const int j = base + u * KS;
      if (j < n_all) {
        if (sub == 0) srow[j] = acc;
        mx = fmaxf(mx, acc);
      }
    }
  }
  if (sub == 0) red[grp] = mx;
  __syncthreads();
  if (tid < N) {
    float m = red[tid * KS];
    for (int p = 1; p < KS; p++) m = fmaxf(m, red[tid * KS + p]);
    cl_max[tid] = m;
  }
  cluster.sync();
  float gmax = -INFINITY;
  if (active)
    for (int c = 0; c < S; c++) gmax = fmaxf(gmax, *cluster.map_shared_rank(&cl_max[qi], c));
  float sum = 0.f;
  for (int j = part + sub * KS; j < n_all; j += LPR * KS) {
    const float p = __expf(srow[j] - gmax);
    srow[j] = p;
    sum += p;
  }
#pragma unroll
  for (int o = LPR / 2; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if (sub == 0) red[grp] = sum;   // the max's reads of red[] finished before the cluster barrier
  __syncthreads();
  if (tid < N) {
    float t = 0.f;
    for (int p = 0; p < KS; p++) t += red[tid * KS + p];
    cl_sum[tid] = t;
  }
  cluster.sync();
  float gsum = 0.f;
  if (active)
    for (int c = 0; c < S; c++) gsum += *cluster.map_shared_rank(&cl_sum[qi], c);
  const float inv = active ? 1.f / gsum : 0.f;
  // ---- phase 2: partial P.V of the local keys (probabilities rounded to the 16-bit type, as P.to(q.dtype))
  float o8[8];
#pragma unroll
  for (int j = 0; j < 8; j++) o8[j] = 0.f;
  for (int base = part; base < n_all; base += step) {
    uint4 raw[4];
    float pk[4];
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const int j = base + u * KS;
      const bool ok = j < n_all;
      raw[u] = ok ? *reinterpret_cast<const uint4*>(vc + off(j)) : make_uint4(0, 0, 0, 0);
      pk[u] = ok ? __bfloat162float(__float2bfloat16_rn(srow[j] * inv)) : 0.f;
    }
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const __nv_bfloat162* hh = reinterpret_cast<const __nv_bfloat162*>(&raw[u]);
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const float2 f = __bfloat1622float2(hh[j]);
        o8[2 * j] += pk[u] * f.x;
        o8[2 * j + 1] += pk[u] * f.y;
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; j++) part_o[grp * D + sub * 8 + j] = o8[j];
  __syncthreads();
  for (int i = tid; i < N * D; i += 256) {
    const int t = i / D, d = i % D;
    float v = 0.f;
    for (int p = 0; p < KS; p++) v += part_o[(t * KS + p) * D + d];
    tot[i] = v;
  }
  cluster.sync();
  if (rank == 0) {
    for (int i = tid; i < N * D; i += 256) {
      float v = 0.f;
      for (int c = 0; c < S; c++) v += cluster.map_shared_rank(tot, c)[i];
      out[(long long)(b * N + i / D) * ldo + (long long)h * D + i % D] = __float2bfloat16_rn(v);
    }
  }
  cluster.sync();   // keep every CTA's shared memory alive until rank 0 has read it
}

}  // namespace g4r

using namespace G4R_NS;

static int launch_kv_append(const void* qkv, long long ld, void* kcache, void* vcache, int B, int Ln, int pos0,
                            const int* pos_dev, const int* pos_rows, int Lmax, int HD, cudaStream_t st) {
  const long long total = (long long)B * Ln * (HD / 8) * 2;
  long long grid = (total + 255) / 256;
  const long long cap = (long long)num_sms() * 16;
  if (grid > cap) grid = cap;
  kv_append_bf16<<<(unsigned)grid, 256, 0, st>>>((const __nv_bfloat16*)qkv, ld, (__nv_bfloat16*)kcache,
                                                 (__nv_bfloat16*)vcache, B, Ln, pos0, pos_dev, pos_rows, Lmax, HD);
  G4R_LAUNCH_CHECK("kv_append");
  return G4R_OK;
}

extern "C" int g4r_kv_append_bf16(const void* qkv, long long ld, void* kcache, void* vcache, int B, int Ln,
                                  int pos0, const int* pos_dev, int Lmax, int HD, void* stream) {
  G4R_REQUIRE(qkv && kcache && vcache && B > 0 && Ln > 0 && pos0 >= 0 && pos0 + Ln <= Lmax && HD % 8 == 0 && ld % 8 == 0,
              "kv_append: bad arguments (pos0=%d Ln=%d Lmax=%d)", pos0, Ln, Lmax);
  return launch_kv_append(qkv, ld, kcache, vcache, B, Ln, pos0, pos_dev, nullptr, Lmax, HD, (cudaStream_t)stream);
}

extern "C" int g4r_kv_append_rows_bf16(const void* qkv, long long ld, void* kcache, void* vcache, int B, int Ln,
                                       const int* pos_rows, int Lmax, int HD, void* stream) {
  G4R_REQUIRE(qkv && kcache && vcache && pos_rows && B > 0 && Ln > 0 && Ln <= Lmax && HD % 8 == 0 && ld % 8 == 0,
              "kv_append_rows: bad arguments (Ln=%d Lmax=%d)", Ln, Lmax);
  return launch_kv_append(qkv, ld, kcache, vcache, B, Ln, 0, nullptr, pos_rows, Lmax, HD, (cudaStream_t)stream);
}

extern "C" int g4r_kv_append_rows_at_bf16(const void* qkv, long long ld, void* kcache, void* vcache, int B, int Ln,
                                          const int* pos_rows, const int* cache_rows, const int* qlen, int Lmax, int HD,
                                          void* stream) {
  G4R_REQUIRE(qkv && kcache && vcache && pos_rows && cache_rows && qlen && B > 0 && Ln > 0 && Ln <= Lmax &&
              HD % 8 == 0 && ld % 8 == 0, "kv_append_rows_at: bad arguments (Ln=%d Lmax=%d)", Ln, Lmax);
  const long long total = (long long)B * Ln * (HD / 8) * 2;
  long long grid = (total + 255) / 256;
  const long long cap = (long long)num_sms() * 16;
  if (grid > cap) grid = cap;
  kv_append_rows_at_bf16<<<(unsigned)grid, 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)qkv, ld, (__nv_bfloat16*)kcache, (__nv_bfloat16*)vcache, B, Ln, pos_rows, cache_rows, qlen,
      Lmax, HD);
  G4R_LAUNCH_CHECK("kv_append_rows_at");
  return G4R_OK;
}

template <int D, bool BEAM>
static int launch_decode_attention(const void* q, long long ldq, const void* kcache, const void* vcache, void* out,
                                   long long ldo, int B, int H, int kv_len, const int* pos_dev, const int* pos_rows,
                                   const int* anc, int Lmax, float scale, cudaStream_t st) {
  // split-KV factor: enough CTAs for >= 2 per SM, slices of >= 64 keys, cluster size <= 8 (portable)
  int S = 1;
  while (S < 8 && H * B * S < 2 * num_sms() && kv_len / (2 * S) >= 64) S *= 2;
  const int per_max = (kv_len + S - 1) / S;
  const int groups = 8 * (32 / (D / 8));
  const size_t smem = ((size_t)per_max + (size_t)groups * D) * sizeof(float);
  G4R_REQUIRE(smem <= 200 * 1024, "decode_attention: kv_len %d too long for the shared-memory score buffer", kv_len);
  static bool set = false;
  if (!set) {
    G4R_CUDA(cudaFuncSetAttribute(decode_attention_bf16<D, BEAM>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    set = true;
  }
  G4R_CUDA(launch_pdl(decode_attention_bf16<D, BEAM>, dim3(H, B, S), dim3(256), smem, st, dim3(1, 1, S),
                      (const __nv_bfloat16*)q, ldq, (const __nv_bfloat16*)kcache, (const __nv_bfloat16*)vcache,
                      (__nv_bfloat16*)out, ldo, H, kv_len, pos_dev, pos_rows, Lmax, scale, per_max, anc));
  return G4R_OK;
}

static int decode_attention(const void* q, long long ldq, const void* kcache, const void* vcache, void* out,
                            long long ldo, int B, int H, int head_dim, int kv_len, const int* pos_dev,
                            const int* pos_rows, const int* anc, int Lmax, float scale, void* stream) {
  G4R_REQUIRE(q && kcache && vcache && out && B > 0 && H > 0 && kv_len > 0 && kv_len <= Lmax, "decode_attention: bad arguments");
  G4R_REQUIRE(head_dim == 64 || head_dim == 128, "decode_attention: head_dim %d", head_dim);
  G4R_REQUIRE(ldq % 8 == 0 && ((uintptr_t)q & 15) == 0, "decode_attention: q rows must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  if (anc) {
    if (head_dim == 128)
      return launch_decode_attention<128, true>(q, ldq, kcache, vcache, out, ldo, B, H, kv_len, pos_dev, pos_rows, anc,
                                                Lmax, scale, st);
    return launch_decode_attention<64, true>(q, ldq, kcache, vcache, out, ldo, B, H, kv_len, pos_dev, pos_rows, anc,
                                             Lmax, scale, st);
  }
  if (head_dim == 128)
    return launch_decode_attention<128, false>(q, ldq, kcache, vcache, out, ldo, B, H, kv_len, pos_dev, pos_rows, nullptr,
                                               Lmax, scale, st);
  return launch_decode_attention<64, false>(q, ldq, kcache, vcache, out, ldo, B, H, kv_len, pos_dev, pos_rows, nullptr,
                                            Lmax, scale, st);
}

extern "C" int g4r_decode_attention_bf16(const void* q, long long ldq, const void* kcache, const void* vcache,
                                         void* out, long long ldo, int B, int H, int head_dim, int kv_len,
                                         const int* pos_dev, int Lmax, float scale, void* stream) {
  return decode_attention(q, ldq, kcache, vcache, out, ldo, B, H, head_dim, kv_len, pos_dev, nullptr, nullptr, Lmax, scale,
                          stream);
}

extern "C" int g4r_decode_attention_rows_bf16(const void* q, long long ldq, const void* kcache, const void* vcache,
                                              void* out, long long ldo, int B, int H, int head_dim, int kv_bound,
                                              const int* pos_rows, int Lmax, float scale, void* stream) {
  G4R_REQUIRE(pos_rows != nullptr, "decode_attention_rows: pos_rows is NULL");
  return decode_attention(q, ldq, kcache, vcache, out, ldo, B, H, head_dim, kv_bound, nullptr, pos_rows, nullptr, Lmax,
                          scale, stream);
}

extern "C" int g4r_decode_attention_beam_bf16(const void* q, long long ldq, const void* kcache, const void* vcache,
                                              void* out, long long ldo, int R, int H, int head_dim, int kv_bound,
                                              const int* pos_rows, const int* anc, int Lmax, float scale, void* stream) {
  G4R_REQUIRE(pos_rows != nullptr && anc != nullptr, "decode_attention_beam: pos_rows and anc are required");
  return decode_attention(q, ldq, kcache, vcache, out, ldo, R, H, head_dim, kv_bound, nullptr, pos_rows, anc, Lmax, scale,
                          stream);
}

extern "C" int g4r_decode_attention_group_bf16(const void* q, long long ldq, const void* kcache, const void* vcache,
                                               void* out, long long ldo, int B, int N, int H, int head_dim,
                                               int prompt_bound, int gen_bound, const int* prompt_lens,
                                               const int* pos_rows, int Lmax, float scale, void* stream) {
  G4R_REQUIRE(q && kcache && vcache && out && prompt_lens && pos_rows, "decode_attention_group: NULL argument");
  G4R_REQUIRE(N >= 1 && N <= GROUP_MAX_N, "decode_attention_group: N=%d rows per prompt; the kernel supports 1..%d", N,
              GROUP_MAX_N);
  G4R_REQUIRE(head_dim == 128, "decode_attention_group: head_dim %d (only 128 is built)", head_dim);
  G4R_REQUIRE(B > 0 && H > 0 && prompt_bound > 0 && gen_bound >= 0 && prompt_bound + gen_bound <= Lmax,
              "decode_attention_group: bad arguments (B=%d H=%d prompt_bound=%d gen_bound=%d Lmax=%d)", B, H,
              prompt_bound, gen_bound, Lmax);
  G4R_REQUIRE(ldq % 8 == 0 && ((uintptr_t)q & 15) == 0, "decode_attention_group: q rows must be 16-byte aligned");
  // split-KV factor as decode_attention's, over the B prompts
  int S = 1;
  while (S < 8 && H * B * S < 2 * num_sms() && prompt_bound / (2 * S) >= 64) S *= 2;
  const int per_max = (prompt_bound + S - 1) / S, gper_max = (gen_bound + S - 1) / S;
  const size_t smem = ((size_t)N * (per_max + gper_max) + (size_t)(16 + N) * head_dim) * sizeof(float);
  G4R_REQUIRE(smem <= 200 * 1024, "decode_attention_group: N=%d rows x (%d prompt + %d generated) keys per CTA exceed "
              "the shared-memory score buffer", N, per_max, gper_max);
  static bool set = false;
  if (!set) {
    G4R_CUDA(cudaFuncSetAttribute(decode_attention_group_bf16, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    set = true;
  }
  G4R_CUDA(launch_pdl(decode_attention_group_bf16, dim3(H, B, S), dim3(256), smem, (cudaStream_t)stream, dim3(1, 1, S),
                      (const __nv_bfloat16*)q, ldq, (const __nv_bfloat16*)kcache, (const __nv_bfloat16*)vcache,
                      (__nv_bfloat16*)out, ldo, H, N, prompt_lens, pos_rows, Lmax, scale, per_max, gper_max));
  return G4R_OK;
}
