// splice.cu -- embedding gather + image-span splice + <bbox> region-token scatter (sm_90a).
//
// Replaces the per-sample python loop of gpt4roi/models/spi_llava.py:99-196 (and the
// embed_tokens lookup at :44-45): ~10 small launches, three full-row copies and several
// device->host syncs per sample in the reference become two launches per batch:
//   splice_plan : one CTA per sample scans input_ids once, validates the reference's
//                 span rules and writes a per-token source code (int32);
//   splice_move : pure HBM copy, one 128-bit load + store per thread per step; each row
//                 (D 16-bit elements) comes from exactly one of {embed table, projected
//                 image patches, region tokens}.
// Data is only moved, never re-rounded, so the result equals the reference's row by row.
#include "common.cuh"

namespace g4r {

constexpr int kPlanThreads = 256;
constexpr int kTagImage = 0x40000000;
constexpr int kTagRegion = 0x20000000;
constexpr int kTagMask = 0x60000000;

__global__ void __launch_bounds__(kPlanThreads)
splice_plan(const int64_t* __restrict__ input_ids, const int32_t* __restrict__ region_offsets,
            int32_t* __restrict__ plan, int32_t* __restrict__ status, int L, int P, int V,
            int64_t tok_patch, int64_t tok_start, int64_t tok_end, int64_t tok_bbox) {
  __shared__ int s_cnt[4];       // patch, start, end, bad-id
  __shared__ int s_start_pos;
  __shared__ int s_scan[kPlanThreads + 1];
  const int b = blockIdx.x;
  const int64_t* ids = input_ids + (size_t)b * L;
  int32_t* pl = plan + (size_t)b * L;
  const int tid = threadIdx.x;
  if (tid < 4) s_cnt[tid] = 0;
  if (tid == 0) s_start_pos = 0x7fffffff;
  __syncthreads();

  // contiguous segment per thread so that <bbox> ordinals come out in token order
  const int seg = (L + kPlanThreads - 1) / kPlanThreads;
  const int t0 = min(L, tid * seg), t1 = min(L, t0 + seg);
  int n_patch = 0, n_start = 0, n_end = 0, n_bbox = 0, n_bad = 0, first_start = 0x7fffffff;
  for (int t = t0; t < t1; t++) {
    const int64_t id = ids[t];
    n_patch += id == tok_patch;
    if (id == tok_start) { n_start++; first_start = min(first_start, t); }
    n_end += id == tok_end;
    n_bbox += id == tok_bbox;
    n_bad += (id < 0 || id >= V);
  }
  if (n_patch) atomicAdd(&s_cnt[0], n_patch);
  if (n_start) { atomicAdd(&s_cnt[1], n_start); atomicMin(&s_start_pos, first_start); }
  if (n_end) atomicAdd(&s_cnt[2], n_end);
  if (n_bad) atomicAdd(&s_cnt[3], n_bad);
  s_scan[tid + 1] = n_bbox;
  if (tid == 0) s_scan[0] = 0;
  __syncthreads();
  if (tid == 0) {
    for (int i = 1; i <= kPlanThreads; i++) s_scan[i] += s_scan[i - 1];  // 256 adds; negligible
  }
  __syncthreads();
  const int total_bbox = s_scan[kPlanThreads];
  const int tot_patch = s_cnt[0], tot_start = s_cnt[1], tot_end = s_cnt[2];
  const int s = s_start_pos;

  int err = 0;
  const bool multimodal = tot_patch > 0;  // spi_llava.py:104-111: otherwise rows stay embeddings
  if (s_cnt[3] > 0) err = 6;
  else if (multimodal) {
    if (tot_start != tot_end) err = 1;                                  // :114-118
    else if (tot_start > 1) err = 4;
    else if (tot_start == 0) err = 5;
    else if (s + P + 1 >= L || ids[s + P + 1] != tok_end) err = 2;      // :124-128
    else {
      const int kb = region_offsets ? region_offsets[b + 1] - region_offsets[b] : 0;
      if (total_bbox != kb) err = 3;                                    // :154 / :158-161
    }
  }
  if (tid == 0) status[b] = err;
  const bool do_splice = multimodal && err == 0;
  const int kbase = (do_splice && region_offsets) ? region_offsets[b] : 0;
  int ord = s_scan[tid];
  for (int t = t0; t < t1; t++) {
    const int64_t id = ids[t];
    int code = (id < 0 || id >= V) ? 0 : (int)id;
    if (do_splice) {
      if (t > s && t <= s + P) code = kTagImage | (t - s - 1);
      if (id == tok_bbox) code = kTagRegion | (kbase + ord);
    }
    ord += id == tok_bbox;
    pl[t] = code;
  }
}

// rows of D 16-bit elements; ROWS rows per CTA, TPR threads per row.
template <int ROWS, int TPR>
__global__ void __launch_bounds__(ROWS * TPR)
splice_move(const int32_t* __restrict__ plan, const uint4* __restrict__ embed,
            const uint4* __restrict__ image, const uint4* __restrict__ region,
            uint4* __restrict__ out, int n_rows, int L, int P, int vec_per_row) {
  const int row = blockIdx.x * ROWS + threadIdx.x / TPR;
  if (row >= n_rows) return;
  const int lane = threadIdx.x % TPR;
  const int code = plan[row];
  const int b = row / L;
  const uint4* src;
  if ((code & kTagMask) == kTagImage) src = image + ((size_t)b * P + (code & ~kTagMask)) * vec_per_row;
  else if ((code & kTagMask) == kTagRegion) src = region + (size_t)(code & ~kTagMask) * vec_per_row;
  else src = embed + (size_t)code * vec_per_row;
  uint4* dst = out + (size_t)row * vec_per_row;
  int v = lane;
  for (; v + 3 * TPR < vec_per_row; v += 4 * TPR) {
    const uint4 a0 = src[v], a1 = src[v + TPR], a2 = src[v + 2 * TPR], a3 = src[v + 3 * TPR];
    dst[v] = a0; dst[v + TPR] = a1; dst[v + 2 * TPR] = a2; dst[v + 3 * TPR] = a3;
  }
  for (; v < vec_per_row; v += TPR) dst[v] = src[v];
}

// ---- backward (training step, SURVEY.md 8(a) row 14) ----------------------------------------------------
// d(inputs_embeds) rows go back where the forward took them from.  Image and region rows have exactly one
// consumer each (a plain row copy); embedding rows are shared by every occurrence of a token id.
template <int ROWS, int TPR>
__global__ void __launch_bounds__(ROWS * TPR)
splice_bwd_move(const int32_t* __restrict__ plan, const uint4* __restrict__ d_out, uint4* __restrict__ d_image,
                uint4* __restrict__ d_region, int n_rows, int L, int P, int vec_per_row) {
  const int row = blockIdx.x * ROWS + threadIdx.x / TPR;
  if (row >= n_rows) return;
  const int lane = threadIdx.x % TPR;
  const int code = plan[row];
  const int b = row / L;
  uint4* dst;
  if ((code & kTagMask) == kTagImage) dst = d_image ? d_image + ((size_t)b * P + (code & ~kTagMask)) * vec_per_row : nullptr;
  else if ((code & kTagMask) == kTagRegion) dst = d_region ? d_region + (size_t)(code & ~kTagMask) * vec_per_row : nullptr;
  else return;
  if (dst == nullptr) return;
  const uint4* src = d_out + (size_t)row * vec_per_row;
  for (int v = lane; v < vec_per_row; v += TPR) dst[v] = src[v];
}

// One CTA per distinct token id u: grad[id_u] = sum of the d_out rows at the positions order[seg[u] .. seg[u+1])
// (positions sorted by id on the host side of the call: fixed order => bitwise reproducible, no atomics).
__global__ void __launch_bounds__(256)
embed_grad_rows(const __nv_bfloat16* __restrict__ d_out, const int32_t* __restrict__ order,
                const int32_t* __restrict__ seg, const int32_t* __restrict__ ids, float* __restrict__ grad, int D) {
  const int u = blockIdx.x;
  const int j0 = seg[u], j1 = seg[u + 1];
  float* g = grad + (size_t)ids[u] * D;
  for (int v = threadIdx.x * 8; v < D; v += 256 * 8) {
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; i++) acc[i] = 0.f;
    for (int j = j0; j < j1; j++) {
      const uint4 raw = *reinterpret_cast<const uint4*>(d_out + (size_t)order[j] * D + v);
      const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const float2 f = __bfloat1622float2(h[i]);
        acc[2 * i] += f.x;
        acc[2 * i + 1] += f.y;
      }
    }
    reinterpret_cast<float4*>(g + v)[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
    reinterpret_cast<float4*>(g + v)[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
  }
}

}  // namespace g4r

using namespace g4r;

extern "C" int g4r_splice_backward(const int32_t* plan, const void* d_out, void* d_image, void* d_region, int B, int L,
                                   int P, int D, void* stream) {
  G4R_REQUIRE(plan && d_out && B > 0 && L > 0 && D % 8 == 0, "splice_backward: bad arguments");
  const int n_rows = B * L;
  constexpr int ROWS = 4, TPR = 64;
  splice_bwd_move<ROWS, TPR><<<(n_rows + ROWS - 1) / ROWS, ROWS * TPR, 0, (cudaStream_t)stream>>>(
      plan, (const uint4*)d_out, (uint4*)d_image, (uint4*)d_region, n_rows, L, P, D / 8);
  G4R_LAUNCH_CHECK("splice_bwd_move");
  return G4R_OK;
}

extern "C" int g4r_embed_grad_rows(const void* d_out, const int32_t* order, const int32_t* seg, const int32_t* ids,
                                   int n_unique, float* grad, int D, void* stream) {
  G4R_REQUIRE(d_out && order && seg && ids && grad && D % 8 == 0, "embed_grad_rows: bad arguments");
  if (n_unique <= 0) return G4R_OK;
  embed_grad_rows<<<n_unique, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)d_out, order, seg, ids, grad, D);
  G4R_LAUNCH_CHECK("embed_grad_rows");
  return G4R_OK;
}

extern "C" int g4r_splice_region_tokens(const int64_t* input_ids, const void* embed_table,
                                        const void* image_rows, const void* region_rows,
                                        const int32_t* region_offsets, void* out, int32_t* plan,
                                        int32_t* status, int B, int L, int P, int D, int V,
                                        int64_t im_patch_token, int64_t im_start_token,
                                        int64_t im_end_token, int64_t bbox_token, void* stream) {
  G4R_REQUIRE(B > 0 && L > 0 && P >= 0 && D > 0 && V > 0, "bad sizes B=%d L=%d P=%d D=%d V=%d", B, L, P, D, V);
  G4R_REQUIRE(input_ids && embed_table && out && plan && status, "null argument");
  G4R_REQUIRE(D % 8 == 0, "D=%d must be a multiple of 8 (128-bit rows of 16-bit elements)", D);
  G4R_REQUIRE(V < kTagRegion, "V too large");
  G4R_REQUIRE((((uintptr_t)embed_table | (uintptr_t)out | (uintptr_t)image_rows | (uintptr_t)region_rows) & 15) == 0,
              "row buffers must be 16-byte aligned");
  G4R_REQUIRE(image_rows || P == 0, "image_rows is NULL with P=%d", P);
  G4R_REQUIRE((region_rows == nullptr) == (region_offsets == nullptr) || region_offsets != nullptr,
              "region_rows given without region_offsets");
  cudaStream_t st = (cudaStream_t)stream;
  splice_plan<<<B, kPlanThreads, 0, st>>>(input_ids, region_offsets, plan, status, L, P, V,
                                          im_patch_token, im_start_token, im_end_token, bbox_token);
  G4R_LAUNCH_CHECK("splice_plan");
  const int n_rows = B * L;
  constexpr int ROWS = 4, TPR = 64;
  splice_move<ROWS, TPR><<<(n_rows + ROWS - 1) / ROWS, ROWS * TPR, 0, st>>>(
      plan, (const uint4*)embed_table, (const uint4*)image_rows, (const uint4*)region_rows, (uint4*)out,
      n_rows, L, P, D / 8);
  G4R_LAUNCH_CHECK("splice_move");
  return G4R_OK;
}
