// clip_preprocess.cu -- the CLIPImageProcessor image path of the demo and the VCR / LLaVA-instruct datasets as two
// launches for a whole ragged batch (gpt4roi/app.py:125-136, gpt4roi/datasets/vcr.py:181-189, det_llava.py:347-389):
//   CLIPImageProcessor.preprocess(image, do_center_crop=False)   PIL BICUBIC resize of the short side to 224, then
//                                                                 float32(u8 * (1/255) in double), (x - mean) / std
//   F.interpolate(x[None], (S, S), mode='bilinear', align_corners=False)   torch's CPU kernel, fp32
// Output [B,3,S,S] fp32 (bit-identical to that path), bf16 or fp16 (one rounding of the fp32 value).
//
// The resize is PIL's separable antialiased resample, pure integer arithmetic once the host has turned each output
// index's tap window into 22-bit fixed-point weights: acc = 2^21 + sum u8 * k, clamp(acc >> 22, 0, 255), one pass into
// uint8, then the other.  PIL runs the horizontal pass first, except for an image taller than 100 x its width that
// shrinks in height (Image.resize), which runs the vertical pass first (`vfirst`).  Only the resized pixels the
// bilinear reads are computed -- at most 2S rows and 2S columns per image -- so the work follows the S x S output, not
// the resized image (16800 rows for a 3000 x 40 image).  The host (gpt4roi_b200/input_pipeline.py: ClipPreprocessor)
// packs per image, with "needed" = read by the bilinear:
//   list  [n]             horizontal first: the source rows the needed resized rows read; vertical first: the
//                         source columns the needed resized columns read (sorted, unique)
//   e1    [n1][2 + k1]    first pass, per needed resized column (row): first source column (row), tap count, k1
//                         fixed-point weights
//   e2    [n2][2 + k2]    second pass, per needed resized row (column): first tap's index into `list`, tap count, k2
//                         weights
//   by/bx [S][4]          per output row / column: the two needed resized rows / columns and torch's two float32
//                         lambdas (bit patterns)
// Pass 1 (clip_resize_1): the first pass into a uint8 [nr][nc][3] intermediate: list x e1 (horizontal first) or
// e1 x list (vertical first).
// Pass 2 (clip_resize_2_sample): per output pixel, the second pass of its four resized pixels, the rescale /
// normalise, and torch's two lerps t_r = fma(v[r][c0], l0x, v[r][c1] * l1x); out = fma(t_0, l0y, t_1 * l1y) (its
// vectorised CPU builds contract them so), all with explicit round-to-nearest intrinsics.
#include "common.cuh"

namespace g4r {

// per-image fields of the int64 meta table [B][CLIP_META]; gpt4roi_b200/input_pipeline.py writes the same layout
enum { M_SRC, M_W, M_VFIRST, M_TMP, M_NR, M_NC, M_LIST, M_E1, M_K1, M_E2, M_K2, M_BY, M_BX, CLIP_META };
constexpr int CLIP_BITS = 22;

__device__ __forceinline__ int clip8(int acc) { return min(max(acc >> CLIP_BITS, 0), 255); }

// acc = 2^21 + sum_t p[t * step] * k[t] for the 3 channels at p
__device__ __forceinline__ void taps3(const unsigned char* p, size_t step, const int* k, int n, int v[3]) {
  int a0 = 1 << (CLIP_BITS - 1), a1 = a0, a2 = a0;
  for (int t = 0; t < n; t++) {
    const unsigned char* q = p + (size_t)t * step;
    a0 += (int)q[0] * k[t];
    a1 += (int)q[1] * k[t];
    a2 += (int)q[2] * k[t];
  }
  v[0] = clip8(a0);
  v[1] = clip8(a1);
  v[2] = clip8(a2);
}

__global__ void __launch_bounds__(256)
clip_resize_1(const long long* __restrict__ meta, const int* __restrict__ tab, unsigned char* __restrict__ tmp) {
  const long long* m = meta + (size_t)blockIdx.y * CLIP_META;
  const int nc = (int)m[M_NC];
  const int idx = blockIdx.x * 256 + threadIdx.x;
  if (idx >= (int)m[M_NR] * nc) return;
  const int r = idx / nc, c = idx - r * nc;
  const bool vfirst = m[M_VFIRST] != 0;
  const size_t w = (size_t)m[M_W];
  const int* e = tab + m[M_E1] + (size_t)(vfirst ? r : c) * (2 + (int)m[M_K1]);
  const size_t at = tab[m[M_LIST] + (vfirst ? c : r)];
  const unsigned char* src = reinterpret_cast<const unsigned char*>(m[M_SRC]);
  const unsigned char* p = src + (vfirst ? (size_t)e[0] * w + at : at * w + e[0]) * 3;
  int v[3];
  taps3(p, vfirst ? w * 3 : 3, e + 2, e[1], v);
  unsigned char* o = tmp + m[M_TMP] + (size_t)idx * 3;
  o[0] = (unsigned char)v[0];
  o[1] = (unsigned char)v[1];
  o[2] = (unsigned char)v[2];
}

// second pass of resized pixel (needed row i, needed column j): 3 channels
__device__ __forceinline__ void resized_px(const long long* m, const int* tab, const unsigned char* tmp, int i, int j,
                                           int v[3]) {
  const bool vfirst = m[M_VFIRST] != 0;
  const size_t nc = (size_t)m[M_NC];
  const int* e = tab + m[M_E2] + (size_t)(vfirst ? j : i) * (2 + (int)m[M_K2]);
  const unsigned char* p = tmp + m[M_TMP] + (vfirst ? (size_t)i * nc + e[0] : (size_t)e[0] * nc + j) * 3;
  taps3(p, vfirst ? 3 : nc * 3, e + 2, e[1], v);
}

struct ClipNorm {
  float mean[3], std[3];
};

__global__ void __launch_bounds__(256)
clip_resize_2_sample(const long long* __restrict__ meta, const int* __restrict__ tab,
                     const unsigned char* __restrict__ tmp, void* __restrict__ out, int S, int out_dtype,
                     const ClipNorm nm) {
  const int b = blockIdx.y;
  const int pix = blockIdx.x * 256 + threadIdx.x;
  if (pix >= S * S) return;
  const long long* m = meta + (size_t)b * CLIP_META;
  const int oy = pix / S, ox = pix - oy * S;
  const int* ey = tab + m[M_BY] + 4 * oy;
  const int* ex = tab + m[M_BX] + 4 * ox;
  const float ly0 = __int_as_float(ey[2]), ly1 = __int_as_float(ey[3]);
  const float lx0 = __int_as_float(ex[2]), lx1 = __int_as_float(ex[3]);
  int v[4][3];
  resized_px(m, tab, tmp, ey[0], ex[0], v[0]);
  resized_px(m, tab, tmp, ey[0], ex[1], v[1]);
  if (ey[1] != ey[0]) {
    resized_px(m, tab, tmp, ey[1], ex[0], v[2]);
    resized_px(m, tab, tmp, ey[1], ex[1], v[3]);
  } else {
#pragma unroll
    for (int c = 0; c < 3; c++) { v[2][c] = v[0][c]; v[3][c] = v[1][c]; }
  }
  const size_t plane = (size_t)S * S;
#pragma unroll
  for (int c = 0; c < 3; c++) {
    float x[4];
#pragma unroll
    for (int q = 0; q < 4; q++)
      x[q] = __fdiv_rn(__fsub_rn((float)__dmul_rn((double)v[q][c], 1.0 / 255.0), nm.mean[c]), nm.std[c]);
    const float t0 = __fmaf_rn(x[0], lx0, __fmul_rn(x[1], lx1));
    const float t1 = __fmaf_rn(x[2], lx0, __fmul_rn(x[3], lx1));
    const float o = __fmaf_rn(t0, ly0, __fmul_rn(t1, ly1));
    const size_t at = ((size_t)b * 3 + c) * plane + pix;
    if (out_dtype == G4R_BF16) reinterpret_cast<__nv_bfloat16*>(out)[at] = __float2bfloat16_rn(o);
    else if (out_dtype == G4R_F16) reinterpret_cast<__half*>(out)[at] = __float2half_rn(o);
    else reinterpret_cast<float*>(out)[at] = o;
  }
}

}  // namespace g4r

using namespace g4r;

extern "C" int g4r_clip_preprocess(const long long* meta, const int* tables, void* tmp, void* out, int B, int S,
                                   long long max_work1, const float* mean3, const float* std3, int out_dtype,
                                   void* stream) {
  G4R_REQUIRE(meta && tables && tmp && out && mean3 && std3, "clip_preprocess: null argument");
  G4R_REQUIRE(B > 0 && B <= 65535 && S > 0 && S <= 4096, "clip_preprocess: bad sizes B=%d S=%d", B, S);
  G4R_REQUIRE(max_work1 > 0 && max_work1 <= 0x7fffffffLL - 255, "clip_preprocess: bad first-pass size %lld", max_work1);
  G4R_REQUIRE(out_dtype == G4R_F32 || out_dtype == G4R_BF16 || out_dtype == G4R_F16,
              "clip_preprocess: out_dtype must be fp32, bf16 or fp16");
  ClipNorm nm;
  for (int c = 0; c < 3; c++) { nm.mean[c] = mean3[c]; nm.std[c] = std3[c]; }
  cudaStream_t st = (cudaStream_t)stream;
  clip_resize_1<<<dim3((unsigned)((max_work1 + 255) / 256), (unsigned)B), 256, 0, st>>>(
      meta, tables, (unsigned char*)tmp);
  G4R_LAUNCH_CHECK("clip_resize_1");
  clip_resize_2_sample<<<dim3((unsigned)((S * S + 255) / 256), (unsigned)B), 256, 0, st>>>(
      meta, tables, (const unsigned char*)tmp, out, S, out_dtype, nm);
  G4R_LAUNCH_CHECK("clip_resize_2_sample");
  return G4R_OK;
}
