// train.cu -- the non-GEMM kernels of the stage-2 training step (SURVEY.md 8(a) row 14:
// gpt4roi/train/train.py:698-712 drives HF Trainer over SPILlavaMPTForCausalLM; the loss is
// llava/model/llava.py:238-249: shift logits/labels, CrossEntropyLoss() = mean over labels != -100).
// Backward GEMMs are g4r_gemm_bf16_t (gemm_wgmma.cu).  Everything here is HBM-bound elementwise /
// row-reduction work: 16-byte vector loads, fp32 math, fixed-order reductions (no atomics, bitwise
// reproducible), bf16 storage like the reference's bf16 autocast.
#include "common.cuh"

namespace g4r {

__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ void unpack8f(const uint4& raw, float (&f)[8]) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const float2 t = __bfloat1622float2(h[j]);
    f[2 * j] = t.x;
    f[2 * j + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 pack8f(const float (&f)[8]) {
  uint4 raw;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&raw);
#pragma unroll
  for (int j = 0; j < 4; j++) h[j] = __floats2bfloat162_rn(f[2 * j], f[2 * j + 1]);
  return raw;
}

// block-wide sum / max over 256 threads; every thread gets the result
__device__ __forceinline__ float block_sum_256(float v, float* red) {
  v = warp_sum_f(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < 8; w++) t += red[w];
  return t;
}
__device__ __forceinline__ float block_max_256(float v, float* red) {
  v = warp_max_f(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = red[0];
#pragma unroll
  for (int w = 1; w < 8; w++) t = fmaxf(t, red[w]);
  return t;
}

// ------------------------------------------------------------------------------------------
// Cross entropy over rows of logits [M, V] (bf16, row stride ld) against int64 targets (-100 = ignore).
// Pass 1 (one CTA per row): row max, log-sum-exp, loss_row = lse - x[target].
// Pass 2 (one CTA): loss = sum(loss_row over valid rows) / count, in a fixed order.
// Pass 3 (one CTA per row): dlogits = (softmax - onehot) * gscale / count, zero for ignored rows.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
ce_rows_fwd(const __nv_bfloat16* __restrict__ logits, long long ld, const long long* __restrict__ targets,
            float* __restrict__ row_loss, float* __restrict__ row_lse, int V) {
  __shared__ float red[8];
  const int r = blockIdx.x, tid = threadIdx.x;
  const long long tgt = targets[r];
  const __nv_bfloat16* x = logits + (long long)r * ld;
  const bool vec = (ld % 8 == 0) && ((reinterpret_cast<uintptr_t>(logits) & 15) == 0);
  const int V8 = vec ? (V & ~7) : 0;
  float mx = -INFINITY;
  for (int v = tid * 8; v < V8; v += 256 * 8) {
    float f[8];
    unpack8f(*reinterpret_cast<const uint4*>(x + v), f);
#pragma unroll
    for (int j = 0; j < 8; j++) mx = fmaxf(mx, f[j]);
  }
  for (int v = V8 + tid; v < V; v += 256) mx = fmaxf(mx, __bfloat162float(x[v]));
  mx = block_max_256(mx, red);
  float s = 0.f;
  for (int v = tid * 8; v < V8; v += 256 * 8) {
    float f[8];
    unpack8f(*reinterpret_cast<const uint4*>(x + v), f);
#pragma unroll
    for (int j = 0; j < 8; j++) s += __expf(f[j] - mx);
  }
  for (int v = V8 + tid; v < V; v += 256) s += __expf(__bfloat162float(x[v]) - mx);
  s = block_sum_256(s, red);
  if (tid == 0) {
    const float lse = mx + logf(s);
    row_lse[r] = lse;
    row_loss[r] = (tgt >= 0 && tgt < V) ? lse - __bfloat162float(x[tgt]) : 0.f;
  }
}

__global__ void __launch_bounds__(256)
ce_reduce(const float* __restrict__ row_loss, const long long* __restrict__ targets, int M, int V,
          float* __restrict__ out /* [0] mean loss, [1] valid count */) {
  __shared__ float red[8];
  float s = 0.f, c = 0.f;
  // fixed assignment of rows to threads + fixed-order tree => bitwise reproducible
  for (int r = threadIdx.x; r < M; r += 256) {
    const long long t = targets[r];
    if (t >= 0 && t < V) { s += row_loss[r]; c += 1.f; }
  }
  s = block_sum_256(s, red);
  c = block_sum_256(c, red);
  if (threadIdx.x == 0) {
    out[0] = c > 0.f ? s / c : 0.f;
    out[1] = c;
  }
}

__global__ void __launch_bounds__(256)
ce_rows_bwd(const __nv_bfloat16* __restrict__ logits, long long ld, const long long* __restrict__ targets,
            const float* __restrict__ row_lse, const float* __restrict__ loss_count,
            __nv_bfloat16* __restrict__ dlogits, long long ldd, int V, float gscale) {
  const int r = blockIdx.x, tid = threadIdx.x;
  const long long tgt = targets[r];
  const bool valid = tgt >= 0 && tgt < V;
  const float cnt = loss_count[1];
  const float k = (valid && cnt > 0.f) ? gscale / cnt : 0.f;
  const float lse = row_lse[r];
  const __nv_bfloat16* x = logits + (long long)r * ld;
  __nv_bfloat16* d = dlogits + (long long)r * ldd;
  const bool vec = (ld % 8 == 0) && (ldd % 8 == 0) && ((reinterpret_cast<uintptr_t>(logits) & 15) == 0) &&
                   ((reinterpret_cast<uintptr_t>(dlogits) & 15) == 0);
  const int V8 = vec ? (V & ~7) : 0;
  for (int v = tid * 8; v < V8; v += 256 * 8) {
    float f[8];
    unpack8f(*reinterpret_cast<const uint4*>(x + v), f);
#pragma unroll
    for (int j = 0; j < 8; j++) f[j] = (__expf(f[j] - lse) - ((long long)(v + j) == tgt ? 1.f : 0.f)) * k;
    *reinterpret_cast<uint4*>(d + v) = pack8f(f);
  }
  for (int v = V8 + tid; v < V; v += 256)
    d[v] = __float2bfloat16_rn((__expf(__bfloat162float(x[v]) - lse) - ((long long)v == tgt ? 1.f : 0.f)) * k);
}

// ------------------------------------------------------------------------------------------
// RMSNorm backward (transformers LlamaRMSNorm: y = w * (x * rsqrt(mean(x^2) + eps)).to(bf16)).
// g = dy * w;  xh = x * r;  dx = r * (g - xh * mean(g * xh));  dw = sum_rows dy * xh.
// One CTA walks rows r = blockIdx.x, blockIdx.x + gridDim.x, ...; each thread keeps its channel slice of
// dw in fp32 registers and writes it to a per-CTA slab; rms_dw_reduce sums the slabs in CTA order.
// ------------------------------------------------------------------------------------------
template <int PER>
__global__ void __launch_bounds__(256)
rmsnorm_bwd_rows(const __nv_bfloat16* __restrict__ x, long long ldx, const __nv_bfloat16* __restrict__ w,
                 const __nv_bfloat16* __restrict__ dy, long long ldy, const __nv_bfloat16* __restrict__ dres,
                 long long ldr, __nv_bfloat16* __restrict__ dx, long long ldd, float* __restrict__ dw_slabs, int M,
                 int D, float eps) {
  __shared__ float red[8];
  const int tid = threadIdx.x;
  const int nvec = D >> 3;
  float wf[PER][8], dwacc[PER][8];
#pragma unroll
  for (int i = 0; i < PER; i++) {
    const int vi = tid + i * 256;
#pragma unroll
    for (int j = 0; j < 8; j++) { wf[i][j] = 0.f; dwacc[i][j] = 0.f; }
    if (vi < nvec) unpack8f(reinterpret_cast<const uint4*>(w)[vi], wf[i]);
  }
  for (int r = blockIdx.x; r < M; r += gridDim.x) {
    float xv[PER][8], gv[PER][8];
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < PER; i++) {
      const int vi = tid + i * 256;
      if (vi < nvec) {
        unpack8f(*reinterpret_cast<const uint4*>(x + (long long)r * ldx + vi * 8), xv[i]);
        unpack8f(*reinterpret_cast<const uint4*>(dy + (long long)r * ldy + vi * 8), gv[i]);
      } else {
#pragma unroll
        for (int j = 0; j < 8; j++) { xv[i][j] = 0.f; gv[i][j] = 0.f; }
      }
#pragma unroll
      for (int j = 0; j < 8; j++) ss += xv[i][j] * xv[i][j];
    }
    ss = block_sum_256(ss, red);
    const float rs = rsqrtf(ss / D + eps);
    float dot = 0.f;
#pragma unroll
    for (int i = 0; i < PER; i++)
#pragma unroll
      for (int j = 0; j < 8; j++) {
        const float xh = xv[i][j] * rs;
        dwacc[i][j] += gv[i][j] * __bfloat162float(__float2bfloat16_rn(xh));  // dy * xhat (xhat as stored: bf16)
        gv[i][j] *= wf[i][j];                                                // g = dy * w
        xv[i][j] = xh;
        dot += gv[i][j] * xh;
      }
    dot = block_sum_256(dot, red) / D;
#pragma unroll
    for (int i = 0; i < PER; i++) {
      const int vi = tid + i * 256;
      if (vi >= nvec) continue;
      float o[8], rr[8];
#pragma unroll
      for (int j = 0; j < 8; j++) rr[j] = 0.f;
      // gradient arriving through the residual connection that bypasses the norm (x -> x + f(norm(x)))
      if (dres != nullptr) unpack8f(*reinterpret_cast<const uint4*>(dres + (long long)r * ldr + vi * 8), rr);
#pragma unroll
      for (int j = 0; j < 8; j++) o[j] = rr[j] + rs * (gv[i][j] - xv[i][j] * dot);
      *reinterpret_cast<uint4*>(dx + (long long)r * ldd + vi * 8) = pack8f(o);
    }
  }
#pragma unroll
  for (int i = 0; i < PER; i++) {
    const int vi = tid + i * 256;
    if (vi >= nvec) continue;
    float* o = dw_slabs + (long long)blockIdx.x * D + vi * 8;
    reinterpret_cast<float4*>(o)[0] = make_float4(dwacc[i][0], dwacc[i][1], dwacc[i][2], dwacc[i][3]);
    reinterpret_cast<float4*>(o)[1] = make_float4(dwacc[i][4], dwacc[i][5], dwacc[i][6], dwacc[i][7]);
  }
}

// Column sums of a bf16 matrix (bias gradients): CTA (x, y) sums the rows r = y, y + S, ... of 2048 columns
// into slab y; slab_reduce_f32 adds the S slabs in order.
__global__ void __launch_bounds__(256)
colsum_rows(const __nv_bfloat16* __restrict__ x, long long ld, int M, int N, float* __restrict__ slabs) {
  const int c0 = (blockIdx.x * 256 + threadIdx.x) * 8;
  if (c0 >= N) return;
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; j++) acc[j] = 0.f;
  for (int r = blockIdx.y; r < M; r += gridDim.y) {
    float f[8];
    unpack8f(*reinterpret_cast<const uint4*>(x + (long long)r * ld + c0), f);
#pragma unroll
    for (int j = 0; j < 8; j++) acc[j] += f[j];
  }
  float* o = slabs + (long long)blockIdx.y * N + c0;
  reinterpret_cast<float4*>(o)[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
  reinterpret_cast<float4*>(o)[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
}

// out[d] = sum_s slabs[s][d] in slab order (fp32)
__global__ void __launch_bounds__(256)
slab_reduce_f32(const float* __restrict__ slabs, int S, int D, float* __restrict__ out) {
  const int d = blockIdx.x * 256 + threadIdx.x;
  if (d >= D) return;
  float a = 0.f;
  for (int s = 0; s < S; s++) a += slabs[(long long)s * D + d];
  out[d] = a;
}

// ------------------------------------------------------------------------------------------
// SwiGLU on an interleaved gate/up buffer gu [M, 2F] (column 2j = gate_j, 2j+1 = up_j; the layout the
// fused weight of engine.py produces): f = silu(g) * u, and its backward
//   dg = df * u * s * (1 + g * (1 - s)),  du = df * g * s,  s = sigmoid(g).
// (transformers LlamaMLP: down_proj(act_fn(gate_proj(x)) * up_proj(x)).)
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
swiglu_fwd(const __nv_bfloat16* __restrict__ gu, long long ldg, __nv_bfloat16* __restrict__ f, long long ldf,
           long long M, int F) {
  const int nv = F >> 2;  // 4 outputs (= 8 interleaved inputs, 16 bytes) per thread-step
  const long long total = M * nv;
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    long long r;
    int c;
    divmod_idx(i, nv, r, c);
    float v[8];
    unpack8f(*reinterpret_cast<const uint4*>(gu + r * ldg + c * 8), v);
    __nv_bfloat162 o[2];
    float t[4];
#pragma unroll
    for (int j = 0; j < 4; j++) t[j] = v[2 * j] / (1.f + __expf(-v[2 * j])) * v[2 * j + 1];
    o[0] = __floats2bfloat162_rn(t[0], t[1]);
    o[1] = __floats2bfloat162_rn(t[2], t[3]);
    *reinterpret_cast<uint2*>(f + r * ldf + c * 4) = *reinterpret_cast<uint2*>(o);
  }
}

__global__ void __launch_bounds__(256)
swiglu_bwd(const __nv_bfloat16* __restrict__ gu, long long ldg, const __nv_bfloat16* __restrict__ df, long long ldf,
           __nv_bfloat16* __restrict__ dgu, long long ldd, long long M, int F) {
  const int nv = F >> 2;
  const long long total = M * nv;
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    long long r;
    int c;
    divmod_idx(i, nv, r, c);
    float v[8], o[8];
    unpack8f(*reinterpret_cast<const uint4*>(gu + r * ldg + c * 8), v);
    const uint2 draw = *reinterpret_cast<const uint2*>(df + r * ldf + c * 4);
    const __nv_bfloat162* dh = reinterpret_cast<const __nv_bfloat162*>(&draw);
    const float2 d01 = __bfloat1622float2(dh[0]), d23 = __bfloat1622float2(dh[1]);
    const float d[4] = {d01.x, d01.y, d23.x, d23.y};
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const float g = v[2 * j], u = v[2 * j + 1];
      const float s = 1.f / (1.f + __expf(-g));
      o[2 * j] = d[j] * u * s * (1.f + g * (1.f - s));
      o[2 * j + 1] = d[j] * g * s;
    }
    *reinterpret_cast<uint4*>(dgu + r * ldd + c * 8) = pack8f(o);
  }
}

// ------------------------------------------------------------------------------------------
// AdamW (torch.optim.AdamW, the HF Trainer default `adamw_torch`): fp32 master weights and moments, gradient
// bf16 or fp32, optional bf16 copy of the updated weight for the next forward.  bias corrections on the host.
// ------------------------------------------------------------------------------------------
// 4 elements per thread-iteration (16-byte p/m/v accesses, 8/16-byte gradient loads); `n4` = n / 4 vectors, the
// (< 4) tail elements are handled by the scalar epilogue of the last CTA.  scale_dev (optional) is a device
// float multiplied into the gradient scale: the global-norm clip coefficient written by grad_clip_coef, so
// that clipping needs no host synchronisation (HF Trainer: clip_grad_norm_(max_grad_norm=1.0) before step()).
template <typename TG>
__global__ void __launch_bounds__(256)
adamw_step(float* __restrict__ p, const TG* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
           __nv_bfloat16* __restrict__ p16, long long n, float lr, float b1, float b2, float eps, float wd,
           float bc1, float bc2_sqrt, float gscale, const float* __restrict__ scale_dev) {
  if (scale_dev) gscale *= scale_dev[0];
  const float decay = 1.f - lr * wd, step = lr / bc1, ib2 = 1.f / bc2_sqrt;
  auto upd = [&](float& pi, float& mi, float& vi, float gi) {
    gi *= gscale;
    pi *= decay;
    mi = b1 * mi + (1.f - b1) * gi;
    vi = b2 * vi + (1.f - b2) * gi * gi;
    pi -= step * (mi / (sqrtf(vi) * ib2 + eps));
  };
  const long long n4 = n >> 2;
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < n4; i += (long long)gridDim.x * 256) {
    float4 P = reinterpret_cast<float4*>(p)[i], M = reinterpret_cast<float4*>(m)[i], V = reinterpret_cast<float4*>(v)[i];
    float g4[4];
    if constexpr (sizeof(TG) == 2) {
      const uint2 raw = reinterpret_cast<const uint2*>(g)[i];
      const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw);
      const float2 a = __bfloat1622float2(h[0]), b = __bfloat1622float2(h[1]);
      g4[0] = a.x; g4[1] = a.y; g4[2] = b.x; g4[3] = b.y;
    } else {
      const float4 G = reinterpret_cast<const float4*>(g)[i];
      g4[0] = G.x; g4[1] = G.y; g4[2] = G.z; g4[3] = G.w;
    }
    upd(P.x, M.x, V.x, g4[0]); upd(P.y, M.y, V.y, g4[1]); upd(P.z, M.z, V.z, g4[2]); upd(P.w, M.w, V.w, g4[3]);
    reinterpret_cast<float4*>(p)[i] = P; reinterpret_cast<float4*>(m)[i] = M; reinterpret_cast<float4*>(v)[i] = V;
    if (p16) {
      uint2 o;
      __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&o);
      h[0] = __floats2bfloat162_rn(P.x, P.y); h[1] = __floats2bfloat162_rn(P.z, P.w);
      reinterpret_cast<uint2*>(p16)[i] = o;
    }
  }
  if (blockIdx.x == gridDim.x - 1) {
    for (long long i = (n4 << 2) + threadIdx.x; i < n; i += 256) {
      float gi;
      if constexpr (sizeof(TG) == 2) gi = __bfloat162float(g[i]); else gi = (float)g[i];
      float pi = p[i], mi = m[i], vi = v[i];
      upd(pi, mi, vi, gi);
      p[i] = pi; m[i] = mi; v[i] = vi;
      if (p16) p16[i] = __float2bfloat16_rn(pi);
    }
  }
}

// Sum of squares of one gradient tensor as kSumsqSlabs per-CTA partials (fixed order: bitwise reproducible).
constexpr int kSumsqSlabs = 296;
template <typename TG>
__global__ void __launch_bounds__(256)
sumsq_partial(const TG* __restrict__ g, long long n, float* __restrict__ slab) {
  __shared__ float red[8];
  float acc = 0.f;
  constexpr int V = 16 / (int)sizeof(TG);
  const bool aligned = (reinterpret_cast<uintptr_t>(g) & 15) == 0;
  const long long nv = aligned ? n / V : 0;
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < nv; i += (long long)gridDim.x * 256) {
    float f[V];
    load16<TG>(g + i * V, f);
#pragma unroll
    for (int j = 0; j < V; j++) acc += f[j] * f[j];
  }
  if (blockIdx.x == 0)
    for (long long i = nv * V + threadIdx.x; i < n; i += 256) { const float x = to_f32<TG>(g[i]); acc += x * x; }
  const float t = block_sum_256(acc, red);
  if (threadIdx.x == 0) slab[blockIdx.x] = t;
}

// total norm and clip coefficient of torch.nn.utils.clip_grad_norm_ (norm_type 2): out[0] = ||g|| * pre_scale,
// out[1] = min(1, max_norm / (out[0] + 1e-6)) (1 when max_norm <= 0).  One CTA, fixed summation order.
__global__ void __launch_bounds__(256)
grad_clip_coef(const float* __restrict__ slabs, long long n, float pre_scale, float max_norm, float* __restrict__ out) {
  __shared__ float red[8];
  float acc = 0.f;
  for (long long i = threadIdx.x; i < n; i += 256) acc += slabs[i];
  const float t = block_sum_256(acc, red);
  if (threadIdx.x == 0) {
    const float norm = sqrtf(t) * pre_scale;
    out[0] = norm;
    out[1] = max_norm > 0.f ? fminf(1.f, max_norm / (norm + 1e-6f)) : 1.f;
  }
}

// Zero-padded NHWC copy for the conv weight-gradient GEMM: x [n, H, W, C] -> rows [guard | n*(H+2)*(W+2) | guard]
// of C channels, zero on the 1-pixel ring and in the guards.
__global__ void __launch_bounds__(256)
pad_nhwc_rows(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ out, int n, int H, int W, int C, int guard) {
  const int nvec = C >> 3;
  const long long rows = 2LL * guard + (long long)n * (H + 2) * (W + 2);
  const long long total = rows * nvec;
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    long long r0;
    int v;
    divmod_idx(i, nvec, r0, v);
    const long long r = r0 - guard;
    uint4 val = make_uint4(0, 0, 0, 0);
    if (r >= 0 && r < (long long)n * (H + 2) * (W + 2)) {
      long long ry, b;
      int xp, yp;
      divmod_idx(r, W + 2, ry, xp);
      divmod_idx(ry, H + 2, b, yp);
      if (xp >= 1 && xp <= W && yp >= 1 && yp <= H)
        val = *reinterpret_cast<const uint4*>(x + (((b * H + (yp - 1)) * W + (xp - 1)) * (long long)C) + v * 8);
    }
    reinterpret_cast<uint4*>(out)[i] = val;
  }
}

// Conv weight for the input-gradient convolution: Wf[ci][ky][kx][co] = W[co][2-ky][2-kx][ci]
// (grad_x = conv(grad_z, flipped and transposed W)).  W rows (one per co) are `w_ld` elements apart so that
// one level of the stacked pconv weight [Cout, L, 3, 3, Cin] can be addressed in place.  32x32 smem transpose.
__global__ void __launch_bounds__(256)
conv_weight_flip_t(const __nv_bfloat16* __restrict__ w, long long w_ld, __nv_bfloat16* __restrict__ wf, int Cin, int Cout) {
  __shared__ __nv_bfloat16 tile[32][33];
  const int tap = blockIdx.z;                    // source tap; destination tap 8 - tap
  const int ci0 = blockIdx.x * 32, co0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 32 x 8
  for (int j = ty; j < 32; j += 8) {
    const int co = co0 + j, ci = ci0 + tx;
    tile[j][tx] = (co < Cout && ci < Cin) ? w[(long long)co * w_ld + (long long)tap * Cin + ci] : __float2bfloat16(0.f);
  }
  __syncthreads();
  for (int j = ty; j < 32; j += 8) {
    const int ci = ci0 + j, co = co0 + tx;
    if (ci < Cin && co < Cout) wf[((long long)ci * 9 + (8 - tap)) * Cout + co] = tile[tx][j];
  }
}

// ------------------------------------------------------------------------------------------
// GroupNorm(64) + ReLU backward for the fuse convs (mmcv ConvModule: conv -> GN -> ReLU, conv_module.py:196-208).
//   z: raw conv output (bf16 NHWC, saved by the forward), y = z*scale + shift (scale/shift from gn_finalize),
//   dy = dA * [y > 0],  xh = (z - mean) * rstd
//   dbeta_c = sum dy,  dgamma_c = sum dy*xh
//   dz = rstd * (dy*gamma - mean_g(dy*gamma) - xh * mean_g(dy*gamma*xh))      (means over the group's H*W*cpg values)
// Pass 1 (gn_bwd_partial): per (image, pixel slab) partial sums of dy and dy*xh per channel -> slabs.
// Pass 2 (gn_bwd_reduce): slabs -> per-(image, channel) sums AB and per-(image, group) sums S1, S2; all in a
//         fixed order.  Pass 3 (gn_bwd_apply): elementwise dz.  gn_param_grad sums AB over the images.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
gn_mean_rstd(const float* __restrict__ stats, float* __restrict__ out, int B, int groups, int slots, float count, float eps) {
  const int w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (w >= B * groups) return;
  const int lane = threadIdx.x & 31;
  const int b = w / groups, g = w % groups;
  float s = 0.f, ss = 0.f;
  for (int t = lane; t < slots; t += 32) {     // same order as gn_finalize (elementwise.cu): identical mean / rstd
    const float2 v = *reinterpret_cast<const float2*>(stats + (((long long)b * slots + t) * groups + g) * 2);
    s += v.x;
    ss += v.y;
  }
  s = warp_sum_f(s);
  ss = warp_sum_f(ss);
  const float mean = s / count;
  float var = ss / count - mean * mean;
  var = var < 0.f ? 0.f : var;
  if (lane == 0) {
    out[(long long)w * 2] = mean;
    out[(long long)w * 2 + 1] = rsqrtf(var + eps);
  }
}

template <typename TA>
__device__ __forceinline__ void load8_any(const TA* p, float (&f)[8]) {
  if constexpr (sizeof(TA) == 2) {
    unpack8f(*reinterpret_cast<const uint4*>(p), f);
  } else {
    const float4 a = reinterpret_cast<const float4*>(p)[0], b = reinterpret_cast<const float4*>(p)[1];
    f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
  }
}

// grid (S, B), block = C/8 threads (one 8-channel vector each)
template <typename TA>
__global__ void gn_bwd_partial(const __nv_bfloat16* __restrict__ z, const TA* __restrict__ dA, const float* __restrict__ scale,
                               const float* __restrict__ shift, const float* __restrict__ mean_rstd,
                               float* __restrict__ slabs, int HW, int C, int groups) {
  const int b = blockIdx.y, s = blockIdx.x, S = gridDim.x;
  const int c0 = threadIdx.x * 8;
  const int cpg = C / groups;
  float sc[8], sh[8], a[8], bb[8];
  const float mean = mean_rstd[((long long)b * groups + c0 / cpg) * 2], rstd = mean_rstd[((long long)b * groups + c0 / cpg) * 2 + 1];
#pragma unroll
  for (int j = 0; j < 8; j++) { sc[j] = scale[(long long)b * C + c0 + j]; sh[j] = shift[(long long)b * C + c0 + j]; a[j] = 0.f; bb[j] = 0.f; }
  for (int pix = s; pix < HW; pix += S) {
    const long long off = ((long long)b * HW + pix) * C + c0;
    float zf[8], df[8];
    unpack8f(*reinterpret_cast<const uint4*>(z + off), zf);
    load8_any<TA>(dA + off, df);
#pragma unroll
    for (int j = 0; j < 8; j++) {
      const float dy = (zf[j] * sc[j] + sh[j] > 0.f) ? df[j] : 0.f;
      a[j] += dy;
      bb[j] += dy * ((zf[j] - mean) * rstd);
    }
  }
  float* o = slabs + (((long long)b * S + s) * 2) * C + c0;
#pragma unroll
  for (int j = 0; j < 8; j++) { o[j] = a[j]; o[C + j] = bb[j]; }
}

// grid B, block 256: AB[b][0/1][c] = sum_s slabs;  gs[b][g] = (sum_c gamma*A, sum_c gamma*B) over the group's channels
__global__ void __launch_bounds__(256)
gn_bwd_reduce(const float* __restrict__ slabs, const __nv_bfloat16* __restrict__ gamma, float* __restrict__ AB,
              float* __restrict__ gs, int S, int C, int groups) {
  extern __shared__ float sm_ab[];   // [2][C]
  const int b = blockIdx.x;
  for (int i = threadIdx.x; i < 2 * C; i += 256) {
    float acc = 0.f;
    for (int s = 0; s < S; s++) acc += slabs[(((long long)b * S + s) * 2) * C + i];
    sm_ab[i] = acc;
    AB[(long long)b * 2 * C + i] = acc;
  }
  __syncthreads();
  const int cpg = C / groups;
  for (int g = threadIdx.x; g < groups; g += 256) {
    float s1 = 0.f, s2 = 0.f;
    for (int j = 0; j < cpg; j++) {
      const float gm = __bfloat162float(gamma[g * cpg + j]);
      s1 += gm * sm_ab[g * cpg + j];
      s2 += gm * sm_ab[C + g * cpg + j];
    }
    gs[((long long)b * groups + g) * 2] = s1;
    gs[((long long)b * groups + g) * 2 + 1] = s2;
  }
}

template <typename TA>
__global__ void __launch_bounds__(256)
gn_bwd_apply(const __nv_bfloat16* __restrict__ z, const TA* __restrict__ dA, const float* __restrict__ scale,
             const float* __restrict__ shift, const float* __restrict__ mean_rstd, const float* __restrict__ gs,
             const __nv_bfloat16* __restrict__ gamma, __nv_bfloat16* __restrict__ dz, int B, int HW, int C, int groups) {
  const int nvec = C >> 3, cpg = C / groups;
  const long long total = (long long)B * HW * nvec;
  const float inv_n = 1.f / ((float)HW * cpg);
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    long long pixel, bq;
    int v, hw_r;
    divmod_idx(i, nvec, pixel, v);
    divmod_idx(pixel, HW, bq, hw_r);
    const int b = (int)bq;
    const int c0 = v * 8, g = c0 / cpg;
    const float mean = mean_rstd[((long long)b * groups + g) * 2], rstd = mean_rstd[((long long)b * groups + g) * 2 + 1];
    const float m1 = gs[((long long)b * groups + g) * 2] * inv_n, m2 = gs[((long long)b * groups + g) * 2 + 1] * inv_n;
    float zf[8], df[8], gm[8], o[8];
    unpack8f(*reinterpret_cast<const uint4*>(z + i * 8), zf);
    load8_any<TA>(dA + i * 8, df);
    unpack8f(*reinterpret_cast<const uint4*>(gamma + c0), gm);
#pragma unroll
    for (int j = 0; j < 8; j++) {
      const float y = zf[j] * scale[(long long)b * C + c0 + j] + shift[(long long)b * C + c0 + j];
      const float dy = y > 0.f ? df[j] : 0.f;
      const float xh = (zf[j] - mean) * rstd;
      o[j] = rstd * (dy * gm[j] - m1 - xh * m2);
    }
    *reinterpret_cast<uint4*>(dz + i * 8) = pack8f(o);
  }
}

// dbeta[c] (+)= sum_b AB[b][0][c];  dgamma[c] (+)= sum_b AB[b][1][c]
__global__ void __launch_bounds__(256)
gn_param_grad(const float* __restrict__ AB, int B, int C, float* __restrict__ dgamma, float* __restrict__ dbeta, int accumulate) {
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c >= C) return;
  float a = 0.f, bsum = 0.f;
  for (int b = 0; b < B; b++) { a += AB[(long long)b * 2 * C + c]; bsum += AB[(long long)b * 2 * C + C + c]; }
  dbeta[c] = (accumulate ? dbeta[c] : 0.f) + a;
  dgamma[c] = (accumulate ? dgamma[c] : 0.f) + bsum;
}

// out = y > 0 ? dy : 0   (ReLU backward from the saved OUTPUT y; bf16, n multiple of 8)
__global__ void __launch_bounds__(256)
relu_bwd_rows(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ y, __nv_bfloat16* __restrict__ out, long long nvec) {
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < nvec; i += (long long)gridDim.x * 256) {
    float d[8], v[8];
    unpack8f(reinterpret_cast<const uint4*>(dy)[i], d);
    unpack8f(reinterpret_cast<const uint4*>(y)[i], v);
#pragma unroll
    for (int j = 0; j < 8; j++) d[j] = v[j] > 0.f ? d[j] : 0.f;
    reinterpret_cast<uint4*>(out)[i] = pack8f(d);
  }
}

static unsigned grid_for(long long work_items) {
  long long g = (work_items + 255) / 256;
  const long long cap = (long long)num_sms() * 16;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (unsigned)g;
}

}  // namespace g4r

using namespace g4r;

extern "C" int g4r_cross_entropy_bf16(const void* logits, long long ld, const long long* targets, int M, int V,
                                      float* row_lse, float* row_loss, float* loss_count, void* dlogits,
                                      long long ldd, float grad_scale, void* stream) {
  G4R_REQUIRE(logits && targets && row_lse && row_loss && loss_count && M > 0 && V > 0 && ld >= V,
              "cross_entropy: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  ce_rows_fwd<<<M, 256, 0, st>>>((const __nv_bfloat16*)logits, ld, targets, row_loss, row_lse, V);
  G4R_LAUNCH_CHECK("ce_rows_fwd");
  ce_reduce<<<1, 256, 0, st>>>(row_loss, targets, M, V, loss_count);
  G4R_LAUNCH_CHECK("ce_reduce");
  if (dlogits) {
    G4R_REQUIRE(ldd >= V, "cross_entropy: ldd < V");
    ce_rows_bwd<<<M, 256, 0, st>>>((const __nv_bfloat16*)logits, ld, targets, row_lse, loss_count,
                                   (__nv_bfloat16*)dlogits, ldd, V, grad_scale);
    G4R_LAUNCH_CHECK("ce_rows_bwd");
  }
  return G4R_OK;
}

extern "C" int g4r_rmsnorm_bwd_slabs(int M) {
  const int cap = 2 * num_sms();
  return M < cap ? M : cap;
}

extern "C" int g4r_rmsnorm_bwd_bf16(const void* x, long long ldx, const void* w, const void* dy, long long ldy,
                                    const void* dres, long long ldr, void* dx, long long ldd, float* dw,
                                    float* dw_slabs, int M, int D, float eps, void* stream) {
  G4R_REQUIRE(dres == nullptr || ldr % 8 == 0, "rmsnorm_bwd: dres rows must be 16-byte aligned");
  G4R_REQUIRE(x && w && dy && dx && dw && dw_slabs && M > 0, "rmsnorm_bwd: null operand");
  G4R_REQUIRE(D % 8 == 0 && D <= 8192 && ldx % 8 == 0 && ldy % 8 == 0 && ldd % 8 == 0, "rmsnorm_bwd: D=%d (multiple of 8, <= 8192), 16-byte rows", D);
  cudaStream_t st = (cudaStream_t)stream;
  const int S = g4r_rmsnorm_bwd_slabs(M);
  const int per = (D / 8 + 255) / 256;
#define G4R_RMSB(P)                                                                                              \
  rmsnorm_bwd_rows<P><<<S, 256, 0, st>>>((const __nv_bfloat16*)x, ldx, (const __nv_bfloat16*)w,                  \
                                         (const __nv_bfloat16*)dy, ldy, (const __nv_bfloat16*)dres, ldr,          \
                                         (__nv_bfloat16*)dx, ldd, dw_slabs, M, D, eps)
  if (per <= 1) G4R_RMSB(1); else if (per <= 2) G4R_RMSB(2); else G4R_RMSB(4);
#undef G4R_RMSB
  G4R_LAUNCH_CHECK("rmsnorm_bwd_rows");
  slab_reduce_f32<<<(D + 255) / 256, 256, 0, st>>>(dw_slabs, S, D, dw);
  G4R_LAUNCH_CHECK("slab_reduce_f32");
  return G4R_OK;
}

static int gn_bwd_slabs(int HW) { return HW < 64 ? HW : 64; }

extern "C" long long g4r_gn_relu_bwd_workspace(int B, int HW, int C, int groups) {
  return (long long)B * gn_bwd_slabs(HW) * 2 * C + (long long)B * 2 * C + (long long)B * groups * 4;
}

extern "C" int g4r_gn_relu_bwd_bf16(const void* z, const void* dA, int dA_f32, const float* scale, const float* shift,
                                    const float* stats, int slots, float count, float eps, const void* gamma, void* dz,
                                    float* dgamma, float* dbeta, int accumulate, float* workspace, int B, int HW, int C,
                                    int groups, void* stream) {
  G4R_REQUIRE(z && dA && scale && shift && stats && gamma && dz && dgamma && dbeta && workspace, "gn_relu_bwd: null argument");
  G4R_REQUIRE(B > 0 && HW > 0 && groups > 0 && C % groups == 0 && (C / groups) % 8 == 0 && C / 8 <= 1024,
              "gn_relu_bwd: C=%d groups=%d (channels per group must be a multiple of 8)", C, groups);
  cudaStream_t st = (cudaStream_t)stream;
  const int S = gn_bwd_slabs(HW);
  float* slabs = workspace;
  float* AB = slabs + (long long)B * S * 2 * C;
  float* gs = AB + (long long)B * 2 * C;
  float* mr = gs + (long long)B * groups * 2;
  gn_mean_rstd<<<(B * groups + 7) / 8, 256, 0, st>>>(stats, mr, B, groups, slots, count, eps);
  G4R_LAUNCH_CHECK("gn_mean_rstd");
  dim3 grid(S, B);
  if (dA_f32) gn_bwd_partial<float><<<grid, C / 8, 0, st>>>((const __nv_bfloat16*)z, (const float*)dA, scale, shift, mr, slabs, HW, C, groups);
  else gn_bwd_partial<__nv_bfloat16><<<grid, C / 8, 0, st>>>((const __nv_bfloat16*)z, (const __nv_bfloat16*)dA, scale, shift, mr, slabs, HW, C, groups);
  G4R_LAUNCH_CHECK("gn_bwd_partial");
  gn_bwd_reduce<<<B, 256, 2 * C * sizeof(float), st>>>(slabs, (const __nv_bfloat16*)gamma, AB, gs, S, C, groups);
  G4R_LAUNCH_CHECK("gn_bwd_reduce");
  const long long total = (long long)B * HW * (C / 8);
  if (dA_f32) gn_bwd_apply<float><<<grid_for(total), 256, 0, st>>>((const __nv_bfloat16*)z, (const float*)dA, scale, shift, mr, gs,
                                                                   (const __nv_bfloat16*)gamma, (__nv_bfloat16*)dz, B, HW, C, groups);
  else gn_bwd_apply<__nv_bfloat16><<<grid_for(total), 256, 0, st>>>((const __nv_bfloat16*)z, (const __nv_bfloat16*)dA, scale, shift, mr, gs,
                                                                     (const __nv_bfloat16*)gamma, (__nv_bfloat16*)dz, B, HW, C, groups);
  G4R_LAUNCH_CHECK("gn_bwd_apply");
  gn_param_grad<<<(C + 255) / 256, 256, 0, st>>>(AB, B, C, dgamma, dbeta, accumulate);
  G4R_LAUNCH_CHECK("gn_param_grad");
  return G4R_OK;
}

extern "C" int g4r_relu_bwd_bf16(const void* dy, const void* y, void* out, long long n, void* stream) {
  G4R_REQUIRE(dy && y && out && n > 0 && n % 8 == 0, "relu_bwd: n must be a positive multiple of 8");
  relu_bwd_rows<<<grid_for(n / 8), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)y, (__nv_bfloat16*)out, n / 8);
  G4R_LAUNCH_CHECK("relu_bwd_rows");
  return G4R_OK;
}

extern "C" int g4r_pad_nhwc_bf16(const void* x, void* out, int n, int H, int W, int C, int guard_rows, void* stream) {
  G4R_REQUIRE(x && out && n > 0 && H > 0 && W > 0 && C % 8 == 0 && guard_rows >= W + 3, "pad_nhwc: bad arguments (guard_rows >= W+3)");
  const long long total = (2LL * guard_rows + (long long)n * (H + 2) * (W + 2)) * (C / 8);
  pad_nhwc_rows<<<grid_for(total), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)out, n, H, W, C, guard_rows);
  G4R_LAUNCH_CHECK("pad_nhwc_rows");
  return G4R_OK;
}

extern "C" int g4r_conv_weight_flip_t_bf16(const void* w, long long w_ld, void* wf, int Cin, int Cout, void* stream) {
  G4R_REQUIRE(w && wf && Cin > 0 && Cout > 0 && w_ld >= 9LL * Cin, "conv_weight_flip_t: bad arguments");
  dim3 grid((Cin + 31) / 32, (Cout + 31) / 32, 9);
  conv_weight_flip_t<<<grid, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)w, w_ld, (__nv_bfloat16*)wf, Cin, Cout);
  G4R_LAUNCH_CHECK("conv_weight_flip_t");
  return G4R_OK;
}

extern "C" int g4r_colsum_slabs(int M) { return M < 64 ? (M > 0 ? M : 1) : 64; }

extern "C" int g4r_colsum_bf16(const void* x, long long ld, int M, int N, float* out, float* slabs, void* stream) {
  G4R_REQUIRE(x && out && slabs && M > 0 && N > 0 && N % 8 == 0 && ld % 8 == 0, "colsum: bad arguments (N, ld multiples of 8)");
  cudaStream_t st = (cudaStream_t)stream;
  const int S = g4r_colsum_slabs(M);
  dim3 grid((N + 2047) / 2048, S);
  colsum_rows<<<grid, 256, 0, st>>>((const __nv_bfloat16*)x, ld, M, N, slabs);
  G4R_LAUNCH_CHECK("colsum_rows");
  slab_reduce_f32<<<(N + 255) / 256, 256, 0, st>>>(slabs, S, N, out);
  G4R_LAUNCH_CHECK("slab_reduce_f32");
  return G4R_OK;
}

extern "C" int g4r_swiglu_fwd_bf16(const void* gu, long long ldg, void* f, long long ldf, long long M, int F,
                                   void* stream) {
  G4R_REQUIRE(gu && f && M > 0 && F > 0 && F % 4 == 0 && ldg % 8 == 0 && ldf % 4 == 0, "swiglu_fwd: bad arguments");
  swiglu_fwd<<<grid_for(M * (F / 4)), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)gu, ldg, (__nv_bfloat16*)f, ldf, M, F);
  G4R_LAUNCH_CHECK("swiglu_fwd");
  return G4R_OK;
}

extern "C" int g4r_swiglu_bwd_bf16(const void* gu, long long ldg, const void* df, long long ldf, void* dgu,
                                   long long ldd, long long M, int F, void* stream) {
  G4R_REQUIRE(gu && df && dgu && M > 0 && F > 0 && F % 4 == 0 && ldg % 8 == 0 && ldf % 4 == 0 && ldd % 8 == 0,
              "swiglu_bwd: bad arguments");
  swiglu_bwd<<<grid_for(M * (F / 4)), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)gu, ldg, (const __nv_bfloat16*)df, ldf,
                                                                    (__nv_bfloat16*)dgu, ldd, M, F);
  G4R_LAUNCH_CHECK("swiglu_bwd");
  return G4R_OK;
}

static int adamw_launch(float* p, const void* g, int g_bf16, float* m, float* v, void* p_bf16, long long n,
                        float lr, float beta1, float beta2, float eps, float weight_decay, int step,
                        float grad_scale, const float* scale_dev, void* stream) {
  G4R_REQUIRE(p && g && m && v && n > 0 && step >= 1, "adamw: bad arguments");
  G4R_REQUIRE(((uintptr_t)p & 15) == 0 && ((uintptr_t)m & 15) == 0 && ((uintptr_t)v & 15) == 0 &&
              ((uintptr_t)g & (g_bf16 ? 7 : 15)) == 0 && ((uintptr_t)p_bf16 & 7) == 0,
              "adamw: tensors must be 16-byte aligned (8 for the bf16 ones)");
  const float bc1 = 1.f - powf(beta1, (float)step);
  const float bc2s = sqrtf(1.f - powf(beta2, (float)step));
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = grid_for((n + 3) / 4);
  if (g_bf16)
    adamw_step<__nv_bfloat16><<<grid, 256, 0, st>>>(p, (const __nv_bfloat16*)g, m, v, (__nv_bfloat16*)p_bf16, n, lr,
                                                     beta1, beta2, eps, weight_decay, bc1, bc2s, grad_scale, scale_dev);
  else
    adamw_step<float><<<grid, 256, 0, st>>>(p, (const float*)g, m, v, (__nv_bfloat16*)p_bf16, n, lr, beta1, beta2,
                                            eps, weight_decay, bc1, bc2s, grad_scale, scale_dev);
  G4R_LAUNCH_CHECK("adamw_step");
  return G4R_OK;
}

extern "C" int g4r_adamw_step(float* p, const void* g, int g_bf16, float* m, float* v, void* p_bf16, long long n,
                              float lr, float beta1, float beta2, float eps, float weight_decay, int step,
                              float grad_scale, void* stream) {
  return adamw_launch(p, g, g_bf16, m, v, p_bf16, n, lr, beta1, beta2, eps, weight_decay, step, grad_scale, nullptr, stream);
}

extern "C" int g4r_adamw_step_ex(float* p, const void* g, int g_bf16, float* m, float* v, void* p_bf16, long long n,
                                 float lr, float beta1, float beta2, float eps, float weight_decay, int step,
                                 float grad_scale, const float* scale_dev, void* stream) {
  return adamw_launch(p, g, g_bf16, m, v, p_bf16, n, lr, beta1, beta2, eps, weight_decay, step, grad_scale, scale_dev, stream);
}

extern "C" int g4r_sumsq_slabs(void) { return kSumsqSlabs; }

extern "C" int g4r_sumsq(const void* g, int g_bf16, long long n, float* slab, void* stream) {
  G4R_REQUIRE(g && slab && n > 0, "sumsq: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (g_bf16) sumsq_partial<__nv_bfloat16><<<kSumsqSlabs, 256, 0, st>>>((const __nv_bfloat16*)g, n, slab);
  else sumsq_partial<float><<<kSumsqSlabs, 256, 0, st>>>((const float*)g, n, slab);
  G4R_LAUNCH_CHECK("sumsq_partial");
  return G4R_OK;
}

extern "C" int g4r_grad_clip_coef(const float* slabs, long long n_slabs, float pre_scale, float max_norm, float* out2,
                                  void* stream) {
  G4R_REQUIRE(slabs && out2 && n_slabs > 0, "grad_clip_coef: bad arguments");
  grad_clip_coef<<<1, 256, 0, (cudaStream_t)stream>>>(slabs, n_slabs, pre_scale, max_norm, out2);
  G4R_LAUNCH_CHECK("grad_clip_coef");
  return G4R_OK;
}
