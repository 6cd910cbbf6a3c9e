// gemm_wgmma.cu -- bf16 x bf16 -> fp32 dense contraction on the Hopper tensor cores (sm_90a, wgmma).
//
// One persistent, warp-specialised kernel serves every dense op of the region-token path:
//   D[M,N] = epilogue( A[M,K] . B[N,K]^T )           (GEMM: nn.Linear weights are [N,K] K-major)
//   D[n,y,x,:] = epilogue( conv3x3(A[n,:,:,:]) )      (implicit GEMM, NHWC, K = 9*Cin, pad 1)
// replacing the library calls the reference makes through ATen (cuBLAS / cuDNN):
//   nn.Linear            : gpt4roi/models/layers.py:260-270 (pos_embedd, updims, flatten_linear),
//                          llava/model/llava.py:52 (mm_projector), :195 (lm_head), HF CLIP / LLaMA linears
//   nn.Conv2d 1x1 / 3x3  : gpt4roi/models/layers.py:129-144 (input_conv, fuse_convs), :257-259 (pconvs)
//
// Structure (per CTA, 1 CTA / SM, persistent over 128 x BN output tiles, BN = 128 or 256; 3 warpgroups):
//   warpgroup 0, one thread : TMA producer -- cp.async.bulk.tensor loads of the A tile [128 x 64] and the
//                B tile [BN x 64] (128-byte swizzle) into a Stages-deep smem ring (4 stages at BN = 128,
//                3 at 256), completion signalled on `full` mbarriers (expect_tx).  In conv mode the A tile
//                is a 4-D box (64 ch, BW, BH, 1) of the NHWC map shifted by the filter tap; out-of-bounds
//                coordinates are zero-filled by TMA = the padding.
//   warpgroups 1, 2 : consumers -- each issues wgmma m64nBNk16 for its 64 rows of the tile (fp32
//                accumulators in registers) and releases the smem slot (`empty`) once its MMAs have read it.
//                After the last k-block a 16-bit output (forward GEMMs, no split-K, 16-bit or no residual,
//                TMA-aligned rows) takes the register epilogue (epilogue_regs): each warpgroup finishes its
//                accumulators in place -- bias / activation / residual / SwiGLU / RoPE -- into 64 x 64 swizzled
//                boxes in shared memory, one thread stores them with TMA, and the warpgroup goes on to its next
//                tile; the residual was loaded by TMA into those boxes while the MMAs ran.  Everything else (fp32
//                outputs and residuals, split-K, convs with GroupNorm statistics, the training GEMMs) stages the
//                accumulators in shared memory, 128 columns at a time, and runs epilogue_tile on each half:
//                thread = (row, half of the columns), 32 columns at a time.  Meanwhile the producer is already
//                loading the next tile's operands.
// The operand majorness (TA, TB) is a template parameter, so each mainloop is straight-line code: every
// k-block's four MMAs and their commit_group sit in one basic block, and wait_group 1 keeps one k-block of
// MMAs in flight.  At BN = 256 the 128 accumulators per consumer thread need setmaxnreg: the producer
// warpgroup gives its registers up (40 per thread) and the consumers grow to 232 (128*40 + 256*232 <= 64 K).
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "ptx.cuh"
#include "act_type.cuh"   // bf16 as written; fp16 twin with -DG4R_ACT_HALF

namespace G4R_NS {

constexpr int kBlockM = 128;
constexpr int kEpiN = 128;   // columns staged and drained per epilogue pass (one 128-dim RoPE head)
constexpr int kBlockK = 64;  // 64 bf16 = 128 B = one swizzle atom
constexpr int kMmaK = 16;
constexpr int kGemmThreads = 384;
constexpr int kConsumerThreads = 256;
constexpr int kProducerRegs = 40;    // setmaxnreg at BN = 256: producer warpgroup ...
constexpr int kConsumerRegs = 232;   // ... and each consumer warpgroup
static_assert(128 * kProducerRegs + kConsumerThreads * kConsumerRegs <= 64 * 1024, "register file");

enum { ACT_NONE = 0, ACT_RELU = 1, ACT_QUICK_GELU = 2, ACT_SWIGLU = 3 };

struct GemmParams {
  int M, N, K;
  int num_m_tiles, num_n_tiles, num_k_blocks;  // num_k_blocks: per split
  int k_splits;
  int n_fast;  // tile order: 1 = n-tile index fastest (conv: the big NHWC input is read from DRAM once and
               // its weight panels stay in L2), 0 = m fastest (GEMM: weight panels stream once)
  // epilogue
  void* D;
  long long ldd;
  const void* bias;      // [N] bf16 or fp32 (bias_f32), or null
  int bias_f32;
  const __nv_bfloat16* residual;  // same row mapping as D, or null (bf16, or fp32 when residual_f32)
  int residual_f32;
  int round_branch;  // round (acc + bias, act) to bf16 before the residual add (bf16 linear output + fp32 stream)
  long long ldr;
  int act;
  int out_f32;   // 1: fp32 output
  int d_vec, r_vec;  // D / residual rows take 16-byte vector accesses: 16-byte aligned base and row pitch (launch_gemm)
  int tma_epi;       // register epilogue with TMA stores (epilogue_regs): tmap_d / tmap_r describe D and the residual
  // conv mode
  int conv;
  int cH, cW, cBH, cBW, tiles_x, tiles_y, cin_blocks, taps;  // taps = 9 (3x3) or 1
  int a_rows;            // rows delivered by the A box (<= 128)
  int levels, lvl_img_stride;  // conv: sum over `levels` inputs (image index + lvl*stride), K concatenated
  // fused rotary embedding (LLaMA QKV GEMM): columns [0, rope_cols) are heads of 128 dims rotated with
  // bf16 cos/sin tables [rope_L][128]; row position = out_row % rope_L
  const __nv_bfloat16* rope_cos;
  const __nv_bfloat16* rope_sin;
  int rope_cols, rope_L, rope_pos0;
  const int* rope_pos_dev;  // optional device-side position base (CUDA-graph decode): pos0 = *rope_pos_dev
  const int* rope_pos_rows; // optional per-sample bases [M / rope_L] (prompts of different lengths); wins over both
  // operand majorness (backward GEMMs): a_mn: A is stored [K][M] (M contiguous); b_mn: B is stored [K][N];
  // b_mn == 2 (conv weight gradient): B is the zero-padded NHWC input seen through a 4-D tensor map
  // {Cin, kx, row, ky} whose kx / ky dimensions alias the row dimension (strides of 1 and W+2 rows), so that
  // column block n = (tap, cin) of the virtual [rows, 9*Cin] matrix is the input shifted by that tap
  int a_mn, b_mn, dw_cin;
  float* gn_stats;       // optional [n_img, groups, 2] (sum, sumsq) of the bf16-rounded output
  int gn_group_ch;       // channels per group (16)
  int gn_groups;         // groups per image (64)
};

// Shared memory: BN = 128: 4 stages x 32 KB + 66 KB staging = 194 KB;
//                BN = 256: 3 stages x 48 KB + 66 KB staging = 210 KB (a 4th stage does not fit beside the staging tile).
// The register epilogue's boxes (2 warpgroups x BN / 64 boxes of 8 KB: 32 or 64 KB) reuse the staging tile.
template <int BN>
struct GemmCfg {
  static constexpr int kStages = BN == 256 ? 3 : 4;
  static constexpr int kABytes = kBlockM * kBlockK * 2;   // 16 KB
  static constexpr int kBBytes = BN * kBlockK * 2;        // 16 or 32 KB
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kAccLd = kEpiN + 4;                // fp32 staging row stride (conflict-free row reads)
  static constexpr int kAccBytes = kBlockM * kAccLd * 4;  // 66 KB
  static constexpr int kBarBytes = (2 * kStages + 2) * 8;
  static constexpr int kSmemBytes = kStages * kStageBytes + kAccBytes + kBarBytes + 1024;  // +1024 alignment slack
  // register epilogue: each consumer warpgroup's 64 x BN output block as BN / 64 TMA boxes of 64 rows x 128 B,
  // in the region of the fp32 staging tile
  static constexpr int kBoxBytes = 64 * 128;
  static constexpr int kWgStageBytes = (BN / 64) * kBoxBytes;
  static_assert(2 * kWgStageBytes <= kAccBytes, "register-epilogue staging exceeds the staging tile");
};
static_assert(GemmCfg<128>::kSmemBytes <= 227 * 1024, "GEMM shared memory exceeds the sm_90 per-block limit");
static_assert(GemmCfg<256>::kSmemBytes <= 227 * 1024, "GEMM shared memory exceeds the sm_90 per-block limit");

__device__ __forceinline__ float act_apply(float x, int act) {
  if (act == ACT_RELU) return fmaxf(x, 0.f);
  if (act == ACT_QUICK_GELU) return x / (1.f + __expf(-1.702f * x));
  return x;
}

// 32 consecutive fp32 accumulator columns of this thread's row from the staging tile
__device__ __forceinline__ void acc_ld32(const float* srow, int c0, float (&f)[32]) {
#pragma unroll
  for (int h = 0; h < 8; h++) {
    const float4 v = *reinterpret_cast<const float4*>(srow + c0 + 4 * h);
    f[4 * h] = v.x; f[4 * h + 1] = v.y; f[4 * h + 2] = v.z; f[4 * h + 3] = v.w;
  }
}

// Epilogue of one 128 x 128 accumulator block staged in shared memory, output columns [col_base, col_base + 128):
// thread (`row`, `half`) handles the 32-column chunks half, half + 2 (RoPE: the head's dims [32*half, 32*half + 32)
// and their partners 64 apart).
template <bool CONV>
__device__ __forceinline__ void epilogue_tile(const GemmParams& p, const float* srow, int m_blk, int col_base,
                                              int split, int row, int half, int lane) {
  constexpr int BLOCK_N = kEpiN;
  // row -> output row offset
  bool row_ok;
  long long out_row;
  int img = 0;
  if (CONV) {
    const int tx = m_blk % p.tiles_x;
    const int ty = (m_blk / p.tiles_x) % p.tiles_y;
    img = m_blk / (p.tiles_x * p.tiles_y);
    const int y = ty * p.cBH + row / p.cBW, x = tx * p.cBW + row % p.cBW;
    row_ok = m_blk < p.num_m_tiles && row < p.a_rows && y < p.cH && x < p.cW;
    out_row = ((long long)img * p.cH + y) * p.cW + x;
  } else {
    out_row = (long long)m_blk * kBlockM + row;
    row_ok = m_blk < p.num_m_tiles && out_row < p.M;
  }
  if (!CONV && p.rope_cos != nullptr && col_base < p.rope_cols) {
    // ---- fused RoPE (transformers modeling_llama.py:138-168): the tile holds one whole head of 128 dims;
    // dims (d, d+64) of a head are 64 columns apart -> load both 32-column chunks, rotate, store.
    // Rounding as in the reference: q/k are bf16 GEMM outputs, each bf16 tensor op rounds:
    //   out = bf16( bf16(x*cos) + bf16(rot*sin) ),  rotate_half(x) = cat(-x2, x1).
    if (!row_ok) return;
    const int base = p.rope_pos_rows ? p.rope_pos_rows[out_row / p.rope_L] : (p.rope_pos_dev ? *p.rope_pos_dev : p.rope_pos0);
    const int pos = base + (int)(out_row % p.rope_L);
    const __nv_bfloat16* ct = p.rope_cos + (long long)pos * 128;
    const __nv_bfloat16* st = p.rope_sin + (long long)pos * 128;
#pragma unroll 1
    for (int hc = half; hc < BLOCK_N / 64; hc += 2) {   // hc = head*2 + half-chunk (0: dims 0-31, 1: dims 32-63)
      const int cA = (hc >> 1) * 128 + (hc & 1) * 32, cB = cA + 64;
      float va[32], vb[32];
      acc_ld32(srow, cA, va);
      acc_ld32(srow, cB, vb);
      const int d0 = (hc & 1) * 32;
      uint32_t oa[16], ob[16];
#pragma unroll
      for (int h8 = 0; h8 < 4; h8++) {
        const uint4 c1r = *reinterpret_cast<const uint4*>(ct + d0 + h8 * 8);
        const uint4 s1r = *reinterpret_cast<const uint4*>(st + d0 + h8 * 8);
        const uint4 c2r = *reinterpret_cast<const uint4*>(ct + 64 + d0 + h8 * 8);
        const uint4 s2r = *reinterpret_cast<const uint4*>(st + 64 + d0 + h8 * 8);
        const __nv_bfloat16* c1 = reinterpret_cast<const __nv_bfloat16*>(&c1r);
        const __nv_bfloat16* s1 = reinterpret_cast<const __nv_bfloat16*>(&s1r);
        const __nv_bfloat16* c2 = reinterpret_cast<const __nv_bfloat16*>(&c2r);
        const __nv_bfloat16* s2 = reinterpret_cast<const __nv_bfloat16*>(&s2r);
        float r1[8], r2[8];
#pragma unroll
        for (int j = 0; j < 8; j++) {
          const float x1 = __bfloat162float(__float2bfloat16_rn(va[h8 * 8 + j]));
          const float x2 = __bfloat162float(__float2bfloat16_rn(vb[h8 * 8 + j]));
          const float a1 = __bfloat162float(__float2bfloat16_rn(x1 * __bfloat162float(c1[j])));
          const float b1 = __bfloat162float(__float2bfloat16_rn(-x2 * __bfloat162float(s1[j])));
          const float a2 = __bfloat162float(__float2bfloat16_rn(x2 * __bfloat162float(c2[j])));
          const float b2 = __bfloat162float(__float2bfloat16_rn(x1 * __bfloat162float(s2[j])));
          r1[j] = a1 + b1;
          r2[j] = a2 + b2;
        }
#pragma unroll
        for (int j = 0; j < 4; j++) {
          __nv_bfloat162 h1 = __floats2bfloat162_rn(r1[2 * j], r1[2 * j + 1]);
          __nv_bfloat162 h2 = __floats2bfloat162_rn(r2[2 * j], r2[2 * j + 1]);
          oa[h8 * 4 + j] = *reinterpret_cast<uint32_t*>(&h1);
          ob[h8 * 4 + j] = *reinterpret_cast<uint32_t*>(&h2);
        }
      }
      __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.D) + out_row * p.ldd + col_base;
#pragma unroll
      for (int h4 = 0; h4 < 4; h4++) {
        reinterpret_cast<uint4*>(o + cA)[h4] = make_uint4(oa[4 * h4], oa[4 * h4 + 1], oa[4 * h4 + 2], oa[4 * h4 + 3]);
        reinterpret_cast<uint4*>(o + cB)[h4] = make_uint4(ob[4 * h4], ob[4 * h4 + 1], ob[4 * h4 + 2], ob[4 * h4 + 3]);
      }
    }
    return;
  }
#pragma unroll 1
  for (int c0 = half * 32; c0 < BLOCK_N; c0 += 64) {
    const int col0 = col_base + c0;
    if (col0 >= p.N) continue;  // (warp-uniform)
    float f[32];
    acc_ld32(srow, c0, f);
    const bool full_chunk = col0 + 32 <= p.N;
    if (p.bias != nullptr && split == 0) {
      if (p.bias_f32) {
        const float* b = reinterpret_cast<const float*>(p.bias) + col0;
#pragma unroll
        for (int j = 0; j < 32; j++) if (full_chunk || col0 + j < p.N) f[j] += b[j];
      } else {
        const __nv_bfloat16* b = reinterpret_cast<const __nv_bfloat16*>(p.bias) + col0;
#pragma unroll
        for (int j = 0; j < 32; j++) if (full_chunk || col0 + j < p.N) f[j] += __bfloat162float(b[j]);
      }
    }
    if (p.act == ACT_RELU || p.act == ACT_QUICK_GELU) {
#pragma unroll
      for (int j = 0; j < 32; j++) f[j] = act_apply(f[j], p.act);
    }
    if (p.act == ACT_SWIGLU) {
      // interleaved weights: column 2j = gate_j, 2j+1 = up_j -> out[:, j] = silu(gate) * up
      if (row_ok) {
        __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.D) + out_row * p.ldd + col0 / 2;
        uint32_t pk[8];
#pragma unroll
        for (int j = 0; j < 8; j++) {
          const float g0 = f[4 * j], u0 = f[4 * j + 1], g1 = f[4 * j + 2], u1 = f[4 * j + 3];
          const float s0 = g0 / (1.f + __expf(-g0)) * u0, s1 = g1 / (1.f + __expf(-g1)) * u1;
          __nv_bfloat162 h = __floats2bfloat162_rn(s0, s1);
          pk[j] = *reinterpret_cast<uint32_t*>(&h);
        }
        if (full_chunk && p.d_vec) {
          reinterpret_cast<uint4*>(o)[0] = make_uint4(pk[0], pk[1], pk[2], pk[3]);
          reinterpret_cast<uint4*>(o)[1] = make_uint4(pk[4], pk[5], pk[6], pk[7]);
        } else {
          const __nv_bfloat16* e = reinterpret_cast<const __nv_bfloat16*>(pk);
          for (int j = 0; j < 16; j++) if (col0 + 2 * j + 1 < p.N) o[j] = e[j];
        }
      }
      continue;
    }
    if (p.round_branch) {
#pragma unroll
      for (int j = 0; j < 32; j++) f[j] = __bfloat162float(__float2bfloat16_rn(f[j]));
    }
    if (p.residual != nullptr && row_ok) {
      if (p.residual_f32) {
        // fp32 residual stream (CLIP under autocast keeps it in fp32: LayerNorm outputs fp32 and
        // `residual + bf16_branch` promotes)
        const float* rr = reinterpret_cast<const float*>(p.residual) + out_row * p.ldr + col0;
        if (full_chunk && p.r_vec) {
#pragma unroll
          for (int h = 0; h < 8; h++) {
            const float4 r4 = reinterpret_cast<const float4*>(rr)[h];
            f[4 * h] += r4.x; f[4 * h + 1] += r4.y; f[4 * h + 2] += r4.z; f[4 * h + 3] += r4.w;
          }
        } else {
          for (int j = 0; j < 32; j++) if (col0 + j < p.N) f[j] += rr[j];
        }
      } else {
        const __nv_bfloat16* rr = p.residual + out_row * p.ldr + col0;
        if (full_chunk && p.r_vec) {
#pragma unroll
          for (int h = 0; h < 4; h++) {
            const uint4 raw = reinterpret_cast<const uint4*>(rr)[h];
            const __nv_bfloat16* e = reinterpret_cast<const __nv_bfloat16*>(&raw);
#pragma unroll
            for (int j = 0; j < 8; j++) f[h * 8 + j] += __bfloat162float(e[j]);
          }
        } else {
          for (int j = 0; j < 32; j++) if (col0 + j < p.N) f[j] += __bfloat162float(rr[j]);
        }
      }
    }
    if (p.out_f32) {
      if (row_ok) {
        // split-K: split s writes slab s of a [k_splits][M][ldd] fp32 buffer (no atomics; the consumer
        // sums the slabs in a fixed order, so the result is bitwise reproducible)
        float* o = reinterpret_cast<float*>(p.D) + ((long long)split * p.M + out_row) * p.ldd + col0;
        if (full_chunk && p.d_vec) {
#pragma unroll
          for (int h = 0; h < 8; h++)
            reinterpret_cast<float4*>(o)[h] = make_float4(f[4 * h], f[4 * h + 1], f[4 * h + 2], f[4 * h + 3]);
        } else {
          for (int j = 0; j < 32; j++) if (col0 + j < p.N) o[j] = f[j];
        }
      }
    } else {
      uint32_t pk[16];
#pragma unroll
      for (int j = 0; j < 16; j++) {
        __nv_bfloat162 h = __floats2bfloat162_rn(f[2 * j], f[2 * j + 1]);
        pk[j] = *reinterpret_cast<uint32_t*>(&h);
      }
      if (row_ok) {
        __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.D) + out_row * p.ldd + col0;
        if (full_chunk && p.d_vec) {
#pragma unroll
          for (int h = 0; h < 4; h++)
            reinterpret_cast<uint4*>(o)[h] = make_uint4(pk[4 * h], pk[4 * h + 1], pk[4 * h + 2], pk[4 * h + 3]);
        } else {
          const __nv_bfloat16* e = reinterpret_cast<const __nv_bfloat16*>(pk);
          for (int j = 0; j < 32; j++) if (col0 + j < p.N) o[j] = e[j];
        }
      }
      if (CONV && p.gn_stats != nullptr) {
        // GroupNorm statistics of the bf16-rounded conv output (what the reference's GN sees:
        // mmcv cnn/bricks/conv_module.py:196-208 runs GN on the conv's bf16 result).
        // 32 columns = 2 groups of 16 channels; reduce over the 32 rows of this warp, then ONE plain
        // store per (tile, warp) slot -- no atomics, so the statistics are bitwise reproducible;
        // gn_finalize sums the slots in a fixed order.  Lane l stores group col0 / 16 + l when that group lies
        // inside N: the last chunk of Cout = 16, 48, 80, ... holds one whole group.
        const __nv_bfloat16* e = reinterpret_cast<const __nv_bfloat16*>(pk);
        float s[2] = {0.f, 0.f}, ss[2] = {0.f, 0.f};
        if (row_ok) {
#pragma unroll
          for (int j = 0; j < 32; j++) {
            const float x = __bfloat162float(e[j]);
            s[j >> 4] += x;
            ss[j >> 4] += x * x;
          }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          s[0] += __shfl_xor_sync(0xffffffffu, s[0], o);
          s[1] += __shfl_xor_sync(0xffffffffu, s[1], o);
          ss[0] += __shfl_xor_sync(0xffffffffu, ss[0], o);
          ss[1] += __shfl_xor_sync(0xffffffffu, ss[1], o);
        }
        if (lane < 2 && col0 + 16 * (lane + 1) <= p.N && m_blk < p.num_m_tiles) {
          const int tiles_per_img = p.tiles_x * p.tiles_y;
          const int slot = (m_blk % tiles_per_img) * 4 + (row >> 5);
          float* st = p.gn_stats + (((long long)img * (tiles_per_img * 4) + slot) * p.gn_groups +
                                    (col0 / p.gn_group_ch + lane)) * 2;
          st[0] = lane == 0 ? s[0] : s[1];
          st[1] = lane == 0 ? ss[0] : ss[1];
        }
      }
    }
  }
}

// Epilogue of one consumer warpgroup's 64 x BN block straight from the accumulators (16-bit output, no split-K,
// no GroupNorm statistics, 16-bit or no residual; gemm_impl decides).  The same fp32 operations in the same order as
// epilogue_tile, so the output is bitwise the same.  The thread holds rows rl and rl + 8 of the block, columns
// 8j + 2(lane & 3) + {0, 1} (acc[4j + 2h + e]: row rl + 8h); each pair is finished, packed to 16 bits and written at
// once into `stg`, BN / 64 boxes of 64 rows x 128 B in the 128-byte swizzle of the D / residual tensor maps.  The
// residual, when there is one, has already been loaded by TMA into exactly those places, so each pair reads its
// residual where it then writes its output.  SwiGLU halves the columns: pair j of row r becomes output column
// 4j + (lane & 3).  Rows at or past M are computed but never stored (TMA clips the box).
template <int BN>
__device__ __forceinline__ void epilogue_regs(const GemmParams& p, float (&acc)[BN / 2], uint32_t stg, int row0,
                                              int col0, int wt) {
  constexpr int kBox = GemmCfg<BN>::kBoxBytes;
  const int lane = wt & 31, c = lane & 3;
  const int rl = (wt >> 5) * 16 + (lane >> 2);
  const int sw = lane >> 2;  // row & 7 of both rows: a row's 16-byte chunk index is xor-ed with it
  const uint32_t srow = stg + rl * 128;
  // pair (j, h): 16-byte chunk j & 7 of box j / 8, row rl + 8h
  auto pair_addr = [&](int j, int h) { return srow + h * 1024 + (j >> 3) * kBox + (((j & 7) ^ sw) << 4) + 4 * c; };
  if (p.rope_cos != nullptr && col0 < p.rope_cols) {
    // RoPE as in epilogue_tile: dims d and d + 64 of a head are accumulator blocks j and j + 8; the cos / sin values
    // of the thread's dims are the same for every head of the tile, so they are loaded once per row, up front
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const long long out_row = row0 + rl + 8 * h;
      int pos = 0;
      if (out_row < p.M) {
        const int base = p.rope_pos_rows ? p.rope_pos_rows[out_row / p.rope_L] : (p.rope_pos_dev ? *p.rope_pos_dev : p.rope_pos0);
        pos = base + (int)(out_row % p.rope_L);
      }
      const uint32_t* ct = reinterpret_cast<const uint32_t*>(p.rope_cos + (long long)pos * 128) + c;
      const uint32_t* st = reinterpret_cast<const uint32_t*>(p.rope_sin + (long long)pos * 128) + c;
      uint32_t c1[8], s1[8], c2[8], s2[8];
#pragma unroll
      for (int j = 0; j < 8; j++) {
        c1[j] = ct[4 * j]; s1[j] = st[4 * j]; c2[j] = ct[32 + 4 * j]; s2[j] = st[32 + 4 * j];
      }
#pragma unroll
      for (int hd = 0; hd < BN / 128; hd++) {
#pragma unroll
        for (int j = 0; j < 8; j++) {
          const int ja = hd * 16 + j, jb = ja + 8;
          const float2 fc1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&c1[j]));
          const float2 fs1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&s1[j]));
          const float2 fc2 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&c2[j]));
          const float2 fs2 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&s2[j]));
          float r1[2], r2[2];
#pragma unroll
          for (int e = 0; e < 2; e++) {
            const float x1 = __bfloat162float(__float2bfloat16_rn(acc[4 * ja + 2 * h + e]));
            const float x2 = __bfloat162float(__float2bfloat16_rn(acc[4 * jb + 2 * h + e]));
            const float cc1 = e ? fc1.y : fc1.x, ss1 = e ? fs1.y : fs1.x;
            const float cc2 = e ? fc2.y : fc2.x, ss2 = e ? fs2.y : fs2.x;
            const float a1 = __bfloat162float(__float2bfloat16_rn(x1 * cc1));
            const float b1 = __bfloat162float(__float2bfloat16_rn(-x2 * ss1));
            const float a2 = __bfloat162float(__float2bfloat16_rn(x2 * cc2));
            const float b2 = __bfloat162float(__float2bfloat16_rn(x1 * ss2));
            r1[e] = a1 + b1;
            r2[e] = a2 + b2;
          }
          __nv_bfloat162 o1 = __floats2bfloat162_rn(r1[0], r1[1]);
          __nv_bfloat162 o2 = __floats2bfloat162_rn(r2[0], r2[1]);
          ptx::st_shared_u32(pair_addr(ja, h), *reinterpret_cast<uint32_t*>(&o1));
          ptx::st_shared_u32(pair_addr(jb, h), *reinterpret_cast<uint32_t*>(&o2));
        }
      }
    }
    return;
  }
  // One branch-free pass over the accumulators per step that applies, so that the code a launch runs stays small
  // (one loop holding every case unrolled over 64 pairs overflows the instruction cache at BN = 256).
  // Columns at or past N get no bias and are never stored.
  if (p.bias != nullptr) {
#pragma unroll
    for (int j = 0; j < BN / 8; j++) {
#pragma unroll
      for (int e = 0; e < 2; e++) {
        const int col = col0 + 8 * j + 2 * c + e;
        if (col < p.N) {
          const float b = p.bias_f32 ? reinterpret_cast<const float*>(p.bias)[col]
                                     : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p.bias)[col]);
          acc[4 * j + e] += b;
          acc[4 * j + 2 + e] += b;
        }
      }
    }
  }
  if (p.act == ACT_RELU) {
#pragma unroll
    for (int i = 0; i < BN / 2; i++) acc[i] = fmaxf(acc[i], 0.f);
  } else if (p.act == ACT_QUICK_GELU) {
#pragma unroll
    for (int i = 0; i < BN / 2; i++) acc[i] = act_apply(acc[i], ACT_QUICK_GELU);
  } else if (p.act == ACT_SWIGLU) {
    // interleaved gate / up: pair j of a row is output column 4j + c of the half-width output
#pragma unroll
    for (int j = 0; j < BN / 8; j++) {
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const float g = acc[4 * j + 2 * h], u = acc[4 * j + 2 * h + 1];
        const __nv_bfloat16 o = __float2bfloat16_rn(g / (1.f + __expf(-g)) * u);
        ptx::st_shared_u16(srow + h * 1024 + (j >> 4) * kBox + ((((j & 15) >> 1) ^ sw) << 4) + 8 * (j & 1) + 2 * c,
                           *reinterpret_cast<const uint16_t*>(&o));
      }
    }
    return;
  }
  if (p.residual != nullptr) {
#pragma unroll
    for (int j = 0; j < BN / 8; j++) {
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const uint32_t a = pair_addr(j, h);
        const uint32_t r = ptx::ld_shared_u32(a);
        const float2 rf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&r));
        __nv_bfloat162 o = __floats2bfloat162_rn(acc[4 * j + 2 * h] + rf.x, acc[4 * j + 2 * h + 1] + rf.y);
        ptx::st_shared_u32(a, *reinterpret_cast<uint32_t*>(&o));
      }
    }
    return;
  }
#pragma unroll
  for (int j = 0; j < BN / 8; j++) {
#pragma unroll
    for (int h = 0; h < 2; h++) {
      __nv_bfloat162 o = __floats2bfloat162_rn(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
      ptx::st_shared_u32(pair_addr(j, h), *reinterpret_cast<uint32_t*>(&o));
    }
  }
}

// One k = 16 MMA of the warpgroup's 64 x BN block; ZERO: the tile's first (scale-d = 0, write-only accumulators).
template <int TA, int TB, int BN, bool ZERO>
__device__ __forceinline__ void mma_k16(float (&acc)[BN / 2], uint64_t da, uint64_t db) {
  if constexpr (BN == 256) {
    if constexpr (ZERO) ptx::wgmma_m64n256_ss_zero<TA, TB>(acc, da, db);
    else ptx::wgmma_m64n256_ss<TA, TB>(acc, da, db, 1);
  } else {
    if constexpr (ZERO) ptx::wgmma_m64n128_ss_zero<TA, TB>(acc, da, db);
    else ptx::wgmma_m64n128_ss<TA, TB>(acc, da, db, 1);
  }
}

// The four MMAs (k = 16 each) of one 64-deep k-block.  K-major operands advance 16 elements = 32 B inside the
// 128 B swizzle atom (+2 in the >>4 start field); MN-major ones advance 16 k-rows of 128 B (+128).
// FIRST: the tile's first k-block, whose first MMA overwrites the accumulators.
template <int TA, int TB, int BN, bool FIRST>
__device__ __forceinline__ void mma_kblock(float (&acc)[BN / 2], uint64_t da, uint64_t db) {
  mma_k16<TA, TB, BN, FIRST>(acc, da, db);
#pragma unroll
  for (int k = 1; k < kBlockK / kMmaK; k++)
    mma_k16<TA, TB, BN, false>(acc, da + (TA ? 128 : 2) * k, db + (TB ? 128 : 2) * k);
}

// CONV: implicit-GEMM conv (TA = TB = 0).  TA / TB = 1: MN-major A / B (TB also covers b_mn == 2).
template <bool CONV, int TA, int TB, int BN>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_bf16_wgmma(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                const __grid_constant__ CUtensorMap tmap_d, const __grid_constant__ CUtensorMap tmap_r,
                const __grid_constant__ GemmParams p) {
  static_assert(BN == 128 || BN == 256, "tile width");
  static_assert(!CONV || (TA == 0 && TB == 0), "conv operands are K-major");
  using Cfg = GemmCfg<BN>;
  constexpr int kStages = Cfg::kStages;
  // the register epilogue serves the forward GEMMs (K-major operands); convs and the training GEMMs stage
  constexpr bool kRegEpi = !CONV && TA == 0 && TB == 0;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kStages * Cfg::kABytes;
  float* acc_s = reinterpret_cast<float*>(smem + kStages * Cfg::kStageBytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kStages * Cfg::kStageBytes + Cfg::kAccBytes);
  uint64_t* full = bars;
  uint64_t* empty = bars + kStages;
  uint64_t* stg_ready = bars + 2 * kStages;  // register epilogue: warpgroup wg's staging boxes may be written

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    ptx::prefetch_tensormap(&tmap_a);
    ptx::prefetch_tensormap(&tmap_b);
    for (int i = 0; i < kStages; i++) {
      ptx::mbar_init(&full[i], 1);
      ptx::mbar_init(&empty[i], 2);  // one arrival per consumer warpgroup
    }
    if (kRegEpi && p.tma_epi) {
      ptx::prefetch_tensormap(&tmap_d);
      if (p.residual) ptx::prefetch_tensormap(&tmap_r);
      ptx::mbar_init(&stg_ready[0], 1);
      ptx::mbar_init(&stg_ready[1], 1);
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  const int tiles_mn = p.num_m_tiles * p.num_n_tiles;
  const int total_tiles = tiles_mn * p.k_splits;

  if (threadIdx.x < kGemmThreads - kConsumerThreads) {
    // ============================ TMA producer (warpgroup 0) ============================
    if constexpr (BN == 256) ptx::setmaxnreg_dec<kProducerRegs>();  // the whole warpgroup, before lanes 1-127 leave
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
        const int split = t / tiles_mn;
        const int mn = t % tiles_mn;
        const int n_blk = p.n_fast ? mn % p.num_n_tiles : mn / p.num_m_tiles;
        const int m_blk = p.n_fast ? mn / p.num_n_tiles : mn % p.num_m_tiles;
        const int kb0 = split * p.num_k_blocks;
        int img = 0, y0 = 0, x0 = 0;
        if (CONV) {
          const int tx = m_blk % p.tiles_x;
          const int ty = (m_blk / p.tiles_x) % p.tiles_y;
          img = m_blk / (p.tiles_x * p.tiles_y);
          y0 = ty * p.cBH;
          x0 = tx * p.cBW;
        }
        for (int kb = 0; kb < p.num_k_blocks; kb++) {
          ptx::mbar_wait(&empty[stage], phase ^ 1);
          ptx::mbar_arrive_expect_tx(&full[stage], (uint32_t)(p.a_rows * kBlockK * 2 + Cfg::kBBytes));
          const int kg = kb0 + kb;
          uint8_t* sa = smem_a + stage * Cfg::kABytes;
          uint8_t* sb = smem_b + stage * Cfg::kBBytes;
          if (CONV) {
            const int tap_all = kg / p.cin_blocks, cc = kg % p.cin_blocks;
            const int lvl = tap_all / p.taps, tap = tap_all % p.taps;
            const int dy = p.taps == 9 ? tap / 3 - 1 : 0, dx = p.taps == 9 ? tap % 3 - 1 : 0;
            ptx::tma_load_4d(sa, &tmap_a, &full[stage], cc * kBlockK, x0 + dx, y0 + dy, img + lvl * p.lvl_img_stride);
          } else if (TA) {
            // MN-major A: two [64 k][64 m] boxes (one 128-byte swizzle atom of m each)
#pragma unroll
            for (int a = 0; a < kBlockM / 64; a++)
              ptx::tma_load_2d(sa + a * (kBlockK * 128), &tmap_a, &full[stage], m_blk * kBlockM + a * 64, kg * kBlockK);
          } else {
            ptx::tma_load_2d(sa, &tmap_a, &full[stage], kg * kBlockK, m_blk * kBlockM);
          }
          if (TB && p.b_mn == 2) {
            const int n0 = n_blk * BN, tap = n0 / p.dw_cin, c0 = n0 % p.dw_cin;
#pragma unroll
            for (int a = 0; a < BN / 64; a++)
              ptx::tma_load_4d(sb + a * (kBlockK * 128), &tmap_b, &full[stage], c0 + a * 64, tap % 3, kg * kBlockK,
                               tap / 3);
          } else if (TB) {
#pragma unroll
            for (int a = 0; a < BN / 64; a++)
              ptx::tma_load_2d(sb + a * (kBlockK * 128), &tmap_b, &full[stage], n_blk * BN + a * 64, kg * kBlockK);
          } else {
            ptx::tma_load_2d(sb, &tmap_b, &full[stage], kg * kBlockK, n_blk * BN);
          }
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ============================ consumers: MMA + epilogue ============================
  if constexpr (BN == 256) ptx::setmaxnreg_inc<kConsumerRegs>();
  const int ct = threadIdx.x - (kGemmThreads - kConsumerThreads);  // 0..255
  const int wg = ct >> 7;    // consumer warpgroup: accumulator rows [64 wg, 64 wg + 64)
  const int wt = ct & 127;   // thread in the warpgroup
  // MN-major B: LBO = the 8 KB stride between its 64-wide n atoms
  const uint32_t lbo_b = TB ? kBlockK * 128 : 0;
  const int row = ct & 127, half = ct >> 7;
  int stage = 0;
  uint32_t phase = 0;
  uint32_t stg_phase = 0;
  // register epilogue: this warpgroup's staging boxes (64 rows each) and the tile's first output row
  uint8_t* stg = smem + kStages * Cfg::kStageBytes + wg * Cfg::kWgStageBytes;
  float acc[BN / 2];
  for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
    const int split = t / tiles_mn;
    const int mn = t % tiles_mn;
    const int n_blk = p.n_fast ? mn % p.num_n_tiles : mn / p.num_m_tiles;
    const int m_blk = p.n_fast ? mn / p.num_n_tiles : mn % p.num_m_tiles;
    const int row0 = m_blk * kBlockM + wg * 64, col0 = n_blk * BN;
    // this warpgroup's 64 rows of A start 8 KB into the stage in both layouts (64 rows x 128 B, or mn atom wg)
    auto desc_a = [&](int s) { return ptx::gmma_desc_sw128(ptx::smem_u32(smem_a + s * Cfg::kABytes + wg * 8192), 0); };
    auto desc_b = [&](int s) { return ptx::gmma_desc_sw128(ptx::smem_u32(smem_b + s * Cfg::kBBytes), lbo_b); };
    // k-block 0: overwrites the accumulators
    ptx::mbar_wait(&full[stage], phase);
    ptx::wgmma_fence();
    mma_kblock<TA, TB, BN, true>(acc, desc_a(stage), desc_b(stage));
    ptx::wgmma_commit();
    int prev = stage;
    if (++stage == kStages) { stage = 0; phase ^= 1; }
    if (kRegEpi && p.tma_epi && wt == 0) {
      // While the MMAs run: once the previous tile's stores have read the staging boxes, load this tile's residual
      // into them (the layout the output takes there), or just hand them back to the warpgroup.
      ptx::bulk_wait_read<0>();
      if (p.residual != nullptr && row0 < p.M) {
        const int nbox = min(BN / 64, (p.N - col0 + 63) / 64);
        ptx::mbar_arrive_expect_tx(&stg_ready[wg], (uint32_t)(nbox * Cfg::kBoxBytes));
        for (int b = 0; b < nbox; b++)
          ptx::tma_load_2d(stg + b * Cfg::kBoxBytes, &tmap_r, &stg_ready[wg], col0 + 64 * b, row0);
      } else {
        ptx::mbar_arrive(&stg_ready[wg]);
      }
    }
    for (int kb = 1; kb < p.num_k_blocks; kb++) {
      ptx::mbar_wait(&full[stage], phase);
      ptx::wgmma_fence();
      mma_kblock<TA, TB, BN, false>(acc, desc_a(stage), desc_b(stage));
      ptx::wgmma_commit();
      ptx::wgmma_wait<1>();  // the MMAs of the previous k-block have completed: its slot can be refilled
      if (wt == 0) ptx::mbar_arrive(&empty[prev]);
      prev = stage;
      if (++stage == kStages) { stage = 0; phase ^= 1; }
    }
    ptx::wgmma_wait<0>();
    ptx::fence_regs(acc);
    if (wt == 0) ptx::mbar_arrive(&empty[prev]);
    if (kRegEpi && p.tma_epi) {
      // ---- register epilogue: finish the accumulators in place into the staging boxes, then one thread stores
      // them with TMA and the warpgroup goes on to its next tile while the stores drain
      ptx::mbar_wait(&stg_ready[wg], stg_phase);
      stg_phase ^= 1;
      epilogue_regs<BN>(p, acc, ptx::smem_u32(stg), row0, col0, wt);
      ptx::fence_proxy_async_smem();
      ptx::named_bar_sync(2 + wg, 128);
      if (wt == 0 && row0 < p.M) {
        const bool glu = p.act == ACT_SWIGLU;
        const int ocol0 = glu ? col0 / 2 : col0, on = glu ? p.N / 2 : p.N;
        const int nbox = min(glu ? BN / 128 : BN / 64, (on - ocol0 + 63) / 64);
        for (int b = 0; b < nbox; b++) ptx::tma_store_2d(&tmap_d, stg + b * Cfg::kBoxBytes, ocol0 + 64 * b, row0);
        ptx::bulk_commit();
      }
      continue;
    }
    // ---- stage the accumulators (fragment layout -> row-major fp32), 128 columns at a time, and run the epilogue
#pragma unroll
    for (int h = 0; h < BN / kEpiN; h++) {
      ptx::named_bar_sync(1, kConsumerThreads);  // the previous pass's epilogue is done reading the staging tile
      {
        const int r = wg * 64 + (wt >> 5) * 16 + ((wt & 31) >> 2);
        float* s = acc_s + r * Cfg::kAccLd + 2 * (wt & 3);
#pragma unroll
        for (int j = 0; j < kEpiN / 8; j++) {
          const int a = h * (kEpiN / 2) + 4 * j;
          *reinterpret_cast<float2*>(s + 8 * j) = make_float2(acc[a], acc[a + 1]);
          *reinterpret_cast<float2*>(s + 8 * Cfg::kAccLd + 8 * j) = make_float2(acc[a + 2], acc[a + 3]);
        }
      }
      ptx::named_bar_sync(1, kConsumerThreads);
      epilogue_tile<CONV>(p, acc_s + row * Cfg::kAccLd, m_blk, n_blk * BN + h * kEpiN, split, row, half, lane);
    }
  }
  if (kRegEpi && p.tma_epi && wt == 0) ptx::bulk_wait<0>();  // the last stores have read shared memory and landed
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess ||
      qres != cudaDriverEntryPointSuccess)
    return nullptr;
  fn = reinterpret_cast<EncodeTiledFn>(p);
  return fn;
}

// bf16 tensor map, rank 2..4; dims/box innermost first; strides (bytes) for dims 1..rank-1.
static int make_tmap(CUtensorMap* m, const void* base, int rank, const cuuint64_t* dims,
                     const cuuint64_t* strides_bytes, const cuuint32_t* box) {
  EncodeTiledFn enc = get_encode();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled unavailable (driver entry point lookup failed)");
    return G4R_ECUDA;
  }
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), dims,
                   strides_bytes, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed: CUresult %d (rank %d, dims %llu,%llu box %u,%u)", (int)r, rank,
              (unsigned long long)dims[0], (unsigned long long)dims[1], box[0], box[1]);
    return G4R_ECUDA;
  }
  return G4R_OK;
}

// A row of D / the residual may be read or written with 16-byte vectors when its base and its row pitch are both
// multiples of 16 bytes; otherwise the epilogue takes its scalar path (e.g. a one-row output at an odd offset).
static int vec16(const void* base, long long ld, int elem_bytes) {
  return ((uintptr_t)base % 16 == 0) && (ld * elem_bytes % 16 == 0);
}

// td / tr: the D and residual maps of the register epilogue (p.tma_epi), unused otherwise
template <bool CONV, int TA, int TB, int BN>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, GemmParams p, cudaStream_t st,
                       const CUtensorMap& td = CUtensorMap{}, const CUtensorMap& tr = CUtensorMap{}) {
  p.d_vec = vec16(p.D, p.ldd, p.out_f32 ? 4 : 2);
  p.r_vec = vec16(p.residual, p.ldr, p.residual_f32 ? 4 : 2);
  static bool attr_set = false;
  auto kern = gemm_bf16_wgmma<CONV, TA, TB, BN>;
  if (!attr_set) {
    G4R_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, GemmCfg<BN>::kSmemBytes));
    attr_set = true;
  }
  const int total = p.num_m_tiles * p.num_n_tiles * p.k_splits;
  const int grid = total < sm_budget() ? total : sm_budget();
  kern<<<grid, kGemmThreads, GemmCfg<BN>::kSmemBytes, st>>>(ta, tb, td, tr, p);
  G4R_LAUNCH_CHECK("gemm_bf16_wgmma");
  return G4R_OK;
}

// Tile width of a forward GEMM / conv launch with `m_tiles` row tiles, N output columns and k_splits.
// G4R_GEMM_BN=128|256 forces a width (read at every launch, so one process can time both); auto / unset applies
// the rule: the persistent grid runs ceil(tiles / grid) rounds, and a 128 x 256 tile costs kTileCost256 / 100 of a
// 128 x 128 tile, so the width with the smaller rounds x cost wins (ties go to 128).
// kTileCost256 from tools/bench_gemm.py (H100 80GB HBM3, 700 W limit, power-capped at 1425-1590 MHz on these
// shapes), time per round at 256 over time per round at 128:
//   LLaMA M = 5648: q|k|v+RoPE 62.8/39.7 us = 1.58 (17 vs 33 rounds), o_proj 60.3/35.7 = 1.69 (6 vs 11),
//   gate/up 57.3/35.4 = 1.62 (30 vs 59), down 148/97 = 1.52 (6 vs 11), lm_head 57.9/37.4 = 1.55 (43 vs 86);
//   3x3 fuse conv 192 px 124/75 = 1.65 (70 vs 140).
// So 256 wins whenever it saves more than ~38 % of the rounds: every LLaMA GEMM (o_proj and down included,
// 0.362 vs 0.393 ms and 0.887 vs 1.069 ms), the big convs and 1x1 convs, while 3 -> 2 round cases such as ViT
// out_proj / fc2 (4616 x 1024: 0.057 vs 0.069 ms, 0.120 vs 0.130 ms) stay at 128.
constexpr int kTileCost256 = 160;   // per cent of a 128 x 128 tile
static int pick_block_n(int m_tiles, int N, int k_splits) {
  const char* e = getenv("G4R_GEMM_BN");
  if (e && !strcmp(e, "128")) return 128;
  if (e && !strcmp(e, "256")) return 256;
  const long long grid = sm_budget();
  const long long t128 = (long long)m_tiles * ((N + 127) / 128) * k_splits;
  const long long t256 = (long long)m_tiles * ((N + 255) / 256) * k_splits;
  const long long r128 = (t128 + grid - 1) / grid, r256 = (t256 + grid - 1) / grid;
  return r256 * kTileCost256 < r128 * 100 ? 256 : 128;
}

}  // namespace g4r

using namespace G4R_NS;

extern "C" int g4r_gemm_bf16(const void* A, long long lda, const void* B, long long ldb, void* D,
                             long long ldd, int M, int N, int K, const void* bias, int bias_f32,
                             const void* residual, long long ldr, int act, int out_f32, int k_splits,
                             void* stream);
extern "C" int g4r_gemm_bf16_ex(const void* A, long long lda, const void* B, long long ldb, void* D,
                                long long ldd, int M, int N, int K, const void* bias, int bias_f32,
                                const void* residual, long long ldr, int residual_f32, int bias_round_bf16,
                                int act, int out_f32, int k_splits, void* stream);
extern "C" int g4r_gemm_bf16(const void* A, long long lda, const void* B, long long ldb, void* D,
                             long long ldd, int M, int N, int K, const void* bias, int bias_f32,
                             const void* residual, long long ldr, int act, int out_f32, int k_splits,
                             void* stream) {
  return g4r_gemm_bf16_ex(A, lda, B, ldb, D, ldd, M, N, K, bias, bias_f32, residual, ldr, 0, 0, act, out_f32,
                          k_splits, stream);
}

static int gemm_impl(const void* A, long long lda, const void* B, long long ldb, void* D, long long ldd, int M,
                     int N, int K, const void* bias, int bias_f32, const void* residual, long long ldr,
                     int residual_f32, int bias_round_bf16, int act, int out_f32, int k_splits,
                     const void* rope_cos, const void* rope_sin, int rope_cols, int rope_L, void* stream,
                     int rope_pos0 = 0, const int* rope_pos_dev = nullptr, const int* rope_pos_rows = nullptr);

namespace G4R_NS {
// gemm_skinny.cu: M <= 16 weight-streaming path; returns -1 when the shape does not qualify
int gemm_skinny_dispatch(const void* A, long long lda, const void* B, long long ldb, void* D, long long ldd, int M,
                         int N, int K, const void* bias, int bias_f32, const void* residual, long long ldr, int act,
                         const void* rope_cos, const void* rope_sin, int rope_cols, int rope_L, int rope_pos0,
                         const int* rope_pos_dev, const int* rope_pos_rows, void* stream);
}

extern "C" int g4r_gemm_bf16_ex(const void* A, long long lda, const void* B, long long ldb, void* D,
                                long long ldd, int M, int N, int K, const void* bias, int bias_f32,
                                const void* residual, long long ldr, int residual_f32, int bias_round_bf16,
                                int act, int out_f32, int k_splits, void* stream) {
  return gemm_impl(A, lda, B, ldb, D, ldd, M, N, K, bias, bias_f32, residual, ldr, residual_f32, bias_round_bf16,
                   act, out_f32, k_splits, nullptr, nullptr, 0, 0, stream);
}

// QKV projection with the rotary embedding fused into the epilogue: D[M, N] = A.B^T, columns
// [0, rope_cols) (the q and k heads, head_dim 128) rotated with cos/sin[row % L].  Replaces
// q_proj/k_proj/v_proj + apply_rotary_pos_emb (transformers modeling_llama.py:138-168,240-260).
extern "C" int g4r_gemm_qkv_rope_bf16(const void* A, long long lda, const void* B, long long ldb, void* D,
                                      long long ldd, int M, int N, int K, const void* rope_cos,
                                      const void* rope_sin, int rope_cols, int L, int pos0, const int* pos0_dev,
                                      void* stream) {
  G4R_REQUIRE(rope_cos && rope_sin && L > 0, "qkv_rope: null tables");
  G4R_REQUIRE(rope_cols % 256 == 0 && rope_cols <= N && N % 128 == 0 && ldd % 8 == 0, "qkv_rope: rope_cols must be a multiple of 256 (whole tiles of 128-dim heads)");  return gemm_impl(A, lda, B, ldb, D, ldd, M, N, K, nullptr, 0, nullptr, 0, 0, 0, ACT_NONE, 0, 1, rope_cos, rope_sin,
                   rope_cols, L, stream, pos0, pos0_dev);
}

// The same with a per-sample position base: row r (sample r / L) is rotated at pos_rows[r / L] + r % L -- a batch of
// prompts of different lengths in the decode step (L = 1).
extern "C" int g4r_gemm_qkv_rope_rows_bf16(const void* A, long long lda, const void* B, long long ldb, void* D,
                                           long long ldd, int M, int N, int K, const void* rope_cos,
                                           const void* rope_sin, int rope_cols, int L, const int* pos_rows,
                                           void* stream) {
  G4R_REQUIRE(rope_cos && rope_sin && pos_rows && L > 0 && M % L == 0, "qkv_rope_rows: null tables / pos_rows, or M %% L != 0");
  G4R_REQUIRE(rope_cols % 256 == 0 && rope_cols <= N && N % 128 == 0 && ldd % 8 == 0, "qkv_rope: rope_cols must be a multiple of 256 (whole tiles of 128-dim heads)");  return gemm_impl(A, lda, B, ldb, D, ldd, M, N, K, nullptr, 0, nullptr, 0, 0, 0, ACT_NONE, 0, 1, rope_cos, rope_sin,
                   rope_cols, L, stream, 0, nullptr, pos_rows);
}

// Backward-pass GEMM: D[M, N] = op(A) . op(B)^T with either operand optionally stored "MN-major":
//   a_mn = 0: A is [M, K] (K contiguous, row stride lda);  a_mn = 1: A is stored [K, M] (M contiguous, lda >= M)
//   b_mn = 0: B is [N, K] (K contiguous, row stride ldb);  b_mn = 1: B is stored [K, N] (N contiguous, ldb >= N)
// so that for y = x W^T (W [N_out, K_in], nn.Linear):
//   dX[M, K_in]      = dY[M, N_out] . W          -> A = dY (a_mn 0), B = W  (b_mn 1, contraction N_out)
//   dW[N_out, K_in]  = dY^T . X                  -> A = dY (a_mn 1), B = X  (b_mn 1, contraction M tokens)
// The transposes happen in the wgmma operand descriptors (transpose immediates), never in memory.
// Replaces the autograd of F.linear inside the stage-2 training step (gpt4roi/train/train.py:698-712).
#if G4R_BF16_ONLY   // training-step only: no fp16 twin
extern "C" int g4r_gemm_bf16_t(const void* A, long long lda, int a_mn, const void* B, long long ldb, int b_mn, void* D,
                               long long ldd, int M, int N, int K, int out_f32, void* stream) {
  G4R_REQUIRE(A && B && D, "null operand");
  G4R_REQUIRE(M > 0 && N > 0 && K > 0, "bad sizes M=%d N=%d K=%d", M, N, K);
  G4R_REQUIRE(lda % 8 == 0 && ldb % 8 == 0, "lda/ldb must be multiples of 8 (16-byte TMA strides)");
  G4R_REQUIRE(lda >= (a_mn ? M : K) && ldb >= (b_mn ? N : K), "lda/ldb smaller than the contiguous extent");
  G4R_REQUIRE(((uintptr_t)A & 15) == 0 && ((uintptr_t)B & 15) == 0, "A/B must be 16-byte aligned");
  GemmParams p{};
  p.M = M; p.N = N; p.K = K;
  p.num_m_tiles = (M + kBlockM - 1) / kBlockM;
  p.k_splits = 1;
  p.num_k_blocks = (K + kBlockK - 1) / kBlockK;
  p.D = D; p.ldd = ldd; p.out_f32 = out_f32;
  p.a_rows = kBlockM;
  p.a_mn = a_mn ? 1 : 0; p.b_mn = b_mn ? 1 : 0;
  p.num_n_tiles = (N + 127) / 128;   // the training GEMMs run 128 x 128 tiles
  CUtensorMap ta, tb;
  {
    cuuint64_t dims[2] = {(cuuint64_t)(a_mn ? M : K), (cuuint64_t)(a_mn ? K : M)};
    cuuint64_t str[1] = {(cuuint64_t)lda * 2};
    cuuint32_t box[2] = {64, (cuuint32_t)(a_mn ? kBlockK : kBlockM)};
    int rc = make_tmap(&ta, A, 2, dims, str, box);
    if (rc) return rc;
  }
  {
    cuuint64_t dims[2] = {(cuuint64_t)(b_mn ? N : K), (cuuint64_t)(b_mn ? K : N)};
    cuuint64_t str[1] = {(cuuint64_t)ldb * 2};
    cuuint32_t box[2] = {64, (cuuint32_t)(b_mn ? kBlockK : 128)};
    int rc = make_tmap(&tb, B, 2, dims, str, box);
    if (rc) return rc;
  }
  const cudaStream_t st = (cudaStream_t)stream;
  if (!a_mn && !b_mn) return launch_gemm<false, 0, 0, 128>(ta, tb, p, st);
  if (!a_mn) return launch_gemm<false, 0, 1, 128>(ta, tb, p, st);
  if (!b_mn) return launch_gemm<false, 1, 0, 128>(ta, tb, p, st);
  return launch_gemm<false, 1, 1, 128>(ta, tb, p, st);
}
#endif

// Weight gradient of a 3x3 / stride 1 / pad 1 convolution (NHWC, bf16) as ONE tensor-core GEMM on the
// zero-padded layout:  dW[co, ky, kx, ci] = sum_rows dz_pad[row, co] * x_pad[row + (ky-1)*(W+2) + (kx-1), ci]
// where rows run over n_img*(H+2)*(W+2) padded pixels (dz_pad is zero on the padding ring, so wrapped
// neighbours contribute nothing).  A = dz_pad as an MN-major operand; B = x_pad through an aliasing 4-D tensor
// map (b_mn == 2), so all nine taps are column blocks of one launch (8 x 72 tiles for 1024 -> 1024).
// x_pad_origin points at the row of x_pad that tap (0,0) pairs with row 0, i.e. (W+2)+1 rows before the first
// real row; the caller keeps >= (W+2)+1 zero guard rows on both ends.  dW is fp32 [Cout, 9*Cin]; accumulate != 0
// adds to it (the four pyramid levels of a fuse round share one weight, gpt4roi/models/layers.py:152-180).
#if G4R_BF16_ONLY   // training-step only: no fp16 twin
extern "C" int g4r_conv3x3_dw_bf16(const void* dz_pad, const void* x_pad_origin, float* dW, long long rows, int Wp,
                                   int Cin, int Cout, int accumulate, void* stream) {
  G4R_REQUIRE(dz_pad && x_pad_origin && dW && rows > 0 && Wp > 2, "conv3x3_dw: bad arguments");
  G4R_REQUIRE(Cin % 256 == 0 && Cout % 8 == 0, "conv3x3_dw: Cin=%d must be a multiple of 256, Cout=%d of 8", Cin, Cout);
  G4R_REQUIRE((((uintptr_t)dz_pad | (uintptr_t)x_pad_origin) & 15) == 0, "conv3x3_dw: misaligned operands");
  GemmParams p{};
  p.M = Cout; p.N = 9 * Cin; p.K = (int)rows;
  p.num_m_tiles = (Cout + kBlockM - 1) / kBlockM;
  p.k_splits = 1;
  p.num_k_blocks = (int)((rows + kBlockK - 1) / kBlockK);
  p.D = dW; p.ldd = 9LL * Cin; p.out_f32 = 1;
  if (accumulate) { p.residual = reinterpret_cast<const __nv_bfloat16*>(dW); p.residual_f32 = 1; p.ldr = p.ldd; }
  p.a_rows = kBlockM;
  p.a_mn = 1; p.b_mn = 2; p.dw_cin = Cin;
  p.num_n_tiles = p.N / 128;
  CUtensorMap ta, tb;
  {
    cuuint64_t dims[2] = {(cuuint64_t)Cout, (cuuint64_t)rows};
    cuuint64_t str[1] = {(cuuint64_t)Cout * 2};
    cuuint32_t box[2] = {64, kBlockK};
    int rc = make_tmap(&ta, dz_pad, 2, dims, str, box);
    if (rc) return rc;
  }
  {
    // dimension order {ci, kx, row, ky}: every stride is a multiple of the previous one (driver requirement)
    cuuint64_t dims[4] = {(cuuint64_t)Cin, 3, (cuuint64_t)rows, 3};
    cuuint64_t str[3] = {(cuuint64_t)Cin * 2, (cuuint64_t)Cin * 2, (cuuint64_t)Wp * Cin * 2};
    cuuint32_t box[4] = {64, 1, kBlockK, 1};
    int rc = make_tmap(&tb, x_pad_origin, 4, dims, str, box);
    if (rc) return rc;
  }
  return launch_gemm<false, 1, 1, 128>(ta, tb, p, (cudaStream_t)stream);
}
#endif

static int gemm_impl(const void* A, long long lda, const void* B, long long ldb, void* D, long long ldd, int M,
                     int N, int K, const void* bias, int bias_f32, const void* residual, long long ldr,
                     int residual_f32, int bias_round_bf16, int act, int out_f32, int k_splits,
                     const void* rope_cos, const void* rope_sin, int rope_cols, int rope_L, void* stream,
                     int rope_pos0, const int* rope_pos_dev, const int* rope_pos_rows) {
  G4R_REQUIRE(A && B && D, "null operand");
  G4R_REQUIRE(M > 0 && N > 0 && K > 0, "bad sizes M=%d N=%d K=%d", M, N, K);
  G4R_REQUIRE(lda % 8 == 0 && ldb % 8 == 0 && lda >= K && ldb >= K, "lda/ldb must be >= K and multiples of 8 (16-byte TMA strides)");
  G4R_REQUIRE(((uintptr_t)A & 15) == 0 && ((uintptr_t)B & 15) == 0, "A/B must be 16-byte aligned");
  G4R_REQUIRE(act >= ACT_NONE && act <= ACT_SWIGLU, "act=%d", act);
  G4R_REQUIRE(k_splits >= 1, "k_splits=%d", k_splits);
  if (act == ACT_SWIGLU) G4R_REQUIRE(N % 2 == 0 && !out_f32 && k_splits == 1 && !residual, "SwiGLU epilogue: even N, bf16 out, no split-K/residual");
  if (k_splits > 1) G4R_REQUIRE(out_f32 && act == ACT_NONE && !residual && !bias, "split-K writes fp32 partial slabs [k_splits][M][ldd]: out_f32, no bias/act/residual");
  // M <= 16 (decode step): HBM-bound weight-streaming kernel instead of a mostly empty 128-row tile
  if (M <= 16 && !out_f32 && k_splits == 1 && !residual_f32 && !bias_round_bf16) {
    const int rc = gemm_skinny_dispatch(A, lda, B, ldb, D, ldd, M, N, K, bias, bias_f32, residual, ldr, act, rope_cos,
                                        rope_sin, rope_cols, rope_L, rope_pos0, rope_pos_dev, rope_pos_rows, stream);
    if (rc >= 0) return rc;
  }
  GemmParams p{};
  p.M = M; p.N = N; p.K = K;
  p.num_m_tiles = (M + kBlockM - 1) / kBlockM;
  const int kb_total = (K + kBlockK - 1) / kBlockK;
  G4R_REQUIRE(kb_total % k_splits == 0, "K blocks (%d) not divisible by k_splits (%d)", kb_total, k_splits);
  p.k_splits = k_splits;
  p.num_k_blocks = kb_total / k_splits;
  p.D = D; p.ldd = ldd; p.bias = bias; p.bias_f32 = bias_f32;
  p.residual = (const __nv_bfloat16*)residual; p.ldr = ldr; p.residual_f32 = residual_f32;
  p.round_branch = bias_round_bf16;
  p.rope_cos = (const __nv_bfloat16*)rope_cos; p.rope_sin = (const __nv_bfloat16*)rope_sin;
  p.rope_cols = rope_cols; p.rope_L = rope_L; p.rope_pos0 = rope_pos0; p.rope_pos_dev = rope_pos_dev;
  p.rope_pos_rows = rope_pos_rows;
  p.act = act; p.out_f32 = out_f32;
  p.conv = 0; p.a_rows = kBlockM;
  const int bn = pick_block_n(p.num_m_tiles, N, k_splits);
  p.num_n_tiles = (N + bn - 1) / bn;
  CUtensorMap ta, tb;
  {
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)M};
    cuuint64_t str[1] = {(cuuint64_t)lda * 2};
    cuuint32_t box[2] = {kBlockK, kBlockM};
    int rc = make_tmap(&ta, A, 2, dims, str, box);
    if (rc) return rc;
  }
  {
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)N};
    cuuint64_t str[1] = {(cuuint64_t)ldb * 2};
    cuuint32_t box[2] = {kBlockK, (cuuint32_t)bn};
    int rc = make_tmap(&tb, B, 2, dims, str, box);
    if (rc) return rc;
  }
  // Register epilogue with TMA stores for a 16-bit output with a 16-bit or no residual, when D and the residual
  // meet TMA's 16-byte base and row-pitch alignment and the row ends on a 16-byte boundary (a TMA store writes
  // whole 16-byte pieces of a row, so a row of 32006 columns would overwrite its two pad columns); fp32 outputs and
  // residuals, split-K and the rounded branch keep the staged epilogue too.  Both store / load 64 x 64 boxes (one
  // consumer warpgroup's rows, 128 B of columns).
  CUtensorMap td{}, tr{};
  const int n_out = act == ACT_SWIGLU ? N / 2 : N;
  p.tma_epi = !out_f32 && k_splits == 1 && !bias_round_bf16 && !residual_f32 && n_out % 8 == 0 &&
              vec16(D, ldd, 2) && (!residual || vec16(residual, ldr, 2));
  if (p.tma_epi) {
    cuuint64_t dims[2] = {(cuuint64_t)n_out, (cuuint64_t)M};
    cuuint64_t str[1] = {(cuuint64_t)ldd * 2};
    cuuint32_t box[2] = {64, 64};
    int rc = make_tmap(&td, D, 2, dims, str, box);
    if (rc) return rc;
    if (residual) {
      cuuint64_t rdims[2] = {(cuuint64_t)N, (cuuint64_t)M};
      cuuint64_t rstr[1] = {(cuuint64_t)ldr * 2};
      rc = make_tmap(&tr, residual, 2, rdims, rstr, box);
      if (rc) return rc;
    }
  }
  return bn == 256 ? launch_gemm<false, 0, 0, 256>(ta, tb, p, (cudaStream_t)stream, td, tr)
                   : launch_gemm<false, 0, 0, 128>(ta, tb, p, (cudaStream_t)stream, td, tr);
}

// spatial tiling used by the conv kernel for an H x W map (also tells callers how many GN partial slots exist)
static void conv_tiling(int H, int W, int* bw_out, int* bh_out) {
  int bw = W >= 16 && W % 16 == 0 ? 16 : (W >= 8 ? 8 : W);
  if (W == 14) bw = 14;
  int bh = kBlockM / bw;
  if (bh > H) bh = H;
  *bw_out = bw;
  *bh_out = bh;
}

#if G4R_BF16_ONLY   // independent of the activation type: built once
extern "C" int g4r_conv_gn_slots(int H, int W) {
  int bw, bh;
  conv_tiling(H, W, &bw, &bh);
  return ((W + bw - 1) / bw) * ((H + bh - 1) / bh) * 4;
}
#endif

extern "C" int g4r_conv_nhwc_bf16(const void* X, const void* Wt, void* Y, int n_img, int H, int W, int Cin,
                                  int Cout, int ksize, int levels, const void* bias, int bias_f32, int act,
                                  float* gn_stats, int gn_groups, void* stream) {
  G4R_REQUIRE(X && Wt && Y, "null operand");
  G4R_REQUIRE(ksize == 3 || ksize == 1, "ksize=%d (1 or 3)", ksize);
  G4R_REQUIRE(Cin % kBlockK == 0, "Cin=%d must be a multiple of 64", Cin);
  G4R_REQUIRE(Cout % 8 == 0, "Cout=%d must be a multiple of 8", Cout);
  G4R_REQUIRE(n_img > 0 && H > 0 && W > 0, "bad sizes");
  G4R_REQUIRE(levels >= 1 && levels <= 8, "levels=%d", levels);
  G4R_REQUIRE(act == ACT_NONE || act == ACT_RELU, "conv epilogue: none or relu");
  if (gn_stats) G4R_REQUIRE(gn_groups > 0 && Cout % gn_groups == 0 && Cout / gn_groups == 16, "GN stats need 16-channel groups");
  GemmParams p{};
  // spatial tile: BW x BH = 128 output pixels (or fewer for small maps)
  int bw, bh;
  conv_tiling(H, W, &bw, &bh);
  p.cBW = bw; p.cBH = bh; p.cH = H; p.cW = W;
  p.tiles_x = (W + bw - 1) / bw;
  p.tiles_y = (H + bh - 1) / bh;
  p.a_rows = bw * bh;
  p.M = n_img * H * W; p.N = Cout; p.K = levels * ksize * ksize * Cin;
  p.levels = levels; p.lvl_img_stride = n_img;
  p.num_m_tiles = n_img * p.tiles_x * p.tiles_y;
  p.cin_blocks = Cin / kBlockK;
  p.taps = ksize * ksize;
  p.num_k_blocks = levels * p.taps * p.cin_blocks;
  p.k_splits = 1;
  p.D = Y; p.ldd = Cout; p.bias = bias; p.bias_f32 = bias_f32; p.act = act;
  p.conv = 1;
  p.n_fast = 1;
  p.gn_stats = gn_stats; p.gn_groups = gn_groups; p.gn_group_ch = gn_groups ? Cout / gn_groups : 0;
  const int bn = pick_block_n(p.num_m_tiles, Cout, 1);
  p.num_n_tiles = (Cout + bn - 1) / bn;
  CUtensorMap ta, tb;
  {
    cuuint64_t dims[4] = {(cuuint64_t)Cin, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)n_img * levels};
    cuuint64_t str[3] = {(cuuint64_t)Cin * 2, (cuuint64_t)W * Cin * 2, (cuuint64_t)H * W * Cin * 2};
    cuuint32_t box[4] = {kBlockK, (cuuint32_t)bw, (cuuint32_t)bh, 1};
    int rc = make_tmap(&ta, X, 4, dims, str, box);
    if (rc) return rc;
  }
  {
    cuuint64_t dims[2] = {(cuuint64_t)p.K, (cuuint64_t)Cout};
    cuuint64_t str[1] = {(cuuint64_t)p.K * 2};
    cuuint32_t box[2] = {kBlockK, (cuuint32_t)bn};
    int rc = make_tmap(&tb, Wt, 2, dims, str, box);
    if (rc) return rc;
  }
  return bn == 256 ? launch_gemm<true, 0, 0, 256>(ta, tb, p, (cudaStream_t)stream)
                   : launch_gemm<true, 0, 0, 128>(ta, tb, p, (cudaStream_t)stream);
}
