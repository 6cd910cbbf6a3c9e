/*
 * oracle/roi_align_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Plain-C restatement of the reference's CPU RoIAlign (forward avg/max and
 * backward), used only by tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline leg as the parity checker.  Nothing under gpt4roi_b200/ may
 * import, link or call it.
 *
 * Reference followed (paths relative to mmcv-1.4.7/mmcv/ops/csrc of the reference checkout):
 *   pytorch/cpu/roi_align.cpp:23-108    pre_calc_for_bilinear_interpolate
 *   pytorch/cpu/roi_align.cpp:110-214   ROIAlignForward<T>
 *   pytorch/cpu/roi_align.cpp:216-262   bilinear_interpolate_gradient
 *   pytorch/cpu/roi_align.cpp:270-382   ROIAlignBackward<T>
 *
 * Pinned against: the mmcv known-answer vectors
 * (mmcv-1.4.7/tests/test_ops/test_roi_align.py:14-32, committed as
 * tests/golden/mmcv_roi_align_kat.json) and against outputs of the reference
 * kernel itself compiled from its own sources (oracle/_ref, tests/golden/
 * roi_align_ref_*.npz).  See tests/test_oracle_cpu.py.
 *
 * Arithmetic contract (what "bit-exact" means): every expression is evaluated
 * in T with the reference's association and WITHOUT fused multiply-add.  Build
 * with -ffp-contract=off and no -march/-mfma (oracle/Makefile does).
 *
 * Differences from the reference that are deliberate:
 *   - layout/stride generalisation: the sample table is computed once per RoI
 *     exactly like PreCalc, but the input may be NCHW (reference layout) or
 *     NHWC (the layout the GPU kernels also accept) -- the VALUES are the same.
 *   - the "aligned && negative RoI size" AT_ASSERTM (cpu/roi_align.cpp:137-139)
 *     is reported as return code 2 instead of throwing.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#define LAYOUT_NCHW 0
#define LAYOUT_NHWC 1

#define DEFINE_ORACLE(T, SUFFIX)                                                                    \
  typedef struct {                                                                                  \
    int pos1, pos2, pos3, pos4; /* y*W+x pixel indices (cpu/roi_align.cpp:94-97) */                 \
    T w1, w2, w3, w4;                                                                               \
    T y, x; /* raw sample coordinates, needed for max-mode argmax */                                \
  } PreCalc_##SUFFIX;                                                                               \
                                                                                                    \
  /* cpu/roi_align.cpp:23-108.  Also exported so the GPU test can compare the                       \
   * index/weight table itself bit-for-bit. */                                                      \
  int roi_oracle_sample_table_##SUFFIX(const T* roi5, int height, int width, int pooled_height,     \
                                       int pooled_width, T spatial_scale, int sampling_ratio,       \
                                       int aligned, int* grid_h_out, int* grid_w_out,               \
                                       PreCalc_##SUFFIX** table_out) {                              \
    T offset = aligned ? (T)0.5 : (T)0.0;                                                           \
    T roi_start_w = roi5[1] * spatial_scale - offset;                                               \
    T roi_start_h = roi5[2] * spatial_scale - offset;                                               \
    T roi_end_w = roi5[3] * spatial_scale - offset;                                                 \
    T roi_end_h = roi5[4] * spatial_scale - offset;                                                 \
    T roi_width = roi_end_w - roi_start_w;                                                          \
    T roi_height = roi_end_h - roi_start_h;                                                         \
    if (aligned) {                                                                                  \
      if (!(roi_width >= 0 && roi_height >= 0)) return 2;                                           \
    } else {                                                                                        \
      roi_width = roi_width > (T)1. ? roi_width : (T)1.;                                            \
      roi_height = roi_height > (T)1. ? roi_height : (T)1.;                                         \
    }                                                                                               \
    T bin_size_h = roi_height / (T)pooled_height;                                                   \
    T bin_size_w = roi_width / (T)pooled_width;                                                     \
    int grid_h = (sampling_ratio > 0) ? sampling_ratio : (int)ceilf((float)(roi_height / pooled_height)); \
    int grid_w = (sampling_ratio > 0) ? sampling_ratio : (int)ceilf((float)(roi_width / pooled_width));   \
    if (grid_h < 0) grid_h = 0;                                                                     \
    if (grid_w < 0) grid_w = 0;                                                                     \
    *grid_h_out = grid_h;                                                                           \
    *grid_w_out = grid_w;                                                                           \
    size_t n = (size_t)grid_h * grid_w * pooled_height * pooled_width;                              \
    PreCalc_##SUFFIX* tab = (PreCalc_##SUFFIX*)malloc((n ? n : 1) * sizeof(PreCalc_##SUFFIX));      \
    if (!tab) return 3;                                                                             \
    size_t k = 0;                                                                                   \
    for (int ph = 0; ph < pooled_height; ph++)                                                      \
      for (int pw = 0; pw < pooled_width; pw++)                                                     \
        for (int iy = 0; iy < grid_h; iy++) {                                                       \
          const T yy = roi_start_h + ph * bin_size_h + (T)(iy + .5f) * bin_size_h / (T)grid_h;      \
          for (int ix = 0; ix < grid_w; ix++) {                                                     \
            const T xx = roi_start_w + pw * bin_size_w + (T)(ix + .5f) * bin_size_w / (T)grid_w;    \
            PreCalc_##SUFFIX pc;                                                                    \
            T x = xx, y = yy;                                                                       \
            pc.y = yy;                                                                              \
            pc.x = xx;                                                                              \
            if (y < -1.0 || y > height || x < -1.0 || x > width) {                                  \
              pc.pos1 = pc.pos2 = pc.pos3 = pc.pos4 = 0;                                            \
              pc.w1 = pc.w2 = pc.w3 = pc.w4 = 0;                                                    \
              tab[k++] = pc;                                                                        \
              continue;                                                                             \
            }                                                                                       \
            if (y <= 0) y = 0;                                                                      \
            if (x <= 0) x = 0;                                                                      \
            int y_low = (int)y, x_low = (int)x, y_high, x_high;                                     \
            if (y_low >= height - 1) {                                                              \
              y_high = y_low = height - 1;                                                          \
              y = (T)y_low;                                                                         \
            } else {                                                                                \
              y_high = y_low + 1;                                                                   \
            }                                                                                       \
            if (x_low >= width - 1) {                                                               \
              x_high = x_low = width - 1;                                                           \
              x = (T)x_low;                                                                         \
            } else {                                                                                \
              x_high = x_low + 1;                                                                   \
            }                                                                                       \
            T ly = y - y_low, lx = x - x_low;                                                       \
            T hy = (T)(1. - ly), hx = (T)(1. - lx);                                                 \
            pc.w1 = hy * hx;                                                                        \
            pc.w2 = hy * lx;                                                                        \
            pc.w3 = ly * hx;                                                                        \
            pc.w4 = ly * lx;                                                                        \
            pc.pos1 = y_low * width + x_low;                                                        \
            pc.pos2 = y_low * width + x_high;                                                       \
            pc.pos3 = y_high * width + x_low;                                                       \
            pc.pos4 = y_high * width + x_high;                                                      \
            tab[k++] = pc;                                                                          \
          }                                                                                         \
        }                                                                                           \
    *table_out = tab;                                                                               \
    return 0;                                                                                       \
  }                                                                                                 \
                                                                                                    \
  void roi_oracle_free_##SUFFIX(void* p) { free(p); }                                               \
                                                                                                    \
  /* cpu/roi_align.cpp:110-214.  output is [K,C,PH,PW] (out_layout NCHW) or                         \
   * [K,PH,PW,C] (NHWC); input [N,C,H,W] or [N,H,W,C]. */                                           \
  int roi_oracle_forward_##SUFFIX(const T* input, const T* rois, T* output, T* argmax_y,            \
                                  T* argmax_x, int n_rois, int channels, int height, int width,     \
                                  int pooled_height, int pooled_width, T spatial_scale,             \
                                  int sampling_ratio, int pool_mode, int aligned, int in_layout,    \
                                  int out_layout) {                                                 \
    const size_t hw = (size_t)height * width;                                                       \
    const size_t phw = (size_t)pooled_height * pooled_width;                                        \
    for (int n = 0; n < n_rois; n++) {                                                              \
      const T* roi = rois + (size_t)n * 5;                                                          \
      int roi_batch_ind = (int)roi[0];                                                              \
      int gh, gw;                                                                                   \
      PreCalc_##SUFFIX* tab = 0;                                                                    \
      int rc = roi_oracle_sample_table_##SUFFIX(roi, height, width, pooled_height, pooled_width,    \
                                                spatial_scale, sampling_ratio, aligned, &gh, &gw,   \
                                                &tab);                                              \
      if (rc) return rc;                                                                            \
      const int cnt_i = gh * gw > 1 ? gh * gw : 1;                                                  \
      const T count = (T)cnt_i;                                                                     \
      for (int c = 0; c < channels; c++) {                                                          \
        const T* base;                                                                              \
        size_t pstride;                                                                             \
        if (in_layout == LAYOUT_NCHW) {                                                             \
          base = input + ((size_t)roi_batch_ind * channels + c) * hw;                               \
          pstride = 1;                                                                              \
        } else {                                                                                    \
          base = input + (size_t)roi_batch_ind * hw * channels + c;                                 \
          pstride = (size_t)channels;                                                               \
        }                                                                                           \
        size_t k = 0;                                                                               \
        for (size_t b = 0; b < phw; b++) {                                                          \
          T output_val = 0.;                                                                        \
          T maxval = -10000;                                                                        \
          T maxidx_y = -1.f, maxidx_x = -1.f;                                                       \
          for (int s = 0; s < gh * gw; s++) {                                                       \
            PreCalc_##SUFFIX pc = tab[k++];                                                         \
            T val = pc.w1 * base[pc.pos1 * pstride] + pc.w2 * base[pc.pos2 * pstride] +             \
                    pc.w3 * base[pc.pos3 * pstride] + pc.w4 * base[pc.pos4 * pstride];              \
            if (val > maxval) {                                                                     \
              maxval = val;                                                                         \
              maxidx_y = pc.y;                                                                      \
              maxidx_x = pc.x;                                                                      \
            }                                                                                       \
            output_val += val;                                                                      \
          }                                                                                         \
          size_t oidx = (out_layout == LAYOUT_NCHW)                                                 \
                            ? ((size_t)n * channels + c) * phw + b                                  \
                            : ((size_t)n * phw + b) * channels + c;                                 \
          if (pool_mode == 0) {                                                                     \
            output[oidx] = maxval;                                                                  \
            argmax_y[oidx] = maxidx_y;                                                              \
            argmax_x[oidx] = maxidx_x;                                                              \
          } else {                                                                                  \
            output[oidx] = output_val / count;                                                      \
          }                                                                                         \
        }                                                                                           \
      }                                                                                             \
      free(tab);                                                                                    \
    }                                                                                               \
    return 0;                                                                                       \
  }                                                                                                 \
                                                                                                    \
  /* cpu/roi_align.cpp:216-262 */                                                                   \
  static void grad_weights_##SUFFIX(int height, int width, T y, T x, T* w1, T* w2, T* w3, T* w4,    \
                                    int* x_low, int* x_high, int* y_low, int* y_high) {             \
    if (y < -1.0 || y > height || x < -1.0 || x > width) {                                          \
      *w1 = *w2 = *w3 = *w4 = 0.;                                                                   \
      *x_low = *x_high = *y_low = *y_high = -1;                                                     \
      return;                                                                                       \
    }                                                                                               \
    if (y <= 0) y = 0;                                                                              \
    if (x <= 0) x = 0;                                                                              \
    *y_low = (int)y;                                                                                \
    *x_low = (int)x;                                                                                \
    if (*y_low >= height - 1) {                                                                     \
      *y_high = *y_low = height - 1;                                                                \
      y = (T)*y_low;                                                                                \
    } else {                                                                                        \
      *y_high = *y_low + 1;                                                                         \
    }                                                                                               \
    if (*x_low >= width - 1) {                                                                      \
      *x_high = *x_low = width - 1;                                                                 \
      x = (T)*x_low;                                                                                \
    } else {                                                                                        \
      *x_high = *x_low + 1;                                                                         \
    }                                                                                               \
    T ly = y - *y_low, lx = x - *x_low;                                                             \
    T hy = (T)(1. - ly), hx = (T)(1. - lx);                                                         \
    *w1 = hy * hx, *w2 = hy * lx, *w3 = ly * hx, *w4 = ly * lx;                                     \
  }                                                                                                 \
                                                                                                    \
  /* cpu/roi_align.cpp:270-382; grad_output contiguous in out_layout, grad_input                    \
   * pre-zeroed by the caller in in_layout (mmcv/ops/roi_align.py:113). Sequential                  \
   * accumulation order = the reference's (index-major), so fp32 results are the                    \
   * reference's bit-for-bit; the GPU path (atomics) is compared with a tolerance. */               \
  int roi_oracle_backward_##SUFFIX(const T* grad_output, const T* rois, const T* argmax_y,          \
                                   const T* argmax_x, T* grad_input, int n_rois, int channels,      \
                                   int height, int width, int pooled_height, int pooled_width,      \
                                   T spatial_scale, int sampling_ratio, int pool_mode, int aligned, \
                                   int in_layout, int out_layout) {                                 \
    const size_t hw = (size_t)height * width;                                                       \
    const size_t phw = (size_t)pooled_height * pooled_width;                                        \
    const size_t nthreads = (size_t)n_rois * channels * phw;                                        \
    for (size_t index = 0; index < nthreads; index++) {                                             \
      int pw = (int)(index % pooled_width);                                                         \
      int ph = (int)((index / pooled_width) % pooled_height);                                       \
      int c = (int)((index / pooled_width / pooled_height) % channels);                             \
      int n = (int)(index / pooled_width / pooled_height / channels);                               \
      const T* roi = rois + (size_t)n * 5;                                                          \
      int roi_batch_ind = (int)roi[0];                                                              \
      T offset = aligned ? (T)0.5 : (T)0.0;                                                         \
      T roi_start_w = roi[1] * spatial_scale - offset;                                              \
      T roi_start_h = roi[2] * spatial_scale - offset;                                              \
      T roi_end_w = roi[3] * spatial_scale - offset;                                                \
      T roi_end_h = roi[4] * spatial_scale - offset;                                                \
      T roi_width = roi_end_w - roi_start_w;                                                        \
      T roi_height = roi_end_h - roi_start_h;                                                       \
      if (aligned) {                                                                                \
        if (!(roi_width >= 0 && roi_height >= 0)) return 2;                                         \
      } else {                                                                                      \
        roi_width = roi_width > (T)1. ? roi_width : (T)1.;                                          \
        roi_height = roi_height > (T)1. ? roi_height : (T)1.;                                       \
      }                                                                                             \
      T bin_size_h = roi_height / (T)pooled_height;                                                 \
      T bin_size_w = roi_width / (T)pooled_width;                                                   \
      T* gbase;                                                                                     \
      size_t pstride;                                                                               \
      if (in_layout == LAYOUT_NCHW) {                                                               \
        gbase = grad_input + ((size_t)roi_batch_ind * channels + c) * hw;                           \
        pstride = 1;                                                                                \
      } else {                                                                                      \
        gbase = grad_input + (size_t)roi_batch_ind * hw * channels + c;                             \
        pstride = (size_t)channels;                                                                 \
      }                                                                                             \
      size_t b = (size_t)ph * pooled_width + pw;                                                    \
      size_t oidx = (out_layout == LAYOUT_NCHW) ? ((size_t)n * channels + c) * phw + b              \
                                                : ((size_t)n * phw + b) * channels + c;             \
      const T g = grad_output[oidx];                                                                \
      if (pool_mode == 0) {                                                                         \
        T y = argmax_y[oidx], x = argmax_x[oidx];                                                   \
        if (y != -1.f) {                                                                            \
          T w1, w2, w3, w4;                                                                         \
          int x_low, x_high, y_low, y_high;                                                         \
          grad_weights_##SUFFIX(height, width, y, x, &w1, &w2, &w3, &w4, &x_low, &x_high, &y_low,   \
                                &y_high);                                                           \
          T g1 = g * w1, g2 = g * w2, g3 = g * w3, g4 = g * w4;                                     \
          if (x_low >= 0 && x_high >= 0 && y_low >= 0 && y_high >= 0) {                             \
            gbase[((size_t)y_low * width + x_low) * pstride] += g1;                                 \
            gbase[((size_t)y_low * width + x_high) * pstride] += g2;                                \
            gbase[((size_t)y_high * width + x_low) * pstride] += g3;                                \
            gbase[((size_t)y_high * width + x_high) * pstride] += g4;                               \
          }                                                                                         \
        }                                                                                           \
      } else {                                                                                      \
        int gh = (sampling_ratio > 0) ? sampling_ratio : (int)ceilf((float)(roi_height / pooled_height)); \
        int gw = (sampling_ratio > 0) ? sampling_ratio : (int)ceilf((float)(roi_width / pooled_width));   \
        const T count = (T)(gh * gw);                                                               \
        for (int iy = 0; iy < gh; iy++) {                                                           \
          const T y = roi_start_h + ph * bin_size_h + (T)(iy + .5f) * bin_size_h / (T)gh;           \
          for (int ix = 0; ix < gw; ix++) {                                                         \
            const T x = roi_start_w + pw * bin_size_w + (T)(ix + .5f) * bin_size_w / (T)gw;         \
            T w1, w2, w3, w4;                                                                       \
            int x_low, x_high, y_low, y_high;                                                       \
            grad_weights_##SUFFIX(height, width, y, x, &w1, &w2, &w3, &w4, &x_low, &x_high,         \
                                  &y_low, &y_high);                                                 \
            T g1 = g * w1 / count, g2 = g * w2 / count, g3 = g * w3 / count, g4 = g * w4 / count;   \
            if (x_low >= 0 && x_high >= 0 && y_low >= 0 && y_high >= 0) {                           \
              gbase[((size_t)y_low * width + x_low) * pstride] += g1;                               \
              gbase[((size_t)y_low * width + x_high) * pstride] += g2;                              \
              gbase[((size_t)y_high * width + x_low) * pstride] += g3;                              \
              gbase[((size_t)y_high * width + x_high) * pstride] += g4;                             \
            }                                                                                       \
          }                                                                                         \
        }                                                                                           \
      }                                                                                             \
    }                                                                                               \
    return 0;                                                                                       \
  }

DEFINE_ORACLE(float, f32)
DEFINE_ORACLE(double, f64)

/* Region-token splice (gpt4roi/models/spi_llava.py:99-196, use_im_start_end
 * branch, orig_embeds_params None).  Pure data movement, restated on raw
 * 16-bit rows so it is dtype-agnostic (bf16/fp16).  row_bytes = D*sizeof(elt).
 * Returns 0 ok; 1 = start/end count mismatch (:114-118); 2 = <im_end> not at
 * start+P+1 (:124-128); 3 = #<bbox> != K_i (the shape error at :154); 4 = more
 * than one <im_start> in a sample (the reference loop :120-162 rebuilds the row
 * block from scratch per start token and walks cur_image_idx off the batch
 * alignment, so its result is ill-defined; both oracle and product reject it).
 * A sample with no <im_patch> keeps embed rows (:104-111).
 * Value semantics: the reference forms x*(~mask)+spi (:156-157), which maps
 * -0.0 to +0.0; rows here are moved verbatim, so tests compare with ==
 * (value equality), under which the two agree exactly.  */
int splice_oracle(const int64_t* input_ids, const uint8_t* embed_table, const uint8_t* image_rows,
                  const uint8_t* region_rows, const int32_t* region_offsets /* [B+1] or NULL */,
                  uint8_t* out, int B, int L, int P, size_t row_bytes, int64_t im_patch,
                  int64_t im_start, int64_t im_end, int64_t bbox_tok) {
  for (int b = 0; b < B; b++) {
    const int64_t* ids = input_ids + (size_t)b * L;
    uint8_t* o = out + (size_t)b * L * row_bytes;
    int n_patch = 0, n_start = 0, n_end = 0, n_bbox = 0;
    for (int t = 0; t < L; t++) {
      n_patch += ids[t] == im_patch;
      n_start += ids[t] == im_start;
      n_end += ids[t] == im_end;
      n_bbox += ids[t] == bbox_tok;
      const uint8_t* src = embed_table + (size_t)ids[t] * row_bytes;
      for (size_t i = 0; i < row_bytes; i++) o[(size_t)t * row_bytes + i] = src[i];
    }
    for (int t = 0; t < L; t++)
      if (ids[t] < 0) return 6; /* (checked before the copy above in the product; ids >= V is the caller's job here) */
    if (n_patch == 0) continue;
    if (n_start != n_end) return 1;
    if (n_start > 1) return 4;
    if (n_start == 0) return 5; /* <im_patch> without <im_start>: reference leaves cur_new_input_embeds unbound */
    for (int t = 0; t < L; t++) {
      if (ids[t] != im_start) continue;
      if (t + P + 1 >= L || ids[t + P + 1] != im_end) return 2;
      const uint8_t* src = image_rows + (size_t)b * P * row_bytes;
      for (size_t i = 0; i < (size_t)P * row_bytes; i++) o[(size_t)(t + 1) * row_bytes + i] = src[i];
    }
    if (!region_offsets && n_bbox != 0) return 3; /* assert at spi_llava.py:158-161 */
    if (region_offsets) {
      int k0 = region_offsets[b], k1 = region_offsets[b + 1];
      if (n_bbox != k1 - k0) return 3;
      int k = k0;
      for (int t = 0; t < L; t++) {
        if (ids[t] != bbox_tok) continue;
        const uint8_t* src = region_rows + (size_t)k * row_bytes;
        for (size_t i = 0; i < row_bytes; i++) o[(size_t)t * row_bytes + i] = src[i];
        k++;
      }
    }
  }
  return 0;
}
