/*
 * gpt4roi_b200.h -- C ABI of libgpt4roi_b200.so (sm_90a).
 *
 * Drop-in boundary for the GPT4RoI region-token forward path.  Every entry
 * point takes raw DEVICE pointers, plain sizes and a cudaStream_t (as void*),
 * returns 0 on success or a negative G4R_E* code (message via
 * g4r_last_error()), allocates nothing that outlives the call, and never
 * synchronises the stream unless stated.  No torch types cross this boundary.
 *
 * Each declaration cites the reference interface it replaces; paths are
 * relative to the reference checkout (jshilong/GPT4RoI).
 */
#ifndef GPT4ROI_B200_H_
#define GPT4ROI_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- enums (ints on the wire) ------------------------------------------- */
enum { G4R_F32 = 0, G4R_F16 = 1, G4R_BF16 = 2, G4R_F64 = 3 };       /* dtype   */
enum { G4R_NCHW = 0, G4R_NHWC = 1 };                                /* layout  */
enum { G4R_POOL_MAX = 0, G4R_POOL_AVG = 1 };  /* mmcv/ops/roi_align.py:77 */

enum {
  G4R_OK = 0,
  G4R_EINVAL = -1,   /* bad argument (message says which)                  */
  G4R_ECUDA = -2,    /* CUDA runtime / launch error                        */
  G4R_EUNSUPPORTED = -3,
  G4R_ENODEVICE = -4
};

#define G4R_MAX_LEVELS 4

/* Thread-local message for the last non-zero return on this thread. */
const char* g4r_last_error(void);
/* Library/ABI version (major*1000+minor) and the SM arch it was built for. */
int g4r_version(void);
int g4r_built_arch(void); /* 90 for sm_90a */
/* Keep n_sms SMs free of the persistent (one CTA per SM) wgmma GEMM kernels -- room for the CTAs of a collective
 * that runs beside the backward (the DDP gradient all-reduce of gpt4roi/train/train.py:698-712).  Returns the
 * previous reserve.  Process-wide; 0 (default) = the GEMMs use every SM. */
int g4r_set_sm_reserve(int n_sms);
/* Programmatic dependent launch for the kernels of the decode step behind generate() (llava/model/llava.py:263-283;
 * gpt4roi/app.py:293-300): while on != 0, the small-M GEMM, RMSNorm and single-query attention kernels are launched so
 * that each may start during its predecessor's tail, fetch its first WEIGHT block, and only then wait for the
 * predecessor.  Sound only for a launch sequence in which no kernel writes weights (the decode step); callers switch
 * it on around such a sequence and off again.  Returns the previous setting.  Process-wide; default off. */
int g4r_set_pdl(int on);

/* ---- RoIAlign: operator seam -------------------------------------------- */
/*
 * Replaces mmcv._ext.roi_align_forward
 *   mmcv-1.4.7/mmcv/ops/csrc/pytorch/pybind.cpp:611-615  (python binding)
 *   mmcv-1.4.7/mmcv/ops/csrc/pytorch/roi_align.cpp:25-32 (dispatch)
 *   mmcv-1.4.7/mmcv/ops/csrc/pytorch/cuda/roi_align_cuda.cu:5-30 (launcher)
 *   mmcv-1.4.7/mmcv/ops/csrc/common/cuda/roi_align_cuda_kernel.cuh:17-108
 * input  [N,C,H,W] (G4R_NCHW) or [N,H,W,C] (G4R_NHWC), contiguous, `dtype`
 * rois   [K,5] = (batch_idx, x1, y1, x2, y2), SAME dtype as input (reference
 *        contract, roi_align_cuda.cu:22)
 * output [K,C,PH,PW] (NCHW) or [K,PH,PW,C] (NHWC), `dtype`; fully overwritten
 * argmax_y/argmax_x: same shape as output for G4R_POOL_MAX, ignored for AVG.
 * Arithmetic: index/bin/weight math in fp32 (fp64 for G4R_F64) with the
 * reference's association and no FMA contraction; fp16/bf16 taps are widened
 * to fp32, accumulated in fp32 and rounded once on store.
 */
int g4r_roi_align_forward(const void* input, const void* rois, void* output,
                          void* argmax_y, void* argmax_x,
                          int N, int C, int H, int W, int K,
                          int pooled_height, int pooled_width,
                          float spatial_scale, int sampling_ratio,
                          int pool_mode, int aligned,
                          int dtype, int layout, void* stream);

/*
 * Same operator with a caller-provided scratch buffer: for the NCHW drop-in layout with enough RoIs
 * (g4r_roi_align_forward_workspace() > 0: avg pooling, fp32/fp16/bf16, C a multiple of the 16-byte vector and
 * >= 64, tap work >= twice the map size) the call runs as NCHW->NHWC transpose, the coalesced NHWC kernel, and
 * the transpose back -- three streaming passes instead of the reference layout's plane gather
 * (roi_align_cuda_kernel.cuh:17-108), bit-identical results.  With workspace == NULL, too small, or a
 * configuration the fast path does not cover, it is exactly g4r_roi_align_forward.  workspace: 256-byte aligned.
 */
size_t g4r_roi_align_forward_workspace(int N, int C, int H, int W, int K, int PH, int PW, int sampling_ratio,
                                       int pool_mode, int dtype, int layout);
int g4r_roi_align_forward_ws(const void* input, const void* rois, void* output, void* argmax_y, void* argmax_x,
                             int N, int C, int H, int W, int K, int PH, int PW, float spatial_scale,
                             int sampling_ratio, int pool_mode, int aligned, int dtype, int layout,
                             void* workspace, size_t workspace_bytes, void* stream);

/*
 * Replaces mmcv._ext.roi_align_backward
 *   pybind.cpp:616-620; roi_align.cpp:34-41; roi_align_cuda.cu:32-57;
 *   roi_align_cuda_kernel.cuh:111-210.
 * grad_output contiguous in `layout`; grad_input must be ZEROED by the caller
 * (mmcv/ops/roi_align.py:113) and is accumulated with atomics.
 */
int g4r_roi_align_backward(const void* grad_output, const void* rois,
                           const void* argmax_y, const void* argmax_x,
                           void* grad_input,
                           int N, int C, int H, int W, int K,
                           int pooled_height, int pooled_width,
                           float spatial_scale, int sampling_ratio,
                           int pool_mode, int aligned,
                           int dtype, int layout, void* stream);

/*
 * Fused multi-level RoIAlign (one launch for all levels and all RoIs).
 * Replaces the per-level loop of gpt4roi/models/layers.py:307-313, i.e.
 * 4x { feats[i].to(float32) -> mmcv RoIAlign -> .to(ori_dtype) }.
 * maps[l]   : NHWC [N,H[l],W[l],C], dtype in_dtype (F32, F16 or BF16)
 * scales[l] : spatial_scale of level l as a C float (1/stride)
 * rois      : fp32 [K,5] in input-pixel units (layers.py:294-302)
 * output    : [n_levels,K,PH,PW,C] NHWC, dtype out_dtype; avg pooling only
 * Optional per-(image,channel) affine+ReLU applied to every tap BEFORE the
 * bilinear weights (fuses the last GroupNorm+ReLU of the fuse stack,
 * layers.py:178 / mmcv cnn/bricks/conv_module.py:196-208): for level l, tap
 * value v -> max(v*gn_scale[l][n*C+c] + gn_shift[l][n*C+c], 0); pass NULL
 * arrays to disable.  fp32 [N,C] each.
 */
int g4r_roi_align_mlvl_forward(const void* const* maps, const int* H, const int* W,
                               const float* scales, int n_levels,
                               const float* rois, void* output,
                               int N, int C, int K,
                               int pooled_height, int pooled_width,
                               int sampling_ratio, int aligned,
                               int in_dtype, int out_dtype,
                               const float* const* gn_scale,
                               const float* const* gn_shift,
                               void* stream);

/* Gradient of the above w.r.t. the maps (fp32 NHWC grad maps, pre-zeroed). */
int g4r_roi_align_mlvl_backward(const void* grad_output, const int* H, const int* W,
                                const float* scales, int n_levels,
                                const float* rois, float* const* grad_maps,
                                int N, int C, int K,
                                int pooled_height, int pooled_width,
                                int sampling_ratio, int aligned,
                                int grad_dtype, void* stream);

/* ---- region-token splice: model seam ------------------------------------- */
/*
 * Replaces the per-sample python loop of gpt4roi/models/spi_llava.py:99-196
 * (use_im_start_end branch) including `embed_tokens(input_ids)` (:44-45):
 *   row t of sample b <- embed_table[ids[b,t]]             (default)
 *                     <- image_rows[b, t-(s+1)]            (s = <im_start> pos, s<t<=s+P)
 *                     <- region_rows[region_offsets[b]+j]  (t is the j-th <bbox> of sample b)
 * All rows are `D` elements of a 16-bit type (bf16/fp16); data is moved, never
 * re-rounded.  status[b] (int32, device) receives 0 or the reference's error:
 *   1 = #<im_start> != #<im_end>            (spi_llava.py:114-118)
 *   2 = <im_end> not at s+P+1               (spi_llava.py:124-128)
 *   3 = #<bbox> != K_b                      (shape error at spi_llava.py:154)
 *   4 = more than one <im_start> (unsupported; see DESIGN.md)
 *   5 = <im_patch> present but no <im_start> (reference: unbound variable)
 *   6 = token id outside [0,V) (reference: embedding index error)
 * region_rows/region_offsets may be NULL (bboxes=None, spi_llava.py:83-87): then
 * a <bbox> token present in a multimodal sample is error 3 (assert :158-161).
 * plan: int32 scratch [B,L] (device).
 */
int g4r_splice_region_tokens(const int64_t* input_ids, const void* embed_table,
                             const void* image_rows, const void* region_rows,
                             const int32_t* region_offsets, void* out,
                             int32_t* plan, int32_t* status,
                             int B, int L, int P, int D, int V,
                             int64_t im_patch_token, int64_t im_start_token,
                             int64_t im_end_token, int64_t bbox_token,
                             void* stream);
/*
 * Continuation chunk (multi-turn generation: the tokens after a prefix already held in the KV cache, past the image
 * span; gpt4roi/app.py:110-188,242-328 re-submits the whole conversation every turn): rows come from the embedding
 * table, and the j-th <bbox> of sample b from region_rows[region_offsets[b]+j].  status: 0, 3 (#<bbox> != K_b), 6,
 * or 7 = an <im_patch> / <im_start> / <im_end> token in the chunk.
 */
int g4r_splice_continuation(const int64_t* input_ids, const void* embed_table, const void* region_rows,
                            const int32_t* region_offsets, void* out, int32_t* plan, int32_t* status,
                            int B, int L, int D, int V, int64_t im_patch_token, int64_t im_start_token,
                            int64_t im_end_token, int64_t bbox_token, void* stream);

/* ---- dense contractions on the wgmma tensor cores -------------------------- */
enum { G4R_ACT_NONE = 0, G4R_ACT_RELU = 1, G4R_ACT_QUICK_GELU = 2, G4R_ACT_SWIGLU = 3 };

/*
 * D[M,N] = epilogue(A[M,K] . B[N,K]^T): bf16 operands (both K-major, i.e. B is an
 * nn.Linear weight [out,in]), fp32 accumulation in registers, TMA-fed, persistent.
 * Replaces the cuBLAS calls behind torch.nn.Linear at
 *   gpt4roi/models/layers.py:260-270,326-329  (pos_embedd, flatten_linear, updims)
 *   llava/model/llava.py:52,76 / gpt4roi/models/spi_llava.py:89-97 (mm_projector)
 *   llava/model/llava.py:195,235-236 (lm_head)
 *   transformers CLIP / LLaMA q,k,v,o,fc1,fc2,gate,up,down projections (third party)
 * epilogue: (+bias[N]) -> act -> (+residual[M,N] bf16) -> store bf16 (or fp32 if out_f32).
 *   G4R_ACT_SWIGLU: B rows interleaved (2j = gate_j, 2j+1 = up_j); D is [M,N/2] = silu(g)*u.
 *   k_splits > 1: D is an fp32 buffer [k_splits][M][ldd]; split s writes slab s (no atomics, no
 *   bias/act/residual); the consumer sums the slabs in a fixed order (bitwise reproducible).
 * lda/ldb/ldd/ldr are row strides in elements; lda, ldb multiples of 8.
 */
int g4r_gemm_bf16(const void* A, long long lda, const void* B, long long ldb,
                  void* D, long long ldd, int M, int N, int K,
                  const void* bias, int bias_f32,
                  const void* residual, long long ldr,
                  int act, int out_f32, int k_splits, void* stream);

/* Extended form: residual may be fp32 (residual_f32=1; CLIP's residual stream is fp32 under autocast)
 * and the branch (acc + bias, act) can be rounded to bf16 before the residual add (bias_round_bf16=1),
 * reproducing "bf16 linear output + fp32 stream". */
int g4r_gemm_bf16_ex(const void* A, long long lda, const void* B, long long ldb,
                     void* D, long long ldd, int M, int N, int K,
                     const void* bias, int bias_f32,
                     const void* residual, long long ldr, int residual_f32, int bias_round_bf16,
                     int act, int out_f32, int k_splits, void* stream);

/* Backward-pass GEMM with operand transposes done in the tensor-core descriptors:
 *   D[M,N] = op(A) . op(B)^T ;  a_mn=0: A [M,K] K-contiguous, a_mn=1: A stored [K,M] M-contiguous (lda >= M)
 *                               b_mn=0: B [N,K] K-contiguous, b_mn=1: B stored [K,N] N-contiguous (ldb >= N)
 * For y = x.W^T (torch.nn.functional.linear; every Linear of the LLaMA stack the stage-2 step trains,
 * gpt4roi/train/train.py:698-712 + llava_trainer.py:59-144):
 *   grad_x = grad_y . W      -> g4r_gemm_bf16_t(grad_y, ., 0, W, ., 1, grad_x, ., M, K_in, N_out, ...)
 *   grad_W = grad_y^T . x    -> g4r_gemm_bf16_t(grad_y, ., 1, x, ., 1, grad_W, ., N_out, K_in, M, ...)
 * bf16 operands, fp32 accumulation, bf16 or fp32 (out_f32) output. */
int g4r_gemm_bf16_t(const void* A, long long lda, int a_mn, const void* B, long long ldb, int b_mn,
                    void* D, long long ldd, int M, int N, int K, int out_f32, void* stream);

/* LLaMA QKV projection with apply_rotary_pos_emb fused into the epilogue (transformers
 * modeling_llama.py:138-168): D[M,N] = A.B^T; columns [0,rope_cols) are 128-dim heads rotated with the
 * bf16 cos/sin tables [>= pos0+L, 128] at position pos0 + (row % L) (pos0 > 0: decode steps);
 * rounding points as in the reference's bf16 ops. */
int g4r_gemm_qkv_rope_bf16(const void* A, long long lda, const void* B, long long ldb,
                           void* D, long long ldd, int M, int N, int K,
                           const void* rope_cos, const void* rope_sin, int rope_cols, int L, int pos0,
                           const int* pos0_dev /* device int32 overriding pos0 (CUDA-graph decode) or NULL */,
                           void* stream);

/* ---- decode loop (KV cache) -------------------------------------------------- */
/* Decode-step GEMM (M = batch <= 16 new tokens, one per sample; the LLaMA stack behind generate(), llava.py:263-283,
 * spi_llava.py:47-48), weight-streaming, with the neighbouring memory-bound steps folded in:
 *   out = [RoPE | SwiGLU | + residual]( x . W^T )
 * rope_cos/sin (optional): rotate columns [0, rope_cols) at position pos0 / *pos_dev;
 * kcache / vcache (optional, with RoPE on the fused q|k|v projection, N == 3 * cache_hd): the rotated key and the value
 * columns of sample m are also written to cache[m, pos, :] -- replaces g4r_gemm_qkv_rope_bf16 + g4r_kv_append_bf16
 * (2 launches) of the unfused step. */
int g4r_decode_gemm_bf16(const void* x, long long ldx, const void* W, long long ldw, void* out, long long ldo, int M,
                         int N, int K, int act, const void* residual, long long ldr,
                         const void* rope_cos, const void* rope_sin, int rope_cols, int pos0, const int* pos_dev,
                         void* kcache, void* vcache, int cache_lmax, int cache_hd, void* stream);

/* Append the k and v parts of packed rows [B*Ln, (q|k|v) of width HD each] to the caches
 * [B, Lmax, HD] at positions pos0..pos0+Ln-1 (prefill: pos0=0, Ln=L; decode: Ln=1).  */
int g4r_kv_append_bf16(const void* qkv, long long ld, void* kcache, void* vcache,
                       int B, int Ln, int pos0, const int* pos_dev /* overrides pos0 when non-NULL */,
                       int Lmax, int HD, void* stream);
/* One new query per sample against the first kv_len cached positions: out[b,h,:] =
 * softmax(q.K^T*scale) V.  Replaces the decode-step attention of transformers' LlamaAttention with a
 * DynamicCache (generate() in gpt4roi/app.py:293-300; vision branch skipped, spi_llava.py:47-48). */
int g4r_decode_attention_bf16(const void* q, long long ldq, const void* kcache, const void* vcache,
                              void* out, long long ldo, int B, int H, int head_dim, int kv_len,
                              const int* pos_dev /* kv_len = *pos_dev + 1 when non-NULL; kv_len then sizes smem */,
                              int Lmax, float scale, void* stream);

/* ---- decode loop over prompts of different lengths (per-sample positions) ------------------
 * The four decode entry points above with one position per sample instead of one for the whole batch: pos_rows is a
 * device int32 [B] vector, sample b's new token sits at position pos_rows[b] and attends over cache rows
 * 0..pos_rows[b].  This is what transformers' generate() does for a padded batch (per-row position_ids from the
 * attention mask, padded keys masked out); here the prompts are packed to the left of the cache instead (right
 * padding) and each sample's length lives on the device, so the step stays capturable in a CUDA graph.  The vector is
 * read where the scalar *pos_dev is read, so it may be updated between graph replays.  Results for a vector whose
 * entries are all equal are bitwise those of the scalar entry at that position.  Caller's contract: pos_rows[b] + Ln
 * <= Lmax (append), pos_rows[b] < kv_bound (attention), and the RoPE tables cover every position. */
/* g4r_gemm_qkv_rope_bf16 with row r (sample r / L) rotated at pos_rows[r / L] + r % L. */
int g4r_gemm_qkv_rope_rows_bf16(const void* A, long long lda, const void* B, long long ldb,
                                void* D, long long ldd, int M, int N, int K,
                                const void* rope_cos, const void* rope_sin, int rope_cols, int L,
                                const int* pos_rows, void* stream);
/* g4r_decode_gemm_bf16 with sample m rotated at, and its k / v columns written to cache[m, pos_rows[m], :]. */
int g4r_decode_gemm_rows_bf16(const void* x, long long ldx, const void* W, long long ldw, void* out, long long ldo,
                              int M, int N, int K, int act, const void* residual,
                              long long ldr, const void* rope_cos, const void* rope_sin, int rope_cols,
                              const int* pos_rows, void* kcache, void* vcache, int cache_lmax, int cache_hd,
                              void* stream);
/* g4r_kv_append_bf16 with sample b's rows at positions pos_rows[b] .. pos_rows[b]+Ln-1. */
int g4r_kv_append_rows_bf16(const void* qkv, long long ld, void* kcache, void* vcache,
                            int B, int Ln, const int* pos_rows, int Lmax, int HD, void* stream);
/* g4r_kv_append_rows_bf16 through a cache-row table (continuous batching with prefix reuse: the chunk prefill of several
 * admitted requests whose rows of the batcher's cache are not adjacent; transformers' generate(past_key_values=...)
 * per request, gpt4roi/app.py:242-328 re-submitting the conversation): kcache / vcache are [rows, Lmax, HD]; chunk
 * row b's first qlen[b] rows go to cache row cache_rows[b] at positions pos_rows[b] .. pos_rows[b]+qlen[b]-1 and its
 * padding rows are not written.  cache_rows, qlen: device int32 [B].  Caller's contract: cache_rows[b] < rows and
 * pos_rows[b] + qlen[b] <= Lmax (positions >= Lmax are dropped, never written into the next row). */
int g4r_kv_append_rows_at_bf16(const void* qkv, long long ld, void* kcache, void* vcache, int B, int Ln,
                               const int* pos_rows, const int* cache_rows, const int* qlen, int Lmax, int HD,
                               void* stream);
/* g4r_decode_attention_bf16 with sample b over its first pos_rows[b] + 1 cached positions; kv_bound (>= every
 * pos_rows[b] + 1, e.g. Lmax in a CUDA graph) sizes the split-KV factor and the shared-memory score buffer. */
int g4r_decode_attention_rows_bf16(const void* q, long long ldq, const void* kcache, const void* vcache,
                                   void* out, long long ldo, int B, int H, int head_dim, int kv_bound,
                                   const int* pos_rows, int Lmax, float scale, void* stream);
/* g4r_decode_attention_rows_bf16 for beam search: the caches are shared by all R rows, and key / value p of row r is
 * read from cache row anc[r * Lmax + p] (device int32 [R, Lmax], the ancestry table) instead of row r. */
int g4r_decode_attention_beam_bf16(const void* q, long long ldq, const void* kcache, const void* vcache,
                                   void* out, long long ldo, int R, int H, int head_dim, int kv_bound,
                                   const int* pos_rows, const int* anc, int Lmax, float scale, void* stream);
/* Decode attention for N sampled rows per prompt that share the prompt's keys (generate(num_return_sequences=N,
 * do_sample=True)): caches [B + B*N, Lmax, H*head_dim], rows 0..B-1 the prompts, row B + r the generated positions of
 * query row r = b*N + i (q: B*N rows of pitch ldq; out: B*N rows of pitch ldo).  Row r attends over positions
 * 0..prompt_lens[b]-1 of cache row b and prompt_lens[b]..pos_rows[r] of cache row B + r (prompt_lens: device int32
 * [B]; pos_rows: device int32 [B*N], pos_rows[r] >= prompt_lens[b] - 1).  Each prompt key / value row is read from HBM
 * once per step for all N rows.  prompt_bound (>= every prompt_lens[b]) and gen_bound (>= every row's count of own
 * keys, pos_rows[r] + 1 - prompt_lens[b]) size the split-KV factor and the score buffer.  1 <= N <= 16, head_dim 128;
 * anything else is refused. */
int g4r_decode_attention_group_bf16(const void* q, long long ldq, const void* kcache, const void* vcache,
                                    void* out, long long ldo, int B, int N, int H, int head_dim, int prompt_bound,
                                    int gen_bound, const int* prompt_lens, const int* pos_rows, int Lmax, float scale,
                                    void* stream);

/* ---- beam search step (the beam decode loop's last two kernels) -----------------------------
 * One step of transformers' GenerationMixin._beam_search with do_sample=False for B samples of N beams, on logits
 * (16-bit rows, pitch ld: B*N rows; row_div = N reads sample b's single row for all its beams, the first step
 * from the prefill logits, else 1).  K = beams_to_keep = max(2, 1 + n_eos) * N; eos_ids: device int32 [n_eos].
 * prompt_len: the padded prompt length, max_length = prompt_len + max_new_tokens, early_stopping 0 (False), 1 (True)
 * or 2 ("never").  G: generated columns of run_seq / fin_seq (int64 [2, B, N, G], double-buffered by the parity of the
 * step).  state: int32 [4B + 2] (per sample: tokens generated, early-stop heuristic unsatisfied, flags; then a ticket
 * and the batch's done word); run_score: fp32 [B*N]; cand_score / cand_tok: [B*N*K] scratch; fin_score: fp32 [B, N];
 * fin_state: int32 [B, N, 2] (finished, generated length).  Writes the next ids (int64 [B*N]), each beam row's
 * position pos_rows = lens[b] + g and the ancestry table anc (int32 [B*N, Lmax]: generated columns permuted to the new
 * parents, the new position pointing at cache row B + r).  Ties in score go to the lower flat index beam * V + token.
 * Capturable: every per-step value is read from device memory. */
int g4r_beam_step_bf16(const void* logits, long long ld, int row_div, int B, int N, int V, int K, const int* eos_ids,
                       int n_eos, int prompt_len, int max_length, double length_penalty, int early_stopping, int G,
                       int Lmax, const int* lens, int* state, float* run_score, float* cand_score, int* cand_tok,
                       long long* run_seq, long long* fin_seq, float* fin_score, int* fin_state, long long* ids,
                       int* pos_rows, int* anc, void* stream);

/* g4r_beam_step_bf16 (same arguments, same step) with transformers' generate() outputs for return_dict_in_generate:
 *   scores / raw_logits (fp32 [n_slots, B*N, V], contiguous, either may be NULL): slot g = state[4b] (the step's
 *     generated-token count) of beam row r gets the row's log_softmax, (x - max) - log sum exp(x - max), before the
 *     running score is added (HF's scores entry), and the widened logits; at the first step (row_div = N) each
 *     sample's single row is written for all its N beams;
 *   run_bidx / fin_bidx (int32 [2, B, N, G], both or neither; initialised to -1): HF's beam_indices beside run_seq /
 *     fin_seq, double-buffered and gathered as they are; column g of a new beam holds b * N + its parent beam. */
int g4r_beam_step_out_bf16(const void* logits, long long ld, int row_div, int B, int N, int V, int K,
                           const int* eos_ids, int n_eos, int prompt_len, int max_length, double length_penalty,
                           int early_stopping, int G, int Lmax, const int* lens, int* state, float* run_score,
                           float* cand_score, int* cand_tok, long long* run_seq, long long* fin_seq, float* fin_score,
                           int* fin_state, long long* ids, int* pos_rows, int* anc, float* scores, float* raw_logits,
                           int n_slots, int* run_bidx, int* fin_bidx, void* stream);

/* ---- next-token selection (the decode loop's last kernel) ------------------------------------
 * logits: 16-bit [B, V] rows, row pitch ld elements.  Writes out_ids[b] (int64, like the decode step's ids buffer).
 * greedy != 0: the arg-max of each row, first index among equal values -- replaces the `argmax` of transformers'
 *   GenerationMixin._sample (and torch.argmax in general; NaN counts as the largest value).
 * greedy == 0: a draw from the processed softmax, in transformers' order (logits_process.py), on the logits widened to
 *   fp32 as HF's `.float()` does: TemperatureLogitsWarper (s = x / temperature, a division), then TopKLogitsWarper when
 *   0 < top_k < V (keep s >= the k-th largest s, duplicates counted), then TopPLogitsWarper when top_p < 1
 *   (min_tokens_to_keep = 1; keep each value whose strictly larger survivors hold less than top_p of the survivors'
 *   softmax mass -- a group of equal values at the boundary is kept whole, where HF's unstable sort may split it),
 *   then the softmax + multinomial of GenerationMixin._sample, by inverse CDF over (value descending, index ascending).
 *   The uniform is Philox4x32-10 with key = seed and counter = (*rng_step, b, 0): (word0 >> 8) * 2^-24.  The result
 *   is a function of the logits, seed and *rng_step alone (no float atomics), so a CUDA graph that captured this call
 *   draws afresh on every replay once the caller advances *rng_step.  Needs V < 65536.
 * eos_id >= 0 and pad_id >= 0 and finished (device int32 [B]) non-NULL: transformers' eos -> pad rule -- a row with
 *   finished[b] set gets pad_id, a row that emits eos_id sets finished[b].
 * Capturable: every per-step value is read from device memory. */
int g4r_sample_tokens_bf16(const void* logits, long long ld, int B, int V, float temperature, int top_k, float top_p,
                           int greedy, unsigned long long seed, const long long* rng_step, int eos_id, int pad_id,
                           int* finished, long long* out_ids, void* stream);

/* ---- next-token selection with transformers' history-dependent logits processors ----------------
 * g4r_sample_tokens_bf16 (same arguments, same selection and eos -> pad rule) on the processed fp32 scores that
 * transformers' GenerationMixin._sample builds before TemperatureLogitsWarper (logits_process.py, in its order):
 *   RepetitionPenaltyLogitsProcessor (repetition_penalty != 1): every id present in the history h gets
 *     x < 0 ? x * penalty : x / penalty (fp32 multiply / IEEE division of the widened logit), once however often it
 *     occurs;
 *   NoRepeatNGramLogitsProcessor (no_repeat_ngram_size n > 0): when len(h) + 1 >= n, t gets -inf if an n-gram lying
 *     wholly in h has its first n - 1 ids equal to the last n - 1 ids of h and ends in t (n = 1: every id of h);
 *   MinLengthLogitsProcessor (len(h) < min_length) and MinNewTokensLengthLogitsProcessor (*rng_step < min_new_tokens):
 *     eos_ids[0 .. n_eos) get -inf.
 * Greedy: the arg-max of the processed scores, first index among equals.  Sampling: temperature -> top-k -> top-p ->
 * inverse CDF as g4r_sample_tokens_bf16, over the processed values; -inf ids have probability 0 and equal processed
 * values form one group whichever ids they come from.
 * history: int64 [B, ld_h], row pitch ld_h; row b's history is h = history[b, 0 .. L + *rng_step) (the prompt as given,
 * then the ids selected so far).  append != 0: after the eos -> pad rule, the selected id is written to
 * history[b, L + *rng_step] (when that is < ld_h), so the next call sees it.  rng_step is required, also for greedy.
 * Sampling with repetition_penalty != 1 needs ld_h <= 8192 (the penalised ids are listed in shared memory).  V < 65536.
 * Capturable: every per-step value is read from device memory. */
int g4r_sample_tokens_proc_bf16(const void* logits, long long ld, int B, int V, float temperature, int top_k,
                                float top_p, int greedy, unsigned long long seed, const long long* rng_step, int eos_id,
                                int pad_id, int* finished, long long* out_ids, long long* history, long long ld_h, int L,
                                float repetition_penalty, int no_repeat_ngram_size, int min_length, int min_new_tokens,
                                const int* eos_ids, int n_eos, int append, void* stream);

/* ---- next-token selection with transformers' generate() outputs (return_dict_in_generate) ------
 * g4r_sample_tokens_proc_bf16 (same arguments, same selection, eos -> pad rule and history append) followed by an
 * output pass into slot s = *rng_step of two fp32 buffers [n_slots, B, V] (contiguous; a slot >= n_slots is not
 * written):
 *   scores[s, b, :]: HF's next_token_scores -- the widened logits through the history-dependent processors, then,
 *     when sampling, / temperature (IEEE division) and -inf below the top-k and top-p thresholds the selection uses
 *     (the top-p group of equal values at the boundary kept whole, as the selection keeps it); greedy: no warpers;
 *   raw_logits[s, b, :]: HF's next_token_logits, the logits widened to fp32.
 * Either pointer may be NULL; with both NULL the call launches exactly what g4r_sample_tokens_bf16 (history NULL) or
 * g4r_sample_tokens_proc_bf16 launches.  history may be NULL: the plain selection, with every processor neutral
 * (repetition_penalty 1, no_repeat_ngram_size 0, n_eos 0), else refused.  With an output rng_step is required.
 * Capturable: every per-step value is read from device memory. */
int g4r_sample_tokens_out_bf16(const void* logits, long long ld, int B, int V, float temperature, int top_k,
                               float top_p, int greedy, unsigned long long seed, const long long* rng_step, int eos_id,
                               int pad_id, int* finished, long long* out_ids, long long* history, long long ld_h, int L,
                               float repetition_penalty, int no_repeat_ngram_size, int min_length, int min_new_tokens,
                               const int* eos_ids, int n_eos, int append, float* scores, float* raw_logits,
                               long long n_slots, void* stream);

/* ---- next-token selection with a rule per row (a continuous batch of independent requests) -------
 * logits: 16-bit [S, V] rows, row pitch ld elements.  Per-row device arrays of S entries: greedy (int32), temperature
 * (fp32), top_k (int32, 0: off), top_p (fp32, 1: off), seed (uint64), step (int64: the row's Philox counter and
 * token count), eos_id (int32, -1: none), active (int32).  For every row r with active[r] != 0, the selection of
 * g4r_sample_tokens_bf16 on row r's parameters, with Philox counter (step[r], 0, 0) -- the token a B = 1 call with
 * the same logits, seed and *rng_step = step[r] selects; greedy and sampled rows may share one launch.  Then
 * out_ids[r] = the token, finished[r] = 1 when it equals eos_id[r] (no pad rule), step[r] += 1, and, when lens
 * (int32 [S], the KV cache's per-row lengths) is non-NULL, lens[r] += 1 as the launch's last write.  A row with
 * active[r] == 0 is left alone: finished, step, lens and out_ids[r] keep their values.  Needs V < 65536; a sampled
 * row needs temperature > 0 and top_p >= 0 (the caller's check: the rule is device data).
 * Capturable: every per-step value is read from device memory. */
int g4r_sample_tokens_rows_bf16(const void* logits, long long ld, int S, int V, const int* greedy,
                                const float* temperature, const int* top_k, const float* top_p,
                                const unsigned long long* seed, long long* step, const int* eos_id, const int* active,
                                int* finished, long long* out_ids, int* lens, void* stream);

/* ---- next-token selection with a rule and history-dependent processors per row -------------------
 * Replaces, per request of a continuous batch, the logits processors transformers' GenerationMixin._sample runs before
 * TemperatureLogitsWarper (RepetitionPenaltyLogitsProcessor, NoRepeatNGramLogitsProcessor, MinLengthLogitsProcessor,
 * MinNewTokensLengthLogitsProcessor), with each request's own values.
 * g4r_sample_tokens_rows_bf16 (same arguments, same per-row rule, Philox counter (step[r], 0, 0), finished / step /
 * lens updates) where row r's processors are g4r_sample_tokens_proc_bf16's with
 *   history: int64 [S, ld_h], row pitch ld_h: row r's history is history[r, 0 .. prompt_len[r] + step[r]);
 *   repetition_penalty (fp32, 1: off), no_repeat_ngram_size, min_length, min_new_tokens (int32): entry r;
 *   eos_ids: int32 [S, 4], the first n_eos[r] of row r are the ids the minimum lengths suppress.
 * An active row whose four processors are neutral (penalty 1, n-gram size 0, and no minimum length or n_eos[r] == 0)
 * selects exactly as g4r_sample_tokens_rows_bf16; any other active row selects as a B = 1 g4r_sample_tokens_proc_bf16
 * call on its logits with L = prompt_len[r] and *rng_step = step[r], and writes its token to
 * history[r, prompt_len[r] + step[r]] (when that is < ld_h).  Inactive rows are left alone.  Sampling with a
 * repetition penalty lists at most min(ld_h, 8192) penalised ids per row (the caller's check).  V < 65536.
 * Capturable: every per-step value is read from device memory. */
int g4r_sample_tokens_rows_proc_bf16(const void* logits, long long ld, int S, int V, const int* greedy,
                                     const float* temperature, const int* top_k, const float* top_p,
                                     const unsigned long long* seed, long long* step, const int* eos_id,
                                     const int* active, int* finished, long long* out_ids, int* lens,
                                     long long* history, long long ld_h, const int* prompt_len,
                                     const float* repetition_penalty, const int* no_repeat_ngram_size,
                                     const int* min_length, const int* min_new_tokens, const int* eos_ids,
                                     const int* n_eos, void* stream);

/* ---- stop strings (after the next-token selection, once per decode step) ---------------------
 * Replaces transformers.generation.stopping_criteria.StopStringCriteria.__call__ (and, per row, the reference's
 * KeywordsStoppingCriteria, llava/model/utils.py:26-46) for the decode loop: a row stops at the first generated token
 * in which an occurrence of a stop string ends.  The matcher is a table built once on the host:
 * step: int16 [V_tok + 1, S], row pitch ld elements; entry (t, s) = the matcher's state after token t is fed from state
 * s (low 15 bits), bit 15 set when an occurrence ended inside token t.  Row V_tok is the reset row.
 * For every row b with finished[b] == 0:  e = step[t][state[b]], t = ids[b] if 0 <= ids[b] < V_tok else V_tok;
 * state[b] = e & 0x7FFF; finished[b] = 1 if e < 0.  Rows with finished[b] != 0 are left untouched.
 * ids: int64 [B] (what g4r_sample_tokens wrote); state, finished: int32 [B].  S in 1..32767.
 * Capturable: every per-step value is read from device memory. */
int g4r_stop_step(const long long* ids, const short* step, long long ld, int V_tok, int S, int B, int* state,
                  int* finished, void* stream);

/* g4r_stop_step with a table per row (transformers' StopStringCriteria of each request of a continuous batch):
 * tables: B device pointers, row b's table int16 [V_tok + 1, S[b]] (row pitch S[b]) or NULL (no stop strings); one
 * V_tok for every table.  For every row b with active[b] != 0, finished[b] == 0 and a table:
 * e = tables[b][t][state[b]], t = ids[b] if 0 <= ids[b] < V_tok else V_tok; state[b] = e & 0x7FFF; finished[b] = 1 if
 * e < 0.  Other rows are left untouched.  ids: int64 [B]; S, active, state, finished: int32 [B].
 * Capturable: every per-step value is read from device memory. */
int g4r_stop_step_rows(const long long* ids, const short* const* tables, const int* S, int V_tok, int B,
                       const int* active, int* state, int* finished, void* stream);

/* ---- prompt-lookup decoding (batch 1; the last launch of each verify step) ---------------------
 * Replaces transformers' PromptLookupCandidateGenerator.get_candidates and the acceptance of
 * GenerationMixin._assisted_decoding (greedy / non-speculative-sampling branch) for generate(prompt_lookup_num_tokens=k).
 * The verify step feeds M = k + 1 rows: ids[0] the last accepted token, ids[1..d] the d drafts (rows past d repeat
 * ids[0]), at positions pos[i] = base[0] + i, and selects sel[i] per row.
 * hist: int64 [ld_h], the prompt then the accepted tokens; state: int32 [5] = {len, d, finished, appended, host_done};
 * base: int32 [1]; pos: int32 [M]; step: int64 [M] (row i's Philox counter, the index of the new token it decides);
 * eos: int32 [n_eos]; readback: int64 [4 + M + k] = {appended, finished, len, d, the appended tokens [M], the next
 * drafts [k] (-1 past d)}.
 * g4r_lookup_step: n = the count of leading drafts ids[1 + i] equal to sel[i]; if the candidate sequence was done
 * (len + d >= max_length, or host_done != 0: the host's stopping criteria on it) and n == d > 0, n -= 1; then
 * min(n + 1, max_length - len) tokens sel[0..] are appended to hist, len advances by as many, and finished is set when
 * one of them is an eos id.  Then, as g4r_lookup_draft, the next draft from hist[0..len): for g = min(max_ngram,
 * len - 1) down to 1, the smallest idx with hist[idx..idx+g) == hist[len-g..len) and idx + g < min(len, max_length)
 * wins; the draft is hist[idx+g .. min(idx+g+k, len, max_length)) cut before its first eos id (no draft when
 * finished, when len + 1 >= max_length, or when no window matches).  Writes ids, pos, base, step (= len - prompt_len
 * + i), state and readback.  max_length: prompt_len + max_new_tokens (<= ld_h).
 * Capturable: every per-step value is read from device memory. */
int g4r_lookup_step(const long long* sel, long long* ids, long long* hist, long long ld_h, int k, int max_ngram,
                    int prompt_len, int max_length, const int* eos, int n_eos, int* state, int* base, int* pos,
                    long long* step, long long* readback, void* stream);
int g4r_lookup_draft(long long* ids, long long* hist, long long ld_h, int k, int max_ngram, int prompt_len,
                     int max_length, const int* eos, int n_eos, int* state, int* base, int* pos, long long* step,
                     long long* readback, void* stream);

/*
 * NHWC convolution as an implicit GEMM (stride 1, pad (ksize-1)/2, ksize 1 or 3):
 *   Y[n,y,x,co] = act( sum_{ky,kx,ci} X[n,y+ky-1,x+kx-1,ci] * Wt[co,(ky*ks+kx)*Cin+ci] + bias[co] )
 * X bf16 [n_img,H,W,Cin]; Wt bf16 [Cout, ks*ks*Cin] (torch [Cout,Cin,kh,kw] permuted to
 * [Cout,kh,kw,Cin] once at load time); Y bf16 [n_img,H,W,Cout].  The A operand is fetched
 * with 4-D TMA boxes shifted by the filter tap; TMA's out-of-bounds zero fill is the padding.
 * Replaces cuDNN behind nn.Conv2d at gpt4roi/models/layers.py:129-144,191,178 (input_conv,
 * fuse_convs[i].conv) and :257-259,320-325 (pconvs).
 * levels > 1 sums `levels` convolutions in one contraction (K concatenated): X is
 * [levels*n_img,H,W,Cin] (level-major), Wt [Cout, levels*ks*ks*Cin]; this is
 * sum_l pconvs[l](roi_feats[l]) of layers.py:320-325 as ONE GEMM.
 * gn_stats (optional, fp32 [n_img, g4r_conv_gn_slots(H,W), gn_groups, 2]): per-(tile,warp) partial
 * sum / sum of squares of the bf16-rounded output per (image, 16-channel group) -- the statistics
 * GroupNorm(64) needs (mmcv cnn/bricks/conv_module.py:196-208) -- written with plain stores
 * (reproducible) and summed in a fixed order by g4r_gn_finalize; no extra pass over Y.
 */
int g4r_conv_gn_slots(int H, int W);
int g4r_conv_nhwc_bf16(const void* X, const void* Wt, void* Y,
                       int n_img, int H, int W, int Cin, int Cout, int ksize, int levels,
                       const void* bias, int bias_f32, int act,
                       float* gn_stats, int gn_groups, void* stream);

/* ---- fused attention ------------------------------------------------------- */
/*
 * out[b,i,h,:] = softmax_j( (q_i.k_j) * scale [+ causal mask] ) . v_j   (scores kept in fp32)
 * q/k/v: bf16, element (b, token, head h, d) at  base + b*bs + token*ld + h*head_dim + d
 * (so the packed [B,L,(q|k|v)] output of the QKV GEMM is read in place); out likewise with
 * ldo/bso.  head_dim 64 (CLIP-ViT-L/14) or 128 (LLaMA-7B).  Replaces transformers'
 * eager_attention_forward (modeling_clip.py / modeling_llama.py:199-222), third party to the
 * reference (pyproject.toml:19).
 */
int g4r_attention_bf16(const void* q, const void* k, const void* v, void* out,
                       long long ld, long long bs, long long ldo, long long bso,
                       int B, int H, int L, int head_dim, int causal, float scale,
                       const int* seqlens /* device int32 [B] or NULL: keys >= seqlens[b] are masked */,
                       void* stream);

/*
 * Same contract on the wgmma tensor cores (TMA-fed, S and O accumulators in registers, V consumed as an
 * MN-major operand); requires the packed layout bs == L*ld.  csrc/attention_wgmma.cu.
 */
int g4r_attention_tc_bf16(const void* q, const void* k, const void* v, void* out,
                          long long ld, long long bs, long long ldo, long long bso,
                          int B, int H, int L, int head_dim, int causal, float scale,
                          const int* seqlens, void* stream);

/*
 * Chunk attention over the KV cache (multi-turn generation: gpt4roi/app.py:110-188,242-328 appends each answer and
 * the next question to the conversation and generates again; transformers' generate(past_key_values=...) reuses the
 * cache of the earlier turns).  q: the chunk's packed, RoPE-rotated rows [B*Lc, >= H*head_dim] (row stride ldq);
 * kcache / vcache: [B, lmax, H*head_dim], the chunk's own K/V already appended at positions start[b]..;
 * start: device int32 [B], the number of cached tokens before row b's chunk; qlen: device int32 [B] valid queries of
 * each right-padded row, or NULL (all Lc).  Query i of row b attends over cache positions 0 .. start[b] + i; output
 * rows >= qlen[b] hold finite filler (zeros for 128-row tiles wholly past qlen[b]).  Cache rows past start[b] + qlen[b], up to the next multiple of 64, must hold finite
 * values (the engine's cache is zero-filled).  head_dim 64 or 128; out [B*Lc, H*head_dim] with row stride ldo.
 */
int g4r_attention_cached_bf16(const void* q, long long ldq, const void* kcache, const void* vcache, int lmax,
                              void* out, long long ldo, int B, int H, int Lc, int head_dim, float scale,
                              const int* start, const int* qlen, void* stream);
/* g4r_attention_cached_bf16 through a cache-row table (the same reuse as g4r_kv_append_rows_at_bf16): kcache / vcache
 * are [rows, lmax, H*head_dim] and chunk row b attends over cache row cache_rows[b] (device int32 [B], each < rows)
 * instead of row b.  The same CACHED rules: key blocks aligned to position 0, 128-row tiles wholly past qlen[b] zeroed,
 * the last key block reading cache row positions up to the next multiple of 64 (finite values required; past the last
 * cache row they read as zeros). */
int g4r_attention_cached_rows_bf16(const void* q, long long ldq, const void* kcache, const void* vcache, int rows,
                                   int lmax, void* out, long long ldo, int B, int H, int Lc, int head_dim, float scale,
                                   const int* start, const int* qlen, const int* cache_rows, void* stream);

/* ---- HBM-bound glue (csrc/elementwise.cu); bf16 rows, fp32 math ------------- */
/* nn.LayerNorm over the last dim (CLIP layer norms; gpt4roi/models/layers.py:263,266). */
int g4r_layernorm_bf16(const void* x, long long ldx, const void* w, const void* b,
                       void* out, long long ldo, int M, int D, float eps, void* stream);
/* LayerNorm with fp32 or bf16 input/output rows (x_f32 / out_f32).  Under autocast the reference's
 * nn.LayerNorm returns fp32, so CLIP's residual stream is fp32: pre_layrnorm is bf16->fp32, layer_norm1/2
 * are fp32->bf16 (their output is cast to bf16 by the following autocast Linear). */
int g4r_layernorm_ex(const void* x, long long ldx, int x_f32, const void* w, const void* b,
                     void* out, long long ldo, int out_f32, int M, int D, float eps, void* stream);
/* fp32 rows [B][rows_per_batch][D] (row stride ld, batch stride bst) -> dense bf16 [B*rows_per_batch, D]
 * (the autocast cast at mm_projector's input, spi_llava.py:89-93, skipping the CLS row). */
int g4r_cast_f32_bf16(const void* x, long long ld, long long bst, void* out,
                      int B, int rows_per_batch, int D, void* stream);
/* LlamaRMSNorm: w * bf16(x * rsqrt(mean(x^2)+eps))  (transformers modeling_llama.py:53-67). */
int g4r_rmsnorm_bf16(const void* x, long long ldx, const void* w,
                     void* out, long long ldo, int M, int D, float eps, void* stream);
/* Same for an fp32 (x_f32=1) or bf16 residual stream; bf16 output rows (the operand of the next GEMM).  With an
 * fp32 stream the normalised value is not rounded before the weight multiply, exactly LlamaRMSNorm on an fp32
 * input (modeling_llama.py:53-67: `self.weight * hidden_states.to(input_dtype)`) -- the reference's residual stream
 * is fp32 whenever its parameters are (training under autocast), bf16 when the model was cast to bf16. */
int g4r_rmsnorm_ex(const void* x, long long ldx, int x_f32, const void* w, void* out, long long ldo, int M, int D,
                   float eps, void* stream);
/* apply_rotary_pos_emb in place on the first n_heads_qk heads of each packed row
 * (modeling_llama.py:138-168); cos/sin bf16 [L, head_dim]; position = row % L. */
int g4r_rope_inplace_bf16(void* qkv, long long ld, const void* cos_t, const void* sin_t,
                          int rows, int L, int n_heads_qk, int head_dim, void* stream);
/* CLIP patchify (im2col of the stride-14 patch_embedding conv, modeling_clip.py:148-154):
 * img bf16 [B,3,S,S] -> out bf16 [B*(S/ps)^2, Kpad], column (c*ps+ky)*ps+kx, zero padded. */
int g4r_patchify_bf16(const void* img, void* out, int B, int S, int ps, int Kpad, void* stream);
/* [CLS | patches] + position_embedding  (modeling_clip.py:209-216). */
int g4r_vit_embed_bf16(const void* patch, const void* cls, const void* pos, void* out,
                       int B, int P, int D, void* stream);
/* ViT tokens [B,G*G,C] (row stride ldt, batch stride bst) -> bilinear align_corners resize to
 * [B,Ho,Ho,Cpad] NHWC with the two coordinate channels appended and zero padding
 * (gpt4roi/models/layers.py:219-232 + :117-126,185-188). */
int g4r_upsample_tokens_coords_bf16(const void* tok, long long ldt, long long bst, void* out,
                                    int B, int G, int Ho, int C, int Cpad, void* stream);
/* same with fp32 tokens (CLIP hidden states are fp32 under autocast) */
int g4r_upsample_tokens_coords_f32(const void* tok, long long ldt, long long bst, void* out,
                                   int B, int G, int Ho, int C, int Cpad, void* stream);
/* One level of MLVLFuseModule._single_shuffle (layers.py:152-180): out = [own[:, :C/2] |
 * resize(top[:, 3C/4:]) | resize(down[:, C/2:3C/4])]; optional per-(image,channel) scale/shift
 * (fp32 [B,C]) apply the previous round's GroupNorm+ReLU to every tap first. */
int g4r_fuse_gather_bf16(const void* own, const float* own_sc, const float* own_sh, int H,
                         const void* top, const float* top_sc, const float* top_sh, int Ht,
                         const void* down, const float* down_sc, const float* down_sh, int Hd,
                         void* out, int B, int C, void* stream);
/* GroupNorm statistics -> per-(image,channel) scale/shift (torch.nn.GroupNorm semantics). */
int g4r_gn_finalize(const float* stats, const void* gamma, const void* beta,
                    float* scale, float* shift, int B, int C, int groups, int slots,
                    float count, float eps, void* stream);
/* pos_embedd MLP of MlvlRoIExtractor (layers.py:260-267,285): boxes fp32 [K,4] -> fp32 [K,1024]. */
int g4r_pos_embed_mlp(const float* boxes, const void* w0, const void* b0, const void* g2,
                      const void* be2, const void* w3, const void* b3, const void* g5,
                      const void* be5, float* out, int K, float eps, void* stream);
/* out = bf16( bf16(sum_s acc[s] + bias) + pos )  (layers.py:327-328). acc fp32 [splits,K,D]
 * (split-K slabs of flatten_linear), pos fp32 [K,D]. */
int g4r_add_bias_pos_cast(const float* acc, int splits, const void* bias, const float* pos, void* out,
                          int K, int D, void* stream);

/* ---- training step (SURVEY.md 8(a) row 14; gpt4roi/train/train.py:698-712 + HF Trainer) ----------------
 * Cross entropy of llava/model/llava.py:238-249 (CrossEntropyLoss(): mean over targets != -100) on rows of
 * bf16 logits [M,V]; `targets` are the already shifted labels (labels[..., 1:], last position -100).
 * Writes row_lse[M], row_loss[M], loss_count[2] = {mean loss, #valid rows} and, if dlogits != NULL,
 * dlogits = (softmax - onehot) * grad_scale / count (bf16, a separate buffer).  No atomics. */
int g4r_cross_entropy_bf16(const void* logits, long long ld, const long long* targets, int M, int V,
                           float* row_lse, float* row_loss, float* loss_count, void* dlogits, long long ldd,
                           float grad_scale, void* stream);

/* LlamaRMSNorm backward (transformers modeling_llama.py LlamaRMSNorm.forward): dx bf16 [M,D], dw fp32 [D].
 * dw_slabs: fp32 scratch [g4r_rmsnorm_bwd_slabs(M)][D] (per-CTA partial sums, reduced in fixed order). */
int g4r_rmsnorm_bwd_slabs(int M);
int g4r_rmsnorm_bwd_bf16(const void* x, long long ldx, const void* w, const void* dy, long long ldy,
                         const void* dres /* optional bf16 [M,D]: added to dx (gradient of the residual branch) */,
                         long long ldr, void* dx, long long ldd, float* dw, float* dw_slabs, int M, int D, float eps,
                         void* stream);

/* SwiGLU on an interleaved gate/up buffer gu [M,2F] (col 2j gate_j, 2j+1 up_j): f = silu(g)*u [M,F], and its
 * backward dgu [M,2F] from df [M,F] (transformers LlamaMLP.forward). */
int g4r_swiglu_fwd_bf16(const void* gu, long long ldg, void* f, long long ldf, long long M, int F, void* stream);
int g4r_swiglu_bwd_bf16(const void* gu, long long ldg, const void* df, long long ldf, void* dgu, long long ldd,
                        long long M, int F, void* stream);

/* Causal attention for training: forward that also writes lse[B,H,L] (fp32 log-sum-exp of the scaled scores),
 * and the backward (autograd of transformers modeling_llama.py:199-222 eager attention): packed dQ|dK|dV rows
 * from q,k,v (after RoPE), the forward output `out`, `dout` and `lse`.  delta: fp32 scratch [B,H,L].
 * q/k/v: row stride ld, batch stride bs (elements); out/dout: ldo, bso; dq/dk/dv: ldg, bsg.  No atomics. */
int g4r_attention_fwd_lse_bf16(const void* q, const void* k, const void* v, void* out, long long ld,
                               long long bs, long long ldo, long long bso, int B, int H, int L,
                               int head_dim, int causal, float scale, float* lse, void* stream);
/* Same contract on the wgmma attention kernel (q, k, v must be one packed [B*L, width] buffer, bs == L*ld):
 * the training forward's default since round 2. */
int g4r_attention_tc_lse_bf16(const void* q, const void* k, const void* v, void* out, long long ld, long long bs,
                              long long ldo, long long bso, int B, int H, int L, int head_dim, int causal, float scale,
                              float* lse, void* stream);
int g4r_attention_bwd_bf16(const void* q, const void* k, const void* v, const void* out, const void* dout,
                           const float* lse, float* delta, void* dq, void* dk, void* dv, long long ld,
                           long long bs, long long ldo, long long bso, long long ldg, long long bsg, int B,
                           int H, int L, int head_dim, int causal, float scale, void* stream);

/* Backward of the splice (spi_llava.py:99-196): rows of d(inputs_embeds) [B*L, D] (16-bit) are copied back to
 * d_image [B*P, D] and d_region [K, D] following the forward's `plan` (either may be NULL to skip it).
 * g4r_embed_grad_rows accumulates the rows that came from the embedding table into a dense fp32 gradient
 * [V, D] (zeroed by the caller): `ids[n_unique]` are the distinct token ids, `order[seg[u] .. seg[u+1])` the
 * row indices (b*L + t) of id u.  One CTA per id, fixed summation order, no atomics. */
int g4r_splice_backward(const int32_t* plan, const void* d_out, void* d_image, void* d_region, int B, int L,
                        int P, int D, void* stream);
int g4r_embed_grad_rows(const void* d_out, const int32_t* order, const int32_t* seg, const int32_t* ids,
                        int n_unique, float* grad, int D, void* stream);

/* Column sums of a bf16 matrix [M,N] into fp32 out[N] (bias gradients of nn.Linear / Conv2d).
 * slabs: fp32 scratch [g4r_colsum_slabs(M)][N]. */
int g4r_colsum_slabs(int M);
int g4r_colsum_bf16(const void* x, long long ld, int M, int N, float* out, float* slabs, void* stream);

/* Backward of a 3x3 / stride 1 / pad 1 NHWC convolution (mmcv ConvModule of MLVLFuseModule, layers.py:133-145, and
 * the pconvs of MlvlRoIExtractor, layers.py:262-268):
 *   grad_x = g4r_conv_nhwc_bf16(grad_z, Wf) with Wf = g4r_conv_weight_flip_t_bf16(W): Wf[ci][ky][kx][co] = W[co][2-ky][2-kx][ci]
 *            (W rows `w_ld` elements apart, so one level of a stacked [Cout, L, 3, 3, Cin] weight works in place);
 *   grad_W = g4r_conv3x3_dw_bf16 on zero-padded copies (g4r_pad_nhwc_bf16: rows [guard | n*(H+2)*(W+2) | guard] x C,
 *            guard_rows >= W+3): one GEMM over all padded pixels, the nine taps being column blocks reached through an
 *            aliasing 4-D TMA tensor map.  x_pad_origin = x_pad + (guard_rows - (W+2) - 1) * Cin elements;
 *            dz_pad = first real row of the padded grad_z (skip its guard).  dW fp32 [Cout, 9*Cin]. */
int g4r_pad_nhwc_bf16(const void* x, void* out, int n, int H, int W, int C, int guard_rows, void* stream);
int g4r_conv_weight_flip_t_bf16(const void* w, long long w_ld, void* wf, int Cin, int Cout, void* stream);
int g4r_conv3x3_dw_bf16(const void* dz_pad, const void* x_pad_origin, float* dW, long long rows, int Wp,
                        int Cin, int Cout, int accumulate, void* stream);

/* GroupNorm(64) + ReLU backward of the fuse ConvModules (mmcv cnn/bricks/conv_module.py:196-208): z = raw conv output
 * (bf16 [B,HW,C], saved), dA = gradient w.r.t. relu(gn(z)) (fp32 when dA_f32, else bf16), scale/shift = g4r_gn_finalize
 * outputs, stats/slots/count/eps = the forward's GroupNorm statistics (mean / rstd are re-derived in the same order).
 * Writes dz (bf16) and dgamma / dbeta (fp32 [C]; accumulate != 0 adds: the four pyramid levels share one GN).
 * workspace: fp32 scratch of g4r_gn_relu_bwd_workspace(B, HW, C, groups) elements.  Fixed-order reductions only. */
long long g4r_gn_relu_bwd_workspace(int B, int HW, int C, int groups);
int g4r_gn_relu_bwd_bf16(const void* z, const void* dA, int dA_f32, const float* scale, const float* shift,
                         const float* stats, int slots, float count, float eps, const void* gamma, void* dz,
                         float* dgamma, float* dbeta, int accumulate, float* workspace, int B, int HW, int C,
                         int groups, void* stream);

/* Adjoint of g4r_fuse_gather_bf16 (MLVLFuseModule._single_shuffle, layers.py:152-180) for pyramid level m:
 * out fp32 [B,H,H,C] = gradient w.r.t. the previous round's activated maps of level m.  d_own = gradient of level
 * m's own conv input; dn0/dn1 = gradients of the conv inputs of the (<= 2) levels that read level m as their
 * `down` source, tp0/tp1 = of those that read it as their `top` source (NULL when absent), each bf16
 * [B,Hx,Hx,C].  Transposed bilinear resize evaluated as a gather (no atomics). */
int g4r_fuse_gather_bwd(const void* d_own, int H, const void* dn0, int Hdn0, const void* dn1, int Hdn1,
                        const void* tp0, int Htp0, const void* tp1, int Htp1, float* out, int B, int C, void* stream);

/* Backward of g4r_pos_embed_mlp (pos_embedd of MlvlRoIExtractor, layers.py:260-267): dout bf16 [K,1024] -> fp32
 * parameter gradients packed as [w0 256x4 | b0 256 | ln2.weight 256 | ln2.bias 256 | w3 1024x256 | b3 1024 |
 * ln5.weight 1024 | ln5.bias 1024] (g4r_pos_embed_mlp_grad_size() floats).  slabs: fp32 scratch [K][that size]. */
int g4r_pos_embed_mlp_grad_size(void);
int g4r_pos_embed_mlp_bwd(const float* boxes, const void* w0, const void* b0, const void* g2, const void* be2,
                          const void* w3, const void* b3, const void* g5, const void* dout, long long ldd,
                          float* grads, float* slabs, int K, float eps, void* stream);

/* ReLU backward from the saved output: out = y > 0 ? dy : 0 (bf16, n elements, n % 8 == 0). */
int g4r_relu_bwd_bf16(const void* dy, const void* y, void* out, long long n, void* stream);

/* ---- input pipeline (SURVEY.md 8(f2)) ------------------------------------------------------------------------
 * Image side of gpt4roi/datasets/coco_det.py:60-71 for a whole batch in one launch: Resize(S,S) [cv2 INTER_LINEAR on
 * uint8, integer-exact] -> RandomShift [zero-filled, per-image (shift_x, shift_y); NULL = none] -> horizontal
 * RandomFlip [per-image flag; NULL = none] -> Normalize(mean, std, to_rgb) [mmcv.imnormalize_ arithmetic] -> CHW.
 * src_packed: decoded uint8 HWC 3-channel images back to back (device); offsets[b] = byte offset of image b;
 * src_hw[b] = (h, w); out [B,3,S,S] fp32 (bit-identical to the reference pipeline) or bf16.  mean3 / std3: HOST float[3].
 * Replaces mmdet/datasets/pipelines/transforms.py:209-243 (Resize), :505-562 (RandomShift), :422-470 (RandomFlip),
 * Normalize / Pad / DefaultFormatBundle, which the reference runs per sample on CPU dataloader workers. */
int g4r_preprocess_images(const void* src_packed, const long long* offsets, const int* src_hw, const int* shift_xy,
                          const int* flip, void* out, int B, int S, const float* mean3, const float* std3, int to_rgb,
                          int out_dtype, void* stream);

/* CLIPImageProcessor image path of the demo and the VCR datasets (gpt4roi/app.py:125-136, gpt4roi/datasets/vcr.py:
 * 181-189): CLIPImageProcessor.preprocess(image, do_center_crop=False) [PIL BICUBIC resize of the short side,
 * integer-exact; float32(u8 * (1/255) in double); (x - mean) / std in float32] -> F.interpolate((S, S), 'bilinear',
 * align_corners=False) [torch's CPU arithmetic] for a ragged batch of uint8 HWC RGB images, in two launches.
 * meta: device int64 [B][13] per-image fields (source address, width, offsets into `tables` and `tmp`, counts; see
 * csrc/clip_preprocess.cu); tables: device int32 tap windows, fixed-point weights and bilinear tables built by
 * gpt4roi_b200.input_pipeline.ClipPreprocessor; tmp: device uint8 intermediate; max_work1 = the largest per-image
 * rows x columns of the first resize pass.  out [B,3,S,S] fp32 (bit-identical to that path), bf16 or fp16.
 * mean3 / std3: HOST float[3]. */
int g4r_clip_preprocess(const long long* meta, const int* tables, void* tmp, void* out, int B, int S,
                        long long max_work1, const float* mean3, const float* std3, int out_dtype, void* stream);

/* Apply a pending GroupNorm affine + ReLU to an NHWC bf16 map: out = relu(z * scale[b,c] + shift[b,c]) with the
 * fp32 [B,C] scale / shift of g4r_gn_finalize.  The activated map is what MLVLFuseModule.forward returns
 * (gpt4roi/models/layers.py:182-195; mmcv ConvModule conv -> GN -> ReLU, conv_module.py:196-208); inside the fused
 * engine the affine stays folded into the consumer's taps, so only the module-level seam calls this. */
int g4r_affine_relu_nhwc_bf16(const void* z, const float* scale, const float* shift, void* out, int B,
                              long long pix_per_img, int C, void* stream);

/* torch.optim.AdamW step (HF Trainer optim="adamw_torch"; param groups llava_trainer.py:59-144): fp32 master
 * weights p and moments m, v; gradient bf16 (g_bf16=1) or fp32, multiplied by grad_scale (1/world, clip factor);
 * p_bf16 (optional) receives the bf16 copy used by the next forward.  step counts from 1. */
int g4r_adamw_step(float* p, const void* g, int g_bf16, float* m, float* v, void* p_bf16, long long n,
                   float lr, float beta1, float beta2, float eps, float weight_decay, int step, float grad_scale,
                   void* stream);
/* Same, with the gradient scale additionally multiplied by the device float *scale_dev (NULL = 1): the clip
 * coefficient of g4r_grad_clip_coef, so that clipping costs no host synchronisation. */
int g4r_adamw_step_ex(float* p, const void* g, int g_bf16, float* m, float* v, void* p_bf16, long long n,
                      float lr, float beta1, float beta2, float eps, float weight_decay, int step, float grad_scale,
                      const float* scale_dev, void* stream);

/* Global gradient-norm clip (HF Trainer max_grad_norm=1.0 -> torch.nn.utils.clip_grad_norm_, called between
 * backward and optimizer.step() by transformers Trainer.training_step; reference gpt4roi/train/train.py:698-712).
 * g4r_sumsq writes g4r_sumsq_slabs() per-CTA partial sums of squares of one gradient tensor (bf16 or fp32) to
 * slab; g4r_grad_clip_coef adds n_slabs partials in a fixed order and writes out2[0] = sqrt(sum) * pre_scale
 * (pre_scale = 1/world for summed, not averaged, DDP gradients) and out2[1] = min(1, max_norm / (out2[0] + 1e-6)). */
int g4r_sumsq_slabs(void);
int g4r_sumsq(const void* g, int g_bf16, long long n, float* slab, void* stream);
int g4r_grad_clip_coef(const float* slabs, long long n_slabs, float pre_scale, float max_norm, float* out2,
                       void* stream);

/* ---- fp16 twins of the inference entry points ---------------------------------------------
 * The demo serves the model in fp16 (gpt4roi/app.py:74-98,271: `model.half()`, `images.half()`, `bboxes.half()`).
 * Every entry point below has the signature, argument meaning and error behaviour of its `_bf16` namesake above,
 * with "bf16" read as "fp16" for every 16-bit tensor (activations, weights, norm / bias vectors, RoPE tables, KV
 * cache); fp32 arguments (statistics, scale / shift, split-K slabs, fp32 residual streams) are unchanged, and the
 * arithmetic is the same (fp32 accumulation, the same rounding points, wgmma with .f16 instead of .bf16
 * operands).  Built from the same sources with -DG4R_ACT_HALF (gpt4roi_b200/csrc/act_type.cuh).  RoIAlign and the
 * splice take a dtype argument / are 2-byte copies and need no twin; the training step is bf16 only
 * (train_stage*.sh --bf16 True). */
int g4r_gemm_f16(const void* A, long long lda, const void* B, long long ldb,
                  void* D, long long ldd, int M, int N, int K,
                  const void* bias, int bias_f32,
                  const void* residual, long long ldr,
                  int act, int out_f32, int k_splits, void* stream);
int g4r_gemm_f16_ex(const void* A, long long lda, const void* B, long long ldb,
                     void* D, long long ldd, int M, int N, int K,
                     const void* bias, int bias_f32,
                     const void* residual, long long ldr, int residual_f32, int bias_round_bf16,
                     int act, int out_f32, int k_splits, void* stream);
int g4r_gemm_qkv_rope_f16(const void* A, long long lda, const void* B, long long ldb,
                           void* D, long long ldd, int M, int N, int K,
                           const void* rope_cos, const void* rope_sin, int rope_cols, int L, int pos0,
                           const int* pos0_dev /* device int32 overriding pos0 (CUDA-graph decode) or NULL */,
                           void* stream);
int g4r_conv_nhwc_f16(const void* X, const void* Wt, void* Y,
                       int n_img, int H, int W, int Cin, int Cout, int ksize, int levels,
                       const void* bias, int bias_f32, int act,
                       float* gn_stats, int gn_groups, void* stream);
int g4r_attention_tc_f16(const void* q, const void* k, const void* v, void* out,
                          long long ld, long long bs, long long ldo, long long bso,
                          int B, int H, int L, int head_dim, int causal, float scale,
                          const int* seqlens, void* stream);
int g4r_attention_f16(const void* q, const void* k, const void* v, void* out,
                       long long ld, long long bs, long long ldo, long long bso,
                       int B, int H, int L, int head_dim, int causal, float scale,
                       const int* seqlens /* device int32 [B] or NULL: keys >= seqlens[b] are masked */,
                       void* stream);
int g4r_layernorm_f16(const void* x, long long ldx, const void* w, const void* b,
                       void* out, long long ldo, int M, int D, float eps, void* stream);
int g4r_rmsnorm_f16(const void* x, long long ldx, const void* w,
                     void* out, long long ldo, int M, int D, float eps, void* stream);
int g4r_rope_inplace_f16(void* qkv, long long ld, const void* cos_t, const void* sin_t,
                          int rows, int L, int n_heads_qk, int head_dim, void* stream);
int g4r_patchify_f16(const void* img, void* out, int B, int S, int ps, int Kpad, void* stream);
int g4r_vit_embed_f16(const void* patch, const void* cls, const void* pos, void* out,
                       int B, int P, int D, void* stream);
int g4r_upsample_tokens_coords_f16(const void* tok, long long ldt, long long bst, void* out,
                                    int B, int G, int Ho, int C, int Cpad, void* stream);
int g4r_upsample_tokens_coords_f32_f16(const void* tok, long long ldt, long long bst, void* out,
                                   int B, int G, int Ho, int C, int Cpad, void* stream);
int g4r_layernorm_ex_f16(const void* x, long long ldx, int x_f32, const void* w, const void* b,
                     void* out, long long ldo, int out_f32, int M, int D, float eps, void* stream);
int g4r_rmsnorm_ex_f16(const void* x, long long ldx, int x_f32, const void* w, void* out, long long ldo, int M, int D,
                   float eps, void* stream);
int g4r_cast_f32_f16(const void* x, long long ld, long long bst, void* out,
                      int B, int rows_per_batch, int D, void* stream);
int g4r_fuse_gather_f16(const void* own, const float* own_sc, const float* own_sh, int H,
                         const void* top, const float* top_sc, const float* top_sh, int Ht,
                         const void* down, const float* down_sc, const float* down_sh, int Hd,
                         void* out, int B, int C, void* stream);
int g4r_gn_finalize_f16(const float* stats, const void* gamma, const void* beta,
                    float* scale, float* shift, int B, int C, int groups, int slots,
                    float count, float eps, void* stream);
int g4r_pos_embed_mlp_f16(const float* boxes, const void* w0, const void* b0, const void* g2,
                      const void* be2, const void* w3, const void* b3, const void* g5,
                      const void* be5, float* out, int K, float eps, void* stream);
int g4r_affine_relu_nhwc_f16(const void* z, const float* scale, const float* shift, void* out, int B,
                              long long pix_per_img, int C, void* stream);
int g4r_add_bias_pos_cast_f16(const float* acc, int splits, const void* bias, const float* pos, void* out,
                          int K, int D, void* stream);
int g4r_decode_gemm_f16(const void* x, long long ldx, const void* W, long long ldw, void* out, long long ldo, int M,
                         int N, int K, int act, const void* residual, long long ldr,
                         const void* rope_cos, const void* rope_sin, int rope_cols, int pos0, const int* pos_dev,
                         void* kcache, void* vcache, int cache_lmax, int cache_hd, void* stream);
int g4r_kv_append_f16(const void* qkv, long long ld, void* kcache, void* vcache,
                       int B, int Ln, int pos0, const int* pos_dev /* overrides pos0 when non-NULL */,
                       int Lmax, int HD, void* stream);
int g4r_decode_attention_f16(const void* q, long long ldq, const void* kcache, const void* vcache,
                              void* out, long long ldo, int B, int H, int head_dim, int kv_len,
                              const int* pos_dev /* kv_len = *pos_dev + 1 when non-NULL; kv_len then sizes smem */,
                              int Lmax, float scale, void* stream);
int g4r_gemm_qkv_rope_rows_f16(const void* A, long long lda, const void* B, long long ldb,
                               void* D, long long ldd, int M, int N, int K,
                               const void* rope_cos, const void* rope_sin, int rope_cols, int L,
                               const int* pos_rows, void* stream);
int g4r_decode_gemm_rows_f16(const void* x, long long ldx, const void* W, long long ldw, void* out, long long ldo,
                             int M, int N, int K, int act, const void* residual,
                             long long ldr, const void* rope_cos, const void* rope_sin, int rope_cols,
                             const int* pos_rows, void* kcache, void* vcache, int cache_lmax, int cache_hd,
                             void* stream);
int g4r_kv_append_rows_f16(const void* qkv, long long ld, void* kcache, void* vcache,
                           int B, int Ln, const int* pos_rows, int Lmax, int HD, void* stream);
int g4r_decode_attention_rows_f16(const void* q, long long ldq, const void* kcache, const void* vcache,
                                  void* out, long long ldo, int B, int H, int head_dim, int kv_bound,
                                  const int* pos_rows, int Lmax, float scale, void* stream);
int g4r_attention_cached_f16(const void* q, long long ldq, const void* kcache, const void* vcache, int lmax,
                             void* out, long long ldo, int B, int H, int Lc, int head_dim, float scale,
                             const int* start, const int* qlen, void* stream);
int g4r_kv_append_rows_at_f16(const void* qkv, long long ld, void* kcache, void* vcache, int B, int Ln,
                              const int* pos_rows, const int* cache_rows, const int* qlen, int Lmax, int HD,
                              void* stream);
int g4r_attention_cached_rows_f16(const void* q, long long ldq, const void* kcache, const void* vcache, int rows,
                                  int lmax, void* out, long long ldo, int B, int H, int Lc, int head_dim, float scale,
                                  const int* start, const int* qlen, const int* cache_rows, void* stream);
int g4r_sample_tokens_f16(const void* logits, long long ld, int B, int V, float temperature, int top_k, float top_p,
                          int greedy, unsigned long long seed, const long long* rng_step, int eos_id, int pad_id,
                          int* finished, long long* out_ids, void* stream);
int g4r_sample_tokens_proc_f16(const void* logits, long long ld, int B, int V, float temperature, int top_k,
                               float top_p, int greedy, unsigned long long seed, const long long* rng_step, int eos_id,
                               int pad_id, int* finished, long long* out_ids, long long* history, long long ld_h, int L,
                               float repetition_penalty, int no_repeat_ngram_size, int min_length, int min_new_tokens,
                               const int* eos_ids, int n_eos, int append, void* stream);
int g4r_decode_attention_beam_f16(const void* q, long long ldq, const void* kcache, const void* vcache,
                                  void* out, long long ldo, int R, int H, int head_dim, int kv_bound,
                                  const int* pos_rows, const int* anc, int Lmax, float scale, void* stream);
int g4r_decode_attention_group_f16(const void* q, long long ldq, const void* kcache, const void* vcache,
                                   void* out, long long ldo, int B, int N, int H, int head_dim, int prompt_bound,
                                   int gen_bound, const int* prompt_lens, const int* pos_rows, int Lmax, float scale,
                                   void* stream);
int g4r_beam_step_f16(const void* logits, long long ld, int row_div, int B, int N, int V, int K, const int* eos_ids,
                      int n_eos, int prompt_len, int max_length, double length_penalty, int early_stopping, int G,
                      int Lmax, const int* lens, int* state, float* run_score, float* cand_score, int* cand_tok,
                      long long* run_seq, long long* fin_seq, float* fin_score, int* fin_state, long long* ids,
                      int* pos_rows, int* anc, void* stream);
int g4r_sample_tokens_out_f16(const void* logits, long long ld, int B, int V, float temperature, int top_k,
                              float top_p, int greedy, unsigned long long seed, const long long* rng_step, int eos_id,
                              int pad_id, int* finished, long long* out_ids, long long* history, long long ld_h, int L,
                              float repetition_penalty, int no_repeat_ngram_size, int min_length, int min_new_tokens,
                              const int* eos_ids, int n_eos, int append, float* scores, float* raw_logits,
                              long long n_slots, void* stream);
int g4r_beam_step_out_f16(const void* logits, long long ld, int row_div, int B, int N, int V, int K,
                          const int* eos_ids, int n_eos, int prompt_len, int max_length, double length_penalty,
                          int early_stopping, int G, int Lmax, const int* lens, int* state, float* run_score,
                          float* cand_score, int* cand_tok, long long* run_seq, long long* fin_seq, float* fin_score,
                          int* fin_state, long long* ids, int* pos_rows, int* anc, float* scores, float* raw_logits,
                          int n_slots, int* run_bidx, int* fin_bidx, void* stream);
int g4r_sample_tokens_rows_f16(const void* logits, long long ld, int S, int V, const int* greedy,
                               const float* temperature, const int* top_k, const float* top_p,
                               const unsigned long long* seed, long long* step, const int* eos_id, const int* active,
                               int* finished, long long* out_ids, int* lens, void* stream);
int g4r_sample_tokens_rows_proc_f16(const void* logits, long long ld, int S, int V, const int* greedy,
                                    const float* temperature, const int* top_k, const float* top_p,
                                    const unsigned long long* seed, long long* step, const int* eos_id,
                                    const int* active, int* finished, long long* out_ids, int* lens,
                                    long long* history, long long ld_h, const int* prompt_len,
                                    const float* repetition_penalty, const int* no_repeat_ngram_size,
                                    const int* min_length, const int* min_new_tokens, const int* eos_ids,
                                    const int* n_eos, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GPT4ROI_B200_H_ */
