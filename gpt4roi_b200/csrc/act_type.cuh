// act_type.cuh -- the 16-bit activation / weight type of the inference kernels.
//
// The demo serves the model in fp16 (gpt4roi/app.py:74-98,271: `model.half()`, `images.half()`, `bboxes.half()`), the
// training scripts and everything else in bf16 (train_stage*.sh --bf16 True).  The six inference sources
// (gemm_wgmma.cu, attention_wgmma.cu, attention.cu, elementwise.cu, gemm_skinny.cu, decode.cu) are therefore built
// twice: as written (bf16), and with -DG4R_ACT_HALF, where this header -- included AFTER common.cuh / ptx.cuh --
// retargets the type, its conversion intrinsics, the tensor-core operand format and the exported names to fp16:
//   * every kernel keeps fp32 accumulation and the same rounding points ("round to the storage type" is now fp16);
//   * wgmma and mma.sync switch their .bf16 operand qualifier to .f16 (G4R_ACT_PTX); TMA tensor maps carry the
//     matching data type;
//   * the C entry points get an _f16 name (`g4r_gemm_bf16` -> `g4r_gemm_f16`, `g4r_rmsnorm_ex` -> `g4r_rmsnorm_ex_f16`)
//     with identical signatures (include/gpt4roi_b200.h), and the C++ symbols move to namespace g4r_h;
//   * entry points only the training step uses are not built for fp16 (G4R_BF16_ONLY).
#pragma once

#ifdef G4R_ACT_HALF
#define G4R_NS g4r_h
#define G4R_ACT_PTX "f16"
#define G4R_BF16_ONLY 0

#define __nv_bfloat16 __half
#define __nv_bfloat162 __half2
#define __bfloat162float __half2float
#define __float2bfloat16_rn __float2half_rn
#define __floats2bfloat162_rn __floats2half2_rn
#define __bfloat1622float2 __half22float2
#define CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 CU_TENSOR_MAP_DATA_TYPE_FLOAT16

#define g4r_gemm_bf16 g4r_gemm_f16
#define g4r_gemm_bf16_ex g4r_gemm_f16_ex
#define g4r_gemm_qkv_rope_bf16 g4r_gemm_qkv_rope_f16
#define g4r_conv_gn_slots g4r_conv_gn_slots_f16
#define g4r_conv_nhwc_bf16 g4r_conv_nhwc_f16
#define g4r_attention_tc_bf16 g4r_attention_tc_f16
#define g4r_attention_bf16 g4r_attention_f16
#define g4r_layernorm_bf16 g4r_layernorm_f16
#define g4r_rmsnorm_bf16 g4r_rmsnorm_f16
#define g4r_rope_inplace_bf16 g4r_rope_inplace_f16
#define g4r_patchify_bf16 g4r_patchify_f16
#define g4r_vit_embed_bf16 g4r_vit_embed_f16
#define g4r_upsample_tokens_coords_bf16 g4r_upsample_tokens_coords_f16
#define g4r_upsample_tokens_coords_f32 g4r_upsample_tokens_coords_f32_f16
#define g4r_layernorm_ex g4r_layernorm_ex_f16
#define g4r_rmsnorm_ex g4r_rmsnorm_ex_f16
#define g4r_cast_f32_bf16 g4r_cast_f32_f16
#define g4r_fuse_gather_bf16 g4r_fuse_gather_f16
#define g4r_gn_finalize g4r_gn_finalize_f16
#define g4r_pos_embed_mlp g4r_pos_embed_mlp_f16
#define g4r_affine_relu_nhwc_bf16 g4r_affine_relu_nhwc_f16
#define g4r_add_bias_pos_cast g4r_add_bias_pos_cast_f16
#define g4r_decode_gemm_bf16 g4r_decode_gemm_f16
#define g4r_kv_append_bf16 g4r_kv_append_f16
#define g4r_decode_attention_bf16 g4r_decode_attention_f16

#else
#define G4R_NS g4r
#define G4R_ACT_PTX "bf16"
#define G4R_BF16_ONLY 1
#endif

namespace g4r {}
namespace G4R_NS { using namespace g4r; }
