/* tokenpacker_b200 — the frozen CLIP-ViT-L/14-336 vision tower in fp16 (libtokenpacker_b200.so).
 *
 * Companion of tokenpacker_b200_clip_tower.h, whose weights struct, conventions and status codes it uses; that header and ABI version 2
 * are unchanged.  The same network as tp_clip_tower_forward with f16 storage: f16 parameters, crops converted to f16, f16 wgmma with
 * fp32 accumulation, one f16 rounding per stored tensor.  This is the precision the LLaVA evaluation and serving scripts run the tower
 * in (vision_tower.to(dtype=torch.float16)), while the LLM and the projector stay in bf16: the four outputs are fp16 and the caller
 * casts them to bf16 for the projector, as clip_encoder.py does (.to(images.dtype)).
 *
 * tp_clip_tower_packed_bytes() and tp_clip_tower_workspace_bytes() serve both precisions.  A packed buffer is valid only for the forward
 * of the precision it was packed for: tp_clip_tower_pack_weights_f16 output for tp_clip_tower_forward_f16, tp_clip_tower_pack_weights
 * output for tp_clip_tower_forward.  Nothing in the buffer records which; mixing them computes garbage.
 */
#ifndef TOKENPACKER_B200_CLIP_TOWER_F16_H_
#define TOKENPACKER_B200_CLIP_TOWER_F16_H_

#include "tokenpacker_b200_clip_tower.h"

#ifdef __cplusplus
extern "C" {
#endif

#define TP_CLIP_CROPS_BF16 1   /* crops_dtype: bf16 crops, converted to f16 exactly as images.to(torch.float16) rounds them */
#define TP_CLIP_CROPS_F16 2    /* crops_dtype: f16 crops, read as they are */

/* Fill ``packed`` (256-byte aligned, >= tp_clip_tower_packed_bytes()) from ``w``, whose pointers are fp16 device pointers (non-NULL,
 * 16-byte aligned): per layer the UNSCALED q/k/v concatenation [3072,1024] in f16 (the 1/8 query scale is applied by the forward after
 * the q bias, with one rounding, because scaling f16 weights by 1/8 would push those below 2^-11 into the subnormals), the biases in
 * fp32, and the patch weight with its rows padded to 592 elements.
 * TP_ERR_INVALID_ARGUMENT / TP_ERR_WORKSPACE_TOO_SMALL before any CUDA call. */
TP_API int tp_clip_tower_pack_weights_f16(const tp_clip_tower_weights* w, void* packed, size_t packed_bytes, void* stream);

/* hidden_states 12, 16, 22 and 23 of n_crops crops, fp16.
 *   packed           tp_clip_tower_pack_weights_f16 output
 *   w                the fp16 weights it was packed from: everything but q/k/v is read in place
 *   crops            [n_crops, 3, 336, 336] of ``crops_dtype`` (TP_CLIP_CROPS_BF16 or TP_CLIP_CROPS_F16; anything else is
 *                    TP_ERR_INVALID_ARGUMENT), crop n at crops + n * crop_stride (elements, >= 3 * 336 * 336), each crop contiguous
 *   out_layers       4 distinct f16 destinations [n_crops, 577, 1024], contiguous (CLS row included), 16-byte aligned; also the residual
 *                    stream the following layers read
 *   workspace        >= tp_clip_tower_workspace_bytes(n_crops), 256-byte aligned
 * Crop n of a batch gets the bits of a call on that crop alone, and bf16 crops the bits of their f16 conversion.
 * TP_ERR_INVALID_ARGUMENT / TP_ERR_WORKSPACE_TOO_SMALL before any CUDA call; TP_ERR_UNSUPPORTED_DEVICE off sm_90. */
TP_API int tp_clip_tower_forward_f16(const void* packed, const tp_clip_tower_weights* w, const void* crops, int crops_dtype, int64_t n_crops,
                                     int64_t crop_stride, void* const* out_layers, void* workspace, size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TOKENPACKER_B200_CLIP_TOWER_F16_H_ */
