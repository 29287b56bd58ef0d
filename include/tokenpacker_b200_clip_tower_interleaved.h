/* tokenpacker_b200 — the frozen CLIP vision tower's four hidden states in one interleaved buffer (libtokenpacker_b200.so).
 *
 * Companion of tokenpacker_b200_clip_tower.h and tokenpacker_b200_clip_tower_f16.h, whose weights struct, packed weights, workspace
 * size, crops conventions and status codes it uses; those headers and ABI version 2 are unchanged.
 *
 * LLaVA's CLIPVisionTower.feature_select (clip_encoder.py:28-44) concatenates hidden states 12, 16, 22 and 23 along the channels into
 * a new [N, 577, 4096] tensor.  These entry points store them there in the first place: out[n][t][1024 j + c] is hidden_states[L_j]
 * [n][t][c] for L = (12, 16, 22, 23).  So out[:, 1:] is the reference's image_features_multi and out[:, 1:, 3072:] its image_features
 * (select_layer -2), with no copy.  The schedule is the one of tp_clip_tower_forward / _f16, the launches are the same, and each
 * 1024-column slice has the bits of the matching dense output: the layers that end in one of the four hidden states store their fc2
 * output at row stride 4096, and the layers that start from one read it there.
 *
 * Element offsets into out pass 2^31 from n_crops = 909 on; every offset is 64-bit.
 */
#ifndef TOKENPACKER_B200_CLIP_TOWER_INTERLEAVED_H_
#define TOKENPACKER_B200_CLIP_TOWER_INTERLEAVED_H_

#include "tokenpacker_b200_clip_tower_f16.h"

#ifdef __cplusplus
extern "C" {
#endif

/* hidden_states 12, 16, 22 and 23 of n_crops crops, bf16, interleaved.
 *   packed, w, crops, n_crops, crop_stride, workspace, workspace_bytes, stream   as for tp_clip_tower_forward (workspace
 *                    >= tp_clip_tower_workspace_bytes(n_crops))
 *   out              bf16 [n_crops, 577, 4096], contiguous (CLS row included), 16-byte aligned; hidden_states[12], [16], [22] and
 *                    [23] at columns 0, 1024, 2048 and 3072
 * Column block j of out has the bits of out_layers[j] of tp_clip_tower_forward on the same crops.
 * TP_ERR_INVALID_ARGUMENT (NULL pointers, n_crops <= 0, a misaligned out, ...) / TP_ERR_WORKSPACE_TOO_SMALL before any CUDA call;
 * TP_ERR_UNSUPPORTED_DEVICE off sm_90. */
TP_API int tp_clip_tower_forward_interleaved(const void* packed, const tp_clip_tower_weights* w, const void* crops, int64_t n_crops,
                                             int64_t crop_stride, void* out, void* workspace, size_t workspace_bytes, void* stream);

/* The same in fp16: packed from tp_clip_tower_pack_weights_f16, crops of crops_dtype (TP_CLIP_CROPS_BF16 or TP_CLIP_CROPS_F16; anything
 * else is TP_ERR_INVALID_ARGUMENT), out f16 [n_crops, 577, 4096].  Column block j has the bits of out_layers[j] of
 * tp_clip_tower_forward_f16 on the same crops. */
TP_API int tp_clip_tower_forward_interleaved_f16(const void* packed, const tp_clip_tower_weights* w, const void* crops, int crops_dtype,
                                                 int64_t n_crops, int64_t crop_stride, void* out, void* workspace, size_t workspace_bytes,
                                                 void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TOKENPACKER_B200_CLIP_TOWER_INTERLEAVED_H_ */
