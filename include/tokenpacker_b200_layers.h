/* tokenpacker_b200 — training straight from the CLIP tower's four hidden states (libtokenpacker_b200.so).
 *
 * Companion of tokenpacker_b200.h, whose conventions, status codes, tp_weights and training entry points it uses.  Kept in a
 * header of its own so that tokenpacker_b200.h, ABI version 2, stays exactly as its consumers compiled it; this header only adds.
 *
 * The reference builds the projector's input with CLIPVisionTower.feature_select (clip_encoder.py:28-44): feat = hidden state 23
 * and feat_multi = torch.cat of hidden states 12 / 16 / 22 / 23, both without the CLS row.  The entry points below take the four
 * hidden states instead, in place:
 *   layers        4 device pointers, layers[i] = token row 0 of crop 0 of hidden state 12 / 16 / 22 / 23 (bf16, 16-byte aligned,
 *                 rows of 1024 channels).  For the tower's [N,577,1024] outputs that is the row after the CLS row.
 *   crop_stride   elements between the token rows 0 of consecutive crops, the same for all four layers: >= 576 * 1024 and a
 *                 multiple of 8 (577 * 1024 for the tower's outputs, 576 * 1024 for contiguous [N,576,1024] tensors)
 * No concatenation and no contiguous copy of feat_multi is ever made.
 */
#ifndef TOKENPACKER_B200_LAYERS_H_
#define TOKENPACKER_B200_LAYERS_H_

#include "tokenpacker_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* tp_forward_train with feat = layers[3] and feat_multi = the concatenation of the four layers.  Same packed weights
 * (tp_pack_weights_train), same ``saved`` size (tp_train_saved_bytes); out and the saved contents are bit-identical to those of
 * tp_forward_train on the concatenation.  TP_ERR_INVALID_ARGUMENT as tp_forward_train, and for a NULL or misaligned layer or a bad
 * crop_stride; TP_ERR_BAD_SCALE_FACTOR as tp_forward_train.  All checks run before any CUDA call. */
TP_API int tp_forward_train_layers(const tp_weights* w, const void* packed, const void* const* layers, int64_t n_crops, int64_t crop_stride,
                                   int scale_factor, int hidden, void* out, void* saved, size_t saved_bytes, void* stream);

/* tp_backward for a tp_forward_train_layers call, reading the four layers in place (the k/v_proj.0 weight gradients), plus the
 * gradients w.r.t. the layers when asked for.
 *   w, n_crops, scale_factor, hidden, grad_out, saved, grads, workspace
 *                 as for tp_backward; the parameter gradients written to ``grads`` are exactly (bit for bit) those of tp_backward on
 *                 the concatenation, and the workspace is the same size (tp_backward_workspace_bytes)
 *   layers, crop_stride
 *                 the tp_forward_train_layers call's
 *   d_layers      NULL, or 4 pointers, each NULL (no gradient for that layer) or token row 0 of crop 0 of a bf16 [n_crops, *, 1024]
 *                 destination, 16-byte aligned.  Only the 576 token rows of each crop are written; CLS rows and anything else are left
 *                 alone.  d_layers[i] = dz_kv . [W_k0; W_v0][:, 1024 i : 1024 (i + 1)] (the feat_multi gradient's quarter i), and
 *                 d_layers[3] has the feat gradient (the point-query stencil run backwards over dq = dy_q . W_q) added in bf16:
 *                 exactly the sum autograd forms for hidden state 23, which is both feat and part of feat_multi
 *   d_crop_stride elements between the crops of every d_layers destination: a multiple of 1024 and >= 576 * 1024
 *   packed        the tp_pack_weights_train buffer of the forward: [W_k0; W_v0] is read from it.  Required when any d_layers[i] is
 *                 given; may be NULL otherwise
 * Each layer gradient adds one GEMM to the last launch tp_backward already makes; d_layers[3] also adds dq to an earlier one and one
 * stencil kernel at the end.
 * TP_ERR_INVALID_ARGUMENT as tp_backward, and for a NULL or misaligned layer, a bad crop_stride or d_crop_stride, a misaligned
 * d_layers[i] or d_layers without packed; TP_ERR_BAD_SCALE_FACTOR as tp_backward.  All checks run before any CUDA call. */
TP_API int tp_backward_layers(const tp_weights* w, const void* packed, const void* const* layers, int64_t crop_stride, int64_t n_crops,
                              int scale_factor, int hidden, const void* grad_out, const void* saved, const tp_weights* grads,
                              void* const* d_layers, int64_t d_crop_stride, void* workspace, size_t workspace_bytes, void* stream);

/* tp_forward_packed from the four layers: the HD packed layout (out_crop_rows rows per crop, the first (24 / s)^2 of them written; 0
 * or (24 / s)^2: dense [N, M, hidden]) stays on the single fused launch.  Same workspace (tp_workspace_bytes) and packed weights
 * (tp_pack_weights) as tp_forward_layers, and the same bits as tp_forward_packed on the concatenation.  TP_ERR_INVALID_ARGUMENT as
 * tp_forward_packed, and for a NULL or misaligned layer or a bad crop_stride; TP_ERR_BAD_SCALE_FACTOR as tp_forward_packed.  All
 * checks run before any CUDA call. */
TP_API int tp_forward_layers_packed(const void* packed, const void* const* layers, int64_t n_crops, int64_t crop_stride, int scale_factor,
                                    int hidden, void* out, int64_t out_crop_rows, void* workspace, size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TOKENPACKER_B200_LAYERS_H_ */
