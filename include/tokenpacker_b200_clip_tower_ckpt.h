/* tokenpacker_b200 — gradient checkpointing for the trainable top of the CLIP-ViT-L/14-336 vision tower (libtokenpacker_b200.so).
 *
 * Companion of tokenpacker_b200_clip_tower_train.h, whose structs, conventions and status codes it uses; that header is unchanged.
 * tp_clip_tower_forward_train keeps a full saved set per trainable layer (20.1 MB per crop and layer).  The pair below keeps, per
 * trainable layer, only its "checkpoint": the layer's derived weights (the q/k/v concatenation with q scaled by 1/8 and the fp32
 * biases, 6.3 MB, packed from ``w`` by every forward) and its input x, bf16 [577 n_crops, 1024] (1.18 MB per crop).
 *
 * The forward runs every layer on the inference schedule (fc1 -> fc2 chained, intermediates in the inference workspace).  The
 * backward walks the trainable layers from the top: for each, it recomputes the layer's saved set from its checkpoint into one scratch
 * set of the workspace (layer_norm1, q|k|v, attention with its softmax statistics, out_proj, layer_norm2, fc1 and quick_gelu; fc2 is
 * not rerun, nothing of the backward reads the layer's output), then runs the layer's backward on it, as tp_clip_tower_backward does.
 * The recompute costs about 70 % of a layer's forward FLOPs.
 *
 * Checkpointing changes memory and time, never bits: the four outputs are those of tp_clip_tower_forward, and every gradient equals
 * that of tp_clip_tower_forward_train + tp_clip_tower_backward.  The recompute launches the same kernels and GEMM items on the same
 * operands as the training forward, and no kernel uses atomics.
 */
#ifndef TOKENPACKER_B200_CLIP_TOWER_CKPT_H_
#define TOKENPACKER_B200_CLIP_TOWER_CKPT_H_

#include "tokenpacker_b200_clip_tower_train.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Bytes of the checkpoints of a forward over n_crops crops with the last trainable_layers (1 .. 23) layers trainable: per layer its
 * derived weights and its input; 0 for arguments out of range. */
TP_API size_t tp_clip_tower_ckpt_saved_bytes(int64_t n_crops, int trainable_layers);

/* Workspace bytes of tp_clip_tower_backward_ckpt: tp_clip_tower_backward's, one layer's saved set and fc1's fp32 pre-activation
 * [577 n_crops, 4096]; the same for every trainable_layers in range, 0 out of range. */
TP_API size_t tp_clip_tower_ckpt_backward_workspace_bytes(int64_t n_crops, int trainable_layers);

/* tp_clip_tower_forward (same packed, w, crops, out_layers and workspace: workspace_bytes >= tp_clip_tower_workspace_bytes) that also
 * fills ``saved`` (256-byte aligned, >= tp_clip_tower_ckpt_saved_bytes) with the checkpoints of layers 23 - trainable_layers .. 22
 * for tp_clip_tower_backward_ckpt.  trainable_layers in 1 .. 23.  TP_ERR_INVALID_ARGUMENT / TP_ERR_WORKSPACE_TOO_SMALL before any CUDA
 * call. */
TP_API int tp_clip_tower_forward_ckpt(const void* packed, const tp_clip_tower_weights* w, const void* crops, int64_t n_crops,
                                      int64_t crop_stride, int trainable_layers, void* const* out_layers, void* saved, size_t saved_bytes,
                                      void* workspace, size_t workspace_bytes, void* stream);

/* tp_clip_tower_backward (same arguments and results) from the checkpoints tp_clip_tower_forward_ckpt left in ``saved``; workspace
 * >= tp_clip_tower_ckpt_backward_workspace_bytes, 256-byte aligned.  Deterministic: no atomics, every reduction in a fixed order.
 * TP_ERR_INVALID_ARGUMENT / TP_ERR_WORKSPACE_TOO_SMALL before any CUDA call. */
TP_API int tp_clip_tower_backward_ckpt(const tp_clip_tower_weights* w, const void* saved, int64_t n_crops, int trainable_layers,
                                       const void* const* d_out_layers, const tp_clip_tower_layer_grads* grads, void* workspace,
                                       size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TOKENPACKER_B200_CLIP_TOWER_CKPT_H_ */
