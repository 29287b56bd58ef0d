/* tokenpacker_b200 — training the top of the CLIP-ViT-L/14-336 vision tower (libtokenpacker_b200.so): a forward that keeps what the
 * backward needs of the last K encoder layers, and the backward through them.
 *
 * Companion of tokenpacker_b200_clip_tower.h, whose structs, conventions and status codes it uses; that header is unchanged.
 * Layers 0 .. 22 - K run exactly as in tp_clip_tower_forward (frozen: nothing of them is kept, they get no gradient); layers
 * 23 - K .. 22 are the trainable ones.  bf16 only.  The four outputs have the bits tp_clip_tower_forward gives.
 *
 * Kept per trainable layer and crop (the "saved set"): the layer's input x, LN1(x), q|k|v (q scaled by 1/8), the log2 softmax
 * denominators (fp32 per head and query), the attention output, the mid-layer residual x' (fp32), LN2(x'), fc1's pre-activation z and
 * quick_gelu(z): 34 KiB + 64 B per token, 20.1 MB per crop and layer, plus 6.3 MB per layer (not per crop) of derived weights.
 *
 * The derived weights of the trainable layers (q/k/v concatenation with q scaled by 1/8, fp32 biases) are rebuilt from ``w`` by every
 * tp_clip_tower_forward_train call, so parameters updated in place between steps are always read as they are; the frozen layers read
 * ``packed``.
 */
#ifndef TOKENPACKER_B200_CLIP_TOWER_TRAIN_H_
#define TOKENPACKER_B200_CLIP_TOWER_TRAIN_H_

#include "tokenpacker_b200_clip_tower.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Destinations of one trainable layer's parameter gradients: bf16 device buffers of the parameters' shapes, 16-byte aligned, every
 * element written (not accumulated).  A NULL pointer skips that gradient (and the weight-gradient GEMM or reduction behind it). */
typedef struct tp_clip_tower_layer_grads {
  void* ln1_w; void* ln1_b;
  void* q_w; void* q_b;                                       /* of the UNSCALED q_proj parameters */
  void* k_w; void* k_b;
  void* v_w; void* v_b;
  void* o_w; void* o_b;
  void* ln2_w; void* ln2_b;
  void* fc1_w; void* fc1_b;
  void* fc2_w; void* fc2_b;
} tp_clip_tower_layer_grads;

/* Bytes of the saved sets of a forward over n_crops crops with the last trainable_layers (1 .. 23) layers trainable; 0 for arguments
 * out of range. */
TP_API size_t tp_clip_tower_train_saved_bytes(int64_t n_crops, int trainable_layers);

/* Workspace bytes of tp_clip_tower_forward_train: tp_clip_tower_forward's plus fc1's fp32 pre-activation [577 n_crops, 4096]. */
TP_API size_t tp_clip_tower_train_workspace_bytes(int64_t n_crops, int trainable_layers);

/* Workspace bytes of tp_clip_tower_backward. */
TP_API size_t tp_clip_tower_backward_workspace_bytes(int64_t n_crops, int trainable_layers);

/* tp_clip_tower_forward (same packed, w, crops, out_layers: see there) that also fills ``saved`` (256-byte aligned,
 * >= tp_clip_tower_train_saved_bytes) for tp_clip_tower_backward.  trainable_layers in 1 .. 23.
 * TP_ERR_INVALID_ARGUMENT / TP_ERR_WORKSPACE_TOO_SMALL before any CUDA call. */
TP_API int tp_clip_tower_forward_train(const void* packed, const tp_clip_tower_weights* w, const void* crops, int64_t n_crops,
                                       int64_t crop_stride, int trainable_layers, void* const* out_layers, void* saved, size_t saved_bytes,
                                       void* workspace, size_t workspace_bytes, void* stream);

/* Parameter gradients of layers 23 - trainable_layers .. 22.
 *   w              the weights of the forward (the trainable layers' are read in place: out_proj, fc1, fc2 and the LayerNorm scales)
 *   saved          as tp_clip_tower_forward_train left it (same n_crops and trainable_layers); read only
 *   d_out_layers   gradients of hidden_states 12, 16, 22 and 23: bf16 [n_crops, 577, 1024], contiguous, 16-byte aligned; any may be
 *                  NULL (no gradient).  One that belongs to a hidden state at or below the first trainable layer's input is ignored.
 *   grads          trainable_layers entries, grads[t] for layer 23 - trainable_layers + t
 *   workspace      >= tp_clip_tower_backward_workspace_bytes, 256-byte aligned
 * Deterministic: no atomics, every reduction in a fixed order.  No gradient is produced for the crops, the embeddings, pre_layrnorm or
 * the frozen layers.  TP_ERR_INVALID_ARGUMENT / TP_ERR_WORKSPACE_TOO_SMALL before any CUDA call. */
TP_API int tp_clip_tower_backward(const tp_clip_tower_weights* w, const void* saved, int64_t n_crops, int trainable_layers,
                                  const void* const* d_out_layers, const tp_clip_tower_layer_grads* grads, void* workspace,
                                  size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TOKENPACKER_B200_CLIP_TOWER_TRAIN_H_ */
