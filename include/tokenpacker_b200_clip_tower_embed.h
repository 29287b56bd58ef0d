/* tokenpacker_b200 — training the whole CLIP-ViT-L/14-336 vision tower (libtokenpacker_b200.so): all 23 encoder layers the tower runs
 * and, below them, pre_layrnorm, the class and position embeddings and the patch embedding.
 *
 * Companion of tokenpacker_b200_clip_tower_ckpt.h (and through it tokenpacker_b200_clip_tower_train.h), whose structs, conventions
 * and status codes it uses; those headers are unchanged.  The number of trainable layers is fixed at 23.  The pair below runs the
 * layers exactly as tp_clip_tower_forward_train / tp_clip_tower_backward do (checkpoint == 0) or as tp_clip_tower_forward_ckpt /
 * tp_clip_tower_backward_ckpt do (checkpoint != 0), with ``saved`` and the workspaces sized by those pairs' queries at 23 layers,
 * and keeps in addition the embedding stage's own saved set (tp_clip_tower_embed_saved_bytes):
 *   the crops' patch rows (im2col), bf16 [576 n_crops, 592] (columns 588.. unused), 0.68 MB per crop, and
 *   the patch GEMM's output rows before pre_layrnorm, bf16 [577 n_crops, 1024] (row 0 of each crop unused), 1.18 MB per crop.
 * The patch weight is read from ``w`` (repacked into 592-element rows by every forward); the class and position embeddings and
 * pre_layrnorm's scale are read from ``w`` too, so parameters updated in place between steps are always read as they are.
 *
 * The four outputs have the bits of tp_clip_tower_forward, and the 23 layers' gradients those of the pair the mode selects.  Below
 * layer 0 the backward runs pre_layrnorm's backward on the fp32 gradient of hidden_states[0], sums the position gradient over the
 * crops (the class-embedding gradient is its token-0 row: the two are equal bit for bit), and forms the patch weight's gradient as
 * one weight-gradient GEMM over every patch row (split-K at 29 crops and more).  Deterministic: no atomics, every reduction in a
 * fixed order.  The crops get no gradient.
 */
#ifndef TOKENPACKER_B200_CLIP_TOWER_EMBED_H_
#define TOKENPACKER_B200_CLIP_TOWER_EMBED_H_

#include "tokenpacker_b200_clip_tower_ckpt.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Destinations of the embedding stage's parameter gradients: bf16 device buffers of the parameters' shapes (patch_w [1024, 3, 14, 14],
 * class_emb [1024], pos_emb [577, 1024], pre_ln_w / pre_ln_b [1024]), 16-byte aligned, every element written (not accumulated).  A NULL
 * pointer skips that gradient; with all five NULL the embedding stage does not run. */
typedef struct tp_clip_tower_embed_grads {
  void* patch_w;
  void* class_emb;
  void* pos_emb;
  void* pre_ln_w;
  void* pre_ln_b;
} tp_clip_tower_embed_grads;

/* Bytes of the embedding stage's saved set of a forward over n_crops crops; 0 for n_crops out of range. */
TP_API size_t tp_clip_tower_embed_saved_bytes(int64_t n_crops);

/* The training forward of the whole tower.  checkpoint == 0: as tp_clip_tower_forward_train with trainable_layers = 23 (``saved`` >=
 * tp_clip_tower_train_saved_bytes(n_crops, 23), workspace >= tp_clip_tower_train_workspace_bytes(n_crops, 23)); checkpoint != 0: as
 * tp_clip_tower_forward_ckpt with trainable_layers = 23 (tp_clip_tower_ckpt_saved_bytes, tp_clip_tower_workspace_bytes).  embed_saved:
 * 256-byte aligned, >= tp_clip_tower_embed_saved_bytes.  TP_ERR_INVALID_ARGUMENT / TP_ERR_WORKSPACE_TOO_SMALL before any CUDA call. */
TP_API int tp_clip_tower_forward_train_embed(const void* packed, const tp_clip_tower_weights* w, const void* crops, int64_t n_crops,
                                             int64_t crop_stride, int checkpoint, void* const* out_layers, void* saved, size_t saved_bytes,
                                             void* embed_saved, size_t embed_saved_bytes, void* workspace, size_t workspace_bytes,
                                             void* stream);

/* Parameter gradients of the 23 layers (grads: 23 entries, grads[i] for layer i, as tp_clip_tower_backward) and of the embedding
 * stage (embed_grads), from what tp_clip_tower_forward_train_embed left in ``saved`` and ``embed_saved`` with the same n_crops and
 * checkpoint.  workspace: tp_clip_tower_backward_workspace_bytes(n_crops, 23) (checkpoint == 0) or
 * tp_clip_tower_ckpt_backward_workspace_bytes(n_crops, 23) (checkpoint != 0), 256-byte aligned.  d_out_layers as in
 * tp_clip_tower_backward.  TP_ERR_INVALID_ARGUMENT / TP_ERR_WORKSPACE_TOO_SMALL before any CUDA call. */
TP_API int tp_clip_tower_backward_embed(const tp_clip_tower_weights* w, const void* saved, const void* embed_saved, int64_t n_crops,
                                        int checkpoint, const void* const* d_out_layers, const tp_clip_tower_layer_grads* grads,
                                        const tp_clip_tower_embed_grads* embed_grads, void* workspace, size_t workspace_bytes,
                                        void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TOKENPACKER_B200_CLIP_TOWER_EMBED_H_ */
