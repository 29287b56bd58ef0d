/* tokenpacker_b200 — the frozen CLIP-ViT-L/14-336 vision tower, forward only (libtokenpacker_b200.so).
 *
 * Companion of tokenpacker_b200.h, whose conventions and status codes it uses; that header and its ABI version 2 are unchanged.
 * Computes transformers' CLIPVisionTransformer (openai/clip-vit-large-patch14-336) up to and including hidden_states[23]:
 *   emb = cat(class_embedding, conv14x14/14(pixels)) + position_embedding;  hidden_states[0] = pre_layrnorm(emb)
 *   layer i (0..22): x = x + out_proj(attn(LN1(x)));  x = x + fc2(quick_gelu(fc1(LN2(x))));  hidden_states[i + 1] = x
 * (LayerNorms as explicit passes; the linears read their weights as they are).
 * Layer 23, post_layernorm and the pooled output are not computed.  bf16 storage, fp32 accumulation, one rounding per stored tensor.
 *
 * Memory is the caller's: device pointers, work enqueued on ``stream`` (a cudaStream_t; NULL = legacy default stream), no
 * synchronisation.  Argument checks run before any CUDA call.
 */
#ifndef TOKENPACKER_B200_CLIP_TOWER_H_
#define TOKENPACKER_B200_CLIP_TOWER_H_

#include "tokenpacker_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#define TP_CLIP_TOWER_LAYERS 23   /* encoder layers run: hidden_states[23] is the output of layer 22 */

/* One encoder layer's parameters, bf16 device pointers in transformers' shapes ([out, in] weights). */
typedef struct tp_clip_tower_layer {
  const void* ln1_w; const void* ln1_b;                       /* layer_norm1 [1024] */
  const void* q_w; const void* q_b;                           /* self_attn.q_proj [1024,1024], [1024] */
  const void* k_w; const void* k_b;
  const void* v_w; const void* v_b;
  const void* o_w; const void* o_b;                           /* self_attn.out_proj */
  const void* ln2_w; const void* ln2_b;                       /* layer_norm2 */
  const void* fc1_w; const void* fc1_b;                       /* mlp.fc1 [4096,1024], [4096] */
  const void* fc2_w; const void* fc2_b;                       /* mlp.fc2 [1024,4096], [1024] */
} tp_clip_tower_layer;

typedef struct tp_clip_tower_weights {
  const void* patch_w;                                        /* embeddings.patch_embedding.weight [1024,3,14,14] */
  const void* class_emb;                                      /* embeddings.class_embedding [1024] */
  const void* pos_emb;                                        /* embeddings.position_embedding.weight [577,1024] */
  const void* pre_ln_w; const void* pre_ln_b;                 /* pre_layrnorm [1024] */
  tp_clip_tower_layer layers[TP_CLIP_TOWER_LAYERS];
} tp_clip_tower_weights;

/* Bytes of the derived weights tp_clip_tower_pack_weights writes (about 147 MB): per layer the q/k/v concatenation [3072,1024] with
 * the q rows scaled by 1/8 (exact: a power of two) and the biases in fp32; and the patch weight with its rows padded to 592 elements
 * (TMA needs 16-byte row strides).  out_proj, fc1, fc2, the LayerNorms and the embeddings are read in place. */
TP_API size_t tp_clip_tower_packed_bytes(void);

/* Fill ``packed`` (256-byte aligned, >= tp_clip_tower_packed_bytes()) from ``w``.  Every pointer of ``w`` must be non-NULL and
 * 16-byte aligned.
 * TP_ERR_INVALID_ARGUMENT / TP_ERR_WORKSPACE_TOO_SMALL before any CUDA call. */
TP_API int tp_clip_tower_pack_weights(const tp_clip_tower_weights* w, void* packed, size_t packed_bytes, void* stream);

/* Workspace bytes of a tp_clip_tower_forward call over n_crops crops (0 when n_crops <= 0). */
TP_API size_t tp_clip_tower_workspace_bytes(int64_t n_crops);

/* hidden_states 12, 16, 22 and 23 of n_crops crops.
 *   packed           tp_clip_tower_pack_weights output
 *   w                the weights it was packed from (non-NULL, 16-byte aligned): everything but q/k/v is read in place
 *   crops            bf16 [n_crops, 3, 336, 336], crop n at crops + n * crop_stride (elements, >= 3 * 336 * 336), each crop contiguous
 *   out_layers       4 distinct bf16 destinations [n_crops, 577, 1024], contiguous (CLS row included), 16-byte aligned.
 *                    They are also the residual stream the following layers read: no hidden state is ever copied.
 *   workspace        >= tp_clip_tower_workspace_bytes(n_crops), 256-byte aligned
 * Crop n of a batch gets the bits of a call on that crop alone.  TP_ERR_INVALID_ARGUMENT / TP_ERR_WORKSPACE_TOO_SMALL before any CUDA
 * call; TP_ERR_UNSUPPORTED_DEVICE off sm_90. */
TP_API int tp_clip_tower_forward(const void* packed, const tp_clip_tower_weights* w, const void* crops, int64_t n_crops, int64_t crop_stride,
                                 void* const* out_layers, void* workspace, size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TOKENPACKER_B200_CLIP_TOWER_H_ */
