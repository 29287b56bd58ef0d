/* tokenpacker_b200 — gradients to the pixels (libtokenpacker_b200.so): the gradient of the CLIP tower's crops, and the backward of the
 * HD tiling block that made them from normalised images.
 *
 * Companion of tokenpacker_b200_clip_tower_embed.h (and through it of the tower's other headers and tokenpacker_b200.h), whose structs,
 * conventions and status codes it uses; those headers are unchanged.
 *
 * tp_clip_tower_backward_crops runs the backward of tp_clip_tower_backward_embed (same saved sets, same workspace, same bits for every
 * parameter gradient asked for) and, below the embedding stage, the patch embedding's input gradient:
 *   d_rows [576 n, 588] = d_patch_out [576 n, 1024] . W_patch [1024, 588]
 * where d_patch_out is the bf16 gradient of the patch GEMM's output rows (token rows 1..576 of every crop: the class token's row gets no
 * crop gradient) and W_patch the live patch weight (repacked into zero-padded 608-element rows in the workspace: a 588-element bf16 row is
 * not a legal TMA stride).  One NN-form GEMM of the tile engine writes d_rows in fp32 into the workspace, and one col2im kernel stores
 * column c * 196 + ky * 14 + kx of row n * 576 + py * 24 + px to d_crops[n][c][14 py + ky][14 px + kx].  Patches do not overlap: every
 * crop element is written exactly once, with no atomics and nothing accumulated.  fp32 crops receive the fp32 values the GEMM
 * accumulated; bf16 crops their one rounding.  Deterministic.
 *
 * tp_hd_tile_batch_backward is the exact adjoint of tp_hd_tile_batch (train.py:695-731): d_images (fp32 [3, h, w] per image) from the
 * gradient of the crops, through the thumbnail resize (when an image has more than one crop), the split into crops, the zero padding
 * (which gets no gradient) and the bilinear resize (align_corners=False).  Gather form: one thread per source pixel and channel, which
 * walks per-axis inverse-tap tables built on the host by tp_hd_tile_batch_backward_plan; each sum runs in a fixed order (the main
 * canvas's contributions, then the thumbnail's).  Deterministic.
 */
#ifndef TOKENPACKER_B200_CLIP_TOWER_CROP_GRAD_H_
#define TOKENPACKER_B200_CLIP_TOWER_CROP_GRAD_H_

#include "tokenpacker_b200_clip_tower_embed.h"

#ifdef __cplusplus
extern "C" {
#endif

#define TP_CROP_GRAD_BF16 0   /* d_crops_dtype: bf16 crop gradients */
#define TP_CROP_GRAD_F32 1    /* d_crops_dtype: fp32 crop gradients */

/* tp_clip_tower_backward_embed (same w, saved, embed_saved, n_crops, checkpoint, d_out_layers, workspace and workspace size) that also
 * writes d_crops [n_crops, 3, 336, 336] (d_crops_dtype TP_CROP_GRAD_BF16 or TP_CROP_GRAD_F32, d_crop_stride elements between crops,
 * >= 3 * 336 * 336; aligned to its element size).  grads (23 entries) and embed_grads may be NULL, and so may every pointer in them: a
 * frozen tower still backpropagates through its 23 layers, pre_layrnorm and the patch embedding.  Every parameter gradient asked for has
 * the bits tp_clip_tower_backward_embed gives.  TP_ERR_INVALID_ARGUMENT / TP_ERR_WORKSPACE_TOO_SMALL before any CUDA call. */
TP_API int tp_clip_tower_backward_crops(const tp_clip_tower_weights* w, const void* saved, const void* embed_saved, int64_t n_crops,
                                        int checkpoint, const void* const* d_out_layers, const tp_clip_tower_layer_grads* grads,
                                        const tp_clip_tower_embed_grads* embed_grads, void* d_crops, int d_crops_dtype,
                                        int64_t d_crop_stride, void* workspace, size_t workspace_bytes, void* stream);

/* Where tp_hd_tile_batch_backward writes one image's gradient, and where that image's inverse-tap tables are (int32 word offsets into the
 * taps buffer).  A table over n indices is n + 1 entry offsets followed by its entries, (index, weight) pairs of int32 words (the weight's
 * float bits): row_taps lists, for each source row, the canvas rows that read it (with their bilinear weights), col_taps the same for
 * columns; thumb_row_taps / thumb_col_taps list, for each canvas row / column inside the resized content, the thumbnail rows / columns
 * that read it (-1 without a thumbnail). */
typedef struct tp_hd_image_grad {
  float* d_image;
  int64_t row_taps, col_taps;
  int64_t thumb_row_taps, thumb_col_taps;
} tp_hd_image_grad;

/* Host function.  For the n_images rows images_host of a tp_hd_tile_batch_plan: fills grads_host[n_images] (d_image = d_images[b], a
 * DEVICE pointer to fp32 [3, h, w]) and taps_host, and reports the words the tables take (*taps_words) and the largest h * w of the
 * batch (*max_pixels).  grads_host, taps_host and d_images may be NULL (count only). */
TP_API int tp_hd_tile_batch_backward_plan(const tp_hd_image* images_host, int64_t n_images, float* const* d_images,
                                          tp_hd_image_grad* grads_host, int32_t* taps_host, int64_t* taps_words, int64_t* max_pixels);

/* The launch: images_dev / grads_dev / taps_dev are device copies of the plans' tables; d_crops fp32 [n_crops, 3, 336, 336], contiguous,
 * the gradient of the crops of the tp_hd_tile_batch launch with the same images_dev; every d_image element is written. */
TP_API int tp_hd_tile_batch_backward(const tp_hd_image* images_dev, const tp_hd_image_grad* grads_dev, const int32_t* taps_dev,
                                     int64_t n_images, int64_t max_pixels, const float* d_crops, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TOKENPACKER_B200_CLIP_TOWER_CROP_GRAD_H_ */
