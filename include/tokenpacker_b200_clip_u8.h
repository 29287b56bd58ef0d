/* tokenpacker_b200 — decoded 8-bit images into the non-HD CLIP input (libtokenpacker_b200.so).
 *
 * Companion of tokenpacker_b200_hd_u8.h, whose tp_hd_u8_source it reuses, and of tokenpacker_b200.h, whose conventions and status
 * codes it follows.  Kept in a header of its own so that both stay exactly as their consumers compiled them (tokenpacker_b200.h is
 * ABI version 2); this header only adds.
 *
 * What it computes, per image, is the input path of the non-HD recipes (image_aspect_ratio 'pad' or 'square'):
 *   pad only: expand2square (llava/mm_utils.py:14-25) onto a virtual L x L canvas, L = max(h, w), of the background colour
 *             (122, 116, 104), the image pasted at ((L - w) / 2, 0) or (0, (L - h) / 2); nothing of size L x L is materialised
 *   then the slow (PIL) CLIPImageProcessor with the openai/clip-vit-large-patch14-336 configuration: shortest edge -> 336
 *             (long edge int(336 * long / short); nothing resized when the short edge is already 336) with PIL's 8-bit BICUBIC
 *             resample, center crop 336 x 336, rescale 1/255 and normalise, as norm_table[c * 256 + byte]
 * The result is PIL's fixed-point resample bit for bit (int32 coefficients with 22 fraction bits, a horizontal pass rounded to
 * uint8, then a vertical pass), so with tokenpacker_b200.hd.norm_table() it is the processor's float32 output bit for bit.
 * (The default CLIPImageProcessor of transformers >= 5 is a torchvision-based "fast" processor whose bits differ.)
 */
#ifndef TOKENPACKER_B200_CLIP_U8_H_
#define TOKENPACKER_B200_CLIP_U8_H_

#include "tokenpacker_b200_hd_u8.h"

#ifdef __cplusplus
extern "C" {
#endif

enum { TP_CLIP_SQUARE = 0, TP_CLIP_PAD = 1 };
#define TP_CLIP_SIZE 336          /* output side: shortest edge and crop */
#define TP_CLIP_MAX_SIDE 32768    /* largest accepted source side */

/* One row of the plan.  A coefficient table is [336] int32 first source index, [336] int32 tap count, then [ksize][336] int32
 * weights (tap-major; zero past the count), for the 336 kept outputs of one axis; coeff_x / coeff_y are its offset in int32
 * elements.  ksize 0 marks a pass that is skipped because its axis keeps its size.  The horizontal pass writes uint8
 * [rows][336][3] for canvas rows row0 .. row0 + rows - 1 at byte workspace_offset (rows = 0 when it is skipped). */
typedef struct tp_clip_image {
  int32_t h, w;                   /* source */
  int32_t canvas_h, canvas_w;     /* L x L in pad mode when h != w, else h x w */
  int32_t pad_y, pad_x;           /* where source pixel (0, 0) lies on the canvas */
  int32_t resized_h, resized_w;   /* size after the resize */
  int32_t top, left;              /* center crop offsets in the resized image */
  int32_t ksize_x, ksize_y;       /* taps of the horizontal / vertical table; 0 = pass skipped */
  int64_t coeff_x, coeff_y;       /* int32 offsets of the tables in coeffs (-1 when skipped) */
  int32_t row0, rows;             /* canvas rows the vertical pass reads, computed by the horizontal pass */
  int64_t workspace_offset;       /* bytes; the horizontal pass's rows of this image */
  int64_t workspace_row;          /* workspace_offset / (336 * 3): the image's first row in the horizontal launch */
} tp_clip_image;

/* Host only, no GPU.  From the source sizes and the mode: every image's geometry, the coefficient tables (deduplicated by
 * (input size, output size, first kept output); in pad mode both axes of a square canvas share one) and the workspace size.
 *   images  [n_images] or NULL, coeffs [*n_coeffs] or NULL: with either NULL nothing is written but the sizes (a size query);
 *   n_coeffs, workspace_bytes  always written: int32 elements of all tables, bytes of the horizontal pass's output
 * TP_ERR_INVALID_ARGUMENT for a bad mode, NULL h / w / n_coeffs / workspace_bytes, n_images < 0, or a side < 1 or above
 * TP_CLIP_MAX_SIDE. */
TP_API int tp_clip_preprocess_plan(const int64_t* h, const int64_t* w, int64_t n_images, int mode, tp_clip_image* images,
                                   int32_t* coeffs, int64_t* n_coeffs, size_t* workspace_bytes);

/* Two launches on the caller's stream for the whole batch, no synchronisation: the horizontal pass into the workspace, then the
 * vertical pass, byte lookup and store into out [n_images, 3, 336, 336].
 *   images_host               the plan's table on the host: it sizes the launches and the workspace check, and is not kept
 *   images_dev / coeffs_dev   device copies of the plan's tables;  sources_dev[n_images]: the images' bytes and element strides
 *                             ((1, 3w, 3) for [h, w, 3], (hw, w, 1) for [3, h, w]; any non-negative strides work)
 *   norm_table_dev            float32 [3][256], device
 *   out_dtype                 0: float32;  1: bfloat16, rounded to nearest even from the float32 value
 *   workspace                 device, at least the plan's workspace_bytes (may be NULL when that is 0)
 * TP_ERR_INVALID_ARGUMENT for a NULL pointer, out_dtype not 0 / 1, n_images < 0, or a grid that does not fit one launch;
 * TP_ERR_WORKSPACE_TOO_SMALL when workspace_bytes is less than the rows of images_host need. */
TP_API int tp_clip_preprocess_batch(const tp_clip_image* images_host, const tp_clip_image* images_dev, const tp_hd_u8_source* sources_dev,
                                    const int32_t* coeffs_dev, int64_t n_images, const float* norm_table_dev, int out_dtype, void* out,
                                    void* workspace, size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TOKENPACKER_B200_CLIP_U8_H_ */
