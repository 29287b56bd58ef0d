/* tokenpacker_b200 — decoded 8-bit images into the batched HD front end (libtokenpacker_b200.so).
 *
 * Companion of tokenpacker_b200.h, whose conventions, status codes and tp_hd_image / tp_hd_tile_batch_plan it uses.  Kept in a
 * header of its own so that tokenpacker_b200.h, ABI version 2, stays exactly as its consumers compiled it; this header only adds.
 */
#ifndef TOKENPACKER_B200_HD_U8_H_
#define TOKENPACKER_B200_HD_U8_H_

#include "tokenpacker_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The batched tiling block of tp_hd_tile_batch on DECODED 8-bit images, with ToTensor + Normalize (train.py:645) folded in: every
 * HD recipe runs Compose([ToTensor(), Normalize(mean, std)]) on the full-resolution image before the tiling block
 * (train.py:695-731).  A byte u of channel c is read as norm_table_dev[c * 256 + u]; with the table built on the host by the CPU
 * ops torchvision runs, (u / 255 - mean[c]) / std[c], the crops have exactly the bits tp_hd_tile_batch gives for the
 * host-normalised float32 image.  The padding of the canvas and of the thumbnail stays 0.0 (normalised space, train.py:710,728),
 * not norm_table[c][0].
 *   images_dev / crop_table_dev  device copies of the tables of tp_hd_tile_batch_plan, called with images = NULL
 *   sources_dev[n_images]        per image: device pointer to pixel (0, 0, 0) and the element strides of channel, row and column;
 *                                (stride_c, stride_y, stride_x) = (1, 3w, 3) for an [h, w, 3] image (np.array(pil_image)),
 *                                (hw, w, 1) for [3, h, w]; any non-negative strides work
 *   norm_table_dev               float32 [3][256], device
 *   out_dtype                    0: crops [n_crops, 3, 336, 336] float32;  1: bfloat16, rounded to nearest even from the float32 value
 * TP_ERR_INVALID_ARGUMENT for a NULL pointer, out_dtype not 0 / 1, n_crops < 0, or more crops than one launch grid holds. */
typedef struct tp_hd_u8_source {
  const uint8_t* pixels;
  int64_t stride_c, stride_y, stride_x;
} tp_hd_u8_source;
TP_API int tp_hd_preprocess_batch(const tp_hd_image* images_dev, const tp_hd_u8_source* sources_dev, const int32_t* crop_table_dev,
                                  int64_t n_crops, const float* norm_table_dev, int out_dtype, void* crops, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TOKENPACKER_B200_HD_U8_H_ */
