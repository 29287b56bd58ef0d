/* Plain-C99 consumer of include/tokenpacker_b200_clip_u8.h, linked against libtokenpacker_b200.so: every entry point it declares
 * resolves at link time, and the plan and argument validation run without a GPU.  Built and run by
 * tests/test_clip_preprocess_host.py::test_plain_c_consumer_of_the_clip_header. */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "tokenpacker_b200_clip_u8.h"

int main(void) {
  /* taking the address of every entry point makes the link fail if one is declared but not exported */
  const void* entry[] = {(const void*)&tp_clip_preprocess_plan, (const void*)&tp_clip_preprocess_batch};
  size_t i;
  for (i = 0; i < sizeof(entry) / sizeof(entry[0]); ++i)
    if (entry[i] == NULL) return 2;
  if (tp_abi_version() != TP_ABI_VERSION) return 3;
  if (sizeof(tp_clip_image) != 88) return 4;
  {
    /* 480 x 640 in pad mode: a 640 x 640 canvas, the image pasted 80 rows down, both axes 640 -> 336 through one shared table */
    const int64_t h[2] = {480, 336}, w[2] = {640, 336};
    tp_clip_image im[2];
    int64_t n = -1;
    size_t ws = 1;
    int32_t* co;
    if (tp_clip_preprocess_plan(h, w, 2, TP_CLIP_PAD, NULL, NULL, &n, &ws) != TP_OK) return 5;
    if (n != (int64_t)(2 + 9) * TP_CLIP_SIZE || ws != (size_t)640 * TP_CLIP_SIZE * 3) return 6;
    co = (int32_t*)malloc((size_t)n * sizeof(int32_t));
    if (co == NULL) return 7;
    if (tp_clip_preprocess_plan(h, w, 2, TP_CLIP_PAD, im, co, &n, &ws) != TP_OK) return 8;
    if (im[0].canvas_h != 640 || im[0].canvas_w != 640 || im[0].pad_y != 80 || im[0].pad_x != 0) return 9;
    if (im[0].resized_h != 336 || im[0].resized_w != 336 || im[0].coeff_x != 0 || im[0].coeff_y != 0 || im[0].ksize_x != 9) return 10;
    if (im[1].ksize_x != 0 || im[1].ksize_y != 0 || im[1].rows != 0 || im[1].workspace_offset != (int64_t)ws) return 11;
    if (co[0] != 0 || co[TP_CLIP_SIZE] != 5) return 12;               /* output 0 reads source 0 .. 4 */
    /* refused before any CUDA call: never dereferenced */
    {
      float norm[768];
      float out[1];
      unsigned char wsb[1];
      tp_hd_u8_source src;
      memset(norm, 0, sizeof(norm));
      memset(&src, 0, sizeof(src));
      if (tp_clip_preprocess_plan(h, w, 2, 2, NULL, NULL, &n, &ws) != TP_ERR_INVALID_ARGUMENT) return 13;
      if (tp_clip_preprocess_plan(NULL, w, 2, TP_CLIP_PAD, NULL, NULL, &n, &ws) != TP_ERR_INVALID_ARGUMENT) return 14;
      if (tp_clip_preprocess_batch(NULL, im, &src, co, 2, norm, 0, out, wsb, 1, NULL) != TP_ERR_INVALID_ARGUMENT) return 15;
      if (tp_clip_preprocess_batch(im, im, &src, co, 2, norm, 2, out, wsb, 1, NULL) != TP_ERR_INVALID_ARGUMENT) return 16;
      if (tp_clip_preprocess_batch(im, im, &src, co, 2, norm, 1, out, wsb, 1, NULL) != TP_ERR_WORKSPACE_TOO_SMALL) return 17;
      if (tp_clip_preprocess_batch(im, im, &src, co, 0, norm, 1, out, wsb, 1, NULL) != TP_OK) return 18;
    }
    free(co);
  }
  printf("abi clip_u8 ok: %u entry points\n", (unsigned)(sizeof(entry) / sizeof(entry[0])));
  return 0;
}
