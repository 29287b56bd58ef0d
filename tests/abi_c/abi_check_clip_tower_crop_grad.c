/* Plain-C99 consumer of include/tokenpacker_b200_clip_tower_crop_grad.h: compiles, links, and exercises the host plan and the argument
 * checks (no GPU needed: every call below is answered or refused before any CUDA work). */
#include <stdio.h>
#include <string.h>

#include "tokenpacker_b200_clip_tower_crop_grad.h"

#define EXPECT(cond)                                          \
  do {                                                        \
    if (!(cond)) {                                            \
      fprintf(stderr, "failed: %s (line %d)\n", #cond, __LINE__); \
      return 1;                                               \
    }                                                         \
  } while (0)

int main(void) {
  int (*bwd)(const tp_clip_tower_weights*, const void*, const void*, int64_t, int, const void* const*, const tp_clip_tower_layer_grads*,
             const tp_clip_tower_embed_grads*, void*, int, int64_t, void*, size_t, void*) = &tp_clip_tower_backward_crops;
  int (*plan)(const tp_hd_image*, int64_t, float* const*, tp_hd_image_grad*, int32_t*, int64_t*, int64_t*) = &tp_hd_tile_batch_backward_plan;
  int (*hd_bwd)(const tp_hd_image*, const tp_hd_image_grad*, const int32_t*, int64_t, int64_t, const float*, void*) = &tp_hd_tile_batch_backward;
  tp_clip_tower_weights w;
  tp_clip_tower_layer_grads grads[23];
  tp_clip_tower_embed_grads eg;
  const void* d_outs[4] = {NULL, NULL, NULL, (const void*)4096};
  const int64_t cs = 3 * 336 * 336;
  const size_t bws = tp_clip_tower_backward_workspace_bytes(1, 23), cws = tp_clip_tower_ckpt_backward_workspace_bytes(1, 23);
  void* P = (void*)4096;
  size_t i;
  for (i = 0; i < sizeof(w) / sizeof(void*); ++i) ((const void**)&w)[i] = (const void*)4096;
  memset(grads, 0, sizeof(grads));
  memset(&eg, 0, sizeof(eg));
  EXPECT(bwd(&w, P, P, 1, 0, d_outs, grads, &eg, P, TP_CROP_GRAD_F32, cs, P, bws - 1, NULL) == TP_ERR_WORKSPACE_TOO_SMALL);
  EXPECT(bwd(&w, P, P, 1, 1, d_outs, NULL, NULL, P, TP_CROP_GRAD_BF16, cs, P, cws - 1, NULL) == TP_ERR_WORKSPACE_TOO_SMALL);
  EXPECT(bwd(&w, P, P, 1, 0, d_outs, grads, &eg, NULL, TP_CROP_GRAD_F32, cs, P, bws, NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(bwd(&w, P, P, 1, 0, d_outs, grads, &eg, P, 2, cs, P, bws, NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(bwd(&w, P, P, 1, 0, d_outs, grads, &eg, P, TP_CROP_GRAD_F32, cs - 1, P, bws, NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(bwd(&w, P, P, 1, 0, d_outs, grads, &eg, (void*)4098, TP_CROP_GRAD_F32, cs, P, bws, NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(bwd(&w, P, NULL, 1, 0, d_outs, grads, &eg, P, TP_CROP_GRAD_F32, cs, P, bws, NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(bwd(&w, P, P, 0, 0, d_outs, grads, &eg, P, TP_CROP_GRAD_F32, cs, P, bws, NULL) == TP_ERR_INVALID_ARGUMENT);
  eg.pos_emb = (void*)4098;
  EXPECT(bwd(&w, P, P, 1, 0, d_outs, grads, &eg, P, TP_CROP_GRAD_BF16, cs, P, bws, NULL) == TP_ERR_INVALID_ARGUMENT);
  {
    /* one 500 x 300 image on a 3 x 2 grid: count, then fill */
    int64_t hs[1] = {500}, ws[1] = {300}, n = 0, words = 0, words2 = 0, most = 0;
    int hb = 0, wb = 0;
    tp_hd_image im;
    tp_hd_image_grad g;
    static int32_t taps[1 << 16];
    float* d = (float*)P;
    EXPECT(tp_hd_tile_batch_plan(hs, ws, NULL, 1, 9, &im, NULL, &hb, &wb, &n) == TP_OK);
    EXPECT(plan(&im, 1, NULL, NULL, NULL, &words, &most) == TP_OK && most == 500 * 300 && words > 0 && words < (1 << 16));
    EXPECT(plan(&im, 1, &d, &g, taps, &words2, &most) == TP_OK && words2 == words && g.d_image == d && g.row_taps == 0);
    EXPECT(taps[0] == 0 && (hb * wb > 1) == (g.thumb_row_taps > 0));
    EXPECT(plan(NULL, 1, NULL, NULL, NULL, &words, &most) == TP_ERR_INVALID_ARGUMENT);
    EXPECT(plan(&im, 1, NULL, NULL, NULL, NULL, &most) == TP_ERR_INVALID_ARGUMENT);
    im.h_r = 0;
    EXPECT(plan(&im, 1, NULL, NULL, NULL, &words, &most) == TP_ERR_INVALID_ARGUMENT);
    EXPECT(hd_bwd(NULL, &g, taps, 1, most, d, NULL) == TP_ERR_INVALID_ARGUMENT);
    EXPECT(hd_bwd(&im, &g, taps, -1, most, d, NULL) == TP_ERR_INVALID_ARGUMENT);
    EXPECT(hd_bwd(&im, &g, taps, 1, most, NULL, NULL) == TP_ERR_INVALID_ARGUMENT);
  }
  EXPECT(tp_abi_version() == 2);
  printf("abi clip tower crop grad ok\n");
  return 0;
}
