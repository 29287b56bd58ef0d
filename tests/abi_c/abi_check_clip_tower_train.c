/* Plain-C99 consumer of include/tokenpacker_b200_clip_tower_train.h: compiles, links, and exercises the size queries and argument
 * checks (no GPU needed: every call below is refused or answered before any CUDA work). */
#include <stdio.h>
#include <string.h>

#include "tokenpacker_b200_clip_tower_train.h"

#define EXPECT(cond)                                          \
  do {                                                        \
    if (!(cond)) {                                            \
      fprintf(stderr, "failed: %s (line %d)\n", #cond, __LINE__); \
      return 1;                                               \
    }                                                         \
  } while (0)

int main(void) {
  size_t (*saved_bytes)(int64_t, int) = &tp_clip_tower_train_saved_bytes;
  size_t (*fwd_ws)(int64_t, int) = &tp_clip_tower_train_workspace_bytes;
  size_t (*bwd_ws)(int64_t, int) = &tp_clip_tower_backward_workspace_bytes;
  int (*fwd)(const void*, const tp_clip_tower_weights*, const void*, int64_t, int64_t, int, void* const*, void*, size_t, void*, size_t, void*) =
      &tp_clip_tower_forward_train;
  int (*bwd)(const tp_clip_tower_weights*, const void*, int64_t, int, const void* const*, const tp_clip_tower_layer_grads*, void*, size_t,
             void*) = &tp_clip_tower_backward;
  tp_clip_tower_weights w;
  tp_clip_tower_layer_grads grads[2];
  void* outs[4] = {(void*)4096, (void*)8192, (void*)12288, (void*)16384};
  const void* d_outs[4] = {NULL, NULL, NULL, (const void*)4096};
  const int64_t cs = 3 * 336 * 336;
  size_t i;
  for (i = 0; i < sizeof(w) / sizeof(void*); ++i) ((const void**)&w)[i] = (const void*)4096;
  memset(grads, 0, sizeof(grads));
  EXPECT(sizeof(tp_clip_tower_layer_grads) == sizeof(tp_clip_tower_layer));
  EXPECT(saved_bytes(0, 1) == 0 && saved_bytes(1, 0) == 0 && saved_bytes(1, 24) == 0);
  EXPECT(saved_bytes(1, 1) > (size_t)577 * 34 * 1024 && saved_bytes(1, 2) == 2 * saved_bytes(1, 1) && saved_bytes(2, 1) > saved_bytes(1, 1));
  EXPECT(fwd_ws(1, 1) > tp_clip_tower_workspace_bytes(1) && fwd_ws(2, 1) > fwd_ws(1, 1) && fwd_ws(1, 0) == 0);
  EXPECT(bwd_ws(1, 1) > 0 && bwd_ws(2, 1) > bwd_ws(1, 1) && bwd_ws(1, 24) == 0);
  EXPECT(fwd((void*)4096, &w, (void*)4096, 1, cs, 0, outs, (void*)4096, saved_bytes(1, 1), (void*)4096, fwd_ws(1, 1), NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(fwd((void*)4096, &w, (void*)4096, 1, cs, 2, outs, NULL, saved_bytes(1, 2), (void*)4096, fwd_ws(1, 2), NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(fwd((void*)4096, &w, (void*)4096, 1, cs, 2, outs, (void*)4096, saved_bytes(1, 2) - 1, (void*)4096, fwd_ws(1, 2), NULL) == TP_ERR_WORKSPACE_TOO_SMALL);
  EXPECT(fwd((void*)4096, &w, (void*)4096, 1, cs, 2, outs, (void*)4096, saved_bytes(1, 2), (void*)4096, fwd_ws(1, 2) - 1, NULL) == TP_ERR_WORKSPACE_TOO_SMALL);
  EXPECT(fwd((void*)4096, &w, NULL, 1, cs, 2, outs, (void*)4096, saved_bytes(1, 2), (void*)4096, fwd_ws(1, 2), NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(bwd(&w, (void*)4096, 1, 2, d_outs, grads, (void*)4096, bwd_ws(1, 2) - 1, NULL) == TP_ERR_WORKSPACE_TOO_SMALL);
  EXPECT(bwd(&w, (void*)4096, 1, 24, d_outs, grads, (void*)4096, bwd_ws(1, 2), NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(bwd(&w, NULL, 1, 2, d_outs, grads, (void*)4096, bwd_ws(1, 2), NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(bwd(&w, (void*)4096, 1, 2, d_outs, NULL, (void*)4096, bwd_ws(1, 2), NULL) == TP_ERR_INVALID_ARGUMENT);
  grads[1].fc1_w = (void*)4098;
  EXPECT(bwd(&w, (void*)4096, 1, 2, d_outs, grads, (void*)4096, bwd_ws(1, 2), NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(tp_abi_version() == 2);
  printf("abi clip tower train ok\n");
  return 0;
}
