/* Plain-C99 consumer of include/tokenpacker_b200_clip_tower_f16.h: compiles, links, and exercises the argument checks of the fp16 tower
 * (no GPU needed: every call below is refused before any CUDA work). */
#include <stdio.h>
#include <string.h>

#include "tokenpacker_b200_clip_tower_f16.h"

#define EXPECT(cond)                                          \
  do {                                                        \
    if (!(cond)) {                                            \
      fprintf(stderr, "failed: %s (line %d)\n", #cond, __LINE__); \
      return 1;                                               \
    }                                                         \
  } while (0)

int main(void) {
  int (*pack)(const tp_clip_tower_weights*, void*, size_t, void*) = &tp_clip_tower_pack_weights_f16;
  int (*fwd)(const void*, const tp_clip_tower_weights*, const void*, int, int64_t, int64_t, void* const*, void*, size_t, void*) =
      &tp_clip_tower_forward_f16;
  tp_clip_tower_weights w;
  void* outs[4] = {(void*)4096, (void*)8192, (void*)12288, (void*)16384};
  const int64_t cs = 3 * 336 * 336;
  size_t i;
  for (i = 0; i < sizeof(w) / sizeof(void*); ++i) ((const void**)&w)[i] = (const void*)4096;
  EXPECT(pack(NULL, (void*)4096, tp_clip_tower_packed_bytes(), NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(pack(&w, (void*)4096, tp_clip_tower_packed_bytes() - 1, NULL) == TP_ERR_WORKSPACE_TOO_SMALL);
  EXPECT(fwd((void*)4096, &w, (void*)4096, 0, 1, cs, outs, (void*)4096, tp_clip_tower_workspace_bytes(1), NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(fwd((void*)4096, &w, (void*)4096, 3, 1, cs, outs, (void*)4096, tp_clip_tower_workspace_bytes(1), NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(fwd((void*)4096, &w, (void*)4096, TP_CLIP_CROPS_F16, 0, cs, outs, (void*)4096, tp_clip_tower_workspace_bytes(1), NULL) ==
         TP_ERR_INVALID_ARGUMENT);
  EXPECT(fwd((void*)4096, &w, (void*)4096, TP_CLIP_CROPS_BF16, 1, cs, outs, (void*)4096, tp_clip_tower_workspace_bytes(1) - 1, NULL) ==
         TP_ERR_WORKSPACE_TOO_SMALL);
  w.layers[22].q_w = NULL;
  EXPECT(fwd((void*)4096, &w, (void*)4096, TP_CLIP_CROPS_F16, 1, cs, outs, (void*)4096, tp_clip_tower_workspace_bytes(1), NULL) ==
         TP_ERR_INVALID_ARGUMENT);
  EXPECT(TP_CLIP_CROPS_BF16 == 1 && TP_CLIP_CROPS_F16 == 2 && TP_CLIP_TOWER_LAYERS == 23 && tp_abi_version() == 2);
  printf("abi clip tower f16 ok\n");
  return 0;
}
