/* Plain-C99 consumer of include/tokenpacker_b200_clip_tower.h: compiles, links, and exercises the size queries and argument checks
 * (no GPU needed: every call below is refused or answered before any CUDA work). */
#include <stdio.h>
#include <string.h>

#include "tokenpacker_b200_clip_tower.h"

#define EXPECT(cond)                                          \
  do {                                                        \
    if (!(cond)) {                                            \
      fprintf(stderr, "failed: %s (line %d)\n", #cond, __LINE__); \
      return 1;                                               \
    }                                                         \
  } while (0)

int main(void) {
  size_t (*packed_bytes)(void) = &tp_clip_tower_packed_bytes;
  int (*pack)(const tp_clip_tower_weights*, void*, size_t, void*) = &tp_clip_tower_pack_weights;
  size_t (*ws_bytes)(int64_t) = &tp_clip_tower_workspace_bytes;
  int (*fwd)(const void*, const tp_clip_tower_weights*, const void*, int64_t, int64_t, void* const*, void*, size_t, void*) =
      &tp_clip_tower_forward;
  tp_clip_tower_weights w;
  void* outs[4] = {(void*)4096, (void*)8192, (void*)12288, (void*)16384};
  size_t i;
  for (i = 0; i < sizeof(w) / sizeof(void*); ++i) ((const void**)&w)[i] = (const void*)4096;
  EXPECT(packed_bytes() > (size_t)23 * 3072 * 1024 * 2);
  EXPECT(ws_bytes(0) == 0 && ws_bytes(1) > 0 && ws_bytes(2) > ws_bytes(1));
  EXPECT(pack(NULL, (void*)4096, packed_bytes(), NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(pack(&w, (void*)4096, packed_bytes() - 1, NULL) == TP_ERR_WORKSPACE_TOO_SMALL);
  EXPECT(fwd((void*)4096, &w, (void*)4096, 0, 3 * 336 * 336, outs, (void*)4096, ws_bytes(1), NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(fwd((void*)4096, &w, (void*)4096, 1, 3 * 336 * 336, outs, (void*)4096, ws_bytes(1) - 1, NULL) == TP_ERR_WORKSPACE_TOO_SMALL);
  w.layers[22].q_w = NULL;
  EXPECT(fwd((void*)4096, &w, (void*)4096, 1, 3 * 336 * 336, outs, (void*)4096, ws_bytes(1), NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(TP_CLIP_TOWER_LAYERS == 23 && tp_abi_version() == 2);
  printf("abi clip tower ok\n");
  return 0;
}
