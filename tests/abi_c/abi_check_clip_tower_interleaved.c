/* Plain-C99 consumer of include/tokenpacker_b200_clip_tower_interleaved.h: compiles, links, and exercises the argument checks of the
 * interleaved forward in both precisions (no GPU needed: every call below is refused before any CUDA work). */
#include <stdio.h>
#include <string.h>

#include "tokenpacker_b200_clip_tower_interleaved.h"

#define EXPECT(cond)                                          \
  do {                                                        \
    if (!(cond)) {                                            \
      fprintf(stderr, "failed: %s (line %d)\n", #cond, __LINE__); \
      return 1;                                               \
    }                                                         \
  } while (0)

int main(void) {
  int (*fwd)(const void*, const tp_clip_tower_weights*, const void*, int64_t, int64_t, void*, void*, size_t, void*) =
      &tp_clip_tower_forward_interleaved;
  int (*fwd16)(const void*, const tp_clip_tower_weights*, const void*, int, int64_t, int64_t, void*, void*, size_t, void*) =
      &tp_clip_tower_forward_interleaved_f16;
  tp_clip_tower_weights w;
  void* P = (void*)4096;
  const int64_t cs = 3 * 336 * 336;
  const size_t ws1 = tp_clip_tower_workspace_bytes(1);
  const int F16 = TP_CLIP_CROPS_F16, BF16 = TP_CLIP_CROPS_BF16;
  size_t i;
  for (i = 0; i < sizeof(w) / sizeof(void*); ++i) ((const void**)&w)[i] = (const void*)4096;
  /* NULLs */
  EXPECT(fwd(NULL, &w, P, 1, cs, P, P, ws1, NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(fwd(P, NULL, P, 1, cs, P, P, ws1, NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(fwd(P, &w, NULL, 1, cs, P, P, ws1, NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(fwd(P, &w, P, 1, cs, NULL, P, ws1, NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(fwd(P, &w, P, 1, cs, P, NULL, ws1, NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(fwd16(P, &w, P, F16, 1, cs, NULL, P, ws1, NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(fwd16(NULL, &w, P, BF16, 1, cs, P, P, ws1, NULL) == TP_ERR_INVALID_ARGUMENT);
  /* batch size, crop stride, crops dtype */
  EXPECT(fwd(P, &w, P, 0, cs, P, P, ws1, NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(fwd(P, &w, P, -1, cs, P, P, ws1, NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(fwd16(P, &w, P, F16, -1, cs, P, P, ws1, NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(fwd(P, &w, P, 1, cs - 1, P, P, ws1, NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(fwd16(P, &w, P, 0, 1, cs, P, P, ws1, NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(fwd16(P, &w, P, 3, 1, cs, P, P, ws1, NULL) == TP_ERR_INVALID_ARGUMENT);
  /* alignment: the output (16 bytes), packed and workspace (256), crops (2) */
  EXPECT(fwd(P, &w, P, 1, cs, (void*)4104, P, ws1, NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(fwd16(P, &w, P, BF16, 1, cs, (void*)4098, P, ws1, NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(fwd(P, &w, P, 1, cs, P, (void*)4112, ws1, NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(fwd((void*)4112, &w, P, 1, cs, P, P, ws1, NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(fwd(P, &w, (void*)4097, 1, cs, P, P, ws1, NULL) == TP_ERR_INVALID_ARGUMENT);
  /* workspace size: tp_clip_tower_workspace_bytes(n), as for the dense outputs */
  EXPECT(fwd(P, &w, P, 1, cs, P, P, ws1 - 1, NULL) == TP_ERR_WORKSPACE_TOO_SMALL);
  EXPECT(fwd16(P, &w, P, F16, 1, cs, P, P, ws1 - 1, NULL) == TP_ERR_WORKSPACE_TOO_SMALL);
  EXPECT(fwd(P, &w, P, 910, cs, P, P, tp_clip_tower_workspace_bytes(910) - 1, NULL) == TP_ERR_WORKSPACE_TOO_SMALL);
  /* an incomplete weights struct */
  w.layers[12].ln1_w = NULL;
  EXPECT(fwd(P, &w, P, 1, cs, P, P, ws1, NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(fwd16(P, &w, P, F16, 1, cs, P, P, ws1, NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(TP_CLIP_TOWER_LAYERS == 23 && tp_abi_version() == 2);
  printf("abi clip tower interleaved ok\n");
  return 0;
}
