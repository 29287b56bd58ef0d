/* Plain-C99 consumer of include/tokenpacker_b200_clip_tower_embed.h: compiles, links, and exercises the size query and argument checks
 * (no GPU needed: every call below is refused or answered before any CUDA work). */
#include <stdio.h>
#include <string.h>

#include "tokenpacker_b200_clip_tower_embed.h"

#define EXPECT(cond)                                          \
  do {                                                        \
    if (!(cond)) {                                            \
      fprintf(stderr, "failed: %s (line %d)\n", #cond, __LINE__); \
      return 1;                                               \
    }                                                         \
  } while (0)

int main(void) {
  size_t (*embed_bytes)(int64_t) = &tp_clip_tower_embed_saved_bytes;
  int (*fwd)(const void*, const tp_clip_tower_weights*, const void*, int64_t, int64_t, int, void* const*, void*, size_t, void*, size_t, void*,
             size_t, void*) = &tp_clip_tower_forward_train_embed;
  int (*bwd)(const tp_clip_tower_weights*, const void*, const void*, int64_t, int, const void* const*, const tp_clip_tower_layer_grads*,
             const tp_clip_tower_embed_grads*, void*, size_t, void*) = &tp_clip_tower_backward_embed;
  tp_clip_tower_weights w;
  tp_clip_tower_layer_grads grads[23];
  tp_clip_tower_embed_grads eg;
  void* outs[4] = {(void*)4096, (void*)8192, (void*)12288, (void*)16384};
  const void* d_outs[4] = {NULL, NULL, NULL, (const void*)4096};
  const int64_t cs = 3 * 336 * 336;
  const size_t eb = embed_bytes(1), sb = tp_clip_tower_ckpt_saved_bytes(1, 23), fwd_ws = tp_clip_tower_workspace_bytes(1);
  const size_t bws = tp_clip_tower_ckpt_backward_workspace_bytes(1, 23);
  void* P = (void*)4096;
  size_t i;
  for (i = 0; i < sizeof(w) / sizeof(void*); ++i) ((const void**)&w)[i] = (const void*)4096;
  memset(grads, 0, sizeof(grads));
  memset(&eg, 0, sizeof(eg));
  EXPECT(embed_bytes(0) == 0 && embed_bytes(-1) == 0);
  EXPECT(eb >= (size_t)576 * 592 * 2 + (size_t)577 * 1024 * 2 && embed_bytes(2) > eb);
  EXPECT(fwd(P, &w, P, 1, cs, 1, outs, P, sb, NULL, eb, P, fwd_ws, NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(fwd(P, &w, P, 1, cs, 1, outs, P, sb, (void*)(4096 + 16), eb, P, fwd_ws, NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(fwd(P, &w, P, 1, cs, 1, outs, P, sb, P, eb - 1, P, fwd_ws, NULL) == TP_ERR_WORKSPACE_TOO_SMALL);
  EXPECT(fwd(P, &w, P, 1, cs, 1, outs, P, sb - 1, P, eb, P, fwd_ws, NULL) == TP_ERR_WORKSPACE_TOO_SMALL);
  EXPECT(fwd(P, &w, P, 1, cs, 0, outs, P, sb, P, eb, P, fwd_ws, NULL) == TP_ERR_WORKSPACE_TOO_SMALL);   /* the full saved sets are larger */
  EXPECT(fwd(P, &w, P, 0, cs, 1, outs, P, sb, P, eb, P, fwd_ws, NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(bwd(&w, P, P, 1, 1, d_outs, grads, &eg, P, bws - 1, NULL) == TP_ERR_WORKSPACE_TOO_SMALL);
  EXPECT(bwd(&w, P, NULL, 1, 1, d_outs, grads, &eg, P, bws, NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(bwd(&w, P, P, 1, 1, d_outs, grads, NULL, P, bws, NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(bwd(&w, P, P, 1, 1, d_outs, NULL, &eg, P, bws, NULL) == TP_ERR_INVALID_ARGUMENT);
  eg.pos_emb = (void*)4098;
  EXPECT(bwd(&w, P, P, 1, 1, d_outs, grads, &eg, P, bws, NULL) == TP_ERR_INVALID_ARGUMENT);
  EXPECT(tp_abi_version() == 2);
  printf("abi clip tower embed ok\n");
  return 0;
}
