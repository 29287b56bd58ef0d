// Test-only entry points into the CLIP tower's embedding-stage backward (libtokenpacker_b200_clip_tower_embed_hooks.so, loaded by
// tests/test_clip_tower_embed_stages_gpu.py; never by the package): the product translation unit plus the tpte_* functions below, which
// run what tp_clip_tower_backward_embed runs below layer 0.  Conventions as in include/tokenpacker_b200.h.
#include "../../tokenpacker_b200/csrc/tp_api.cu"

extern "C" {

// Byte offsets over n crops: out[0..2] = the embedding saved set's patches, rows, total; out[3..8] = the backward workspace's carry32,
// carry16, ln_part, splitk, unused_grad, total
TP_API int tpte_offsets(int64_t n, int64_t* out) {
  if (n <= 0 || out == nullptr) return TP_ERR_INVALID_ARGUMENT;
  const ClipEmbedSavedLayout E = clip_embed_saved_layout(n);
  const ClipBwdLayout B = clip_bwd_layout(n);
  const size_t o[9] = {E.patches, E.rows, E.total, B.carry32, B.carry16, B.ln_part, B.splitk, B.unused_grad, B.total};
  for (int i = 0; i < 9; ++i) out[i] = static_cast<int64_t>(o[i]);
  return TP_OK;
}

// The embedding stage's backward alone (run_clip_embed_backward) up to step last_step (1 .. 3, the numbering of
// tp_clip_tower_embed.inl), from an embedding saved set of tp_clip_tower_forward_train_embed over n crops.  The carry is NOT
// initialised: the caller writes carry32 (the fp32 gradient of hidden_states[0]) into ws.
TP_API int tpte_embed_backward(const tp_clip_tower_weights* w, const void* embed_saved, int64_t n, const tp_clip_tower_embed_grads* grads,
                               void* ws, size_t ws_bytes, int last_step, void* stream) {
  if (w == nullptr || embed_saved == nullptr || grads == nullptr || ws == nullptr || n <= 0 || last_step < 1 || last_step > 3 ||
      !clip_weights_complete(w))
    return TP_ERR_INVALID_ARGUMENT;
  if ((reinterpret_cast<uintptr_t>(embed_saved) & 255) != 0 || (reinterpret_cast<uintptr_t>(ws) & 255) != 0) return TP_ERR_INVALID_ARGUMENT;
  const ClipBwdLayout B = clip_bwd_layout(n);
  if (ws_bytes < B.total) return TP_ERR_WORKSPACE_TOO_SMALL;
  DeviceInfo dev;
  TP_TRY(device_info(&dev));
  return run_clip_embed_backward(w, static_cast<const uint8_t*>(embed_saved), *grads, static_cast<uint8_t*>(ws), B, n, dev.sms,
                                 static_cast<cudaStream_t>(stream), last_step);
}

}  // extern "C"
