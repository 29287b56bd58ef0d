// Test-only entry points into the kernels of the CLIP tower's training path (libtokenpacker_b200_clip_tower_train_hooks.so, loaded by
// tests/test_clip_tower_train_gpu.py; never by the package): the product translation unit plus the tptt_* functions below, which
// launch the same kernels tp_clip_tower_forward_train and tp_clip_tower_backward launch.  Conventions as in include/tokenpacker_b200.h.
#include "../../tokenpacker_b200/csrc/tp_api.cu"

extern "C" {

// the forward attention with its softmax statistics: ctx [n * 577, 1024], lse fp32 [n, 16, 640] (tokens >= 577 not written)
TP_API int tptt_attention_lse(const void* qkv, void* ctx, float* lse, int64_t n, void* stream) {
  if (qkv == nullptr || ctx == nullptr || lse == nullptr || n <= 0) return TP_ERR_INVALID_ARGUMENT;
  DeviceInfo dev;
  TP_TRY(device_info(&dev));
  return launch_clip_attn(qkv, ctx, n, static_cast<cudaStream_t>(stream), false, lse);
}

// dqkv [n * 577, 3072] = the attention backward of dctx; delta: fp32 [n, 16, 640] scratch (D is left there)
TP_API int tptt_attention_bwd(const void* qkv, const float* lse, const void* ctx, const void* dctx, float* delta, void* dqkv, int64_t n,
                              void* stream) {
  if (qkv == nullptr || lse == nullptr || ctx == nullptr || dctx == nullptr || delta == nullptr || dqkv == nullptr || n <= 0)
    return TP_ERR_INVALID_ARGUMENT;
  DeviceInfo dev;
  TP_TRY(device_info(&dev));
  return launch_clip_attn_bwd(qkv, lse, ctx, dctx, delta, dqkv, n, static_cast<cudaStream_t>(stream));
}

// dh [rows, 4096] *= quick_gelu'(z) in place, db [4096] = its column sums; col_part: fp32 [592 * 4096] scratch
TP_API int tptt_quick_gelu_bwd(void* dh, const void* z, int64_t rows, void* db, float* col_part, void* stream) {
  if (dh == nullptr || z == nullptr || db == nullptr || col_part == nullptr || rows <= 0) return TP_ERR_INVALID_ARGUMENT;
  return quick_gelu_bwd_bias(static_cast<__nv_bfloat16*>(dh), static_cast<const __nv_bfloat16*>(z), rows, db, col_part,
                             static_cast<cudaStream_t>(stream));
}

// carry32 += dLN(g) (+ add), carry16 = bf16(carry32), dgamma / dbeta / dsum [1024]; x_f32: x is fp32 (layer_norm2) or bf16 (layer_norm1);
// partial: fp32 [296 * 3 * 1024] scratch
TP_API int tptt_ln_bwd(const void* g, const void* x, int x_f32, const void* gamma, const void* add, float* carry32, void* carry16,
                       float* partial, int64_t rows, void* dgamma, void* dbeta, void* dsum, void* stream_) {
  if (g == nullptr || x == nullptr || gamma == nullptr || carry32 == nullptr || carry16 == nullptr || partial == nullptr || rows <= 0 ||
      dgamma == nullptr || dbeta == nullptr || dsum == nullptr)
    return TP_ERR_INVALID_ARGUMENT;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (x_f32) return launch_clip_ln_bwd<float>(g, x, gamma, add, carry32, carry16, partial, rows, dgamma, dbeta, dsum, nullptr, stream);
  return launch_clip_ln_bwd<__nv_bfloat16>(g, x, gamma, add, carry32, carry16, partial, rows, dgamma, dbeta, dsum, nullptr, stream);
}

// Byte offsets inside one layer's saved set of a tp_clip_tower_forward_train call over n crops: pack, x, y1, qkv, lse, ctx, x', y2, z, h;
// out[10] = the bytes of one set; out[11] = the offset of the q|k|v weight inside pack
TP_API int tptt_saved_offsets(int64_t n, int64_t* out) {
  if (n <= 0 || out == nullptr) return TP_ERR_INVALID_ARGUMENT;
  const ClipSavedLayout L = clip_saved_layout(n);
  const size_t o[12] = {L.pack, L.x, L.y1, L.qkv, L.lse, L.ctx, L.xp, L.y2, L.z, L.h, L.layer_bytes, clip_packed_layout().w_qkv};
  for (int i = 0; i < 12; ++i) out[i] = static_cast<int64_t>(o[i]);
  return TP_OK;
}

// Byte offsets inside a tp_clip_tower_backward workspace over n crops: carry32, carry16, dh, g, delta, ln_part, col_part, splitk,
// unused_grad; out[9] = its total size
TP_API int tptt_bwd_offsets(int64_t n, int64_t* out) {
  if (n <= 0 || out == nullptr) return TP_ERR_INVALID_ARGUMENT;
  const ClipBwdLayout B = clip_bwd_layout(n);
  const size_t o[10] = {B.carry32, B.carry16, B.dh, B.g, B.delta, B.ln_part, B.col_part, B.splitk, B.unused_grad, B.total};
  for (int i = 0; i < 10; ++i) out[i] = static_cast<int64_t>(o[i]);
  return TP_OK;
}

// The backward of encoder layer `layer` alone (run_clip_layer_backward, as tp_clip_tower_backward runs it), from its saved set
// `saved_set` of a tp_clip_tower_forward_train call over n crops, up to step last_step (1 .. 8, the numbering of
// tp_clip_tower_train.inl).  The carry is NOT initialised: the caller writes carry32 and carry16 = bf16(carry32) into ws, so a test can
// start from fp32 values bf16 cannot represent.  d_x: the caller's gradient of the layer's input hidden state (or NULL).
TP_API int tptt_layer_backward(const tp_clip_tower_weights* w, int layer, const void* saved_set, int64_t n, const void* d_x,
                               const tp_clip_tower_layer_grads* grads, void* ws, size_t ws_bytes, int last_step, void* stream) {
  if (w == nullptr || saved_set == nullptr || grads == nullptr || ws == nullptr || n <= 0 || layer < 0 || layer >= TP_CLIP_TOWER_LAYERS ||
      last_step < 1 || last_step > 8 || !clip_weights_complete(w))
    return TP_ERR_INVALID_ARGUMENT;
  if ((reinterpret_cast<uintptr_t>(saved_set) & 255) != 0 || (reinterpret_cast<uintptr_t>(ws) & 255) != 0) return TP_ERR_INVALID_ARGUMENT;
  const ClipBwdLayout B = clip_bwd_layout(n);
  if (ws_bytes < B.total) return TP_ERR_WORKSPACE_TOO_SMALL;
  DeviceInfo dev;
  TP_TRY(device_info(&dev));
  return run_clip_layer_backward(w->layers[layer], static_cast<const uint8_t*>(saved_set), clip_saved_layout(n), d_x, *grads,
                                 static_cast<uint8_t*>(ws), B, n, dev.sms, static_cast<cudaStream_t>(stream), last_step);
}

// z = bf16(z32), h = bf16(quick_gelu(z32)) over n elements (a multiple of 8): the training forward's clip_quick_gelu_fwd_kernel launch
TP_API int tptt_quick_gelu_fwd(const float* z32, void* z, void* h, int64_t n, void* stream) {
  if (z32 == nullptr || z == nullptr || h == nullptr || n <= 0 || n % 8 != 0) return TP_ERR_INVALID_ARGUMENT;
  return launch_clip_quick_gelu_fwd(z32, z, h, n, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
