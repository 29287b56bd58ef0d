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

}  // extern "C"
