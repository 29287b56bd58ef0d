// Test-only entry points into the CLIP tower's kernels (libtokenpacker_b200_clip_tower_hooks.so, loaded by
// tests/test_clip_tower_gpu.py; never by the package): the product translation unit plus the tpc_* functions below, which launch the
// same kernels and GEMM items tp_clip_tower_forward launches.  Conventions as in include/tokenpacker_b200.h.
#include "../../tokenpacker_b200/csrc/tp_api.cu"

extern "C" {

// C[M, N] = epilogue(A[M, K] . B[N, K]^T) with the tower's epilogue: bias (fp32, may be NULL), residual R [M, ldr] (NULL: none),
// gelu 0 / 2 (quick_gelu).  mode: 0 = the engine's own choice, 1 = one-CTA 128 x 256 tiles, 2 = the pair kernel.
TP_API int tpc_gemm(const void* a, int64_t lda, const void* b, int64_t ldb, void* c, int64_t ldc, int64_t m, int64_t n, int64_t k,
                    const float* bias, const void* resid, int64_t ldr, int gelu, int mode, void* stream_) {
  if (a == nullptr || b == nullptr || c == nullptr || mode < 0 || mode > 2) return TP_ERR_INVALID_ARGUMENT;
  DeviceInfo dev;
  TP_TRY(device_info(&dev));
  GemmItem it{AOperand{a, lda, 0, 0}, b, ldb, m, n, k, clip_epilogue(c, ldc)};
  it.ep.col_b = bias;
  it.ep.resid = static_cast<const __nv_bfloat16*>(resid);
  it.ep.ldr = ldr;
  it.ep.gelu = gelu;
  TP_TRY(check_item(it));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (mode == 0) return launch_gemms(&it, 1, dev.sms, stream);
  if (mode == 2) return launch_gemm_pair_group(&it, 1, dev.sms, stream);
  if (n % 256 != 0) return TP_ERR_INVALID_ARGUMENT;
  CUtensorMap ma, mb;
  TP_TRY(make_one_cta_maps(it, 256, &ma, &mb));
  return launch_gemm_t<256>(it, ma, mb, dev.sms, stream);
}

// ctx [n * 577, 1024] = attention of qkv [n * 577, 3072] (q pre-scaled), the kernel tp_clip_tower_forward runs in every layer
TP_API int tpc_attention(const void* qkv, void* ctx, int64_t n, void* stream) {
  if (qkv == nullptr || ctx == nullptr || n <= 0) return TP_ERR_INVALID_ARGUMENT;
  DeviceInfo dev;
  TP_TRY(device_info(&dev));
  return launch_clip_attn(qkv, ctx, n, static_cast<cudaStream_t>(stream));
}

// Byte offsets inside the workspace of a tp_clip_tower_forward call over n crops: y1 (layer_norm1 out), qkv, ctx, x' (after the
// attention residual), y2 (layer_norm2 out), h (quick_gelu(fc1)), in this order; out[6] = the workspace size.
TP_API int tpc_workspace_offsets(int64_t n, int64_t* out) {
  if (n <= 0 || out == nullptr) return TP_ERR_INVALID_ARGUMENT;
  const ClipWorkLayout L = clip_work_layout(n);
  const size_t o[7] = {L.y1, L.qkv, L.ctx, L.xp, L.y2, L.h, L.total};
  for (int i = 0; i < 7; ++i) out[i] = static_cast<int64_t>(o[i]);
  return TP_OK;
}

// Encoder layer ``layer`` alone, exactly as tp_clip_tower_forward runs it: x [n * 577, 1024] -> x_out, every intermediate left in the
// workspace at the offsets above.
TP_API int tpc_layer(const void* packed, const tp_clip_tower_weights* w, int layer, const void* x, void* x_out, int64_t n, void* workspace,
                     size_t workspace_bytes, void* stream_) {
  if (packed == nullptr || w == nullptr || !clip_weights_complete(w) || x == nullptr || x_out == nullptr || workspace == nullptr || n <= 0 ||
      layer < 0 || layer >= TP_CLIP_TOWER_LAYERS)
    return TP_ERR_INVALID_ARGUMENT;
  const ClipWorkLayout WL = clip_work_layout(n);
  if (workspace_bytes < WL.total) return TP_ERR_WORKSPACE_TOO_SMALL;
  DeviceInfo dev;
  TP_TRY(device_info(&dev));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  uint8_t* W = static_cast<uint8_t*>(workspace);
  int* flags = reinterpret_cast<int*>(W + WL.flags);
  TP_CUDA(cudaMemsetAsync(flags, 0, static_cast<size_t>(WL.flags_per_layer) * 4, stream));
  return run_clip_layer(static_cast<const uint8_t*>(packed), w, layer, x, x_out, W, WL, n, flags, dev.sms, stream);
}

}  // extern "C"
