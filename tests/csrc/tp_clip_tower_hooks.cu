// Test-only entry points into the CLIP tower's kernels (libtokenpacker_b200_clip_tower_hooks.so, loaded by
// tests/test_clip_tower_gpu.py and tests/test_clip_tower_forward_stages_gpu.py; never by the package): the product translation unit plus
// the tpc_* functions below, which launch the same kernels and GEMM items tp_clip_tower_forward launches.  Conventions as in
// include/tokenpacker_b200.h.
#include "../../tokenpacker_b200/csrc/tp_api.cu"

extern "C" {

// C[M, N] = epilogue(A[M, K] . B[N, K]^T) with the tower's epilogue: bias (fp32, may be NULL), residual R [M, ldr] (NULL: none; bf16,
// or fp32 with resid_f32: the tower's mid-layer residual x'), gelu 0 / 2 (quick_gelu).  mode: 0 = the engine's own choice, 1 = one-CTA
// 128 x 256 tiles, 2 = the pair kernel.
TP_API int tpc_gemm_resid(const void* a, int64_t lda, const void* b, int64_t ldb, void* c, int64_t ldc, int64_t m, int64_t n, int64_t k,
                          const float* bias, const void* resid, int64_t ldr, int resid_f32, int gelu, int mode, void* stream_) {
  if (a == nullptr || b == nullptr || c == nullptr || mode < 0 || mode > 2) return TP_ERR_INVALID_ARGUMENT;
  DeviceInfo dev;
  TP_TRY(device_info(&dev));
  GemmItem it{AOperand{a, lda, 0, 0}, b, ldb, m, n, k, clip_epilogue(c, ldc)};
  it.ep.col_b = bias;
  it.ep.resid = resid;
  it.ep.ldr = ldr;
  it.ep.resid_f32 = resid_f32;
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

// tpc_gemm_resid with a bf16 residual
TP_API int tpc_gemm(const void* a, int64_t lda, const void* b, int64_t ldb, void* c, int64_t ldc, int64_t m, int64_t n, int64_t k,
                    const float* bias, const void* resid, int64_t ldr, int gelu, int mode, void* stream) {
  return tpc_gemm_resid(a, lda, b, ldb, c, ldc, m, n, k, bias, resid, ldr, 0, gelu, mode, stream);
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
  const ClipPackedLayout PL = clip_packed_layout();
  return run_clip_layer(static_cast<const uint8_t*>(packed) + PL.layer0 + layer * PL.layer_bytes, w, layer, x, x_out, W, WL, n, flags, dev.sms,
                        stream);
}

// Byte offsets inside the workspace of a tp_clip_tower_forward(_f16) call over n crops for the embedding stage: h (the im2col patch rows,
// [576 n, 592]), xa (hidden_states[0], [577 n, 1024]); out[2] = the workspace size.
TP_API int tpc_embed_offsets(int64_t n, int64_t* out) {
  if (n <= 0 || out == nullptr) return TP_ERR_INVALID_ARGUMENT;
  const ClipWorkLayout L = clip_work_layout(n);
  const size_t o[3] = {L.h, L.xa, L.total};
  for (int i = 0; i < 3; ++i) out[i] = static_cast<int64_t>(o[i]);
  return TP_OK;
}

// The embedding stage of tp_clip_tower_forward alone (run_clip_embed) up to step last_step (1 = im2col, 2 = + the patch GEMM, 3 = +
// embeddings and pre_layrnorm), on the caller's workspace.  crops_dtype and crop_stride as in the C ABI (bf16 crops only here).
TP_API int tpc_embed(const void* packed, const tp_clip_tower_weights* w, const void* crops, int crops_dtype, int64_t n, int64_t crop_stride,
                     void* workspace, size_t workspace_bytes, int last_step, void* stream) {
  if (packed == nullptr || w == nullptr || !clip_weights_complete(w) || crops == nullptr || workspace == nullptr || n <= 0 ||
      crops_dtype != TP_CLIP_CROPS_BF16 || crop_stride < 3ll * kClipImage * kClipImage || last_step < 1 || last_step > 3)
    return TP_ERR_INVALID_ARGUMENT;
  const ClipWorkLayout WL = clip_work_layout(n);
  if (workspace_bytes < WL.total) return TP_ERR_WORKSPACE_TOO_SMALL;
  DeviceInfo dev;
  TP_TRY(device_info(&dev));
  return run_clip_embed(static_cast<const uint8_t*>(packed), w, crops, crops_dtype, n, crop_stride, static_cast<uint8_t*>(workspace), WL,
                        dev.sms, static_cast<cudaStream_t>(stream), false, nullptr, last_step);
}

// y [rows, 1024] = LayerNorm(x) gamma + beta, the tower's launch_clip_ln: x_kind 0 = x has the storage type, 1 = x is fp32; f16 = 0: bf16
// storage (layer_norm1: bf16 -> bf16, layer_norm2: fp32 -> bf16), 1: f16 storage (f16 -> f16, fp32 -> f16)
TP_API int tpc_layernorm(const void* x, int x_kind, int64_t rows, const void* gamma, const void* beta, void* y, int f16, void* stream_) {
  if (x == nullptr || gamma == nullptr || beta == nullptr || y == nullptr || rows <= 0 || (x_kind != 0 && x_kind != 1) || (f16 != 0 && f16 != 1))
    return TP_ERR_INVALID_ARGUMENT;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (f16) return x_kind ? launch_clip_ln<float, __half>(x, rows, gamma, beta, y, stream) : launch_clip_ln<__half, __half>(x, rows, gamma, beta, y, stream);
  return x_kind ? launch_clip_ln<float>(x, rows, gamma, beta, y, stream) : launch_clip_ln<__nv_bfloat16>(x, rows, gamma, beta, y, stream);
}

// The fields of the packed derived weights' layout (tp_clip_tower_pack_weights / _f16), in bytes: patch_w, layer0, layer_bytes, and
// inside a layer's block w_qkv, b_qkv, b_o, b_fc1, b_fc2; out[8] = the total
TP_API int tpc_packed_layout(int64_t* out) {
  if (out == nullptr) return TP_ERR_INVALID_ARGUMENT;
  const ClipPackedLayout L = clip_packed_layout();
  const size_t o[9] = {L.patch_w, L.layer0, L.layer_bytes, L.w_qkv, L.b_qkv, L.b_o, L.b_fc1, L.b_fc2, L.total};
  for (int i = 0; i < 9; ++i) out[i] = static_cast<int64_t>(o[i]);
  return TP_OK;
}

}  // extern "C"
