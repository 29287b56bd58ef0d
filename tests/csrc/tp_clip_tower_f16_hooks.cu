// Test-only entry points into the fp16 CLIP tower (libtokenpacker_b200_clip_tower_f16_hooks.so, loaded by tests/test_clip_tower_f16_gpu.py
// and tests/test_clip_tower_f16_host.py; never by the package): the product translation unit plus the tpc_*_f16 functions below, which
// launch the same kernels and GEMM items tp_clip_tower_forward_f16 launches.  Conventions as in include/tokenpacker_b200.h.
#include "../../tokenpacker_b200/csrc/tp_api.cu"

extern "C" {

// Byte offsets inside the workspace of a tp_clip_tower_forward_f16 call over n crops (the bf16 tower's layout; f16 and bf16 elements
// are both 2 bytes): y1, qkv, ctx, x' (fp32), y2, h, in this order; out[6] = the workspace size.
TP_API int tpc_workspace_offsets_f16(int64_t n, int64_t* out) {
  if (n <= 0 || out == nullptr) return TP_ERR_INVALID_ARGUMENT;
  const ClipWorkLayout L = clip_work_layout(n);
  const size_t o[7] = {L.y1, L.qkv, L.ctx, L.xp, L.y2, L.h, L.total};
  for (int i = 0; i < 7; ++i) out[i] = static_cast<int64_t>(o[i]);
  return TP_OK;
}

// C[M, N] = epilogue(A[M, K] . B[N, K]^T) on the f16 instantiations (GemmEpilogue::f16): A, B, C f16; R f16, or fp32 with resid_f32;
// out_f32: C is fp32; alpha after the bias / residual / quick_gelu; seg_len != 0: C row r goes to row (r / seg_len) * seg_stride +
// r % seg_len (the patch GEMM's store).  mode: 0 = the engine's own choice, 1 = one-CTA 128 x 256 tiles, 2 = the pair kernel.
TP_API int tpc_gemm_f16(const void* a, int64_t lda, const void* b, int64_t ldb, void* c, int64_t ldc, int64_t m, int64_t n, int64_t k,
                        const float* bias, const void* resid, int64_t ldr, int resid_f32, int gelu, int out_f32, float alpha, int seg_len,
                        int seg_stride, int mode, void* stream_) {
  if (a == nullptr || b == nullptr || c == nullptr || mode < 0 || mode > 2) return TP_ERR_INVALID_ARGUMENT;
  DeviceInfo dev;
  TP_TRY(device_info(&dev));
  GemmItem it{AOperand{a, lda, 0, 0}, b, ldb, m, n, k, clip_epilogue(c, ldc, true)};
  it.ep.col_b = bias;
  it.ep.resid = resid;
  it.ep.ldr = ldr;
  it.ep.resid_f32 = resid_f32;
  it.ep.gelu = gelu;
  it.ep.out_f32 = out_f32;
  it.ep.alpha = alpha;
  it.ep.seg_len = seg_len;
  it.ep.seg_stride = seg_stride;
  TP_TRY(check_item(it));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (mode == 0) return launch_gemms(&it, 1, dev.sms, stream);
  if (mode == 2) return launch_gemm_pair_group(&it, 1, dev.sms, stream);
  if (n % 256 != 0) return TP_ERR_INVALID_ARGUMENT;
  CUtensorMap ma, mb;
  TP_TRY(make_one_cta_maps(it, 256, &ma, &mb));
  return launch_gemm_t<256>(it, ma, mb, dev.sms, stream);
}

// ctx [n * 577, 1024] = attention of f16 qkv [n * 577, 3072] (q already scaled by 1/8)
TP_API int tpc_attention_f16(const void* qkv, void* ctx, int64_t n, void* stream) {
  if (qkv == nullptr || ctx == nullptr || n <= 0) return TP_ERR_INVALID_ARGUMENT;
  DeviceInfo dev;
  TP_TRY(device_info(&dev));
  return launch_clip_attn(qkv, ctx, n, static_cast<cudaStream_t>(stream), true);
}

// Encoder layer ``layer`` of the fp16 tower alone (packed by tp_clip_tower_pack_weights_f16), exactly as tp_clip_tower_forward_f16 runs
// it: x [n * 577, 1024] -> x_out, every intermediate left in the workspace at tpc_workspace_offsets_f16's offsets.
TP_API int tpc_layer_f16(const void* packed, const tp_clip_tower_weights* w, int layer, const void* x, void* x_out, int64_t n, void* workspace,
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
                        stream, true);
}

// Status of a launch that mixes one bf16 and one f16 tower item (fc1 -> fc2 shapes, addresses that are never dereferenced): as a
// group (how = 0: launch_gemms), as a chain (1: launch_chain), and as one pair-kernel group (2: build_pair_group).  All three are
// refused before any CUDA call, so this runs without a GPU.
TP_API int tpc_mixed_precision(int how) {
  char* base = reinterpret_cast<char*>(static_cast<uintptr_t>(1) << 20);
  const long long M = 577 * 2;
  GemmItem items[2];
  items[0] = GemmItem{AOperand{base, kC, 0, 0}, base, kC, M, 4 * kC, kC, clip_epilogue(base + (1 << 24), 4 * kC, false)};
  items[0].ep.gelu = 2;
  items[1] = GemmItem{AOperand{base + (1 << 24), 4 * kC, 0, 0}, base, 4 * kC, M, kC, 4 * kC, clip_epilogue(base + (1 << 26), kC, true)};
  items[1].ep.resid = base;
  items[1].ep.ldr = kC;
  if (how == 0) return launch_gemms(items, 2, 132, nullptr);
  if (how == 1) {
    items[1].stage = 1;
    items[1].dep = 0;
    return launch_chain(items, 2, reinterpret_cast<int*>(base), 1 << 20, nullptr, 132, nullptr);
  }
  BuiltLaunch b;
  return build_pair_group(items, 2, 132, nullptr, &b);
}

// The embedding stage of tp_clip_tower_forward_f16 alone (run_clip_embed) up to step last_step, as tpc_embed (tp_clip_tower_hooks.cu):
// crops_dtype TP_CLIP_CROPS_BF16 (converted to f16 rows by im2col) or TP_CLIP_CROPS_F16 (read as they are); offsets from tpc_embed_offsets
TP_API int tpc_embed_f16(const void* packed, const tp_clip_tower_weights* w, const void* crops, int crops_dtype, int64_t n,
                         int64_t crop_stride, void* workspace, size_t workspace_bytes, int last_step, void* stream) {
  if (packed == nullptr || w == nullptr || !clip_weights_complete(w) || crops == nullptr || workspace == nullptr || n <= 0 ||
      (crops_dtype != TP_CLIP_CROPS_BF16 && crops_dtype != TP_CLIP_CROPS_F16) || crop_stride < 3ll * kClipImage * kClipImage ||
      last_step < 1 || last_step > 3)
    return TP_ERR_INVALID_ARGUMENT;
  const ClipWorkLayout WL = clip_work_layout(n);
  if (workspace_bytes < WL.total) return TP_ERR_WORKSPACE_TOO_SMALL;
  DeviceInfo dev;
  TP_TRY(device_info(&dev));
  return run_clip_embed(static_cast<const uint8_t*>(packed), w, crops, crops_dtype, n, crop_stride, static_cast<uint8_t*>(workspace), WL,
                        dev.sms, static_cast<cudaStream_t>(stream), true, nullptr, last_step);
}

}  // extern "C"
