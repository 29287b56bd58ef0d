// Test-only entry points into the backward's internal kernels and the forward's buffer layouts (libtokenpacker_b200_testhooks.so,
// loaded by tests/test_train_kernels_gpu.py, tests/test_forward_stages_gpu.py and tests/test_train_stages_gpu.py; never by the
// package).  The library is the product translation unit plus the tpt_* functions
// below, which call the same launch functions tp_backward calls (tp_train.inl), so every kernel runs with the launch configuration
// of a training step.  Conventions as in include/tokenpacker_b200.h: device pointers, caller-owned buffers, work enqueued on
// ``stream``, a tp_status returned.
#include "../../tokenpacker_b200/csrc/tp_api.cu"

extern "C" {

// Kernels launched by this library (its own counter: the product library keeps another).
TP_API uint64_t tpt_launch_count(void) { return g_launch_count.load(std::memory_order_relaxed); }

// out[0..3] = LayerNorm-backward CTAs, column-sum row chunks, split-K slices of tp_backward, fewest rows that take split-K there.
TP_API int tpt_constants(int64_t* out) {
  if (out == nullptr) return TP_ERR_INVALID_ARGUMENT;
  out[0] = kLnBlocks;
  out[1] = kColChunks;
  out[2] = kWgradSplits;
  out[3] = 64ll * kBlockK * kWgradSplits;
  return TP_OK;
}

// partial[s][n_out, n_in] (fp32) = slice s of dY^T X over rows (dY: [rows, n_out], X: [rows, n_in]), one TN item with k_splits =
// splits.  d_a != NULL: launched in one group with the NN dgrad item  d_c[d_rows, d_n_in] = d_alpha * d_a . d_w  (d_w: [d_n_out,
// d_n_in] as stored), split-K item first, as tp_backward groups them.
TP_API int tpt_wgrad_splitk(const void* dy, int64_t ld_dy, const void* x, int64_t ld_x, int64_t rows, int n_out, int n_in, int splits,
                            float* partial, size_t partial_floats, const void* d_a, int64_t ld_da, const void* d_w, int64_t ld_dw, void* d_c,
                            int64_t ld_dc, int64_t d_rows, int d_n_in, int d_n_out, float d_alpha, void* stream) {
  if (dy == nullptr || x == nullptr || partial == nullptr || rows <= 0 || n_out <= 0 || n_in <= 0 || splits < 2) return TP_ERR_INVALID_ARGUMENT;
  if (partial_floats < static_cast<size_t>(splits) * n_out * n_in) return TP_ERR_WORKSPACE_TOO_SMALL;
  if (d_a != nullptr && (d_w == nullptr || d_c == nullptr || d_n_in % 256 != 0)) return TP_ERR_INVALID_ARGUMENT;
  DeviceInfo dev;
  TP_TRY(device_info(&dev));
  GemmItem gi[2];
  int n = 0;
  gi[n++] = wgrad_split(dy, ld_dy, x, ld_x, rows, n_out, n_in, splits, partial);
  if (d_a != nullptr) gi[n++] = dgrad_nn_item(d_a, ld_da, d_w, ld_dw, d_c, ld_dc, d_rows, d_n_in, d_n_out, d_alpha);
  return launch_gemms(gi, n, dev.sms, static_cast<cudaStream_t>(stream));
}

// out[i] = bf16(alpha * sum_s partial[s * elems + i])
TP_API int tpt_splitk_reduce(const float* partial, int splits, int64_t elems, float alpha, void* out, void* stream) {
  if (partial == nullptr || out == nullptr || splits < 1 || elems <= 0 || elems % 4 != 0) return TP_ERR_INVALID_ARGUMENT;
  return wgrad_reduce(partial, splits, elems, alpha, out, static_cast<cudaStream_t>(stream));
}

// LayerNorm backward (1024 wide) of rows rows: dy, and dgamma / dbeta / dbias (dbias may be NULL) through caller-owned partials
TP_API int tpt_ln_bwd(const void* g, const void* y, const float* stats, const void* gamma, void* dy, float* partial, size_t partial_floats,
                      int64_t rows, void* dgamma, void* dbeta, void* dbias, void* stream) {
  if (g == nullptr || y == nullptr || stats == nullptr || gamma == nullptr || dy == nullptr || partial == nullptr || dgamma == nullptr ||
      dbeta == nullptr || rows <= 0)
    return TP_ERR_INVALID_ARGUMENT;
  if (partial_floats < 3ull * kLnBlocks * kC) return TP_ERR_WORKSPACE_TOO_SMALL;
  return launch_ln_bwd(g, y, stats, gamma, dy, partial, rows, dgamma, dbeta, dbias, static_cast<cudaStream_t>(stream));
}

TP_API int tpt_ln_apply(const void* y, const float* stats, const void* gamma, const void* beta, void* out, int64_t rows, void* stream) {
  if (y == nullptr || stats == nullptr || gamma == nullptr || beta == nullptr || out == nullptr || rows <= 0) return TP_ERR_INVALID_ARGUMENT;
  return ln_apply(static_cast<const __nv_bfloat16*>(y), stats, gamma, beta, static_cast<__nv_bfloat16*>(out), rows, static_cast<cudaStream_t>(stream));
}

// window-attention backward of the first n_queries queries (crops of 576 key/value rows, 24 / s x 24 / s queries per crop)
TP_API int tpt_window_attn_bwd(const void* qp, const void* kp, const void* vp, const void* dctx, void* dqp, void* dkp, void* dvp, int64_t n_queries,
                               int s, void* stream) {
  if (s <= 0 || kGrid % s != 0) return TP_ERR_BAD_SCALE_FACTOR;
  if (qp == nullptr || kp == nullptr || vp == nullptr || dctx == nullptr || dqp == nullptr || dkp == nullptr || dvp == nullptr || n_queries <= 0)
    return TP_ERR_INVALID_ARGUMENT;
  auto b = [](const void* p) { return static_cast<const __nv_bfloat16*>(p); };
  auto m = [](void* p) { return static_cast<__nv_bfloat16*>(p); };
  return launch_attn_bwd_s(s, b(qp), b(kp), b(vp), b(dctx), m(dqp), m(dkp), m(dvp), n_queries, static_cast<cudaStream_t>(stream));
}

TP_API int tpt_gelu_fwd(const void* z, void* h, int64_t elems, void* stream) {
  if (z == nullptr || h == nullptr || elems <= 0 || elems % 8 != 0) return TP_ERR_INVALID_ARGUMENT;
  return launch_gelu_fwd(z, h, static_cast<size_t>(elems), static_cast<cudaStream_t>(stream));
}

// dh <- dh GELU'(z) in place, out (and out_hi, if not NULL: columns [cols/2, cols)) = column sums of the stored result
TP_API int tpt_gelu_bwd_bias(void* dh, const void* z, int64_t ld, int64_t rows, int cols, void* out, void* out_hi, float* partial,
                             size_t partial_floats, void* stream) {
  if (dh == nullptr || z == nullptr || out == nullptr || partial == nullptr || rows <= 0 || cols <= 0 || ld % 8 != 0) return TP_ERR_INVALID_ARGUMENT;
  return gelu_bwd_bias(static_cast<__nv_bfloat16*>(dh), static_cast<const __nv_bfloat16*>(z), ld, rows, cols, out, out_hi, partial, partial_floats,
                       static_cast<cudaStream_t>(stream));
}

// out[c] = bf16(scale * sum_r in[r, c])
TP_API int tpt_colsum(const void* in, int64_t ld, int64_t rows, int cols, float scale, float* partial, size_t partial_floats, void* out,
                      void* stream) {
  if (in == nullptr || out == nullptr || partial == nullptr || rows <= 0 || cols <= 0 || ld % 8 != 0) return TP_ERR_INVALID_ARGUMENT;
  return bias_grad(in, ld, rows, cols, scale, out, partial, partial_floats, static_cast<cudaStream_t>(stream));
}

// Workspace layout of tp_forward for (n_crops, s, hidden), so that a test reads each stage's output where the forward put it:
// out[2 i], out[2 i + 1] = byte offset and byte size of region i in WorkLayout order (h_kv, y_k, y_v, k_p, v_p, stats, q, y_q, q_p,
// ctx, h_m, flags); out[24] = total.  The sizes are the regions' shapes (WorkLayout's comments); the gaps up to the next offset are
// alignment padding that nothing writes.
TP_API int tpt_work_layout(int64_t n_crops, int s, int hidden, int64_t* out) {
  if (out == nullptr || n_crops <= 0 || s <= 0 || kGrid % s != 0 || !valid_hidden(hidden)) return TP_ERR_INVALID_ARGUMENT;
  const WorkLayout L = work_layout(n_crops, s, hidden);
  const long long R = n_crops * kTokens, Q = n_crops * (kGrid / s) * (kGrid / s);
  const size_t off[12] = {L.h_kv, L.y_k, L.y_v, L.k_p, L.v_p, L.stats, L.q, L.y_q, L.q_p, L.ctx, L.h_m, L.flags};
  const long long bytes[12] = {R * 2 * kC * 2, R * kC * 2, R * kC * 2, R * kC * 2, R * kC * 2, (2 * R + Q) * kStatSlots * 2 * 4,
                               Q * kC * 2, Q * kC * 2, Q * kC * 2, Q * kC * 2, Q * hidden * 2, L.n_flags * 4};
  for (int i = 0; i < 12; ++i) {
    out[2 * i] = static_cast<int64_t>(off[i]);
    out[2 * i + 1] = bytes[i];
  }
  out[24] = static_cast<int64_t>(L.total);
  return TP_OK;
}

// Buffer layouts of the training step for (n_crops, s, hidden), so that a test reads every activation tp_forward_train saves and
// every intermediate tp_backward forms where they were put: out[2 i], out[2 i + 1] = byte offset and byte size of region i, first
// the 14 SavedLayout regions of ``saved`` (z_kv, h_kv, y_k, y_v, stats, k_p, v_p, q, y_q, q_p, ctx, o, z_m, h_m), then the 22
// BwdLayout regions of the backward workspace (w_m2t, g_t, hm_t, dzm, d_o, dctx, dqp, dkp, dvp, lnq_t, lnk_t, lnv_t, dqh, dkh, dvh,
// dyq, dyk, dyv, dzkv, ln_part, col_part, splitk); out[72] = the saved total, out[73] = the workspace total.  A region the
// configuration does not allocate (the transposing fallback's scratch when hidden % 256 == 0) has size 0.  The sizes are the
// regions' shapes (the layouts' comments); the gaps up to the next offset are alignment padding that nothing writes.
TP_API int tpt_train_layout(int64_t n_crops, int s, int hidden, int64_t* out) {
  if (out == nullptr || n_crops <= 0 || s <= 0 || kGrid % s != 0 || !valid_hidden(hidden)) return TP_ERR_INVALID_ARGUMENT;
  const SavedLayout S = saved_layout(n_crops, s, hidden);
  const BwdLayout B = bwd_layout(n_crops, s, hidden);
  const long long R = n_crops * kTokens, Q = n_crops * (kGrid / s) * (kGrid / s), H = hidden;
  const long long act = R * kC * 2, qry = Q * kC * 2, fb = (H % 256 != 0) ? H * B.Qp * 2 : 0;
  const size_t off[36] = {S.z_kv, S.h_kv, S.y_k, S.y_v, S.stats, S.k_p, S.v_p, S.q, S.y_q, S.q_p, S.ctx, S.o, S.z_m, S.h_m,
                          B.w_m2t, B.g_t, B.hm_t, B.dzm, B.d_o, B.dctx, B.dqp, B.dkp, B.dvp, B.lnq_t, B.lnk_t, B.lnv_t, B.dqh, B.dkh,
                          B.dvh, B.dyq, B.dyk, B.dyv, B.dzkv, B.ln_part, B.col_part, B.splitk};
  const long long bytes[36] = {2 * act, 2 * act, act, act, (2 * R + Q) * kStatSlots * 2 * 4, act, act, qry, qry, qry, qry, qry, Q * H * 2,
                               Q * H * 2,
                               (H % 256 != 0) ? H * H * 2 : 0, fb, fb, Q * H * 2, qry, qry, qry, act, act, qry, act, act, qry, act, act,
                               qry, act, act, 2 * act, 3ll * kLnBlocks * 3 * kC * 4, static_cast<long long>(kColChunks) * (H > 2048 ? H : 2048) * 4,
                               2ll * kWgradSplits * kC * kC * 4};
  for (int i = 0; i < 36; ++i) {
    out[2 * i] = static_cast<int64_t>(off[i]);
    out[2 * i + 1] = bytes[i];
  }
  out[72] = static_cast<int64_t>(S.total);
  out[73] = static_cast<int64_t>(B.total);
  return TP_OK;
}

// Packed-weight layout of tp_pack_weights for hidden: every PackedLayout byte offset in declaration order (w_kv0, b_kv0, w_k2, b_k2,
// w_v2, b_v2, w_ik, wsum_k, c_k, w_iv, wsum_v, c_v, w_q, w_iq, wsum_q, c_q, w_ot, w_om, b_om, w_m2, b_m2, w_o, b_o, w_m0, b_m0), then
// the total: 26 values.
TP_API int tpt_packed_layout(int hidden, int64_t* out) {
  if (out == nullptr || !valid_hidden(hidden)) return TP_ERR_INVALID_ARGUMENT;
  const PackedLayout L = packed_layout(hidden);
  const size_t f[26] = {L.w_kv0, L.b_kv0, L.w_k2, L.b_k2, L.w_v2, L.b_v2, L.w_ik, L.wsum_k, L.c_k, L.w_iv, L.wsum_v, L.c_v, L.w_q,
                        L.w_iq, L.wsum_q, L.c_q, L.w_ot, L.w_om, L.b_om, L.w_m2, L.b_m2, L.w_o, L.b_o, L.w_m0, L.b_m0, L.total};
  for (int i = 0; i < 26; ++i) out[i] = static_cast<int64_t>(f[i]);
  return TP_OK;
}

// out[c, r] = in[r, c]
TP_API int tpt_transpose(const void* in, int64_t ld_in, void* out, int64_t ld_out, int64_t rows, int cols, void* stream) {
  if (in == nullptr || out == nullptr || rows <= 0 || cols <= 0 || ld_in < cols || ld_out < rows) return TP_ERR_INVALID_ARGUMENT;
  return launch_transpose(in, ld_in, out, ld_out, rows, cols, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
