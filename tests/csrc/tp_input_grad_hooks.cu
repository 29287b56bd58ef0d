// Test-only entry points into the input-gradient part of the backward (libtokenpacker_b200_input_grad_hooks.so, loaded by
// tests/test_input_grad_gpu.py; never by the package).  Like libtokenpacker_b200_testhooks.so, the library is the product
// translation unit plus the tpt_* functions below, which call the same launch functions tp_backward_inputs calls (tp_train.inl).
// Conventions as in include/tokenpacker_b200.h: device pointers, caller-owned buffers, work enqueued on ``stream``, a tp_status
// returned.
#include "../../tokenpacker_b200/csrc/tp_api.cu"

extern "C" {

// point-query stencil backwards: dx0 [n_crops * 576, 1024] (every element written) from dq [n_crops (24 / s)^2, 1024]
TP_API int tpt_point_query_bwd(const void* dq, void* dx0, int64_t n_crops, int s, void* stream) {
  if (s <= 0 || kGrid % s != 0) return TP_ERR_BAD_SCALE_FACTOR;
  if (dq == nullptr || dx0 == nullptr || n_crops <= 0) return TP_ERR_INVALID_ARGUMENT;
  return launch_front_bwd_s(s, static_cast<const __nv_bfloat16*>(dq), static_cast<__nv_bfloat16*>(dx0), n_crops * kTokens,
                            static_cast<cudaStream_t>(stream));
}

// Workspace layout of tp_backward / tp_backward_inputs for (n_crops, s, hidden): out[0..2] = byte offsets of dzkv (dz_kv [R, 2048]
// at the end of the backward), dqh (dq [Q, 1024] at the end, when d_x0 was asked for) and dyq (dy_q [Q, 1024]); out[3] = total.
TP_API int tpt_bwd_layout(int64_t n_crops, int s, int hidden, int64_t* out) {
  if (out == nullptr || n_crops <= 0 || s <= 0 || kGrid % s != 0 || !valid_hidden(hidden)) return TP_ERR_INVALID_ARGUMENT;
  const BwdLayout L = bwd_layout(n_crops, s, hidden);
  out[0] = static_cast<int64_t>(L.dzkv);
  out[1] = static_cast<int64_t>(L.dqh);
  out[2] = static_cast<int64_t>(L.dyq);
  out[3] = static_cast<int64_t>(L.total);
  return TP_OK;
}

}  // extern "C"
