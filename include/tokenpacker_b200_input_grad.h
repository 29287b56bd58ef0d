/* tokenpacker_b200 — gradients w.r.t. the CLIP features in the training path (libtokenpacker_b200.so).
 *
 * Companion of tokenpacker_b200.h, whose conventions, status codes, tp_weights and training entry points it uses.  Kept in a
 * header of its own so that tokenpacker_b200.h, ABI version 2, stays exactly as its consumers compiled it; this header only adds.
 */
#ifndef TOKENPACKER_B200_INPUT_GRAD_H_
#define TOKENPACKER_B200_INPUT_GRAD_H_

#include "tokenpacker_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* tp_backward, plus the gradients w.r.t. the projector's inputs: the CLIP features x0 (feat) and xm (feat_multi) of the
 * tp_forward_train call that filled ``saved``.  The reference's builder.py:107-137 is ordinary autograd, so these are what it
 * gives whenever the vision tower, a LoRA / adapter on it, or an attribution method asks for them.
 *   w, xm, xm_crop_stride, n_crops, scale_factor, hidden, grad_out, saved, grads, workspace
 *                 as for tp_backward; the parameter gradients written to ``grads`` are exactly (bit for bit) those of tp_backward,
 *                 and the workspace is the same size (tp_backward_workspace_bytes)
 *   d_x0          [n_crops, 576, 1024] bf16, contiguous, 16-byte aligned, or NULL (no x0 gradient).  Every element is written, zeros
 *                 included: the point-query stencil (builder.py:117-118) run backwards over dq = dy_q . W_q.  Given the same dq it
 *                 has exactly the bits of the reference's upsample_bilinear2d backward followed by the bf16 rounding of .float()'s
 *                 backward: odd s, dq at each window's centre token; even s, bf16(0.25 dq) on its centre 2x2; 0 elsewhere
 *   d_xm          [n_crops, 576, 4096] bf16, contiguous, 16-byte aligned, or NULL (no xm gradient):  dz_kv . [W_k0; W_v0], one
 *                 GEMM of the size of the forward's k/v_proj.0 GEMM
 *   packed        the tp_pack_weights_train (or tp_pack_weights) buffer of the same forward: [W_k0; W_v0] is read from it.  Required
 *                 only when d_xm is not NULL; may be NULL otherwise
 * Each gradient asked for adds one GEMM to a launch tp_backward already makes (and, for d_x0, one stencil kernel); with both NULL
 * the launches are exactly those of tp_backward.
 * TP_ERR_INVALID_ARGUMENT as tp_backward, and for d_xm without packed or a misaligned d_x0 / d_xm; TP_ERR_BAD_SCALE_FACTOR as
 * tp_backward.  All checks run before any CUDA call. */
TP_API int tp_backward_inputs(const tp_weights* w, const void* packed, const void* xm, int64_t xm_crop_stride, int64_t n_crops,
                              int scale_factor, int hidden, const void* grad_out, const void* saved, const tp_weights* grads,
                              void* d_x0, void* d_xm, void* workspace, size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TOKENPACKER_B200_INPUT_GRAD_H_ */
