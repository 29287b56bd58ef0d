/* tokenpacker_b200 — C ABI of the H100 (sm_90a) TokenPacker hot path (libtokenpacker_b200.so).
 *
 * The reference (CircleRadon/TokenPacker) is pure Python and has no FFI of its own: its boundary for this path is
 * the nn.Module ``TokenPacker`` (llava/model/multimodal_projector/builder.py:39-137) plus the HD front end
 * (llava/patch_divide.py:71-105, llava/train/train.py:695-731, llava/model/llava_arch.py:139-155).  This header is
 * the seam a maintainer binds instead (ctypes stub in INTEGRATION.md); each entry point cites what it replaces.
 *
 * Conventions
 *   - plain pointers and sizes only; no torch / C++ types cross the ABI
 *   - every buffer is owned by the caller; the library allocates nothing that outlives a call
 *   - device pointers unless the name says "host"; bf16 storage, fp32 accumulation
 *   - every function returns a tp_status (0 = ok) and never throws, exits or synchronises the device
 *     (except the *_host helpers, which synchronise their own stream before returning)
 *   - work is enqueued on the ``stream`` argument (a cudaStream_t passed as void*); re-entrant, no global state
 */
#ifndef TOKENPACKER_B200_H_
#define TOKENPACKER_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TP_ABI_VERSION 2

#if defined(__GNUC__)
#define TP_API __attribute__((visibility("default")))
#else
#define TP_API
#endif

typedef enum tp_status {
  TP_OK = 0,
  TP_ERR_INVALID_ARGUMENT = 1, /* null pointer, bad shape, hidden size not a multiple of 32 ... */
  TP_ERR_BAD_SCALE_FACTOR = 2, /* 24 % scale_factor != 0  (reference: ValueError, builder.py:51-52) */
  TP_ERR_WORKSPACE_TOO_SMALL = 3,
  TP_ERR_CUDA = 4,             /* a CUDA runtime / driver call failed; see tp_last_cuda_error() */
  TP_ERR_UNSUPPORTED_DEVICE = 5, /* not a compute-capability 9.x device */
  TP_ERR_BAD_PATCH_NUM = 6     /* patch_num not in {9,16,25} (reference: NotImplementedError, patch_divide.py:79-80) */
} tp_status;

TP_API const char* tp_strerror(int status);
TP_API int tp_abi_version(void);
/* Name of the last failing CUDA call on this thread ("" if none); diagnostic only. */
TP_API const char* tp_last_cuda_error(void);
/* Number of kernels this library has launched so far, over all host threads of the process (diagnostic: the benchmark's gpu_launches). */
TP_API uint64_t tp_launch_count(void);

/* ---------------------------------------------------------------------------------------------------------------
 * Parameters.  Raw module parameters exactly as the reference state_dict holds them (builder.py:59-83), bf16,
 * row-major [out, in], on the device.  Replaces: TokenPacker.__init__ / load_state_dict (llava_arch.py:78-83).
 * ------------------------------------------------------------------------------------------------------------- */
typedef struct tp_weights {
  const void* q_proj_w;                        /* q_proj_1.weight            [1024,1024]  (no bias)            */
  const void* k_proj_0_w; const void* k_proj_0_b; /* k_proj_1.0             [1024,4096], [1024]               */
  const void* k_proj_2_w; const void* k_proj_2_b; /* k_proj_1.2             [1024,1024], [1024]               */
  const void* v_proj_0_w; const void* v_proj_0_b; /* v_proj_1.0                                               */
  const void* v_proj_2_w; const void* v_proj_2_b; /* v_proj_1.2                                               */
  const void* ln_q_w; const void* ln_q_b;      /* ln_q_1  [1024] x2, eps 1e-6                                   */
  const void* ln_k_w; const void* ln_k_b;
  const void* ln_v_w; const void* ln_v_b;
  const void* in_proj_w; const void* in_proj_b;   /* clip_attn.in_proj_{weight,bias}  [3072,1024], [3072]     */
  const void* out_proj_w; const void* out_proj_b; /* clip_attn.out_proj               [1024,1024], [1024]     */
  const void* mlp_0_w; const void* mlp_0_b;    /* mlp.0  [H,1024], [H]                                          */
  const void* mlp_2_w; const void* mlp_2_b;    /* mlp.2  [H,H],    [H]                                          */
} tp_weights;

/* Size of the derived ("packed") weight cache for hidden size H: concatenated K/V first layers, LayerNorm affine
 * folded into the MHA in-projections, fp32 biases.  The cache must be rebuilt whenever a parameter changes. */
TP_API size_t tp_packed_bytes(int hidden);
TP_API int tp_pack_weights(const tp_weights* w, int hidden, void* packed, size_t packed_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Projector forward.  Replaces TokenPacker.forward (builder.py:107-137).
 *   x0  [n_crops, 576, 1024] bf16 — CLIP layer-23 patch features        (x[0] of the reference's input tuple)
 *   xm  [n_crops, 576, 4096] bf16 — concatenated layers 12/16/22/23     (x[1])
 *   x0_crop_stride / xm_crop_stride: elements between consecutive crops (576*1024 / 576*4096 when contiguous;
 *        577*C for the [:,1:] views CLIPVisionTower.feature_select hands over, clip_encoder.py:37-38)
 *   out [n_crops, M, H] bf16 contiguous, M = (24/scale_factor)^2 — or, when seg_row_offset != NULL, crop i's M
 *        rows are written to rows seg_row_offset[i] .. +M-1 of ``out`` (row stride H): the packed HD layout
 *        of llava_arch.py:139-155 without a second pass.  seg_row_offset is a DEVICE int64 array [n_crops].
 * ------------------------------------------------------------------------------------------------------------- */
TP_API size_t tp_workspace_bytes(int64_t n_crops, int scale_factor, int hidden);

TP_API int tp_forward(const void* packed, const void* x0, const void* xm, int64_t n_crops, int64_t x0_crop_stride,
               int64_t xm_crop_stride, int scale_factor, int hidden, void* out, const int64_t* seg_row_offset,
               void* workspace, size_t workspace_bytes, void* stream);

/* Same forward with the HD packed layout as a UNIFORM row stride: crop i's M rows go to rows i*out_crop_rows .. +M-1 of ``out``
 * (row stride H).  llava_arch.py:139-155 follows every crop's tokens with exactly one separator row (',' between columns, '\n'
 * at the end of a grid row and after the thumbnail), so the packed sequence of any batch of images is this layout with
 * out_crop_rows = M + 1 and the separator rows (tp_hd_fill_separators) in the gaps.  Unlike the seg_row_offset form the output
 * stays on the TMA-store path: each 128-row slab leaves as one clipped 3-D box per crop it touches.  out_crop_rows = 0 or M: dense. */
TP_API int tp_forward_packed(const void* packed, const void* x0, const void* xm, int64_t n_crops, int64_t x0_crop_stride,
                             int64_t xm_crop_stride, int scale_factor, int hidden, void* out, int64_t out_crop_rows,
                             void* workspace, size_t workspace_bytes, void* stream);

/* Same forward, taking the multi-level stack as its FOUR layers instead of their concatenation: layers[0..3] are the CLIP
 * hidden states 12 / 16 / 22 / 23 that CLIPVisionTower.feature_select concatenates (clip_encoder.py:28-44), each
 * [n_crops, 576, 1024] bf16 with row stride 1024 and crop stride ``crop_stride`` (577*1024 for the [:,1:] views of the raw
 * hidden states); layers[3] is also x0 (select_layer = -2).  The first GEMM reads its K range from four tensor maps, so the
 * 4.7 MB/crop concatenated copy upstream never has to exist (SURVEY.md §8f N3). */
TP_API int tp_forward_layers(const void* packed, const void* const* layers, int64_t n_crops, int64_t crop_stride, int scale_factor,
                             int hidden, void* out, const int64_t* seg_row_offset, void* workspace, size_t workspace_bytes, void* stream);

/* Multi-GPU form with the all-gather FUSED into the last GEMM's epilogue.  peer_out[p] (p < n_peers <= 8) is the base of an
 * output buffer [total_crops * R, H] bf16 on GPU p (R = out_crop_rows, or M when out_crop_rows is 0: the dense gathered
 * [total_crops, M, H] form), mapped into this process (CUDA IPC / symmetric memory; own buffer included).  This rank's n_crops
 * crops are written to rows (crop_offset + i)*R .. +M-1 of EVERY peer buffer by TMA stores over NVLink, tile by tile as the GEMM
 * produces them — no separate collective kernel, no staging copy and, with R = M + 1, no assembly pass either: the stores land
 * in the packed per-image sequences of llava_arch.py:139-155 directly (separator rows: tp_hd_fill_separators on each rank).
 * The caller must run a cross-rank barrier after the stream reaches this call before any rank reads its buffer.
 * Needs hidden % 256 == 0.  Replaces: encode_images on sharded crops + the cross-rank reassembly of llava_arch.py:139-155. */
TP_API int tp_forward_allgather(const void* packed, const void* x0, const void* xm, int64_t n_crops, int64_t x0_crop_stride,
                                int64_t xm_crop_stride, int scale_factor, int hidden, void* const* peer_out, int n_peers,
                                int64_t crop_offset, int64_t out_crop_rows, void* workspace, size_t workspace_bytes, void* stream);

/* Same call with HOST buffers (pinned recommended): copies inputs in, runs, copies the result out, pipelined over
 * chunks of ``chunk_crops`` crops (the last few chunks shrink, so that the part not hidden behind the copies in — the final
 * chunk's compute and copy out — is short) on internal streams, and returns after the result is in ``out_host``.  The workspace
 * must cover tp_workspace_bytes(chunk_crops, ...).  d_* are caller-provided
 * device staging buffers of at least the sizes tp_forward needs for n_crops.  This is the end-to-end entry point
 * the benchmark times (host<->device traffic inside the call). */
TP_API int tp_forward_host(const void* packed, const void* x0_host, const void* xm_host, int64_t n_crops, int scale_factor,
                    int hidden, void* out_host, void* d_x0, void* d_xm, void* d_out, void* workspace,
                    size_t workspace_bytes, int64_t chunk_crops, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Training path.  The reference trains this module through PyTorch autograd over builder.py:107-137 (it is the only
 * trainable module of stage 1, train.py:950-953).  tp_forward_train computes the same output as tp_forward while keeping
 * the intermediates the backward needs in ``saved`` (caller-owned, tp_train_saved_bytes); tp_backward turns dL/d(out)
 * into dL/d(parameter) for every entry of tp_weights (``grads``: same struct, device bf16 buffers of the parameter shapes,
 * overwritten).  No gradient is produced for x0 / xm (frozen CLIP tower).  xm must be contiguous for tp_backward.
 * ------------------------------------------------------------------------------------------------------------- */
TP_API size_t tp_train_saved_bytes(int64_t n_crops, int scale_factor, int hidden);
TP_API size_t tp_backward_workspace_bytes(int64_t n_crops, int scale_factor, int hidden);
/* ``w`` NULL: every weight matrix is read from ``packed`` (a full tp_pack_weights buffer).  ``w`` non-NULL: the matrices that need no
 * transformation (k/v_proj.2, q_proj, out_proj, mlp.0, mlp.2) are read from the live parameters IN PLACE and ``packed`` only has to hold
 * what tp_pack_weights_train writes (fp32 biases, the LayerNorm-folded in-projections, the concatenated k/v_proj.0): a training step
 * repacks every forward (the optimizer moved the weights), so the 50 MB of copies and the inference-only out_proj fold are skipped. */
TP_API int tp_pack_weights_train(const tp_weights* w, int hidden, void* packed, size_t packed_bytes, void* stream);
TP_API int tp_forward_train(const tp_weights* w, const void* packed, const void* x0, const void* xm, int64_t n_crops, int64_t x0_crop_stride,
                            int64_t xm_crop_stride, int scale_factor, int hidden, void* out, void* saved, size_t saved_bytes,
                            void* stream);
TP_API int tp_backward(const tp_weights* w, const void* xm, int64_t xm_crop_stride, int64_t n_crops, int scale_factor, int hidden,
                       const void* grad_out, const void* saved, const tp_weights* grads, void* workspace, size_t workspace_bytes,
                       void* stream);

/* A single fused-epilogue GEMM of the path, exposed for unit tests and microbenchmarks:
 *   C[M,N] = alpha * act( A[M,K] . B[N,K]^T + bias ),  bf16 in/out, fp32 accumulate; bias fp32 [N] or NULL. */
TP_API int tp_gemm_bf16(const void* a, int64_t lda, const void* b, int64_t ldb, void* c, int64_t ldc, int64_t m, int64_t n,
                 int64_t k, const float* bias, int gelu, float alpha, void* stream);

/* The wgrad form of the same kernel:  C[M,N] = alpha * A^T . B  with A given as a row-major [K, M] matrix and B as [K, N]
 * (contraction over ROWS; both operands reach the tensor cores as MN-major shared-memory tiles — no transposes).
 * Needs N % 256 == 0. */
TP_API int tp_gemm_tn_bf16(const void* a, int64_t lda, const void* b, int64_t ldb, void* c, int64_t ldc, int64_t m, int64_t n,
                           int64_t k, float alpha, void* stream);

/* The dgrad form:  C[M,N] = alpha * A . B  with A the usual row-major [M, K] and B given as a row-major [K, N] matrix (a weight
 * as stored, [out, in]): B reaches the tensor cores as MN-major tiles — no transposed copy of the weight.  Needs N % 256 == 0. */
TP_API int tp_gemm_nn_bf16(const void* a, int64_t lda, const void* b, int64_t ldb, void* c, int64_t ldc, int64_t m, int64_t n,
                           int64_t k, float alpha, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * TokenPacker-HD front end.
 * ------------------------------------------------------------------------------------------------------------- */
/* Image_Patch(image_size, patch_num).calculate(h, w)  (patch_divide.py:96-105).  Host function, no CUDA. */
TP_API int tp_hd_grid(int64_t h, int64_t w, int patch_num, int image_size, int* h_block, int* w_block);

/* Sizes produced by the tiling block for an h x w image on an hb x wb grid (train.py:701-708, :719-726):
 * resized size of the main canvas content and of the thumbnail content.  Host function. */
TP_API int tp_hd_fit(int64_t h, int64_t w, int h_block, int w_block, int* h_resized, int* w_resized, int* h_thumb, int* w_thumb);

/* Tiling block (train.py:695-731): bilinear resize (align_corners=False, no antialias) of image[3,h,w] fp32 into a
 * zero-padded 336*hb x 336*wb canvas, row-major 336x336 crops, plus — when hb*wb > 1 — the thumbnail resized
 * from the PADDED canvas.  crops: [hb*wb (+1), 3, 336, 336] fp32.  All device pointers. */
TP_API int tp_hd_tile(const float* image, int64_t h, int64_t w, int h_block, int w_block, float* crops, void* stream);

/* Batched form of the tiling block: the collator concatenates the crops of a batch (train.py:797-800), so the front end of a
 * batch is ONE launch over variable-size images, thumbnails included.
 *   tp_hd_tile_batch_plan  host function: per image grid selection (tp_hd_grid) + fitted sizes (tp_hd_fit), fills
 *                          images_host[n_images] (image = images[b], a DEVICE pointer to [3,h,w] fp32), crop_table_host[3*n_crops]
 *                          = (image, grid row, grid column; column -1 = the thumbnail), h_block / w_block, *n_crops.  Any output
 *                          pointer may be NULL (count only).  Crop order = the reference's: image by image, row-major, thumbnail last.
 *   tp_hd_tile_batch       the launch: images_dev / crop_table_dev are device copies of the two tables; crops [n_crops,3,336,336] fp32. */
typedef struct tp_hd_image {
  const float* image;
  int32_t h, w, hb, wb;
  int32_t h_r, w_r;
  int32_t h_t, w_t;
  int64_t crop0;
  float sy, sx, ty, tx;   /* bilinear scales (source extent / resized extent) of the main canvas and of the thumbnail */
} tp_hd_image;
TP_API int tp_hd_tile_batch_plan(const int64_t* h, const int64_t* w, const void* const* images, int64_t n_images, int patch_num,
                                 tp_hd_image* images_host, int32_t* crop_table_host, int* h_block, int* w_block, int64_t* n_crops);
TP_API int tp_hd_tile_batch(const tp_hd_image* images_dev, const int32_t* crop_table_dev, int64_t n_crops, float* crops, void* stream);

/* Slice assembly (llava_arch.py:139-155).  Host helper: fills seg_row_offset_host[n_crops] (destination row of each
 * crop's first token), sep_rows / ret_rows (destination rows of the ',' and '\n' embedding rows; capacities are the
 * exact counts returned in *n_sep / *n_ret) and cu_seqlens_host[n_images+1].  Pass NULL outputs to only count. */
TP_API int tp_hd_plan(const int* h_block, const int* w_block, int64_t n_images, int tokens_per_crop, int64_t* seg_row_offset_host,
               int64_t* sep_rows_host, int64_t* ret_rows_host, int64_t* cu_seqlens_host, int64_t* n_crops, int64_t* n_sep,
               int64_t* n_ret);

/* Stand-alone form of the crop scatter (used after the multi-GPU all-gather, where the projector's own scatter epilogue
 * cannot be used): out[seg_row_offset[c] + m, :] = feats[c, m, :].  Device pointers, bf16. */
TP_API int tp_hd_scatter_crops(const void* feats, int64_t n_crops, int tokens_per_crop, int hidden, const int64_t* seg_row_offset,
                               void* out, void* stream);

/* Text/vision splice as ONE gather (replaces the Python list / torch.cat loops of llava_arch.py:119-233): row i of ``out``
 * [n_rows, hidden] bf16 is table[src_index[i]] (text token embedding) when src_index[i] >= 0, a zero row (right padding) when
 * it is -1, and visual[-src_index[i] - 2] (a projected visual token) otherwise.  All device pointers. */
TP_API int tp_gather_rows(const void* table, const void* visual, int hidden, const int64_t* src_index, int64_t n_rows, void* out,
                          void* stream);

/* Writes the separator rows of the packed output: out[sep_rows[i], :] = sep_row, out[ret_rows[i], :] = ret_row
 * (bf16 vectors of length hidden).  Device pointers. */
TP_API int tp_hd_fill_separators(void* out, int hidden, const int64_t* sep_rows, int64_t n_sep, const void* sep_row,
                          const int64_t* ret_rows, int64_t n_ret, const void* ret_row, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TOKENPACKER_B200_H_ */
