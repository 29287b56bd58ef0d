// Non-GEMM kernels of the TokenPacker path: point-query stencil, local-window attention, weight packing,
// and the HD front end (tiling, separator rows).  All HBM-bound: 16-byte vector accesses along the channel dim.
#pragma once

#include "tp_ptx.cuh"

namespace tp {

constexpr int kGrid = 24;       // builder.py:42 raw_grid
constexpr int kTokens = 576;    // 24*24
constexpr int kC = 1024;        // embed_dim / kv_dim (builder.py:43,45)
constexpr int kCm = 4096;       // multi-level stack width (builder.py:61,67)
constexpr int kHeads = 8;       // builder.py:44
constexpr int kHeadDim = 128;

__device__ __forceinline__ void unpack8(const uint4& v, float (&f)[8]) {
  f[0] = bf16_lo(v.x); f[1] = bf16_hi(v.x); f[2] = bf16_lo(v.y); f[3] = bf16_hi(v.y);
  f[4] = bf16_lo(v.z); f[5] = bf16_hi(v.z); f[6] = bf16_lo(v.w); f[7] = bf16_hi(v.w);
}

__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  return make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
}

// ------------------------------------------------------------------------------------------------
// Point queries (builder.py:117-118): bilinear 24x24 -> g x g with align_corners=False is a fixed stencil per
// s x s window: the source coordinate of output i is s*i + s/2 - 0.5, so an odd s reads the window's centre token
// (weight exactly 1) and an even s the mean of its centre 2x2 (weights exactly 0.5 each) — s=2: mean of the 2x2;
// s=3: the centre; s=4: mean of the centre 2x2; s=1: the token itself.  Computed in fp32 (the reference upcasts
// with .float()) and rounded once to bf16 (.to(x.dtype)).
// One thread per 8 channels of one query.
// ------------------------------------------------------------------------------------------------
template <int S>
__global__ void point_query_kernel(const __nv_bfloat16* __restrict__ x0, long long crop_stride, __nv_bfloat16* __restrict__ q,
                                   long long n_queries) {
  constexpr int G = kGrid / S;
  constexpr int M = G * G;
  grid_dependency_wait();        // PDL: inputs may come from the previous kernel on the stream
  grid_launch_dependents();
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long query = idx >> 7;          // 128 vectors of 8 channels per query
  const int vec = static_cast<int>(idx & 127);
  if (query >= n_queries) return;
  const long long n = query / M;
  const int m = static_cast<int>(query - n * M);
  const int hb = m / G, wb = m - hb * G;
  const __nv_bfloat16* base = x0 + n * crop_stride + vec * 8;
  auto tok = [&](int r, int c) { return __ldg(reinterpret_cast<const uint4*>(base + static_cast<long long>(r * kGrid + c) * kC)); };
  uint4 out;
  if (S % 2 == 1) {
    out = tok(hb * S + (S - 1) / 2, wb * S + (S - 1) / 2);
  } else {
    const int r0 = hb * S + S / 2 - 1;
    const int c0 = wb * S + S / 2 - 1;
    float a[8], b[8], c[8], d[8], o[8];
    unpack8(tok(r0, c0), a);
    unpack8(tok(r0, c0 + 1), b);
    unpack8(tok(r0 + 1, c0), c);
    unpack8(tok(r0 + 1, c0 + 1), d);
    // (0.25a + 0.25b) + (0.25c + 0.25d): each tap is scaled BEFORE the adds, so taps in bf16's top binade (|x| >= 2^127) cannot
    // overflow a partial sum.  0.25 x is exact for every bf16 x (bf16's smallest subnormal is 2^-133, fp32's 2^-149), so the bits
    // are those of the reference's 0.5 (0.5a + 0.5b) + 0.5 (0.5c + 0.5d), and — wherever the scaled taps and partial sums are
    // normal numbers — those of the former 0.25 ((a + b) + (c + d)).  Explicit intrinsics: no FMA contraction.
#pragma unroll
    for (int i = 0; i < 8; ++i)
      o[i] = __fadd_rn(__fadd_rn(__fmul_rn(0.25f, a[i]), __fmul_rn(0.25f, b[i])), __fadd_rn(__fmul_rn(0.25f, c[i]), __fmul_rn(0.25f, d[i])));
    out = pack8(o);
  }
  *reinterpret_cast<uint4*>(q + query * kC + vec * 8) = out;
}

// ------------------------------------------------------------------------------------------------
// Local-window cross attention core (builder.py:122-130 == nn.MultiheadAttention with L=1, S=s*s):
//   per query (n, hb, wb) and head h:  p = softmax_j( q'_h . k'_{j,h} ),  ctx_h = sum_j p_j v'_{j,h}
// q' is already scaled by 1/sqrt(128) (fused into the in_proj_q GEMM epilogue).  The window gather
// (divide_feature, builder.py:96-105) is pure address arithmetic here: fine token (hb*s+hi, wb*s+wi).
// One warp per query; lane l owns channels {256*i + 8*l .. +7 : i=0..3}; channel block i of lanes 0-15 is head 2i,
// of lanes 16-31 head 2i+1, so a head's dot product is a 16-lane shuffle reduction.
// ------------------------------------------------------------------------------------------------
template <int S>
__global__ void __launch_bounds__(256) window_attn_kernel(const __nv_bfloat16* __restrict__ qp, const __nv_bfloat16* __restrict__ kp,
                                                          const __nv_bfloat16* __restrict__ vp, __nv_bfloat16* __restrict__ ctx,
                                                          long long n_queries) {
  constexpr int G = kGrid / S;
  constexpr int M = G * G;
  constexpr int W = S * S;
  grid_dependency_wait();        // PDL: q', k', v' come from the previous GEMM launch
  grid_launch_dependents();
  const long long query = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (query >= n_queries) return;
  const long long n = query / M;
  const int m = static_cast<int>(query - n * M);
  const int hb = m / G, wb = m - hb * G;
  const long long tok0 = n * kTokens + static_cast<long long>(hb * S) * kGrid + wb * S;

  float qf[4][8];
#pragma unroll
  for (int i = 0; i < 4; ++i) unpack8(__ldg(reinterpret_cast<const uint4*>(qp + query * kC + i * 256 + lane * 8)), qf[i]);

  float sc[4][W];
#pragma unroll
  for (int j = 0; j < W; ++j) {
    const long long tok = tok0 + (j / S) * kGrid + (j % S);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float kf[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(kp + tok * kC + i * 256 + lane * 8)), kf);
      float d = 0.f;
#pragma unroll
      for (int e = 0; e < 8; ++e) d = fmaf(qf[i][e], kf[e], d);
      sc[i][j] = d;
    }
  }
  // 16-lane reductions (lanes 0-15 and 16-31 hold different heads)
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < W; ++j) {
      float d = sc[i][j];
      d += __shfl_xor_sync(0xffffffffu, d, 8);
      d += __shfl_xor_sync(0xffffffffu, d, 4);
      d += __shfl_xor_sync(0xffffffffu, d, 2);
      d += __shfl_xor_sync(0xffffffffu, d, 1);
      sc[i][j] = d;
    }
  // softmax over the W keys, fp32
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float mx = sc[i][0];
#pragma unroll
    for (int j = 1; j < W; ++j) mx = fmaxf(mx, sc[i][j]);
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < W; ++j) {
      sc[i][j] = __expf(sc[i][j] - mx);
      sum += sc[i][j];
    }
    const float inv = 1.0f / sum;
#pragma unroll
    for (int j = 0; j < W; ++j) sc[i][j] *= inv;
  }
  float of[4][8];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int e = 0; e < 8; ++e) of[i][e] = 0.f;
#pragma unroll
  for (int j = 0; j < W; ++j) {
    const long long tok = tok0 + (j / S) * kGrid + (j % S);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float vf[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(vp + tok * kC + i * 256 + lane * 8)), vf);
#pragma unroll
      for (int e = 0; e < 8; ++e) of[i][e] = fmaf(sc[i][j], vf[e], of[i][e]);
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) *reinterpret_cast<uint4*>(ctx + query * kC + i * 256 + lane * 8) = pack8(of[i]);
}

// Same computation for any window size (scale_factor 1, 6, 8, 12, 24: 1 ... 576 keys per query — constructor-valid upstream,
// builder.py:51-52, though no released model uses them): the keys are streamed through an online softmax instead of being
// held in registers.  Same warp / lane ownership as window_attn_kernel.
__global__ void __launch_bounds__(256) window_attn_stream_kernel(const __nv_bfloat16* __restrict__ qp, const __nv_bfloat16* __restrict__ kp,
                                                                 const __nv_bfloat16* __restrict__ vp, __nv_bfloat16* __restrict__ ctx,
                                                                 long long n_queries, int s) {
  const int G = kGrid / s;
  const int M = G * G;
  const int W = s * s;
  grid_dependency_wait();
  grid_launch_dependents();
  const long long query = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (query >= n_queries) return;
  const long long n = query / M;
  const int m = static_cast<int>(query - n * M);
  const int hb = m / G, wb = m - hb * G;
  const long long tok0 = n * kTokens + static_cast<long long>(hb * s) * kGrid + wb * s;

  float qf[4][8], of[4][8], mx[4], den[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    unpack8(__ldg(reinterpret_cast<const uint4*>(qp + query * kC + i * 256 + lane * 8)), qf[i]);
    mx[i] = -INFINITY;
    den[i] = 0.f;
#pragma unroll
    for (int e = 0; e < 8; ++e) of[i][e] = 0.f;
  }
  for (int j = 0; j < W; ++j) {
    const int hi = j / s;
    const long long tok = tok0 + static_cast<long long>(hi) * kGrid + (j - hi * s);
    float sc[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float kf[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(kp + tok * kC + i * 256 + lane * 8)), kf);
      float d = 0.f;
#pragma unroll
      for (int e = 0; e < 8; ++e) d = fmaf(qf[i][e], kf[e], d);
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) d += __shfl_xor_sync(0xffffffffu, d, off);
      sc[i] = d;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float m_new = fmaxf(mx[i], sc[i]);
      const float corr = __expf(mx[i] - m_new);       // 0 on the first key (mx = -inf)
      const float pj = __expf(sc[i] - m_new);
      den[i] = fmaf(den[i], corr, pj);
      mx[i] = m_new;
      float vf[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(vp + tok * kC + i * 256 + lane * 8)), vf);
#pragma unroll
      for (int e = 0; e < 8; ++e) of[i][e] = fmaf(pj, vf[e], of[i][e] * corr);
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float inv = 1.0f / den[i];
#pragma unroll
    for (int e = 0; e < 8; ++e) of[i][e] *= inv;
    *reinterpret_cast<uint4*>(ctx + query * kC + i * 256 + lane * 8) = pack8(of[i]);
  }
}

// ------------------------------------------------------------------------------------------------
// Weight packing
// ------------------------------------------------------------------------------------------------
// bf16 -> fp32 vectors in one launch (the packed biases): blockIdx.y = segment
struct CastSeg { const __nv_bfloat16* src; float* dst; int n; };
struct CastSegs { CastSeg s[8]; };
__global__ void bf16_to_f32_multi_kernel(CastSegs segs) {
  const CastSeg g = segs.s[blockIdx.y];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < g.n; i += gridDim.x * blockDim.x) g.dst[i] = __bfloat162float(g.src[i]);
}
// The same for segments whose src holds IEEE half values (the fp16 CLIP tower's biases)
__global__ void f16_to_f32_multi_kernel(CastSegs segs) {
  const CastSeg g = segs.s[blockIdx.y];
  const __half* src = reinterpret_cast<const __half*>(g.src);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < g.n; i += gridDim.x * blockDim.x) g.dst[i] = __half2float(src[i]);
}

// LayerNorm folded into the following linear (one warp per output feature o):
//   LN(y) W^T + b = rstd * ( y (gamma.W)^T - mu * rowsum(gamma.W) ) + ( W beta + b )
//   w_out[o,:] = bf16(W[o,:] * gamma),  wsum[o] = sum_i w_out[o,i] (of the ROUNDED values),  cst[o] = W[o,:].beta + b[o]
__global__ void fold_layernorm_kernel(const __nv_bfloat16* __restrict__ w, const __nv_bfloat16* __restrict__ bias,
                                      const __nv_bfloat16* __restrict__ gamma, const __nv_bfloat16* __restrict__ beta,
                                      __nv_bfloat16* __restrict__ w_out, float* __restrict__ wsum, float* __restrict__ cst,
                                      int out_dim, int in_dim) {
  const int o = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (o >= out_dim) return;
  float s = 0.f, c = 0.f;
  for (int i = lane; i < in_dim; i += 32) {
    const float wv = __bfloat162float(w[static_cast<long long>(o) * in_dim + i]);
    const __nv_bfloat16 folded = __float2bfloat16_rn(wv * __bfloat162float(gamma[i]));
    w_out[static_cast<long long>(o) * in_dim + i] = folded;
    s += __bfloat162float(folded);
    c = fmaf(wv, __bfloat162float(beta[i]), c);
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, off);
    c += __shfl_xor_sync(0xffffffffu, c, off);
  }
  if (lane == 0) {
    wsum[o] = s;
    cst[o] = c + __bfloat162float(bias[o]);
  }
}

// out[o] = sum_i w[o, i] * x[i] + b[o]   (fp32 out; one warp per output; pack time only)
__global__ void matvec_bias_kernel(const __nv_bfloat16* __restrict__ w, const __nv_bfloat16* __restrict__ x,
                                   const __nv_bfloat16* __restrict__ b, float* __restrict__ out, int out_dim, int in_dim) {
  const int o = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (o >= out_dim) return;
  float acc = 0.f;
  for (int i = lane; i < in_dim; i += 32) acc = fmaf(__bfloat162float(w[static_cast<long long>(o) * in_dim + i]), __bfloat162float(x[i]), acc);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  if (lane == 0) out[o] = acc + __bfloat162float(b[o]);
}

// ------------------------------------------------------------------------------------------------
// HD front end
// ------------------------------------------------------------------------------------------------
constexpr int kBlockPx = 336;   // train.py:699 block_size

struct LinearTap {
  int i0, i1;
  float w0, w1;
};

// ATen upsample_bilinear2d, align_corners=False, scales derived from sizes: src = (in/out)*(dst+0.5)-0.5 clamped at 0.
__device__ __forceinline__ LinearTap linear_tap_scaled(int dst, int in_size, float scale);

__device__ __forceinline__ LinearTap linear_tap(int dst, int in_size, int out_size) {
  return linear_tap_scaled(dst, in_size, static_cast<float>(in_size) / static_cast<float>(out_size));
}

// same with the scale (in_size / out_size as one IEEE float division) supplied by the caller
__device__ __forceinline__ LinearTap linear_tap_scaled(int dst, int in_size, float scale) {
  float src = __fmaf_rn(scale, static_cast<float>(dst) + 0.5f, -0.5f);   // ONE fused multiply-add, like ATen's CPU kernel (see oracle/hd_oracle.py)
  src = fmaxf(src, 0.f);
  LinearTap t;
  t.i0 = min(static_cast<int>(src), in_size - 1);
  t.i1 = t.i0 + (t.i0 < in_size - 1 ? 1 : 0);
  t.w1 = fminf(fmaxf(src - static_cast<float>(t.i0), 0.f), 1.f);
  t.w0 = 1.f - t.w1;
  return t;
}

__device__ __forceinline__ float bilerp(float a, float b, float c, float d, const LinearTap& ty, const LinearTap& tx) {
  const float top = __fadd_rn(__fmul_rn(tx.w0, a), __fmul_rn(tx.w1, b));
  const float bot = __fadd_rn(__fmul_rn(tx.w0, c), __fmul_rn(tx.w1, d));
  return __fadd_rn(__fmul_rn(ty.w0, top), __fmul_rn(ty.w1, bot));
}

// Pass 1 (train.py:709-717): crops[(i*wb+j), ch, y, x] = canvas[ch, 336 i + y, 336 j + x], canvas = zero-padded
// bilinear resize of image[3,h,w] to (h_r, w_r).
__global__ void hd_tile_main_kernel(const float* __restrict__ image, int h, int w, int hb, int wb, int h_r, int w_r,
                                    float* __restrict__ crops) {
  const long long total = 3ll * hb * kBlockPx * wb * kBlockPx;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cw = wb * kBlockPx, chh = hb * kBlockPx;
  const int X = static_cast<int>(idx % cw);
  const int Y = static_cast<int>((idx / cw) % chh);
  const int ch = static_cast<int>(idx / (static_cast<long long>(cw) * chh));
  float v = 0.f;
  if (Y < h_r && X < w_r) {
    const LinearTap ty = linear_tap(Y, h, h_r), tx = linear_tap(X, w, w_r);
    const float* p = image + static_cast<long long>(ch) * h * w;
    v = bilerp(p[static_cast<long long>(ty.i0) * w + tx.i0], p[static_cast<long long>(ty.i0) * w + tx.i1],
               p[static_cast<long long>(ty.i1) * w + tx.i0], p[static_cast<long long>(ty.i1) * w + tx.i1], ty, tx);
  }
  const int ci = Y / kBlockPx, cj = X / kBlockPx;
  const int y = Y - ci * kBlockPx, x = X - cj * kBlockPx;
  crops[((static_cast<long long>(ci * wb + cj) * 3 + ch) * kBlockPx + y) * kBlockPx + x] = v;
}

// Pass 2 (train.py:718-730): thumbnail = zero-padded bilinear resize of the PADDED canvas (read back from the crop
// layout written by pass 1) to (h_t, w_t); stored as crop index hb*wb.
__global__ void hd_tile_thumb_kernel(int hb, int wb, int h_t, int w_t, float* __restrict__ crops) {
  const int total = 3 * kBlockPx * kBlockPx;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int x = idx % kBlockPx;
  const int y = (idx / kBlockPx) % kBlockPx;
  const int ch = idx / (kBlockPx * kBlockPx);
  float v = 0.f;
  if (y < h_t && x < w_t) {
    const LinearTap ty = linear_tap(y, hb * kBlockPx, h_t), tx = linear_tap(x, wb * kBlockPx, w_t);
    auto canvas = [&](int Y, int X) {
      const int ci = Y / kBlockPx, cj = X / kBlockPx;
      return crops[((static_cast<long long>(ci * wb + cj) * 3 + ch) * kBlockPx + (Y - ci * kBlockPx)) * kBlockPx + (X - cj * kBlockPx)];
    };
    v = bilerp(canvas(ty.i0, tx.i0), canvas(ty.i0, tx.i1), canvas(ty.i1, tx.i0), canvas(ty.i1, tx.i1), ty, tx);
  }
  crops[((static_cast<long long>(hb * wb) * 3 + ch) * kBlockPx + y) * kBlockPx + x] = v;
}

// ------------------------------------------------------------------------------------------------
// Batched form of the tiling block: ONE launch tiles a whole batch of variable-size images (the collator concatenates the
// crops of a batch, train.py:797-800), thumbnails included, float4 stores.  Every thread produces 4 consecutive pixels of one
// crop row.  The thumbnail is resized from the PADDED canvas (train.py:710,718-730); instead of reading pass-1 output back, each
// canvas tap is recomputed from the source image with exactly the arithmetic the main crops use, so the bits are those of
// the two-pass kernels above.
// ------------------------------------------------------------------------------------------------
struct HdImage {            // mirrors tp_hd_image (include/tokenpacker_b200.h)
  const float* image;       // [3, h, w] fp32, normalised
  int h, w, hb, wb;
  int h_r, w_r;             // resized content of the main canvas
  int h_t, w_t;             // resized content of the thumbnail (0 when hb*wb == 1)
  long long crop0;          // index of this image's first crop in the batch output
  float sy, sx;             // h / h_r, w / w_r as float divisions (ATen's scale), computed once per image on the host
  float ty, tx;             // (336 hb) / h_t, (336 wb) / w_t
};

struct HdU8Image {          // mirrors tp_hd_u8_source (include/tokenpacker_b200_hd_u8.h)
  const unsigned char* pixels;
  long long stride_c, stride_y, stride_x;   // element strides of channel, row and column
};

// Source readers of hd_tile_batch_kernel.  view() binds a reader to one image; View::at(row(y), ch, x) is source pixel (ch, y, x) as
// the float32 value the tap arithmetic consumes.  The arithmetic is the same for every reader, so equal values give equal bits.
struct HdF32Source {        // HdImage::image: the normalised float32 [3, h, w] image, contiguous
  struct View {
    const float* p;
    long long plane;
    int w;
    __device__ __forceinline__ long long row(int y) const { return static_cast<long long>(y) * w; }
    __device__ __forceinline__ float at(long long r, int ch, int x) const { return __ldg(p + r + ch * plane + x); }
  };
  __device__ __forceinline__ View view(const HdImage& im, int) const { return {im.image, static_cast<long long>(im.h) * im.w, im.w}; }
};

// Decoded 8-bit pixels at any (channel, row, column) strides, normalised through table[c][u] = (u / 255 - mean[c]) / std[c]
// (ToTensor + Normalize, train.py:645), which the host computes with the CPU ops torchvision uses.  The 768 floats are staged in
// shared memory once per CTA: lanes look up different bytes, and constant memory would serialise such divergent reads.
constexpr int kNormTable = 3 * 256;
struct HdU8Source {
  const HdU8Image* sources;   // [n_images], indexed like HdImage
  const float* table;         // [3][256] float32
  struct View {
    const unsigned char* p;
    long long sc, sy, sx;
    const float* lut;         // shared memory
    __device__ __forceinline__ long long row(int y) const { return y * sy; }
    __device__ __forceinline__ float at(long long r, int ch, int x) const { return lut[ch * 256 + __ldg(p + r + ch * sc + x * sx)]; }
  };
  // every thread of the CTA calls this once (it synchronises the CTA)
  __device__ __forceinline__ View view(const HdImage&, int img) const {
    __shared__ float lut[kNormTable];
    for (int i = threadIdx.x; i < kNormTable; i += blockDim.x) lut[i] = __ldg(table + i);
    __syncthreads();
    const HdU8Image s = sources[img];
    return {s.pixels, s.stride_c, s.stride_y, s.stride_x, lut};
  }
};

__device__ __forceinline__ void hd_store(float* p, float v) { *p = v; }
__device__ __forceinline__ void hd_store(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }   // == fp32 crops .to(bfloat16)

__device__ __forceinline__ float hd_canvas_value(const HdImage& im, const float* __restrict__ plane, int Y, int X) {
  if (Y >= im.h_r || X >= im.w_r) return 0.f;
  const LinearTap ty = linear_tap_scaled(Y, im.h, im.sy), tx = linear_tap_scaled(X, im.w, im.sx);
  const float* r0 = plane + static_cast<long long>(ty.i0) * im.w;
  const float* r1 = plane + static_cast<long long>(ty.i1) * im.w;
  return bilerp(__ldg(r0 + tx.i0), __ldg(r0 + tx.i1), __ldg(r1 + tx.i0), __ldg(r1 + tx.i1), ty, tx);
}

// crop_table[c] = (image index, grid row, grid column); grid column -1 marks the image's thumbnail.
// One CTA = kHdRows rows of one crop; thread = one pixel COLUMN: its column tap is computed once and reused by the kHdRows x 3 (row,
// channel) pairs, and the lanes of a warp read neighbouring source pixels (a warp's load touches 4-6 sectors; with 4 pixels per
// thread it was 16 sectors of which 6.5 bytes each were used, and the kernel sat at 18 % of DRAM waiting for L1).  Scalar stores of
// 32 consecutive floats per warp.  The tap arithmetic is unchanged, so the bits are.
constexpr int kHdRows = 8;                                     // rows per thread; 336 = 42 x 8
constexpr int kHdUnroll = 2;                                   // rows in flight per thread (loads of the next row issue under the math of this one)
static_assert(kBlockPx % kHdRows == 0, "rows per CTA must divide the crop height");
// Src: HdF32Source (tp_hd_tile_batch) or HdU8Source (tp_hd_preprocess_batch); Out: float or __nv_bfloat16.
template <class Src, class Out>
__global__ void __launch_bounds__(kBlockPx) hd_tile_batch_kernel(const HdImage* __restrict__ images, const int* __restrict__ crop_table,
                                                                 long long n_crops, Src src, Out* __restrict__ crops) {
  constexpr int kRowGroups = kBlockPx / kHdRows;
  const long long crop = blockIdx.x / kRowGroups;
  const int y0 = static_cast<int>(blockIdx.x % kRowGroups) * kHdRows;
  const int x = threadIdx.x;
  if (crop >= n_crops) return;                                                     // uniform over the CTA
  const int img = crop_table[crop * 3], ci = crop_table[crop * 3 + 1], cj = crop_table[crop * 3 + 2];
  const HdImage im = images[img];
  const typename Src::View s = src.view(im, img);
  Out* out_base = crops + (crop * 3 * kBlockPx + y0) * kBlockPx + x;              // channel stride 336 * 336, row stride 336
  if (cj >= 0) {
    const int X = cj * kBlockPx + x;
    const bool okx = X < im.w_r;
    const LinearTap tx = linear_tap_scaled(okx ? X : 0, im.w, im.sx);
#pragma unroll kHdUnroll
    for (int r = 0; r < kHdRows; ++r) {
      const int Y = ci * kBlockPx + y0 + r;
      const bool ok = okx && Y < im.h_r;
      const LinearTap ty = linear_tap_scaled(ok ? Y : 0, im.h, im.sy);
      const long long r0 = s.row(ty.i0), r1 = s.row(ty.i1);
#pragma unroll
      for (int ch = 0; ch < 3; ++ch)
        hd_store(out_base + (static_cast<long long>(ch) * kBlockPx + r) * kBlockPx,
                 ok ? bilerp(s.at(r0, ch, tx.i0), s.at(r0, ch, tx.i1), s.at(r1, ch, tx.i0), s.at(r1, ch, tx.i1), ty, tx) : 0.f);
    }
  } else {
    // thumbnail: resized from the PADDED canvas; a canvas tap = the main crops' arithmetic at that canvas pixel (zero outside the content)
    const int ch_h = im.hb * kBlockPx, ch_w = im.wb * kBlockPx;
    const bool okx = x < im.w_t;
    const LinearTap cx = linear_tap_scaled(okx ? x : 0, ch_w, im.tx);                 // canvas column tap ...
    const bool okx0 = cx.i0 < im.w_r, okx1 = cx.i1 < im.w_r;
    const LinearTap sx0 = linear_tap_scaled(okx0 ? cx.i0 : 0, im.w, im.sx);           // ... and the source taps of its two canvas columns
    const LinearTap sx1 = linear_tap_scaled(okx1 ? cx.i1 : 0, im.w, im.sx);
#pragma unroll kHdUnroll
    for (int r = 0; r < kHdRows; ++r) {
      const int y = y0 + r;
      const bool ok = okx && y < im.h_t;
      const LinearTap cy = linear_tap_scaled(ok ? y : 0, ch_h, im.ty);
      const bool oky0 = cy.i0 < im.h_r, oky1 = cy.i1 < im.h_r;
      const LinearTap sy0 = linear_tap_scaled(oky0 ? cy.i0 : 0, im.h, im.sy), sy1 = linear_tap_scaled(oky1 ? cy.i1 : 0, im.h, im.sy);
      const long long a0 = s.row(sy0.i0), a1 = s.row(sy0.i1);   // source rows of canvas row cy.i0
      const long long b0 = s.row(sy1.i0), b1 = s.row(sy1.i1);   // ... of canvas row cy.i1
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        float o = 0.f;
        if (ok) {
          auto canvas = [&](long long q0, long long q1, const LinearTap& sy, bool rowok, const LinearTap& sx, bool colok) {
            return (rowok && colok) ? bilerp(s.at(q0, ch, sx.i0), s.at(q0, ch, sx.i1), s.at(q1, ch, sx.i0), s.at(q1, ch, sx.i1), sy, sx) : 0.f;
          };
          o = bilerp(canvas(a0, a1, sy0, oky0, sx0, okx0), canvas(a0, a1, sy0, oky0, sx1, okx1),
                     canvas(b0, b1, sy1, oky1, sx0, okx0), canvas(b0, b1, sy1, oky1, sx1, okx1), cy, cx);
        }
        hd_store(out_base + (static_cast<long long>(ch) * kBlockPx + r) * kBlockPx, o);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Non-HD CLIP input (tp_clip_preprocess_batch): expand2square onto a virtual canvas (pad mode), PIL's 8-bit BICUBIC resize of the
// short edge to 336, center crop, and the (channel, byte) table.  PIL's fixed-point arithmetic exactly: int32 weights with 22 fraction
// bits from the host plan, an accumulator that starts at 1 << 21, clamp(acc >> 22, 0, 255); the horizontal pass first, rounded to
// uint8 in the workspace, then the vertical pass.  Every sum is an exact integer sum (255 * sum |k| < 2^31), so its order is free.
// Only the 336 kept columns and the canvas rows the kept output rows read are computed.
// ------------------------------------------------------------------------------------------------
struct ClipImage {          // mirrors tp_clip_image (include/tokenpacker_b200_clip_u8.h)
  int h, w, canvas_h, canvas_w, pad_y, pad_x, resized_h, resized_w, top, left, ksize_x, ksize_y;
  long long coeff_x, coeff_y;
  int row0, rows;
  long long workspace_offset, workspace_row;
};

constexpr int kClipPrecision = 22;
constexpr int kClipRowBytes = kBlockPx * 3;                   // one workspace row: 336 kept columns x 3 channels, uint8

__device__ __forceinline__ int clip_u8(int acc) { return min(max(acc >> kClipPrecision, 0), 255); }   // Resample.c clip8

// Pixel (y, x, ch) of the canvas: the source inside the pasted rectangle, expand2square's background (122, 116, 104), the CLIP mean
// as int(x * 255), outside it.  In square mode the canvas is the source and every read is inside.
struct ClipCanvas {
  const unsigned char* p;
  long long sc, sy, sx;
  int h, w, py, px;
  __device__ __forceinline__ ClipCanvas(const ClipImage& im, const HdU8Image& s)
      : p(s.pixels), sc(s.stride_c), sy(s.stride_y), sx(s.stride_x), h(im.h), w(im.w), py(im.pad_y), px(im.pad_x) {}
  __device__ __forceinline__ int at(int y, int x, int ch) const {
    const int yy = y - py, xx = x - px;
    if (static_cast<unsigned>(yy) < static_cast<unsigned>(h) && static_cast<unsigned>(xx) < static_cast<unsigned>(w))
      return __ldg(p + yy * sy + xx * sx + ch * sc);
    return ch == 0 ? 122 : (ch == 1 ? 116 : 104);
  }
};

// Horizontal pass.  CTA = one workspace row (one canvas row of one image), thread = one kept output column, 3 channels.  The image is
// the last one whose first workspace row is <= this row (images skipping this pass own no rows).  Weight table: tap-major
// [ksize][336], so the lanes of a warp read consecutive weights.
__global__ void __launch_bounds__(kBlockPx) clip_resample_h_kernel(const ClipImage* __restrict__ images, long long n_images,
                                                                   const HdU8Image* __restrict__ sources, const int* __restrict__ coeffs,
                                                                   unsigned char* __restrict__ workspace) {
  const long long row = blockIdx.x;
  long long lo = 0, hi = n_images - 1;
  while (lo < hi) {                                              // uniform over the CTA
    const long long mid = (lo + hi + 1) / 2;
    if (images[mid].workspace_row <= row) lo = mid; else hi = mid - 1;
  }
  const ClipImage im = images[lo];
  const int r = static_cast<int>(row - im.workspace_row);
  if (im.ksize_x == 0 || r >= im.rows) return;                   // only past the last image's rows (an oversized workspace)
  const ClipCanvas cv(im, sources[lo]);
  const int y = im.row0 + r, x = threadIdx.x;
  const int* tab = coeffs + im.coeff_x;
  const int xmin = __ldg(tab + x), n = __ldg(tab + kBlockPx + x);
  const int* k = tab + 2 * kBlockPx + x;
  int a0 = 1 << (kClipPrecision - 1), a1 = a0, a2 = a0;
  for (int i = 0; i < n; ++i) {
    const int kk = __ldg(k + i * kBlockPx);
    a0 += kk * cv.at(y, xmin + i, 0);
    a1 += kk * cv.at(y, xmin + i, 1);
    a2 += kk * cv.at(y, xmin + i, 2);
  }
  unsigned char* o = workspace + im.workspace_offset + static_cast<long long>(r) * kClipRowBytes + x * 3;
  o[0] = static_cast<unsigned char>(clip_u8(a0));
  o[1] = static_cast<unsigned char>(clip_u8(a1));
  o[2] = static_cast<unsigned char>(clip_u8(a2));
}

// Vertical pass, byte lookup and store.  CTA = one output row of one image, thread = one output column, 3 channels.  The row's taps
// are the same for every thread (broadcast loads).  Its input is the workspace when the horizontal pass ran, else the canvas at the
// crop's columns; when the vertical pass is skipped the output row is input row `top + y`, as PIL leaves it.
template <class Out>
__global__ void __launch_bounds__(kBlockPx) clip_resample_v_kernel(const ClipImage* __restrict__ images, const HdU8Image* __restrict__ sources,
                                                                   const int* __restrict__ coeffs, const unsigned char* __restrict__ workspace,
                                                                   const float* __restrict__ table, Out* __restrict__ out) {
  __shared__ float lut[kNormTable];
  for (int i = threadIdx.x; i < kNormTable; i += blockDim.x) lut[i] = __ldg(table + i);
  __syncthreads();
  const long long b = blockIdx.x / kBlockPx;
  const int y = static_cast<int>(blockIdx.x % kBlockPx), x = threadIdx.x;
  const ClipImage im = images[b];
  const ClipCanvas cv(im, sources[b]);
  const bool from_ws = im.ksize_x > 0;
  const unsigned char* ws = workspace + (from_ws ? im.workspace_offset : 0) + x * 3;
  auto in = [&](int canvas_row, int ch) -> int {                 // pixel (canvas_row, kept column x) after the horizontal pass
    return from_ws ? __ldg(ws + static_cast<long long>(canvas_row - im.row0) * kClipRowBytes + ch) : cv.at(canvas_row, im.left + x, ch);
  };
  int v[3];
  if (im.ksize_y > 0) {
    const int* tab = coeffs + im.coeff_y;
    const int ymin = __ldg(tab + y), n = __ldg(tab + kBlockPx + y);
    const int* k = tab + 2 * kBlockPx + y;
    int a0 = 1 << (kClipPrecision - 1), a1 = a0, a2 = a0;
    for (int i = 0; i < n; ++i) {
      const int kk = __ldg(k + i * kBlockPx);
      a0 += kk * in(ymin + i, 0);
      a1 += kk * in(ymin + i, 1);
      a2 += kk * in(ymin + i, 2);
    }
    v[0] = clip_u8(a0); v[1] = clip_u8(a1); v[2] = clip_u8(a2);
  } else {
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) v[ch] = in(im.top + y, ch);
  }
  Out* o = out + (b * 3 * kBlockPx + y) * kBlockPx + x;
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) hd_store(o + static_cast<long long>(ch) * kBlockPx * kBlockPx, lut[ch * 256 + v[ch]]);
}

// out[seg_row_offset[c] + m, :] = feats[c, m, :]  (bf16; one thread per 8 channels): crop token blocks -> packed rows.
__global__ void scatter_crops_kernel(const __nv_bfloat16* __restrict__ feats, long long n_crops, int tokens, int hidden,
                                     const long long* __restrict__ seg_row_offset, __nv_bfloat16* __restrict__ out) {
  const int vecs = hidden / 8;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long rows = n_crops * tokens;
  if (idx >= rows * vecs) return;
  const long long r = idx / vecs;
  const int v = static_cast<int>(idx - r * vecs);
  const long long c = r / tokens;
  const long long dst = seg_row_offset[c] + (r - c * tokens);
  *reinterpret_cast<uint4*>(out + dst * hidden + v * 8) = __ldg(reinterpret_cast<const uint4*>(feats + r * hidden + v * 8));
}

// Text/vision splice (llava_arch.py:119-233 as one gather): out[i,:] = table[src[i]] if src[i] >= 0, zeros if src[i] == -1,
// visual[-src[i]-2] otherwise.  bf16 rows, one thread per 8 channels.
__global__ void gather_rows_kernel(const __nv_bfloat16* __restrict__ table, const __nv_bfloat16* __restrict__ visual, int hidden,
                                   const long long* __restrict__ src, long long n_rows, __nv_bfloat16* __restrict__ out) {
  const int vecs = hidden / 8;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= n_rows * vecs) return;
  const long long r = idx / vecs;
  const int v = static_cast<int>(idx - r * vecs);
  const long long sidx = src[r];
  uint4 val = make_uint4(0u, 0u, 0u, 0u);
  if (sidx >= 0) val = __ldg(reinterpret_cast<const uint4*>(table + sidx * hidden + v * 8));
  else if (sidx <= -2) val = __ldg(reinterpret_cast<const uint4*>(visual + (-sidx - 2) * hidden + v * 8));
  *reinterpret_cast<uint4*>(out + r * hidden + v * 8) = val;
}

// out[rows[i], :] = row (bf16 [hidden]); one thread per 8 channels.
__global__ void fill_rows_kernel(__nv_bfloat16* __restrict__ out, int hidden, const long long* __restrict__ rows, long long n_rows,
                                 const __nv_bfloat16* __restrict__ row) {
  const int vecs = hidden / 8;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= n_rows * vecs) return;
  const long long r = idx / vecs;
  const int v = static_cast<int>(idx - r * vecs);
  *reinterpret_cast<uint4*>(out + rows[r] * hidden + v * 8) = __ldg(reinterpret_cast<const uint4*>(row + v * 8));
}

}  // namespace tp
