// Kernels of the projector's backward pass that are not GEMMs: GELU forward/backward as elementwise passes, LayerNorm apply /
// backward, window-attention backward, deterministic column sums (bias gradients), a plain transpose (weights for the
// dgrad GEMMs; activations only in the small-hidden wgrad fallback), and the point-query stencil backwards (the gradient w.r.t.
// the CLIP feature x0, when asked for).  All HBM-bound, 16-byte vector accesses.
// The GEMMs of the backward run on the forward's wgmma kernels: dgrad (dX = dY . W) takes a transposed copy of the weight as
// its K-major B operand; wgrad (dW = dY^T . X) uses the TN form, reading both activations in place as MN-major tiles.
#pragma once

#include "tp_kernels.cuh"

namespace tp {

constexpr int kStatSlotsBwd = kC / 128;

// per-row LayerNorm statistics from the per-128-column (mean, M2) pairs the forward GEMM epilogue left (same combination, same
// order, same bits as the folded LayerNorm in tp_gemm.cuh)
__device__ __forceinline__ void row_mean_rstd(const float* stats, long long row, float& mu, float& rstd) {
  const float2* st = reinterpret_cast<const float2*>(stats) + row * kStatSlotsBwd;
  float t1 = 0.f, m2 = 0.f;
#pragma unroll
  for (int i = 0; i < kStatSlotsBwd; ++i) t1 = __fadd_rn(t1, st[i].x);
  const float inv_slots = __frcp_rn(static_cast<float>(kStatSlotsBwd));
  mu = __fmul_rn(t1, inv_slots);
  float between = 0.f;
#pragma unroll
  for (int i = 0; i < kStatSlotsBwd; ++i) {
    const float2 v = st[i];
    const float d = __fsub_rn(v.x, mu);
    between = fmaf(d, d, between);
    m2 = __fadd_rn(m2, v.y);
  }
  const float inv_dim = 1.0f / kC;
  const float var = __fmul_rn(fmaf(between, __fmul_rn(inv_slots, __frcp_rn(inv_dim)), m2), inv_dim);
  rstd = rsqrtf(__fadd_rn(var, 1e-6f));
}

// d/dz [ z * Phi(z) ] = Phi(z) + z * phi(z)
__device__ __forceinline__ float gelu_grad(float z) {
  const float t = fabsf(z) * 0.70710678118654752440f;
  float p = 0.0000430638f;
  p = fmaf(p, t, 0.0002765672f);
  p = fmaf(p, t, 0.0001520143f);
  p = fmaf(p, t, 0.0092705272f);
  p = fmaf(p, t, 0.0422820123f);
  p = fmaf(p, t, 0.0705230784f);
  p = fmaf(p, t, 1.0f);
  p *= p; p *= p; p *= p; p *= p;
  const float e = 1.0f - rcp_approx(p);                 // erf(|z|/sqrt2)
  const float cdf = 0.5f * (1.0f + copysignf(e, z));
  const float pdf = 0.3989422804014327f * __expf(-0.5f * z * z);
  return fmaf(z, pdf, cdf);
}

// ------------------------------------------------------------------------------------------------
// Transpose  out[c, r] = in[r, c]   (bf16; in: [rows, cols] row stride ld_in; out: [cols, rows] row stride ld_out)
// ------------------------------------------------------------------------------------------------
__global__ void transpose_kernel(const __nv_bfloat16* __restrict__ in, long long ld_in, __nv_bfloat16* __restrict__ out, long long ld_out,
                                 long long rows, int cols) {
  __shared__ __nv_bfloat16 tile[32][34];
  const long long r0 = static_cast<long long>(blockIdx.x) * 32;     // row tiles on grid.x (up to 2^31 - 1 of them; grid.y stops at 65535)
  const int c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const long long r = r0 + i;
    const int c = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (r < rows && c < cols) ? in[r * ld_in + c] : __float2bfloat16_rn(0.f);
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i;
    const long long r = r0 + threadIdx.x;
    if (c < cols && r < rows) out[static_cast<long long>(c) * ld_out + r] = tile[threadIdx.x][i];
  }
}

// h = GELU(z), 8 elements per thread (n8 = number of 8-element vectors)
__global__ void gelu_fwd_kernel(const __nv_bfloat16* __restrict__ z, __nv_bfloat16* __restrict__ h, long long n8) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n8) return;
  float f[8];
  unpack8(__ldg(reinterpret_cast<const uint4*>(z) + i), f);
#pragma unroll
  for (int j = 0; j < 8; ++j) f[j] = gelu_erf(f[j]);
  reinterpret_cast<uint4*>(h)[i] = pack8(f);
}

// dz = dh * GELU'(z) in place over dh, FUSED with the first stage of the bias gradient that follows it (column sums of dz): the
// thread layout of colsum_partial_kernel (8 columns per thread, a chunk of rows per CTA row), so dz is never re-read.  The sums
// are taken over the ROUNDED values that were stored, in row order: the same bits as colsum_partial_kernel over the stored dz.
// grid = (ceil(cols / 1024), n_chunks), 128 threads; dh and z share the row stride ld.
__global__ void __launch_bounds__(128) gelu_bwd_colsum_kernel(__nv_bfloat16* __restrict__ dh, const __nv_bfloat16* __restrict__ z, long long ld,
                                                              long long rows, int cols, int n_chunks, float* __restrict__ partial) {
  const int c0 = (blockIdx.x * 128 + threadIdx.x) * 8;
  if (c0 >= cols) return;
  const long long per = (rows + n_chunks - 1) / n_chunks;
  const long long r0 = per * blockIdx.y, r1 = min(rows, r0 + per);
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  auto one = [&](const uint4& gv, const uint4& zv, long long r) {
    float g[8], zz[8];
    unpack8(gv, g);
    unpack8(zv, zz);
#pragma unroll
    for (int j = 0; j < 8; ++j) g[j] *= gelu_grad(zz[j]);
    const uint4 o = pack8(g);
    *reinterpret_cast<uint4*>(dh + r * ld + c0) = o;
    unpack8(o, g);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] += g[j];
  };
  long long r = r0;
  for (; r + 4 <= r1; r += 4) {          // four rows of loads in flight before the first (aliasing) store
    uint4 gv[4], zv[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      gv[u] = *reinterpret_cast<const uint4*>(dh + (r + u) * ld + c0);
      zv[u] = __ldg(reinterpret_cast<const uint4*>(z + (r + u) * ld + c0));
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) one(gv[u], zv[u], r + u);
  }
  for (; r < r1; ++r) one(*reinterpret_cast<const uint4*>(dh + r * ld + c0), __ldg(reinterpret_cast<const uint4*>(z + r * ld + c0)), r);
#pragma unroll
  for (int j = 0; j < 8; ++j) partial[static_cast<long long>(blockIdx.y) * cols + c0 + j] = acc[j];
}

// LayerNorm output  out[r,:] = (y[r,:] - mu_r) rstd_r gamma + beta  (bf16; one warp per row): B operand of the in-projection wgrad
__global__ void __launch_bounds__(256) ln_apply_kernel(const __nv_bfloat16* __restrict__ y, const float* __restrict__ stats,
                                                       const __nv_bfloat16* __restrict__ gamma, const __nv_bfloat16* __restrict__ beta,
                                                       __nv_bfloat16* __restrict__ out, long long rows) {
  const long long row = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  float mu, rstd;
  row_mean_rstd(stats, row, mu, rstd);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float v[8], g[8], b[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(y + row * kC + i * 256 + lane * 8)), v);
    unpack8(__ldg(reinterpret_cast<const uint4*>(gamma + i * 256 + lane * 8)), g);
    unpack8(__ldg(reinterpret_cast<const uint4*>(beta + i * 256 + lane * 8)), b);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = fmaf((v[j] - mu) * rstd, g[j], b[j]);
    *reinterpret_cast<uint4*>(out + row * kC + i * 256 + lane * 8) = pack8(v);
  }
}

// Column sums (bias gradients), deterministic two-stage:  partial[chunk][c] = sum over the chunk's rows of in[r, c]
// grid = (ceil(cols / 1024), n_chunks), 128 threads x 8 columns
__global__ void colsum_partial_kernel(const __nv_bfloat16* __restrict__ in, long long ld, long long rows, int cols, int n_chunks,
                                      float* __restrict__ partial) {
  const int c0 = (blockIdx.x * 128 + threadIdx.x) * 8;
  if (c0 >= cols) return;
  const long long per = (rows + n_chunks - 1) / n_chunks;
  const long long r0 = per * blockIdx.y, r1 = min(rows, r0 + per);
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (long long r = r0; r < r1; ++r) {
    float f[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(in + r * ld + c0)), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] += f[j];
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) partial[static_cast<long long>(blockIdx.y) * cols + c0 + j] = acc[j];
}

// Second stage: out[c] = scale * sum_i partial[i][c] (partial rows ld_part floats apart).  Block = 32 columns x 16 chunk lanes: every thread sums chunks ty, ty+16, ...
// (independent loads), the 16 lane sums are added in fixed order — deterministic, and ~10x faster than one thread walking all
// chunks of a column with dependent loads (45 us per call at 592 chunks: 10 calls were 11 % of the training step).
constexpr int kReduceLanes = 16;
__global__ void __launch_bounds__(32 * kReduceLanes) colsum_reduce_kernel(const float* __restrict__ partial, int n_chunks, int cols, int ld_part,
                                                                          float scale, __nv_bfloat16* __restrict__ out) {
  __shared__ float s_sum[kReduceLanes][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  float a = 0.f;
  if (c < cols)
    for (int i = threadIdx.y; i < n_chunks; i += kReduceLanes) a += partial[static_cast<long long>(i) * ld_part + c];
  s_sum[threadIdx.y][threadIdx.x] = a;
  __syncthreads();
  if (threadIdx.y == 0 && c < cols) {
    float t = 0.f;
#pragma unroll
    for (int j = 0; j < kReduceLanes; ++j) t += s_sum[j][threadIdx.x];
    out[c] = __float2bfloat16_rn(t * scale);
  }
}

// ------------------------------------------------------------------------------------------------
// LayerNorm backward (eps 1e-6, 1024 wide).  g = dL/d(LN output) [rows,1024], y = LN input, stats = its partial sums.
//   yhat = (y - mu) rstd;  gg = gamma * g;  dy = rstd (gg - mean(gg) - yhat mean(gg yhat))
// One warp per row (lane owns 4 x 8 channels), rows strided over the grid; per-CTA column partials of
// dgamma = sum_r g yhat, dbeta = sum_r g and sum_r dy (the bias gradient of the linear layer that feeds this LayerNorm, summed over
// the ROUNDED dy that is stored) are written to partial[blockIdx][3][1024] (fp32) for ln_param_reduce_kernel.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) ln_bwd_kernel(const __nv_bfloat16* __restrict__ g, const __nv_bfloat16* __restrict__ y,
                                                     const float* __restrict__ stats, const __nv_bfloat16* __restrict__ gamma,
                                                     __nv_bfloat16* __restrict__ dy, float* __restrict__ partial, long long rows) {
  __shared__ float s_part[8][3][kC / 4];   // staged in 4 passes of 256 columns to keep smem small
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float gam[4][8];
#pragma unroll
  for (int i = 0; i < 4; ++i) unpack8(__ldg(reinterpret_cast<const uint4*>(gamma + i * 256 + lane * 8)), gam[i]);
  float dg[4][8], db[4][8], ds[4][8];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) dg[i][j] = db[i][j] = ds[i][j] = 0.f;
  for (long long row = static_cast<long long>(blockIdx.x) * 8 + warp; row < rows; row += static_cast<long long>(gridDim.x) * 8) {
    float mu, rstd;
    row_mean_rstd(stats, row, mu, rstd);
    float gv[4][8], yh[4][8];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float yv[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(g + row * kC + i * 256 + lane * 8)), gv[i]);
      unpack8(__ldg(reinterpret_cast<const uint4*>(y + row * kC + i * 256 + lane * 8)), yv);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        yh[i][j] = (yv[j] - mu) * rstd;
        const float gg = gam[i][j] * gv[i][j];
        s1 += gg;
        s2 = fmaf(gg, yh[i][j], s2);
        dg[i][j] = fmaf(gv[i][j], yh[i][j], dg[i][j]);
        db[i][j] += gv[i][j];
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      s1 += __shfl_xor_sync(0xffffffffu, s1, off);
      s2 += __shfl_xor_sync(0xffffffffu, s2, off);
    }
    const float c1 = s1 * (1.0f / kC), c2 = s2 * (1.0f / kC);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = rstd * (gam[i][j] * gv[i][j] - c1 - yh[i][j] * c2);
      const uint4 pk = pack8(o);
      *reinterpret_cast<uint4*>(dy + row * kC + i * 256 + lane * 8) = pk;
      unpack8(pk, o);
#pragma unroll
      for (int j = 0; j < 8; ++j) ds[i][j] += o[j];
    }
  }
  // cross-warp reduction of the column partials, 256 columns (one channel block i) at a time
#pragma unroll
  for (int i = 0; i < 4; ++i) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      s_part[warp][0][lane * 8 + j] = dg[i][j];
      s_part[warp][1][lane * 8 + j] = db[i][j];
      s_part[warp][2][lane * 8 + j] = ds[i][j];
    }
    __syncthreads();
    for (int idx = threadIdx.x; idx < 3 * 256; idx += blockDim.x) {
      const int which = idx >> 8, c = idx & 255;
      float acc = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) acc += s_part[w][which][c];
      partial[(static_cast<long long>(blockIdx.x) * 3 + which) * kC + i * 256 + c] = acc;
    }
    __syncthreads();
  }
}

// dgamma / dbeta / dbias = sum over CTAs of the partials (fixed order -> deterministic); dbias (the column sums of dy) may be nullptr
__global__ void __launch_bounds__(32 * kReduceLanes) ln_param_reduce_kernel(const float* __restrict__ partial, int n_blocks,
                                                                            __nv_bfloat16* __restrict__ dgamma, __nv_bfloat16* __restrict__ dbeta,
                                                                            __nv_bfloat16* __restrict__ dbias) {
  __shared__ float s_a[kReduceLanes][33], s_b[kReduceLanes][33], s_c[kReduceLanes][33];
  const int c = blockIdx.x * 32 + threadIdx.x;        // kC is a multiple of 32
  float a = 0.f, b = 0.f, d = 0.f;
  for (int i = threadIdx.y; i < n_blocks; i += kReduceLanes) {
    a += partial[(static_cast<long long>(i) * 3 + 0) * kC + c];
    b += partial[(static_cast<long long>(i) * 3 + 1) * kC + c];
    d += partial[(static_cast<long long>(i) * 3 + 2) * kC + c];
  }
  s_a[threadIdx.y][threadIdx.x] = a;
  s_b[threadIdx.y][threadIdx.x] = b;
  s_c[threadIdx.y][threadIdx.x] = d;
  __syncthreads();
  if (threadIdx.y == 0) {
    float ta = 0.f, tb = 0.f, tc = 0.f;
#pragma unroll
    for (int j = 0; j < kReduceLanes; ++j) {
      ta += s_a[j][threadIdx.x];
      tb += s_b[j][threadIdx.x];
      tc += s_c[j][threadIdx.x];
    }
    dgamma[c] = __float2bfloat16_rn(ta);
    dbeta[c] = __float2bfloat16_rn(tb);
    if (dbias != nullptr) dbias[c] = __float2bfloat16_rn(tc);
  }
}

// ------------------------------------------------------------------------------------------------
// Window attention backward.  Forward (window_attn_kernel): p = softmax_j(q'_h . k'_{j,h}), ctx_h = sum_j p_j v'_{j,h}.
//   dv'_j = p_j dctx_h;  dp_j = dctx_h . v'_j;  ds_j = p_j (dp_j - sum_i p_i dp_i);  dq'_h = sum_j ds_j k'_j;  dk'_j = ds_j q'_h
// Every fine token belongs to exactly one query window, so dk'/dv' rows are written once: no atomics.  One warp per query,
// same channel ownership as the forward kernel.
// ------------------------------------------------------------------------------------------------
template <int S>
__global__ void __launch_bounds__(256) window_attn_bwd_kernel(const __nv_bfloat16* __restrict__ qp, const __nv_bfloat16* __restrict__ kp,
                                                              const __nv_bfloat16* __restrict__ vp, const __nv_bfloat16* __restrict__ dctx,
                                                              __nv_bfloat16* __restrict__ dqp, __nv_bfloat16* __restrict__ dkp,
                                                              __nv_bfloat16* __restrict__ dvp, long long n_queries) {
  constexpr int G = kGrid / S;
  constexpr int M = G * G;
  constexpr int W = S * S;
  const long long query = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (query >= n_queries) return;
  const long long n = query / M;
  const int m = static_cast<int>(query - n * M);
  const int hb = m / G, wb = m - hb * G;
  const long long tok0 = n * kTokens + static_cast<long long>(hb * S) * kGrid + wb * S;

  float qf[4][8], dc[4][8];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    unpack8(__ldg(reinterpret_cast<const uint4*>(qp + query * kC + i * 256 + lane * 8)), qf[i]);
    unpack8(__ldg(reinterpret_cast<const uint4*>(dctx + query * kC + i * 256 + lane * 8)), dc[i]);
  }
  float sc[4][W], dp[4][W];
#pragma unroll
  for (int j = 0; j < W; ++j) {
    const long long tok = tok0 + (j / S) * kGrid + (j % S);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float kf[8], vf[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(kp + tok * kC + i * 256 + lane * 8)), kf);
      unpack8(__ldg(reinterpret_cast<const uint4*>(vp + tok * kC + i * 256 + lane * 8)), vf);
      float d = 0.f, e = 0.f;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        d = fmaf(qf[i][c], kf[c], d);
        e = fmaf(dc[i][c], vf[c], e);
      }
      sc[i][j] = d;
      dp[i][j] = e;
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < W; ++j) {
      float d = sc[i][j], e = dp[i][j];
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) {
        d += __shfl_xor_sync(0xffffffffu, d, off);
        e += __shfl_xor_sync(0xffffffffu, e, off);
      }
      sc[i][j] = d;
      dp[i][j] = e;
    }
  // p (into sc) and ds (into dp)
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
    float dot = 0.f;
#pragma unroll
    for (int j = 0; j < W; ++j) {
      sc[i][j] *= inv;
      dot = fmaf(sc[i][j], dp[i][j], dot);
    }
#pragma unroll
    for (int j = 0; j < W; ++j) dp[i][j] = sc[i][j] * (dp[i][j] - dot);
  }
  float dq[4][8];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int c = 0; c < 8; ++c) dq[i][c] = 0.f;
#pragma unroll
  for (int j = 0; j < W; ++j) {
    const long long tok = tok0 + (j / S) * kGrid + (j % S);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float kf[8], dk[8], dv[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(kp + tok * kC + i * 256 + lane * 8)), kf);
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        dq[i][c] = fmaf(dp[i][j], kf[c], dq[i][c]);
        dk[c] = dp[i][j] * qf[i][c];
        dv[c] = sc[i][j] * dc[i][c];
      }
      *reinterpret_cast<uint4*>(dkp + tok * kC + i * 256 + lane * 8) = pack8(dk);
      *reinterpret_cast<uint4*>(dvp + tok * kC + i * 256 + lane * 8) = pack8(dv);
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) *reinterpret_cast<uint4*>(dqp + query * kC + i * 256 + lane * 8) = pack8(dq[i]);
}

// Backward for any window size (scale_factor 1, 6, 8, 12, 24): two passes over the window's keys.  Pass A streams
// (s_j, dp_j) through an online softmax to get the row maximum, the denominator and sum_j p_j dp_j; pass B recomputes
// p_j and emits dk'_j, dv'_j (written once: every fine token belongs to exactly one window) and accumulates dq'.
__global__ void __launch_bounds__(256) window_attn_bwd_stream_kernel(const __nv_bfloat16* __restrict__ qp, const __nv_bfloat16* __restrict__ kp,
                                                                     const __nv_bfloat16* __restrict__ vp, const __nv_bfloat16* __restrict__ dctx,
                                                                     __nv_bfloat16* __restrict__ dqp, __nv_bfloat16* __restrict__ dkp,
                                                                     __nv_bfloat16* __restrict__ dvp, long long n_queries, int s) {
  const int G = kGrid / s;
  const int M = G * G;
  const int W = s * s;
  const long long query = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (query >= n_queries) return;
  const long long n = query / M;
  const int m = static_cast<int>(query - n * M);
  const int hb = m / G, wb = m - hb * G;
  const long long tok0 = n * kTokens + static_cast<long long>(hb * s) * kGrid + wb * s;

  float qf[4][8], dc[4][8];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    unpack8(__ldg(reinterpret_cast<const uint4*>(qp + query * kC + i * 256 + lane * 8)), qf[i]);
    unpack8(__ldg(reinterpret_cast<const uint4*>(dctx + query * kC + i * 256 + lane * 8)), dc[i]);
  }
  // (s_j, dp_j) for channel block i of key j, reduced over the head's 16 lanes
  auto scores = [&](long long tok, int i, float& sc, float& dp) {
    float kf[8], vf[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(kp + tok * kC + i * 256 + lane * 8)), kf);
    unpack8(__ldg(reinterpret_cast<const uint4*>(vp + tok * kC + i * 256 + lane * 8)), vf);
    float d = 0.f, e = 0.f;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      d = fmaf(qf[i][c], kf[c], d);
      e = fmaf(dc[i][c], vf[c], e);
    }
#pragma unroll
    for (int off = 8; off > 0; off >>= 1) {
      d += __shfl_xor_sync(0xffffffffu, d, off);
      e += __shfl_xor_sync(0xffffffffu, e, off);
    }
    sc = d;
    dp = e;
  };
  float mx[4], den[4], num[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    mx[i] = -INFINITY;
    den[i] = 0.f;
    num[i] = 0.f;
  }
  for (int j = 0; j < W; ++j) {
    const int hi = j / s;
    const long long tok = tok0 + static_cast<long long>(hi) * kGrid + (j - hi * s);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float sc, dp;
      scores(tok, i, sc, dp);
      const float m_new = fmaxf(mx[i], sc);
      const float corr = __expf(mx[i] - m_new);
      const float pj = __expf(sc - m_new);
      den[i] = fmaf(den[i], corr, pj);
      num[i] = fmaf(num[i], corr, pj * dp);
      mx[i] = m_new;
    }
  }
  float inv[4], dot[4], dq[4][8];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    inv[i] = 1.0f / den[i];
    dot[i] = num[i] * inv[i];
#pragma unroll
    for (int c = 0; c < 8; ++c) dq[i][c] = 0.f;
  }
  for (int j = 0; j < W; ++j) {
    const int hi = j / s;
    const long long tok = tok0 + static_cast<long long>(hi) * kGrid + (j - hi * s);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float sc, dp;
      scores(tok, i, sc, dp);
      const float pj = __expf(sc - mx[i]) * inv[i];
      const float ds = pj * (dp - dot[i]);
      float kf[8], dk[8], dv[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(kp + tok * kC + i * 256 + lane * 8)), kf);
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        dq[i][c] = fmaf(ds, kf[c], dq[i][c]);
        dk[c] = ds * qf[i][c];
        dv[c] = pj * dc[i][c];
      }
      *reinterpret_cast<uint4*>(dkp + tok * kC + i * 256 + lane * 8) = pack8(dk);
      *reinterpret_cast<uint4*>(dvp + tok * kC + i * 256 + lane * 8) = pack8(dv);
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) *reinterpret_cast<uint4*>(dqp + query * kC + i * 256 + lane * 8) = pack8(dq[i]);
}

// Split-K epilogue: out[i] = bf16(alpha * sum_s partial[s][i]), slices summed in fixed order (deterministic).  4 elements per thread.
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const float* __restrict__ partial, int splits, long long slice_elems,
                                                            float alpha, __nv_bfloat16* __restrict__ out) {
  const long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 4;
  if (i >= slice_elems) return;
  float4 acc = __ldg(reinterpret_cast<const float4*>(partial + i));
  for (int s = 1; s < splits; ++s) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(partial + s * slice_elems + i));
    acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
  }
  uint2 o;
  o.x = pack_bf16x2(acc.x * alpha, acc.y * alpha);
  o.y = pack_bf16x2(acc.z * alpha, acc.w * alpha);
  *reinterpret_cast<uint2*>(out + i) = o;
}

// ------------------------------------------------------------------------------------------------
// Point-query stencil backwards (the transpose of point_query_kernel): dx0 [n_tokens, 1024] from dq [N g^2, 1024].
// With align_corners=False and no edge clamping for any divisor s of 24, every fine token is a tap of at most one query, its own
// window's, so the transpose is a gather: per fine token (r, c) of crop n, with m = (r / s) g + c / s,
//   odd s:  dx0 = dq[n, m] at the window's centre token, 0 elsewhere;
//   even s: dx0 = bf16(0.25 float(dq[n, m])) on the centre 2x2, 0 elsewhere (s = 2: every token).
// That is the reference's upsample_bilinear2d backward (weights 0.5 x 0.5, fp32) followed by the bf16 rounding of .float()'s
// backward; 0.25 x is exact in fp32, so the bits match given the same dq.  Writes every element, zeros included.
// One thread per 8 channels of one fine token.
// ------------------------------------------------------------------------------------------------
// The 8 bf16 values of fine token t of crop n, channels [8 vec, 8 vec + 8)
template <int S>
__device__ __forceinline__ uint4 point_query_bwd_value(const __nv_bfloat16* __restrict__ dq, long long n, int t, int vec) {
  constexpr int G = kGrid / S;
  constexpr int M = G * G;
  constexpr int kLo = (S % 2 == 1) ? (S - 1) / 2 : S / 2 - 1;     // first tap row / column inside the window
  constexpr int kHi = (S % 2 == 1) ? kLo : kLo + 1;               // last
  const int r = t / kGrid, c = t - r * kGrid;
  const int hb = r / S, wb = c / S;
  const int ri = r - hb * S, ci = c - wb * S;
  uint4 out = make_uint4(0u, 0u, 0u, 0u);
  if (ri >= kLo && ri <= kHi && ci >= kLo && ci <= kHi) {
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(dq + (n * M + hb * G + wb) * kC + vec * 8));
    if (S % 2 == 1) {
      out = v;
    } else {
      float f[8];
      unpack8(v, f);
#pragma unroll
      for (int i = 0; i < 8; ++i) f[i] = __fmul_rn(0.25f, f[i]);
      out = pack8(f);
    }
  }
  return out;
}

template <int S>
__global__ void __launch_bounds__(256) point_query_bwd_kernel(const __nv_bfloat16* __restrict__ dq, __nv_bfloat16* __restrict__ dx0,
                                                              long long n_tokens) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long tok = idx >> 7;            // 128 vectors of 8 channels per token
  const int vec = static_cast<int>(idx & 127);
  if (tok >= n_tokens) return;
  const long long n = tok / kTokens;
  const int t = static_cast<int>(tok - n * kTokens);
  *reinterpret_cast<uint4*>(dx0 + tok * kC + vec * 8) = point_query_bwd_value<S>(dq, n, t, vec);
}

// The same stencil ADDED to a crop-strided destination that already holds another gradient of the same tensor (CLIP layer 23 is both
// feat and the last quarter of feat_multi): dx = bf16(float(dx) + float(v)) with v the bf16 value point_query_bwd_kernel stores —
// autograd's bf16 sum of the two paths.  Every token is read, modified and written, so a -0.0 left by the other path becomes
// -0.0 + +0.0 = +0.0 on the tokens the stencil does not touch, exactly as the sum makes it.
template <int S>
__global__ void __launch_bounds__(256) point_query_bwd_acc_kernel(const __nv_bfloat16* __restrict__ dq, __nv_bfloat16* __restrict__ dx,
                                                                  long long crop_stride, long long n_tokens) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long tok = idx >> 7;
  const int vec = static_cast<int>(idx & 127);
  if (tok >= n_tokens) return;
  const long long n = tok / kTokens;
  const int t = static_cast<int>(tok - n * kTokens);
  uint4* p = reinterpret_cast<uint4*>(dx + n * crop_stride + static_cast<long long>(t) * kC + vec * 8);
  float a[8], b[8];
  unpack8(*p, a);
  unpack8(point_query_bwd_value<S>(dq, n, t, vec), b);
#pragma unroll
  for (int i = 0; i < 8; ++i) a[i] = __fadd_rn(a[i], b[i]);
  *p = pack8(a);
}

}  // namespace tp
