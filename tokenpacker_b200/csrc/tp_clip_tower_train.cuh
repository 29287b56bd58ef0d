// Kernels of the CLIP tower's training path that are not GEMMs (include/tokenpacker_b200_clip_tower_train.h):
//   clip_quick_gelu_fwd_kernel      fc1's fp32 pre-activation -> z (bf16, kept for the backward) and quick_gelu(z) with the fused epilogue's bits
//   quick_gelu_bwd_colsum_kernel    dz = dh quick_gelu'(z) in place + the column partials of fc1's bias gradient
//   clip_ln_bwd_kernel              LayerNorm backward (statistics recomputed from the row) + the residual carry, dgamma / dbeta partials
//   clip_carry_init_kernel          the carry of the top layer from the caller's gradient of hidden_states[23]
//   clip_attn_delta_kernel          D = rowsum(dO o O) per (crop, head, token)
//   clip_attn_bwd_kernel            the 577-token attention backward on wgmma: dQ (kKV = false) or dK and dV (kKV = true)
// bf16 storage, fp32 arithmetic.  The forward's kernels are tp_clip_tower.cuh's (clip_attn_kernel with kLse = true keeps the softmax
// statistics).
#pragma once

#include "tp_backward.cuh"
#include "tp_clip_tower.cuh"

namespace tp {

// z32 [n8 * 8] fp32 (fc1's accumulator + bias, unrounded) -> z = bf16(z32), h = bf16(quick_gelu(z32)): the value and the single rounding
// of the inference path's fused fc1 epilogue (tp_gemm.cuh: quick_gelu_pk on the fp32 sum, then pack_x2)
__global__ void __launch_bounds__(256) clip_quick_gelu_fwd_kernel(const float* __restrict__ z32, __nv_bfloat16* __restrict__ z,
                                                                  __nv_bfloat16* __restrict__ h, long long n8) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n8) return;
  const float4 a = *reinterpret_cast<const float4*>(z32 + i * 8), b = *reinterpret_cast<const float4*>(z32 + i * 8 + 4);
  const float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
  uint32_t zo[4], ho[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    float lo, hi;
    upk2(quick_gelu_pk(pk2(f[2 * k], f[2 * k + 1])), lo, hi);
    zo[k] = pack_bf16x2(f[2 * k], f[2 * k + 1]);
    ho[k] = pack_bf16x2(lo, hi);
  }
  *reinterpret_cast<uint4*>(z + i * 8) = make_uint4(zo[0], zo[1], zo[2], zo[3]);
  *reinterpret_cast<uint4*>(h + i * 8) = make_uint4(ho[0], ho[1], ho[2], ho[3]);
}

// d/dz [z sigmoid(1.702 z)] = s (1 + 1.702 z (1 - s)), s = sigmoid(1.702 z).  Large |z|: exp overflows to +inf -> s = 0 -> 0; exp
// underflows to 0 -> s = 1 -> 1; (1 - s) z is formed first so that no inf * 0 appears for any finite z.  Below z = -2e38, 1.702 z itself
// overflows to -inf inside the fma and 0 * -inf would be NaN: (1 - s) z is clamped at -1e38 (s = 0 there already, so no other z changes).
__device__ __forceinline__ float quick_gelu_grad(float z) {
  const float s = 1.0f / (1.0f + __expf(-1.702f * z));
  return s * fmaf(1.702f, fmaxf((1.0f - s) * z, -1e38f), 1.0f);
}

// gelu_bwd_colsum_kernel (tp_backward.cuh) for quick_gelu: dz = dh quick_gelu'(z) in place over dh, fused with the first stage of fc1's
// bias gradient (column sums of the ROUNDED dz, in row order).  grid = (ceil(cols / 1024), n_chunks), 128 threads.
__global__ void __launch_bounds__(128) quick_gelu_bwd_colsum_kernel(__nv_bfloat16* __restrict__ dh, const __nv_bfloat16* __restrict__ z,
                                                                    long long ld, long long rows, int cols, int n_chunks,
                                                                    float* __restrict__ partial) {
  const int c0 = (blockIdx.x * 128 + threadIdx.x) * 8;
  if (c0 >= cols) return;
  const long long per = (rows + n_chunks - 1) / n_chunks;
  const long long r0 = per * blockIdx.y, r1 = min(rows, r0 + per);
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (long long r = r0; r < r1; ++r) {
    float g[8], zz[8];
    unpack8(*reinterpret_cast<const uint4*>(dh + r * ld + c0), g);
    unpack8(__ldg(reinterpret_cast<const uint4*>(z + r * ld + c0)), zz);
#pragma unroll
    for (int j = 0; j < 8; ++j) g[j] *= quick_gelu_grad(zz[j]);
    const uint4 o = pack8(g);
    *reinterpret_cast<uint4*>(dh + r * ld + c0) = o;
    unpack8(o, g);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] += g[j];
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) partial[static_cast<long long>(blockIdx.y) * cols + c0 + j] = acc[j];
}

// carry32 = fp32(d_out), carry16 = d_out (d_out == nullptr: zeros): the gradient of the top layer's output
__global__ void __launch_bounds__(256) clip_carry_init_kernel(const __nv_bfloat16* __restrict__ d_out, float* __restrict__ carry32,
                                                              __nv_bfloat16* __restrict__ carry16, long long n8) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n8) return;
  const uint4 v = d_out != nullptr ? __ldg(reinterpret_cast<const uint4*>(d_out + i * 8)) : make_uint4(0, 0, 0, 0);
  float f[8];
  unpack8(v, f);
  *reinterpret_cast<float4*>(carry32 + i * 8) = make_float4(f[0], f[1], f[2], f[3]);
  *reinterpret_cast<float4*>(carry32 + i * 8 + 4) = make_float4(f[4], f[5], f[6], f[7]);
  *reinterpret_cast<uint4*>(carry16 + i * 8) = v;
}

// ------------------------------------------------------------------------------------------------
// LayerNorm backward of the tower (eps 1e-5, 1024 wide) with the residual carry.  g = dL/d(LN output) [rows, 1024] bf16; x = the LN
// input (T = bf16: a hidden state, layer_norm1; T = float: the mid-layer residual x', layer_norm2), whose mean and rstd are
// recomputed exactly as clip_ln_row_store computes them;
//   xhat = (x - mu) rstd;  gg = gamma g;  dLN = rstd (gg - mean(gg) - xhat mean(gg xhat))
//   carry32 <- carry32 + dLN (+ add, the caller's gradient of this hidden state);  carry16 = bf16(carry32)
// The carry is the gradient of the residual stream: fp32 in memory (one bf16 rounding per use as a GEMM operand, none accumulated
// from layer to layer).  One warp per row, rows strided over the grid; per-CTA column partials [blockIdx][3][1024] of
// dgamma = sum g xhat, dbeta = sum g and sum carry16 (the bias gradient of the linear whose output this residual stream is, summed over
// the ROUNDED values its weight gradient reads) for ln_param_reduce_kernel.
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) clip_ln_bwd_kernel(const __nv_bfloat16* __restrict__ g, const T* __restrict__ x,
                                                          const __nv_bfloat16* __restrict__ gamma, const __nv_bfloat16* __restrict__ add,
                                                          float* __restrict__ carry32, __nv_bfloat16* __restrict__ carry16,
                                                          float* __restrict__ partial, long long rows) {
  __shared__ float s_part[8][3][kC / 4];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float gam[32], dg[32], db[32], ds[32];
  clip_load_row(gamma, gam, lane);
#pragma unroll
  for (int i = 0; i < 32; ++i) dg[i] = db[i] = ds[i] = 0.f;
  for (long long row = static_cast<long long>(blockIdx.x) * 8 + warp; row < rows; row += static_cast<long long>(gridDim.x) * 8) {
    float e[32], gv[32];
    clip_load_row(x + row * kC, e, lane);
    clip_load_row(g + row * kC, gv, lane);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 32; ++i) s += e[i];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    const float mean = s * (1.0f / 1024);
    float v = 0.f;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      e[i] -= mean;
      v = fmaf(e[i], e[i], v);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    const float rstd = rsqrtf(v * (1.0f / 1024) + kClipLnEps);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      e[i] *= rstd;                                  // xhat
      const float gg = gam[i] * gv[i];
      s1 += gg;
      s2 = fmaf(gg, e[i], s2);
      dg[i] = fmaf(gv[i], e[i], dg[i]);
      db[i] += gv[i];
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      s1 += __shfl_xor_sync(0xffffffffu, s1, off);
      s2 += __shfl_xor_sync(0xffffffffu, s2, off);
    }
    const float c1 = s1 * (1.0f / kC), c2 = s2 * (1.0f / kC);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long long at = row * kC + 256 * j + 8 * lane;
      const float4 ca = *reinterpret_cast<const float4*>(carry32 + at), cb = *reinterpret_cast<const float4*>(carry32 + at + 4);
      float o[8] = {ca.x, ca.y, ca.z, ca.w, cb.x, cb.y, cb.z, cb.w};
      if (add != nullptr) {
        float a[8];
        unpack8(__ldg(reinterpret_cast<const uint4*>(add + at)), a);
#pragma unroll
        for (int k = 0; k < 8; ++k) o[k] += a[k];
      }
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int i = 8 * j + k;
        o[k] += rstd * (gam[i] * gv[i] - c1 - e[i] * c2);
      }
      *reinterpret_cast<float4*>(carry32 + at) = make_float4(o[0], o[1], o[2], o[3]);
      *reinterpret_cast<float4*>(carry32 + at + 4) = make_float4(o[4], o[5], o[6], o[7]);
      const uint4 pk = pack8(o);
      *reinterpret_cast<uint4*>(carry16 + at) = pk;
      unpack8(pk, o);
#pragma unroll
      for (int k = 0; k < 8; ++k) ds[8 * j + k] += o[k];
    }
  }
  // cross-warp reduction of the column partials, 256 columns (one channel block j) at a time
#pragma unroll
  for (int j = 0; j < 4; ++j) {
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      s_part[warp][0][lane * 8 + k] = dg[8 * j + k];
      s_part[warp][1][lane * 8 + k] = db[8 * j + k];
      s_part[warp][2][lane * 8 + k] = ds[8 * j + k];
    }
    __syncthreads();
    for (int idx = threadIdx.x; idx < 3 * 256; idx += blockDim.x) {
      const int which = idx >> 8, col = idx & 255;
      float acc = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) acc += s_part[w][which][col];
      partial[(static_cast<long long>(blockIdx.x) * 3 + which) * kC + j * 256 + col] = acc;
    }
    __syncthreads();
  }
}

// D[crop][head][t] = sum over the head's 64 channels of dO o O (dctx and ctx, [rows, 1024] bf16): one warp per token row.  Lane l
// holds channels 256 j + 8 l + [0, 8): head 4 j + l / 8, so eight lanes share a head.
__global__ void __launch_bounds__(256) clip_attn_delta_kernel(const __nv_bfloat16* __restrict__ dctx, const __nv_bfloat16* __restrict__ ctx,
                                                              float* __restrict__ delta, long long rows) {
  const long long row = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  float a[32], b[32];
  clip_load_row(dctx + row * kC, a, lane);
  clip_load_row(ctx + row * kC, b, lane);
  const long long crop = row / kClipTokens;
  const int t = static_cast<int>(row - crop * kClipTokens);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) s = fmaf(a[8 * j + k], b[8 * j + k], s);
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    s += __shfl_xor_sync(0xffffffffu, s, 4);
    if ((lane & 7) == 0) delta[(crop * kClipHeads + 4 * j + (lane >> 3)) * kClipStatLd + t] = s;
  }
}

// ------------------------------------------------------------------------------------------------
// Attention backward over the 577 tokens of one crop and one head.  With q (scaled), k, v as the forward read them, dO = dctx,
// LSE = log2 of the forward's softmax denominator (clip_attn_kernel, kLse) and D as above:
//   S = Q K^T;  P = exp2(S log2 e - LSE);  dP = dO V^T;  dS = P o (dP - D);  dV = P^T dO;  dK = dS^T Q;  dQ = dS K
// Two instantiations of one kernel, as in FlashAttention-2's split.  A CTA owns a block of 128 "rows" (two warpgroups of 64) and
// walks all 640 "columns" in blocks of 64; nothing is accumulated across CTAs, so there are no atomics and the result is deterministic:
//   kKV = false  rows = queries (R1 = Q, R2 = dO), columns = keys (C1 = K, C2 = V):   X = R1 C1^T = S,   Y = R2 C2^T = dP,
//                acc1 = dS C1 = dQ
//   kKV = true   rows = keys (R1 = K, R2 = V), columns = queries (C1 = Q, C2 = dO):   X = S^T, Y = dP^T (LSE and D indexed by column),
//                acc1 = dS^T C1 = dK,  acc2 = P^T C2 = dV
// so both have the forward's operand forms: X and Y are K-major x K-major wgmma m64n64k16 (contraction over the 64 channels), P and
// dS are rounded to bf16 into shared memory as K-major A tiles, and C1 / C2 are their MN-major B operands (contraction over the
// block's 64 columns).  Operands arrive by TMA through the forward's 3-D (column, token, crop) maps with token extent 577: rows past
// token 576 are zero-filled.  A column >= 577 gets P = dS = 0 by selection (a zero-filled key scores 0, not -inf; a padded query's
// LSE and D are never written), so it contributes nothing; a row >= 577 only ever touches its own accumulator row, which is not stored.
// ------------------------------------------------------------------------------------------------
constexpr int kAttnBwdColBoxes = 10;                      // 640 >= 577 columns in boxes of 64
struct ClipAttnBwdSmem {
  static constexpr int kR1 = 0;                           // [2 warpgroups][64 x 64]
  static constexpr int kR2 = kR1 + 2 * kAttnBoxBytes;
  static constexpr int kC1 = kR2 + 2 * kAttnBoxBytes;     // [640 x 64]
  static constexpr int kC2 = kC1 + kAttnBwdColBoxes * kAttnBoxBytes;
  static constexpr int kP = kC2 + kAttnBwdColBoxes * kAttnBoxBytes;   // [2 warpgroups][64 x 64]  (kKV only)
  static constexpr int kDS = kP + 2 * kAttnBoxBytes;      // [2 warpgroups][64 x 64]
  static constexpr int kBar = kDS + 2 * kAttnBoxBytes;
  static constexpr int kBytes = kBar + 16 + 1024;         // + alignment slack
};
static_assert(ClipAttnBwdSmem::kBytes <= 232448, "shared memory budget of an sm_90 SM (227 KiB)");

template <bool kKV>
__global__ void __launch_bounds__(256, 1)
clip_attn_bwd_kernel(const __grid_constant__ CUtensorMap tmap_qkv, const __grid_constant__ CUtensorMap tmap_do,
                     const float* __restrict__ lse, const float* __restrict__ delta, __nv_bfloat16* __restrict__ dqkv) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + ClipAttnBwdSmem::kBar);
  const int rb = blockIdx.x, head = blockIdx.y, crop = blockIdx.z;
  const int tid = threadIdx.x;
  if (tid == 0) {
    tma_prefetch_desc(&tmap_qkv);
    tma_prefetch_desc(&tmap_do);
    mbar_init(bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  const int ch = head * kClipHeadDim;
  if (tid == 0) {
    mbar_arrive_expect_tx(bar, (4 + 2 * kAttnBwdColBoxes) * kAttnBoxBytes);
    for (int w = 0; w < 2; ++w) {
      const int t0 = rb * 128 + w * 64;
      if (kKV) {
        tma_load_3d(smem + ClipAttnBwdSmem::kR1 + w * kAttnBoxBytes, &tmap_qkv, bar, 1024 + ch, t0, crop);
        tma_load_3d(smem + ClipAttnBwdSmem::kR2 + w * kAttnBoxBytes, &tmap_qkv, bar, 2048 + ch, t0, crop);
      } else {
        tma_load_3d(smem + ClipAttnBwdSmem::kR1 + w * kAttnBoxBytes, &tmap_qkv, bar, ch, t0, crop);
        tma_load_3d(smem + ClipAttnBwdSmem::kR2 + w * kAttnBoxBytes, &tmap_do, bar, ch, t0, crop);
      }
    }
    for (int b = 0; b < kAttnBwdColBoxes; ++b) {
      if (kKV) {
        tma_load_3d(smem + ClipAttnBwdSmem::kC1 + b * kAttnBoxBytes, &tmap_qkv, bar, ch, b * 64, crop);
        tma_load_3d(smem + ClipAttnBwdSmem::kC2 + b * kAttnBoxBytes, &tmap_do, bar, ch, b * 64, crop);
      } else {
        tma_load_3d(smem + ClipAttnBwdSmem::kC1 + b * kAttnBoxBytes, &tmap_qkv, bar, 1024 + ch, b * 64, crop);
        tma_load_3d(smem + ClipAttnBwdSmem::kC2 + b * kAttnBoxBytes, &tmap_qkv, bar, 2048 + ch, b * 64, crop);
      }
    }
  }
  const int wg = tid >> 7;                                 // warpgroup: rows 64 wg .. + 63 of the block
  const int warp = (tid >> 5) & 3, lane = tid & 31;
  const int g = lane >> 2, q = lane & 3;
  const uint32_t sr1 = smem_u32(smem + ClipAttnBwdSmem::kR1 + wg * kAttnBoxBytes);
  const uint32_t sr2 = smem_u32(smem + ClipAttnBwdSmem::kR2 + wg * kAttnBoxBytes);
  const uint32_t sc1 = smem_u32(smem + ClipAttnBwdSmem::kC1), sc2 = smem_u32(smem + ClipAttnBwdSmem::kC2);
  const uint32_t sp = smem_u32(smem + ClipAttnBwdSmem::kP + wg * kAttnBoxBytes);
  const uint32_t sds = smem_u32(smem + ClipAttnBwdSmem::kDS + wg * kAttnBoxBytes);
  constexpr float kLog2e = 1.4426950408889634f;
  const float* lse_h = lse + (static_cast<long long>(crop) * kClipHeads + head) * kClipStatLd;
  const float* delta_h = delta + (static_cast<long long>(crop) * kClipHeads + head) * kClipStatLd;
  const int row0 = rb * 128 + wg * 64 + 16 * warp + g;     // this thread's rows: row0 and row0 + 8 (< 640)
  float lse_r[2] = {0.f, 0.f}, d_r[2] = {0.f, 0.f};
  if (!kKV) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      lse_r[h] = __ldg(lse_h + row0 + 8 * h);
      d_r[h] = __ldg(delta_h + row0 + 8 * h);
    }
  }
  float acc1[32], acc2[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc1[i] = acc2[i] = 0.f;
  mbar_wait(bar, 0);
  for (int cb = 0; cb < kAttnBwdColBoxes; ++cb) {
    float s[32], dp[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) s[i] = dp[i] = 0.f;
    fence_regs(s);
    fence_regs(dp);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kClipHeadDim / kUmmaK; ++k)
      wgmma_m64n64<0, 0>(s, make_smem_desc_kmajor_sw128(sr1) + static_cast<uint64_t>(k * 2),
                         make_smem_desc_kmajor_sw128(sc1 + cb * kAttnBoxBytes) + static_cast<uint64_t>(k * 2), static_cast<uint32_t>(k != 0));
#pragma unroll
    for (int k = 0; k < kClipHeadDim / kUmmaK; ++k)
      wgmma_m64n64<0, 0>(dp, make_smem_desc_kmajor_sw128(sr2) + static_cast<uint64_t>(k * 2),
                         make_smem_desc_kmajor_sw128(sc2 + cb * kAttnBoxBytes) + static_cast<uint64_t>(k * 2), static_cast<uint32_t>(k != 0));
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);
    fence_regs(dp);
    named_bar_sync(1 + wg, 128);                           // the previous block's wgmmas of the whole warpgroup have read P and dS
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int h = (i >> 1) & 1;
      const int col = 8 * (i >> 2) + 2 * q;                // columns col, col + 1 of the block
      const int tok = cb * 64 + col;
      float l0 = lse_r[h], l1 = lse_r[h], d0 = d_r[h], d1 = d_r[h];
      if (kKV) {
        const float2 lv = __ldg(reinterpret_cast<const float2*>(lse_h + tok)), dv = __ldg(reinterpret_cast<const float2*>(delta_h + tok));
        l0 = lv.x; l1 = lv.y; d0 = dv.x; d1 = dv.y;
      }
      const bool ok0 = tok < kClipTokens, ok1 = tok + 1 < kClipTokens;
      const float p0 = ok0 ? ex2_approx(fmaf(s[i], kLog2e, -l0)) : 0.f;
      const float p1 = ok1 ? ex2_approx(fmaf(s[i + 1], kLog2e, -l1)) : 0.f;
      const float ds0 = ok0 ? p0 * (dp[i] - d0) : 0.f;
      const float ds1 = ok1 ? p1 * (dp[i + 1] - d1) : 0.f;
      // K-major, 128-byte swizzle: row r's 16-byte chunk c lies at r * 128 + ((c ^ (r & 7)) << 4)
      const int r = 16 * warp + g + 8 * h;
      const uint32_t off = r * 128 + ((((col >> 3) ^ (r & 7)) << 4) | ((col & 7) * 2));
      const uint32_t dsk = pack_bf16x2(ds0, ds1);
      asm volatile("st.shared.b32 [%0], %1;" ::"r"(sds + off), "r"(dsk) : "memory");
      if (kKV) {
        const uint32_t pk = pack_bf16x2(p0, p1);
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(sp + off), "r"(pk) : "memory");
      }
    }
    fence_proxy_async_smem();                              // generic-proxy stores -> visible to wgmma's reads
    named_bar_sync(1 + wg, 128);
    fence_regs(acc1);
    fence_regs(acc2);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 64 / kUmmaK; ++k)
      wgmma_m64n64<0, 1>(acc1, make_smem_desc_kmajor_sw128(sds) + static_cast<uint64_t>(k * 2),
                         make_smem_desc_mnmajor_sw128(sc1 + cb * kAttnBoxBytes, kAttnBoxBytes) + static_cast<uint64_t>(k * 128), 1u);
    if (kKV) {
#pragma unroll
      for (int k = 0; k < 64 / kUmmaK; ++k)
        wgmma_m64n64<0, 1>(acc2, make_smem_desc_kmajor_sw128(sp) + static_cast<uint64_t>(k * 2),
                           make_smem_desc_mnmajor_sw128(sc2 + cb * kAttnBoxBytes, kAttnBoxBytes) + static_cast<uint64_t>(k * 128), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(acc1);
    fence_regs(acc2);
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int t = row0 + 8 * h;
    if (t >= kClipTokens) continue;
    __nv_bfloat16* dst = dqkv + (static_cast<long long>(crop) * kClipTokens + t) * (3 * kC) + (kKV ? kC : 0) + ch + 2 * q;
#pragma unroll
    for (int i = 2 * h; i < 32; i += 4) {
      *reinterpret_cast<uint32_t*>(dst + 8 * (i >> 2)) = pack_bf16x2(acc1[i], acc1[i + 1]);
      if (kKV) *reinterpret_cast<uint32_t*>(dst + kC + 8 * (i >> 2)) = pack_bf16x2(acc2[i], acc2[i + 1]);
    }
  }
}

}  // namespace tp
