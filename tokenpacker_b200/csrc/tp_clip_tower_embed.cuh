// Kernels of the CLIP tower's embedding-stage backward (include/tokenpacker_b200_clip_tower_embed.h):
//   clip_preln_bwd_kernel           pre_layrnorm backward from the fp32 gradient of hidden_states[0], in place, + dgamma / dbeta partials
//   clip_pos_grad_kernel            d position_embedding = the sum over crops of d emb, in crop order (token 0: d class_embedding)
//   clip_patch_grad_reduce_kernel   the patch weight's gradient from the split-K partials of dW^T, transposed to [1024, 588]
// The weight gradient itself is a TN item of the pair GEMM.  bf16 storage, fp32 arithmetic, no atomics.
#pragma once

#include "tp_clip_tower_train.cuh"

namespace tp {

// pre_layrnorm backward, one warp per token row of [rows, 1024] (rows n * 577 + t).  The LayerNorm input is rebuilt exactly as
// clip_embed_preln_kernel formed it, e = fl32((t == 0 ? class_embedding : patch row) + position_embedding[t]), and its statistics as
// clip_ln_row_store computes them.  g is the fp32 gradient of hidden_states[0] (carry32, never rounded);
//   xhat = (e - mu) rstd;  gg = gamma g;  de = rstd (gg - mean(gg) - xhat mean(gg xhat))
// de overwrites carry32 and its bf16 rounding carry16 (the patch weight gradient's operand).  Per-CTA column partials
// [blockIdx][3][1024] of dgamma = sum g xhat and dbeta = sum g (the third slot zero) for ln_param_reduce_kernel.
__global__ void __launch_bounds__(256) clip_preln_bwd_kernel(float* __restrict__ carry32, __nv_bfloat16* __restrict__ carry16,
                                                             const __nv_bfloat16* __restrict__ patch_rows, const __nv_bfloat16* __restrict__ cls,
                                                             const __nv_bfloat16* __restrict__ pos, const __nv_bfloat16* __restrict__ gamma,
                                                             float* __restrict__ partial, long long rows) {
  __shared__ float s_part[8][2][kC / 4];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float gam[32], dg[32], db[32];
  clip_load_row(gamma, gam, lane);
#pragma unroll
  for (int i = 0; i < 32; ++i) dg[i] = db[i] = 0.f;
  for (long long row = static_cast<long long>(blockIdx.x) * 8 + warp; row < rows; row += static_cast<long long>(gridDim.x) * 8) {
    const int t = static_cast<int>(row % kClipTokens);
    float e[32], p[32], gv[32];
    clip_load_row(t == 0 ? cls : patch_rows + row * kC, e, lane);
    clip_load_row(pos + static_cast<long long>(t) * kC, p, lane);
    clip_load_row(carry32 + row * kC, gv, lane);
#pragma unroll
    for (int i = 0; i < 32; ++i) e[i] = __fadd_rn(e[i], p[i]);
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
      float o[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int i = 8 * j + k;
        o[k] = rstd * (gam[i] * gv[i] - c1 - e[i] * c2);
      }
      *reinterpret_cast<float4*>(carry32 + at) = make_float4(o[0], o[1], o[2], o[3]);
      *reinterpret_cast<float4*>(carry32 + at + 4) = make_float4(o[4], o[5], o[6], o[7]);
      *reinterpret_cast<uint4*>(carry16 + at) = pack8(o);
    }
  }
  // cross-warp reduction of the column partials, 256 columns (one channel block j) at a time
#pragma unroll
  for (int j = 0; j < 4; ++j) {
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      s_part[warp][0][lane * 8 + k] = dg[8 * j + k];
      s_part[warp][1][lane * 8 + k] = db[8 * j + k];
    }
    __syncthreads();
    for (int idx = threadIdx.x; idx < 3 * 256; idx += blockDim.x) {
      const int which = idx >> 8, col = idx & 255;
      float acc = 0.f;
      if (which < 2) {
#pragma unroll
        for (int w = 0; w < 8; ++w) acc += s_part[w][which][col];
      }
      partial[(static_cast<long long>(blockIdx.x) * 3 + which) * kC + j * 256 + col] = acc;
    }
    __syncthreads();
  }
}

// dpos[t][c] = bf16(sum over n = 0, 1, .. of de[n * 577 + t][c]), an fp32 sum in crop order; dcls = dpos[0] (the class embedding is
// added where position 0 is, so its gradient is that row, with the same bits).  One thread per (token, 4 columns); dpos or dcls may be
// nullptr.
__global__ void __launch_bounds__(256) clip_pos_grad_kernel(const float* __restrict__ de, long long n_crops, __nv_bfloat16* __restrict__ dpos,
                                                            __nv_bfloat16* __restrict__ dcls) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= kClipTokens * (kC / 4)) return;
  const int t = idx / (kC / 4), c = (idx - t * (kC / 4)) * 4;
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  for (long long n = 0; n < n_crops; ++n) {
    const float4 v = *reinterpret_cast<const float4*>(de + (n * kClipTokens + t) * kC + c);
    s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
  }
  const uint2 pk = make_uint2(pack_bf16x2(s.x, s.y), pack_bf16x2(s.z, s.w));
  if (dpos != nullptr) *reinterpret_cast<uint2*>(dpos + static_cast<long long>(t) * kC + c) = pk;
  if (t == 0 && dcls != nullptr) *reinterpret_cast<uint2*>(dcls + c) = pk;
}

// dw[o][k] = bf16(sum over s = 0, 1, .. of part[s][k][o]) for o < 1024, k < 588: the split-K slices of dW^T [588, 1024] summed in slice
// order and transposed into the conv weight's [1024, 3, 14, 14] (k = (c, ky, kx), the im2col column order).  32 x 32 tiles through
// shared memory; grid (1024 / 32, ceil(588 / 32)), block (32, 8).
__global__ void __launch_bounds__(256) clip_patch_grad_reduce_kernel(const float* __restrict__ part, int splits,
                                                                     __nv_bfloat16* __restrict__ dw) {
  __shared__ float tile[32][33];
  const int o0 = blockIdx.x * 32, k0 = blockIdx.y * 32;
  const long long slice = static_cast<long long>(kClipPatchK) * kC;
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int k = k0 + r;
    float s = 0.f;
    if (k < kClipPatchK)
      for (int q = 0; q < splits; ++q) s += part[q * slice + static_cast<long long>(k) * kC + o0 + threadIdx.x];
    tile[r][threadIdx.x] = s;
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int k = k0 + threadIdx.x;
    if (k < kClipPatchK) dw[static_cast<long long>(o0 + r) * kClipPatchK + k] = __float2bfloat16_rn(tile[threadIdx.x][r]);
  }
}

}  // namespace tp
