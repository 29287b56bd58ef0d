// Kernels of the frozen CLIP-ViT-L/14-336 vision tower that are not GEMMs (the linears run on tp_gemm.cuh's engine):
//   clip_im2col_kernel         crops [N,3,336,336] -> patch rows [N*576, 588] in the conv weight's (c, ky, kx) order
//   clip_embed_preln_kernel    + class / position embedding, pre_layrnorm -> hidden_states[0]
//   clip_layernorm_kernel      layer_norm1 / layer_norm2 of a layer
//   clip_attn_kernel           softmax(q k^T) v per (crop, head, 128-query block) over the 577 tokens, wgmma + online softmax
// Each is instantiated for the bf16 tower and for the fp16 one (__half storage, f16 wgmma); the arithmetic is fp32 in both.
#pragma once

#include <type_traits>

#include "tp_ptx.cuh"

namespace tp {

constexpr int kClipTokens = 577;            // CLS + 24 x 24 patches
constexpr int kClipPatch = 14;
constexpr int kClipImage = 336;
constexpr int kClipPatchK = 3 * kClipPatch * kClipPatch;   // 588
constexpr int kClipPatchLd = 592;           // patch rows padded to a 16-byte multiple (TMA strides); columns 588.. are never read
constexpr int kClipHeads = 16;
constexpr int kClipHeadDim = 64;
constexpr float kClipLnEps = 1e-5f;
constexpr int kClipStatLd = 640;            // tokens per (crop, head) row of the training path's softmax statistics: 5 query blocks of 128

// One thread per (patch row, channel, kernel row): 14 consecutive pixels in, 14 consecutive patch-row elements out.  bf16 crops into
// f16 patch rows are converted as images.to(torch.float16) does (clip_encoder.py:59): through fp32, one round-to-nearest-even.
template <typename Tin, typename Tout>
__global__ void clip_im2col_kernel(const Tin* __restrict__ crops, long long crop_stride, long long n_crops, Tout* __restrict__ patches) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= n_crops * 576 * 3 * kClipPatch) return;
  const int cy = static_cast<int>(idx % (3 * kClipPatch));
  const long long prow = idx / (3 * kClipPatch);
  const long long n = prow / 576;
  const int p = static_cast<int>(prow - n * 576);
  const int c = cy / kClipPatch, ky = cy - c * kClipPatch;
  const int py = p / 24, px = p - py * 24;
  const Tin* src = crops + n * crop_stride + (static_cast<long long>(c) * kClipImage + py * kClipPatch + ky) * kClipImage + px * kClipPatch;
  Tout* dst = patches + prow * kClipPatchLd + cy * kClipPatch;
#pragma unroll
  for (int kx = 0; kx < kClipPatch; ++kx) {
    if constexpr (std::is_same_v<Tin, Tout>) dst[kx] = src[kx];
    else dst[kx] = __float2half_rn(__bfloat162float(src[kx]));
  }
}

// LayerNorm of one 1024-wide row held by a warp in fp32 (lane l: columns 256 j + 8 l + [0, 8), j = 0..3), one rounding to T (bf16 or
// f16, the type of gamma and beta too): mean, then the variance from the deviations (two passes over registers), rstd = rsqrt(var + 1e-5)
template <typename T>
__device__ __forceinline__ void clip_ln_row_store(const float (&e)[32], const T* __restrict__ gamma, const T* __restrict__ beta,
                                                  T* __restrict__ out, int lane) {
  constexpr bool kF16 = std::is_same_v<T, __half>;
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 32; ++i) s += e[i];
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  const float mean = s * (1.0f / 1024);
  float v = 0.f;
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    const float d = e[i] - mean;
    v = fmaf(d, d, v);
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  const float rstd = rsqrtf(v * (1.0f / 1024) + kClipLnEps);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int col = 256 * j + 8 * lane;
    const uint4 g = __ldg(reinterpret_cast<const uint4*>(gamma + col)), b = __ldg(reinterpret_cast<const uint4*>(beta + col));
    const uint32_t gw[4] = {g.x, g.y, g.z, g.w}, bw[4] = {b.x, b.y, b.z, b.w};
    uint32_t o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k)
      o[k] = pack_x2<kF16>(fmaf((e[8 * j + 2 * k] - mean) * rstd, x2_lo<kF16>(gw[k]), x2_lo<kF16>(bw[k])),
                           fmaf((e[8 * j + 2 * k + 1] - mean) * rstd, x2_hi<kF16>(gw[k]), x2_hi<kF16>(bw[k])));
    *reinterpret_cast<uint4*>(out + col) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

__device__ __forceinline__ void clip_load_row(const float* __restrict__ src, float (&e)[32], int lane) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float4 a = *reinterpret_cast<const float4*>(src + 256 * j + 8 * lane);
    const float4 b = *reinterpret_cast<const float4*>(src + 256 * j + 8 * lane + 4);
    e[8 * j] = a.x; e[8 * j + 1] = a.y; e[8 * j + 2] = a.z; e[8 * j + 3] = a.w;
    e[8 * j + 4] = b.x; e[8 * j + 5] = b.y; e[8 * j + 6] = b.z; e[8 * j + 7] = b.w;
  }
}

__device__ __forceinline__ void clip_load_row(const __nv_bfloat16* __restrict__ src, float (&e)[32], int lane) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint4 a = *reinterpret_cast<const uint4*>(src + 256 * j + 8 * lane);
    const uint32_t aw[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      e[8 * j + 2 * k] = bf16_lo(aw[k]);
      e[8 * j + 2 * k + 1] = bf16_hi(aw[k]);
    }
  }
}

__device__ __forceinline__ void clip_load_row(const __half* __restrict__ src, float (&e)[32], int lane) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint4 a = *reinterpret_cast<const uint4*>(src + 256 * j + 8 * lane);
    const uint32_t aw[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      e[8 * j + 2 * k] = f16_lo(aw[k]);
      e[8 * j + 2 * k + 1] = f16_hi(aw[k]);
    }
  }
}

// One warp per token row of x ([N*577, 1024], rows n*577 + t; rows t >= 1 hold the patch embedding, row 0 is ignored):
//   x[row] = T(pre_layrnorm((t == 0 ? class_embedding : x[row]) + position_embedding[t]))    (fp32 sum, in place, one rounding)
template <typename T>
__global__ void clip_embed_preln_kernel(T* __restrict__ x, long long rows, const T* __restrict__ cls, const T* __restrict__ pos,
                                        const T* __restrict__ gamma, const T* __restrict__ beta) {
  const long long row = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const int t = static_cast<int>(row % kClipTokens);
  float e[32], p[32];
  clip_load_row(t == 0 ? cls : x + row * 1024, e, lane);
  clip_load_row(pos + static_cast<long long>(t) * 1024, p, lane);
#pragma unroll
  for (int i = 0; i < 32; ++i) e[i] = __fadd_rn(e[i], p[i]);
  clip_ln_row_store(e, gamma, beta, x + row * 1024, lane);
}

// y = Tp(LayerNorm(x) * gamma + beta), one warp per row of [rows, 1024]: layer_norm1 (x: the bf16 / f16 hidden state) / layer_norm2 (x:
// the fp32 mid-layer residual) of a layer, as an explicit pass (statistics from the row itself, in fp32) so that the following linear
// reads its weights as they are.  Tp: the tower's storage type (gamma, beta and y).  ldx: elements between x's rows (1024, or 4096 when
// x is a hidden state stored into the interleaved output of tp_clip_tower_forward_interleaved); y is dense.
template <typename T, typename Tp = __nv_bfloat16>
__global__ void clip_layernorm_kernel(const T* __restrict__ x, long long ldx, long long rows, const Tp* __restrict__ gamma,
                                      const Tp* __restrict__ beta, Tp* __restrict__ y) {
  const long long row = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  float e[32];
  clip_load_row(x + row * ldx, e, lane);
  clip_ln_row_store(e, gamma, beta, y + row * 1024, lane);
}

// ------------------------------------------------------------------------------------------------
// Attention over the 577 tokens of one crop, one head, 128 queries (two warpgroups of 64):
//   qkv  [N*577, 3072] T: q (already scaled by 1/8: in the packed bf16 weights, by the q GEMM's alpha in f16) | k | v, head h at columns
//        64 h of each third
//   ctx  [N*577, 1024] T: heads side by side (HF's reshape of [N, 577, 16, 64])
// T = bf16 or f16: the wgmmas take T operands, P is rounded to T.
// Thread 0 loads the CTA's Q rows and the whole K and V of the (crop, head) by TMA through a 3-D (column, token, crop) map whose
// token extent is 577: boxes reaching past token 576 are zero-filled, never the next crop's rows.  Per 128-key block:
//   S = Q K^T (wgmma m64n128k16, both K-major), keys >= 577 set to -inf BEFORE the row max (a zero-filled key scores 0 and would take
//   weight), online softmax in fp32 (exp2 on log2(e)-scaled scores), P rounded to bf16 into shared memory (K-major, 128-byte
//   swizzle), O += P V (wgmma m64n64k16, V as the MN-major B operand).  The row sum is taken over the ROUNDED P that multiplies V.
// kLse (the training forward): also writes lse[crop][head][t] = m log2(e) + log2(l), the log2 of the softmax denominator on the scale of
// the exp2 above ([N, 16, 640] fp32, tokens >= 577 not written), from which the backward recomputes P = exp2(s log2(e) - lse).
// ------------------------------------------------------------------------------------------------
constexpr int kAttnKeyBoxes = 10;                         // 640 >= 577 keys in boxes of 64
constexpr int kAttnBoxBytes = 64 * 128;                   // 64 tokens x 64 channels bf16
struct ClipAttnSmem {
  static constexpr int kQ = 0;                            // [2 warpgroups][64 x 64]
  static constexpr int kK = kQ + 2 * kAttnBoxBytes;       // [640 x 64]
  static constexpr int kV = kK + kAttnKeyBoxes * kAttnBoxBytes;
  static constexpr int kP = kV + kAttnKeyBoxes * kAttnBoxBytes;   // [2 warpgroups][2 key halves][64 x 64]
  static constexpr int kBar = kP + 4 * kAttnBoxBytes;
  static constexpr int kBytes = kBar + 16 + 1024;         // + alignment slack
};
static_assert(ClipAttnSmem::kBytes <= 232448, "shared memory budget of an sm_90 SM (227 KiB)");

template <typename T, bool kLse = false>
__global__ void __launch_bounds__(256, 1)
clip_attn_kernel(const __grid_constant__ CUtensorMap tmap_qkv, T* __restrict__ ctx, float* __restrict__ lse) {
  constexpr bool kF16 = std::is_same_v<T, __half>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + ClipAttnSmem::kBar);
  const int qb = blockIdx.x, head = blockIdx.y, crop = blockIdx.z;
  const int tid = threadIdx.x;
  if (tid == 0) {
    tma_prefetch_desc(&tmap_qkv);
    mbar_init(bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(bar, (2 + 2 * kAttnKeyBoxes) * kAttnBoxBytes);
    for (int w = 0; w < 2; ++w)
      tma_load_3d(smem + ClipAttnSmem::kQ + w * kAttnBoxBytes, &tmap_qkv, bar, head * kClipHeadDim, qb * 128 + w * 64, crop);
    for (int b = 0; b < kAttnKeyBoxes; ++b) {
      tma_load_3d(smem + ClipAttnSmem::kK + b * kAttnBoxBytes, &tmap_qkv, bar, 1024 + head * kClipHeadDim, b * 64, crop);
      tma_load_3d(smem + ClipAttnSmem::kV + b * kAttnBoxBytes, &tmap_qkv, bar, 2048 + head * kClipHeadDim, b * 64, crop);
    }
  }
  const int wg = tid >> 7;                                 // warpgroup: queries 64 wg .. + 63 of the block
  const int warp = (tid >> 5) & 3, lane = tid & 31;
  const int g = lane >> 2, q = lane & 3;
  const uint32_t sq = smem_u32(smem + ClipAttnSmem::kQ + wg * kAttnBoxBytes);
  const uint32_t sk = smem_u32(smem + ClipAttnSmem::kK), sv = smem_u32(smem + ClipAttnSmem::kV);
  const uint32_t sp = smem_u32(smem + ClipAttnSmem::kP + wg * 2 * kAttnBoxBytes);
  constexpr float kLog2e = 1.4426950408889634f;
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};   // rows 16 warp + g + 8 h of the warpgroup's 64
  mbar_wait(bar, 0);
  for (int kb = 0; kb < 5; ++kb) {
    float s[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) s[i] = 0.f;
    fence_regs(s);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kClipHeadDim / kUmmaK; ++k)
      wgmma_m64n128<0, 0, kF16>(s, make_smem_desc_kmajor_sw128(sq) + static_cast<uint64_t>(k * 2),
                          make_smem_desc_kmajor_sw128(sk + kb * 2 * kAttnBoxBytes) + static_cast<uint64_t>(k * 2), static_cast<uint32_t>(k != 0));
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);
    if (kb == 4) {                                         // keys 512 + col >= 577: padding zero-filled by TMA
#pragma unroll
      for (int i = 0; i < 64; ++i)
        if (512 + 8 * (i >> 2) + 2 * q + (i & 1) >= kClipTokens) s[i] = -INFINITY;
    }
    float corr[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = m[h];
#pragma unroll
      for (int i = 0; i < 64; ++i)
        if (((i >> 1) & 1) == h) mx = fmaxf(mx, s[i]);
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      corr[h] = ex2_approx(__fmul_rn(m[h] - mx, kLog2e));  // m = -inf on the first block: 0 (O and l are 0 anyway)
      m[h] = mx;
      l[h] *= corr[h];
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] *= corr[(i >> 1) & 1];
    // P = exp2((s - m) log2 e), rounded to T; the rounded values are summed and stored (K-major, 128-byte swizzle: row r's 16-byte
    // chunk c of a 64-key half lies at r * 128 + ((c ^ (r & 7)) << 4))
    const float nm0 = -m[0] * kLog2e, nm1 = -m[1] * kLog2e;
    named_bar_sync(1 + wg, 128);                           // the previous block's P V wgmmas of the whole warpgroup have retired
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
      const int h = (i >> 1) & 1;
      const float nm = h ? nm1 : nm0;
      const uint32_t pk = pack_x2<kF16>(ex2_approx(fmaf(s[i], kLog2e, nm)), ex2_approx(fmaf(s[i + 1], kLog2e, nm)));
      l[h] += x2_lo<kF16>(pk) + x2_hi<kF16>(pk);
      const int r = 16 * warp + g + 8 * h;
      const int col = 8 * (i >> 2) + 2 * q;
      const int half = col >> 6, c64 = col & 63;
      const uint32_t addr = sp + half * kAttnBoxBytes + r * 128 + ((((c64 >> 3) ^ (r & 7)) << 4) | ((c64 & 7) * 2));
      asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(pk) : "memory");
    }
    fence_proxy_async_smem();                              // generic-proxy stores -> visible to wgmma's reads
    named_bar_sync(1 + wg, 128);
    fence_regs(o);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 128 / kUmmaK; ++k)
      wgmma_m64n64<0, 1, kF16>(o, make_smem_desc_kmajor_sw128(sp + (k >> 2) * kAttnBoxBytes) + static_cast<uint64_t>((k & 3) * 2),
                         make_smem_desc_mnmajor_sw128(sv + (kb * 2 + (k >> 2)) * kAttnBoxBytes, kAttnBoxBytes) + static_cast<uint64_t>((k & 3) * 128),
                         1u);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(o);
  }
  float inv[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
    inv[h] = rcp_rn_normal(l[h]);                          // l >= 1: the row maximum contributes exp2(0) = 1
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int t = qb * 128 + wg * 64 + 16 * warp + g + 8 * h;
    if (t >= kClipTokens) continue;
    if (kLse && q == 0) lse[(static_cast<long long>(crop) * kClipHeads + head) * kClipStatLd + t] = fmaf(m[h], kLog2e, lg2_approx(l[h]));
    T* dst = ctx + (static_cast<long long>(crop) * kClipTokens + t) * 1024 + head * kClipHeadDim + 2 * q;
#pragma unroll
    for (int i = 2 * h; i < 32; i += 4)
      *reinterpret_cast<uint32_t*>(dst + 8 * (i >> 2)) = pack_x2<kF16>(__fmul_rn(o[i], inv[h]), __fmul_rn(o[i + 1], inv[h]));
  }
}

// The q third of the packed [3072, 1024] qkv weight and its fp32 bias times 1/8 (exact: a power of two in bf16, whose exponent range is
// fp32's, except that weights below 2^-123 become bf16 subnormals and round once to nearest even; the f16 tower applies 1/8 as the q
// GEMM's alpha instead, since weights below 2^-11 would lose bits as f16 subnormals)
__global__ void clip_scale_q_kernel(__nv_bfloat16* __restrict__ w, float* __restrict__ bias) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 1024 * 1024) w[i] = __float2bfloat16_rn(__bfloat162float(w[i]) * 0.125f);
  if (i < 1024) bias[i] *= 0.125f;
}

}  // namespace tp
