// Persistent warp-specialised wgmma GEMMs for sm_90a with the fused epilogues the TokenPacker path needs.
//
//   C[M,N] (bf16) = epilogue( A[M,K] (bf16, K-major) . B[N,K]^T (bf16, K-major) ),  fp32 accumulation in registers.
//   (The CLIP tower's fp16 instantiations, kF16: the same with f16 operands and output, GemmEpilogue::f16.)
//
// Every nn.Linear on the reference hot path (builder.py:59-83; MHA in/out projections builder.py:77) is an
// instance of these kernels: activations are [rows, in] and weights are [out, in], both K-major, which is exactly the
// operand form wgmma takes from shared memory, so no transposes exist anywhere.
//
// Two kernels share one epilogue:
//   tp_gemm_kernel<BN>   one CTA per SM, 128 x BN tiles (small problems, BN = 128 | 256)
//   tp_gemm2_kernel      256 x 256 tiles handled by two CTAs ("a pair": CTA 2p + r computes rows r * 128 .. + 127 of the tile), each
//                        with a 3-stage TMA ring of its 128 rows of A and the whole 256-row B tile, and double-buffered output
//                        slabs for the TMA stores.  Also the home of the TN form (MN-major operands, wgrad), multi-part A (four
//                        CLIP layers side by side along K), grouped launches and the peer (all-gather) stores.
//
// CTA = 384 threads, persistent over output tiles:
//   warps 0-7   two MMA + epilogue warpgroups, one per 64-row block of the CTA's 128 rows: one wgmma m64nNk16 per k16 step over
//               the whole N-column tile (N/2 fp32 accumulators per thread), so each warpgroup reads its A block once and the B tile
//               once per k-step; then the epilogue on the same registers.  Pair-kernel tiles stored through TMA (every
//               instantiation): fused per-row / per-column math on the fragments in place, stmatrix into the swizzled shared-memory
//               slabs (epilogue_tile_frag, the only slab writer).  Tiles with direct global stores (the one-CTA kernel; the pair
//               kernel's scattered segment rows and fp32 outputs) and KV-attention tiles: each warp turns its fragments into
//               thread == output row form (lanes 0-15: column half 0, lanes 16-31: column half 1 of the warp's 16 rows) through a
//               2 KiB shared-memory transpose (32 columns at a time), then fused per-row / per-column math and 16-byte global stores
//               (epilogue_tile).  KV-attention tiles: the window softmax on the fragments (attn_scores / attn_pv)
//   warps 8, 9  store warps of the pair kernel (one per column half): wait for a finished slab on an mbarrier, issue its TMA
//               store(s), hand the buffer back, and — for GEMMs that other GEMMs of the same launch depend on — publish each
//               finished tile to a global counter.  The epilogue warps never wait for a store.
//   warp 10     TMA producer   (warp-uniform loop, elect.sync around the issue): cp.async.bulk.tensor boxes, 128B swizzle, mbarrier
//               ring; spins on the producer GEMM's tile counter before the first load of a dependent tile
//   (warps 8-11 run with 72 registers a thread, setmaxnreg, so that the accumulator warpgroups can hold 216)
//
// Fused epilogue (all optional, selected at run time, warp-uniform branches):
//   v = acc
//   v = fma(rstd_r, fma(-mu_r, col_a[c], v), col_b[c])    LayerNorm folded into the NEXT linear: (mu, rstd) from per-row sums,
//                                                col_b = the folded constant W.beta + b    -- or, without a fold --
//   v = v + col_b[c]                             bias
//   v = v + R[r, c]                              residual add (bf16 operand read from global memory)
//   v = gelu_erf(v)  |  v = quick_gelu(v)        exact erf GELU (nn.GELU default) | x sigmoid(1.702 x) (CLIP)
//   v = alpha * v                                1/sqrt(head_dim) query scaling
//   y = bf16(v);  stats_out[r][slot] = (mean, M2) of y over this thread's 128 columns -> next LayerNorm fold (deterministic:
//                                                one slot per 128-column block, combined Chan-style in fixed order by the consumer)
//   C[dst_row(r), c] = y                         optional segment scatter (HD packed output)
#pragma once

#include "tp_ptx.cuh"

namespace tp {

struct GemmEpilogue {
  void* c;                 // output: bf16 [M, ldc] (f16 with f16, float with out_f32)
  long long ldc;           // elements between output rows
  const float* col_a;      // [N]  LN fold: row-sum of the gamma-folded weight      (nullptr: no LN fold)
  const float* col_b;      // [N]  bias                                             (nullptr: none)
  const float* stats_in;   // [M, stats_in_slots, 2] per-block (mean, M2) of the A rows (required with col_a)
  float* stats_out;        // [M, stats_out_slots, 2]                               (nullptr: none)
  const long long* seg_row_offset;  // [M / seg_len] destination row of each segment's first row (nullptr: identity / uniform stride)
  int seg_len;             // rows per segment (one crop's tokens)
  int seg_stride;          // uniform-stride form (seg_row_offset == nullptr): segment i starts at output row i * seg_stride
                           // (0: contiguous).  The HD packed layout (llava_arch.py:139-155) is exactly this with stride = seg_len + 1:
                           // every crop is followed by ONE separator row (',' or '\n').  Kept on the TMA-store path (3-D C map).
  int stats_in_slots;
  int stats_out_slots;     // = N / 128 (host-checked; statistics need 256-column tiles): slot = col / 128
  float ln_inv_dim;        // 1 / ln_dim
  float ln_eps;
  float alpha;
  int gelu;
  int wm_s;                // != 0: rows are tokens in raster order (24 x 24 per crop) and C is stored WINDOW-MAJOR for scale factor
                           // wm_s: row (crop, hb, wb, hi, wi) of [crops * 576] — the s x s keys of a window become wm_s^2 consecutive
                           // rows (divide_feature, builder.py:96-105, done by the store instead of five permute copies).  The row
                           // statistics go to the permuted row too.  Pair kernel / TMA stores only; wm_s in {2, 4, 8}.
  int out_f32;             // 1: C is float [M, ldc] (split-K partial sums of the wgrads): fp32 direct stores, no bf16 rounding
  int dual;                // 1 (with gelu): the bf16-rounded PRE-activation (after bias / LN fold, before GELU and alpha) is stored too,
                           // through GemmProblem::tmap_cx[0] (the training forward keeps z for GELU'(z); builder.py:66-75 under autograd).
                           // Pair kernel, plain (unsegmented) TMA-store output, two 64-column staging buffers per half.
  const void* resid;            // != nullptr: v += resid[row * ldr + c] after bias / LN fold (the CLIP tower's residual stream), read
  long long ldr;                // straight from global memory (the pair kernel's shared memory is full); row = the GEMM row; bf16
                                // values (f16 with f16)
  int resid_f32;                // 1: resid points to float values (the tower's unrounded mid-layer residual x')
  int f16;                      // 1: A, B, C and a 16-bit resid are IEEE half: the tower's f16 instantiations run the item (kF16)
};
// f16 fills the padding after resid_f32: every other field keeps its offset, so the kernels' parameter blocks are laid out as before
static_assert(sizeof(GemmEpilogue) == 128 && offsetof(GemmEpilogue, f16) == 124, "GemmEpilogue layout");

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;     // 64 bf16 = 128 bytes = one swizzle-128B row
constexpr int kUmmaK = 16;
constexpr int kGemmThreads = 384;
// Warp roles: warps 0-7 are the two MMA + epilogue warpgroups (warpgroup = 64-row block of the CTA's 128 rows, warp % 4 =
// "quarter": the 16 rows of that block its wgmma fragments hold), warps 8-11 the producer / store warpgroup.
constexpr int kEpiWarp0 = 0;
constexpr int kTmaWarp = 10;
constexpr int kStoreWarp0 = 8;      // pair kernel: warps 8 and 9 issue the TMA stores of column half 0 / 1
constexpr int kNumEpiWarps = 8;
constexpr int kEpiThreads = kNumEpiWarps * 32;
constexpr int kEpiBarrierId = 1;
constexpr uint32_t kMmaRegs = 216;  // setmaxnreg: 256 x 216 + 128 x 72 <= 64 K registers of an SM
constexpr uint32_t kAuxRegs = 72;
constexpr int kScratchBytesPerWarp = 32 * 16 * 4;     // accumulator transpose: 32 rows x 16 fp32 columns
constexpr int kScratchBytes = kNumEpiWarps * kScratchBytesPerWarp;

// Pair kernel: tile row of epilogue thread (warpgroup wg, quarter, lane): the 16 rows whose wgmma fragments warp `quarter` of
// warpgroup wg holds, once for each column half (lanes 0-15: half 0, lanes 16-31: half 1: epi_half), so the fragment -> row
// transpose never leaves the warp.
__device__ __forceinline__ int epi_row(int wg, int quarter, uint32_t lane) {
  return 64 * wg + 16 * quarter + static_cast<int>(lane & 15u);
}
__device__ __forceinline__ int epi_half(uint32_t lane) { return static_cast<int>(lane >> 4); }

// One-CTA kernel (warpgroup = column half): tile row of epilogue thread (quarter, lane): the 16 rows of each 64-row block whose
// fragments warp `quarter` holds, lanes 0-15 in block 0 and lanes 16-31 in block 1.
__device__ __forceinline__ int epi_row_1cta(int quarter, uint32_t lane) {
  return 16 * quarter + static_cast<int>(lane & 15u) + 64 * static_cast<int>(lane >> 4);
}

// 32 accumulator columns [32 chunk, +32) of each of the warp's two fragment parts into r: lane l gets row l & 15 of part l >> 4.
// acc[h] is part h: in the pair kernel the column-half-h registers of the m64n256 fragment (registers 64 h ...), in the one-CTA
// kernel the fragment of 64-row block h.  Both parts go through the warp's scratch, 16 columns at a time, XOR-swizzled so that
// both the 8-byte fragment stores and the 16-byte row loads are free of bank conflicts.  `chunk` must be a compile-time constant
// after unrolling.
__device__ __forceinline__ uint32_t scratch_swz(uint32_t row) { return (((row >> 1) & 1u) << 1) | ((row >> 2) & 1u); }

template <int kAccN>
__device__ __forceinline__ void acc_chunk(const float (&acc)[2][kAccN], int chunk, uint32_t scratch, uint32_t (&r)[32]) {
  const uint32_t lane = lane_id();
  const uint32_t g = lane >> 2, q = lane & 3u;
#pragma unroll
  for (int t = 0; t < 2; ++t) {
    __syncwarp();                                      // the previous reads of the scratch are done
#pragma unroll
    for (int ch = 0; ch < 2; ++ch)
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int jj = 0; jj < 2; ++jj) {
          const int i = (chunk * 4 + t * 2 + jj) * 4 + 2 * h;
          const uint32_t row = g + 8u * h + 16u * ch;
          const uint32_t unit = ((2u * jj) + (q >> 1)) ^ scratch_swz(row);
          sts_f2(scratch + row * 64u + unit * 16u + (q & 1u) * 8u, acc[ch][i], acc[ch][i + 1]);
        }
    __syncwarp();
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const float4 v = lds_f4_ordered(scratch + lane * 64u + ((static_cast<uint32_t>(u) ^ scratch_swz(lane)) * 16u));
      r[16 * t + 4 * u + 0] = __float_as_uint(v.x);
      r[16 * t + 4 * u + 1] = __float_as_uint(v.y);
      r[16 * t + 4 * u + 2] = __float_as_uint(v.z);
      r[16 * t + 4 * u + 3] = __float_as_uint(v.w);
    }
  }
}

// One warpgroup's MMAs for a tile: kRowBlocks 64-row blocks of A starting `a_off` bytes into the stage x kN rows of B starting
// `b_off` bytes into it, over n_kb k-blocks of the ring: per k16 step one m64nNk16 per row block.  The pair kernel: one row block
// (its warpgroup's) x the whole 256-row B tile, m64n256.  The one-CTA kernel: both row blocks x its warpgroup's column half.
// A stage is released (one arrive per warp on empty_bar) once the wgmmas reading it have retired; one k-block of wgmmas stays
// in flight while the next one is issued.
template <int kN, int kRowBlocks, int kTransA, int kTransB, bool kF16 = false>
__device__ __forceinline__ void mma_tile(float (&acc)[2][kN * kRowBlocks / 4], const uint8_t* smem, int stage_bytes, int a_off, int b_off,
                                         uint64_t* full_bar, uint64_t* empty_bar, int n_stages, int& stage, uint32_t& phase, int n_kb) {
  static_assert(kN == 64 || kN == 128 || kN == 256, "wgmma N");
  float (&d)[kRowBlocks][kN / 2] = reinterpret_cast<float (&)[kRowBlocks][kN / 2]>(acc);   // per row block: its fragment, wgmma order
  int prev = -1;
  for (int kb = 0; kb < n_kb; ++kb) {
    mbar_wait(&full_bar[stage], phase);         // TMA bytes have landed
    const uint32_t sa = smem_u32(smem + stage * stage_bytes) + static_cast<uint32_t>(a_off);
    const uint32_t sb = smem_u32(smem + stage * stage_bytes) + static_cast<uint32_t>(b_off);
#pragma unroll
    for (int mb = 0; mb < kRowBlocks; ++mb) fence_regs(d[mb]);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kBlockK / kUmmaK; ++k) {
      // K-major: advance 16 elements = 32 bytes along the 128-byte swizzle row (+2 in the address field);
      // MN-major: one k16 step = two 8-row K groups = 2 KiB (+128); 64-row blocks of A and 64-wide MN atoms are 8 KiB apart
      const uint64_t db = kTransB ? make_smem_desc_mnmajor_sw128(sb, 8192) + static_cast<uint64_t>(k * 128)
                                  : make_smem_desc_kmajor_sw128(sb) + static_cast<uint64_t>(k * 2);
      const uint32_t accumulate = static_cast<uint32_t>((kb | k) != 0);
#pragma unroll
      for (int mb = 0; mb < kRowBlocks; ++mb) {
        const uint32_t sam = sa + static_cast<uint32_t>(mb * 8192);
        const uint64_t da = kTransA ? make_smem_desc_mnmajor_sw128(sam, 8192) + static_cast<uint64_t>(k * 128)
                                    : make_smem_desc_kmajor_sw128(sam) + static_cast<uint64_t>(k * 2);
        if constexpr (kN == 256) wgmma_m64n256<kTransA, kTransB, kF16>(d[mb], da, db, accumulate);
        else if constexpr (kN == 128) wgmma_m64n128<kTransA, kTransB, kF16>(d[mb], da, db, accumulate);
        else wgmma_m64n64<kTransA, kTransB, kF16>(d[mb], da, db, accumulate);
      }
    }
    wgmma_commit();
#pragma unroll
    for (int mb = 0; mb < kRowBlocks; ++mb) fence_regs(d[mb]);
    wgmma_wait<1>();                                   // the previous k-block's wgmmas have retired
    if (prev >= 0) {
      __syncwarp();
      if (lane_id() == 0) mbar_arrive(&empty_bar[prev]);
    }
    prev = stage;
    if (++stage == n_stages) { stage = 0; phase ^= 1u; }
  }
  wgmma_wait<0>();
#pragma unroll
  for (int mb = 0; mb < kRowBlocks; ++mb) fence_regs(d[mb]);
  if (prev >= 0) {
    __syncwarp();
    if (lane_id() == 0) mbar_arrive(&empty_bar[prev]);
  }
}

// ------------------------------------------------------------------------------------------------
// Output staging for the pair kernel's TMA stores: each column half of the tile owns two 16 KiB buffers holding a 128-row x 64-col
// slab in the 128B-swizzled layout, 16 rows of it from each of the 8 epilogue warps.  epilogue_tile_frag writes a slab with stmatrix
// and hands it over with one mbarrier arrive per warp; the half's store warp sends it to the TMA unit (full 128-byte row segments
// instead of 16-byte scattered stores: less L1/L2 work and less power).
constexpr int kMaxPeers = 8;
// Fused all-gather: tensor maps of the SAME output slot in every peer GPU's gathered buffer (peer-mapped over NVLink);
// each finished slab is TMA-stored to all of them instead of to one local matrix.
constexpr int kBoxLevels = 4;   // exact-size store boxes: rows = unit << level
constexpr int kWholeLevels = 3; // ... and boxes of 1, 2 or 3 WHOLE segments (crops that lie entirely inside a 128-row slab)
struct PeerStores {
  CUtensorMap m[kMaxPeers][kBoxLevels + kWholeLevels];   // [destination][level]; plain (unsegmented) output uses level 0 only
  int count;                 // 0: ordinary local output through GemmProblem::tmap_c
  int whole;                 // 1: the whole-segment maps m[.][kBoxLevels + k - 1] (k segments) are valid (seg_len <= 128)
};

// Output slab = 128 rows x 64 columns of 16-bit values: 128-byte rows in TMA's SWIZZLE_128B layout.
constexpr int kSlabCols = 64;
constexpr int kSlabRowBytes = kSlabCols * 2;
constexpr int kOutSlabBytes = 128 * kSlabRowBytes;

// Shared staging of a tile's per-column vectors: [col_a | col_b] x [column half 0 | kColPad | column half 1 | kColPad] floats.
// In the pair kernel the two halves of a warp read the same offset of their half at once; the padding puts those two addresses
// in different banks.
constexpr int kColPad = 4;
template <int kTileN>
__host__ __device__ constexpr int col_slot(int vec, int c) { return vec * (kTileN + 2 * kColPad) + c + (c >= kTileN / 2 ? kColPad : 0); }

// raster row (crop n, token row tr, token column tc) -> window-major row (crop n, window (hb, wb), key (hi, wi)) for windows of s x s
__device__ __forceinline__ long long window_major_row(long long row, int s) {
  const long long n = row / 576;
  const int t = static_cast<int>(row - n * 576);
  const int tr = t / 24, tc = t - tr * 24;
  const int hb = tr / s, hi = tr - hb * s, wb = tc / s, wi = tc - wb * s;
  return n * 576 + ((hb * (24 / s) + wb) * s + hi) * s + wi;
}

// (mean, rstd) of a LayerNorm row from its per-128-column (mean, M2) pairs st[0 .. slots), combined Chan-style in fixed order
__device__ __forceinline__ void ln_stats_combine(const float2* st, int slots, float inv_dim, float eps, float& mu, float& rstd) {
  float t1 = 0.f, m2 = 0.f;
  for (int i = 0; i < slots; ++i) t1 = __fadd_rn(t1, st[i].x);
  const float inv_slots = rcp_rn_normal(static_cast<float>(slots));      // slots in [1, 64], inv_dim in [2^-13, 1]: call-free
  mu = __fmul_rn(t1, inv_slots);
  float between = 0.f;
  for (int i = 0; i < slots; ++i) {
    const float2 v = st[i];
    const float d = __fsub_rn(v.x, mu);
    between = fmaf(d, d, between);
    m2 = __fadd_rn(m2, v.y);
  }
  const float var = __fmul_rn(fmaf(between, __fmul_rn(inv_slots, rcp_rn_normal(inv_dim)), m2), inv_dim);
  rstd = rsqrtf(__fadd_rn(var, eps));
}
__device__ __forceinline__ void ln_row_stats(const float* stats, long long row, int slots, float inv_dim, float eps, float& mu, float& rstd) {
  ln_stats_combine(reinterpret_cast<const float2*>(stats) + row * slots, slots, inv_dim, eps, mu, rstd);
}

// ------------------------------------------------------------------------------------------------
// Direct-store epilogue for one 128-row x kTileN-column accumulator tile held in the registers of the CTA's two MMA warpgroups: the
// one-CTA kernel's tiles, and the pair kernel's tiles without TMA stores (scattered segment rows, fp32 output and split-K slices).
// Each warp turns its fragments into thread == output row form through the transpose scratch, then stores 16 bytes at a time.
//   acc      : this warpgroup's wgmma accumulators, [column half (pair kernel) | 64-row block (one-CTA kernel)][fragment registers]
//   scratch  : shared address of this warp's transpose scratch (kScratchBytesPerWarp)
//   row      : global output row of this thread (epi_row / epi_row_1cta)
//   col_tile0: global column of the tile's first column
//   half     : the column half this thread owns
//   s_col    : shared staging for this tile's col_a / col_b slices, col_slot layout (already filled + synced)
// kTower: the CLIP tower's instantiations (bias, bf16 or fp32 residual add, quick_gelu, alpha, fp32 output) — and none of the
// projector's LayerNorm fold and row statistics, so that neither set of instantiations carries the other's registers.
// kF16 (tower only): the same with an f16 residual and f16 output (one __floats2half2_rn rounding).
// kSubPairs: packed column pairs (2 columns each) that go through every step together: each run-time option is ONE warp-uniform
// branch around a basic block of kSubPairs independent dependency chains for the scheduler to interleave (more chains, more
// registers).  8 in the one-CTA kernel; 4 in the pair kernel, where the column half is a per-lane value and 8 chains spill at
// the 216-register limit.
template <int kTileN, bool kTower = false, bool kF16 = false, int kSubPairs = 8>
__device__ __forceinline__ void epilogue_tile(const GemmEpilogue& ep, int M, int N, const float (&acc)[2][kTileN / 4], uint32_t scratch,
                                              int row, int col_tile0, int half, const float* s_col, long long c_extra = 0) {
  constexpr int kColsPerHalf = kTileN / 2;
  constexpr int kChunks = kColsPerHalf / 32;
  const bool ln_fold = !kTower && ep.col_a != nullptr;
  const bool row_ok = row < M;
  float mu = 0.f, rstd = 1.f;
  // Row statistics arrive as one (mean_i, M2_i) pair per 128-column block (M2 = sum of squared deviations from the block's own
  // mean) and are combined Chan-style in a fixed order: no E[y^2] - mu^2 cancellation when |mean| >> std, bitwise reproducible.
  // (explicit intrinsics throughout the epilogue math: no FMA-contraction freedom for the compiler, so the one-CTA and CTA-pair
  // instantiations produce the same bits for the same row)
  if (ln_fold && row_ok) ln_row_stats(ep.stats_in, row, ep.stats_in_slots, ep.ln_inv_dim, ep.ln_eps, mu, rstd);
  long long dst_row = row;
  if (ep.seg_row_offset != nullptr && row_ok) {
    const int seg = row / ep.seg_len;
    dst_row = ep.seg_row_offset[seg] + (row - seg * ep.seg_len);
  } else if (ep.seg_stride != 0 && row_ok) {
    const int seg = row / ep.seg_len;
    dst_row = static_cast<long long>(seg) * ep.seg_stride + (row - seg * ep.seg_len);
  }
  __nv_bfloat16* c_row = static_cast<__nv_bfloat16*>(ep.c) + dst_row * ep.ldc;     // 16-bit elements (bf16 or f16: stored as raw bits)
  float* c_row32 = reinterpret_cast<float*>(ep.c) + c_extra + dst_row * ep.ldc;     // out_f32 only (c_extra: split-K slice)
  const uint32_t sa_addr = smem_u32(s_col + col_slot<kTileN>(0, half * kColsPerHalf));
  const uint32_t sb_addr = smem_u32(s_col + col_slot<kTileN>(1, half * kColsPerHalf));

  float s1 = 0.f, s2 = 0.f, shift = 0.f;     // statistics of (y - shift), shift = the block's first value: sums stay small
  const bool do_stats = !kTower && ep.stats_out != nullptr;
  const bool scale = ep.alpha != 1.0f;
  const uint64_t rstd2 = pk2(rstd), nmu2 = pk2(-mu), alpha2 = pk2(ep.alpha);
  uint32_t r[32];
#pragma unroll
  for (int chunk = 0; chunk < kChunks; ++chunk) {
    acc_chunk(acc, chunk, scratch, r);
    const int col0 = col_tile0 + half * kColsPerHalf + chunk * 32;
    if (col0 < N) {        // N is a multiple of 32 (checked on the host) -> whole chunk in or out
#pragma unroll
      for (int sub = 0; sub < 16 / kSubPairs; ++sub) {
        const int lc = chunk * 32 + sub * kSubPairs * 2;             // first column of this sub-block inside the warp's slice
        uint64_t v[kSubPairs];
#pragma unroll
        for (int j = 0; j < kSubPairs; ++j)
          v[j] = pk2(__uint_as_float(r[sub * kSubPairs * 2 + 2 * j]), __uint_as_float(r[sub * kSubPairs * 2 + 2 * j + 1]));
        const uint32_t sb4 = sb_addr + static_cast<uint32_t>(lc) * 4u;
        if (ln_fold) {     // v = fma(rstd, fma(-mu, col_a, v), col_b): explicit fmas, the same in every instantiation
          const uint32_t sa4 = sa_addr + static_cast<uint32_t>(lc) * 4u;
#pragma unroll
          for (int q = 0; q < kSubPairs / 2; ++q) {
            const float4 a = lds_f4(sa4 + q * 16), b = lds_f4(sb4 + q * 16);
            v[2 * q] = fma2(rstd2, fma2(nmu2, pk2(a.x, a.y), v[2 * q]), pk2(b.x, b.y));
            v[2 * q + 1] = fma2(rstd2, fma2(nmu2, pk2(a.z, a.w), v[2 * q + 1]), pk2(b.z, b.w));
          }
        } else {
#pragma unroll
          for (int q = 0; q < kSubPairs / 2; ++q) {
            const float4 b = lds_f4(sb4 + q * 16);
            v[2 * q] = add2(v[2 * q], pk2(b.x, b.y));
            v[2 * q + 1] = add2(v[2 * q + 1], pk2(b.z, b.w));
          }
        }
        if constexpr (kTower) {
          if (ep.resid != nullptr && row_ok && ep.resid_f32) {
            const float4* rp = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(ep.resid) + static_cast<long long>(row) * ep.ldr +
                                                               col0 + sub * kSubPairs * 2);
#pragma unroll
            for (int g = 0; g < kSubPairs / 2; ++g) {
              const float4 r4 = rp[g];
              v[2 * g] = add2(v[2 * g], pk2(r4.x, r4.y));
              v[2 * g + 1] = add2(v[2 * g + 1], pk2(r4.z, r4.w));
            }
          } else if (ep.resid != nullptr && row_ok) {   // one rounding of acc + bias + R: the residual add of a CLIP layer
            const uint4* rp = reinterpret_cast<const uint4*>(static_cast<const __nv_bfloat16*>(ep.resid) + static_cast<long long>(row) * ep.ldr +
                                                             col0 + sub * kSubPairs * 2);
#pragma unroll
            for (int g = 0; g < kSubPairs / 4; ++g) {
              const uint4 r4 = rp[g];
              v[4 * g] = add2(v[4 * g], pk2(x2_lo<kF16>(r4.x), x2_hi<kF16>(r4.x)));
              v[4 * g + 1] = add2(v[4 * g + 1], pk2(x2_lo<kF16>(r4.y), x2_hi<kF16>(r4.y)));
              v[4 * g + 2] = add2(v[4 * g + 2], pk2(x2_lo<kF16>(r4.z), x2_hi<kF16>(r4.z)));
              v[4 * g + 3] = add2(v[4 * g + 3], pk2(x2_lo<kF16>(r4.w), x2_hi<kF16>(r4.w)));
            }
          }
          if (ep.gelu == 2) {
#pragma unroll
            for (int j = 0; j < kSubPairs; ++j) v[j] = quick_gelu_pk(v[j]);
          }
        } else if (ep.gelu) {
#pragma unroll
          for (int j = 0; j < kSubPairs; ++j) v[j] = gelu_erf_pk(v[j]);
        }
        if (scale) {       // alpha == 1 (every GEMM but in_proj_q): x * 1 is x, skip the multiply
#pragma unroll
          for (int j = 0; j < kSubPairs; ++j) v[j] = mul2(v[j], alpha2);
        }
        uint32_t pk[kSubPairs];
#pragma unroll
        for (int j = 0; j < kSubPairs; ++j) {
          float lo, hi;
          upk2(v[j], lo, hi);
          pk[j] = pack_x2<kF16>(lo, hi);
        }
        if (do_stats) {    // LayerNorm statistics of the ROUNDED values the next GEMM will read (column order: deterministic)
          if (chunk == 0 && sub == 0) shift = bf16_lo(pk[0]);
#pragma unroll
          for (int j = 0; j < kSubPairs; ++j) {
            const float y0 = __fsub_rn(bf16_lo(pk[j]), shift), y1 = __fsub_rn(bf16_hi(pk[j]), shift);
            s1 = __fadd_rn(s1, __fadd_rn(y0, y1));
            s2 = fmaf(y0, y0, fmaf(y1, y1, s2));
          }
        }
        if (row_ok) {
          if (ep.out_f32) {
#pragma unroll
            for (int g = 0; g < kSubPairs / 2; ++g) {
              float4 f;
              upk2(v[2 * g], f.x, f.y);
              upk2(v[2 * g + 1], f.z, f.w);
              *reinterpret_cast<float4*>(c_row32 + col0 + sub * kSubPairs * 2 + g * 4) = f;
            }
          } else {
#pragma unroll
            for (int g = 0; g < kSubPairs / 4; ++g)
              *reinterpret_cast<uint4*>(c_row + col0 + sub * kSubPairs * 2 + g * 8) = make_uint4(pk[4 * g], pk[4 * g + 1], pk[4 * g + 2], pk[4 * g + 3]);
          }
        }
      }
    }
  }
  if (do_stats && row_ok) {
    const int slot = (col_tile0 + half * kColsPerHalf) / kColsPerHalf;
    if (slot < ep.stats_out_slots) {
      // (mean, M2) of this 128-column block: mean = shift + s1/n, M2 = s2 - s1^2/n  (deviations from `shift` are O(std): no cancellation)
      constexpr float inv_n = 1.0f / kColsPerHalf;
      const float dm = __fmul_rn(s1, inv_n);
      reinterpret_cast<float2*>(ep.stats_out)[static_cast<long long>(row) * ep.stats_out_slots + slot] =
          make_float2(__fadd_rn(shift, dm), fmaxf(fmaf(-s1, dm, s2), 0.f));
    }
  }
}

// ------------------------------------------------------------------------------------------------
// KV-attention tiles (problem kind 1): the MHA in-projections of the keys and values FUSED with the local-window attention core
// (builder.py:122-130 == nn.MultiheadAttention, L = 1 query, S = s*s keys per window, 8 heads x 128).
//   A tile = 256 window-major rows (CTA pair) x TWO heads, in two accumulator phases of the ordinary 256 x 256 x K pipeline:
//     phase K: k' = y_k . (gamma_k W_ik)^T for the two heads  -> epilogue: folded LayerNorm, dot with the window's q' (already scaled
//              by 1/sqrt 128), softmax over the window's s*s consecutive rows  -> p stays in registers
//     phase V: v' = y_v . (gamma_v W_iv)^T                     -> epilogue: folded LayerNorm, p * v', summed over the window's rows,
//              store the window's 128 context channels of each head
//   Both phases use the same accumulator registers one after the other; the producer keeps the ring full in the meantime.
//   k' and v' never exist in memory (fp32, unrounded, in registers): the [R,1024] x 2 round trip through HBM and the separate
//   attention kernel are gone.
//   Both epilogues work on the wgmma m64n256 fragments where they are: lane (g = lane / 4, q = lane % 4) of a warp holds rows g and
//   g + 8 of the warp's 16 rows, acc[h][4 j + 2 r + e] = row g + 8 r, column 8 j + 2 q + e of column half h == head h of the pair.
//   A window is W = s*s consecutive rows, W-aligned: for s = 2 the rows g = 4 a .. 4 a + 3 of one r (lanes xor 4, 8), for s = 4
//   all 16 rows of the warp (the lane's two rows, lanes xor 4, 8, 16).
//   Order of the sums: a row's score is the lane's 32 products in column order, then the 4 lanes of the row (xor 1, then xor 2);
//   the softmax denominator and the context sums are pairwise trees over the window's rows (s = 4: the lane's rows g + g + 8 first).
//   What the epilogues read after the mainloop is fetched while the tensor pipe is busy: the (mean, M2) slots of the warp's rows of
//   y_k and y_v into registers (attn_load_stats), the q' rows of the CTA's windows into the (otherwise unused) transpose scratch
//   (attn_load_q).
// ------------------------------------------------------------------------------------------------
struct AttnParams {
  const __nv_bfloat16* qp;      // [Q, 1024] q', row = window index (= query index), scaled
  __nv_bfloat16* ctx;           // [Q, 1024]
  const float* stats_k;         // [R, slots, 2] (window-major rows) per-block (mean, M2) of y_k / y_v
  const float* stats_v;
  const float* wsum_k;          // [1024] LayerNorm-fold column vectors of the two in-projections
  const float* cst_k;
  const float* wsum_v;
  const float* cst_v;
  int s;                        // scale factor: W = s*s consecutive rows per window (2 or 4)
  int stats_slots;              // = kAttnSlots (host-checked)
  float ln_inv_dim, ln_eps;
  int* done_counter;            // ctx row blocks of 256 queries: counter[(m_blk * 256 / W) / 256] += 1 per (CTA, head pair)
  // dependencies of a tile: the raster row blocks of y_k / y_v covering the crops it touches, and its queries' q' row block
  const int* k_counter;
  const int* v_counter;
  int kv_target;
  const int* q_counter;
  int q_target;
};

constexpr int kAttnSlots = 8;         // (mean, M2) slots of a y_k / y_v row: 1024 columns / 128
constexpr int kAttnQBytes = 512;      // q' of one window in the scratch: the tile's two heads x 128 bf16
static_assert(kBlockM / 4 * kAttnQBytes <= kScratchBytes, "q' of a CTA's windows (s = 2) fits the transpose scratch");

// The (mean, M2) slots of the warp's 16 rows of y_k or y_v: lane l loads slots 4 (l / 16) .. + 3 of row row_w0 + l % 16 (zeros past
// M).  Phase K's are issued before its MMAs, phase V's before its epilogue, so that both land while the tensor pipe is busy.
__device__ __forceinline__ void attn_load_stats(const float* stats, int M, int row_w0, float4 (&st)[2]) {
  const uint32_t lane = lane_id();
  const int row = row_w0 + static_cast<int>(lane & 15u);
  const float4* src = reinterpret_cast<const float4*>(stats + static_cast<long long>(row) * (2 * kAttnSlots)) + 2 * (lane >> 4);
#pragma unroll
  for (int i = 0; i < 2; ++i) st[i] = row < M ? __ldcg(src + i) : make_float4(0.f, 0.f, 0.f, 0.f);
}

// (mu, rstd) of row row_w0 + l % 16 in lanes l < 16 from attn_load_stats (0, 0 past M: k' = v' = the folded constant there)
__device__ __forceinline__ void attn_row_stats(const AttnParams& at, const float4 (&st)[2], int M, int row_w0, float& mu, float& rstd) {
  float4 hi[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    hi[i].x = __shfl_down_sync(0xffffffffu, st[i].x, 16);
    hi[i].y = __shfl_down_sync(0xffffffffu, st[i].y, 16);
    hi[i].z = __shfl_down_sync(0xffffffffu, st[i].z, 16);
    hi[i].w = __shfl_down_sync(0xffffffffu, st[i].w, 16);
  }
  const float2 v[kAttnSlots] = {make_float2(st[0].x, st[0].y), make_float2(st[0].z, st[0].w), make_float2(st[1].x, st[1].y),
                                make_float2(st[1].z, st[1].w), make_float2(hi[0].x, hi[0].y), make_float2(hi[0].z, hi[0].w),
                                make_float2(hi[1].x, hi[1].y), make_float2(hi[1].z, hi[1].w)};
  mu = 0.f;
  rstd = 0.f;
  if (row_w0 + static_cast<int>(lane_id() & 15u) < M) ln_stats_combine(v, kAttnSlots, at.ln_inv_dim, at.ln_eps, mu, rstd);
}

// q' of the CTA's 128 / W windows for the tile's two heads into the transpose scratch (cp.async; issued before phase K's MMAs, landed
// by col_vectors_ready): window wl at scratch + wl * kAttnQBytes, its 16-byte piece u (channels 8 u ..) XOR-swizzled to
// (u ^ (wl & 7)) * 16, so that the two windows one warp instruction reads (s = 2) sit in different banks; zeros past the last window
__device__ __forceinline__ void attn_load_q(const AttnParams& at, int M, int row_cta0, int n_blk, uint32_t scratch, int epi_tid) {
  const int W = at.s * at.s;
  const long long win0 = row_cta0 / W, n_win = M / W;
  for (int i = epi_tid; i < (kBlockM / W) * 32; i += kEpiThreads) {
    const int wl = i >> 5, u = i & 31;
    const long long w = win0 + wl;
    const bool ok = w < n_win;
    cp_async_16(scratch + static_cast<uint32_t>(wl * kAttnQBytes + ((u ^ (wl & 7)) << 4)), at.qp + (ok ? w : 0) * 1024 + n_blk * 256 + u * 8,
                ok ? 16u : 0u);
  }
}

// Phase K epilogue: p[h][r] = the softmax weight of the lane's row g + 8 r for head h of the pair.
//   mu_own / rstd_own: attn_row_stats of y_k (lanes 0-15); rloc_w0: CTA row of the warp's first row; scratch: the q' rows
//   (attn_load_q); s_vec: wsum | cst of the tile's two heads (col_slot)
__device__ __forceinline__ void attn_scores(const AttnParams& at, const float (&acc)[2][64], float mu_own, float rstd_own, int rloc_w0,
                                            uint32_t scratch, const float* s_vec, float (&p)[2][2]) {
  const uint32_t lane = lane_id();
  const uint32_t g = lane >> 2, q = lane & 3u;
  const int W = at.s * at.s;
  float mu[2], rstd[2];
  uint32_t qa[2], swz[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    mu[r] = __shfl_sync(0xffffffffu, mu_own, static_cast<int>(g) + 8 * r);
    rstd[r] = __shfl_sync(0xffffffffu, rstd_own, static_cast<int>(g) + 8 * r);
    const int wl = (rloc_w0 + static_cast<int>(g) + 8 * r) / W;
    qa[r] = scratch + static_cast<uint32_t>(wl * kAttnQBytes) + 4u * q;
    swz[r] = static_cast<uint32_t>(wl & 7);
  }
  const uint32_t sa = smem_u32(s_vec + col_slot<256>(0, 0)), sb = smem_u32(s_vec + col_slot<256>(1, 0));
  float part[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const uint32_t c = static_cast<uint32_t>(h * 128 + 8 * j + (h ? kColPad : 0)) + 2u * q;    // col_slot offset
      float w0, w1, c0, c1;
      upk2(lds_f2(sa + c * 4u), w0, w1);
      upk2(lds_f2(sb + c * 4u), c0, c1);
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const uint32_t qw = lds_u32(qa[r] + (((16u * h + j) ^ swz[r]) << 4));
        const float k0 = fmaf(rstd[r], fmaf(-mu[r], w0, acc[h][4 * j + 2 * r]), c0);
        const float k1 = fmaf(rstd[r], fmaf(-mu[r], w1, acc[h][4 * j + 2 * r + 1]), c1);
        part[h][r] = fmaf(bf16_lo(qw), k0, part[h][r]);
        part[h][r] = fmaf(bf16_hi(qw), k1, part[h][r]);
      }
    }
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      part[h][r] += __shfl_xor_sync(0xffffffffu, part[h][r], 1);
      part[h][r] += __shfl_xor_sync(0xffffffffu, part[h][r], 2);
    }
  // softmax over the window's W rows (every lane of the window gets the same max and denominator: a + b == b + a)
  if (W == 4) {
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        float mx = part[h][r];
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 4));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 8));
        const float e = __expf(part[h][r] - mx);
        float den = e + __shfl_xor_sync(0xffffffffu, e, 4);
        den += __shfl_xor_sync(0xffffffffu, den, 8);
        p[h][r] = e * rcp_rn_normal(den);               // den in [1, 4]: the correctly rounded 1 / den, without a call
      }
  } else {                                              // W == 16
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = fmaxf(part[h][0], part[h][1]);
#pragma unroll
      for (int off = 4; off < 32; off <<= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
      const float e0 = __expf(part[h][0] - mx), e1 = __expf(part[h][1] - mx);
      float den = e0 + e1;
#pragma unroll
      for (int off = 4; off < 32; off <<= 1) den += __shfl_xor_sync(0xffffffffu, den, off);
      const float inv = rcp_rn_normal(den);             // den in [1, 16]
      p[h][0] = e0 * inv;
      p[h][1] = e1 * inv;
    }
  }
}

// Phase V epilogue: ctx = sum over the window's rows of p * v'.  Halving exchange: each step sends half of the lane's live values to
// the partner lane and adds the other half of the partner's, so that afterwards the 4 (s = 2) or 16 (s = 4) lanes of a window hold
// disjoint shares of its two heads x 128 channels, and store them as bf16 pairs (no value is stored twice).  Four rounds of 4
// 8-column groups each, so that few values are live at a time; acc itself is only read (the next tile's wgmmas take it over).
//   mu_own / rstd_own: attn_row_stats of y_v (lanes 0-15); row_w0: global row of the warp's first row
__device__ __forceinline__ void attn_pv(const AttnParams& at, int M, const float (&acc)[2][64], float mu_own, float rstd_own, int row_w0,
                                        int n_blk, const float (&p)[2][2], const float* s_vec) {
  const uint32_t lane = lane_id();
  const uint32_t g = lane >> 2, q = lane & 3u;
  const int W = at.s * at.s;
  float mu[2], rstd[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    mu[r] = __shfl_sync(0xffffffffu, mu_own, static_cast<int>(g) + 8 * r);
    rstd[r] = __shfl_sync(0xffffffffu, rstd_own, static_cast<int>(g) + 8 * r);
  }
  const uint32_t sa = smem_u32(s_vec + col_slot<256>(0, 0)), sb = smem_u32(s_vec + col_slot<256>(1, 0));
  const bool up4 = (lane & 4u) != 0, up8 = (lane & 8u) != 0, up16 = (lane & 16u) != 0;
  const int head = 2 * n_blk + (up4 ? 1 : 0);
  // o[r][e] = p v' of (head h, 8-column group j, row g + 8 r, column 8 j + 2 q + e)
  auto pv = [&](int h, int j, float (&o)[2][2]) {
    const uint32_t c = static_cast<uint32_t>(h * 128 + 8 * j + (h ? kColPad : 0)) + 2u * q;    // col_slot offset
    float w[2], cs[2];
    upk2(lds_f2(sa + c * 4u), w[0], w[1]);
    upk2(lds_f2(sb + c * 4u), cs[0], cs[1]);
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
      for (int e = 0; e < 2; ++e) o[r][e] = p[h][r] * fmaf(rstd[r], fmaf(-mu[r], w[e], acc[h][4 * j + 2 * r + e]), cs[e]);
  };
  // keep `up ? hi : lo`, add the partner's (lane ^ off) copy of it
  auto halve = [](float lo, float hi, bool up, int off) {
    const float send = up ? lo : hi, keep = up ? hi : lo;
    return keep + __shfl_xor_sync(0xffffffffu, send, off);
  };
  if (W == 4) {
    // window = rows g = 4 a .. 4 a + 3 of one r: xor 4 keeps head up4, xor 8 keeps row g + 8 up8; round jc: groups j = 4 jc .. + 3
    const int row = row_w0 + static_cast<int>(g) + (up8 ? 8 : 0);
    __nv_bfloat16* dst = at.ctx + static_cast<long long>(row / 4) * 1024 + head * 128 + 2 * static_cast<int>(q);
#pragma unroll
    for (int jc = 0; jc < 4; ++jc) {
      float v[4][2][2];                                 // [j][r][e]
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        float o0[2][2], o1[2][2];
        pv(0, 4 * jc + jj, o0);
        pv(1, 4 * jc + jj, o1);
#pragma unroll
        for (int r = 0; r < 2; ++r)
#pragma unroll
          for (int e = 0; e < 2; ++e) v[jj][r][e] = halve(o0[r][e], o1[r][e], up4, 4);
      }
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const float c0 = halve(v[jj][0][0], v[jj][1][0], up8, 8), c1 = halve(v[jj][0][1], v[jj][1][1], up8, 8);
        if (row < M) *reinterpret_cast<uint32_t*>(dst + 8 * (4 * jc + jj)) = pack_bf16x2(c0, c1);
      }
    }
  } else {
    // W == 16: window = all 16 rows: the lane's two rows first, then xor 4 keeps head up4, xor 8 keeps groups j = 8 up8 + .., xor 16
    // j = 8 up8 + 4 up16 + ..; round jc: groups jc, jc + 4, jc + 8, jc + 12, of which the lane stores jc + 4 up16 + 8 up8
    __nv_bfloat16* dst = at.ctx + static_cast<long long>(row_w0 / 16) * 1024 + head * 128 + 2 * static_cast<int>(q);
#pragma unroll
    for (int jc = 0; jc < 4; ++jc) {
      float v[4][2];                                    // [group jc + 4 k][e]
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        float o0[2][2], o1[2][2];
        pv(0, jc + 4 * k, o0);
        pv(1, jc + 4 * k, o1);
#pragma unroll
        for (int e = 0; e < 2; ++e) v[k][e] = halve(o0[0][e] + o0[1][e], o1[0][e] + o1[1][e], up4, 4);
      }
      float c[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float a = halve(v[0][e], v[2][e], up8, 8), b = halve(v[1][e], v[3][e], up8, 8);   // groups jc + 8 up8, jc + 4 + 8 up8
        c[e] = halve(a, b, up16, 16);
      }
      const int j = jc + (up16 ? 4 : 0) + (up8 ? 8 : 0);
      if (row_w0 < M) *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack_bf16x2(c[0], c[1]);
    }
  }
}

// Stage this tile's slices of col_a / col_b into shared memory (coalesced), then sync the 256 epilogue threads.
template <int kTileN>
__device__ __forceinline__ void stage_col_vectors(const GemmEpilogue& ep, int N, int col_tile0, float* s_col, int epi_tid,
                                                  bool single_buffer = false) {
  if (single_buffer) named_bar_sync(kEpiBarrierId, kEpiThreads);      // everyone is done reading the previous tile's vectors
  for (int c = epi_tid; c < kTileN; c += kEpiThreads) {
    const int col = col_tile0 + c;
    const bool ok = col < N;
    s_col[col_slot<kTileN>(0, c)] = (ok && ep.col_a != nullptr) ? __ldg(ep.col_a + col) : 0.f;
    s_col[col_slot<kTileN>(1, c)] = (ok && ep.col_b != nullptr) ? __ldg(ep.col_b + col) : 0.f;
  }
  named_bar_sync(kEpiBarrierId, kEpiThreads);
}

// The pair kernel's form of the same: the copies are issued with cp.async (zero fill for columns >= N and null vectors) and land
// while the tile's MMAs run; col_vectors_ready() before the epilogue reads them.  The caller has passed a barrier since the
// previous tile's vectors were last read (the buffer is single).  16-byte pieces (col_slot keeps them 16-byte aligned in shared
// memory) unless a vector's address is not 16-byte aligned; a null vector is zeroed with plain shared stores (no copy, no source
// address), and a piece past N reads 0 bytes from the vector's first element.
template <int kTileN>
__device__ __forceinline__ void stage_col_vectors_async(const float* col_a, const float* col_b, int N, int col_tile0, float* s_col,
                                                        int epi_tid) {
#pragma unroll
  for (int vec = 0; vec < 2; ++vec) {
    const float* v = vec == 0 ? col_a : col_b;
    if ((reinterpret_cast<uintptr_t>(v) & 15u) == 0) {
      for (int c = 4 * epi_tid; c < kTileN; c += 4 * kEpiThreads) {      // N is a multiple of 32: a piece is all in or all out
        const int col = col_tile0 + c;
        const uint32_t dst = smem_u32(s_col + col_slot<kTileN>(vec, c));
        if (v == nullptr) sts_u4(dst, 0u, 0u, 0u, 0u);               // made visible by col_vectors_ready's barrier
        else cp_async_16(dst, col < N ? v + col : v, col < N ? 16u : 0u);
      }
    } else {
      for (int c = epi_tid; c < kTileN; c += kEpiThreads) {
        const int col = col_tile0 + c;
        cp_async_4(smem_u32(s_col + col_slot<kTileN>(vec, c)), col < N ? v + col : v, col < N ? 4u : 0u);
      }
    }
  }
}
__device__ __forceinline__ void col_vectors_ready() {
  cp_async_wait_all();
  named_bar_sync(kEpiBarrierId, kEpiThreads);
}

// ------------------------------------------------------------------------------------------------
// Pair kernel, tiles stored through the TMA slabs (every instantiation): the epilogue works on the wgmma m64n256 fragments where
// they are, with no transpose.  Lane (g = lane / 4, q = lane % 4) of a warp holds rows g and g + 8 of the warp's 16 rows, columns
// 8 j + 2 q, +1 of both column halves; every value goes through the same explicit fma / add / mul sequence as in epilogue_tile, so
// the bits do not depend on which thread computes them.  The packed 16-bit pairs are already in the m8n8 matrix fragment form:
// stmatrix writes each 8 x 8 block's rows to their 128B-swizzled slab positions.  The warp writes both column halves, slab by slab
// with the halves interleaved so that both store warps stay busy, and hands each half-slab over with one arrive.
//   Row statistics keep epilogue_tile's order (sequential over the 128 rounded columns of a row and half): once both halves of a
// slab are written, lane l re-reads row l % 16, column half l / 16 of it in column order — before the next slab is written, which
// with dual output reuses the same activation buffer; the last slab of each half is handed over only once the statistics are
// stored, so that the store warp's tile-done release covers them.
//   kTower / kF16 as in epilogue_tile: the tower's residual is read at the lane's own fragment positions (one 4-byte load per
// 16-bit pair, one 8-byte load per fp32 pair); the projector's LayerNorm fold, row statistics, dual output and erf GELU are
// compiled out of the tower's instantiations.
//   acc: [column half][fragment registers]; rloc_w0 / row_w0: tile row / global row of the warp's first row; s_out: the [2 halves]
// [kOutBufs] slabs; full_bar / empty_bar: [2 halves][kOutBufs]; slab_seq: running slab number (both halves share it).
// ------------------------------------------------------------------------------------------------
template <int kOutBufs, bool kTower = false, bool kF16 = false>
__device__ __forceinline__ void epilogue_tile_frag(const GemmEpilogue& ep, int M, int N, const float (&acc)[2][64], int row_w0, int rloc_w0,
                                                   int col_tile0, const float* s_col, uint8_t* s_out, uint64_t* full_bar,
                                                   uint64_t* empty_bar, uint32_t slab_seq) {
  static_assert(kOutBufs == 2, "slab numbering: buffer = seq % 2");
  constexpr int kColsPerHalf = 128;
  const uint32_t lane = lane_id();
  const uint32_t g = lane >> 2, q = lane & 3u;
  const bool ln_fold = !kTower && ep.col_a != nullptr;
  const bool dual = !kTower && ep.dual != 0;
  const bool scale = ep.alpha != 1.0f;
  const bool do_stats = !kTower && ep.stats_out != nullptr;
  // the tower's residual rows g and g + 8 (nullptr: no residual, or the row is past M)
  const uint8_t* resid_row[2] = {nullptr, nullptr};
  if constexpr (kTower) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int row = row_w0 + static_cast<int>(g) + 8 * r;
      if (ep.resid != nullptr && row < M)
        resid_row[r] = static_cast<const uint8_t*>(ep.resid) + static_cast<long long>(row) * ep.ldr * (ep.resid_f32 ? 4 : 2);
    }
  }
  uint64_t rstd2[2], nmu2[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = row_w0 + static_cast<int>(g) + 8 * r;
    float mu = 0.f, rstd = 1.f;
    if (ln_fold && row < M) ln_row_stats(ep.stats_in, row, ep.stats_in_slots, ep.ln_inv_dim, ep.ln_eps, mu, rstd);
    rstd2[r] = pk2(rstd);
    nmu2[r] = pk2(-mu);
  }
  const uint64_t alpha2 = pk2(ep.alpha);
  // this lane's stmatrix row address: matrix m = lane / 8 of an x4 is (8-column group m / 2, rows 8 (m % 2) ..); rloc_w0 is a
  // multiple of 16, so the row's swizzle (row & 7) is lane & 7
  const uint32_t m_row = static_cast<uint32_t>(rloc_w0) + 8u * ((lane >> 3) & 1u) + (lane & 7u);
  const uint32_t m_grp = lane >> 4;
  const uint32_t out_addr = smem_u32(s_out);
  const uint32_t sa_addr = smem_u32(s_col + col_slot<256>(0, 0)), sb_addr = smem_u32(s_col + col_slot<256>(1, 0));
  // row statistics: this lane's row and column half, and its running sums of (y - shift), shift = the block's first value
  const int st_r = static_cast<int>(lane & 15u), st_h = static_cast<int>(lane >> 4);
  const uint32_t st_addr = out_addr + static_cast<uint32_t>(st_h * kOutBufs * kOutSlabBytes + (rloc_w0 + st_r) * kSlabRowBytes);
  float s1 = 0.f, s2 = 0.f, shift = 0.f;
#pragma unroll
  for (int s = 0; s < kColsPerHalf / kSlabCols; ++s) {
    // dual output: every 64-column slab exists twice — pre-activation (even slab number, buffer 0) and activation (odd, buffer 1)
    const uint32_t slab_pre = slab_seq + 2u * static_cast<uint32_t>(s);
    const uint32_t slab_q = dual ? slab_pre + 1u : slab_seq + static_cast<uint32_t>(s);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      uint64_t* full = full_bar + h * kOutBufs;
      uint64_t* empty = empty_bar + h * kOutBufs;
      // the TMA store that last used this staging buffer must have finished READING it (signalled by the store warp)
      if (dual) mbar_wait(&empty[slab_pre & 1u], ((slab_pre >> 1) & 1u) ^ 1u);
      mbar_wait(&empty[slab_q & 1u], ((slab_q >> 1) & 1u) ^ 1u);
      const uint32_t half_addr = out_addr + static_cast<uint32_t>(h * kOutBufs * kOutSlabBytes) + m_row * kSlabRowBytes;
#pragma unroll
      for (int x = 0; x < kSlabCols / 16; ++x) {
        // 8-column groups j0 = 8 s + 2 x and j0 + 1 of the half: v[2 jj + r] = row g + 8 r, columns 8 (j0 + jj) + 2 q, +1
        uint64_t v[4];
#pragma unroll
        for (int jj = 0; jj < 2; ++jj) {
          const int j = 8 * s + 2 * x + jj;
          const uint32_t c = static_cast<uint32_t>(h * kColsPerHalf + 8 * j + (h ? kColPad : 0)) + 2u * q;    // col_slot offset
          const uint64_t b2 = lds_f2(sb_addr + c * 4u);
          if (ln_fold) {     // v = fma(rstd, fma(-mu, col_a, v), col_b): explicit fmas, the same in every instantiation
            const uint64_t a2 = lds_f2(sa_addr + c * 4u);
#pragma unroll
            for (int r = 0; r < 2; ++r)
              v[2 * jj + r] = fma2(rstd2[r], fma2(nmu2[r], a2, pk2(acc[h][4 * j + 2 * r], acc[h][4 * j + 2 * r + 1])), b2);
          } else {
#pragma unroll
            for (int r = 0; r < 2; ++r) v[2 * jj + r] = add2(pk2(acc[h][4 * j + 2 * r], acc[h][4 * j + 2 * r + 1]), b2);
          }
          if constexpr (kTower) {   // one rounding of acc + bias + R: the residual add of a CLIP layer
            const long long col = col_tile0 + h * kColsPerHalf + 8 * j + 2 * static_cast<int>(q);
#pragma unroll
            for (int r = 0; r < 2; ++r) {
              if (resid_row[r] == nullptr || col >= N) continue;
              if (ep.resid_f32) {
                const float2 x = *reinterpret_cast<const float2*>(resid_row[r] + col * 4);
                v[2 * jj + r] = add2(v[2 * jj + r], pk2(x.x, x.y));
              } else {
                const uint32_t x = *reinterpret_cast<const uint32_t*>(resid_row[r] + col * 2);
                v[2 * jj + r] = add2(v[2 * jj + r], pk2(x2_lo<kF16>(x), x2_hi<kF16>(x)));
              }
            }
          }
        }
        // 16-byte piece of the slab row: groups 2 x + m_grp, XOR-swizzled like TMA's SWIZZLE_128B
        const uint32_t piece = ((2u * static_cast<uint32_t>(x) + m_grp) ^ (lane & 7u)) << 4;
        uint32_t w[4];
        if (dual) {        // the pre-activation slab
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            float lo, hi;
            upk2(v[k], lo, hi);
            w[k] = pack_bf16x2(lo, hi);
          }
          stmatrix_x4(half_addr + (slab_pre & 1u) * kOutSlabBytes + piece, w[0], w[1], w[2], w[3]);
        }
        if constexpr (kTower) {
          if (ep.gelu == 2) {
#pragma unroll
            for (int k = 0; k < 4; ++k) v[k] = quick_gelu_pk(v[k]);
          }
        } else if (ep.gelu) {
#pragma unroll
          for (int k = 0; k < 4; ++k) v[k] = gelu_erf_pk(v[k]);
        }
        if (scale) {       // alpha == 1 (every GEMM but in_proj_q): x * 1 is x, skip the multiply
#pragma unroll
          for (int k = 0; k < 4; ++k) v[k] = mul2(v[k], alpha2);
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          float lo, hi;
          upk2(v[k], lo, hi);
          w[k] = pack_x2<kF16>(lo, hi);
        }
        stmatrix_x4(half_addr + (slab_q & 1u) * kOutSlabBytes + piece, w[0], w[1], w[2], w[3]);
      }
      // slab written: make the generic-proxy writes visible to the async proxy, then one arrive per warp hands it to the store warp
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0 && !(do_stats && s == kColsPerHalf / kSlabCols - 1)) {
        if (dual) mbar_arrive(&full[slab_pre & 1u]);
        mbar_arrive(&full[slab_q & 1u]);
      }
    }
    if (do_stats) {
      // LayerNorm statistics of the ROUNDED values the next GEMM will read, from the warp's own rows of this slab (ordered by the
      // __syncwarp above; only this warp writes them, and only after this read), in column order (deterministic)
#pragma unroll
      for (int ci = 0; ci < kSlabRowBytes / 16; ++ci) {
        const uint4 u = lds_u4_ordered(st_addr + (slab_q & 1u) * kOutSlabBytes + static_cast<uint32_t>((ci ^ (st_r & 7)) << 4));
        const uint32_t pk[4] = {u.x, u.y, u.z, u.w};
        if (s == 0 && ci == 0) shift = bf16_lo(pk[0]);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float y0 = __fsub_rn(bf16_lo(pk[j]), shift), y1 = __fsub_rn(bf16_hi(pk[j]), shift);
          s1 = __fadd_rn(s1, __fadd_rn(y0, y1));
          s2 = fmaf(y0, y0, fmaf(y1, y1, s2));
        }
      }
    }
  }
  if (do_stats) {
    const int row = row_w0 + st_r;
    const int slot = (col_tile0 + st_h * kColsPerHalf) / kColsPerHalf;
    if (row < M && slot < ep.stats_out_slots) {
      const long long srow = ep.wm_s != 0 ? window_major_row(row, ep.wm_s) : row;
      // (mean, M2) of this 128-column block: mean = shift + s1/n, M2 = s2 - s1^2/n  (deviations from `shift` are O(std): no cancellation)
      constexpr float inv_n = 1.0f / kColsPerHalf;
      const float dm = __fmul_rn(s1, inv_n);
      reinterpret_cast<float2*>(ep.stats_out)[srow * ep.stats_out_slots + slot] = make_float2(__fadd_rn(shift, dm), fmaxf(fmaf(-s1, dm, s2), 0.f));
    }
    __syncwarp();                              // every lane's statistics are stored before the last slabs are handed over
    if (lane == 0) {
      const uint32_t slab_pre = slab_seq + 2u * static_cast<uint32_t>(kColsPerHalf / kSlabCols - 1);
      const uint32_t slab_q = dual ? slab_pre + 1u : slab_seq + static_cast<uint32_t>(kColsPerHalf / kSlabCols - 1);
#pragma unroll
      for (int h2 = 0; h2 < 2; ++h2) {
        if (dual) mbar_arrive(&full_bar[h2 * kOutBufs + (slab_pre & 1u)]);
        mbar_arrive(&full_bar[h2 * kOutBufs + (slab_q & 1u)]);
      }
    }
  }
}

// ================================================================================================
// One-CTA kernel: 128 x kBlockN tiles
// ================================================================================================
template <int kBlockN>
struct GemmConfig {
  static constexpr int kStages = 4;
  static constexpr int kABytes = kBlockM * kBlockK * 2;
  static constexpr int kBBytes = kBlockN * kBlockK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kColStageBytes = col_slot<kBlockN>(2, 0) * 4;   // [col_a | col_b], col_slot layout
  static constexpr int kBarrierBytes = 2 * kStages * 8;
  static constexpr int kSmemBytes = kStages * kStageBytes + kScratchBytes + kColStageBytes + kBarrierBytes + 1024;  // +1024: manual alignment
  static_assert(kSmemBytes <= 232448, "shared memory budget of an sm_90 SM (227 KiB)");
};

template <int kBlockN, bool kTower = false, bool kF16 = false>
__global__ void __launch_bounds__(kGemmThreads, 1)
tp_gemm_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, int M, int N, int K,
               int a_seg_rows, GemmEpilogue ep) {
  using Cfg = GemmConfig<kBlockN>;
  constexpr int kStages = Cfg::kStages;
  static_assert(kBlockN == 128 || kBlockN == 256, "BLOCK_N");
  static_assert(kTower || !kF16, "f16 instantiations are the tower's");

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* s_scratch = smem + kStages * Cfg::kStageBytes;
  float* s_col = reinterpret_cast<float*>(s_scratch + kScratchBytes);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(s_scratch + kScratchBytes + Cfg::kColStageBytes);
  uint64_t* empty_bar = full_bar + kStages;

  const int warp_idx = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
  const uint32_t lane = lane_id();

  const int num_m_blocks = (M + kBlockM - 1) / kBlockM;
  const int num_n_blocks = (N + kBlockN - 1) / kBlockN;
  const int num_tiles = num_m_blocks * num_n_blocks;
  const int num_k_blocks = (K + kBlockK - 1) / kBlockK;

  if (warp_idx == kTmaWarp && lane == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], kNumEpiWarps);      // one arrive per MMA warp
    }
    fence_barrier_init();
  }
  __syncthreads();
  grid_dependency_wait();                  // PDL: the prologue above overlapped the previous kernel's tail
  grid_launch_dependents();

  if (warp_idx >= kNumEpiWarps) {
    setmaxnreg_dec<kAuxRegs>();
    if (warp_idx == kTmaWarp && lane == 0) {
      // ======================================= TMA producer =======================================
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m_blk = tile / num_n_blocks;
        const int n_blk = tile - m_blk * num_n_blocks;
        for (int kb = 0; kb < num_k_blocks; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1u);
          uint8_t* sa = smem + stage * Cfg::kStageBytes;
          uint8_t* sb = sa + Cfg::kABytes;
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          if (a_seg_rows == 0) {
            tma_load_2d(sa, &tmap_a, &full_bar[stage], kb * kBlockK, m_blk * kBlockM);
          } else {
            // segmented A (3-D map, 64-row boxes): global row g -> (segment g / seg_rows, row g % seg_rows)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int g = m_blk * kBlockM + h * 64;
              const int seg = g / a_seg_rows;
              tma_load_3d(sa + h * (Cfg::kABytes / 2), &tmap_a, &full_bar[stage], kb * kBlockK, g - seg * a_seg_rows, seg);
            }
          }
          tma_load_2d(sb, &tmap_b, &full_bar[stage], kb * kBlockK, n_blk * kBlockN);
          if (++stage == kStages) { stage = 0; phase ^= 1u; }
        }
      }
    }
    __syncwarp();
  } else {
    // ======================================= MMA + epilogue (warpgroup = column half) =============
    setmaxnreg_inc<kMmaRegs>();
    const int e = warp_idx - kEpiWarp0;
    const int half = e >> 2;
    const int rloc = epi_row_1cta(warp_idx & 3, lane);
    const int epi_tid = e * 32 + static_cast<int>(lane);
    const uint32_t scratch = smem_u32(s_scratch + e * kScratchBytesPerWarp);
    constexpr int kN = kBlockN / 2;                  // columns per warpgroup
    int stage = 0;
    uint32_t phase = 0;
    float acc[2][kN / 2];
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int m_blk = tile / num_n_blocks;
      const int n_blk = tile - m_blk * num_n_blocks;
      stage_col_vectors<kBlockN>(ep, N, n_blk * kBlockN, s_col, epi_tid, true);
      mma_tile<kN, 2, 0, 0, kF16>(acc, smem, Cfg::kStageBytes, 0, Cfg::kABytes + half * kN * kBlockK * 2, full_bar, empty_bar, kStages, stage,
                                  phase, num_k_blocks);
      epilogue_tile<kBlockN, kTower, kF16>(ep, M, N, acc, scratch, m_blk * kBlockM + rloc, n_blk * kBlockN, half, s_col);
    }
  }
}

// ================================================================================================
// Pair kernel: 256 x 256 tiles (two CTAs of 128 rows each), GROUPED: one launch runs up to kMaxGroup independent GEMM problems
// (e.g. k_proj_1.2 | v_proj_1.2 | q_proj_1, which share no data but would each leave the machine with a partial last
// wave and pay launch + prologue + drain on their own).  Tiles are numbered across the problems of the group; every warp
// role walks the same sequence.
// ================================================================================================
struct Gemm2Config {
  static constexpr int kTileM = 256;
  static constexpr int kTileN = 256;
  static constexpr int kStages = 3;
  static constexpr int kOutBufs = 2;                             // staging buffers per column half: consecutive slabs alternate
  static constexpr int kABytes = kBlockM * kBlockK * 2;          // this CTA's 128 rows of A
  static constexpr int kBBytes = kTileN * kBlockK * 2;           // the whole B tile
  static constexpr int kStageBytes = kABytes + kBBytes;          // 48 KiB
  static constexpr int kOutBytes = 2 * kOutBufs * kOutSlabBytes; // [2 column halves][kOutBufs] output slabs for TMA stores
  static constexpr int kColStageBytes = col_slot<kTileN>(2, 0) * 4;   // [col_a | col_b], col_slot layout, ONE buffer (barrier before it is rewritten)
  static constexpr int kBarrierBytes = (2 * kStages + 4 * kOutBufs) * 8;   // ring + slab full/empty per half
  // 3 stages x 48 KiB + 4 x 16 KiB slabs + 16 KiB transpose scratch + 2 KiB + barriers = 226.1 KiB of the 227 KiB an SM offers: the
  // dynamic shared memory is declared 1024-byte aligned (no alignment slack), and the per-column vectors are single-buffered
  static constexpr int kSmemBytes = kStages * kStageBytes + kOutBytes + kScratchBytes + kColStageBytes + kBarrierBytes;
  static_assert(kSmemBytes <= 232448, "shared memory budget of an sm_90 SM (227 KiB)");
};

constexpr int kMaxGroup = 8;

constexpr int kMaxAParts = 4;

struct GemmProblem {
  CUtensorMap tmap_a, tmap_b, tmap_c;
  CUtensorMap tmap_cx[kBoxLevels - 1];       // further C maps of the segmented / window-major stores (see the store warps): boxes of
                                             // c_unit << level rows (segmented) or 8 * (level + 1) tokens (window-major); level 0 = tmap_c
  CUtensorMap tmap_a2, tmap_b2;              // kind 1: the value operands (tmap_a / tmap_b: the key operands)
  int kind;              // 0: GEMM with the fused epilogue; 1: KV-attention tile (see attn_epilogue_tile)
  int c_wm_s;            // != 0: tmap_c is the 5-D window-major map of GemmEpilogue::wm_s
  AttnParams attn;
  CUtensorMap tmap_a_more[kMaxAParts - 1];   // A given as several tensors side by side along K (e.g. the four CLIP hidden states
                                             // that the reference concatenates, clip_encoder.py:28-44): part p covers k-blocks
                                             // [p * a_kblocks_per_part, (p+1) * a_kblocks_per_part)
  int a_parts;           // 1: a single A tensor
  int a_kblocks_per_part;
  // TN form (ab_mn_major == 1) only, where A is never split: B given as several tensors side by side along N (the four CLIP hidden
  // states as the wgrad operand of k/v_proj.0), part p > 0 in tmap_a_more[p - 1]; part = n-block / b_nblocks_per_part
  int b_parts;           // 0 or 1: a single B tensor
  int b_nblocks_per_part;
  int b_seg_rows;        // TN form: 0: plain 2-D B; else rows per segment of the 3-D (cols, row, segment) B map (a multiple of 64)
  int M, N, K;
  int a_seg_rows;        // 0: plain 2-D A; else rows per segment of the 3-D (crop-strided) A map
  int ab_mn_major;       // 1: BOTH operands are given as row-major [K, M] / [K, N] matrices (wgrad: C = A^T . B, contraction over rows)
                         // 2: only B is ([K, N] row-major: dgrad C = A . B with the weight as stored); A is the usual K-major [M, K]
  int use_tma_store;     // C through TMA stores (0 when rows are scattered to arbitrary segment offsets)
  int c_seg_len;         // != 0: tmap_c (and the peer maps) are 3-D (cols, row in segment, segment): uniform-stride segmented output
  int c_unit;            //       gcd(c_seg_len, 128): every piece of a slab that belongs to one segment is a multiple of it
  int num_n_blocks;
  int num_tiles;         // = tiles_mn * k_splits
  int num_k_blocks;
  // split-K (wgrads whose output is a few tiles but whose contraction runs over every row of the batch): tile = (split, m, n),
  // split s covers k-blocks [s * kb_per_split, (s+1) * kb_per_split) and writes its fp32 partial to slice s of C (ep.out_f32)
  int k_splits;          // >= 1
  int kb_per_split;
  int tiles_mn;
  long long c_split_stride;   // floats between consecutive split slices of C
  // Dependencies between GEMMs of ONE launch (a chain of linears runs as a single persistent kernel: no ramp / drain / partial
  // last wave per layer).  Tiles are numbered problem after problem and every CTA pair walks its tiles in increasing order, so a
  // tile only ever waits for lower-numbered tiles: no deadlock as long as all CTAs are co-resident (grid <= one CTA per SM).
  int* done_counter;     // != nullptr: [ceil(M/256)] tile counter of THIS problem's output row blocks, +1 per (CTA, column half)
                         //             once that part of a tile is in global memory (bumped by the store warps)
  const int* dep_counter;// != nullptr: the A operand's row block m_blk is ready when dep_counter[m_blk >> dep_shift] >= dep_target
  int dep_target;        //             (= 4 * num_n_blocks of the producing problem: 2 CTAs x 2 column halves per tile)
  int dep_shift;         //             0 for GEMM -> GEMM (same row blocks); 31 for a single launch-wide counter (front work)
  int dep_span;          // != 0: the producer is a KV-attention problem: row block m_blk (256 queries) is complete after dep_per arrivals
  int dep_src_blocks;    //       from each of its source tiles [m_blk * dep_span, min((m_blk + 1) * dep_span, dep_src_blocks))
  int dep_per;
  int peer_out;          // C of this problem goes to the PeerStores maps (fused all-gather) instead of tmap_c
  GemmEpilogue ep;
};

// Optional prologue work of a chained launch: the point queries (builder.py:117-118: bilinear 24x24 -> g x g, align_corners=False
// == a fixed stencil per s x s window: the centre token for odd s, the mean of the centre 2x2 for even s; fp32, one bf16 rounding).
// Done by the epilogue warps of every CTA BEFORE their first tile — that time is otherwise idle (the first accumulator of the
// K=4096 GEMM takes ~33k cycles to appear), so the stencil costs nothing and needs no launch of its own.  Every CTA handles a
// strided share of the (query, 8-channel vector) items and then bumps done_counter once; the GEMM that reads q waits for
// gridDim.x arrivals.
struct FrontWork {
  const __nv_bfloat16* x0;   // nullptr: no front work in this launch
  __nv_bfloat16* q;          // [n_queries, 1024]
  long long crop_stride;     // elements between crops of x0
  long long n_queries;
  int s;                     // scale factor
  int* done_counter;
};

struct GemmGroup {
  GemmProblem p[kMaxGroup];
  int count;
  int total_tiles;            // tiles are numbered problem after problem
  FrontWork front;
};


// __grid_constant__ parameters of tp_gemm2_kernel: the kernel parameter space of sm_90 holds 32764 bytes
static_assert(sizeof(GemmGroup) + sizeof(PeerStores) <= 32764, "tp_gemm2_kernel's parameter block exceeds the 32 KB limit");

struct TileRef {
  const GemmProblem* pr;
  int m_blk, n_blk;
  int kb0, kb1;          // k-block range of this tile (the whole K unless the problem is split)
  int split;
};

__device__ __forceinline__ TileRef decode_tile(const GemmGroup& g, int tile) {
  int p = 0;
  while (p + 1 < g.count && tile >= g.p[p].num_tiles) {
    tile -= g.p[p].num_tiles;
    ++p;
  }
  TileRef t;
  t.pr = &g.p[p];
  t.split = 0;
  if (t.pr->k_splits > 1) {
    t.split = tile / t.pr->tiles_mn;
    tile -= t.split * t.pr->tiles_mn;
  }
  t.m_blk = tile / t.pr->num_n_blocks;
  t.n_blk = tile - t.m_blk * t.pr->num_n_blocks;
  t.kb0 = t.split * t.pr->kb_per_split;
  t.kb1 = t.kb0 + t.pr->kb_per_split < t.pr->num_k_blocks ? t.kb0 + t.pr->kb_per_split : t.pr->num_k_blocks;
  return t;
}

template <bool kTower = false, bool kF16 = false>
__global__ void __launch_bounds__(kGemmThreads, 1)
tp_gemm2_kernel(const __grid_constant__ GemmGroup grp, const __grid_constant__ PeerStores peers) {
  static_assert(kTower || !kF16, "f16 instantiations are the tower's");
  using Cfg = Gemm2Config;
  constexpr int kStages = Cfg::kStages;
  constexpr int kTileN = Cfg::kTileN;

  extern __shared__ __align__(1024) uint8_t smem_raw[];     // 1 KiB aligned: swizzle atoms of the operand tiles and output slabs
  uint8_t* smem = smem_raw;
  uint8_t* s_out = smem + kStages * Cfg::kStageBytes;                                  // 1 KiB aligned (swizzle atoms)
  uint8_t* s_scratch = s_out + Cfg::kOutBytes;
  float* s_col_base = reinterpret_cast<float*>(s_scratch + kScratchBytes);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(s_scratch + kScratchBytes + Cfg::kColStageBytes);
  uint64_t* empty_bar = full_bar + kStages;
  uint64_t* slab_full_bar = empty_bar + kStages;                // [2 halves][kOutBufs]
  uint64_t* slab_empty_bar = slab_full_bar + 2 * Cfg::kOutBufs; // [2 halves][kOutBufs]

  const int warp_idx = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
  const uint32_t lane = lane_id();
  const uint32_t cta_rank = blockIdx.x & 1u;                   // which 128 rows of the pair's 256-row tile this CTA computes
  const int num_tiles = grp.total_tiles;
  const int pair_idx = static_cast<int>(blockIdx.x >> 1);
  const int num_pairs = static_cast<int>(gridDim.x >> 1);

  if (warp_idx == kTmaWarp && lane == 0) {
    for (int i = 0; i < grp.count; ++i) {
      tma_prefetch_desc(&grp.p[i].tmap_a);
      for (int q = 1; q < grp.p[i].a_parts; ++q) tma_prefetch_desc(&grp.p[i].tmap_a_more[q - 1]);
      tma_prefetch_desc(&grp.p[i].tmap_b);
      if (grp.p[i].kind == 1) {
        tma_prefetch_desc(&grp.p[i].tmap_a2);
        tma_prefetch_desc(&grp.p[i].tmap_b2);
      }
      if (grp.p[i].use_tma_store) tma_prefetch_desc(&grp.p[i].tmap_c);
    }
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);                        // the producer's expect-tx arrive
      mbar_init(&empty_bar[i], kNumEpiWarps);            // one arrive per MMA warp
    }
    for (int i = 0; i < 2 * Cfg::kOutBufs; ++i) {
      mbar_init(&slab_full_bar[i], kNumEpiWarps);        // one arrive per epilogue warp (from its 16 lanes of the column half)
      mbar_init(&slab_empty_bar[i], 1);                  // the half's store warp
    }
    fence_barrier_init();
  }
  __syncthreads();
  // Programmatic dependent launch: everything above overlapped the tail of the previous kernel on the stream; from here
  // on we read what it wrote.  (No-op when the launch carries no PDL attribute.)
  grid_dependency_wait();
  grid_launch_dependents();                // the next kernel's CTAs may take over SMs as ours exit (they block in their own wait)
  if (warp_idx < kNumEpiWarps) {
    setmaxnreg_inc<kMmaRegs>();
    // ======================================= MMA + epilogue (own 128 rows, warpgroup = 64-row block) =
    const int e = warp_idx - kEpiWarp0;
    const int wg = e >> 2;
    const int rloc = epi_row(wg, warp_idx & 3, lane);
    const int half = epi_half(lane);
    const int epi_tid = e * 32 + static_cast<int>(lane);
    const uint32_t scratch = smem_u32(s_scratch + e * kScratchBytesPerWarp);
    int stage = 0;
    uint32_t phase = 0;
    uint32_t slab_seq = 0;
    float acc[2][kTileN / 4];
    if (!kTower && grp.front.x0 != nullptr) {
      // point queries: this CTA's share of the (query, 8-channel vector) items, 128 vectors per query
      const FrontWork& fw = grp.front;
      const int g = 24 / fw.s, mq = g * g;
      const int lo = (fw.s & 1) ? (fw.s - 1) / 2 : fw.s / 2 - 1;          // first tap inside the window (row and column)
      const long long items = fw.n_queries * 128;
      for (long long idx = static_cast<long long>(blockIdx.x) * kEpiThreads + epi_tid; idx < items; idx += static_cast<long long>(gridDim.x) * kEpiThreads) {
        const long long query = idx >> 7;
        const int vec = static_cast<int>(idx & 127);
        const long long n = query / mq;
        const int m = static_cast<int>(query - n * mq);
        const int hb = m / g, wb = m - hb * g;
        const __nv_bfloat16* base = fw.x0 + n * fw.crop_stride + vec * 8 + static_cast<long long>((hb * fw.s + lo) * 24 + wb * fw.s + lo) * 1024;
        uint4 o = __ldg(reinterpret_cast<const uint4*>(base));
        if (!(fw.s & 1)) {
          const uint4 b = __ldg(reinterpret_cast<const uint4*>(base + 1024)), c = __ldg(reinterpret_cast<const uint4*>(base + 24 * 1024)),
                      d = __ldg(reinterpret_cast<const uint4*>(base + 25 * 1024));
          // (0.25a + 0.25b) + (0.25c + 0.25d): the sequence of point_query_kernel, so both give the same bits; taps are scaled before
          // the adds, so no partial sum overflows when taps lie in bf16's top binade
          auto mean4 = [](uint32_t a_, uint32_t b_, uint32_t c_, uint32_t d_) {
            auto m4 = [](float a, float b, float c, float d) {
              return __fadd_rn(__fadd_rn(__fmul_rn(0.25f, a), __fmul_rn(0.25f, b)), __fadd_rn(__fmul_rn(0.25f, c), __fmul_rn(0.25f, d)));
            };
            return pack_bf16x2(m4(bf16_lo(a_), bf16_lo(b_), bf16_lo(c_), bf16_lo(d_)), m4(bf16_hi(a_), bf16_hi(b_), bf16_hi(c_), bf16_hi(d_)));
          };
          o = make_uint4(mean4(o.x, b.x, c.x, d.x), mean4(o.y, b.y, c.y, d.y), mean4(o.z, b.z, c.z, d.z), mean4(o.w, b.w, c.w, d.w));
        }
        *reinterpret_cast<uint4*>(fw.q + query * 1024 + vec * 8) = o;
      }
      named_bar_sync(kEpiBarrierId, kEpiThreads);           // every epilogue thread's stores are issued ...
      if (epi_tid == 0) {
        __threadfence();                                     // ... and ordered (cumulatively) before the release below
        red_release_gpu_add(fw.done_counter, 1);
      }
    }
    for (int tile = pair_idx; tile < num_tiles; tile += num_pairs) {
      const TileRef t = decode_tile(grp, tile);
      const GemmProblem& pr = *t.pr;
      float* s_col = s_col_base;
      const int row_tile0 = t.m_blk * Cfg::kTileM + static_cast<int>(cta_rank) * kBlockM;
      const int row = row_tile0 + rloc;
      if (!kTower && pr.kind == 1) {
        const AttnParams& at = pr.attn;
        const int rloc_w0 = 64 * wg + 16 * (warp_idx & 3);
        const uint32_t q_scratch = smem_u32(s_scratch);
        named_bar_sync(kEpiBarrierId, kEpiThreads);          // everyone is done reading the previous tile's vectors and scratch
        stage_col_vectors_async<kTileN>(at.wsum_k, at.cst_k, pr.N, t.n_blk * kTileN, s_col, epi_tid);
        // the first stage is full: the producer has acquired y_k, y_v, their statistics and q' (tile counters); mma_tile's own wait
        // on it returns at once
        mbar_wait(&full_bar[stage], phase);
        float4 st[2];
        attn_load_stats(at.stats_k, pr.M, row_tile0 + rloc_w0, st);
        attn_load_q(at, pr.M, row_tile0, t.n_blk, q_scratch, epi_tid);
        mma_tile<kTileN, 1, 0, 0>(acc, smem, Cfg::kStageBytes, wg * 8192, Cfg::kABytes, full_bar, empty_bar, kStages, stage, phase, pr.num_k_blocks);
        float mu, rstd;                                      // lanes 0-15: of row row_tile0 + rloc_w0 + lane
        attn_row_stats(at, st, pr.M, row_tile0 + rloc_w0, mu, rstd);
        attn_load_stats(at.stats_v, pr.M, row_tile0 + rloc_w0, st);
        col_vectors_ready();                                 // also the q' copies
        float p[2][2];
        attn_scores(at, acc, mu, rstd, rloc_w0, q_scratch, s_col, p);
        attn_row_stats(at, st, pr.M, row_tile0 + rloc_w0, mu, rstd);
        named_bar_sync(kEpiBarrierId, kEpiThreads);          // everyone is done reading phase K's vectors
        stage_col_vectors_async<kTileN>(at.wsum_v, at.cst_v, pr.N, t.n_blk * kTileN, s_col, epi_tid);
        mma_tile<kTileN, 1, 0, 0>(acc, smem, Cfg::kStageBytes, wg * 8192, Cfg::kABytes, full_bar, empty_bar, kStages, stage, phase, pr.num_k_blocks);
        col_vectors_ready();
        attn_pv(at, pr.M, acc, mu, rstd, row_tile0 + rloc_w0, t.n_blk, p, s_col);
        if (at.done_counter != nullptr) {
          named_bar_sync(kEpiBarrierId, kEpiThreads);       // every epilogue thread's ctx stores are issued ...
          if (epi_tid == 0) {
            __threadfence();                                 // ... and ordered (cumulatively) before the release
            red_release_gpu_add(at.done_counter + ((static_cast<long long>(t.m_blk) * Cfg::kTileM / (at.s * at.s)) >> 8), 1);
          }
        }
        continue;
      }
      named_bar_sync(kEpiBarrierId, kEpiThreads);            // everyone is done reading the previous tile's vectors
      stage_col_vectors_async<kTileN>(pr.ep.col_a, pr.ep.col_b, pr.N, t.n_blk * kTileN, s_col, epi_tid);
      const int n_kb = t.kb1 - t.kb0;
      if (!kTower && pr.ab_mn_major == 1)
        mma_tile<kTileN, 1, 1, 1>(acc, smem, Cfg::kStageBytes, wg * 8192, Cfg::kABytes, full_bar, empty_bar, kStages, stage, phase, n_kb);
      else if (!kTower && pr.ab_mn_major == 2)
        mma_tile<kTileN, 1, 0, 1>(acc, smem, Cfg::kStageBytes, wg * 8192, Cfg::kABytes, full_bar, empty_bar, kStages, stage, phase, n_kb);
      else
        mma_tile<kTileN, 1, 0, 0, kF16>(acc, smem, Cfg::kStageBytes, wg * 8192, Cfg::kABytes, full_bar, empty_bar, kStages, stage, phase, n_kb);
      col_vectors_ready();
      if (pr.use_tma_store) {
        const int rloc_w0 = 64 * wg + 16 * (warp_idx & 3);
        epilogue_tile_frag<Cfg::kOutBufs, kTower, kF16>(pr.ep, pr.M, pr.N, acc, row_tile0 + rloc_w0, rloc_w0, t.n_blk * kTileN, s_col, s_out,
                                                        slab_full_bar, slab_empty_bar, slab_seq);
        slab_seq += (kTileN / 2 / kSlabCols) * (pr.ep.dual ? 2 : 1);                        // slabs per tile and column half
      } else {
        epilogue_tile<kTileN, kTower, kF16, 4>(pr.ep, pr.M, pr.N, acc, scratch, row, t.n_blk * kTileN, half, s_col,
                                               static_cast<long long>(t.split) * pr.c_split_stride);
      }
    }
  } else {
    setmaxnreg_dec<kAuxRegs>();
  if (warp_idx == kTmaWarp) {
    // ======================================= TMA producer (both CTAs) ============================
    // Whole warp runs the loop (uniform control flow); one elected lane issues the arrive + TMA instructions.
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = pair_idx; tile < num_tiles; tile += num_pairs) {
      const TileRef t = decode_tile(grp, tile);
      const GemmProblem& pr = *t.pr;
      const int row0 = t.m_blk * Cfg::kTileM + static_cast<int>(cta_rank) * kBlockM;          // my 128 rows of A
      const int brow0 = t.n_blk * kTileN;                                                     // the whole B tile
      // segmented A (3-D map, 64-row boxes): global row g -> (segment g / seg_rows, row g % seg_rows); hoisted per tile
      if (pr.dep_counter != nullptr) {
        // A's row block is written by an earlier problem of this launch: wait until all its tiles have been published (acquire),
        // then order the TMA (async proxy) reads after the acquire
        int target = pr.dep_target;
        if (pr.dep_span != 0) {
          const int lo = t.m_blk * pr.dep_span;
          const int hi = lo + pr.dep_span < pr.dep_src_blocks ? lo + pr.dep_span : pr.dep_src_blocks;
          target = (hi - lo) * pr.dep_per;
        }
        wait_counter_at_least(pr.dep_counter + (t.m_blk >> pr.dep_shift), target);
        fence_proxy_async_all();
      }
      if (pr.kind == 1) {
        // KV-attention tile: y_k . W_ik(head pair)^T, then y_v . W_iv(head pair)^T, through the same ring
        const AttnParams& at = pr.attn;
        if (at.k_counter != nullptr) {
          // y_k / y_v were stored window-major by raster-ordered GEMMs of this launch: wait for every raster row block of the
          // crops this tile touches, and for the q' row block of its windows
          const long long r_lo = static_cast<long long>(t.m_blk) * Cfg::kTileM;
          const long long r_hi = r_lo + Cfg::kTileM < pr.M ? r_lo + Cfg::kTileM : pr.M;
          const int n_blocks = (pr.M + Cfg::kTileM - 1) / Cfg::kTileM;
          int b_lo = static_cast<int>((r_lo / 576) * 576 / Cfg::kTileM);
          int b_hi = static_cast<int>((((r_hi - 1) / 576 + 1) * 576 + Cfg::kTileM - 1) / Cfg::kTileM);
          if (b_hi > n_blocks) b_hi = n_blocks;
          for (int b = b_lo; b < b_hi; ++b) {
            wait_counter_at_least(at.k_counter + b, at.kv_target);
            wait_counter_at_least(at.v_counter + b, at.kv_target);
          }
          if (at.q_counter != nullptr) wait_counter_at_least(at.q_counter + ((r_lo / (at.s * at.s)) >> 8), at.q_target);
          fence_proxy_async_all();
        }
        for (int op = 0; op < 2; ++op) {            // phase K, then phase V: two ordinary 256-wide k-loops (brow0: the head pair's weight rows)
          const CUtensorMap* ta = op == 0 ? &pr.tmap_a : &pr.tmap_a2;
          const CUtensorMap* tb = op == 0 ? &pr.tmap_b : &pr.tmap_b2;
          for (int kb = 0; kb < pr.num_k_blocks; ++kb) {
            mbar_wait(&empty_bar[stage], phase ^ 1u);
            if (elect_one()) {
              uint8_t* sa = smem + stage * Cfg::kStageBytes;
              mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
              tma_load_2d(sa, ta, &full_bar[stage], kb * kBlockK, row0);
              tma_load_2d(sa + Cfg::kABytes, tb, &full_bar[stage], kb * kBlockK, brow0);
              tma_load_2d(sa + Cfg::kABytes + Cfg::kBBytes / 2, tb, &full_bar[stage], kb * kBlockK, brow0 + kTileN / 2);
            }
            __syncwarp();
            if (++stage == kStages) { stage = 0; phase ^= 1u; }
          }
        }
        continue;
      }
      int seg0 = 0, srow0 = 0, seg1 = 0, srow1 = 0;
      if (pr.a_seg_rows != 0) {
        seg0 = row0 / pr.a_seg_rows;
        srow0 = row0 - seg0 * pr.a_seg_rows;
        seg1 = (row0 + 64) / pr.a_seg_rows;
        srow1 = row0 + 64 - seg1 * pr.a_seg_rows;
      }
      for (int kb = t.kb0; kb < t.kb1; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1u);
        if (elect_one()) {
          uint8_t* sa = smem + stage * Cfg::kStageBytes;
          uint8_t* sb = sa + Cfg::kABytes;
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          if (pr.ab_mn_major == 1) {
            // boxes of [64 K-rows x 64 MN-elements]: coordinates (mn, k); two MN atoms of A, four of B per CTA
            tma_load_2d(sa, &pr.tmap_a, &full_bar[stage], row0, kb * kBlockK);
            tma_load_2d(sa + Cfg::kABytes / 2, &pr.tmap_a, &full_bar[stage], row0 + 64, kb * kBlockK);
          } else {
            const int part = pr.a_parts > 1 ? kb / pr.a_kblocks_per_part : 0;
            const CUtensorMap* ta = part == 0 ? &pr.tmap_a : &pr.tmap_a_more[part - 1];
            const int ka = (kb - part * pr.a_kblocks_per_part) * kBlockK;      // K coordinate inside this part
            if (pr.a_seg_rows == 0) {
              tma_load_2d(sa, ta, &full_bar[stage], ka, row0);
            } else {
              tma_load_3d(sa, ta, &full_bar[stage], ka, srow0, seg0);
              tma_load_3d(sa + Cfg::kABytes / 2, ta, &full_bar[stage], ka, srow1, seg1);
            }
          }
          if (pr.ab_mn_major == 0) {
            tma_load_2d(sb, &pr.tmap_b, &full_bar[stage], kb * kBlockK, brow0);
            tma_load_2d(sb + Cfg::kBBytes / 2, &pr.tmap_b, &full_bar[stage], kb * kBlockK, brow0 + kTileN / 2);
          } else if (pr.b_parts <= 1 && pr.b_seg_rows == 0) {   // 1 (TN) and 2 (NN): B is a row-major [K, N] matrix
#pragma unroll
            for (int a4 = 0; a4 < 4; ++a4)
              tma_load_2d(sb + a4 * (Cfg::kBBytes / 4), &pr.tmap_b, &full_bar[stage], brow0 + a4 * 64, kb * kBlockK);
          } else {
            // TN form with B split along N: the part that holds this tile's 256 columns, and the tile's first column inside it
            const int bpart = pr.b_parts > 1 ? t.n_blk / pr.b_nblocks_per_part : 0;
            const CUtensorMap* tb = bpart == 0 ? &pr.tmap_b : &pr.tmap_a_more[bpart - 1];
            const int bcol0 = bpart == 0 ? brow0 : (t.n_blk - bpart * pr.b_nblocks_per_part) * kTileN;
            if (pr.b_seg_rows == 0) {
#pragma unroll
              for (int a4 = 0; a4 < 4; ++a4)
                tma_load_2d(sb + a4 * (Cfg::kBBytes / 4), tb, &full_bar[stage], bcol0 + a4 * 64, kb * kBlockK);
            } else {
              // segmented K rows (TN form, 3-D map): K row g -> (segment g / seg_rows, row g % seg_rows); seg_rows is a multiple of
              // 64, so a k-block never straddles two segments (576 = 9 x 64: one crop of a [:,1:] CLIP hidden state)
              const int g = kb * kBlockK;
              const int seg = g / pr.b_seg_rows;
#pragma unroll
              for (int a4 = 0; a4 < 4; ++a4)
                tma_load_3d(sb + a4 * (Cfg::kBBytes / 4), tb, &full_bar[stage], bcol0 + a4 * 64, g - seg * pr.b_seg_rows, seg);
            }
          }
        }
        __syncwarp();
        if (++stage == kStages) { stage = 0; phase ^= 1u; }
      }
    }
  } else if (warp_idx == kStoreWarp0 || warp_idx == kStoreWarp0 + 1) {
    // ======================================= store warps (both CTAs, one per column half) =========
    // Walks the same tile sequence as the epilogue warps.  Per slab: wait until the 8 epilogue warps have written their rows of
    // it (mbarrier), issue the TMA store(s) — plain 2-D box, clipped 3-D boxes for segmented rows, one per peer GPU for the
    // fused all-gather —, wait until the copy engine has READ the buffer and hand it back.  Per tile of a GEMM that others in
    // this launch depend on: wait for the stores to be PERFORMED, then publish the tile (release) on its row block's counter.
    const int half = warp_idx - kStoreWarp0;
    uint64_t* full = slab_full_bar + half * Cfg::kOutBufs;
    uint64_t* empty = slab_empty_bar + half * Cfg::kOutBufs;
    uint32_t q = 0;
    for (int tile = pair_idx; tile < num_tiles; tile += num_pairs) {
      const TileRef t = decode_tile(grp, tile);
      const GemmProblem& pr = *t.pr;
      if (!pr.use_tma_store) continue;
      const int row_tile0 = t.m_blk * Cfg::kTileM + static_cast<int>(cta_rank) * kBlockM;
      const bool to_peers = pr.peer_out != 0 && peers.count > 0;
      const int n_maps = to_peers ? peers.count : 1;
      const int dual = pr.ep.dual != 0 ? 1 : 0;     // every column slab twice: pre-activation (tmap_cx[0]) then activation (tmap_c)
      for (int slab = 0; slab < (kTileN / 2 / kSlabCols) << dual; ++slab, ++q) {
        const uint32_t buf = q & 1u;
        mbar_wait(&full[buf], (q >> 1) & 1u);
        {
          // Every TMA store of this slab is a JOB; lane l issues jobs l, l + 32, ...  All lanes walk the same (cheap) enumeration of the
          // slab's pieces and keep the parameters of their own jobs, then issue them together: the up to 88 stores of a packed-row
          // slab that goes to eight GPUs leave the warp in two or three instructions instead of one lane issuing them one by one.
          const uint8_t* src = s_out + (half * Cfg::kOutBufs + static_cast<int>(buf)) * kOutSlabBytes;
          const int col = t.n_blk * kTileN + half * (kTileN / 2) + (slab >> dual) * kSlabCols;
          constexpr int kJobsPerLane = 3;                  // 96 jobs per slab at most (host-checked: pieces x destinations)
          const CUtensorMap* jmap[kJobsPerLane];
          int jlo[kJobsPerLane], jc1[kJobsPerLane], jc2[kJobsPerLane], jc3[kJobsPerLane], jc4[kJobsPerLane];
#pragma unroll
          for (int k = 0; k < kJobsPerLane; ++k) jmap[k] = nullptr;
          int job = 0;
          auto add = [&](const CUtensorMap* mp, int lo, int c1, int c2, int c3, int c4) {
#pragma unroll
            for (int k = 0; k < kJobsPerLane; ++k)
              if (job == static_cast<int>(lane) + 32 * k) { jmap[k] = mp; jlo[k] = lo; jc1[k] = c1; jc2[k] = c2; jc3[k] = c3; jc4[k] = c4; }
            ++job;
          };
          // TMA stores must lie entirely inside the tensor (a box that sticks out of a segment is not relied on), so every piece of
          // a slab goes out through boxes of EXACTLY its size: a few maps per destination with box heights unit << level.
          int kind = 2;                                    // dimensionality of this problem's stores: 2, 3 or 5
          if (pr.c_wm_s != 0) {
            // Raster rows -> window-major rows: the slab is cut at token-row boundaries (24 tokens; crops are 24 token rows, so
            // token row R24 = global row / 24 = (crop * g + hb) * s + hi).  Slab edges fall on multiples of 8 tokens — a whole
            // number of windows for s in {2, 4, 8} —, so a piece holds 8, 16 or 24 tokens: map (tokens / 8 - 1), a
            // (channel, wi, -, wb) box of that many windows at (hi, crop-and-hb).
            kind = 5;
            const int sf = pr.c_wm_s;
            const int n_r24 = pr.M / 24;
            int r24 = row_tile0 / 24;
            for (int a = r24 * 24 - row_tile0; a < kBlockM && r24 < n_r24; a += 24, ++r24) {
              const int lo = max(a, 0), hi = min(a + 24, kBlockM);
              const int lvl = (hi - lo) / 8 - 1;
              add(lvl == 0 ? &pr.tmap_c : &pr.tmap_cx[lvl - 1], lo, 0, r24 % sf, (lo - a) / sf, r24 / sf);    // (c, wi, hi, wb, crop-and-hb)
            }
          } else if (pr.c_seg_len == 0) {
            if (dual && (slab & 1) == 0) add(&pr.tmap_cx[0], 0, row_tile0, 0, 0, 0);
            else
              for (int p = 0; p < n_maps; ++p) add(to_peers ? &peers.m[p][0] : &pr.tmap_c, 0, row_tile0, 0, 0, 0);
          } else {
            // Segmented output rows (global row g = seg * seg_len + r  ->  map coordinate (col, r, seg)): the slab's 128 rows are
            // cut at segment boundaries.  Runs of up to 3 WHOLE segments leave as one (cols, seg_len, k) box per destination; a
            // partial piece of L = n * unit rows leaves as one box per set bit of n (largest first).
            kind = 3;
            const int n_segs = pr.M / pr.c_seg_len;
            const bool whole_ok = to_peers && peers.whole != 0;
            int seg = row_tile0 / pr.c_seg_len;
            int a = seg * pr.c_seg_len - row_tile0;
            while (a < kBlockM && seg < n_segs) {
              if (whole_ok && a >= 0 && a + pr.c_seg_len <= kBlockM) {
                int k = 1;
                while (k < kWholeLevels && a + (k + 1) * pr.c_seg_len <= kBlockM && seg + k < n_segs) ++k;
                for (int p = 0; p < n_maps; ++p) add(&peers.m[p][kBoxLevels + k - 1], a, 0, seg, 0, 0);
                a += k * pr.c_seg_len;
                seg += k;
                continue;
              }
              int lo = max(a, 0);
              const int hi = min(a + pr.c_seg_len, kBlockM);
              for (int lvl = kBoxLevels - 1; lvl >= 0; --lvl) {
                const int rows = pr.c_unit << lvl;
                while (hi - lo >= rows) {
                  for (int p = 0; p < n_maps; ++p)
                    add(to_peers ? &peers.m[p][lvl] : (lvl == 0 ? &pr.tmap_c : &pr.tmap_cx[lvl - 1]), lo, lo - a, seg, 0, 0);
                  lo += rows;
                }
              }
              a += pr.c_seg_len;
              ++seg;
            }
          }
          if (job > 32 * kJobsPerLane) __trap();       // cannot happen: the host rejects shapes whose worst slab needs more jobs
#pragma unroll
          for (int k = 0; k < kJobsPerLane; ++k) {
            if (jmap[k] != nullptr) {
              const uint8_t* from = src + jlo[k] * kSlabRowBytes;
              if (kind == 2) tma_store_2d(jmap[k], from, col, jc1[k]);
              else if (kind == 3) tma_store_3d(jmap[k], from, col, jc1[k], jc2[k]);
              else tma_store_5d(jmap[k], from, col, jc1[k], jc2[k], jc3[k], jc4[k]);
            }
          }
          bulk_commit_group();
          bulk_wait_group_read<0>();               // this lane's stores have read the buffer ...
          __syncwarp();                            // ... and so have everybody else's: the epilogue warps may overwrite it
          if (lane == 0) mbar_arrive(&empty[buf]);
        }
        __syncwarp();
      }
      if (pr.done_counter != nullptr) {
        bulk_wait_group<0>();                      // every lane: its stores of this CTA-half's part of the tile are in global memory ...
        fence_proxy_async_all();                   // ... (async-proxy writes) ordered before the generic-proxy release below
        __syncwarp();
        if (lane == 0) red_release_gpu_add(pr.done_counter + t.m_blk, 1);
        __syncwarp();
      }
    }
    bulk_wait_group<0>();                          // my half's last TMA stores have been performed
    if (peers.count > 0) __threadfence_system();   // ... and are ordered before the cross-GPU barrier that follows the kernel
    __syncwarp();
  }
  }
}

}  // namespace tp
