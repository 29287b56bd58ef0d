// C ABI of libtokenpacker_b200.so (see include/tokenpacker_b200.h).  Host-side orchestration only: tensor-map
// encoding, workspace carving and kernel launches on the caller's stream.  No allocation, no synchronisation
// (except tp_forward_host), no global mutable state.
#include <limits.h>
#include <atomic>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <map>
#include <tuple>
#include <vector>

#include "../../include/tokenpacker_b200.h"
#include "../../include/tokenpacker_b200_clip_tower.h"
#include "../../include/tokenpacker_b200_clip_tower_f16.h"
#include "../../include/tokenpacker_b200_clip_tower_train.h"
#include "../../include/tokenpacker_b200_clip_tower_ckpt.h"
#include "../../include/tokenpacker_b200_clip_tower_embed.h"
#include "../../include/tokenpacker_b200_clip_tower_crop_grad.h"
#include "../../include/tokenpacker_b200_clip_tower_interleaved.h"
#include "../../include/tokenpacker_b200_clip_u8.h"
#include "../../include/tokenpacker_b200_hd_u8.h"
#include "../../include/tokenpacker_b200_input_grad.h"
#include "../../include/tokenpacker_b200_layers.h"
#include "../../include/tokenpacker_b200_jpeg.h"
#include "../../include/tokenpacker_b200_png.h"
#include "tp_gemm.cuh"
#include "tp_kernels.cuh"
#include "tp_backward.cuh"
#include "tp_clip_tower.cuh"
#include "tp_clip_tower_train.cuh"
#include "tp_clip_tower_embed.cuh"
#include "tp_jpeg.cuh"
#include "tp_png.cuh"

namespace {

using namespace tp;

thread_local char g_last_cuda_error[256] = "";
std::atomic<unsigned long long> g_launch_count{0};   // kernels launched by this library, all host threads (autograd runs backward on its own thread)

#define TP_CUDA(call)                                                                                        \
  do {                                                                                                       \
    cudaError_t err__ = (call);                                                                              \
    if (err__ != cudaSuccess) {                                                                              \
      snprintf(g_last_cuda_error, sizeof(g_last_cuda_error), "%s: %s", #call, cudaGetErrorString(err__));    \
      return TP_ERR_CUDA;                                                                                    \
    }                                                                                                        \
  } while (0)

#define TP_TRY(expr)                  \
  do {                                \
    int st__ = (expr);                \
    if (st__ != TP_OK) return st__;   \
  } while (0)

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// ------------------------------------------------------------------------------------------------
// TMA tensor maps.  cuTensorMapEncodeTiled is resolved through the runtime so that the library has no link-time
// dependency on libcuda.so (it must dlopen on a box without a driver for the CPU-side ABI test).
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_tiled_fn() {
  static EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
      p = nullptr;
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  return fn;
}

// bf16 tensor of `rank` dimensions, innermost first: extents `dims`, byte strides `strides` of dimensions 1 .. rank-1, boxes of
// `box` elements.  Every box is 64 columns wide (128 bytes: one row of the 128-byte swizzle the operand tiles and output slabs use).
static_assert(kSlabCols == kBlockK, "output slabs and operand tiles share the 64-column, 128-byte swizzle rows");
int encode_bf16_map(CUtensorMap* map, const void* ptr, int rank, const cuuint64_t* dims, const cuuint64_t* strides, const cuuint32_t* box) {
  EncodeTiledFn fn = encode_tiled_fn();
  if (fn == nullptr) {
    snprintf(g_last_cuda_error, sizeof(g_last_cuda_error), "cuTensorMapEncodeTiled entry point not found");
    return TP_ERR_CUDA;
  }
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) != 0) return TP_ERR_INVALID_ARGUMENT;
  for (int i = 0; i < rank - 1; ++i)
    if (strides[i] % 16 != 0) return TP_ERR_INVALID_ARGUMENT;
  const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, static_cast<cuuint32_t>(rank), const_cast<void*>(ptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    snprintf(g_last_cuda_error, sizeof(g_last_cuda_error), "cuTensorMapEncodeTiled(%dd) failed: %d", rank, static_cast<int>(r));
    return TP_ERR_CUDA;
  }
  return TP_OK;
}

// bf16 matrix [rows, cols] with row stride ld (elements); box = 64 columns x box_rows rows.
int make_map_2d(CUtensorMap* map, const void* ptr, long long rows, long long cols, long long ld, int box_rows) {
  const cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  const cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld) * 2};
  const cuuint32_t box[2] = {static_cast<cuuint32_t>(kBlockK), static_cast<cuuint32_t>(box_rows)};
  return encode_bf16_map(map, ptr, 2, dims, strides, box);
}

// bf16 tensor [segs, seg_rows, cols] with row stride ld and segment stride seg_stride (elements); box 64 x box_rows x box_segs.
int make_map_3d(CUtensorMap* map, const void* ptr, long long segs, long long seg_rows, long long cols, long long ld,
                long long seg_stride, int box_rows = 64, int box_segs = 1) {
  const cuuint64_t dims[3] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(seg_rows), static_cast<cuuint64_t>(segs)};
  const cuuint64_t strides[2] = {static_cast<cuuint64_t>(ld) * 2, static_cast<cuuint64_t>(seg_stride) * 2};
  const cuuint32_t box[3] = {static_cast<cuuint32_t>(kBlockK), static_cast<cuuint32_t>(box_rows), static_cast<cuuint32_t>(box_segs)};
  return encode_bf16_map(map, ptr, 3, dims, strides, box);
}

// Window-major destination of a raster-ordered [crops * 576, cols] bf16 matrix (scale factor s, g = 24 / s): dims
// (channel, wi, hi, wb, crop-and-hb) — ordered by increasing stride, as the tensor-map encoder wants —, box = 64 channels x s x 1 x
// (box_tokens / s) x 1 = box_tokens consecutive tokens of one token row (hi has extent 1 in the box, so the box is traversed
// wi-then-wb: raster order).  box_tokens in {8, 16, 24}: stores never stick out of the tensor (that faults), so each piece of a
// slab uses the map of exactly its size.
int make_map_wm(CUtensorMap* map, const void* ptr, long long rows, long long cols, long long ld, int s, int box_tokens) {
  if (rows % 576 != 0 || (s != 2 && s != 4 && s != 8) || box_tokens % s != 0 || box_tokens > 24) return TP_ERR_INVALID_ARGUMENT;
  const int g = 24 / s;
  const cuuint64_t dims[5] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(s), static_cast<cuuint64_t>(s), static_cast<cuuint64_t>(g),
                              static_cast<cuuint64_t>(rows / 576 * g)};
  const cuuint64_t row_b = static_cast<cuuint64_t>(ld) * 2;
  const cuuint64_t strides[4] = {row_b, row_b * s, row_b * s * s, row_b * s * s * g};
  const cuuint32_t box[5] = {static_cast<cuuint32_t>(kSlabCols), static_cast<cuuint32_t>(s), 1, static_cast<cuuint32_t>(box_tokens / s), 1};
  return encode_bf16_map(map, ptr, 5, dims, strides, box);
}

// Height of the smallest store box of a uniform-stride segmented output (packed HD rows): gcd(seg_len, 128).  Every piece of a
// 128-row slab that belongs to one segment is a multiple of it.  The pair kernel's segmented stores need it to be at least 4, which
// rules out scale factors 8 and 24 (M = 9, 1); the one-CTA kernels store such rows one by one.
int seg_store_unit(long long seg_len) {
  int unit = 128;
  while (seg_len % unit != 0) unit >>= 1;
  return unit;
}

struct DeviceInfo {
  int sms;
};

int device_info(DeviceInfo* info) {
  int dev = 0, major = 0;
  TP_CUDA(cudaGetDevice(&dev));
  TP_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  if (major != 9) return TP_ERR_UNSUPPORTED_DEVICE;
  TP_CUDA(cudaDeviceGetAttribute(&info->sms, cudaDevAttrMultiProcessorCount, dev));
  return TP_OK;
}

// ------------------------------------------------------------------------------------------------
// GEMM launch
// ------------------------------------------------------------------------------------------------
struct AOperand {
  const void* ptr;
  long long ld;          // row stride (elements)
  long long seg_rows;    // 0: plain 2-D [M,K]; else rows per segment of a 3-D [M/seg_rows, seg_rows, K] tensor
  long long seg_stride;  // elements between segments
  const void* more[3] = {nullptr, nullptr, nullptr};   // further A tensors side by side along K (same ld / segmentation), pair kernel only
  int parts = 1;
};

// Every kernel of the path is launched with the programmatic-stream-serialization attribute (PDL): its CTAs may be
// scheduled while the previous kernel on the stream drains, run their prologue (barrier init, tensor-map
// prefetch) and then block in griddepcontrol.wait until the previous kernel's memory is visible.
template <typename... KArgs, typename... Args>
cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  ++g_launch_count;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

struct GemmItem {
  AOperand a;
  const void* b;
  long long ldb;
  long long M, N, K;
  GemmEpilogue ep;
  void* const* peer_c = nullptr;   // fused all-gather: the same output slot in every peer's gathered buffer
  int n_peers = 0;
  int tn = 0;                      // 1: C[M,N] = A^T . B with A given as [K, M] (ld = a.ld) and B as [K, N] (ld = ldb), both row-major
                                   // 2: C[M,N] = A . B with A the usual [M, K] and B given as [K, N] row-major (dgrad with the weight as stored)
  // tn == 1 only: B as b_parts tensors side by side along N (b, then b_more; same ldb and segmentation), each [K, N / b_parts], and
  // b_seg_rows != 0: B's K rows in segments of b_seg_rows rows, b_seg_stride elements apart (a [:,1:] view of CLIP hidden states)
  const void* b_more[3] = {nullptr, nullptr, nullptr};
  int b_parts = 1;
  long long b_seg_rows = 0, b_seg_stride = 0;
  // kind 1 (KV-attention, pair kernel only): a / b = y_k (window-major rows) and the gamma-folded W_ik; a2 / b2 = y_v and W_iv;
  // M = rows of y_k, N = K = 1024; attn holds everything else; dep / dep2 / dep3 = the producers of y_k, y_v and q'
  int kind = 0;
  const void* a2 = nullptr;
  const void* b2 = nullptr;
  void* c_pre = nullptr;           // ep.dual: destination of the pre-activation copy [M, N], row stride ld_pre
  long long ld_pre = 0;
  AttnParams attn = {};
  int dep2 = -1, dep3 = -1;
  int k_splits = 1;                // > 1: split-K; ep.c must then be a float buffer [k_splits][M, ldc] (ep.out_f32 = 1, pair kernel only)
  // chains (launch_chain): GEMMs of consecutive stages in ONE persistent launch, ordered by per-row-block tile counters
  int stage = 0;                   // items of equal stage are independent of each other
  int dep = -1;                    // index (in the chain) of the item whose C is this item's A: same M, plain 2-D A
  int* done_counter = nullptr;     // filled by launch_chain
  const int* dep_counter = nullptr;
  int dep_target = 0;
  int dep_shift = 0;
  int dep_span = 0, dep_src_blocks = 0, dep_per = 0;     // producer is a KV-attention item (see GemmProblem)
};
constexpr int kDepFront = -2;      // GemmItem::dep: the A operand is the point-query output of the launch's front work

int gemm_variant(const GemmEpilogue& ep);

int check_item(const GemmItem& it) {
  if (it.kind == 1) return (it.M > 0 && it.M % 16 == 0 && it.attn.qp != nullptr && it.attn.ctx != nullptr) ? TP_OK : TP_ERR_INVALID_ARGUMENT;
  if (it.M <= 0 || it.N <= 0 || it.K <= 0 || it.N % 32 != 0 || it.M > 0x7fffff00ll) return TP_ERR_INVALID_ARGUMENT;   // K: any (TMA zero-fills)
  if ((reinterpret_cast<uintptr_t>(it.ep.c) & 15) != 0 || (it.ep.ldc * 2) % 16 != 0) return TP_ERR_INVALID_ARGUMENT;
  if (it.k_splits < 1 || (it.k_splits > 1 && !it.ep.out_f32) || (it.ep.out_f32 && (it.ep.seg_row_offset != nullptr || it.ep.seg_stride != 0)))
    return TP_ERR_INVALID_ARGUMENT;
  if (it.ep.stats_out != nullptr && (it.N % 256 != 0 || it.ep.stats_out_slots != it.N / 128)) return TP_ERR_INVALID_ARGUMENT;
  if (it.ep.col_a != nullptr && (it.ep.stats_in == nullptr || it.ep.stats_in_slots <= 0)) return TP_ERR_INVALID_ARGUMENT;
  if ((it.b_parts != 1 || it.b_seg_rows != 0) && it.tn != 1) return TP_ERR_INVALID_ARGUMENT;
  // the tower's epilogue instantiations (gemm_variant 1 and 2) have no erf GELU, LayerNorm fold, row statistics, dual, window-major or fp32
  // output, no KV-attention tiles and no TN / NN operand forms; R is read 16 bytes at a time
  if (gemm_variant(it.ep) != 0 && (it.ep.gelu == 1 || it.ep.col_a != nullptr || it.ep.stats_out != nullptr || it.ep.dual || it.ep.wm_s != 0 ||
                                it.k_splits != 1 || it.kind != 0 || it.tn != 0 ||
                                (reinterpret_cast<uintptr_t>(it.ep.resid) & 15) != 0 || it.ep.ldr % 8 != 0))
    return TP_ERR_INVALID_ARGUMENT;
  if (it.ep.resid_f32 && it.ep.resid == nullptr) return TP_ERR_INVALID_ARGUMENT;
  if (it.ep.gelu < 0 || it.ep.gelu > 2) return TP_ERR_INVALID_ARGUMENT;
  return TP_OK;
}

int make_a_map(CUtensorMap* map, const AOperand& a, long long M, long long K) {
  if (a.seg_rows == 0) return make_map_2d(map, a.ptr, M, K, a.ld, kBlockM);
  if (a.seg_rows % 64 != 0 || M % a.seg_rows != 0) return TP_ERR_INVALID_ARGUMENT;
  return make_map_3d(map, a.ptr, M / a.seg_rows, a.seg_rows, K, a.ld, a.seg_stride);
}

// Operand maps of a one-CTA launch with 128 x block_n tiles (encoded before anything of the call is launched).
int make_one_cta_maps(const GemmItem& it, int block_n, CUtensorMap* map_a, CUtensorMap* map_b) {
  TP_TRY(make_a_map(map_a, it.a, it.M, it.K));
  return make_map_2d(map_b, it.b, it.N, it.K, it.ldb, block_n);
}

// The CLIP tower's epilogue features (residual add, quick_gelu) run in instantiations of their own (tp_gemm.cuh: kTower)
bool tower_epilogue(const GemmEpilogue& ep) { return ep.resid != nullptr || ep.gelu == 2; }   // (an fp32 output alone stays on the projector's)

// The instantiation that runs an item: 0 the projector's, 1 the bf16 tower's (inferred from the epilogue features, so that a bf16 tower's
// plain items — patch embedding, qkv — run on the projector's), 2 the f16 tower's (selected by GemmEpilogue::f16 alone: every f16 item,
// plain ones included, runs there)
int gemm_variant(const GemmEpilogue& ep) { return ep.f16 ? 2 : tower_epilogue(ep) ? 1 : 0; }

// One launch runs one instantiation, and a chain's stages hand 16-bit data from one to the next: f16 and bf16 items never share either
bool mixed_precision(const GemmItem* items, int count) {
  for (int i = 1; i < count; ++i)
    if (items[i].ep.f16 != items[0].ep.f16) return true;
  return false;
}

template <int kBlockN, bool kTower, bool kF16 = false>
int launch_gemm_tt(const GemmItem& it, const CUtensorMap& map_a, const CUtensorMap& map_b, int sms, cudaStream_t stream) {
  using Cfg = GemmConfig<kBlockN>;
  {
    static thread_local unsigned attr_done = 0;        // bit per device: the attribute is per (function, device)
    int dev = 0;
    TP_CUDA(cudaGetDevice(&dev));
    if (dev >= 32 || !(attr_done & (1u << dev))) {
      TP_CUDA(cudaFuncSetAttribute(tp_gemm_kernel<kBlockN, kTower, kF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
      if (dev < 32) attr_done |= 1u << dev;
    }
  }
  const long long tiles = ((it.M + kBlockM - 1) / kBlockM) * ((it.N + kBlockN - 1) / kBlockN);
  const int grid = static_cast<int>(tiles < sms ? tiles : sms);
  GemmEpilogue ep = it.ep;
  TP_CUDA(launch_pdl(tp_gemm_kernel<kBlockN, kTower, kF16>, dim3(grid), dim3(kGemmThreads), Cfg::kSmemBytes, stream, map_a, map_b,
                     static_cast<int>(it.M), static_cast<int>(it.N), static_cast<int>(it.K), static_cast<int>(it.a.seg_rows), ep));
  return TP_OK;
}

template <int kBlockN>
int launch_gemm_t(const GemmItem& it, const CUtensorMap& map_a, const CUtensorMap& map_b, int sms, cudaStream_t stream) {
  switch (gemm_variant(it.ep)) {
    case 2: return launch_gemm_tt<kBlockN, true, true>(it, map_a, map_b, sms, stream);
    case 1: return launch_gemm_tt<kBlockN, true>(it, map_a, map_b, sms, stream);
    default: return launch_gemm_tt<kBlockN, false>(it, map_a, map_b, sms, stream);
  }
}

// Everything a launch of the pair kernel needs, as built from a list of items: kept by the forward plan cache below (encoding
// ~100 tensor maps per call costs more host time than the whole 32-crop forward takes on the GPU).
struct BuiltLaunch {
  GemmGroup g;
  PeerStores peers;
  int grid;
};

// Up to kMaxGroup independent problems for ONE launch of the CTA-pair kernel: every check, tensor map and the grid, nothing launched.
int build_pair_group(const GemmItem* items, int count, int sms, const FrontWork* front, BuiltLaunch* out) {
  using Cfg = Gemm2Config;
  GemmGroup& g = out->g;
  memset(&g, 0, sizeof(g));
  g.count = count;
  // one launch runs one instantiation (launch_built): tower epilogues and the projector's features, f16 and bf16 items never share a group
  for (int i = 1; i < count; ++i)
    if (gemm_variant(items[i].ep) != gemm_variant(items[0].ep)) return TP_ERR_INVALID_ARGUMENT;
  if (count > 0 && gemm_variant(items[0].ep) != 0 && front != nullptr) return TP_ERR_INVALID_ARGUMENT;   // no front work there either
  long long total = 0;
  for (int i = 0; i < count; ++i) {
    const GemmItem& it = items[i];
    GemmProblem& p = g.p[i];
    if (it.kind == 1) {
      if (it.N != kC || it.K != kC || it.a2 == nullptr || it.b2 == nullptr || (it.attn.s != 2 && it.attn.s != 4) ||
          it.attn.stats_slots != kAttnSlots)
        return TP_ERR_INVALID_ARGUMENT;
      TP_TRY(make_map_2d(&p.tmap_a, it.a.ptr, it.M, it.K, it.a.ld, kBlockM));
      TP_TRY(make_map_2d(&p.tmap_a2, it.a2, it.M, it.K, it.a.ld, kBlockM));
      TP_TRY(make_map_2d(&p.tmap_b, it.b, it.N, it.K, it.ldb, Cfg::kTileN / 2));   // the head pair's 256 weight rows: 128 per CTA
      TP_TRY(make_map_2d(&p.tmap_b2, it.b2, it.N, it.K, it.ldb, Cfg::kTileN / 2));
      p.kind = 1;
      p.attn = it.attn;
      p.a_parts = 1;
      p.M = static_cast<int>(it.M);
      p.N = static_cast<int>(it.N);
      p.K = static_cast<int>(it.K);
      p.num_n_blocks = 4;                                                      // one tile column per PAIR of heads
      p.num_k_blocks = static_cast<int>(it.K / kBlockK);
      p.tiles_mn = static_cast<int>((it.M + Cfg::kTileM - 1) / Cfg::kTileM) * p.num_n_blocks;
      p.k_splits = 1;
      p.kb_per_split = p.num_k_blocks;
      p.num_tiles = p.tiles_mn;
      p.dep_counter = nullptr;                                                 // its dependencies live in attn.{k,v,q}_counter
      total += p.num_tiles;
      continue;
    }
    if (it.tn == 1 && (it.b_parts > 1 || it.b_seg_rows != 0)) {
      // row-major [K, M] A as below; B split along N into parts of whole 256-column tiles, each a 2-D [K, N / parts] map or a 3-D
      // (cols, row in segment, segment) map with the same 64 x 64 boxes
      if (it.b_parts < 1 || it.b_parts > kMaxAParts || it.N % (it.b_parts * Cfg::kTileN) != 0 || it.a.parts > 1 || it.a.seg_rows != 0 ||
          (it.b_seg_rows != 0 && (it.b_seg_rows % kBlockK != 0 || it.K % it.b_seg_rows != 0)))
        return TP_ERR_INVALID_ARGUMENT;
      TP_TRY(make_map_2d(&p.tmap_a, it.a.ptr, it.K, it.M, it.a.ld, 64));
      const long long np = it.N / it.b_parts;
      for (int q = 0; q < it.b_parts; ++q) {
        const void* ptr = q == 0 ? it.b : it.b_more[q - 1];
        CUtensorMap* map = q == 0 ? &p.tmap_b : &p.tmap_a_more[q - 1];
        if (ptr == nullptr) return TP_ERR_INVALID_ARGUMENT;
        if (it.b_seg_rows == 0) TP_TRY(make_map_2d(map, ptr, it.K, np, it.ldb, 64));
        else TP_TRY(make_map_3d(map, ptr, it.K / it.b_seg_rows, it.b_seg_rows, np, it.ldb, it.b_seg_stride, 64));
      }
      p.b_parts = it.b_parts;
      p.b_nblocks_per_part = static_cast<int>(np / Cfg::kTileN);
      p.b_seg_rows = static_cast<int>(it.b_seg_rows);
      p.ab_mn_major = 1;
    } else if (it.tn == 1) {
      // row-major [K, M] / [K, N] operands: box = 64 MN-elements x 64 K-rows
      TP_TRY(make_map_2d(&p.tmap_a, it.a.ptr, it.K, it.M, it.a.ld, 64));
      TP_TRY(make_map_2d(&p.tmap_b, it.b, it.K, it.N, it.ldb, 64));
      p.ab_mn_major = 1;
    } else if (it.tn == 2) {
      // C = A . B with B row-major [K, N]: the usual A boxes, B as 64 N-elements x 64 K-rows boxes
      if (it.a.parts > 1) return TP_ERR_INVALID_ARGUMENT;
      TP_TRY(make_a_map(&p.tmap_a, it.a, it.M, it.K));
      TP_TRY(make_map_2d(&p.tmap_b, it.b, it.K, it.N, it.ldb, 64));
      p.ab_mn_major = 2;
    } else if (it.a.parts > 1) {
      if (it.a.parts > kMaxAParts || it.K % (it.a.parts * kBlockK) != 0) return TP_ERR_INVALID_ARGUMENT;
      const long long kp = it.K / it.a.parts;
      AOperand part = it.a;
      TP_TRY(make_a_map(&p.tmap_a, part, it.M, kp));
      for (int q = 1; q < it.a.parts; ++q) {
        part.ptr = it.a.more[q - 1];
        if (part.ptr == nullptr) return TP_ERR_INVALID_ARGUMENT;
        TP_TRY(make_a_map(&p.tmap_a_more[q - 1], part, it.M, kp));
      }
      TP_TRY(make_map_2d(&p.tmap_b, it.b, it.N, it.K, it.ldb, Cfg::kTileN / 2));
      p.a_parts = it.a.parts;
      p.a_kblocks_per_part = static_cast<int>(kp / kBlockK);
    } else {
      TP_TRY(make_a_map(&p.tmap_a, it.a, it.M, it.K));
      TP_TRY(make_map_2d(&p.tmap_b, it.b, it.N, it.K, it.ldb, Cfg::kTileN / 2));
    }
    if (p.a_parts == 0) { p.a_parts = 1; p.a_kblocks_per_part = static_cast<int>((it.K + kBlockK - 1) / kBlockK); }
    // C goes out through TMA stores (64-col x 128-row swizzled slabs) unless rows are scattered to ARBITRARY segment offsets;
    // uniformly strided segments (the HD packed layout) stay on the TMA path through a 3-D (cols, row in segment, segment) map
    p.use_tma_store = (it.ep.seg_row_offset == nullptr && !it.ep.out_f32) ? 1 : 0;
    const bool c_segmented = p.use_tma_store && it.ep.seg_stride != 0 && it.ep.seg_stride != it.ep.seg_len;
    if (it.ep.wm_s != 0) {
      if (!p.use_tma_store || c_segmented || it.n_peers > 0) return TP_ERR_INVALID_ARGUMENT;
      p.c_wm_s = it.ep.wm_s;
      TP_TRY(make_map_wm(&p.tmap_c, it.ep.c, it.M, it.N, it.ep.ldc, it.ep.wm_s, 8));
      TP_TRY(make_map_wm(&p.tmap_cx[0], it.ep.c, it.M, it.N, it.ep.ldc, it.ep.wm_s, 16));
      TP_TRY(make_map_wm(&p.tmap_cx[1], it.ep.c, it.M, it.N, it.ep.ldc, it.ep.wm_s, 24));
    } else if (c_segmented) {
      if (it.ep.seg_len <= 0 || it.M % it.ep.seg_len != 0 || it.ep.seg_stride < it.ep.seg_len) return TP_ERR_INVALID_ARGUMENT;
      p.c_seg_len = it.ep.seg_len;
      p.c_unit = seg_store_unit(it.ep.seg_len);
      if (p.c_unit < 4) return TP_ERR_INVALID_ARGUMENT;             // (choose_kernel sends these to the one-CTA kernels' row stores)
      for (int lvl = 0; lvl < kBoxLevels; ++lvl) {
        int rows = p.c_unit << lvl;
        if (rows > kBlockM || rows > it.ep.seg_len) rows = p.c_unit;  // level never used (pieces are at most min(seg_len, 128) rows)
        TP_TRY(make_map_3d(lvl == 0 ? &p.tmap_c : &p.tmap_cx[lvl - 1], it.ep.c, it.M / it.ep.seg_len, it.ep.seg_len, it.N, it.ep.ldc,
                           it.ep.seg_stride * it.ep.ldc, rows));
      }
    } else {
      TP_TRY(make_map_2d(&p.tmap_c, it.ep.c, it.M, it.N, it.ep.ldc, kBlockM));
    }
    if (it.ep.dual) {
      // pre-activation copy: plain TMA-store output only (z and GELU(z) slabs side by side in the half's two staging buffers)
      if (!p.use_tma_store || c_segmented || it.ep.wm_s != 0 || it.n_peers > 0 || !it.ep.gelu || it.c_pre == nullptr || it.k_splits > 1)
        return TP_ERR_INVALID_ARGUMENT;
      TP_TRY(make_map_2d(&p.tmap_cx[0], it.c_pre, it.M, it.N, it.ld_pre, kBlockM));
    }
    p.M = static_cast<int>(it.M);
    p.N = static_cast<int>(it.N);
    p.K = static_cast<int>(it.K);
    p.a_seg_rows = static_cast<int>(it.a.seg_rows);
    p.num_n_blocks = static_cast<int>((it.N + Cfg::kTileN - 1) / Cfg::kTileN);
    p.num_k_blocks = static_cast<int>((it.K + kBlockK - 1) / kBlockK);
    p.tiles_mn = static_cast<int>((it.M + Cfg::kTileM - 1) / Cfg::kTileM) * p.num_n_blocks;
    p.k_splits = it.k_splits;
    p.kb_per_split = (p.num_k_blocks + p.k_splits - 1) / p.k_splits;
    if (static_cast<long long>(p.k_splits - 1) * p.kb_per_split >= p.num_k_blocks) return TP_ERR_INVALID_ARGUMENT;   // no empty split
    p.c_split_stride = it.M * it.ep.ldc;
    p.num_tiles = p.tiles_mn * p.k_splits;
    p.ep = it.ep;
    p.done_counter = it.done_counter;
    p.dep_counter = it.dep_counter;
    p.dep_target = it.dep_target;
    p.dep_shift = it.dep_shift;
    p.dep_span = it.dep_span;
    p.dep_src_blocks = it.dep_src_blocks;
    p.dep_per = it.dep_per;
    if ((p.done_counter != nullptr && !p.use_tma_store) || (p.dep_counter != nullptr && (it.tn || it.a.seg_rows != 0)))
      return TP_ERR_INVALID_ARGUMENT;          // tile counters are published by the store warps / index plain 256-row blocks of A
    p.peer_out = it.n_peers > 0 ? 1 : 0;
    total += p.num_tiles;
  }
  if (total > 0x7fffffffll) return TP_ERR_INVALID_ARGUMENT;
  g.total_tiles = static_cast<int>(total);
  if (front != nullptr) g.front = *front;
  PeerStores& peers = out->peers;
  memset(&peers, 0, sizeof(peers));
  int peer_item = -1;
  // The destination maps of the launch: the peers of a fused all-gather, or — for a segmented (packed-row) output that stays on this
  // GPU — the local buffer as the one "destination" (same store path, including the whole-segment boxes).  Further local segmented
  // outputs whose segments exceed a slab (no whole-segment boxes: the input gradients of the four CLIP layers, 576-row crops) store
  // through their own tmap_c / tmap_cx maps, which cut a slab into the same pieces; a slab of such an output is at most two pieces of
  // at most 7 boxes each (unit >= 4), well inside the store warp's 96 job slots.
  for (int i = 0; i < count; ++i)
    if (items[i].n_peers > 0 || g.p[i].c_seg_len != 0) {
      if (peer_item >= 0 && items[i].n_peers == 0 && items[peer_item].n_peers == 0 && g.p[i].c_seg_len > kBlockM) continue;
      if (peer_item >= 0) return TP_ERR_INVALID_ARGUMENT;      // one set of destination maps per launch
      peer_item = i;
    }
  if (peer_item >= 0) {
    const GemmItem& it0 = items[peer_item];
    const GemmProblem& p0 = g.p[peer_item];
    void* const local_dst[1] = {it0.ep.c};
    void* const* dst = it0.n_peers > 0 ? it0.peer_c : local_dst;
    const int n_dst = it0.n_peers > 0 ? it0.n_peers : 1;
    if (n_dst > kMaxPeers || it0.ep.seg_row_offset != nullptr) return TP_ERR_INVALID_ARGUMENT;
    const bool whole = p0.c_seg_len != 0 && p0.c_seg_len <= kBlockM;
    if (p0.c_seg_len != 0) {
      // worst number of store pieces one 128-row slab is cut into (slab starts fall on multiples of unit inside a segment): the store
      // warp has 96 job slots per slab (pieces x destinations)
      int worst = 0;
      for (int a0 = 0; a0 > -p0.c_seg_len; a0 -= p0.c_unit) {
        int pieces = 0, a = a0;
        while (a < kBlockM) {
          if (whole && a >= 0 && a + p0.c_seg_len <= kBlockM) {
            int k = 1;
            while (k < kWholeLevels && a + (k + 1) * p0.c_seg_len <= kBlockM) ++k;
            ++pieces;
            a += k * p0.c_seg_len;
            continue;
          }
          int len = (a + p0.c_seg_len < kBlockM ? a + p0.c_seg_len : kBlockM) - (a > 0 ? a : 0);
          for (int lvl = kBoxLevels - 1; lvl >= 0; --lvl)
            while (len >= (p0.c_unit << lvl)) { ++pieces; len -= p0.c_unit << lvl; }
          a += p0.c_seg_len;
        }
        if (pieces > worst) worst = pieces;
      }
      if (worst * n_dst > 96) return TP_ERR_INVALID_ARGUMENT;
    }
    for (int p = 0; p < n_dst; ++p) {
      if (p0.c_seg_len != 0) {
        const long long n_segs = it0.M / it0.ep.seg_len;
        for (int lvl = 0; lvl < kBoxLevels; ++lvl) {
          int rows = p0.c_unit << lvl;
          if (rows > kBlockM || rows > it0.ep.seg_len) rows = p0.c_unit;
          TP_TRY(make_map_3d(&peers.m[p][lvl], dst[p], n_segs, it0.ep.seg_len, it0.N, it0.ep.ldc, it0.ep.seg_stride * it0.ep.ldc, rows));
        }
        for (int k = 1; k <= kWholeLevels; ++k) {
          // k whole segments; a level that can never be used (k segments do not fit a slab, or there are fewer segments) repeats k = 1
          const int kk = (whole && k * it0.ep.seg_len <= kBlockM && k <= n_segs) ? k : 1;
          if (whole)
            TP_TRY(make_map_3d(&peers.m[p][kBoxLevels + k - 1], dst[p], n_segs, it0.ep.seg_len, it0.N, it0.ep.ldc,
                               it0.ep.seg_stride * it0.ep.ldc, it0.ep.seg_len, kk));
          else
            peers.m[p][kBoxLevels + k - 1] = peers.m[p][0];
        }
      } else {
        TP_TRY(make_map_2d(&peers.m[p][0], dst[p], it0.M, it0.N, it0.ep.ldc, kBlockM));
      }
    }
    peers.count = n_dst;
    peers.whole = whole ? 1 : 0;
    g.p[peer_item].peer_out = 1;
  }
  const long long max_pairs = sms / 2;
  const int grid = 2 * static_cast<int>(total < max_pairs ? total : max_pairs);
  for (int i = 0; i < count; ++i)
    if (g.p[i].dep_shift == 31) g.p[i].dep_target = grid;        // front work: one arrival per CTA of this launch
  out->grid = grid;
  return TP_OK;
}

template <bool kTower, bool kF16 = false>
int launch_built_t(const BuiltLaunch& b, cudaStream_t stream) {
  using Cfg = Gemm2Config;
  {
    static thread_local unsigned attr_done = 0;
    int dev = 0;
    TP_CUDA(cudaGetDevice(&dev));
    if (dev >= 32 || !(attr_done & (1u << dev))) {
      TP_CUDA(cudaFuncSetAttribute(tp_gemm2_kernel<kTower, kF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
      if (dev < 32) attr_done |= 1u << dev;
    }
  }
  TP_CUDA(launch_pdl(tp_gemm2_kernel<kTower, kF16>, dim3(b.grid), dim3(kGemmThreads), Cfg::kSmemBytes, stream, b.g, b.peers));
  return TP_OK;
}

int launch_built(const BuiltLaunch& b, cudaStream_t stream) {
  int variant = 0;                                     // the same for every problem (build_pair_group)
  for (int i = 0; i < b.g.count; ++i) variant = gemm_variant(b.g.p[i].ep) > variant ? gemm_variant(b.g.p[i].ep) : variant;
  switch (variant) {
    case 2: return launch_built_t<true, true>(b, stream);
    case 1: return launch_built_t<true>(b, stream);
    default: return launch_built_t<false>(b, stream);
  }
}

// Build and launch; built != nullptr: the launch is kept there for replay (the forward plan cache)
int launch_gemm_pair_group(const GemmItem* items, int count, int sms, cudaStream_t stream, const FrontWork* front = nullptr,
                           BuiltLaunch* built = nullptr) {
  BuiltLaunch local;
  BuiltLaunch* b = built != nullptr ? built : &local;
  TP_TRY(build_pair_group(items, count, sms, front, b));
  return launch_built(*b, stream);
}

// Kernel selection: CTA-pair 256x256 tiles whenever the problem fills them (independent problems of one stage share a
// launch), else one-CTA 128 x {256,128} tiles.  TP_GEMM_MODE=1 forces the one-CTA kernels, =2 forces the pair kernel,
// =3 pair kernel without grouping (A/B experiments; read per call, no caching).
// Returns 0 pair, 1 one-CTA 256, 2 one-CTA 128, or -1 (invalid).
int choose_kernel(const GemmItem& it, int count, int sms, int mode) {
  // a uniform-stride segmented output whose crops are not a multiple of 4 rows cannot leave through the pair kernel's boxes
  // (launch_gemm_pair_group rejects it): cost-based, forced and chained selection all fall back to the one-CTA kernels then
  const bool c_segmented = it.ep.seg_row_offset == nullptr && !it.ep.out_f32 && it.ep.seg_stride != 0 && it.ep.seg_stride != it.ep.seg_len;
  const bool pair_ok = (it.N % 256 == 0) && sms >= 2 && !(c_segmented && seg_store_unit(it.ep.seg_len) < 4);
  const bool pair_only = it.n_peers > 0 || it.tn || it.ep.dual || it.a.parts > 1 || it.k_splits > 1 || it.ep.out_f32 || it.kind == 1 || it.ep.wm_s != 0;   // pair-kernel-only features
  if (pair_only && !pair_ok) return -1;
  const bool needs_256 = it.ep.stats_out != nullptr;                        // statistics slots assume 256-column tiles
  // Estimated tensor-pipe cycles of each candidate = waves x k-blocks x cycles per k-block of one CTA.  An H100 SM does 4096 dense
  // bf16 FLOP per cycle (989 TFLOP/s over 132 SMs at 1.83 GHz), so a 128 x 256 x 64 k-block takes 1024 cycles and a 128 x 128 x 64
  // one 512; a pair tile is two CTAs of 128 x 256 side by side.  Large problems always land on the pair kernel; small ones
  // (single crops: the serving latency case) get the tile shape that fills more SMs.  All kernels produce identical bits, so the
  // choice never changes results.
  const long long kb = (it.K + kBlockK - 1) / kBlockK;
  auto waves = [](long long tiles, long long units) { return (tiles + units - 1) / units; };
  const long long t_pair = ((it.M + 255) / 256) * ((it.N + 255) / 256);
  const long long t_256 = ((it.M + 127) / 128) * ((it.N + 255) / 256);
  const long long t_128 = ((it.M + 127) / 128) * ((it.N + 127) / 128);
  // The pair kernel's ring is one stage shallower (3 x 48 KiB next to its output slabs, against 4 in the one-CTA kernels): on an
  // H100 at equal waves it ran 10 - 25 % behind the one-CTA 128 x 256 kernel (bias + GELU GEMMs, M = 576 .. 36864 rows, N = 1024 /
  // 2048, K = 1024 / 4096), so it is charged 1/8 over its nominal MMA time.  The 128-wide kernel reads every A tile once per 128
  // columns instead of per 256: at 36864 x 2048 x 4096 it took 1.21x the 256-wide kernel's time at equal waves, so it is charged 1/5.
  const long long c_pair = pair_ok ? waves(t_pair, sms / 2) * kb * 1024 * 9 / 8 : LLONG_MAX;
  const long long c_256 = (it.N % 256 == 0) ? waves(t_256, sms) * kb * 1024 : LLONG_MAX;
  const long long c_128 = needs_256 ? LLONG_MAX : waves(t_128, sms) * kb * 512 * 6 / 5;
  // a launch costs ~10k cycles of ramp and drain; pair-kernel items of one call share a single (grouped) launch
  const long long launch = 10000;
  const long long l_pair = pair_ok ? c_pair + launch / count : LLONG_MAX;
  const long long l_256 = c_256 == LLONG_MAX ? LLONG_MAX : c_256 + launch;
  const long long l_128 = c_128 == LLONG_MAX ? LLONG_MAX : c_128 + launch;
  int choice;
  if (pair_only || mode == 2 || mode == 3) choice = 0;
  else if (mode == 1) choice = (it.N % 256 == 0) ? 1 : 2;
  else if (l_pair <= l_256 && l_pair <= l_128) choice = 0;                  // ties go to the pair kernel (TMA stores, grouping)
  else choice = (l_256 <= l_128) ? 1 : 2;
  if (choice == 0 && !pair_ok) choice = (it.N % 256 == 0) ? 1 : 2;
  return choice;
}

int gemm_mode() {
  const char* mode_env = getenv("TP_GEMM_MODE");
  return mode_env != nullptr ? atoi(mode_env) : 0;
}

int launch_gemms(const GemmItem* items, int count, int sms, cudaStream_t stream) {
  if (count <= 0 || count > kMaxGroup || mixed_precision(items, count)) return TP_ERR_INVALID_ARGUMENT;
  const int mode = gemm_mode();
  // Every item is checked, placed and encoded before the first launch: an invalid item anywhere in the list launches nothing.
  int choice[kMaxGroup];
  CUtensorMap map_a[kMaxGroup], map_b[kMaxGroup];     // one-CTA items
  GemmItem grouped[kMaxGroup];
  int n_grouped = 0;
  BuiltLaunch pair;
  for (int i = 0; i < count; ++i) {
    TP_TRY(check_item(items[i]));
    const GemmItem& it = items[i];
    if (it.n_peers > 0 && count != 1) return TP_ERR_INVALID_ARGUMENT;
    choice[i] = choose_kernel(it, count, sms, mode);
    if (choice[i] < 0) return TP_ERR_INVALID_ARGUMENT;
    if (choice[i] == 0) {
      if (mode == 3) TP_TRY(build_pair_group(&it, 1, sms, nullptr, &pair));     // validated here, rebuilt at its launch below
      else grouped[n_grouped++] = it;
    } else {
      TP_TRY(make_one_cta_maps(it, choice[i] == 1 ? 256 : 128, &map_a[i], &map_b[i]));
    }
  }
  if (n_grouped > 0) TP_TRY(build_pair_group(grouped, n_grouped, sms, nullptr, &pair));
  for (int i = 0; i < count; ++i) {
    if (choice[i] == 0) {
      if (mode == 3) TP_TRY(launch_gemm_pair_group(&items[i], 1, sms, stream));
    } else if (choice[i] == 1) {
      TP_TRY(launch_gemm_t<256>(items[i], map_a[i], map_b[i], sms, stream));
    } else {
      TP_TRY(launch_gemm_t<128>(items[i], map_a[i], map_b[i], sms, stream));
    }
  }
  if (n_grouped > 0) TP_TRY(launch_built(pair, stream));
  return TP_OK;
}

int launch_front_s(int s, const __nv_bfloat16* x0, long long x0_stride, __nv_bfloat16* q, long long Q, cudaStream_t stream);

// A chain of dependent GEMM stages (items sorted by stage; items[i].dep names the producer of items[i]'s A operand, kDepFront =
// the point queries described by ``front``).  When every item lands on the CTA-pair kernel the whole chain is ONE persistent
// launch: tiles are numbered stage after stage, consumers wait on per-row-block tile counters (``flags``, zeroed earlier on the
// stream) instead of on kernel boundaries — no ramp, drain or partial last wave between the linears — and the point queries are
// computed by the epilogue warps while the first accumulators are still being produced.  Otherwise (small problems on one-CTA
// tiles, TP_CHAIN=0, forced modes) the point queries and the stages run as separate launches exactly as before; either way the
// bits are the same.
bool chain_enabled(int mode) {
  const char* e = getenv("TP_CHAIN");                // A/B aid, read per call: TP_CHAIN=0 -> one launch per stage
  const bool chain_off = e != nullptr && atoi(e) == 0;
  return !chain_off && (mode == 0 || mode == 2);
}

// Can these items run as one chained launch of the pair kernel?  (every item on 256-row pair tiles, nothing scattered to arbitrary
// rows).  by_cost: additionally require that the size-based kernel choice lands on the pair kernel for every item (chains whose
// unchained form computes the same bits); without it the chain is taken whenever the pair kernel CAN run it (the fused-attention
// plan: its results must not depend on the batch size, so neither may the decision).
bool chain_feasible(const GemmItem* items, int count, int sms, bool by_cost = true) {
  const int mode = gemm_mode();
  if (!chain_enabled(mode) || count <= 0 || count > kMaxGroup || sms < 2) return false;
  for (int i = 0; i < count; ++i) {
    if (check_item(items[i]) != TP_OK || items[i].ep.seg_row_offset != nullptr || items[i].N % 256 != 0) return false;
    if (by_cost && choose_kernel(items[i], count, sms, mode) != 0) return false;
  }
  return true;
}

int launch_chain(GemmItem* items, int count, int* flags, long long flag_capacity, const FrontWork* front, int sms, cudaStream_t stream,
                 BuiltLaunch* built = nullptr) {
  if (count <= 0 || count > kMaxGroup || mixed_precision(items, count)) return TP_ERR_INVALID_ARGUMENT;
  for (int i = 0; i < count; ++i) {
    const int deps[3] = {items[i].dep, items[i].dep2, items[i].dep3};
    for (int d : deps) {
      if (d == kDepFront ? front == nullptr : (d >= 0 && (d >= i || items[d].stage >= items[i].stage))) return TP_ERR_INVALID_ARGUMENT;
      // GEMM -> GEMM: the consumer's A row blocks are the producer's C row blocks
      if (d >= 0 && items[i].kind == 0 && items[d].kind == 0 && (items[d].M != items[i].M || items[i].a.seg_rows != 0)) return TP_ERR_INVALID_ARGUMENT;
    }
  }
  bool fused_items = false;
  for (int i = 0; i < count; ++i) fused_items = fused_items || items[i].kind == 1 || items[i].ep.wm_s != 0;
  const bool chain = flags != nullptr && chain_feasible(items, count, sms, !fused_items);
  if (chain) {
    long long used = 0;
    FrontWork fw;
    memset(&fw, 0, sizeof(fw));
    if (front != nullptr) {
      if (used + 1 > flag_capacity) return TP_ERR_WORKSPACE_TOO_SMALL;
      fw = *front;
      fw.done_counter = flags + used;
      used += 1;
    }
    for (int i = 0; i < count; ++i) {
      bool produces = false;
      for (int j = 0; j < count; ++j) produces = produces || items[j].dep == i || items[j].dep2 == i || items[j].dep3 == i;
      if (!produces) continue;
      // a KV-attention item produces ctx: one counter per block of 256 queries; a GEMM: one per block of 256 output rows
      const long long out_rows = items[i].kind == 1 ? items[i].M / (items[i].attn.s * items[i].attn.s) : items[i].M;
      const long long blocks = (out_rows + 255) / 256;
      if (used + blocks > flag_capacity) return TP_ERR_WORKSPACE_TOO_SMALL;
      items[i].done_counter = flags + used;
      if (items[i].kind == 1) {
        items[i].attn.done_counter = items[i].done_counter;
        items[i].done_counter = nullptr;            // published by the epilogue warps, not by the store warps
      }
      used += blocks;
    }
    auto counter_of = [&](int d) { return items[d].kind == 1 ? items[d].attn.done_counter : items[d].done_counter; };
    auto gemm_target = [&](int d) { return 4 * static_cast<int>((items[d].N + 255) / 256); };   // 2 CTAs x 2 column halves per tile
    for (int i = 0; i < count; ++i) {
      GemmItem& it = items[i];
      if (it.kind == 1) {
        if (it.dep < 0 || it.dep2 < 0 || it.dep3 < 0 || items[it.dep].M != it.M || items[it.dep2].M != it.M) return TP_ERR_INVALID_ARGUMENT;
        it.attn.k_counter = counter_of(it.dep);
        it.attn.v_counter = counter_of(it.dep2);
        it.attn.kv_target = gemm_target(it.dep);
        it.attn.q_counter = counter_of(it.dep3);
        it.attn.q_target = gemm_target(it.dep3);
        continue;
      }
      const int d = it.dep;
      if (d == kDepFront) {
        it.dep_counter = fw.done_counter;
        it.dep_shift = 31;                                                 // one launch-wide counter; target = grid size
      } else if (d >= 0 && items[d].kind == 1) {
        it.dep_counter = counter_of(d);
        it.dep_span = items[d].attn.s * items[d].attn.s;                   // KV tiles per block of 256 queries
        it.dep_src_blocks = static_cast<int>((items[d].M + 255) / 256);
        it.dep_per = 8;                                                    // 4 head pairs x 2 CTAs per KV row block
      } else if (d >= 0) {
        it.dep_counter = counter_of(d);
        it.dep_target = gemm_target(d);
      }
    }
    return launch_gemm_pair_group(items, count, sms, stream, front != nullptr ? &fw : nullptr, built);
  }
  for (int i = 0; i < count; ++i)
    if (items[i].kind == 1 || items[i].ep.wm_s != 0) return TP_ERR_INVALID_ARGUMENT;      // fused-attention items exist only inside a chain
  if (front != nullptr) TP_TRY(launch_front_s(front->s, front->x0, front->crop_stride, front->q, front->n_queries, stream));
  for (int first = 0; first < count;) {
    int last = first;
    while (last + 1 < count && items[last + 1].stage == items[first].stage) ++last;
    TP_TRY(launch_gemms(items + first, last - first + 1, sms, stream));
    first = last + 1;
  }
  return TP_OK;
}

int launch_gemm(const AOperand& a, const void* b, long long ldb, long long M, long long N, long long K, const GemmEpilogue& ep,
                int sms, cudaStream_t stream) {
  const GemmItem it{a, b, ldb, M, N, K, ep};
  return launch_gemms(&it, 1, sms, stream);
}

GemmEpilogue plain_epilogue(void* c, long long ldc, const float* bias, int gelu) {
  GemmEpilogue ep;
  memset(&ep, 0, sizeof(ep));
  ep.c = static_cast<__nv_bfloat16*>(c);
  ep.ldc = ldc;
  ep.col_b = bias;
  ep.gelu = gelu;
  ep.alpha = 1.0f;
  ep.ln_inv_dim = 1.0f / kC;
  ep.ln_eps = 1e-6f;     // builder.py:48
  return ep;
}

// ------------------------------------------------------------------------------------------------
// Packed weights layout
// ------------------------------------------------------------------------------------------------
struct PackedLayout {
  size_t w_kv0, b_kv0;                 // [2048,4096] bf16 (k rows then v rows), [2048] f32
  size_t w_k2, b_k2, w_v2, b_v2;       // [1024,1024] bf16, [1024] f32
  size_t w_ik, wsum_k, c_k;            // gamma_k-folded in_proj K weight, its row sums, folded constant
  size_t w_iv, wsum_v, c_v;
  size_t w_q;                          // q_proj_1
  size_t w_iq, wsum_q, c_q;
  size_t w_ot;                         // W_o^T scratch (pack time only)
  size_t w_om, b_om;                   // out_proj folded into mlp.0: W_m0 W_o [H,1024] bf16, W_m0 b_o + b_m0 [H] f32
  size_t w_m2, b_m2;
  size_t w_o, b_o, w_m0, b_m0;         // unfolded copies for the training forward (gradients go to the original parameters)
  size_t total;
};

PackedLayout packed_layout(int H) {
  PackedLayout L;
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return o; };
  const size_t mat = static_cast<size_t>(kC) * kC * 2, vec = static_cast<size_t>(kC) * 4;
  L.w_kv0 = take(2ull * kC * kCm * 2); L.b_kv0 = take(2 * vec);
  L.w_k2 = take(mat); L.b_k2 = take(vec); L.w_v2 = take(mat); L.b_v2 = take(vec);
  L.w_ik = take(mat); L.wsum_k = take(vec); L.c_k = take(vec);
  L.w_iv = take(mat); L.wsum_v = take(vec); L.c_v = take(vec);
  L.w_q = take(mat);
  L.w_iq = take(mat); L.wsum_q = take(vec); L.c_q = take(vec);
  L.w_ot = take(mat);
  L.w_om = take(static_cast<size_t>(H) * kC * 2); L.b_om = take(static_cast<size_t>(H) * 4);
  L.w_m2 = take(static_cast<size_t>(H) * H * 2); L.b_m2 = take(static_cast<size_t>(H) * 4);
  L.w_o = take(mat); L.b_o = take(vec);
  L.w_m0 = take(static_cast<size_t>(H) * kC * 2); L.b_m0 = take(static_cast<size_t>(H) * 4);
  L.total = off;
  return L;
}

// ------------------------------------------------------------------------------------------------
// Workspace layout (per call; all intermediates bf16 unless noted)
// ------------------------------------------------------------------------------------------------
constexpr int kStatSlots = kC / 128;   // one (mean, M2) slot per 128 output columns of a 1024-wide linear

struct WorkLayout {
  size_t h_kv;      // [R,2048]  GELU(W0 xm + b) for k|v
  size_t y_k, y_v;  // [R,1024]  second linear outputs (pre-LayerNorm)
  size_t k_p, v_p;  // [R,1024]  MHA in-projections of the keys / values
  size_t stats;     // f32 [2R + Q, 8, 2]  per-row (mean, M2) of each 128-column block: k rows, v rows, q rows
  size_t q, y_q, q_p, ctx, h_m;      // [Q,1024] x4, [Q,H]
  size_t flags;     // int32 [n_flags]  per-row-block tile counters of the chained GEMM launches (zeroed by the point-query kernel)
  long long n_flags;
  size_t total;
};

WorkLayout work_layout(long long n_crops, int s, int H) {
  const size_t R = static_cast<size_t>(n_crops) * kTokens;
  const int g = kGrid / s;
  const size_t Q = static_cast<size_t>(n_crops) * g * g;
  WorkLayout L;
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 1024); return o; };
  L.h_kv = take(R * 2 * kC * 2);
  L.y_k = take(R * kC * 2);
  L.y_v = take(R * kC * 2);
  L.k_p = take(R * kC * 2);
  L.v_p = take(R * kC * 2);
  L.stats = take((2 * R + Q) * kStatSlots * 2 * 4);
  L.q = take(Q * kC * 2); L.y_q = take(Q * kC * 2); L.q_p = take(Q * kC * 2); L.ctx = take(Q * kC * 2);
  L.h_m = take(Q * static_cast<size_t>(H) * 2);
  L.n_flags = 3 * static_cast<long long>((R + 255) / 256) + 4 * static_cast<long long>((Q + 255) / 256) + 2;
  L.flags = take(static_cast<size_t>(L.n_flags) * 4);
  L.total = off;
  return L;
}

bool valid_hidden(int H) { return H >= 32 && H % 32 == 0 && H <= 65536; }

// Most crops one projector call takes, forward or backward: 576 N token rows stay within the GEMMs' 32-bit row count (0x7fff0000).
// The size queries return 0 past it.
constexpr long long kMaxCrops = 0x7fff0000ll / kTokens;

template <int S>
int launch_front(const __nv_bfloat16* x0, long long x0_stride, __nv_bfloat16* q, long long Q, cudaStream_t stream) {
  const long long threads = Q * 128;
  TP_CUDA(launch_pdl(point_query_kernel<S>, dim3(static_cast<unsigned>((threads + 255) / 256)), dim3(256), 0, stream, x0, x0_stride, q, Q));
  return TP_OK;
}

template <int S>
int launch_attn(const __nv_bfloat16* qp, const __nv_bfloat16* kp, const __nv_bfloat16* vp, __nv_bfloat16* ctx, long long Q,
                cudaStream_t stream) {
  const long long threads = Q * 32;
  TP_CUDA(launch_pdl(window_attn_kernel<S>, dim3(static_cast<unsigned>((threads + 255) / 256)), dim3(256), 0, stream, qp, kp, vp, ctx, Q));
  return TP_OK;
}

// scale_factor dispatch: every divisor of 24 (builder.py:51-52).  2 / 3 / 4 (the released 144 / 64 / 36-token models) keep
// the window in registers; the others stream it.
int launch_front_s(int s, const __nv_bfloat16* x0, long long x0_stride, __nv_bfloat16* q, long long Q, cudaStream_t stream) {
  switch (s) {
    case 1: return launch_front<1>(x0, x0_stride, q, Q, stream);
    case 2: return launch_front<2>(x0, x0_stride, q, Q, stream);
    case 3: return launch_front<3>(x0, x0_stride, q, Q, stream);
    case 4: return launch_front<4>(x0, x0_stride, q, Q, stream);
    case 6: return launch_front<6>(x0, x0_stride, q, Q, stream);
    case 8: return launch_front<8>(x0, x0_stride, q, Q, stream);
    case 12: return launch_front<12>(x0, x0_stride, q, Q, stream);
    case 24: return launch_front<24>(x0, x0_stride, q, Q, stream);
    default: return TP_ERR_BAD_SCALE_FACTOR;
  }
}

int launch_attn_s(int s, const __nv_bfloat16* qp, const __nv_bfloat16* kp, const __nv_bfloat16* vp, __nv_bfloat16* ctx, long long Q,
                  cudaStream_t stream) {
  switch (s) {
    case 2: return launch_attn<2>(qp, kp, vp, ctx, Q, stream);
    case 3: return launch_attn<3>(qp, kp, vp, ctx, Q, stream);
    case 4: return launch_attn<4>(qp, kp, vp, ctx, Q, stream);
    default: {
      const long long threads = Q * 32;
      TP_CUDA(launch_pdl(window_attn_stream_kernel, dim3(static_cast<unsigned>((threads + 255) / 256)), dim3(256), 0, stream, qp, kp, vp, ctx,
                         Q, s));
      return TP_OK;
    }
  }
}

// out[c, r] = in[r, c]  (in: [rows, cols] bf16, row stride ld_in; out: [cols, rows], row stride ld_out)
// Row tiles go on grid.x, column tiles on grid.y (at most 65535: cols <= 2,097,120; a projector's hidden size is at most 65536).
int launch_transpose(const void* in, long long ld_in, void* out, long long ld_out, long long rows, int cols, cudaStream_t stream) {
  if ((rows + 31) / 32 > 0x7fffffffll || (cols + 31) / 32 > 65535) return TP_ERR_INVALID_ARGUMENT;
  const dim3 grid(static_cast<unsigned>((rows + 31) / 32), static_cast<unsigned>((cols + 31) / 32));
  transpose_kernel<<<grid, dim3(32, 8), 0, stream>>>(static_cast<const __nv_bfloat16*>(in), ld_in, static_cast<__nv_bfloat16*>(out), ld_out, rows,
                                                      cols);
  TP_CUDA(cudaGetLastError()); ++g_launch_count;
  return TP_OK;
}

}  // namespace

// ==================================================================================================
// extern "C"
// ==================================================================================================
extern "C" {

const char* tp_strerror(int status) {
  switch (status) {
    case TP_OK: return "ok";
    case TP_ERR_INVALID_ARGUMENT: return "invalid argument";
    case TP_ERR_BAD_SCALE_FACTOR: return "scale_factor must be divisible by grid size";   // builder.py:52 message
    case TP_ERR_WORKSPACE_TOO_SMALL: return "workspace too small";
    case TP_ERR_CUDA: return "CUDA error";
    case TP_ERR_UNSUPPORTED_DEVICE: return "unsupported device: tokenpacker_b200 needs an sm_90a (H100) GPU";
    case TP_ERR_BAD_PATCH_NUM: return "patch_num must be 9, 16 or 25";
    default: return "unknown status";
  }
}

int tp_abi_version(void) { return TP_ABI_VERSION; }

const char* tp_last_cuda_error(void) { return g_last_cuda_error; }

uint64_t tp_launch_count(void) { return g_launch_count.load(std::memory_order_relaxed); }

size_t tp_packed_bytes(int hidden) { return valid_hidden(hidden) ? packed_layout(hidden).total : 0; }

int tp_pack_weights_train(const tp_weights* w, int hidden, void* packed, size_t packed_bytes, void* stream_) {
  if (w == nullptr || packed == nullptr || !valid_hidden(hidden)) return TP_ERR_INVALID_ARGUMENT;
  const void* const* fields = reinterpret_cast<const void* const*>(w);
  for (size_t i = 0; i < sizeof(tp_weights) / sizeof(void*); ++i)
    if (fields[i] == nullptr) return TP_ERR_INVALID_ARGUMENT;
  const PackedLayout L = packed_layout(hidden);
  if (packed_bytes < L.total) return TP_ERR_WORKSPACE_TOO_SMALL;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  uint8_t* P = static_cast<uint8_t*>(packed);
  // k/v_proj.0 side by side: ONE GEMM of N = 2048 reads every row block of the 4096-wide features once
  const size_t kv0 = static_cast<size_t>(kC) * kCm * 2;
  TP_CUDA(cudaMemcpyAsync(P + L.w_kv0, w->k_proj_0_w, kv0, cudaMemcpyDeviceToDevice, stream));
  TP_CUDA(cudaMemcpyAsync(P + L.w_kv0 + kv0, w->v_proj_0_w, kv0, cudaMemcpyDeviceToDevice, stream));
  CastSegs segs;
  auto seg = [&](int i, const void* src, size_t off, int n) {
    segs.s[i] = CastSeg{static_cast<const __nv_bfloat16*>(src), reinterpret_cast<float*>(P + off), n};
  };
  seg(0, w->k_proj_0_b, L.b_kv0, kC);
  seg(1, w->v_proj_0_b, L.b_kv0 + kC * 4, kC);
  seg(2, w->k_proj_2_b, L.b_k2, kC);
  seg(3, w->v_proj_2_b, L.b_v2, kC);
  seg(4, w->out_proj_b, L.b_o, kC);
  seg(5, w->mlp_0_b, L.b_m0, hidden);
  seg(6, w->mlp_2_b, L.b_m2, hidden);
  bf16_to_f32_multi_kernel<<<dim3(4, 7), 256, 0, stream>>>(segs);
  TP_CUDA(cudaGetLastError()); ++g_launch_count;
  const __nv_bfloat16* in_w = static_cast<const __nv_bfloat16*>(w->in_proj_w);
  const __nv_bfloat16* in_b = static_cast<const __nv_bfloat16*>(w->in_proj_b);
  auto fold = [&](size_t w_off, size_t wsum_off, size_t c_off, const void* wsrc, const void* bsrc, const void* gamma, const void* beta) {
    fold_layernorm_kernel<<<(kC * 32 + 255) / 256, 256, 0, stream>>>(
        static_cast<const __nv_bfloat16*>(wsrc), static_cast<const __nv_bfloat16*>(bsrc), static_cast<const __nv_bfloat16*>(gamma),
        static_cast<const __nv_bfloat16*>(beta), reinterpret_cast<__nv_bfloat16*>(P + w_off), reinterpret_cast<float*>(P + wsum_off),
        reinterpret_cast<float*>(P + c_off), kC, kC);
    ++g_launch_count;
    return cudaGetLastError();
  };
  // clip_attn.in_proj_weight rows [0,C) = q, [C,2C) = k, [2C,3C) = v   (torch MHA packed in-projection)
  TP_CUDA(fold(L.w_iq, L.wsum_q, L.c_q, in_w, in_b, w->ln_q_w, w->ln_q_b));
  TP_CUDA(fold(L.w_ik, L.wsum_k, L.c_k, in_w + static_cast<size_t>(kC) * kC, in_b + kC, w->ln_k_w, w->ln_k_b));
  TP_CUDA(fold(L.w_iv, L.wsum_v, L.c_v, in_w + 2 * static_cast<size_t>(kC) * kC, in_b + 2 * kC, w->ln_v_w, w->ln_v_b));
  return TP_OK;
}

// Everything tp_pack_weights_train packs, and what only the inference forward reads: the weights it uses unchanged, and out_proj folded
// into mlp.0 (exact re-association, no nonlinearity in between):
//   mlp.0(out_proj(x)) = (W_m0 W_o) x + (W_m0 b_o + b_m0);  W_m0 W_o computed by our own GEMM with B = W_o^T (K-major)
int tp_pack_weights(const tp_weights* w, int hidden, void* packed, size_t packed_bytes, void* stream_) {
  TP_TRY(tp_pack_weights_train(w, hidden, packed, packed_bytes, stream_));
  const PackedLayout L = packed_layout(hidden);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  uint8_t* P = static_cast<uint8_t*>(packed);
  const size_t mat = static_cast<size_t>(kC) * kC * 2;
  const struct { size_t off; const void* src; size_t bytes; } copies[] = {
      {L.w_k2, w->k_proj_2_w, mat}, {L.w_v2, w->v_proj_2_w, mat}, {L.w_q, w->q_proj_w, mat}, {L.w_o, w->out_proj_w, mat},
      {L.w_m0, w->mlp_0_w, static_cast<size_t>(hidden) * kC * 2}, {L.w_m2, w->mlp_2_w, static_cast<size_t>(hidden) * hidden * 2}};
  for (const auto& c : copies) TP_CUDA(cudaMemcpyAsync(P + c.off, c.src, c.bytes, cudaMemcpyDeviceToDevice, stream));
  DeviceInfo dev;
  TP_TRY(device_info(&dev));
  TP_TRY(launch_transpose(w->out_proj_w, kC, P + L.w_ot, kC, kC, kC, stream));
  TP_TRY(launch_gemm(AOperand{w->mlp_0_w, kC, 0, 0}, P + L.w_ot, kC, hidden, kC, kC, plain_epilogue(P + L.w_om, kC, nullptr, 0), dev.sms, stream));
  matvec_bias_kernel<<<(hidden * 32 + 255) / 256, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(w->mlp_0_w),
                                                                    static_cast<const __nv_bfloat16*>(w->out_proj_b),
                                                                    static_cast<const __nv_bfloat16*>(w->mlp_0_b),
                                                                    reinterpret_cast<float*>(P + L.b_om), hidden, kC);
  TP_CUDA(cudaGetLastError()); ++g_launch_count;
  return TP_OK;
}

size_t tp_workspace_bytes(int64_t n_crops, int scale_factor, int hidden) {
  if (n_crops <= 0 || n_crops > kMaxCrops || scale_factor <= 0 || kGrid % scale_factor != 0 || !valid_hidden(hidden)) return 0;
  return work_layout(n_crops, scale_factor, hidden).total;
}

}  // extern "C"

namespace {
// Plan cache of the single-launch forward: the launch is a pure function of these values (tensor maps depend on addresses and shapes
// only), so a call that repeats them — a serving loop, the chunks of tp_forward_host, the ranks of a sharded HD batch — skips the
// ~100 cuTensorMapEncodeTiled calls and replays the stored launch.  Per host thread, 4 entries, round-robin replacement.  (TP_FUSE_ATTN,
// TP_CHAIN and TP_GEMM_MODE only decide whether this plan runs at all, and are read before the cache is probed.)
struct FwdKey {
  const void* packed; const void* x0; const void* xm[4]; void* out; void* ws; const void* peers[kMaxPeers];
  long long n, s0, sm, crop_rows;
  int s, H, n_peers, sms, parts;
};
struct FwdPlan {
  FwdKey key;
  bool valid = false;
  BuiltLaunch launch;
  size_t flag_bytes;
  int* flags;
};
thread_local FwdPlan g_fwd_plans[4];
thread_local int g_fwd_next = 0;

// Checks of the entry points in include/tokenpacker_b200_layers.h, before any CUDA call: every layer given and 16-byte aligned, crops
// crop_stride elements apart (at least 576 rows of 1024, a 16-byte multiple: TMA strides)
int check_layers(const void* const* layers, int64_t crop_stride) {
  if (layers == nullptr || crop_stride < static_cast<int64_t>(kTokens) * kC || crop_stride % 8 != 0) return TP_ERR_INVALID_ARGUMENT;
  for (int i = 0; i < 4; ++i)
    if (layers[i] == nullptr || (reinterpret_cast<uintptr_t>(layers[i]) & 15) != 0) return TP_ERR_INVALID_ARGUMENT;
  return TP_OK;
}

// What the forward and the backward read from the CLIP tower: feat, and the multi-level stack either as one [n_crops, 576, 4096]
// concatenation (parts = 1) or as its four [n_crops, 576, 1024] layers side by side (parts = 4), crops xm_crop_stride elements apart.
// The k/v_proj.0 GEMMs read the four layers in place as four parts of one operand: each walks the same k-blocks (forward) or output
// tiles (weight gradient) in the same order as the concatenation, so both forms give the same bits.  Only the methods below branch on
// the form.
struct Features {
  const void* x0;
  int64_t x0_crop_stride;
  const void* xm[4];        // the concatenation, or the four layers
  int64_t xm_crop_stride;
  int parts;

  static Features cat(const void* x0, int64_t x0_crop_stride, const void* xm, int64_t xm_crop_stride) {
    return Features{x0, x0_crop_stride, {xm, nullptr, nullptr, nullptr}, xm_crop_stride, 1};
  }
  // the four hidden states of include/tokenpacker_b200_layers.h: the last one is feat as well
  static Features layers(const void* const* l, int64_t crop_stride) {
    return Features{l[3], crop_stride, {l[0], l[1], l[2], l[3]}, crop_stride, 4};
  }
  long long ld() const { return kCm / parts; }
  // both operands given, crops at least 576 rows apart and a 16-byte multiple apart (TMA strides)
  bool valid() const {
    return x0 != nullptr && xm[0] != nullptr && x0_crop_stride >= static_cast<int64_t>(kTokens) * kC && x0_crop_stride % 8 == 0 &&
           xm_crop_stride >= kTokens * ld() && xm_crop_stride % 8 == 0;
  }
  // A of stage [1] (xm [W_k0; W_v0]^T): crop-strided rows are a 3-D [n_crops, 576, K] operand
  AOperand stage1_a() const {
    AOperand a{xm[0], ld(), 0, 0};
    if (xm_crop_stride != kTokens * ld()) a = AOperand{xm[0], ld(), kTokens, xm_crop_stride};
    a.parts = parts;
    for (int i = 1; i < 4; ++i) a.more[i - 1] = xm[i];
    return a;
  }
  // The concatenation is the k/v_proj.0 weight gradients' B operand as one plain [R, 4096] matrix, so its crops must be contiguous;
  // the layers are read crop-strided.
  bool wgrad_b_ok() const { return parts == 4 || xm_crop_stride == static_cast<int64_t>(kTokens) * kCm; }
  // B of those weight gradients: the four layers side by side along N, K rows = tokens in 576-row crops
  void set_wgrad_b(GemmItem* it) const {
    it->b = xm[0];
    it->ldb = ld();
    if (parts == 1) return;
    it->b_parts = parts;
    for (int i = 1; i < 4; ++i) it->b_more[i - 1] = xm[i];
    it->b_seg_rows = kTokens;
    it->b_seg_stride = xm_crop_stride;
  }
};

// The forward's buffers that stages [1] - [3] write and read: the inference workspace, or the activations the training forward saves
struct StageBufs {
  __nv_bfloat16 *h_kv, *q, *y_k, *y_v, *y_q, *k_p, *v_p, *q_p;
  float *stats_k, *stats_v, *stats_q;
};

// it[0] = [1] h_kv = GELU(xm [W_k0; W_v0]^T + b); it[1..3] = [2] y_k | y_v | y_q = the second linears of k / v and q_proj_1, each
// storing its rows' LayerNorm statistics.  Their weights are the live parameters when w != NULL, else the packed copies.
void stage12_items(GemmItem* it, const Features& f, const uint8_t* P, const PackedLayout& L, const tp_weights* w, const StageBufs& b,
                   long long R, long long Q) {
  auto wf = [&](size_t off) { return reinterpret_cast<const float*>(P + off); };
  it[0] = GemmItem{f.stage1_a(), P + L.w_kv0, kCm, R, 2 * kC, kCm, plain_epilogue(b.h_kv, 2 * kC, wf(L.b_kv0), 1)};
  it[1] = GemmItem{AOperand{b.h_kv, 2 * kC, 0, 0}, w != nullptr ? w->k_proj_2_w : P + L.w_k2, kC, R, kC, kC,
                   plain_epilogue(b.y_k, kC, wf(L.b_k2), 0)};
  it[1].ep.stats_out = b.stats_k;
  it[2] = GemmItem{AOperand{b.h_kv + kC, 2 * kC, 0, 0}, w != nullptr ? w->v_proj_2_w : P + L.w_v2, kC, R, kC, kC,
                   plain_epilogue(b.y_v, kC, wf(L.b_v2), 0)};
  it[2].ep.stats_out = b.stats_v;
  it[3] = GemmItem{AOperand{b.q, kC, 0, 0}, w != nullptr ? w->q_proj_w : P + L.w_q, kC, Q, kC, kC, plain_epilogue(b.y_q, kC, nullptr, 0)};
  it[3].ep.stats_out = b.stats_q;
  for (int i = 1; i <= 3; ++i) it[i].ep.stats_out_slots = kStatSlots;
}

// it[0..2] = [3] k' | v' | q' = the LayerNorms folded into the MHA in-projections (q' scaled by 1/sqrt 128)
void stage3_items(GemmItem* it, const uint8_t* P, const PackedLayout& L, const StageBufs& b, long long R, long long Q) {
  auto wf = [&](size_t off) { return reinterpret_cast<const float*>(P + off); };
  it[0] = GemmItem{AOperand{b.y_k, kC, 0, 0}, P + L.w_ik, kC, R, kC, kC, plain_epilogue(b.k_p, kC, wf(L.c_k), 0)};
  it[0].ep.col_a = wf(L.wsum_k);
  it[0].ep.stats_in = b.stats_k;
  it[1] = GemmItem{AOperand{b.y_v, kC, 0, 0}, P + L.w_iv, kC, R, kC, kC, plain_epilogue(b.v_p, kC, wf(L.c_v), 0)};
  it[1].ep.col_a = wf(L.wsum_v);
  it[1].ep.stats_in = b.stats_v;
  it[2] = GemmItem{AOperand{b.y_q, kC, 0, 0}, P + L.w_iq, kC, Q, kC, kC, plain_epilogue(b.q_p, kC, wf(L.c_q), 0)};
  it[2].ep.col_a = wf(L.wsum_q);
  it[2].ep.stats_in = b.stats_q;
  it[2].ep.alpha = 0.08838834764831845f;   // 1/sqrt(head_dim = 128): torch MHA scales q after the in-projection
  for (int i = 0; i < 3; ++i) it[i].ep.stats_in_slots = kStatSlots;
}

int forward_impl(const void* packed, const Features& f, int64_t n_crops, int scale_factor, int hidden, void* out, const int64_t* seg_row_offset,
                 int64_t out_crop_rows, void* const* peer_out, int n_peers, void* workspace, size_t workspace_bytes, void* stream_) {
  if (scale_factor <= 0 || kGrid % scale_factor != 0) return TP_ERR_BAD_SCALE_FACTOR;          // builder.py:51-52
  if (packed == nullptr || !f.valid() || out == nullptr || workspace == nullptr || n_crops <= 0 || !valid_hidden(hidden) ||
      n_crops > kMaxCrops)
    return TP_ERR_INVALID_ARGUMENT;
  DeviceInfo dev;
  TP_TRY(device_info(&dev));
  const int s = scale_factor, H = hidden;
  const int g = kGrid / s, Mq = g * g;
  const long long R = n_crops * kTokens, Q = n_crops * Mq;
  const WorkLayout W = work_layout(n_crops, s, H);
  if (workspace_bytes < W.total) return TP_ERR_WORKSPACE_TOO_SMALL;
  const PackedLayout L = packed_layout(H);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const uint8_t* P = static_cast<const uint8_t*>(packed);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  auto wf = [&](size_t off) { return reinterpret_cast<const float*>(P + off); };
  auto bf = [&](size_t off) { return reinterpret_cast<__nv_bfloat16*>(ws + off); };

  // k' / v' have buffers of their own: in a chained launch [3] runs while other row blocks of [2] still read h_kv, so the
  // round-1 trick of writing them over the dead h_kv buffer is no longer legal
  StageBufs bufs{bf(W.h_kv), bf(W.q), bf(W.y_k), bf(W.y_v), bf(W.y_q), bf(W.k_p), bf(W.v_p), bf(W.q_p)};
  bufs.stats_k = reinterpret_cast<float*>(ws + W.stats);
  bufs.stats_v = bufs.stats_k + 2 * kStatSlots * R;
  bufs.stats_q = bufs.stats_v + 2 * kStatSlots * R;     // every slot is written by the producing GEMM: no memset needed

  // Launch plan.  s = 2 / 4 with hidden % 256 == 0: the fused plan below, one launch at every batch size.  Otherwise chain A =
  // {[S], [1], [2], [3]} and chain B = {[4], [5]} would each run as ONE persistent CTA-pair launch (stages ordered by per-row-block
  // tile counters) if choose_kernel, costing the chain's items as one launch, put every one of them on the pair kernel; on an H100
  // (132 SMs) it never does at the default mode (some item of each chain goes to a one-CTA kernel at every N), so the stages run as
  // separate launches, [A] in between: 7 to 11 launches depending on N (tests/test_projector_batches_gpu.py records the plans and
  // which items block each chain).  TP_GEMM_MODE=2 takes the chains: 3 launches.
  //   [S] point queries            builder.py:117-118   (inside chain A: done by the epilogue warps before their first tile)
  //   [1] h_kv = GELU(xm [W_k0;W_v0]^T + b)                                 :112-113 first linears, xm read once
  //   [2] y_k | y_v | y_q   = second linears k/v + q_proj_1 (+ row statistics for the LayerNorms)   :112-113, :120
  //   [3] k'  | v'  | q'    = LayerNorm folded into the MHA in-projections (q' scaled by 1/sqrt 128)   MHA in_proj
  //   [A] window attention core                                              :122-130
  //   [4] h_m = GELU(ctx (W_m0 W_o)^T + (W_m0 b_o + b_m0))                   out_proj folded into mlp.0  (:130,:136)
  //   [5] out = h_m W_m2^T + b_m2  -> final [N,M,H] (or packed HD) layout    :136
  int* flags = reinterpret_cast<int*>(ws + W.flags);
  const long long flags_a = 3 * ((R + 255) / 256);          // chain A: [1], [2]k, [2]v produce for later stages ([2]q: Q rows, below)
  TP_CUDA(cudaMemsetAsync(flags, 0, static_cast<size_t>(W.n_flags) * 4, stream));      // tile counters of the chained launches
  FrontWork front;
  memset(&front, 0, sizeof(front));
  front.x0 = static_cast<const __nv_bfloat16*>(f.x0);
  front.q = bufs.q;
  front.crop_stride = f.x0_crop_stride;
  front.n_queries = Q;
  front.s = s;
  // ---- fully fused plan (scale factors 2 and 4, batches large enough for pair tiles): ONE launch for the whole forward.
  //   [2] stores y_k / y_v WINDOW-MAJOR (the s x s keys of a window become consecutive rows: divide_feature done by the TMA store),
  //   and the K / V in-projections run as KV-attention tiles whose epilogue is the window attention itself: k', v' never reach memory.
  //   Stages: [1] | [2]k [2]v [2]q | [3]q | KV-attention | [4] | [5], ordered by tile counters; point queries as front work.
  const char* fuse_env = getenv("TP_FUSE_ATTN");       // A/B aid, read per call: TP_FUSE_ATTN=0 -> separate attention kernel
  const bool fuse_off = fuse_env != nullptr && atoi(fuse_env) == 0;
  if ((s == 2 || s == 4) && !fuse_off && seg_row_offset == nullptr) {
    GemmItem g[8], in_proj[3];
    stage12_items(g, f, P, L, nullptr, bufs, R, Q);
    for (int i = 1; i <= 3; ++i) g[i].stage = 1;
    g[1].ep.wm_s = g[2].ep.wm_s = s;
    g[1].dep = g[2].dep = 0;
    g[3].dep = kDepFront;
    stage3_items(in_proj, P, L, bufs, R, Q);
    g[4] = in_proj[2];
    g[4].stage = 2;
    g[4].dep = 3;
    g[5] = GemmItem{AOperand{bf(W.y_k), kC, 0, 0}, P + L.w_ik, kC, R, kC, kC, plain_epilogue(nullptr, kC, nullptr, 0)};
    g[5].kind = 1;
    g[5].a2 = bf(W.y_v);
    g[5].b2 = P + L.w_iv;
    g[5].attn.qp = bf(W.q_p);
    g[5].attn.ctx = bf(W.ctx);
    g[5].attn.stats_k = bufs.stats_k;
    g[5].attn.stats_v = bufs.stats_v;
    g[5].attn.wsum_k = wf(L.wsum_k);
    g[5].attn.cst_k = wf(L.c_k);
    g[5].attn.wsum_v = wf(L.wsum_v);
    g[5].attn.cst_v = wf(L.c_v);
    g[5].attn.s = s;
    g[5].attn.stats_slots = kStatSlots;
    g[5].attn.ln_inv_dim = 1.0f / kC;
    g[5].attn.ln_eps = 1e-6f;
    g[5].stage = 3;
    g[5].dep = 1;
    g[5].dep2 = 2;
    g[5].dep3 = 4;
    g[6] = GemmItem{AOperand{bf(W.ctx), kC, 0, 0}, P + L.w_om, kC, Q, H, kC, plain_epilogue(bf(W.h_m), H, wf(L.b_om), 1)};
    g[6].stage = 4;
    g[6].dep = 5;
    GemmEpilogue ep = plain_epilogue(out, H, wf(L.b_m2), 0);
    if (out_crop_rows != 0 && out_crop_rows != Mq) {
      if (out_crop_rows < Mq || out_crop_rows > 0x7fffffffll / H) return TP_ERR_INVALID_ARGUMENT;
      ep.seg_len = Mq;
      ep.seg_stride = static_cast<int>(out_crop_rows);
    }
    g[7] = GemmItem{AOperand{bf(W.h_m), H, 0, 0}, P + L.w_m2, H, Q, H, H, ep};
    g[7].peer_c = peer_out;
    g[7].n_peers = n_peers;
    g[7].stage = 5;
    g[7].dep = 6;
    FwdKey key;
    memset(&key, 0, sizeof(key));
    key.packed = packed; key.x0 = f.x0; key.out = out; key.ws = workspace;
    for (int i = 0; i < 4; ++i) key.xm[i] = f.xm[i];
    for (int i = 0; i < n_peers && i < kMaxPeers; ++i) key.peers[i] = peer_out[i];
    key.n = n_crops; key.s0 = f.x0_crop_stride; key.sm = f.xm_crop_stride; key.crop_rows = out_crop_rows;
    key.s = s; key.H = H; key.n_peers = n_peers; key.sms = dev.sms; key.parts = f.parts;
    if (chain_feasible(g, 8, dev.sms, false)) {
      for (FwdPlan& fp : g_fwd_plans)
        if (fp.valid && memcmp(&fp.key, &key, sizeof(key)) == 0) {
          // (the counters were already reset by the memset above)
          TP_CUDA(launch_pdl(tp_gemm2_kernel<false>, dim3(fp.launch.grid), dim3(kGemmThreads), Gemm2Config::kSmemBytes, stream, fp.launch.g, fp.launch.peers));
          return TP_OK;
        }
      FwdPlan& slot = g_fwd_plans[g_fwd_next];
      g_fwd_next = (g_fwd_next + 1) % 4;
      slot.valid = false;
      TP_TRY(launch_chain(g, 8, flags, W.n_flags, &front, dev.sms, stream, &slot.launch));
      slot.key = key;
      slot.valid = true;
      return TP_OK;
    }
  }
  {
    GemmItem g[7];
    stage12_items(g, f, P, L, nullptr, bufs, R, Q);
    stage3_items(g + 4, P, L, bufs, R, Q);
    g[1].stage = g[2].stage = g[3].stage = 1;
    g[1].dep = g[2].dep = 0;
    g[3].dep = kDepFront;
    g[4].stage = g[5].stage = g[6].stage = 2;
    g[4].dep = 1;
    g[5].dep = 2;
    g[6].dep = 3;
    TP_TRY(launch_chain(g, 7, flags, flags_a + (Q + 255) / 256 + 1, &front, dev.sms, stream));
  }
  TP_TRY(launch_attn_s(s, bufs.q_p, bufs.k_p, bufs.v_p, bf(W.ctx), Q, stream));
  {
    GemmItem g[2];
    g[0] = GemmItem{AOperand{bf(W.ctx), kC, 0, 0}, P + L.w_om, kC, Q, H, kC, plain_epilogue(bf(W.h_m), H, wf(L.b_om), 1)};
    g[0].stage = 0;
    GemmEpilogue ep = plain_epilogue(out, H, wf(L.b_m2), 0);
    if (seg_row_offset != nullptr) {
      ep.seg_row_offset = reinterpret_cast<const long long*>(seg_row_offset);
      ep.seg_len = Mq;
    } else if (out_crop_rows != 0 && out_crop_rows != Mq) {
      if (out_crop_rows < Mq || out_crop_rows > 0x7fffffffll / H) return TP_ERR_INVALID_ARGUMENT;
      ep.seg_len = Mq;
      ep.seg_stride = static_cast<int>(out_crop_rows);
    }
    g[1] = GemmItem{AOperand{bf(W.h_m), H, 0, 0}, P + L.w_m2, H, Q, H, H, ep};
    g[1].peer_c = peer_out;
    g[1].n_peers = n_peers;
    g[1].stage = 1;
    g[1].dep = 0;
    int* flags_b = flags + flags_a + (Q + 255) / 256 + 1;
    TP_TRY(launch_chain(g, 2, flags_b, (Q + 255) / 256, nullptr, dev.sms, stream));
  }
  return TP_OK;
}
}  // namespace

extern "C" {

int tp_forward(const void* packed, const void* x0, const void* xm, int64_t n_crops, int64_t x0_crop_stride, int64_t xm_crop_stride,
               int scale_factor, int hidden, void* out, const int64_t* seg_row_offset, void* workspace, size_t workspace_bytes,
               void* stream) {
  return forward_impl(packed, Features::cat(x0, x0_crop_stride, xm, xm_crop_stride), n_crops, scale_factor, hidden, out, seg_row_offset, 0,
                      nullptr, 0, workspace, workspace_bytes, stream);
}

int tp_forward_packed(const void* packed, const void* x0, const void* xm, int64_t n_crops, int64_t x0_crop_stride, int64_t xm_crop_stride,
                      int scale_factor, int hidden, void* out, int64_t out_crop_rows, void* workspace, size_t workspace_bytes, void* stream) {
  return forward_impl(packed, Features::cat(x0, x0_crop_stride, xm, xm_crop_stride), n_crops, scale_factor, hidden, out, nullptr, out_crop_rows,
                      nullptr, 0, workspace, workspace_bytes, stream);
}

int tp_forward_layers(const void* packed, const void* const* layers, int64_t n_crops, int64_t crop_stride, int scale_factor, int hidden,
                      void* out, const int64_t* seg_row_offset, void* workspace, size_t workspace_bytes, void* stream) {
  // (a missing layer is reported before a bad scale factor)
  if (layers == nullptr || layers[0] == nullptr || layers[1] == nullptr || layers[2] == nullptr || layers[3] == nullptr)
    return TP_ERR_INVALID_ARGUMENT;
  if (scale_factor <= 0 || kGrid % scale_factor != 0) return TP_ERR_BAD_SCALE_FACTOR;
  TP_TRY(check_layers(layers, crop_stride));
  return forward_impl(packed, Features::layers(layers, crop_stride), n_crops, scale_factor, hidden, out, seg_row_offset, 0, nullptr, 0,
                      workspace, workspace_bytes, stream);
}

int tp_forward_layers_packed(const void* packed, const void* const* layers, int64_t n_crops, int64_t crop_stride, int scale_factor,
                             int hidden, void* out, int64_t out_crop_rows, void* workspace, size_t workspace_bytes, void* stream) {
  if (scale_factor <= 0 || kGrid % scale_factor != 0) return TP_ERR_BAD_SCALE_FACTOR;
  TP_TRY(check_layers(layers, crop_stride));
  const int64_t mq = static_cast<int64_t>(kGrid / scale_factor) * (kGrid / scale_factor);
  if ((reinterpret_cast<uintptr_t>(out) & 15) != 0 || !valid_hidden(hidden) ||
      (out_crop_rows != 0 && (out_crop_rows < mq || out_crop_rows > 0x7fffffffll / hidden)))
    return TP_ERR_INVALID_ARGUMENT;
  return forward_impl(packed, Features::layers(layers, crop_stride), n_crops, scale_factor, hidden, out, nullptr, out_crop_rows, nullptr, 0,
                      workspace, workspace_bytes, stream);
}

int tp_forward_allgather(const void* packed, const void* x0, const void* xm, int64_t n_crops, int64_t x0_crop_stride,
                         int64_t xm_crop_stride, int scale_factor, int hidden, void* const* peer_out, int n_peers, int64_t crop_offset,
                         int64_t out_crop_rows, void* workspace, size_t workspace_bytes, void* stream) {
  if (peer_out == nullptr || n_peers <= 0 || n_peers > kMaxPeers || crop_offset < 0 || hidden % 256 != 0) return TP_ERR_INVALID_ARGUMENT;
  if (scale_factor <= 0 || kGrid % scale_factor != 0) return TP_ERR_BAD_SCALE_FACTOR;
  const int g = kGrid / scale_factor;
  if (out_crop_rows != 0 && out_crop_rows < g * g) return TP_ERR_INVALID_ARGUMENT;
  // packed rows reach the peers only through the pair kernel's segmented stores: rejected here, before anything is launched, for the
  // scale factors those stores cannot serve (8 and 24)
  if (out_crop_rows != 0 && out_crop_rows != g * g && seg_store_unit(g * g) < 4) return TP_ERR_INVALID_ARGUMENT;
  const size_t crop_rows = out_crop_rows != 0 ? static_cast<size_t>(out_crop_rows) : static_cast<size_t>(g) * g;
  const size_t slot = static_cast<size_t>(crop_offset) * crop_rows * hidden * 2;   // this rank's first row in every peer's output buffer
  void* dst[kMaxPeers];
  for (int p = 0; p < n_peers; ++p) {
    if (peer_out[p] == nullptr) return TP_ERR_INVALID_ARGUMENT;
    dst[p] = static_cast<uint8_t*>(peer_out[p]) + slot;
  }
  return forward_impl(packed, Features::cat(x0, x0_crop_stride, xm, xm_crop_stride), n_crops, scale_factor, hidden, dst[0], nullptr,
                      out_crop_rows, dst, n_peers, workspace, workspace_bytes, stream);
}

namespace {
// Copy streams and events of the host-buffer path: created once per (host thread, device) and kept for the life of the thread —
// creating and destroying two streams and 2 events per chunk on every call cost more host time than the launches themselves.
// (The only state the library keeps; it holds no memory and never outlives its thread's CUDA context use.)
constexpr int kHostEvents = 64;      // ring of (copy-in done, compute done) event pairs; a 64-crop call uses ~12
struct HostPipe {
  int device = -1;
  cudaStream_t s_in = nullptr, s_out = nullptr;
  cudaEvent_t ev_start = nullptr, ev_in[kHostEvents] = {}, ev_done[kHostEvents] = {};
};
thread_local HostPipe g_host_pipe[16];

int host_pipe(HostPipe** out) {
  int dev = 0;
  TP_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 16) return TP_ERR_INVALID_ARGUMENT;
  HostPipe& hp = g_host_pipe[dev];
  if (hp.device != dev) {
    TP_CUDA(cudaStreamCreateWithFlags(&hp.s_in, cudaStreamNonBlocking));
    TP_CUDA(cudaStreamCreateWithFlags(&hp.s_out, cudaStreamNonBlocking));
    TP_CUDA(cudaEventCreateWithFlags(&hp.ev_start, cudaEventDisableTiming));
    for (int i = 0; i < kHostEvents; ++i) {
      TP_CUDA(cudaEventCreateWithFlags(&hp.ev_in[i], cudaEventDisableTiming));
      TP_CUDA(cudaEventCreateWithFlags(&hp.ev_done[i], cudaEventDisableTiming));
    }
    hp.device = dev;
  }
  *out = &hp;
  return TP_OK;
}
}  // namespace

int tp_forward_host(const void* packed, const void* x0_host, const void* xm_host, int64_t n_crops, int scale_factor, int hidden,
                    void* out_host, void* d_x0, void* d_xm, void* d_out, void* workspace, size_t workspace_bytes, int64_t chunk_crops,
                    void* stream_) {
  if (x0_host == nullptr || xm_host == nullptr || out_host == nullptr || d_x0 == nullptr || d_xm == nullptr || d_out == nullptr ||
      n_crops <= 0)
    return TP_ERR_INVALID_ARGUMENT;
  if (scale_factor <= 0 || kGrid % scale_factor != 0) return TP_ERR_BAD_SCALE_FACTOR;
  if (chunk_crops <= 0 || chunk_crops > n_crops) chunk_crops = n_crops;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int g = kGrid / scale_factor;
  const size_t x0_b = static_cast<size_t>(kTokens) * kC * 2, xm_b = static_cast<size_t>(kTokens) * kCm * 2;
  const size_t out_b = static_cast<size_t>(g) * g * hidden * 2;
  HostPipe* hp = nullptr;
  TP_TRY(host_pipe(&hp));
  int status = TP_OK;
  cudaError_t err = cudaSuccess;
  const char* where = "";
  // every CUDA call of the pipeline is checked; the first failure stops issuing and is reported after the common drain below
#define TP_HOST_STEP(call)                                   \
  do {                                                       \
    if (err == cudaSuccess && status == TP_OK) {             \
      err = (call);                                          \
      if (err != cudaSuccess) where = #call;                 \
    }                                                        \
  } while (0)
  TP_HOST_STEP(cudaEventRecord(hp->ev_start, stream));          // copies must not start before prior work on the caller's stream
  TP_HOST_STEP(cudaStreamWaitEvent(hp->s_in, hp->ev_start, 0));
  TP_HOST_STEP(cudaStreamWaitEvent(hp->s_out, hp->ev_start, 0));
  // Full chunks, then a tapered tail (remaining/2, ..., 2, 1, 1): the copies in are the bottleneck (PCIe), so what is NOT hidden
  // behind them is the last chunk's compute + copy out — keep that chunk small.
  int slot = 0;
  for (int64_t c0 = 0, nc = 0; c0 < n_crops && status == TP_OK && err == cudaSuccess; c0 += nc, ++slot) {
    const int64_t remaining = n_crops - c0;
    nc = remaining > chunk_crops ? chunk_crops : (remaining > 1 ? (remaining + 1) / 2 : 1);
    if (slot == kHostEvents) {          // ring exhausted (very long calls): drain before reusing the events
      TP_HOST_STEP(cudaStreamSynchronize(hp->s_out));
      slot = 0;
    }
    TP_HOST_STEP(cudaMemcpyAsync(static_cast<uint8_t*>(d_x0) + c0 * x0_b, static_cast<const uint8_t*>(x0_host) + c0 * x0_b, nc * x0_b,
                                 cudaMemcpyHostToDevice, hp->s_in));
    TP_HOST_STEP(cudaMemcpyAsync(static_cast<uint8_t*>(d_xm) + c0 * xm_b, static_cast<const uint8_t*>(xm_host) + c0 * xm_b, nc * xm_b,
                                 cudaMemcpyHostToDevice, hp->s_in));
    TP_HOST_STEP(cudaEventRecord(hp->ev_in[slot], hp->s_in));
    TP_HOST_STEP(cudaStreamWaitEvent(stream, hp->ev_in[slot], 0));
    if (err == cudaSuccess)
      status = tp_forward(packed, static_cast<uint8_t*>(d_x0) + c0 * x0_b, static_cast<uint8_t*>(d_xm) + c0 * xm_b, nc,
                          static_cast<int64_t>(kTokens) * kC, static_cast<int64_t>(kTokens) * kCm, scale_factor, hidden,
                          static_cast<uint8_t*>(d_out) + c0 * out_b, nullptr, workspace, workspace_bytes, stream);
    TP_HOST_STEP(cudaEventRecord(hp->ev_done[slot], stream));
    TP_HOST_STEP(cudaStreamWaitEvent(hp->s_out, hp->ev_done[slot], 0));
    TP_HOST_STEP(cudaMemcpyAsync(static_cast<uint8_t*>(out_host) + c0 * out_b, static_cast<uint8_t*>(d_out) + c0 * out_b, nc * out_b,
                                 cudaMemcpyDeviceToHost, hp->s_out));
  }
#undef TP_HOST_STEP
  // common drain: whatever was issued completes before the caller's buffers may be touched again
  const cudaError_t e1 = cudaStreamSynchronize(hp->s_out);
  const cudaError_t e2 = cudaStreamSynchronize(stream);
  const cudaError_t e3 = cudaStreamSynchronize(hp->s_in);
  if (status != TP_OK) return status;
  if (err != cudaSuccess) {
    snprintf(g_last_cuda_error, sizeof(g_last_cuda_error), "%s: %s", where, cudaGetErrorString(err));
    return TP_ERR_CUDA;
  }
  TP_CUDA(e1);
  TP_CUDA(e2);
  TP_CUDA(e3);
  return TP_OK;
}

int tp_gemm_tn_bf16(const void* a, int64_t lda, const void* b, int64_t ldb, void* c, int64_t ldc, int64_t m, int64_t n, int64_t k,
                    float alpha, void* stream) {
  if (a == nullptr || b == nullptr || c == nullptr) return TP_ERR_INVALID_ARGUMENT;
  DeviceInfo dev;
  TP_TRY(device_info(&dev));
  GemmItem it{AOperand{a, lda, 0, 0}, b, ldb, m, n, k, plain_epilogue(c, ldc, nullptr, 0)};
  it.ep.alpha = alpha;
  it.tn = 1;
  return launch_gemms(&it, 1, dev.sms, static_cast<cudaStream_t>(stream));
}

int tp_gemm_nn_bf16(const void* a, int64_t lda, const void* b, int64_t ldb, void* c, int64_t ldc, int64_t m, int64_t n, int64_t k,
                    float alpha, void* stream) {
  if (a == nullptr || b == nullptr || c == nullptr) return TP_ERR_INVALID_ARGUMENT;
  DeviceInfo dev;
  TP_TRY(device_info(&dev));
  GemmItem it{AOperand{a, lda, 0, 0}, b, ldb, m, n, k, plain_epilogue(c, ldc, nullptr, 0)};
  it.ep.alpha = alpha;
  it.tn = 2;
  return launch_gemms(&it, 1, dev.sms, static_cast<cudaStream_t>(stream));
}

int tp_gemm_bf16(const void* a, int64_t lda, const void* b, int64_t ldb, void* c, int64_t ldc, int64_t m, int64_t n, int64_t k,
                 const float* bias, int gelu, float alpha, void* stream) {
  if (a == nullptr || b == nullptr || c == nullptr) return TP_ERR_INVALID_ARGUMENT;
  DeviceInfo dev;
  TP_TRY(device_info(&dev));
  GemmEpilogue ep = plain_epilogue(c, ldc, bias, gelu != 0 ? 1 : 0);     // any nonzero flag is the erf GELU, as documented
  ep.alpha = alpha;
  return launch_gemm(AOperand{a, lda, 0, 0}, b, ldb, m, n, k, ep, dev.sms, static_cast<cudaStream_t>(stream));
}

#include "tp_train.inl"

// ------------------------------------------------------------------------------------------------
// HD front end
// ------------------------------------------------------------------------------------------------
namespace {
struct GridPair { int h, w; };
// Candidate tables: data of patch_divide.py:4-54 (argmax takes the FIRST maximum, so order is part of the contract;
// the 25-table really lists (4,6),(6,4) twice).
const GridPair kGrid9[] = {{1,1},{1,2},{2,1},{1,3},{3,1},{2,2},{1,4},{4,1},{1,5},{5,1},{1,6},{6,1},{2,3},{3,2},{1,7},{7,1},
                           {4,2},{2,4},{1,8},{8,1},{3,3},{1,9},{9,1}};
const GridPair kGrid16x[] = {{2,5},{5,2},{2,6},{6,2},{3,4},{4,3},{2,7},{7,2},{3,5},{5,3},{2,8},{8,2},{4,4}};
const GridPair kGrid25x[] = {{3,6},{6,3},{2,9},{9,2},{4,5},{5,4},{2,10},{10,2},{3,7},{7,3},{11,2},{2,11},{4,6},{6,4},{12,2},{2,12},
                             {3,8},{8,3},{4,6},{6,4},{5,5}};

int grid_table(int patch_num, GridPair* out) {
  int n = 0;
  for (const GridPair& p : kGrid9) out[n++] = p;
  if (patch_num == 9) return n;
  for (const GridPair& p : kGrid16x) out[n++] = p;
  if (patch_num == 16) return n;
  for (const GridPair& p : kGrid25x) out[n++] = p;
  return n;
}

// Python round(): round-half-to-even on doubles.
long long py_round(double v) { return static_cast<long long>(nearbyint(v)); }
}  // namespace

int tp_hd_grid(int64_t h, int64_t w, int patch_num, int image_size, int* h_block, int* w_block) {
  if (h_block == nullptr || w_block == nullptr || h <= 0 || w <= 0 || image_size <= 0) return TP_ERR_INVALID_ARGUMENT;
  if (patch_num != 9 && patch_num != 16 && patch_num != 25) return TP_ERR_BAD_PATCH_NUM;
  GridPair table[64];
  const int n = grid_table(patch_num, table);
  // float32 arithmetic op-for-op like the torch expression (patch_divide.py:96-105, box_iou :57-69); volatile keeps
  // every intermediate rounded to float (no fused multiply-add, no excess precision).
  const float fh = static_cast<float>(h), fw = static_cast<float>(w);
  volatile float bh = fh * 1.4f, bw = fw * 1.4f;
  volatile float area2 = bh * bw;
  int best = 0;
  float best_score = 0.f;
  for (int i = 0; i < n; ++i) {
    const long long ph = static_cast<long long>(table[i].h) * image_size, pw = static_cast<long long>(table[i].w) * image_size;
    const float fph = static_cast<float>(ph), fpw = static_cast<float>(pw);
    const float farea1 = static_cast<float>(ph * pw);
    volatile float r0 = fph / fh, r1 = fpw / fw;
    const float ratio = r0 < r1 ? r0 : r1;
    volatile float hr = fh * ratio, wr = fw * ratio;
    volatile float prod = nearbyintf(hr) * nearbyintf(wr);
    volatile float score = prod / farea1;
    const float wh0 = fph < bh ? fph : bh, wh1 = fpw < bw ? fpw : bw;
    volatile float inter = wh0 * wh1;
    volatile float uni = farea1 + area2;
    uni = uni - inter;
    volatile float den = uni + 1e-5f;
    volatile float iou = inter / den;
    volatile float iou01 = iou * 0.1f;
    const float total = score + iou01;
    if (i == 0 || total > best_score) { best_score = total; best = i; }
  }
  *h_block = table[best].h;
  *w_block = table[best].w;
  return TP_OK;
}

int tp_hd_fit(int64_t h, int64_t w, int h_block, int w_block, int* h_resized, int* w_resized, int* h_thumb, int* w_thumb) {
  if (h <= 0 || w <= 0 || h_block <= 0 || w_block <= 0) return TP_ERR_INVALID_ARGUMENT;
  auto fit = [&](int hb, int wb, int* oh, int* ow) {
    // train.py:701-708 — Python float (double) ratios, round() half-to-even, min clamp
    const double h_ratio = static_cast<double>(kBlockPx * hb) / static_cast<double>(h);
    const double w_ratio = static_cast<double>(kBlockPx * wb) / static_cast<double>(w);
    if (h_ratio <= w_ratio) {
      *oh = kBlockPx * hb;
      const long long r = py_round(static_cast<double>(w) * h_ratio);
      *ow = static_cast<int>(r < kBlockPx * wb ? r : kBlockPx * wb);
    } else {
      *ow = kBlockPx * wb;
      const long long r = py_round(static_cast<double>(h) * w_ratio);
      *oh = static_cast<int>(r < kBlockPx * hb ? r : kBlockPx * hb);
    }
  };
  int a, b;
  fit(h_block, w_block, &a, &b);
  if (h_resized) *h_resized = a;
  if (w_resized) *w_resized = b;
  fit(1, 1, &a, &b);
  if (h_thumb) *h_thumb = a;
  if (w_thumb) *w_thumb = b;
  return TP_OK;
}

int tp_hd_tile(const float* image, int64_t h, int64_t w, int h_block, int w_block, float* crops, void* stream_) {
  if (image == nullptr || crops == nullptr || h <= 0 || w <= 0 || h_block <= 0 || w_block <= 0 || h > 32768 || w > 32768)
    return TP_ERR_INVALID_ARGUMENT;
  int h_r, w_r, h_t, w_t;
  TP_TRY(tp_hd_fit(h, w, h_block, w_block, &h_r, &w_r, &h_t, &w_t));
  if (h_r <= 0 || w_r <= 0) return TP_ERR_INVALID_ARGUMENT;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const long long total = 3ll * h_block * kBlockPx * w_block * kBlockPx;
  hd_tile_main_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(image, static_cast<int>(h), static_cast<int>(w),
                                                                                      h_block, w_block, h_r, w_r, crops);
  TP_CUDA(cudaGetLastError()); ++g_launch_count;
  if (h_block * w_block > 1) {
    if (h_t <= 0 || w_t <= 0) return TP_ERR_INVALID_ARGUMENT;
    const int t = 3 * kBlockPx * kBlockPx;
    hd_tile_thumb_kernel<<<(t + 255) / 256, 256, 0, stream>>>(h_block, w_block, h_t, w_t, crops);
    TP_CUDA(cudaGetLastError()); ++g_launch_count;
  }
  return TP_OK;
}

int tp_hd_tile_batch_plan(const int64_t* h, const int64_t* w, const void* const* images, int64_t n_images, int patch_num,
                          tp_hd_image* images_host, int32_t* crop_table_host, int* h_block, int* w_block, int64_t* n_crops) {
  if (h == nullptr || w == nullptr || n_images < 0 || n_crops == nullptr) return TP_ERR_INVALID_ARGUMENT;
  if (patch_num != 9 && patch_num != 16 && patch_num != 25) return TP_ERR_BAD_PATCH_NUM;
  int64_t crop = 0;
  for (int64_t b = 0; b < n_images; ++b) {
    if (h[b] <= 0 || w[b] <= 0 || h[b] > 32768 || w[b] > 32768) return TP_ERR_INVALID_ARGUMENT;
    int hb = 0, wb = 0, h_r = 0, w_r = 0, h_t = 0, w_t = 0;
    TP_TRY(tp_hd_grid(h[b], w[b], patch_num, kBlockPx, &hb, &wb));
    TP_TRY(tp_hd_fit(h[b], w[b], hb, wb, &h_r, &w_r, &h_t, &w_t));
    if (h_r <= 0 || w_r <= 0 || (hb * wb > 1 && (h_t <= 0 || w_t <= 0))) return TP_ERR_INVALID_ARGUMENT;
    if (h_block) h_block[b] = hb;
    if (w_block) w_block[b] = wb;
    if (images_host) {
      tp_hd_image& im = images_host[b];
      im.image = images ? static_cast<const float*>(images[b]) : nullptr;
      im.h = static_cast<int>(h[b]); im.w = static_cast<int>(w[b]); im.hb = hb; im.wb = wb;
      im.h_r = h_r; im.w_r = w_r; im.h_t = hb * wb > 1 ? h_t : 0; im.w_t = hb * wb > 1 ? w_t : 0;
      im.crop0 = crop;
      // ATen derives the bilinear scale from the sizes as ONE float division; done here once per image instead of per pixel
      im.sy = static_cast<float>(im.h) / static_cast<float>(h_r);
      im.sx = static_cast<float>(im.w) / static_cast<float>(w_r);
      im.ty = im.h_t > 0 ? static_cast<float>(kBlockPx * hb) / static_cast<float>(im.h_t) : 1.f;
      im.tx = im.w_t > 0 ? static_cast<float>(kBlockPx * wb) / static_cast<float>(im.w_t) : 1.f;
    }
    for (int i = 0; i < hb; ++i)
      for (int j = 0; j < wb; ++j, ++crop)
        if (crop_table_host) { crop_table_host[crop * 3] = static_cast<int32_t>(b); crop_table_host[crop * 3 + 1] = i; crop_table_host[crop * 3 + 2] = j; }
    if (hb * wb > 1) {       // train.py:718: the thumbnail is appended only when the image was split
      if (crop_table_host) { crop_table_host[crop * 3] = static_cast<int32_t>(b); crop_table_host[crop * 3 + 1] = 0; crop_table_host[crop * 3 + 2] = -1; }
      ++crop;
    }
  }
  *n_crops = crop;
  return TP_OK;
}

int tp_hd_tile_batch(const tp_hd_image* images_dev, const int32_t* crop_table_dev, int64_t n_crops, float* crops, void* stream_) {
  static_assert(sizeof(tp_hd_image) == sizeof(HdImage), "tp_hd_image and the kernel's HdImage must have the same layout");
  if (images_dev == nullptr || crop_table_dev == nullptr || crops == nullptr || n_crops < 0) return TP_ERR_INVALID_ARGUMENT;
  if (n_crops == 0) return TP_OK;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const long long blocks = n_crops * (kBlockPx / kHdRows);          // a CTA: kHdRows rows of one crop, one thread per pixel column, 3 channels
  if (blocks > 0x7fffffffll) return TP_ERR_INVALID_ARGUMENT;
  hd_tile_batch_kernel<<<static_cast<unsigned>(blocks), kBlockPx, 0, stream>>>(reinterpret_cast<const HdImage*>(images_dev), crop_table_dev, n_crops,
                                                                              HdF32Source{}, crops);
  TP_CUDA(cudaGetLastError()); ++g_launch_count;
  return TP_OK;
}

int tp_hd_preprocess_batch(const tp_hd_image* images_dev, const tp_hd_u8_source* sources_dev, const int32_t* crop_table_dev, int64_t n_crops,
                           const float* norm_table_dev, int out_dtype, void* crops, void* stream_) {
  static_assert(sizeof(tp_hd_u8_source) == sizeof(HdU8Image), "tp_hd_u8_source and the kernel's HdU8Image must have the same layout");
  if (images_dev == nullptr || sources_dev == nullptr || crop_table_dev == nullptr || norm_table_dev == nullptr || crops == nullptr ||
      n_crops < 0 || (out_dtype != 0 && out_dtype != 1))
    return TP_ERR_INVALID_ARGUMENT;
  if (n_crops == 0) return TP_OK;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const long long blocks = n_crops * (kBlockPx / kHdRows);          // the launch shape of tp_hd_tile_batch
  if (blocks > 0x7fffffffll) return TP_ERR_INVALID_ARGUMENT;
  const HdImage* images = reinterpret_cast<const HdImage*>(images_dev);
  const HdU8Source src{reinterpret_cast<const HdU8Image*>(sources_dev), norm_table_dev};
  if (out_dtype == 0)
    hd_tile_batch_kernel<<<static_cast<unsigned>(blocks), kBlockPx, 0, stream>>>(images, crop_table_dev, n_crops, src, static_cast<float*>(crops));
  else
    hd_tile_batch_kernel<<<static_cast<unsigned>(blocks), kBlockPx, 0, stream>>>(images, crop_table_dev, n_crops, src,
                                                                                static_cast<__nv_bfloat16*>(crops));
  TP_CUDA(cudaGetLastError()); ++g_launch_count;
  return TP_OK;
}

// ------------------------------------------------------------------------------------------------
// Non-HD CLIP input: expand2square + PIL 8-bit BICUBIC resize + center crop (include/tokenpacker_b200_clip_u8.h)
// ------------------------------------------------------------------------------------------------
namespace {
// The coefficient arithmetic below restates Pillow's Resample.c (bicubic_filter, precompute_coeffs, normalize_coeffs_8bpc) operation
// for operation in double precision; PIL's bits depend on every product being rounded before the following addition.  A compiler
// that contracts a * b + c into one fused multiply-add (g++ does by default on aarch64, where FMA is part of the base ISA) would
// round once instead of twice and move some weights by one unit, so contraction is switched off for these functions.
__attribute__((optimize("fp-contract=off"))) double pil_bicubic(double x) {
  const double a = -0.5;
  if (x < 0.0) x = -x;
  if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
  if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
  return 0.0;
}

int pil_bicubic_ksize(int in_size, int out_size) {
  const double scale = static_cast<double>(in_size) / out_size;
  return static_cast<int>(ceil(2.0 * (scale < 1.0 ? 1.0 : scale))) * 2 + 1;
}

// Weights of the outputs first .. first + 336 - 1 of an in_size -> out_size BICUBIC resample, laid out as tp_clip_image documents:
// [336] first source index, [336] tap count, [ksize][336] int32 weights (zero past the count).  tab may be NULL (bounds only).
__attribute__((optimize("fp-contract=off"))) void pil_bicubic_table(int in_size, int out_size, int first, int32_t* tab, int* lo, int* hi) {
  const double scale = static_cast<double>(in_size) / out_size;
  const double filterscale = scale < 1.0 ? 1.0 : scale;
  const double support = 2.0 * filterscale;
  const double ss = 1.0 / filterscale;
  const int ksize = pil_bicubic_ksize(in_size, out_size);
  std::vector<double> w(ksize);
  *lo = INT_MAX; *hi = 0;
  for (int j = 0; j < kBlockPx; ++j) {
    const int xx = first + j;
    const double center = (xx + 0.5) * scale;
    int xmin = static_cast<int>(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = static_cast<int>(center + support + 0.5);
    if (xmax > in_size) xmax = in_size;
    xmax -= xmin;
    if (xmin < *lo) *lo = xmin;
    if (xmin + xmax > *hi) *hi = xmin + xmax;
    if (tab == nullptr) continue;
    double ww = 0.0;
    for (int x = 0; x < xmax; ++x) {
      w[x] = pil_bicubic((x + xmin - center + 0.5) * ss);
      ww += w[x];
    }
    tab[j] = xmin;
    tab[kBlockPx + j] = xmax;
    for (int x = 0; x < ksize; ++x) {
      int32_t k = 0;
      if (x < xmax) {
        const double v = ww != 0.0 ? w[x] / ww : w[x];
        k = static_cast<int32_t>(v < 0 ? -0.5 + v * (1 << kClipPrecision) : 0.5 + v * (1 << kClipPrecision));
      }
      tab[(2 + x) * kBlockPx + j] = k;
    }
  }
}
}  // namespace

int tp_clip_preprocess_plan(const int64_t* h, const int64_t* w, int64_t n_images, int mode, tp_clip_image* images, int32_t* coeffs,
                            int64_t* n_coeffs, size_t* workspace_bytes) {
  static_assert(sizeof(tp_clip_image) == sizeof(ClipImage), "tp_clip_image and the kernel's ClipImage must have the same layout");
  if (h == nullptr || w == nullptr || n_coeffs == nullptr || workspace_bytes == nullptr || n_images < 0 ||
      (mode != TP_CLIP_SQUARE && mode != TP_CLIP_PAD))
    return TP_ERR_INVALID_ARGUMENT;
  for (int64_t b = 0; b < n_images; ++b)
    if (h[b] < 1 || w[b] < 1 || h[b] > TP_CLIP_MAX_SIDE || w[b] > TP_CLIP_MAX_SIDE) return TP_ERR_INVALID_ARGUMENT;
  const bool write = images != nullptr && coeffs != nullptr;
  struct Table { int in, out, first; int64_t offset; int lo, hi; };
  std::map<std::tuple<int, int, int>, Table> tables;         // one table per (input size, output size, first kept output)
  int64_t n_co = 0, ws_rows = 0;
  auto table = [&](int in, int out, int first) -> const Table& {
    auto it = tables.find(std::make_tuple(in, out, first));
    if (it == tables.end()) {
      Table t{in, out, first, n_co, 0, 0};
      pil_bicubic_table(in, out, first, write ? coeffs + n_co : nullptr, &t.lo, &t.hi);
      n_co += static_cast<int64_t>(2 + pil_bicubic_ksize(in, out)) * kBlockPx;
      it = tables.emplace(std::make_tuple(in, out, first), t).first;
    }
    return it->second;
  };
  for (int64_t b = 0; b < n_images; ++b) {
    tp_clip_image im;
    memset(&im, 0, sizeof(im));
    im.h = static_cast<int32_t>(h[b]); im.w = static_cast<int32_t>(w[b]);
    im.canvas_h = im.h; im.canvas_w = im.w;
    if (mode == TP_CLIP_PAD && im.h != im.w) {               // expand2square (mm_utils.py:14-25): paste into the middle of L x L
      const int side = im.h > im.w ? im.h : im.w;
      im.canvas_h = im.canvas_w = side;
      if (im.w > im.h) im.pad_y = (im.w - im.h) / 2; else im.pad_x = (im.h - im.w) / 2;
    }
    // get_resize_output_image_size(default_to_square=False): the short edge becomes 336, the long edge int(336 * long / short)
    // (Python's true division, float64, truncated); nothing is resized when the short edge is already 336
    const bool w_short = im.canvas_w <= im.canvas_h;
    const int s = w_short ? im.canvas_w : im.canvas_h, l = w_short ? im.canvas_h : im.canvas_w;
    im.resized_h = im.canvas_h; im.resized_w = im.canvas_w;
    if (s != kBlockPx) {
      const int new_l = static_cast<int>(static_cast<double>(static_cast<int64_t>(kBlockPx) * l) / static_cast<double>(s));
      im.resized_h = w_short ? new_l : kBlockPx;
      im.resized_w = w_short ? kBlockPx : new_l;
    }
    im.top = (im.resized_h - kBlockPx) / 2;
    im.left = (im.resized_w - kBlockPx) / 2;
    im.coeff_x = im.coeff_y = -1;
    if (im.resized_w != im.canvas_w) {
      const Table& t = table(im.canvas_w, im.resized_w, im.left);
      im.ksize_x = pil_bicubic_ksize(t.in, t.out);
      im.coeff_x = t.offset;
    }
    im.row0 = im.top;
    im.rows = kBlockPx;
    if (im.resized_h != im.canvas_h) {
      const Table& t = table(im.canvas_h, im.resized_h, im.top);
      im.ksize_y = pil_bicubic_ksize(t.in, t.out);
      im.coeff_y = t.offset;
      im.row0 = t.lo;
      im.rows = t.hi - t.lo;
    }
    if (im.ksize_x == 0) im.rows = 0;                         // no horizontal pass: the vertical pass reads the canvas
    im.workspace_row = ws_rows;
    im.workspace_offset = ws_rows * kClipRowBytes;
    ws_rows += im.rows;
    if (write) images[b] = im;
  }
  *n_coeffs = n_co;
  *workspace_bytes = static_cast<size_t>(ws_rows) * kClipRowBytes;
  return TP_OK;
}

int tp_clip_preprocess_batch(const tp_clip_image* images_host, const tp_clip_image* images_dev, const tp_hd_u8_source* sources_dev,
                             const int32_t* coeffs_dev, int64_t n_images, const float* norm_table_dev, int out_dtype, void* out,
                             void* workspace, size_t workspace_bytes, void* stream_) {
  if (images_host == nullptr || images_dev == nullptr || sources_dev == nullptr || coeffs_dev == nullptr || norm_table_dev == nullptr ||
      out == nullptr || n_images < 0 || (out_dtype != 0 && out_dtype != 1))
    return TP_ERR_INVALID_ARGUMENT;
  if (n_images == 0) return TP_OK;
  if (n_images > 0x7fffffffll / kBlockPx) return TP_ERR_INVALID_ARGUMENT;      // the vertical launch: one CTA per output row
  int64_t rows = 0;
  for (int64_t b = 0; b < n_images; ++b) {
    const tp_clip_image& im = images_host[b];
    if (im.rows < 0 || im.workspace_row < 0) return TP_ERR_INVALID_ARGUMENT;
    if (im.ksize_x > 0 && im.workspace_row + im.rows > rows) rows = im.workspace_row + im.rows;
  }
  if (rows > 0x7fffffffll) return TP_ERR_INVALID_ARGUMENT;                       // the horizontal launch: one CTA per workspace row
  if (static_cast<uint64_t>(rows) * kClipRowBytes > workspace_bytes) return TP_ERR_WORKSPACE_TOO_SMALL;
  if (rows > 0 && workspace == nullptr) return TP_ERR_INVALID_ARGUMENT;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const ClipImage* images = reinterpret_cast<const ClipImage*>(images_dev);
  const HdU8Image* sources = reinterpret_cast<const HdU8Image*>(sources_dev);
  unsigned char* ws = static_cast<unsigned char*>(workspace);
  if (rows > 0) {
    clip_resample_h_kernel<<<static_cast<unsigned>(rows), kBlockPx, 0, stream>>>(images, n_images, sources, coeffs_dev, ws);
    TP_CUDA(cudaGetLastError()); ++g_launch_count;
  }
  const unsigned blocks = static_cast<unsigned>(n_images * kBlockPx);
  if (out_dtype == 0)
    clip_resample_v_kernel<<<blocks, kBlockPx, 0, stream>>>(images, sources, coeffs_dev, ws, norm_table_dev, static_cast<float*>(out));
  else
    clip_resample_v_kernel<<<blocks, kBlockPx, 0, stream>>>(images, sources, coeffs_dev, ws, norm_table_dev, static_cast<__nv_bfloat16*>(out));
  TP_CUDA(cudaGetLastError()); ++g_launch_count;
  return TP_OK;
}

int tp_hd_plan(const int* h_block, const int* w_block, int64_t n_images, int tokens_per_crop, int64_t* seg_row_offset_host,
               int64_t* sep_rows_host, int64_t* ret_rows_host, int64_t* cu_seqlens_host, int64_t* n_crops, int64_t* n_sep, int64_t* n_ret) {
  if (h_block == nullptr || w_block == nullptr || n_images < 0 || tokens_per_crop <= 0) return TP_ERR_INVALID_ARGUMENT;
  int64_t row = 0, crop = 0, sep = 0, ret = 0;
  if (cu_seqlens_host) cu_seqlens_host[0] = 0;
  for (int64_t b = 0; b < n_images; ++b) {
    const int hb = h_block[b], wb = w_block[b];
    if (hb <= 0 || wb <= 0) return TP_ERR_INVALID_ARGUMENT;
    // llava_arch.py:141-152
    for (int i = 0; i < hb; ++i) {
      for (int j = 0; j < wb; ++j) {
        if (seg_row_offset_host) seg_row_offset_host[crop] = row;
        ++crop;
        row += tokens_per_crop;
        if (j < wb - 1) {
          if (sep_rows_host) sep_rows_host[sep] = row;
          ++sep;
          ++row;
        }
      }
      if (ret_rows_host) ret_rows_host[ret] = row;
      ++ret;
      ++row;
    }
    if (hb * wb > 1) {
      if (seg_row_offset_host) seg_row_offset_host[crop] = row;
      ++crop;
      row += tokens_per_crop;
      if (ret_rows_host) ret_rows_host[ret] = row;
      ++ret;
      ++row;
    }
    if (cu_seqlens_host) cu_seqlens_host[b + 1] = row;
  }
  if (n_crops) *n_crops = crop;
  if (n_sep) *n_sep = sep;
  if (n_ret) *n_ret = ret;
  return TP_OK;
}

int tp_hd_scatter_crops(const void* feats, int64_t n_crops, int tokens_per_crop, int hidden, const int64_t* seg_row_offset, void* out,
                        void* stream_) {
  if (feats == nullptr || out == nullptr || seg_row_offset == nullptr || n_crops <= 0 || tokens_per_crop <= 0 || hidden <= 0 ||
      hidden % 8 != 0)
    return TP_ERR_INVALID_ARGUMENT;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const long long threads = n_crops * tokens_per_crop * (hidden / 8);
  scatter_crops_kernel<<<static_cast<unsigned>((threads + 255) / 256), 256, 0, stream>>>(
      static_cast<const __nv_bfloat16*>(feats), n_crops, tokens_per_crop, hidden, reinterpret_cast<const long long*>(seg_row_offset),
      static_cast<__nv_bfloat16*>(out));
  TP_CUDA(cudaGetLastError()); ++g_launch_count;
  return TP_OK;
}

int tp_gather_rows(const void* table, const void* visual, int hidden, const int64_t* src_index, int64_t n_rows, void* out, void* stream_) {
  if (table == nullptr || out == nullptr || src_index == nullptr || hidden <= 0 || hidden % 8 != 0 || n_rows < 0) return TP_ERR_INVALID_ARGUMENT;
  if (n_rows == 0) return TP_OK;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const long long threads = n_rows * (hidden / 8);
  gather_rows_kernel<<<static_cast<unsigned>((threads + 255) / 256), 256, 0, stream>>>(
      static_cast<const __nv_bfloat16*>(table), static_cast<const __nv_bfloat16*>(visual), hidden, reinterpret_cast<const long long*>(src_index),
      n_rows, static_cast<__nv_bfloat16*>(out));
  TP_CUDA(cudaGetLastError()); ++g_launch_count;
  return TP_OK;
}

int tp_hd_fill_separators(void* out, int hidden, const int64_t* sep_rows, int64_t n_sep, const void* sep_row, const int64_t* ret_rows,
                          int64_t n_ret, const void* ret_row, void* stream_) {
  if (out == nullptr || hidden <= 0 || hidden % 8 != 0 || n_sep < 0 || n_ret < 0) return TP_ERR_INVALID_ARGUMENT;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int vecs = hidden / 8;
  if (n_sep > 0) {
    if (sep_rows == nullptr || sep_row == nullptr) return TP_ERR_INVALID_ARGUMENT;
    fill_rows_kernel<<<static_cast<unsigned>((n_sep * vecs + 255) / 256), 256, 0, stream>>>(
        static_cast<__nv_bfloat16*>(out), hidden, reinterpret_cast<const long long*>(sep_rows), n_sep, static_cast<const __nv_bfloat16*>(sep_row));
    TP_CUDA(cudaGetLastError()); ++g_launch_count;
  }
  if (n_ret > 0) {
    if (ret_rows == nullptr || ret_row == nullptr) return TP_ERR_INVALID_ARGUMENT;
    fill_rows_kernel<<<static_cast<unsigned>((n_ret * vecs + 255) / 256), 256, 0, stream>>>(
        static_cast<__nv_bfloat16*>(out), hidden, reinterpret_cast<const long long*>(ret_rows), n_ret, static_cast<const __nv_bfloat16*>(ret_row));
    TP_CUDA(cudaGetLastError()); ++g_launch_count;
  }
  return TP_OK;
}

}  // extern "C"

#include "tp_clip_tower.inl"
#include "tp_clip_tower_train.inl"
#include "tp_clip_tower_embed.inl"
#include "tp_clip_tower_crop_grad.inl"
#include "tp_jpeg.inl"
#include "tp_png.inl"
