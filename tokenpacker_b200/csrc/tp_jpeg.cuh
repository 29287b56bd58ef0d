// Baseline JPEG decode on sm_90a (include/tokenpacker_b200_jpeg.h): unstuff, self-synchronising parallel Huffman decode with DC
// prediction, jpeg_idct_islow, fancy upsampling and YCbCr -> RGB.  Integer arithmetic as libjpeg-turbo does it, so the bytes equal
// PIL's; oracle/jpeg_oracle.py states the same decoder in numpy and the tests pin both against PIL.
#pragma once
#include <cub/block/block_scan.cuh>
#include <stdint.h>

#include "../../include/tokenpacker_b200_jpeg.h"

namespace tpjpeg {

constexpr int kUnstuffThreads = 512;
constexpr int kUnstuffBytesPerThread = 8;
constexpr int kHuffThreads = 512;
constexpr int kSubBits = TP_JPEG_SUBSEQUENCE_BYTES * 8;
constexpr int kIdctThreads = 256;                       // 8 threads per block: 32 blocks per CTA
constexpr int kColourThreads = 256;
constexpr int kPoisoned = -1;                           // exit state of a decode that met an error: its successors wait

// One subsequence: [start, end) bits of the file's unstuffed bytes, inside restart interval seg whose data ends at seg_end.
// State = (bit position, block in the MCU << 8 | coefficient index); coefficient index 0 means a DC code comes next.
struct JpegSub {
  long long start, end, seg_end;
  long long entry_pos, exit_pos;
  int seg;
  int entry_bk, exit_bk;
  int started;    // DC codes decoded from the entry to the exit
  int bad;        // first block, counted from this subsequence's first DC, that an error touched; INT_MAX when none
  int first;      // interval-relative index of the block of this subsequence's first DC (after the scan)
};
static_assert(sizeof(JpegSub) == 64, "subsequence records are 64 bytes");

// natural index of the k-th coefficient in the stream
__constant__ unsigned char kJpegZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                              41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                              30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// Per block of the MCU: component, and block row / column inside the component's part of the MCU.
__device__ __forceinline__ void jpeg_block_of_mcu(const tp_jpeg_image& im, int b, int* c, int* dy, int* dx) {
  const int n0 = im.hs * im.vs;
  if (b < n0) { *c = 0; *dy = b / im.hs; *dx = b % im.hs; }
  else { *c = b - n0 + 1; *dy = 0; *dx = 0; }
}

// ------------------------------------------------------------------------------------------------
// 1. unstuff: one CTA per file
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kUnstuffThreads) jpeg_unstuff_kernel(const tp_jpeg_image* __restrict__ images,
                                                                        const uint8_t* __restrict__ staged, uint8_t* ws,
                                                                        tp_jpeg_status* status) {
  const tp_jpeg_image& im = images[blockIdx.x];
  if (im.reason != TP_JPEG_SUPPORTED) return;
  using Scan = cub::BlockScan<int2, kUnstuffThreads>;
  using Scan1 = cub::BlockScan<int, kUnstuffThreads>;
  __shared__ union { typename Scan::TempStorage s2; typename Scan1::TempStorage s1; } tmp;
  const uint8_t* src = staged + im.scan_offset;
  const long long n = im.scan_bytes;
  uint8_t* dst = ws + im.unstuffed_offset;
  long long* segs = reinterpret_cast<long long*>(ws + im.seg_offset);
  long long out_base = 0, rst_base = 0;
  for (long long base = 0; base < n; base += static_cast<long long>(kUnstuffThreads) * kUnstuffBytesPerThread) {
    const long long i0 = base + static_cast<long long>(threadIdx.x) * kUnstuffBytesPerThread;
    // kind per byte: 1 = emit, 2 = RSTn starts here, 0 = dropped
    unsigned char kind[kUnstuffBytesPerThread], val[kUnstuffBytesPerThread];
    int2 cnt = make_int2(0, 0);
#pragma unroll
    for (int j = 0; j < kUnstuffBytesPerThread; ++j) {
      const long long i = i0 + j;
      kind[j] = 0; val[j] = 0;
      if (i < n) {
        const unsigned cur = src[i], prev = i > 0 ? src[i - 1] : 0u, next = i + 1 < n ? src[i + 1] : 0u;
        if (cur == 0xFF) {
          if (next == 0x00) kind[j] = 1;
          else if (next >= 0xD0 && next <= 0xD7) kind[j] = 2;
        } else if (!(prev == 0xFF && (cur == 0x00 || (cur >= 0xD0 && cur <= 0xD7)))) {
          kind[j] = 1;
        }
        val[j] = static_cast<unsigned char>(cur);
        cnt.x += kind[j] == 1;
        cnt.y += kind[j] == 2;
      }
    }
    int2 excl, total;
    Scan(tmp.s2).ExclusiveScan(cnt, excl, make_int2(0, 0),
                               [](const int2& a, const int2& b) { return make_int2(a.x + b.x, a.y + b.y); }, total);
    long long o = out_base + excl.x, r = rst_base + excl.y;
#pragma unroll
    for (int j = 0; j < kUnstuffBytesPerThread; ++j) {
      if (kind[j] == 1) dst[o++] = val[j];
      else if (kind[j] == 2) {
        ++r;                                   // interval r starts here
        if (r < im.n_segments) segs[r] = o;
      }
    }
    out_base += total.x;
    rst_base += total.y;
    __syncthreads();                           // tmp is reused
  }
  if (threadIdx.x == 0) {
    segs[0] = 0;
    if (rst_base != im.n_segments - 1) status[blockIdx.x].status = TP_JPEG_STATUS_RESTART;
  }
  // intervals the markers did not delimit are empty: decoding them reports the missing blocks
  const long long found = rst_base < im.n_segments - 1 ? rst_base : im.n_segments - 1;
  for (long long s = found + 1 + threadIdx.x; s <= im.n_segments; s += kUnstuffThreads) segs[s] = out_base;
  __syncthreads();
  // subsequences: every interval cut into TP_JPEG_SUBSEQUENCE_BYTES pieces (at least one)
  JpegSub* subs = reinterpret_cast<JpegSub*>(ws + im.sub_offset);
  int sub_base = 0;
  for (int s0 = 0; s0 < im.n_segments; s0 += kUnstuffThreads) {
    const int s = s0 + threadIdx.x;
    long long a = 0, e = 0;
    int cnt = 0;
    if (s < im.n_segments) {
      a = segs[s];
      e = segs[s + 1];
      if (e < a) e = a;
      cnt = static_cast<int>((e - a + TP_JPEG_SUBSEQUENCE_BYTES - 1) / TP_JPEG_SUBSEQUENCE_BYTES);
      if (cnt == 0) cnt = 1;
    }
    int excl, total;
    Scan1(tmp.s1).ExclusiveSum(cnt, excl, total);
    for (int q = 0; q < cnt; ++q) {
      const long long idx = static_cast<long long>(sub_base) + excl + q;
      if (idx >= im.sub_capacity) break;       // cannot happen: the capacity bounds the count
      JpegSub sub;
      sub.start = a * 8 + static_cast<long long>(q) * kSubBits;
      sub.end = min(sub.start + kSubBits, e * 8);
      sub.seg_end = e * 8;
      sub.entry_pos = sub.exit_pos = sub.start;
      sub.seg = s;
      sub.entry_bk = sub.exit_bk = 0;
      sub.started = 0;
      sub.bad = 0x7fffffff;
      sub.first = 0;
      subs[idx] = sub;
    }
    sub_base += total;
    __syncthreads();
  }
  if (threadIdx.x == 0) status[blockIdx.x].subsequences = static_cast<int>(min(static_cast<long long>(sub_base), static_cast<long long>(im.sub_capacity)));
}

// ------------------------------------------------------------------------------------------------
// 2. Huffman decode: one CTA per file
// ------------------------------------------------------------------------------------------------
struct BitReader {
  const uint8_t* p;
  long long next, end;     // bytes: next to load, end of the interval (zeros are read past it)
  unsigned long long buf;  // left-aligned
  int nbits;
  long long pos;           // bits consumed, from the start of the file's unstuffed bytes

  __device__ __forceinline__ void init(const uint8_t* bytes, long long at, long long end_bits) {
    p = bytes;
    end = end_bits >> 3;
    next = at >> 3;
    buf = 0;
    nbits = 0;
    pos = next * 8;
    refill();
    skip(static_cast<int>(at & 7));
  }
  __device__ __forceinline__ void refill() {
    while (nbits <= 56) {
      const unsigned long long b = next < end ? p[next] : 0ull;
      buf |= b << (56 - nbits);
      nbits += 8;
      ++next;
    }
  }
  __device__ __forceinline__ unsigned peek(int n) const { return static_cast<unsigned>(buf >> (64 - n)); }
  __device__ __forceinline__ void skip(int n) { buf <<= n; nbits -= n; pos += n; }
  __device__ __forceinline__ int get(int n) {       // n <= 16
    if (n == 0) return 0;
    const int v = static_cast<int>(peek(n));
    skip(n);
    return v;
  }
};

// Decodes one Huffman symbol (the reader holds at least 41 bits); -1 for an invalid code.
__device__ __forceinline__ int jpeg_huff_decode(const tp_jpeg_huff& t, BitReader& br) {
  const unsigned e = t.lookup[br.peek(9)];
  if (e != 0) {
    br.skip(static_cast<int>(e >> 8));
    return static_cast<int>(e & 255);
  }
  const int code16 = static_cast<int>(br.peek(16));
  for (int l = 10; l <= 16; ++l) {
    const int c = code16 >> (16 - l);
    if (c <= t.maxcode[l]) {
      br.skip(l);
      return t.values[(c + t.valoff[l]) & 255];
    }
  }
  return -1;
}

__device__ __forceinline__ int jpeg_extend(int v, int s) { return (s != 0 && v < (1 << (s - 1))) ? v - (1 << s) + 1 : v; }

struct JpegSmem {
  tp_jpeg_tables t;
  unsigned char zz[64];
  int flag;
};

// Decodes from (pos, bk) while pos < stop.  Counting pass (kWrite false): returns the exit state, the DC codes decoded and the first
// block an error touched.  Writing pass: also stores the coefficients of blocks cur = first - 1 + (DC codes so far) while
// cur < needed (interval-relative), in natural order with the DC difference in [0]; every position of a block is written once.
template <bool kWrite>
__device__ __forceinline__ void jpeg_decode_span(const JpegSmem& sm, const tp_jpeg_image& im, const uint8_t* bytes, const JpegSub& sub, long long pos,
                                 int bk, long long* exit_pos, int* exit_bk, int* started_out, int* bad_out, int16_t* coef,
                                 long long interval_block0, int first, int needed) {
  int b = bk >> 8, k = bk & 255;
  int started = 0, bad = 0x7fffffff;
  BitReader br;
  br.init(bytes, pos, sub.seg_end);
  int cur = first - 1;                       // interval-relative block being decoded
  int16_t* blk = nullptr;
  int c, dy, dx;
  jpeg_block_of_mcu(im, b, &c, &dy, &dx);
  auto locate = [&]() -> int16_t* {
    if (!kWrite || cur < 0 || cur >= needed) return nullptr;
    const long long t = interval_block0 + cur;
    const long long mcu = t / im.blocks_per_mcu;
    const long long my = mcu / im.mcus_x, mx = mcu % im.mcus_x;
    long long base = 0;
    for (int cc = 0; cc < c; ++cc) base += static_cast<long long>(im.comp_bx[cc]) * im.comp_by[cc];
    const long long by = my * (c == 0 ? im.vs : 1) + dy, bx = mx * (c == 0 ? im.hs : 1) + dx;
    return coef + (base + by * im.comp_bx[c] + bx) * 64;
  };
  if (kWrite && k > 0) blk = locate();
  bool err = false;
  while (br.pos < sub.end) {
    br.refill();
    if (k == 0) {
      const int s = jpeg_huff_decode(sm.t.dc[c], br);
      if (s < 0 || s > 15) { err = true; break; }
      const int v = jpeg_extend(br.get(s), s);
      ++started;
      ++cur;
      if (kWrite) {
        blk = locate();
        if (blk) blk[0] = static_cast<int16_t>(v);
      }
      k = 1;
      if (br.pos > sub.seg_end) { err = true; break; }    // read past the end of the interval: this block is not whole
    } else {
      const int rs = jpeg_huff_decode(sm.t.ac[c], br);
      if (rs < 0) { err = true; break; }
      const int r = rs >> 4, s = rs & 15;
      if (s == 0) {
        const int kend = r == 15 ? k + 16 : 64;
        if (kend > 64) { err = true; break; }
        if (blk) for (int j = k; j < kend; ++j) blk[sm.zz[j]] = 0;
        k = kend;
      } else {
        if (k + r > 63) { err = true; break; }
        const int v = jpeg_extend(br.get(s), s);
        if (blk) {
          for (int j = k; j < k + r; ++j) blk[sm.zz[j]] = 0;
          blk[sm.zz[k + r]] = static_cast<int16_t>(v);
        }
        k += r + 1;
      }
      // checked before the block is closed, so that the error names the block whose code or value read the zeros past the end
      if (br.pos > sub.seg_end) { err = true; break; }
      if (k == 64) {
        k = 0;
        b = b + 1 == im.blocks_per_mcu ? 0 : b + 1;
        jpeg_block_of_mcu(im, b, &c, &dy, &dx);
        blk = nullptr;
      }
    }
  }
  if (err) {
    bad = started - (k > 0 ? 1 : 0);
    *exit_pos = sub.end;
    *exit_bk = kPoisoned;
  } else {
    *exit_pos = br.pos;
    *exit_bk = (b << 8) | k;
  }
  *started_out = started;
  *bad_out = bad;
}

__device__ __forceinline__ bool jpeg_first_of_interval(const JpegSub* subs, int i) { return i == 0 || subs[i - 1].seg != subs[i].seg; }

__device__ __forceinline__ int jpeg_blocks_in_interval(const tp_jpeg_image& im, int seg) {
  const long long mcus = static_cast<long long>(im.mcus_x) * im.mcus_y;
  const long long left = mcus - static_cast<long long>(seg) * im.restart;
  return static_cast<int>((left < im.restart ? left : im.restart) * im.blocks_per_mcu);
}

struct SegPair { int flag, v; };

__global__ void __launch_bounds__(kHuffThreads, 1) jpeg_huffman_kernel(const tp_jpeg_image* __restrict__ images,
                                                                     const tp_jpeg_tables* __restrict__ tables, uint8_t* ws,
                                                                     tp_jpeg_status* status) {
  const tp_jpeg_image& im = images[blockIdx.x];
  if (im.reason != TP_JPEG_SUPPORTED) return;
  using Scan = cub::BlockScan<SegPair, kHuffThreads>;
  __shared__ JpegSmem sm;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ int s_err;
  {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(&tables[blockIdx.x]);
    uint32_t* dst = reinterpret_cast<uint32_t*>(&sm.t);
    for (int i = threadIdx.x; i < static_cast<int>(sizeof(tp_jpeg_tables) / 4); i += kHuffThreads) dst[i] = src[i];
  }
  if (threadIdx.x < 64) sm.zz[threadIdx.x] = kJpegZigzag[threadIdx.x];
  if (threadIdx.x == 0) { sm.flag = 1; s_err = 0; }
  const uint8_t* bytes = ws + im.unstuffed_offset;
  JpegSub* subs = reinterpret_cast<JpegSub*>(ws + im.sub_offset);
  int16_t* coef = reinterpret_cast<int16_t*>(ws + im.coef_offset);
  __syncthreads();
  const int n = status[blockIdx.x].subsequences;
  // speculative decode: every subsequence from its first bit, as if a block started there
  for (int i = threadIdx.x; i < n; i += kHuffThreads) {
    JpegSub& s = subs[i];
    jpeg_decode_span<false>(sm, im, bytes, s, s.start, 0, &s.exit_pos, &s.exit_bk, &s.started, &s.bad, nullptr, 0, 0, 0);
  }
  // rounds: a subsequence whose entry differs from its predecessor's exit decodes again from that exit; a decode from the true entry
  // reproduces the true exit, so after at most n rounds (one per subsequence, a sequential decode) every entry is true
  int rounds = 0;
  for (;;) {
    __syncthreads();
    if (threadIdx.x == 0) sm.flag = 0;
    __syncthreads();
    // phase A reads only exits and writes only entries
    for (int i = threadIdx.x; i < n; i += kHuffThreads) {
      if (jpeg_first_of_interval(subs, i)) continue;
      const JpegSub& p = subs[i - 1];
      JpegSub& s = subs[i];
      if (p.exit_pos != s.entry_pos || p.exit_bk != s.entry_bk) {
        s.entry_pos = p.exit_pos;
        s.entry_bk = p.exit_bk;
        s.first = -1;                          // marks the record for phase B
        sm.flag = 1;
      }
    }
    __syncthreads();
    if (sm.flag == 0) break;
    ++rounds;
    for (int i = threadIdx.x; i < n; i += kHuffThreads) {
      JpegSub& s = subs[i];
      if (s.first != -1) continue;
      s.first = 0;
      // behind an error the exit stays as it was, so that a speculative error does not travel down the chain one subsequence per
      // round; after a true error nothing here is written (its blocks lie past the error, which the check below reports)
      if (s.entry_bk == kPoisoned) continue;
      if (s.entry_pos >= s.end) {                // the predecessor's last code ran past this subsequence: nothing starts here
        s.exit_pos = s.entry_pos;
        s.exit_bk = s.entry_bk;
        s.started = 0;
        s.bad = 0x7fffffff;
        continue;
      }
      jpeg_decode_span<false>(sm, im, bytes, s, s.entry_pos, s.entry_bk, &s.exit_pos, &s.exit_bk, &s.started, &s.bad, nullptr, 0, 0, 0);
    }
  }
  // place the blocks: exclusive scan of the DC counts, restarted at every interval
  {
    int carry = 0;
    for (int i0 = 0; i0 < n; i0 += kHuffThreads) {
      const int i = i0 + threadIdx.x;
      SegPair in{0, 0};
      if (i < n) in = SegPair{jpeg_first_of_interval(subs, i) ? 1 : 0, subs[i].started};
      SegPair out, total;
      Scan(tmp).InclusiveScan(in, out, [](const SegPair& a, const SegPair& b) { return SegPair{a.flag | b.flag, b.flag ? b.v : a.v + b.v}; },
                              total);
      if (i < n) {
        const int incl = out.flag ? out.v : out.v + carry;        // no interval start in this chunk up to i: continue the carry
        subs[i].first = incl - subs[i].started;
      }
      carry = total.flag ? total.v : total.v + carry;
      __syncthreads();
    }
  }
  __syncthreads();
  // check every interval: an error before its last block, or too few complete blocks
  for (int i = threadIdx.x; i < n; i += kHuffThreads) {
    const JpegSub& s = subs[i];
    const int needed = jpeg_blocks_in_interval(im, s.seg);
    if (s.bad != 0x7fffffff && static_cast<long long>(s.first) + s.bad < needed) s_err = 1;
    const bool last = i == n - 1 || subs[i + 1].seg != s.seg;
    if (last && s.entry_bk != kPoisoned && s.exit_bk != kPoisoned && s.bad == 0x7fffffff) {
      const int complete = s.first + s.started - ((s.exit_bk & 255) != 0 ? 1 : 0);
      if (complete < needed) s_err = 1;
    }
  }
  // second decode: the coefficients
  for (int i = threadIdx.x; i < n; i += kHuffThreads) {
    const JpegSub& s = subs[i];
    if (s.entry_bk == kPoisoned || s.entry_pos >= s.end) continue;
    const int needed = jpeg_blocks_in_interval(im, s.seg);
    if (s.first > needed) continue;
    long long ep;
    int eb, st, bd;
    const long long block0 = static_cast<long long>(s.seg) * im.restart * im.blocks_per_mcu;
    jpeg_decode_span<true>(sm, im, bytes, s, s.entry_pos, s.entry_bk, &ep, &eb, &st, &bd, coef, block0, s.first, needed);
  }
  __syncthreads();
  // DC prediction: per component, a running sum of the differences in decode order, restarted at every interval
  for (int c = 0; c < im.ncomp; ++c) {
    const int per_mcu = c == 0 ? im.hs * im.vs : 1;
    const long long n_e = static_cast<long long>(im.mcus_x) * im.mcus_y * per_mcu;
    long long base = 0;
    for (int cc = 0; cc < c; ++cc) base += static_cast<long long>(im.comp_bx[cc]) * im.comp_by[cc];
    int carry = 0;
    for (long long e0 = 0; e0 < n_e; e0 += kHuffThreads) {
      const long long e = e0 + threadIdx.x;
      int16_t* dc = nullptr;
      SegPair in{0, 0};
      if (e < n_e) {
        const long long mcu = e / per_mcu;
        const int j = static_cast<int>(e % per_mcu);
        const long long my = mcu / im.mcus_x, mx = mcu % im.mcus_x;
        const int hs = c == 0 ? im.hs : 1;
        const long long by = my * (c == 0 ? im.vs : 1) + j / hs, bx = mx * hs + j % hs;
        dc = coef + (base + by * im.comp_bx[c] + bx) * 64;
        in = SegPair{(mcu % im.restart == 0 && j == 0) ? 1 : 0, *dc};
      }
      SegPair out, total;
      Scan(tmp).InclusiveScan(in, out, [](const SegPair& a, const SegPair& b) { return SegPair{a.flag | b.flag, b.flag ? b.v : a.v + b.v}; },
                              total);
      if (dc) *dc = static_cast<int16_t>(out.flag ? out.v : out.v + carry);
      carry = total.flag ? total.v : total.v + carry;
      __syncthreads();
    }
  }
  if (threadIdx.x == 0) {
    tp_jpeg_status& st = status[blockIdx.x];
    if (s_err && st.status == TP_JPEG_STATUS_OK) st.status = TP_JPEG_STATUS_ENTROPY;
    st.sync_rounds = rounds;
  }
}

// ------------------------------------------------------------------------------------------------
// 3. dequantise + jpeg_idct_islow: 8 threads per block
// ------------------------------------------------------------------------------------------------
constexpr int kConstBits = 13, kPass1Bits = 2;
constexpr int FIX_0_298631336 = 2446, FIX_0_390180644 = 3196, FIX_0_541196100 = 4433, FIX_0_765366865 = 6270, FIX_0_899976223 = 7373,
              FIX_1_175875602 = 9633, FIX_1_501321110 = 12299, FIX_1_847759065 = 15137, FIX_1_961570560 = 16069,
              FIX_2_053119869 = 16819, FIX_2_562915447 = 20995, FIX_3_072711026 = 25172;

__device__ __forceinline__ int jpeg_w16(int x) { return static_cast<int16_t>(x); }            // a 16-bit SIMD add or multiply
__device__ __forceinline__ int jpeg_sat16(int x) { return x < -32768 ? -32768 : (x > 32767 ? 32767 : x); }

// One islow pass over in[0], in[st], .. in[7 st] (int16 values), descaled by shift and saturated to int16 into o[0 .. 7]: the
// arithmetic of libjpeg-turbo's SIMD islow, which PIL runs on x86.  The sums in0 +- in4, in7 + in3 and in5 + in1 are 16-bit (they
// wrap), every product pairs 16-bit operands into 32-bit sums, and the outputs are packed to int16 with saturation.  This equals
// jidctint.c's C code whenever no value leaves 16 bits (every file with quantisers up to a few thousand); past that the SIMD and C
// builds of libjpeg-turbo differ and PIL's bits are the SIMD build's.  oracle/jpeg_oracle.py states the same.
__device__ __forceinline__ void jpeg_idct_1d(const int* in, int st, int shift, int* o) {
  const int z2 = in[2 * st], z3 = in[6 * st];
  const int tmp3 = z2 * (FIX_0_541196100 + FIX_0_765366865) + z3 * FIX_0_541196100;
  const int tmp2 = z2 * FIX_0_541196100 + z3 * (FIX_0_541196100 - FIX_1_847759065);
  const int tmp0 = jpeg_w16(in[0] + in[4 * st]) * (1 << kConstBits);
  const int tmp1 = jpeg_w16(in[0] - in[4 * st]) * (1 << kConstBits);
  const int t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
  const int a0 = in[7 * st], a1 = in[5 * st], a2 = in[3 * st], a3 = in[st];
  const int y3 = jpeg_w16(a0 + a2), y4 = jpeg_w16(a1 + a3);
  const int z3p = y3 * (FIX_1_175875602 - FIX_1_961570560) + y4 * FIX_1_175875602;
  const int z4p = y3 * FIX_1_175875602 + y4 * (FIX_1_175875602 - FIX_0_390180644);
  const int b0 = a0 * (FIX_0_298631336 - FIX_0_899976223) - a3 * FIX_0_899976223 + z3p;
  const int b3 = -a0 * FIX_0_899976223 + a3 * (FIX_1_501321110 - FIX_0_899976223) + z4p;
  const int b1 = a1 * (FIX_2_053119869 - FIX_2_562915447) - a2 * FIX_2_562915447 + z4p;
  const int b2 = -a1 * FIX_2_562915447 + a2 * (FIX_3_072711026 - FIX_2_562915447) + z3p;
  const int r = 1 << (shift - 1);
  o[0] = jpeg_sat16((t10 + b3 + r) >> shift); o[7] = jpeg_sat16((t10 - b3 + r) >> shift);
  o[1] = jpeg_sat16((t11 + b2 + r) >> shift); o[6] = jpeg_sat16((t11 - b2 + r) >> shift);
  o[2] = jpeg_sat16((t12 + b1 + r) >> shift); o[5] = jpeg_sat16((t12 - b1 + r) >> shift);
  o[3] = jpeg_sat16((t13 + b0 + r) >> shift); o[4] = jpeg_sat16((t13 - b0 + r) >> shift);
}

// the output byte: saturated to -128 .. 127, plus 128 (a saturating pack to signed bytes, then the centre added)
__device__ __forceinline__ unsigned jpeg_range_limit(int v) { return static_cast<unsigned>((v < -128 ? -128 : (v > 127 ? 127 : v)) + 128); }

// Index of the file holding item g of a batch-wide numbering where file i holds [first[i], first[i] + count[i]).
template <typename F>
__device__ __forceinline__ int jpeg_find_image(int n_images, long long g, F end_of) {
  int lo = 0, hi = n_images - 1;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (end_of(mid) > g) hi = mid; else lo = mid + 1;
  }
  return lo;
}

__global__ void __launch_bounds__(kIdctThreads) jpeg_idct_kernel(const tp_jpeg_image* __restrict__ images, int n_images,
                                                                  const tp_jpeg_tables* __restrict__ tables, uint8_t* ws,
                                                                  long long total_blocks) {
  __shared__ int sblk[kIdctThreads / 8][64];
  const long long g = static_cast<long long>(blockIdx.x) * (kIdctThreads / 8) + threadIdx.x / 8;
  const int r = threadIdx.x & 7;
  int* s = sblk[threadIdx.x / 8];
  if (g >= total_blocks) return;                  // whole 8-thread groups leave together; only __syncwarp below
  const int img = jpeg_find_image(n_images, g, [&](int i) { return images[i].block0 + images[i].n_blocks; });
  const tp_jpeg_image& im = images[img];
  long long local = g - im.block0, plane = im.plane_offset;
  int c = 0;
  for (; c < im.ncomp - 1; ++c) {
    const long long nb = static_cast<long long>(im.comp_bx[c]) * im.comp_by[c];
    if (local < nb) break;
    local -= nb;
    plane += nb * 64;
  }
  const int stride = im.comp_bx[c] * 8;
  const long long by = local / im.comp_bx[c], bx = local % im.comp_bx[c];
  // row r of coefficients, dequantised: the 16-bit product of the SIMD dequantisation
  const int4 raw = *reinterpret_cast<const int4*>(ws + im.coef_offset + (g - im.block0) * 128 + r * 16);
  const int16_t* cv = reinterpret_cast<const int16_t*>(&raw);
  const uint16_t* q = tables[img].quant[c] + r * 8;
#pragma unroll
  for (int j = 0; j < 8; ++j) s[r * 8 + j] = jpeg_w16(static_cast<int>(cv[j]) * static_cast<int>(q[j]));
  __syncwarp();
  int o[8];
  jpeg_idct_1d(s + r, 8, kConstBits - kPass1Bits, o);                 // pass 1: column r
#pragma unroll
  for (int j = 0; j < 8; ++j) s[j * 8 + r] = o[j];
  __syncwarp();
  jpeg_idct_1d(s + r * 8, 1, kConstBits + kPass1Bits + 3, o);         // pass 2: row r
  unsigned lo = 0, hi = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    lo |= jpeg_range_limit(o[j]) << (8 * j);
    hi |= jpeg_range_limit(o[j + 4]) << (8 * j);
  }
  *reinterpret_cast<uint2*>(ws + plane + (by * 8 + r) * stride + bx * 8) = make_uint2(lo, hi);
}

// ------------------------------------------------------------------------------------------------
// 4. upsampling + colour conversion: one thread per output pixel
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kColourThreads) jpeg_colour_kernel(const tp_jpeg_image* __restrict__ images, int n_images,
                                                                      const uint8_t* __restrict__ ws, uint8_t* __restrict__ out,
                                                                      long long total_pixels) {
  const long long g = static_cast<long long>(blockIdx.x) * kColourThreads + threadIdx.x;
  if (g >= total_pixels) return;
  const int img = jpeg_find_image(n_images, g, [&](int i) { return images[i].pixel0 + static_cast<long long>(images[i].h) * images[i].w; });
  const tp_jpeg_image& im = images[img];
  const long long p = g - im.pixel0;
  const int y = static_cast<int>(p / im.w), x = static_cast<int>(p % im.w);
  const uint8_t* P0 = ws + im.plane_offset;
  const int s0 = im.comp_bx[0] * 8;
  const int Y = P0[static_cast<long long>(y) * s0 + x];
  uint8_t* o = out + im.out_offset + p * 3;
  if (im.ncomp == 1) {
    o[0] = o[1] = o[2] = static_cast<uint8_t>(Y);
    return;
  }
  const int cs = im.comp_bx[1] * 8;
  const long long csize = static_cast<long long>(cs) * im.comp_by[1] * 8;
  const long long l0 = static_cast<long long>(im.comp_bx[0]) * im.comp_by[0] * 64;
  const int cw = (im.w + im.hs - 1) / im.hs, ch = (im.h + im.vs - 1) / im.vs;   // downsampled width / height of the chroma
  int cc[2];
  for (int k = 0; k < 2; ++k) {
    const uint8_t* P = P0 + l0 + k * csize;
    if (im.hs == 1 && im.vs == 1) {
      cc[k] = P[static_cast<long long>(y) * cs + x];
    } else if (cw <= 2) {                          // jinit_upsampler: fancy upsampling needs downsampled_width > 2
      cc[k] = P[static_cast<long long>(y / im.vs) * cs + x / im.hs];
    } else if (im.vs == 1) {                       // h2v1_fancy_upsample
      const int j = x >> 1;
      const uint8_t* row = P + static_cast<long long>(y) * cs;
      const int v = row[j];
      if ((x & 1) == 0) cc[k] = j == 0 ? v : (v * 3 + row[j - 1] + 1) >> 2;
      else cc[k] = j == cw - 1 ? v : (v * 3 + row[j + 1] + 2) >> 2;
    } else {                                       // h2v2_fancy_upsample, edge rows replicated as context
      const int i = y >> 1, j = x >> 1;
      const int near = (y & 1) ? (i + 1 < ch ? i + 1 : ch - 1) : (i > 0 ? i - 1 : 0);
      const uint8_t* r0 = P + static_cast<long long>(i) * cs;
      const uint8_t* r1 = P + static_cast<long long>(near) * cs;
      auto colsum = [&](int jj) { return r0[jj] * 3 + r1[jj]; };
      const int t = colsum(j);
      if ((x & 1) == 0) cc[k] = j == 0 ? (t * 4 + 8) >> 4 : (t * 3 + colsum(j - 1) + 8) >> 4;
      else cc[k] = j == cw - 1 ? (t * 4 + 7) >> 4 : (t * 3 + colsum(j + 1) + 7) >> 4;
    }
  }
  // ycc_rgb_convert: SCALEBITS 16, FIX(1.40200) = 91881, FIX(1.77200) = 116130, FIX(0.71414) = 46802, FIX(0.34414) = 22554
  const int cb = cc[0] - 128, cr = cc[1] - 128;
  const int R = Y + ((91881 * cr + 32768) >> 16);
  const int G = Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16);
  const int B = Y + ((116130 * cb + 32768) >> 16);
  o[0] = static_cast<uint8_t>(R < 0 ? 0 : (R > 255 ? 255 : R));
  o[1] = static_cast<uint8_t>(G < 0 ? 0 : (G > 255 ? 255 : G));
  o[2] = static_cast<uint8_t>(B < 0 ? 0 : (B > 255 ? 255 : B));
}

}  // namespace tpjpeg
