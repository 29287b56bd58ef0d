// PNG decode (include/tokenpacker_b200_png.h): the scalar core.  The bit reader, the Huffman table builder, the block decoders, the
// per-thread bodies of every stage, the PNG filters and the unpack / palette rules are plain functions free of CUDA intrinsics, so
// that the kernels of tp_png.inl call them on the GPU and tests/test_png_sanitized_host.py compiles the very same functions with
// g++ -fsanitize=address,undefined.  The host-only part (chunk walk, CRC, IHDR / PLTE / zlib header checks) sits at the end.
//
// Every reader returns zeros past the end of its stream and flags it; every writer checks the extent of the region it writes; every
// loop is bounded by the bits it consumes or the bytes it produces.
#pragma once
#include <stdint.h>
#include <string.h>

#include "../../include/tokenpacker_b200_png.h"

#if defined(__CUDACC__)
#define TP_PNG_HD __host__ __device__ inline
#else
#define TP_PNG_HD inline
#endif

namespace tppng {

constexpr int kMaxCodeBits = 15;
constexpr uint32_t kAdlerMod = 65521;

// ------------------------------------------------------------------------------------------------
// bit reader: deflate's LSB-first bit order over bytes [0, nbits / 8)
// ------------------------------------------------------------------------------------------------
struct Bits {
  const uint8_t* p;
  int64_t nbits;    // 8 * bytes of the stream
  int64_t pos;      // next bit
  int over;         // a read went past the end (the bits read there were zeros)
};

// The next 25 or more bits (zeros past the end), without consuming them.
TP_PNG_HD uint32_t bits_peek(const Bits& b) {
  const int64_t byte = b.pos >> 3, nbytes = b.nbits >> 3;
  uint32_t v = 0;
  for (int k = 0; k < 4; ++k)
    if (byte + k < nbytes) v |= static_cast<uint32_t>(b.p[byte + k]) << (8 * k);
  return v >> (b.pos & 7);
}

TP_PNG_HD void bits_drop(Bits& b, int n) {
  if (b.pos + n > b.nbits) b.over = 1;
  b.pos += n;
}

// n <= 16 bits
TP_PNG_HD uint32_t bits_get(Bits& b, int n) {
  const uint32_t v = bits_peek(b) & ((1u << n) - 1u);
  bits_drop(b, n);
  return v;
}

// ------------------------------------------------------------------------------------------------
// canonical Huffman codes (RFC 1951 3.2.2) in counts-and-symbols form
// ------------------------------------------------------------------------------------------------
struct Huff {
  int16_t count[kMaxCodeBits + 1];   // codes of each length; count[0]: symbols without a code
  int16_t symbol[288];               // symbols ordered by code
};

// Builds h from the code lengths of n <= 288 symbols.  Returns 0 for a complete code (or no codes at all: count[0] == n), > 0 for an
// incomplete one and < 0 for an over-subscribed one.
TP_PNG_HD int huff_build(Huff& h, const uint8_t* length, int n) {
  for (int l = 0; l <= kMaxCodeBits; ++l) h.count[l] = 0;
  for (int s = 0; s < n; ++s) h.count[length[s] <= kMaxCodeBits ? length[s] : 0]++;
  if (h.count[0] == n) return 0;
  int left = 1;
  for (int l = 1; l <= kMaxCodeBits; ++l) {
    left <<= 1;
    left -= h.count[l];
    if (left < 0) return left;
  }
  int16_t offs[kMaxCodeBits + 1];
  offs[1] = 0;
  for (int l = 1; l < kMaxCodeBits; ++l) offs[l + 1] = static_cast<int16_t>(offs[l] + h.count[l]);
  for (int s = 0; s < n; ++s)
    if (length[s] != 0 && length[s] <= kMaxCodeBits) h.symbol[offs[length[s]]++] = static_cast<int16_t>(s);
  return left;
}

// zlib's rule for literal / length and distance codes: complete, or a single code of length 1 (or, for distances, no code at all).
TP_PNG_HD bool huff_acceptable(const Huff& h, int n, int built) {
  return built == 0 || (built > 0 && n - h.count[0] == 1 && h.count[1] == 1);
}

// The next symbol, or -1 when the bits match no code (an incomplete code).
TP_PNG_HD int huff_decode(Bits& b, const Huff& h) {
  const uint32_t v = bits_peek(b);
  int code = 0, first = 0, index = 0;
  for (int len = 1; len <= kMaxCodeBits; ++len) {
    code |= static_cast<int>((v >> (len - 1)) & 1u);
    const int count = h.count[len];
    if (code - count < first) {
      bits_drop(b, len);
      return h.symbol[index + (code - first)];
    }
    index += count;
    first += count;
    first <<= 1;
    code <<= 1;
  }
  return -1;
}

struct Tables {
  Huff lit, dist;
};

TP_PNG_HD void build_fixed(Tables& t) {
  uint8_t len[288];
  for (int s = 0; s < 288; ++s) len[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8;
  huff_build(t.lit, len, 288);
  for (int s = 0; s < 30; ++s) len[s] = 5;
  huff_build(t.dist, len, 30);     // symbols 30 and 31 have no code here, so they decode as invalid, as in zlib
}

// A dynamic block's header after BFINAL / BTYPE, with every check zlib makes.  Returns a TP_PNG_STATUS_* code.
TP_PNG_HD int read_dynamic(Bits& b, Tables& t) {
  const uint8_t order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
  const int nlen = static_cast<int>(bits_get(b, 5)) + 257, ndist = static_cast<int>(bits_get(b, 5)) + 1;
  const int ncode = static_cast<int>(bits_get(b, 4)) + 4;
  if (b.over) return TP_PNG_STATUS_TRUNCATED;
  if (nlen > 286 || ndist > 30) return TP_PNG_STATUS_CODE_LENGTHS;
  uint8_t len[286 + 30];
  for (int i = 0; i < 19; ++i) len[i] = 0;
  for (int i = 0; i < ncode; ++i) len[order[i]] = static_cast<uint8_t>(bits_get(b, 3));
  if (b.over) return TP_PNG_STATUS_TRUNCATED;
  Huff& cl = t.lit;                // the code-length code lives in the literal table until the literal code replaces it
  if (huff_build(cl, len, 19) != 0 || cl.count[0] == 19) return TP_PNG_STATUS_CODE_LENGTHS;
  int index = 0;
  while (index < nlen + ndist) {   // every pass writes at least one length
    const int sym = huff_decode(b, cl);
    if (b.over) return TP_PNG_STATUS_TRUNCATED;
    if (sym < 0) return TP_PNG_STATUS_CODE_LENGTHS;
    if (sym < 16) {
      len[index++] = static_cast<uint8_t>(sym);
      continue;
    }
    uint8_t value = 0;
    int rep;
    if (sym == 16) {
      if (index == 0) return TP_PNG_STATUS_CODE_LENGTHS;
      value = len[index - 1];
      rep = 3 + static_cast<int>(bits_get(b, 2));
    } else if (sym == 17) {
      rep = 3 + static_cast<int>(bits_get(b, 3));
    } else {
      rep = 11 + static_cast<int>(bits_get(b, 7));
    }
    if (b.over) return TP_PNG_STATUS_TRUNCATED;
    if (index + rep > nlen + ndist) return TP_PNG_STATUS_CODE_LENGTHS;
    for (int k = 0; k < rep; ++k) len[index++] = value;
  }
  if (len[256] == 0) return TP_PNG_STATUS_CODE_LENGTHS;
  if (!huff_acceptable(t.lit, nlen, huff_build(t.lit, len, nlen))) return TP_PNG_STATUS_CODE_LENGTHS;
  if (!huff_acceptable(t.dist, ndist, huff_build(t.dist, len + nlen, ndist))) return TP_PNG_STATUS_CODE_LENGTHS;
  return TP_PNG_STATUS_OK;
}

// ------------------------------------------------------------------------------------------------
// block decoders, generic over where the bytes go
// ------------------------------------------------------------------------------------------------

// Counts the bytes a block produces, up to limit (the speculative and the chain's dry decodes).
struct CountSink {
  uint32_t n, limit;
  TP_PNG_HD int literal(uint32_t) {
    if (n >= limit) return TP_PNG_STATUS_DATA_SIZE;
    ++n;
    return TP_PNG_STATUS_OK;
  }
  TP_PNG_HD int match(uint32_t len, uint32_t) {
    if (len > limit - n) return TP_PNG_STATUS_DATA_SIZE;
    n += len;
    return TP_PNG_STATUS_OK;
  }
  TP_PNG_HD int bytes(const uint8_t*, uint32_t len) { return match(len, 0); }
};

// Writes a block's literals to raw[pos] and, for every byte, the position it copies (itself for a literal) to src[pos].  pos runs from
// the block's out_offset to end; a distance past the bytes before pos or past the zlib window is a status, not a read.
struct WriteSink {
  uint8_t* raw;
  uint32_t* src;
  uint32_t pos, end, window;
  TP_PNG_HD int literal(uint32_t v) {
    if (pos >= end) return TP_PNG_STATUS_DATA_SIZE;
    raw[pos] = static_cast<uint8_t>(v);
    src[pos] = pos;
    ++pos;
    return TP_PNG_STATUS_OK;
  }
  TP_PNG_HD int match(uint32_t len, uint32_t dist) {
    if (len > end - pos) return TP_PNG_STATUS_DATA_SIZE;
    if (dist > pos || dist > window) return TP_PNG_STATUS_DISTANCE;
    for (uint32_t k = 0; k < len; ++k, ++pos) src[pos] = pos - dist;
    return TP_PNG_STATUS_OK;
  }
  TP_PNG_HD int bytes(const uint8_t* p, uint32_t len) {
    if (len > end - pos) return TP_PNG_STATUS_DATA_SIZE;
    for (uint32_t k = 0; k < len; ++k, ++pos) {
      raw[pos] = p[k];
      src[pos] = pos;
    }
    return TP_PNG_STATUS_OK;
  }
};

template <class Sink>
TP_PNG_HD int inflate_codes(Bits& b, const Tables& t, Sink& s) {
  const uint16_t lbase[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
  const uint8_t lextra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
  const uint16_t dbase[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073,
                              4097, 6145, 8193, 12289, 16385, 24577};
  const uint8_t dextra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
  for (;;) {                       // every pass consumes at least one bit, and reading past the end returns
    int sym = huff_decode(b, t.lit);
    if (b.over) return TP_PNG_STATUS_TRUNCATED;
    if (sym < 0) return TP_PNG_STATUS_SYMBOL;
    if (sym < 256) {
      const int st = s.literal(static_cast<uint32_t>(sym));
      if (st) return st;
      continue;
    }
    if (sym == 256) return TP_PNG_STATUS_OK;
    sym -= 257;
    if (sym >= 29) return TP_PNG_STATUS_SYMBOL;
    const uint32_t len = lbase[sym] + bits_get(b, lextra[sym]);
    const int ds = huff_decode(b, t.dist);
    if (b.over) return TP_PNG_STATUS_TRUNCATED;
    if (ds < 0 || ds >= 30) return TP_PNG_STATUS_SYMBOL;
    const uint32_t dist = dbase[ds] + bits_get(b, dextra[ds]);
    if (b.over) return TP_PNG_STATUS_TRUNCATED;
    const int st = s.match(len, dist);
    if (st) return st;
  }
}

// One block from b.pos: BFINAL, BTYPE and the block to its end.  Returns a TP_PNG_STATUS_* code; *final / *type are set once read.
template <class Sink>
TP_PNG_HD int inflate_block(Bits& b, Tables& t, Sink& s, int* final, int* type) {
  *final = static_cast<int>(bits_get(b, 1));
  *type = static_cast<int>(bits_get(b, 2));
  if (b.over) return TP_PNG_STATUS_TRUNCATED;
  if (*type == 0) {
    b.pos = (b.pos + 7) & ~static_cast<int64_t>(7);
    const uint32_t len = bits_get(b, 16), nlen = bits_get(b, 16);
    if (b.over) return TP_PNG_STATUS_TRUNCATED;
    if (len != (~nlen & 0xffffu)) return TP_PNG_STATUS_STORED;
    if (b.pos + 8 * static_cast<int64_t>(len) > b.nbits) {
      b.over = 1;
      return TP_PNG_STATUS_TRUNCATED;
    }
    const int st = s.bytes(b.p + (b.pos >> 3), len);
    b.pos += 8 * static_cast<int64_t>(len);
    return st;
  }
  if (*type == 1) {
    build_fixed(t);
  } else if (*type == 2) {
    const int st = read_dynamic(b, t);
    if (st) return st;
  } else {
    return TP_PNG_STATUS_BLOCK_TYPE;
  }
  return inflate_codes(b, t, s);
}

// ------------------------------------------------------------------------------------------------
// the per-thread bodies of the stages
// ------------------------------------------------------------------------------------------------

// Stage 1, test: does a dynamic block header that zlib accepts start at bit?
TP_PNG_HD bool is_dynamic_header(const uint8_t* stream, int64_t nbits, int64_t bit, Tables& t) {
  Bits b{stream, nbits, bit, 0};
  bits_get(b, 1);
  if (bits_get(b, 2) != 2 || b.over) return false;
  return read_dynamic(b, t) == TP_PNG_STATUS_OK;
}

// Stages 1 and 2, dry decode: the block at bit to its end-of-block code, producing at most limit bytes.  Writes only *r.
TP_PNG_HD void dry_block(const uint8_t* stream, int64_t nbits, int64_t bit, uint32_t limit, Tables& t, tp_png_block* r) {
  Bits b{stream, nbits, bit, 0};
  CountSink s{0, limit};
  int final = 0, type = 0;
  const int st = inflate_block(b, t, s, &final, &type);
  r->start_bit = static_cast<uint32_t>(bit);
  r->end_bit = static_cast<uint32_t>(b.pos < nbits ? b.pos : nbits);
  r->out_offset = 0;
  r->out_bytes = s.n;
  r->flags = static_cast<uint32_t>(final) | (static_cast<uint32_t>(type) << 1) | (static_cast<uint32_t>(st) << 8);
}

TP_PNG_HD int popc32(uint32_t x) {
  x = x - ((x >> 1) & 0x55555555u);
  x = (x & 0x33333333u) + ((x >> 2) & 0x33333333u);
  x = (x + (x >> 4)) & 0x0f0f0f0fu;
  return static_cast<int>((x * 0x01010101u) >> 24);
}

// Rank of candidate bit among the candidates of its span (the speculative slot it was decoded into when the rank is below
// TP_PNG_SLOTS), or -1 when bit is not a candidate.
TP_PNG_HD int candidate_rank(const uint32_t* mask, int64_t bit) {
  const int64_t w = bit >> 5;
  if (((mask[w] >> (bit & 31)) & 1u) == 0) return -1;
  int rank = popc32(mask[w] & ((1u << (bit & 31)) - 1u));
  for (int64_t k = (bit / TP_PNG_SPAN_BITS) * (TP_PNG_SPAN_BITS / 32); k < w; ++k) rank += popc32(mask[k]);
  return rank;
}

// Stage 3, one thread per file: the true blocks from the first one, each either taken from its speculative slot or dry-decoded here.
// Writes blocks [0, status->blocks) and the status row's status, blocks and serial_blocks.
TP_PNG_HD void chain(const tp_png_image& im, const uint8_t* stream, const uint32_t* mask, const tp_png_block* spec, tp_png_block* blocks,
                     Tables& t, tp_png_status* status) {
  const int64_t nbits = 8 * im.stream_bytes;
  const uint32_t raw = static_cast<uint32_t>(im.raw_bytes);
  int64_t pos = 16;                // after the zlib header
  uint32_t out = 0;
  int64_t nb = 0;
  int serial = 0, st = TP_PNG_STATUS_OK, final = 0;
  while (!final) {
    if (nb >= im.block_capacity || pos >= nbits) {   // every block takes at least TP_PNG_MIN_BLOCK_BITS bits
      st = TP_PNG_STATUS_TRUNCATED;
      break;
    }
    tp_png_block r;
    const int rank = candidate_rank(mask, pos);
    if (rank >= 0 && rank < TP_PNG_SLOTS && spec[(pos / TP_PNG_SPAN_BITS) * TP_PNG_SLOTS + rank].start_bit == static_cast<uint32_t>(pos)) {
      r = spec[(pos / TP_PNG_SPAN_BITS) * TP_PNG_SLOTS + rank];
    } else {
      dry_block(stream, nbits, pos, raw - out, t, &r);
      ++serial;
    }
    st = static_cast<int>(r.flags >> 8);
    if (st == TP_PNG_STATUS_OK && r.out_bytes > raw - out) st = TP_PNG_STATUS_DATA_SIZE;
    if (st != TP_PNG_STATUS_OK) break;
    r.out_offset = out;
    blocks[nb++] = r;
    out += r.out_bytes;
    pos = r.end_bit;
    final = static_cast<int>(r.flags & 1u);
  }
  if (st == TP_PNG_STATUS_OK && ((pos + 7) >> 3) + 4 > im.stream_bytes) st = TP_PNG_STATUS_TRUNCATED;   // the Adler-32 trailer
  if (st == TP_PNG_STATUS_OK && out != raw) st = TP_PNG_STATUS_DATA_SIZE;
  status->status = st;
  status->blocks = static_cast<int32_t>(nb);
  status->serial_blocks = serial;
}

// Stage 4, one thread per true block: the block again, literals into raw and every byte's source into src.
TP_PNG_HD int decode_block(const uint8_t* stream, int64_t nbits, const tp_png_block& blk, uint32_t raw_bytes, uint32_t window,
                           uint8_t* raw, uint32_t* src, Tables& t) {
  Bits b{stream, nbits, static_cast<int64_t>(blk.start_bit), 0};
  const uint32_t end = blk.out_bytes <= raw_bytes && blk.out_offset <= raw_bytes - blk.out_bytes ? blk.out_offset + blk.out_bytes : raw_bytes;
  WriteSink s{raw, src, blk.out_offset < raw_bytes ? blk.out_offset : raw_bytes, end, window};
  int final = 0, type = 0;
  const int st = inflate_block(b, t, s, &final, &type);
  if (st) return st;
  return s.pos == end ? TP_PNG_STATUS_OK : TP_PNG_STATUS_DATA_SIZE;
}

// Stage 5, one step of pointer jumping for byte i of n: src[i] = src[src[i]].  Sources lie strictly earlier; a literal is its own.
TP_PNG_HD void jump(uint32_t* src, uint32_t i, uint32_t n) {
  const uint32_t p = src[i];
  if (p >= i || p >= n) return;
  const uint32_t q = src[p];
  if (q < p) src[i] = q;
}

// Gather: byte i takes the value of the literal its resolved source points at.
TP_PNG_HD void gather(uint8_t* raw, const uint32_t* src, uint32_t i, uint32_t n) {
  const uint32_t p = src[i];
  if (p < i && p < n) raw[i] = raw[p];
}

// Adler-32 as a combinable reduction: a part of m bytes is (A, B) = (sum d_j, sum (m - j) d_j) mod 65521.
TP_PNG_HD void adler_part(const uint8_t* p, int64_t m, uint32_t* A, uint32_t* B) {
  uint32_t a = 0, b = 0;
  for (int64_t j = 0; j < m; ++j) {
    a += p[j];
    if (a >= kAdlerMod) a -= kAdlerMod;
    b += a;
    if (b >= kAdlerMod) b -= kAdlerMod;
  }
  *A = a;
  *B = b;
}

// (A, B) of x followed by y, where y has my bytes
TP_PNG_HD void adler_combine(uint32_t* A, uint32_t* B, uint32_t Ay, uint32_t By, int64_t my) {
  const uint64_t m = static_cast<uint64_t>(my) % kAdlerMod;
  *B = static_cast<uint32_t>((static_cast<uint64_t>(*B) + m * *A + By) % kAdlerMod);
  *A = static_cast<uint32_t>((static_cast<uint64_t>(*A) + Ay) % kAdlerMod);
}

// The Adler-32 of n bytes whose parts combine to (A, B).
TP_PNG_HD uint32_t adler_final(uint32_t A, uint32_t B, int64_t n) {
  const uint32_t a = (1u + A) % kAdlerMod;
  const uint32_t b = static_cast<uint32_t>((static_cast<uint64_t>(n) % kAdlerMod + B) % kAdlerMod);
  return (b << 16) | a;
}

TP_PNG_HD int paeth(int a, int b, int c) {
  const int p = a + b - c;
  const int pa = p > a ? p - a : a - p, pb = p > b ? p - b : b - p, pc = p > c ? p - c : c - p;
  return pa <= pb && pa <= pc ? a : pb <= pc ? b : c;
}

// Stage 6, unfilter bytes [begin, end) of a row (after its filter-type byte) in place.  prev: the row above, already unfiltered, or
// NULL for the first row.  The bytes of this row left of begin must be unfiltered already.  type <= 4.
TP_PNG_HD void unfilter_span(uint8_t* row, const uint8_t* prev, int begin, int end, int bpp, int type) {
  for (int j = begin; j < end; ++j) {
    const int a = j >= bpp ? row[j - bpp] : 0;
    const int b = prev ? prev[j] : 0;
    const int c = prev && j >= bpp ? prev[j - bpp] : 0;
    int v = row[j];
    if (type == 1) v += a;
    else if (type == 2) v += b;
    else if (type == 3) v += (a + b) >> 1;
    else if (type == 4) v += paeth(a, b, c);
    row[j] = static_cast<uint8_t>(v);
  }
}

// Sample x of an unfiltered row at depth < 8 bits, the first sample in the high bits of a byte.
TP_PNG_HD int sub_byte_sample(const uint8_t* row, int x, int depth) {
  const int64_t bit = static_cast<int64_t>(x) * depth;
  return (row[bit >> 3] >> (8 - depth - (bit & 7))) & ((1 << depth) - 1);
}

// Pixel x of an unfiltered row as convert('RGB') gives it: gray replicated (1-bit to 0 / 255, 2- and 4-bit scaled by 85 and 17),
// palette looked up (black past the end of PLTE), alpha dropped.
TP_PNG_HD void convert_pixel(const tp_png_image& im, const uint8_t* row, const uint8_t* palette, int x, uint8_t* rgb) {
  int r, g, b;
  if (im.color_type == 3) {
    const int i = im.depth == 8 ? row[x] : sub_byte_sample(row, x, im.depth);
    if (i < im.palette_entries) { r = palette[3 * i]; g = palette[3 * i + 1]; b = palette[3 * i + 2]; }
    else { r = g = b = 0; }
  } else if (im.color_type == 2 || im.color_type == 6) {
    const uint8_t* p = row + static_cast<int64_t>(x) * im.channels;
    r = p[0]; g = p[1]; b = p[2];
  } else {
    int v;
    if (im.depth == 8) v = row[static_cast<int64_t>(x) * im.channels];
    else {
      v = sub_byte_sample(row, x, im.depth);
      v = im.depth == 1 ? v * 255 : im.depth == 2 ? v * 85 : v * 17;
    }
    r = g = b = v;
  }
  rgb[0] = static_cast<uint8_t>(r);
  rgb[1] = static_cast<uint8_t>(g);
  rgb[2] = static_cast<uint8_t>(b);
}

// ------------------------------------------------------------------------------------------------
// host only: the file's chunks
// ------------------------------------------------------------------------------------------------
inline uint32_t be32(const uint8_t* p) {
  return (static_cast<uint32_t>(p[0]) << 24) | (static_cast<uint32_t>(p[1]) << 16) | (static_cast<uint32_t>(p[2]) << 8) | p[3];
}

inline uint32_t crc32(const uint8_t* p, int64_t n, uint32_t crc) {
  static const struct Table {
    uint32_t v[256];
    Table() {
      for (uint32_t i = 0; i < 256; ++i) {
        uint32_t c = i;
        for (int k = 0; k < 8; ++k) c = (c >> 1) ^ (0xEDB88320u & (0u - (c & 1u)));
        v[i] = c;
      }
    }
  } table;
  crc = ~crc;
  for (int64_t i = 0; i < n; ++i) crc = table.v[(crc ^ p[i]) & 0xffu] ^ (crc >> 8);
  return ~crc;
}

// Bytes a zlib stream inflates to, stopping at limit (returns limit when it reaches it); 0 for a stream zlib reports an error on
// first.  PIL inflates iCCP, zTXt and iTXt payloads and raises when one exceeds PngImagePlugin.MAX_TEXT_CHUNK.
inline int64_t zlib_inflated_size(const uint8_t* p, int64_t n, uint32_t limit) {
  if (n < 2 || (p[0] & 15) != 8 || (p[0] >> 4) > 7 || ((p[0] << 8) | p[1]) % 31 != 0 || (p[1] & 32)) return 0;
  Tables t;
  int64_t pos = 16;
  uint32_t out = 0;
  for (;;) {                       // every block consumes bits, and the decode stops at the stream's end
    tp_png_block r;
    dry_block(p, 8 * n, pos, limit - out, t, &r);
    const int st = static_cast<int>(r.flags >> 8);
    if (st == TP_PNG_STATUS_DATA_SIZE) return limit;
    if (st != TP_PNG_STATUS_OK) return 0;
    out += r.out_bytes;
    if (r.flags & 1u) return out;
    pos = r.end_bit;
  }
}

struct Parsed {
  int w = 0, h = 0, depth = 0, color_type = 0;
  int palette_entries = 0;
  uint8_t palette[768];
  int window = 0;
  int64_t idat_bytes = 0;
};

constexpr int64_t kMaxTextChunk = 1 << 20;        // PngImagePlugin.MAX_TEXT_CHUNK
constexpr int64_t kMaxTextMemory = 64 << 20;      // PngImagePlugin.MAX_TEXT_MEMORY

inline bool chunk_type_is_word(const uint8_t* t) {
  for (int k = 0; k < 4; ++k) {
    const uint8_t c = t[k];
    if (!((c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') || (c >= '0' && c <= '9') || c == '_')) return false;
  }
  return true;
}

// The ancillary chunks whose content PIL parses and raises on: too short, an unknown compression method, a compressed payload past
// MAX_TEXT_CHUNK, or more than MAX_TEXT_MEMORY of text.  True when PIL reads the chunk without raising.
inline bool ancillary_ok(const uint8_t* type, const uint8_t* s, int64_t len, int color_type, int depth, int64_t* text_memory) {
  const void* z;
  if (!memcmp(type, "tRNS", 4)) {
    if (color_type == 0 && depth <= 8) return len >= 2;
    if (color_type == 2) return len >= 6;
    return true;
  }
  if (!memcmp(type, "gAMA", 4)) return len >= 4;
  if (!memcmp(type, "cHRM", 4)) return len % 4 == 0;
  if (!memcmp(type, "sRGB", 4)) return len >= 1;
  if (!memcmp(type, "pHYs", 4)) return len >= 9;
  if (!memcmp(type, "tEXt", 4)) {
    *text_memory += len;
    return *text_memory <= kMaxTextMemory;
  }
  if (!memcmp(type, "iCCP", 4)) {
    z = memchr(s, 0, static_cast<size_t>(len));
    if (z == nullptr) return false;
    const int64_t i = static_cast<const uint8_t*>(z) - s;
    if (i + 1 >= len || s[i + 1] != 0) return false;
    return zlib_inflated_size(s + i + 2, len - i - 2, kMaxTextChunk) < kMaxTextChunk;
  }
  if (!memcmp(type, "zTXt", 4)) {
    z = memchr(s, 0, static_cast<size_t>(len));
    if (z == nullptr) return true;
    const int64_t i = static_cast<const uint8_t*>(z) - s;
    if (i + 1 >= len) return true;
    if (s[i + 1] != 0) return false;
    const int64_t m = zlib_inflated_size(s + i + 2, len - i - 2, kMaxTextChunk);
    *text_memory += m;
    return m < kMaxTextChunk && *text_memory <= kMaxTextMemory;
  }
  if (!memcmp(type, "iTXt", 4)) {
    z = memchr(s, 0, static_cast<size_t>(len));
    if (z == nullptr) return true;
    int64_t i = static_cast<const uint8_t*>(z) - s + 1;
    if (len - i < 2) return true;
    const int cf = s[i], cm = s[i + 1];
    i += 2;
    const void* z1 = memchr(s + i, 0, static_cast<size_t>(len - i));
    if (z1 == nullptr) return true;
    i = static_cast<const uint8_t*>(z1) - s + 1;
    const void* z2 = memchr(s + i, 0, static_cast<size_t>(len - i));
    if (z2 == nullptr) return true;
    i = static_cast<const uint8_t*>(z2) - s + 1;
    int64_t m = len - i;
    if (cf != 0 && cm == 0) {
      m = zlib_inflated_size(s + i, len - i, kMaxTextChunk);
      if (m >= kMaxTextChunk) return false;
    }
    *text_memory += m;
    return *text_memory <= kMaxTextMemory;
  }
  return true;
}

// Walks one file's chunks into p and returns the refusal reason.  The CRCs of the chunks before the image data are checked, as PIL
// checks them when it opens the file; IDAT CRCs are not (PIL does not read them).
inline int parse(const uint8_t* d, int64_t n, Parsed* p) {
  static const uint8_t sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1a, '\n'};
  if (n < 8 || memcmp(d, sig, 8) != 0) return TP_PNG_NOT_PNG;
  bool ihdr = false, idat_seen = false, idat_done = false;
  int64_t text_memory = 0, staged_at = 0;
  int interlace = 0;
  memset(p->palette, 0, sizeof(p->palette));
  for (int64_t i = 8; i < n;) {
    if (n - i < 12) return TP_PNG_MALFORMED;
    const uint32_t len = be32(d + i);
    const uint8_t* type = d + i + 4;
    const uint8_t* s = d + i + 8;
    if (len > 0x7fffffffu || static_cast<int64_t>(len) > n - i - 12 || !chunk_type_is_word(type)) return TP_PNG_MALFORMED;
    if (!memcmp(type, "IEND", 4)) break;
    const bool is_idat = !memcmp(type, "IDAT", 4);
    if (!ihdr && memcmp(type, "IHDR", 4) != 0) return TP_PNG_MALFORMED;
    if (!is_idat && !idat_seen && crc32(type, 4 + static_cast<int64_t>(len), 0) != be32(s + len)) return TP_PNG_BAD_CRC;
    if (is_idat) {
      if (idat_done) return TP_PNG_MALFORMED;
      staged_at += len;
      idat_seen = true;
    } else {
      if (idat_seen) idat_done = true;
      if (!memcmp(type, "IHDR", 4)) {
        if (ihdr || len != 13) return TP_PNG_MALFORMED;
        ihdr = true;
        const uint32_t w = be32(s), h = be32(s + 4);
        p->depth = s[8];
        p->color_type = s[9];
        interlace = s[12];
        if (w == 0 || h == 0 || w > 0x7fffffffu || h > 0x7fffffffu || s[10] != 0 || s[11] != 0) return TP_PNG_MALFORMED;
        const int ct = p->color_type, dp = p->depth;
        const bool valid = (ct == 0 && (dp == 1 || dp == 2 || dp == 4 || dp == 8 || dp == 16)) ||
                           (ct == 3 && (dp == 1 || dp == 2 || dp == 4 || dp == 8)) ||
                           ((ct == 2 || ct == 4 || ct == 6) && (dp == 8 || dp == 16));
        if (!valid) return TP_PNG_MALFORMED;
        p->w = static_cast<int>(w);
        p->h = static_cast<int>(h);
      } else if (!memcmp(type, "PLTE", 4)) {
        if (idat_seen || len == 0 || len % 3 != 0 || len > 768) return TP_PNG_MALFORMED;
        p->palette_entries = static_cast<int>(len / 3);
        memcpy(p->palette, s, len);
      } else if (!memcmp(type, "acTL", 4) || !memcmp(type, "fcTL", 4) || !memcmp(type, "fdAT", 4)) {
        return TP_PNG_ANIMATED;
      } else if (!ancillary_ok(type, s, len, p->color_type, p->depth, &text_memory)) {
        return TP_PNG_METADATA;
      }
    }
    i += 12 + static_cast<int64_t>(len);
  }
  if (!ihdr || !idat_seen) return TP_PNG_MALFORMED;
  if (p->depth == 16) return TP_PNG_DEPTH;
  if (interlace != 0) return TP_PNG_INTERLACED;
  if (p->color_type == 3 && p->palette_entries == 0) return TP_PNG_MALFORMED;
  if (p->color_type != 3) p->palette_entries = 0;
  if (static_cast<int64_t>(p->w) * p->h > TP_PNG_MAX_PIXELS || staged_at >= TP_PNG_MAX_STREAM_BYTES) return TP_PNG_TOO_LARGE;
  p->idat_bytes = staged_at;
  // the zlib header: deflate, a window of at most 32 KB, FCHECK, no preset dictionary
  if (staged_at < 2) return TP_PNG_MALFORMED;
  uint8_t zh[2];
  int64_t got = 0;
  for (int64_t i = 8; got < 2;) {  // the first two bytes of the IDAT payloads
    const uint32_t len = be32(d + i);
    if (!memcmp(d + i + 4, "IDAT", 4))
      for (uint32_t k = 0; k < len && got < 2; ++k) zh[got++] = d[i + 8 + k];
    i += 12 + static_cast<int64_t>(len);
  }
  if ((zh[0] & 15) != 8 || (zh[0] >> 4) > 7 || ((zh[0] << 8) | zh[1]) % 31 != 0 || (zh[1] & 32)) return TP_PNG_ZLIB;
  p->window = 1 << ((zh[0] >> 4) + 8);
  return TP_PNG_SUPPORTED;
}

// The IDAT payloads of a file parse() accepted, concatenated into staged (p->idat_bytes bytes).
inline void copy_idat(const uint8_t* d, int64_t n, uint8_t* staged) {
  for (int64_t i = 8; i + 12 <= n;) {
    const uint32_t len = be32(d + i);
    if (!memcmp(d + i + 4, "IEND", 4)) break;
    if (!memcmp(d + i + 4, "IDAT", 4)) {
      memcpy(staged, d + i + 8, len);
      staged += len;
    }
    i += 12 + static_cast<int64_t>(len);
  }
}

}  // namespace tppng
