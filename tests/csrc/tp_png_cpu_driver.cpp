// The PNG decoder's scalar core (tokenpacker_b200/csrc/tp_png.cuh) run on the CPU, stage by stage in the order the kernels run it:
// candidate test at every bit offset, speculative dry decode of each span's first candidates, the chain, the second decode of every
// true block, pointer jumping, gather, Adler-32 in parts, the unfilter wavefront and the conversion.  Each region is its own heap
// allocation of exactly the size the plan gives it, so that tests/test_png_sanitized_host.py, which builds this file with
// g++ -fsanitize=address,undefined, catches any access outside one.
//
// Usage: tp_png_cpu_driver FILE...; for each FILE writes FILE.out:
//   int32 reason, status, blocks, serial blocks, candidates; int64 raw bytes; the inflated bytes (when status is 0); the [h, w, 3] bytes
#include <stdio.h>
#include <stdlib.h>

#include <vector>

#include "../../tokenpacker_b200/csrc/tp_png.cuh"

using namespace tppng;

static std::vector<uint8_t> read_file(const char* path) {
  std::vector<uint8_t> d;
  FILE* f = fopen(path, "rb");
  if (!f) return d;
  uint8_t buf[65536];
  size_t n;
  while ((n = fread(buf, 1, sizeof(buf), f)) > 0) d.insert(d.end(), buf, buf + n);
  fclose(f);
  return d;
}

int main(int argc, char** argv) {
  for (int a = 1; a < argc; ++a) {
    const std::vector<uint8_t> file = read_file(argv[a]);
    Parsed p;
    int32_t head[5] = {0, 0, 0, 0, 0};
    int64_t raw_bytes = 0;
    std::vector<uint8_t> inflated, rgb;
    head[0] = file.empty() ? TP_PNG_NOT_PNG : parse(file.data(), static_cast<int64_t>(file.size()), &p);
    if (head[0] == TP_PNG_SUPPORTED) {
      std::vector<uint8_t> stream(static_cast<size_t>(p.idat_bytes));
      copy_idat(file.data(), static_cast<int64_t>(file.size()), stream.data());
      tp_png_image im;
      memset(&im, 0, sizeof(im));
      static const int kChannels[7] = {1, 0, 3, 1, 2, 0, 4};
      im.h = p.h; im.w = p.w; im.depth = p.depth; im.color_type = p.color_type; im.channels = kChannels[p.color_type];
      const int64_t bits = static_cast<int64_t>(im.channels) * im.depth;
      im.row_bytes = static_cast<int32_t>((static_cast<int64_t>(p.w) * bits + 7) / 8);
      im.filter_bpp = static_cast<int32_t>(bits >= 8 ? bits / 8 : 1);
      im.palette_entries = p.palette_entries;
      im.window = p.window;
      im.stream_bytes = p.idat_bytes;
      im.raw_bytes = raw_bytes = static_cast<int64_t>(p.h) * (im.row_bytes + 1);
      const int64_t nbits = 8 * im.stream_bytes;
      im.block_capacity = nbits / TP_PNG_MIN_BLOCK_BITS + 2;
      std::vector<uint32_t> mask(static_cast<size_t>((nbits + 31) / 32), 0);
      std::vector<tp_png_block> spec(static_cast<size_t>((nbits + TP_PNG_SPAN_BITS - 1) / TP_PNG_SPAN_BITS * TP_PNG_SLOTS));
      std::vector<tp_png_block> blocks(static_cast<size_t>(im.block_capacity));
      std::vector<uint8_t> raw(static_cast<size_t>(raw_bytes));
      std::vector<uint32_t> src(static_cast<size_t>(raw_bytes));
      Tables t;
      tp_png_status st = {0, 0, 0, 0};
      // 1. speculate
      for (int64_t span = 0; span * TP_PNG_SPAN_BITS < nbits; ++span) {
        int rank = 0;
        for (int64_t bit = span * TP_PNG_SPAN_BITS; bit < (span + 1) * TP_PNG_SPAN_BITS && bit < nbits; ++bit) {
          if (!(bit == 16 || (bit > 16 && is_dynamic_header(stream.data(), nbits, bit, t)))) continue;
          mask[bit >> 5] |= 1u << (bit & 31);
          ++st.candidates;
          if (rank < TP_PNG_SLOTS) dry_block(stream.data(), nbits, bit, static_cast<uint32_t>(raw_bytes), t, &spec[span * TP_PNG_SLOTS + rank]);
          ++rank;
        }
      }
      // 2. chain
      chain(im, stream.data(), mask.data(), spec.data(), blocks.data(), t, &st);
      // 3. decode, in reverse block order (the kernel runs them in any order)
      for (int k = st.status == 0 ? st.blocks - 1 : -1; k >= 0; --k) {
        const int s = decode_block(stream.data(), nbits, blocks[k], static_cast<uint32_t>(raw_bytes), static_cast<uint32_t>(im.window),
                                   raw.data(), src.data(), t);
        if (s > st.status) st.status = s;
      }
      if (st.status == 0) {
        // 4. jump, from the end down (so that each pass resolves one more step, as a synchronous round does), then gather
        int rounds = 0;
        while ((static_cast<int64_t>(1) << rounds) < raw_bytes) ++rounds;
        for (int r = 0; r < rounds; ++r)
          for (int64_t i = raw_bytes - 1; i >= 0; --i) jump(src.data(), static_cast<uint32_t>(i), static_cast<uint32_t>(raw_bytes));
        for (int64_t i = 0; i < raw_bytes; ++i) gather(raw.data(), src.data(), static_cast<uint32_t>(i), static_cast<uint32_t>(raw_bytes));
        inflated = raw;
        // 5. Adler-32 in 7 parts
        uint32_t A = 0, B = 0;
        const int64_t per = (raw_bytes + 6) / 7;
        for (int k = 0; k < 7; ++k) {
          const int64_t b0 = per * k < raw_bytes ? per * k : raw_bytes, b1 = b0 + per < raw_bytes ? b0 + per : raw_bytes;
          uint32_t a2, bb2;
          adler_part(raw.data() + b0, b1 - b0, &a2, &bb2);
          if (k == 0) { A = a2; B = bb2; } else adler_combine(&A, &B, a2, bb2, b1 - b0);
        }
        const uint8_t* tr = stream.data() + ((static_cast<int64_t>(blocks[st.blocks - 1].end_bit) + 7) >> 3);
        const uint32_t want = (static_cast<uint32_t>(tr[0]) << 24) | (static_cast<uint32_t>(tr[1]) << 16) | (static_cast<uint32_t>(tr[2]) << 8) | tr[3];
        if (adler_final(A, B, raw_bytes) != want) st.status = TP_PNG_STATUS_ADLER;
      }
      if (st.status == 0) {
        // 6. the wavefront with 256 column chunks, then the conversion
        const int rb = im.row_bytes, bpp = im.filter_bpp, threads = 256;
        int chunk = (rb + threads - 1) / threads;
        chunk = (chunk + bpp - 1) / bpp * bpp;
        const int active = (rb + chunk - 1) / chunk;
        for (int64_t step = 0; step < static_cast<int64_t>(im.h) + active - 1; ++step)
          for (int c = 0; c < active; ++c) {
            const int64_t r = step - c;
            if (r < 0 || r >= im.h) continue;
            uint8_t* row = raw.data() + r * (rb + 1);
            if (row[0] > 4) st.status = TP_PNG_STATUS_FILTER;
            else unfilter_span(row + 1, r > 0 ? row - rb : nullptr, c * chunk, (c + 1) * chunk < rb ? (c + 1) * chunk : rb, bpp, row[0]);
          }
      }
      if (st.status == 0) {
        rgb.resize(static_cast<size_t>(im.h) * im.w * 3);
        for (int64_t y = 0; y < im.h; ++y)
          for (int x = 0; x < im.w; ++x)
            convert_pixel(im, raw.data() + y * (im.row_bytes + 1) + 1, p.palette, x, rgb.data() + 3 * (y * im.w + x));
      } else {
        inflated.clear();
      }
      head[1] = st.status; head[2] = st.blocks; head[3] = st.serial_blocks; head[4] = st.candidates;
    }
    char path[4096];
    snprintf(path, sizeof(path), "%s.out", argv[a]);
    FILE* f = fopen(path, "wb");
    if (!f) return 1;
    fwrite(head, sizeof(head), 1, f);
    fwrite(&raw_bytes, sizeof(raw_bytes), 1, f);
    if (!inflated.empty()) fwrite(inflated.data(), 1, inflated.size(), f);
    if (!rgb.empty()) fwrite(rgb.data(), 1, rgb.size(), f);
    fclose(f);
  }
  return 0;
}
