/* Plain-C99 consumer of include/tokenpacker_b200_png.h, linked against libtokenpacker_b200.so: every entry point it declares
 * resolves at link time, and the plan and argument validation run without a GPU.  Built and run by
 * tests/test_png_host.py::test_plain_c_consumer_of_the_png_header.  argv[1]: a PNG file (24 x 16 RGB, one IDAT). */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "tokenpacker_b200_png.h"

int main(int argc, char** argv) {
  const void* entry[] = {(const void*)&tp_png_plan, (const void*)&tp_png_workspace_bytes, (const void*)&tp_png_reason_string,
                         (const void*)&tp_png_decode_batch};
  size_t i;
  for (i = 0; i < sizeof(entry) / sizeof(entry[0]); ++i)
    if (entry[i] == NULL) return 2;
  if (tp_abi_version() != TP_ABI_VERSION) return 3;
  if (sizeof(tp_png_image) != 136 || sizeof(tp_png_block) != 20 || sizeof(tp_png_status) != 16) return 4;
  if (argc < 2) return 5;
  {
    FILE* f = fopen(argv[1], "rb");
    static uint8_t file[1 << 16];
    static const uint8_t not_png[4] = {'G', 'I', 'F', '8'};
    const uint8_t* data[2];
    int64_t sizes[2];
    tp_png_image im[2];
    uint8_t pal[2 * 768];
    uint8_t* staged;
    tp_png_totals tot;
    if (f == NULL) return 6;
    sizes[0] = (int64_t)fread(file, 1, sizeof(file), f);
    fclose(f);
    data[0] = file;
    data[1] = not_png;
    sizes[1] = 4;
    staged = (uint8_t*)malloc((size_t)sizes[0] + 32);
    if (staged == NULL) return 7;
    if (tp_png_plan(data, sizes, 2, im, pal, staged, &tot) != TP_OK) return 8;
    if (im[0].reason != TP_PNG_SUPPORTED || im[1].reason != TP_PNG_NOT_PNG) return 9;
    if (im[0].h != 16 || im[0].w != 24 || im[0].color_type != 2 || im[0].row_bytes != 72 || im[0].raw_bytes != 16 * 73) return 10;
    if (tot.output_bytes != 16 * 24 * 3 || tot.pixels != 16 * 24 || tot.max_raw_bytes != 16 * 73) return 11;
    if (tp_png_workspace_bytes(im, 2) != (size_t)tot.workspace_bytes || tot.workspace_bytes <= 0) return 12;
    if (memcmp(staged, file + 8 + 25 + 8, (size_t)im[0].stream_bytes) != 0) return 13;   /* the IDAT payload after IHDR */
    if (strcmp(tp_png_reason_string(TP_PNG_INTERLACED), "interlaced PNG") != 0 || tp_png_reason_string(99) != NULL) return 14;
    /* refused before any CUDA call: never dereferenced */
    {
      tp_png_status st[2];
      uint8_t out[1];
      if (tp_png_plan(NULL, sizes, 2, im, NULL, NULL, &tot) != TP_ERR_INVALID_ARGUMENT) return 15;
      if (tp_png_decode_batch(im, im, pal, staged, 2, out, staged, 1, st, NULL) != TP_ERR_INVALID_ARGUMENT) return 16;  /* a refused row */
      if (tp_png_decode_batch(im, im, pal, staged, 1, out, staged + 16 - ((uintptr_t)staged & 15), 1, st, NULL) !=
          TP_ERR_WORKSPACE_TOO_SMALL) return 17;
      if (tp_png_decode_batch(im, im, pal, staged, 0, out, staged, 1, st, NULL) != TP_OK) return 18;
    }
    free(staged);
  }
  printf("abi png ok: %u entry points\n", (unsigned)(sizeof(entry) / sizeof(entry[0])));
  return 0;
}
