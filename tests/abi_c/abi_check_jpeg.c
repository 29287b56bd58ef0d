/* Plain-C99 consumer of include/tokenpacker_b200_jpeg.h, linked against libtokenpacker_b200.so: every entry point it declares
 * resolves at link time, and the plan and argument validation run without a GPU.  Built and run by
 * tests/test_jpeg_host.py::test_plain_c_consumer_of_the_jpeg_header.  argv[1]: a JPEG file (16 x 24, 4:2:0, DRI of 2 MCUs). */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "tokenpacker_b200_jpeg.h"

int main(int argc, char** argv) {
  const void* entry[] = {(const void*)&tp_jpeg_plan, (const void*)&tp_jpeg_workspace_bytes, (const void*)&tp_jpeg_reason_string,
                         (const void*)&tp_jpeg_decode_batch};
  size_t i;
  for (i = 0; i < sizeof(entry) / sizeof(entry[0]); ++i)
    if (entry[i] == NULL) return 2;
  if (tp_abi_version() != TP_ABI_VERSION) return 3;
  if (sizeof(tp_jpeg_image) != 168 || sizeof(tp_jpeg_tables) != 8928 || sizeof(tp_jpeg_status) != 16) return 4;
  if (argc < 2) return 5;
  {
    FILE* f = fopen(argv[1], "rb");
    static uint8_t file[1 << 16];
    static const uint8_t not_jpeg[4] = {'G', 'I', 'F', '8'};
    const uint8_t* data[2];
    int64_t sizes[2];
    tp_jpeg_image im[2];
    tp_jpeg_tables* tab;
    uint8_t* staged;
    tp_jpeg_totals tot;
    if (f == NULL) return 6;
    sizes[0] = (int64_t)fread(file, 1, sizeof(file), f);
    fclose(f);
    data[0] = file;
    data[1] = not_jpeg;
    sizes[1] = 4;
    tab = (tp_jpeg_tables*)malloc(2 * sizeof(tp_jpeg_tables));
    staged = (uint8_t*)malloc((size_t)sizes[0] + 32);
    if (tab == NULL || staged == NULL) return 7;
    if (tp_jpeg_plan(data, sizes, 2, im, tab, staged, &tot) != TP_OK) return 8;
    if (im[0].reason != TP_JPEG_SUPPORTED || im[1].reason != TP_JPEG_NOT_JPEG) return 9;
    if (im[0].h != 16 || im[0].w != 24 || im[0].ncomp != 3 || im[0].hs != 2 || im[0].vs != 2 || im[0].blocks_per_mcu != 6) return 10;
    if (im[0].mcus_x != 2 || im[0].mcus_y != 1 || im[0].restart != 1 || im[0].n_segments != 2) return 11;
    if (im[0].n_blocks != 12 || tot.blocks != 12 || tot.pixels != 16 * 24 || tot.output_bytes != 16 * 24 * 3) return 12;
    if (tp_jpeg_workspace_bytes(im, 2) != (size_t)tot.workspace_bytes || tot.workspace_bytes <= 0) return 13;
    if (memcmp(staged, file + (sizes[0] - 2 - im[0].scan_bytes), (size_t)im[0].scan_bytes) != 0) return 14;  /* the scan, then EOI */
    if (strcmp(tp_jpeg_reason_string(TP_JPEG_PROGRESSIVE), "progressive JPEG") != 0 || tp_jpeg_reason_string(99) != NULL) return 15;
    /* refused before any CUDA call: never dereferenced */
    {
      tp_jpeg_status st[2];
      uint8_t out[1];
      if (tp_jpeg_plan(NULL, sizes, 2, im, NULL, NULL, &tot) != TP_ERR_INVALID_ARGUMENT) return 16;
      if (tp_jpeg_decode_batch(im, im, tab, staged, 2, out, staged, 1, st, NULL) != TP_ERR_INVALID_ARGUMENT) return 17;  /* a refused row */
      if (tp_jpeg_decode_batch(im, im, tab, staged, 1, out, staged + 16 - ((uintptr_t)staged & 15), 1, st, NULL) !=
          TP_ERR_WORKSPACE_TOO_SMALL) return 18;
      if (tp_jpeg_decode_batch(im, im, tab, staged, 0, out, staged, 1, st, NULL) != TP_OK) return 19;
    }
    free(tab);
    free(staged);
  }
  printf("abi jpeg ok: %u entry points\n", (unsigned)(sizeof(entry) / sizeof(entry[0])));
  return 0;
}
