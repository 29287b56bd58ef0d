/* Plain-C99 consumer of include/tokenpacker_b200_hd_u8.h, linked against libtokenpacker_b200.so: every entry point it declares
 * resolves at link time, and argument validation runs without a GPU.  Built and run by
 * tests/test_hd_preprocess_host.py::test_plain_c_consumer_of_the_u8_header. */
#include <stdio.h>
#include <string.h>

#include "tokenpacker_b200_hd_u8.h"

int main(void) {
  /* taking the address of every entry point makes the link fail if one is declared but not exported */
  const void* entry[] = {(const void*)&tp_hd_preprocess_batch};
  size_t i;
  for (i = 0; i < sizeof(entry) / sizeof(entry[0]); ++i)
    if (entry[i] == NULL) return 2;
  if (tp_abi_version() != TP_ABI_VERSION) return 3;
  if (sizeof(tp_hd_u8_source) != 32) return 4;
  {
    /* refused before any CUDA call: never dereferenced */
    tp_hd_image im;
    tp_hd_u8_source src;
    int32_t table[3];
    float norm[768];
    float crop[1];
    memset(&im, 0, sizeof(im));
    memset(&src, 0, sizeof(src));
    memset(table, 0, sizeof(table));
    memset(norm, 0, sizeof(norm));
    memset(crop, 0, sizeof(crop));
    if (tp_hd_preprocess_batch(NULL, &src, table, 1, norm, 0, crop, NULL) != TP_ERR_INVALID_ARGUMENT) return 5;
    if (tp_hd_preprocess_batch(&im, NULL, table, 1, norm, 0, crop, NULL) != TP_ERR_INVALID_ARGUMENT) return 6;
    if (tp_hd_preprocess_batch(&im, &src, table, 1, norm, 2, crop, NULL) != TP_ERR_INVALID_ARGUMENT) return 7;
    if (tp_hd_preprocess_batch(&im, &src, table, -1, norm, 1, crop, NULL) != TP_ERR_INVALID_ARGUMENT) return 8;
    if (tp_hd_preprocess_batch(&im, &src, table, 0, norm, 1, crop, NULL) != TP_OK) return 9;
  }
  printf("abi hd_u8 ok: %u entry points\n", (unsigned)(sizeof(entry) / sizeof(entry[0])));
  return 0;
}
