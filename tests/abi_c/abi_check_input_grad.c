/* Plain-C99 consumer of include/tokenpacker_b200_input_grad.h, linked against libtokenpacker_b200.so: every entry point it declares
 * resolves at link time, and argument validation runs without a GPU.  Built and run by
 * tests/test_input_grad_host.py::test_plain_c_consumer_of_the_input_grad_header. */
#include <stdio.h>
#include <string.h>

#include "tokenpacker_b200_input_grad.h"

int main(void) {
  /* taking the address of every entry point makes the link fail if one is declared but not exported */
  const void* entry[] = {(const void*)&tp_backward_inputs};
  size_t i;
  for (i = 0; i < sizeof(entry) / sizeof(entry[0]); ++i)
    if (entry[i] == NULL) return 2;
  if (tp_abi_version() != TP_ABI_VERSION) return 3;
  {
    /* refused before any CUDA call: never dereferenced */
    static char buf[64] __attribute__((aligned(16)));
    void* p = buf;
    tp_weights w, g;
    void** fw = (void**)&w;
    void** fg = (void**)&g;
    for (i = 0; i < sizeof(tp_weights) / sizeof(void*); ++i) {
      fw[i] = p;
      fg[i] = p;
    }
    /* d_xm without the packed weights it reads [W_k0; W_v0] from */
    if (tp_backward_inputs(&w, NULL, p, 576 * 4096, 1, 2, 4096, p, p, &g, NULL, p, p, 1, NULL) != TP_ERR_INVALID_ARGUMENT) return 4;
    /* 5 does not divide 24 */
    if (tp_backward_inputs(&w, p, p, 576 * 4096, 1, 5, 4096, p, p, &g, p, p, p, 1, NULL) != TP_ERR_BAD_SCALE_FACTOR) return 5;
    /* no grad_out */
    if (tp_backward_inputs(&w, p, p, 576 * 4096, 1, 2, 4096, NULL, p, &g, p, p, p, 1, NULL) != TP_ERR_INVALID_ARGUMENT) return 6;
    /* a d_x0 that is not 16-byte aligned */
    if (tp_backward_inputs(&w, p, p, 576 * 4096, 1, 2, 4096, p, p, &g, buf + 2, p, p, 1, NULL) != TP_ERR_INVALID_ARGUMENT) return 7;
  }
  printf("abi input_grad ok: %u entry points\n", (unsigned)(sizeof(entry) / sizeof(entry[0])));
  return 0;
}
