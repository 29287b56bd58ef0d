/* Plain-C99 consumer of include/tokenpacker_b200_layers.h, linked against libtokenpacker_b200.so: every entry point it declares
 * resolves at link time, and argument validation runs without a GPU.  Built and run by
 * tests/test_hidden_states_host.py::test_plain_c_consumer_of_the_layers_header. */
#include <stdio.h>
#include <string.h>

#include "tokenpacker_b200_layers.h"

int main(void) {
  /* taking the address of every entry point makes the link fail if one is declared but not exported */
  const void* entry[] = {(const void*)&tp_forward_train_layers, (const void*)&tp_backward_layers, (const void*)&tp_forward_layers_packed};
  size_t i;
  for (i = 0; i < sizeof(entry) / sizeof(entry[0]); ++i)
    if (entry[i] == NULL) return 2;
  if (tp_abi_version() != TP_ABI_VERSION) return 3;
  {
    /* refused before any CUDA call: never dereferenced */
    static char buf[64] __attribute__((aligned(16)));
    void* p = buf;
    const int64_t cs = 577 * 1024;
    tp_weights w, g;
    void** fw = (void**)&w;
    void** fg = (void**)&g;
    const void* layers[4] = {p, p, p, p};
    const void* no_layer[4] = {p, p, NULL, p};
    void* d_layers[4] = {NULL, NULL, NULL, p};
    for (i = 0; i < sizeof(tp_weights) / sizeof(void*); ++i) {
      fw[i] = p;
      fg[i] = p;
    }
    /* a NULL layer */
    if (tp_forward_train_layers(&w, p, no_layer, 1, cs, 2, 4096, p, p, 1, NULL) != TP_ERR_INVALID_ARGUMENT) return 4;
    /* 5 does not divide 24 */
    if (tp_forward_train_layers(&w, p, layers, 1, cs, 5, 4096, p, p, 1, NULL) != TP_ERR_BAD_SCALE_FACTOR) return 5;
    /* layer gradients without the packed weights they read [W_k0; W_v0] from */
    if (tp_backward_layers(&w, NULL, layers, cs, 1, 2, 4096, p, p, &g, d_layers, cs, p, 1, NULL) != TP_ERR_INVALID_ARGUMENT) return 6;
    /* a gradient crop stride that is not a whole number of 1024-channel rows */
    if (tp_backward_layers(&w, p, layers, cs, 1, 2, 4096, p, p, &g, d_layers, cs + 8, p, 1, NULL) != TP_ERR_INVALID_ARGUMENT) return 7;
    /* a crop stride shorter than 576 rows */
    if (tp_forward_layers_packed(p, layers, 1, 575 * 1024, 2, 4096, p, 0, p, 1, NULL) != TP_ERR_INVALID_ARGUMENT) return 8;
  }
  printf("abi layers ok: %u entry points\n", (unsigned)(sizeof(entry) / sizeof(entry[0])));
  return 0;
}
