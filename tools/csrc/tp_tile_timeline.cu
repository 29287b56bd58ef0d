// The product translation unit with the pair kernel's per-tile timeline: a measurement library of tools/bench_tile_timeline.py,
// which compiles it from a copy of the sources with the timeline added (its PATCHES); never loaded by the package or the tests.
// Every tp_* entry point behaves as in libtokenpacker_b200.so; while a buffer is set, every launch of tp_gemm2_kernel writes its
// tiles' timestamps there.
#include "../../tokenpacker_b200/csrc/tp_api.cu"

extern "C" {

// buf: nullptr (no timeline), or device memory of [grid][kTimelineTiles][kTimelineSlots] unsigned 64-bit values
TP_API int tpl_set_timeline(void* buf) {
  g_tile_timeline = static_cast<unsigned long long*>(buf);
  return TP_OK;
}

TP_API int tpl_timeline_shape(int64_t* out) {
  if (out == nullptr) return TP_ERR_INVALID_ARGUMENT;
  out[0] = kTimelineTiles;
  out[1] = kTimelineSlots;
  return TP_OK;
}

}  // extern "C"
