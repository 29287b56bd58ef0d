// Test-only entry point into the PNG decoder's stages (libtokenpacker_b200_png_hooks.so, loaded by tests/test_png_gpu.py;
// never by the package): the product translation unit plus tpp_decode_stages, which runs tp_png_decode_batch's launches up to one
// stage so that each stage's output can be read from the workspace.  Conventions as in include/tokenpacker_b200_png.h.
#include "../../tokenpacker_b200/csrc/tp_api.cu"

extern "C" {

// tp_png_decode_batch up to stage last_stage: 1 speculate, 2 chain, 3 decode, 4 jump and gather, 5 finish (all of it).
TP_API int tpp_decode_stages(const tp_png_image* images_host, const tp_png_image* images_dev, const uint8_t* palettes_dev,
                             const uint8_t* staged_dev, int64_t n_images, uint8_t* out, void* workspace, size_t workspace_bytes,
                             tp_png_status* status_dev, int last_stage, void* stream) {
  if (last_stage < 1 || last_stage > 5) return TP_ERR_INVALID_ARGUMENT;
  return png_decode_stages(images_host, images_dev, palettes_dev, staged_dev, n_images, out, workspace, workspace_bytes, status_dev,
                           static_cast<cudaStream_t>(stream), last_stage);
}

}  // extern "C"
