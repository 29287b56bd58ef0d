// Test-only entry point into the JPEG decoder's stages (libtokenpacker_b200_jpeg_hooks.so, loaded by tests/test_jpeg_stages_gpu.py;
// never by the package): the product translation unit plus tpj_decode_stages, which runs tp_jpeg_decode_batch's launches up to one
// stage so that each stage's output can be read from the workspace.  Conventions as in include/tokenpacker_b200_jpeg.h.
#include "../../tokenpacker_b200/csrc/tp_api.cu"

extern "C" {

// tp_jpeg_decode_batch up to stage last_stage: 1 unstuff, 2 Huffman decode and DC prediction, 3 IDCT, 4 colour (all of it).
TP_API int tpj_decode_stages(const tp_jpeg_image* images_host, const tp_jpeg_image* images_dev, const tp_jpeg_tables* tables_dev,
                             const uint8_t* staged_dev, int64_t n_images, uint8_t* out, void* workspace, size_t workspace_bytes,
                             tp_jpeg_status* status_dev, int last_stage, void* stream) {
  if (last_stage < 1 || last_stage > 4) return TP_ERR_INVALID_ARGUMENT;
  return jpeg_decode_stages(images_host, images_dev, tables_dev, staged_dev, n_images, out, workspace, workspace_bytes, status_dev,
                            static_cast<cudaStream_t>(stream), last_stage);
}

// sizeof(JpegSub): the workspace's subsequence records
TP_API int tpj_subsequence_record_bytes(void) { return static_cast<int>(sizeof(tpjpeg::JpegSub)); }

}  // extern "C"
