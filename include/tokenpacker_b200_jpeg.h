/* tokenpacker_b200 — baseline JPEG decoding on the GPU, bit for bit as PIL decodes (libtokenpacker_b200.so).
 *
 * Companion of tokenpacker_b200.h, whose conventions and status codes it follows; tokenpacker_b200.h (ABI version 2) is unchanged and
 * this header only adds.
 *
 * What it computes, per file, is np.array(Image.open(f).convert('RGB')): libjpeg-turbo's decode with PIL's defaults (JDCT_ISLOW,
 * fancy upsampling, no merged upsampling), integer arithmetic from the entropy decode to the colour conversion, so equal bit for bit.
 * Supported: baseline and extended sequential Huffman (SOF0 / SOF1), 8-bit samples, one scan of 1 component (grayscale, replicated
 * into RGB) or 3 interleaved YCbCr components with luma sampling 1x1, 2x1 or 2x2 and chroma 1x1, 8- and 16-bit quantisation tables,
 * any Huffman tables, restart intervals, any size.  Everything else is refused by the host plan, with a reason, before any launch.
 *
 * The decode of a batch is one host plan (tp_jpeg_plan), one upload of [plan rows | tables | staged scan bytes] and four launches:
 *   1 unstuff   per file: drop the 0x00 after each stuffed 0xFF, split the scan at RSTn into restart intervals, cut every interval
 *               into subsequences of TP_JPEG_SUBSEQUENCE_BYTES
 *   2 huffman   per file: decode every subsequence speculatively, then repeat rounds until each subsequence's entry state equals its
 *               predecessor's exit state (self-synchronisation); a scan places each subsequence's blocks; a second decode writes the
 *               coefficients in natural order; a segmented scan per component turns DC differences into DC values
 *   3 idct      per 8x8 block: dequantise and jpeg_idct_islow into component planes padded to whole MCUs
 *   4 colour    per output pixel: h2v1 / h2v2 fancy upsampling, ycc_rgb_convert, the [h, w, 3] bytes
 * A corrupt or truncated entropy-coded segment is reported in the file's tp_jpeg_status; the kernels read only the file's scan bytes.
 */
#ifndef TOKENPACKER_B200_JPEG_H_
#define TOKENPACKER_B200_JPEG_H_

#include "tokenpacker_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* why the plan refuses a file (tp_jpeg_image.reason); tp_jpeg_reason_string gives the text */
enum {
  TP_JPEG_SUPPORTED = 0,
  TP_JPEG_NOT_JPEG = 1,       /* no SOI marker */
  TP_JPEG_MALFORMED = 2,      /* malformed or truncated header */
  TP_JPEG_PROGRESSIVE = 3,    /* SOF2 / SOF6 */
  TP_JPEG_ARITHMETIC = 4,     /* arithmetic coding (SOF9 .. SOF15, DAC) */
  TP_JPEG_LOSSLESS = 5,       /* lossless or hierarchical (SOF3, SOF5, SOF7) */
  TP_JPEG_PRECISION = 6,      /* sample precision other than 8 bits */
  TP_JPEG_MULTI_SCAN = 7,     /* a sequential file with more than one scan */
  TP_JPEG_COLOUR = 8,         /* CMYK, YCCK or RGB-coded colour (3 components: no JFIF marker and either Adobe transform 0, or no
                                 Adobe marker and component ids 'R', 'G', 'B', as libjpeg decides), or a component count other than
                                 1 and 3 */
  TP_JPEG_SAMPLING = 9,       /* sampling factors other than 4:4:4, 4:2:2 and 4:2:0 */
  TP_JPEG_SCAN_ORDER = 10     /* the scan lists its components in another order than the frame (T.81 B.2.3 forbids it; libjpeg
                                 reads it) */
};

/* what the GPU reports per file (tp_jpeg_status.status) */
enum {
  TP_JPEG_STATUS_OK = 0,
  TP_JPEG_STATUS_ENTROPY = 1, /* the entropy-coded data is corrupt or truncated: an invalid code, a run past coefficient 63, bits
                                 read past the end of a restart interval, or an interval with too few blocks */
  TP_JPEG_STATUS_RESTART = 2  /* the scan has a different number of RSTn markers than its restart interval implies */
};

#define TP_JPEG_SUBSEQUENCE_BYTES 128   /* unit of the parallel Huffman decode */

/* One row of the plan.  Offsets are bytes: scan_offset into the staged bytes, out_offset into the output, the rest into the
 * workspace.  A refused file (reason != 0) has zero blocks, bytes and pixels and is skipped by every launch. */
typedef struct tp_jpeg_image {
  int32_t reason;
  int32_t h, w;
  int32_t ncomp;                  /* 1 or 3 */
  int32_t hs, vs;                 /* luma sampling factors (1, 1 for grayscale); chroma is 1 x 1 */
  int32_t mcus_x, mcus_y;
  int32_t blocks_per_mcu;         /* 1, 3, 4 or 6 */
  int32_t restart;                /* MCUs per restart interval (all of them without DRI) */
  int32_t n_segments;             /* restart intervals */
  int32_t comp_bx[3], comp_by[3]; /* component plane size in 8 x 8 blocks, whole MCUs */
  int32_t reserved;
  int64_t scan_offset, scan_bytes;/* the scan's entropy-coded bytes (markers included) */
  int64_t unstuffed_offset;       /* uint8 [scan_bytes]: the scan without stuffing and RSTn */
  int64_t seg_offset;             /* int64 [n_segments + 1]: byte starts of the restart intervals in the unstuffed bytes */
  int64_t sub_offset;             /* subsequence records, 64 bytes each */
  int64_t sub_capacity;           /* records reserved: ceil(scan_bytes / TP_JPEG_SUBSEQUENCE_BYTES) + n_segments */
  int64_t coef_offset;            /* int16 [n_blocks][64], natural order, component planes one after another, row-major */
  int64_t n_blocks, block0;       /* blocks of the file, and of the files before it in the batch */
  int64_t plane_offset;           /* uint8 component planes one after another, comp_bx * 8 wide and comp_by * 8 high */
  int64_t out_offset, pixel0;     /* uint8 [h][w][3] in the output; pixels of the files before it */
} tp_jpeg_image;

/* A Huffman table in the form the kernels decode from. */
typedef struct tp_jpeg_huff {
  uint16_t lookup[512];           /* next 9 bits -> (code length << 8) | symbol; 0 when the code is longer than 9 bits */
  int32_t maxcode[18];            /* [l]: largest code of length l, -1 when there is none (l = 1 .. 16) */
  int32_t valoff[18];             /* [l]: index in values of the code of length l minus that code */
  uint8_t values[256];
} tp_jpeg_huff;

/* The tables one file's scan uses, per scan component (component order of the frame). */
typedef struct tp_jpeg_tables {
  tp_jpeg_huff dc[3], ac[3];
  uint16_t quant[3][64];          /* natural order */
} tp_jpeg_tables;

/* What the plan sums up over the batch. */
typedef struct tp_jpeg_totals {
  int64_t staged_bytes;           /* scan bytes, each file's at a 16-byte-aligned offset */
  int64_t output_bytes;           /* sum of h * w * 3 */
  int64_t workspace_bytes;        /* = tp_jpeg_workspace_bytes(images, n_images) */
  int64_t blocks, pixels;
} tp_jpeg_totals;

/* Per file, written by launch 2 (status) and launch 1 (subsequences). */
typedef struct tp_jpeg_status {
  int32_t status;                 /* TP_JPEG_STATUS_* */
  int32_t sync_rounds;            /* decode rounds after the speculative one until every subsequence was synchronised */
  int32_t subsequences;
  int32_t reserved;
} tp_jpeg_status;

/* Host only, no GPU.  Parses the markers of every file: frame and scan headers, DQT, DHT, DRI, the scan's byte range, and lays out
 * the batch.  data[i] / sizes[i]: the files (any host memory).
 *   images   [n_images], always written: one row per file; reason says whether and why it is refused
 *   tables   [n_images] or NULL: the Huffman and quantisation tables of each supported file
 *   staged   NULL, or at least totals->staged_bytes bytes: receives each supported file's scan bytes at its scan_offset
 *   totals   always written
 * Returns TP_OK with refusals in the rows; TP_ERR_INVALID_ARGUMENT for NULL data / sizes / images / totals, n_images < 0, a NULL
 * file pointer with a non-zero size or a negative size. */
TP_API int tp_jpeg_plan(const uint8_t* const* data, const int64_t* sizes, int64_t n_images, tp_jpeg_image* images, tp_jpeg_tables* tables,
                        uint8_t* staged, tp_jpeg_totals* totals);

/* The workspace the plan rows need, in bytes (the end of the last region); 0 for NULL images or n_images <= 0. */
TP_API size_t tp_jpeg_workspace_bytes(const tp_jpeg_image* images, int64_t n_images);

/* Text of a refusal reason ("" for TP_JPEG_SUPPORTED, NULL for an unknown code). */
TP_API const char* tp_jpeg_reason_string(int reason);

/* Four launches on the caller's stream for the whole batch, no synchronisation.
 *   images_host        the plan rows on the host: they size the launches and the workspace check, and are not kept
 *   images_dev / tables_dev / staged_dev   device copies of the plan rows, the tables and the staged bytes
 *   out                device, totals.output_bytes;  workspace: device, tp_jpeg_workspace_bytes, 16-byte aligned
 *   status_dev         device, tp_jpeg_status [n_images]
 * TP_ERR_INVALID_ARGUMENT for a NULL pointer, n_images < 0, a refused row, a misaligned workspace or a grid that does not fit one
 * launch; TP_ERR_WORKSPACE_TOO_SMALL when workspace_bytes is less than the rows need. */
TP_API int tp_jpeg_decode_batch(const tp_jpeg_image* images_host, const tp_jpeg_image* images_dev, const tp_jpeg_tables* tables_dev,
                                const uint8_t* staged_dev, int64_t n_images, uint8_t* out, void* workspace, size_t workspace_bytes,
                                tp_jpeg_status* status_dev, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TOKENPACKER_B200_JPEG_H_ */
