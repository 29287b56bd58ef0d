/* tokenpacker_b200 — PNG decoding on the GPU, byte for byte as PIL decodes (libtokenpacker_b200.so).
 *
 * Companion of tokenpacker_b200.h, whose conventions and status codes it follows; tokenpacker_b200.h (ABI version 2) and
 * tokenpacker_b200_jpeg.h are unchanged and this header only adds.
 *
 * What it computes, per file, is np.array(Image.open(f).convert('RGB')).  Supported: non-interlaced PNG at bit depth <= 8 in every
 * colour type: gray at 1, 2, 4 or 8 bits (1-bit gray becomes 0 / 255, 2- and 4-bit gray is scaled by 85 and 17), RGB, palette at 1, 2,
 * 4 or 8 bits (an index past the end of PLTE is black), gray + alpha and RGBA (alpha dropped).  tRNS, gAMA, iCCP and sRGB are not
 * applied, as convert('RGB') does not apply them.  Everything else is refused by the host plan, with a reason, before any launch.
 *
 * The decode of a batch is one host plan (tp_png_plan), one upload of [plan rows | palettes | zlib streams] and
 * 5 + ceil(log2(largest raw size)) kernel launches, a number that follows from the plan alone:
 *   1 speculate  per 256 bit offsets of a stream: test whether a valid dynamic deflate block header starts at each offset (every check
 *                zlib makes), and dry-decode the first TP_PNG_SLOTS candidates of the 256 to their end-of-block code
 *   2 chain      per file, one thread: follow the true blocks from the first one, taking a speculative result where a candidate sits at
 *                the block's start and dry-decoding the block there otherwise (stored and fixed blocks, missed candidates); a false
 *                candidate is never used, because only offsets the chain reaches are looked up
 *   3 decode     per true block: literals to their final place in the inflated bytes, every byte the position it copies from
 *   4 jump       ceil(log2(largest raw size)) launches of src[i] = src[src[i]]: every byte's source lies strictly earlier and a literal
 *                is its own source, so afterwards every byte points at the literal it copies
 *   5 gather     per byte: the literal's value
 *   6 finish     per file, one CTA: Adler-32 of the inflated bytes against the trailer, the five PNG filters undone as a wavefront
 *                (row r, column chunk c at step r + c), and the [h, w, 3] bytes
 * Every read stays inside the file's staged stream and workspace regions and every write inside the file's own; a malformed stream is
 * reported in the file's tp_png_status.
 */
#ifndef TOKENPACKER_B200_PNG_H_
#define TOKENPACKER_B200_PNG_H_

#include "tokenpacker_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* why the plan refuses a file (tp_png_image.reason); tp_png_reason_string gives the text */
enum {
  TP_PNG_SUPPORTED = 0,
  TP_PNG_NOT_PNG = 1,         /* no PNG signature */
  TP_PNG_MALFORMED = 2,       /* malformed or truncated chunks, an invalid IHDR or PLTE, no IDAT, IDAT chunks that are not
                                 consecutive, a palette image without PLTE */
  TP_PNG_BAD_CRC = 3,         /* a CRC mismatch on a chunk before the first IDAT (PIL checks those, and no IDAT CRC) */
  TP_PNG_DEPTH = 4,           /* 16-bit samples */
  TP_PNG_INTERLACED = 5,      /* Adam7 interlacing */
  TP_PNG_ANIMATED = 6,        /* APNG (an acTL chunk) */
  TP_PNG_ZLIB = 7,            /* a zlib header PIL's zlib refuses or that sets a preset dictionary, or a method other than deflate */
  TP_PNG_TOO_LARGE = 8,       /* more than TP_PNG_MAX_PIXELS pixels (PIL raises DecompressionBombError), or image data of
                                 TP_PNG_MAX_STREAM_BYTES or more */
  TP_PNG_METADATA = 9         /* an ancillary chunk PIL raises on: tRNS, gAMA, sRGB or pHYs too short, cHRM not whole 32-bit
                                 values, an iCCP / zTXt / iTXt compression method other than deflate or a payload that inflates
                                 past PngImagePlugin.MAX_TEXT_CHUNK, more text than MAX_TEXT_MEMORY */
};

/* what the GPU reports per file (tp_png_status.status) */
enum {
  TP_PNG_STATUS_OK = 0,
  TP_PNG_STATUS_BLOCK_TYPE = 1,   /* a block of type 3 */
  TP_PNG_STATUS_CODE_LENGTHS = 2, /* a dynamic block's code-length set is invalid (counts, code lengths or codes zlib refuses) */
  TP_PNG_STATUS_SYMBOL = 3,       /* an invalid literal / length or distance code */
  TP_PNG_STATUS_DISTANCE = 4,     /* a distance that reaches before the file's first byte or past the zlib window */
  TP_PNG_STATUS_STORED = 5,       /* a stored block whose LEN and NLEN disagree */
  TP_PNG_STATUS_TRUNCATED = 6,    /* the stream ends before its final block or its Adler-32 trailer */
  TP_PNG_STATUS_DATA_SIZE = 7,    /* the inflated data is not exactly h rows (PIL pads too little with zeros and ignores too much) */
  TP_PNG_STATUS_ADLER = 8,        /* Adler-32 mismatch */
  TP_PNG_STATUS_FILTER = 9        /* a row filter type above 4 */
};

#define TP_PNG_MAX_PIXELS 178956970ll          /* 2 * PIL's Image.MAX_IMAGE_PIXELS */
#define TP_PNG_MAX_STREAM_BYTES (1ll << 29)    /* streams are shorter, so that every bit offset, the end included, fits 32 bits */
#define TP_PNG_SPAN_BITS 256                   /* bit offsets per CTA of the speculative decode */
#define TP_PNG_SLOTS 4                         /* candidates of a span that are decoded speculatively */
#define TP_PNG_MIN_BLOCK_BITS 10               /* the shortest deflate block: a fixed block with only its end-of-block code */

/* One row of the plan.  stream_offset is into the staged bytes, out_offset into the output, the other offsets into the workspace;
 * all are bytes.  A refused file (reason != 0) has zero sizes and is skipped by every launch.  The workspace a file needs follows
 * from its row alone and holds for any stream:
 *   mask     uint32 [ceil(8 * stream_bytes / 32)]                         candidate bit per bit offset
 *   spec     tp_png_block [ceil(8 * stream_bytes / 256) * TP_PNG_SLOTS]   speculative results
 *   blocks   tp_png_block [block_capacity = 8 * stream_bytes / 10 + 2]    the true blocks, in stream order
 *   raw      uint8 [raw_bytes = h * (row_bytes + 1)]                      the inflated (filtered) rows
 *   src      uint32 [raw_bytes]                                           the position each inflated byte copies
 * each region 16-byte aligned: at most 19.5 * stream_bytes + 5 * raw_bytes + 200 bytes. */
typedef struct tp_png_image {
  int32_t reason;
  int32_t h, w;
  int32_t depth;                  /* bits per sample: 1, 2, 4 or 8 */
  int32_t color_type;             /* 0 gray, 2 RGB, 3 palette, 4 gray + alpha, 6 RGBA */
  int32_t channels;               /* samples per pixel: 1, 3, 1, 2, 4 */
  int32_t row_bytes;              /* bytes of a row after its filter-type byte */
  int32_t filter_bpp;             /* the byte distance the Sub, Avg and Paeth filters look back: max(1, bits per pixel / 8) */
  int32_t palette_entries;        /* PLTE entries (palette images), 0 otherwise */
  int32_t window;                 /* the zlib header's window in bytes, 256 .. 32768 */
  int64_t palette_offset;         /* uint8 [768] in the upload, relative to the palettes' start: RGB, unused entries zero */
  int64_t stream_offset, stream_bytes;  /* the zlib stream (header, deflate blocks, Adler-32): the IDAT payloads concatenated */
  int64_t raw_bytes;
  int64_t block_capacity;
  int64_t mask_offset, spec_offset, block_offset, raw_offset, src_offset;
  int64_t out_offset, pixel0;     /* uint8 [h][w][3] in the output; pixels of the files before it */
} tp_png_image;

/* A deflate block: bits are offsets in the file's zlib stream, out_offset / out_bytes bytes of the inflated data.  flags: bit 0
 * BFINAL, bits 1-2 BTYPE, bits 8.. a TP_PNG_STATUS_* code (0: the block decoded to its end-of-block code). */
typedef struct tp_png_block {
  uint32_t start_bit, end_bit;
  uint32_t out_offset, out_bytes;
  uint32_t flags;
} tp_png_block;

/* What the plan sums up over the batch. */
typedef struct tp_png_totals {
  int64_t staged_bytes;           /* zlib streams, each file's at a 16-byte-aligned offset */
  int64_t output_bytes;           /* sum of h * w * 3 */
  int64_t workspace_bytes;        /* = tp_png_workspace_bytes(images, n_images) */
  int64_t max_raw_bytes;          /* the largest raw_bytes of the batch: it sets the number of pointer-jumping launches */
  int64_t pixels;
} tp_png_totals;

/* Per file, written by the launches. */
typedef struct tp_png_status {
  int32_t status;                 /* TP_PNG_STATUS_* */
  int32_t blocks;                 /* true deflate blocks */
  int32_t serial_blocks;          /* true blocks the chain decoded itself: no speculative result sat at their start */
  int32_t candidates;             /* bit offsets that passed the dynamic-header test */
} tp_png_status;

/* Host only, no GPU.  Walks the chunks of every file, checks IHDR, PLTE and the zlib header, and lays out the batch.
 *   images    [n_images], always written: one row per file; reason says whether and why it is refused
 *   palettes  NULL, or [n_images * 768] bytes: each palette file's PLTE at its palette_offset, zero-padded
 *   staged    NULL, or at least totals->staged_bytes bytes: receives each supported file's concatenated IDAT payloads
 *   totals    always written
 * Returns TP_OK with refusals in the rows; TP_ERR_INVALID_ARGUMENT for NULL data / sizes / images / totals, n_images < 0, a NULL
 * file pointer with a non-zero size or a negative size. */
TP_API int tp_png_plan(const uint8_t* const* data, const int64_t* sizes, int64_t n_images, tp_png_image* images, uint8_t* palettes,
                       uint8_t* staged, tp_png_totals* totals);

/* The workspace the plan rows need, in bytes (the end of the last region); 0 for NULL images or n_images <= 0. */
TP_API size_t tp_png_workspace_bytes(const tp_png_image* images, int64_t n_images);

/* Text of a refusal reason ("" for TP_PNG_SUPPORTED, NULL for an unknown code). */
TP_API const char* tp_png_reason_string(int reason);

/* The launches on the caller's stream for the whole batch, no synchronisation.
 *   images_host        the plan rows on the host: they size the launches and the workspace check, and are not kept
 *   images_dev / palettes_dev / staged_dev   device copies of the plan rows, the palettes and the staged streams
 *   out                device, totals.output_bytes;  workspace: device, tp_png_workspace_bytes, 16-byte aligned
 *   status_dev         device, tp_png_status [n_images]
 * TP_ERR_INVALID_ARGUMENT for a NULL pointer, n_images < 0, a refused row or a misaligned workspace; TP_ERR_WORKSPACE_TOO_SMALL when
 * workspace_bytes is less than the rows need. */
TP_API int tp_png_decode_batch(const tp_png_image* images_host, const tp_png_image* images_dev, const uint8_t* palettes_dev,
                               const uint8_t* staged_dev, int64_t n_images, uint8_t* out, void* workspace, size_t workspace_bytes,
                               tp_png_status* status_dev, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TOKENPACKER_B200_PNG_H_ */
