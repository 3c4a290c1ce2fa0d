/*
 * rawspeed_b200.h -- C ABI of the H100-native RAW decompression engine.
 *
 * This is the drop-in boundary for rawspeed's per-pixel decode hot path.  The
 * reference (darktable-org/rawspeed) has no FFI layer; its seam is four C++
 * decompressor classes whose method bodies are the hot path.  Each entry point
 * below replaces one of those bodies (paths relative to
 * /root/reference/src/librawspeed):
 *
 *   rsb200_unpack_plan_create + rsb200_plan_run
 *       <- UncompressedDecompressor::readUncompressedRaw / decodePackedInt<Pump>
 *          decompressors/UncompressedDecompressor.cpp:188-200, 202-268
 *          (and AbstractDngDecompressor::decompressThread<1>,
 *           decompressors/AbstractDngDecompressor.cpp:54-110, one job per tile)
 *   rsb200_ljpeg_plan_create + rsb200_plan_run
 *       <- LJpegDecompressor::decode / decodeN / decodeRowN
 *          decompressors/LJpegDecompressor.cpp:184-370
 *          (and AbstractDngDecompressor::decompressThread<7>,
 *           decompressors/AbstractDngDecompressor.cpp:112-131: all tiles of a
 *           frame -- or of a batch of frames -- in one plan)
 *   rsb200_cr2_plan_create + rsb200_plan_run
 *       <- Cr2Decompressor<PrefixCodeDecoder<>>::decompress / decompressN_X_Y
 *          decompressors/Cr2DecompressorImpl.h:396-487
 *   rsb200_huff_table
 *       <- HuffmanCode<BaselineCodeTag> + PrefixCodeDecoder<>::setup
 *          codes/HuffmanCode.h:66-166, codes/PrefixCodeLUTDecoder.h:95-148
 *          (the DHT contents; the device LUT is built by the library)
 *
 * Everything the reference does *around* those bodies -- marker parsing,
 * geometry validation, exceptions, RawImage allocation -- stays on the host
 * (rawspeed_b200/csrc/host/, the C++ mirror of the reference classes, calls
 * this ABI).  Signatures are POD only: plain pointers and sizes, no C++/torch
 * types.  The caller owns every buffer it passes; the library owns its device
 * staging/scratch memory.
 *
 * There is NO CPU fallback: every entry point fails with RSB200_ERR_CUDA if no
 * CUDA device / kernel image is usable.
 *
 * Threading: a ctx/plan is single-use-at-a-time (like a reference decoder
 * instance, decoders/RawDecoder.h:39-43); different contexts may run
 * concurrently.
 */
#ifndef RAWSPEED_B200_H
#define RAWSPEED_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RSB200_ABI_VERSION 1

/* Status codes.  RDE/IOE map onto the reference's exception classes
 * (common/RawspeedException.h:33-95): the host shim turns them into
 * RawDecoderException / IOException. */
enum {
  RSB200_OK = 0,
  RSB200_ERR_RDE = 1,  /* -> RawDecoderException (e.g. "bad Huffman code") */
  RSB200_ERR_IOE = 2,  /* -> IOException (bit stream over-read)            */
  RSB200_ERR_CUDA = 3, /* CUDA failure; message in rsb200_last_error()     */
  RSB200_ERR_ARG = 4   /* malformed descriptor                             */
};

/* bitstreams/BitStreams.h:28-35 (enum class BitOrder), same values. */
enum { RSB200_LSB = 0, RSB200_MSB = 1, RSB200_MSB16 = 2, RSB200_MSB32 = 3 };

typedef struct rsb200_ctx rsb200_ctx;
typedef struct rsb200_plan rsb200_plan;

int rsb200_abi_version(void);

/* Bind a context to CUDA device `device` (one process per GPU). */
int rsb200_create(int device, rsb200_ctx** ctx);
void rsb200_destroy(rsb200_ctx* ctx);
/* Text of the last failure on this context ("" if none). */
const char* rsb200_last_error(const rsb200_ctx* ctx);
/* Number of kernels this context has launched so far (bench: gpu_launches). */
uint64_t rsb200_kernel_launches(const rsb200_ctx* ctx);
/* Name of the dominant kernel of a plan kind + its per-launch resource use. */
int rsb200_device_sm_count(const rsb200_ctx* ctx);

/* ------------------------------------------------------------------ */
/* K1: packed N-bit unpack.  One job = one strip/tile (one                */
/* UncompressedDecompressor instance).                                 */
/* ------------------------------------------------------------------ */
typedef struct {
  uint64_t in_offset;  /* byte offset of the strip inside the input buffer       */
  uint64_t in_size;    /* bytes of the strip (>= rows*in_pitch; bytes past it read
                          as 0, BitStreamer.h:100-131)                           */
  uint64_t out_offset; /* byte offset of image row 0 inside the output buffer;
                          even                                                   */
  int32_t out_pitch;   /* bytes between output rows (RawImageData::pitch); even  */
  int32_t row0;        /* first output row  (offset.y)                           */
  int32_t rows;        /* rows to decode    (min(h+oy, dim.y) - oy)              */
  int32_t samples;     /* samples per row   (size.x * cpp)                       */
  int32_t out_col0;    /* first output sample column: 0 for packed integers (the
                          reference ignores offset.x there,
                          UncompressedDecompressor.cpp:196); offset.x*cpp for the
                          16-bit LSB row-copy form (:255-264)                    */
  int32_t in_pitch;    /* bytes between input rows                               */
  int32_t bps;         /* 1..16                                                  */
  int32_t order;       /* RSB200_LSB/MSB/MSB16/MSB32                             */
} rsb200_unpack_job;

int rsb200_unpack_plan_create(rsb200_ctx* ctx, const rsb200_unpack_job* jobs,
                              int njobs, rsb200_plan** plan);

/* ------------------------------------------------------------------ */
/* K1b: the remaining UncompressedDecompressor forms (fixed layouts).   */
/*   decode8BitRaw<uncorrected>          UncompressedDecompressor.cpp:270-294 */
/*   decode12BitRawWithControl<e>        UncompressedDecompressor.cpp:299-359 */
/*   decode12BitRawUnpackedLeftAligned<e> UncompressedDecompressor.cpp:366-390 */
/*   decodePackedFP<Pump, Binary16/24>   UncompressedDecompressor.cpp:171-186 */
/*   32-bit float row copy               UncompressedDecompressor.cpp:214-224 */
/* ------------------------------------------------------------------ */
enum {
  RSB200_RAW_8BIT = 1,             /* out = in byte (uncorrectedRawValues, or no table) */
  RSB200_RAW_8BIT_TABLE = 2,       /* out = table[in byte] (RawImageDataU16::setWithLookUp,
                                      common/RawImage.h:335-353; the dither counter of
                                      decode8BitRaw starts at 0 and therefore stays 0, so
                                      the dithered form is table[2*v] exactly)           */
  RSB200_RAW_12BIT_CONTROL_BE = 3, /* 3 bytes -> 2 px, 1 control byte after every 10 px */
  RSB200_RAW_12BIT_CONTROL_LE = 4,
  RSB200_RAW_12BIT_LEFT_BE = 5,    /* 16-bit words, value = word >> 4                   */
  RSB200_RAW_12BIT_LEFT_LE = 6,
  RSB200_RAW_FP16_MSB = 7,         /* binary16 -> binary32 (common/FloatingPoint.h:116-160) */
  RSB200_RAW_FP16_LSB = 8,
  RSB200_RAW_FP24_MSB = 9,         /* binary24 -> binary32                              */
  RSB200_RAW_FP24_LSB = 10,
  RSB200_RAW_F32_COPY = 11         /* 32-bit rows copied as they are                    */
};

typedef struct {
  uint64_t in_offset;  /* byte offset of the strip inside the input buffer          */
  uint64_t in_size;    /* bytes of the strip (>= rows * in_pitch, checked)          */
  uint64_t out_offset; /* byte offset of image row 0 inside the output buffer; a
                          multiple of the output sample size (2, or 4 for 7-11)     */
  int32_t out_pitch;   /* bytes between output rows; a multiple of the sample size  */
  int32_t row0;        /* first output row                                          */
  int32_t rows;
  int32_t samples;     /* samples per row (w, or w*cpp for the float forms)         */
  int32_t out_col0;    /* first output sample column (0 for the integer forms;
                          offset.x for decodePackedFP, offset.x*cpp for the copy)   */
  int32_t in_pitch;    /* bytes between input rows (8-bit: w; control: perline;
                          left-aligned: 2w; float: inputPitchBytes)                 */
  int32_t format;      /* RSB200_RAW_*                                              */
  int32_t table;       /* RSB200_RAW_8BIT_TABLE: index into the plan's tables       */
} rsb200_raw_job;

/* `tables`: ntables x 65536 uint16 entries (TableLookUp::getTable content for the
 * non-dithered form; for a dithered table pass entries 2*v, see above), may be
 * NULL when no job uses RSB200_RAW_8BIT_TABLE.  Output samples are uint16 for
 * formats 1-6 and 32-bit for 7-11. */
int rsb200_raw_plan_create(rsb200_ctx* ctx, const rsb200_raw_job* jobs, int njobs,
                           const uint16_t* tables, int ntables, rsb200_plan** plan);

/* ------------------------------------------------------------------ */
/* K6: Sony ARW2 block codec (SURVEY 8(f)4).                            */
/*   SonyArw2Decompressor::decompressRow / decompress                   */
/*   decompressors/SonyArw2Decompressor.cpp:58-112, 114-148             */
/* ------------------------------------------------------------------ */
typedef struct {
  uint64_t in_offset;  /* first byte of the image's data: width*height bytes       */
  uint64_t out_offset; /* byte offset of image row 0; multiple of 16               */
  uint32_t out_pitch;  /* bytes between output rows; multiple of 16, >= 2*width    */
  uint32_t width;      /* multiple of 32, <= 9600                                  */
  uint32_t height;     /* <= 6376                                                  */
  int32_t table;       /* index into the plan's tables, -1 = image has no table    */
} rsb200_arw2_job;

/* `tables`: ntables tables in TableLookUp's storage layout (common/TableLookUp.cpp:
 * 48-85): dither == 0 -> 65536 uint16 each, dither != 0 -> 2*65536 uint16 each
 * (base, delta pairs).  Only entries of values <= 0xFFE are ever used (a value is
 * an 11-bit number << 1).  A block whose imax == imin makes rsb200_plan_results
 * report RSB200_ERR_RDE for its job (the reference throws "ARW2 invariant
 * failed, ..." for the row and gives up on the image).                          */
int rsb200_arw2_plan_create(rsb200_ctx* ctx, const rsb200_arw2_job* jobs, int njobs,
                            const uint16_t* tables, int ntables, int dither,
                            rsb200_plan** plan);

/* ------------------------------------------------------------------ */
/* K7: Panasonic RW2 block codecs V4 / V5 / V6 / V7 (SURVEY 8(f)4).     */
/*   PanasonicV4Decompressor::processBlock (+ ProxyStream section swap) */
/*       decompressors/PanasonicV4Decompressor.cpp:129-236               */
/*   PanasonicV5Decompressor::processBlock (+ ProxyStream section swap) */
/*       decompressors/PanasonicV5Decompressor.cpp:147-232              */
/*   PanasonicV6Decompressor::decompressBlock  PanasonicV6Decompressor.cpp:88-221 */
/*   PanasonicV7Decompressor::decompressBlock  PanasonicV7Decompressor.cpp:66-73  */
/* ------------------------------------------------------------------ */
typedef struct {
  uint64_t in_offset;  /* first byte of the image's data                          */
  uint64_t in_size;    /* bytes available (checked against the block count)       */
  uint64_t out_offset; /* byte offset of image row 0; multiple of 2               */
  uint32_t out_pitch;  /* bytes between output rows; multiple of 2, >= 2*width    */
  uint32_t width;      /* multiple of the pixels per 16-byte unit (V4: 14,        */
  uint32_t height;     /* V5: 10 / 9, V6: 14 / 11, V7: 9)                         */
  uint8_t version;     /* 4, 5, 6 or 7                                            */
  uint8_t bps;         /* 12 or 14 (V7: 14; V4: ignored)                          */
  uint8_t zero_is_not_bad; /* V4: 0 = positions of pixels decoded as 0 are kept
                              for rsb200_plan_bad_pixels()                        */
  uint8_t reserved;
  uint32_t section_split_offset; /* V4: 0 .. 0x4000 (0 = blocks are not swapped)  */
  uint32_t reserved1;
} rsb200_pana_job;

int rsb200_pana_plan_create(rsb200_ctx* ctx, const rsb200_pana_job* jobs, int njobs,
                            rsb200_plan** plan);
/* V4 jobs with zero_is_not_bad == 0: the positions ((row << 16) | col) of the pixels the
 * plan's last run decoded as 0 -- what the reference appends to mRaw->mBadPixelPositions
 * (PanasonicV4Decompressor.cpp:206-207, :228-235), in no particular order (the reference's
 * order depends on its thread schedule).  *count = how many there were; at most `cap` (and at
 * most RSB200_PANA_BAD_CAP) are stored.  Waits for the run. */
#define RSB200_PANA_BAD_CAP (1u << 22)
/* (For a DNG opcode plan `job` is the index of a BAD_CONSTANT opcode, see K10.) */
int rsb200_plan_bad_pixels(rsb200_plan* plan, int job, uint32_t* positions, uint32_t cap,
                           uint32_t* count);

/* ------------------------------------------------------------------ */
/* K8: Phase One IIQ row codec (SURVEY 8(f)4).                          */
/*   PhaseOneDecompressor::decompressStrip / decompress                 */
/*   decompressors/PhaseOneDecompressor.cpp:85-168                      */
/* ------------------------------------------------------------------ */
typedef struct {
  uint64_t in_offset; /* first byte of the strip (one image row)                  */
  uint32_t in_size;   /* bytes of the strip                                       */
  uint32_t row;       /* image row it decodes (PhaseOneStrip::n)                  */
} rsb200_phaseone_strip;

typedef struct {
  uint64_t out_offset;  /* byte offset of image row 0; multiple of 4              */
  uint32_t out_pitch;   /* bytes between output rows; multiple of 4, >= 2*width   */
  uint32_t width;       /* even, <= 11976                                         */
  uint32_t height;      /* <= 8854; the job owns `height` strips                  */
  uint32_t first_strip; /* index of its first strip in the plan's strip array; the
                           strips of a job may be in any order but must name every
                           row exactly once (prepareStrips, :61-83)               */
} rsb200_phaseone_job;

/* rsb200_plan_results: RSB200_ERR_RDE for a job with a row that cannot be decoded
 * (lengths not initialised at column 0, bit stream over-read) -- the reference's
 * "Too many errors encountered. Giving up." */
int rsb200_phaseone_plan_create(rsb200_ctx* ctx, const rsb200_phaseone_job* jobs, int njobs,
                                const rsb200_phaseone_strip* strips, int nstrips,
                                rsb200_plan** plan);

/* ------------------------------------------------------------------ */
/* K13: Samsung SRW V0 row codec (SURVEY 8(f)4).                       */
/*   SamsungV0Decompressor::decompress / decompressStrip                */
/*   decompressors/SamsungV0Decompressor.cpp:92-204                     */
/*   (one MSB32 bit stream per image row; blocks of 16 pixels predicted  */
/*   from the left or from one / two rows above; red/blue swap after)   */
/* ------------------------------------------------------------------ */
typedef struct {
  uint64_t in_offset; /* first byte of the row's stream                           */
  uint32_t in_size;   /* bytes of the row's stream (< 2^28)                       */
  uint32_t reserved;  /* 0                                                        */
} rsb200_samsung0_strip;

typedef struct {
  uint64_t out_offset;  /* byte offset of image row 0; even                       */
  uint32_t out_pitch;   /* bytes between output rows; even, >= 2*width            */
  uint32_t width;       /* 16..5546 and height 1..3714: the constructor's check   */
  uint32_t height;      /* (SamsungV0Decompressor.cpp:51-55)                      */
  uint32_t first_strip; /* its `height` strips, rows 0..height-1 in order, start
                           here in the plan's strip array (computeStripes, :61-90) */
} rsb200_samsung0_job;

/* Dimensions the constructor rejects fail plan creation with RSB200_ERR_RDE
 * ("Unexpected image dimensions found"); an odd out_offset or out_pitch, a pitch
 * below 2*width or strips outside the array with RSB200_ERR_ARG.  Rows with 4-byte
 * aligned out_offset and out_pitch are written 4 bytes at a time.
 * rsb200_plan_results() per job: RSB200_ERR_RDE or RSB200_ERR_IOE with consumed ==
 * code << 24 | row << 9 | block of the first failure (rows in order, blocks of 16
 * pixels), code one of RSB200_S0_*.  The image is then as the reference leaves it:
 * rows before the failing one decoded, that row up to the failing operation, the
 * rest untouched, and no red/blue swap. */
#define RSB200_S0_LEN_NEG 1u  /* RDE "Bit length less than 0."                             */
#define RSB200_S0_LEN_BIG 2u  /* RDE "Bit Length more than 16."                            */
#define RSB200_S0_UP_FIRST 3u /* RDE "Upward prediction for the first two rows. Raw corrupt" */
#define RSB200_S0_UP_LAST 4u  /* RDE "Upward prediction for the last block of pixels. ..."   */
#define RSB200_S0_OVERREAD 5u /* IOE "Buffer overflow read in BitStreamer"                  */
#define RSB200_S0_SHORT 6u    /* IOE "Bit stream size is smaller than MaxProcessBytes"      */
int rsb200_samsung0_plan_create(rsb200_ctx* ctx, const rsb200_samsung0_job* jobs, int njobs,
                                const rsb200_samsung0_strip* strips, int nstrips,
                                rsb200_plan** plan);

/* ------------------------------------------------------------------ */
/* K9: black / white level scaling, in place (SURVEY 8(f)3).            */
/*   RawImageDataU16::scaleValues  common/RawImageDataU16.cpp:185-399   */
/*   (the SCALE_VALUES worker of scaleBlackWhite(), :147-183)           */
/* The job scales the crop rows of one uint16 image that already lives  */
/* in the plan's OUTPUT buffer (a decode plan's output): run it with     */
/* rsb200_plan_run(plan, NULL, 0, d_image, bytes, stream).              */
/* ------------------------------------------------------------------ */
typedef struct {
  uint64_t offset;     /* byte offset of row 0 of the UNCROPPED image; multiple of 16 */
  uint32_t pitch;      /* bytes between rows; multiple of 16 (RawImageData::pitch)    */
  uint32_t width;      /* uncropped_dim.x (pixels)                                    */
  uint32_t height;     /* uncropped_dim.y                                             */
  uint32_t cpp;        /* components per pixel                                        */
  uint32_t crop_x;     /* mOffset.x                                                   */
  uint32_t crop_y;     /* mOffset.y                                                   */
  uint32_t crop_w;     /* dim.x                                                       */
  uint32_t crop_h;     /* dim.y                                                       */
  int32_t black_separate[4]; /* blackLevelSeparate, index 2*row + col                 */
  int32_t white_point;       /* whitePoint; must differ from black_separate[0]        */
  uint8_t dither;      /* mDitherScale                                                */
  uint8_t path;        /* RSB200_SCALE_AUTO: what an x86 build of the reference runs
                          (SSE2 loop iff 65535 / (white - black[0]) < 63, :185-202);
                          RSB200_SCALE_SSE2 / RSB200_SCALE_PLAIN force one            */
  uint8_t reserved[2];
} rsb200_scale_job;
#define RSB200_SCALE_AUTO 0
#define RSB200_SCALE_SSE2 1
#define RSB200_SCALE_PLAIN 2

int rsb200_scale_plan_create(rsb200_ctx* ctx, const rsb200_scale_job* jobs, int njobs,
                             rsb200_plan** plan);

/* ------------------------------------------------------------------ */
/* K10: a DNG opcode list applied in one pass, in place (SURVEY 8(f)3). */
/*   DngOpcodes::applyOpCodes            common/DngOpcodes.cpp:730-735  */
/*   PixelOpcode::applyOP (lattice walk) :390-409, LookupOpcode :417-438,*/
/*   OffsetPerRowOrCol :591-623, ScalePerRowOrCol :625-662,              */
/*   FixBadPixelsConstant::apply :172-183                                */
/* The list is parsed and validated on the host (the mirror's DngOpcodes */
/* class does what the reference's constructor and setup() do); what     */
/* reaches the device are the per-sample maps, with their ROI in         */
/* UNCROPPED pixel coordinates.  Run with rsb200_plan_run(plan, NULL, 0, */
/* d_image, bytes, stream).                                              */
/* ------------------------------------------------------------------ */
#define RSB200_DNGOP_LOOKUP 0       /* MapTable / MapPolynomial: v = table[v] (uint16)       */
#define RSB200_DNGOP_OFFSET_ROW 1   /* DeltaPerRow: clampBits(delta[y] + v, 16) | d[y] + v    */
#define RSB200_DNGOP_OFFSET_COL 2   /* DeltaPerColumn                                        */
#define RSB200_DNGOP_SCALE_ROW 3    /* ScalePerRow: clampBits((d[y]*v + 512) >> 10, 16) | d*v */
#define RSB200_DNGOP_SCALE_COL 4    /* ScalePerColumn                                        */
#define RSB200_DNGOP_BAD_CONSTANT 5 /* FixBadPixelsConstant: collect samples == value        */
typedef struct {
  uint32_t kind;
  uint32_t top, left, bottom, right; /* pixels top..bottom-1 x left..right-1 (uncropped)     */
  uint32_t first_plane, planes;      /* components first_plane .. first_plane+planes-1       */
  uint32_t row_pitch, col_pitch;     /* every row_pitch-th row / col_pitch-th column of the ROI */
  uint32_t table;  /* LOOKUP: index into `tables`; OFFSET / SCALE: first element in `deltas`
                      (one per affected row resp. column: int32 = (int)(f2iScale * f) for
                      uint16 images, the float itself for float images)                      */
  uint32_t value;  /* BAD_CONSTANT                                                           */
  uint32_t reserved;
} rsb200_dng_op;

typedef struct {
  uint64_t offset;   /* byte offset of row 0 of the uncropped image; multiple of 16          */
  uint32_t pitch;    /* bytes between rows; multiple of 16                                   */
  uint32_t width;    /* uncropped pixels per row                                             */
  uint32_t height;
  uint32_t cpp;      /* 1 .. 4                                                               */
  uint32_t is_f32;   /* samples are 32-bit floats instead of uint16                          */
  uint32_t first_op; /* this image's opcodes: ops[first_op .. first_op + num_ops)            */
  uint32_t num_ops;
  uint32_t reserved;
} rsb200_dngop_job;

/* tables: ntables x 65536 uint16; deltas: ndeltas 32-bit words.  The positions a
 * BAD_CONSTANT opcode collected ((row << 16) | col, uncropped coordinates, unordered) are
 * read with rsb200_plan_bad_pixels(plan, index of the opcode in `ops`, ...). */
int rsb200_dngop_plan_create(rsb200_ctx* ctx, const rsb200_dngop_job* jobs, int njobs,
                             const rsb200_dng_op* ops, int nops, const uint16_t* tables,
                             int ntables, const uint32_t* deltas, int ndeltas,
                             rsb200_plan** plan);

/* ------------------------------------------------------------------ */
/* K11: bad-pixel interpolation, in place (SURVEY 8(f)3).               */
/*   RawImageData::fixBadPixels / transferBadPixelsToMap /               */
/*   fixBadPixelsThread       common/RawImage.cpp:201-239, :297-323      */
/*   RawImageDataU16::fixBadPixel  common/RawImageDataU16.cpp:399-485    */
/* uint16 images with one component per pixel (the reference's indexing  */
/* for cpp > 1 makes the result depend on its visiting order; refused).  */
/* Run with rsb200_plan_run(plan, NULL, 0, d_image, bytes, stream).      */
/* ------------------------------------------------------------------ */
typedef struct {
  uint64_t offset;         /* byte offset of row 0 of the uncropped image; multiple of 2   */
  uint32_t pitch;          /* bytes between rows; multiple of 2                            */
  uint32_t width;          /* uncropped_dim                                                */
  uint32_t height;
  uint32_t is_cfa;         /* RawImageData::isCFA: neighbours at distance 2, else 1        */
  uint32_t first_position; /* mBadPixelPositions of this image: positions[first ..         */
  uint32_t num_positions;  /* first + num), each (y << 16) | x in uncropped coordinates    */
  const uint8_t* prior_map; /* an existing mBadPixelMap (map pitch roundUp(ceil(width/8),  */
                            /* 16) x height bytes) to OR the positions into, or NULL       */
} rsb200_badpix_job;

int rsb200_badpix_plan_create(rsb200_ctx* ctx, const rsb200_badpix_job* jobs, int njobs,
                              const uint32_t* positions, uint32_t npositions,
                              rsb200_plan** plan);

/* ------------------------------------------------------------------ */
/* K12: 16-bit table lookup of a whole image, in place (SURVEY 8(f)3).  */
/*   RawImageData::sixteenBitLookup        common/RawImage.cpp:373-378  */
/*   RawImageDataU16::doLookup      common/RawImageDataU16.cpp:487-520  */
/* (what DngDecoder does with a LinearizationTable, DngDecoder.cpp:614,  */
/* and Cr2Decoder with its curve, Cr2Decoder.cpp:117).  Every sample of  */
/* every row of the uncropped buffer; run with rsb200_plan_run(plan,     */
/* NULL, 0, d_image, bytes, stream).                                     */
/* ------------------------------------------------------------------ */
typedef struct {
  uint64_t offset;  /* byte offset of row 0 of the uncropped image; multiple of 16 */
  uint32_t pitch;   /* bytes between rows; multiple of 16                          */
  uint32_t width;   /* uncropped_dim.x (pixels)                                    */
  uint32_t height;
  uint32_t cpp;
  uint32_t table;   /* index into the plan's tables                                */
  uint32_t reserved;
} rsb200_lookup_job;

/* tables: ntables tables in TableLookUp's storage layout (common/TableLookUp.cpp:48-85):
 * dither == 0 -> 65536 uint16 each, dither != 0 -> 2*65536 uint16 each ({base, delta}). */
int rsb200_lookup_plan_create(rsb200_ctx* ctx, const rsb200_lookup_job* jobs, int njobs,
                              const uint16_t* tables, int ntables, int dither,
                              rsb200_plan** plan);

/* ------------------------------------------------------------------ */
/* K5: Canon sRaw interpolation (SURVEY 8(f)2).                         */
/*   Cr2sRawInterpolator::interpolate(version)                          */
/*   interpolators/Cr2sRawInterpolator.cpp:96-187 (4:2:2), :189-453     */
/*   (4:2:0), YUV_TO_RGB<0|1|2> + STORE_RGB :455-497                    */
/* ------------------------------------------------------------------ */
typedef struct {
  uint64_t in_offset;  /* byte offset of row 0 of the subsampled uint16 image (the
                          output of the CR2 decode: 4 (4:2:2) or 6 (4:2:0) samples
                          per MCU); multiple of 4                               */
  uint32_t in_pitch;   /* bytes between its rows; multiple of 4                  */
  uint32_t num_mcus;   /* MCUs per input row (input.width() / 4 or / 6), >= 2    */
  uint32_t in_rows;    /* rows of the subsampled image                           */
  uint8_t sub_x;       /* ImageMetaData::subsampling: (2,1) = 4:2:2, (2,2) = 4:2:0 */
  uint8_t sub_y;
  uint8_t version;     /* 0, 1, 2 (4:2:0: 1 or 2)                                */
  uint8_t reserved;
  int32_t sraw_coeffs[3];
  int32_t hue;
  uint64_t out_offset; /* byte offset of the 3-component output image; multiple of 4 */
  uint32_t out_pitch;  /* bytes; rows written: in_rows * sub_y, 2*num_mcus pixels each */
  uint32_t reserved1;
} rsb200_sraw_job;

int rsb200_sraw_plan_create(rsb200_ctx* ctx, const rsb200_sraw_job* jobs, int njobs,
                            rsb200_plan** plan);

/* ------------------------------------------------------------------ */
/* K2+K3: lossless JPEG (Huffman + predictor 1).                        */
/* ------------------------------------------------------------------ */
typedef struct {
  uint8_t ncodes_per_len[16]; /* DHT Li, i = 1..16                               */
  uint8_t values[162];        /* DHT Vij: SSSS per code, in code order           */
  uint16_t nvalues;
  uint8_t fix_dng16; /* PrefixCodeDecoder::setup(fullDecode=true, fixDNGBug16)   */
  uint8_t reserved[3];
} rsb200_huff_table;

/* One entropy-coded segment: one restart interval of one tile (or the whole
 * tile when DRI is absent).  Geometry follows LJpegDecompressor
 * (LJpegDecompressor.cpp:52-152). */
typedef struct {
  uint64_t in_offset; /* first entropy-coded byte inside the input buffer        */
  uint32_t in_size;   /* bytes available from there (to the end of the tile's
                         buffer); the first FFxx (xx!=0) ends the data           */
  uint32_t rows;      /* LJPEG rows decoded in this segment                      */
  uint32_t frame_w;   /* MCUs per LJPEG row (Frame::dim.x); all are decoded, only
                         the first ceil(store_w/mcu_w) are kept                  */
  uint8_t mcu_w;      /* Frame::mcu: {1,1} {2,1} {3,1} {4,1} {2,2}               */
  uint8_t mcu_h;
  uint8_t table[4];   /* index into the plan's table array, per component       */
  uint8_t reserved[2];
  uint16_t init_pred[4]; /* PerComponentRecipe::initPred                        */
  uint64_t out_offset;   /* byte offset of the image (row 0, col 0); even       */
  uint32_t out_pitch;    /* bytes; even                                         */
  uint32_t out_x;        /* first output sample column = cpp * imgFrame.pos.x   */
  uint32_t out_y;        /* first output row of this segment                    */
  uint32_t store_w;      /* samples kept per row = cpp * imgFrame.dim.x         */
} rsb200_ljpeg_scan;

typedef struct {
  uint32_t status;   /* RSB200_OK / RSB200_ERR_RDE / RSB200_ERR_IOE              */
  uint32_t consumed; /* BitStreamerJPEG::getStreamPosition() after the segment
                        (BitStreamerJPEG.h:185-189): bytes from in_offset       */
} rsb200_scan_result;

/* Segments are independent (DNG tiles, restart intervals).  The plan picks the kernel:
 * block-per-segment (K2F; multi-CTA K2R for segments > 256 KiB) or, when the plan holds
 * >= 16384 eligible segments (e.g. a batch of >= 23 frames of 726 tiles), an unstuffing
 * pre-pass plus one thread per segment (K2C + K2T, ljpeg_clean.cuh / ljpeg_thread.cuh).
 * Results are identical; the environment variable RSB200_LJPEG_PATH=fused|thread, read at
 * plan creation, forces the choice (tests).  The thread path allocates a scratch copy of
 * the compressed bytes of its segments with the plan. */
int rsb200_ljpeg_plan_create(rsb200_ctx* ctx, const rsb200_huff_table* tables,
                             int ntables, const rsb200_ljpeg_scan* scans,
                             int nscans, rsb200_plan** plan);

/* Canon CR2: one job = one frame = one entropy-coded stream
 * (Cr2DecompressorImpl.h:396-468).  Values are the *validated* ones the
 * Cr2Decompressor ctor (:279-363) works with. */
typedef struct {
  uint64_t in_offset;
  uint32_t in_size;
  uint8_t n_comp, x_s_f, y_s_f; /* format <N_COMP, X_S_F, Y_S_F>                 */
  uint8_t reserved0;
  uint8_t table[4];
  uint16_t init_pred[4];
  int32_t frame_w, frame_h;  /* LJPEG frame (SOF3 w,h after the Canon height fix) */
  int32_t num_slices;        /* Cr2SliceWidths (CANONCR2SLICE): widths in sample   */
  int32_t slice_w;           /*   columns, as passed to the Cr2Decompressor ctor   */
  int32_t last_slice_w;
  int32_t img_w, img_h;      /* RawImage dim (cpp == 1)                           */
  uint64_t out_offset;       /* byte offset of image row 0; even                  */
  uint32_t out_pitch;        /* bytes; even, >= 2 * img_w                         */
  uint32_t reserved1;
} rsb200_cr2_job;

int rsb200_cr2_plan_create(rsb200_ctx* ctx, const rsb200_huff_table* tables,
                           int ntables, const rsb200_cr2_job* jobs, int njobs,
                           rsb200_plan** plan);

/* ------------------------------------------------------------------ */
/* Pentax PEF Huffman codec (SURVEY 8(f)2).                              */
/*   PentaxDecompressor::decompress  decompressors/PentaxDecompressor.cpp:158-176 */
/*   (plain MSB bit stream, one table, per-parity left predictor, row   */
/*   starts from two rows up).  The table comes from the host:          */
/*   SetupPrefixCodeDecoder_Legacy/_Modern :69-141.                     */
/* ------------------------------------------------------------------ */
typedef struct {
  uint64_t in_offset; /* first byte of the compressed stream                    */
  uint32_t in_size;   /* bytes available                                        */
  uint32_t table;     /* index into the plan's table array                      */
  int32_t width;      /* image width (even, <= 8384) and height (<= 6208)       */
  int32_t height;
  uint64_t out_offset; /* byte offset of image row 0                            */
  uint32_t out_pitch;  /* bytes                                                 */
  uint32_t reserved;
} rsb200_pentax_job;

/* rsb200_plan_results() for such a plan: status RSB200_ERR_RDE with consumed ==
 * 0 = "bad Huffman code"; with consumed == 0x80000000 | (row << 14) | col =
 * "decoded value out of bounds at col:row" (the first such pixel in stream order);
 * RSB200_ERR_IOE = stream exhausted. */
#define RSB200_PENTAX_OOB 0x80000000u
int rsb200_pentax_plan_create(rsb200_ctx* ctx, const rsb200_huff_table* tables, int ntables,
                              const rsb200_pentax_job* jobs, int njobs, rsb200_plan** plan);

/* ------------------------------------------------------------------ */
/* Sony ARW1 (SURVEY 8(f)2).                                             */
/*   SonyArw1Decompressor::decompress  decompressors/SonyArw1Decompressor.cpp:58-92 */
/*   (plain MSB bit stream, fixed prefix code, one running predictor    */
/*   over the frame, walked column by column from the right: even rows, */
/*   then odd rows; every value must stay in 0..4095).                  */
/* ------------------------------------------------------------------ */
typedef struct {
  uint64_t in_offset; /* first byte of the stream                                 */
  uint32_t in_size;   /* bytes available (the rest of the file in ArwDecoder);   */
                      /* < 2^28 (stream bit positions are 32-bit on the device)  */
  uint32_t reserved0; /* 0                                                       */
  int32_t width;      /* 1..4600 and height (even, 2..3072): the constructor's    */
  int32_t height;     /* checks, SonyArw1Decompressor.cpp:39-50                   */
  uint64_t out_offset; /* byte offset of image row 0 (even)                      */
  uint32_t out_pitch;  /* bytes (even, >= 2 * width)                             */
  uint32_t reserved;   /* 0                                                      */
} rsb200_arw1_job;

/* Dimensions the reference's constructor rejects fail plan creation with
 * RSB200_ERR_RDE ("Unexpected image dimensions found").  rsb200_plan_results()
 * for such a plan: RSB200_ERR_RDE with consumed == RSB200_PENTAX_OOB | (row << 14)
 * | col = "Error decompressing" at the first pixel (stream order) whose value left
 * 0..4095; RSB200_ERR_IOE = a refill of the bit pump started more than 8 bytes
 * behind the stream, before that pixel, or a stream of fewer than 4 bytes.  Pixels up to the error are written, as
 * the reference does; the rest of the image is left as it was. */
int rsb200_arw1_plan_create(rsb200_ctx* ctx, const rsb200_arw1_job* jobs, int njobs,
                            rsb200_plan** plan);

/* ------------------------------------------------------------------ */
/* Samsung SRW V1, compression 32772 (SURVEY 8(f)4).                     */
/*   SamsungV1Decompressor::decompress                                   */
/*   decompressors/SamsungV1Decompressor.cpp:81-140                      */
/*   (plain MSB bit stream, fixed prefix code, per-parity left predictor,*/
/*   rows start from two rows up; every value must stay in 0..4095).     */
/* ------------------------------------------------------------------ */
typedef struct {
  uint64_t in_offset; /* first byte of the stream                                 */
  uint32_t in_size;   /* bytes available; < 2^28                                  */
  uint32_t bits;      /* the container's bits per sample (must be 12)            */
  int32_t width;      /* multiple of 32, 32..5664, and height (even, 2..3714):    */
  int32_t height;     /* the constructor's checks, SamsungV1Decompressor.cpp:52-60 */
  uint64_t out_offset; /* byte offset of image row 0; multiple of 4               */
  uint32_t out_pitch;  /* bytes; multiple of 4, >= 2 * width                     */
  uint32_t reserved;   /* 0                                                      */
} rsb200_samsung1_job;

/* A bit count other than 12 or dimensions the reference's constructor rejects fail
 * plan creation with RSB200_ERR_RDE ("Unexpected bit per pixel" / "Unexpected image
 * dimensions found"); an out_offset or out_pitch that is not a multiple of 4, a pitch
 * below 2 * width, in_size >= 2^28 or a non-zero reserved field with RSB200_ERR_ARG.
 * rsb200_plan_results() per job: RSB200_ERR_RDE with consumed == RSB200_PENTAX_OOB |
 * (row << 14) | col = "decoded value out of bounds" at the first pixel (row-major)
 * whose value left 0..4095; RSB200_ERR_IOE with consumed == (row << 14) | col of the
 * pixel whose refill started more than 8 bytes behind the stream (0 for a stream of
 * fewer than 4 bytes), when it comes first.  Pixels before the error are written; the
 * rest of the image is left as it was. */
int rsb200_samsung1_plan_create(rsb200_ctx* ctx, const rsb200_samsung1_job* jobs, int njobs,
                                rsb200_plan** plan);

/* ------------------------------------------------------------------ */
/* Samsung SRW V2, compression 32773 (SURVEY 8(f)4).                     */
/*   SamsungV2Decompressor::SamsungV2Decompressor / decompress           */
/*   decompressors/SamsungV2Decompressor.cpp:85-355                      */
/*   (one MSB32 stream per row, each starting at the next multiple of 16 */
/*   bytes of the data; blocks of 16 pixels predicted from the left or   */
/*   from one / two rows up, every pixel clamped to the bit depth).       */
/* ------------------------------------------------------------------ */
typedef struct {
  uint64_t in_offset;  /* first byte of the strip, its 16-byte header included    */
  uint32_t in_size;    /* bytes of the strip; < 2^28                              */
  uint32_t bits;       /* the container's bits per sample (12 or 14)              */
  int32_t width;       /* the RawImage's dimensions, which must equal the         */
  int32_t height;      /* header's                                                */
  uint8_t header[16];  /* the strip's first 16 bytes (the device reads from
                          in_offset + 16)                                         */
  uint64_t out_offset; /* byte offset of image row 0; multiple of 4               */
  uint32_t out_pitch;  /* bytes; multiple of 4, >= 2 * width                      */
  uint32_t reserved;   /* 0                                                       */
} rsb200_samsung2_job;

/* Plan creation runs the constructor's checks in its order (SamsungV2Decompressor.cpp:88-142): bits
 * other than 12 / 14 (RSB200_ERR_RDE "Unexpected bit per pixel"), in_size < 16 (RSB200_ERR_IOE "Out of
 * bounds access in ByteStream"), then from the header a bit depth other than bits, opt flags > 7,
 * dimensions the constructor rejects and dimensions other than width x height (RSB200_ERR_RDE with the
 * reference's messages).  An out_offset or out_pitch that is not a multiple of 4, a pitch below
 * 2 * width, in_size >= 2^28 or a non-zero reserved field are refused with RSB200_ERR_ARG.
 * rsb200_plan_results() per job: RSB200_ERR_RDE or RSB200_ERR_IOE with consumed ==
 * code << 28 | value << 22 | row << 9 | block of the first failure, code one of RSB200_S2_*, value the
 * number the message prints (the motion, or the difference bits) and block the block of 16 pixels
 * (0 for a failure in front of the row's first block, width / 16 for the skip behind its last).  The
 * image is then as the reference leaves it: the rows before the failing one and the blocks of that
 * row before the failing block written (the whole row for a failure behind it), nothing else. */
#define RSB200_S2_START_MOTION 1u /* RDE "At start of image and motion isn't 7. File corrupted?" */
#define RSB200_S2_MOTION_BEGIN 2u /* RDE "Bad motion %d at the beginning of the row"             */
#define RSB200_S2_MOTION_END 3u   /* RDE "Bad motion %d at the end of the row"                   */
#define RSB200_S2_UNDERFLOW 4u    /* RDE "Difference bits underflow. File corrupted?"            */
#define RSB200_S2_TOO_MANY 5u     /* RDE "Too many difference bits (%u). File corrupted?"        */
#define RSB200_S2_OVERREAD 6u     /* IOE "Buffer overflow read in BitStreamer"                   */
#define RSB200_S2_SHORT 7u        /* IOE "Bit stream size is smaller than MaxProcessBytes"       */
#define RSB200_S2_BYTESTREAM 8u   /* IOE "Out of bounds access in ByteStream"                    */
int rsb200_samsung2_plan_create(rsb200_ctx* ctx, const rsb200_samsung2_job* jobs, int njobs,
                                rsb200_plan** plan);

/* ------------------------------------------------------------------ */
/* Kodak DCR, compression 65000 (DESIGN 8(f)4).                          */
/*   KodakDecompressor::KodakDecompressor / decompress                   */
/*   decompressors/KodakDecompressor.cpp:46-150                          */
/*   (rows cut into segments of up to 256 pixels; a segment is a header  */
/*   of 4-bit lengths, then the differences as a bit string, predicted   */
/*   per parity from 0 at every segment).                                */
/* ------------------------------------------------------------------ */
typedef struct {
  uint64_t in_offset;  /* first byte of the stream                                 */
  uint32_t in_size;    /* bytes of the stream; <= 2^28                             */
  int32_t width;       /* the RawImage's dimensions                                */
  int32_t height;
  int32_t bps;         /* bits per sample (10 or 12)                               */
  int32_t table;       /* index into the plan's tables, -1 = none (uncorrectedRawValues,
                          or an image without a table)                             */
  uint64_t out_offset; /* byte offset of image row 0; multiple of 4                */
  uint32_t out_pitch;  /* bytes; multiple of 4, >= 2 * width                       */
  uint32_t reserved;   /* 0                                                        */
} rsb200_kodak_job;

/* `tables`: ntables x 65536 uint16 entries, as for rsb200_raw_plan_create (for a dithered table pass
 * entries 2*v: the dither counter of decompress starts at 0 and stays there, RawImage.h:335-353).
 * Plan creation runs the constructor's checks in its order (KodakDecompressor.cpp:50-64): dimensions
 * (RSB200_ERR_RDE "Unexpected image dimensions found: (%d; %d)"), bps ("Unexpected bits per sample: %i"),
 * then in_size < width * height / 2 (RSB200_ERR_IOE "Out of bounds access in ByteStream").  An
 * out_offset or out_pitch that is not a multiple of 4, a pitch below 2 * width, in_size > 2^28, a table
 * outside 0..ntables - 1 (other than -1) or a non-zero reserved field are refused with RSB200_ERR_ARG.
 * rsb200_plan_results() per job: RSB200_ERR_RDE or RSB200_ERR_IOE with consumed ==
 * code << 28 | row << 13 | column, code one of RSB200_KODAK_*, column the failing pixel's (RDE) or the
 * first of the segment that reads past the end (IOE).  The image then holds every pixel in front of
 * that one in raster order and nothing else.  The value the RDE message prints comes from
 * rsb200_kodak_plan_values. */
#define RSB200_KODAK_VALUE 1u    /* RDE "Value out of bounds %d (bps = %i)"          */
#define RSB200_KODAK_OVERFLOW 2u /* IOE "Buffer overflow: image file may be truncated" */
int rsb200_kodak_plan_create(rsb200_ctx* ctx, const rsb200_kodak_job* jobs, int njobs, const uint16_t* tables,
                             int ntables, rsb200_plan** plan);
/* After a run of a Kodak plan: values[i] (i < n) = the value job i's RSB200_KODAK_VALUE failure prints,
 * 0 for a job without one.  RSB200_ERR_ARG for another kind of plan or one that has not run. */
int rsb200_kodak_plan_values(rsb200_plan* plan, int32_t* values, int n);

/* ------------------------------------------------------------------ */
/* GoPro VC-5, DNG compression 9 (DESIGN 4 VC5).                         */
/*   VC5Decompressor::decode  decompressors/VC5Decompressor.cpp:137-960  */
/*   (4 channels x 10 subbands: a low-pass band of fixed-width values    */
/*   and nine run-length / prefix-code bands per channel, three inverse  */
/*   wavelet levels, a Bayer combine through a log table).  The tag walk */
/*   (parseVC5) runs on the host: a plan sees band payloads only.        */
/* ------------------------------------------------------------------ */
typedef struct {
  uint32_t size;  /* code length in bits, 1..26                         */
  uint32_t bits;  /* code word, right-justified                         */
  uint32_t count; /* run length, 0..511 (0: a marker)                   */
  uint32_t value; /* run value magnitude, 0..255 (decompanded by the plan) */
} rsb200_vc5_code;

typedef struct {
  uint64_t in_offset; /* first byte of the band's payload                            */
  uint32_t in_size;   /* bytes; high pass: a multiple of 4, <= 2^28; low pass: at least
                         8 * ceil(w * h * precision / 64)                            */
  int32_t param;      /* high pass: quantization (-32768..32767); low pass: precision 8..16 */
} rsb200_vc5_band;

typedef struct {
  int32_t width;         /* the image: even, 34..65534 (a level-3 band of 3 or more)  */
  int32_t height;
  int32_t output_bits;   /* bit length of the white level, 1..16                      */
  int32_t phase;         /* RSB200_VC5_RGGB or RSB200_VC5_GBRG                        */
  uint8_t prescale[4][3]; /* [channel][wavelet 1..3]: PrescaleShift, 0..3 (2: descale) */
  uint32_t first_band;   /* its 40 bands are bands[first_band + channel * 10 + subband] */
  uint64_t out_offset;   /* byte offset of image row 0; multiple of 4                 */
  uint32_t out_pitch;    /* bytes; multiple of 4, >= 2 * width                        */
  uint32_t reserved;     /* 0                                                         */
} rsb200_vc5_job;

/* `codes`: ncodes entries, a complete prefix code (the Kraft sum is exactly 1, no code is a prefix of
 * another), each size 1..26, count <= 511, value <= 255; else RSB200_ERR_ARG.  The plan builds its
 * decode tables and decompanded values from it.  Refused with RSB200_ERR_ARG: a job whose width or
 * height is odd, <= 32 (the reference reads outside its bands there) or > 65534, output_bits outside
 * 1..16, a phase other than the two, a prescale > 3, bands outside 0..nbands - 1, an out_offset or
 * out_pitch that is not a multiple of 4, a pitch below 2 * width, a non-zero reserved field, or a band
 * that breaks the in_size / param rules above.
 * rsb200_plan_results() per job: RSB200_ERR_RDE or RSB200_ERR_IOE (the two RSB200_VC5_* marked IOE)
 * with consumed == code << 28 | channel << 4 | subband of the band the reference's decode (one worker)
 * meets first among the failing ones: subbands 3, 2, 1, 6, 5, 4, 9, 8, 7, each for channels 0..3.
 * Within a band, the failure is that of the first failing symbol in stream order.  A failed job's
 * image is left untouched. */
#define RSB200_VC5_RGGB 0
#define RSB200_VC5_GBRG 2
#define RSB200_VC5_QUANT 1u     /* RDE "Impossible RLV value given current quantum"          */
#define RSB200_VC5_EARLY_END 2u /* RDE "Got EndOfBand marker while looking for next pixel"   */
#define RSB200_VC5_OVERRUN 3u   /* RDE "Not all pixels consumed?"                            */
#define RSB200_VC5_NO_END 4u    /* RDE "EndOfBand marker not found"                          */
#define RSB200_VC5_SHORT 5u     /* IOE "Bit stream size is smaller than MaxProcessBytes"     */
#define RSB200_VC5_OVERREAD 6u  /* IOE "Buffer overflow read in BitStreamer"                 */
int rsb200_vc5_plan_create(rsb200_ctx* ctx, const rsb200_vc5_code* codes, int ncodes, const rsb200_vc5_job* jobs,
                           int njobs, const rsb200_vc5_band* bands, int nbands, rsb200_plan** plan);

/* ------------------------------------------------------------------ */
/* Nikon NEF Huffman codec without split (SURVEY 8(f)2).                 */
/*   NikonDecompressor::decompress  decompressors/NikonDecompressor.cpp:513-560 */
/*   (plain MSB bit stream, nikon_tree table, per-parity left predictor, */
/*   rows start from pUp[row & 1], clampBits(15), dithered curve).  The  */
/*   constructor work (:380-511: version bytes, tree selection, pUp,     */
/*   createCurve, split) stays on the host.                              */
/* ------------------------------------------------------------------ */
typedef struct {
  uint64_t in_offset;  /* first byte of the compressed stream                   */
  uint32_t in_size;    /* bytes available (>= 4)                                */
  uint32_t table;      /* index into the plan's Huffman tables                  */
  int32_t width;       /* even, <= 8288                                         */
  int32_t height;      /* <= 5520                                               */
  uint64_t out_offset; /* byte offset of image row 0; multiple of 4             */
  uint32_t out_pitch;  /* bytes; multiple of 4                                  */
  int32_t lut;         /* index into the plan's curve tables, -1 = none
                          (uncorrectedRawValues)                                */
  uint16_t pup[4];     /* pUp[0][0], pUp[0][1], pUp[1][0], pUp[1][1]            */
} rsb200_nikon_job;

/* `luts`: nluts curve tables in TableLookUp's DITHERED storage layout (2*65536
 * uint16 each: base, delta per value; common/TableLookUp.cpp:62-84).  Status as for
 * the LJPEG plans: RSB200_ERR_RDE = bad Huffman code, RSB200_ERR_IOE = stream
 * exhausted. */
int rsb200_nikon_plan_create(rsb200_ctx* ctx, const rsb200_huff_table* tables, int ntables,
                             const rsb200_nikon_job* jobs, int njobs, const uint16_t* luts,
                             int nluts, rsb200_plan** plan);



/* ------------------------------------------------------------------ */
/* Plan execution                                                       */
/* ------------------------------------------------------------------ */
/* Device-resident: d_in / d_out are device pointers (16-byte aligned; d_in must
 * be readable up to the next 16-byte boundary past in_bytes).  Enqueues the
 * kernels on `stream` (a cudaStream_t, may be 0) and returns without waiting. */
int rsb200_plan_run(rsb200_plan* plan, const void* d_in, size_t in_bytes,
                    void* d_out, size_t out_bytes, void* stream);
/* Host buffers: H2D copy of `in`, kernels, D2H copy of `out` (pinned staging is
 * the library's), then waits.  `out` must hold the current image contents for
 * bytes the decode does not write (it is uploaded first when partial != 0; always
 * for the in-place plans K9 - K12, which take in == NULL, in_bytes == 0). */
int rsb200_plan_run_host(rsb200_plan* plan, const uint8_t* in, size_t in_bytes,
                         uint8_t* out, size_t out_bytes, int partial);
/* Same, for a plan whose output is ONE RawImage (pitch bytes between rows): only
 * row_bytes of every row are copied back, so the host's row padding is left
 * untouched (RawImageData::createData(), common/RawImage.cpp:68-113). */
int rsb200_plan_run_host_image(rsb200_plan* plan, const uint8_t* in, size_t in_bytes,
                               uint8_t* out, uint32_t pitch, uint32_t row_bytes,
                               uint32_t rows, int partial);
/* Waits for the plan's last run and returns per-segment status/consumed
 * (nresults = number of scans/jobs; unpack plans report RSB200_OK only).
 * Return value: first non-OK status, or RSB200_OK. */
int rsb200_plan_results(rsb200_plan* plan, rsb200_scan_result* results,
                        int nresults);
/* Algorithmic byte counts of one run (input bytes read + output bytes written),
 * for roofline accounting. */
int rsb200_plan_bytes(const rsb200_plan* plan, uint64_t* in_bytes,
                      uint64_t* out_bytes, uint64_t* pixels);
/* ------------------------------------------------------------------ */
/* HasselbladDecompressor (reference: decompressors/HasselbladDecompressor.h:37-64 ctor + decompress(),
 * HasselbladDecompressor.cpp:39-100; caller HasselbladLJpegDecoder::decodeScan,
 * HasselbladLJpegDecoder.cpp:50-69).  One frame is ONE Huffman stream over the MSB32 bit source
 * (32-bit little-endian chunks, most significant bit first), per pair of pixels
 * [len1 code][len2 code][len1 bits][len2 bits]; both predictors restart at init_pred in every row.
 * The table's values are difference lengths 0..16; a difference of 16 one-bits means -32768.
 * rsb200_plan_results: per job RSB200_ERR_RDE for a code that is not in the table ("bad Huffman
 * code"), RSB200_ERR_IOE where the reference's replenisher throws (a refill more than 8 bytes behind
 * the buffer), whichever comes first in stream order; consumed = the reference's
 * BitStreamerMSB32::getStreamPosition() after the last pair. */
typedef struct rsb200_hasselblad_job {
  uint64_t in_offset;  /* first byte of the stream in the input buffer; multiple of 4 */
  uint32_t in_size;    /* bytes of the stream (what the reference's Array1DRef input holds) */
  uint32_t width;      /* pixels, even, <= 12000 */
  uint32_t height;     /* <= 8842 */
  uint32_t out_pitch;  /* bytes, multiple of 4 */
  uint64_t out_offset; /* first byte of the image in the output buffer; multiple of 4 */
  uint16_t init_pred;  /* PerComponentRecipe::initPred */
  uint8_t table;       /* index into `tables` */
  uint8_t reserved[5];
} rsb200_hasselblad_job;
int rsb200_hasselblad_plan_create(rsb200_ctx* ctx, const rsb200_huff_table* tables, int ntables,
                                  const rsb200_hasselblad_job* jobs, int njobs, rsb200_plan** plan);

/* Kernels launched by one rsb200_plan_run(). */
int rsb200_plan_launches(const rsb200_plan* plan);
/* Which kernels one rsb200_plan_run() of this plan launches, as a short static string (for logs and
 * the benchmark's JSON line), e.g. "k2_stream_kernel (one thread per segment) [+ k2_tile_kernel<1>
 * second opinion]" for an LJPEG plan; "unpack_fast_kernel", "unpack_kernel" or
 * "unpack_fast_kernel + unpack_kernel" for an unpack plan; "rawform_kernel" for a raw-form plan
 * ("(empty unpack plan)" / "(empty raw-form plan)" when every job has 0 rows); "(not an LJPEG
 * plan)" for the other kinds; "" for a null plan. */
const char* rsb200_plan_kernels(const rsb200_plan* plan);
void rsb200_plan_destroy(rsb200_plan* plan);

/* ------------------------------------------------------------------ */
/* Multi-GPU: frames are sharded across the GPUs of one box, one process */
/* per GPU (SURVEY 8e); the only exchange is the gather of the decoded   */
/* uint16 images over NVLink.  The reference has no counterpart (its     */
/* fan-out is OpenMP over tiles, AbstractDngDecompressor.cpp:240-252);   */
/* this is the `rsgpu_gather` of SURVEY 8b.  NCCL is taken from the      */
/* process at run time (dlopen of libnccl.so.2, the copy that is already  */
/* loaded if there is one); without it these calls return RSB200_ERR_CUDA.*/
/* ------------------------------------------------------------------ */
typedef struct rsb200_comm rsb200_comm;
enum {
  RSB200_GATHER_NONE = 0, /* decode only: every rank keeps its slab               */
  RSB200_GATHER_ALL = 1,  /* every rank ends up with every slab                   */
  RSB200_GATHER_ROOT = 2  /* only `root` does (the consumer GPU)                  */
};
/* Rank 0 makes the 128-byte id, the caller ships it to the other ranks (any
 * side channel), then every rank creates its communicator. */
int rsb200_comm_unique_id(uint8_t id[128]);
int rsb200_comm_create(rsb200_ctx* ctx, const uint8_t id[128], int world, int rank,
                       rsb200_comm** comm);
void rsb200_comm_destroy(rsb200_comm* comm);
/* Decode + gather.  d_out_all holds `world` slabs of slab_bytes each; this rank
 * decodes into slab `rank` (the plan's output offsets are relative to the slab)
 * and, as soon as a group of segments (~8 MB of pixels) has been decoded, that
 * part of the slab travels on the communicator's own stream, so the transfer
 * overlaps the decode of the following groups.  Every rank must run a plan of
 * the same geometry (same output spans).  `stream` orders the whole call: when
 * work queued behind it on `stream` runs, decode and gather are complete. */
int rsb200_plan_run_gather(rsb200_plan* plan, rsb200_comm* comm, const void* d_in,
                           size_t in_bytes, void* d_out_all, size_t slab_bytes, int mode,
                           int root, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* RAWSPEED_B200_H */
