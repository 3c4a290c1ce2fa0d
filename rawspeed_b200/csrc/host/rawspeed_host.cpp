// rawspeed_host.cpp -- host side of the drop-in: the reference's decompressor
// classes re-implemented above the C ABI (see rawspeed_host.h for the map of
// reference files).  Everything here is header parsing / validation / exception
// plumbing; every per-pixel loop of the reference is a call into
// librawspeed_b200.so (CUDA).  There is no CPU decode path in this file.
#include "../vc5_parse.h"
#include "rawspeed_host.h"

#include <algorithm>
#include <thread>
#include <atomic>
#include <cstdlib>
#include <cmath>
#include <cstring>
#include <limits>

namespace rawspeed_b200 {

// ------------------------------------------------------------------ exceptions
static std::string vfmt(const char* fmt, va_list ap) {
  char buf[512];
  vsnprintf(buf, sizeof buf, fmt, ap);
  return buf;
}
void ThrowRDE(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  std::string s = vfmt(fmt, ap);
  va_end(ap);
  throw RawDecoderException(s);
}
void ThrowIOE(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  std::string s = vfmt(fmt, ap);
  va_end(ap);
  throw IOException(s);
}

// ------------------------------------------------------------------ engine
rsb200_ctx* engine() {
  static rsb200_ctx* ctx = nullptr;
  static std::mutex m;
  std::lock_guard<std::mutex> g(m);
  if (!ctx) {
    int dev = 0;
    if (const char* e = std::getenv("RSB200_DEVICE"))
      dev = std::atoi(e);
    if (rsb200_create(dev, &ctx) != RSB200_OK || !ctx)
      ThrowRDE("rawspeed_b200: no usable CUDA device (there is no CPU fallback)");
  }
  return ctx;
}

void engineCheck(int rc, const char* what) {
  if (rc == RSB200_OK)
    return;
  const char* msg = rsb200_last_error(engine());
  if (rc == RSB200_ERR_IOE)
    ThrowIOE("%s", (msg && *msg) ? msg : "Buffer overflow read in BitStreamer");
  ThrowRDE("%s: %s", what, (msg && *msg) ? msg : "device error");
}

namespace {
struct PlanGuard {
  rsb200_plan* p = nullptr;
  ~PlanGuard() {
    if (p)
      rsb200_plan_destroy(p);
  }
};

// run a plan whose output is (part of) a RawImage held in host memory
void runOnImage(rsb200_plan* plan, const uint8_t* in, size_t inBytes, RawImage& img,
                bool partial) {
  engineCheck(rsb200_plan_run_host_image(plan, in, inBytes, img->getByteData(),
                                         (uint32_t)img->pitch,
                                         (uint32_t)(img->dim.x * (int)img->getBpp()),
                                         (uint32_t)img->dim.y, partial ? 1 : 0),
              "rsb200_plan_run_host_image");
}
} // namespace

// ------------------------------------------------------------------ RawImage
void RawImageData::setCpp(uint32_t v) {
  if (isAllocated())
    ThrowRDE("Attempted to set Components per pixel after data allocation");
  if (v > 4)
    ThrowRDE("Only up to 4 components per pixel is support - attempted to set: %u", v);
  bpp = bpp / cpp * v;
  cpp = v;
}

void RawImageData::createData() {
  if (dim.x > 65535 || dim.y > 65535)
    ThrowRDE("Dimensions too large for allocation.");
  if (dim.x <= 0 || dim.y <= 0)
    ThrowRDE("Dimension of one sides is less than 1 - cannot allocate image.");
  if (cpp <= 0 || bpp <= 0)
    ThrowRDE("Unspecified component count - cannot allocate image.");
  if (isAllocated())
    ThrowRDE("Duplicate data allocation in createData.");
  pitch = (int)(((size_t)dim.x * bpp + 15) / 16 * 16);
  data.resize((size_t)pitch * dim.y + 16);
  storage = reinterpret_cast<uint8_t*>(((uintptr_t)data.data() + 15) & ~(uintptr_t)15);
  uncropped_dim = dim;
}

// RawImageData::subFrame (common/RawImage.cpp:175-199); the CFA shift is metadata outside
// this path
void RawImageData::subFrame(iRectangle2D crop) {
  if (!crop.hasPositiveArea())
    ThrowRDE("No positive crop area");
  if (!(crop.dim.x <= dim.x - crop.pos.x && crop.dim.y <= dim.y - crop.pos.y))
    return; // "Attempted to create new subframe larger than original size. Crop skipped."
  if (crop.pos.x < 0 || crop.pos.y < 0 || crop.dim.x < 0 || crop.dim.y < 0)
    return; // "Negative crop offset. Crop skipped."
  mOffset.x += crop.pos.x;
  mOffset.y += crop.pos.y;
  dim = crop.dim;
}

// RawImageData::sixteenBitLookup (common/RawImage.cpp:373-378) -> doLookup over the full image
void RawImageData::sixteenBitLookup() {
  if (!hasTable())
    return;
  if (dataType != RawImageType::UINT16)
    ThrowRDE("rawspeed_b200: sixteenBitLookup is implemented for UINT16 images");
  if (!isAllocated())
    ThrowRDE("sixteenBitLookup: image has no data");
  rsb200_lookup_job job;
  std::memset(&job, 0, sizeof job);
  job.offset = 0;
  job.pitch = (uint32_t)pitch;
  job.width = (uint32_t)uncropped_dim.x;
  job.height = (uint32_t)uncropped_dim.y;
  job.cpp = cpp;
  job.table = 0;
  PlanGuard pg;
  engineCheck(rsb200_lookup_plan_create(engine(), &job, 1, tableStorage.data(), 1, ditherTable ? 1 : 0,
                                        &pg.p),
              "rsb200_lookup_plan_create");
  engineCheck(rsb200_plan_run_host_image(pg.p, nullptr, 0, storage, (uint32_t)pitch,
                                         (uint32_t)(uncropped_dim.x * (int)bpp),
                                         (uint32_t)uncropped_dim.y, /*partial=*/1),
              "rsb200_plan_run_host_image");
}

// RawImageData::createBadPixelMap + transferBadPixelsToMap (common/RawImage.cpp:201-229)
void RawImageData::transferBadPixelsToMap() {
  std::lock_guard<std::mutex> guard(mBadPixelMutex);
  if (mBadPixelPositions.empty())
    return;
  if (mBadPixelMap.empty()) {
    if (!isAllocated())
      ThrowRDE("(internal) Bad pixel map cannot be allocated before image.");
    mBadPixelMapPitch = (uint32_t)((((uint32_t)uncropped_dim.x + 7) / 8 + 15) / 16 * 16);
    mBadPixelMap.assign((size_t)mBadPixelMapPitch * (size_t)uncropped_dim.y, 0);
  }
  for (const uint32_t pos : mBadPixelPositions) {
    const uint32_t pos_x = pos & 0xffff, pos_y = pos >> 16;
    if ((int)pos_x >= uncropped_dim.x || (int)pos_y >= uncropped_dim.y) // (an assert in the reference)
      ThrowRDE("Bad pixel position (%u, %u) outside the image", pos_x, pos_y);
    mBadPixelMap[(size_t)mBadPixelMapPitch * pos_y + (pos_x >> 3)] |= (uint8_t)(1 << (pos_x & 7));
  }
  mBadPixelPositions.clear();
}

// RawImageData::fixBadPixels (:231-239): FIX_BAD_PIXELS over the whole map, on the device
void RawImageData::fixBadPixels() {
  transferBadPixelsToMap();
  if (mBadPixelMap.empty())
    return;
  if (dataType != RawImageType::UINT16)
    ThrowRDE("rawspeed_b200: fixBadPixels is implemented for UINT16 images");
  if (cpp != 1)
    ThrowRDE("rawspeed_b200: fixBadPixels is implemented for 1 component per pixel (the "
             "reference's result for %u depends on its visiting order)", cpp);
  rsb200_badpix_job job;
  std::memset(&job, 0, sizeof job);
  job.offset = 0;
  job.pitch = (uint32_t)pitch;
  job.width = (uint32_t)uncropped_dim.x;
  job.height = (uint32_t)uncropped_dim.y;
  job.is_cfa = isCFA ? 1u : 0u;
  job.first_position = 0;
  job.num_positions = 0;
  job.prior_map = mBadPixelMap.data();
  PlanGuard pg;
  engineCheck(rsb200_badpix_plan_create(engine(), &job, 1, nullptr, 0, &pg.p),
              "rsb200_badpix_plan_create");
  engineCheck(rsb200_plan_run_host_image(pg.p, nullptr, 0, storage, (uint32_t)pitch,
                                         (uint32_t)(uncropped_dim.x * (int)bpp),
                                         (uint32_t)uncropped_dim.y, /*partial=*/1),
              "rsb200_plan_run_host_image");
}

// RawImageDataU16::calculateBlackAreas (common/RawImageDataU16.cpp:60-145): per CFA position,
// the median of the masked areas -- 16-bit histogram counters and the one sampled column / row
// (the FIXMEs at :87, :103) as the reference has them.  Host work: the areas are a few rows.
void RawImageData::calculateBlackAreas() {
  const uint16_t* img = reinterpret_cast<const uint16_t*>(storage);
  const size_t pitchElts = (size_t)pitch / 2;
  std::vector<uint16_t> histogram(4 * 65536, 0);
  int totalpixels = 0;
  for (BlackArea area : blackAreas) {
    area.size = area.size - (area.size & 1);
    if (!area.isVertical) {
      if ((int)area.offset + (int)area.size > uncropped_dim.y)
        ThrowRDE("Offset + size is larger than height of image");
      for (uint32_t y = area.offset; y < area.offset + area.size; y++)
        for (int x = mOffset.x; x < dim.x + mOffset.x; x++)
          histogram[(size_t)((2 * (y & 1)) + (x & 1)) * 65536 + img[y * pitchElts + mOffset.x]]++;
      totalpixels += area.size * dim.x;
    } else {
      if ((int)area.offset + (int)area.size > uncropped_dim.x)
        ThrowRDE("Offset + size is larger than width of image");
      for (int y = mOffset.y; y < dim.y + mOffset.y; y++)
        for (uint32_t x = area.offset; x < area.size + area.offset; x++)
          histogram[(size_t)((2 * (y & 1)) + (x & 1)) * 65536 + img[(size_t)y * pitchElts + area.offset]]++;
      totalpixels += area.size * dim.y;
    }
  }
  blackLevelSeparate = Array2DRef<int>(blackLevelSeparateStorage.data(), 2, 2);
  if (!totalpixels) {
    for (int& i : blackLevelSeparateStorage)
      i = blackLevel;
    return;
  }
  totalpixels /= 4 * 2;
  for (int i = 0; i < 4; i++) {
    const uint16_t* localhist = &histogram[(size_t)i * 65536];
    int acc_pixels = localhist[0];
    int pixel_value = 0;
    while (acc_pixels <= totalpixels && pixel_value < 65535) {
      pixel_value++;
      acc_pixels += localhist[pixel_value];
    }
    blackLevelSeparateStorage[i] = pixel_value;
  }
  if (!isCFA) {
    int total = 0;
    for (int i : blackLevelSeparateStorage)
      total += i;
    for (int& i : blackLevelSeparateStorage)
      i = (total + 2) >> 2;
  }
}

// RawImageDataU16::scaleBlackWhite (common/RawImageDataU16.cpp:147-183) up to the worker
// launch: false = the reference returns without scaling
bool RawImageData::prepareScaleBlackWhite() {
  if (dataType != RawImageType::UINT16)
    ThrowRDE("rawspeed_b200: scaleBlackWhite is implemented for UINT16 images");
  if (!isAllocated())
    ThrowRDE("scaleBlackWhite: image has no data");
  const int skipBorder = 250;
  const int gw = (dim.x - skipBorder) * (int)cpp;
  if ((blackAreas.empty() && !blackLevelSeparate && blackLevel < 0) || !whitePoint) { // estimate
    int b = 65536;
    int m = 0;
    const uint16_t* img = reinterpret_cast<const uint16_t*>(storage);
    for (int row = skipBorder; row < (dim.y - skipBorder); row++) {
      const uint16_t* p = img + (size_t)(mOffset.y + row) * ((size_t)pitch / 2) + (size_t)mOffset.x * cpp;
      for (int col = skipBorder; col < gw; col++) {
        const int pixel = p[skipBorder + col];
        b = std::min(pixel, b);
        m = std::max(pixel, m);
      }
    }
    if (blackLevel < 0)
      blackLevel = b;
    if (!whitePoint)
      whitePoint = m;
  }
  // nothing to do (:173-177)
  if ((blackAreas.empty() && blackLevel == 0 && whitePoint == 65535 && !blackLevelSeparate) ||
      dim.area() <= 0)
    return false;
  if (!blackLevelSeparate)
    calculateBlackAreas();
  return true;
}

void RawImageData::scaleBlackWhite(int path) {
  if (!prepareScaleBlackWhite())
    return;
  // startWorker(SCALE_VALUES): the per-sample pass, on the device
  rsb200_scale_job job;
  std::memset(&job, 0, sizeof job);
  job.offset = 0;
  job.pitch = (uint32_t)pitch;
  job.width = (uint32_t)uncropped_dim.x;
  job.height = (uint32_t)uncropped_dim.y;
  job.cpp = cpp;
  job.crop_x = (uint32_t)mOffset.x;
  job.crop_y = (uint32_t)mOffset.y;
  job.crop_w = (uint32_t)dim.x;
  job.crop_h = (uint32_t)dim.y;
  for (int i = 0; i < 4; ++i)
    job.black_separate[i] = blackLevelSeparateStorage[i];
  job.white_point = *whitePoint;
  job.dither = mDitherScale ? 1 : 0;
  job.path = (uint8_t)path;
  PlanGuard pg;
  engineCheck(rsb200_scale_plan_create(engine(), &job, 1, &pg.p), "rsb200_scale_plan_create");
  engineCheck(rsb200_plan_run_host_image(pg.p, nullptr, 0, storage, (uint32_t)pitch,
                                         (uint32_t)(uncropped_dim.x * (int)bpp),
                                         (uint32_t)uncropped_dim.y, /*partial=*/1),
              "rsb200_plan_run_host_image");
}

void RawImageData::setError(const std::string& err) {
  std::lock_guard<std::mutex> g(errMutex);
  errors.push_back(err);
}
bool RawImageData::isTooManyErrors(unsigned many, std::string* firstErr) {
  std::lock_guard<std::mutex> g(errMutex);
  if (errors.size() < many)
    return false;
  if (firstErr)
    *firstErr = errors[0];
  return true;
}
std::vector<std::string> RawImageData::getErrors() {
  std::lock_guard<std::mutex> g(errMutex);
  return errors;
}

RawImage RawImage::create(const iPoint2D& dim, RawImageType type, uint32_t cpp) {
  RawImage r;
  r.p_ = std::make_shared<RawImageData>();
  r.p_->dim = dim;
  r.p_->dataType = type;
  r.p_->cpp = cpp;
  r.p_->bpp = (type == RawImageType::F32 ? 4u : 2u) * cpp; // RawImageDataFloat / U16 ctors
  r.p_->createData();
  return r;
}

// TableLookUp::TableLookUp(1, dither) + setTable(0, table) (common/TableLookUp.cpp:40-85)
void RawImageData::setTable(const std::vector<uint16_t>& table, bool dither) {
  constexpr int MAXE = 65536;
  const int nfilled = (int)table.size();
  if (nfilled == 0)
    ThrowRDE("Table lookup with 0 entries is unsupported");
  if (nfilled > MAXE)
    ThrowRDE("Table lookup with %i entries is unsupported", nfilled);
  ditherTable = dither;
  tableStorage.assign((size_t)MAXE * 2, 0);
  if (!dither) {
    for (int i = 0; i < MAXE; ++i)
      tableStorage[i] = (i < nfilled) ? table[i] : table[nfilled - 1];
    return;
  }
  for (int i = 0; i < nfilled; ++i) {
    const int center = table[i];
    int lower = i > 0 ? table[i - 1] : center;
    int upper = i < (nfilled - 1) ? table[i + 1] : center;
    lower = std::min(lower, center); // non-monotonic LUT: no interpolation across the cross-over
    upper = std::max(upper, center);
    const int delta = upper - lower;
    const int base = center - ((upper - lower + 2) / 4);
    tableStorage[(size_t)i * 2] = (uint16_t)std::min(std::max(base, 0), 65535);
    tableStorage[(size_t)i * 2 + 1] = (uint16_t)delta;
  }
  for (int i = nfilled; i < MAXE; ++i) {
    tableStorage[(size_t)i * 2] = table[nfilled - 1];
    tableStorage[(size_t)i * 2 + 1] = 0;
  }
}

// ------------------------------------------------------------------ Huffman
template <typename Tag> uint32_t HuffmanCode<Tag>::setNCodesPerLength(Buffer data) {
  if (data.getSize() != 16)
    ThrowRDE("Codes-per-length table must have 16 entries");
  uint32_t cnt = 0;
  int maxLen = 0;
  for (int l = 1; l <= 16; ++l) {
    nCodesPerLength[l - 1] = data.begin()[l - 1];
    cnt += nCodesPerLength[l - 1];
    if (nCodesPerLength[l - 1])
      maxLen = l;
  }
  if (maxLen == 0)
    ThrowRDE("Codes-per-length table is empty");
  if (cnt > 162)
    ThrowRDE("Too big code-values table");
  // a code of length l needs a free node at depth l (Kraft)
  unsigned freeNodes = 2;
  for (int l = 1; l <= maxLen; ++l) {
    const unsigned n = nCodesPerLength[l - 1];
    if (n > (1U << l))
      ThrowRDE("Corrupt Huffman. Can never have %u codes in %d-bit len", n, l);
    if (n > freeNodes)
      ThrowRDE("Corrupt Huffman. Can only fit %u out of %u codes in %d-bit len", freeNodes, n, l);
    freeNodes = (freeNodes - n) * 2;
  }
  count = cnt;
  return cnt;
}

template <typename Tag> void HuffmanCode<Tag>::setCodeValues(const uint8_t* values, int n) {
  if ((uint32_t)n != count)
    ThrowRDE("Malformed code");
  codeValues.assign(values, values + n);
}

template <typename Tag> void PrefixCodeDecoder<Tag>::setup(bool fullDecode_, bool fixDNGBug16_) {
  fullDecode = fullDecode_;
  fixDNGBug16 = fixDNGBug16_;
  if (code.codeValues.empty())
    ThrowRDE("Empty code alphabet?");
  if (fullDecode)
    for (uint8_t v : code.codeValues)
      if (v > 16)
        ThrowRDE("Corrupt Huffman code: difference length %u longer than %u", v, 16);
}

template <typename Tag> rsb200_huff_table PrefixCodeDecoder<Tag>::deviceTable() const {
  rsb200_huff_table t;
  std::memset(&t, 0, sizeof t);
  std::memcpy(t.ncodes_per_len, code.nCodesPerLength.data(), 16);
  std::memcpy(t.values, code.codeValues.data(), code.codeValues.size());
  t.nvalues = (uint16_t)code.codeValues.size();
  t.fix_dng16 = fixDNGBug16 ? 1 : 0;
  return t;
}

template class HuffmanCode<BaselineCodeTag>;
template class PrefixCodeDecoder<BaselineCodeTag>;

static uint8_t tableIndex(std::vector<rsb200_huff_table>& tables, const rsb200_huff_table& t) {
  for (size_t i = 0; i < tables.size(); ++i)
    if (!std::memcmp(&tables[i], &t, sizeof t))
      return (uint8_t)i;
  if (tables.size() >= 255)
    ThrowRDE("Too many distinct Huffman tables in one batch");
  tables.push_back(t);
  return (uint8_t)(tables.size() - 1);
}

// ------------------------------------------------------------------ K1
UncompressedDecompressor::UncompressedDecompressor(ByteStream input_, RawImage img_,
                                                   const iRectangle2D& crop,
                                                   int inputPitchBytes_, int bitPerPixel_,
                                                   BitOrder order_)
    : input(input_.getStream((uint32_t)crop.dim.y, (uint32_t)inputPitchBytes_)),
      mRaw(std::move(img_)), size(crop.dim), offset(crop.pos),
      inputPitchBytes(inputPitchBytes_), bitPerPixel(bitPerPixel_), order(order_) {
  if (!size.hasPositiveArea())
    ThrowRDE("Empty tile.");
  if (inputPitchBytes < 1)
    ThrowRDE("Input pitch is non-positive");
  if (order == BitOrder::JPEG)
    ThrowRDE("JPEG bit order not supported.");
  const uint32_t w = size.x, h = size.y, cpp = mRaw->getCpp();
  const uint64_t ox = offset.x, oy = offset.y;
  if (cpp < 1 || cpp > 3)
    ThrowRDE("Unsupported number of components per pixel: %u", cpp);
  if (bitPerPixel < 1 || bitPerPixel > 32 ||
      (bitPerPixel > 16 && mRaw->getDataType() == RawImageType::UINT16))
    ThrowRDE("Unsupported bit depth");
  const uint64_t outPixelBits = (uint64_t)w * cpp * bitPerPixel;
  if (outPixelBits % 8 != 0)
    ThrowRDE("Bad combination of cpp (%u), bps (%d) and width (%u), the pitch is %llu bits, "
             "which is not a multiple of 8 (1 byte)",
             cpp, bitPerPixel, w, (unsigned long long)outPixelBits);
  const uint64_t outPixelBytes = outPixelBits / 8;
  if ((uint64_t)(unsigned)inputPitchBytes < outPixelBytes)
    ThrowRDE("Specified pitch is smaller than minimally-required pitch");
  const uint32_t fullRows = input.getRemainSize() / (uint32_t)inputPitchBytes;
  if (fullRows < h) {
    if (fullRows == 0)
      ThrowIOE("Not enough data to decode a single line. Image file truncated.");
    ThrowIOE("Image truncated, only %u of %u lines found", fullRows, h);
  }
  skipBytes = (uint32_t)(inputPitchBytes - outPixelBytes);
  if (oy > (uint64_t)mRaw->dim.y)
    ThrowRDE("Invalid y offset");
  if (ox + size.x > (uint64_t)mRaw->dim.x)
    ThrowRDE("Invalid x offset");
}

bool UncompressedDecompressor::describe(const uint8_t* fileBase, rsb200_unpack_job* job) const {
  const uint32_t cpp = mRaw->getCpp();
  const uint64_t oy = offset.y;
  const uint64_t hEnd = std::min<uint64_t>((uint64_t)size.y + oy, (uint64_t)mRaw->dim.y);
  const bool copy16 = (order == BitOrder::LSB && bitPerPixel == 16);
  if (!copy16 && input.getRemainSize() < 4) // BitStreamer ctor (BitStreamer.h:56-60)
    ThrowIOE("Bit stream size is smaller than MaxProcessBytes");
  if (hEnd <= oy)
    return false;
  std::memset(job, 0, sizeof *job);
  job->in_offset = (uint64_t)(input.begin() - fileBase);
  job->in_size = input.getRemainSize();
  job->out_offset = 0;
  job->out_pitch = mRaw->pitch;
  job->row0 = (int32_t)oy;
  job->rows = (int32_t)(hEnd - oy);
  job->samples = (int32_t)(size.x * (int)cpp);
  // packed integers ignore the crop's x offset (UncompressedDecompressor.cpp:196),
  // the 16-bit little-endian row copy honours it (:255-264)
  job->out_col0 = copy16 ? (int32_t)(offset.x * (int)cpp) : 0;
  job->in_pitch = inputPitchBytes;
  job->bps = bitPerPixel;
  job->order = (int32_t)order;
  return true;
}

// sanityCheck(const uint32_t* h, int bytesPerLine) (UncompressedDecompressor.cpp:52-74)
void UncompressedDecompressor::sanityCheck(uint32_t h, int bytesPerLine) const {
  const uint32_t fullRows = input.getRemainSize() / (uint32_t)bytesPerLine;
  if (fullRows >= h)
    return;
  if (fullRows == 0)
    ThrowIOE("Not enough data to decode a single line. Image file truncated.");
  ThrowIOE("Image truncated, only %u of %u lines found", fullRows, h);
}

// one device job over the whole stream for a fixed-layout form
void UncompressedDecompressor::runFixed(int format, uint32_t w, uint32_t h,
                                        uint32_t bytesPerLine) {
  if ((uint64_t)bytesPerLine * h > input.getRemainSize()) // ByteStream::getData
    ThrowIOE("Buffer overflow: image file may be truncated");
  rsb200_raw_job job;
  std::memset(&job, 0, sizeof job);
  job.in_offset = 0;
  job.in_size = input.getRemainSize();
  job.out_pitch = mRaw->pitch;
  job.rows = (int32_t)h;
  job.samples = (int32_t)w;
  job.in_pitch = (int32_t)bytesPerLine;
  job.format = format;
  PlanGuard pg;
  const uint16_t* tables = nullptr;
  std::vector<uint16_t> dev;
  if (format == RSB200_RAW_8BIT_TABLE) {
    // dithered table: decode8BitRaw's dither counter starts at 0 and the update
    // 15700*(r&65535)+(r>>16) keeps it there, so pix == base == tables[2*v]
    // (RawImage.h:335-353); the device gets one 65536-entry table either way
    const std::vector<uint16_t>& t = mRaw->tableData();
    dev.resize(65536);
    for (int i = 0; i < 65536; ++i)
      dev[i] = mRaw->tableDither() ? t[(size_t)2 * i] : t[i];
    tables = dev.data();
  }
  engineCheck(rsb200_raw_plan_create(engine(), &job, 1, tables, tables ? 1 : 0, &pg.p),
              "rsb200_raw_plan_create");
  runOnImage(pg.p, input.begin(), input.getRemainSize(), mRaw, /*partial=*/true);
}

template <bool uncorrectedRawValues> void UncompressedDecompressor::decode8BitRaw() {
  const uint32_t w = size.x, h = size.y;
  sanityCheck(h, (int)w);
  const bool lut = !uncorrectedRawValues && mRaw->hasTable();
  runFixed(lut ? RSB200_RAW_8BIT_TABLE : RSB200_RAW_8BIT, w, h, w);
}
template void UncompressedDecompressor::decode8BitRaw<false>();
template void UncompressedDecompressor::decode8BitRaw<true>();

template <Endianness e> void UncompressedDecompressor::decode12BitRawWithControl() {
  const uint32_t w = size.x, h = size.y;
  if ((12 * w) % 8 != 0) // bytesPerLine (UncompressedDecompressor.cpp:86-104)
    ThrowIOE("Bad image width");
  const uint32_t perline = (12 * w) / 8 + ((w + 2) / 10);
  sanityCheck(h, (int)perline);
  runFixed(e == Endianness::big ? RSB200_RAW_12BIT_CONTROL_BE : RSB200_RAW_12BIT_CONTROL_LE, w, h,
           perline);
}
template void UncompressedDecompressor::decode12BitRawWithControl<Endianness::little>();
template void UncompressedDecompressor::decode12BitRawWithControl<Endianness::big>();

template <Endianness e> void UncompressedDecompressor::decode12BitRawUnpackedLeftAligned() {
  const uint32_t w = size.x, h = size.y;
  sanityCheck(h, (int)(2 * w));
  runFixed(e == Endianness::big ? RSB200_RAW_12BIT_LEFT_BE : RSB200_RAW_12BIT_LEFT_LE, w, h, 2 * w);
}
template void UncompressedDecompressor::decode12BitRawUnpackedLeftAligned<Endianness::little>();
template void UncompressedDecompressor::decode12BitRawUnpackedLeftAligned<Endianness::big>();

// readUncompressedRaw() on an F32 image (UncompressedDecompressor.cpp:214-247): the job
// it amounts to.  false = nothing to decode.
bool UncompressedDecompressor::describeF32(const uint8_t* fileBase, rsb200_raw_job* job) const {
  const uint32_t cpp = mRaw->getCpp();
  const uint64_t oy = offset.y;
  const uint64_t hEnd = std::min<uint64_t>((uint64_t)size.y + oy, (uint64_t)mRaw->dim.y);
  int format;
  int32_t col0;
  if (bitPerPixel == 32) {
    format = RSB200_RAW_F32_COPY;
    col0 = (int32_t)(offset.x * (int)cpp);
    if (hEnd > oy && (uint64_t)inputPitchBytes * (hEnd - oy) > input.getRemainSize())
      ThrowIOE("Buffer overflow: image file may be truncated");
  } else if ((order == BitOrder::MSB || order == BitOrder::LSB) &&
             (bitPerPixel == 16 || bitPerPixel == 24)) {
    const bool msb = order == BitOrder::MSB;
    format = bitPerPixel == 16 ? (msb ? RSB200_RAW_FP16_MSB : RSB200_RAW_FP16_LSB)
                               : (msb ? RSB200_RAW_FP24_MSB : RSB200_RAW_FP24_LSB);
    col0 = (int32_t)offset.x; // decodePackedFP: out(row, offset.x + col)
    if (input.getRemainSize() < 4) // BitStreamer ctor (BitStreamer.h:56-60)
      ThrowIOE("Bit stream size is smaller than MaxProcessBytes");
  } else {
    ThrowRDE("Unsupported floating-point input bitwidth/bit packing: %d / %u", bitPerPixel,
             (unsigned)order);
  }
  if (hEnd <= oy)
    return false;
  std::memset(job, 0, sizeof *job);
  job->in_offset = (uint64_t)(input.begin() - fileBase);
  job->in_size = input.getRemainSize();
  job->out_pitch = mRaw->pitch;
  job->row0 = (int32_t)oy;
  job->rows = (int32_t)(hEnd - oy);
  job->samples = (int32_t)(size.x * (int)cpp);
  job->out_col0 = col0;
  job->in_pitch = inputPitchBytes;
  job->format = format;
  return true;
}

void UncompressedDecompressor::readF32() {
  rsb200_raw_job job;
  if (!describeF32(input.begin(), &job))
    return;
  PlanGuard pg;
  engineCheck(rsb200_raw_plan_create(engine(), &job, 1, nullptr, 0, &pg.p),
              "rsb200_raw_plan_create");
  runOnImage(pg.p, input.begin(), input.getRemainSize(), mRaw, /*partial=*/true);
}

void UncompressedDecompressor::readUncompressedRaw() {
  if (mRaw->getDataType() == RawImageType::F32) {
    readF32();
    return;
  }
  rsb200_unpack_job job;
  if (!describe(input.begin(), &job))
    return;
  PlanGuard pg;
  engineCheck(rsb200_unpack_plan_create(engine(), &job, 1, &pg.p), "rsb200_unpack_plan_create");
  runOnImage(pg.p, input.begin(), input.getRemainSize(), mRaw, /*partial=*/true);
}

// ------------------------------------------------------------------ Pentax
PentaxDecompressor::PentaxDecompressor(RawImage img, const ByteStream* metaData)
    : mRaw(std::move(img)), ht(SetupPrefixCodeDecoder(metaData)) {
  if (mRaw->getCpp() != 1 || mRaw->getDataType() != RawImageType::UINT16 ||
      mRaw->getBpp() != sizeof(uint16_t))
    ThrowRDE("Unexpected component count / data type");
  if (!mRaw->dim.x || !mRaw->dim.y || mRaw->dim.x % 2 != 0 || mRaw->dim.x > 8384 ||
      mRaw->dim.y > 6208)
    ThrowRDE("Unexpected image dimensions found: (%d; %d)", mRaw->dim.x, mRaw->dim.y);
}

HuffmanCode<> PentaxDecompressor::SetupPrefixCodeDecoder_Legacy() {
  // PentaxDecompressor::pentax_tree (PentaxDecompressor.cpp:46-53)
  static const uint8_t ncpl[16] = {0, 2, 3, 1, 1, 1, 1, 1, 1, 2, 0, 0, 0, 0, 0, 0};
  static const uint8_t vals[13] = {3, 4, 2, 5, 1, 6, 0, 7, 8, 9, 10, 11, 12};
  HuffmanCode<> hc;
  hc.setNCodesPerLength(Buffer(ncpl, 16));
  hc.setCodeValues(vals, 13);
  return hc;
}

HuffmanCode<> PentaxDecompressor::SetupPrefixCodeDecoder_Modern(ByteStream stream) {
  const uint32_t depth = (uint32_t)stream.getU16() + 12;
  if (depth > 15)
    ThrowRDE("Depth of huffman table is too great (%u).", depth);
  stream.skipBytes(12);
  uint32_t v0[16], v1[16], v2[16];
  for (uint32_t i = 0; i < depth; i++)
    v0[i] = stream.getU16();
  for (uint32_t i = 0; i < depth; i++) {
    v1[i] = stream.getByte();
    if (v1[i] == 0 || v1[i] > 12)
      ThrowRDE("Data corrupt: v1[%u]=%u, expected [1..12]", depth, v1[i]);
  }
  uint8_t nCodesPerLength[17] = {0};
  for (uint32_t c = 0; c < depth; c++) {
    v2[c] = v0[c] >> (12 - v1[c]); // extractHighBits(v0, v1, effectiveBitwidth = 12)
    nCodesPerLength[v1[c]]++;
  }
  HuffmanCode<> hc;
  hc.setNCodesPerLength(Buffer(nCodesPerLength + 1, 16));
  // code values in increasing code order: repeatedly the LAST index holding the minimum
  uint8_t codeValues[16];
  for (uint32_t i = 0; i < depth; i++) {
    uint32_t sm_val = 0xfffffff, sm_num = 0xff;
    for (uint32_t j = 0; j < depth; j++) {
      if (v2[j] <= sm_val) {
        sm_num = j;
        sm_val = v2[j];
      }
    }
    codeValues[i] = (uint8_t)sm_num;
    v2[sm_num] = 0xffffffff;
  }
  hc.setCodeValues(codeValues, (int)depth);
  return hc;
}

PrefixCodeDecoder<> PentaxDecompressor::SetupPrefixCodeDecoder(const ByteStream* metaData) {
  PrefixCodeDecoder<> d(metaData ? SetupPrefixCodeDecoder_Modern(*metaData)
                                 : SetupPrefixCodeDecoder_Legacy());
  d.setup(true, false);
  return d;
}

void PentaxDecompressor::decompress(ByteStream data) const {
  if (data.getRemainSize() < 4) // BitStreamerMSB ctor (BitStreamer.h:56-60)
    ThrowIOE("Bit stream size is smaller than MaxProcessBytes");
  rsb200_huff_table t = ht.deviceTable();
  rsb200_pentax_job job;
  std::memset(&job, 0, sizeof job);
  job.in_offset = 0;
  job.in_size = data.getRemainSize();
  job.table = 0;
  job.width = mRaw->dim.x;
  job.height = mRaw->dim.y;
  job.out_offset = 0;
  job.out_pitch = (uint32_t)mRaw->pitch;
  PlanGuard pg;
  engineCheck(rsb200_pentax_plan_create(engine(), &t, 1, &job, 1, &pg.p),
              "rsb200_pentax_plan_create");
  RawImage img = mRaw;
  runOnImage(pg.p, data.begin() + data.getPosition(), data.getRemainSize(), img,
             /*partial=*/true);
  rsb200_scan_result res;
  const int rc = rsb200_plan_results(pg.p, &res, 1);
  if (rc == RSB200_OK)
    return;
  if (res.status == RSB200_ERR_RDE && (res.consumed & RSB200_PENTAX_OOB)) {
    const uint32_t key = res.consumed & ~RSB200_PENTAX_OOB;
    ThrowRDE("decoded value out of bounds at %d:%d", (int)(key & 0x3FFFu), (int)(key >> 14));
  }
  if (res.status == RSB200_ERR_RDE)
    ThrowRDE("bad Huffman code");
  if (res.status == RSB200_ERR_IOE)
    ThrowIOE("Buffer overflow read in BitStreamer");
  engineCheck(rc, "rsb200_plan_results");
}

// ------------------------------------------------------------------ Samsung V0
SamsungV0Decompressor::SamsungV0Decompressor(const RawImage& image, ByteStream bso, ByteStream bsr)
    : mRaw(image) {
  if (mRaw->getCpp() != 1 || mRaw->getDataType() != RawImageType::UINT16 ||
      mRaw->getBpp() != sizeof(uint16_t))
    ThrowRDE("Unexpected component count / data type");
  const uint32_t width = mRaw->dim.x;
  const uint32_t height = mRaw->dim.y;
  if (width == 0 || height == 0 || width < 16 || width > 5546 || height > 3714)
    ThrowRDE("Unexpected image dimensions found: (%u; %u)", width, height);
  computeStripes(bso.getStream(height, 4), bsr); // (peekStream of a copy: the same check)
}

// SamsungV0Decompressor::computeStripes (SamsungV0Decompressor.cpp:61-90)
void SamsungV0Decompressor::computeStripes(ByteStream bso, ByteStream bsr) {
  const uint32_t height = mRaw->dim.y;
  std::vector<uint32_t> offsets;
  offsets.reserve(1 + height);
  for (uint32_t y = 0; y < height; y++)
    offsets.emplace_back(bso.getU32());
  offsets.emplace_back(bsr.getSize());
  stripes.reserve(height);
  bsr.skipBytes(offsets[0]);
  for (uint32_t y = 0; y < height; y++) {
    if (offsets[y] >= offsets[y + 1])
      ThrowRDE("Line offsets are out of sequence or slice is empty.");
    stripes.emplace_back(bsr.getStream(offsets[y + 1] - offsets[y]));
  }
}

void SamsungV0Decompressor::decompress() const {
  const uint32_t h = mRaw->dim.y;
  const uint8_t* base = stripes[0].begin();
  std::vector<rsb200_samsung0_strip> st(h);
  for (uint32_t r = 0; r < h; ++r) {
    st[r].in_offset = (uint64_t)(stripes[r].begin() - base);
    st[r].in_size = stripes[r].getSize();
    st[r].reserved = 0;
  }
  const size_t bytes = (size_t)(stripes[h - 1].begin() + stripes[h - 1].getSize() - base);
  rsb200_samsung0_job job;
  std::memset(&job, 0, sizeof job);
  job.out_offset = 0;
  job.out_pitch = (uint32_t)mRaw->pitch;
  job.width = mRaw->dim.x;
  job.height = h;
  job.first_strip = 0;
  PlanGuard pg;
  engineCheck(rsb200_samsung0_plan_create(engine(), &job, 1, st.data(), (int)h, &pg.p),
              "rsb200_samsung0_plan_create");
  RawImage img = mRaw;
  runOnImage(pg.p, base, bytes, img, /*partial=*/true);
  rsb200_scan_result res;
  const int rc = rsb200_plan_results(pg.p, &res, 1);
  if (rc == RSB200_OK)
    return;
  switch (res.consumed >> 24) { // SamsungV0Decompressor.cpp:147-160, BitStreamer.h:56-59, :96-104
  case RSB200_S0_LEN_NEG:
    ThrowRDE("Bit length less than 0.");
  case RSB200_S0_LEN_BIG:
    ThrowRDE("Bit Length more than 16.");
  case RSB200_S0_UP_FIRST:
    ThrowRDE("Upward prediction for the first two rows. Raw corrupt");
  case RSB200_S0_UP_LAST:
    ThrowRDE("Upward prediction for the last block of pixels. Raw corrupt");
  case RSB200_S0_OVERREAD:
    ThrowIOE("Buffer overflow read in BitStreamer");
  case RSB200_S0_SHORT:
    ThrowIOE("Bit stream size is smaller than MaxProcessBytes");
  default:
    engineCheck(rc, "rsb200_plan_results");
  }
}

// ------------------------------------------------------------------ Samsung V1
SamsungV1Decompressor::SamsungV1Decompressor(const RawImage& image, ByteStream bs_, int bit)
    : mRaw(image), bs(bs_) {
  if (mRaw->getCpp() != 1 || mRaw->getDataType() != RawImageType::UINT16 ||
      mRaw->getBpp() != sizeof(uint16_t))
    ThrowRDE("Unexpected component count / data type");
  if (bit != 12)
    ThrowRDE("Unexpected bit per pixel (%d)", bit);
  const uint32_t w = mRaw->dim.x;
  const uint32_t h = mRaw->dim.y;
  if (w == 0 || h == 0 || w % 32 != 0 || h % 2 != 0 || w > 5664 || h > 3714)
    ThrowRDE("Unexpected image dimensions found: (%u; %u)", w, h);
}

void SamsungV1Decompressor::decompress() const {
  if (bs.getRemainSize() < 4) // BitStreamerMSB ctor (BitStreamer.h:56-60)
    ThrowIOE("Bit stream size is smaller than MaxProcessBytes");
  rsb200_samsung1_job job;
  std::memset(&job, 0, sizeof job);
  job.in_offset = 0;
  job.in_size = bs.getRemainSize();
  job.bits = 12;
  job.width = mRaw->dim.x;
  job.height = mRaw->dim.y;
  job.out_offset = 0;
  job.out_pitch = (uint32_t)mRaw->pitch;
  PlanGuard pg;
  engineCheck(rsb200_samsung1_plan_create(engine(), &job, 1, &pg.p), "rsb200_samsung1_plan_create");
  RawImage img = mRaw;
  runOnImage(pg.p, bs.begin() + bs.getPosition(), bs.getRemainSize(), img, /*partial=*/true);
  rsb200_scan_result res;
  const int rc = rsb200_plan_results(pg.p, &res, 1);
  if (rc == RSB200_OK)
    return;
  if (res.status == RSB200_ERR_RDE)
    ThrowRDE("decoded value out of bounds"); // SamsungV1Decompressor.cpp:135-136
  if (res.status == RSB200_ERR_IOE)
    ThrowIOE("Buffer overflow read in BitStreamer");
  engineCheck(rc, "rsb200_plan_results");
}

// ------------------------------------------------------------------ Samsung V2
// bits [pos, pos + n) of the 16-byte header read as MSB32 (SamsungV2Decompressor.cpp:103-131)
static uint32_t samsung2HeaderBits(const uint8_t* hd, uint32_t pos, uint32_t n) {
  uint32_t v = 0;
  for (uint32_t b = pos; b < pos + n; ++b) {
    const uint8_t* w = hd + 4 * (b >> 5);
    const uint32_t word = (uint32_t)w[0] | (uint32_t)w[1] << 8 | (uint32_t)w[2] << 16 | (uint32_t)w[3] << 24;
    v = v << 1 | ((word >> (31u - (b & 31u))) & 1u);
  }
  return v;
}

SamsungV2Decompressor::SamsungV2Decompressor(const RawImage& image, ByteStream bs_, unsigned bits_)
    : mRaw(image), bs(bs_), bits(bits_) {
  if (mRaw->getCpp() != 1 || mRaw->getDataType() != RawImageType::UINT16 ||
      mRaw->getBpp() != sizeof(uint16_t))
    ThrowRDE("Unexpected component count / data type");
  if (bits != 12 && bits != 14)
    ThrowRDE("Unexpected bit per pixel (%u)", bits);
  (void)bs.check(16);
  const uint8_t* hd = bs.begin() + bs.getPosition();
  const uint32_t depth = samsung2HeaderBits(hd, 20, 4) + 1;
  if (depth != bits)
    ThrowRDE("Bit depth mismatch with container, %u vs %u", depth, bits);
  const uint32_t flags = samsung2HeaderBits(hd, 84, 4);
  if (flags > 7)
    ThrowRDE("Invalid opt flags %x", flags);
  const int width = (int)samsung2HeaderBits(hd, 32, 16), height = (int)samsung2HeaderBits(hd, 48, 16);
  if (width == 0 || height == 0 || width % 16 != 0 || width > 6496 || height > 4336)
    ThrowRDE("Unexpected image dimensions found: (%i; %i)", width, height);
  if (width != mRaw->dim.x || height != mRaw->dim.y)
    ThrowRDE("EXIF image dimensions do not match dimensions from raw header");
}

void SamsungV2Decompressor::decompress() const {
  rsb200_samsung2_job job;
  std::memset(&job, 0, sizeof job);
  job.in_offset = 0;
  // A frame reads at most 283 bits per block (scale 2 + 12, motion 1 + 3, skip 1, flags 8, lengths 16,
  // differences 16 x 15) and skips at most 15 bytes per row; more data behind that (and the pump's
  // 8-byte over-read) changes no outcome, so the plan gets no more of it.
  const uint64_t most = 16 + (uint64_t)mRaw->dim.y * ((283ull * (mRaw->dim.x / 16) + 7) / 8 + 15) + 64;
  job.in_size = (uint32_t)std::min<uint64_t>(bs.getRemainSize(), most);
  job.bits = bits;
  job.width = mRaw->dim.x;
  job.height = mRaw->dim.y;
  std::memcpy(job.header, bs.begin() + bs.getPosition(), 16);
  job.out_offset = 0;
  job.out_pitch = (uint32_t)mRaw->pitch;
  PlanGuard pg;
  engineCheck(rsb200_samsung2_plan_create(engine(), &job, 1, &pg.p), "rsb200_samsung2_plan_create");
  RawImage img = mRaw;
  runOnImage(pg.p, bs.begin() + bs.getPosition(), job.in_size, img, /*partial=*/true);
  rsb200_scan_result res;
  const int rc = rsb200_plan_results(pg.p, &res, 1);
  if (rc == RSB200_OK)
    return;
  const unsigned value = (res.consumed >> 22) & 31u;
  switch (res.consumed >> 28) { // SamsungV2Decompressor.cpp:180-247, 329-350; BitStreamer.h; ByteStream.h
  case RSB200_S2_START_MOTION:
    ThrowRDE("At start of image and motion isn't 7. File corrupted?");
  case RSB200_S2_MOTION_BEGIN:
    ThrowRDE("Bad motion %d at the beginning of the row", (int)value);
  case RSB200_S2_MOTION_END:
    ThrowRDE("Bad motion %d at the end of the row", (int)value);
  case RSB200_S2_UNDERFLOW:
    ThrowRDE("Difference bits underflow. File corrupted?");
  case RSB200_S2_TOO_MANY:
    ThrowRDE("Too many difference bits (%u). File corrupted?", value);
  case RSB200_S2_OVERREAD:
    ThrowIOE("Buffer overflow read in BitStreamer");
  case RSB200_S2_SHORT:
    ThrowIOE("Bit stream size is smaller than MaxProcessBytes");
  case RSB200_S2_BYTESTREAM:
    ThrowIOE("Out of bounds access in ByteStream");
  default:
    engineCheck(rc, "rsb200_plan_results");
  }
}

// ------------------------------------------------------------------ Kodak DCR
KodakDecompressor::KodakDecompressor(RawImage img, ByteStream bs, int bps_, bool uncorrectedRawValues_)
    : mRaw(std::move(img)), input(bs), bps(bps_), uncorrectedRawValues(uncorrectedRawValues_) {
  if (mRaw->getCpp() != 1 || mRaw->getDataType() != RawImageType::UINT16 ||
      mRaw->getBpp() != sizeof(uint16_t))
    ThrowRDE("Unexpected component count / data type");
  if (!mRaw->dim.hasPositiveArea() || mRaw->dim.x % 4 != 0 || mRaw->dim.x > 4516 || mRaw->dim.y > 3012)
    ThrowRDE("Unexpected image dimensions found: (%d; %d)", mRaw->dim.x, mRaw->dim.y);
  if (bps != 10 && bps != 12)
    ThrowRDE("Unexpected bits per sample: %i", bps);
  // Lower estimate: this decompressor requires *at least* half a byte per output pixel
  (void)input.check((uint32_t)((uint64_t)mRaw->dim.area() / 2ULL));
}

void KodakDecompressor::decompress() const {
  rsb200_kodak_job job;
  std::memset(&job, 0, sizeof job);
  job.in_offset = 0;
  // A row reads at most 608 bytes per full segment (128 of lengths, 4 * ceil(15 * 256 / 32) of
  // differences) and the tail's maximum; more data behind that changes no outcome.
  const uint32_t w = (uint32_t)mRaw->dim.x, t = w % 256u, e = (t & 7u) == 4u ? 2u : 0u;
  const uint64_t tailMax = t ? t / 2u + e + 4u * ((15u * t > 8u * e ? 15u * t - 8u * e + 31u : 0u) / 32u) : 0u;
  const uint64_t most = (uint64_t)mRaw->dim.y * (608ull * (w / 256u) + tailMax);
  job.in_size = (uint32_t)std::min<uint64_t>(input.getRemainSize(), most);
  job.width = mRaw->dim.x;
  job.height = mRaw->dim.y;
  job.bps = bps;
  job.out_offset = 0;
  job.out_pitch = (uint32_t)mRaw->pitch;
  // setWithLookUp (RawImage.h:335-353): the dither counter starts at 0 and stays there, so a dithered
  // table reads entry 2 * v exactly; the device gets one 65536-entry table either way
  const bool lut = !uncorrectedRawValues && mRaw->hasTable();
  std::vector<uint16_t> dev;
  if (lut) {
    const std::vector<uint16_t>& tab = mRaw->tableData();
    dev.resize(65536);
    for (int i = 0; i < 65536; ++i)
      dev[i] = mRaw->tableDither() ? tab[(size_t)2 * i] : tab[i];
  }
  job.table = lut ? 0 : -1;
  PlanGuard pg;
  engineCheck(rsb200_kodak_plan_create(engine(), &job, 1, lut ? dev.data() : nullptr, lut ? 1 : 0, &pg.p),
              "rsb200_kodak_plan_create");
  RawImage img = mRaw;
  runOnImage(pg.p, input.begin() + input.getPosition(), job.in_size, img, /*partial=*/true);
  rsb200_scan_result res;
  const int rc = rsb200_plan_results(pg.p, &res, 1);
  if (rc == RSB200_OK)
    return;
  switch (res.consumed >> 28) { // KodakDecompressor.cpp:137-138; Buffer.h:78-83
  case RSB200_KODAK_VALUE: {
    int32_t value = 0;
    engineCheck(rsb200_kodak_plan_values(pg.p, &value, 1), "rsb200_kodak_plan_values");
    ThrowRDE("Value out of bounds %d (bps = %i)", (int)value, bps);
  }
  case RSB200_KODAK_OVERFLOW:
    ThrowIOE("Buffer overflow: image file may be truncated");
  default:
    engineCheck(rc, "rsb200_plan_results");
  }
}

// ------------------------------------------------------------------ GoPro VC-5
VC5Decompressor::VC5Decompressor(ByteStream bs, const RawImage& img, int phase, const rsb200_vc5_code* codes_,
                                 int ncodes)
    : mRaw(img), mBs(bs), codes(codes_, codes_ + (ncodes > 0 ? ncodes : 0)) {
  if (mRaw->getCpp() != 1 || mRaw->getDataType() != RawImageType::UINT16 || mRaw->getBpp() != sizeof(uint16_t))
    ThrowRDE("Unexpected component count / data type");
  rsb200_vc5::Parsed p;
  const rsb200_vc5::Outcome o = rsb200_vc5::parse(mBs.begin() + mBs.getPosition(), mBs.getRemainSize(), mRaw->dim.x,
                                                  mRaw->dim.y, mRaw->whitePoint.value_or(0), phase, p);
  if (o.cls == rsb200_vc5::IOE)
    ThrowIOE("%s", o.msg.c_str());
  if (o.cls != rsb200_vc5::OK)
    ThrowRDE("%s", o.msg.c_str());
  job = p.job;
  std::memcpy(bands, p.bands, sizeof bands);
}

void VC5Decompressor::decode(unsigned int offsetX, unsigned int offsetY, unsigned int width, unsigned int height) {
  if (offsetX || offsetY || mRaw->dim.x != (int)width || mRaw->dim.y != (int)height)
    ThrowRDE("VC5Decompressor expects to fill the whole image, not some tile.");
  job.out_offset = 0;
  job.out_pitch = (uint32_t)mRaw->pitch;
  PlanGuard pg;
  engineCheck(rsb200_vc5_plan_create(engine(), codes.data(), (int)codes.size(), &job, 1, bands, 40, &pg.p),
              "rsb200_vc5_plan_create");
  RawImage img = mRaw;
  // partial: a failed frame leaves the image as it was
  runOnImage(pg.p, mBs.begin() + mBs.getPosition(), mBs.getRemainSize(), img, /*partial=*/true);
  rsb200_scan_result res;
  const int rc = rsb200_plan_results(pg.p, &res, 1);
  if (rc == RSB200_OK)
    return;
  if (rc != RSB200_ERR_RDE && rc != RSB200_ERR_IOE)
    engineCheck(rc, "rsb200_plan_results");
  mRaw->setError(rsb200_vc5::band_failure(res.consumed).msg);
  std::string firstErr;
  if (mRaw->isTooManyErrors(1, &firstErr))
    ThrowRDE("Too many errors encountered. Giving up. First Error:\n%s", firstErr.c_str());
}

// ------------------------------------------------------------------ Sony ARW1
SonyArw1Decompressor::SonyArw1Decompressor(RawImage img) : mRaw(std::move(img)) {
  if (mRaw->getCpp() != 1 || mRaw->getDataType() != RawImageType::UINT16 ||
      mRaw->getBpp() != sizeof(uint16_t))
    ThrowRDE("Unexpected component count / data type");
  const uint32_t w = mRaw->dim.x;
  const uint32_t h = mRaw->dim.y;
  if (w == 0 || h == 0 || h % 2 != 0 || w > 4600 || h > 3072)
    ThrowRDE("Unexpected image dimensions found: (%u; %u)", w, h);
}

void SonyArw1Decompressor::decompress(ByteStream input) const {
  if (input.getRemainSize() < 4) // BitStreamerMSB ctor (BitStreamer.h:56-60)
    ThrowIOE("Bit stream size is smaller than MaxProcessBytes");
  rsb200_arw1_job job;
  std::memset(&job, 0, sizeof job);
  job.in_offset = 0;
  job.in_size = input.getRemainSize();
  job.width = mRaw->dim.x;
  job.height = mRaw->dim.y;
  job.out_offset = 0;
  job.out_pitch = (uint32_t)mRaw->pitch;
  PlanGuard pg;
  engineCheck(rsb200_arw1_plan_create(engine(), &job, 1, &pg.p), "rsb200_arw1_plan_create");
  RawImage img = mRaw;
  runOnImage(pg.p, input.begin() + input.getPosition(), input.getRemainSize(), img,
             /*partial=*/true);
  rsb200_scan_result res;
  const int rc = rsb200_plan_results(pg.p, &res, 1);
  if (rc == RSB200_OK)
    return;
  if (res.status == RSB200_ERR_RDE)
    ThrowRDE("Error decompressing"); // SonyArw1Decompressor.cpp:86-87
  if (res.status == RSB200_ERR_IOE)
    ThrowIOE("Buffer overflow read in BitStreamer");
  engineCheck(rc, "rsb200_plan_results");
}

// ------------------------------------------------------------------ Nikon
namespace {
// NikonDecompressor::nikon_tree (NikonDecompressor.cpp:47-67)
const uint8_t kNikonTree[6][2][16] = {
    {{0, 1, 5, 1, 1, 1, 1, 1, 1, 2, 0, 0, 0, 0, 0, 0}, {5, 4, 3, 6, 2, 7, 1, 0, 8, 9, 11, 10, 12}},
    {{0, 1, 5, 1, 1, 1, 1, 1, 1, 2, 0, 0, 0, 0, 0, 0},
     {0x39, 0x5a, 0x38, 0x27, 0x16, 5, 4, 3, 2, 1, 0, 11, 12, 12}},
    {{0, 1, 4, 2, 3, 1, 2, 0, 0, 0, 0, 0, 0, 0, 0, 0}, {5, 4, 6, 3, 7, 2, 8, 1, 9, 0, 10, 11, 12}},
    {{0, 1, 4, 3, 1, 1, 1, 1, 1, 2, 0, 0, 0, 0, 0, 0},
     {5, 6, 4, 7, 8, 3, 9, 2, 1, 0, 10, 11, 12, 13, 14}},
    {{0, 1, 5, 1, 1, 1, 1, 1, 1, 1, 2, 0, 0, 0, 0, 0},
     {8, 0x5c, 0x4b, 0x3a, 0x29, 7, 6, 5, 4, 3, 2, 1, 0, 13, 14}},
    {{0, 1, 4, 2, 2, 3, 1, 2, 0, 0, 0, 0, 0, 0, 0, 0},
     {7, 6, 8, 5, 9, 4, 10, 3, 11, 12, 2, 0, 1, 13, 14}},
};
} // namespace

// createPrefixCodeDecoder<PrefixCodeDecoder<>> (:458-471)
PrefixCodeDecoder<> NikonDecompressor::createPrefixCodeDecoder(uint32_t sel) {
  HuffmanCode<> hc;
  const uint32_t count = hc.setNCodesPerLength(Buffer(kNikonTree[sel][0], 16));
  hc.setCodeValues(kNikonTree[sel][1], (int)count);
  PrefixCodeDecoder<> ht(std::move(hc));
  ht.setup(true, false);
  return ht;
}

// createCurve (:380-441)
std::vector<uint16_t> NikonDecompressor::createCurve(ByteStream& metadata, uint32_t bitsPS,
                                                     uint32_t v0, uint32_t v1, uint32_t* split) {
  if (v0 == 68 && v1 == 64) // Nikon Z7 12/14 bit compressed hack
    bitsPS -= 2;
  std::vector<uint16_t> curve(((1u << bitsPS) & 0x7fffu) + 1u);
  for (size_t i = 0; i < curve.size(); i++)
    curve[i] = (uint16_t)i;
  uint32_t step = 0;
  const uint32_t csize = metadata.getU16();
  if (csize > 1)
    step = (uint32_t)(curve.size() / (csize - 1));
  if (v0 == 68 && (v1 == 32 || v1 == 64) && step > 0) {
    if ((csize - 1) * step != curve.size() - 1)
      ThrowRDE("Bad curve segment count (%u)", csize);
    for (size_t i = 0; i < csize; i++)
      curve[i * step] = metadata.getU16();
    for (size_t i = 0; i < curve.size() - 1; i++) {
      const uint32_t b_scale = (uint32_t)(i % step);
      const uint32_t a_pos = (uint32_t)(i - b_scale), b_pos = a_pos + step;
      const uint32_t a_scale = step - b_scale;
      curve[i] = (uint16_t)((a_scale * curve[a_pos] + b_scale * curve[b_pos]) / step);
    }
    metadata.setPosition(562);
    *split = metadata.getU16();
  } else if (v0 != 70) {
    if (csize == 0 || csize > 0x4001)
      ThrowRDE("Don't know how to compute curve! csize = %u", csize);
    curve.resize(csize + 1UL);
    for (uint32_t i = 0; i < csize; i++)
      curve[i] = metadata.getU16();
  }
  curve.resize(curve.size() - 1); // and drop the last value
  return curve;
}

// ctor (:473-511)
NikonDecompressor::NikonDecompressor(RawImage raw, ByteStream metadata, uint32_t bitsPS_)
    : mRaw(std::move(raw)), bitsPS(bitsPS_) {
  if (mRaw->getCpp() != 1 || mRaw->getDataType() != RawImageType::UINT16 ||
      mRaw->getBpp() != sizeof(uint16_t))
    ThrowRDE("Unexpected component count / data type");
  if (!(mRaw->dim.x > 0 && mRaw->dim.y > 0) || mRaw->dim.x % 2 != 0 || mRaw->dim.x > 8288 ||
      mRaw->dim.y > 5520)
    ThrowRDE("Unexpected image dimensions found: (%d; %d)", mRaw->dim.x, mRaw->dim.y);
  if (bitsPS != 12 && bitsPS != 14)
    ThrowRDE("Invalid bpp found: %u", bitsPS);
  const uint32_t v0 = metadata.getByte();
  const uint32_t v1 = metadata.getByte();
  if (v0 == 73 || v1 == 88)
    metadata.skipBytes(2110);
  if (v0 == 70)
    huffSelect = 2;
  if (bitsPS == 14)
    huffSelect += 3;
  pUp[0][0] = metadata.getU16();
  pUp[1][0] = metadata.getU16();
  pUp[0][1] = metadata.getU16();
  pUp[1][1] = metadata.getU16();
  curve = createCurve(metadata, bitsPS, v0, v1, &split);
  // If the 'split' happens outside of the image, it does not actually happen.
  if (split >= (unsigned)mRaw->dim.y)
    split = 0;
}

// decompress (:540-560)
void NikonDecompressor::decompress(Buffer input, bool uncorrectedRawValues) {
  if (split != 0)
    ThrowRDE("rawspeed_b200: Nikon streams with a split (lossy after split) are not supported yet");
  if (input.getSize() < 4) // BitStreamerMSB ctor (BitStreamer.h:56-60)
    ThrowIOE("Bit stream size is smaller than MaxProcessBytes");
  // RawImageCurveGuard (common/RawImage.h): the curve is applied while decoding, dithered
  if (!uncorrectedRawValues)
    mRaw->setTable(curve, true);
  const PrefixCodeDecoder<> ht = createPrefixCodeDecoder(huffSelect);
  rsb200_huff_table t = ht.deviceTable();
  rsb200_nikon_job job;
  std::memset(&job, 0, sizeof job);
  job.in_offset = 0;
  job.in_size = input.getSize();
  job.table = 0;
  job.width = mRaw->dim.x;
  job.height = mRaw->dim.y;
  job.out_offset = 0;
  job.out_pitch = (uint32_t)mRaw->pitch;
  job.lut = uncorrectedRawValues ? -1 : 0;
  job.pup[0] = (uint16_t)pUp[0][0];
  job.pup[1] = (uint16_t)pUp[0][1];
  job.pup[2] = (uint16_t)pUp[1][0];
  job.pup[3] = (uint16_t)pUp[1][1];
  PlanGuard pg;
  engineCheck(rsb200_nikon_plan_create(engine(), &t, 1, &job, 1,
                                       uncorrectedRawValues ? nullptr : mRaw->tableData().data(),
                                       uncorrectedRawValues ? 0 : 1, &pg.p),
              "rsb200_nikon_plan_create");
  RawImage img = mRaw;
  runOnImage(pg.p, input.begin(), input.getSize(), img, /*partial=*/true);
  rsb200_scan_result res;
  const int rc = rsb200_plan_results(pg.p, &res, 1);
  // ~RawImageCurveGuard: the table stays (plain) for the consumer only when uncorrected
  if (uncorrectedRawValues)
    mRaw->setTable(curve, false);
  else
    mRaw->clearTable();
  if (rc == RSB200_OK)
    return;
  if (res.status == RSB200_ERR_RDE)
    ThrowRDE("bad Huffman code");
  if (res.status == RSB200_ERR_IOE)
    ThrowIOE("Buffer overflow read in BitStreamer");
  engineCheck(rc, "rsb200_plan_results");
}

// ------------------------------------------------------------------ Panasonic
namespace {
void panaCheckImage(const RawImage& mRaw) {
  if (mRaw->getCpp() != 1 || mRaw->getDataType() != RawImageType::UINT16 ||
      mRaw->getBpp() != sizeof(uint16_t))
    ThrowRDE("Unexpected component count / data type");
}
// the constructors' block accounting (V5 :87-112, V6 :163-175, V7 :50-63)
void panaCheckInput(const RawImage& mRaw, const ByteStream& input, int pixelsPerUnit,
                    uint64_t unitBytes, uint64_t unitsPerBlock) {
  if (!(mRaw->dim.x > 0 && mRaw->dim.y > 0) || mRaw->dim.x % pixelsPerUnit != 0)
    ThrowRDE("Unexpected image dimensions found: (%i; %i)", mRaw->dim.x, mRaw->dim.y);
  const uint64_t units = (uint64_t)mRaw->dim.x * (uint64_t)mRaw->dim.y / (uint64_t)pixelsPerUnit;
  const uint64_t numBlocks = (units + unitsPerBlock - 1) / unitsPerBlock;
  if ((uint64_t)input.getRemainSize() / (unitBytes * unitsPerBlock) < numBlocks)
    ThrowRDE("Insufficient count of input blocks for a given image");
}
void panaRun(const RawImage& mRaw, const ByteStream& input, int version, int bps) {
  rsb200_pana_job job;
  std::memset(&job, 0, sizeof job);
  job.in_offset = 0;
  job.in_size = input.getRemainSize();
  job.out_offset = 0;
  job.out_pitch = (uint32_t)mRaw->pitch;
  job.width = (uint32_t)mRaw->dim.x;
  job.height = (uint32_t)mRaw->dim.y;
  job.version = (uint8_t)version;
  job.bps = (uint8_t)bps;
  PlanGuard pg;
  engineCheck(rsb200_pana_plan_create(engine(), &job, 1, &pg.p), "rsb200_pana_plan_create");
  RawImage img = mRaw;
  runOnImage(pg.p, input.begin() + input.getPosition(), input.getRemainSize(), img,
             /*partial=*/false);
  engineCheck(rsb200_plan_results(pg.p, nullptr, 0), "rsb200_plan_results");
}
} // namespace

// ctor (decompressors/PanasonicV4Decompressor.cpp:49-90)
PanasonicV4Decompressor::PanasonicV4Decompressor(RawImage img, ByteStream input_,
                                                 bool zero_is_not_bad,
                                                 uint32_t section_split_offset_)
    : mRaw(std::move(img)), input(input_), zero_is_bad(!zero_is_not_bad),
      section_split_offset(section_split_offset_) {
  constexpr uint32_t BlockSize = 0x4000, PixelsPerPacket = 14, BytesPerPacket = 16;
  panaCheckImage(mRaw);
  if (!(mRaw->dim.x > 0 && mRaw->dim.y > 0) || mRaw->dim.x % (int)PixelsPerPacket != 0)
    ThrowRDE("Unexpected image dimensions found: (%i; %i)", mRaw->dim.x, mRaw->dim.y);
  if (BlockSize < section_split_offset)
    ThrowRDE("Bad section_split_offset: %u, less than BlockSize (%u)", section_split_offset,
             BlockSize);
  const uint64_t bytesTotal = mRaw->dim.area() / PixelsPerPacket * BytesPerPacket;
  const uint64_t bufSize = section_split_offset == 0
                               ? bytesTotal
                               : (bytesTotal + BlockSize - 1) / BlockSize * BlockSize;
  if (bufSize > 0xFFFFFFFFull)
    ThrowRDE("Raw dimensions require input buffer larger than supported");
  if (bufSize > input.getRemainSize()) // input_.peekStream(bufSize)
    ThrowIOE("Out of bounds access in ByteStream");
}

// decompress (:238-266): blocks / packets in parallel on the device
void PanasonicV4Decompressor::decompress() const {
  rsb200_pana_job job;
  std::memset(&job, 0, sizeof job);
  job.in_offset = 0;
  job.in_size = input.getRemainSize();
  job.out_offset = 0;
  job.out_pitch = (uint32_t)mRaw->pitch;
  job.width = (uint32_t)mRaw->dim.x;
  job.height = (uint32_t)mRaw->dim.y;
  job.version = 4;
  job.bps = 12;
  job.zero_is_not_bad = zero_is_bad ? 0 : 1;
  job.section_split_offset = section_split_offset;
  PlanGuard pg;
  engineCheck(rsb200_pana_plan_create(engine(), &job, 1, &pg.p), "rsb200_pana_plan_create");
  RawImage img = mRaw;
  runOnImage(pg.p, input.begin() + input.getPosition(), input.getRemainSize(), img,
             /*partial=*/false);
  engineCheck(rsb200_plan_results(pg.p, nullptr, 0), "rsb200_plan_results");
  if (!zero_is_bad)
    return;
  uint32_t count = 0;
  engineCheck(rsb200_plan_bad_pixels(pg.p, 0, nullptr, 0, &count), "rsb200_plan_bad_pixels");
  if (!count)
    return;
  if (count > RSB200_PANA_BAD_CAP)
    ThrowRDE("rawspeed_b200: %u bad pixels, more than the device list holds (%u)", count,
             RSB200_PANA_BAD_CAP);
  std::vector<uint32_t> zero_pos(count);
  engineCheck(rsb200_plan_bad_pixels(pg.p, 0, zero_pos.data(), count, &count),
              "rsb200_plan_bad_pixels");
  std::lock_guard<std::mutex> guard(mRaw->mBadPixelMutex);
  mRaw->mBadPixelPositions.insert(mRaw->mBadPixelPositions.end(), zero_pos.begin(), zero_pos.end());
}

PanasonicV5Decompressor::PanasonicV5Decompressor(RawImage img, ByteStream input_, uint32_t bps_)
    : mRaw(std::move(img)), input(input_), bps(bps_) {
  panaCheckImage(mRaw);
  if (bps != 12 && bps != 14)
    ThrowRDE("Unsupported bps: %u", bps);
  panaCheckInput(mRaw, input, (int)(128 / bps), 16, 1024);
}
void PanasonicV5Decompressor::decompress() const { panaRun(mRaw, input, 5, (int)bps); }

PanasonicV6Decompressor::PanasonicV6Decompressor(RawImage img, ByteStream input_, uint32_t bps_)
    : mRaw(std::move(img)), input(input_), bps(bps_) {
  panaCheckImage(mRaw);
  if (bps != 12 && bps != 14)
    ThrowRDE("Unsupported bps: %u", bps);
  panaCheckInput(mRaw, input, bps == 14 ? 11 : 14, 16, 1);
}
void PanasonicV6Decompressor::decompress() const { panaRun(mRaw, input, 6, (int)bps); }

PanasonicV7Decompressor::PanasonicV7Decompressor(RawImage img, ByteStream input_)
    : mRaw(std::move(img)), input(input_) {
  panaCheckImage(mRaw);
  panaCheckInput(mRaw, input, 9, 16, 1);
}
void PanasonicV7Decompressor::decompress() const { panaRun(mRaw, input, 7, 14); }

// ------------------------------------------------------------------ Phase One
// ctor (decompressors/PhaseOneDecompressor.cpp:42-59)
PhaseOneDecompressor::PhaseOneDecompressor(RawImage img, std::vector<PhaseOneStrip>&& strips_)
    : mRaw(std::move(img)), strips(std::move(strips_)) {
  if (mRaw->getDataType() != RawImageType::UINT16)
    ThrowRDE("Unexpected data type");
  if (mRaw->getCpp() != 1 || mRaw->getBpp() != sizeof(uint16_t))
    ThrowRDE("Unexpected cpp: %u", mRaw->getCpp());
  if (!(mRaw->dim.x > 0 && mRaw->dim.y > 0) || mRaw->dim.x % 2 != 0 || mRaw->dim.x > 11976 ||
      mRaw->dim.y > 8854)
    ThrowRDE("Unexpected image dimensions found: (%d; %d)", mRaw->dim.x, mRaw->dim.y);
  prepareStrips();
}

// prepareStrips (:61-83): every row exactly once
void PhaseOneDecompressor::prepareStrips() {
  if (strips.size() != (size_t)mRaw->dim.y)
    ThrowRDE("Height (%d) vs strip count %zu mismatch", mRaw->dim.y, strips.size());
  std::sort(strips.begin(), strips.end(),
            [](const PhaseOneStrip& a, const PhaseOneStrip& b) { return a.n < b.n; });
  for (size_t i = 0; i < strips.size(); ++i)
    if ((size_t)strips[i].n != i)
      ThrowRDE("Strips validation issue.");
}

// decompress (:152-168): rows in parallel on the device
void PhaseOneDecompressor::decompress() const {
  // one contiguous input window that covers every strip
  const uint8_t* lo = nullptr;
  const uint8_t* hi = nullptr;
  for (const PhaseOneStrip& s : strips) {
    const uint8_t* b = s.bs.begin() + s.bs.getPosition();
    const uint8_t* e = b + s.bs.getRemainSize();
    lo = (!lo || b < lo) ? b : lo;
    hi = (!hi || e > hi) ? e : hi;
  }
  std::vector<rsb200_phaseone_strip> st(strips.size());
  for (size_t i = 0; i < strips.size(); ++i) {
    const uint8_t* b = strips[i].bs.begin() + strips[i].bs.getPosition();
    st[i].in_offset = (uint64_t)(b - lo);
    st[i].in_size = strips[i].bs.getRemainSize();
    st[i].row = (uint32_t)strips[i].n;
  }
  rsb200_phaseone_job job;
  std::memset(&job, 0, sizeof job);
  job.out_offset = 0;
  job.out_pitch = (uint32_t)mRaw->pitch;
  job.width = (uint32_t)mRaw->dim.x;
  job.height = (uint32_t)mRaw->dim.y;
  job.first_strip = 0;
  PlanGuard pg;
  engineCheck(rsb200_phaseone_plan_create(engine(), &job, 1, st.data(), (int)st.size(), &pg.p),
              "rsb200_phaseone_plan_create");
  RawImage img = mRaw;
  runOnImage(pg.p, lo, (size_t)(hi - lo), img, /*partial=*/true);
  rsb200_scan_result res;
  const int rc = rsb200_plan_results(pg.p, &res, 1);
  if (rc == RSB200_OK)
    return;
  if (res.status == RSB200_ERR_RDE)
    ThrowRDE("Too many errors encountered. Giving up. First Error:\n"
             "a Phase One row cannot be decoded (lengths / bit stream)");
  engineCheck(rc, "rsb200_plan_results");
}

// ------------------------------------------------------------------ Sony ARW2
// SonyArw2Decompressor ctor (decompressors/SonyArw2Decompressor.cpp:41-56)
SonyArw2Decompressor::SonyArw2Decompressor(RawImage img, ByteStream input_)
    : mRaw(std::move(img)), input(input_) {
  if (mRaw->getCpp() != 1 || mRaw->getDataType() != RawImageType::UINT16 ||
      mRaw->getBpp() != sizeof(uint16_t))
    ThrowRDE("Unexpected component count / data type");
  if (!(mRaw->dim.x > 0 && mRaw->dim.y > 0) || mRaw->dim.x % 32 != 0 || mRaw->dim.x > 9600 ||
      mRaw->dim.y > 6376)
    ThrowRDE("Unexpected image dimensions found: (%d; %d)", mRaw->dim.x, mRaw->dim.y);
  // 1 byte per pixel: input_.peekStream(dim.x * dim.y)
  if ((uint64_t)mRaw->dim.x * (uint64_t)mRaw->dim.y > input.getRemainSize())
    ThrowIOE("Out of bounds access in ByteStream");
}

// SonyArw2Decompressor::decompress (:135-148); rows / blocks in parallel on the device
void SonyArw2Decompressor::decompress() const {
  rsb200_arw2_job job;
  std::memset(&job, 0, sizeof job);
  job.in_offset = 0;
  job.out_offset = 0;
  job.out_pitch = (uint32_t)mRaw->pitch;
  job.width = (uint32_t)mRaw->dim.x;
  job.height = (uint32_t)mRaw->dim.y;
  job.table = mRaw->hasTable() ? 0 : -1;
  PlanGuard pg;
  engineCheck(rsb200_arw2_plan_create(engine(), &job, 1,
                                      mRaw->hasTable() ? mRaw->tableData().data() : nullptr,
                                      mRaw->hasTable() ? 1 : 0, mRaw->tableDither() ? 1 : 0, &pg.p),
              "rsb200_arw2_plan_create");
  RawImage img = mRaw;
  const size_t bytes = (size_t)mRaw->dim.x * (size_t)mRaw->dim.y;
  runOnImage(pg.p, input.begin() + input.getPosition(), bytes, img, /*partial=*/false);
  rsb200_scan_result res;
  const int rc = rsb200_plan_results(pg.p, &res, 1);
  if (rc == RSB200_OK)
    return;
  if (res.status == RSB200_ERR_RDE)
    ThrowRDE("Too many errors encountered. Giving up. First Error:\n"
             "ARW2 invariant failed, same pixel is both min and max");
  engineCheck(rc, "rsb200_plan_results");
}

// ------------------------------------------------------------------ DngOpcodes
// ROIOpcode ctor (common/DngOpcodes.cpp:193-226): inside {0, 0, dim}, inclusive
void DngOpcodes::readRoi(ByteStream& bs, const iPoint2D& dim, Op& op) {
  const uint32_t top = bs.getU32(), left = bs.getU32(), bottom = bs.getU32(), right = bs.getU32();
  const int tx = (int)left, ty = (int)top, bx = (int)right, by = (int)bottom;
  const bool ok = tx >= 0 && ty >= 0 && tx <= dim.x && ty <= dim.y && bx >= 0 && by >= 0 &&
                  bx <= dim.x && by <= dim.y && bx >= tx && by >= ty;
  if (!ok)
    ThrowRDE("Rectangle (%d, %d, %d, %d) not inside image (%d, %d, %d, %d).", tx, ty, bx, by, 0, 0,
             dim.x, dim.y);
  op.roi = iRectangle2D(tx, ty, bx - tx, by - ty);
}

// PixelOpcode ctor (:353-381)
void DngOpcodes::readPixelOpcode(const RawImage& ri, ByteStream& bs, const iPoint2D& dim, Op& op) {
  readRoi(bs, dim, op);
  op.firstPlane = bs.getU32();
  op.planes = bs.getU32();
  if (op.planes == 0 || op.firstPlane > ri->getCpp() || op.planes > ri->getCpp() ||
      op.firstPlane + op.planes > ri->getCpp())
    ThrowRDE("Bad plane params (first %u, num %u), got planes = %u", op.firstPlane, op.planes,
             ri->getCpp());
  op.rowPitch = bs.getU32();
  op.colPitch = bs.getU32();
  if (op.rowPitch < 1 || op.rowPitch > (uint32_t)op.roi.dim.y || op.colPitch < 1 ||
      op.colPitch > (uint32_t)op.roi.dim.x)
    ThrowRDE("Invalid pitch");
}

namespace {
uint64_t roundUpDivisionSafe(uint64_t a, uint64_t b) { return a ? 1 + (a - 1) / b : 0; }
} // namespace

// DngOpcodes::DngOpcodes (:666-726) and the opcode constructors it dispatches to
DngOpcodes::DngOpcodes(const RawImage& ri, ByteStream bs) {
  bs.setByteOrder(Endianness::big);
  const uint32_t opcode_count = bs.getU32();
  const auto origPos = bs.getPosition();
  for (uint32_t i = 0; i < opcode_count; i++) {
    bs.skipBytes(4);
    bs.skipBytes(4);
    bs.skipBytes(4);
    const uint32_t opcode_size = bs.getU32();
    bs.skipBytes(opcode_size);
  }
  bs.setPosition(origPos);
  opcodes.reserve(opcode_count);
  // integrated_subimg: the crop the list will see as TrimBounds opcodes narrow it
  iPoint2D subDim = ri->dim;
  const iPoint2D fullDim = ri->getUncroppedDim();
  for (uint32_t i = 0; i < opcode_count; i++) {
    const uint32_t code = bs.getU32();
    bs.skipBytes(4); // version
    const uint32_t flags = bs.getU32();
    const uint32_t opcode_size = bs.getU32();
    ByteStream ob = bs.getStream(opcode_size);
    Op op;
    op.code = code;
    bool keep = true;
    switch (code) {
    case 1:
    case 2:
    case 3:
    case 9: { // known, not implemented (:751-757, :776)
      static const char* const names[] = {"", "WarpRectilinear", "WarpFisheye", "FixVignetteRadial",
                                          "", "", "", "", "", "GainMap"};
      if (!(flags & 1))
        ThrowRDE("Unsupported Opcode: %u (%s)", code, names[code]);
      keep = false;
      break;
    }
    case 4: // FixBadPixelsConstant (:149-160)
      op.value = ob.getU32();
      ob.getU32(); // Bayer phase
      break;
    case 5: { // FixBadPixelsList (:263-317): uncropped coordinates
      ob.getU32(); // phase
      const uint32_t badPointCount = ob.getU32();
      const uint32_t badRectCount = ob.getU32();
      const auto pos0 = ob.getPosition();
      ob.skipBytes(badPointCount, 2 * 4);
      ob.skipBytes(badRectCount, 4 * 4);
      ob.setPosition(pos0);
      op.badPixels.reserve(badPointCount);
      for (uint32_t k = 0; k < badPointCount; ++k) {
        const uint32_t y = ob.getU32(), x = ob.getU32();
        const int px = (int)x, py = (int)y;
        if (!(px >= 0 && py >= 0 && px < fullDim.x && py < fullDim.y))
          ThrowRDE("Bad point not inside image.");
        op.badPixels.emplace_back(y << 16 | x);
      }
      for (uint32_t k = 0; k < badRectCount; ++k) {
        Op r;
        readRoi(ob, fullDim, r);
        for (int y = 0; y < r.roi.dim.y; ++y)
          for (int x = 0; x < r.roi.dim.x; ++x)
            op.badPixels.emplace_back((uint32_t)(r.roi.pos.y + y) << 16 | (uint32_t)(r.roi.pos.x + x));
      }
      break;
    }
    case 6: // TrimBounds (:332-346)
      readRoi(ob, subDim, op);
      subDim = op.roi.dim;
      break;
    case 7: { // MapTable (:446-466)
      readPixelOpcode(ri, ob, subDim, op);
      const uint32_t count = ob.getU32();
      if (count == 0 || count > 65536)
        ThrowRDE("Invalid size of lookup table");
      op.lookup.assign(65536, 0);
      for (uint32_t k = 0; k < count; ++k)
        op.lookup[k] = ob.getU16();
      for (uint32_t k = count; k < 65536; ++k)
        op.lookup[k] = op.lookup[count - 1];
      break;
    }
    case 8: { // MapPolynomial (:473-505)
      readPixelOpcode(ri, ob, subDim, op);
      const uint64_t polynomial_size = (uint64_t)ob.getU32() + 1;
      (void)ob.check((uint64_t)(uint32_t)(8 * polynomial_size)); // implicit_cast<size_type>(8UL * n)
      if (polynomial_size > 9)
        ThrowRDE("A polynomial with more than 8 degrees not allowed");
      std::vector<double> polynomial;
      for (uint64_t k = 0; k < polynomial_size; ++k) {
        const uint64_t hi = ob.getU32(), lo = ob.getU32();
        const uint64_t bits = (hi << 32) | lo;
        double d;
        std::memcpy(&d, &bits, 8);
        polynomial.push_back(d);
      }
      op.lookup.assign(65536, 0);
      for (size_t k = 0; k < op.lookup.size(); ++k) {
        double val = polynomial[0];
        for (size_t j = 1; j < polynomial.size(); ++j)
          val += polynomial[j] * std::pow((double)k / 65536.0, (double)j);
        op.lookup[k] = (uint16_t)std::clamp<double>(val * 65535.5, 0.0, 65535.0);
      }
      break;
    }
    case 10:
    case 11:
    case 12:
    case 13: { // DeltaRowOrCol (:535-589): 10 / 12 index by row, 11 / 13 by column
      readPixelOpcode(ri, ob, subDim, op);
      const uint32_t deltaF_count = ob.getU32();
      (void)ob.check(deltaF_count, 4);
      const bool byRow = code == 10 || code == 12;
      const uint64_t expectedSize = byRow ? roundUpDivisionSafe((uint64_t)op.roi.dim.y, op.rowPitch)
                                          : roundUpDivisionSafe((uint64_t)op.roi.dim.x, op.colPitch);
      if (expectedSize != deltaF_count)
        ThrowRDE("Got unexpected number of elements (%llu), expected %u.",
                 (unsigned long long)expectedSize, deltaF_count);
      op.deltaF.reserve(deltaF_count);
      for (uint32_t k = 0; k < deltaF_count; ++k) {
        const uint32_t bits = ob.getU32();
        float f;
        std::memcpy(&f, &bits, 4);
        if (!std::isfinite(f))
          ThrowRDE("Got bad float %f.", (double)f);
        op.deltaF.push_back(f);
      }
      break;
    }
    default:
      ThrowRDE("Unknown unhandled Opcode: %u", code);
    }
    if (ob.getRemainSize() != 0)
      ThrowRDE("Inconsistent length of opcode");
    if (keep)
      opcodes.push_back(std::move(op));
  }
}

DngOpcodes::~DngOpcodes() = default;

// setup() of every opcode in list order (:160-170, :425-430, :538-552) and the device form of
// its apply(); the first failing opcode ends the list and its exception is kept
DngOpcodes::Lowered DngOpcodes::lower(const RawImage& ri) const {
  Lowered L;
  iPoint2D off = ri->getCropOffset(), dim = ri->dim; // the crop as the list narrows it
  const bool isU16 = ri->getDataType() == RawImageType::UINT16;
  try {
    for (uint32_t i = 0; i < opcodes.size(); ++i) {
      const Op& op = opcodes[i];
      rsb200_dng_op d;
      std::memset(&d, 0, sizeof d);
      switch (op.code) {
      case 4:
        if (!isU16)
          ThrowRDE("Only 16 bit images supported");
        if (ri->getCpp() > 1)
          ThrowRDE("Only 1 component images supported");
        d.kind = RSB200_DNGOP_BAD_CONSTANT;
        d.top = (uint32_t)off.y;
        d.left = (uint32_t)off.x;
        d.bottom = (uint32_t)(off.y + dim.y);
        d.right = (uint32_t)(off.x + dim.x);
        d.first_plane = 0;
        d.planes = 1;
        d.row_pitch = d.col_pitch = 1;
        d.value = op.value;
        L.actions.push_back({Action::BadConstant, (uint32_t)L.ops.size()});
        L.ops.push_back(d);
        break;
      case 5:
        L.actions.push_back({Action::BadList, i});
        break;
      case 6: // ri->subFrame(roi) (common/RawImage.cpp:175-199)
        if (!op.roi.hasPositiveArea())
          ThrowRDE("No positive crop area");
        L.actions.push_back({Action::Trim, i});
        if (op.roi.dim.x <= dim.x - op.roi.pos.x && op.roi.dim.y <= dim.y - op.roi.pos.y) {
          off.x += op.roi.pos.x;
          off.y += op.roi.pos.y;
          dim = op.roi.dim;
        }
        break;
      default: {
        d.top = (uint32_t)(off.y + op.roi.pos.y);
        d.left = (uint32_t)(off.x + op.roi.pos.x);
        d.bottom = d.top + (uint32_t)op.roi.dim.y;
        d.right = d.left + (uint32_t)op.roi.dim.x;
        d.first_plane = op.firstPlane;
        d.planes = op.planes;
        d.row_pitch = op.rowPitch;
        d.col_pitch = op.colPitch;
        if (op.code == 7 || op.code == 8) {
          if (!isU16)
            ThrowRDE("Only 16 bit images supported");
          d.kind = RSB200_DNGOP_LOOKUP;
          d.table = (uint32_t)(L.tables.size() / 65536);
          L.tables.insert(L.tables.end(), op.lookup.begin(), op.lookup.end());
        } else {
          const bool scale = op.code == 12 || op.code == 13;
          d.kind = op.code == 10   ? RSB200_DNGOP_OFFSET_ROW
                   : op.code == 11 ? RSB200_DNGOP_OFFSET_COL
                   : op.code == 12 ? RSB200_DNGOP_SCALE_ROW
                                   : RSB200_DNGOP_SCALE_COL;
          d.table = (uint32_t)L.deltas.size();
          if (isU16) {
            // DeltaRowOrCol::setup (:538-552) with valueIsOk of Offset (:598-600) / Scale (:636-638)
            const float f2iScale = scale ? 1024.0F : 65535.0F;
            const double absLimit = 65535.0 / (double)65535.0F;
            const double maxLimit = ((double)(2147483647 - 512) / 65535.0) / (double)1024.0F;
            std::vector<uint32_t> conv;
            conv.reserve(op.deltaF.size());
            for (const float f : op.deltaF) {
              const bool ok = scale ? (f >= 0.0F && (double)f <= maxLimit)
                                    : ((double)std::abs(f) <= absLimit);
              if (!ok)
                ThrowRDE("Got float %f which is unacceptable.", (double)f);
              conv.push_back((uint32_t)static_cast<int>(f2iScale * f));
            }
            L.deltas.insert(L.deltas.end(), conv.begin(), conv.end());
          } else {
            for (const float f : op.deltaF) {
              uint32_t bits;
              std::memcpy(&bits, &f, 4);
              L.deltas.push_back(bits);
            }
          }
        }
        L.ops.push_back(d);
        break;
      }
      }
    }
  } catch (...) {
    L.error = std::current_exception();
  }
  return L;
}

// DngOpcodes::applyOpCodes (:730-735): the opcodes that set up run as one pass over the image;
// then the crop and mBadPixelPositions are brought to the state the reference's sequential walk
// leaves them in, and the error of the opcode that failed (if any) is rethrown
void DngOpcodes::applyOpCodes(const RawImage& ri) const {
  const Lowered L = lower(ri);
  std::vector<std::vector<uint32_t>> constant(L.ops.size());
  if (!L.ops.empty()) {
    if (!ri->isAllocated())
      ThrowRDE("applyOpCodes: image has no data");
    const iPoint2D full = ri->getUncroppedDim();
    rsb200_dngop_job job;
    std::memset(&job, 0, sizeof job);
    job.offset = 0;
    job.pitch = (uint32_t)ri->pitch;
    job.width = (uint32_t)full.x;
    job.height = (uint32_t)full.y;
    job.cpp = ri->getCpp();
    job.is_f32 = ri->getDataType() == RawImageType::F32 ? 1u : 0u;
    job.first_op = 0;
    job.num_ops = (uint32_t)L.ops.size();
    PlanGuard pg;
    engineCheck(rsb200_dngop_plan_create(engine(), &job, 1, L.ops.data(), (int)L.ops.size(),
                                         L.tables.data(), (int)(L.tables.size() / 65536),
                                         L.deltas.data(), (int)L.deltas.size(), &pg.p),
                "rsb200_dngop_plan_create");
    engineCheck(rsb200_plan_run_host_image(pg.p, nullptr, 0, ri->getByteData(), (uint32_t)ri->pitch,
                                           (uint32_t)(full.x * (int)ri->getBpp()), (uint32_t)full.y,
                                           /*partial=*/1),
                "rsb200_plan_run_host_image");
    for (size_t k = 0; k < L.ops.size(); ++k) {
      if (L.ops[k].kind != RSB200_DNGOP_BAD_CONSTANT)
        continue;
      uint32_t count = 0;
      engineCheck(rsb200_plan_bad_pixels(pg.p, (int)k, nullptr, 0, &count), "rsb200_plan_bad_pixels");
      if (count > RSB200_PANA_BAD_CAP)
        ThrowRDE("rawspeed_b200: %u bad pixels, more than the device list holds (%u)", count,
                 RSB200_PANA_BAD_CAP);
      constant[k].resize(count);
      if (count)
        engineCheck(rsb200_plan_bad_pixels(pg.p, (int)k, constant[k].data(), count, &count),
                    "rsb200_plan_bad_pixels");
      // the reference walks the crop row by row (:175-182): ascending (row << 16 | col)
      std::sort(constant[k].begin(), constant[k].end());
    }
  }
  {
    std::lock_guard<std::mutex> guard(ri->mBadPixelMutex);
    for (const Action& a : L.actions) {
      if (a.kind == Action::BadList) {
        const auto& b = opcodes[a.index].badPixels;
        ri->mBadPixelPositions.insert(ri->mBadPixelPositions.begin(), b.begin(), b.end());
      } else if (a.kind == Action::BadConstant) {
        ri->mBadPixelPositions.insert(ri->mBadPixelPositions.end(), constant[a.index].begin(),
                                      constant[a.index].end());
      } else {
        ri->subFrame(opcodes[a.index].roi);
      }
    }
  }
  if (L.error)
    std::rethrow_exception(L.error);
}

// ------------------------------------------------------------------ sRaw
// Cr2sRawInterpolator::interpolate (interpolators/Cr2sRawInterpolator.cpp:499-542)
void Cr2sRawInterpolator::interpolate(int version) {
  const iPoint2D sub = mRaw->subsampling;
  const bool is422 = sub.y == 1 && sub.x == 2, is420 = sub.y == 2 && sub.x == 2;
  if (!is422 && !is420)
    ThrowRDE("Unknown subsampling: (%i; %i)", sub.x, sub.y);
  if (version < 0 || version > 2 || (is420 && version == 0))
    ThrowRDE("rawspeed_b200: sRaw version %d is not defined for this subsampling", version);
  const int per = is420 ? 6 : 4;
  rsb200_sraw_job job;
  std::memset(&job, 0, sizeof job);
  job.in_offset = 0;
  job.in_pitch = (uint32_t)input.pitch() * 2u;
  job.num_mcus = (uint32_t)(input.width() / per);
  job.in_rows = (uint32_t)input.height();
  job.sub_x = (uint8_t)sub.x;
  job.sub_y = (uint8_t)sub.y;
  job.version = (uint8_t)version;
  for (int i = 0; i < 3; ++i)
    job.sraw_coeffs[i] = sraw_coeffs[(size_t)i];
  job.hue = hue;
  job.out_offset = 0;
  job.out_pitch = (uint32_t)mRaw->pitch;
  if (mRaw->getCpp() != 3 || (int)(job.num_mcus * 2) > mRaw->dim.x ||
      (int)(job.in_rows * (uint32_t)sub.y) > mRaw->dim.y)
    ThrowRDE("rawspeed_b200: sRaw output image does not match the subsampled input");
  PlanGuard pg;
  engineCheck(rsb200_sraw_plan_create(engine(), &job, 1, &pg.p), "rsb200_sraw_plan_create");
  RawImage img = mRaw;
  const size_t inBytes = (size_t)(input.height() - 1) * job.in_pitch + (size_t)input.width() * 2;
  runOnImage(pg.p, reinterpret_cast<const uint8_t*>(input.begin()), inBytes, img,
             /*partial=*/true);
}

// ------------------------------------------------------------------ LJPEG
LJpegDecompressor::LJpegDecompressor(RawImage img, iRectangle2D imgFrame_, Frame frame_,
                                     std::vector<PerComponentRecipe> rec_,
                                     int numLJpegRowsPerRestartInterval_, Buffer input_)
    : mRaw(std::move(img)), input(input_), imgFrame(imgFrame_), frame(frame_),
      rec(std::move(rec_)), numLJpegRowsPerRestartInterval(numLJpegRowsPerRestartInterval_) {
  const int cpp = (int)mRaw->getCpp();
  if (cpp < 1 || cpp > 3)
    ThrowRDE("Unexpected component count (%u)", mRaw->getCpp());
  if (!mRaw->dim.hasPositiveArea())
    ThrowRDE("Image has zero size");
  if (!imgFrame.hasPositiveArea())
    ThrowRDE("Tile has zero size");
  if (imgFrame.pos.x >= mRaw->dim.x)
    ThrowRDE("X offset outside of image");
  if (imgFrame.pos.y >= mRaw->dim.y)
    ThrowRDE("Y offset outside of image");
  if (imgFrame.dim.x > mRaw->dim.x)
    ThrowRDE("Tile wider than image");
  if (imgFrame.dim.y > mRaw->dim.y)
    ThrowRDE("Tile taller than image");
  if (imgFrame.pos.x + imgFrame.dim.x > mRaw->dim.x)
    ThrowRDE("Tile overflows image horizontally");
  if (imgFrame.pos.y + imgFrame.dim.y > mRaw->dim.y)
    ThrowRDE("Tile overflows image vertically");
  if (!frame.dim.hasPositiveArea())
    ThrowRDE("Frame has zero size");
  const iPoint2D m = frame.mcu;
  const bool mcuOk = (m.y == 1 && m.x >= 1 && m.x <= 4) || (m.x == 2 && m.y == 2);
  if (!mcuOk)
    ThrowRDE("Unexpected MCU size: {%i, %i}", m.x, m.y);
  if (rec.size() != (size_t)(m.x * m.y))
    ThrowRDE("Must have exactly one recepie per component");
  for (const auto& r : rec)
    if (!r.ht.isFullDecode())
      ThrowRDE("Huffman table is not of a full decoding variety");
  if (numLJpegRowsPerRestartInterval < 1)
    ThrowRDE("Number of rows per restart interval must be positives");
  if ((int64_t)m.x * frame.dim.x > std::numeric_limits<int>::max() ||
      (int64_t)m.y * frame.dim.y > std::numeric_limits<int>::max())
    ThrowRDE("LJpeg frame is too big");
  if ((int64_t)cpp * imgFrame.dim.x > std::numeric_limits<int>::max())
    ThrowRDE("Img frame is too big");
  if (imgFrame.dim.x < m.x || imgFrame.dim.y < m.y)
    ThrowRDE("Tile size is smaller than a single frame MCU");
  if (imgFrame.dim.y % m.y != 0)
    ThrowRDE("Output row count is not a multiple of MCU row count");
  const int tileRequiredWidth = cpp * imgFrame.dim.x;
  const int mcusToConsume = (tileRequiredWidth + m.x - 1) / m.x;
  if (frame.dim.x < mcusToConsume || m.y * frame.dim.y < imgFrame.dim.y ||
      m.x * frame.dim.x < tileRequiredWidth)
    ThrowRDE("LJpeg frame (%d, %d) is smaller than expected (%d, %d)", m.x * frame.dim.x,
             m.y * frame.dim.y, tileRequiredWidth, imgFrame.dim.y);
  const int rows = imgFrame.dim.y / m.y;
  numRestartIntervals = (rows + numLJpegRowsPerRestartInterval - 1) / numLJpegRowsPerRestartInterval;
}

void LJpegDecompressor::describe(const uint8_t* fileBase, std::vector<rsb200_huff_table>& tables,
                                 std::vector<rsb200_ljpeg_scan>& scans,
                                 uint64_t outOffset) const {
  const int cpp = (int)mRaw->getCpp();
  const iPoint2D m = frame.mcu;
  const int totalRows = imgFrame.dim.y / m.y;
  const uint8_t* data = input.begin();
  const uint32_t size = input.getSize();
  uint8_t tab[4] = {0, 0, 0, 0};
  for (size_t c = 0; c < rec.size(); ++c)
    tab[c] = tableIndex(tables, rec[c].ht.deviceTable());
  intervalStart.assign(1, 0);
  markerPos.clear();
  // Restart intervals: the entropy data of interval k ends at the first FFxx
  // (xx != 00); it must be RST((k) % 8) (LJpegDecompressor.cpp:286-297).
  for (int k = 1; k < numRestartIntervals; ++k) {
    uint32_t p = intervalStart.back();
    bool foundMarker = false;
    while (p + 1 < size) {
      const uint8_t* q = (const uint8_t*)std::memchr(data + p, 0xFF, size - 1 - p);
      if (!q)
        break;
      p = (uint32_t)(q - data);
      if (data[p + 1] != 0x00) {
        foundMarker = true;
        break;
      }
      p += 2;
    }
    if (!foundMarker)
      ThrowRDE("Jpeg marker not encountered");
    const uint8_t c1 = data[p + 1];
    if (c1 == 0xFF)
      ThrowRDE("Jpeg marker not encountered");
    if (c1 < 0xD0 || c1 > 0xD7)
      ThrowRDE("Not a restart marker!");
    if ((c1 - 0xD0) != ((k - 1) % 8))
      ThrowRDE("Unexpected restart marker found");
    markerPos.push_back(p);
    intervalStart.push_back(p + 2);
  }
  for (int k = 0; k < numRestartIntervals; ++k) {
    const uint32_t start = intervalStart[(size_t)k];
    if (size < start || size - start < 8) // BitStreamerJPEG: MaxProcessBytes == 8
      ThrowIOE("Bit stream size is smaller than MaxProcessBytes");
    rsb200_ljpeg_scan s;
    std::memset(&s, 0, sizeof s);
    s.in_offset = (uint64_t)(data - fileBase) + start;
    s.in_size = size - start;
    s.rows = (uint32_t)std::min(numLJpegRowsPerRestartInterval,
                                totalRows - k * numLJpegRowsPerRestartInterval);
    s.frame_w = (uint32_t)frame.dim.x;
    s.mcu_w = (uint8_t)m.x;
    s.mcu_h = (uint8_t)m.y;
    for (size_t c = 0; c < rec.size(); ++c) {
      s.table[c] = tab[c];
      s.init_pred[c] = rec[c].initPred;
    }
    s.out_offset = outOffset;
    s.out_pitch = (uint32_t)mRaw->pitch;
    s.out_x = (uint32_t)(cpp * imgFrame.pos.x);
    s.out_y = (uint32_t)(imgFrame.pos.y + m.y * numLJpegRowsPerRestartInterval * k);
    s.store_w = (uint32_t)(cpp * imgFrame.dim.x);
    scans.push_back(s);
  }
}

uint32_t LJpegDecompressor::finish(const rsb200_scan_result* res, int nres) const {
  if (nres != numRestartIntervals)
    ThrowRDE("internal: result count mismatch");
  for (int k = 0; k < numRestartIntervals; ++k) {
    if (res[k].status == RSB200_ERR_RDE)
      ThrowRDE("bad Huffman code");
    if (res[k].status == RSB200_ERR_IOE)
      ThrowIOE("Buffer overflow read in BitStreamer");
    if (res[k].status != RSB200_OK)
      ThrowRDE("device error %u", res[k].status);
    if (k + 1 < numRestartIntervals) {
      // the pump must have stopped exactly on the restart marker
      if ((uint64_t)intervalStart[(size_t)k] + res[k].consumed != markerPos[(size_t)k])
        ThrowRDE("Jpeg marker not encountered");
    }
  }
  const uint64_t pos = (uint64_t)intervalStart.back() + res[numRestartIntervals - 1].consumed;
  if (pos > input.getSize()) // inputStream.skipBytes(bs.getStreamPosition())
    ThrowIOE("Out of bounds access in ByteStream");
  return (uint32_t)pos;
}

uint32_t LJpegDecompressor::decode() const {
  std::vector<rsb200_huff_table> tables;
  std::vector<rsb200_ljpeg_scan> scans;
  describe(input.begin(), tables, scans);
  PlanGuard pg;
  engineCheck(rsb200_ljpeg_plan_create(engine(), tables.data(), (int)tables.size(), scans.data(),
                                       (int)scans.size(), &pg.p),
              "rsb200_ljpeg_plan_create");
  RawImage img = mRaw;
  runOnImage(pg.p, input.begin(), input.getSize(), img, /*partial=*/true);
  std::vector<rsb200_scan_result> res(scans.size());
  (void)rsb200_plan_results(pg.p, res.data(), (int)res.size());
  return finish(res.data(), (int)res.size());
}

// ------------------------------------------------------------------ marker walk
AbstractLJpegDecoder::AbstractLJpegDecoder(ByteStream bs, RawImage img)
    : input(bs), mRaw(std::move(img)) {
  input.setByteOrder(Endianness::big);
  if (!mRaw->dim.hasPositiveArea())
    ThrowRDE("Image has zero size");
}

uint8_t AbstractLJpegDecoder::getNextMarker(bool allowskip) {
  // first FF xx with xx not in {00, FF}; without skipping it must be right here
  ByteStream probe = input;
  bool found = false;
  while (probe.getRemainSize() >= 2) {
    const uint8_t c0 = probe.peekByte(0), c1 = probe.peekByte(1);
    if (c0 == 0xFF && c1 != 0 && c1 != 0xFF) {
      found = true;
      break;
    }
    if (!allowskip)
      break;
    probe.skipBytes(1);
  }
  if (!found)
    ThrowRDE("(Noskip) Expected marker not found. Probably corrupt file.");
  input = probe;
  const uint8_t m = input.peekByte(1);
  input.skipBytes(2);
  return m;
}

void AbstractLJpegDecoder::parseSOF(ByteStream s, SOFInfo* sof) {
  sof->prec = s.getByte();
  sof->h = s.getU16();
  sof->w = s.getU16();
  sof->cps = s.getByte();
  if (sof->prec < 2 || sof->prec > 16)
    ThrowRDE("Invalid precision (%u).", sof->prec);
  if (sof->h == 0 || sof->w == 0)
    ThrowRDE("Frame width or height set to zero");
  if (sof->cps > 4 || sof->cps < 1)
    ThrowRDE("Only from 1 to 4 components are supported.");
  if (sof->cps < mRaw->getCpp())
    ThrowRDE("Component count should be no less than sample count (%u vs %u).", sof->cps,
             mRaw->getCpp());
  if (sof->cps > (uint32_t)mRaw->dim.x)
    ThrowRDE("Component count should be no greater than row length (%u vs %d).", sof->cps,
             mRaw->dim.x);
  if (s.getRemainSize() != 3 * sof->cps)
    ThrowRDE("Header size mismatch.");
  for (uint32_t i = 0; i < sof->cps; i++) {
    sof->compInfo[i].componentId = s.getByte();
    const uint32_t subs = s.getByte();
    sof->compInfo[i].superV = subs & 0xf;
    sof->compInfo[i].superH = subs >> 4;
    if (sof->compInfo[i].superV < 1 || sof->compInfo[i].superV > 4)
      ThrowRDE("Horizontal sampling factor is invalid.");
    if (sof->compInfo[i].superH < 1 || sof->compInfo[i].superH > 4)
      ThrowRDE("Horizontal sampling factor is invalid.");
    if (s.getByte() != 0)
      ThrowRDE("Quantized components not supported.");
  }
  if ((int)sof->compInfo[0].superH != mRaw->subsampling.x ||
      (int)sof->compInfo[0].superV != mRaw->subsampling.y)
    ThrowRDE("LJpeg's subsampling does not match image's subsampling.");
  sof->initialized = true;
}

void AbstractLJpegDecoder::parseDHT(ByteStream dht) {
  while (dht.getRemainSize() > 0) {
    const uint32_t b = dht.getByte();
    if ((b >> 4) != 0)
      ThrowRDE("Unsupported Table class.");
    const uint32_t htIndex = b & 0xf;
    if (htIndex >= huff.size())
      ThrowRDE("Invalid huffman table destination id.");
    if (huff[htIndex] != nullptr)
      ThrowRDE("Duplicate table definition");
    HuffmanCode<> hc;
    const uint32_t nCodes = hc.setNCodesPerLength(dht.getBuffer(16));
    if (nCodes > 17) // Hasselblad uses 17
      ThrowRDE("Invalid DHT table.");
    const Buffer vals = dht.getBuffer(nCodes);
    hc.setCodeValues(vals.begin(), (int)nCodes);
    for (size_t i = 0; i < huffmanCodeStore.size(); ++i)
      if (*huffmanCodeStore[i] == hc)
        huff[htIndex] = PrefixCodeDecoderStore[i].get();
    if (!huff[htIndex]) {
      huffmanCodeStore.emplace_back(std::make_unique<HuffmanCode<>>(hc));
      auto dHT = std::make_unique<PrefixCodeDecoder<>>(std::move(hc));
      dHT->setup(fullDecodeHT, fixDng16Bug);
      huff[htIndex] = dHT.get();
      PrefixCodeDecoderStore.emplace_back(std::move(dHT));
    }
  }
}

void AbstractLJpegDecoder::parseDRI(ByteStream dri) {
  if (dri.getRemainSize() != 2)
    ThrowRDE("Invalid DRI header length.");
  numMCUsPerRestartInterval = dri.getU16();
}

void AbstractLJpegDecoder::parseSOS(ByteStream sos) {
  if (sos.getRemainSize() != 1 + 2 * frame.cps + 3)
    ThrowRDE("Invalid SOS header length.");
  if (const uint32_t soscps = sos.getByte(); frame.cps != soscps)
    ThrowRDE("Component number mismatch.");
  for (uint32_t i = 0; i < frame.cps; i++) {
    const uint32_t cs = sos.getByte();
    const uint32_t td = sos.getByte() >> 4;
    if (td >= huff.size() || !huff[td])
      ThrowRDE("Invalid Huffman table selection.");
    int ciIndex = -1;
    for (uint32_t j = 0; j < frame.cps; ++j)
      if (frame.compInfo[j].componentId == cs)
        ciIndex = (int)j;
    if (ciIndex == -1)
      ThrowRDE("Invalid Component Selector");
    frame.compInfo[(size_t)ciIndex].dcTblNo = td;
  }
  predictorMode = sos.getByte();
  if (predictorMode > 8) // Hasselblad uses '8'
    ThrowRDE("Invalid predictor mode.");
  if (sos.getByte() != 0)
    ThrowRDE("Se/Ah not zero.");
  Pt = sos.getByte();
  if (Pt > 15)
    ThrowRDE("Invalid Point transform.");
  if (Pt != 0)
    ThrowRDE("Point transform not supported.");
  prepareScan(); // == the validating half of decodeScan()
  pendingScan = true;
}

std::vector<const PrefixCodeDecoder<>*>
AbstractLJpegDecoder::getPrefixCodeDecoders(int N_COMP) const {
  std::vector<const PrefixCodeDecoder<>*> ht((size_t)N_COMP);
  for (int i = 0; i < N_COMP; ++i) {
    const unsigned t = frame.compInfo[(size_t)i].dcTblNo;
    if (t >= huff.size())
      ThrowRDE("Decoding table %u for comp %i does not exist (tables = %u)", t, i,
               (unsigned)huff.size());
    ht[(size_t)i] = huff[t];
  }
  return ht;
}

std::vector<uint16_t> AbstractLJpegDecoder::getInitialPredictors(int N_COMP) const {
  if (frame.prec < (Pt + 1))
    ThrowRDE("Invalid precision (%u) and point transform (%u) combination!", frame.prec, Pt);
  return std::vector<uint16_t>((size_t)N_COMP, (uint16_t)(1u << (frame.prec - Pt - 1)));
}

void AbstractLJpegDecoder::markerLoop(bool resume) {
  if (!resume) {
    if (getNextMarker(false) != 0xD8)
      ThrowRDE("Image did not start with SOI. Probably not an LJPEG");
  }
  for (uint8_t m; (m = getNextMarker(true)) != 0xD9;) {
    ByteStream data(input.getStream(input.peekU16()));
    data.setByteOrder(Endianness::big);
    data.skipBytes(2);
    switch (m) {
    case 0xC4: // DHT
      if (found.SOS)
        ThrowRDE("Found second DHT marker after SOS");
      parseDHT(data);
      found.DHT = true;
      break;
    case 0xC3: // SOF3
      if (found.SOS)
        ThrowRDE("Found second SOF marker after SOS");
      if (found.SOF)
        ThrowRDE("Found second SOF marker");
      parseSOF(data, &frame);
      found.SOF = true;
      break;
    case 0xDA: // SOS
      if (found.SOS)
        ThrowRDE("Found second SOS marker");
      if (!found.DHT)
        ThrowRDE("Did not find DHT marker before SOS.");
      if (!found.SOF)
        ThrowRDE("Did not find SOF marker before SOS.");
      parseSOS(data);
      if (immediate) {
        const uint32_t scanLength = runScan();
        pendingScan = false;
        input.skipBytes(scanLength);
        found.SOS = true;
        break;
      }
      return; // batch mode: resume in decodeSOIAfterScan()
    case 0xDB: // DQT
      ThrowRDE("Not a valid RAW file.");
    case 0xDD: // DRI
      if (found.DRI)
        ThrowRDE("Found second DRI marker");
      parseDRI(data);
      found.DRI = true;
      break;
    default:
      break;
    }
  }
  if (!found.SOS)
    ThrowRDE("Did not find SOS marker.");
}

void AbstractLJpegDecoder::decodeSOI() {
  immediate = true;
  markerLoop(false);
}
void AbstractLJpegDecoder::decodeSOIUntilScan() {
  immediate = false;
  markerLoop(false);
}
void AbstractLJpegDecoder::decodeSOIAfterScan(uint32_t scanLength) {
  pendingScan = false;
  input.skipBytes(scanLength);
  found.SOS = true;
  markerLoop(true);
}

// ------------------------------------------------------------------ LJpegDecoder
LJpegDecoder::LJpegDecoder(ByteStream bs, const RawImage& img) : AbstractLJpegDecoder(bs, img) {
  const uint32_t cpp = mRaw->getCpp();
  if (cpp < 1 || cpp > 3)
    ThrowRDE("Unexpected component count (%u)", cpp);
  if (!mRaw->dim.hasPositiveArea())
    ThrowRDE("Image has zero size");
}

bool LJpegDecoder::prepare(uint32_t offsetX, uint32_t offsetY, uint32_t width, uint32_t height,
                           iPoint2D maxDim_, bool fixDng16Bug_) {
  if (offsetX >= (unsigned)mRaw->dim.x)
    ThrowRDE("X offset outside of image");
  if (offsetY >= (unsigned)mRaw->dim.y)
    ThrowRDE("Y offset outside of image");
  if (width > (unsigned)mRaw->dim.x)
    ThrowRDE("Tile wider than image");
  if (height > (unsigned)mRaw->dim.y)
    ThrowRDE("Tile taller than image");
  if (offsetX + width > (unsigned)mRaw->dim.x)
    ThrowRDE("Tile overflows image horizontally");
  if (offsetY + height > (unsigned)mRaw->dim.y)
    ThrowRDE("Tile overflows image vertically");
  if (width == 0 || height == 0)
    return false; // nothing needed from this tile
  if (!maxDim_.hasPositiveArea() || (unsigned)maxDim_.x < width || (unsigned)maxDim_.y < height)
    ThrowRDE("Requested tile is larger than tile's maximal dimensions");
  offX = offsetX;
  offY = offsetY;
  w = width;
  h = height;
  maxDim = maxDim_;
  fixDng16Bug = fixDng16Bug_;
  decodeSOIUntilScan();
  return scanPending();
}

void LJpegDecoder::decode(uint32_t offsetX, uint32_t offsetY, uint32_t width, uint32_t height,
                          iPoint2D maxDim_, bool fixDng16Bug_) {
  if (!prepare(offsetX, offsetY, width, height, maxDim_, fixDng16Bug_))
    return;
  const uint32_t consumed = runScan();
  decodeSOIAfterScan(consumed);
}

void LJpegDecoder::prepareScan() {
  if (predictorMode != 1)
    ThrowRDE("Unsupported predictor mode: %u", predictorMode);
  for (uint32_t i = 0; i < frame.cps; i++)
    if (frame.compInfo[i].superH != 1 || frame.compInfo[i].superV != 1)
      ThrowRDE("Unsupported subsampling");
  const int N_COMP = (int)frame.cps;
  const auto hts = getPrefixCodeDecoders(N_COMP);
  const auto initPred = getInitialPredictors(N_COMP);
  std::vector<LJpegDecompressor::PerComponentRecipe> rec;
  rec.reserve((size_t)N_COMP);
  for (int i = 0; i < N_COMP; ++i)
    rec.push_back({*hts[(size_t)i], initPred[(size_t)i]});
  const iRectangle2D imgFrame((int)offX, (int)offY, (int)w, (int)h);
  const iPoint2D jpegFrameDim((int)frame.w, (int)frame.h);
  if ((int64_t)maxDim.x * (int)mRaw->getCpp() > std::numeric_limits<int>::max())
    ThrowRDE("Maximal output tile is too large");
  const iPoint2D maxRes((int)mRaw->getCpp() * maxDim.x, maxDim.y);
  if (maxRes.area() != (uint64_t)N_COMP * jpegFrameDim.area())
    ThrowRDE("LJpeg frame area does not match maximal tile area");
  if (maxRes.x % jpegFrameDim.x != 0 || maxRes.y % jpegFrameDim.y != 0)
    ThrowRDE("Maximal output tile size is not a multiple of LJpeg frame size");
  const iPoint2D MCUSize(maxRes.x / jpegFrameDim.x, maxRes.y / jpegFrameDim.y);
  if (MCUSize.area() != (uint64_t)N_COMP)
    ThrowRDE("Unexpected MCU size, does not match LJpeg component count");
  int rowsPerInterval;
  if (numMCUsPerRestartInterval == 0)
    rowsPerInterval = jpegFrameDim.y;
  else {
    if (numMCUsPerRestartInterval % jpegFrameDim.x != 0)
      ThrowRDE("Restart interval is not a multiple of frame row size");
    rowsPerInterval = numMCUsPerRestartInterval / jpegFrameDim.x;
  }
  d = std::make_unique<LJpegDecompressor>(mRaw, imgFrame,
                                          LJpegDecompressor::Frame{MCUSize, jpegFrameDim}, rec,
                                          rowsPerInterval, input.peekRemainingBuffer());
}

uint32_t LJpegDecoder::runScan() { return d->decode(); }

// ------------------------------------------------------------------ CR2
Cr2SliceWidths::Cr2SliceWidths(uint16_t numSlices_, uint16_t sliceWidth_, uint16_t lastSliceWidth_)
    : numSlices(numSlices_), sliceWidth(sliceWidth_), lastSliceWidth(lastSliceWidth_) {
  if (numSlices < 1)
    ThrowRDE("Bad slice count: %d", numSlices);
}

namespace {
struct Cr2Dsc { // Dsc of Cr2DecompressorImpl.h:250-275
  int N_COMP, X_S_F, Y_S_F, sliceColStep, pixelsPerGroup, groupSize;
  bool subSampled;
  explicit Cr2Dsc(std::tuple<int, int, int> f)
      : N_COMP(std::get<0>(f)), X_S_F(std::get<1>(f)), Y_S_F(std::get<2>(f)),
        sliceColStep(N_COMP * X_S_F), pixelsPerGroup(X_S_F * Y_S_F),
        groupSize((X_S_F != 1 || Y_S_F != 1) ? 2 + X_S_F * Y_S_F : N_COMP),
        subSampled(X_S_F != 1 || Y_S_F != 1) {}
};
struct Rect {
  int x, y, w, h;
};
} // namespace

template <typename HT>
Cr2Decompressor<HT>::Cr2Decompressor(RawImage mRaw_, std::tuple<int, int, int> format_,
                                     iPoint2D frame_, Cr2SliceWidths slicing_,
                                     std::vector<PerComponentRecipe> rec_, Buffer input_)
    : mRaw(std::move(mRaw_)), format(format_), frame(frame_), slicing(slicing_),
      rawSlicing(slicing_), rawFrame(frame_), rec(std::move(rec_)), input(input_) {
  if (mRaw->getCpp() != 1 || mRaw->getBpp() != 2)
    ThrowRDE("Unexpected cpp: %u", mRaw->getCpp());
  const auto f = format;
  const bool known = f == std::make_tuple(3, 2, 2) || f == std::make_tuple(3, 2, 1) ||
                     f == std::make_tuple(2, 1, 1) || f == std::make_tuple(4, 1, 1);
  if (!known)
    ThrowRDE("Unknown format <%i,%i,%i>", std::get<0>(f), std::get<1>(f), std::get<2>(f));
  const Cr2Dsc dsc(format);
  dim = mRaw->dim;
  if (!dim.hasPositiveArea() || dim.x % dsc.groupSize != 0)
    ThrowRDE("Unexpected image dimension multiplicity");
  dim.x /= dsc.groupSize;
  if (!frame.hasPositiveArea() || frame.x % dsc.X_S_F != 0 || frame.y % dsc.Y_S_F != 0)
    ThrowRDE("Unexpected LJpeg frame dimension multiplicity");
  frame.x /= dsc.X_S_F;
  frame.y /= dsc.Y_S_F;
  if (mRaw->dim.x > 19440 || mRaw->dim.y > 5920)
    ThrowRDE("Unexpected image dimensions found: (%d; %d)", mRaw->dim.x, mRaw->dim.y);
  for (int s = 0; s < slicing.numSlices; s++)
    if (slicing.widthOfSlice(s) <= 0)
      ThrowRDE("Bad slice width: %i", slicing.widthOfSlice(s));
  if (dsc.subSampled == mRaw->isCFA)
    ThrowRDE("Cannot decode subsampled image to CFA data or vice versa");
  if ((int)rec.size() != dsc.N_COMP)
    ThrowRDE("HT/Initial predictor count does not match component count");
  for (const auto& r : rec)
    if (!r.ht.isFullDecode())
      ThrowRDE("Huffman table is not of a full decoding variety");
  for (int* width : {&slicing.sliceWidth, &slicing.lastSliceWidth}) {
    if (*width % dsc.sliceColStep != 0)
      ThrowRDE("Slice width (%d) should be multiple of pixel group size (%d)", *width,
               dsc.sliceColStep);
    *width /= dsc.sliceColStep;
  }
  if (frame.area() < dim.area())
    ThrowRDE("Frame area smaller than the image area");
  // Walk the output tiles of the slices in stream order (slices are frame.y tall
  // and wrap into the next image column when they hit the bottom) and validate
  // the tiling like the reference's ctor does (Cr2DecompressorImpl.h:336-362).
  int sliceId = 0, sliceRow = 0, px = 0, py = 0;
  bool haveLast = false;
  Rect last{0, 0, 0, 0};
  while (sliceId < slicing.numSlices) {
    const int wS = slicing.widthOfSlice(sliceId);
    const Rect t{px, py, wS, std::min(dim.y - py, frame.y - sliceRow)};
    if (haveLast) {
      const bool continues = last.x == t.x && last.y + last.h == t.y && last.w == t.w;
      const bool newColumn = t.y == 0 && t.x == last.x + last.w;
      if (!continues && !newColumn)
        ThrowRDE("Invalid tiling - slice width change mid-output row?");
    }
    if (t.x + t.w <= dim.x && t.y + t.h <= dim.y) {
      last = t;
      haveLast = true;
    } else {
      if (t.x < dim.x && t.y < dim.y)
        ThrowRDE("Output tile partially outside of image");
      break;
    }
    sliceRow += t.h;
    py += t.h;
    if (sliceRow == frame.y) {
      ++sliceId;
      sliceRow = 0;
    }
    if (py == dim.y) {
      py = 0;
      px += t.w;
    }
  }
  if (!haveLast)
    ThrowRDE("No tiles are provided");
  if (last.x + last.w != dim.x || last.y + last.h != dim.y)
    ThrowRDE("Tiles do not cover the entire image area.");
}

template <typename HT> uint32_t Cr2Decompressor<HT>::decompress() const {
  if (input.getSize() < 8) // BitStreamerJPEG ctor
    ThrowIOE("Bit stream size is smaller than MaxProcessBytes");
  std::vector<rsb200_huff_table> tables;
  rsb200_cr2_job j;
  std::memset(&j, 0, sizeof j);
  j.in_offset = 0;
  j.in_size = input.getSize();
  j.n_comp = (uint8_t)std::get<0>(format);
  j.x_s_f = (uint8_t)std::get<1>(format);
  j.y_s_f = (uint8_t)std::get<2>(format);
  for (size_t c = 0; c < rec.size(); ++c) {
    j.table[c] = tableIndex(tables, rec[c].ht.deviceTable());
    j.init_pred[c] = rec[c].initPred;
  }
  j.frame_w = rawFrame.x;
  j.frame_h = rawFrame.y;
  j.num_slices = rawSlicing.numSlices;
  j.slice_w = rawSlicing.sliceWidth;
  j.last_slice_w = rawSlicing.lastSliceWidth;
  j.img_w = mRaw->dim.x;
  j.img_h = mRaw->dim.y;
  j.out_offset = 0;
  j.out_pitch = (uint32_t)mRaw->pitch;
  PlanGuard pg;
  engineCheck(rsb200_cr2_plan_create(engine(), tables.data(), (int)tables.size(), &j, 1, &pg.p),
              "rsb200_cr2_plan_create");
  RawImage img = mRaw;
  runOnImage(pg.p, input.begin(), input.getSize(), img, /*partial=*/false);
  rsb200_scan_result res{};
  (void)rsb200_plan_results(pg.p, &res, 1);
  if (res.status == RSB200_ERR_RDE)
    ThrowRDE("bad Huffman code");
  if (res.status == RSB200_ERR_IOE)
    ThrowIOE("Buffer overflow read in BitStreamer");
  if (res.status != RSB200_OK)
    ThrowRDE("device error %u", res.status);
  return res.consumed;
}

template class Cr2Decompressor<PrefixCodeDecoder<>>;

Cr2LJpegDecoder::Cr2LJpegDecoder(ByteStream bs, const RawImage& img)
    : AbstractLJpegDecoder(bs, img) {
  if (mRaw->getCpp() != 1 || mRaw->getBpp() != 2)
    ThrowRDE("Unexpected cpp: %u", mRaw->getCpp());
  if (!mRaw->dim.x || !mRaw->dim.y || mRaw->dim.x > 19440 || mRaw->dim.y > 5920)
    ThrowRDE("Unexpected image dimensions found: (%d; %d)", mRaw->dim.x, mRaw->dim.y);
}

void Cr2LJpegDecoder::prepareScan() {
  if (numMCUsPerRestartInterval != 0)
    ThrowRDE("Non-zero restart interval not supported.");
  if (predictorMode != 1)
    ThrowRDE("Unsupported predictor mode.");
  if (slicing.empty()) {
    const int slicesWidth = (int)(frame.w * frame.cps);
    if (slicesWidth > mRaw->dim.x)
      ThrowRDE("Don't know slicing pattern, and failed to guess it.");
    slicing = Cr2SliceWidths(1, 0, (uint16_t)slicesWidth);
  }
  bool isSubSampled = false;
  for (uint32_t i = 0; i < frame.cps; i++)
    isSubSampled = isSubSampled || frame.compInfo[i].superH != 1 || frame.compInfo[i].superV != 1;
  if (frame.cps != 3 && frame.w * frame.cps > 2 * frame.h)
    frame.h *= 2; // Canon doubled the width and halved the height (e.g. 5Ds)
  std::tuple<int, int, int> format;
  if (isSubSampled) {
    if (mRaw->isCFA)
      ThrowRDE("Cannot decode subsampled image to CFA data");
    if (frame.cps != 3)
      ThrowRDE("Unsupported number of subsampled components: %u", frame.cps);
    bool ok = frame.compInfo[0].superH == 2 &&
              (frame.compInfo[0].superV == 1 || frame.compInfo[0].superV == 2);
    for (uint32_t i = 1; i < frame.cps; i++)
      ok = ok && frame.compInfo[i].superH == 1 && frame.compInfo[i].superV == 1;
    if (!ok)
      ThrowRDE("Unsupported subsampling ([[%u, %u], [%u, %u], [%u, %u]])",
               frame.compInfo[0].superH, frame.compInfo[0].superV, frame.compInfo[1].superH,
               frame.compInfo[1].superV, frame.compInfo[2].superH, frame.compInfo[2].superV);
    if (frame.compInfo[0].superV == 2)
      format = {3, 2, 2};
    else {
      slicing.sliceWidth = slicing.sliceWidth * 3 / 2; // sRaw slice-width quirk
      slicing.lastSliceWidth = slicing.lastSliceWidth * 3 / 2;
      format = {3, 2, 1};
    }
  } else {
    if (frame.cps == 2)
      format = {2, 1, 1};
    else if (frame.cps == 4)
      format = {4, 1, 1};
    else
      ThrowRDE("Unsupported number of components: %u", frame.cps);
  }
  const int N_COMP = std::get<0>(format);
  const auto hts = getPrefixCodeDecoders(N_COMP);
  const auto initPred = getInitialPredictors(N_COMP);
  std::vector<Cr2Decompressor<>::PerComponentRecipe> rec;
  for (int i = 0; i < N_COMP; ++i)
    rec.push_back({*hts[(size_t)i], initPred[(size_t)i]});
  d = std::make_unique<Cr2Decompressor<>>(mRaw, format, iPoint2D((int)frame.w, (int)frame.h),
                                          slicing, rec, input.peekRemainingBuffer());
}

uint32_t Cr2LJpegDecoder::runScan() { return d->decompress(); }

void Cr2LJpegDecoder::decode(const Cr2SliceWidths& slicing_) {
  slicing = slicing_;
  for (int s = 0; s < slicing.numSlices; s++)
    if (slicing.widthOfSlice(s) <= 0)
      ThrowRDE("Bad slice width: %i", slicing.widthOfSlice(s));
  decodeSOI();
}

// ------------------------------------------------------------------ Hasselblad
// ctor (decompressors/HasselbladDecompressor.cpp:39-58)
HasselbladDecompressor::HasselbladDecompressor(RawImage mRaw_, const PerComponentRecipe& rec_, Buffer input_)
    : mRaw(std::move(mRaw_)), rec(rec_), input(input_) {
  if (mRaw->getDataType() != RawImageType::UINT16)
    ThrowRDE("Unexpected data type");
  if (mRaw->getCpp() != 1 || mRaw->getBpp() != sizeof(uint16_t))
    ThrowRDE("Unexpected cpp: %u", mRaw->getCpp());
  // FIXME (reference): could be wrong. max "active pixels" - "100 MP"
  if (!mRaw->dim.hasPositiveArea() || mRaw->dim.x % 2 != 0 || mRaw->dim.x > 12000 || mRaw->dim.y > 8842)
    ThrowRDE("Unexpected image dimensions found: (%d; %d)", mRaw->dim.x, mRaw->dim.y);
  if (rec.ht.isFullDecode())
    ThrowRDE("Huffman table is of a full decoding variety");
}

// decompress (:72-100)
uint32_t HasselbladDecompressor::decompress() {
  // ht.verifyCodeValuesAsDiffLengths() (codes/AbstractPrefixCode.h)
  for (const uint8_t v : rec.ht.code.codeValues)
    if (v > 16)
      ThrowRDE("Corrupt Huffman code: difference length %u longer than 16", (unsigned)v);
  if (input.getSize() < 4) // BitStreamerMSB32 ctor
    ThrowIOE("Bit stream size is smaller than MaxProcessBytes");
  rsb200_huff_table t = rec.ht.deviceTable();
  rsb200_hasselblad_job j;
  std::memset(&j, 0, sizeof j);
  j.in_offset = 0;
  j.in_size = input.getSize();
  j.width = (uint32_t)mRaw->dim.x;
  j.height = (uint32_t)mRaw->dim.y;
  j.out_pitch = (uint32_t)mRaw->pitch;
  j.out_offset = 0;
  j.init_pred = rec.initPred;
  j.table = 0;
  PlanGuard pg;
  engineCheck(rsb200_hasselblad_plan_create(engine(), &t, 1, &j, 1, &pg.p), "rsb200_hasselblad_plan_create");
  RawImage img = mRaw;
  runOnImage(pg.p, input.begin(), input.getSize(), img, /*partial=*/false);
  rsb200_scan_result res{};
  (void)rsb200_plan_results(pg.p, &res, 1);
  if (res.status == RSB200_ERR_RDE)
    ThrowRDE("bad Huffman code");
  if (res.status == RSB200_ERR_IOE)
    ThrowIOE("Buffer overflow read in BitStreamer");
  if (res.status != RSB200_OK)
    ThrowRDE("device error %u", res.status);
  return res.consumed;
}

// HasselbladLJpegDecoder.cpp:35-48
HasselbladLJpegDecoder::HasselbladLJpegDecoder(ByteStream bs, const RawImage& img)
    : AbstractLJpegDecoder(bs, img) {
  if (mRaw->getCpp() != 1 || mRaw->getDataType() != RawImageType::UINT16 || mRaw->getBpp() != sizeof(uint16_t))
    ThrowRDE("Unexpected component count / data type");
  if (!mRaw->dim.hasPositiveArea() || mRaw->dim.x % 2 != 0 || mRaw->dim.x > 12000 || mRaw->dim.y > 8842)
    ThrowRDE("Unexpected image dimensions found: (%d; %d)", mRaw->dim.x, mRaw->dim.y);
}

// decodeScan (:50-69)
void HasselbladLJpegDecoder::prepareScan() {
  if (numMCUsPerRestartInterval != 0)
    ThrowRDE("Non-zero restart interval not supported.");
  if (frame.w != (unsigned)mRaw->dim.x || frame.h != (unsigned)mRaw->dim.y)
    ThrowRDE("LJPEG frame does not match EXIF dimensions: (%u; %u) vs (%i; %i)", frame.w, frame.h,
             mRaw->dim.x, mRaw->dim.y);
  const HasselbladDecompressor::PerComponentRecipe rec = {*getPrefixCodeDecoders(1)[0],
                                                          getInitialPredictors(1)[0]};
  d = std::make_unique<HasselbladDecompressor>(mRaw, rec, input.peekRemainingBuffer());
}

uint32_t HasselbladLJpegDecoder::runScan() { return d->decompress(); }

// decode (:71-77): the pair stream cannot use a fully decoding table
void HasselbladLJpegDecoder::decode() {
  fullDecodeHT = false;
  decodeSOI();
}

// ------------------------------------------------------------------ DNG
namespace {
// the byte span of the file covered by the tiles (they all view one file buffer)
void tileSpan(const std::vector<DngSliceElement>& slices, const uint8_t** base, size_t* len) {
  const uint8_t* lo = nullptr;
  const uint8_t* hi = nullptr;
  for (const auto& e : slices) {
    const uint8_t* b = e.bs.begin();
    const uint8_t* en = b + e.bs.getSize();
    if (!lo || b < lo)
      lo = b;
    if (!hi || en > hi)
      hi = en;
  }
  *base = lo;
  *len = (size_t)(hi - lo);
}
} // namespace

void AbstractDngDecompressor::decompressUncompressed() const {
  const uint8_t* base;
  size_t span;
  tileSpan(slices, &base, &span);
  std::vector<rsb200_unpack_job> jobs;
  std::vector<rsb200_raw_job> fjobs; // floating-point DNG: F32 image
  const bool f32 = mRaw->getDataType() == RawImageType::F32;
  for (const auto& e : slices) {
    try {
      bool big_endian = e.bs.getByteOrder() == Endianness::big;
      if (mBps != 8 && mBps != 16 && mBps != 32 && !f32)
        big_endian = true; // DNG: not 8/16/32 bit => always big endian (UINT16 images only,
                           // AbstractDngDecompressor.cpp:66-77)
      const uint32_t inputPixelBits = mRaw->getCpp() * mBps;
      if (e.dsc.tileW > (uint32_t)std::numeric_limits<int>::max() / inputPixelBits)
        ThrowIOE("Integer overflow when calculating input pitch");
      const int inputPitchBits = (int)(inputPixelBits * e.dsc.tileW);
      if (inputPitchBits % 8 != 0)
        ThrowRDE("Bad combination of cpp (%u), bps (%u) and width (%u), the pitch is %d bits, "
                 "which is not a multiple of 8 (1 byte)",
                 mRaw->getCpp(), mBps, e.width, inputPitchBits);
      const int inputPitch = inputPitchBits / 8;
      if (inputPitch == 0)
        ThrowRDE("Data input pitch is too short. Can not decode!");
      UncompressedDecompressor u(e.bs, mRaw,
                                 iRectangle2D((int)e.offX, (int)e.offY, (int)e.width,
                                              (int)e.height),
                                 inputPitch, (int)mBps, big_endian ? BitOrder::MSB : BitOrder::LSB);
      if (f32) {
        rsb200_raw_job fjob;
        if (u.describeF32(base, &fjob))
          fjobs.push_back(fjob);
        continue;
      }
      rsb200_unpack_job job;
      if (u.describe(base, &job))
        jobs.push_back(job);
    } catch (const RawDecoderException& err) {
      mRaw->setError(err.what());
    } catch (const IOException& err) {
      mRaw->setError(err.what());
    }
  }
  if (jobs.empty() && fjobs.empty())
    return;
  PlanGuard pg;
  if (f32)
    engineCheck(rsb200_raw_plan_create(engine(), fjobs.data(), (int)fjobs.size(), nullptr, 0, &pg.p),
                "rsb200_raw_plan_create");
  else
    engineCheck(rsb200_unpack_plan_create(engine(), jobs.data(), (int)jobs.size(), &pg.p),
                "rsb200_unpack_plan_create");
  RawImage img = mRaw;
  runOnImage(pg.p, base, span, img, /*partial=*/true);
}

AbstractDngDecompressor::PreparedLJpeg AbstractDngDecompressor::prepareLJpeg(unsigned threads) const {
  PreparedLJpeg out;
  tileSpan(slices, &out.base, &out.span);
  struct One {
    std::unique_ptr<LJpegDecoder> dec;
    bool use = false;
    bool ioe = false;
    std::string err;
    std::vector<rsb200_huff_table> tables; // this tile's tables and scans (table indices local)
    std::vector<rsb200_ljpeg_scan> scans;
  };
  std::vector<One> one(slices.size());
  const uint8_t* const base = out.base;
  auto work = [&](size_t i) {
    const DngSliceElement& e = slices[i];
    One& o = one[i];
    try {
      auto dec = std::make_unique<LJpegDecoder>(e.bs, mRaw);
      o.use = dec->prepare(e.offX, e.offY, e.width, e.height,
                           iPoint2D((int)e.dsc.tileW, (int)e.dsc.tileH), mFixLjpeg);
      if (o.use) // restart-marker scan (a memchr walk over the tile's entropy data) + descriptors
        dec->scan()->describe(base, o.tables, o.scans);
      o.dec = std::move(dec);
    } catch (const RawDecoderException& err) {
      o.err = err.what();
      o.scans.clear();
    } catch (const IOException& err) {
      o.err = err.what();
      o.ioe = true;
      o.scans.clear();
    } catch (const std::exception& err) {
      // (bad_alloc, system_error ...: must not escape a std::thread; reported like a tile error)
      o.err = std::string("rawspeed_b200 host half: ") + err.what();
      o.scans.clear();
    } catch (...) {
      o.err = "rawspeed_b200 host half: unknown exception";
      o.scans.clear();
    }
  };
  bool forced = false;
  if (threads == 0) {
    threads = std::min(16u, std::max(1u, std::thread::hardware_concurrency()));
    if (const char* env = std::getenv("RSB200_HOST_THREADS")) {
      threads = (unsigned)std::max(1, std::atoi(env));
      forced = true; // the override is taken as is (it may raise the count above the default clamp)
    }
  }
  // worth a thread: >= 16 tiles and >= 1 MiB of tile data each
  if (!forced)
    threads = (unsigned)std::min<size_t>(threads, std::min((slices.size() + 15) / 16, out.span / (1u << 20) + 1));
  threads = (unsigned)std::min<size_t>(threads, std::max<size_t>(1, slices.size()));
  if (threads <= 1) {
    for (size_t i = 0; i < slices.size(); ++i)
      work(i);
  } else {
    // tiles are independent (each decoder only reads the image's shape): a shared counter
    // hands them out; results land in per-tile slots, so the order of the outcome is fixed
    std::atomic<size_t> next{0};
    std::vector<std::thread> pool;
    pool.reserve(threads);
    for (unsigned t = 0; t < threads; ++t)
      pool.emplace_back([&] {
        for (size_t i = next.fetch_add(1); i < slices.size(); i = next.fetch_add(1))
          work(i);
      });
    for (auto& th : pool)
      th.join();
  }
  // merge in tile order: de-duplicate the tables across tiles, re-index the scans
  {
    size_t total = 0;
    for (const One& o : one)
      total += o.scans.size();
    out.scans.reserve(total);
    out.tiles.reserve(slices.size());
  }
  for (size_t i = 0; i < slices.size(); ++i) {
    One& o = one[i];
    if (!o.err.empty()) {
      out.errors.push_back(o.err);
      out.errorIsIOE.push_back(o.ioe ? 1 : 0);
      continue;
    }
    if (!o.use)
      continue;
    uint8_t remap[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    try {
      for (size_t t = 0; t < o.tables.size() && t < 8; ++t)
        remap[t] = tableIndex(out.tables, o.tables[t]);
    } catch (const RawDecoderException& err) { // more than 255 distinct tables in the batch
      out.errors.emplace_back(err.what());
      out.errorIsIOE.push_back(0);
      continue;
    }
    PreparedLJpeg::Tile t;
    t.firstScan = (int)out.scans.size();
    t.nScans = (int)o.scans.size();
    for (rsb200_ljpeg_scan sc : o.scans) {
      const size_t ncomp = std::min<size_t>((size_t)sc.mcu_w * sc.mcu_h, sizeof sc.table / sizeof sc.table[0]);
      for (size_t c = 0; c < ncomp; ++c)
        sc.table[c] = remap[sc.table[c] & 7];
      out.scans.push_back(sc);
    }
    t.dec = std::move(o.dec);
    out.tiles.push_back(std::move(t));
  }
  return out;
}

void AbstractDngDecompressor::decompressLJpeg() const {
  PreparedLJpeg pl = prepareLJpeg();
  for (const std::string& err : pl.errors)
    mRaw->setError(err);
  if (pl.scans.empty())
    return;
  PlanGuard pg;
  engineCheck(rsb200_ljpeg_plan_create(engine(), pl.tables.data(), (int)pl.tables.size(),
                                       pl.scans.data(), (int)pl.scans.size(), &pg.p),
              "rsb200_ljpeg_plan_create");
  RawImage img = mRaw;
  // every tile was prepared: together they cover the whole image (DngTilingDescription), so its
  // current contents need not travel to the device first
  const bool covers = pl.errors.empty() && pl.tiles.size() == slices.size() && slices.size() == dsc.numTiles;
  runOnImage(pg.p, pl.base, pl.span, img, /*partial=*/!covers);
  std::vector<rsb200_scan_result> res(pl.scans.size());
  // (ADVICE r1: a CUDA / argument failure must not read as "every tile decoded")
  const int rrc = rsb200_plan_results(pg.p, res.data(), (int)res.size());
  if (rrc != RSB200_OK && rrc != RSB200_ERR_RDE && rrc != RSB200_ERR_IOE)
    engineCheck(rrc, "rsb200_plan_results");
  for (auto& t : pl.tiles) {
    try {
      const uint32_t consumed = t.dec->scan()->finish(res.data() + t.firstScan, t.nScans);
      t.dec->decodeSOIAfterScan(consumed);
    } catch (const RawDecoderException& err) {
      mRaw->setError(err.what());
    } catch (const IOException& err) {
      mRaw->setError(err.what());
    }
  }
}

void AbstractDngDecompressor::decompress() const {
  if (compression == 1)
    decompressUncompressed();
  else if (compression == 7)
    decompressLJpeg();
  else if (compression == 8)
    mRaw->setError("deflate support is disabled.");
  else if (compression == 9)
    mRaw->setError("VC-5 is not on the accelerated path.");
  else if (compression == 0x884c)
    mRaw->setError("jpeg support is disabled.");
  else
    mRaw->setError("AbstractDngDecompressor: Unknown compression");
  std::string firstErr;
  if (mRaw->isTooManyErrors(1, &firstErr))
    ThrowRDE("Too many errors encountered. Giving up. First Error:\n%s", firstErr.c_str());
}

} // namespace rawspeed_b200
