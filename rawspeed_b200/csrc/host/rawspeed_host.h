// rawspeed_host.h -- C++ host mirror of the reference's hot-path interface.
//
// The reference (darktable-org/rawspeed) has no FFI: callers (DngDecoder,
// Cr2Decoder, RawDecoder::decodeUncompressed, NefDecoder, the fuzzers) use four
// C++ decompressor classes.  This header re-declares those classes with the
// SAME names, constructor arguments, return values and exception behaviour, so
// a maintainer can point the callers at them unchanged; the method bodies that
// were the per-pixel CPU loops now build descriptors and call the C ABI
// (include/rawspeed_b200.h) -- marker parsing, Huffman-table validation,
// geometry checks, RawImage allocation and exceptions stay on the host exactly
// like the reference (paths relative to /root/reference/src/librawspeed):
//
//   UncompressedDecompressor   decompressors/UncompressedDecompressor.h:39-101
//   LJpegDecompressor          decompressors/LJpegDecompressor.h:38-95
//   AbstractLJpegDecoder       decompressors/AbstractLJpegDecoder.h:74-146
//   LJpegDecoder               decompressors/LJpegDecoder.h:31-49
//   Cr2SliceWidths/Cr2Decompressor  decompressors/Cr2Decompressor.h:50-174
//   Cr2LJpegDecoder            decompressors/Cr2LJpegDecoder.h:30-40
//   AbstractDngDecompressor    decompressors/AbstractDngDecompressor.h:37-151
//   RawImage / RawImageData    common/RawImage.h:111-263
//   Buffer / ByteStream        io/Buffer.h:47-121, io/ByteStream.h:42-140
//   HuffmanCode / PrefixCodeDecoder  codes/HuffmanCode.h, codes/PrefixCodeDecoder.h
//
// Written from the behaviour of those classes, not from their text.
#pragma once

#include <array>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <exception>
#include <memory>
#include <mutex>
#include <optional>
#include <stdexcept>
#include <string>
#include <tuple>
#include <vector>

#include "rawspeed_b200.h"

namespace rawspeed_b200 {

// ---------------------------------------------------------------- exceptions
class RawspeedException : public std::runtime_error {
public:
  explicit RawspeedException(const std::string& m) : std::runtime_error(m) {}
};
class RawDecoderException : public RawspeedException {
public:
  using RawspeedException::RawspeedException;
};
class IOException : public RawspeedException {
public:
  using RawspeedException::RawspeedException;
};

[[noreturn]] void ThrowRDE(const char* fmt, ...) __attribute__((format(printf, 1, 2)));
[[noreturn]] void ThrowIOE(const char* fmt, ...) __attribute__((format(printf, 1, 2)));

// ---------------------------------------------------------------- geometry
struct iPoint2D {
  int x = 0, y = 0;
  iPoint2D() = default;
  iPoint2D(int a, int b) : x(a), y(b) {}
  bool operator==(const iPoint2D& o) const { return x == o.x && y == o.y; }
  bool operator!=(const iPoint2D& o) const { return !(*this == o); }
  bool hasPositiveArea() const { return x > 0 && y > 0; }
  uint64_t area() const {
    return (uint64_t)(x < 0 ? -(int64_t)x : x) * (uint64_t)(y < 0 ? -(int64_t)y : y);
  }
};
struct iRectangle2D {
  iPoint2D pos, dim;
  iRectangle2D() = default;
  iRectangle2D(iPoint2D p, iPoint2D d) : pos(p), dim(d) {}
  iRectangle2D(int w, int h) : dim(w, h) {}
  iRectangle2D(int x, int y, int w, int h) : pos(x, y), dim(w, h) {}
  bool hasPositiveArea() const { return dim.x > 0 && dim.y > 0; }
};

enum class Endianness { little, big };
enum class BitOrder : uint8_t { LSB, MSB, MSB16, MSB32, JPEG }; // bitstreams/BitStreams.h:28-35

// ---------------------------------------------------------------- io
class Buffer {
public:
  using size_type = uint32_t;
  Buffer() = default;
  Buffer(const uint8_t* d, size_type s) : data_(d), size_(s) {}
  const uint8_t* begin() const { return data_; }
  size_type getSize() const { return size_; }
  bool isValid(uint64_t offset, uint64_t count = 1) const { return offset + count <= size_; }
  Buffer getSubView(size_type offset, size_type size) const {
    if (!isValid(offset, size))
      ThrowIOE("Buffer overflow: image file may be truncated");
    return {data_ + offset, size};
  }
  Buffer getSubView(size_type offset) const {
    if (!isValid(offset, 0))
      ThrowIOE("Buffer overflow: image file may be truncated");
    return {data_ + offset, size_ - offset};
  }

protected:
  const uint8_t* data_ = nullptr;
  size_type size_ = 0;
};

class ByteStream : public Buffer {
public:
  ByteStream() = default;
  explicit ByteStream(Buffer b, Endianness e = Endianness::little) : Buffer(b), order(e) {}
  ByteStream(const uint8_t* d, size_type s, Endianness e = Endianness::little)
      : Buffer(d, s), order(e) {}
  void setByteOrder(Endianness e) { order = e; }
  Endianness getByteOrder() const { return order; }
  size_type check(uint64_t bytes) const {
    if ((uint64_t)pos + bytes > size_)
      ThrowIOE("Out of bounds access in ByteStream");
    return (size_type)bytes;
  }
  size_type getPosition() const {
    check(0);
    return pos;
  }
  size_type getRemainSize() const {
    check(0);
    return size_ - pos;
  }
  uint8_t peekByte(size_type i = 0) const {
    check((uint64_t)i + 1);
    return data_[pos + i];
  }
  uint8_t getByte() {
    uint8_t v = peekByte();
    pos += 1;
    return v;
  }
  uint16_t peekU16() const {
    check(2);
    return order == Endianness::big ? (uint16_t)((data_[pos] << 8) | data_[pos + 1])
                                    : (uint16_t)((data_[pos + 1] << 8) | data_[pos]);
  }
  uint16_t getU16() {
    uint16_t v = peekU16();
    pos += 2;
    return v;
  }
  void skipBytes(uint64_t n) { pos += check(n); }
  // check(nmemb, size) / skipBytes(nmemb, size) (io/ByteStream.h:71-75, :130-132)
  size_type check(size_type nmemb, size_type size) const {
    if (size && nmemb > UINT32_MAX / size)
      ThrowIOE("Integer overflow when calculating stream length");
    return check((uint64_t)nmemb * size);
  }
  void skipBytes(size_type nmemb, size_type size) { pos += check(nmemb, size); }
  uint32_t getU32() {
    check(4);
    const uint8_t* p = data_ + pos;
    pos += 4;
    return order == Endianness::big
               ? ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]
               : ((uint32_t)p[3] << 24) | ((uint32_t)p[2] << 16) | ((uint32_t)p[1] << 8) | p[0];
  }
  void setPosition(size_type newPos) {
    pos = newPos;
    check(0);
  }
  Buffer getBuffer(size_type n) {
    Buffer b = getSubView(pos, n);
    pos += n;
    return b;
  }
  Buffer peekRemainingBuffer() const { return getSubView(pos, getRemainSize()); }
  ByteStream getStream(size_type n) {
    ByteStream s(getSubView(pos, n), order);
    pos += n;
    return s;
  }
  ByteStream getStream(size_type nmemb, size_type size) {
    if (size && nmemb > UINT32_MAX / size)
      ThrowIOE("Integer overflow when calculating stream length");
    return getStream(nmemb * size);
  }

private:
  size_type pos = 0;
  Endianness order = Endianness::little;
};

// ---------------------------------------------------------------- RawImage
// adt/Array2DRef.h: non-owning 2-D view (pitch in elements)
template <typename T> class Array2DRef {
public:
  Array2DRef(T* data_, int width_, int height_, int pitch_)
      : data(data_), w(width_), h(height_), pitchElts(pitch_) {}
  Array2DRef(T* data_, int width_, int height_)
      : data(data_), w(width_), h(height_), pitchElts(width_) {}
  int width() const { return w; }
  int height() const { return h; }
  int pitch() const { return pitchElts; }
  T* begin() const { return data; }
  T& operator()(int row, int col) const { return data[(size_t)row * pitchElts + col]; }

private:
  T* data;
  int w, h, pitchElts;
};

template <typename T> using Optional = std::optional<T>; // adt/Optional.h

// metadata/BlackArea.h:27-34
class BlackArea final {
public:
  BlackArea(int offset_, int size_, bool isVertical_)
      : offset(offset_), size(size_), isVertical(isVertical_) {}
  uint32_t offset; // in bayer pixels
  uint32_t size;
  bool isVertical; // otherwise horizontal
};

enum class RawImageType { UINT16, F32 };

class RawImageData {
public:
  iPoint2D dim;
  int pitch = 0;
  bool isCFA = true;
  iPoint2D subsampling{1, 1}; // ImageMetaData::subsampling
  // black / white levels (common/RawImage.h:163-174) and the scaling they drive
  int blackLevel = -1;
  std::array<int, 4> blackLevelSeparateStorage{};
  Optional<Array2DRef<int>> blackLevelSeparate;
  Optional<int> whitePoint;
  std::vector<BlackArea> blackAreas;
  bool mDitherScale = true; // common/RawImage.h:205
  // (y << 16) | x of pixels a decoder marked bad (common/RawImage.h:179-186)
  std::vector<uint32_t> mBadPixelPositions;
  std::mutex mBadPixelMutex;
  // bitmap of bad pixels, mBadPixelMapPitch bytes per row (common/RawImage.h:190-197)
  std::vector<uint8_t> mBadPixelMap;
  uint32_t mBadPixelMapPitch = 0;
  // RawImageData::transferBadPixelsToMap / fixBadPixels (common/RawImage.cpp:211-239): the
  // positions move into the bitmap on the host, the interpolation runs on the device (K11)
  void transferBadPixelsToMap();
  void fixBadPixels();
  // RawImageData::sixteenBitLookup (common/RawImage.cpp:373-378): the table set with
  // setTable() applied to every sample of the uncropped buffer, on the device (K12)
  void sixteenBitLookup();
  // RawImageData::subFrame (common/RawImage.cpp:175-199): dim becomes the crop, the data and
  // pitch stay those of the uncropped image
  void subFrame(iRectangle2D crop);
  iPoint2D getUncroppedDim() const { return uncropped_dim; }
  iPoint2D getCropOffset() const { return mOffset; }
  // RawImageDataU16::scaleBlackWhite (common/RawImageDataU16.cpp:147-183): the estimate and the
  // masked-area medians (calculateBlackAreas :60-145) on the host, the SCALE_VALUES pass over
  // the image on the device (K9).  `path`: RSB200_SCALE_AUTO = what an x86 build runs.
  void scaleBlackWhite(int path = RSB200_SCALE_AUTO);
  // its host half alone (estimate + calculateBlackAreas); false: nothing to scale
  bool prepareScaleBlackWhite();
  uint32_t getCpp() const { return cpp; }
  uint32_t getBpp() const { return bpp; }
  RawImageType getDataType() const { return dataType; }
  // RawImageData::setTable(table, dither) -> TableLookUp (common/TableLookUp.cpp:40-85)
  void setTable(const std::vector<uint16_t>& table_, bool dither);
  void clearTable() { tableStorage.clear(); }
  bool hasTable() const { return !tableStorage.empty(); }
  bool tableDither() const { return ditherTable; }
  // TableLookUp::tables of table 0: 65536 entries, or 2*65536 {base, delta} when dithered
  const std::vector<uint16_t>& tableData() const { return tableStorage; }
  void setCpp(uint32_t v);
  void createData(); // pitch = roundUp(dim.x*bpp, 16) (RawImage.cpp:68-113)
  bool isAllocated() const { return !data.empty(); }
  uint16_t* getData() { return reinterpret_cast<uint16_t*>(storage); }
  uint8_t* getByteData() { return storage; }
  size_t getByteSize() const { return (size_t)pitch * (size_t)uncropped_dim.y; }
  // ErrorLog (common/ErrorLog.h)
  void setError(const std::string& err);
  bool isTooManyErrors(unsigned many, std::string* firstErr = nullptr);
  std::vector<std::string> getErrors();

private:
  friend class RawImage;
  void calculateBlackAreas();
  iPoint2D uncropped_dim, mOffset;
  uint32_t cpp = 1, bpp = 2;
  RawImageType dataType = RawImageType::UINT16;
  std::vector<uint16_t> tableStorage;
  bool ditherTable = false;
  std::vector<uint8_t> data;
  uint8_t* storage = nullptr; // 16-byte aligned start inside `data`
  std::mutex errMutex;
  std::vector<std::string> errors;
};

class RawImage {
public:
  static RawImage create(const iPoint2D& dim, RawImageType type = RawImageType::UINT16,
                         uint32_t componentsPerPixel = 1);
  RawImageData* operator->() const { return p_.get(); }
  RawImageData& operator*() const { return *p_; }

private:
  std::shared_ptr<RawImageData> p_;
};

// ---------------------------------------------------------------- Huffman
struct BaselineCodeTag {};

template <typename Tag = BaselineCodeTag> class HuffmanCode {
public:
  // returns the number of codes; validates like HuffmanCode.h:100-147
  uint32_t setNCodesPerLength(Buffer data);
  void setCodeValues(const uint8_t* values, int n); // HuffmanCode.h:149-164
  bool operator==(const HuffmanCode& o) const {
    return nCodesPerLength == o.nCodesPerLength && codeValues == o.codeValues;
  }
  std::array<uint8_t, 16> nCodesPerLength{};
  std::vector<uint8_t> codeValues;
  uint32_t count = 0;
};

// PrefixCodeDecoder<> = LUT + lookup decoder in the reference; here it owns the
// validated table and hands it to the device (rsb200_huff_table).
template <typename Tag = BaselineCodeTag> class PrefixCodeDecoder {
public:
  explicit PrefixCodeDecoder(HuffmanCode<Tag> hc) : code(std::move(hc)) {}
  void setup(bool fullDecode_, bool fixDNGBug16_); // AbstractPrefixCodeTranscoder.h:70-83
  bool isFullDecode() const { return fullDecode; }
  bool handleDNGBug16() const { return fixDNGBug16; }
  rsb200_huff_table deviceTable() const;
  HuffmanCode<Tag> code;

private:
  bool fullDecode = true, fixDNGBug16 = false;
};

// ---------------------------------------------------------------- engine
// One process-wide device context (one process per GPU).
rsb200_ctx* engine();
void engineCheck(int rc, const char* what); // RSB200_* -> exception

// ---------------------------------------------------------------- K1
class UncompressedDecompressor {
public:
  UncompressedDecompressor(ByteStream input, RawImage img, const iRectangle2D& crop,
                           int inputPitchBytes, int bitPerPixel, BitOrder order);
  void readUncompressedRaw();
  // the fixed-layout members (UncompressedDecompressor.cpp:270-390); all write the
  // image from (0,0) and use only the crop's size, like the reference
  template <bool uncorrectedRawValues> void decode8BitRaw();
  template <Endianness e> void decode12BitRawWithControl();
  template <Endianness e> void decode12BitRawUnpackedLeftAligned();
  // batch support (AbstractDngDecompressor): describe instead of decode
  bool describe(const uint8_t* fileBase, rsb200_unpack_job* job) const;
  bool describeF32(const uint8_t* fileBase, rsb200_raw_job* job) const; // F32 image

private:
  void sanityCheck(uint32_t h, int bytesPerLine) const;
  void runFixed(int format, uint32_t w, uint32_t h, uint32_t bytesPerLine);
  void readF32();
  ByteStream input;
  RawImage mRaw;
  iPoint2D size, offset;
  int inputPitchBytes, bitPerPixel;
  BitOrder order;
  uint32_t skipBytes = 0;
};

// ---------------------------------------------------------------- LJPEG
class LJpegDecompressor {
public:
  struct Frame {
    iPoint2D mcu, dim;
  };
  struct PerComponentRecipe {
    const PrefixCodeDecoder<>& ht;
    uint16_t initPred;
  };
  LJpegDecompressor(RawImage img, iRectangle2D imgFrame, Frame frame,
                    std::vector<PerComponentRecipe> rec, int numLJpegRowsPerRestartInterval,
                    Buffer input);
  // decodes the scan; returns the number of input bytes consumed
  // (== BitStreamerJPEG::getStreamPosition() bookkeeping of the reference)
  uint32_t decode() const;

  // ---- batch interface used by AbstractDngDecompressor ----
  struct Segment {
    uint32_t start; // offset of the first entropy-coded byte inside `input`
  };
  // splits the scan into restart intervals (host-side RSTn marker scan) and
  // appends one rsb200_ljpeg_scan per interval; `fileBase` anchors in_offset.
  void describe(const uint8_t* fileBase, std::vector<rsb200_huff_table>& tables,
                std::vector<rsb200_ljpeg_scan>& scans, uint64_t outOffset = 0) const;
  // turns the per-interval device results into the reference's outcome
  uint32_t finish(const rsb200_scan_result* res, int nres) const;
  int numIntervals() const { return numRestartIntervals; }

private:
  RawImage mRaw;
  Buffer input;
  iRectangle2D imgFrame;
  Frame frame;
  std::vector<PerComponentRecipe> rec;
  int numLJpegRowsPerRestartInterval;
  int numRestartIntervals = 1;
  mutable std::vector<uint32_t> intervalStart; // offsets inside `input`
  mutable std::vector<uint32_t> markerPos;     // offsets of the RSTn markers
};

struct JpegComponentInfo {
  uint32_t componentId = ~0U, dcTblNo = ~0U, superH = ~0U, superV = ~0U;
};
struct SOFInfo {
  std::array<JpegComponentInfo, 4> compInfo;
  uint32_t w = 0, h = 0, cps = 0, prec = 0;
  bool initialized = false;
};

class AbstractLJpegDecoder {
public:
  AbstractLJpegDecoder(ByteStream bs, RawImage img);
  virtual ~AbstractLJpegDecoder() = default;
  int getSamplePrecision() const { return (int)frame.prec; }

  // Resumable marker walk (AbstractLJpegDecoder.cpp:65-125): runs until the SOS
  // header has been parsed (the scan is then described, not yet decoded) ...
  void decodeSOIUntilScan();
  // ... and, once the device has reported how many bytes the scan consumed,
  // continues to EOI exactly like the reference.
  void decodeSOIAfterScan(uint32_t scanLength);
  bool scanPending() const { return pendingScan; }

protected:
  bool fixDng16Bug = false;
  bool fullDecodeHT = true;
  void decodeSOI(); // immediate mode: parse, decode (device), finish
  void parseSOF(ByteStream data, SOFInfo* i);
  void parseSOS(ByteStream data);
  void parseDHT(ByteStream data);
  void parseDRI(ByteStream dri);
  uint8_t getNextMarker(bool allowskip);
  std::vector<const PrefixCodeDecoder<>*> getPrefixCodeDecoders(int N_COMP) const;
  std::vector<uint16_t> getInitialPredictors(int N_COMP) const;
  // builds the decompressor for the scan (validation happens here, as in the
  // reference's decodeScan()); decoding is deferred to runScan()
  virtual void prepareScan() = 0;
  virtual uint32_t runScan() = 0; // immediate-mode decode, returns bytes consumed

  ByteStream input;
  RawImage mRaw;
  SOFInfo frame;
  uint16_t numMCUsPerRestartInterval = 0;
  uint32_t predictorMode = 0;
  uint32_t Pt = 0;
  std::array<const PrefixCodeDecoder<>*, 4> huff{{}};
  std::vector<std::unique_ptr<HuffmanCode<>>> huffmanCodeStore;
  std::vector<std::unique_ptr<PrefixCodeDecoder<>>> PrefixCodeDecoderStore;

private:
  void markerLoop(bool resume);
  bool pendingScan = false;
  bool immediate = true;
  struct {
    bool DRI = false, DHT = false, SOF = false, SOS = false;
  } found;
};

class LJpegDecoder final : public AbstractLJpegDecoder {
public:
  LJpegDecoder(ByteStream bs, const RawImage& img);
  // immediate decode of one tile (AbstractDngDecompressor.cpp:118-121 call shape)
  void decode(uint32_t offsetX, uint32_t offsetY, uint32_t width, uint32_t height,
              iPoint2D maxDim, bool fixDng16Bug);
  // batch: validate + parse up to the scan; false if the tile needs nothing
  bool prepare(uint32_t offsetX, uint32_t offsetY, uint32_t width, uint32_t height,
               iPoint2D maxDim, bool fixDng16Bug);
  const LJpegDecompressor* scan() const { return d.get(); }

private:
  void prepareScan() override;
  uint32_t runScan() override;
  uint32_t offX = 0, offY = 0, w = 0, h = 0;
  iPoint2D maxDim;
  std::unique_ptr<LJpegDecompressor> d;
};

// ---------------------------------------------------------------- CR2
class Cr2SliceWidths {
public:
  Cr2SliceWidths() = default;
  Cr2SliceWidths(uint16_t numSlices_, uint16_t sliceWidth_, uint16_t lastSliceWidth_);
  bool empty() const { return 0 == numSlices && 0 == sliceWidth && 0 == lastSliceWidth; }
  int widthOfSlice(int sliceId) const {
    return (sliceId + 1) == numSlices ? lastSliceWidth : sliceWidth;
  }
  int numSlices = 0, sliceWidth = 0, lastSliceWidth = 0;
};

template <typename HT = PrefixCodeDecoder<>> class Cr2Decompressor {
public:
  struct PerComponentRecipe {
    const HT& ht;
    uint16_t initPred;
  };
  Cr2Decompressor(RawImage mRaw, std::tuple<int, int, int> format, iPoint2D frame,
                  Cr2SliceWidths slicing, std::vector<PerComponentRecipe> rec, Buffer input);
  uint32_t decompress() const;

private:
  RawImage mRaw;
  std::tuple<int, int, int> format;
  iPoint2D dim, frame;
  Cr2SliceWidths slicing; // already divided by the slice column step
  Cr2SliceWidths rawSlicing;
  iPoint2D rawFrame;
  std::vector<PerComponentRecipe> rec;
  Buffer input;
};

class Cr2LJpegDecoder final : public AbstractLJpegDecoder {
public:
  Cr2LJpegDecoder(ByteStream bs, const RawImage& img);
  void decode(const Cr2SliceWidths& slicing);

private:
  void prepareScan() override;
  uint32_t runScan() override;
  Cr2SliceWidths slicing;
  std::unique_ptr<Cr2Decompressor<>> d;
};

// ---------------------------------------------------------------- Hasselblad
// decompressors/HasselbladDecompressor.h:37-64 / HasselbladLJpegDecoder.h: same constructors and
// decompress() / decode().  Header walk and validation on the host, the pair stream on the device
// (rsb200_hasselblad_plan_create).
class HasselbladDecompressor final {
public:
  struct PerComponentRecipe {
    const PrefixCodeDecoder<>& ht;
    uint16_t initPred;
  };
  HasselbladDecompressor(RawImage mRaw, const PerComponentRecipe& rec, Buffer input);
  uint32_t decompress(); // returns BitStreamerMSB32::getStreamPosition()

private:
  RawImage mRaw;
  PerComponentRecipe rec;
  Buffer input;
};

class HasselbladLJpegDecoder final : public AbstractLJpegDecoder {
public:
  HasselbladLJpegDecoder(ByteStream bs, const RawImage& img);
  void decode();

private:
  void prepareScan() override;
  uint32_t runScan() override;
  std::unique_ptr<HasselbladDecompressor> d;
};

// ---------------------------------------------------------------- Pentax
// decompressors/PentaxDecompressor.h: same constructor (image + optional table
// description from the maker note) and decompress(ByteStream).  Table set-up and
// validation on the host (PentaxDecompressor.cpp:55-153), the Huffman decode and
// the predictor on the device.
class PentaxDecompressor final {
public:
  // metaData == nullptr: the built-in legacy table
  PentaxDecompressor(RawImage img, const ByteStream* metaData);
  void decompress(ByteStream data) const;
  const PrefixCodeDecoder<>& table() const { return ht; }

private:
  static HuffmanCode<> SetupPrefixCodeDecoder_Legacy();
  static HuffmanCode<> SetupPrefixCodeDecoder_Modern(ByteStream stream);
  static PrefixCodeDecoder<> SetupPrefixCodeDecoder(const ByteStream* metaData);
  RawImage mRaw;
  const PrefixCodeDecoder<> ht;
};

// ---------------------------------------------------------------- Samsung V0
// decompressors/SamsungV0Decompressor.h: same constructor (image, offset table bso, row data bsr;
// its checks and computeStripes, SamsungV0Decompressor.cpp:44-90, on the host) and decompress().
// The rows are decoded on the device (samsung0.cuh); errors are thrown with the reference's classes
// and messages.
class SamsungV0Decompressor final {
public:
  SamsungV0Decompressor(const RawImage& image, ByteStream bso, ByteStream bsr);
  void decompress() const;

private:
  void computeStripes(ByteStream bso, ByteStream bsr);
  RawImage mRaw;
  std::vector<ByteStream> stripes;
};

// ---------------------------------------------------------------- Samsung V1
// decompressors/SamsungV1Decompressor.h: same constructor (image, stream, bits per sample; its
// checks, SamsungV1Decompressor.cpp:45-61) and decompress().  The whole decode runs on the device
// (samsung1.cuh); errors are thrown with the reference's classes and messages.
class SamsungV1Decompressor final {
public:
  SamsungV1Decompressor(const RawImage& image, ByteStream bs, int bit);
  void decompress() const;

private:
  RawImage mRaw;
  ByteStream bs;
};

// ---------------------------------------------------------------- Samsung V2
// decompressors/SamsungV2Decompressor.h: same constructor (image, stream, bits per sample; its checks,
// SamsungV2Decompressor.cpp:85-143, in its order, with the 16-byte header read on the host) and
// decompress().  The rows are decoded on the device (samsung2.cuh); errors are thrown with the
// reference's classes and messages, printed values included.
class SamsungV2Decompressor final {
public:
  SamsungV2Decompressor(const RawImage& image, ByteStream bs, unsigned bits);
  void decompress() const;

private:
  RawImage mRaw;
  ByteStream bs;
  unsigned bits;
};

// ---------------------------------------------------------------- Kodak DCR
// decompressors/KodakDecompressor.h: same constructor (image, stream, bits per sample,
// uncorrectedRawValues; its checks, KodakDecompressor.cpp:46-65, in its order) and decompress().  The
// segments are decoded on the device (kodak.cuh) through the image's table (none, plain or dithered);
// errors are thrown with the reference's classes and messages, printed values included.
class KodakDecompressor final {
public:
  KodakDecompressor(RawImage img, ByteStream bs, int bps, bool uncorrectedRawValues);
  void decompress() const;

private:
  RawImage mRaw;
  ByteStream input;
  int bps;
  bool uncorrectedRawValues;
};

// ---------------------------------------------------------------- GoPro VC-5
// decompressors/VC5Decompressor.h: the constructor (stream, image; its checks and the tag walk,
// VC5Decompressor.cpp:382-618, with the reference's messages) and decode(offsetX, offsetY, width,
// height).  Two arguments more than the reference's: the image's Bayer phase (0..3 as BayerPhase, -1
// for a CFA that is not 2x2; this RawImage carries no CFA), and the codebook (the entries of the
// reference's table17.inc), which goes to the plan as it is.  The bands are decoded and the wavelets
// reconstructed on the device (vc5.cuh); a band failure goes through setError and is rethrown as
// "Too many errors encountered. Giving up. First Error:\n..." as VC5Decompressor::decode does.
// Images of 32 or fewer columns or rows, where the reference reads outside its bands, are refused.
class VC5Decompressor final {
public:
  VC5Decompressor(ByteStream bs, const RawImage& img, int phase, const rsb200_vc5_code* codes, int ncodes);
  void decode(unsigned int offsetX, unsigned int offsetY, unsigned int width, unsigned int height);

private:
  RawImage mRaw;
  ByteStream mBs;
  std::vector<rsb200_vc5_code> codes;
  rsb200_vc5_job job;
  rsb200_vc5_band bands[40];
};

// ---------------------------------------------------------------- Sony ARW1
// decompressors/SonyArw1Decompressor.h: same constructor (image; its checks,
// SonyArw1Decompressor.cpp:39-50) and decompress(ByteStream).  The whole decode runs
// on the device (arw1.cuh); errors are thrown with the reference's classes.
class SonyArw1Decompressor final {
public:
  explicit SonyArw1Decompressor(RawImage img);
  void decompress(ByteStream input) const;

private:
  RawImage mRaw;
};

// ---------------------------------------------------------------- Nikon
// decompressors/NikonDecompressor.h: same constructor (image, maker-note stream,
// bits per sample) and decompress(input, uncorrectedRawValues).  The constructor work
// (version bytes, tree selection, start predictors, createCurve, split;
// NikonDecompressor.cpp:380-511) is host code; Huffman decode, predictor, clamp and
// the dithered curve run on the device.  Streams with a non-zero split ("lossy after
// split", NikonLASDecompressor) are not supported yet and throw.
class NikonDecompressor final {
public:
  NikonDecompressor(RawImage raw, ByteStream metadata, uint32_t bitsPS);
  void decompress(Buffer input, bool uncorrectedRawValues);
  const std::vector<uint16_t>& getCurve() const { return curve; }
  uint32_t getSplit() const { return split; }

private:
  static std::vector<uint16_t> createCurve(ByteStream& metadata, uint32_t bitsPS, uint32_t v0,
                                           uint32_t v1, uint32_t* split);
  static PrefixCodeDecoder<> createPrefixCodeDecoder(uint32_t huffSelect);
  RawImage mRaw;
  uint32_t bitsPS;
  uint32_t huffSelect = 0;
  uint32_t split = 0;
  int pUp[2][2];
  std::vector<uint16_t> curve;
};

// ---------------------------------------------------------------- Panasonic
// decompressors/PanasonicV{5,6,7}Decompressor.h: same constructors (image, byte
// stream[, bps]) with the reference's validation, decompress() runs on the device.
// decompressors/PanasonicV4Decompressor.h:37-98: zero_is_not_bad = false makes decompress()
// append the positions of the pixels decoded as 0 to mRaw->mBadPixelPositions (unordered, as
// the reference's thread schedule leaves them)
class PanasonicV4Decompressor final {
public:
  PanasonicV4Decompressor(RawImage img, ByteStream input_, bool zero_is_not_bad,
                          uint32_t section_split_offset_);
  void decompress() const;

private:
  RawImage mRaw;
  ByteStream input;
  bool zero_is_bad;
  uint32_t section_split_offset;
};
class PanasonicV5Decompressor final {
public:
  PanasonicV5Decompressor(RawImage img, ByteStream input_, uint32_t bps_);
  void decompress() const;

private:
  RawImage mRaw;
  ByteStream input;
  uint32_t bps;
};
class PanasonicV6Decompressor final {
public:
  PanasonicV6Decompressor(RawImage img, ByteStream input_, uint32_t bps_);
  void decompress() const;

private:
  RawImage mRaw;
  ByteStream input;
  uint32_t bps;
};
class PanasonicV7Decompressor final {
public:
  PanasonicV7Decompressor(RawImage img, ByteStream input_);
  void decompress() const;

private:
  RawImage mRaw;
  ByteStream input;
};

// ---------------------------------------------------------------- Phase One
// decompressors/PhaseOneDecompressor.h: one strip per image row.
struct PhaseOneStrip final {
  int n = 0;
  ByteStream bs;
  PhaseOneStrip() = default;
  PhaseOneStrip(int block, ByteStream bs_) : n(block), bs(bs_) {}
};

class PhaseOneDecompressor final {
public:
  PhaseOneDecompressor(RawImage img, std::vector<PhaseOneStrip>&& strips_);
  void decompress() const;

private:
  void prepareStrips();
  RawImage mRaw;
  std::vector<PhaseOneStrip> strips;
};

// ---------------------------------------------------------------- Sony ARW2
// decompressors/SonyArw2Decompressor.h: same constructor (image + the byte stream,
// one byte per pixel) and decompress().  The image's table (RawImageData::setTable,
// set by ArwDecoder through RawImageCurveGuard) is applied on the device, including
// the dithered form.
class SonyArw2Decompressor final {
public:
  SonyArw2Decompressor(RawImage img, ByteStream input);
  void decompress() const;

private:
  RawImage mRaw;
  ByteStream input;
};

// ---------------------------------------------------------------- sRaw
// ---------------------------------------------------------------- DngOpcodes
// common/DngOpcodes.h:41-88 -- same constructor (parses and validates the big-endian list
// against the image and its crop, common/DngOpcodes.cpp:666-726) and applyOpCodes(); the
// per-sample work of all opcodes runs as ONE pass on the device (K10), the bad-pixel list and
// crop bookkeeping on the host in the reference's order.
class DngOpcodes final {
public:
  DngOpcodes(const RawImage& ri, ByteStream bs);
  ~DngOpcodes();
  void applyOpCodes(const RawImage& ri) const;

  // The list in device form for `ri` in its current state (setup() of every opcode done, in
  // order; ROIs in uncropped coordinates) + the host-side actions, in list order.
  struct Action {
    enum Kind { BadList, BadConstant, Trim } kind;
    uint32_t index; // BadList: opcode; BadConstant: index into Lowered::ops; Trim: opcode
  };
  struct Lowered {
    std::vector<rsb200_dng_op> ops;
    std::vector<uint16_t> tables; // 65536 per table
    std::vector<uint32_t> deltas;
    std::vector<Action> actions;
    std::exception_ptr error; // setup()/apply() error of the first opcode that failed, if any
  };
  Lowered lower(const RawImage& ri) const;
  // opcode `i`: its bad-pixel list (FixBadPixelsList) / ROI (TrimBounds)
  const std::vector<uint32_t>& badPixels(uint32_t i) const { return opcodes[i].badPixels; }
  iRectangle2D roi(uint32_t i) const { return opcodes[i].roi; }

private:
  struct Op {
    uint32_t code = 0;
    uint32_t value = 0;
    std::vector<uint32_t> badPixels;
    iRectangle2D roi;
    uint32_t firstPlane = 0, planes = 0, rowPitch = 0, colPitch = 0;
    std::vector<uint16_t> lookup;
    std::vector<float> deltaF;
  };
  std::vector<Op> opcodes;
  static void readRoi(ByteStream& bs, const iPoint2D& dim, Op& op);
  static void readPixelOpcode(const RawImage& ri, ByteStream& bs, const iPoint2D& dim, Op& op);
};

// interpolators/Cr2sRawInterpolator.h:36-60 -- same constructor and interpolate();
// the per-pixel work (chroma interpolation + YCbCr->RGB) runs on the device.
class Cr2sRawInterpolator final {
public:
  Cr2sRawInterpolator(const RawImage& mRaw_, Array2DRef<const uint16_t> input_,
                      std::array<int, 3> sraw_coeffs_, int hue_)
      : mRaw(mRaw_), input(input_), sraw_coeffs(sraw_coeffs_), hue(hue_) {}
  void interpolate(int version);

private:
  const RawImage& mRaw;
  const Array2DRef<const uint16_t> input;
  std::array<int, 3> sraw_coeffs;
  int hue;
};

// ---------------------------------------------------------------- DNG
struct DngTilingDescription {
  const iPoint2D& dim;
  const uint32_t tileW, tileH, tilesX, tilesY;
  const unsigned numTiles;
  DngTilingDescription(const iPoint2D& dim_, uint32_t tileW_, uint32_t tileH_)
      : dim(dim_), tileW(tileW_), tileH(tileH_), tilesX((dim_.x + tileW_ - 1) / tileW_),
        tilesY((dim_.y + tileH_ - 1) / tileH_), numTiles(tilesX * tilesY) {}
};

struct DngSliceElement {
  const DngTilingDescription& dsc;
  const unsigned n;
  const ByteStream bs;
  const unsigned column, row;
  const bool lastColumn, lastRow;
  const unsigned offX, offY, width, height;
  DngSliceElement(const DngTilingDescription& dsc_, unsigned n_, ByteStream bs_)
      : dsc(dsc_), n(n_), bs(bs_), column(n_ % dsc_.tilesX), row(n_ / dsc_.tilesX),
        lastColumn((column + 1) == dsc_.tilesX), lastRow((row + 1) == dsc_.tilesY),
        offX(dsc_.tileW * column), offY(dsc_.tileH * row),
        width(!lastColumn ? dsc_.tileW : dsc_.dim.x - offX),
        height(!lastRow ? dsc_.tileH : dsc_.dim.y - offY) {}
};

class AbstractDngDecompressor {
public:
  AbstractDngDecompressor(RawImage img, const DngTilingDescription& dsc_, int compression_,
                          bool mFixLjpeg_, uint32_t mBps_, uint32_t mPredictor_)
      : dsc(dsc_), compression(compression_), mFixLjpeg(mFixLjpeg_), mBps(mBps_),
        mPredictor(mPredictor_), mRaw(std::move(img)) {}
  // all tiles of the frame go to the device in ONE plan (the reference fans them
  // out over OpenMP threads, AbstractDngDecompressor.cpp:54-131,240-252)
  void decompress() const;
  // The host half of the LJPEG path: per tile the marker walk / validation / restart-marker
  // scan (LJpegDecoder::prepare, on `threads` host threads: 0 = min(16, hardware threads),
  // RSB200_HOST_THREADS overrides) and, in tile order, the scan descriptors and de-duplicated
  // tables the device plan is made of.  Tile errors come back in tile order, as the serial walk
  // of the reference's single-threaded build reports them.
  struct PreparedLJpeg {
    struct Tile {
      std::unique_ptr<LJpegDecoder> dec;
      int firstScan = 0, nScans = 0;
    };
    std::vector<Tile> tiles;
    std::vector<rsb200_huff_table> tables;
    std::vector<rsb200_ljpeg_scan> scans;
    std::vector<std::string> errors;
    std::vector<uint8_t> errorIsIOE; // per entry of `errors`: IOException (1) or RawDecoderException (0)
    const uint8_t* base = nullptr; // the file span the scans' offsets refer to
    size_t span = 0;
  };
  PreparedLJpeg prepareLJpeg(unsigned threads = 0) const;
  const DngTilingDescription dsc;
  std::vector<DngSliceElement> slices;
  const int compression;
  const bool mFixLjpeg;
  const uint32_t mBps, mPredictor;

private:
  RawImage mRaw;
  void decompressUncompressed() const;
  void decompressLJpeg() const;
};

} // namespace rawspeed_b200
