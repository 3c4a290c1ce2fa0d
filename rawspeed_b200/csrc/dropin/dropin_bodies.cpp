// dropin_bodies.cpp -- the reference-side half of the drop-in: OUR bodies for the four hot-path
// methods of darktable-org/rawspeed, written against the reference's own headers (RawImage,
// ByteStream, PrefixCodeDecoder<>, iRectangle2D ...) and calling the rawspeed_b200 C ABI
// (include/rawspeed_b200.h).  Everything else of the reference -- parsers, TIFF, decoders, marker
// walks, constructors with their checks, exceptions -- is compiled unmodified
// (oracle/Makefile.dropin: the original bodies just get another name), so RawParser ->
// RawDecoder::decodeRaw() -> RawDecoder::decodeRawInternal() runs the reference's code up to the
// per-pixel loops and this file from there:
//
//   UncompressedDecompressor::readUncompressedRaw   decompressors/UncompressedDecompressor.cpp:202-268
//   LJpegDecompressor::decode                        decompressors/LJpegDecompressor.cpp:339-370
//   Cr2Decompressor<PrefixCodeDecoder<>>::decompress decompressors/Cr2DecompressorImpl.h:470-487
//   AbstractDngDecompressor::decompress              decompressors/AbstractDngDecompressor.cpp:240-252
//
// There is no CPU fallback: forms the engine does not take raise RawDecoderException.
#include "rawspeedconfig.h"
#include "codes/PrefixCodeDecoder.h"
#include "common/BayerPhase.h"
#include "common/RawImage.h"
#include "common/RawspeedException.h"
#include "decoders/RawDecoderException.h"
#include "decompressors/AbstractDngDecompressor.h"
#include "decompressors/Cr2Decompressor.h"
#include "decompressors/LJpegDecoder.h"
#include "decompressors/LJpegDecompressor.h"
#include "decompressors/UncompressedDecompressor.h"
#include "io/IOException.h"

#include "rawspeed_b200.h"
#include "../vc5_parse.h"

#include <algorithm>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

extern "C" int rawspeed_get_number_of_processor_cores();

namespace rawspeed {
namespace {

// one engine context per process (device 0 or RSB200_DEVICE)
rsb200_ctx* engine() {
  static rsb200_ctx* ctx = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    int dev = 0;
    if (const char* e = getenv("RSB200_DEVICE"))
      dev = atoi(e);
    if (rsb200_create(dev, &ctx) != RSB200_OK)
      ctx = nullptr;
  });
  if (!ctx)
    ThrowRDE("rawspeed_b200: no usable CUDA device (there is no CPU fallback)");
  return ctx;
}
std::mutex& engine_mutex() {
  static std::mutex m;
  return m;
}

[[noreturn]] void throw_status(int rc, const char* what) {
  if (rc == RSB200_ERR_IOE)
    ThrowIOE("%s: %s", what, rsb200_last_error(engine()));
  ThrowRDE("%s: %s", what, rsb200_last_error(engine()));
}

struct PlanGuard {
  rsb200_plan* p = nullptr;
  ~PlanGuard() {
    if (p)
      rsb200_plan_destroy(p);
  }
};

// The VC-5 codebook of the integrator's reference checkout (src/external/gopro/vc5/table17.inc, on the
// include path of this unit), in the shapes that file expects; it reaches the plan as an argument.
struct RLV final {
  uint_fast8_t size; // code length in bits
  uint32_t bits;     // code word, right-justified
  uint16_t count;    // run length
  uint16_t value;    // run value (unsigned)
};
#define RLVTABLE(n)                                                                                    \
  struct {                                                                                             \
    const uint32_t length;                                                                             \
    const RLV entries[n];                                                                              \
  } constexpr
#include "gopro/vc5/table17.inc"
#undef RLVTABLE

const std::vector<rsb200_vc5_code>& vc5_codebook() {
  static const std::vector<rsb200_vc5_code> codes = [] {
    std::vector<rsb200_vc5_code> c;
    for (const RLV& e : table17.entries)
      c.push_back(rsb200_vc5_code{e.size, e.bits, e.count, e.value});
    return c;
  }();
  return codes;
}

[[noreturn]] void throw_outcome(const rsb200_vc5::Outcome& o) {
  if (o.cls == rsb200_vc5::IOE)
    ThrowIOE("%s", o.msg.c_str());
  ThrowRDE("%s", o.msg.c_str());
}

// VC5Decompressor(bs, mRaw) + decode(offX, offY, width, height) of one DNG tile (the reference's
// decompressThread<9>, AbstractDngDecompressor.cpp:161-179): the constructor's checks and the tag walk on
// the host (vc5_parse.h), the bands and wavelets on the device, a band failure rethrown as decode() does.
void vc5_tile(const RawImage& mRaw, const ByteStream& bs, int offX, int offY, int width, int height) {
  if (mRaw->getCpp() != 1 || mRaw->getDataType() != RawImageType::UINT16 || mRaw->getBpp() != sizeof(uint16_t))
    ThrowRDE("Unexpected component count / data type");
  const Optional<BayerPhase> phase = getAsBayerPhase(mRaw->cfa);
  const uint8_t* data = bs.peekData(bs.getRemainSize());
  const uint32_t size = static_cast<uint32_t>(bs.getRemainSize());
  rsb200_vc5::Parsed p;
  const rsb200_vc5::Outcome o = rsb200_vc5::parse(data, size, mRaw->dim.x, mRaw->dim.y,
                                                  mRaw->whitePoint ? *mRaw->whitePoint : 0,
                                                  phase ? static_cast<int>(*phase) : -1, p);
  if (o.cls != rsb200_vc5::OK)
    throw_outcome(o);
  if (offX || offY || mRaw->dim != iPoint2D(width, height))
    ThrowRDE("VC5Decompressor expects to fill the whole image, not some tile.");
  const auto img = mRaw->getU16DataAsUncroppedArray2DRef();
  const uint32_t pitch = static_cast<uint32_t>(img.pitch()) * 2u;
  p.job.out_offset = 0;
  p.job.out_pitch = pitch;
  const std::vector<rsb200_vc5_code>& codes = vc5_codebook();
  std::lock_guard<std::mutex> g(engine_mutex());
  PlanGuard pg;
  int rc = rsb200_vc5_plan_create(engine(), codes.data(), static_cast<int>(codes.size()), &p.job, 1, p.bands, 40,
                                  &pg.p);
  if (rc != RSB200_OK)
    throw_status(rc, "VC5Decompressor");
  // partial: a failed frame leaves the image as it was
  rc = rsb200_plan_run_host_image(pg.p, data, size, reinterpret_cast<uint8_t*>(&img(0, 0)), pitch,
                                  static_cast<uint32_t>(mRaw->dim.x) * 2u, static_cast<uint32_t>(mRaw->dim.y), 1);
  if (rc != RSB200_OK)
    throw_status(rc, "VC5Decompressor");
  rsb200_scan_result res;
  rc = rsb200_plan_results(pg.p, &res, 1);
  if (rc == RSB200_OK)
    return;
  if (rc != RSB200_ERR_RDE && rc != RSB200_ERR_IOE)
    throw_status(rc, "VC5Decompressor");
  mRaw->setError(rsb200_vc5::band_failure(res.consumed).msg);
  std::string firstErr;
  if (mRaw->isTooManyErrors(1, &firstErr))
    ThrowRDE("Too many errors encountered. Giving up. First Error:\n%s", firstErr.c_str());
}

rsb200_huff_table table_of(const PrefixCodeDecoder<>& ht) {
  rsb200_huff_table t;
  memset(&t, 0, sizeof t);
  const auto& n = ht.code.nCodesPerLength; // index = code length
  for (size_t l = 1; l < n.size() && l <= 16; ++l)
    t.ncodes_per_len[l - 1] = static_cast<uint8_t>(n[l]);
  const auto& v = ht.code.codeValues;
  t.nvalues = static_cast<uint16_t>(std::min<size_t>(v.size(), 162));
  for (size_t i = 0; i < t.nvalues; ++i)
    t.values[i] = static_cast<uint8_t>(v[i]);
  t.fix_dng16 = ht.handleDNGBug16() ? 1 : 0;
  return t;
}

int add_table(std::vector<rsb200_huff_table>& tabs, const rsb200_huff_table& t) {
  for (size_t i = 0; i < tabs.size(); ++i)
    if (!memcmp(&tabs[i], &t, sizeof t))
      return static_cast<int>(i);
  tabs.push_back(t);
  return static_cast<int>(tabs.size()) - 1;
}

// ---- a batch of LJPEG tiles collected while the reference's own tile loop runs ----
struct TileJob {
  const uint8_t* data; // entropy-coded bytes (behind SOS)
  uint32_t size;
  iRectangle2D imgFrame;
  iPoint2D mcu, frameDim;
  int rowsPerRestart;
  rsb200_huff_table tab[4];
  uint16_t initPred[4];
  unsigned tile; // which DngSliceElement
};
struct Batch {
  std::mutex m;
  std::vector<TileJob> jobs;
};
thread_local Batch* t_batch = nullptr;
thread_local unsigned t_tile = 0;

// offsets of the restart intervals of one tile (LJpegDecompressor.cpp:283-297: interval k > 0
// starts behind the marker FF D0+((k-1)%8) that follows the previous interval's data)
std::vector<uint32_t> interval_starts(const uint8_t* p, uint32_t n, int nIntervals) {
  std::vector<uint32_t> s{0u};
  uint32_t pos = 0;
  for (int k = 1; k < nIntervals; ++k) {
    bool found = false;
    while (pos + 1 < n) {
      const auto* q = static_cast<const uint8_t*>(memchr(p + pos, 0xFF, n - 1 - pos));
      if (!q)
        break;
      pos = static_cast<uint32_t>(q - p);
      const uint8_t m = p[pos + 1];
      if (m == 0x00 || m == 0xFF) {
        pos += (m == 0x00) ? 2 : 1;
        continue;
      }
      if (m < 0xD0 || m > 0xD7)
        ThrowRDE("Not a restart marker!");
      if (m - 0xD0 != ((k - 1) % 8))
        ThrowRDE("Unexpected restart marker found");
      pos += 2;
      s.push_back(pos);
      found = true;
      break;
    }
    if (!found)
      ThrowRDE("Jpeg marker not encountered");
  }
  return s;
}

void append_scans(const TileJob& j, const uint8_t* base, uint32_t cpp, uint64_t out_offset,
                  uint32_t out_pitch, std::vector<rsb200_huff_table>& tabs,
                  std::vector<rsb200_ljpeg_scan>& scans, std::vector<unsigned>* owner) {
  const int rowsTotal = j.imgFrame.dim.y / j.mcu.y;
  const int nIntervals = (rowsTotal + j.rowsPerRestart - 1) / j.rowsPerRestart;
  const auto starts = interval_starts(j.data, j.size, nIntervals);
  int tid[4] = {0, 0, 0, 0};
  const int ncomp = j.mcu.x * j.mcu.y;
  for (int c = 0; c < ncomp; ++c)
    tid[c] = add_table(tabs, j.tab[c]);
  for (int k = 0; k < nIntervals; ++k) {
    rsb200_ljpeg_scan s;
    memset(&s, 0, sizeof s);
    s.in_offset = static_cast<uint64_t>(j.data - base) + starts[static_cast<size_t>(k)];
    s.in_size = j.size - starts[static_cast<size_t>(k)];
    s.rows = static_cast<uint32_t>(std::min(j.rowsPerRestart, rowsTotal - k * j.rowsPerRestart));
    s.frame_w = static_cast<uint32_t>(j.frameDim.x);
    s.mcu_w = static_cast<uint8_t>(j.mcu.x);
    s.mcu_h = static_cast<uint8_t>(j.mcu.y);
    for (int c = 0; c < ncomp; ++c) {
      s.table[c] = static_cast<uint8_t>(tid[c]);
      s.init_pred[c] = j.initPred[c];
    }
    s.out_offset = out_offset;
    s.out_pitch = out_pitch;
    s.out_x = cpp * static_cast<uint32_t>(j.imgFrame.pos.x);
    s.out_y = static_cast<uint32_t>(j.imgFrame.pos.y + k * j.rowsPerRestart * j.mcu.y);
    s.store_w = cpp * static_cast<uint32_t>(j.imgFrame.dim.x);
    scans.push_back(s);
    if (owner)
      owner->push_back(j.tile);
  }
}

} // namespace

// ======================= LJpegDecompressor::decode =======================
// One tile (S2b).  Inside AbstractDngDecompressor::decompress() (below) the call only RECORDS the
// tile: the whole frame then goes to the device as one plan.
ByteStream::size_type LJpegDecompressor::decode() const {
  if (mRaw->getDataType() != RawImageType::UINT16)
    ThrowRDE("rawspeed_b200: LJPEG into a non-uint16 image");
  TileJob j;
  j.data = input.begin();
  j.size = static_cast<uint32_t>(input.size());
  j.imgFrame = imgFrame;
  j.mcu = frame.mcu;
  j.frameDim = frame.dim;
  j.rowsPerRestart = numLJpegRowsPerRestartInterval;
  j.tile = t_tile;
  for (size_t c = 0; c < rec.size() && c < 4; ++c) {
    j.tab[c] = table_of(rec[c].ht);
    j.initPred[c] = rec[c].initPred;
  }
  if (t_batch) {
    {
      std::lock_guard<std::mutex> g(t_batch->m);
      t_batch->jobs.push_back(j);
    }
    // The caller (AbstractLJpegDecoder::parseSOS) skips this many bytes and then looks for the
    // next marker; the exact position is known only after the batch has run, so point it at the
    // EOI that ends the tile (its last FF D9).
    for (uint32_t p = j.size; p >= 2; --p)
      if (j.data[p - 2] == 0xFF && j.data[p - 1] == 0xD9)
        return static_cast<ByteStream::size_type>(p - 2);
    return static_cast<ByteStream::size_type>(j.size);
  }
  // stand-alone: this tile alone, rows [pos.y, pos.y + dim.y) of the image through host buffers
  const auto img = mRaw->getU16DataAsUncroppedArray2DRef();
  const uint32_t pitch = static_cast<uint32_t>(img.pitch()) * 2u;
  auto* rows0 = reinterpret_cast<uint8_t*>(&img(imgFrame.pos.y, 0));
  TileJob rel = j;
  rel.imgFrame.pos.y = 0;
  std::vector<rsb200_huff_table> tabs;
  std::vector<rsb200_ljpeg_scan> scans;
  append_scans(rel, j.data, mRaw->getCpp(), 0, pitch, tabs, scans, nullptr);
  std::lock_guard<std::mutex> g(engine_mutex());
  PlanGuard pg;
  int rc = rsb200_ljpeg_plan_create(engine(), tabs.data(), static_cast<int>(tabs.size()), scans.data(),
                                    static_cast<int>(scans.size()), &pg.p);
  if (rc != RSB200_OK)
    throw_status(rc, "LJpegDecompressor");
  rc = rsb200_plan_run_host_image(pg.p, j.data, j.size, rows0, pitch,
                                  static_cast<uint32_t>(img.width()) * 2u,
                                  static_cast<uint32_t>(imgFrame.dim.y), /*partial=*/1);
  if (rc != RSB200_OK)
    throw_status(rc, "LJpegDecompressor");
  std::vector<rsb200_scan_result> res(scans.size());
  rc = rsb200_plan_results(pg.p, res.data(), static_cast<int>(res.size()));
  if (rc == RSB200_ERR_IOE)
    ThrowIOE("Buffer overflow read in BitStreamer");
  if (rc != RSB200_OK)
    ThrowRDE("bad Huffman code (rawspeed_b200 status %d)", rc);
  return static_cast<ByteStream::size_type>(scans.back().in_offset + res.back().consumed);
}

// ======================= AbstractDngDecompressor::decompress =======================
template <> void AbstractDngDecompressor::decompressThread<7>() const noexcept;

void AbstractDngDecompressor::decompress() const {
  if (compression == 7 && mRaw->getDataType() == RawImageType::UINT16) {
    // The reference's own tile loop (LJpegDecoder: SOI/SOF3/DHT/DRI/SOS walk, validation) runs
    // on the host cores with OpenMP exactly as before; each tile's LJpegDecompressor::decode()
    // records its job instead of decoding; then ONE plan decodes every tile of the frame.
    Batch batch;
    batch.jobs.reserve(slices.size());
    // (decompressThread<7> holds an orphaned `omp for`: it shares the tiles of the enclosing team)
#pragma omp parallel num_threads(rawspeed_get_number_of_processor_cores()) if (slices.size() > 1)
    {
      t_batch = &batch;
      decompressThread<7>();
      t_batch = nullptr;
    }
    if (!batch.jobs.empty()) {
      const auto img = mRaw->getU16DataAsUncroppedArray2DRef();
      const uint32_t pitch = static_cast<uint32_t>(img.pitch()) * 2u;
      const uint8_t* lo = batch.jobs[0].data;
      const uint8_t* hi = lo;
      for (const TileJob& j : batch.jobs) {
        lo = std::min(lo, j.data);
        hi = std::max(hi, j.data + j.size);
      }
      std::sort(batch.jobs.begin(), batch.jobs.end(),
                [](const TileJob& a, const TileJob& b) { return a.data < b.data; });
      std::vector<rsb200_huff_table> tabs;
      std::vector<rsb200_ljpeg_scan> scans;
      // every tile was recorded: together they cover the whole image (DngTilingDescription), so the
      // current image contents need not travel to the device first
      const bool covers_image = batch.jobs.size() == slices.size() && slices.size() == dsc.numTiles;
      try {
        for (const TileJob& j : batch.jobs)
          append_scans(j, lo, mRaw->getCpp(), 0, pitch, tabs, scans, nullptr);
        std::lock_guard<std::mutex> g(engine_mutex());
        PlanGuard pg;
        int rc = rsb200_ljpeg_plan_create(engine(), tabs.data(), static_cast<int>(tabs.size()),
                                          scans.data(), static_cast<int>(scans.size()), &pg.p);
        if (rc != RSB200_OK)
          throw_status(rc, "AbstractDngDecompressor");
        rc = rsb200_plan_run_host_image(pg.p, lo, static_cast<size_t>(hi - lo),
                                        reinterpret_cast<uint8_t*>(&img(0, 0)), pitch,
                                        static_cast<uint32_t>(img.width()) * 2u,
                                        static_cast<uint32_t>(img.height()),
                                        /*partial=*/covers_image ? 0 : 1);
        if (rc != RSB200_OK)
          throw_status(rc, "AbstractDngDecompressor");
        std::vector<rsb200_scan_result> res(scans.size());
        rsb200_plan_results(pg.p, res.data(), static_cast<int>(res.size()));
        for (const rsb200_scan_result& r : res) {
          if (r.status == RSB200_ERR_IOE)
            mRaw->setError("Buffer overflow read in BitStreamer");
          else if (r.status != RSB200_OK)
            mRaw->setError("bad Huffman code");
        }
      } catch (const RawDecoderException& err) {
        mRaw->setError(err.what());
      } catch (const IOException& err) {
        mRaw->setError(err.what());
      }
    }
  } else if (compression == 9) {
    // VC-5 (GoPro): every tile through the device, in the reference's tile order
    for (const auto& e : slices) {
      try {
        vc5_tile(mRaw, e.bs, static_cast<int>(e.offX), static_cast<int>(e.offY), static_cast<int>(e.width),
                 static_cast<int>(e.height));
      } catch (const RawDecoderException& err) {
        mRaw->setError(err.what());
      } catch (const IOException& err) {
        mRaw->setError(err.what());
      }
    }
  } else {
    // uncompressed tiles go through UncompressedDecompressor::readUncompressedRaw() (below);
    // Deflate / lossy JPEG tiles are outside the hot path and stay the reference's
#pragma omp parallel num_threads(rawspeed_get_number_of_processor_cores()) if (slices.size() > 1)
    decompressThread();
  }
  std::string firstErr;
  if (mRaw->isTooManyErrors(1, &firstErr)) {
    ThrowRDE("Too many errors encountered. Giving up. First Error:\n%s", firstErr.c_str());
  }
}

// ======================= UncompressedDecompressor::readUncompressedRaw =======================
void UncompressedDecompressor::readUncompressedRaw() {
  if (mRaw->getDataType() != RawImageType::UINT16)
    ThrowRDE("rawspeed_b200: floating-point strips are not part of the drop-in");
  if (bitPerPixel < 1 || bitPerPixel > 16)
    ThrowRDE("rawspeed_b200: %d bits per sample", bitPerPixel);
  const uint32_t cpp = mRaw->getCpp();
  const auto img = mRaw->getU16DataAsUncroppedArray2DRef();
  const uint32_t pitch = static_cast<uint32_t>(img.pitch()) * 2u;
  const uint32_t h = static_cast<uint32_t>(size.y);
  const uint64_t need = static_cast<uint64_t>(inputPitchBytes) * h;
  const Buffer in = input.peekRemainingBuffer();
  if (in.getSize() < need)
    ThrowIOE("Not enough data to decode. Image file truncated.");
  rsb200_unpack_job j;
  memset(&j, 0, sizeof j);
  j.in_offset = 0;
  j.in_size = static_cast<uint32_t>(std::min<uint64_t>(in.getSize(), 0xFFFFFFFFull));
  j.out_offset = 0;
  j.out_pitch = pitch;
  j.row0 = 0;
  j.rows = h;
  j.samples = cpp * static_cast<uint32_t>(size.x);
  j.out_col0 = 0; // (the reference ignores offset.x for packed integers, UncompressedDecompressor.cpp:196)
  j.in_pitch = static_cast<uint32_t>(inputPitchBytes);
  j.bps = static_cast<uint8_t>(bitPerPixel);
  j.order = order == BitOrder::LSB ? RSB200_LSB
            : order == BitOrder::MSB ? RSB200_MSB
            : order == BitOrder::MSB16 ? RSB200_MSB16 : RSB200_MSB32;
  std::lock_guard<std::mutex> g(engine_mutex());
  PlanGuard pg;
  int rc = rsb200_unpack_plan_create(engine(), &j, 1, &pg.p);
  if (rc != RSB200_OK)
    throw_status(rc, "UncompressedDecompressor");
  rc = rsb200_plan_run_host_image(pg.p, in.begin(), j.in_size,
                                  reinterpret_cast<uint8_t*>(&img(offset.y, 0)), pitch,
                                  static_cast<uint32_t>(img.width()) * 2u, h, /*partial=*/1);
  if (rc != RSB200_OK)
    throw_status(rc, "UncompressedDecompressor");
}

// ======================= Cr2Decompressor::decompress =======================
// (the header declares `extern template class Cr2Decompressor<PrefixCodeDecoder<>>`: the member is
// defined as a template here and instantiated explicitly below)
template <typename HT> ByteStream::size_type Cr2Decompressor<HT>::decompress() const {
  const auto [N_COMP, X_S_F, Y_S_F] = format;
  rsb200_cr2_job j;
  memset(&j, 0, sizeof j);
  std::vector<rsb200_huff_table> tabs;
  for (int c = 0; c < N_COMP && c < 4; ++c) {
    j.table[c] = static_cast<uint8_t>(add_table(tabs, table_of(rec[static_cast<size_t>(c)].ht)));
    j.init_pred[c] = rec[static_cast<size_t>(c)].initPred;
  }
  j.in_offset = 0;
  j.in_size = static_cast<uint32_t>(input.size());
  j.n_comp = static_cast<uint8_t>(N_COMP);
  j.x_s_f = static_cast<uint8_t>(X_S_F);
  j.y_s_f = static_cast<uint8_t>(Y_S_F);
  j.frame_w = frame.x;
  j.frame_h = frame.y;
  j.num_slices = slicing.numSlices;
  j.slice_w = slicing.sliceWidth;
  j.last_slice_w = slicing.lastSliceWidth;
  j.img_w = mRaw->dim.x * static_cast<int>(mRaw->getCpp());
  j.img_h = mRaw->dim.y;
  const auto img = mRaw->getU16DataAsUncroppedArray2DRef();
  j.out_offset = 0;
  j.out_pitch = static_cast<uint32_t>(img.pitch()) * 2u;
  std::lock_guard<std::mutex> g(engine_mutex());
  PlanGuard pg;
  int rc = rsb200_cr2_plan_create(engine(), tabs.data(), static_cast<int>(tabs.size()), &j, 1, &pg.p);
  if (rc != RSB200_OK)
    throw_status(rc, "Cr2Decompressor");
  rc = rsb200_plan_run_host_image(pg.p, input.begin(), j.in_size, reinterpret_cast<uint8_t*>(&img(0, 0)),
                                  j.out_pitch, static_cast<uint32_t>(img.width()) * 2u,
                                  static_cast<uint32_t>(img.height()), /*partial=*/1);
  if (rc != RSB200_OK)
    throw_status(rc, "Cr2Decompressor");
  rsb200_scan_result res;
  rc = rsb200_plan_results(pg.p, &res, 1);
  if (rc == RSB200_ERR_IOE)
    ThrowIOE("Buffer overflow read in BitStreamer");
  if (rc != RSB200_OK)
    ThrowRDE("bad Huffman code (rawspeed_b200 status %d)", rc);
  return static_cast<ByteStream::size_type>(res.consumed);
}
template ByteStream::size_type Cr2Decompressor<PrefixCodeDecoder<>>::decompress() const;

} // namespace rawspeed
