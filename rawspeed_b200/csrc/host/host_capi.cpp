// host_capi.cpp -- plain-C entry points over the C++ host mirror, so that the
// Python parity tests (and any C consumer) can drive the reference-shaped
// classes: same inputs as the reference's fuzz drivers
// (fuzz/librawspeed/decompressors/*.cpp), exceptions reported as codes.
#include "rawspeed_host.h"

#include <chrono>
#include <cstring>

using namespace rawspeed_b200;

extern "C" {

struct rsb200h_err {
  int code; // 0 ok, 1 RawDecoderException, 2 IOException
  char msg[240];
};

struct rsb200h_huff {
  uint8_t ncpl[16];
  uint8_t values[162];
  int nvalues;
};
}

namespace {
template <typename F> int guarded(rsb200h_err* e, F&& f) {
  if (e) {
    e->code = 0;
    e->msg[0] = 0;
  }
  try {
    f();
    return 0;
  } catch (const IOException& ex) {
    if (e) {
      e->code = 2;
      std::snprintf(e->msg, sizeof e->msg, "%s", ex.what());
    }
    return 2;
  } catch (const RawspeedException& ex) {
    if (e) {
      e->code = 1;
      std::snprintf(e->msg, sizeof e->msg, "%s", ex.what());
    }
    return 1;
  }
}

RawImage makeImage(const uint16_t* src, int w, int h, int cpp, int pitch, bool isCfa, int subX,
                   int subY) {
  RawImage img = RawImage::create(iPoint2D(w, h), RawImageType::UINT16, (uint32_t)cpp);
  img->isCFA = isCfa;
  img->subsampling = iPoint2D(subX, subY);
  if (img->pitch != pitch)
    ThrowRDE("test harness: pitch mismatch (%d vs %d)", img->pitch, pitch);
  std::memcpy(img->getByteData(), src, (size_t)pitch * h);
  return img;
}
void copyOut(RawImage& img, uint16_t* dst) {
  std::memcpy(dst, img->getByteData(), img->getByteSize());
}

PrefixCodeDecoder<> makeHT(const rsb200h_huff& t, bool fix16) {
  HuffmanCode<> hc;
  hc.setNCodesPerLength(Buffer(t.ncpl, 16));
  hc.setCodeValues(t.values, t.nvalues);
  PrefixCodeDecoder<> ht(std::move(hc));
  ht.setup(true, fix16);
  return ht;
}
} // namespace

extern "C" {

int rsb200h_unpack(const uint8_t* in, uint32_t in_size, uint16_t* img_data, int w, int h,
                   int cpp, int pitch, int crop_x, int crop_y, int crop_w, int crop_h,
                   int in_pitch, int bps, int order, rsb200h_err* e) {
  return guarded(e, [&] {
    RawImage img = makeImage(img_data, w, h, cpp, pitch, true, 1, 1);
    UncompressedDecompressor u(ByteStream(in, in_size), img,
                               iRectangle2D(crop_x, crop_y, crop_w, crop_h), in_pitch, bps,
                               static_cast<BitOrder>(order));
    u.readUncompressedRaw();
    copyOut(img, img_data);
  });
}

// The other UncompressedDecompressor members.  form: 0 readUncompressedRaw (is_f32: on
// an F32 image), 1/2 decode8BitRaw<false/true>, 3/4 decode12BitRawWithControl<big/
// little>, 5/6 decode12BitRawUnpackedLeftAligned<big/little>; curve != NULL ->
// mRaw->setTable(curve, dither) first.
int rsb200h_unpack_form(const uint8_t* in, uint32_t in_size, void* img_data, int is_f32, int w,
                        int h, int cpp, int pitch, int crop_x, int crop_y, int crop_w,
                        int crop_h, int in_pitch, int bps, int order, int form,
                        const uint16_t* curve, int ncurve, int dither, rsb200h_err* e) {
  return guarded(e, [&] {
    RawImage img = RawImage::create(iPoint2D(w, h),
                                    is_f32 ? RawImageType::F32 : RawImageType::UINT16,
                                    (uint32_t)cpp);
    if (img->pitch != pitch)
      ThrowRDE("test harness: pitch mismatch (%d vs %d)", img->pitch, pitch);
    std::memcpy(img->getByteData(), img_data, (size_t)pitch * h);
    if (curve)
      img->setTable(std::vector<uint16_t>(curve, curve + ncurve), dither != 0);
    UncompressedDecompressor u(ByteStream(in, in_size), img,
                               iRectangle2D(crop_x, crop_y, crop_w, crop_h), in_pitch, bps,
                               static_cast<BitOrder>(order));
    switch (form) {
    case 0: u.readUncompressedRaw(); break;
    case 1: u.decode8BitRaw<false>(); break;
    case 2: u.decode8BitRaw<true>(); break;
    case 3: u.decode12BitRawWithControl<Endianness::big>(); break;
    case 4: u.decode12BitRawWithControl<Endianness::little>(); break;
    case 5: u.decode12BitRawUnpackedLeftAligned<Endianness::big>(); break;
    case 6: u.decode12BitRawUnpackedLeftAligned<Endianness::little>(); break;
    default: ThrowRDE("unknown form");
    }
    std::memcpy(img_data, img->getByteData(), img->getByteSize());
  });
}

int rsb200h_ljpeg_decompress(uint16_t* img_data, int w, int h, int cpp, int pitch, int fx, int fy,
                             int fw, int fh, int mcu_x, int mcu_y, int dim_x, int dim_y,
                             const rsb200h_huff* tabs, const int* tab_of_comp,
                             const uint16_t* init_pred, int nrec, int fix16,
                             int rows_per_restart, const uint8_t* in, uint32_t in_size,
                             uint32_t* consumed, rsb200h_err* e) {
  return guarded(e, [&] {
    RawImage img = makeImage(img_data, w, h, cpp, pitch, true, 1, 1);
    std::vector<std::unique_ptr<PrefixCodeDecoder<>>> hts;
    int maxTab = 0;
    for (int i = 0; i < nrec; ++i)
      maxTab = std::max(maxTab, tab_of_comp[i]);
    for (int t = 0; t <= maxTab; ++t)
      hts.emplace_back(std::make_unique<PrefixCodeDecoder<>>(makeHT(tabs[t], fix16)));
    std::vector<LJpegDecompressor::PerComponentRecipe> rec;
    for (int i = 0; i < nrec; ++i)
      rec.push_back({*hts[(size_t)tab_of_comp[i]], init_pred[i]});
    LJpegDecompressor d(img, iRectangle2D(fx, fy, fw, fh),
                        LJpegDecompressor::Frame{iPoint2D(mcu_x, mcu_y), iPoint2D(dim_x, dim_y)},
                        rec, rows_per_restart, Buffer(in, in_size));
    const uint32_t c = d.decode();
    if (consumed)
      *consumed = c;
    copyOut(img, img_data);
  });
}

int rsb200h_ljpeg_decode(const uint8_t* in, uint32_t in_size, uint16_t* img_data, int w, int h,
                         int cpp, int pitch, uint32_t off_x, uint32_t off_y, uint32_t tw,
                         uint32_t th, int max_w, int max_h, int fix16, rsb200h_err* e) {
  return guarded(e, [&] {
    RawImage img = makeImage(img_data, w, h, cpp, pitch, true, 1, 1);
    LJpegDecoder d(ByteStream(in, in_size), img);
    d.decode(off_x, off_y, tw, th, iPoint2D(max_w, max_h), fix16 != 0);
    copyOut(img, img_data);
  });
}

static thread_local double g_last_call_ms = 0.0;

int rsb200h_dng_decompress(const uint8_t* file, uint64_t file_size, const uint64_t* tile_off,
                           const uint32_t* tile_len, int ntiles, void* img_data, int is_f32, int w,
                           int h, int cpp, int pitch, int tile_w, int tile_h, int compression,
                           int fix_ljpeg, int bps, int big_endian, rsb200h_err* e) {
  return guarded(e, [&] {
    RawImage img = RawImage::create(iPoint2D(w, h),
                                    is_f32 ? RawImageType::F32 : RawImageType::UINT16,
                                    (uint32_t)cpp);
    if (img->pitch != pitch)
      ThrowRDE("test harness: pitch mismatch (%d vs %d)", img->pitch, pitch);
    std::memcpy(img->getByteData(), img_data, (size_t)pitch * h);
    const iPoint2D dim(w, h);
    DngTilingDescription dsc(dim, (uint32_t)tile_w, (uint32_t)tile_h);
    AbstractDngDecompressor d(img, dsc, compression, fix_ljpeg != 0, (uint32_t)bps, 1);
    const Buffer whole(file, (Buffer::size_type)file_size);
    d.slices.reserve((size_t)ntiles);
    for (int n = 0; n < ntiles; ++n)
      d.slices.emplace_back(d.dsc, (unsigned)n,
                            ByteStream(whole.getSubView((Buffer::size_type)tile_off[n], tile_len[n]),
                                       big_endian ? Endianness::big : Endianness::little));
    // (the member call alone is timed: allocating the RawImage and copying the caller's numpy
    //  array in and out of it belong to this test harness, not to the decompressor)
    const auto t0 = std::chrono::steady_clock::now();
    try {
      d.decompress();
    } catch (...) {
      std::memcpy(img_data, img->getByteData(), img->getByteSize());
      throw;
    }
    g_last_call_ms =
        std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    std::memcpy(img_data, img->getByteData(), img->getByteSize());
  });
}

// wall time of the decompressor's member call inside the last rsb200h_dng_decompress() of this thread
double rsb200h_last_call_ms(void) { return g_last_call_ms; }

// The host half of AbstractDngDecompressor::decompress() for LJPEG tiles, alone
// (AbstractDngDecompressor::prepareLJpeg: per tile LJpegDecoder::prepare() -- marker walk, SOF3 /
// DHT / SOS validation, restart-marker scan -- then scan descriptors and table de-duplication):
// everything that happens before rsb200_ljpeg_plan_create.  No GPU involved: a measurement and
// test hook (best wall ms of `reps`; a digest of the descriptors so that thread counts can be
// compared); the image is only a shape here.
int rsb200h_dng_ljpeg_host_half(const uint8_t* file, uint64_t file_size, const uint64_t* tile_off,
                                const uint32_t* tile_len, int ntiles, int w, int h, int cpp,
                                int tile_w, int tile_h, int fix_ljpeg, int threads, int reps,
                                double* best_ms, uint32_t* nscans, uint32_t* ntables,
                                uint32_t* nerrors, uint64_t* digest, rsb200_ljpeg_scan* scans_out,
                                uint32_t scans_cap, char* first_error, int first_error_cap,
                                rsb200h_err* e) {
  return guarded(e, [&] {
    const iPoint2D dim(w, h); // (DngTilingDescription keeps a reference to it)
    RawImage img = RawImage::create(dim, RawImageType::UINT16, (uint32_t)cpp);
    DngTilingDescription dsc(dim, (uint32_t)tile_w, (uint32_t)tile_h);
    AbstractDngDecompressor d(img, dsc, 7, fix_ljpeg != 0, 16, 1);
    const Buffer whole(file, (Buffer::size_type)file_size);
    d.slices.reserve((size_t)ntiles);
    for (int n = 0; n < ntiles; ++n)
      d.slices.emplace_back(d.dsc, (unsigned)n,
                            ByteStream(whole.getSubView((Buffer::size_type)tile_off[n], tile_len[n]),
                                       Endianness::little));
    *best_ms = 1e30;
    for (int r = 0; r < std::max(1, reps); ++r) {
      const auto t0 = std::chrono::steady_clock::now();
      const AbstractDngDecompressor::PreparedLJpeg pl = d.prepareLJpeg((unsigned)threads);
      const double ms =
          std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
      *best_ms = std::min(*best_ms, ms);
      *nscans = (uint32_t)pl.scans.size();
      *ntables = (uint32_t)pl.tables.size();
      *nerrors = (uint32_t)pl.errors.size();
      // FNV-1a over the descriptors, the tables and the error texts, in order
      uint64_t hsh = 1469598103934665603ull;
      auto mix = [&](const void* p, size_t nb) {
        const uint8_t* b = static_cast<const uint8_t*>(p);
        for (size_t i = 0; i < nb; ++i)
          hsh = (hsh ^ b[i]) * 1099511628211ull;
      };
      if (!pl.scans.empty())
        mix(pl.scans.data(), sizeof(rsb200_ljpeg_scan) * pl.scans.size());
      if (!pl.tables.empty())
        mix(pl.tables.data(), sizeof(rsb200_huff_table) * pl.tables.size());
      for (const std::string& er : pl.errors)
        mix(er.data(), er.size());
      for (const auto& t : pl.tiles)
        mix(&t.firstScan, sizeof t.firstScan);
      *digest = hsh;
      if (first_error && first_error_cap > 0) {
        first_error[0] = 0;
        if (!pl.errors.empty()) { // "IOE: ..." / "RDE: ..."
          const std::string tagged = std::string(pl.errorIsIOE[0] ? "IOE: " : "RDE: ") + pl.errors[0];
          std::strncpy(first_error, tagged.c_str(), (size_t)first_error_cap - 1);
          first_error[first_error_cap - 1] = 0;
        }
      }
      // the descriptors themselves (offsets relative to `file`), for comparison in tests
      for (size_t i = 0; scans_out && i < pl.scans.size() && i < scans_cap; ++i) {
        scans_out[i] = pl.scans[i];
        scans_out[i].in_offset += (uint64_t)(pl.base - file);
      }
    }
  });
}

int rsb200h_cr2_decompress(uint16_t* img_data, int w, int h, int pitch, int is_cfa, int n_comp,
                           int x_s_f, int y_s_f, int frame_w, int frame_h, int num_slices,
                           int slice_w, int last_slice_w, const rsb200h_huff* tabs,
                           const int* tab_of_comp, const uint16_t* init_pred, int nrec,
                           const uint8_t* in, uint32_t in_size, uint32_t* consumed,
                           rsb200h_err* e) {
  return guarded(e, [&] {
    RawImage img = makeImage(img_data, w, h, 1, pitch, is_cfa != 0, 1, 1);
    std::vector<std::unique_ptr<PrefixCodeDecoder<>>> hts;
    int maxTab = 0;
    for (int i = 0; i < nrec; ++i)
      maxTab = std::max(maxTab, tab_of_comp[i]);
    for (int t = 0; t <= maxTab; ++t)
      hts.emplace_back(std::make_unique<PrefixCodeDecoder<>>(makeHT(tabs[t], false)));
    std::vector<Cr2Decompressor<>::PerComponentRecipe> rec;
    for (int i = 0; i < nrec; ++i)
      rec.push_back({*hts[(size_t)tab_of_comp[i]], init_pred[i]});
    Cr2Decompressor<> d(img, std::make_tuple(n_comp, x_s_f, y_s_f), iPoint2D(frame_w, frame_h),
                        Cr2SliceWidths((uint16_t)num_slices, (uint16_t)slice_w,
                                       (uint16_t)last_slice_w),
                        rec, Buffer(in, in_size));
    const uint32_t c = d.decompress();
    if (consumed)
      *consumed = c;
    copyOut(img, img_data);
  });
}

int rsb200h_cr2_ljpeg_decode(const uint8_t* in, uint32_t in_size, uint16_t* img_data, int w, int h,
                             int pitch, int is_cfa, int sub_x, int sub_y, int num_slices,
                             int slice_w, int last_slice_w, rsb200h_err* e) {
  return guarded(e, [&] {
    RawImage img = makeImage(img_data, w, h, 1, pitch, is_cfa != 0, sub_x, sub_y);
    Cr2LJpegDecoder d(ByteStream(in, in_size), img);
    if (num_slices == 0 && slice_w == 0 && last_slice_w == 0)
      d.decode(Cr2SliceWidths());
    else
      d.decode(Cr2SliceWidths((uint16_t)num_slices, (uint16_t)slice_w, (uint16_t)last_slice_w));
    copyOut(img, img_data);
  });
}

// HasselbladLJpegDecoder(bs, img).decode(): the LJPEG container walk on the host, the pair stream on
// the device
int rsb200h_hasselblad_ljpeg_decode(const uint8_t* in, uint32_t in_size, uint16_t* img_data, int w, int h,
                                    int pitch, rsb200h_err* e) {
  return guarded(e, [&] {
    RawImage img = makeImage(img_data, w, h, 1, pitch, true, 1, 1);
    HasselbladLJpegDecoder d(ByteStream(in, in_size), img);
    d.decode();
    copyOut(img, img_data);
  });
}

int rsb200h_pentax_decompress(uint16_t* img_data, int w, int h, int pitch, const uint8_t* meta,
                              int meta_size, int meta_be, const uint8_t* data, uint32_t size,
                              rsb200h_err* e) {
  return guarded(e, [&] {
    RawImage img = makeImage(img_data, w, h, 1, pitch, true, 1, 1);
    ByteStream md(meta, meta ? (Buffer::size_type)meta_size : 0,
                  meta_be ? Endianness::big : Endianness::little);
    PentaxDecompressor p(img, meta ? &md : nullptr);
    try {
      p.decompress(ByteStream(data, size));
    } catch (...) {
      copyOut(img, img_data);
      throw;
    }
    copyOut(img, img_data);
  });
}

int rsb200h_samsung_v0(uint16_t* img_data, int w, int h, int pitch, const uint8_t* bso, uint32_t bso_size,
                       const uint8_t* bsr, uint32_t bsr_size, rsb200h_err* e) {
  return guarded(e, [&] {
    RawImage img = makeImage(img_data, w, h, 1, pitch, true, 1, 1);
    SamsungV0Decompressor d(img, ByteStream(bso, bso_size), ByteStream(bsr, bsr_size));
    try {
      d.decompress();
    } catch (...) {
      copyOut(img, img_data);
      throw;
    }
    copyOut(img, img_data);
  });
}

// cpp: components per pixel of the image (the constructor refuses anything but 1)
int rsb200h_samsung_v1(uint16_t* img_data, int w, int h, int cpp, int pitch, const uint8_t* data,
                       uint32_t size, int bit, rsb200h_err* e) {
  return guarded(e, [&] {
    RawImage img = makeImage(img_data, w, h, cpp, pitch, true, 1, 1);
    SamsungV1Decompressor d(img, ByteStream(data, size), bit);
    try {
      d.decompress();
    } catch (...) {
      copyOut(img, img_data);
      throw;
    }
    copyOut(img, img_data);
  });
}

// cpp: components per pixel of the image (the constructor refuses anything but 1)
int rsb200h_samsung_v2(uint16_t* img_data, int w, int h, int cpp, int pitch, const uint8_t* data,
                       uint32_t size, unsigned bits, rsb200h_err* e) {
  return guarded(e, [&] {
    RawImage img = makeImage(img_data, w, h, cpp, pitch, true, 1, 1);
    SamsungV2Decompressor d(img, ByteStream(data, size), bits);
    try {
      d.decompress();
    } catch (...) {
      copyOut(img, img_data);
      throw;
    }
    copyOut(img, img_data);
  });
}

// cpp: components per pixel of the image (the constructor refuses anything but 1); curve != NULL ->
// mRaw->setTable(curve, dither) first
int rsb200h_kodak(uint16_t* img_data, int w, int h, int cpp, int pitch, const uint8_t* data, uint32_t size, int bps,
                  int uncorrected, const uint16_t* curve, int ncurve, int dither, rsb200h_err* e) {
  return guarded(e, [&] {
    RawImage img = makeImage(img_data, w, h, cpp, pitch, true, 1, 1);
    if (curve)
      img->setTable(std::vector<uint16_t>(curve, curve + ncurve), dither != 0);
    KodakDecompressor d(img, ByteStream(data, size), bps, uncorrected != 0);
    try {
      d.decompress();
    } catch (...) {
      copyOut(img, img_data);
      throw;
    }
    copyOut(img, img_data);
  });
}

// VC5Decompressor(bs, img, phase, codes).decode(0, 0, w, h) on an image with white level `white`;
// codes: ncodes entries of {size, bits, count, value}
int rsb200h_vc5(uint16_t* img_data, int w, int h, int pitch, const uint8_t* data, uint32_t size, int white, int phase,
                const rsb200_vc5_code* codes, int ncodes, rsb200h_err* e) {
  return guarded(e, [&] {
    RawImage img = makeImage(img_data, w, h, 1, pitch, true, 1, 1);
    img->whitePoint = white;
    try {
      VC5Decompressor d(ByteStream(data, size), img, phase, codes, ncodes);
      d.decode(0, 0, (unsigned)w, (unsigned)h);
    } catch (...) {
      copyOut(img, img_data);
      throw;
    }
    copyOut(img, img_data);
  });
}

int rsb200h_sony_arw1_decompress(uint16_t* img_data, int w, int h, int pitch, const uint8_t* data,
                                 uint32_t size, rsb200h_err* e) {
  return guarded(e, [&] {
    RawImage img = makeImage(img_data, w, h, 1, pitch, true, 1, 1);
    SonyArw1Decompressor d(img);
    try {
      d.decompress(ByteStream(data, size));
    } catch (...) {
      copyOut(img, img_data);
      throw;
    }
    copyOut(img, img_data);
  });
}

int rsb200h_nikon_decompress(uint16_t* img_data, int w, int h, int pitch, const uint8_t* meta,
                             uint32_t meta_size, int meta_be, int bitsPS, const uint8_t* data,
                             uint32_t size, int uncorrected, rsb200h_err* e) {
  return guarded(e, [&] {
    RawImage img = makeImage(img_data, w, h, 1, pitch, true, 1, 1);
    NikonDecompressor n(img, ByteStream(meta, meta_size, meta_be ? Endianness::big : Endianness::little),
                        (uint32_t)bitsPS);
    try {
      n.decompress(Buffer(data, size), uncorrected != 0);
    } catch (...) {
      copyOut(img, img_data);
      throw;
    }
    copyOut(img, img_data);
  });
}

int rsb200h_panasonic(int version, uint16_t* img_data, int w, int h, int pitch,
                      const uint8_t* data, uint32_t size, int bps, rsb200h_err* e) {
  return guarded(e, [&] {
    RawImage img = makeImage(img_data, w, h, 1, pitch, true, 1, 1);
    const ByteStream in(data, size);
    if (version == 5) {
      PanasonicV5Decompressor d(img, in, (uint32_t)bps);
      d.decompress();
    } else if (version == 6) {
      PanasonicV6Decompressor d(img, in, (uint32_t)bps);
      d.decompress();
    } else if (version == 7) {
      PanasonicV7Decompressor d(img, in);
      d.decompress();
    } else {
      ThrowRDE("unknown Panasonic version");
    }
    copyOut(img, img_data);
  });
}

// PanasonicV4Decompressor(img, data, zero_is_not_bad, split).decompress(); the bad-pixel
// positions it appended to mRaw->mBadPixelPositions come back in zero_pos (at most cap) / nzero.
// construct_only != 0: the constructor's checks alone (no GPU needed).
int rsb200h_panasonic_v4(uint16_t* img_data, int w, int h, int pitch, const uint8_t* data,
                         uint32_t size, int zero_is_not_bad, uint32_t split, uint32_t* zero_pos,
                         uint32_t cap, uint32_t* nzero, int construct_only, rsb200h_err* e) {
  return guarded(e, [&] {
    RawImage img = makeImage(img_data, w, h, 1, pitch, true, 1, 1);
    PanasonicV4Decompressor d(img, ByteStream(data, size), zero_is_not_bad != 0, split);
    if (construct_only)
      return;
    d.decompress();
    copyOut(img, img_data);
    const auto& z = img->mBadPixelPositions;
    *nzero = (uint32_t)z.size();
    for (size_t i = 0; i < z.size() && i < cap; ++i)
      zero_pos[i] = z[i];
  });
}

// mRaw->setTable(curve, dither); mRaw->sixteenBitLookup()
int rsb200h_sixteen_bit_lookup(uint16_t* img_data, int w, int h, int cpp, int pitch,
                               const uint16_t* curve, int ncurve, int dither, rsb200h_err* e) {
  return guarded(e, [&] {
    RawImage img = makeImage(img_data, w, h, cpp, pitch, true, 1, 1);
    if (curve)
      img->setTable(std::vector<uint16_t>(curve, curve + ncurve), dither != 0);
    img->sixteenBitLookup();
    copyOut(img, img_data);
  });
}

// RawImageData::fixBadPixels() with mBadPixelPositions = positions[0..n); map_only != 0: stop
// after transferBadPixelsToMap() and return the bitmap (no GPU needed): map_out must hold
// roundUp(ceil(w / 8), 16) * h bytes.
int rsb200h_fix_bad_pixels(uint16_t* img_data, int w, int h, int cpp, int pitch, int is_cfa,
                           const uint32_t* positions, uint32_t n, int map_only, uint8_t* map_out,
                           rsb200h_err* e) {
  return guarded(e, [&] {
    RawImage img = makeImage(img_data, w, h, cpp, pitch, is_cfa != 0, 1, 1);
    img->mBadPixelPositions.assign(positions, positions + n);
    if (map_only) {
      img->transferBadPixelsToMap();
      if (map_out && !img->mBadPixelMap.empty())
        std::memcpy(map_out, img->mBadPixelMap.data(), img->mBadPixelMap.size());
      return;
    }
    img->fixBadPixels();
    copyOut(img, img_data);
  });
}

namespace {
RawImage makeAnyImage(const void* src, int is_f32, int w, int h, int cpp, int pitch, const int* crop) {
  RawImage img = RawImage::create(iPoint2D(w, h), is_f32 ? RawImageType::F32 : RawImageType::UINT16,
                                  (uint32_t)cpp);
  if (img->pitch != pitch)
    ThrowRDE("test harness: pitch mismatch (%d vs %d)", img->pitch, pitch);
  std::memcpy(img->getByteData(), src, (size_t)pitch * h);
  if (crop[0] || crop[1] || crop[2] != w || crop[3] != h)
    img->subFrame(iRectangle2D(crop[0], crop[1], crop[2], crop[3]));
  return img;
}
} // namespace

// DngOpcodes(ri, data) + applyOpCodes(ri) on a uint16 / float image with the crop crop[4] =
// (mOffset.x, mOffset.y, dim.x, dim.y); reports crop and mBadPixelPositions afterwards (also
// when applyOpCodes throws: the opcodes before the failing one stay applied).  stage: which
// half threw (1 constructor, 2 applyOpCodes), 0 if none.
int rsb200h_dng_opcodes(void* img_data, int is_f32, int w, int h, int cpp, int pitch, int* crop,
                        const uint8_t* data, uint32_t size, uint32_t* bad, uint32_t bad_cap,
                        uint32_t* nbad, int* stage, rsb200h_err* e) {
  *stage = 0;
  return guarded(e, [&] {
    RawImage img = makeAnyImage(img_data, is_f32, w, h, cpp, pitch, crop);
    auto copyBack = [&] {
      std::memcpy(img_data, img->getByteData(), img->getByteSize());
      const iPoint2D o = img->getCropOffset();
      crop[0] = o.x;
      crop[1] = o.y;
      crop[2] = img->dim.x;
      crop[3] = img->dim.y;
      *nbad = (uint32_t)img->mBadPixelPositions.size();
      for (uint32_t i = 0; i < *nbad && i < bad_cap; ++i)
        bad[i] = img->mBadPixelPositions[i];
    };
    *stage = 1;
    DngOpcodes codes(img, ByteStream(data, size));
    *stage = 2;
    try {
      codes.applyOpCodes(img);
    } catch (...) {
      copyBack();
      throw;
    }
    *stage = 0;
    copyBack();
  });
}

// The list in device form (DngOpcodes::lower) without running anything: what applyOpCodes would
// upload.  Buffers are caller-allocated (capacities in elements); counts come back in n[4] =
// {ops, tables, deltas, actions}; actions as pairs (kind: 0 list / 1 constant / 2 trim, index),
// followed for a list action by nothing -- the lists themselves are read with list_of.
// has_error: the first failing opcode's setup()/apply() error is in *e (class code returned).
int rsb200h_dngop_lower(const void* img_data, int is_f32, int w, int h, int cpp, int pitch,
                        const int* crop, const uint8_t* data, uint32_t size, rsb200_dng_op* ops,
                        uint32_t ops_cap, uint16_t* tables, uint32_t tables_cap, uint32_t* deltas,
                        uint32_t deltas_cap, uint32_t* actions, uint32_t actions_cap, uint32_t* n,
                        uint32_t* lists, uint32_t lists_cap, uint32_t* rois, rsb200h_err* e) {
  return guarded(e, [&] {
    RawImage img = makeAnyImage(img_data, is_f32, w, h, cpp, pitch, crop);
    DngOpcodes codes(img, ByteStream(data, size));
    const DngOpcodes::Lowered L = codes.lower(img);
    n[0] = (uint32_t)L.ops.size();
    n[1] = (uint32_t)(L.tables.size() / 65536);
    n[2] = (uint32_t)L.deltas.size();
    n[3] = (uint32_t)L.actions.size();
    if (n[0] > ops_cap || n[1] > tables_cap || n[2] > deltas_cap || n[3] > actions_cap)
      ThrowRDE("test harness: buffers too small");
    std::copy(L.ops.begin(), L.ops.end(), ops);
    std::copy(L.tables.begin(), L.tables.end(), tables);
    std::copy(L.deltas.begin(), L.deltas.end(), deltas);
    // per action: kind, index, then (list: count + offset into `lists`) / (trim: roi x, y, w, h in rois)
    uint32_t lpos = 0;
    for (size_t i = 0; i < L.actions.size(); ++i) {
      const auto& a = L.actions[i];
      actions[4 * i] = (uint32_t)a.kind;
      actions[4 * i + 1] = a.index;
      actions[4 * i + 2] = actions[4 * i + 3] = 0;
      if (a.kind == DngOpcodes::Action::BadList) {
        const auto& b = codes.badPixels(a.index);
        if (lpos + b.size() > lists_cap)
          ThrowRDE("test harness: buffers too small");
        actions[4 * i + 2] = (uint32_t)b.size();
        actions[4 * i + 3] = lpos;
        std::copy(b.begin(), b.end(), lists + lpos);
        lpos += (uint32_t)b.size();
      } else if (a.kind == DngOpcodes::Action::Trim) {
        const iRectangle2D r = codes.roi(a.index);
        rois[4 * i] = (uint32_t)r.pos.x;
        rois[4 * i + 1] = (uint32_t)r.pos.y;
        rois[4 * i + 2] = (uint32_t)r.dim.x;
        rois[4 * i + 3] = (uint32_t)r.dim.y;
      }
    }
    if (L.error)
      std::rethrow_exception(L.error);
  });
}

int rsb200h_phaseone(uint16_t* img_data, int w, int h, int pitch, const uint8_t* file,
                     uint64_t file_size, const uint64_t* off, const uint32_t* len,
                     const int32_t* rown, int nstrips, rsb200h_err* e) {
  return guarded(e, [&] {
    RawImage img = makeImage(img_data, w, h, 1, pitch, true, 1, 1);
    std::vector<PhaseOneStrip> strips;
    for (int k = 0; k < nstrips; ++k) {
      if (off[k] + len[k] > file_size)
        ThrowIOE("Out of bounds access in ByteStream");
      strips.emplace_back(rown[k], ByteStream(file + off[k], len[k]));
    }
    PhaseOneDecompressor d(img, std::move(strips));
    try {
      d.decompress();
    } catch (...) {
      copyOut(img, img_data);
      throw;
    }
    copyOut(img, img_data);
  });
}

int rsb200h_sony_arw2(uint16_t* img_data, int w, int h, int pitch, const uint8_t* data,
                      uint32_t size, const uint16_t* curve, int ncurve, int dither,
                      rsb200h_err* e) {
  return guarded(e, [&] {
    RawImage img = makeImage(img_data, w, h, 1, pitch, true, 1, 1);
    if (curve)
      img->setTable(std::vector<uint16_t>(curve, curve + ncurve), dither != 0);
    SonyArw2Decompressor a(img, ByteStream(data, size));
    a.decompress();
    copyOut(img, img_data);
  });
}

// RawImageData::scaleBlackWhite(): blackLevel, optional blackLevelSeparate / whitePoint,
// blackAreas as triples (is_vertical, offset, size); reports what it settled on.
// stage: 0 = everything (device pass included), 1 = host part only (estimate + black areas;
// needs no GPU).
int rsb200h_scale_black_white(uint16_t* img_data, int w, int h, int cpp, int pitch, int is_cfa,
                              int off_x, int off_y, int crop_w, int crop_h, int black_level,
                              int* black_sep, int has_sep, int* white, int has_white,
                              const int* areas, int n_areas, int dither, int path, int stage,
                              int* sep_set, rsb200h_err* e) {
  return guarded(e, [&] {
    RawImage img = makeImage(img_data, w, h, cpp, pitch, is_cfa != 0, 1, 1);
    img->subFrame(iRectangle2D(off_x, off_y, crop_w, crop_h));
    img->blackLevel = black_level;
    if (has_sep) {
      img->blackLevelSeparate = Array2DRef<int>(img->blackLevelSeparateStorage.data(), 2, 2);
      for (int i = 0; i < 4; ++i)
        img->blackLevelSeparateStorage[i] = black_sep[i];
    }
    if (has_white)
      img->whitePoint = *white;
    for (int i = 0; i < n_areas; ++i)
      img->blackAreas.emplace_back(areas[3 * i + 1], areas[3 * i + 2], areas[3 * i] != 0);
    img->mDitherScale = dither != 0;
    if (stage == 0)
      img->scaleBlackWhite(path);
    else
      img->prepareScaleBlackWhite();
    copyOut(img, img_data);
    *sep_set = img->blackLevelSeparate.has_value();
    if (img->blackLevelSeparate)
      for (int i = 0; i < 4; ++i)
        black_sep[i] = img->blackLevelSeparateStorage[i];
    *white = img->whitePoint.has_value() ? *img->whitePoint : -1;
  });
}

int rsb200h_sraw_interpolate(const uint16_t* in, int in_w, int in_h, int in_pitch,
                             uint16_t* out_data, int out_w, int out_h, int out_pitch, int sub_x,
                             int sub_y, const int* coeffs, int hue, int version,
                             rsb200h_err* e) {
  return guarded(e, [&] {
    RawImage img = makeImage(out_data, out_w, out_h, 3, out_pitch, false, sub_x, sub_y);
    Cr2sRawInterpolator i(img, Array2DRef<const uint16_t>(in, in_w, in_h, in_pitch / 2),
                          {coeffs[0], coeffs[1], coeffs[2]}, hue);
    i.interpolate(version);
    copyOut(img, out_data);
  });
}

int rsb200h_huff_check(const uint8_t* ncpl, const uint8_t* values, int nvalues, int full,
                       int fix16, rsb200h_err* e) {
  return guarded(e, [&] {
    HuffmanCode<> hc;
    hc.setNCodesPerLength(Buffer(ncpl, 16));
    hc.setCodeValues(values, nvalues);
    PrefixCodeDecoder<> ht(std::move(hc));
    ht.setup(full != 0, fix16 != 0);
  });
}

} // extern "C"
