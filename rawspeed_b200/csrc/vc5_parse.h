// vc5_parse.h -- the host half of GoPro VC-5: VC5Decompressor's constructor checks and its tag walk
// (decompressors/VC5Decompressor.cpp:382-432, :490-618, :744-816), which cut a datablock into the 40
// band payloads a plan of rsb200_vc5_plan_create takes, and the texts of the plan's band outcomes.
// Used by the host mirror (csrc/host) and the drop-in (csrc/dropin), which throw the failures with
// their own exception classes.
#pragma once
#include "../../include/rawspeed_b200.h"

#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>

namespace rsb200_vc5 {

enum : int { OK = 0, RDE = 1, IOE = 2 };

struct Outcome {
  int cls = OK;     // OK, RDE or IOE
  std::string msg;  // the reference's text, without its "function, line" prefix
};

struct Parsed {
  rsb200_vc5_job job;          // first_band 0, out_offset 0, out_pitch left to the caller
  rsb200_vc5_band bands[40];   // channel * 10 + subband; in_offset relative to the datablock
};

inline Outcome fail(int cls, const char* fmt, ...) __attribute__((format(printf, 2, 3)));
inline Outcome fail(int cls, const char* fmt, ...) {
  char buf[256];
  va_list ap;
  va_start(ap, fmt);
  std::vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  return Outcome{cls, buf};
}

// The constructor's checks after the component count / data type (the caller's, with its image) and
// the tag walk.  phase: the image's BayerPhase 0..3 (RGGB, GRBG, GBRG, BGGR), or -1 for a CFA that is
// not a 2x2 Bayer pattern.  white: the image's white level.
inline Outcome parse(const uint8_t* d, uint32_t size, int w, int h, int white, int phase, Parsed& out) {
  std::memset(&out, 0, sizeof out);
  if (w <= 0 || h <= 0)
    return fail(RDE, "Bad image dimensions.");
  if (w % 2 != 0)
    return fail(RDE, "Width %i is not a multiple of %i", w, 2);
  if (h % 2 != 0)
    return fail(RDE, "Height %i is not a multiple of %i", h, 2);
  if (phase < 0)
    return fail(RDE, "Image has invalid CFA.");
  if (phase != RSB200_VC5_RGGB && phase != RSB200_VC5_GBRG)
    return fail(RDE, "Unexpected bayer phase, please file a bug.");
  if (white <= 0 || white > 65535)
    return fail(RDE, "Bad white level %i", white);
  int bits = 0;
  for (int wp = white; wp != 0; wp >>= 1)
    ++bits;
  out.job.width = w, out.job.height = h, out.job.output_bits = bits, out.job.phase = phase;
  int bw3 = w, bh3 = h;
  for (int k = 0; k < 4; ++k)
    bw3 = (bw3 + 1) / 2, bh3 = (bh3 + 1) / 2;
  // ByteStream reads past the end: Buffer::getSubView
  const Outcome trunc = fail(IOE, "Buffer overflow: image file may be truncated");
  uint32_t pos = 0;
  auto get16 = [&](int& v) {
    if (size - pos < 2)
      return false;
    v = d[pos] << 8 | d[pos + 1];
    pos += 2;
    return true;
  };
  if (size < 4)
    return trunc;
  if (!(d[0] == 0x56 && d[1] == 0x43 && d[2] == 0x2d && d[3] == 0x35))
    return fail(RDE, "not a valid VC-5 datablock");
  pos = 4;
  int chan = 0, subband = -1, prec = -1, quant = 0;
  bool hasQuant = false;
  int valid[4][4] = {{0}};  // [channel][wavelet 0..3]: bands seen
  for (;;) {
    int t, val;
    if (!get16(t) || !get16(val))
      return trunc;
    int16_t tag = (int16_t)t;
    const bool optional = (tag & (int16_t)0x8000) != 0;
    if (optional)
      tag = (int16_t)-tag;
    const unsigned u = (unsigned)val;
    switch (tag) {
    case 0x000c:
      if (val != 4)
        return fail(RDE, "Bad channel count %u, expected %i", u, 4);
      break;
    case 0x0014:
      if (val != w)
        return fail(RDE, "Image width mismatch: %u vs %i", u, w);
      break;
    case 0x0015:
      if (val != h)
        return fail(RDE, "Image height mismatch: %u vs %i", u, h);
      break;
    case 0x0023:
      if (val < 8 || val > 16)
        return fail(RDE, "Invalid precision %i", val);
      prec = val;
      break;
    case 0x003e:
      if (val >= 4)
        return fail(RDE, "Bad channel number (%u)", u);
      chan = val;
      break;
    case 0x0054:
      if (val != 4)
        return fail(RDE, "Image format %i is not 4(RAW)", val);
      break;
    case 0x000e:
      if (val != 10)
        return fail(RDE, "Unexpected subband count %u, expected %i", u, 10);
      break;
    case 0x0066:
      if (val != 12)
        return fail(RDE, "Bad bits per componend %u, not %i", u, 12);
      break;
    case 0x006a:
      if (val != 2)
        return fail(RDE, "Bad pattern width %u, not %u", u, 2u);
      break;
    case 0x006b:
      if (val != 2)
        return fail(RDE, "Bad pattern height %u, not %u", u, 2u);
      break;
    case 0x0030:
      if (val >= 10)
        return fail(RDE, "Bad subband number %u", u);
      subband = val;
      break;
    case 0x0035:
      quant = (int16_t)val;
      hasQuant = true;
      break;
    case 0x006c:
      if (val != 1)
        return fail(RDE, "Bad component per sample count %u, not %u", u, 1u);
      break;
    case 0x006d:
      // applies to the CURRENT channel, as in the reference (the FIXME at VC5Decompressor.cpp:568).  A
      // wavelet whose prescale is never set is left indeterminate by the reference; here it is 0.
      for (int k = 0; k < 3; ++k)
        out.job.prescale[chan][k] = (uint8_t)((val >> (14 - 2 * k)) & 3);
      break;
    default: {
      uint64_t chunk = 0;
      if (tag & 0x2000)
        chunk = (uint64_t)(tag & 0xff) << 16 | (uint64_t)val;
      else if (tag & 0x4000)
        chunk = (uint64_t)val;
      if ((tag & 0x6000) == 0x6000) {  // LargeCodeblock: parseLargeCodeblock(getStream(chunk, 4))
        if ((uint64_t)(size - pos) < 4 * chunk)
          return trunc;
        const uint32_t off = pos, len = (uint32_t)(4 * chunk);
        pos += len;
        if (subband < 0)
          return fail(RDE, "Did not see VC5Tag::SubbandNumber yet");
        const int wl = subband == 0 ? 3 : 3 - (subband - 1) / 3;  // wavelet 1..3
        const int bi = subband == 0 ? 0 : 1 + (subband - 1) % 3;
        if (valid[chan][wl] & (1 << bi))
          return fail(RDE, "Band %i for wavelet %i on channel %u was already seen", bi, wl - 1, (unsigned)chan);
        rsb200_vc5_band& b = out.bands[chan * 10 + subband];
        b.in_offset = off;
        if (subband == 0) {
          if (prec < 0)
            return fail(RDE, "Did not see VC5Tag::LowpassPrecision yet");
          const uint64_t bytes = 8 * (((uint64_t)bw3 * (uint64_t)bh3 * (uint64_t)prec + 63) / 64);
          if (bytes > len)
            return trunc;
          b.in_size = (uint32_t)bytes, b.param = prec;
          prec = -1;
        } else {
          if (!hasQuant)
            return fail(RDE, "Did not see VC5Tag::Quantization yet");
          b.in_size = len, b.param = quant;
          hasQuant = false;
        }
        valid[chan][wl] |= 1 << bi;
        if (valid[chan][wl] == 15)
          valid[chan][wl - 1] |= 1;
        subband = -1;
        break;
      }
      bool opt = optional;
      if (tag & 0x2000)
        opt = true, chunk = 0;
      if (!opt)
        return fail(RDE, "Unknown (unhandled) non-optional Tag 0x%04hx", (unsigned short)tag);
      if (chunk) {  // skipBytes(chunk, 4): ByteStream::check
        if ((uint64_t)(size - pos) < 4 * chunk)
          return fail(IOE, "Out of bounds access in ByteStream");
        pos += (uint32_t)(4 * chunk);
      }
    }
    }
    if (valid[0][0] & valid[1][0] & valid[2][0] & valid[3][0] & 1)
      return Outcome{};
  }
}

// The band failure a plan reports for a job (its `consumed`), as VC5Decompressor::decode throws it.
inline Outcome band_failure(uint32_t consumed) {
  static const char* const text[7] = {"device error",
                                      "Impossible RLV value given current quantum",
                                      "Got EndOfBand marker while looking for next pixel",
                                      "Not all pixels consumed?",
                                      "EndOfBand marker not found",
                                      "Bit stream size is smaller than MaxProcessBytes",
                                      "Buffer overflow read in BitStreamer"};
  const uint32_t code = consumed >> 28;
  return Outcome{code == RSB200_VC5_SHORT || code == RSB200_VC5_OVERREAD ? IOE : RDE, text[code <= 6 ? code : 0]};
}

}  // namespace rsb200_vc5
