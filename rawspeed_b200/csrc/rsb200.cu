// rsb200.cu -- C ABI of the H100-native RAW decompression engine
// (include/rawspeed_b200.h).  Host-side plan construction + kernel launches.
// No CPU fallback lives here: every entry point needs a CUDA device.

#include "../../include/rawspeed_b200.h"

#include "ljpeg.cuh"
#include "ljpeg_fused.cuh"
#include "ljpeg_ranges.cuh"
#include "ljpeg_thread.cuh"
#include "ljpeg_stream.cuh"
#include "ljpeg_par.cuh"
#include "hasselblad.cuh"
#include "ljpeg_tile.cuh"
#include "ljpeg_host.h"
#include "rawforms.cuh"
#include "lookup.cuh"
#include "lookup_host.h"
#include "scale.cuh"
#include "scale_host.h"
#include "sraw.cuh"
#include "arw2.cuh"
#include "badpix.cuh"
#include "badpix_host.h"
#include "dngop.cuh"
#include "dngop_host.h"
#include "pana.cuh"
#include "phaseone.cuh"
#include "pentax.cuh"
#include "nikon.cuh"
#include "unpack.cuh"

#include <algorithm>
#include <cstdarg>
#include <cstdlib>
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <new>
#include <string>
#include <chrono>
#include <thread>
#include <vector>

using namespace rsb200;

// ---- allocation: plans are created and destroyed per frame by the drop-in callers (one
// AbstractDngDecompressor::decompress() = one plan), so their device memory comes from the
// device's stream-ordered pool (kept, not returned to the driver) and their small pinned result
// buffers from a process-wide cache; cudaMalloc / cudaFree (which synchronises the device) and
// cudaMallocHost (milliseconds) are off that path.  The big grow-only staging buffers of a
// context (ensure_cap / ensure_host_cap) keep using the plain calls. ----
#include <mutex>
static cudaError_t rsb_dev_alloc(void** p, size_t n) {
  cudaError_t e = cudaMallocAsync(p, n, (cudaStream_t)0);
  if (e == cudaSuccess)
    e = cudaStreamSynchronize((cudaStream_t)0);
  if (e != cudaSuccess) { // (no pool support: fall back to the plain allocator)
    cudaGetLastError();
    e = cudaMalloc(p, n);
  }
  return e;
}
template <typename T> static cudaError_t rsb_dev_alloc(T** p, size_t n) {
  return rsb_dev_alloc(reinterpret_cast<void**>(p), n);
}
static cudaError_t rsb_dev_free(void* p) {
  if (!p)
    return cudaSuccess;
  cudaError_t e = cudaFreeAsync(p, (cudaStream_t)0);
  if (e != cudaSuccess) {
    cudaGetLastError();
    e = cudaFree(p);
  }
  return e;
}
namespace {
struct HostCache {
  std::mutex m;
  std::multimap<size_t, void*> free_blocks;
  std::map<void*, size_t> live;
};
HostCache& host_cache() {
  static HostCache* c = new HostCache(); // (never destroyed: pinned blocks live as long as the process)
  return *c;
}
} // namespace
static cudaError_t rsb_host_alloc(void** p, size_t n) {
  size_t cap = 256;
  while (cap < n)
    cap <<= 1;
  HostCache& c = host_cache();
  {
    std::lock_guard<std::mutex> g(c.m);
    auto it = c.free_blocks.find(cap);
    if (it != c.free_blocks.end()) {
      *p = it->second;
      c.free_blocks.erase(it);
      c.live[*p] = cap;
      return cudaSuccess;
    }
  }
  const cudaError_t e = cudaMallocHost(p, cap);
  if (e == cudaSuccess) {
    std::lock_guard<std::mutex> g(c.m);
    c.live[*p] = cap;
  }
  return e;
}
template <typename T> static cudaError_t rsb_host_alloc(T** p, size_t n) {
  return rsb_host_alloc(reinterpret_cast<void**>(p), n);
}
static cudaError_t rsb_host_free(void* p) {
  if (!p)
    return cudaSuccess;
  HostCache& c = host_cache();
  std::lock_guard<std::mutex> g(c.m);
  auto it = c.live.find(p);
  if (it == c.live.end())
    return cudaFreeHost(p);
  c.free_blocks.emplace(it->second, p);
  c.live.erase(it);
  return cudaSuccess;
}

// ------------------------------------------------------------------
constexpr int N_PIPE = 8;
struct rsb200_ctx {
  int device = 0;
  int sm_count = 0;
  uint64_t launches = 0;
  char err[512] = {0};
  // host-API staging (grow only)
  uint8_t* d_in = nullptr;
  size_t d_in_cap = 0;
  uint8_t* d_out = nullptr;
  size_t d_out_cap = 0;
  cudaStream_t stream = nullptr;
  // H2D / kernel / D2H overlap of pipelined host-buffer runs: a group's upload, decode and download
  // are chained on one stream; a decode of ~70 tiles takes ~0.25 ms however few CTAs it has, so it
  // takes more than three groups in flight to keep the D2H engine busy
  cudaStream_t pipe[N_PIPE] = {};
  // pinned staging for callers whose buffers are pageable (a RawImage is): grow only
  uint8_t* h_in = nullptr;
  size_t h_in_cap = 0;
  uint8_t* h_out = nullptr;
  size_t h_out_cap = 0;
  std::vector<cudaEvent_t> stage_events;
};

static int set_err(rsb200_ctx* c, int code, const char* fmt, ...) {
  if (c) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(c->err, sizeof c->err, fmt, ap);
    va_end(ap);
  }
  return code;
}


// offset + extent without wrap-around: a sum that does not fit saturates, so the plan asks for
// more bytes than any caller has and rsb200_plan_run refuses it
static inline uint64_t sat_add(uint64_t a, uint64_t b) { return a + b < a ? ~0ull : a + b; }

#define CUDA_TRY(ctx, expr)                                                    \
  do {                                                                         \
    cudaError_t e_ = (expr);                                                   \
    if (e_ != cudaSuccess)                                                     \
      return set_err((ctx), RSB200_ERR_CUDA, "%s failed: %s", #expr,           \
                     cudaGetErrorString(e_));                                  \
  } while (0)

struct UnpackGroup {
  int bps_t;  // template bps (0 = generic)
  bool lsb;
  UnpackJobDev* d_jobs = nullptr;
  int njobs = 0;
  uint32_t nblocks = 0;
};

struct RawGroup {
  int format = 0;
  RawJobDev* d_jobs = nullptr;
  int njobs = 0;
  uint32_t total_items = 0;
};

struct PanaGroup {
  int version = 0, bps = 0;
  PanaJobDev* d_jobs = nullptr;
  int njobs = 0;
  uint32_t total_units = 0;
};

struct SrawGroup {
  int version = 0;
  bool is420 = false;
  SrawJobDev* d_jobs = nullptr;
  int njobs = 0;
  uint32_t total_mcus = 0;
};

struct ScaleGroup {
  int mode = 0; // 0: SSE2 loop semantics, 1: plain loop semantics
  ScaleJobDev* d_jobs = nullptr;
  int njobs = 0;
  uint32_t total_quads = 0;
  uint32_t nseg = 1; // column segments per row quad (mode 1)
};

struct UnpackFastGroup {
  int bps;
  bool lsb;
  UnpackFastJobDev* d_jobs = nullptr;
  int njobs = 0;
  uint32_t nblocks = 0;
  std::vector<UnpackFastJobDev> h_jobs; // host copy (pipelined host runs)
};

struct rsb200_plan {
  rsb200_ctx* ctx = nullptr;
  int kind = 0; // 0 unpack, 1 ljpeg/cr2, 2 fixed-layout raw forms, 3 sRaw interpolation, 4 ARW2, 5 Panasonic, 6 Phase One, 7 black/white scaling (in place), 8 DNG opcode list (in place), 9 bad-pixel interpolation (in place), 10 whole-image table lookup (in place), 11 Hasselblad
  int nunits = 0;
  uint64_t in_bytes = 0, out_bytes = 0, pixels = 0;
  int launches_per_run = 0;
  // required extents (validation of run() arguments)
  uint64_t need_in = 0, need_out = 0;
  // unpack
  std::vector<UnpackGroup> groups;
  std::vector<UnpackFastGroup> fast_groups;
  // fixed-layout raw forms
  std::vector<RawGroup> raw_groups;
  uint16_t* d_raw_tables = nullptr;
  std::vector<SrawGroup> sraw_groups;
  std::vector<PanaGroup> pana_groups;
  // Panasonic V4 bad-pixel lists: slot per job that asked for them (-1 otherwise)
  std::vector<int> pana_zero_slot;
  uint32_t* d_pana_zero_count = nullptr;
  uint32_t* d_pana_zero_list = nullptr;
  int pana_zero_slots = 0;
  std::vector<ScaleGroup> scale_groups;
  // DNG opcode pass (K10); bad-pixel lists share pana_zero_slot / d_pana_zero_* (slot per
  // BAD_CONSTANT opcode, indexed by opcode)
  DngOpJobDev* d_dngop_jobs = nullptr;
  DngOpDev* d_dngop_ops = nullptr;
  uint16_t* d_dngop_tables = nullptr;
  uint32_t* d_dngop_deltas = nullptr;
  int dngop_njobs = 0;
  uint32_t dngop_units = 0;
  // whole-image table lookup (K12)
  LookupJobDev* d_lookup_jobs = nullptr;
  uint16_t* d_lookup_tables = nullptr;
  int lookup_njobs = 0;
  uint32_t lookup_quads = 0;
  uint32_t lookup_nseg = 1; // column segments per row quad (more warps for few rows)
  bool lookup_dither = false;
  bool lookup_smem = false; // RSB200_LUT_SMEM=1 at plan creation: the shared-memory-table kernel (A/B candidate, lookup.cuh)
  int lookup_ntables = 0;
  // bad-pixel interpolation (K11)
  BadPixJobDev* d_badpix_jobs = nullptr;
  uint32_t* d_badpix_list = nullptr;
  uint8_t* d_badpix_maps = nullptr;
  int badpix_njobs = 0;
  uint32_t badpix_total = 0;
  // Phase One (shares d_arw2_bad / h_arw2_bad as the per-job error flags)
  // Hasselblad (K2H)
  DevHassJob* d_hass_jobs = nullptr;
  DevHassCta* d_hass_ctas = nullptr;
  DevHassState* d_hass_states = nullptr;
  DevHassState* h_hass_states = nullptr; // pinned
  uint32_t* d_hass_seg_job = nullptr;
  uint32_t* d_hass_u32 = nullptr;        // start | parsed | exit | count (nseg each) | cta_sum | cta_base | changed
  uint32_t* d_hass_row_begin = nullptr;
  uint32_t hass_nseg = 0, hass_ncta = 0, hass_rows = 0;
  P1StripDev* d_p1_strips = nullptr;
  P1JobDev* d_p1_jobs = nullptr;
  uint32_t* d_p1_gdesc = nullptr;   // third version: one word per group of 8 pixels (+ 1 per row)
  uint32_t* d_p1_rowflag = nullptr; // ... and per row: failed before anything was stored
  uint32_t p1_gstride = 0;          // words of gdesc per row
  int p1_ver = 3;                   // which version of the kernel this plan runs (RSB200_P1)
  int p1_walk1 = 0;                 // RSB200_P1W = 1 .. 6: other forms of the third version's walk (A/B; see p1_walk_kernel)
  uint32_t p1_nstrips = 0;
  // Sony ARW2
  Arw2JobDev* d_arw2_jobs = nullptr;
  uint16_t* d_arw2_tables = nullptr;
  uint32_t* d_arw2_bad = nullptr;
  uint32_t* h_arw2_bad = nullptr; // pinned
  uint32_t arw2_groups = 0;
  int arw2_mode = 0, arw2_ntables = 0;
  // ljpeg
  DevTable* d_tables = nullptr;
  DevScan* d_scans = nullptr;
  DevStrip* d_strips = nullptr;
  K3RowRef* d_rows = nullptr;
  uint16_t* d_diffs = nullptr;
  uint16_t* d_colvals = nullptr;
  DevResult* d_results = nullptr;
  DevResult* h_results = nullptr; // pinned
  uint32_t nrows = 0;
  int nscans = 0;
  int ntab_slots = 4;
  // small LJPEG tile segments: one fused CTA each; big segments (CR2 frames,
  // untiled strips): multi-CTA count/verify/diffs + K3
  uint32_t* d_small_ids = nullptr;
  int nsmall = 0;
  uint32_t* d_tile_ids = nullptr; // segments decoded by k2_tile_kernel<R> (ljpeg_tile.cuh)
  // host-buffer runs of a plan that holds only such segments are pipelined group by group
  // (upload / decode / download of consecutive groups overlap on three streams)
  struct TileGroup {
    uint32_t first, count;
    uint64_t in_lo, in_hi, out_lo, out_hi;
  };
  std::vector<TileGroup> tile_groups;
  DevTileParam* d_tile_params = nullptr;
  int ntile = 0;
  int tile_r = 1;
  bool clean2 = false; // thread path: k2_clean2_kernel instead of k2_clean_kernel
  int par_ctas = 0;        // k2_par_kernel: 0 = one CTA per segment; n = persistent, n CTAs per SM (RSB200_PAR_CTAS; an experiment)
  bool use_par = false;    // thread path for small launches: k2_clean_kernel + k2_par_kernel (one CTA per segment)
  bool use_stream = false; // thread path: k2_stream_kernel (unstuffing inside the thread) instead of K2C + K2T
  int stream_form = 0;     // k2_stream_kernel: 0 = by launch size, 1 = prefetch form, 2 = full-launch form (RSB200_STREAM_FORM)
  bool host_tiles_only = false; // tile_groups / d_tile_ids describe the thread path's segments for host-buffer runs only
  std::vector<uint32_t> h_in_size; // per scan: bytes of a plain LJPEG segment (kind 0), else 0xFFFFFFFF
  DevTileParam* d_thread_tile_params = nullptr; // thread path: parameters of the exact second opinion
  uint32_t* d_redo = nullptr;                   // ... and which segments need it (written by K2T)
  int nthread_redo = 0;                         // segments of the thread path the tile kernel can take
  uint32_t* d_thread_ids = nullptr; // segments decoded one per thread (K2C + K2T)
  DevTScan* d_tscans = nullptr;
  DevTInfo* d_tinfos = nullptr;
  uint32_t* d_clean = nullptr;      // unstuffed data of those segments
  uint32_t* d_anchors = nullptr;
  int nthread = 0;
  int ntables = 0;
  uint32_t* d_big_ids = nullptr;
  int nbig = 0;
  BigScanInfo* d_big = nullptr;
  DevRange* d_ranges = nullptr;
  RangeState* d_states = nullptr;
  RangeFinal* d_finals = nullptr;
  uint32_t* d_fallback = nullptr;
  int nranges = 0;
  // Pentax segments (DevScan::kind == 2): first out-of-bounds pixel per segment
  uint32_t* d_oob = nullptr;
  uint32_t* h_oob = nullptr; // pinned
  bool has_pentax = false, has_k3 = false, has_nikon = false;
  uint16_t* d_nikon_luts = nullptr;
  cudaStream_t last_stream = nullptr;
  bool ran = false;
};

extern "C" int rsb200_abi_version(void) { return RSB200_ABI_VERSION; }

extern "C" int rsb200_create(int device, rsb200_ctx** out) {
  if (!out)
    return RSB200_ERR_ARG;
  *out = nullptr;
  rsb200_ctx* c = new (std::nothrow) rsb200_ctx();
  if (!c)
    return RSB200_ERR_CUDA;
  c->device = device;
  cudaError_t e = cudaSetDevice(device);
  if (e == cudaSuccess) {
    cudaDeviceProp prop;
    e = cudaGetDeviceProperties(&prop, device);
    if (e == cudaSuccess) {
      c->sm_count = prop.multiProcessorCount;
      if (prop.major != 9 || prop.minor != 0)
        e = cudaErrorNoKernelImageForDevice; // sm_90a only, no fallback path
    }
  }
  if (e == cudaSuccess)
    e = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking);
  for (int i = 0; i < N_PIPE && e == cudaSuccess; ++i)
    e = cudaStreamCreateWithFlags(&c->pipe[i], cudaStreamNonBlocking);
  if (e != cudaSuccess) {
    fprintf(stderr, "rsb200_create: no usable CUDA device (%s); there is no CPU "
                    "fallback\n",
            cudaGetErrorString(e));
    delete c;
    return RSB200_ERR_CUDA;
  }
  // opt in to the dynamic shared memory the kernels need
  cudaFuncSetAttribute(k2_entropy_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                       (int)sizeof(K2Shared));
  cudaFuncSetAttribute(k2_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                       (int)fused_smem_bytes(4));
  cudaFuncSetAttribute(lookup_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, LUT_SMEM_BYTES);
  cudaDeviceGetAttribute(&c->sm_count, cudaDevAttrMultiProcessorCount, device);
  {
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
      uint64_t keep = ~0ull;
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
    } else {
      cudaGetLastError();
    }
  }
  cudaFuncSetAttribute(k2_tile_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                       (int)tile_smem_bytes<1>());
  cudaFuncSetAttribute(k2_clean2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                       (int)tile_smem_bytes<1>());
  cudaFuncSetAttribute(k2_tile_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                       (int)tile_smem_bytes<2>());
  cudaFuncSetAttribute(k2_range_count_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                       (int)fused_smem_bytes(4));
  cudaFuncSetAttribute(k2_range_diffs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                       (int)fused_smem_bytes(4));
  *out = c;
  return RSB200_OK;
}

extern "C" void rsb200_destroy(rsb200_ctx* c) {
  if (!c)
    return;
  cudaSetDevice(c->device);
  cudaFree(c->d_in);
  cudaFree(c->d_out);
  if (c->h_in)
    cudaFreeHost(c->h_in);
  if (c->h_out)
    cudaFreeHost(c->h_out);
  for (cudaEvent_t e : c->stage_events)
    cudaEventDestroy(e);
  if (c->stream)
    cudaStreamDestroy(c->stream);
  for (int i = 0; i < N_PIPE; ++i)
    if (c->pipe[i])
      cudaStreamDestroy(c->pipe[i]);
  delete c;
}

extern "C" const char* rsb200_last_error(const rsb200_ctx* c) { return c ? c->err : ""; }
extern "C" uint64_t rsb200_kernel_launches(const rsb200_ctx* c) { return c ? c->launches : 0; }
extern "C" int rsb200_device_sm_count(const rsb200_ctx* c) { return c ? c->sm_count : 0; }

#ifdef RSB200_PHASE_TIMING
// profiling builds only (tools/phase_timing.py): read/reset the per-phase cycle sums
extern "C" int rsb200_debug_phase_cycles(unsigned long long* out16, int reset) {
  cudaDeviceSynchronize();
  if (out16 && cudaMemcpyFromSymbol(out16, rsb200::g_phase_cycles, 16 * sizeof(unsigned long long)) != cudaSuccess)
    return RSB200_ERR_CUDA;
  if (reset) {
    unsigned long long z[16] = {0};
    if (cudaMemcpyToSymbol(rsb200::g_phase_cycles, z, sizeof z) != cudaSuccess)
      return RSB200_ERR_CUDA;
  }
  return RSB200_OK;
}
extern "C" int rsb200_debug_tile_phase_cycles(unsigned long long* out16, int reset) {
  cudaDeviceSynchronize();
  if (out16 && cudaMemcpyFromSymbol(out16, rsb200::g_tile_phase_cycles, 16 * sizeof(unsigned long long)) != cudaSuccess)
    return RSB200_ERR_CUDA;
  if (reset) {
    unsigned long long z[16] = {0};
    if (cudaMemcpyToSymbol(rsb200::g_tile_phase_cycles, z, sizeof z) != cudaSuccess)
      return RSB200_ERR_CUDA;
  }
  return RSB200_OK;
}
#endif

// ------------------------------------------------------------------
// unpack plan
// ------------------------------------------------------------------
static int unpack_template_bps(int bps) {
  return (bps == 8 || bps == 10 || bps == 12 || bps == 14 || bps == 16) ? bps : 0;
}

extern "C" int rsb200_unpack_plan_create(rsb200_ctx* ctx, const rsb200_unpack_job* jobs,
                                         int njobs, rsb200_plan** out) {
  if (!ctx || !jobs || njobs <= 0 || !out)
    return set_err(ctx, RSB200_ERR_ARG, "unpack_plan_create: bad arguments");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  rsb200_plan* p = new (std::nothrow) rsb200_plan();
  if (!p)
    return RSB200_ERR_CUDA;
  p->ctx = ctx;
  p->kind = 0;
  p->nunits = njobs;
  std::map<std::pair<int, bool>, std::vector<UnpackJobDev>> buckets;
  std::map<std::pair<int, bool>, std::vector<UnpackFastJobDev>> fast_buckets;
  for (int i = 0; i < njobs; ++i) {
    const rsb200_unpack_job& j = jobs[i];
    if (j.bps < 1 || j.bps > 16 || j.order < 0 || j.order > 3 || j.rows < 0 ||
        j.samples <= 0 || j.in_pitch <= 0 || j.out_pitch <= 0 || j.row0 < 0 ||
        j.out_col0 < 0 ||
        ((uint64_t)j.samples * (uint64_t)j.bps) % 8 != 0 ||
        (uint64_t)j.in_pitch < ((uint64_t)j.samples * j.bps) / 8 ||
        (uint64_t)j.rows * (uint64_t)j.in_pitch > j.in_size ||
        ((uint64_t)j.out_col0 + j.samples) * 2 > (uint64_t)j.out_pitch) {
      delete p;
      return set_err(ctx, RSB200_ERR_ARG, "unpack job %d: malformed descriptor", i);
    }
    if (j.rows == 0)
      continue;
    UnpackJobDev d;
    memset(&d, 0, sizeof d);
    d.in_offset = j.in_offset;
    d.in_size = j.in_size;
    d.out_offset = j.out_offset;
    d.out_pitch = j.out_pitch;
    d.row0 = j.row0;
    d.rows = j.rows;
    d.samples = j.samples;
    d.out_col0 = j.out_col0;
    d.in_pitch = j.in_pitch;
    d.bps = j.bps;
    d.order = j.order;
    const int groups = (j.samples + 7) / 8;
    d.nchunks = (groups + UNPACK_MAX_CHUNK_GROUPS - 1) / UNPACK_MAX_CHUNK_GROUPS;
    d.chunk_groups = (groups + d.nchunks - 1) / d.nchunks;
    d.vec_ok = ((j.out_offset % 16) == 0 && (j.out_pitch % 16) == 0 &&
                (j.out_col0 % 8) == 0)
                   ? 1u
                   : 0u;
    const uint32_t ipr = (uint32_t)((j.samples + 15) / 16);
    const bool fast = unpack_template_bps(j.bps) != 0 && (j.in_offset % 4) == 0 &&
                      (j.in_pitch % 4) == 0 && ipr >= 64 &&
                      (uint64_t)j.rows * ipr < 0xFFFF0000ull;
    if (fast) {
      UnpackFastJobDev f;
      memset(&f, 0, sizeof f);
      f.in_offset = j.in_offset;
      f.out_offset = j.out_offset;
      f.out_pitch = j.out_pitch;
      f.row0 = j.row0;
      f.rows = j.rows;
      f.samples = j.samples;
      f.out_col0 = j.out_col0;
      f.in_pitch = j.in_pitch;
      f.order = j.order;
      f.ipr = ipr;
      f.total_items = (uint32_t)j.rows * ipr;
      f.vec_ok = d.vec_ok;
      f.row_bytes = (uint32_t)((uint64_t)j.samples * j.bps / 8);
      fast_buckets[{j.bps, j.order == RSB200_LSB}].push_back(f);
    } else {
      buckets[{unpack_template_bps(j.bps), j.order == RSB200_LSB}].push_back(d);
    }
    p->in_bytes += (uint64_t)j.rows * ((uint64_t)j.samples * j.bps / 8);
    p->out_bytes += (uint64_t)j.rows * (uint64_t)j.samples * 2;
    p->pixels += (uint64_t)j.rows * (uint64_t)j.samples;
    p->need_in = std::max<uint64_t>(p->need_in, sat_add(j.in_offset, (uint64_t)j.rows * j.in_pitch));
    p->need_out = std::max<uint64_t>(p->need_out, sat_add(j.out_offset, ((uint64_t)j.row0 + j.rows - 1) * j.out_pitch +
                         2ull * ((uint64_t)j.out_col0 + j.samples)));
  }
  for (auto& kv : buckets) {
    UnpackGroup g;
    g.bps_t = kv.first.first;
    g.lsb = kv.first.second;
    uint32_t nb = 0;
    for (auto& d : kv.second) {
      d.block_begin = nb;
      nb += (uint32_t)d.rows * (uint32_t)d.nchunks;
    }
    g.njobs = (int)kv.second.size();
    g.nblocks = nb;
    cudaError_t e = rsb_dev_alloc(&g.d_jobs, sizeof(UnpackJobDev) * kv.second.size());
    if (e == cudaSuccess)
      e = cudaMemcpy(g.d_jobs, kv.second.data(), sizeof(UnpackJobDev) * kv.second.size(),
                     cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
      rsb200_plan_destroy(p);
      return set_err(ctx, RSB200_ERR_CUDA, "unpack plan upload failed: %s",
                     cudaGetErrorString(e));
    }
    p->groups.push_back(g);
  }
  for (auto& kv : fast_buckets) {
    UnpackFastGroup g;
    g.bps = kv.first.first;
    g.lsb = kv.first.second;
    uint32_t nb = 0;
    for (auto& f : kv.second) {
      f.block_begin = nb;
      nb += (f.total_items + UNPACK_IPB - 1) / UNPACK_IPB;
    }
    g.njobs = (int)kv.second.size();
    g.nblocks = nb;
    g.h_jobs = kv.second;
    cudaError_t e = rsb_dev_alloc(&g.d_jobs, sizeof(UnpackFastJobDev) * kv.second.size());
    if (e == cudaSuccess)
      e = cudaMemcpy(g.d_jobs, kv.second.data(), sizeof(UnpackFastJobDev) * kv.second.size(),
                     cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
      rsb200_plan_destroy(p);
      return set_err(ctx, RSB200_ERR_CUDA, "unpack plan upload failed: %s",
                     cudaGetErrorString(e));
    }
    p->fast_groups.push_back(g);
  }
  p->launches_per_run = (int)(p->groups.size() + p->fast_groups.size());
  *out = p;
  return RSB200_OK;
}

// ------------------------------------------------------------------
// fixed-layout raw forms (K1b)
// ------------------------------------------------------------------
extern "C" int rsb200_raw_plan_create(rsb200_ctx* ctx, const rsb200_raw_job* jobs, int njobs,
                                      const uint16_t* tables, int ntables, rsb200_plan** out) {
  if (!ctx || !jobs || njobs <= 0 || !out || ntables < 0 || (ntables > 0 && !tables))
    return set_err(ctx, RSB200_ERR_ARG, "raw_plan_create: bad arguments");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  rsb200_plan* p = new (std::nothrow) rsb200_plan();
  if (!p)
    return RSB200_ERR_CUDA;
  p->ctx = ctx;
  p->kind = 2;
  p->nunits = njobs;
  std::map<int, std::vector<RawJobDev>> buckets;
  for (int i = 0; i < njobs; ++i) {
    const rsb200_raw_job& j = jobs[i];
    const bool fmt_ok = j.format >= RSB200_RAW_8BIT && j.format <= RSB200_RAW_F32_COPY;
    const uint32_t ob = fmt_ok ? raw_out_sample_bytes(j.format) : 2u;
    bool ok = fmt_ok && j.rows >= 0 && j.samples > 0 && j.in_pitch > 0 && j.out_pitch > 0 &&
              j.row0 >= 0 && j.out_col0 >= 0 && (j.out_offset % ob) == 0 &&
              ((uint32_t)j.out_pitch % ob) == 0 &&
              ((uint64_t)j.out_col0 + j.samples) * ob <= (uint64_t)j.out_pitch &&
              (uint64_t)j.rows * (uint64_t)j.in_pitch <= j.in_size;
    if (ok) {
      // bytes one row really occupies
      uint64_t need = raw_in_bytes(j.format, (uint32_t)j.samples);
      if (j.format == RSB200_RAW_12BIT_CONTROL_BE || j.format == RSB200_RAW_12BIT_CONTROL_LE) {
        ok = (j.samples % 2) == 0; // (12*w) % 8 == 0, UncompressedDecompressor.cpp:89-90
        need += (uint64_t)(j.samples + 2) / 10;
      }
      ok = ok && need <= (uint64_t)j.in_pitch;
      if (j.format == RSB200_RAW_8BIT_TABLE)
        ok = ok && j.table >= 0 && j.table < ntables;
    }
    if (!ok) {
      delete p;
      return set_err(ctx, RSB200_ERR_ARG, "raw job %d: malformed descriptor", i);
    }
    if (j.rows == 0)
      continue;
    RawJobDev d;
    memset(&d, 0, sizeof d);
    d.in_offset = j.in_offset;
    d.out_offset = j.out_offset;
    d.out_pitch = (uint32_t)j.out_pitch;
    d.in_pitch = (uint32_t)j.in_pitch;
    d.row0 = (uint32_t)j.row0;
    d.rows = (uint32_t)j.rows;
    d.samples = (uint32_t)j.samples;
    d.out_col0 = (uint32_t)j.out_col0;
    d.format = (uint32_t)j.format;
    d.table = (uint32_t)j.table;
    const uint32_t K = raw_item_samples(j.format);
    d.ipr = ((uint32_t)j.samples + K - 1) / K;
    if ((uint64_t)d.ipr * d.rows >= 0xFFFF0000ull) {
      delete p;
      return set_err(ctx, RSB200_ERR_ARG, "raw job %d: too large", i);
    }
    buckets[j.format].push_back(d);
    p->in_bytes += (uint64_t)j.rows * raw_in_bytes(j.format, (uint32_t)j.samples);
    p->out_bytes += (uint64_t)j.rows * (uint64_t)j.samples * ob;
    p->pixels += (uint64_t)j.rows * (uint64_t)j.samples;
    p->need_in = std::max<uint64_t>(p->need_in, sat_add(j.in_offset, (uint64_t)j.rows * j.in_pitch));
    p->need_out = std::max<uint64_t>(p->need_out, sat_add(j.out_offset, ((uint64_t)j.row0 + j.rows - 1) * j.out_pitch +
                         (uint64_t)ob * ((uint64_t)j.out_col0 + j.samples)));
  }
  if (ntables > 0) {
    const size_t tb = (size_t)ntables * 65536u * sizeof(uint16_t);
    cudaError_t e = rsb_dev_alloc(&p->d_raw_tables, tb);
    if (e == cudaSuccess)
      e = cudaMemcpy(p->d_raw_tables, tables, tb, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
      rsb200_plan_destroy(p);
      return set_err(ctx, RSB200_ERR_CUDA, "raw plan upload failed: %s", cudaGetErrorString(e));
    }
  }
  for (auto& kv : buckets) {
    RawGroup g;
    g.format = kv.first;
    uint64_t items = 0;
    for (auto& d : kv.second) {
      d.item_begin = (uint32_t)items;
      items += (uint64_t)d.ipr * d.rows;
    }
    if (items >= 0xFFFF0000ull) {
      rsb200_plan_destroy(p);
      return set_err(ctx, RSB200_ERR_ARG, "raw plan: too many items of format %d", g.format);
    }
    g.total_items = (uint32_t)items;
    g.njobs = (int)kv.second.size();
    cudaError_t e = rsb_dev_alloc(&g.d_jobs, sizeof(RawJobDev) * kv.second.size());
    if (e == cudaSuccess)
      e = cudaMemcpy(g.d_jobs, kv.second.data(), sizeof(RawJobDev) * kv.second.size(),
                     cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
      rsb200_plan_destroy(p);
      return set_err(ctx, RSB200_ERR_CUDA, "raw plan upload failed: %s", cudaGetErrorString(e));
    }
    p->raw_groups.push_back(g);
  }
  p->launches_per_run = (int)p->raw_groups.size();
  *out = p;
  return RSB200_OK;
}

template <int FORMAT>
static cudaError_t launch_rawform(const RawGroup& g, const uint8_t* in, uint64_t in_total,
                                  uint8_t* outp, const uint16_t* tables, cudaStream_t st) {
  const uint32_t nb = (g.total_items + RAW_NT - 1) / RAW_NT;
  rawform_kernel<FORMAT><<<nb, RAW_NT, 0, st>>>(in, in_total, outp, g.d_jobs, g.njobs,
                                                g.total_items, tables);
  return cudaGetLastError();
}

static cudaError_t run_raw_group(const RawGroup& g, const uint8_t* in, uint64_t in_total,
                                 uint8_t* outp, const uint16_t* tables, cudaStream_t st) {
  switch (g.format) {
#define RSB_CASE(F)                                                               \
  case F:                                                                         \
    return launch_rawform<F>(g, in, in_total, outp, tables, st);
    RSB_CASE(RSB200_RAW_8BIT)
    RSB_CASE(RSB200_RAW_8BIT_TABLE)
    RSB_CASE(RSB200_RAW_12BIT_CONTROL_BE)
    RSB_CASE(RSB200_RAW_12BIT_CONTROL_LE)
    RSB_CASE(RSB200_RAW_12BIT_LEFT_BE)
    RSB_CASE(RSB200_RAW_12BIT_LEFT_LE)
    RSB_CASE(RSB200_RAW_FP16_MSB)
    RSB_CASE(RSB200_RAW_FP16_LSB)
    RSB_CASE(RSB200_RAW_FP24_MSB)
    RSB_CASE(RSB200_RAW_FP24_LSB)
    RSB_CASE(RSB200_RAW_F32_COPY)
#undef RSB_CASE
  default:
    return cudaErrorInvalidValue;
  }
}

// ------------------------------------------------------------------
// sRaw interpolation (K5)
// ------------------------------------------------------------------
// K12: whole-image table lookup (RawImageData::sixteenBitLookup)
extern "C" int rsb200_lookup_plan_create(rsb200_ctx* ctx, const rsb200_lookup_job* jobs, int njobs,
                                         const uint16_t* tables, int ntables, int dither,
                                         rsb200_plan** out) {
  if (!ctx || !jobs || njobs <= 0 || !out || !tables || ntables <= 0)
    return set_err(ctx, RSB200_ERR_ARG, "lookup_plan_create: bad arguments");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  std::unique_ptr<rsb200_plan, void (*)(rsb200_plan*)> holder(new rsb200_plan, rsb200_plan_destroy);
  rsb200_plan* p = holder.get();
  p->ctx = ctx;
  p->kind = 10;
  p->nunits = njobs;
  p->lookup_dither = dither != 0;
  {
    const char* smem_env = getenv("RSB200_LUT_SMEM");
    p->lookup_smem = smem_env && smem_env[0] == '1';
  }
  p->lookup_ntables = ntables;
  std::vector<LookupJobDev> hj((size_t)njobs);
  uint64_t quads = 0;
  for (int i = 0; i < njobs; ++i) {
    if (const char* why = lookup_build_job(jobs[i], ntables, (uint32_t)quads, &hj[i]))
      return set_err(ctx, RSB200_ERR_ARG, "lookup job %d: %s", i, why);
    quads += lookup_job_quads(jobs[i]);
    if (quads > 0x7FFFFFFFull)
      return set_err(ctx, RSB200_ERR_ARG, "lookup plan: too many rows");
    const uint64_t bytes = (uint64_t)hj[i].ncols * jobs[i].height * 2;
    p->in_bytes += bytes;
    p->out_bytes += bytes;
    p->pixels += (uint64_t)jobs[i].width * jobs[i].height;
    p->need_out = std::max<uint64_t>(p->need_out, sat_add(jobs[i].offset, (uint64_t)jobs[i].height * jobs[i].pitch));
  }
  p->lookup_njobs = njobs;
  p->lookup_quads = (uint32_t)quads;
  {
    // enough warps to fill the machine (~32 per SM), but at least 2 iterations of 32 groups each
    uint32_t min_groups = 0xFFFFFFFFu;
    for (int i = 0; i < njobs; ++i)
      min_groups = std::min(min_groups, hj[(size_t)i].ngroups);
    const uint32_t want = (uint32_t)((32ull * (uint64_t)ctx->sm_count + quads - 1) / std::max<uint64_t>(quads, 1));
    p->lookup_nseg = std::max(1u, std::min(std::min(want, 8u), std::max(1u, min_groups / 64u)));
    if (const char* e = getenv("RSB200_LUT_NSEG"))
      p->lookup_nseg = (uint32_t)std::max(1, std::min(64, atoi(e)));
  }
  const size_t tbytes = sizeof(uint16_t) * (size_t)ntables * (dither ? 131072u : 65536u);
  CUDA_TRY(ctx, rsb_dev_alloc((void**)&p->d_lookup_jobs, sizeof(LookupJobDev) * hj.size()));
  CUDA_TRY(ctx, cudaMemcpy(p->d_lookup_jobs, hj.data(), sizeof(LookupJobDev) * hj.size(),
                           cudaMemcpyHostToDevice));
  CUDA_TRY(ctx, rsb_dev_alloc((void**)&p->d_lookup_tables, tbytes));
  CUDA_TRY(ctx, cudaMemcpy(p->d_lookup_tables, tables, tbytes, cudaMemcpyHostToDevice));
  p->launches_per_run = 1;
  *out = holder.release();
  return RSB200_OK;
}

// K11: bad-pixel interpolation (RawImageData::fixBadPixels)
extern "C" int rsb200_badpix_plan_create(rsb200_ctx* ctx, const rsb200_badpix_job* jobs, int njobs,
                                         const uint32_t* positions, uint32_t npositions,
                                         rsb200_plan** out) {
  if (!ctx || !jobs || njobs <= 0 || !out || (npositions && !positions))
    return set_err(ctx, RSB200_ERR_ARG, "badpix_plan_create: bad arguments");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  std::unique_ptr<rsb200_plan, void (*)(rsb200_plan*)> holder(new rsb200_plan, rsb200_plan_destroy);
  rsb200_plan* p = holder.get();
  p->ctx = ctx;
  p->kind = 9;
  p->nunits = njobs;
  std::vector<BadPixJobDev> hj((size_t)njobs);
  std::vector<uint8_t> maps;
  std::vector<uint32_t> list;
  for (int i = 0; i < njobs; ++i) {
    if (const char* why = badpix_build(jobs[i], positions, npositions, jobs[i].prior_map, &hj[i],
                                       &maps, &list))
      return set_err(ctx, RSB200_ERR_ARG, "badpix job %d: %s", i, why);
    p->pixels += hj[i].count;
    p->in_bytes += (uint64_t)hj[i].count * 2 * 4; // up to four neighbours read per bad pixel
    p->out_bytes += (uint64_t)hj[i].count * 2;
    p->need_out = std::max<uint64_t>(p->need_out, sat_add(jobs[i].offset, (uint64_t)jobs[i].height * jobs[i].pitch));
  }
  if (list.size() > 0x7FFFFFFFull)
    return set_err(ctx, RSB200_ERR_ARG, "badpix plan: too many bad pixels");
  p->badpix_njobs = njobs;
  p->badpix_total = (uint32_t)list.size();
  CUDA_TRY(ctx, rsb_dev_alloc((void**)&p->d_badpix_jobs, sizeof(BadPixJobDev) * hj.size()));
  CUDA_TRY(ctx, cudaMemcpy(p->d_badpix_jobs, hj.data(), sizeof(BadPixJobDev) * hj.size(),
                           cudaMemcpyHostToDevice));
  CUDA_TRY(ctx, rsb_dev_alloc((void**)&p->d_badpix_list, sizeof(uint32_t) * (list.size() + 1)));
  if (!list.empty())
    CUDA_TRY(ctx, cudaMemcpy(p->d_badpix_list, list.data(), sizeof(uint32_t) * list.size(),
                             cudaMemcpyHostToDevice));
  CUDA_TRY(ctx, rsb_dev_alloc((void**)&p->d_badpix_maps, maps.size() + 16));
  if (!maps.empty())
    CUDA_TRY(ctx, cudaMemcpy(p->d_badpix_maps, maps.data(), maps.size(), cudaMemcpyHostToDevice));
  p->launches_per_run = p->badpix_total ? 1 : 0;
  *out = holder.release();
  return RSB200_OK;
}

// K10: a DNG opcode list in one pass (DngOpcodes::applyOpCodes)
static_assert(DNGOP_BAD_CAP == RSB200_PANA_BAD_CAP, "one list capacity for both users");
extern "C" int rsb200_dngop_plan_create(rsb200_ctx* ctx, const rsb200_dngop_job* jobs, int njobs,
                                        const rsb200_dng_op* ops, int nops, const uint16_t* tables,
                                        int ntables, const uint32_t* deltas, int ndeltas,
                                        rsb200_plan** out) {
  if (!ctx || !jobs || njobs <= 0 || !out || nops < 0 || (nops > 0 && !ops) || ntables < 0 ||
      (ntables > 0 && !tables) || ndeltas < 0 || (ndeltas > 0 && !deltas))
    return set_err(ctx, RSB200_ERR_ARG, "dngop_plan_create: bad arguments");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  std::unique_ptr<rsb200_plan, void (*)(rsb200_plan*)> holder(new rsb200_plan, rsb200_plan_destroy);
  rsb200_plan* p = holder.get();
  p->ctx = ctx;
  p->kind = 8;
  p->nunits = njobs;
  std::vector<DngOpJobDev> hj((size_t)njobs);
  std::vector<DngOpDev> ho((size_t)nops);
  p->pana_zero_slot.assign((size_t)nops, -1);
  uint64_t units = 0;
  if (const char* why = dngop_build(jobs, njobs, ops, nops, ntables, ndeltas, hj.data(), ho.data(),
                                    p->pana_zero_slot.data(), &p->pana_zero_slots, &units))
    return set_err(ctx, RSB200_ERR_ARG, "dngop plan: %s", why);
  for (int i = 0; i < njobs; ++i) {
    const uint64_t bytes = (uint64_t)(hj[i].row1 - hj[i].row0) * hj[i].samples * (jobs[i].is_f32 ? 4u : 2u);
    p->in_bytes += bytes;
    p->out_bytes += bytes;
    p->pixels += (uint64_t)(hj[i].row1 - hj[i].row0) * jobs[i].width;
    p->need_out = std::max<uint64_t>(p->need_out, sat_add(jobs[i].offset, (uint64_t)jobs[i].height * jobs[i].pitch));
  }
  p->dngop_njobs = njobs;
  p->dngop_units = (uint32_t)units;
  CUDA_TRY(ctx, rsb_dev_alloc((void**)&p->d_dngop_jobs, sizeof(DngOpJobDev) * hj.size()));
  CUDA_TRY(ctx, cudaMemcpy(p->d_dngop_jobs, hj.data(), sizeof(DngOpJobDev) * hj.size(),
                           cudaMemcpyHostToDevice));
  CUDA_TRY(ctx, rsb_dev_alloc((void**)&p->d_dngop_ops, sizeof(DngOpDev) * (ho.size() + 1)));
  if (!ho.empty())
    CUDA_TRY(ctx, cudaMemcpy(p->d_dngop_ops, ho.data(), sizeof(DngOpDev) * ho.size(),
                             cudaMemcpyHostToDevice));
  CUDA_TRY(ctx, rsb_dev_alloc((void**)&p->d_dngop_tables, sizeof(uint16_t) * 65536 * (size_t)(ntables + 1)));
  if (ntables)
    CUDA_TRY(ctx, cudaMemcpy(p->d_dngop_tables, tables, sizeof(uint16_t) * 65536 * (size_t)ntables,
                             cudaMemcpyHostToDevice));
  CUDA_TRY(ctx, rsb_dev_alloc((void**)&p->d_dngop_deltas, sizeof(uint32_t) * (size_t)(ndeltas + 1)));
  if (ndeltas)
    CUDA_TRY(ctx, cudaMemcpy(p->d_dngop_deltas, deltas, sizeof(uint32_t) * (size_t)ndeltas,
                             cudaMemcpyHostToDevice));
  if (p->pana_zero_slots) {
    CUDA_TRY(ctx, rsb_dev_alloc((void**)&p->d_pana_zero_count, sizeof(uint32_t) * (size_t)p->pana_zero_slots));
    CUDA_TRY(ctx, rsb_dev_alloc((void**)&p->d_pana_zero_list,
                             sizeof(uint32_t) * (size_t)DNGOP_BAD_CAP * (size_t)p->pana_zero_slots));
  }
  p->launches_per_run = units ? 1 : 0;
  *out = holder.release();
  return RSB200_OK;
}

// K9: black / white scaling in place (RawImageDataU16::scaleValues)
extern "C" int rsb200_scale_plan_create(rsb200_ctx* ctx, const rsb200_scale_job* jobs, int njobs,
                                        rsb200_plan** out) {
  if (!ctx || !jobs || njobs <= 0 || !out)
    return set_err(ctx, RSB200_ERR_ARG, "scale_plan_create: bad arguments");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  std::unique_ptr<rsb200_plan, void (*)(rsb200_plan*)> holder(new rsb200_plan, rsb200_plan_destroy);
  rsb200_plan* p = holder.get();
  p->ctx = ctx;
  p->kind = 7;
  p->nunits = njobs;
  std::vector<ScaleJobDev> dev[2];
  uint32_t quads[2] = {0, 0};
  for (int i = 0; i < njobs; ++i) {
    ScaleJobDev d;
    int mode = 0;
    if (const char* why = scale_build_job(jobs[i], 0, &d, &mode))
      return set_err(ctx, RSB200_ERR_ARG, "scale job %d: %s", i, why);
    d.quad_begin = quads[mode];
    const uint64_t q = (uint64_t)quads[mode] + scale_job_quads(jobs[i]);
    if (q > 0x7FFFFFFFull)
      return set_err(ctx, RSB200_ERR_ARG, "scale plan: too many rows");
    quads[mode] = (uint32_t)q;
    dev[mode].push_back(d);
    // what one run reads and writes: the samples of the rows it walks
    const uint64_t samples = (uint64_t)d.ncols * jobs[i].crop_h;
    p->in_bytes += samples * 2;
    p->out_bytes += samples * 2;
    p->pixels += (uint64_t)jobs[i].crop_w * jobs[i].crop_h;
    p->need_out = std::max<uint64_t>(p->need_out, sat_add(jobs[i].offset, (uint64_t)jobs[i].height * jobs[i].pitch));
  }
  for (int mode = 0; mode < 2; ++mode) {
    if (dev[mode].empty())
      continue;
    ScaleGroup g;
    g.mode = mode;
    g.njobs = (int)dev[mode].size();
    g.total_quads = quads[mode];
    {
      uint32_t min_groups = 0xFFFFFFFFu;
      for (const ScaleJobDev& d : dev[mode])
        min_groups = std::min(min_groups, d.ngroups);
      const uint32_t want = (uint32_t)((32ull * (uint64_t)ctx->sm_count + g.total_quads - 1) / std::max(g.total_quads, 1u));
      g.nseg = mode == 0 ? 1u : std::max(1u, std::min(std::min(want, 8u), std::max(1u, min_groups / 64u)));
    }
    CUDA_TRY(ctx, rsb_dev_alloc((void**)&g.d_jobs, sizeof(ScaleJobDev) * dev[mode].size()));
    p->scale_groups.push_back(g); // owned by the plan from here on
    CUDA_TRY(ctx, cudaMemcpy(g.d_jobs, dev[mode].data(), sizeof(ScaleJobDev) * dev[mode].size(),
                             cudaMemcpyHostToDevice));
  }
  p->launches_per_run = (int)p->scale_groups.size();
  *out = holder.release();
  return RSB200_OK;
}

extern "C" int rsb200_sraw_plan_create(rsb200_ctx* ctx, const rsb200_sraw_job* jobs, int njobs,
                                       rsb200_plan** out) {
  if (!ctx || !jobs || njobs <= 0 || !out)
    return set_err(ctx, RSB200_ERR_ARG, "sraw_plan_create: bad arguments");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  rsb200_plan* p = new (std::nothrow) rsb200_plan();
  if (!p)
    return RSB200_ERR_CUDA;
  p->ctx = ctx;
  p->kind = 3;
  p->nunits = njobs;
  std::map<std::pair<int, bool>, std::vector<SrawJobDev>> buckets;
  for (int i = 0; i < njobs; ++i) {
    const rsb200_sraw_job& j = jobs[i];
    const bool is422 = j.sub_x == 2 && j.sub_y == 1, is420 = j.sub_x == 2 && j.sub_y == 2;
    const uint32_t per = is420 ? 6u : 4u;
    const bool ok = (is422 || is420) && j.version <= 2 && !(is420 && j.version == 0) &&
                    j.num_mcus >= 2 && j.in_rows >= 1 && (j.in_offset % 4) == 0 &&
                    (j.in_pitch % 4) == 0 && (j.out_offset % 4) == 0 && (j.out_pitch % 4) == 0 &&
                    (uint64_t)j.num_mcus * per * 2 <= j.in_pitch &&
                    (uint64_t)j.num_mcus * 12 <= j.out_pitch &&
                    (uint64_t)j.num_mcus * j.in_rows < 0xFFFF0000ull;
    if (!ok) {
      delete p;
      return set_err(ctx, RSB200_ERR_ARG, "sraw job %d: malformed descriptor", i);
    }
    SrawJobDev d;
    memset(&d, 0, sizeof d);
    d.in_offset = j.in_offset;
    d.out_offset = j.out_offset;
    d.in_pitch = j.in_pitch;
    d.out_pitch = j.out_pitch;
    d.num_mcus = j.num_mcus;
    d.in_rows = j.in_rows;
    d.k0 = j.sraw_coeffs[0];
    d.k1 = j.sraw_coeffs[1];
    d.k2 = j.sraw_coeffs[2];
    d.hue = j.hue;
    buckets[{(int)j.version, is420}].push_back(d);
    const uint64_t out_rows = (uint64_t)j.in_rows * j.sub_y;
    p->in_bytes += (uint64_t)j.in_rows * j.num_mcus * per * 2;
    p->out_bytes += out_rows * j.num_mcus * 12;
    p->pixels += out_rows * j.num_mcus * 2;
    p->need_in = std::max<uint64_t>(p->need_in, sat_add(j.in_offset, ((uint64_t)j.in_rows - 1) * j.in_pitch +
                                                    (uint64_t)j.num_mcus * per * 2));
    p->need_out = std::max<uint64_t>(p->need_out, sat_add(j.out_offset, (out_rows - 1) * j.out_pitch +
                                                      (uint64_t)j.num_mcus * 12));
  }
  for (auto& kv : buckets) {
    SrawGroup g;
    g.version = kv.first.first;
    g.is420 = kv.first.second;
    uint64_t n = 0;
    for (auto& d : kv.second) {
      d.mcu_begin = (uint32_t)n;
      n += (uint64_t)d.num_mcus * d.in_rows;
    }
    if (n >= 0xFFFF0000ull) {
      rsb200_plan_destroy(p);
      return set_err(ctx, RSB200_ERR_ARG, "sraw plan: too many MCUs");
    }
    g.total_mcus = (uint32_t)n;
    g.njobs = (int)kv.second.size();
    cudaError_t e = rsb_dev_alloc(&g.d_jobs, sizeof(SrawJobDev) * kv.second.size());
    if (e == cudaSuccess)
      e = cudaMemcpy(g.d_jobs, kv.second.data(), sizeof(SrawJobDev) * kv.second.size(),
                     cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
      rsb200_plan_destroy(p);
      return set_err(ctx, RSB200_ERR_CUDA, "sraw plan upload failed: %s", cudaGetErrorString(e));
    }
    p->sraw_groups.push_back(g);
  }
  p->launches_per_run = (int)p->sraw_groups.size();
  *out = p;
  return RSB200_OK;
}

// ------------------------------------------------------------------
// Hasselblad (K2H, hasselblad.cuh)
// ------------------------------------------------------------------
extern "C" int rsb200_hasselblad_plan_create(rsb200_ctx* ctx, const rsb200_huff_table* tables, int ntables,
                                             const rsb200_hasselblad_job* jobs, int njobs,
                                             rsb200_plan** out) {
  if (!ctx || !tables || ntables <= 0 || !jobs || njobs <= 0 || !out)
    return set_err(ctx, RSB200_ERR_ARG, "hasselblad_plan_create: bad arguments");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  std::vector<DevTable> ht((size_t)ntables);
  for (int i = 0; i < ntables; ++i)
    if (!build_dev_table(tables[i], ht[(size_t)i]))
      return set_err(ctx, RSB200_ERR_ARG, "huffman table %d is malformed", i);
  rsb200_plan* p = new (std::nothrow) rsb200_plan();
  if (!p)
    return RSB200_ERR_CUDA;
  p->ctx = ctx;
  p->kind = 11;
  p->nunits = njobs;
  std::vector<DevHassJob> dj((size_t)njobs);
  std::vector<DevHassCta> ctas;
  std::vector<uint32_t> seg_job, row_begin((size_t)njobs + 1, 0);
  uint64_t nseg_total = 0, rows_total = 0;
  for (int i = 0; i < njobs; ++i) {
    const rsb200_hasselblad_job& j = jobs[i];
    // HasselbladDecompressor ctor (HasselbladDecompressor.cpp:39-58) + what the kernels need
    const bool ok = j.width > 0 && j.height > 0 && j.width % 2 == 0 && j.width <= 12000 && j.height <= 8842 &&
                    (j.in_offset % 4) == 0 && j.in_size < (1u << 28) && (j.out_offset % 4) == 0 &&
                    (j.out_pitch % 4) == 0 && (uint64_t)j.width * 2 <= j.out_pitch && j.table < ntables;
    if (!ok) {
      delete p;
      return set_err(ctx, RSB200_ERR_ARG, "hasselblad job %d: malformed descriptor", i);
    }
    DevHassJob& d = dj[(size_t)i];
    memset(&d, 0, sizeof d);
    d.in_offset = j.in_offset;
    d.in_size = j.in_size;
    d.w = j.width;
    d.h = j.height;
    d.out_pitch = j.out_pitch;
    d.out_offset = j.out_offset;
    d.init_pred = j.init_pred;
    d.table = j.table;
    d.seg_begin = (uint32_t)nseg_total;
    // the pump may read (as zero) up to 12 bytes behind the buffer before it throws
    d.nseg = (uint32_t)((((uint64_t)j.in_size + 24) * 8 + H_SEG_BITS - 1) / H_SEG_BITS);
    d.cta_begin = (uint32_t)ctas.size();
    for (uint32_t s0 = 0; s0 < d.nseg; s0 += H_NT)
      ctas.push_back(DevHassCta{(uint32_t)i, s0});
    seg_job.insert(seg_job.end(), d.nseg, (uint32_t)i);
    nseg_total += d.nseg;
    row_begin[(size_t)i] = (uint32_t)rows_total;
    rows_total += j.height;
    p->h_in_size.push_back(j.in_size);
    p->in_bytes += j.in_size;
    p->out_bytes += (uint64_t)j.width * j.height * 2;
    p->pixels += (uint64_t)j.width * j.height;
    p->need_in = std::max<uint64_t>(p->need_in, sat_add(j.in_offset, j.in_size));
    p->need_out = std::max<uint64_t>(p->need_out, sat_add(j.out_offset, ((uint64_t)j.height - 1) * j.out_pitch +
                                                                            (uint64_t)j.width * 2));
  }
  row_begin[(size_t)njobs] = (uint32_t)rows_total;
  if (nseg_total >= 0x7FFFFFFFull || rows_total >= 0x7FFFFFFull) {
    delete p;
    return set_err(ctx, RSB200_ERR_ARG, "hasselblad plan: too large");
  }
  p->hass_nseg = (uint32_t)nseg_total;
  p->hass_ncta = (uint32_t)ctas.size();
  p->hass_rows = (uint32_t)rows_total;
  p->ntables = ntables;
  cudaError_t e = cudaSuccess;
  auto up = [&](void** dptr, const void* src, size_t bytes) {
    if (e != cudaSuccess)
      return;
    e = rsb_dev_alloc(dptr, bytes ? bytes : 16);
    if (e == cudaSuccess && bytes)
      e = cudaMemcpy(*dptr, src, bytes, cudaMemcpyHostToDevice);
  };
  up((void**)&p->d_tables, ht.data(), sizeof(DevTable) * ht.size());
  up((void**)&p->d_hass_jobs, dj.data(), sizeof(DevHassJob) * dj.size());
  up((void**)&p->d_hass_ctas, ctas.data(), sizeof(DevHassCta) * ctas.size());
  up((void**)&p->d_hass_seg_job, seg_job.data(), sizeof(uint32_t) * seg_job.size());
  up((void**)&p->d_hass_row_begin, row_begin.data(), sizeof(uint32_t) * row_begin.size());
  if (e == cudaSuccess)
    e = rsb_dev_alloc((void**)&p->d_hass_u32,
                      sizeof(uint32_t) * (4ull * nseg_total + 2ull * ctas.size() + H_ROUNDS + 8));
  if (e == cudaSuccess)
    e = rsb_dev_alloc((void**)&p->d_hass_states, sizeof(DevHassState) * (size_t)njobs);
  if (e == cudaSuccess)
    e = rsb_host_alloc((void**)&p->h_hass_states, sizeof(DevHassState) * (size_t)njobs);
  if (e != cudaSuccess) {
    rsb200_plan_destroy(p);
    return set_err(ctx, RSB200_ERR_CUDA, "hasselblad plan allocation failed: %s", cudaGetErrorString(e));
  }
  p->launches_per_run = 1 + 2 * H_ROUNDS + 1 + 2 + 1 + 1;
  *out = p;
  return RSB200_OK;
}

static cudaError_t run_hasselblad(const rsb200_plan* p, const uint8_t* in, uint8_t* outp, cudaStream_t st) {
  const uint32_t n = p->hass_nseg, nc = p->hass_ncta;
  uint32_t* start = p->d_hass_u32;
  uint32_t* parsed = start + n;
  uint32_t* exitp = parsed + n;
  uint32_t* count = exitp + n;
  uint32_t* cta_sum = count + n;
  uint32_t* cta_base = cta_sum + nc;
  uint32_t* changed = cta_base + nc;
  const size_t smem = sizeof(HassShared);
  const uint32_t nb = (std::max<uint32_t>(std::max<uint32_t>(n, (uint32_t)p->nunits), H_ROUNDS + 1) + 255) / 256;
  hass_init_kernel<<<nb, 256, 0, st>>>(p->d_hass_jobs, p->nunits, n, p->d_hass_seg_job, start, parsed,
                                       p->d_hass_states, changed);
  for (int r = 0; r < H_ROUNDS; ++r) {
    hass_parse_kernel<<<nc, H_NT, smem, st>>>(in, p->d_hass_jobs, p->d_tables, p->d_hass_ctas, start, parsed,
                                              exitp, count);
    hass_link_kernel<<<(n + 255) / 256, 256, 0, st>>>(p->d_hass_jobs, p->nunits, n, p->d_hass_seg_job, start,
                                                      exitp, changed + r);
  }
  hass_serial_kernel<<<p->nunits, 32, 0, st>>>(in, p->d_hass_jobs, p->d_tables, start, parsed, exitp, count,
                                               changed + (H_ROUNDS - 1));
  hass_ctasum_kernel<<<nc, H_NT, smem, st>>>(p->d_hass_jobs, p->d_hass_ctas, count, cta_sum);
  hass_ctascan_kernel<<<(p->nunits + 63) / 64, 64, 0, st>>>(p->d_hass_jobs, p->nunits, cta_sum, cta_base);
  hass_decode_kernel<<<nc, H_NT, smem, st>>>(in, p->d_hass_jobs, p->d_tables, p->d_hass_ctas, start, exitp,
                                             count, cta_base, outp, p->d_hass_states);
  hass_rows_kernel<<<(p->hass_rows * 32 + 255) / 256, 256, 0, st>>>(p->d_hass_jobs, p->nunits,
                                                                   p->d_hass_row_begin, outp);
  return cudaGetLastError();
}

// ------------------------------------------------------------------
// Phase One (K8)
// ------------------------------------------------------------------
// RSB200_P1 = 1 / 2 select the first (per-lane refills) / second (a thread per row, loads at group
// boundaries) version for A/B runs; default: the third (group headers walked per row, pixels in parallel)
// (read when a plan is created)
static int p1_version() {
  const char* e = getenv("RSB200_P1");
  return (e && (e[0] == '1' || e[0] == '2') && !e[1]) ? e[0] - '0' : 3;
}

extern "C" int rsb200_phaseone_plan_create(rsb200_ctx* ctx, const rsb200_phaseone_job* jobs,
                                           int njobs, const rsb200_phaseone_strip* strips,
                                           int nstrips, rsb200_plan** out) {
  if (!ctx || !jobs || njobs <= 0 || !strips || nstrips <= 0 || !out)
    return set_err(ctx, RSB200_ERR_ARG, "phaseone_plan_create: bad arguments");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  rsb200_plan* p = new (std::nothrow) rsb200_plan();
  if (!p)
    return RSB200_ERR_CUDA;
  p->ctx = ctx;
  p->kind = 6;
  p->nunits = njobs;
  std::vector<P1JobDev> dj((size_t)njobs);
  std::vector<P1StripDev> ds;
  for (int i = 0; i < njobs; ++i) {
    const rsb200_phaseone_job& j = jobs[i];
    // PhaseOneDecompressor ctor + prepareStrips (PhaseOneDecompressor.cpp:42-83)
    bool ok = j.width > 0 && j.height > 0 && j.width % 2 == 0 && j.width <= 11976 &&
              j.height <= 8854 && (j.out_offset % 4) == 0 && (j.out_pitch % 4) == 0 &&
              (uint64_t)j.width * 2 <= j.out_pitch &&
              (uint64_t)j.first_strip + j.height <= (uint64_t)nstrips;
    std::vector<uint8_t> seen(ok ? j.height : 0, 0);
    for (uint32_t k = 0; ok && k < j.height; ++k) {
      const rsb200_phaseone_strip& st = strips[j.first_strip + k];
      ok = st.row < j.height && !seen[st.row];
      if (ok) {
        seen[st.row] = 1;
        P1StripDev d;
        d.in_offset = st.in_offset;
        d.in_size = st.in_size;
        d.row = st.row;
        d.job = (uint32_t)i;
        d.pad = 0;
        ds.push_back(d);
        p->in_bytes += st.in_size;
        p->need_in = std::max<uint64_t>(p->need_in, sat_add(st.in_offset, st.in_size));
      }
    }
    if (!ok) {
      delete p;
      return set_err(ctx, RSB200_ERR_ARG, "phaseone job %d: malformed descriptor or strips", i);
    }
    dj[(size_t)i].out_offset = j.out_offset;
    dj[(size_t)i].out_pitch = j.out_pitch;
    dj[(size_t)i].width = j.width;
    p->out_bytes += (uint64_t)j.width * j.height * 2;
    p->pixels += (uint64_t)j.width * j.height;
    p->need_out = std::max<uint64_t>(p->need_out, sat_add(j.out_offset, ((uint64_t)j.height - 1) * j.out_pitch +
                                                      2ull * j.width));
  }
  p->p1_nstrips = (uint32_t)ds.size();
  for (int i = 0; i < njobs; ++i)
    p->p1_gstride = std::max<uint32_t>(p->p1_gstride, (jobs[i].width / 8u + 1u + 3u) & ~3u); // (16-byte rows)
  cudaError_t e = rsb_dev_alloc((void**)&p->d_p1_strips, sizeof(P1StripDev) * ds.size());
  if (e == cudaSuccess)
    e = rsb_dev_alloc((void**)&p->d_p1_gdesc, sizeof(uint32_t) * (size_t)p->p1_gstride * ds.size());
  if (e == cudaSuccess)
    e = rsb_dev_alloc((void**)&p->d_p1_rowflag, sizeof(uint32_t) * ds.size());
  if (e == cudaSuccess)
    e = cudaMemcpy(p->d_p1_strips, ds.data(), sizeof(P1StripDev) * ds.size(), cudaMemcpyHostToDevice);
  if (e == cudaSuccess)
    e = rsb_dev_alloc((void**)&p->d_p1_jobs, sizeof(P1JobDev) * dj.size());
  if (e == cudaSuccess)
    e = cudaMemcpy(p->d_p1_jobs, dj.data(), sizeof(P1JobDev) * dj.size(), cudaMemcpyHostToDevice);
  if (e == cudaSuccess)
    e = rsb_dev_alloc((void**)&p->d_arw2_bad, sizeof(uint32_t) * (size_t)njobs);
  if (e == cudaSuccess)
    e = rsb_host_alloc((void**)&p->h_arw2_bad, sizeof(uint32_t) * (size_t)njobs);
  if (e != cudaSuccess) {
    rsb200_plan_destroy(p);
    return set_err(ctx, RSB200_ERR_CUDA, "phaseone plan upload failed: %s", cudaGetErrorString(e));
  }
  p->p1_ver = p1_version();
  {
    const char* e = getenv("RSB200_P1W");
    p->p1_walk1 = (e && e[0] >= '1' && e[0] <= '8' && !e[1]) ? e[0] - '0' : 0;
  }
  p->launches_per_run = p->p1_ver == 3 ? 2 : 1;
  *out = p;
  return RSB200_OK;
}

static cudaError_t run_phaseone(const rsb200_plan* p, const uint8_t* in, uint8_t* outp,
                                cudaStream_t st) {
  cudaError_t e = cudaMemsetAsync(p->d_arw2_bad, 0, sizeof(uint32_t) * (size_t)p->nunits, st);
  if (e != cudaSuccess)
    return e;
  const int v = p->p1_ver;
  const uint32_t nb = (p->p1_nstrips + P1_NT - 1) / P1_NT;
  if (v == 1) {
    p1_kernel<<<nb, P1_NT, 0, st>>>(in, outp, p->d_p1_strips, p->p1_nstrips, p->d_p1_jobs,
                                    p->d_arw2_bad);
  } else if (v == 2) {
    p1_kernel_v2<<<nb, P1_NT, 0, st>>>(in, outp, p->d_p1_strips, p->p1_nstrips, p->d_p1_jobs,
                                       p->d_arw2_bad);
  } else {
    p1_walk_kernel<<<(p->p1_nstrips + P1W_NT - 1) / P1W_NT, P1W_NT, 0, st>>>(
        in, p->d_p1_strips, p->p1_nstrips, p->d_p1_jobs, p->p1_gstride, p->d_p1_gdesc, p->d_p1_rowflag,
        p->p1_walk1);
    p1_decode_kernel<<<(p->p1_nstrips * 32u + P1D_NT - 1) / P1D_NT, P1D_NT, 0, st>>>(
        in, outp, p->d_p1_strips, p->p1_nstrips, p->d_p1_jobs, p->p1_gstride, p->d_p1_gdesc,
        p->d_p1_rowflag, p->d_arw2_bad);
  }
  return cudaGetLastError();
}

// ------------------------------------------------------------------
// Panasonic V5 / V6 / V7 (K7)
// ------------------------------------------------------------------
extern "C" int rsb200_pana_plan_create(rsb200_ctx* ctx, const rsb200_pana_job* jobs, int njobs,
                                       rsb200_plan** out) {
  if (!ctx || !jobs || njobs <= 0 || !out)
    return set_err(ctx, RSB200_ERR_ARG, "pana_plan_create: bad arguments");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  rsb200_plan* p = new (std::nothrow) rsb200_plan();
  if (!p)
    return RSB200_ERR_CUDA;
  p->ctx = ctx;
  p->kind = 5;
  p->nunits = njobs;
  std::map<std::pair<int, int>, std::vector<PanaJobDev>> buckets;
  for (int i = 0; i < njobs; ++i) {
    const rsb200_pana_job& j = jobs[i];
    const int bps = j.version == 7 ? 14 : (j.version == 4 ? 12 : j.bps);
    const bool vok = (j.version == 4 || j.version == 5 || j.version == 6 || j.version == 7) &&
                     (bps == 12 || bps == 14);
    const uint32_t npix = !vok ? 1u
                               : (j.version == 4 ? 14u
                                                 : (j.version == 6 ? (bps == 14 ? 11u : 14u)
                                                                   : 128u / (uint32_t)bps));
    const uint64_t area = (uint64_t)j.width * j.height;
    const uint64_t units = area / npix;
    // the constructors' checks (PanasonicV4Decompressor.cpp:49-90, V5 :58-116, V6 :146-176,
    // V7 :40-64)
    uint64_t need = units * 16;
    if (j.version == 5 || (j.version == 4 && j.section_split_offset != 0))
      need = ((units + 1023) / 1024) * 0x4000ull;
    const bool ok = vok && j.width > 0 && j.height > 0 && j.width % npix == 0 &&
                    j.in_size >= need && (j.out_offset % 2) == 0 && (j.out_pitch % 2) == 0 &&
                    (uint64_t)j.width * 2 <= j.out_pitch && area < 0xFFFF0000ull &&
                    (j.version != 4 || (j.section_split_offset <= 0x4000u && j.width <= 0xFFFFu &&
                                        j.height <= 0xFFFFu));
    if (!ok) {
      delete p;
      return set_err(ctx, RSB200_ERR_ARG, "pana job %d: malformed descriptor", i);
    }
    PanaJobDev d;
    memset(&d, 0, sizeof d);
    d.in_offset = j.in_offset;
    d.out_offset = j.out_offset;
    d.out_pitch = j.out_pitch;
    d.width = j.width;
    d.height = j.height;
    d.units = (uint32_t)units;
    p->pana_zero_slot.push_back(-1);
    if (j.version == 4) {
      d.split = j.section_split_offset;
      if (!j.zero_is_not_bad) {
        p->pana_zero_slot.back() = p->pana_zero_slots;
        d.zero_slot = (uint32_t)++p->pana_zero_slots;
      }
    }
    buckets[{(int)j.version, bps}].push_back(d);
    p->in_bytes += units * 16;
    p->out_bytes += area * 2;
    p->pixels += area;
    p->need_in = std::max<uint64_t>(p->need_in, sat_add(j.in_offset, need));
    p->need_out = std::max<uint64_t>(p->need_out, sat_add(j.out_offset, ((uint64_t)j.height - 1) * j.out_pitch +
                                                      2ull * j.width));
  }
  for (auto& kv : buckets) {
    PanaGroup g;
    g.version = kv.first.first;
    g.bps = kv.first.second;
    uint64_t n = 0;
    for (auto& d : kv.second) {
      d.unit_begin = (uint32_t)n;
      n += d.units;
    }
    if (n >= 0xFFFF0000ull) {
      rsb200_plan_destroy(p);
      return set_err(ctx, RSB200_ERR_ARG, "pana plan: too many blocks");
    }
    g.total_units = (uint32_t)n;
    g.njobs = (int)kv.second.size();
    cudaError_t e = rsb_dev_alloc(&g.d_jobs, sizeof(PanaJobDev) * kv.second.size());
    if (e == cudaSuccess)
      e = cudaMemcpy(g.d_jobs, kv.second.data(), sizeof(PanaJobDev) * kv.second.size(),
                     cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
      rsb200_plan_destroy(p);
      return set_err(ctx, RSB200_ERR_CUDA, "pana plan upload failed: %s", cudaGetErrorString(e));
    }
    p->pana_groups.push_back(g);
  }
  if (p->pana_zero_slots) {
    cudaError_t e = rsb_dev_alloc(&p->d_pana_zero_count, sizeof(uint32_t) * (size_t)p->pana_zero_slots);
    if (e == cudaSuccess)
      e = rsb_dev_alloc(&p->d_pana_zero_list,
                     sizeof(uint32_t) * (size_t)PANA_ZERO_CAP * (size_t)p->pana_zero_slots);
    if (e != cudaSuccess) {
      rsb200_plan_destroy(p);
      return set_err(ctx, RSB200_ERR_CUDA, "pana plan: bad-pixel lists: %s", cudaGetErrorString(e));
    }
  }
  p->launches_per_run = (int)p->pana_groups.size();
  *out = p;
  return RSB200_OK;
}

static_assert(PANA_ZERO_CAP == RSB200_PANA_BAD_CAP, "header and kernel disagree");

static cudaError_t run_pana_group(const rsb200_plan* p, const PanaGroup& g, const uint8_t* in,
                                  uint8_t* outp, cudaStream_t st) {
  const uint32_t nb = (g.total_units + PANA_NT - 1) / PANA_NT;
#define RSB_PANA(V, B)                                                                     \
  pana_kernel<V, B><<<nb, PANA_NT, 0, st>>>(in, outp, g.d_jobs, g.njobs, g.total_units,    \
                                            p->d_pana_zero_count, p->d_pana_zero_list)
  if (g.version == 4) {
    if (p->pana_zero_slots) {
      const cudaError_t e = cudaMemsetAsync(p->d_pana_zero_count, 0,
                                            sizeof(uint32_t) * (size_t)p->pana_zero_slots, st);
      if (e != cudaSuccess)
        return e;
    }
    RSB_PANA(4, 12);
  } else if (g.version == 5 && g.bps == 12)
    RSB_PANA(5, 12);
  else if (g.version == 5)
    RSB_PANA(5, 14);
  else if (g.version == 6 && g.bps == 12)
    RSB_PANA(6, 12);
  else if (g.version == 6)
    RSB_PANA(6, 14);
  else
    RSB_PANA(7, 14);
#undef RSB_PANA
  return cudaGetLastError();
}

// ------------------------------------------------------------------
// Sony ARW2 (K6)
// ------------------------------------------------------------------
extern "C" int rsb200_arw2_plan_create(rsb200_ctx* ctx, const rsb200_arw2_job* jobs, int njobs,
                                       const uint16_t* tables, int ntables, int dither,
                                       rsb200_plan** out) {
  if (!ctx || !jobs || njobs <= 0 || !out || ntables < 0 || (ntables > 0 && !tables))
    return set_err(ctx, RSB200_ERR_ARG, "arw2_plan_create: bad arguments");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  rsb200_plan* p = new (std::nothrow) rsb200_plan();
  if (!p)
    return RSB200_ERR_CUDA;
  p->ctx = ctx;
  p->kind = 4;
  p->nunits = njobs;
  std::vector<Arw2JobDev> dev((size_t)njobs);
  uint64_t groups = 0;
  bool any_table = false, any_plain = false;
  for (int i = 0; i < njobs; ++i) {
    const rsb200_arw2_job& j = jobs[i];
    // SonyArw2Decompressor ctor (SonyArw2Decompressor.cpp:41-56)
    const bool ok = j.width > 0 && j.height > 0 && j.width % 32 == 0 && j.width <= 9600 &&
                    j.height <= 6376 && (j.out_offset % 16) == 0 && (j.out_pitch % 16) == 0 &&
                    (uint64_t)j.width * 2 <= j.out_pitch && j.table < ntables;
    if (!ok) {
      delete p;
      return set_err(ctx, RSB200_ERR_ARG, "arw2 job %d: malformed descriptor", i);
    }
    (j.table >= 0 ? any_table : any_plain) = true;
    Arw2JobDev& d = dev[(size_t)i];
    d.in_offset = j.in_offset;
    d.out_offset = j.out_offset;
    d.out_pitch = j.out_pitch;
    d.width = j.width;
    d.height = j.height;
    d.groups_per_row = j.width / 32;
    d.group_begin = (uint32_t)groups;
    d.table = j.table;
    groups += (uint64_t)d.groups_per_row * j.height;
    const uint64_t px = (uint64_t)j.width * j.height;
    p->in_bytes += px;
    p->out_bytes += px * 2;
    p->pixels += px;
    p->need_in = std::max<uint64_t>(p->need_in, sat_add(j.in_offset, px));
    p->need_out = std::max<uint64_t>(p->need_out, sat_add(j.out_offset, ((uint64_t)j.height - 1) * j.out_pitch +
                                                      2ull * j.width));
  }
  if (any_table && any_plain) {
    delete p;
    return set_err(ctx, RSB200_ERR_ARG, "arw2 plan: jobs with and without a table cannot be mixed");
  }
  if (groups >= 0xFFFF0000ull) {
    delete p;
    return set_err(ctx, RSB200_ERR_ARG, "arw2 plan: too many blocks");
  }
  p->arw2_groups = (uint32_t)groups;
  p->arw2_mode = !any_table ? 0 : (dither ? 2 : 1);
  p->arw2_ntables = any_table ? ntables : 0;
  // the part of the tables a value can reach: entries 0 .. 4095
  std::vector<uint16_t> tcut;
  if (any_table) {
    const size_t per_in = dither ? 2u * 65536u : 65536u, per_out = dither ? 8192u : 4096u;
    tcut.resize(per_out * (size_t)ntables);
    for (int t = 0; t < ntables; ++t)
      memcpy(&tcut[per_out * (size_t)t], tables + per_in * (size_t)t, per_out * sizeof(uint16_t));
  }
  {
    // 15700^(32 g) mod m (one modular multiplication takes a thread to its 32 calls)
    static uint32_t jump[ARW2_MAX_GROUPS];
    uint64_t step = 1;
    for (int k = 0; k < 32; ++k)
      step = step * 15700ull % ARW2_M;
    uint64_t v = 1;
    for (int gq = 0; gq < ARW2_MAX_GROUPS; ++gq) {
      jump[gq] = (uint32_t)v;
      v = v * step % ARW2_M;
    }
    cudaError_t e = cudaMemcpyToSymbol(c_arw2_jump, jump, sizeof jump);
    if (e == cudaSuccess)
      e = rsb_dev_alloc(&p->d_arw2_jobs, sizeof(Arw2JobDev) * dev.size());
    if (e == cudaSuccess)
      e = cudaMemcpy(p->d_arw2_jobs, dev.data(), sizeof(Arw2JobDev) * dev.size(),
                     cudaMemcpyHostToDevice);
    if (e == cudaSuccess)
      e = rsb_dev_alloc(&p->d_arw2_tables, tcut.size() * sizeof(uint16_t) + 16);
    if (e == cudaSuccess && !tcut.empty())
      e = cudaMemcpy(p->d_arw2_tables, tcut.data(), tcut.size() * sizeof(uint16_t),
                     cudaMemcpyHostToDevice);
    if (e == cudaSuccess)
      e = rsb_dev_alloc(&p->d_arw2_bad, sizeof(uint32_t) * (size_t)njobs);
    if (e == cudaSuccess)
      e = rsb_host_alloc((void**)&p->h_arw2_bad, sizeof(uint32_t) * (size_t)njobs);
    if (e != cudaSuccess) {
      rsb200_plan_destroy(p);
      return set_err(ctx, RSB200_ERR_CUDA, "arw2 plan upload failed: %s", cudaGetErrorString(e));
    }
  }
  p->launches_per_run = 1;
  *out = p;
  return RSB200_OK;
}

static cudaError_t run_arw2(const rsb200_plan* p, const uint8_t* in, uint8_t* outp,
                            cudaStream_t st) {
  cudaError_t e = cudaMemsetAsync(p->d_arw2_bad, 0, sizeof(uint32_t) * (size_t)p->nunits, st);
  if (e != cudaSuccess)
    return e;
  const uint32_t per_cta = ARW2_NT * ARW2_GPT;
  const uint32_t nb = (p->arw2_groups + per_cta - 1) / per_cta;
  const bool sm = p->arw2_ntables == 1; // one table: staged in shared memory
#define RSB_ARW2(M, S)                                                                     \
  arw2_kernel<M, S><<<nb, ARW2_NT, 0, st>>>(in, outp, p->d_arw2_jobs, p->nunits,           \
                                            p->arw2_groups, p->d_arw2_tables, p->d_arw2_bad)
  if (p->arw2_mode == 0)
    RSB_ARW2(0, false);
  else if (p->arw2_mode == 1) {
    if (sm)
      RSB_ARW2(1, true);
    else
      RSB_ARW2(1, false);
  } else {
    if (sm)
      RSB_ARW2(2, true);
    else
      RSB_ARW2(2, false);
  }
#undef RSB_ARW2
  return cudaGetLastError();
}

static cudaError_t run_sraw_group(const SrawGroup& g, const uint8_t* in, uint8_t* outp,
                                  cudaStream_t st) {
  const uint32_t nb = (g.total_mcus + SRAW_NT - 1) / SRAW_NT;
#define RSB_SRAW(V, T)                                                                     \
  sraw_kernel<V, T><<<nb, SRAW_NT, 0, st>>>(in, outp, g.d_jobs, g.njobs, g.total_mcus)
  if (g.is420) {
    if (g.version == 1)
      RSB_SRAW(1, true);
    else
      RSB_SRAW(2, true);
  } else {
    if (g.version == 0)
      RSB_SRAW(0, false);
    else if (g.version == 1)
      RSB_SRAW(1, false);
    else
      RSB_SRAW(2, false);
  }
#undef RSB_SRAW
  return cudaGetLastError();
}

template <int BPS, bool LSBO>
static cudaError_t launch_unpack(const UnpackGroup& g, const uint8_t* in, uint64_t in_total,
                                 uint8_t* outp, cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(unpack_kernel<BPS, LSBO>,
                         cudaFuncAttributeMaxDynamicSharedMemorySize, UNPACK_SMEM_BYTES);
    attr_set = true;
  }
  unpack_kernel<BPS, LSBO><<<g.nblocks, UNPACK_THREADS, UNPACK_SMEM_BYTES, st>>>(
      in, in_total, outp, g.d_jobs, g.njobs);
  return cudaGetLastError();
}

static cudaError_t run_unpack_group(const UnpackGroup& g, const uint8_t* in,
                                    uint64_t in_total, uint8_t* outp, cudaStream_t st) {
#define RSB_CASE(B)                                                            \
  case B:                                                                      \
    return g.lsb ? launch_unpack<B, true>(g, in, in_total, outp, st)           \
                 : launch_unpack<B, false>(g, in, in_total, outp, st);
  switch (g.bps_t) {
    RSB_CASE(8)
    RSB_CASE(10)
    RSB_CASE(12)
    RSB_CASE(14)
    RSB_CASE(16)
  default:
    return g.lsb ? launch_unpack<0, true>(g, in, in_total, outp, st)
                 : launch_unpack<0, false>(g, in, in_total, outp, st);
  }
#undef RSB_CASE
}

template <int BPS, bool LSBO>
static cudaError_t launch_unpack_fast(const UnpackFastGroup& g, const uint8_t* in,
                                      uint8_t* outp, cudaStream_t st, uint32_t block_base = 0,
                                      uint32_t nblocks = 0) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(unpack_fast_kernel<BPS, LSBO>,
                         cudaFuncAttributeMaxDynamicSharedMemorySize, UNPACK_FAST_SMEM);
    attr_set = true;
  }
  unpack_fast_kernel<BPS, LSBO><<<nblocks ? nblocks : g.nblocks, UNPACK_THREADS,
                                  UNPACK_FAST_SMEM, st>>>(in, outp, g.d_jobs, g.njobs, block_base);
  return cudaGetLastError();
}

static cudaError_t run_unpack_fast_group(const UnpackFastGroup& g, const uint8_t* in,
                                         uint8_t* outp, cudaStream_t st,
                                         uint32_t block_base = 0, uint32_t nblocks = 0) {
#define RSB_CASE(B)                                                            \
  case B:                                                                      \
    return g.lsb ? launch_unpack_fast<B, true>(g, in, outp, st, block_base, nblocks) \
                 : launch_unpack_fast<B, false>(g, in, outp, st, block_base, nblocks);
  switch (g.bps) {
    RSB_CASE(8)
    RSB_CASE(10)
    RSB_CASE(12)
    RSB_CASE(14)
    RSB_CASE(16)
  default:
    return cudaErrorInvalidValue;
  }
#undef RSB_CASE
}

struct ScanBuild {
  std::vector<DevScan> scans;
  std::vector<DevStrip> strips;
  std::vector<K3RowRef> rows;
  uint64_t diff_elems = 0;
  uint64_t col_elems = 0;
};

constexpr uint32_t BIG_SEGMENT_BYTES = 256u << 10; // above this a segment gets several CTAs

// Segments the one-thread-per-segment kernel handles: plain LJPEG tiles whose rows
// are whole 8-sample units written with aligned 128-bit stores.
#ifndef RSB200_STREAM_DEFAULT
#define RSB200_STREAM_DEFAULT 1
#endif
// k2_stream_kernel: an L2 prefetch ahead of every sector is meant for launches too small to fill the
// machine (latency bound) and left out of full ones (it adds requests); the split, like the WIDE form of the
// full launches (a pair of units leaves as two back-to-back 128-bit stores), has not been measured on H100
constexpr size_t K2P_MAX_SEGMENTS = 0; // (k2_par_kernel: off by default until measured; RSB200_PAR_MAX / RSB200_LJPEG_PATH=par)
// half a wave: for sm_90a ptxas gives k2_stream_kernel 80 registers, so 6 CTAs of 128 threads fit an SM
constexpr int K2S_PREFETCH_CTAS_PER_SM = 3;
// k2_stream_kernel<true> (no prefetch, whole-sector stores) for launches of more than half a wave of
// thread-path segments, k2_stream_kernel<false> up to that; RSB200_STREAM_FORM overrides it
static bool stream_full_launch(const rsb200_ctx* ctx, const rsb200_plan* p) {
  if (p->stream_form)
    return p->stream_form == 2;
  const bool prefetch = p->nthread <= ctx->sm_count * K2S_PREFETCH_CTAS_PER_SM * T_NT;
  return !prefetch;
}
// the thread path needs enough independent segments to fill the machine (~22 frames of 726 tiles); this
// crossover has not been re-measured on H100
constexpr size_t K2T_MIN_SEGMENTS = 16384;
static bool thread_eligible(const DevScan& d) {
  return d.kind == 0 && d.pump == 0 && d.mcu_h == 1 &&
         (d.group == 1 || d.group == 2 || d.group == 4) && (d.row_samples & 7u) == 0 &&
         ((d.out_offset | d.out_pitch) & 15u) == 0 && (d.out_x & 7u) == 0;
}

// k2_par_kernel additionally needs one table for all components (the speculative parse does not
// know its component phase)
static bool par_eligible(const DevScan& d) {
  return thread_eligible(d) && !d.multi_table && d.n_samples >= 8 && d.in_size >= 8;
}

static int finish_ljpeg_plan(rsb200_ctx* ctx, rsb200_plan* p,
                             const rsb200_huff_table* tables, int ntables, ScanBuild& b,
                             bool /*unused*/) {
  std::vector<DevTable> ht((size_t)ntables);
  for (int i = 0; i < ntables; ++i)
    if (!build_dev_table(tables[i], ht[(size_t)i])) {
      delete p;
      return set_err(ctx, RSB200_ERR_ARG, "huffman table %d is malformed", i);
    }
  p->kind = 1;
  p->ntab_slots = 1;
  for (const DevScan& d : b.scans)
    for (int sl = 0; sl < 4; ++sl)
      if (d.table_idx[sl] >= 0)
        p->ntab_slots = std::max(p->ntab_slots, sl + 1);
  p->nscans = (int)b.scans.size();
  p->nunits = p->nscans;
  // classify the segments and lay out the scratch of the multi-CTA path
  std::vector<uint32_t> small_ids, big_ids, thread_ids, tile_ids;
  std::vector<DevTileParam> tile_prm;
  // K2T (one thread per segment) pays off once the launch holds enough independent
  // segments to fill the machine with serial decoders; RSB200_LJPEG_PATH=thread|fused
  // forces the choice (tests exercise both kernels on the same inputs).
  bool use_thread = false;
  if (ntables <= T_MAXTAB) {
    size_t n_el = 0;
    for (const DevScan& d : b.scans)
      if (d.kind == 0 && d.in_size <= BIG_SEGMENT_BYTES && thread_eligible(d))
        ++n_el;
    use_thread = n_el >= K2T_MIN_SEGMENTS;
    if (const char* e = getenv("RSB200_LJPEG_PATH")) {
      if (!strcmp(e, "thread") || !strcmp(e, "stream"))
        use_thread = true;
      else if (!strcmp(e, "fused") || !strcmp(e, "tile"))
        use_thread = false;
    }
  }
  // small launches: one CTA per segment on the clean stream (k2_par_kernel) when every plain
  // segment qualifies; RSB200_LJPEG_PATH=par forces it, RSB200_PAR_MAX moves the threshold (A/B)
  {
    size_t n_plain = 0, n_par = 0;
    for (const DevScan& d : b.scans)
      if (d.kind == 0 && d.in_size <= BIG_SEGMENT_BYTES) {
        ++n_plain;
        n_par += par_eligible(d) ? 1 : 0;
      }
    size_t par_max = K2P_MAX_SEGMENTS;
    if (const char* e = getenv("RSB200_PAR_MAX"))
      par_max = (size_t)atoll(e);
    p->use_par = ntables <= T_MAXTAB && n_plain > 0 && n_par == n_plain && n_plain <= par_max;
    if (const char* e = getenv("RSB200_LJPEG_PATH")) {
      if (!strcmp(e, "par"))
        p->use_par = ntables <= T_MAXTAB && n_par > 0;
      else
        p->use_par = false;
    }
    if (p->use_par)
      use_thread = true;
    if (const char* e = getenv("RSB200_PAR_CTAS"))
      p->par_ctas = std::max(0, std::min(8, atoi(e)));
  }
  // the thread path's kernel: k2_stream_kernel (raw bytes, unstuffed by the thread itself) or
  // k2_clean_kernel + k2_thread_kernel; RSB200_LJPEG_PATH=stream|thread forces one (tests run both)
  p->use_stream = RSB200_STREAM_DEFAULT != 0 && !p->use_par;
  if (const char* e = getenv("RSB200_THREAD_KERNEL"))
    p->use_stream = !strcmp(e, "stream");
  if (const char* e = getenv("RSB200_LJPEG_PATH")) {
    if (!strcmp(e, "stream"))
      p->use_stream = true;
    else if (!strcmp(e, "thread"))
      p->use_stream = false;
  }
  if (p->use_par)
    p->use_stream = false;
  // RSB200_STREAM_FORM=prefetch|wide fixes the form of k2_stream_kernel whatever the launch size
  // (stream_full_launch; tests run both forms on small batches)
  if (const char* e = getenv("RSB200_STREAM_FORM")) {
    if (!strcmp(e, "prefetch"))
      p->stream_form = 1;
    else if (!strcmp(e, "wide"))
      p->stream_form = 2;
  }
  // k2_tile_kernel<R> takes the plain single-table tiles; RSB200_LJPEG_PATH=fused keeps them on
  // k2_fused_kernel (tests run both), RSB200_TILE_R=1|2 picks the geometry, RSB200_TILE_PREROLL /
  // RSB200_TILE_NPIECES override the plan-time parameters (A/B runs)
  bool use_tile = true;
  int tile_r = 1, preroll_override = -1, npieces_override = 0;
  if (const char* e = getenv("RSB200_LJPEG_PATH"))
    if (!strcmp(e, "fused"))
      use_tile = false;
  if (const char* e = getenv("RSB200_TILE_R"))
    tile_r = atoi(e) == 2 ? 2 : 1;
  if (const char* e = getenv("RSB200_TILE_PREROLL"))
    preroll_override = atoi(e);
  if (const char* e = getenv("RSB200_TILE_NPIECES"))
    npieces_override = atoi(e);
  p->tile_r = tile_r;
  const int tile_min_rs = tile_r == 2 ? TileGeom<2>::MIN_RS : TileGeom<1>::MIN_RS;
  const int tile_npiece = tile_r == 2 ? TileGeom<2>::NPIECE : TileGeom<1>::NPIECE;
  const int tile_dcap = tile_r == 2 ? TileGeom<2>::DCAP : TileGeom<1>::DCAP;
  std::vector<BigScanInfo> big;
  std::vector<DevRange> ranges;
  b.rows.clear();
  b.diff_elems = 0;
  b.col_elems = 0;
  for (size_t i = 0; i < b.scans.size(); ++i) {
    DevScan& d = b.scans[i];
    const bool is_big = d.kind != 0 || d.in_size > BIG_SEGMENT_BYTES;
    if (is_big)
      (d.kind == 2 ? p->has_pentax : (d.kind == 3 ? p->has_nikon : p->has_k3)) = true;
    if (!is_big) {
      if (use_thread && (p->use_par ? par_eligible(d) : thread_eligible(d))) {
        thread_ids.push_back((uint32_t)i);
        if (p->use_par) { // differences in stream order (scratch), groups of 8
          d.diff_offset = b.diff_elems;
          b.diff_elems += (((uint64_t)d.rows * d.row_samples) + 7) & ~7ull;
        }
      } else if (use_tile && tile_eligible(d, tile_min_rs)) {
        DevTileParam tp;
        tile_params(d, tile_npiece, tile_dcap, preroll_override, tp.npieces, tp.preroll);
        if (npieces_override > 0)
          tp.npieces = (uint32_t)std::min(npieces_override, tile_npiece);
        tile_ids.push_back((uint32_t)i);
        tile_prm.push_back(tp);
      } else {
        small_ids.push_back((uint32_t)i);
      }
      continue;
    }
    big_ids.push_back((uint32_t)i);
    d.diff_offset = b.diff_elems;
    b.diff_elems += (((uint64_t)d.rows * d.row_samples) + 7) & ~7ull;
    d.col_offset = b.col_elems;
    b.col_elems += (uint64_t)d.rows * 4;
    d.row_begin = (uint32_t)b.rows.size();
    for (uint32_t r = 0; r < d.rows; ++r)
      b.rows.push_back(K3RowRef{(uint32_t)i, r});
    const uint32_t skew = (uint32_t)(d.in_offset & 15ull);
    const uint32_t range_bytes = (uint32_t)R_CHUNKS * F_RAW;
    const uint32_t nr = (skew + d.in_size + range_bytes - 1) / range_bytes;
    BigScanInfo bi;
    bi.scan = (uint32_t)i;
    bi.first_range = (uint32_t)ranges.size();
    bi.nranges = std::max(nr, 1u);
    bi.pad = 0;
    big.push_back(bi);
    for (uint32_t r = 0; r < bi.nranges; ++r)
      ranges.push_back(DevRange{(uint32_t)i, r});
  }
  p->nsmall = (int)small_ids.size();
  p->ntile = (int)tile_ids.size();
  // host-buffer runs of a plan made of tile-kernel segments only are pipelined: groups of
  // consecutive segments worth ~16 MB of output each (32 MB in plans of more than 1 GB): a download has a
  // fixed cost of tens of microseconds, so groups must be large, and small enough to overlap
  auto build_groups = [&](const std::vector<uint32_t>& ids) {
    uint64_t total = 0;
    for (uint32_t i : ids)
      total += (uint64_t)b.scans[i].rows * b.scans[i].store_w * 2;
    uint64_t kGroupOut = total > (1ull << 30) ? (32ull << 20) : (16ull << 20);
    if (const char* e = getenv("RSB200_GROUP_MB"))
      kGroupOut = (uint64_t)std::max(1, atoi(e)) << 20;
    rsb200_plan::TileGroup g{0, 0, ~0ull, 0, ~0ull, 0};
    uint64_t acc = 0;
    for (size_t k = 0; k < ids.size(); ++k) {
      const DevScan& d = b.scans[ids[k]];
      const uint64_t i0 = d.in_offset & ~15ull, i1 = (d.in_offset + d.in_size + 15) & ~15ull;
      const uint64_t o0 = d.out_offset + (uint64_t)d.out_y * d.out_pitch + 2ull * d.out_x;
      const uint64_t o1 = d.out_offset + ((uint64_t)d.out_y + d.rows - 1) * d.out_pitch +
                          2ull * ((uint64_t)d.out_x + d.store_w);
      g.in_lo = std::min(g.in_lo, i0);
      g.in_hi = std::max(g.in_hi, i1);
      g.out_lo = std::min(g.out_lo, o0);
      g.out_hi = std::max(g.out_hi, o1);
      ++g.count;
      acc += (uint64_t)d.rows * d.store_w * 2;
      if (acc >= kGroupOut || k + 1 == ids.size()) {
        p->tile_groups.push_back(g);
        g = rsb200_plan::TileGroup{(uint32_t)(k + 1), 0, ~0ull, 0, ~0ull, 0};
        acc = 0;
      }
    }
  };
  if (!tile_ids.empty() && small_ids.empty() && thread_ids.empty() && big_ids.empty())
    build_groups(tile_ids);
  // A plan on the thread path decodes device-resident input fastest with one thread per segment,
  // but a host-buffer run is bound by the PCIe link (2 B/px down at ~50 GB/s): there the tile
  // kernel, group by group between the upload and the download, hides the decode completely.
  if (!thread_ids.empty() && tile_ids.empty() && small_ids.empty() && big_ids.empty() && use_tile &&
      tile_r == 1 && !getenv("RSB200_NO_HOST_TILES")) {
    bool all = true;
    for (uint32_t i : thread_ids)
      all = all && tile_eligible(b.scans[i], TileGeom<1>::MIN_RS);
    if (all) {
      tile_ids = thread_ids;
      tile_prm.resize(tile_ids.size());
      for (size_t k = 0; k < tile_ids.size(); ++k)
        tile_params(b.scans[tile_ids[k]], TileGeom<1>::NPIECE, TileGeom<1>::DCAP, -1, tile_prm[k].npieces,
                    tile_prm[k].preroll);
      build_groups(tile_ids);
      p->host_tiles_only = true;
    }
  }
  p->h_in_size.resize(b.scans.size());
  for (size_t i = 0; i < b.scans.size(); ++i)
    p->h_in_size[i] = b.scans[i].kind == 0 ? b.scans[i].in_size : 0xFFFFFFFFu;
  p->nthread = (int)thread_ids.size();
  if (!thread_ids.empty()) {
    uint64_t bytes = 0;
    for (uint32_t i : thread_ids)
      bytes += b.scans[i].in_size;
    // the warp-per-segment pre-pass is the default: one CTA per small segment (k2_clean2_kernel) is
    // latency bound
    (void)bytes;
    p->clean2 = false;
    if (const char* e = getenv("RSB200_CLEAN"))
      p->clean2 = atoi(e) == 2;
  }
  p->ntables = ntables;
  p->nbig = (int)big_ids.size();
  p->nranges = (int)ranges.size();
  p->nrows = (uint32_t)b.rows.size();
  cudaError_t e = cudaSuccess;
  auto up = [&](void** dptr, const void* src, size_t bytes) {
    if (e != cudaSuccess)
      return;
    e = rsb_dev_alloc(dptr, bytes ? bytes : 16);
    if (e == cudaSuccess && bytes)
      e = cudaMemcpy(*dptr, src, bytes, cudaMemcpyHostToDevice);
  };
  auto alloc = [&](void** dptr, size_t bytes) {
    if (e == cudaSuccess)
      e = rsb_dev_alloc(dptr, bytes ? bytes : 16);
  };
  up((void**)&p->d_tables, ht.data(), sizeof(DevTable) * ht.size());
  up((void**)&p->d_scans, b.scans.data(), sizeof(DevScan) * b.scans.size());
  up((void**)&p->d_strips, b.strips.data(), sizeof(DevStrip) * b.strips.size());
  up((void**)&p->d_rows, b.rows.data(), sizeof(K3RowRef) * b.rows.size());
  up((void**)&p->d_small_ids, small_ids.data(), sizeof(uint32_t) * small_ids.size());
  {
    // k2_stream_kernel reads "the tile kernel can give this segment a second opinion" from bit 31
    std::vector<uint32_t> ids = thread_ids;
    if (p->use_stream)
      for (uint32_t& i : ids)
        if (tile_eligible(b.scans[i], TileGeom<1>::MIN_RS))
          i |= 0x80000000u;
    up((void**)&p->d_thread_ids, ids.data(), sizeof(uint32_t) * ids.size());
  }
  up((void**)&p->d_tile_ids, tile_ids.data(), sizeof(uint32_t) * tile_ids.size());
  up((void**)&p->d_tile_params, tile_prm.data(), sizeof(DevTileParam) * tile_prm.size());
  if (!thread_ids.empty()) {
    std::vector<DevTScan> tsc(thread_ids.size());
    uint64_t clean_words = 0, n_anchor = 0;
    for (size_t k = 0; k < thread_ids.size(); ++k) {
      const DevScan& d = b.scans[thread_ids[k]];
      const uint32_t skew = (uint32_t)(d.in_offset & 15ull);
      DevTScan t;
      t.clean_off = clean_words;
      t.cap_words = (((d.in_size + 15u) & ~15u) + 64u) / 4u;
      t.anchor_off = (uint32_t)n_anchor;
      t.n_anchor = ((skew + d.in_size) >> T_ANCHOR_SHIFT) + 1u;
      t.pad = tile_eligible(d, TileGeom<1>::MIN_RS) ? 1u : 0u; // may get the tile kernel's second opinion
      clean_words += t.cap_words;
      n_anchor += t.n_anchor;
      tsc[k] = t;
    }
    if (n_anchor >= (1ull << 32) && !p->use_stream)
      e = cudaErrorInvalidValue;
    if (!p->use_stream)
      up((void**)&p->d_tscans, tsc.data(), sizeof(DevTScan) * tsc.size());
    {
      std::vector<DevTileParam> tp(tsc.size());
      for (size_t k = 0; k < tsc.size(); ++k) {
        tile_params(b.scans[thread_ids[k]], TileGeom<1>::NPIECE, TileGeom<1>::DCAP, -1, tp[k].npieces,
                    tp[k].preroll);
        p->nthread_redo += tsc[k].pad ? 1 : 0;
      }
      up((void**)&p->d_thread_tile_params, tp.data(), sizeof(DevTileParam) * tp.size());
      alloc((void**)&p->d_redo, sizeof(uint32_t) * tsc.size());
    }
    if (!p->use_stream) {
      alloc((void**)&p->d_tinfos, sizeof(DevTInfo) * tsc.size());
      alloc((void**)&p->d_clean, clean_words * 4 + 256);
      alloc((void**)&p->d_anchors, n_anchor * 4 + 256);
    }
  }
  up((void**)&p->d_big_ids, big_ids.data(), sizeof(uint32_t) * big_ids.size());
  up((void**)&p->d_big, big.data(), sizeof(BigScanInfo) * big.size());
  up((void**)&p->d_ranges, ranges.data(), sizeof(DevRange) * ranges.size());
  alloc((void**)&p->d_states, sizeof(RangeState) * ranges.size());
  alloc((void**)&p->d_finals, sizeof(RangeFinal) * ranges.size());
  alloc((void**)&p->d_fallback, sizeof(uint32_t) * big.size());
  alloc((void**)&p->d_diffs, (b.diff_elems + 64) * sizeof(uint16_t));
  alloc((void**)&p->d_colvals, (b.col_elems + 64) * sizeof(uint16_t));
  alloc((void**)&p->d_results, sizeof(DevResult) * b.scans.size());
  if (e == cudaSuccess)
    e = rsb_host_alloc((void**)&p->h_results, sizeof(DevResult) * b.scans.size());
  if (p->has_pentax) {
    alloc((void**)&p->d_oob, sizeof(uint32_t) * b.scans.size());
    if (e == cudaSuccess)
      e = rsb_host_alloc((void**)&p->h_oob, sizeof(uint32_t) * b.scans.size());
  }
  if (e != cudaSuccess) {
    rsb200_plan_destroy(p);
    return set_err(ctx, RSB200_ERR_CUDA, "ljpeg plan allocation failed: %s",
                   cudaGetErrorString(e));
  }
  p->launches_per_run = (p->nsmall ? 1 : 0) + (p->ntile ? 1 : 0) + (p->nthread ? (p->use_stream ? 1 : 2) + (p->nthread_redo ? 1 : 0) : 0) +
                        (p->nbig ? 5 + (p->has_k3 ? 2 : 0) + (p->has_pentax ? 2 : 0) + (p->has_nikon ? 2 : 0) : 0);
  return RSB200_OK;
}

// ------------------------------------------------------------------
// Pentax: one long plain-MSB Huffman stream per image (K2R + K3P)
// ------------------------------------------------------------------
extern "C" int rsb200_pentax_plan_create(rsb200_ctx* ctx, const rsb200_huff_table* tables,
                                         int ntables, const rsb200_pentax_job* jobs, int njobs,
                                         rsb200_plan** out) {
  if (!ctx || !tables || ntables <= 0 || !jobs || njobs <= 0 || !out)
    return set_err(ctx, RSB200_ERR_ARG, "pentax_plan_create: bad arguments");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  rsb200_plan* p = new (std::nothrow) rsb200_plan();
  if (!p)
    return RSB200_ERR_CUDA;
  p->ctx = ctx;
  ScanBuild b;
  for (int i = 0; i < njobs; ++i) {
    const rsb200_pentax_job& j = jobs[i];
    // PentaxDecompressor ctor (PentaxDecompressor.cpp:55-67)
    const bool ok = j.width > 0 && j.height > 0 && j.width % 2 == 0 && j.width <= 8384 &&
                    j.height <= 6208 && (int)j.table < ntables && j.in_size < (1u << 28) &&
                    (uint64_t)j.width * 2 <= j.out_pitch && (j.out_offset % 4) == 0 &&
                    (j.out_pitch % 4) == 0;
    if (!ok) {
      delete p;
      return set_err(ctx, RSB200_ERR_ARG, "pentax job %d: malformed descriptor", i);
    }
    DevScan d;
    memset(&d, 0, sizeof d);
    d.in_offset = j.in_offset;
    d.in_size = j.in_size;
    d.row_samples = (uint32_t)j.width;
    d.rows = (uint32_t)j.height;
    d.n_samples = (uint32_t)j.width * (uint32_t)j.height;
    d.group = 2;
    d.ncomp = 2;
    d.kind = 2;
    d.pump = 1;
    d.pattern = PAT_PLAIN;
    const uint8_t tab[4] = {(uint8_t)j.table, (uint8_t)j.table, 0, 0};
    const uint8_t comp_of_pos[2] = {0, 1};
    assign_tables(d, tab, 2, comp_of_pos, 2);
    d.first_idx[0] = 0;
    d.first_idx[1] = 1;
    d.out_offset = j.out_offset;
    d.out_pitch = j.out_pitch;
    d.mcu_w = 2;
    d.mcu_h = 1;
    d.store_w = (uint32_t)j.width;
    b.scans.push_back(d);
    p->in_bytes += j.in_size;
    p->out_bytes += (uint64_t)j.width * j.height * 2;
    p->pixels += (uint64_t)j.width * j.height;
    p->need_in = std::max<uint64_t>(p->need_in, sat_add(j.in_offset, j.in_size));
    p->need_out = std::max<uint64_t>(p->need_out, sat_add(j.out_offset, ((uint64_t)j.height - 1) * j.out_pitch + 2ull * j.width));
  }
  int rc = finish_ljpeg_plan(ctx, p, tables, ntables, b, /*fused=*/false);
  if (rc != RSB200_OK)
    return rc;
  *out = p;
  return RSB200_OK;
}

// ------------------------------------------------------------------
// Nikon: one long plain-MSB Huffman stream per image (K2R + K3N)
// ------------------------------------------------------------------
extern "C" int rsb200_nikon_plan_create(rsb200_ctx* ctx, const rsb200_huff_table* tables,
                                        int ntables, const rsb200_nikon_job* jobs, int njobs,
                                        const uint16_t* luts, int nluts, rsb200_plan** out) {
  if (!ctx || !tables || ntables <= 0 || !jobs || njobs <= 0 || !out || nluts < 0 ||
      nluts > 254 || (nluts > 0 && !luts))
    return set_err(ctx, RSB200_ERR_ARG, "nikon_plan_create: bad arguments");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  rsb200_plan* p = new (std::nothrow) rsb200_plan();
  if (!p)
    return RSB200_ERR_CUDA;
  p->ctx = ctx;
  ScanBuild b;
  for (int i = 0; i < njobs; ++i) {
    const rsb200_nikon_job& j = jobs[i];
    // NikonDecompressor ctor (NikonDecompressor.cpp:478-489); BitStreamerMSB needs 4 bytes
    const bool ok = j.width > 0 && j.height > 0 && j.width % 2 == 0 && j.width <= 8288 &&
                    j.height <= 5520 && (int)j.table < ntables && j.in_size >= 4 &&
                    j.in_size < (1u << 28) && (uint64_t)j.width * 2 <= j.out_pitch &&
                    (j.out_offset % 4) == 0 && (j.out_pitch % 4) == 0 && j.lut < nluts;
    if (!ok) {
      delete p;
      return set_err(ctx, RSB200_ERR_ARG, "nikon job %d: malformed descriptor", i);
    }
    DevScan d;
    memset(&d, 0, sizeof d);
    d.in_offset = j.in_offset;
    d.in_size = j.in_size;
    d.row_samples = (uint32_t)j.width;
    d.rows = (uint32_t)j.height;
    d.n_samples = (uint32_t)j.width * (uint32_t)j.height;
    d.group = 2;
    d.ncomp = 2;
    d.kind = 3;
    d.pump = 1;
    d.pattern = PAT_PLAIN;
    d.pad0[0] = (uint8_t)(j.lut < 0 ? 0 : j.lut + 1);
    const uint8_t tab[4] = {(uint8_t)j.table, (uint8_t)j.table, 0, 0};
    const uint8_t comp_of_pos[2] = {0, 1};
    assign_tables(d, tab, 2, comp_of_pos, 2);
    d.first_idx[0] = 0;
    d.first_idx[1] = 1;
    for (int k = 0; k < 4; ++k)
      d.init_pred[k] = j.pup[k];
    d.out_offset = j.out_offset;
    d.out_pitch = j.out_pitch;
    d.mcu_w = 2;
    d.mcu_h = 1;
    d.store_w = (uint32_t)j.width;
    b.scans.push_back(d);
    p->in_bytes += j.in_size;
    p->out_bytes += (uint64_t)j.width * j.height * 2;
    p->pixels += (uint64_t)j.width * j.height;
    p->need_in = std::max<uint64_t>(p->need_in, sat_add(j.in_offset, j.in_size));
    p->need_out = std::max<uint64_t>(p->need_out, sat_add(j.out_offset, ((uint64_t)j.height - 1) * j.out_pitch + 2ull * j.width));
  }
  int rc = finish_ljpeg_plan(ctx, p, tables, ntables, b, /*fused=*/false);
  if (rc != RSB200_OK)
    return rc;
  {
    const size_t bytes = (size_t)nluts * 2u * 65536u * sizeof(uint16_t);
    cudaError_t e = rsb_dev_alloc((void**)&p->d_nikon_luts, bytes + 16);
    if (e == cudaSuccess && bytes)
      e = cudaMemcpy(p->d_nikon_luts, luts, bytes, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
      rsb200_plan_destroy(p);
      return set_err(ctx, RSB200_ERR_CUDA, "nikon plan upload failed: %s", cudaGetErrorString(e));
    }
  }
  *out = p;
  return RSB200_OK;
}

extern "C" int rsb200_ljpeg_plan_create(rsb200_ctx* ctx, const rsb200_huff_table* tables,
                                        int ntables, const rsb200_ljpeg_scan* scans,
                                        int nscans, rsb200_plan** out) {
  if (!ctx || !tables || ntables <= 0 || !scans || nscans <= 0 || !out)
    return set_err(ctx, RSB200_ERR_ARG, "ljpeg_plan_create: bad arguments");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  rsb200_plan* p = new (std::nothrow) rsb200_plan();
  if (!p)
    return RSB200_ERR_CUDA;
  p->ctx = ctx;
  ScanBuild b;
  b.scans.reserve((size_t)nscans);
  for (int i = 0; i < nscans; ++i) {
    const rsb200_ljpeg_scan& s = scans[i];
    const int group = s.mcu_w * s.mcu_h;
    DevScan d;
    // validation (every sum in 64 bits, out_offset 2-byte aligned) + descriptor: ljpeg_host.h
    if (!ljpeg_scan_to_dev(s, ntables, d)) {
      delete p;
      return set_err(ctx, RSB200_ERR_ARG, "ljpeg scan %d: malformed descriptor", i);
    }
    (void)group;
    d.diff_offset = b.diff_elems;
    b.diff_elems += ((uint64_t)d.n_samples + 7) & ~7ull;
    d.col_offset = b.col_elems;
    b.col_elems += (uint64_t)d.rows * 4;
    d.row_begin = (uint32_t)b.rows.size();
    for (uint32_t r = 0; r < d.rows; ++r)
      b.rows.push_back(K3RowRef{(uint32_t)i, r});
    b.scans.push_back(d);
    p->in_bytes += s.in_size;
    p->out_bytes += (uint64_t)s.rows * s.mcu_h * s.store_w * 2;
    p->pixels += (uint64_t)s.rows * s.mcu_h * s.store_w;
    p->need_in = std::max<uint64_t>(p->need_in, sat_add(s.in_offset, s.in_size));
    const uint64_t last_row = (uint64_t)s.out_y + (uint64_t)s.rows * s.mcu_h - 1;
    const uint64_t extent = last_row * s.out_pitch + 2ull * ((uint64_t)s.out_x + s.store_w);
    if (s.out_offset + extent < s.out_offset || s.in_offset + (uint64_t)s.in_size < s.in_offset) {
      delete p;
      return set_err(ctx, RSB200_ERR_ARG, "ljpeg scan %d: offset + extent overflows", i);
    }
    p->need_out = std::max<uint64_t>(p->need_out, sat_add(s.out_offset, extent));
  }
  int rc = finish_ljpeg_plan(ctx, p, tables, ntables, b, /*fused=*/true);
  if (rc != RSB200_OK)
    return rc;
  *out = p;
  return RSB200_OK;
}

// Vertical output strips of a CR2 frame, restating the slice iterators of
// Cr2DecompressorImpl.h:76-248 (slices in stream order -> output tiles clamped
// to the image height -> vertically adjacent tiles coalesced).
static bool cr2_strips(int dimX /*groups*/, int dimY, int frameY, int numSlices,
                       int sliceW, int lastSliceW, std::vector<DevStrip>& out) {
  int sliceId = 0, sliceRow = 0, px = 0, py = 0;
  uint32_t g = 0;
  bool done = false;
  while (sliceId < numSlices && !done) {
    const int w = (sliceId + 1 == numSlices) ? lastSliceW : sliceW;
    const int h = std::min(dimY - py, frameY - sliceRow);
    if (w <= 0 || h <= 0)
      return false;
    if (px + w > dimX || py + h > dimY)
      return false;
    if (!out.empty() && out.back().x == px && out.back().w == w &&
        out.back().y + out.back().h == py) {
      out.back().h += h; // ContinuesColumn
    } else {
      if (!out.empty() && !(py == 0 && px == out.back().x + out.back().w))
        return false; // invalid tiling
      out.push_back(DevStrip{g, px, py, w, h});
    }
    g += (uint32_t)w * (uint32_t)h;
    if (px + w == dimX && py + h == dimY)
      done = true;
    sliceRow += h;
    py += h;
    if (sliceRow == frameY) {
      ++sliceId;
      sliceRow = 0;
    }
    if (py == dimY) {
      py = 0;
      px += w;
    }
  }
  return done;
}

extern "C" int rsb200_cr2_plan_create(rsb200_ctx* ctx, const rsb200_huff_table* tables,
                                      int ntables, const rsb200_cr2_job* jobs, int njobs,
                                      rsb200_plan** out) {
  if (!ctx || !tables || ntables <= 0 || !jobs || njobs <= 0 || !out)
    return set_err(ctx, RSB200_ERR_ARG, "cr2_plan_create: bad arguments");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  rsb200_plan* p = new (std::nothrow) rsb200_plan();
  if (!p)
    return RSB200_ERR_CUDA;
  p->ctx = ctx;
  ScanBuild b;
  for (int i = 0; i < njobs; ++i) {
    const rsb200_cr2_job& j = jobs[i];
    const bool sub = (j.x_s_f != 1 || j.y_s_f != 1);
    const bool fmt_ok = (j.n_comp == 2 && !sub) || (j.n_comp == 4 && !sub) ||
                        (j.n_comp == 3 && j.x_s_f == 2 && (j.y_s_f == 1 || j.y_s_f == 2));
    // Dsc (Cr2DecompressorImpl.h:250-275)
    const int pixelsPerGroup = j.x_s_f * j.y_s_f;
    const int groupSize = !sub ? j.n_comp : 2 + pixelsPerGroup;
    const int sliceColStep = j.n_comp * j.x_s_f;
    bool ok = fmt_ok && j.img_w > 0 && j.img_h > 0 && j.img_w % groupSize == 0 &&
              j.frame_w > 0 && j.frame_h > 0 && j.frame_w % j.x_s_f == 0 &&
              j.frame_h % j.y_s_f == 0 && j.num_slices >= 1 &&
              j.last_slice_w > 0 && (j.num_slices == 1 || j.slice_w > 0) &&
              j.slice_w % sliceColStep == 0 && j.last_slice_w % sliceColStep == 0 &&
              (uint64_t)j.img_w * 2 <= j.out_pitch && j.in_size < (1u << 28);
    for (int c = 0; ok && c < j.n_comp; ++c)
      ok = j.table[c] < ntables;
    DevScan d;
    memset(&d, 0, sizeof d);
    if (ok) {
      const int dimX = j.img_w / groupSize, dimY = j.img_h;
      const int frameX = j.frame_w / j.x_s_f, frameY = j.frame_h / j.y_s_f;
      ok = (uint64_t)frameX * frameY >= (uint64_t)dimX * dimY;
      d.strip_begin = (uint32_t)b.strips.size();
      if (ok)
        ok = cr2_strips(dimX, dimY, frameY, j.num_slices, j.slice_w / sliceColStep,
                        j.last_slice_w / sliceColStep, b.strips);
      d.n_strips = (uint16_t)(b.strips.size() - d.strip_begin);
      const uint64_t total_groups = (uint64_t)dimX * dimY;
      d.row_samples = (uint32_t)frameX * (uint32_t)groupSize;
      d.rows = (uint32_t)((total_groups + frameX - 1) / frameX);
      d.n_samples = (uint32_t)(total_groups * groupSize);
      ok = ok && total_groups * groupSize < (1ull << 32);
    }
    if (!ok) {
      delete p;
      return set_err(ctx, RSB200_ERR_ARG, "cr2 job %d: malformed descriptor", i);
    }
    d.in_offset = j.in_offset;
    d.in_size = j.in_size;
    d.group = (uint8_t)groupSize;
    d.ncomp = j.n_comp;
    d.kind = 1;
    d.pattern = !sub ? PAT_PLAIN : (j.y_s_f == 1 ? PAT_H2V1 : PAT_H2V2);
    uint8_t comp_of_pos[12];
    for (int q = 0; q < groupSize; ++q)
      comp_of_pos[q] = (uint8_t)(!sub ? q : (q < pixelsPerGroup ? 0 : q - pixelsPerGroup + 1));
    assign_tables(d, j.table, j.n_comp, comp_of_pos, groupSize);
    for (int c = 0; c < j.n_comp; ++c) {
      d.first_idx[c] = (uint8_t)(c == 0 ? 0 : groupSize - (j.n_comp - c));
      d.init_pred[c] = j.init_pred[c];
    }
    d.out_offset = j.out_offset;
    d.out_pitch = j.out_pitch;
    d.mcu_w = (uint8_t)groupSize;
    d.mcu_h = 1;
    d.store_w = (uint32_t)j.img_w;
    d.diff_offset = b.diff_elems;
    b.diff_elems += (((uint64_t)d.rows * d.row_samples) + 7) & ~7ull;
    d.col_offset = b.col_elems;
    b.col_elems += (uint64_t)d.rows * 4;
    d.row_begin = (uint32_t)b.rows.size();
    for (uint32_t r = 0; r < d.rows; ++r)
      b.rows.push_back(K3RowRef{(uint32_t)i, r});
    b.scans.push_back(d);
    p->in_bytes += j.in_size;
    p->out_bytes += (uint64_t)j.img_w * j.img_h * 2;
    p->pixels += (uint64_t)j.img_w * j.img_h;
    p->need_in = std::max<uint64_t>(p->need_in, sat_add(j.in_offset, j.in_size));
    p->need_out = std::max<uint64_t>(p->need_out, sat_add(j.out_offset, ((uint64_t)j.img_h - 1) * j.out_pitch + 2ull * j.img_w));
  }
  int rc = finish_ljpeg_plan(ctx, p, tables, ntables, b, /*fused=*/false);
  if (rc != RSB200_OK)
    return rc;
  *out = p;
  return RSB200_OK;
}

// ------------------------------------------------------------------
// execution
// ------------------------------------------------------------------
namespace {
struct DeviceGuard {
  int prev = -1;
  bool changed = false, ok = true;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess)
      prev = -1;
    if (prev != dev) {
      ok = cudaSetDevice(dev) == cudaSuccess;
      changed = ok;
    }
  }
  ~DeviceGuard() {
    if (changed && prev >= 0)
      cudaSetDevice(prev);
  }
};
} // namespace

extern "C" int rsb200_plan_run(rsb200_plan* p, const void* d_in, size_t in_bytes,
                               void* d_out, size_t out_bytes, void* stream) {
  if (!p || !d_out || (!d_in && p->need_in))
    return RSB200_ERR_ARG;
  rsb200_ctx* ctx = p->ctx;
  if (in_bytes < p->need_in || out_bytes < p->need_out)
    return set_err(ctx, RSB200_ERR_ARG,
                   "plan_run: buffers too small (in %zu < %llu or out %zu < %llu)",
                   in_bytes, (unsigned long long)p->need_in, out_bytes,
                   (unsigned long long)p->need_out);
  if ((reinterpret_cast<uintptr_t>(d_in) & 15) || (reinterpret_cast<uintptr_t>(d_out) & 15))
    return set_err(ctx, RSB200_ERR_ARG, "plan_run: device pointers must be 16-byte aligned");
  // launches go to the plan's device whatever the caller's current device is (restored on return)
  DeviceGuard guard(ctx->device);
  if (!guard.ok)
    return set_err(ctx, RSB200_ERR_CUDA, "plan_run: cannot select device %d", ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  const uint8_t* in = (const uint8_t*)d_in;
  uint8_t* outp = (uint8_t*)d_out;
  if (p->kind == 0) {
    for (const UnpackFastGroup& g : p->fast_groups) {
      if (!g.nblocks)
        continue;
      CUDA_TRY(ctx, run_unpack_fast_group(g, in, outp, st));
      ctx->launches++;
    }
    for (const UnpackGroup& g : p->groups) {
      if (!g.nblocks)
        continue;
      CUDA_TRY(ctx, run_unpack_group(g, in, (uint64_t)in_bytes, outp, st));
      ctx->launches++;
    }
  } else if (p->kind == 10) {
    const uint32_t nbs = (uint32_t)(((uint64_t)p->lookup_quads * p->lookup_nseg + LUT_WARPS - 1) / LUT_WARPS);
    if (p->lookup_smem && !p->lookup_dither && p->lookup_ntables == 1) {
      const int sms = ctx->sm_count;
      lookup_smem_kernel<<<(unsigned)std::max(1, sms), LUT_SMEM_NT, LUT_SMEM_BYTES, st>>>(
          outp, p->d_lookup_jobs, p->lookup_njobs, p->lookup_quads, p->d_lookup_tables);
    } else if (p->lookup_dither)
      lookup_kernel<true><<<nbs, LUT_NT, 0, st>>>(outp, p->d_lookup_jobs, p->lookup_njobs, p->lookup_quads,
                                                  p->d_lookup_tables, p->lookup_nseg);
    else
      lookup_kernel<false><<<nbs, LUT_NT, 0, st>>>(outp, p->d_lookup_jobs, p->lookup_njobs, p->lookup_quads,
                                                   p->d_lookup_tables, p->lookup_nseg);
    CUDA_TRY(ctx, cudaGetLastError());
    ctx->launches++;
  } else if (p->kind == 9) {
    if (p->badpix_total) {
      badpix_kernel<<<(p->badpix_total + BADPIX_NT - 1) / BADPIX_NT, BADPIX_NT, 0, st>>>(
          outp, p->d_badpix_jobs, p->badpix_njobs, p->d_badpix_list, p->badpix_total, p->d_badpix_maps);
      CUDA_TRY(ctx, cudaGetLastError());
      ctx->launches++;
    }
  } else if (p->kind == 8) {
    if (p->pana_zero_slots)
      CUDA_TRY(ctx, cudaMemsetAsync(p->d_pana_zero_count, 0,
                                    sizeof(uint32_t) * (size_t)p->pana_zero_slots, st));
    if (p->dngop_units) {
      dngop_kernel<<<(p->dngop_units + DNGOP_NT - 1) / DNGOP_NT, DNGOP_NT, 0, st>>>(
          outp, p->d_dngop_jobs, p->dngop_njobs, p->dngop_units, p->d_dngop_ops, p->d_dngop_tables,
          p->d_dngop_deltas, p->d_pana_zero_count, p->d_pana_zero_list);
      CUDA_TRY(ctx, cudaGetLastError());
      ctx->launches++;
    }
  } else if (p->kind == 7) {
    for (const ScaleGroup& g : p->scale_groups) {
      const uint32_t nb = (g.total_quads + SCALE_WARPS - 1) / SCALE_WARPS;
      if (g.mode == 0)
        scale_kernel<0><<<nb, SCALE_NT, 0, st>>>(outp, g.d_jobs, g.njobs, g.total_quads, 1u);
      else
        scale_kernel<1><<<(uint32_t)(((uint64_t)g.total_quads * g.nseg + SCALE_WARPS - 1) / SCALE_WARPS), SCALE_NT,
                          0, st>>>(outp, g.d_jobs, g.njobs, g.total_quads, g.nseg);
      CUDA_TRY(ctx, cudaGetLastError());
      ctx->launches++;
    }
  } else if (p->kind == 11) {
    CUDA_TRY(ctx, run_hasselblad(p, in, outp, st));
    ctx->launches += (uint64_t)p->launches_per_run;
  } else if (p->kind == 6) {
    CUDA_TRY(ctx, run_phaseone(p, in, outp, st));
    ctx->launches++;
  } else if (p->kind == 5) {
    for (const PanaGroup& g : p->pana_groups) {
      CUDA_TRY(ctx, run_pana_group(p, g, in, outp, st));
      ctx->launches++;
    }
  } else if (p->kind == 4) {
    CUDA_TRY(ctx, run_arw2(p, in, outp, st));
    ctx->launches++;
  } else if (p->kind == 3) {
    for (const SrawGroup& g : p->sraw_groups) {
      CUDA_TRY(ctx, run_sraw_group(g, in, outp, st));
      ctx->launches++;
    }
  } else if (p->kind == 2) {
    for (const RawGroup& g : p->raw_groups) {
      if (!g.total_items)
        continue;
      CUDA_TRY(ctx, run_raw_group(g, in, (uint64_t)in_bytes, outp, p->d_raw_tables, st));
      ctx->launches++;
    }
  } else {
    const size_t fsm = fused_smem_bytes(p->ntab_slots);
    if (p->ntile) {
      if (p->tile_r == 2)
        k2_tile_kernel<2><<<p->ntile, TL_NT, tile_smem_bytes<2>(), st>>>(
            in, (uint64_t)in_bytes, p->d_scans, p->d_tables, outp, p->d_results, p->d_tile_ids,
            p->d_tile_params, nullptr);
      else
        k2_tile_kernel<1><<<p->ntile, TL_NT, tile_smem_bytes<1>(), st>>>(
            in, (uint64_t)in_bytes, p->d_scans, p->d_tables, outp, p->d_results, p->d_tile_ids,
            p->d_tile_params, nullptr);
      CUDA_TRY(ctx, cudaGetLastError());
      ctx->launches += 1;
    }
    if (p->nsmall) {
      k2_fused_kernel<<<p->nsmall, F_NT, fsm, st>>>(in, (uint64_t)in_bytes, p->d_scans,
                                                     p->d_tables, outp, p->d_results,
                                                     p->d_small_ids);
      CUDA_TRY(ctx, cudaGetLastError());
      ctx->launches += 1;
    }
    if (p->nthread && p->use_stream) {
      // small launches are latency bound (L2 prefetch ahead, 128-bit stores), full ones are bound
      // by the number of memory requests (no prefetch, whole-sector stores)
      if (!stream_full_launch(ctx, p))
        k2_stream_kernel<false><<<(p->nthread + T_NT - 1) / T_NT, T_NT, stream_smem_bytes(p->ntables), st>>>(
            in, (uint64_t)in_bytes, p->d_scans, p->d_tables, p->ntables, outp, p->d_results,
            p->d_thread_ids, (uint32_t)p->nthread, p->d_redo, 1);
      else
        k2_stream_kernel<true><<<(p->nthread + T_NT - 1) / T_NT, T_NT, stream_smem_bytes(p->ntables), st>>>(
            in, (uint64_t)in_bytes, p->d_scans, p->d_tables, p->ntables, outp, p->d_results,
            p->d_thread_ids, (uint32_t)p->nthread, p->d_redo, 0);
      CUDA_TRY(ctx, cudaGetLastError());
      ctx->launches += 1;
    } else if (p->nthread && p->use_par) {
      k2_clean_kernel<<<(p->nthread + C_WARPS - 1) / C_WARPS, 32 * C_WARPS, 0, st>>>(
          in, (uint64_t)in_bytes, p->d_scans, p->d_thread_ids, (uint32_t)p->nthread, p->d_tscans,
          p->d_clean, p->d_anchors, p->d_tinfos);
      k2_par_kernel<<<p->par_ctas > 0 ? std::min(p->nthread, ctx->sm_count * p->par_ctas) : p->nthread, P_NT, 0, st>>>(
          in, p->d_scans, p->d_tables, outp, p->d_results, p->d_thread_ids, (uint32_t)p->nthread, p->d_tscans,
          p->d_tinfos, p->d_clean, p->d_anchors, p->d_diffs, p->d_redo);
      CUDA_TRY(ctx, cudaGetLastError());
      ctx->launches += 2;
    } else if (p->nthread) {
      // unstuffing pre-pass: one CTA per segment with the tile kernel's stage B for DNG-size
      // segments (k2_clean2_kernel), one warp per segment for small ones (k2_clean_kernel)
      if (p->clean2)
        k2_clean2_kernel<<<p->nthread, TL_NT, tile_smem_bytes<1>(), st>>>(
            in, (uint64_t)in_bytes, p->d_scans, p->d_thread_ids, (uint32_t)p->nthread, p->d_tscans,
            p->d_clean, p->d_anchors, p->d_tinfos);
      else
      k2_clean_kernel<<<(p->nthread + C_WARPS - 1) / C_WARPS, 32 * C_WARPS, 0, st>>>(
          in, (uint64_t)in_bytes, p->d_scans, p->d_thread_ids, (uint32_t)p->nthread, p->d_tscans,
          p->d_clean, p->d_anchors, p->d_tinfos);
      k2_thread_kernel<<<(p->nthread + T_NT - 1) / T_NT, T_NT, thread_smem_bytes(p->ntables), st>>>(
          in, p->d_scans, p->d_tables, p->ntables, outp, p->d_results, p->d_thread_ids,
          (uint32_t)p->nthread, p->d_tscans, p->d_tinfos, p->d_clean, p->d_anchors, p->d_redo);
      CUDA_TRY(ctx, cudaGetLastError());
      ctx->launches += 2;
    }
    if (p->nthread) {
      if (p->nthread_redo) {
        // exact end-of-stream semantics for the segments K2T flagged (CTAs of the others exit at once)
        k2_tile_kernel<1><<<p->nthread, TL_NT, tile_smem_bytes<1>(), st>>>(
            in, (uint64_t)in_bytes, p->d_scans, p->d_tables, outp, p->d_results, p->d_thread_ids,
            p->d_thread_tile_params, p->d_redo);
        CUDA_TRY(ctx, cudaGetLastError());
        ctx->launches += 1;
      }
    }
    if (p->nbig) {
      k2_clear_results_kernel<<<(p->nbig + 127) / 128, 128, 0, st>>>(p->d_big, p->nbig,
                                                                     p->d_results, p->d_oob);
      k2_range_count_kernel<<<p->nranges, F_NT, fsm, st>>>(in, (uint64_t)in_bytes, p->d_scans,
                                                           p->d_tables, p->d_ranges, p->d_states);
      k2_range_verify_kernel<<<p->nbig, V_NT, 0, st>>>(p->d_scans, p->d_big, p->d_states,
                                                       p->d_finals, p->d_fallback);
      k2_range_diffs_kernel<<<p->nranges, F_NT, fsm, st>>>(in, (uint64_t)in_bytes, p->d_scans,
                                                           p->d_tables, p->d_ranges, p->d_finals,
                                                           p->d_diffs, p->d_results);
      // exact redo of segments whose speculative parse failed verification (no-op otherwise)
      k2_entropy_kernel<<<p->nbig, K2_THREADS, sizeof(K2Shared), st>>>(
          in, (uint64_t)in_bytes, p->d_scans, p->d_tables, p->d_diffs, p->d_results,
          p->d_big_ids, p->d_fallback);
      const int col_warps = p->nbig * 4;
      const uint32_t rows_per_block = K3_THREADS / 32;
      int nk3 = 0;
      if (p->has_k3) {
        k3_column_kernel<<<(col_warps * 32 + 127) / 128, 128, 0, st>>>(
            p->d_scans, p->d_big_ids, p->nbig, p->d_diffs, p->d_colvals);
        k3_row_kernel<<<(p->nrows + rows_per_block - 1) / rows_per_block, K3_THREADS, 0, st>>>(
            p->d_scans, p->d_rows, p->nrows, p->d_diffs, p->d_colvals, p->d_strips, outp);
        nk3 += 2;
      }
      if (p->has_pentax) {
        k3p_column_kernel<<<(col_warps * 32 + 127) / 128, 128, 0, st>>>(
            p->d_scans, p->d_big_ids, p->nbig, p->d_diffs, p->d_colvals, p->d_oob);
        k3p_row_kernel<<<(p->nrows + rows_per_block - 1) / rows_per_block, K3_THREADS, 0, st>>>(
            p->d_scans, p->d_rows, p->nrows, p->d_diffs, p->d_colvals, outp, p->d_oob);
        nk3 += 2;
      }
      if (p->has_nikon) {
        k3n_column_kernel<<<(col_warps * 32 + 127) / 128, 128, 0, st>>>(
            p->d_scans, p->d_big_ids, p->nbig, p->d_diffs, p->d_colvals);
        k3n_row_kernel<<<(p->nrows + rows_per_block - 1) / rows_per_block, K3_THREADS, 0, st>>>(
            in, p->d_scans, p->d_rows, p->nrows, p->d_diffs, p->d_colvals, p->d_nikon_luts, outp);
        nk3 += 2;
      }
      CUDA_TRY(ctx, cudaGetLastError());
      ctx->launches += 5 + nk3;
    }
  }
  p->last_stream = st;
  p->ran = true;
  return RSB200_OK;
}

static int ensure_cap(rsb200_ctx* ctx, uint8_t** buf, size_t* cap, size_t need) {
  need = (need + 255) & ~(size_t)255;
  if (*cap >= need)
    return RSB200_OK;
  if (*buf)
    cudaFree(*buf);
  *buf = nullptr;
  *cap = 0;
  CUDA_TRY(ctx, cudaMalloc((void**)buf, need + 256));
  *cap = need;
  return RSB200_OK;
}

// A batch of packed frames (one job per frame, disjoint input and output spans):
// job j's H2D copy, kernel and D2H copy are chained on stream j % 3, so the
// upload of the next frame and the download of the previous one overlap the
// unpack of the current one (both PCIe directions busy).
static bool unpack_pipeline_ok(const rsb200_plan* p) {
  if (p->kind != 0 || !p->groups.empty() || p->fast_groups.size() != 1)
    return false;
  const auto& jobs = p->fast_groups[0].h_jobs;
  if (jobs.size() < 2)
    return false;
  for (size_t j = 0; j + 1 < jobs.size(); ++j) {
    const uint64_t in_end = jobs[j].in_offset + (uint64_t)jobs[j].rows * jobs[j].in_pitch;
    const uint64_t out_end = jobs[j].out_offset +
                             (uint64_t)(jobs[j].row0 + jobs[j].rows) * jobs[j].out_pitch;
    if (in_end > jobs[j + 1].in_offset || out_end > jobs[j + 1].out_offset)
      return false;
  }
  return true;
}

static int run_host_unpack_pipelined(rsb200_plan* p, const uint8_t* in, size_t in_bytes,
                                     uint8_t* out, size_t out_bytes) {
  rsb200_ctx* ctx = p->ctx;
  const UnpackFastGroup& g = p->fast_groups[0];
  for (size_t j = 0; j < g.h_jobs.size(); ++j) {
    const UnpackFastJobDev& jb = g.h_jobs[j];
    cudaStream_t st = ctx->pipe[j % N_PIPE];
    const uint64_t i0 = jb.in_offset & ~15ull;
    uint64_t i1 = jb.in_offset + (uint64_t)jb.rows * jb.in_pitch;
    i1 = std::min<uint64_t>((i1 + 15) & ~15ull, in_bytes);
    const uint64_t o0 = jb.out_offset + (uint64_t)jb.row0 * jb.out_pitch;
    const uint64_t o1 = std::min<uint64_t>(o0 + (uint64_t)jb.rows * jb.out_pitch, out_bytes);
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_in + i0, in + i0, i1 - i0, cudaMemcpyHostToDevice, st));
    const uint32_t nb = (jb.total_items + UNPACK_IPB - 1) / UNPACK_IPB;
    CUDA_TRY(ctx, run_unpack_fast_group(g, ctx->d_in, ctx->d_out, st, jb.block_begin, nb));
    ctx->launches++;
    CUDA_TRY(ctx, cudaMemcpyAsync(out + o0, ctx->d_out + o0, o1 - o0, cudaMemcpyDeviceToHost, st));
  }
  for (int i = 0; i < N_PIPE; ++i)
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->pipe[i]));
  p->last_stream = ctx->pipe[0];
  p->ran = true;
  return RSB200_OK;
}

// ---- host buffers that are not page-locked ----
// cudaMemcpyAsync from / to pageable memory is staged by the driver on one thread (~9 GB/s
// measured: 15 ms for the 137 MB of a 45 MP frame).  The library stages such buffers itself
// through its own pinned memory with several copying threads, slice by slice, overlapped with the
// transfers and the kernels.
constexpr size_t STAGE_LIMIT = 768ull << 20; // beyond this the driver's path is used
static bool host_is_pageable(const void* ptr) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, ptr) != cudaSuccess) {
    cudaGetLastError();
    return true;
  }
  return a.type == cudaMemoryTypeUnregistered;
}
static int copy_threads(size_t bytes) {
  int nt = (int)std::min<size_t>(12, bytes / (1ull << 20));
  if (const char* e = getenv("RSB200_COPY_THREADS"))
    nt = std::max(1, atoi(e));
  return std::max(nt, 1);
}
// (OpenMP: a persistent team -- spawning threads per call costs more than the copies)
static void parallel_copy(uint8_t* dst, const uint8_t* src, size_t n) {
  const long kSlice = 1l << 20;
  const long ns = (long)((n + kSlice - 1) / kSlice);
  const int nt = copy_threads(n);
  if (nt <= 1 || ns <= 1) {
    memcpy(dst, src, n);
    return;
  }
#pragma omp parallel for num_threads(nt) schedule(static)
  for (long i = 0; i < ns; ++i) {
    const size_t a = (size_t)i * kSlice, b2 = std::min(n, a + (size_t)kSlice);
    memcpy(dst + a, src + a, b2 - a);
  }
}
// rows of row_bytes out of a pitch-strided source into a pitch-strided destination
static void parallel_copy_rows(uint8_t* dst, const uint8_t* src, size_t pitch, size_t row_bytes,
                               size_t rows) {
  if (row_bytes == pitch) {
    parallel_copy(dst, src, pitch * rows);
    return;
  }
  const int nt = copy_threads(row_bytes * rows);
#pragma omp parallel for num_threads(nt) schedule(static) if (nt > 1)
  for (long r = 0; r < (long)rows; ++r)
    memcpy(dst + (size_t)r * pitch, src + (size_t)r * pitch, row_bytes);
}
static int ensure_host_cap(rsb200_ctx* ctx, uint8_t** buf, size_t* cap, size_t need) {
  need = (need + 4095) & ~(size_t)4095;
  if (*cap >= need)
    return RSB200_OK;
  if (*buf)
    cudaFreeHost(*buf);
  *buf = nullptr;
  *cap = 0;
  CUDA_TRY(ctx, cudaHostAlloc((void**)buf, need + 4096, cudaHostAllocDefault));
  *cap = need;
  return RSB200_OK;
}

static cudaError_t launch_tile_range(const rsb200_plan* p, const uint8_t* d_in, uint64_t in_bytes,
                                     uint8_t* d_out, uint32_t first, uint32_t count,
                                     cudaStream_t st) {
  if (p->tile_r == 2)
    k2_tile_kernel<2><<<count, TL_NT, tile_smem_bytes<2>(), st>>>(
        d_in, in_bytes, p->d_scans, p->d_tables, d_out, p->d_results, p->d_tile_ids + first,
        p->d_tile_params + first, nullptr);
  else
    k2_tile_kernel<1><<<count, TL_NT, tile_smem_bytes<1>(), st>>>(
        d_in, in_bytes, p->d_scans, p->d_tables, d_out, p->d_results, p->d_tile_ids + first,
        p->d_tile_params + first, nullptr);
  return cudaGetLastError();
}

// LJPEG plan made of tile-kernel segments only: group g's upload, kernel and download are chained
// on stream g % 3, so the upload of the next group and the download of the previous one overlap
// the decode of the current one.  Spans of neighbouring groups may overlap (tiles of one tile row
// in two groups): every byte's last download happens after its last write, whatever the order.
static int run_host_tile_pipelined(rsb200_plan* p, const uint8_t* in, size_t in_bytes,
                                   uint8_t* out, size_t out_bytes, uint32_t pitch = 0,
                                   uint32_t row_bytes = 0) {
  rsb200_ctx* ctx = p->ctx;
  const bool stage_in = in_bytes <= STAGE_LIMIT && host_is_pageable(in);
  const bool stage_out = out_bytes <= STAGE_LIMIT && host_is_pageable(out);
  if (stage_in) {
    const int rc = ensure_host_cap(ctx, &ctx->h_in, &ctx->h_in_cap, in_bytes + 16);
    if (rc)
      return rc;
  }
  if (stage_out) {
    const int rc = ensure_host_cap(ctx, &ctx->h_out, &ctx->h_out_cap, out_bytes);
    if (rc)
      return rc;
    while (ctx->stage_events.size() < p->tile_groups.size()) {
      cudaEvent_t e;
      CUDA_TRY(ctx, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
      ctx->stage_events.push_back(e);
    }
  }
  const bool rows2d = pitch && row_bytes && row_bytes < pitch;
  // RSB200_PIPE_TRACE=1: a timeline of the groups on stderr (timed events after every upload,
  // kernel and download; debugging aid for the pipeline itself, slows the run down a little)
  const bool trace = getenv("RSB200_PIPE_TRACE") != nullptr;
  std::vector<cudaEvent_t> tev;
  auto mark = [&](cudaStream_t s) {
    if (!trace)
      return;
    cudaEvent_t e;
    cudaEventCreate(&e);
    cudaEventRecord(e, s);
    tev.push_back(e);
  };
  if (trace) {
    for (int i = 0; i < N_PIPE; ++i)
      cudaStreamSynchronize(ctx->pipe[i]);
    mark(ctx->pipe[0]);
  }
  const auto trace_t0 = std::chrono::steady_clock::now();
  for (size_t gi = 0; gi < p->tile_groups.size(); ++gi) {
    const rsb200_plan::TileGroup& g = p->tile_groups[gi];
    cudaStream_t st = ctx->pipe[gi % N_PIPE];
    const uint64_t i1c = std::min<uint64_t>(g.in_hi, in_bytes);
    const uint64_t o1 = std::min<uint64_t>(g.out_hi, out_bytes);
    if (i1c > g.in_lo) {
      const uint8_t* src = in + g.in_lo;
      if (stage_in) {
        parallel_copy(ctx->h_in + g.in_lo, src, i1c - g.in_lo);
        src = ctx->h_in + g.in_lo;
      }
      CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_in + g.in_lo, src, i1c - g.in_lo, cudaMemcpyHostToDevice, st));
    }
    mark(st);
    CUDA_TRY(ctx, launch_tile_range(p, ctx->d_in, (uint64_t)in_bytes, ctx->d_out, g.first, g.count, st));
    ctx->launches++;
    mark(st);
    if (o1 > g.out_lo) {
      uint8_t* dst = (stage_out ? ctx->h_out : out) + g.out_lo;
      if (rows2d && !stage_out) {
        // whole rows of the span, only row_bytes of each (the caller's row padding stays untouched)
        const uint64_t r0 = g.out_lo / pitch, r1 = (o1 + pitch - 1) / pitch;
        CUDA_TRY(ctx, cudaMemcpy2DAsync(out + r0 * pitch, pitch, ctx->d_out + r0 * pitch, pitch, row_bytes,
                                        r1 - r0, cudaMemcpyDeviceToHost, st));
      } else {
        CUDA_TRY(ctx, cudaMemcpyAsync(dst, ctx->d_out + g.out_lo, o1 - g.out_lo, cudaMemcpyDeviceToHost, st));
      }
      if (stage_out)
        CUDA_TRY(ctx, cudaEventRecord(ctx->stage_events[gi], st));
    }
    mark(st);
  }
  const double trace_submit_ms =
      std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - trace_t0).count();
  if (stage_out) {
    // copy every group out of the staging as soon as its download has landed
    for (size_t gi = 0; gi < p->tile_groups.size(); ++gi) {
      const rsb200_plan::TileGroup& g = p->tile_groups[gi];
      const uint64_t o1 = std::min<uint64_t>(g.out_hi, out_bytes);
      if (o1 <= g.out_lo)
        continue;
      CUDA_TRY(ctx, cudaEventSynchronize(ctx->stage_events[gi]));
      if (rows2d) {
        const uint64_t r0 = g.out_lo / pitch, r1 = (o1 + pitch - 1) / pitch;
        // (rows shared with a neighbouring group are copied by both, after both downloads: the
        //  later copy carries the final bytes, see above)
        parallel_copy_rows(out + r0 * pitch, ctx->h_out + r0 * pitch, pitch, row_bytes, r1 - r0);
      } else {
        parallel_copy(out + g.out_lo, ctx->h_out + g.out_lo, o1 - g.out_lo);
      }
    }
  }
  for (int i = 0; i < N_PIPE; ++i)
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->pipe[i]));
  if (trace) {
    const double total_ms =
        std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - trace_t0).count();
    fprintf(stderr, "PIPE_TRACE groups %zu submit %.3f ms total %.3f ms (group: upload done, kernel done, download done; ms)\n",
            p->tile_groups.size(), trace_submit_ms, total_ms);
    for (size_t gi = 0; gi < p->tile_groups.size() && 3 * gi + 3 < tev.size(); ++gi) {
      float a = 0, b = 0, c = 0;
      cudaEventElapsedTime(&a, tev[0], tev[3 * gi + 1]);
      cudaEventElapsedTime(&b, tev[0], tev[3 * gi + 2]);
      cudaEventElapsedTime(&c, tev[0], tev[3 * gi + 3]);
      if (gi < 16 || gi + 4 > p->tile_groups.size())
        fprintf(stderr, "PIPE_TRACE %3zu  %8.3f %8.3f %8.3f\n", gi, a, b, c);
    }
    for (cudaEvent_t e : tev)
      cudaEventDestroy(e);
  }
  p->last_stream = ctx->pipe[0];
  p->ran = true;
  return RSB200_OK;
}

extern "C" int rsb200_plan_run_host(rsb200_plan* p, const uint8_t* in, size_t in_bytes,
                                    uint8_t* out, size_t out_bytes, int partial) {
  if (!p || !out || (!in && in_bytes))
    return RSB200_ERR_ARG;
  rsb200_ctx* ctx = p->ctx;
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  int rc = ensure_cap(ctx, &ctx->d_in, &ctx->d_in_cap, in_bytes + 16);
  if (rc)
    return rc;
  rc = ensure_cap(ctx, &ctx->d_out, &ctx->d_out_cap, out_bytes);
  if (rc)
    return rc;
  if (in_bytes < p->need_in || out_bytes < p->need_out)
    return set_err(ctx, RSB200_ERR_ARG, "plan_run_host: buffers too small");
  if (p->kind >= 7 && p->kind <= 10)
    partial = 1; // in-place plans work on the image the caller holds: it always goes up first
  if (!partial && unpack_pipeline_ok(p))
    return run_host_unpack_pipelined(p, in, in_bytes, out, out_bytes);
  if (!partial && p->kind == 1 && p->tile_groups.size() >= 2 && !getenv("RSB200_NO_PIPELINE"))
    return run_host_tile_pipelined(p, in, in_bytes, out, out_bytes);
  cudaStream_t st = ctx->stream;
  const bool stage_in = in_bytes && in_bytes <= STAGE_LIMIT && host_is_pageable(in);
  const bool stage_out = out_bytes <= STAGE_LIMIT && host_is_pageable(out);
  const uint8_t* hin = in;
  if (stage_in) {
    rc = ensure_host_cap(ctx, &ctx->h_in, &ctx->h_in_cap, in_bytes + 16);
    if (rc)
      return rc;
    parallel_copy(ctx->h_in, in, in_bytes);
    hin = ctx->h_in;
  }
  if (stage_out) {
    rc = ensure_host_cap(ctx, &ctx->h_out, &ctx->h_out_cap, out_bytes);
    if (rc)
      return rc;
  }
  if (in_bytes)
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_in, hin, in_bytes, cudaMemcpyHostToDevice, st));
  if (partial) {
    const uint8_t* hout = out;
    if (stage_out) {
      parallel_copy(ctx->h_out, out, out_bytes);
      hout = ctx->h_out;
    }
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_out, hout, out_bytes, cudaMemcpyHostToDevice, st));
  }
  rc = rsb200_plan_run(p, ctx->d_in, in_bytes, ctx->d_out, out_bytes, (void*)st);
  if (rc)
    return rc;
  CUDA_TRY(ctx, cudaMemcpyAsync(stage_out ? ctx->h_out : out, ctx->d_out, out_bytes, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaStreamSynchronize(st));
  if (stage_out)
    parallel_copy(out, ctx->h_out, out_bytes);
  return RSB200_OK;
}

extern "C" int rsb200_plan_run_host_image(rsb200_plan* p, const uint8_t* in, size_t in_bytes,
                                          uint8_t* out, uint32_t pitch, uint32_t row_bytes,
                                          uint32_t rows, int partial) {
  if (!p || !out || (!in && in_bytes) || row_bytes > pitch)
    return RSB200_ERR_ARG;
  rsb200_ctx* ctx = p->ctx;
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  const size_t out_bytes = (size_t)pitch * rows;
  if (p->kind >= 7 && p->kind <= 10)
    partial = 1; // in-place plans: the image always goes up first
  int rc = ensure_cap(ctx, &ctx->d_in, &ctx->d_in_cap, in_bytes + 16);
  if (rc)
    return rc;
  rc = ensure_cap(ctx, &ctx->d_out, &ctx->d_out_cap, out_bytes);
  if (rc)
    return rc;
  if (in_bytes < p->need_in || out_bytes < p->need_out)
    return set_err(ctx, RSB200_ERR_ARG, "plan_run_host_image: buffers too small");
  if (!partial && p->kind == 1 && p->tile_groups.size() >= 2 && !getenv("RSB200_NO_PIPELINE"))
    return run_host_tile_pipelined(p, in, in_bytes, out, out_bytes, pitch, row_bytes);
  cudaStream_t st = ctx->stream;
  // pageable buffers go through the library's pinned staging (several copying threads)
  const bool stage_in = in_bytes && in_bytes <= STAGE_LIMIT && host_is_pageable(in);
  const bool stage_out = out_bytes <= STAGE_LIMIT && host_is_pageable(out);
  const uint8_t* hin = in;
  if (stage_in) {
    rc = ensure_host_cap(ctx, &ctx->h_in, &ctx->h_in_cap, in_bytes + 16);
    if (rc)
      return rc;
    parallel_copy(ctx->h_in, in, in_bytes);
    hin = ctx->h_in;
  }
  if (stage_out) {
    rc = ensure_host_cap(ctx, &ctx->h_out, &ctx->h_out_cap, out_bytes);
    if (rc)
      return rc;
  }
  if (in_bytes)
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_in, hin, in_bytes, cudaMemcpyHostToDevice, st));
  if (partial) {
    const uint8_t* hout = out;
    if (stage_out) {
      parallel_copy(ctx->h_out, out, out_bytes);
      hout = ctx->h_out;
    }
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_out, hout, out_bytes, cudaMemcpyHostToDevice, st));
  }
  rc = rsb200_plan_run(p, ctx->d_in, in_bytes, ctx->d_out, out_bytes, (void*)st);
  if (rc)
    return rc;
  if (stage_out) {
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->h_out, ctx->d_out, out_bytes, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaStreamSynchronize(st));
    parallel_copy_rows(out, ctx->h_out, pitch, row_bytes, rows);
  } else {
    CUDA_TRY(ctx, cudaMemcpy2DAsync(out, pitch, ctx->d_out, pitch, row_bytes, rows,
                                    cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaStreamSynchronize(st));
  }
  return RSB200_OK;
}

// ------------------------------------------------------------------
// Multi-GPU output gather over NCCL (resolved at run time)
// ------------------------------------------------------------------
#include <dlfcn.h>
struct Id128 { // ncclUniqueId: 128 opaque bytes, passed by value
  char internal[128];
};
namespace {
struct NcclApi {
  void* lib = nullptr;
  int (*GetUniqueId)(void*) = nullptr;
  int (*CommInitRank)(void**, int, Id128, int) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  int (*GroupStart)() = nullptr;
  int (*GroupEnd)() = nullptr;
  int (*Broadcast)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*Send)(const void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*Recv)(void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  bool ok = false;
};
} // namespace
static NcclApi& nccl_api() {
  static NcclApi a;
  static bool tried = false;
  if (tried)
    return a;
  tried = true;
  // the copy the process already has (e.g. the one PyTorch brought), else the system's
  a.lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
  if (!a.lib)
    a.lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!a.lib)
    a.lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!a.lib)
    return a;
#define RSB_SYM(field, name) *(void**)(&a.field) = dlsym(a.lib, name)
  RSB_SYM(GetUniqueId, "ncclGetUniqueId");
  RSB_SYM(CommInitRank, "ncclCommInitRank");
  RSB_SYM(CommDestroy, "ncclCommDestroy");
  RSB_SYM(GroupStart, "ncclGroupStart");
  RSB_SYM(GroupEnd, "ncclGroupEnd");
  RSB_SYM(Broadcast, "ncclBroadcast");
  RSB_SYM(Send, "ncclSend");
  RSB_SYM(Recv, "ncclRecv");
  RSB_SYM(GetErrorString, "ncclGetErrorString");
#undef RSB_SYM
  a.ok = a.GetUniqueId && a.CommInitRank && a.CommDestroy && a.GroupStart && a.GroupEnd &&
         a.Broadcast && a.Send && a.Recv;
  return a;
}

struct rsb200_comm {
  rsb200_ctx* ctx = nullptr;
  void* comm = nullptr;
  int world = 1, rank = 0;
  cudaStream_t stream = nullptr; // the transfers run here, beside the decode stream
  std::vector<cudaEvent_t> events;
  cudaEvent_t done = nullptr;
};

#define NCCL_TRY(ctx, expr)                                                                \
  do {                                                                                     \
    const int rc_ = (expr);                                                                \
    if (rc_ != 0)                                                                          \
      return set_err(ctx, RSB200_ERR_CUDA, "%s failed: %s", #expr,                         \
                     nccl_api().GetErrorString ? nccl_api().GetErrorString(rc_) : "?");    \
  } while (0)

extern "C" int rsb200_comm_unique_id(uint8_t id[128]) {
  NcclApi& a = nccl_api();
  if (!a.ok || !id)
    return RSB200_ERR_CUDA;
  return a.GetUniqueId(id) == 0 ? RSB200_OK : RSB200_ERR_CUDA;
}

extern "C" int rsb200_comm_create(rsb200_ctx* ctx, const uint8_t id[128], int world, int rank,
                                  rsb200_comm** out) {
  if (!ctx || !id || !out || world < 1 || rank < 0 || rank >= world)
    return set_err(ctx, RSB200_ERR_ARG, "comm_create: bad arguments");
  NcclApi& a = nccl_api();
  if (!a.ok)
    return set_err(ctx, RSB200_ERR_CUDA, "comm_create: NCCL (libnccl.so.2) is not available");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  rsb200_comm* c = new (std::nothrow) rsb200_comm();
  if (!c)
    return RSB200_ERR_CUDA;
  c->ctx = ctx;
  c->world = world;
  c->rank = rank;
  Id128 uid;
  memcpy(uid.internal, id, 128);
  const int rc = a.CommInitRank(&c->comm, world, uid, rank);
  if (rc != 0) {
    delete c;
    return set_err(ctx, RSB200_ERR_CUDA, "ncclCommInitRank failed: %s",
                   a.GetErrorString ? a.GetErrorString(rc) : "?");
  }
  cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking);
  cudaEventCreateWithFlags(&c->done, cudaEventDisableTiming);
  *out = c;
  return RSB200_OK;
}

extern "C" void rsb200_comm_destroy(rsb200_comm* c) {
  if (!c)
    return;
  cudaSetDevice(c->ctx->device);
  if (c->stream)
    cudaStreamSynchronize(c->stream);
  if (c->comm)
    nccl_api().CommDestroy(c->comm);
  for (cudaEvent_t e : c->events)
    cudaEventDestroy(e);
  if (c->done)
    cudaEventDestroy(c->done);
  if (c->stream)
    cudaStreamDestroy(c->stream);
  delete c;
}

// one span [lo, hi) of every rank's slab, on the communicator's stream
static int gather_span(rsb200_comm* c, uint8_t* all, size_t slab, uint64_t lo, uint64_t hi, int mode,
                       int root) {
  NcclApi& a = nccl_api();
  rsb200_ctx* ctx = c->ctx;
  const size_t n = (size_t)(hi - lo);
  if (!n || c->world == 1 || mode == RSB200_GATHER_NONE)
    return RSB200_OK;
  // Point-to-point transfers inside one group; a large span is cut into several of them so that
  // NCCL spreads it over more channels.
  // GATHER_ALL = every rank sends its span to every other rank (all-gather with explicit
  // placement: slab r lands at the same offset everywhere).
  const size_t kPart = 32ull << 20;
  const int parts = (int)std::min<size_t>(8, std::max<size_t>(1, n / kPart));
  const size_t per = ((n + parts - 1) / parts + 15) & ~(size_t)15;
  NCCL_TRY(ctx, a.GroupStart());
  for (int k = 0; k < parts; ++k) {
    const size_t a0 = std::min(n, per * k), a1 = std::min(n, per * (k + 1));
    if (a1 <= a0)
      continue;
    if (mode == RSB200_GATHER_ALL) {
      for (int r = 0; r < c->world; ++r) {
        if (r == c->rank)
          continue;
        NCCL_TRY(ctx, a.Send(all + (size_t)c->rank * slab + lo + a0, a1 - a0, 1, r, c->comm, c->stream));
        NCCL_TRY(ctx, a.Recv(all + (size_t)r * slab + lo + a0, a1 - a0, 1, r, c->comm, c->stream));
      }
    } else if (c->rank == root) {
      for (int r = 0; r < c->world; ++r)
        if (r != root)
          NCCL_TRY(ctx, a.Recv(all + (size_t)r * slab + lo + a0, a1 - a0, 1, r, c->comm, c->stream));
    } else {
      NCCL_TRY(ctx, a.Send(all + (size_t)c->rank * slab + lo + a0, a1 - a0, 1, root, c->comm, c->stream));
    }
  }
  NCCL_TRY(ctx, a.GroupEnd());
  return RSB200_OK;
}

extern "C" int rsb200_plan_run_gather(rsb200_plan* p, rsb200_comm* c, const void* d_in,
                                      size_t in_bytes, void* d_out_all, size_t slab_bytes, int mode,
                                      int root, void* stream) {
  if (!p || !c || !d_out_all || root < 0 || root >= c->world || mode < 0 || mode > 2)
    return RSB200_ERR_ARG;
  rsb200_ctx* ctx = p->ctx;
  if (slab_bytes < p->need_out || (slab_bytes & 15))
    return set_err(ctx, RSB200_ERR_ARG, "plan_run_gather: slab smaller than the plan's output or not a multiple of 16");
  DeviceGuard guard(ctx->device);
  if (!guard.ok)
    return set_err(ctx, RSB200_ERR_CUDA, "plan_run_gather: cannot select device %d", ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* all = (uint8_t*)d_out_all;
  uint8_t* mine = all + (size_t)c->rank * slab_bytes;
  // the transfers start behind whatever the caller queued on `stream` so far
  CUDA_TRY(ctx, cudaEventRecord(c->done, st));
  CUDA_TRY(ctx, cudaStreamWaitEvent(c->stream, c->done, 0));
  if (p->kind == 1 && !p->tile_groups.empty() && !p->host_tiles_only) {
    if (in_bytes < p->need_in)
      return set_err(ctx, RSB200_ERR_ARG, "plan_run_gather: input too small");
    while (c->events.size() < p->tile_groups.size()) {
      cudaEvent_t e;
      CUDA_TRY(ctx, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
      c->events.push_back(e);
    }
    for (size_t gi = 0; gi < p->tile_groups.size(); ++gi) {
      const rsb200_plan::TileGroup& g = p->tile_groups[gi];
      CUDA_TRY(ctx, launch_tile_range(p, (const uint8_t*)d_in, (uint64_t)in_bytes, mine, g.first, g.count, st));
      ctx->launches++;
      CUDA_TRY(ctx, cudaEventRecord(c->events[gi], st));
      CUDA_TRY(ctx, cudaStreamWaitEvent(c->stream, c->events[gi], 0));
      const int rc = gather_span(c, all, slab_bytes, g.out_lo & ~15ull,
                                 std::min<uint64_t>((g.out_hi + 15) & ~15ull, slab_bytes), mode, root);
      if (rc)
        return rc;
    }
    p->last_stream = st;
    p->ran = true;
  } else {
    const int rc0 = rsb200_plan_run(p, d_in, in_bytes, mine, slab_bytes, stream);
    if (rc0)
      return rc0;
    CUDA_TRY(ctx, cudaEventRecord(c->done, st));
    CUDA_TRY(ctx, cudaStreamWaitEvent(c->stream, c->done, 0));
    for (uint64_t lo = 0; lo < p->need_out; lo += (512ull << 20)) {
      const int rc = gather_span(c, all, slab_bytes, lo, std::min<uint64_t>(p->need_out, lo + (512ull << 20)),
                                 mode, root);
      if (rc)
        return rc;
    }
  }
  // `stream` continues only when the transfers are done
  CUDA_TRY(ctx, cudaEventRecord(c->done, c->stream));
  CUDA_TRY(ctx, cudaStreamWaitEvent(st, c->done, 0));
  return RSB200_OK;
}

extern "C" int rsb200_plan_results(rsb200_plan* p, rsb200_scan_result* results, int n) {
  if (!p)
    return RSB200_ERR_ARG;
  rsb200_ctx* ctx = p->ctx;
  if (!p->ran)
    return set_err(ctx, RSB200_ERR_ARG, "plan_results: plan has not been run");
  if (p->kind == 4 || p->kind == 6) {
    CUDA_TRY(ctx, cudaMemcpyAsync(p->h_arw2_bad, p->d_arw2_bad, sizeof(uint32_t) * (size_t)p->nunits,
                                  cudaMemcpyDeviceToHost, p->last_stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(p->last_stream));
    int first = RSB200_OK;
    for (int i = 0; i < p->nunits; ++i) {
      const bool bad = p->h_arw2_bad[i] != 0;
      if (results && i < n) {
        results[i].status = bad ? RSB200_ERR_RDE : RSB200_OK;
        results[i].consumed = 0;
      }
      if (bad && first == RSB200_OK) {
        first = RSB200_ERR_RDE;
        set_err(ctx, first, p->kind == 4
                                ? "Too many errors encountered. Giving up. First Error:\n"
                                  "ARW2 invariant failed, same pixel is both min and max"
                                : "Too many errors encountered. Giving up. First Error:\n"
                                  "a Phase One row cannot be decoded (lengths / bit stream)");
      }
    }
    return first;
  }
  if (p->kind == 11) {
    CUDA_TRY(ctx, cudaMemcpyAsync(p->h_hass_states, p->d_hass_states, sizeof(DevHassState) * (size_t)p->nunits,
                                  cudaMemcpyDeviceToHost, p->last_stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(p->last_stream));
    int first = RSB200_OK;
    for (int i = 0; i < p->nunits; ++i) {
      const DevHassState& hs = p->h_hass_states[i];
      // the first failure in stream order decides (a refill is checked before the code it feeds)
      // (a stream shorter than one chunk: the BitStreamerMSB32 constructor throws, BitStreamer.h:60-64)
      const int status = (p->h_in_size[(size_t)i] < 4 || (hs.key_ioe != H_NOKEY && hs.key_ioe <= hs.key_bad))
                             ? RSB200_ERR_IOE
                             : (hs.key_bad != H_NOKEY ? RSB200_ERR_RDE : RSB200_OK);
      if (results && i < n) {
        results[i].status = (uint32_t)status;
        results[i].consumed = status == RSB200_OK ? hs.consumed : 0u;
      }
      if (status != RSB200_OK && first == RSB200_OK) {
        first = status;
        set_err(ctx, first, status == RSB200_ERR_RDE ? "job %d: bad Huffman code"
                                                     : "job %d: Buffer overflow read in BitStreamer", i);
      }
    }
    return first;
  }
  if (p->kind != 1) {
    CUDA_TRY(ctx, cudaStreamSynchronize(p->last_stream));
    for (int i = 0; results && i < n; ++i) {
      results[i].status = RSB200_OK;
      results[i].consumed = 0;
    }
    return RSB200_OK;
  }
  CUDA_TRY(ctx, cudaMemcpyAsync(p->h_results, p->d_results, sizeof(DevResult) * p->nscans,
                                cudaMemcpyDeviceToHost, p->last_stream));
  if (p->d_oob)
    CUDA_TRY(ctx, cudaMemcpyAsync(p->h_oob, p->d_oob, sizeof(uint32_t) * p->nscans,
                                  cudaMemcpyDeviceToHost, p->last_stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(p->last_stream));
  int first = RSB200_OK;
  for (int i = 0; i < p->nscans; ++i) {
    if (p->d_oob && p->h_results[i].status == 0 && p->h_oob[i] != 0xFFFFFFFFu) {
      // Pentax: a decoded value left 0..65535 (PentaxDecompressor.cpp:170-171)
      p->h_results[i].status = RSB200_ERR_RDE;
      p->h_results[i].consumed = RSB200_PENTAX_OOB | p->h_oob[i];
      if (results && i < n) {
        results[i].status = p->h_results[i].status;
        results[i].consumed = p->h_results[i].consumed;
      }
      if (first == RSB200_OK) {
        first = RSB200_ERR_RDE;
        set_err(ctx, first, "decoded value out of bounds at %u:%u", p->h_oob[i] & 0x3FFFu,
                p->h_oob[i] >> 14);
      }
      continue;
    }
    // The reference skips `consumed` bytes of its input when a scan is done
    // (LJpegDecompressor.cpp:339 inputStream.skipBytes(bs.getStreamPosition())) and throws when
    // the buffer is shorter: a buffer that ends inside the last refill of the pump is an
    // IOException even though every symbol was there.  One rule for every LJPEG kernel.
    if (p->h_results[i].status == 0 && (size_t)i < p->h_in_size.size() &&
        p->h_results[i].consumed > p->h_in_size[(size_t)i])
      p->h_results[i].status = RSB200_ERR_IOE;
    if (results && i < n) {
      results[i].status = p->h_results[i].status;
      results[i].consumed = p->h_results[i].consumed;
    }
    if (first == RSB200_OK && p->h_results[i].status != 0) {
      first = (int)p->h_results[i].status;
      set_err(ctx, first,
              first == RSB200_ERR_RDE ? "segment %d: bad Huffman code"
                                      : "segment %d: Buffer overflow read in BitStreamer",
              i);
    }
  }
  return first;
}

extern "C" int rsb200_plan_bad_pixels(rsb200_plan* p, int job, uint32_t* positions, uint32_t cap,
                                      uint32_t* count) {
  if (!p || !count)
    return RSB200_ERR_ARG;
  rsb200_ctx* ctx = p->ctx;
  *count = 0;
  if ((p->kind != 5 && p->kind != 8) || job < 0 || job >= (int)p->pana_zero_slot.size())
    return set_err(ctx, RSB200_ERR_ARG,
                   "plan_bad_pixels: not a job of a Panasonic plan / an opcode of a DNG opcode plan");
  if (!p->ran)
    return set_err(ctx, RSB200_ERR_ARG, "plan_bad_pixels: plan has not been run");
  const int slot = p->pana_zero_slot[job];
  if (slot < 0)
    return RSB200_OK; // zero_is_not_bad (or not V4): the reference collects nothing
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  CUDA_TRY(ctx, cudaStreamSynchronize(p->last_stream));
  uint32_t n = 0;
  CUDA_TRY(ctx, cudaMemcpy(&n, p->d_pana_zero_count + slot, sizeof n, cudaMemcpyDeviceToHost));
  *count = n;
  const uint32_t take = std::min(std::min(n, cap), (uint32_t)PANA_ZERO_CAP);
  if (take && positions)
    CUDA_TRY(ctx, cudaMemcpy(positions, p->d_pana_zero_list + (size_t)slot * PANA_ZERO_CAP,
                             sizeof(uint32_t) * take, cudaMemcpyDeviceToHost));
  return RSB200_OK;
}

extern "C" int rsb200_plan_bytes(const rsb200_plan* p, uint64_t* in_bytes,
                                 uint64_t* out_bytes, uint64_t* pixels) {
  if (!p)
    return RSB200_ERR_ARG;
  if (in_bytes)
    *in_bytes = p->in_bytes;
  if (out_bytes)
    *out_bytes = p->out_bytes;
  if (pixels)
    *pixels = p->pixels;
  return RSB200_OK;
}

extern "C" int rsb200_plan_launches(const rsb200_plan* p) {
  return p ? p->launches_per_run : 0;
}

extern "C" const char* rsb200_plan_kernels(const rsb200_plan* p) {
  if (!p)
    return "";
  if (p->kind != 1)
    return "(not an LJPEG plan)";
  const bool only_thread = p->nthread && !p->ntile && !p->nsmall && !p->nbig;
  const bool only_tile = p->ntile && !p->nthread && !p->nsmall && !p->nbig;
  if (only_thread && p->use_par)
    return "k2_clean_kernel + k2_par_kernel (one CTA per segment: speculative parse of the clean stream to a "
           "fixed point, decode, row sums)";
  if (only_thread && p->use_stream) {
    if (stream_full_launch(p->ctx, p))
      return p->nthread_redo ? "k2_stream_kernel (one thread per segment, unstuffing in the thread), full-launch form + "
                               "k2_tile_kernel<1> for flagged ends of stream"
                             : "k2_stream_kernel (one thread per segment, unstuffing in the thread), full-launch form";
    return p->nthread_redo ? "k2_stream_kernel (one thread per segment, unstuffing in the thread), prefetch form + "
                             "k2_tile_kernel<1> for flagged ends of stream"
                           : "k2_stream_kernel (one thread per segment, unstuffing in the thread), prefetch form";
  }
  if (only_thread)
    return p->clean2 ? "k2_clean2_kernel + k2_thread_kernel (one thread per segment)"
                     : "k2_clean_kernel + k2_thread_kernel (one thread per segment)";
  if (only_tile)
    return p->tile_r == 2 ? "k2_tile_kernel<2> (one CTA per tile)" : "k2_tile_kernel<1> (one CTA per tile)";
  if (p->nsmall && !p->nthread && !p->ntile && !p->nbig)
    return "k2_fused_kernel (one CTA per segment)";
  return "mixed (k2_fused / k2_tile / thread path / multi-CTA ranges + K3)";
}

extern "C" void rsb200_plan_destroy(rsb200_plan* p) {
  if (!p)
    return;
  if (p->ctx)
    cudaSetDevice(p->ctx->device);
  if (p->ran && p->last_stream)
    cudaStreamSynchronize(p->last_stream); // (the frees below are stream ordered, not device-wide syncs)
  for (UnpackGroup& g : p->groups)
    rsb_dev_free(g.d_jobs);
  for (UnpackFastGroup& g : p->fast_groups)
    rsb_dev_free(g.d_jobs);
  for (RawGroup& g : p->raw_groups)
    rsb_dev_free(g.d_jobs);
  for (PanaGroup& g : p->pana_groups)
    rsb_dev_free(g.d_jobs);
  for (ScaleGroup& g : p->scale_groups)
    rsb_dev_free(g.d_jobs);
  rsb_dev_free(p->d_pana_zero_count);
  rsb_dev_free(p->d_pana_zero_list);
  rsb_dev_free(p->d_lookup_jobs);
  rsb_dev_free(p->d_lookup_tables);
  rsb_dev_free(p->d_badpix_jobs);
  rsb_dev_free(p->d_badpix_list);
  rsb_dev_free(p->d_badpix_maps);
  rsb_dev_free(p->d_dngop_jobs);
  rsb_dev_free(p->d_dngop_ops);
  rsb_dev_free(p->d_dngop_tables);
  rsb_dev_free(p->d_dngop_deltas);
  rsb_dev_free(p->d_hass_jobs);
  rsb_dev_free(p->d_hass_ctas);
  rsb_dev_free(p->d_hass_states);
  rsb_host_free(p->h_hass_states);
  rsb_dev_free(p->d_hass_seg_job);
  rsb_dev_free(p->d_hass_u32);
  rsb_dev_free(p->d_hass_row_begin);
  rsb_dev_free(p->d_p1_strips);
  rsb_dev_free(p->d_p1_jobs);
  rsb_dev_free(p->d_p1_gdesc);
  rsb_dev_free(p->d_p1_rowflag);
  rsb_dev_free(p->d_nikon_luts);
  rsb_dev_free(p->d_arw2_jobs);
  rsb_dev_free(p->d_arw2_tables);
  rsb_dev_free(p->d_arw2_bad);
  if (p->h_arw2_bad)
    rsb_host_free(p->h_arw2_bad);
  for (SrawGroup& g : p->sraw_groups)
    rsb_dev_free(g.d_jobs);
  rsb_dev_free(p->d_raw_tables);
  rsb_dev_free(p->d_tables);
  rsb_dev_free(p->d_scans);
  rsb_dev_free(p->d_strips);
  rsb_dev_free(p->d_rows);
  rsb_dev_free(p->d_diffs);
  rsb_dev_free(p->d_colvals);
  rsb_dev_free(p->d_results);
  rsb_dev_free(p->d_small_ids);
  rsb_dev_free(p->d_tile_ids);
  rsb_dev_free(p->d_tile_params);
  rsb_dev_free(p->d_thread_tile_params);
  rsb_dev_free(p->d_redo);
  rsb_dev_free(p->d_thread_ids);
  rsb_dev_free(p->d_tscans);
  rsb_dev_free(p->d_tinfos);
  rsb_dev_free(p->d_clean);
  rsb_dev_free(p->d_anchors);
  rsb_dev_free(p->d_big_ids);
  rsb_dev_free(p->d_big);
  rsb_dev_free(p->d_ranges);
  rsb_dev_free(p->d_states);
  rsb_dev_free(p->d_finals);
  rsb_dev_free(p->d_fallback);
  rsb_dev_free(p->d_oob);
  if (p->h_oob)
    rsb_host_free(p->h_oob);
  if (p->h_results)
    rsb_host_free(p->h_results);
  delete p;
}
