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
#include "arw1.cuh"
#include "samsung0.cuh"
#include "samsung1.cuh"
#include "samsung2.cuh"
#include "kodak.cuh"
#include "vc5.cuh"
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
#include <cmath>
#include <functional>
#include <thread>
#include <variant>
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

// Owners of a plan's device memory and of its pinned result buffers (read on the host by index);
// null means "not allocated".
struct DevFree {
  void operator()(void* p) const { rsb_dev_free(p); }
};
struct HostFree {
  void operator()(void* p) const { rsb_host_free(p); }
};
template <class T> using DevPtr = std::unique_ptr<T, DevFree>;
template <class T> using PinnedPtr = std::unique_ptr<T[], HostFree>;

// A create chains its allocations through `e`: each step does nothing once an earlier one failed,
// so the create checks `e` once.  An empty request still gets 16 bytes (kernels are never handed null).
template <class T> static void dev_alloc(cudaError_t& e, DevPtr<T>& d, size_t bytes) {
  void* raw = nullptr;
  if (e == cudaSuccess)
    e = rsb_dev_alloc(&raw, bytes ? bytes : 16);
  if (e == cudaSuccess)
    d.reset(static_cast<T*>(raw));
}
// ... and copies `bytes` from the host into it; `pad` more bytes behind them are allocated, not copied
template <class T>
static void dev_upload(cudaError_t& e, DevPtr<T>& d, const void* src, size_t bytes, size_t pad = 0) {
  dev_alloc(e, d, bytes + pad);
  if (e == cudaSuccess && bytes)
    e = cudaMemcpy(d.get(), src, bytes, cudaMemcpyHostToDevice);
}
template <class T> static void host_alloc(cudaError_t& e, PinnedPtr<T>& h, size_t bytes) {
  void* raw = nullptr;
  if (e == cudaSuccess)
    e = rsb_host_alloc(&raw, bytes);
  if (e == cudaSuccess)
    h.reset(static_cast<T*>(raw));
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
  DevPtr<UnpackJobDev> d_jobs;
  int njobs = 0;
  uint32_t nblocks = 0;
};

struct RawGroup {
  int format = 0;
  DevPtr<RawJobDev> d_jobs;
  int njobs = 0;
  uint32_t total_items = 0;
};

struct PanaGroup {
  int version = 0, bps = 0;
  DevPtr<PanaJobDev> d_jobs;
  int njobs = 0;
  uint32_t total_units = 0;
};

struct SrawGroup {
  int version = 0;
  bool is420 = false;
  DevPtr<SrawJobDev> d_jobs;
  int njobs = 0;
  uint32_t total_mcus = 0;
};

struct ScaleGroup {
  int mode = 0; // 0: SSE2 loop semantics, 1: plain loop semantics
  DevPtr<ScaleJobDev> d_jobs;
  int njobs = 0;
  uint32_t total_quads = 0;
  uint32_t nseg = 1; // column segments per row quad (mode 1)
};

struct UnpackFastGroup {
  int bps;
  bool lsb;
  DevPtr<UnpackFastJobDev> d_jobs;
  int njobs = 0;
  uint32_t nblocks = 0;
  std::vector<UnpackFastJobDev> h_jobs; // host copy (pipelined host runs)
};

// ---- the state of each plan kind: what its create fills and its run reads ----
struct UnpackPlan {
  std::vector<UnpackGroup> groups;
  std::vector<UnpackFastGroup> fast_groups;
};

// fixed-layout raw forms
struct RawFormPlan {
  std::vector<RawGroup> groups;
  DevPtr<uint16_t> d_tables;
};

struct SrawPlan {
  std::vector<SrawGroup> groups;
};

struct ScalePlan {
  std::vector<ScaleGroup> groups;
};

// bad-pixel lists of Panasonic V4 jobs and of DNG BAD_CONSTANT opcodes: slot per job / opcode
// that asked for one (-1 otherwise)
struct BadList {
  std::vector<int> slot;
  DevPtr<uint32_t> d_count;
  DevPtr<uint32_t> d_list;
  int nslots = 0;
};

struct PanaPlan {
  std::vector<PanaGroup> groups;
  BadList bad;
};

// DNG opcode pass (K10)
struct DngOpPlan {
  DevPtr<DngOpJobDev> d_dngop_jobs;
  DevPtr<DngOpDev> d_dngop_ops;
  DevPtr<uint16_t> d_dngop_tables;
  DevPtr<uint32_t> d_dngop_deltas;
  int dngop_njobs = 0;
  uint32_t dngop_units = 0;
  BadList bad;
};

// whole-image table lookup (K12)
struct LookupPlan {
  DevPtr<LookupJobDev> d_lookup_jobs;
  DevPtr<uint16_t> d_lookup_tables;
  int lookup_njobs = 0;
  uint32_t lookup_quads = 0;
  uint32_t lookup_nseg = 1; // column segments per row quad (more warps for few rows)
  bool lookup_dither = false;
  bool lookup_smem = false; // RSB200_LUT_SMEM=1 at plan creation: the shared-memory-table kernel (A/B candidate, lookup.cuh)
  int lookup_ntables = 0;
};

// bad-pixel interpolation (K11)
struct BadPixPlan {
  DevPtr<BadPixJobDev> d_badpix_jobs;
  DevPtr<uint32_t> d_badpix_list;
  DevPtr<uint8_t> d_badpix_maps;
  int badpix_njobs = 0;
  uint32_t badpix_total = 0;
};

// Hasselblad (K2H)
struct HasselbladPlan {
  DevPtr<DevTable> d_tables;
  DevPtr<DevHassJob> d_hass_jobs;
  DevPtr<DevHassCta> d_hass_ctas;
  DevPtr<DevHassState> d_hass_states;
  PinnedPtr<DevHassState> h_hass_states;
  DevPtr<uint32_t> d_hass_seg_job;
  DevPtr<uint32_t> d_hass_u32; // start | parsed | exit | count (nseg each) | cta_sum | cta_base | changed
  DevPtr<uint32_t> d_hass_row_begin;
  uint32_t hass_nseg = 0, hass_ncta = 0, hass_rows = 0;
  std::vector<uint32_t> h_in_size; // per job
};

// Phase One (K8)
struct PhaseOnePlan {
  DevPtr<P1StripDev> d_p1_strips;
  DevPtr<P1JobDev> d_p1_jobs;
  DevPtr<uint32_t> d_p1_gdesc;   // third version: one word per group of 8 pixels (+ 1 per row)
  DevPtr<uint32_t> d_p1_rowflag; // ... and per row: failed before anything was stored
  uint32_t p1_gstride = 0;          // words of gdesc per row
  int p1_ver = 3;                   // which version of the kernel this plan runs (RSB200_P1)
  int p1_walk1 = 0;                 // RSB200_P1W = 1 .. 6: other forms of the third version's walk (A/B; see p1_walk_kernel)
  uint32_t p1_nstrips = 0;
  // per-job error flags
  DevPtr<uint32_t> d_job_bad;
  PinnedPtr<uint32_t> h_job_bad;
};

// Samsung V0 (K13, samsung0.cuh)
struct SamsungV0Plan {
  DevPtr<S0RowDev> d_s0_rows;
  DevPtr<S0JobDev> d_s0_jobs;
  DevPtr<uint2> d_s0_desc;     // per block
  DevPtr<uint16_t> d_s0_adj;   // per pixel (rows of 16 * blocks)
  DevPtr<uint2> d_s0_nodes;    // two ping-pong buffers of s0_nnodes
  DevPtr<uint32_t> d_s0_carry; // per row tile, column and chain
  DevPtr<uint32_t> d_s0_rowfail;
  DevPtr<uint32_t> d_s0_jobfail;
  uint32_t s0_nrows = 0, s0_nnodes = 0, s0_max_nodes = 0, s0_max_w = 0, s0_max_tiles = 0;
  int s0_rounds = 0;
  // per-job results
  DevPtr<uint2> d_job_res;
  PinnedPtr<uint2> h_job_res;
};

// Samsung V2 (samsung2.cuh)
struct SamsungV2Plan {
  DevPtr<S2FrameDev> d_s2_frames;
  DevPtr<uint32_t> d_s2_starts; // per frame, four searches: candidate entries, pair steps, rows, checkpoints
  DevPtr<uint32_t> d_s2_tab;    // candidate entries
  DevPtr<uint32_t> d_s2_jump;   // two ping-pong buffers of s2_njump
  DevPtr<uint32_t> d_s2_rowstart;
  DevPtr<uint32_t> d_s2_cp;
  DevPtr<uint32_t> d_s2_ncp;
  DevPtr<uint2> d_s2_fail;
  DevPtr<uint2> d_s2_desc;
  DevPtr<int16_t> d_s2_px;
  uint32_t s2_ntab = 0, s2_njump = 0, s2_nrows = 0, s2_ncp = 0;
  // per-job results
  DevPtr<uint2> d_job_res;
  PinnedPtr<uint2> h_job_res;
};

// Kodak DCR (kodak.cuh)
struct KodakPlan {
  DevPtr<KdFrameDev> d_kd_frames;
  DevPtr<uint32_t> d_kd_starts; // per frame, four searches: tiles, candidates, checkpoints, segments
  DevPtr<uint16_t> d_kd_tables;
  DevPtr<uint32_t> d_kd_tsum;   // per prefix tile
  DevPtr<uint32_t> d_kd_q;      // nibble-sum prefix
  DevPtr<uint32_t> d_kd_tab;    // candidate entries
  DevPtr<uint32_t> d_kd_jump;   // two ping-pong buffers of kd_ncand
  DevPtr<uint32_t> d_kd_rowstart;
  DevPtr<uint32_t> d_kd_cp;
  DevPtr<uint32_t> d_kd_ncp;
  DevPtr<uint2> d_kd_fail;
  DevPtr<uint32_t> d_kd_key;
  uint32_t kd_ntiles = 0, kd_ncand = 0, kd_ncp = 0, kd_nsegs = 0;
  // per-job results and printed values
  DevPtr<uint2> d_job_res;
  PinnedPtr<uint2> h_job_res;
  DevPtr<int32_t> d_kd_values;
};

// GoPro VC-5 (vc5.cuh)
struct Vc5Plan {
  DevPtr<uint32_t> d_code;      // multi-level decode table
  DevPtr<Vc5FrameDev> d_frames;
  DevPtr<Vc5BandDev> d_bands;   // 40 per frame
  DevPtr<uint32_t> d_seg_band;  // per segment: its band
  DevPtr<uint2> d_map;          // two ping-pong buffers of nsegs * VC5_CAND
  DevPtr<unsigned long long> d_err;  // per band: first failure, bit position << 3 | code
  DevPtr<int16_t> d_coef;       // bands and the level-3 / level-2 reconstructions
  DevPtr<uint16_t> d_luts;      // log tables of output bits 1..16
  uint64_t ncoef = 0;
  uint32_t nsegs = 0, rounds = 0;
  uint32_t max_low = 0, max_rec[2] = {0, 0}, max_quads = 0;  // grid sizes
  DevPtr<uint2> d_job_res;
  PinnedPtr<uint2> h_job_res;
};

// Sony ARW2
struct Arw2Plan {
  DevPtr<Arw2JobDev> d_arw2_jobs;
  DevPtr<uint16_t> d_arw2_tables;
  uint32_t arw2_groups = 0;
  int arw2_mode = 0, arw2_ntables = 0;
  // per-job error flags
  DevPtr<uint32_t> d_job_bad;
  PinnedPtr<uint32_t> h_job_bad;
};

// every LJPEG-family create: ljpeg, cr2, pentax, nikon, arw1, samsung1
struct LjpegPlan {
  DevPtr<DevTable> d_tables;
  DevPtr<DevScan> d_scans;
  DevPtr<DevStrip> d_strips;
  DevPtr<K3RowRef> d_rows;
  DevPtr<uint16_t> d_diffs;
  DevPtr<uint16_t> d_colvals;
  DevPtr<DevResult> d_results;
  PinnedPtr<DevResult> h_results;
  uint32_t nrows = 0;
  int nscans = 0;
  int ntab_slots = 4;
  // small LJPEG tile segments: one fused CTA each; big segments (CR2 frames,
  // untiled strips): multi-CTA count/verify/diffs + K3
  DevPtr<uint32_t> d_small_ids;
  int nsmall = 0;
  DevPtr<uint32_t> d_tile_ids; // segments decoded by k2_tile_kernel<R> (ljpeg_tile.cuh)
  // host-buffer runs of a plan that holds only such segments are pipelined group by group
  // (upload / decode / download of consecutive groups overlap on three streams)
  struct TileGroup {
    uint32_t first, count;
    uint64_t in_lo, in_hi, out_lo, out_hi;
  };
  std::vector<TileGroup> tile_groups;
  DevPtr<DevTileParam> d_tile_params;
  int ntile = 0;
  int tile_r = 1;
  bool clean2 = false; // thread path: k2_clean2_kernel instead of k2_clean_kernel
  int par_ctas = 0;        // k2_par_kernel: 0 = one CTA per segment; n = persistent, n CTAs per SM (RSB200_PAR_CTAS; an experiment)
  bool use_par = false;    // thread path for small launches: k2_clean_kernel + k2_par_kernel (one CTA per segment)
  bool use_stream = false; // thread path: k2_stream_kernel (unstuffing inside the thread) instead of K2C + K2T
  int stream_form = 0;     // k2_stream_kernel: 0 = by launch size, 1 = prefetch form, 2 = full-launch form (RSB200_STREAM_FORM)
  bool host_tiles_only = false; // tile_groups / d_tile_ids describe the thread path's segments for host-buffer runs only
  std::vector<uint32_t> h_in_size; // per scan: bytes of a plain LJPEG segment (kind 0), else 0xFFFFFFFF
  DevPtr<DevTileParam> d_thread_tile_params; // thread path: parameters of the exact second opinion
  DevPtr<uint32_t> d_redo;                   // ... and which segments need it (written by K2T)
  int nthread_redo = 0;                         // segments of the thread path the tile kernel can take
  DevPtr<uint32_t> d_thread_ids; // segments decoded one per thread (K2C + K2T)
  DevPtr<DevTScan> d_tscans;
  DevPtr<DevTInfo> d_tinfos;
  DevPtr<uint32_t> d_clean;      // unstuffed data of those segments
  DevPtr<uint32_t> d_anchors;
  int nthread = 0;
  int ntables = 0;
  DevPtr<uint32_t> d_big_ids;
  std::vector<uint32_t> h_big_ids; // (for rsb200_debug_range_redo)
  int nbig = 0;
  DevPtr<BigScanInfo> d_big;
  DevPtr<DevRange> d_ranges;
  DevPtr<RangeState> d_states;
  DevPtr<RangeFinal> d_finals;
  DevPtr<uint32_t> d_fallback;
  int nranges = 0;
  // Pentax segments (DevScan::kind == 2): first out-of-bounds pixel per segment
  DevPtr<uint32_t> d_oob;
  PinnedPtr<uint32_t> h_oob;
  bool has_pentax = false, has_k3 = false, has_nikon = false;
  DevPtr<uint16_t> d_nikon_luts;
  // Sony ARW1 frames (DevScan::kind == 4, arw1.cuh): the range decoder reads their complemented
  // streams from d_arw1_in
  bool has_arw1 = false;
  int narw1 = 0;
  DevPtr<DevArw1> d_arw1;
  DevPtr<uint8_t> d_arw1_in;
  uint64_t arw1_in_bytes = 0;
  DevPtr<Arw1Run> d_arw1_runs;
  DevPtr<uint32_t> d_arw1_lastoff;
  DevPtr<int2> d_arw1_runpre;
  DevPtr<Arw1Info> d_arw1_info;
  uint32_t arw1_max_runs = 0, arw1_max_tiles = 0, arw1_max_words = 0;
  // Samsung V1 frames (DevScan::kind == 5, samsung1.cuh): reconstruction and end-of-stream scratch
  bool has_samsung1 = false;
  int ns1 = 0;
  DevPtr<DevS1> d_s1;
  DevPtr<uint16_t> d_s1_colvals; // 2 per row
  DevPtr<uint2> d_s1_rowbits;    // per row
  DevPtr<uint32_t> d_s1_oob;     // per frame: first out-of-range pixel
  DevPtr<uint32_t> d_s1_lim;     // per frame: first pixel not written
  uint32_t s1_max_h = 0;
};

// A plan holds what every kind has, and its kind's state.  Each kind's section below has its create,
// and the overloads run(), results() and kernels() that rsb200_plan_run, rsb200_plan_results and
// rsb200_plan_kernels reach through std::visit: a kind without one of them does not compile.
struct rsb200_plan {
  rsb200_ctx* ctx = nullptr;
  int nunits = 0;
  uint64_t in_bytes = 0, out_bytes = 0, pixels = 0;
  int launches_per_run = 0;
  // required extents (validation of run() arguments)
  uint64_t need_in = 0, need_out = 0;
  cudaStream_t last_stream = nullptr;
  bool ran = false;
  std::variant<UnpackPlan, LjpegPlan, RawFormPlan, SrawPlan, Arw2Plan, PanaPlan, PhaseOnePlan, ScalePlan, DngOpPlan,
               BadPixPlan, LookupPlan, HasselbladPlan, SamsungV0Plan, SamsungV2Plan, KodakPlan, Vc5Plan>
      state;
};

// A create builds its plan in a holder, so that every refusal frees whatever it allocated so far,
// and hands it out with `*out = holder.release()`.  Null when out of memory.
using PlanHolder = std::unique_ptr<rsb200_plan, decltype(&rsb200_plan_destroy)>;
static PlanHolder new_plan(rsb200_ctx* ctx) {
  PlanHolder holder(new (std::nothrow) rsb200_plan(), rsb200_plan_destroy);
  if (holder)
    holder->ctx = ctx;
  return holder;
}

// in-place plans work on the image the caller holds
static bool in_place(const rsb200_plan& p) {
  return std::holds_alternative<ScalePlan>(p.state) || std::holds_alternative<DngOpPlan>(p.state) ||
         std::holds_alternative<BadPixPlan>(p.state) || std::holds_alternative<LookupPlan>(p.state);
}

// rsb200_plan_results of a kind with per-job outcomes: copies the per-job array `d` to its pinned copy
// `h` on the plan's last stream, waits, and walks the jobs in order.  outcome(i) gives job i's
// {status, consumed}, written to out[i] when i < n; message(i, r) sets the error text of the first
// failing job only, right after outcome(i).  Returns the status of that job (RSB200_OK if none).
template <class T, class Outcome, class Message>
static int report_jobs(const rsb200_plan* p, const DevPtr<T>& d, const PinnedPtr<T>& h, rsb200_scan_result* out,
                       int n, Outcome outcome, Message message) {
  rsb200_ctx* ctx = p->ctx;
  CUDA_TRY(ctx, cudaMemcpyAsync(h.get(), d.get(), sizeof(T) * (size_t)p->nunits, cudaMemcpyDeviceToHost,
                                p->last_stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(p->last_stream));
  int first = RSB200_OK;
  for (int i = 0; i < p->nunits; ++i) {
    const rsb200_scan_result r = outcome(i);
    if (out && i < n)
      out[i] = r;
    if (r.status != RSB200_OK && first == RSB200_OK) {
      first = (int)r.status;
      message(i, r);
    }
  }
  return first;
}

// ... of ARW2 and Phase One: a job whose error flag is set fails with RDE, and the first one sets `text`
static int report_job_bad(const rsb200_plan* p, const DevPtr<uint32_t>& d, const PinnedPtr<uint32_t>& h,
                          rsb200_scan_result* out, int n, const char* text) {
  return report_jobs(
      p, d, h, out, n, [&](int i) { return rsb200_scan_result{h[i] != 0 ? (uint32_t)RSB200_ERR_RDE : 0u, 0u}; },
      [&](int, const rsb200_scan_result& r) { set_err(p->ctx, (int)r.status, "%s", text); });
}

// rsb200_plan_results of a kind without per-job outcomes: waits for the run, every job is OK
static int report_ok(const rsb200_plan* p, rsb200_scan_result* out, int n) {
  CUDA_TRY(p->ctx, cudaStreamSynchronize(p->last_stream));
  for (int i = 0; out && i < n; ++i) {
    out[i].status = RSB200_OK;
    out[i].consumed = 0;
  }
  return RSB200_OK;
}

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

#ifdef RSB200_FLUSH_COUNT
// profiling builds only (tools/flush_count.py): read/reset the 64-byte runs k2_stream_kernel's output
// stage stored by whole warps (out2[0]) and by single lanes (out2[1])
extern "C" int rsb200_debug_flush_runs(unsigned long long* out2, int reset) {
  cudaDeviceSynchronize();
  if (out2 && cudaMemcpyFromSymbol(out2, rsb200::g_flush_runs, 2 * sizeof(unsigned long long)) != cudaSuccess)
    return RSB200_ERR_CUDA;
  if (reset) {
    unsigned long long z[2] = {0, 0};
    if (cudaMemcpyToSymbol(rsb200::g_flush_runs, z, sizeof z) != cudaSuccess)
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
  PlanHolder holder = new_plan(ctx);
  if (!holder)
    return RSB200_ERR_CUDA;
  rsb200_plan* p = holder.get();
  UnpackPlan& s = p->state.emplace<UnpackPlan>();
  p->nunits = njobs;
  std::map<std::pair<int, bool>, std::vector<UnpackJobDev>> buckets;
  std::map<std::pair<int, bool>, std::vector<UnpackFastJobDev>> fast_buckets;
  for (int i = 0; i < njobs; ++i) {
    const rsb200_unpack_job& j = jobs[i];
    if (j.bps < 1 || j.bps > 16 || j.order < 0 || j.order > 3 || j.rows < 0 ||
        j.samples <= 0 || j.in_pitch <= 0 || j.out_pitch <= 0 || j.row0 < 0 ||
        j.out_col0 < 0 || (j.out_offset % 2) != 0 || (j.out_pitch % 2) != 0 ||
        ((uint64_t)j.samples * (uint64_t)j.bps) % 8 != 0 ||
        (uint64_t)j.in_pitch < ((uint64_t)j.samples * j.bps) / 8 ||
        (uint64_t)j.rows * (uint64_t)j.in_pitch > j.in_size ||
        ((uint64_t)j.out_col0 + j.samples) * 2 > (uint64_t)j.out_pitch)
      return set_err(ctx, RSB200_ERR_ARG, "unpack job %d: malformed descriptor", i);
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
    cudaError_t e = cudaSuccess;
    dev_upload(e, g.d_jobs, kv.second.data(), sizeof(UnpackJobDev) * kv.second.size());
    if (e != cudaSuccess)
      return set_err(ctx, RSB200_ERR_CUDA, "unpack plan upload failed: %s",
                     cudaGetErrorString(e));
    s.groups.push_back(std::move(g));
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
    cudaError_t e = cudaSuccess;
    dev_upload(e, g.d_jobs, kv.second.data(), sizeof(UnpackFastJobDev) * kv.second.size());
    if (e != cudaSuccess)
      return set_err(ctx, RSB200_ERR_CUDA, "unpack plan upload failed: %s",
                     cudaGetErrorString(e));
    s.fast_groups.push_back(std::move(g));
  }
  p->launches_per_run = (int)(s.groups.size() + s.fast_groups.size());
  *out = holder.release();
  return RSB200_OK;
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
      in, in_total, outp, g.d_jobs.get(), g.njobs);
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
                                  UNPACK_FAST_SMEM, st>>>(in, outp, g.d_jobs.get(), g.njobs, block_base);
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

static int run(const rsb200_plan* p, const UnpackPlan& s, const uint8_t* in, uint64_t in_bytes, uint8_t* outp,
               cudaStream_t st) {
  rsb200_ctx* ctx = p->ctx;
  for (const UnpackFastGroup& g : s.fast_groups) {
    if (!g.nblocks)
      continue;
    CUDA_TRY(ctx, run_unpack_fast_group(g, in, outp, st));
    ctx->launches++;
  }
  for (const UnpackGroup& g : s.groups) {
    if (!g.nblocks)
      continue;
    CUDA_TRY(ctx, run_unpack_group(g, in, in_bytes, outp, st));
    ctx->launches++;
  }
  return RSB200_OK;
}

static int results(const rsb200_plan* p, UnpackPlan&, rsb200_scan_result* out, int n) { return report_ok(p, out, n); }
static const char* kernels(const rsb200_plan*, const UnpackPlan& s) {
  // jobs of bit depth 8/10/12/14/16 with 4-byte aligned input rows of >= 64 items (1024
  // samples) take the fast kernel, the others the generic one
  if (!s.fast_groups.empty() && !s.groups.empty())
    return "unpack_fast_kernel + unpack_kernel";
  if (!s.fast_groups.empty())
    return "unpack_fast_kernel";
  return s.groups.empty() ? "(empty unpack plan)" : "unpack_kernel";
}

// ------------------------------------------------------------------
// fixed-layout raw forms (K1b)
// ------------------------------------------------------------------
extern "C" int rsb200_raw_plan_create(rsb200_ctx* ctx, const rsb200_raw_job* jobs, int njobs,
                                      const uint16_t* tables, int ntables, rsb200_plan** out) {
  if (!ctx || !jobs || njobs <= 0 || !out || ntables < 0 || (ntables > 0 && !tables))
    return set_err(ctx, RSB200_ERR_ARG, "raw_plan_create: bad arguments");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  PlanHolder holder = new_plan(ctx);
  if (!holder)
    return RSB200_ERR_CUDA;
  rsb200_plan* p = holder.get();
  RawFormPlan& s = p->state.emplace<RawFormPlan>();
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
    if (!ok)
      return set_err(ctx, RSB200_ERR_ARG, "raw job %d: malformed descriptor", i);
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
    if ((uint64_t)d.ipr * d.rows >= 0xFFFF0000ull)
      return set_err(ctx, RSB200_ERR_ARG, "raw job %d: too large", i);
    buckets[j.format].push_back(d);
    p->in_bytes += (uint64_t)j.rows * raw_in_bytes(j.format, (uint32_t)j.samples);
    p->out_bytes += (uint64_t)j.rows * (uint64_t)j.samples * ob;
    p->pixels += (uint64_t)j.rows * (uint64_t)j.samples;
    p->need_in = std::max<uint64_t>(p->need_in, sat_add(j.in_offset, (uint64_t)j.rows * j.in_pitch));
    p->need_out = std::max<uint64_t>(p->need_out, sat_add(j.out_offset, ((uint64_t)j.row0 + j.rows - 1) * j.out_pitch +
                         (uint64_t)ob * ((uint64_t)j.out_col0 + j.samples)));
  }
  if (ntables > 0) {
    cudaError_t e = cudaSuccess;
    dev_upload(e, s.d_tables, tables, (size_t)ntables * 65536u * sizeof(uint16_t));
    if (e != cudaSuccess)
      return set_err(ctx, RSB200_ERR_CUDA, "raw plan upload failed: %s", cudaGetErrorString(e));
  }
  for (auto& kv : buckets) {
    RawGroup g;
    g.format = kv.first;
    uint64_t items = 0;
    for (auto& d : kv.second) {
      d.item_begin = (uint32_t)items;
      items += (uint64_t)d.ipr * d.rows;
    }
    if (items >= 0xFFFF0000ull)
      return set_err(ctx, RSB200_ERR_ARG, "raw plan: too many items of format %d", g.format);
    g.total_items = (uint32_t)items;
    g.njobs = (int)kv.second.size();
    cudaError_t e = cudaSuccess;
    dev_upload(e, g.d_jobs, kv.second.data(), sizeof(RawJobDev) * kv.second.size());
    if (e != cudaSuccess)
      return set_err(ctx, RSB200_ERR_CUDA, "raw plan upload failed: %s", cudaGetErrorString(e));
    s.groups.push_back(std::move(g));
  }
  p->launches_per_run = (int)s.groups.size();
  *out = holder.release();
  return RSB200_OK;
}

template <int FORMAT>
static cudaError_t launch_rawform(const RawGroup& g, const uint8_t* in, uint64_t in_total,
                                  uint8_t* outp, const uint16_t* tables, cudaStream_t st) {
  const uint32_t nb = (g.total_items + RAW_NT - 1) / RAW_NT;
  rawform_kernel<FORMAT><<<nb, RAW_NT, 0, st>>>(in, in_total, outp, g.d_jobs.get(), g.njobs,
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

static int run(const rsb200_plan* p, const RawFormPlan& s, const uint8_t* in, uint64_t in_bytes, uint8_t* outp,
               cudaStream_t st) {
  rsb200_ctx* ctx = p->ctx;
  for (const RawGroup& g : s.groups) {
    if (!g.total_items)
      continue;
    CUDA_TRY(ctx, run_raw_group(g, in, in_bytes, outp, s.d_tables.get(), st));
    ctx->launches++;
  }
  return RSB200_OK;
}

static int results(const rsb200_plan* p, RawFormPlan&, rsb200_scan_result* out, int n) { return report_ok(p, out, n); }
static const char* kernels(const rsb200_plan*, const RawFormPlan& s) {
  return s.groups.empty() ? "(empty raw-form plan)" : "rawform_kernel";
}

// K12: whole-image table lookup (RawImageData::sixteenBitLookup)
extern "C" int rsb200_lookup_plan_create(rsb200_ctx* ctx, const rsb200_lookup_job* jobs, int njobs,
                                         const uint16_t* tables, int ntables, int dither,
                                         rsb200_plan** out) {
  if (!ctx || !jobs || njobs <= 0 || !out || !tables || ntables <= 0)
    return set_err(ctx, RSB200_ERR_ARG, "lookup_plan_create: bad arguments");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  PlanHolder holder = new_plan(ctx);
  if (!holder)
    return RSB200_ERR_CUDA;
  rsb200_plan* p = holder.get();
  LookupPlan& s = p->state.emplace<LookupPlan>();
  p->nunits = njobs;
  s.lookup_dither = dither != 0;
  {
    const char* smem_env = getenv("RSB200_LUT_SMEM");
    s.lookup_smem = smem_env && smem_env[0] == '1';
  }
  s.lookup_ntables = ntables;
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
  s.lookup_njobs = njobs;
  s.lookup_quads = (uint32_t)quads;
  {
    // enough warps to fill the machine (~32 per SM), but at least 2 iterations of 32 groups each
    uint32_t min_groups = 0xFFFFFFFFu;
    for (int i = 0; i < njobs; ++i)
      min_groups = std::min(min_groups, hj[(size_t)i].ngroups);
    const uint32_t want = (uint32_t)((32ull * (uint64_t)ctx->sm_count + quads - 1) / std::max<uint64_t>(quads, 1));
    s.lookup_nseg = std::max(1u, std::min(std::min(want, 8u), std::max(1u, min_groups / 64u)));
    if (const char* e = getenv("RSB200_LUT_NSEG"))
      s.lookup_nseg = (uint32_t)std::max(1, std::min(64, atoi(e)));
  }
  cudaError_t e = cudaSuccess;
  dev_upload(e, s.d_lookup_jobs, hj.data(), sizeof(LookupJobDev) * hj.size());
  dev_upload(e, s.d_lookup_tables, tables, sizeof(uint16_t) * (size_t)ntables * (dither ? 131072u : 65536u));
  if (e != cudaSuccess)
    return set_err(ctx, RSB200_ERR_CUDA, "lookup plan upload failed: %s", cudaGetErrorString(e));
  p->launches_per_run = 1;
  *out = holder.release();
  return RSB200_OK;
}

static int run(const rsb200_plan* p, const LookupPlan& s, const uint8_t*, uint64_t, uint8_t* outp, cudaStream_t st) {
  rsb200_ctx* ctx = p->ctx;
  const uint32_t nbs = (uint32_t)(((uint64_t)s.lookup_quads * s.lookup_nseg + LUT_WARPS - 1) / LUT_WARPS);
  if (s.lookup_smem && !s.lookup_dither && s.lookup_ntables == 1) {
    const int sms = ctx->sm_count;
    lookup_smem_kernel<<<(unsigned)std::max(1, sms), LUT_SMEM_NT, LUT_SMEM_BYTES, st>>>(
        outp, s.d_lookup_jobs.get(), s.lookup_njobs, s.lookup_quads, s.d_lookup_tables.get());
  } else if (s.lookup_dither)
    lookup_kernel<true><<<nbs, LUT_NT, 0, st>>>(outp, s.d_lookup_jobs.get(), s.lookup_njobs, s.lookup_quads,
                                                s.d_lookup_tables.get(), s.lookup_nseg);
  else
    lookup_kernel<false><<<nbs, LUT_NT, 0, st>>>(outp, s.d_lookup_jobs.get(), s.lookup_njobs, s.lookup_quads,
                                                 s.d_lookup_tables.get(), s.lookup_nseg);
  CUDA_TRY(ctx, cudaGetLastError());
  ctx->launches++;
  return RSB200_OK;
}

static int results(const rsb200_plan* p, LookupPlan&, rsb200_scan_result* out, int n) { return report_ok(p, out, n); }
static const char* kernels(const rsb200_plan*, const LookupPlan&) { return "(not an LJPEG plan)"; }

// K11: bad-pixel interpolation (RawImageData::fixBadPixels)
extern "C" int rsb200_badpix_plan_create(rsb200_ctx* ctx, const rsb200_badpix_job* jobs, int njobs,
                                         const uint32_t* positions, uint32_t npositions,
                                         rsb200_plan** out) {
  if (!ctx || !jobs || njobs <= 0 || !out || (npositions && !positions))
    return set_err(ctx, RSB200_ERR_ARG, "badpix_plan_create: bad arguments");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  PlanHolder holder = new_plan(ctx);
  if (!holder)
    return RSB200_ERR_CUDA;
  rsb200_plan* p = holder.get();
  BadPixPlan& s = p->state.emplace<BadPixPlan>();
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
  s.badpix_njobs = njobs;
  s.badpix_total = (uint32_t)list.size();
  cudaError_t e = cudaSuccess;
  dev_upload(e, s.d_badpix_jobs, hj.data(), sizeof(BadPixJobDev) * hj.size());
  dev_upload(e, s.d_badpix_list, list.data(), sizeof(uint32_t) * list.size(), sizeof(uint32_t));
  dev_upload(e, s.d_badpix_maps, maps.data(), maps.size(), 16);
  if (e != cudaSuccess)
    return set_err(ctx, RSB200_ERR_CUDA, "badpix plan upload failed: %s", cudaGetErrorString(e));
  p->launches_per_run = s.badpix_total ? 1 : 0;
  *out = holder.release();
  return RSB200_OK;
}

static int run(const rsb200_plan* p, const BadPixPlan& s, const uint8_t*, uint64_t, uint8_t* outp, cudaStream_t st) {
  rsb200_ctx* ctx = p->ctx;
  if (s.badpix_total) {
    badpix_kernel<<<(s.badpix_total + BADPIX_NT - 1) / BADPIX_NT, BADPIX_NT, 0, st>>>(
        outp, s.d_badpix_jobs.get(), s.badpix_njobs, s.d_badpix_list.get(), s.badpix_total, s.d_badpix_maps.get());
    CUDA_TRY(ctx, cudaGetLastError());
    ctx->launches++;
  }
  return RSB200_OK;
}

static int results(const rsb200_plan* p, BadPixPlan&, rsb200_scan_result* out, int n) { return report_ok(p, out, n); }
static const char* kernels(const rsb200_plan*, const BadPixPlan&) { return "(not an LJPEG plan)"; }

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
  PlanHolder holder = new_plan(ctx);
  if (!holder)
    return RSB200_ERR_CUDA;
  rsb200_plan* p = holder.get();
  DngOpPlan& s = p->state.emplace<DngOpPlan>();
  p->nunits = njobs;
  std::vector<DngOpJobDev> hj((size_t)njobs);
  std::vector<DngOpDev> ho((size_t)nops);
  s.bad.slot.assign((size_t)nops, -1);
  uint64_t units = 0;
  if (const char* why = dngop_build(jobs, njobs, ops, nops, ntables, ndeltas, hj.data(), ho.data(),
                                    s.bad.slot.data(), &s.bad.nslots, &units))
    return set_err(ctx, RSB200_ERR_ARG, "dngop plan: %s", why);
  for (int i = 0; i < njobs; ++i) {
    const uint64_t bytes = (uint64_t)(hj[i].row1 - hj[i].row0) * hj[i].samples * (jobs[i].is_f32 ? 4u : 2u);
    p->in_bytes += bytes;
    p->out_bytes += bytes;
    p->pixels += (uint64_t)(hj[i].row1 - hj[i].row0) * jobs[i].width;
    p->need_out = std::max<uint64_t>(p->need_out, sat_add(jobs[i].offset, (uint64_t)jobs[i].height * jobs[i].pitch));
  }
  s.dngop_njobs = njobs;
  s.dngop_units = (uint32_t)units;
  cudaError_t e = cudaSuccess;
  dev_upload(e, s.d_dngop_jobs, hj.data(), sizeof(DngOpJobDev) * hj.size());
  dev_upload(e, s.d_dngop_ops, ho.data(), sizeof(DngOpDev) * ho.size(), sizeof(DngOpDev));
  dev_upload(e, s.d_dngop_tables, tables, sizeof(uint16_t) * 65536 * (size_t)ntables, sizeof(uint16_t) * 65536);
  dev_upload(e, s.d_dngop_deltas, deltas, sizeof(uint32_t) * (size_t)ndeltas, sizeof(uint32_t));
  if (s.bad.nslots) {
    dev_alloc(e, s.bad.d_count, sizeof(uint32_t) * (size_t)s.bad.nslots);
    dev_alloc(e, s.bad.d_list, sizeof(uint32_t) * (size_t)DNGOP_BAD_CAP * (size_t)s.bad.nslots);
  }
  if (e != cudaSuccess)
    return set_err(ctx, RSB200_ERR_CUDA, "dngop plan upload failed: %s", cudaGetErrorString(e));
  p->launches_per_run = units ? 1 : 0;
  *out = holder.release();
  return RSB200_OK;
}

static int run(const rsb200_plan* p, const DngOpPlan& s, const uint8_t*, uint64_t, uint8_t* outp, cudaStream_t st) {
  rsb200_ctx* ctx = p->ctx;
  if (s.bad.nslots)
    CUDA_TRY(ctx, cudaMemsetAsync(s.bad.d_count.get(), 0,
                                  sizeof(uint32_t) * (size_t)s.bad.nslots, st));
  if (s.dngop_units) {
    dngop_kernel<<<(s.dngop_units + DNGOP_NT - 1) / DNGOP_NT, DNGOP_NT, 0, st>>>(
        outp, s.d_dngop_jobs.get(), s.dngop_njobs, s.dngop_units, s.d_dngop_ops.get(), s.d_dngop_tables.get(),
        s.d_dngop_deltas.get(), s.bad.d_count.get(), s.bad.d_list.get());
    CUDA_TRY(ctx, cudaGetLastError());
    ctx->launches++;
  }
  return RSB200_OK;
}

static int results(const rsb200_plan* p, DngOpPlan&, rsb200_scan_result* out, int n) { return report_ok(p, out, n); }
static const char* kernels(const rsb200_plan*, const DngOpPlan&) { return "(not an LJPEG plan)"; }

// K9: black / white scaling in place (RawImageDataU16::scaleValues)
extern "C" int rsb200_scale_plan_create(rsb200_ctx* ctx, const rsb200_scale_job* jobs, int njobs,
                                        rsb200_plan** out) {
  if (!ctx || !jobs || njobs <= 0 || !out)
    return set_err(ctx, RSB200_ERR_ARG, "scale_plan_create: bad arguments");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  PlanHolder holder = new_plan(ctx);
  if (!holder)
    return RSB200_ERR_CUDA;
  rsb200_plan* p = holder.get();
  ScalePlan& s = p->state.emplace<ScalePlan>();
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
    cudaError_t e = cudaSuccess;
    dev_upload(e, g.d_jobs, dev[mode].data(), sizeof(ScaleJobDev) * dev[mode].size());
    if (e != cudaSuccess)
      return set_err(ctx, RSB200_ERR_CUDA, "scale plan upload failed: %s", cudaGetErrorString(e));
    s.groups.push_back(std::move(g));
  }
  p->launches_per_run = (int)s.groups.size();
  *out = holder.release();
  return RSB200_OK;
}

static int run(const rsb200_plan* p, const ScalePlan& s, const uint8_t*, uint64_t, uint8_t* outp, cudaStream_t st) {
  rsb200_ctx* ctx = p->ctx;
  for (const ScaleGroup& g : s.groups) {
    const uint32_t nb = (g.total_quads + SCALE_WARPS - 1) / SCALE_WARPS;
    if (g.mode == 0)
      scale_kernel<0><<<nb, SCALE_NT, 0, st>>>(outp, g.d_jobs.get(), g.njobs, g.total_quads, 1u);
    else
      scale_kernel<1><<<(uint32_t)(((uint64_t)g.total_quads * g.nseg + SCALE_WARPS - 1) / SCALE_WARPS), SCALE_NT,
                        0, st>>>(outp, g.d_jobs.get(), g.njobs, g.total_quads, g.nseg);
    CUDA_TRY(ctx, cudaGetLastError());
    ctx->launches++;
  }
  return RSB200_OK;
}

static int results(const rsb200_plan* p, ScalePlan&, rsb200_scan_result* out, int n) { return report_ok(p, out, n); }
static const char* kernels(const rsb200_plan*, const ScalePlan&) { return "(not an LJPEG plan)"; }

// ------------------------------------------------------------------
// sRaw interpolation (K5)
// ------------------------------------------------------------------
extern "C" int rsb200_sraw_plan_create(rsb200_ctx* ctx, const rsb200_sraw_job* jobs, int njobs,
                                       rsb200_plan** out) {
  if (!ctx || !jobs || njobs <= 0 || !out)
    return set_err(ctx, RSB200_ERR_ARG, "sraw_plan_create: bad arguments");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  PlanHolder holder = new_plan(ctx);
  if (!holder)
    return RSB200_ERR_CUDA;
  rsb200_plan* p = holder.get();
  SrawPlan& s = p->state.emplace<SrawPlan>();
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
    if (!ok)
      return set_err(ctx, RSB200_ERR_ARG, "sraw job %d: malformed descriptor", i);
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
    if (n >= 0xFFFF0000ull)
      return set_err(ctx, RSB200_ERR_ARG, "sraw plan: too many MCUs");
    g.total_mcus = (uint32_t)n;
    g.njobs = (int)kv.second.size();
    cudaError_t e = cudaSuccess;
    dev_upload(e, g.d_jobs, kv.second.data(), sizeof(SrawJobDev) * kv.second.size());
    if (e != cudaSuccess)
      return set_err(ctx, RSB200_ERR_CUDA, "sraw plan upload failed: %s", cudaGetErrorString(e));
    s.groups.push_back(std::move(g));
  }
  p->launches_per_run = (int)s.groups.size();
  *out = holder.release();
  return RSB200_OK;
}

static cudaError_t run_sraw_group(const SrawGroup& g, const uint8_t* in, uint8_t* outp,
                                  cudaStream_t st) {
  const uint32_t nb = (g.total_mcus + SRAW_NT - 1) / SRAW_NT;
#define RSB_SRAW(V, T)                                                                     \
  sraw_kernel<V, T><<<nb, SRAW_NT, 0, st>>>(in, outp, g.d_jobs.get(), g.njobs, g.total_mcus)
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

static int run(const rsb200_plan* p, const SrawPlan& s, const uint8_t* in, uint64_t, uint8_t* outp, cudaStream_t st) {
  rsb200_ctx* ctx = p->ctx;
  for (const SrawGroup& g : s.groups) {
    CUDA_TRY(ctx, run_sraw_group(g, in, outp, st));
    ctx->launches++;
  }
  return RSB200_OK;
}

static int results(const rsb200_plan* p, SrawPlan&, rsb200_scan_result* out, int n) { return report_ok(p, out, n); }
static const char* kernels(const rsb200_plan*, const SrawPlan&) { return "(not an LJPEG plan)"; }

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
  PlanHolder holder = new_plan(ctx);
  if (!holder)
    return RSB200_ERR_CUDA;
  rsb200_plan* p = holder.get();
  HasselbladPlan& s = p->state.emplace<HasselbladPlan>();
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
    if (!ok)
      return set_err(ctx, RSB200_ERR_ARG, "hasselblad job %d: malformed descriptor", i);
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
    s.h_in_size.push_back(j.in_size);
    p->in_bytes += j.in_size;
    p->out_bytes += (uint64_t)j.width * j.height * 2;
    p->pixels += (uint64_t)j.width * j.height;
    p->need_in = std::max<uint64_t>(p->need_in, sat_add(j.in_offset, j.in_size));
    p->need_out = std::max<uint64_t>(p->need_out, sat_add(j.out_offset, ((uint64_t)j.height - 1) * j.out_pitch +
                                                                            (uint64_t)j.width * 2));
  }
  row_begin[(size_t)njobs] = (uint32_t)rows_total;
  if (nseg_total >= 0x7FFFFFFFull || rows_total >= 0x7FFFFFFull)
    return set_err(ctx, RSB200_ERR_ARG, "hasselblad plan: too large");
  s.hass_nseg = (uint32_t)nseg_total;
  s.hass_ncta = (uint32_t)ctas.size();
  s.hass_rows = (uint32_t)rows_total;
  cudaError_t e = cudaSuccess;
  dev_upload(e, s.d_tables, ht.data(), sizeof(DevTable) * ht.size());
  dev_upload(e, s.d_hass_jobs, dj.data(), sizeof(DevHassJob) * dj.size());
  dev_upload(e, s.d_hass_ctas, ctas.data(), sizeof(DevHassCta) * ctas.size());
  dev_upload(e, s.d_hass_seg_job, seg_job.data(), sizeof(uint32_t) * seg_job.size());
  dev_upload(e, s.d_hass_row_begin, row_begin.data(), sizeof(uint32_t) * row_begin.size());
  dev_alloc(e, s.d_hass_u32, sizeof(uint32_t) * (4ull * nseg_total + 2ull * ctas.size() + H_ROUNDS + 8));
  dev_alloc(e, s.d_hass_states, sizeof(DevHassState) * (size_t)njobs);
  host_alloc(e, s.h_hass_states, sizeof(DevHassState) * (size_t)njobs);
  if (e != cudaSuccess)
    return set_err(ctx, RSB200_ERR_CUDA, "hasselblad plan allocation failed: %s", cudaGetErrorString(e));
  p->launches_per_run = 1 + 2 * H_ROUNDS + 1 + 2 + 1 + 1;
  *out = holder.release();
  return RSB200_OK;
}

static int run(const rsb200_plan* p, const HasselbladPlan& s, const uint8_t* in, uint64_t, uint8_t* outp,
               cudaStream_t st) {
  const uint32_t n = s.hass_nseg, nc = s.hass_ncta;
  uint32_t* start = s.d_hass_u32.get();
  uint32_t* parsed = start + n;
  uint32_t* exitp = parsed + n;
  uint32_t* count = exitp + n;
  uint32_t* cta_sum = count + n;
  uint32_t* cta_base = cta_sum + nc;
  uint32_t* changed = cta_base + nc;
  const size_t smem = sizeof(HassShared);
  const uint32_t nb = (std::max<uint32_t>(std::max<uint32_t>(n, (uint32_t)p->nunits), H_ROUNDS + 1) + 255) / 256;
  hass_init_kernel<<<nb, 256, 0, st>>>(s.d_hass_jobs.get(), p->nunits, n, s.d_hass_seg_job.get(), start, parsed,
                                       s.d_hass_states.get(), changed);
  for (int r = 0; r < H_ROUNDS; ++r) {
    hass_parse_kernel<<<nc, H_NT, smem, st>>>(in, s.d_hass_jobs.get(), s.d_tables.get(), s.d_hass_ctas.get(), start, parsed,
                                              exitp, count);
    hass_link_kernel<<<(n + 255) / 256, 256, 0, st>>>(s.d_hass_jobs.get(), p->nunits, n, s.d_hass_seg_job.get(), start,
                                                      exitp, changed + r);
  }
  hass_serial_kernel<<<p->nunits, 32, 0, st>>>(in, s.d_hass_jobs.get(), s.d_tables.get(), start, parsed, exitp, count,
                                               changed + (H_ROUNDS - 1));
  hass_ctasum_kernel<<<nc, H_NT, smem, st>>>(s.d_hass_jobs.get(), s.d_hass_ctas.get(), count, cta_sum);
  hass_ctascan_kernel<<<(p->nunits + 63) / 64, 64, 0, st>>>(s.d_hass_jobs.get(), p->nunits, cta_sum, cta_base);
  hass_decode_kernel<<<nc, H_NT, smem, st>>>(in, s.d_hass_jobs.get(), s.d_tables.get(), s.d_hass_ctas.get(), start, exitp,
                                             count, cta_base, outp, s.d_hass_states.get());
  hass_rows_kernel<<<(s.hass_rows * 32 + 255) / 256, 256, 0, st>>>(s.d_hass_jobs.get(), p->nunits,
                                                                   s.d_hass_row_begin.get(), outp);
  CUDA_TRY(p->ctx, cudaGetLastError());
  p->ctx->launches += (uint64_t)p->launches_per_run;
  return RSB200_OK;
}

static int results(const rsb200_plan* p, HasselbladPlan& s, rsb200_scan_result* out, int n) {
  return report_jobs(
      p, s.d_hass_states, s.h_hass_states, out, n,
      [&](int i) {
        const DevHassState& hs = s.h_hass_states[i];
        // the first failure in stream order decides (a refill is checked before the code it feeds)
        // (a stream shorter than one chunk: the BitStreamerMSB32 constructor throws, BitStreamer.h:60-64)
        const int status = (s.h_in_size[(size_t)i] < 4 || (hs.key_ioe != H_NOKEY && hs.key_ioe <= hs.key_bad))
                               ? RSB200_ERR_IOE
                               : (hs.key_bad != H_NOKEY ? RSB200_ERR_RDE : RSB200_OK);
        return rsb200_scan_result{(uint32_t)status, status == RSB200_OK ? hs.consumed : 0u};
      },
      [&](int i, const rsb200_scan_result& r) {
        set_err(p->ctx, (int)r.status, r.status == RSB200_ERR_RDE ? "job %d: bad Huffman code"
                                                                   : "job %d: Buffer overflow read in BitStreamer", i);
      });
}

static const char* kernels(const rsb200_plan*, const HasselbladPlan&) { return "(not an LJPEG plan)"; }

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
  PlanHolder holder = new_plan(ctx);
  if (!holder)
    return RSB200_ERR_CUDA;
  rsb200_plan* p = holder.get();
  PhaseOnePlan& s = p->state.emplace<PhaseOnePlan>();
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
    if (!ok)
      return set_err(ctx, RSB200_ERR_ARG, "phaseone job %d: malformed descriptor or strips", i);
    dj[(size_t)i].out_offset = j.out_offset;
    dj[(size_t)i].out_pitch = j.out_pitch;
    dj[(size_t)i].width = j.width;
    p->out_bytes += (uint64_t)j.width * j.height * 2;
    p->pixels += (uint64_t)j.width * j.height;
    p->need_out = std::max<uint64_t>(p->need_out, sat_add(j.out_offset, ((uint64_t)j.height - 1) * j.out_pitch +
                                                      2ull * j.width));
  }
  s.p1_nstrips = (uint32_t)ds.size();
  for (int i = 0; i < njobs; ++i)
    s.p1_gstride = std::max<uint32_t>(s.p1_gstride, (jobs[i].width / 8u + 1u + 3u) & ~3u); // (16-byte rows)
  cudaError_t e = cudaSuccess;
  dev_upload(e, s.d_p1_strips, ds.data(), sizeof(P1StripDev) * ds.size());
  dev_alloc(e, s.d_p1_gdesc, sizeof(uint32_t) * (size_t)s.p1_gstride * ds.size());
  dev_alloc(e, s.d_p1_rowflag, sizeof(uint32_t) * ds.size());
  dev_upload(e, s.d_p1_jobs, dj.data(), sizeof(P1JobDev) * dj.size());
  dev_alloc(e, s.d_job_bad, sizeof(uint32_t) * (size_t)njobs);
  host_alloc(e, s.h_job_bad, sizeof(uint32_t) * (size_t)njobs);
  if (e != cudaSuccess)
    return set_err(ctx, RSB200_ERR_CUDA, "phaseone plan upload failed: %s", cudaGetErrorString(e));
  s.p1_ver = p1_version();
  {
    const char* e = getenv("RSB200_P1W");
    s.p1_walk1 = (e && e[0] >= '1' && e[0] <= '8' && !e[1]) ? e[0] - '0' : 0;
  }
  p->launches_per_run = s.p1_ver == 3 ? 2 : 1;
  *out = holder.release();
  return RSB200_OK;
}

static int run(const rsb200_plan* p, const PhaseOnePlan& s, const uint8_t* in, uint64_t, uint8_t* outp,
               cudaStream_t st) {
  CUDA_TRY(p->ctx, cudaMemsetAsync(s.d_job_bad.get(), 0, sizeof(uint32_t) * (size_t)p->nunits, st));
  const int v = s.p1_ver;
  const uint32_t nb = (s.p1_nstrips + P1_NT - 1) / P1_NT;
  if (v == 1) {
    p1_kernel<<<nb, P1_NT, 0, st>>>(in, outp, s.d_p1_strips.get(), s.p1_nstrips, s.d_p1_jobs.get(),
                                    s.d_job_bad.get());
  } else if (v == 2) {
    p1_kernel_v2<<<nb, P1_NT, 0, st>>>(in, outp, s.d_p1_strips.get(), s.p1_nstrips, s.d_p1_jobs.get(),
                                       s.d_job_bad.get());
  } else {
    p1_walk_kernel<<<(s.p1_nstrips + P1W_NT - 1) / P1W_NT, P1W_NT, 0, st>>>(
        in, s.d_p1_strips.get(), s.p1_nstrips, s.d_p1_jobs.get(), s.p1_gstride, s.d_p1_gdesc.get(), s.d_p1_rowflag.get(),
        s.p1_walk1);
    p1_decode_kernel<<<(s.p1_nstrips * 32u + P1D_NT - 1) / P1D_NT, P1D_NT, 0, st>>>(
        in, outp, s.d_p1_strips.get(), s.p1_nstrips, s.d_p1_jobs.get(), s.p1_gstride, s.d_p1_gdesc.get(),
        s.d_p1_rowflag.get(), s.d_job_bad.get());
  }
  CUDA_TRY(p->ctx, cudaGetLastError());
  p->ctx->launches += (uint64_t)p->launches_per_run;
  return RSB200_OK;
}

static int results(const rsb200_plan* p, PhaseOnePlan& s, rsb200_scan_result* out, int n) {
  return report_job_bad(p, s.d_job_bad, s.h_job_bad, out, n,
                        "Too many errors encountered. Giving up. First Error:\n"
                        "a Phase One row cannot be decoded (lengths / bit stream)");
}

static const char* kernels(const rsb200_plan*, const PhaseOnePlan&) { return "(not an LJPEG plan)"; }

// ------------------------------------------------------------------
// Samsung V0 (K13): one MSB32 stream per row (samsung0.cuh)
// ------------------------------------------------------------------
extern "C" int rsb200_samsung0_plan_create(rsb200_ctx* ctx, const rsb200_samsung0_job* jobs, int njobs,
                                           const rsb200_samsung0_strip* strips, int nstrips,
                                           rsb200_plan** out) {
  if (!ctx || !jobs || njobs <= 0 || !strips || nstrips <= 0 || !out)
    return set_err(ctx, RSB200_ERR_ARG, "samsung0_plan_create: bad arguments");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  for (int i = 0; i < njobs; ++i) {
    const rsb200_samsung0_job& j = jobs[i];
    // SamsungV0Decompressor ctor (SamsungV0Decompressor.cpp:51-55)
    if (j.width < 16 || j.width > 5546 || j.height == 0 || j.height > 3714)
      return set_err(ctx, RSB200_ERR_RDE, "job %d: Unexpected image dimensions found: (%u; %u)", i, j.width,
                     j.height);
    bool ok = (j.out_offset % 2) == 0 && (j.out_pitch % 2) == 0 && (uint64_t)j.width * 2 <= j.out_pitch &&
              (uint64_t)j.first_strip + j.height <= (uint64_t)nstrips;
    for (uint32_t r = 0; ok && r < j.height; ++r) {
      const rsb200_samsung0_strip& st = strips[j.first_strip + r];
      ok = st.in_size < (1u << 28) && st.reserved == 0;
    }
    if (!ok)
      return set_err(ctx, RSB200_ERR_ARG, "samsung0 job %d: malformed descriptor or strips", i);
  }
  PlanHolder holder = new_plan(ctx);
  if (!holder)
    return RSB200_ERR_CUDA;
  rsb200_plan* p = holder.get();
  SamsungV0Plan& s = p->state.emplace<SamsungV0Plan>();
  p->nunits = njobs;
  std::vector<S0JobDev> dj((size_t)njobs);
  std::vector<S0RowDev> dr;
  uint64_t blk = 0, px = 0, carry = 0, nodes = 0;
  uint32_t depth = 0;
  for (int i = 0; i < njobs; ++i) {
    const rsb200_samsung0_job& j = jobs[i];
    S0JobDev& d = dj[(size_t)i];
    memset(&d, 0, sizeof d);
    d.out_offset = j.out_offset;
    d.out_pitch = j.out_pitch;
    d.w = j.width;
    d.h = j.height;
    d.nb = (j.width + 15) / 16;
    d.blk_base = blk;
    d.px_base = px;
    d.carry_base = carry;
    d.node_base = (uint32_t)nodes;
    d.row_base = (uint32_t)dr.size();
    d.rtiles = (j.height + S0C_TH - 1) / S0C_TH;
    blk += (uint64_t)d.h * d.nb;
    px += (uint64_t)d.h * d.nb * 16;
    carry += (uint64_t)d.rtiles * d.nb * 32;
    nodes += (uint64_t)d.h * d.nb * 2;
    depth = std::max(depth, d.h + d.nb + 1); // (a node chain moves up a row or left a block per step)
    s.s0_max_nodes = std::max(s.s0_max_nodes, d.h * d.nb * 2);
    s.s0_max_w = std::max(s.s0_max_w, d.w);
    s.s0_max_tiles = std::max(s.s0_max_tiles, d.rtiles);
    for (uint32_t r = 0; r < j.height; ++r) {
      const rsb200_samsung0_strip& st = strips[j.first_strip + r];
      dr.push_back(S0RowDev{st.in_offset, st.in_size, (uint32_t)i, r, 0});
      p->in_bytes += st.in_size;
      p->need_in = std::max<uint64_t>(p->need_in, sat_add(st.in_offset, st.in_size));
    }
    p->out_bytes += (uint64_t)j.width * j.height * 2;
    p->pixels += (uint64_t)j.width * j.height;
    p->need_out = std::max<uint64_t>(p->need_out, sat_add(j.out_offset, ((uint64_t)j.height - 1) * j.out_pitch +
                                                      2ull * j.width));
  }
  if (nodes >= S0_ROOT)
    return set_err(ctx, RSB200_ERR_ARG, "samsung0 plan: too many frames for one plan");
  s.s0_nrows = (uint32_t)dr.size();
  s.s0_nnodes = (uint32_t)nodes;
  while ((1u << s.s0_rounds) < depth)
    ++s.s0_rounds;
  cudaError_t e = cudaSuccess;
  dev_upload(e, s.d_s0_rows, dr.data(), sizeof(S0RowDev) * dr.size());
  dev_upload(e, s.d_s0_jobs, dj.data(), sizeof(S0JobDev) * dj.size());
  dev_alloc(e, s.d_s0_desc, sizeof(uint2) * blk);
  dev_alloc(e, s.d_s0_adj, sizeof(uint16_t) * px);
  dev_alloc(e, s.d_s0_nodes, sizeof(uint2) * 2 * nodes);
  dev_alloc(e, s.d_s0_carry, sizeof(uint32_t) * carry);
  dev_alloc(e, s.d_s0_rowfail, sizeof(uint32_t) * dr.size());
  dev_alloc(e, s.d_s0_jobfail, sizeof(uint32_t) * (size_t)njobs);
  dev_alloc(e, s.d_job_res, sizeof(uint2) * (size_t)njobs);
  host_alloc(e, s.h_job_res, sizeof(uint2) * (size_t)njobs);
  if (e != cudaSuccess)
    return set_err(ctx, RSB200_ERR_CUDA, "samsung0 plan allocation failed: %s", cudaGetErrorString(e));
  p->launches_per_run = 6 + s.s0_rounds;
  *out = holder.release();
  return RSB200_OK;
}

static int run(const rsb200_plan* p, const SamsungV0Plan& s, const uint8_t* in, uint64_t, uint8_t* outp,
               cudaStream_t st) {
  CUDA_TRY(p->ctx, cudaMemsetAsync(s.d_s0_jobfail.get(), 0xFF, sizeof(uint32_t) * (size_t)p->nunits, st));
  const uint32_t nj = (uint32_t)p->nunits;
  s0_walk_kernel<<<(s.s0_nrows + S0W_NT - 1) / S0W_NT, S0W_NT, 0, st>>>(
      in, s.d_s0_rows.get(), s.s0_nrows, s.d_s0_jobs.get(), s.d_s0_desc.get(), s.d_s0_rowfail.get(), s.d_s0_jobfail.get());
  s0_diff_kernel<<<(s.s0_nrows + S0D_NT / 32 - 1) / (S0D_NT / 32), S0D_NT, 0, st>>>(
      in, s.d_s0_rows.get(), s.s0_nrows, s.d_s0_jobs.get(), s.d_s0_desc.get(), s.d_s0_adj.get());
  s0_node_kernel<<<dim3((s.s0_max_nodes + S0N_NT - 1) / S0N_NT, nj), S0N_NT, 0, st>>>(
      s.d_s0_jobs.get(), s.d_s0_desc.get(), s.d_s0_adj.get(), s.d_s0_nodes.get());
  uint2* src = s.d_s0_nodes.get();
  uint2* dst = s.d_s0_nodes.get() + s.s0_nnodes;
  for (int r = 0; r < s.s0_rounds; ++r) {
    s0_jump_kernel<<<(s.s0_nnodes + S0N_NT - 1) / S0N_NT, S0N_NT, 0, st>>>(src, dst, s.s0_nnodes);
    std::swap(src, dst);
  }
  const dim3 tiles((s.s0_max_w + S0C_NT - 1) / S0C_NT, s.s0_max_tiles, nj);
  s0_scan_kernel<<<tiles, S0C_NT, 0, st>>>(s.d_s0_jobs.get(), s.d_s0_desc.get(), s.d_s0_adj.get(), src, s.d_s0_carry.get());
  s0_carry_kernel<<<dim3((2 * s.s0_max_w + S0C_NT - 1) / S0C_NT, nj), S0C_NT, 0, st>>>(s.d_s0_jobs.get(),
                                                                                     s.d_s0_carry.get());
  s0_store_kernel<<<tiles, S0C_NT, 0, st>>>(s.d_s0_jobs.get(), s.d_s0_desc.get(), s.d_s0_adj.get(), src, s.d_s0_carry.get(),
                                            s.d_s0_rowfail.get(), s.d_s0_jobfail.get(), outp, s.d_job_res.get());
  CUDA_TRY(p->ctx, cudaGetLastError());
  p->ctx->launches += (uint64_t)p->launches_per_run;
  return RSB200_OK;
}

static int results(const rsb200_plan* p, SamsungV0Plan& s, rsb200_scan_result* out, int n) {
  static const char* const msgs[7] = {"", "Bit length less than 0.", "Bit Length more than 16.",
                                      "Upward prediction for the first two rows. Raw corrupt",
                                      "Upward prediction for the last block of pixels. Raw corrupt",
                                      "Buffer overflow read in BitStreamer",
                                      "Bit stream size is smaller than MaxProcessBytes"};
  return report_jobs(
      p, s.d_job_res, s.h_job_res, out, n, [&](int i) { return rsb200_scan_result{s.h_job_res[i].x, s.h_job_res[i].y}; },
      [&](int i, const rsb200_scan_result& r) {
        set_err(p->ctx, (int)r.status, "job %d: %s (row %u, block %u)", i, msgs[std::min(r.consumed >> 24, 6u)],
                (r.consumed >> 9) & 0x7FFFu, r.consumed & 0x1FFu);
      });
}

static const char* kernels(const rsb200_plan*, const SamsungV0Plan&) {
  return "s0_walk_kernel + s0_diff_kernel + s0_node_kernel + s0_jump_kernel + s0_scan_kernel + s0_carry_kernel + "
         "s0_store_kernel";
}

// ------------------------------------------------------------------
// Samsung V2: one strip per frame, a stream per row at 16-byte boundaries (samsung2.cuh)
// ------------------------------------------------------------------
extern "C" int rsb200_samsung2_plan_create(rsb200_ctx* ctx, const rsb200_samsung2_job* jobs, int njobs,
                                           rsb200_plan** out) {
  if (!ctx || !jobs || njobs <= 0 || !out)
    return set_err(ctx, RSB200_ERR_ARG, "samsung2_plan_create: bad arguments");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  for (int i = 0; i < njobs; ++i) {
    const rsb200_samsung2_job& j = jobs[i];
    // SamsungV2Decompressor ctor (SamsungV2Decompressor.cpp:88-142), in its order
    if (j.bits != 12 && j.bits != 14)
      return set_err(ctx, RSB200_ERR_RDE, "job %d: Unexpected bit per pixel (%u)", i, j.bits);
    if (j.in_size < 16)
      return set_err(ctx, RSB200_ERR_IOE, "job %d: Out of bounds access in ByteStream", i);
    const uint32_t depth = s2_header_bits(j.header, 20, 4) + 1;
    if (depth != j.bits)
      return set_err(ctx, RSB200_ERR_RDE, "job %d: Bit depth mismatch with container, %u vs %u", i, depth, j.bits);
    const uint32_t flags = s2_header_bits(j.header, 84, 4);
    if (flags > 7)
      return set_err(ctx, RSB200_ERR_RDE, "job %d: Invalid opt flags %x", i, flags);
    const uint32_t hw = s2_header_bits(j.header, 32, 16), hh = s2_header_bits(j.header, 48, 16);
    if (hw == 0 || hh == 0 || hw % 16 != 0 || hw > 6496 || hh > 4336)
      return set_err(ctx, RSB200_ERR_RDE, "job %d: Unexpected image dimensions found: (%i; %i)", i, (int)hw, (int)hh);
    if ((int32_t)hw != j.width || (int32_t)hh != j.height)
      return set_err(ctx, RSB200_ERR_RDE, "job %d: EXIF image dimensions do not match dimensions from raw header", i);
    // the reconstruction stores two pixels as one 32-bit word
    if (j.in_size >= (1u << 28) || (uint64_t)j.width * 2 > j.out_pitch || (j.out_offset % 4) || (j.out_pitch % 4) ||
        j.reserved)
      return set_err(ctx, RSB200_ERR_ARG, "samsung2 job %d: malformed descriptor", i);
  }
  PlanHolder holder = new_plan(ctx);
  if (!holder)
    return RSB200_ERR_CUDA;
  rsb200_plan* p = holder.get();
  SamsungV2Plan& s = p->state.emplace<SamsungV2Plan>();
  p->nunits = njobs;
  std::vector<S2FrameDev> fr((size_t)njobs);
  std::vector<uint32_t> starts((size_t)njobs * 4);
  S2Totals t;
  for (int i = 0; i < njobs; ++i) {
    const rsb200_samsung2_job& j = jobs[i];
    S2FrameDev& f = fr[(size_t)i];
    s2_place_frame(f, t, starts.data(), (uint32_t)njobs, (uint32_t)i, j.in_offset, j.in_size, j.header, j.bits,
                   (uint32_t)j.width, (uint32_t)j.height, j.out_offset, j.out_pitch);
    if (t.tab >= (1ull << 31) || t.rows >= (1ull << 31))
      return set_err(ctx, RSB200_ERR_ARG, "samsung2 plan: too many frames for one plan");
    p->in_bytes += j.in_size;
    p->out_bytes += (uint64_t)f.w * f.h * 2;
    p->pixels += (uint64_t)f.w * f.h;
    p->need_in = std::max<uint64_t>(p->need_in, sat_add(j.in_offset, j.in_size));
    p->need_out = std::max<uint64_t>(p->need_out, sat_add(j.out_offset, ((uint64_t)f.h - 1) * j.out_pitch + 2ull * f.w));
  }
  const uint64_t tab = t.tab, jump = t.jump, rows = t.rows, cps = t.cps, desc = t.desc, px = t.px;
  s.s2_ntab = (uint32_t)tab;
  s.s2_njump = (uint32_t)jump;
  s.s2_nrows = (uint32_t)rows;
  s.s2_ncp = (uint32_t)cps;
  cudaError_t e = cudaSuccess;
  dev_upload(e, s.d_s2_frames, fr.data(), sizeof(S2FrameDev) * fr.size());
  dev_upload(e, s.d_s2_starts, starts.data(), sizeof(uint32_t) * starts.size());
  dev_alloc(e, s.d_s2_tab, sizeof(uint32_t) * tab);
  dev_alloc(e, s.d_s2_jump, sizeof(uint32_t) * 2 * jump);
  dev_alloc(e, s.d_s2_rowstart, sizeof(uint32_t) * rows);
  dev_alloc(e, s.d_s2_cp, sizeof(uint32_t) * cps);
  dev_alloc(e, s.d_s2_ncp, sizeof(uint32_t) * (size_t)njobs);
  dev_alloc(e, s.d_s2_fail, sizeof(uint2) * (size_t)njobs);
  dev_alloc(e, s.d_s2_desc, sizeof(uint2) * desc);
  dev_alloc(e, s.d_s2_px, sizeof(int16_t) * px);
  dev_alloc(e, s.d_job_res, sizeof(uint2) * (size_t)njobs);
  host_alloc(e, s.h_job_res, sizeof(uint2) * (size_t)njobs);
  if (e != cudaSuccess)
    return set_err(ctx, RSB200_ERR_CUDA, "samsung2 plan allocation failed: %s", cudaGetErrorString(e));
  p->launches_per_run = 7 + S2_JUMP;
  *out = holder.release();
  return RSB200_OK;
}

static int run(const rsb200_plan* p, const SamsungV2Plan& s, const uint8_t* in, uint64_t, uint8_t* outp,
               cudaStream_t st) {
  const uint32_t nf = (uint32_t)p->nunits;
  const uint32_t* starts = s.d_s2_starts.get();
  s2_cand_kernel<<<(s.s2_ntab + S2W_NT - 1) / S2W_NT, S2W_NT, 0, st>>>(in, s.d_s2_frames.get(), starts, nf, s.s2_ntab,
                                                                         s.d_s2_tab.get());
  uint32_t* src = s.d_s2_jump.get();
  uint32_t* dst = s.d_s2_jump.get() + s.s2_njump;
  const uint32_t gj = (s.s2_njump + S2J_NT - 1) / S2J_NT;
  s2_pair_kernel<<<gj, S2J_NT, 0, st>>>(s.d_s2_frames.get(), starts + nf, nf, s.s2_njump, s.d_s2_tab.get(), src);
  for (int r = 0; r < S2_JUMP; ++r) {
    s2_double_kernel<<<gj, S2J_NT, 0, st>>>(s.d_s2_frames.get(), starts + nf, nf, s.s2_njump, src, dst);
    std::swap(src, dst);
  }
  s2_coarse_kernel<<<(nf + S2J_NT - 1) / S2J_NT, S2J_NT, 0, st>>>(s.d_s2_frames.get(), nf, s.d_s2_tab.get(), src,
                                                                   s.d_s2_rowstart.get(), s.d_s2_cp.get(), s.d_s2_ncp.get(),
                                                                   s.d_s2_fail.get());
  s2_fine_kernel<<<(s.s2_ncp + S2J_NT - 1) / S2J_NT, S2J_NT, 0, st>>>(s.d_s2_frames.get(), starts + 3 * nf, nf, s.s2_ncp,
                                                                        s.d_s2_tab.get(), s.d_s2_cp.get(), s.d_s2_ncp.get(),
                                                                        s.d_s2_rowstart.get(), s.d_s2_fail.get());
  s2_desc_kernel<<<(s.s2_nrows + S2W_NT - 1) / S2W_NT, S2W_NT, 0, st>>>(
      in, s.d_s2_frames.get(), starts + 2 * nf, nf, s.s2_nrows, s.d_s2_rowstart.get(), s.d_s2_fail.get(), s.d_s2_desc.get());
  s2_diff_kernel<<<s.s2_nrows, S2X_NT, 0, st>>>(in, s.d_s2_frames.get(), starts + 2 * nf, nf, s.d_s2_fail.get(), s.d_s2_desc.get(),
                                                 s.d_s2_px.get());
  s2_recon_kernel<<<nf, S2R_NT, 0, st>>>(s.d_s2_frames.get(), s.d_s2_fail.get(), s.d_s2_desc.get(), s.d_s2_px.get(), outp,
                                         s.d_job_res.get());
  CUDA_TRY(p->ctx, cudaGetLastError());
  p->ctx->launches += (uint64_t)p->launches_per_run;
  return RSB200_OK;
}

static int results(const rsb200_plan* p, SamsungV2Plan& s, rsb200_scan_result* out, int n) {
  // SamsungV2Decompressor.cpp:180-247, 329-350; BitStreamer.h; ByteStream::check
  static const char* const msgs[9] = {"", "At start of image and motion isn't 7. File corrupted?",
                                      "Bad motion %u at the beginning of the row",
                                      "Bad motion %u at the end of the row",
                                      "Difference bits underflow. File corrupted?",
                                      "Too many difference bits (%u). File corrupted?",
                                      "Buffer overflow read in BitStreamer",
                                      "Bit stream size is smaller than MaxProcessBytes",
                                      "Out of bounds access in ByteStream"};
  return report_jobs(
      p, s.d_job_res, s.h_job_res, out, n, [&](int i) { return rsb200_scan_result{s.h_job_res[i].x, s.h_job_res[i].y}; },
      [&](int i, const rsb200_scan_result& r) {
        char m[96];
        snprintf(m, sizeof m, msgs[std::min(r.consumed >> 28, 8u)], (r.consumed >> 22) & 31u);
        set_err(p->ctx, (int)r.status, "job %d: %s (row %u, block %u)", i, m, (r.consumed >> 9) & 0x1FFFu,
                r.consumed & 0x1FFu);
      });
}

static const char* kernels(const rsb200_plan*, const SamsungV2Plan&) {
  return "s2_cand_kernel + s2_pair_kernel + s2_double_kernel + s2_coarse_kernel + s2_fine_kernel + s2_desc_kernel + "
         "s2_diff_kernel + s2_recon_kernel";
}

// ------------------------------------------------------------------
// Kodak DCR: segments of up to 256 pixels, row starts resolved from every candidate (kodak.cuh)
// ------------------------------------------------------------------
extern "C" int rsb200_kodak_plan_create(rsb200_ctx* ctx, const rsb200_kodak_job* jobs, int njobs,
                                        const uint16_t* tables, int ntables, rsb200_plan** out) {
  if (!ctx || !jobs || njobs <= 0 || ntables < 0 || (ntables > 0 && !tables) || !out)
    return set_err(ctx, RSB200_ERR_ARG, "kodak_plan_create: bad arguments");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  for (int i = 0; i < njobs; ++i) {
    const rsb200_kodak_job& j = jobs[i];
    // KodakDecompressor ctor (KodakDecompressor.cpp:50-64), in its order
    if (j.width <= 0 || j.height <= 0 || j.width % 4 != 0 || j.width > (int32_t)KD_MAXW || j.height > (int32_t)KD_MAXH)
      return set_err(ctx, RSB200_ERR_RDE, "job %d: Unexpected image dimensions found: (%d; %d)", i, j.width, j.height);
    if (j.bps != 10 && j.bps != 12)
      return set_err(ctx, RSB200_ERR_RDE, "job %d: Unexpected bits per sample: %i", i, j.bps);
    if ((uint64_t)j.in_size < (uint64_t)j.width * (uint64_t)j.height / 2u)
      return set_err(ctx, RSB200_ERR_IOE, "job %d: Out of bounds access in ByteStream", i);
    // the stores write two pixels as one 32-bit word
    if (j.in_size > KD_MAX_IN || (uint64_t)j.width * 2 > j.out_pitch || (j.out_offset % 4) || (j.out_pitch % 4) ||
        j.table < -1 || j.table >= ntables || j.reserved)
      return set_err(ctx, RSB200_ERR_ARG, "kodak job %d: malformed descriptor", i);
  }
  PlanHolder holder = new_plan(ctx);
  if (!holder)
    return RSB200_ERR_CUDA;
  rsb200_plan* p = holder.get();
  KodakPlan& s = p->state.emplace<KodakPlan>();
  p->nunits = njobs;
  std::vector<KdFrameDev> fr((size_t)njobs);
  std::vector<uint32_t> starts((size_t)njobs * 4);
  KdTotals t;
  for (int i = 0; i < njobs; ++i) {
    const rsb200_kodak_job& j = jobs[i];
    kd_place_frame(fr[(size_t)i], t, starts.data(), (uint32_t)njobs, (uint32_t)i, j.in_offset, j.in_size,
                   (uint32_t)j.width, (uint32_t)j.height, (uint32_t)j.bps,
                   j.table < 0 ? ~0u : (uint32_t)j.table * 65536u, j.out_offset, j.out_pitch);
    if (t.q >= (1ull << 31) || t.cand >= (1ull << 31) || t.segs >= (1ull << 31))
      return set_err(ctx, RSB200_ERR_ARG, "kodak plan: too many frames for one plan");
    p->in_bytes += j.in_size;
    p->out_bytes += (uint64_t)j.width * j.height * 2;
    p->pixels += (uint64_t)j.width * j.height;
    p->need_in = std::max<uint64_t>(p->need_in, sat_add(j.in_offset, j.in_size));
    p->need_out = std::max<uint64_t>(p->need_out,
                                     sat_add(j.out_offset, ((uint64_t)j.height - 1) * j.out_pitch + 2ull * j.width));
  }
  s.kd_ntiles = (uint32_t)t.tiles;
  s.kd_ncand = (uint32_t)t.cand;
  s.kd_ncp = (uint32_t)t.cps;
  s.kd_nsegs = (uint32_t)t.segs;
  cudaError_t e = cudaSuccess;
  dev_upload(e, s.d_kd_frames, fr.data(), sizeof(KdFrameDev) * fr.size());
  dev_upload(e, s.d_kd_starts, starts.data(), sizeof(uint32_t) * starts.size());
  dev_upload(e, s.d_kd_tables, tables, sizeof(uint16_t) * 65536 * (size_t)ntables);
  dev_alloc(e, s.d_kd_tsum, sizeof(uint32_t) * t.tiles);
  dev_alloc(e, s.d_kd_q, sizeof(uint32_t) * t.q);
  dev_alloc(e, s.d_kd_tab, sizeof(uint32_t) * t.cand);
  dev_alloc(e, s.d_kd_jump, sizeof(uint32_t) * 2 * t.cand);
  dev_alloc(e, s.d_kd_rowstart, sizeof(uint32_t) * t.rows);
  dev_alloc(e, s.d_kd_cp, sizeof(uint32_t) * t.cps);
  dev_alloc(e, s.d_kd_ncp, sizeof(uint32_t) * (size_t)njobs);
  dev_alloc(e, s.d_kd_fail, sizeof(uint2) * (size_t)njobs);
  dev_alloc(e, s.d_kd_key, sizeof(uint32_t) * (size_t)njobs);
  dev_alloc(e, s.d_job_res, sizeof(uint2) * (size_t)njobs);
  host_alloc(e, s.h_job_res, sizeof(uint2) * (size_t)njobs);
  dev_alloc(e, s.d_kd_values, sizeof(int32_t) * (size_t)njobs);
  if (e != cudaSuccess)
    return set_err(ctx, RSB200_ERR_CUDA, "kodak plan allocation failed: %s", cudaGetErrorString(e));
  p->launches_per_run = 8 + KD_JUMP;
  *out = holder.release();
  return RSB200_OK;
}

static int run(const rsb200_plan* p, const KodakPlan& s, const uint8_t* in, uint64_t, uint8_t* outp, cudaStream_t st) {
  const uint32_t nf = (uint32_t)p->nunits;
  const uint32_t* starts = s.d_kd_starts.get();
  const KdFrameDev* fr = s.d_kd_frames.get();
  kd_tsum_kernel<<<s.kd_ntiles, KD_NT, 0, st>>>(in, fr, starts, nf, s.d_kd_tsum.get());
  kd_tscan_kernel<<<nf, KD_NT, 0, st>>>(fr, s.d_kd_tsum.get());
  kd_prefix_kernel<<<s.kd_ntiles, KD_NT, 0, st>>>(in, fr, starts, nf, s.d_kd_tsum.get(), s.d_kd_q.get());
  const uint32_t gc = (s.kd_ncand + KD_NT - 1) / KD_NT;
  kd_cand_kernel<<<gc, KD_NT, 0, st>>>(fr, starts + nf, nf, s.kd_ncand, s.d_kd_q.get(), s.d_kd_tab.get());
  const uint32_t* src = s.d_kd_tab.get();
  uint32_t* dst = s.d_kd_jump.get();
  for (int r = 0; r < KD_JUMP; ++r) {
    kd_double_kernel<<<gc, KD_NT, 0, st>>>(fr, starts + nf, nf, s.kd_ncand, src, dst);
    src = dst;
    dst = dst == s.d_kd_jump.get() ? s.d_kd_jump.get() + s.kd_ncand : s.d_kd_jump.get();
  }
  kd_coarse_kernel<<<(nf + KD_NT - 1) / KD_NT, KD_NT, 0, st>>>(fr, nf, src, s.d_kd_cp.get(), s.d_kd_ncp.get(),
                                                               s.d_kd_fail.get(), s.d_kd_key.get());
  kd_fine_kernel<<<(s.kd_ncp + KD_NT - 1) / KD_NT, KD_NT, 0, st>>>(fr, starts + 2 * nf, nf, s.kd_ncp, s.d_kd_tab.get(),
                                                                   s.d_kd_cp.get(), s.d_kd_ncp.get(),
                                                                   s.d_kd_rowstart.get(), s.d_kd_fail.get());
  const uint32_t gs = (s.kd_nsegs + KD_NT / 32 - 1) / (KD_NT / 32);
  kd_check_kernel<<<gs, KD_NT, 0, st>>>(in, fr, starts + 3 * nf, nf, s.kd_nsegs, s.d_kd_q.get(), s.d_kd_rowstart.get(),
                                        s.d_kd_fail.get(), s.d_kd_key.get());
  kd_store_kernel<<<gs, KD_NT, 0, st>>>(in, fr, starts + 3 * nf, nf, s.kd_nsegs, s.d_kd_q.get(), s.d_kd_rowstart.get(),
                                        s.d_kd_fail.get(), s.d_kd_key.get(), s.d_kd_tables.get(), outp,
                                        s.d_job_res.get(), s.d_kd_values.get());
  CUDA_TRY(p->ctx, cudaGetLastError());
  p->ctx->launches += (uint64_t)p->launches_per_run;
  return RSB200_OK;
}

static int results(const rsb200_plan* p, KodakPlan& s, rsb200_scan_result* out, int n) {
  // KodakDecompressor.cpp:137-138; Buffer.h:78-83
  return report_jobs(
      p, s.d_job_res, s.h_job_res, out, n, [&](int i) { return rsb200_scan_result{s.h_job_res[i].x, s.h_job_res[i].y}; },
      [&](int i, const rsb200_scan_result& r) {
        set_err(p->ctx, (int)r.status, "job %d: %s (row %u, column %u)", i,
                r.status == RSB200_ERR_RDE ? "Value out of bounds" : "Buffer overflow: image file may be truncated",
                (r.consumed >> 13) & 0x7FFFu, r.consumed & 0x1FFFu);
      });
}

static const char* kernels(const rsb200_plan*, const KodakPlan&) {
  return "kd_tsum_kernel + kd_tscan_kernel + kd_prefix_kernel + kd_cand_kernel + kd_double_kernel + kd_coarse_kernel + "
         "kd_fine_kernel + kd_check_kernel + kd_store_kernel";
}

extern "C" int rsb200_kodak_plan_values(rsb200_plan* p, int32_t* values, int n) {
  if (!p || (n > 0 && !values))
    return RSB200_ERR_ARG;
  rsb200_ctx* ctx = p->ctx;
  const KodakPlan* s = std::get_if<KodakPlan>(&p->state);
  if (!s)
    return set_err(ctx, RSB200_ERR_ARG, "kodak_plan_values: not a Kodak plan");
  if (!p->ran)
    return set_err(ctx, RSB200_ERR_ARG, "kodak_plan_values: plan has not been run");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  CUDA_TRY(ctx, cudaStreamSynchronize(p->last_stream));
  const int take = std::min(n, p->nunits);
  if (take > 0)
    CUDA_TRY(ctx, cudaMemcpy(values, s->d_kd_values.get(), sizeof(int32_t) * (size_t)take, cudaMemcpyDeviceToHost));
  return RSB200_OK;
}

// ------------------------------------------------------------------
// GoPro VC-5: band payloads cut into segments, exact entries by a scan of candidate walks (vc5.cuh)
// ------------------------------------------------------------------
extern "C" int rsb200_vc5_plan_create(rsb200_ctx* ctx, const rsb200_vc5_code* codes, int ncodes,
                                      const rsb200_vc5_job* jobs, int njobs, const rsb200_vc5_band* bands, int nbands,
                                      rsb200_plan** out) {
  if (!ctx || !codes || !jobs || njobs <= 0 || njobs > 16383 || !bands || nbands <= 0 || !out)
    return set_err(ctx, RSB200_ERR_ARG, "vc5_plan_create: bad arguments");
  std::vector<uint32_t> code;
  if (!vc5_build_code(codes, ncodes, code))
    return set_err(ctx, RSB200_ERR_ARG, "vc5_plan_create: the codebook is not a complete prefix code within limits");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  PlanHolder holder = new_plan(ctx);
  if (!holder)
    return RSB200_ERR_CUDA;
  rsb200_plan* p = holder.get();
  Vc5Plan& s = p->state.emplace<Vc5Plan>();
  p->nunits = njobs;
  Vc5Layout L;
  const char* why = nullptr;
  const int bad = vc5_layout(jobs, njobs, bands, nbands, L, &why);
  if (bad >= 0)
    return set_err(ctx, RSB200_ERR_ARG, "vc5 job %d: %s", bad, why);
  for (int i = 0; i < njobs; ++i) {
    const rsb200_vc5_job& j = jobs[i];
    for (int b = 0; b < 40; ++b) {
      const rsb200_vc5_band& band = bands[j.first_band + (uint32_t)b];
      p->in_bytes += band.in_size;
      p->need_in = std::max<uint64_t>(p->need_in, sat_add(band.in_offset, band.in_size));
    }
    p->out_bytes += (uint64_t)j.width * j.height * 2;
    p->pixels += (uint64_t)j.width * j.height;
    p->need_out = std::max<uint64_t>(p->need_out,
                                     sat_add(j.out_offset, ((uint64_t)j.height - 1) * j.out_pitch + 2ull * j.width));
  }
  s.ncoef = L.ncoef;
  s.nsegs = (uint32_t)L.seg_band.size();
  s.rounds = L.rounds;
  s.max_low = L.max_low, s.max_rec[0] = L.max_rec[0], s.max_rec[1] = L.max_rec[1], s.max_quads = L.max_quads;
  const std::vector<uint16_t> luts = vc5_luts();
  cudaError_t e = cudaSuccess;
  dev_upload(e, s.d_code, code.data(), sizeof(uint32_t) * code.size());
  dev_upload(e, s.d_frames, L.frames.data(), sizeof(Vc5FrameDev) * L.frames.size());
  dev_upload(e, s.d_bands, L.bands.data(), sizeof(Vc5BandDev) * L.bands.size());
  dev_upload(e, s.d_seg_band, L.seg_band.data(), sizeof(uint32_t) * L.seg_band.size());
  dev_upload(e, s.d_luts, luts.data(), sizeof(uint16_t) * luts.size());
  dev_alloc(e, s.d_map, sizeof(uint2) * 2 * (size_t)s.nsegs * VC5_CAND);
  dev_alloc(e, s.d_err, sizeof(unsigned long long) * L.bands.size());
  dev_alloc(e, s.d_coef, sizeof(int16_t) * L.ncoef);
  dev_alloc(e, s.d_job_res, sizeof(uint2) * (size_t)njobs);
  host_alloc(e, s.h_job_res, sizeof(uint2) * (size_t)njobs);
  if (e != cudaSuccess)
    return set_err(ctx, RSB200_ERR_CUDA, "vc5 plan allocation failed: %s", cudaGetErrorString(e));
  p->launches_per_run = 7 + (int)s.rounds;
  *out = holder.release();
  return RSB200_OK;
}

static int run(const rsb200_plan* p, const Vc5Plan& s, const uint8_t* in, uint64_t, uint8_t* outp, cudaStream_t st) {
  const uint32_t nf = (uint32_t)p->nunits;
  auto blocks = [](uint64_t n) { return (uint32_t)std::max<uint64_t>(1, (n + VC5_NT - 1) / VC5_NT); };
  const Vc5FrameDev* fr = s.d_frames.get();
  const Vc5BandDev* bd = s.d_bands.get();
  int16_t* coef = s.d_coef.get();
  CUDA_TRY(p->ctx, cudaMemsetAsync(s.d_err.get(), 0xFF, sizeof(unsigned long long) * 40 * nf, st));
  CUDA_TRY(p->ctx, cudaMemsetAsync(coef, 0, sizeof(int16_t) * s.ncoef, st));
  vc5_lowpass_kernel<<<dim3(blocks(s.max_low), 4 * nf), VC5_NT, 0, st>>>(in, bd, coef);
  const uint32_t gm = blocks((uint64_t)s.nsegs * VC5_CAND);
  uint2* a = s.d_map.get();
  uint2* b = a + (size_t)s.nsegs * VC5_CAND;
  vc5_walk_kernel<<<gm, VC5_NT, 0, st>>>(in, bd, s.d_seg_band.get(), s.nsegs, s.d_code.get(), a);
  for (uint32_t r = 0; r < s.rounds; ++r) {
    vc5_scan_kernel<<<gm, VC5_NT, 0, st>>>(bd, s.d_seg_band.get(), s.nsegs, r, a, b);
    std::swap(a, b);
  }
  vc5_store_kernel<<<blocks(s.nsegs), VC5_NT, 0, st>>>(in, bd, s.d_seg_band.get(), s.nsegs, s.d_code.get(), a,
                                                       s.d_err.get(), coef);
  vc5_result_kernel<<<blocks(nf), VC5_NT, 0, st>>>(fr, nf, bd, s.d_err.get(), s.d_job_res.get());
  vc5_recon_kernel<<<dim3(blocks(s.max_rec[0]), 4 * nf), VC5_NT, 0, st>>>(fr, bd, 0, coef);
  vc5_recon_kernel<<<dim3(blocks(s.max_rec[1]), 4 * nf), VC5_NT, 0, st>>>(fr, bd, 1, coef);
  vc5_final_kernel<<<dim3(blocks(s.max_quads), nf), VC5_NT, 0, st>>>(fr, bd, coef, s.d_luts.get(),
                                                                       s.d_job_res.get(), outp);
  CUDA_TRY(p->ctx, cudaGetLastError());
  p->ctx->launches += (uint64_t)p->launches_per_run;
  return RSB200_OK;
}

static int results(const rsb200_plan* p, Vc5Plan& s, rsb200_scan_result* out, int n) {
  // VC5Decompressor.cpp:683-742, :849-873; BitStreamer.h:58-59, :125-127
  static const char* const text[7] = {"",
                                      "Impossible RLV value given current quantum",
                                      "Got EndOfBand marker while looking for next pixel",
                                      "Not all pixels consumed?",
                                      "EndOfBand marker not found",
                                      "Bit stream size is smaller than MaxProcessBytes",
                                      "Buffer overflow read in BitStreamer"};
  return report_jobs(
      p, s.d_job_res, s.h_job_res, out, n, [&](int i) { return rsb200_scan_result{s.h_job_res[i].x, s.h_job_res[i].y}; },
      [&](int i, const rsb200_scan_result& r) {
        set_err(p->ctx, (int)r.status, "job %d: Too many errors encountered. Giving up. First Error:\n%s (channel %u, subband %u)",
                i, text[std::min<uint32_t>(r.consumed >> 28, 6u)], (r.consumed >> 4) & 15u, r.consumed & 15u);
      });
}

static const char* kernels(const rsb200_plan*, const Vc5Plan&) {
  return "vc5_lowpass_kernel + vc5_walk_kernel + vc5_scan_kernel + vc5_store_kernel + vc5_result_kernel + "
         "vc5_recon_kernel + vc5_final_kernel";
}

// ------------------------------------------------------------------
// Panasonic V5 / V6 / V7 (K7)
// ------------------------------------------------------------------
extern "C" int rsb200_pana_plan_create(rsb200_ctx* ctx, const rsb200_pana_job* jobs, int njobs,
                                       rsb200_plan** out) {
  if (!ctx || !jobs || njobs <= 0 || !out)
    return set_err(ctx, RSB200_ERR_ARG, "pana_plan_create: bad arguments");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  PlanHolder holder = new_plan(ctx);
  if (!holder)
    return RSB200_ERR_CUDA;
  rsb200_plan* p = holder.get();
  PanaPlan& s = p->state.emplace<PanaPlan>();
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
    if (!ok)
      return set_err(ctx, RSB200_ERR_ARG, "pana job %d: malformed descriptor", i);
    PanaJobDev d;
    memset(&d, 0, sizeof d);
    d.in_offset = j.in_offset;
    d.out_offset = j.out_offset;
    d.out_pitch = j.out_pitch;
    d.width = j.width;
    d.height = j.height;
    d.units = (uint32_t)units;
    s.bad.slot.push_back(-1);
    if (j.version == 4) {
      d.split = j.section_split_offset;
      if (!j.zero_is_not_bad) {
        s.bad.slot.back() = s.bad.nslots;
        d.zero_slot = (uint32_t)++s.bad.nslots;
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
    if (n >= 0xFFFF0000ull)
      return set_err(ctx, RSB200_ERR_ARG, "pana plan: too many blocks");
    g.total_units = (uint32_t)n;
    g.njobs = (int)kv.second.size();
    cudaError_t e = cudaSuccess;
    dev_upload(e, g.d_jobs, kv.second.data(), sizeof(PanaJobDev) * kv.second.size());
    if (e != cudaSuccess)
      return set_err(ctx, RSB200_ERR_CUDA, "pana plan upload failed: %s", cudaGetErrorString(e));
    s.groups.push_back(std::move(g));
  }
  if (s.bad.nslots) {
    cudaError_t e = cudaSuccess;
    dev_alloc(e, s.bad.d_count, sizeof(uint32_t) * (size_t)s.bad.nslots);
    dev_alloc(e, s.bad.d_list, sizeof(uint32_t) * (size_t)PANA_ZERO_CAP * (size_t)s.bad.nslots);
    if (e != cudaSuccess)
      return set_err(ctx, RSB200_ERR_CUDA, "pana plan: bad-pixel lists: %s", cudaGetErrorString(e));
  }
  p->launches_per_run = (int)s.groups.size();
  *out = holder.release();
  return RSB200_OK;
}

static_assert(PANA_ZERO_CAP == RSB200_PANA_BAD_CAP, "header and kernel disagree");

static cudaError_t run_pana_group(const PanaPlan& s, const PanaGroup& g, const uint8_t* in,
                                  uint8_t* outp, cudaStream_t st) {
  const uint32_t nb = (g.total_units + PANA_NT - 1) / PANA_NT;
#define RSB_PANA(V, B)                                                                     \
  pana_kernel<V, B><<<nb, PANA_NT, 0, st>>>(in, outp, g.d_jobs.get(), g.njobs, g.total_units,    \
                                            s.bad.d_count.get(), s.bad.d_list.get())
  if (g.version == 4) {
    if (s.bad.nslots) {
      const cudaError_t e = cudaMemsetAsync(s.bad.d_count.get(), 0,
                                            sizeof(uint32_t) * (size_t)s.bad.nslots, st);
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

static int run(const rsb200_plan* p, const PanaPlan& s, const uint8_t* in, uint64_t, uint8_t* outp, cudaStream_t st) {
  rsb200_ctx* ctx = p->ctx;
  for (const PanaGroup& g : s.groups) {
    CUDA_TRY(ctx, run_pana_group(s, g, in, outp, st));
    ctx->launches++;
  }
  return RSB200_OK;
}

static int results(const rsb200_plan* p, PanaPlan&, rsb200_scan_result* out, int n) { return report_ok(p, out, n); }
static const char* kernels(const rsb200_plan*, const PanaPlan&) { return "(not an LJPEG plan)"; }

// ------------------------------------------------------------------
// Sony ARW2 (K6)
// ------------------------------------------------------------------
extern "C" int rsb200_arw2_plan_create(rsb200_ctx* ctx, const rsb200_arw2_job* jobs, int njobs,
                                       const uint16_t* tables, int ntables, int dither,
                                       rsb200_plan** out) {
  if (!ctx || !jobs || njobs <= 0 || !out || ntables < 0 || (ntables > 0 && !tables))
    return set_err(ctx, RSB200_ERR_ARG, "arw2_plan_create: bad arguments");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  PlanHolder holder = new_plan(ctx);
  if (!holder)
    return RSB200_ERR_CUDA;
  rsb200_plan* p = holder.get();
  Arw2Plan& s = p->state.emplace<Arw2Plan>();
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
    if (!ok)
      return set_err(ctx, RSB200_ERR_ARG, "arw2 job %d: malformed descriptor", i);
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
  if (any_table && any_plain)
    return set_err(ctx, RSB200_ERR_ARG, "arw2 plan: jobs with and without a table cannot be mixed");
  if (groups >= 0xFFFF0000ull)
    return set_err(ctx, RSB200_ERR_ARG, "arw2 plan: too many blocks");
  s.arw2_groups = (uint32_t)groups;
  s.arw2_mode = !any_table ? 0 : (dither ? 2 : 1);
  s.arw2_ntables = any_table ? ntables : 0;
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
    dev_upload(e, s.d_arw2_jobs, dev.data(), sizeof(Arw2JobDev) * dev.size());
    dev_upload(e, s.d_arw2_tables, tcut.data(), tcut.size() * sizeof(uint16_t), 16);
    dev_alloc(e, s.d_job_bad, sizeof(uint32_t) * (size_t)njobs);
    host_alloc(e, s.h_job_bad, sizeof(uint32_t) * (size_t)njobs);
    if (e != cudaSuccess)
      return set_err(ctx, RSB200_ERR_CUDA, "arw2 plan upload failed: %s", cudaGetErrorString(e));
  }
  p->launches_per_run = 1;
  *out = holder.release();
  return RSB200_OK;
}

static int run(const rsb200_plan* p, const Arw2Plan& s, const uint8_t* in, uint64_t, uint8_t* outp,
               cudaStream_t st) {
  CUDA_TRY(p->ctx, cudaMemsetAsync(s.d_job_bad.get(), 0, sizeof(uint32_t) * (size_t)p->nunits, st));
  const uint32_t per_cta = ARW2_NT * ARW2_GPT;
  const uint32_t nb = (s.arw2_groups + per_cta - 1) / per_cta;
  const bool sm = s.arw2_ntables == 1; // one table: staged in shared memory
#define RSB_ARW2(M, S)                                                                     \
  arw2_kernel<M, S><<<nb, ARW2_NT, 0, st>>>(in, outp, s.d_arw2_jobs.get(), p->nunits,           \
                                            s.arw2_groups, s.d_arw2_tables.get(), s.d_job_bad.get())
  if (s.arw2_mode == 0)
    RSB_ARW2(0, false);
  else if (s.arw2_mode == 1) {
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
  CUDA_TRY(p->ctx, cudaGetLastError());
  p->ctx->launches++;
  return RSB200_OK;
}

static int results(const rsb200_plan* p, Arw2Plan& s, rsb200_scan_result* out, int n) {
  return report_job_bad(p, s.d_job_bad, s.h_job_bad, out, n,
                        "Too many errors encountered. Giving up. First Error:\n"
                        "ARW2 invariant failed, same pixel is both min and max");
}

static const char* kernels(const rsb200_plan*, const Arw2Plan&) { return "(not an LJPEG plan)"; }

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
// machine (latency bound) and left out of full ones (it adds requests); the split has not been measured on
// H100.  The full launches stage their output in shared memory and store it in 64-byte runs (DESIGN.md, K2S)
constexpr size_t K2P_MAX_SEGMENTS = 0; // (k2_par_kernel: off by default until measured; RSB200_PAR_MAX / RSB200_LJPEG_PATH=par)
// half a wave: for sm_90a ptxas gives k2_stream_kernel 80 registers, so 6 CTAs of 128 threads fit an SM
constexpr int K2S_PREFETCH_CTAS_PER_SM = 3;
// k2_stream_kernel<true, *> (no prefetch; output staged where the tables leave room, else pairs of units
// stored as whole sectors) for launches of more than half a wave of thread-path segments,
// k2_stream_kernel<false, false> up to that; RSB200_STREAM_FORM overrides it
static bool stream_full_launch(const rsb200_ctx* ctx, const LjpegPlan& s) {
  if (s.stream_form)
    return s.stream_form == 2;
  const bool prefetch = s.nthread <= ctx->sm_count * K2S_PREFETCH_CTAS_PER_SM * T_NT;
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

static int finish_ljpeg_plan_tables(rsb200_ctx* ctx, PlanHolder& plan, const std::vector<DevTable>& ht,
                                    ScanBuild& b);

// Lays out and uploads an LJPEG-family plan; on a refusal the caller's holder still owns the plan.
static int finish_ljpeg_plan(rsb200_ctx* ctx, PlanHolder& plan, const rsb200_huff_table* tables, int ntables,
                             ScanBuild& b) {
  std::vector<DevTable> ht((size_t)ntables);
  for (int i = 0; i < ntables; ++i)
    if (!build_dev_table(tables[i], ht[(size_t)i]))
      return set_err(ctx, RSB200_ERR_ARG, "huffman table %d is malformed", i);
  return finish_ljpeg_plan_tables(ctx, plan, ht, b);
}

// the rest of finish_ljpeg_plan, for plans whose device tables are built by their codec
static int finish_ljpeg_plan_tables(rsb200_ctx* ctx, PlanHolder& plan, const std::vector<DevTable>& ht,
                                    ScanBuild& b) {
  rsb200_plan* p = plan.get();
  LjpegPlan& s = std::get<LjpegPlan>(p->state);
  const int ntables = (int)ht.size();
  s.ntab_slots = 1;
  for (const DevScan& d : b.scans)
    for (int sl = 0; sl < 4; ++sl)
      if (d.table_idx[sl] >= 0)
        s.ntab_slots = std::max(s.ntab_slots, sl + 1);
  s.nscans = (int)b.scans.size();
  p->nunits = s.nscans;
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
    s.use_par = ntables <= T_MAXTAB && n_plain > 0 && n_par == n_plain && n_plain <= par_max;
    if (const char* e = getenv("RSB200_LJPEG_PATH")) {
      if (!strcmp(e, "par"))
        s.use_par = ntables <= T_MAXTAB && n_par > 0;
      else
        s.use_par = false;
    }
    if (s.use_par)
      use_thread = true;
    if (const char* e = getenv("RSB200_PAR_CTAS"))
      s.par_ctas = std::max(0, std::min(8, atoi(e)));
  }
  // the thread path's kernel: k2_stream_kernel (raw bytes, unstuffed by the thread itself) or
  // k2_clean_kernel + k2_thread_kernel; RSB200_LJPEG_PATH=stream|thread forces one (tests run both)
  s.use_stream = RSB200_STREAM_DEFAULT != 0 && !s.use_par;
  if (const char* e = getenv("RSB200_THREAD_KERNEL"))
    s.use_stream = !strcmp(e, "stream");
  if (const char* e = getenv("RSB200_LJPEG_PATH")) {
    if (!strcmp(e, "stream"))
      s.use_stream = true;
    else if (!strcmp(e, "thread"))
      s.use_stream = false;
  }
  if (s.use_par)
    s.use_stream = false;
  // RSB200_STREAM_FORM=prefetch|wide fixes the form of k2_stream_kernel whatever the launch size
  // (stream_full_launch; tests run both forms on small batches)
  if (const char* e = getenv("RSB200_STREAM_FORM")) {
    if (!strcmp(e, "prefetch"))
      s.stream_form = 1;
    else if (!strcmp(e, "wide"))
      s.stream_form = 2;
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
  s.tile_r = tile_r;
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
      (d.kind == 2 ? s.has_pentax
                   : (d.kind == 3 ? s.has_nikon
                                  : (d.kind == 4 ? s.has_arw1
                                                 : (d.kind == 5 ? s.has_samsung1 : s.has_k3)))) = true;
    if (!is_big) {
      if (use_thread && (s.use_par ? par_eligible(d) : thread_eligible(d))) {
        thread_ids.push_back((uint32_t)i);
        if (s.use_par) { // differences in stream order (scratch), groups of 8
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
    for (uint32_t r = 0; d.kind < 4 && r < d.rows; ++r) // (ARW1, Samsung V1: their own kernels)
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
  s.nsmall = (int)small_ids.size();
  s.ntile = (int)tile_ids.size();
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
    LjpegPlan::TileGroup g{0, 0, ~0ull, 0, ~0ull, 0};
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
        s.tile_groups.push_back(g);
        g = LjpegPlan::TileGroup{(uint32_t)(k + 1), 0, ~0ull, 0, ~0ull, 0};
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
      s.host_tiles_only = true;
    }
  }
  // The thread path decodes its segments by shape (thread_shape_order), so that whole warps flush the
  // output stage together.  Everything below that is indexed by position (the ids with their bit 31,
  // the per-thread scratch, the redo flags and parameters) is built in this order; the host-buffer
  // groups above keep scan order.
  {
    const std::vector<uint32_t> perm = thread_shape_order(b.scans.data(), thread_ids);
    std::vector<uint32_t> ordered(perm.size());
    for (size_t k = 0; k < perm.size(); ++k)
      ordered[k] = thread_ids[perm[k]];
    thread_ids.swap(ordered);
  }
  s.h_in_size.resize(b.scans.size());
  for (size_t i = 0; i < b.scans.size(); ++i)
    s.h_in_size[i] = b.scans[i].kind == 0 ? b.scans[i].in_size : 0xFFFFFFFFu;
  s.nthread = (int)thread_ids.size();
  if (!thread_ids.empty()) {
    uint64_t bytes = 0;
    for (uint32_t i : thread_ids)
      bytes += b.scans[i].in_size;
    // the warp-per-segment pre-pass is the default: one CTA per small segment (k2_clean2_kernel) is
    // latency bound
    (void)bytes;
    s.clean2 = false;
    if (const char* e = getenv("RSB200_CLEAN"))
      s.clean2 = atoi(e) == 2;
  }
  s.ntables = ntables;
  s.nbig = (int)big_ids.size();
  s.h_big_ids = big_ids;
  s.nranges = (int)ranges.size();
  s.nrows = (uint32_t)b.rows.size();
  cudaError_t e = cudaSuccess;
  dev_upload(e, s.d_tables, ht.data(), sizeof(DevTable) * ht.size());
  dev_upload(e, s.d_scans, b.scans.data(), sizeof(DevScan) * b.scans.size());
  dev_upload(e, s.d_strips, b.strips.data(), sizeof(DevStrip) * b.strips.size());
  dev_upload(e, s.d_rows, b.rows.data(), sizeof(K3RowRef) * b.rows.size());
  dev_upload(e, s.d_small_ids, small_ids.data(), sizeof(uint32_t) * small_ids.size());
  {
    // k2_stream_kernel reads "the tile kernel can give this segment a second opinion" from bit 31
    std::vector<uint32_t> ids = thread_ids;
    if (s.use_stream)
      for (uint32_t& i : ids)
        if (tile_eligible(b.scans[i], TileGeom<1>::MIN_RS))
          i |= 0x80000000u;
    dev_upload(e, s.d_thread_ids, ids.data(), sizeof(uint32_t) * ids.size());
  }
  dev_upload(e, s.d_tile_ids, tile_ids.data(), sizeof(uint32_t) * tile_ids.size());
  dev_upload(e, s.d_tile_params, tile_prm.data(), sizeof(DevTileParam) * tile_prm.size());
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
    if (n_anchor >= (1ull << 32) && !s.use_stream)
      e = cudaErrorInvalidValue;
    if (!s.use_stream)
      dev_upload(e, s.d_tscans, tsc.data(), sizeof(DevTScan) * tsc.size());
    {
      std::vector<DevTileParam> tp(tsc.size());
      for (size_t k = 0; k < tsc.size(); ++k) {
        tile_params(b.scans[thread_ids[k]], TileGeom<1>::NPIECE, TileGeom<1>::DCAP, -1, tp[k].npieces,
                    tp[k].preroll);
        s.nthread_redo += tsc[k].pad ? 1 : 0;
      }
      dev_upload(e, s.d_thread_tile_params, tp.data(), sizeof(DevTileParam) * tp.size());
      dev_alloc(e, s.d_redo, sizeof(uint32_t) * tsc.size());
    }
    if (!s.use_stream) {
      dev_alloc(e, s.d_tinfos, sizeof(DevTInfo) * tsc.size());
      dev_alloc(e, s.d_clean, clean_words * 4 + 256);
      dev_alloc(e, s.d_anchors, n_anchor * 4 + 256);
    }
  }
  dev_upload(e, s.d_big_ids, big_ids.data(), sizeof(uint32_t) * big_ids.size());
  dev_upload(e, s.d_big, big.data(), sizeof(BigScanInfo) * big.size());
  dev_upload(e, s.d_ranges, ranges.data(), sizeof(DevRange) * ranges.size());
  dev_alloc(e, s.d_states, sizeof(RangeState) * ranges.size());
  dev_alloc(e, s.d_finals, sizeof(RangeFinal) * ranges.size());
  dev_alloc(e, s.d_fallback, sizeof(uint32_t) * big.size());
  dev_alloc(e, s.d_diffs, (b.diff_elems + 64) * sizeof(uint16_t));
  dev_alloc(e, s.d_colvals, (b.col_elems + 64) * sizeof(uint16_t));
  dev_alloc(e, s.d_results, sizeof(DevResult) * b.scans.size());
  host_alloc(e, s.h_results, sizeof(DevResult) * b.scans.size());
  if (s.has_pentax) {
    dev_alloc(e, s.d_oob, sizeof(uint32_t) * b.scans.size());
    host_alloc(e, s.h_oob, sizeof(uint32_t) * b.scans.size());
  }
  if (e != cudaSuccess)
    return set_err(ctx, RSB200_ERR_CUDA, "ljpeg plan allocation failed: %s",
                   cudaGetErrorString(e));
  p->launches_per_run = (s.nsmall ? 1 : 0) + (s.ntile ? 1 : 0) + (s.nthread ? (s.use_stream ? 1 : 2) + (s.nthread_redo ? 1 : 0) : 0) +
                        (s.nbig ? 5 + (s.has_k3 ? 2 : 0) + (s.has_pentax ? 2 : 0) + (s.has_nikon ? 2 : 0) : 0);
  return RSB200_OK;
}

static int run(const rsb200_plan* p, const LjpegPlan& s, const uint8_t* in, uint64_t in_bytes, uint8_t* outp,
               cudaStream_t st) {
  rsb200_ctx* ctx = p->ctx;
  const size_t fsm = fused_smem_bytes(s.ntab_slots);
  if (s.ntile) {
    if (s.tile_r == 2)
      k2_tile_kernel<2><<<s.ntile, TL_NT, tile_smem_bytes<2>(), st>>>(
          in, (uint64_t)in_bytes, s.d_scans.get(), s.d_tables.get(), outp, s.d_results.get(), s.d_tile_ids.get(),
          s.d_tile_params.get(), nullptr);
    else
      k2_tile_kernel<1><<<s.ntile, TL_NT, tile_smem_bytes<1>(), st>>>(
          in, (uint64_t)in_bytes, s.d_scans.get(), s.d_tables.get(), outp, s.d_results.get(), s.d_tile_ids.get(),
          s.d_tile_params.get(), nullptr);
    CUDA_TRY(ctx, cudaGetLastError());
    ctx->launches += 1;
  }
  if (s.nsmall) {
    k2_fused_kernel<<<s.nsmall, F_NT, fsm, st>>>(in, (uint64_t)in_bytes, s.d_scans.get(),
                                                   s.d_tables.get(), outp, s.d_results.get(),
                                                   s.d_small_ids.get());
    CUDA_TRY(ctx, cudaGetLastError());
    ctx->launches += 1;
  }
  if (s.nthread && s.use_stream) {
    // small launches are latency bound (L2 prefetch ahead, 128-bit stores), full ones are bound
    // by the number of memory requests (no prefetch, output stored in 64-byte runs)
    // (the output stage where the plan's tables leave room for it, see stream_staged)
    const int nb = (s.nthread + T_NT - 1) / T_NT;
    const size_t smem = stream_smem_bytes(s.ntables);
    if (!stream_full_launch(ctx, s))
      k2_stream_kernel<false, false><<<nb, T_NT, smem, st>>>(
          in, (uint64_t)in_bytes, s.d_scans.get(), s.d_tables.get(), s.ntables, outp, s.d_results.get(),
          s.d_thread_ids.get(), (uint32_t)s.nthread, s.d_redo.get(), 1);
    else if (stream_staged(s.ntables))
      k2_stream_kernel<true, true><<<nb, T_NT, smem, st>>>(
          in, (uint64_t)in_bytes, s.d_scans.get(), s.d_tables.get(), s.ntables, outp, s.d_results.get(),
          s.d_thread_ids.get(), (uint32_t)s.nthread, s.d_redo.get(), 0);
    else
      k2_stream_kernel<true, false><<<nb, T_NT, smem, st>>>(
          in, (uint64_t)in_bytes, s.d_scans.get(), s.d_tables.get(), s.ntables, outp, s.d_results.get(),
          s.d_thread_ids.get(), (uint32_t)s.nthread, s.d_redo.get(), 0);
    CUDA_TRY(ctx, cudaGetLastError());
    ctx->launches += 1;
  } else if (s.nthread && s.use_par) {
    k2_clean_kernel<<<(s.nthread + C_WARPS - 1) / C_WARPS, 32 * C_WARPS, 0, st>>>(
        in, (uint64_t)in_bytes, s.d_scans.get(), s.d_thread_ids.get(), (uint32_t)s.nthread, s.d_tscans.get(),
        s.d_clean.get(), s.d_anchors.get(), s.d_tinfos.get());
    k2_par_kernel<<<s.par_ctas > 0 ? std::min(s.nthread, ctx->sm_count * s.par_ctas) : s.nthread, P_NT, 0, st>>>(
        in, s.d_scans.get(), s.d_tables.get(), outp, s.d_results.get(), s.d_thread_ids.get(), (uint32_t)s.nthread, s.d_tscans.get(),
        s.d_tinfos.get(), s.d_clean.get(), s.d_anchors.get(), s.d_diffs.get(), s.d_redo.get());
    CUDA_TRY(ctx, cudaGetLastError());
    ctx->launches += 2;
  } else if (s.nthread) {
    // unstuffing pre-pass: one CTA per segment with the tile kernel's stage B for DNG-size
    // segments (k2_clean2_kernel), one warp per segment for small ones (k2_clean_kernel)
    if (s.clean2)
      k2_clean2_kernel<<<s.nthread, TL_NT, tile_smem_bytes<1>(), st>>>(
          in, (uint64_t)in_bytes, s.d_scans.get(), s.d_thread_ids.get(), (uint32_t)s.nthread, s.d_tscans.get(),
          s.d_clean.get(), s.d_anchors.get(), s.d_tinfos.get());
    else
    k2_clean_kernel<<<(s.nthread + C_WARPS - 1) / C_WARPS, 32 * C_WARPS, 0, st>>>(
        in, (uint64_t)in_bytes, s.d_scans.get(), s.d_thread_ids.get(), (uint32_t)s.nthread, s.d_tscans.get(),
        s.d_clean.get(), s.d_anchors.get(), s.d_tinfos.get());
    k2_thread_kernel<<<(s.nthread + T_NT - 1) / T_NT, T_NT, thread_smem_bytes(s.ntables), st>>>(
        in, s.d_scans.get(), s.d_tables.get(), s.ntables, outp, s.d_results.get(), s.d_thread_ids.get(),
        (uint32_t)s.nthread, s.d_tscans.get(), s.d_tinfos.get(), s.d_clean.get(), s.d_anchors.get(), s.d_redo.get());
    CUDA_TRY(ctx, cudaGetLastError());
    ctx->launches += 2;
  }
  if (s.nthread) {
    if (s.nthread_redo) {
      // exact end-of-stream semantics for the segments K2T flagged (CTAs of the others exit at once)
      k2_tile_kernel<1><<<s.nthread, TL_NT, tile_smem_bytes<1>(), st>>>(
          in, (uint64_t)in_bytes, s.d_scans.get(), s.d_tables.get(), outp, s.d_results.get(), s.d_thread_ids.get(),
          s.d_thread_tile_params.get(), s.d_redo.get());
      CUDA_TRY(ctx, cudaGetLastError());
      ctx->launches += 1;
    }
  }
  if (s.nbig) {
    k2_clear_results_kernel<<<(s.nbig + 127) / 128, 128, 0, st>>>(s.d_big.get(), s.nbig,
                                                                   s.d_results.get(), s.d_oob.get());
    // ARW1 frames: the range decoder reads the complemented copies (arw1.cuh)
    const uint8_t* kin = in;
    uint64_t kin_bytes = (uint64_t)in_bytes;
    if (s.has_arw1) {
      arw1_prep_kernel<<<dim3((s.arw1_max_words + 255) / 256, s.narw1), 256, 0, st>>>(
          in, s.d_arw1_in.get(), s.d_arw1.get());
      kin = s.d_arw1_in.get();
      kin_bytes = s.arw1_in_bytes;
    }
    k2_range_count_kernel<<<s.nranges, F_NT, fsm, st>>>(kin, kin_bytes, s.d_scans.get(),
                                                         s.d_tables.get(), s.d_ranges.get(), s.d_states.get());
    k2_range_verify_kernel<<<s.nbig, V_NT, 0, st>>>(s.d_scans.get(), s.d_big.get(), s.d_states.get(),
                                                     s.d_finals.get(), s.d_fallback.get(), s.d_results.get());
    k2_range_diffs_kernel<<<s.nranges, F_NT, fsm, st>>>(kin, kin_bytes, s.d_scans.get(),
                                                         s.d_tables.get(), s.d_ranges.get(), s.d_finals.get(),
                                                         s.d_diffs.get(), s.d_results.get());
    // exact redo of segments whose speculative parse failed verification (no-op otherwise)
    k2_entropy_kernel<<<s.nbig, K2_THREADS, sizeof(K2Shared), st>>>(
        kin, kin_bytes, s.d_scans.get(), s.d_tables.get(), s.d_diffs.get(), s.d_results.get(),
        s.d_big_ids.get(), s.d_fallback.get());
    const int col_warps = s.nbig * 4;
    const uint32_t rows_per_block = K3_THREADS / 32;
    int nk3 = 0;
    if (s.has_k3) {
      k3_column_kernel<<<(col_warps * 32 + 127) / 128, 128, 0, st>>>(
          s.d_scans.get(), s.d_big_ids.get(), s.nbig, s.d_diffs.get(), s.d_colvals.get());
      k3_row_kernel<<<(s.nrows + rows_per_block - 1) / rows_per_block, K3_THREADS, 0, st>>>(
          s.d_scans.get(), s.d_rows.get(), s.nrows, s.d_diffs.get(), s.d_colvals.get(), s.d_strips.get(), outp);
      nk3 += 2;
    }
    if (s.has_pentax) {
      k3p_column_kernel<<<(col_warps * 32 + 127) / 128, 128, 0, st>>>(
          s.d_scans.get(), s.d_big_ids.get(), s.nbig, s.d_diffs.get(), s.d_colvals.get(), s.d_oob.get());
      k3p_row_kernel<<<(s.nrows + rows_per_block - 1) / rows_per_block, K3_THREADS, 0, st>>>(
          s.d_scans.get(), s.d_rows.get(), s.nrows, s.d_diffs.get(), s.d_colvals.get(), outp, s.d_oob.get());
      nk3 += 2;
    }
    if (s.has_nikon) {
      k3n_column_kernel<<<(col_warps * 32 + 127) / 128, 128, 0, st>>>(
          s.d_scans.get(), s.d_big_ids.get(), s.nbig, s.d_diffs.get(), s.d_colvals.get());
      k3n_row_kernel<<<(s.nrows + rows_per_block - 1) / rows_per_block, K3_THREADS, 0, st>>>(
          in, s.d_scans.get(), s.d_rows.get(), s.nrows, s.d_diffs.get(), s.d_colvals.get(), s.d_nikon_luts.get(), outp);
      nk3 += 2;
    }
    if (s.has_arw1) {
      arw1_runsum_kernel<<<dim3((s.arw1_max_runs + ARW1_NT / 32 - 1) / (ARW1_NT / 32), s.narw1),
                           ARW1_NT, 0, st>>>(s.d_arw1.get(), s.d_diffs.get(), s.d_arw1_runs.get(),
                                             s.d_arw1_lastoff.get());
      arw1_scan_kernel<<<s.narw1, ARW1_SCAN_NT, 0, st>>>(s.d_arw1.get(), s.d_arw1_runs.get(),
                                                          s.d_arw1_lastoff.get(), s.d_arw1_runpre.get(),
                                                          s.d_arw1_info.get(), s.d_results.get());
      arw1_apply_kernel<<<dim3(s.arw1_max_tiles, s.narw1), ARW1_NT, 0, st>>>(
          s.d_arw1.get(), s.d_diffs.get(), s.d_arw1_runpre.get(), s.d_arw1_info.get(), outp, s.d_results.get());
      nk3 += 4;
    }
    if (s.has_samsung1) {
      CUDA_TRY(ctx, cudaMemsetAsync(s.d_s1_oob.get(), 0xFF, sizeof(uint32_t) * (size_t)s.ns1, st));
      const uint32_t rb = (s.s1_max_h + S1_ROWS_PER_CTA - 1) / S1_ROWS_PER_CTA;
      const uint32_t rows_grid = rb * (uint32_t)s.ns1; // (< 2^31: checked at plan creation)
      s1_column_kernel<<<(s.ns1 * 4 * 32 + 127) / 128, 128, 0, st>>>(s.d_s1.get(), s.ns1, s.d_diffs.get(),
                                                                      s.d_s1_colvals.get(), s.d_s1_oob.get());
      s1_row_kernel<<<rows_grid, S1_NT, 0, st>>>(s.d_s1.get(), rb, s.d_diffs.get(), s.d_s1_colvals.get(),
                                                 s.d_s1_rowbits.get(), s.d_s1_oob.get());
      s1_scan_kernel<<<s.ns1, S1_SCAN_NT, 0, st>>>(s.d_s1.get(), s.d_diffs.get(), s.d_s1_rowbits.get(),
                                                    s.d_s1_oob.get(), s.d_s1_lim.get(), s.d_results.get());
      s1_store_kernel<<<rows_grid, S1_NT, 0, st>>>(s.d_s1.get(), rb, s.d_diffs.get(), s.d_s1_colvals.get(),
                                                   s.d_s1_lim.get(), outp);
      nk3 += 4;
    }
    CUDA_TRY(ctx, cudaGetLastError());
    ctx->launches += 5 + nk3;
  }
  return RSB200_OK;
}

static int results(const rsb200_plan* p, LjpegPlan& s, rsb200_scan_result* out, int n) {
  rsb200_ctx* ctx = p->ctx;
  if (s.d_oob)
    CUDA_TRY(ctx, cudaMemcpyAsync(s.h_oob.get(), s.d_oob.get(), sizeof(uint32_t) * s.nscans,
                                  cudaMemcpyDeviceToHost, p->last_stream));
  bool oob = false; // the job outcome() just gave is a Pentax value out of range
  return report_jobs(
      p, s.d_results, s.h_results, out, n,
      [&](int i) {
        DevResult& r = s.h_results[i];
        oob = s.d_oob && r.status == 0 && s.h_oob[i] != 0xFFFFFFFFu;
        if (oob) {
          // Pentax: a decoded value left 0..65535 (PentaxDecompressor.cpp:170-171)
          r.status = RSB200_ERR_RDE;
          r.consumed = RSB200_PENTAX_OOB | s.h_oob[i];
        } else if (r.status == 0 && (size_t)i < s.h_in_size.size() && r.consumed > s.h_in_size[(size_t)i]) {
          // The reference skips `consumed` bytes of its input when a scan is done
          // (LJpegDecompressor.cpp:339 inputStream.skipBytes(bs.getStreamPosition())) and throws when
          // the buffer is shorter: a buffer that ends inside the last refill of the pump is an
          // IOException even though every symbol was there.  One rule for every LJPEG kernel.
          r.status = RSB200_ERR_IOE;
        }
        return rsb200_scan_result{r.status, r.consumed};
      },
      [&](int i, const rsb200_scan_result& r) {
        const int first = (int)r.status;
        if (oob) {
          set_err(ctx, first, "decoded value out of bounds at %u:%u", s.h_oob[i] & 0x3FFFu, s.h_oob[i] >> 14);
        } else if (s.has_samsung1) {
          // SamsungV1Decompressor.cpp:135-136 / BitStreamer.h:58-59, 125-127
          if (first == RSB200_ERR_RDE)
            set_err(ctx, first, "job %d: decoded value out of bounds (col %u, row %u)", i, r.consumed & 0x3FFFu,
                    (r.consumed >> 14) & 0xFFFu);
          else if (r.consumed == 0) // (T* >= 106 for 4 bytes and more: only a short stream)
            set_err(ctx, first, "job %d: Bit stream size is smaller than MaxProcessBytes", i);
          else
            set_err(ctx, first, "job %d: Buffer overflow read in BitStreamer (col %u, row %u)", i,
                    r.consumed & 0x3FFFu, r.consumed >> 14);
        } else if (s.has_arw1) {
          // SonyArw1Decompressor.cpp:86-87 / BitStreamer.h:100-131
          if (first == RSB200_ERR_RDE)
            set_err(ctx, first, "job %d: Error decompressing (col %u, row %u)", i, r.consumed & 0x3FFFu,
                    (r.consumed >> 14) & 0xFFFu);
          else
            set_err(ctx, first, "job %d: Buffer overflow read in BitStreamer", i);
        } else {
          set_err(ctx, first,
                  first == RSB200_ERR_RDE ? "segment %d: bad Huffman code"
                                          : "segment %d: Buffer overflow read in BitStreamer",
                  i);
        }
      });
}

static const char* kernels(const rsb200_plan* p, const LjpegPlan& s) {
  const bool only_thread = s.nthread && !s.ntile && !s.nsmall && !s.nbig;
  const bool only_tile = s.ntile && !s.nthread && !s.nsmall && !s.nbig;
  if (only_thread && s.use_par)
    return "k2_clean_kernel + k2_par_kernel (one CTA per segment: speculative parse of the clean stream to a "
           "fixed point, decode, row sums)";
  if (only_thread && s.use_stream) {
    if (stream_full_launch(p->ctx, s))
      return s.nthread_redo ? "k2_stream_kernel (one thread per segment, unstuffing in the thread), full-launch form + "
                              "k2_tile_kernel<1> for flagged ends of stream"
                            : "k2_stream_kernel (one thread per segment, unstuffing in the thread), full-launch form";
    return s.nthread_redo ? "k2_stream_kernel (one thread per segment, unstuffing in the thread), prefetch form + "
                            "k2_tile_kernel<1> for flagged ends of stream"
                          : "k2_stream_kernel (one thread per segment, unstuffing in the thread), prefetch form";
  }
  if (only_thread)
    return s.clean2 ? "k2_clean2_kernel + k2_thread_kernel (one thread per segment)"
                    : "k2_clean_kernel + k2_thread_kernel (one thread per segment)";
  if (only_tile)
    return s.tile_r == 2 ? "k2_tile_kernel<2> (one CTA per tile)" : "k2_tile_kernel<1> (one CTA per tile)";
  if (s.nsmall && !s.nthread && !s.ntile && !s.nbig)
    return "k2_fused_kernel (one CTA per segment)";
  return "mixed (k2_fused / k2_tile / thread path / multi-CTA ranges + K3)";
}

// the tile-kernel segments first .. first + count - 1 (host-buffer and gather pipelines)
static cudaError_t launch_tile_range(const LjpegPlan& s, const uint8_t* d_in, uint64_t in_bytes,
                                     uint8_t* d_out, uint32_t first, uint32_t count,
                                     cudaStream_t st) {
  if (s.tile_r == 2)
    k2_tile_kernel<2><<<count, TL_NT, tile_smem_bytes<2>(), st>>>(
        d_in, in_bytes, s.d_scans.get(), s.d_tables.get(), d_out, s.d_results.get(), s.d_tile_ids.get() + first,
        s.d_tile_params.get() + first, nullptr);
  else
    k2_tile_kernel<1><<<count, TL_NT, tile_smem_bytes<1>(), st>>>(
        d_in, in_bytes, s.d_scans.get(), s.d_tables.get(), d_out, s.d_results.get(), s.d_tile_ids.get() + first,
        s.d_tile_params.get() + first, nullptr);
  return cudaGetLastError();
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
  PlanHolder holder = new_plan(ctx);
  if (!holder)
    return RSB200_ERR_CUDA;
  rsb200_plan* p = holder.get();
  p->state.emplace<LjpegPlan>();
  ScanBuild b;
  for (int i = 0; i < njobs; ++i) {
    const rsb200_pentax_job& j = jobs[i];
    // PentaxDecompressor ctor (PentaxDecompressor.cpp:55-67)
    const bool ok = j.width > 0 && j.height > 0 && j.width % 2 == 0 && j.width <= 8384 &&
                    j.height <= 6208 && (int)j.table < ntables && j.in_size < (1u << 28) &&
                    (uint64_t)j.width * 2 <= j.out_pitch && (j.out_offset % 4) == 0 &&
                    (j.out_pitch % 4) == 0;
    if (!ok)
      return set_err(ctx, RSB200_ERR_ARG, "pentax job %d: malformed descriptor", i);
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
  int rc = finish_ljpeg_plan(ctx, holder, tables, ntables, b);
  if (rc != RSB200_OK)
    return rc;
  *out = holder.release();
  return RSB200_OK;
}

// ------------------------------------------------------------------
// Sony ARW1: one plain-MSB stream per frame (arw1.cuh: complemented copy, K2R, frame-wide scan)
// ------------------------------------------------------------------
// The prefix code of the complemented ARW1 stream (arw1.cuh): counts per code length 1..16 and
// the extra bits of each code, in canonical order; length 17 is two 16-bit codes whose 16 extra
// bits (DNG rule) make up its 17
static rsb200_huff_table arw1_table() {
  rsb200_huff_table t;
  memset(&t, 0, sizeof t);
  const uint8_t counts[16] = {0, 2, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 2};
  const uint8_t values[19] = {1, 2, 0, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 16, 16};
  memcpy(t.ncodes_per_len, counts, sizeof counts);
  memcpy(t.values, values, sizeof values);
  t.nvalues = 19;
  t.fix_dng16 = 1;
  return t;
}

extern "C" int rsb200_arw1_plan_create(rsb200_ctx* ctx, const rsb200_arw1_job* jobs, int njobs,
                                       rsb200_plan** out) {
  if (!ctx || !jobs || njobs <= 0 || !out)
    return set_err(ctx, RSB200_ERR_ARG, "arw1_plan_create: bad arguments");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  for (int i = 0; i < njobs; ++i) {
    const rsb200_arw1_job& j = jobs[i];
    // SonyArw1Decompressor ctor (SonyArw1Decompressor.cpp:39-50)
    if (j.width <= 0 || j.height <= 0 || j.height % 2 != 0 || j.width > 4600 || j.height > 3072)
      return set_err(ctx, RSB200_ERR_RDE, "job %d: Unexpected image dimensions found: (%u; %u)", i,
                     (unsigned)j.width, (unsigned)j.height);
    if (j.in_size >= (1u << 28) || (uint64_t)j.width * 2 > j.out_pitch || (j.out_offset % 2) ||
        (j.out_pitch % 2) || j.reserved0 || j.reserved)
      return set_err(ctx, RSB200_ERR_ARG, "arw1 job %d: malformed descriptor", i);
  }
  PlanHolder holder = new_plan(ctx);
  if (!holder)
    return RSB200_ERR_CUDA;
  rsb200_plan* p = holder.get();
  LjpegPlan& s = p->state.emplace<LjpegPlan>();
  ScanBuild b;
  std::vector<DevArw1> fr((size_t)njobs);
  uint64_t koff = 0, runs = 0;
  for (int i = 0; i < njobs; ++i) {
    const rsb200_arw1_job& j = jobs[i];
    const uint32_t w = (uint32_t)j.width, h = (uint32_t)j.height;
    DevArw1& f = fr[(size_t)i];
    memset(&f, 0, sizeof f);
    f.in_offset = j.in_offset;
    f.in_size = j.in_size;
    f.k_offset = koff;
    f.w = w;
    f.h = h;
    f.out_offset = j.out_offset;
    f.out_pitch = j.out_pitch;
    f.nrh = (h + 63) / 64;
    // plain_overread (ljpeg.cuh): the first bit T with (T >> 5) + 1 + (T & 31 ? 1 : 0) refills
    // >= (size + 8) / 4 + 2
    f.tstar = 32u * ((j.in_size + 8u) / 4u) + 1u;
    if (j.in_size < 4) // BitStreamerMSB's constructor throws (BitStreamer.h:56-60): before symbol 0
      f.tstar = 0;
    f.scan = (uint32_t)i;
    f.run_offset = runs;
    runs += (uint64_t)w * 2 * f.nrh;
    s.arw1_max_runs = std::max(s.arw1_max_runs, w * 2 * f.nrh);
    s.arw1_max_tiles = std::max(s.arw1_max_tiles, f.nrh * ((w + 63) / 64));
    s.arw1_max_words = std::max(s.arw1_max_words, (j.in_size + 16u + 3u) / 4u);
    DevScan d;
    memset(&d, 0, sizeof d);
    d.in_offset = koff;
    d.in_size = j.in_size + 16u; // + the 0xFF bytes: zero bits of the original stream
    d.row_samples = w;
    d.rows = h;
    d.n_samples = w * h;
    d.group = 1;
    d.ncomp = 1;
    d.kind = 4;
    d.pump = 1;
    d.pattern = PAT_PLAIN;
    const uint8_t tab[4] = {0, 0, 0, 0};
    const uint8_t comp_of_pos[1] = {0};
    assign_tables(d, tab, 1, comp_of_pos, 1);
    d.out_offset = j.out_offset;
    d.out_pitch = j.out_pitch;
    d.mcu_w = 1;
    d.mcu_h = 1;
    d.store_w = w;
    b.scans.push_back(d);
    koff += ((uint64_t)j.in_size + 16u + 15u) & ~15ull;
    p->in_bytes += j.in_size;
    p->out_bytes += (uint64_t)w * h * 2;
    p->pixels += (uint64_t)w * h;
    p->need_in = std::max<uint64_t>(p->need_in, sat_add(j.in_offset, j.in_size));
    p->need_out = std::max<uint64_t>(p->need_out, sat_add(j.out_offset, ((uint64_t)h - 1) * j.out_pitch + 2ull * w));
  }
  const rsb200_huff_table t = arw1_table();
  int rc = finish_ljpeg_plan(ctx, holder, &t, 1, b);
  if (rc != RSB200_OK)
    return rc;
  for (size_t i = 0; i < fr.size(); ++i)
    fr[i].diff_offset = b.scans[i].diff_offset;
  s.narw1 = njobs;
  s.arw1_in_bytes = koff;
  cudaError_t e = cudaSuccess;
  dev_upload(e, s.d_arw1, fr.data(), sizeof(DevArw1) * fr.size());
  dev_alloc(e, s.d_arw1_in, koff + 256);
  dev_alloc(e, s.d_arw1_runs, sizeof(Arw1Run) * runs);
  dev_alloc(e, s.d_arw1_lastoff, sizeof(uint32_t) * runs);
  dev_alloc(e, s.d_arw1_runpre, sizeof(int2) * runs);
  dev_alloc(e, s.d_arw1_info, sizeof(Arw1Info) * fr.size());
  if (e != cudaSuccess)
    return set_err(ctx, RSB200_ERR_CUDA, "arw1 plan allocation failed: %s", cudaGetErrorString(e));
  p->launches_per_run += 4;
  *out = holder.release();
  return RSB200_OK;
}

// ------------------------------------------------------------------
// Samsung V1: one plain-MSB stream per frame (K2R with the LUT-only table, samsung1.cuh)
// ------------------------------------------------------------------
extern "C" int rsb200_samsung1_plan_create(rsb200_ctx* ctx, const rsb200_samsung1_job* jobs,
                                           int njobs, rsb200_plan** out) {
  if (!ctx || !jobs || njobs <= 0 || !out)
    return set_err(ctx, RSB200_ERR_ARG, "samsung1_plan_create: bad arguments");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  for (int i = 0; i < njobs; ++i) {
    const rsb200_samsung1_job& j = jobs[i];
    // SamsungV1Decompressor ctor (SamsungV1Decompressor.cpp:52-60)
    if (j.bits != 12)
      return set_err(ctx, RSB200_ERR_RDE, "job %d: Unexpected bit per pixel (%d)", i, (int)j.bits);
    if (j.width <= 0 || j.height <= 0 || j.width % 32 != 0 || j.height % 2 != 0 || j.width > 5664 ||
        j.height > 3714)
      return set_err(ctx, RSB200_ERR_RDE, "job %d: Unexpected image dimensions found: (%u; %u)", i,
                     (unsigned)j.width, (unsigned)j.height);
    // the stores write two pixels as one 32-bit word
    if (j.in_size >= (1u << 28) || (uint64_t)j.width * 2 > j.out_pitch || (j.out_offset % 4) ||
        (j.out_pitch % 4) || j.reserved)
      return set_err(ctx, RSB200_ERR_ARG, "samsung1 job %d: malformed descriptor", i);
  }
  PlanHolder holder = new_plan(ctx);
  if (!holder)
    return RSB200_ERR_CUDA;
  rsb200_plan* p = holder.get();
  LjpegPlan& s = p->state.emplace<LjpegPlan>();
  ScanBuild b;
  std::vector<DevS1> fr((size_t)njobs);
  uint64_t rows = 0;
  for (int i = 0; i < njobs; ++i) {
    const rsb200_samsung1_job& j = jobs[i];
    const uint32_t w = (uint32_t)j.width, h = (uint32_t)j.height;
    DevS1& f = fr[(size_t)i];
    memset(&f, 0, sizeof f);
    f.w = w;
    f.h = h;
    f.out_offset = j.out_offset;
    f.out_pitch = j.out_pitch;
    f.tstar = samsung1_tstar(j.in_size);
    f.scan = (uint32_t)i;
    f.row_base = (uint32_t)rows;
    rows += h;
    s.s1_max_h = std::max(s.s1_max_h, h);
    DevScan d;
    memset(&d, 0, sizeof d);
    d.in_offset = j.in_offset;
    d.in_size = j.in_size;
    d.row_samples = w;
    d.rows = h;
    d.n_samples = w * h;
    d.group = 1;
    d.ncomp = 1;
    d.kind = 5;
    d.pump = 1;
    d.pattern = PAT_PLAIN;
    const uint8_t tab[4] = {0, 0, 0, 0};
    const uint8_t comp_of_pos[1] = {0};
    assign_tables(d, tab, 1, comp_of_pos, 1);
    d.out_offset = j.out_offset;
    d.out_pitch = j.out_pitch;
    d.mcu_w = 1;
    d.mcu_h = 1;
    d.store_w = w;
    b.scans.push_back(d);
    p->in_bytes += j.in_size;
    p->out_bytes += (uint64_t)w * h * 2;
    p->pixels += (uint64_t)w * h;
    p->need_in = std::max<uint64_t>(p->need_in, sat_add(j.in_offset, j.in_size));
    p->need_out = std::max<uint64_t>(p->need_out, sat_add(j.out_offset, ((uint64_t)h - 1) * j.out_pitch + 2ull * w));
  }
  // (the row kernels' 1-D grids: one CTA per 8 rows of the tallest frame, per frame)
  if (rows >= (1ull << 31) ||
      (uint64_t)njobs * ((s.s1_max_h + S1_ROWS_PER_CTA - 1) / S1_ROWS_PER_CTA) >= (1ull << 31))
    return set_err(ctx, RSB200_ERR_ARG, "samsung1 plan: too many frames for one plan");
  std::vector<DevTable> ht(1);
  samsung1_dev_table(ht[0]);
  int rc = finish_ljpeg_plan_tables(ctx, holder, ht, b);
  if (rc != RSB200_OK)
    return rc;
  for (size_t i = 0; i < fr.size(); ++i)
    fr[i].diff_offset = b.scans[i].diff_offset;
  s.ns1 = njobs;
  cudaError_t e = cudaSuccess;
  dev_upload(e, s.d_s1, fr.data(), sizeof(DevS1) * fr.size());
  dev_alloc(e, s.d_s1_colvals, sizeof(uint16_t) * 2 * rows);
  dev_alloc(e, s.d_s1_rowbits, sizeof(uint2) * rows);
  dev_alloc(e, s.d_s1_oob, sizeof(uint32_t) * fr.size());
  dev_alloc(e, s.d_s1_lim, sizeof(uint32_t) * fr.size());
  if (e != cudaSuccess)
    return set_err(ctx, RSB200_ERR_CUDA, "samsung1 plan allocation failed: %s", cudaGetErrorString(e));
  p->launches_per_run += 4;
  *out = holder.release();
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
  PlanHolder holder = new_plan(ctx);
  if (!holder)
    return RSB200_ERR_CUDA;
  rsb200_plan* p = holder.get();
  LjpegPlan& s = p->state.emplace<LjpegPlan>();
  ScanBuild b;
  for (int i = 0; i < njobs; ++i) {
    const rsb200_nikon_job& j = jobs[i];
    // NikonDecompressor ctor (NikonDecompressor.cpp:478-489); BitStreamerMSB needs 4 bytes
    const bool ok = j.width > 0 && j.height > 0 && j.width % 2 == 0 && j.width <= 8288 &&
                    j.height <= 5520 && (int)j.table < ntables && j.in_size >= 4 &&
                    j.in_size < (1u << 28) && (uint64_t)j.width * 2 <= j.out_pitch &&
                    (j.out_offset % 4) == 0 && (j.out_pitch % 4) == 0 && j.lut < nluts;
    if (!ok)
      return set_err(ctx, RSB200_ERR_ARG, "nikon job %d: malformed descriptor", i);
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
  int rc = finish_ljpeg_plan(ctx, holder, tables, ntables, b);
  if (rc != RSB200_OK)
    return rc;
  cudaError_t e = cudaSuccess;
  dev_upload(e, s.d_nikon_luts, luts, (size_t)nluts * 2u * 65536u * sizeof(uint16_t), 16);
  if (e != cudaSuccess)
    return set_err(ctx, RSB200_ERR_CUDA, "nikon plan upload failed: %s", cudaGetErrorString(e));
  *out = holder.release();
  return RSB200_OK;
}

extern "C" int rsb200_ljpeg_plan_create(rsb200_ctx* ctx, const rsb200_huff_table* tables,
                                        int ntables, const rsb200_ljpeg_scan* scans,
                                        int nscans, rsb200_plan** out) {
  if (!ctx || !tables || ntables <= 0 || !scans || nscans <= 0 || !out)
    return set_err(ctx, RSB200_ERR_ARG, "ljpeg_plan_create: bad arguments");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  PlanHolder holder = new_plan(ctx);
  if (!holder)
    return RSB200_ERR_CUDA;
  rsb200_plan* p = holder.get();
  p->state.emplace<LjpegPlan>();
  ScanBuild b;
  b.scans.reserve((size_t)nscans);
  for (int i = 0; i < nscans; ++i) {
    const rsb200_ljpeg_scan& s = scans[i];
    const int group = s.mcu_w * s.mcu_h;
    DevScan d;
    // validation (every sum in 64 bits, out_offset 2-byte aligned) + descriptor: ljpeg_host.h
    if (!ljpeg_scan_to_dev(s, ntables, d))
      return set_err(ctx, RSB200_ERR_ARG, "ljpeg scan %d: malformed descriptor", i);
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
    if (s.out_offset + extent < s.out_offset || s.in_offset + (uint64_t)s.in_size < s.in_offset)
      return set_err(ctx, RSB200_ERR_ARG, "ljpeg scan %d: offset + extent overflows", i);
    p->need_out = std::max<uint64_t>(p->need_out, sat_add(s.out_offset, extent));
  }
  int rc = finish_ljpeg_plan(ctx, holder, tables, ntables, b);
  if (rc != RSB200_OK)
    return rc;
  *out = holder.release();
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
  PlanHolder holder = new_plan(ctx);
  if (!holder)
    return RSB200_ERR_CUDA;
  rsb200_plan* p = holder.get();
  p->state.emplace<LjpegPlan>();
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
              (uint64_t)j.img_w * 2 <= j.out_pitch && (j.out_offset % 2) == 0 &&
              (j.out_pitch % 2) == 0 && j.in_size < (1u << 28);
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
    if (!ok)
      return set_err(ctx, RSB200_ERR_ARG, "cr2 job %d: malformed descriptor", i);
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
  int rc = finish_ljpeg_plan(ctx, holder, tables, ntables, b);
  if (rc != RSB200_OK)
    return rc;
  *out = holder.release();
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
  const int rc = std::visit([&](const auto& s) { return run(p, s, in, (uint64_t)in_bytes, outp, st); }, p->state);
  if (rc)
    return rc;
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
static bool unpack_pipeline_ok(const UnpackPlan& s) {
  if (!s.groups.empty() || s.fast_groups.size() != 1)
    return false;
  const auto& jobs = s.fast_groups[0].h_jobs;
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

static int run_host_unpack_pipelined(rsb200_plan* p, const UnpackFastGroup& g, const uint8_t* in, size_t in_bytes,
                                     uint8_t* out, size_t out_bytes) {
  rsb200_ctx* ctx = p->ctx;
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

// LJPEG plan made of tile-kernel segments only: group g's upload, kernel and download are chained
// on stream g % 3, so the upload of the next group and the download of the previous one overlap
// the decode of the current one.  Spans of neighbouring groups may overlap (tiles of one tile row
// in two groups): every byte's last download happens after its last write, whatever the order.
static int run_host_tile_pipelined(rsb200_plan* p, const LjpegPlan& s, const uint8_t* in, size_t in_bytes,
                                   uint8_t* out, size_t out_bytes, uint32_t pitch, uint32_t row_bytes) {
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
    while (ctx->stage_events.size() < s.tile_groups.size()) {
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
  for (size_t gi = 0; gi < s.tile_groups.size(); ++gi) {
    const LjpegPlan::TileGroup& g = s.tile_groups[gi];
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
    CUDA_TRY(ctx, launch_tile_range(s, ctx->d_in, (uint64_t)in_bytes, ctx->d_out, g.first, g.count, st));
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
    for (size_t gi = 0; gi < s.tile_groups.size(); ++gi) {
      const LjpegPlan::TileGroup& g = s.tile_groups[gi];
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
            s.tile_groups.size(), trace_submit_ms, total_ms);
    for (size_t gi = 0; gi < s.tile_groups.size() && 3 * gi + 3 < tev.size(); ++gi) {
      float a = 0, b = 0, c = 0;
      cudaEventElapsedTime(&a, tev[0], tev[3 * gi + 1]);
      cudaEventElapsedTime(&b, tev[0], tev[3 * gi + 2]);
      cudaEventElapsedTime(&c, tev[0], tev[3 * gi + 3]);
      if (gi < 16 || gi + 4 > s.tile_groups.size())
        fprintf(stderr, "PIPE_TRACE %3zu  %8.3f %8.3f %8.3f\n", gi, a, b, c);
    }
    for (cudaEvent_t e : tev)
      cudaEventDestroy(e);
  }
  p->last_stream = ctx->pipe[0];
  p->ran = true;
  return RSB200_OK;
}

// The body of rsb200_plan_run_host and rsb200_plan_run_host_image.  `image`: only `row_bytes` of each of
// the output's `rows` rows (every `pitch` bytes) are written back; otherwise all `out_bytes` are.
static int run_host(rsb200_plan* p, const uint8_t* in, size_t in_bytes, uint8_t* out, size_t out_bytes, bool image,
                    uint32_t pitch, uint32_t row_bytes, uint32_t rows, int partial, const char* too_small) {
  rsb200_ctx* ctx = p->ctx;
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  int rc = ensure_cap(ctx, &ctx->d_in, &ctx->d_in_cap, in_bytes + 16);
  if (rc)
    return rc;
  rc = ensure_cap(ctx, &ctx->d_out, &ctx->d_out_cap, out_bytes);
  if (rc)
    return rc;
  if (in_bytes < p->need_in || out_bytes < p->need_out)
    return set_err(ctx, RSB200_ERR_ARG, "%s", too_small);
  if (in_place(*p))
    partial = 1; // in-place plans work on the image the caller holds: it always goes up first
  const UnpackPlan* unpack = std::get_if<UnpackPlan>(&p->state);
  if (!partial && !image && unpack && unpack_pipeline_ok(*unpack))
    return run_host_unpack_pipelined(p, unpack->fast_groups[0], in, in_bytes, out, out_bytes);
  const LjpegPlan* lj = std::get_if<LjpegPlan>(&p->state);
  if (!partial && lj && lj->tile_groups.size() >= 2 && !getenv("RSB200_NO_PIPELINE"))
    return run_host_tile_pipelined(p, *lj, in, in_bytes, out, out_bytes, pitch, row_bytes);
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
  if (image && !stage_out) {
    CUDA_TRY(ctx, cudaMemcpy2DAsync(out, pitch, ctx->d_out, pitch, row_bytes, rows,
                                    cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaStreamSynchronize(st));
    return RSB200_OK;
  }
  CUDA_TRY(ctx, cudaMemcpyAsync(stage_out ? ctx->h_out : out, ctx->d_out, out_bytes, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaStreamSynchronize(st));
  if (stage_out && image)
    parallel_copy_rows(out, ctx->h_out, pitch, row_bytes, rows);
  else if (stage_out)
    parallel_copy(out, ctx->h_out, out_bytes);
  return RSB200_OK;
}

extern "C" int rsb200_plan_run_host(rsb200_plan* p, const uint8_t* in, size_t in_bytes,
                                    uint8_t* out, size_t out_bytes, int partial) {
  if (!p || !out || (!in && in_bytes))
    return RSB200_ERR_ARG;
  return run_host(p, in, in_bytes, out, out_bytes, false, 0, 0, 0, partial, "plan_run_host: buffers too small");
}

extern "C" int rsb200_plan_run_host_image(rsb200_plan* p, const uint8_t* in, size_t in_bytes,
                                          uint8_t* out, uint32_t pitch, uint32_t row_bytes,
                                          uint32_t rows, int partial) {
  if (!p || !out || (!in && in_bytes) || row_bytes > pitch)
    return RSB200_ERR_ARG;
  return run_host(p, in, in_bytes, out, (size_t)pitch * rows, true, pitch, row_bytes, rows, partial,
                  "plan_run_host_image: buffers too small");
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
  const LjpegPlan* lj = std::get_if<LjpegPlan>(&p->state);
  if (lj && !lj->tile_groups.empty() && !lj->host_tiles_only) {
    const LjpegPlan& s = *lj;
    if (in_bytes < p->need_in)
      return set_err(ctx, RSB200_ERR_ARG, "plan_run_gather: input too small");
    while (c->events.size() < s.tile_groups.size()) {
      cudaEvent_t e;
      CUDA_TRY(ctx, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
      c->events.push_back(e);
    }
    for (size_t gi = 0; gi < s.tile_groups.size(); ++gi) {
      const LjpegPlan::TileGroup& g = s.tile_groups[gi];
      CUDA_TRY(ctx, launch_tile_range(s, (const uint8_t*)d_in, (uint64_t)in_bytes, mine, g.first, g.count, st));
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

extern "C" int rsb200_plan_results(rsb200_plan* p, rsb200_scan_result* out, int n) {
  if (!p)
    return RSB200_ERR_ARG;
  if (!p->ran)
    return set_err(p->ctx, RSB200_ERR_ARG, "plan_results: plan has not been run");
  return std::visit([&](auto& s) { return results(p, s, out, n); }, p->state);
}

// Debug entry (not in the public header; tests reach it through ctypes): after the last run of
// `p`, flags[i] = 1 if scan i went through the multi-CTA range path (ljpeg_ranges.cuh) and a seam
// failed its check, so that k2_entropy_kernel redid the whole segment; 0 otherwise (also for scans
// that are not big).  Reads the flags P2 wrote; launches nothing.
extern "C" int rsb200_debug_range_redo(const rsb200_plan* p, uint32_t* flags, int n) {
  if (!p || n < 0 || (n > 0 && !flags))
    return RSB200_ERR_ARG;
  rsb200_ctx* ctx = p->ctx;
  if (!p->ran)
    return set_err(ctx, RSB200_ERR_ARG, "debug_range_redo: plan has not been run");
  for (int i = 0; i < n; ++i)
    flags[i] = 0;
  const LjpegPlan* lj = std::get_if<LjpegPlan>(&p->state);
  if (!lj || lj->h_big_ids.empty())
    return RSB200_OK;
  const LjpegPlan& s = *lj;
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  CUDA_TRY(ctx, cudaStreamSynchronize(p->last_stream));
  std::vector<uint32_t> fb(s.h_big_ids.size());
  CUDA_TRY(ctx, cudaMemcpy(fb.data(), s.d_fallback.get(), sizeof(uint32_t) * fb.size(), cudaMemcpyDeviceToHost));
  for (size_t k = 0; k < fb.size(); ++k)
    if ((int)s.h_big_ids[k] < n)
      flags[s.h_big_ids[k]] = fb[k] ? 1u : 0u;
  return RSB200_OK;
}

extern "C" int rsb200_plan_bad_pixels(rsb200_plan* p, int job, uint32_t* positions, uint32_t cap,
                                      uint32_t* count) {
  if (!p || !count)
    return RSB200_ERR_ARG;
  rsb200_ctx* ctx = p->ctx;
  *count = 0;
  const BadList* bad = nullptr;
  if (const PanaPlan* pana = std::get_if<PanaPlan>(&p->state))
    bad = &pana->bad;
  else if (const DngOpPlan* dngop = std::get_if<DngOpPlan>(&p->state))
    bad = &dngop->bad;
  if (!bad || job < 0 || job >= (int)bad->slot.size())
    return set_err(ctx, RSB200_ERR_ARG,
                   "plan_bad_pixels: not a job of a Panasonic plan / an opcode of a DNG opcode plan");
  if (!p->ran)
    return set_err(ctx, RSB200_ERR_ARG, "plan_bad_pixels: plan has not been run");
  const int slot = bad->slot[job];
  if (slot < 0)
    return RSB200_OK; // zero_is_not_bad (or not V4): the reference collects nothing
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  CUDA_TRY(ctx, cudaStreamSynchronize(p->last_stream));
  uint32_t n = 0;
  CUDA_TRY(ctx, cudaMemcpy(&n, bad->d_count.get() + slot, sizeof n, cudaMemcpyDeviceToHost));
  *count = n;
  const uint32_t take = std::min(std::min(n, cap), (uint32_t)PANA_ZERO_CAP);
  if (take && positions)
    CUDA_TRY(ctx, cudaMemcpy(positions, bad->d_list.get() + (size_t)slot * PANA_ZERO_CAP,
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
  return std::visit([&](const auto& s) { return kernels(p, s); }, p->state);
}

extern "C" void rsb200_plan_destroy(rsb200_plan* p) {
  if (!p)
    return;
  if (p->ctx)
    cudaSetDevice(p->ctx->device);
  if (p->ran && p->last_stream)
    cudaStreamSynchronize(p->last_stream); // (the owners free stream ordered, not with device-wide syncs)
  delete p;
}
