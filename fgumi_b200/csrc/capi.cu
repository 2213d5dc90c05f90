// C-ABI implementation (include/fgumi_b200.h): handle lifecycle, tile planner, vote launches,
// the chunked host-buffer pipeline, strand-combine launches and the device counters.
// There is no CPU fallback anywhere in this file: without a CUDA device every compute entry point
// returns FGB_ERR_NO_DEVICE / FGB_ERR_CUDA.
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "../../include/fgumi_b200.h"
#include "assemble_kernel.cuh"
#include "combine_kernels.cuh"
#include "dedup_kernels.cuh"
#include "fgb_config.h"
#include "filter_kernel.cuh"
#include "filter_records_kernels.cuh"
#include "inflate_kernel.cuh"
#include "host_tables.h"
#include "planner.h"
#include "sort_kernels.cuh"
#include "umi_kernels.cuh"
#include "unpack_kernels.cuh"
#include "host/dedup_device.h"
#include "host/filter_device.h"
#include "host/record_link.h"
#include "host/sort_device.h"
#include "host/umi_host.h"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include "vote_kernel.cuh"

using namespace fgb;

static_assert(sizeof(fgb_unit) == 16, "fgb_unit must be 16 bytes");
static_assert(sizeof(fgb_tile) == 32, "fgb_tile must be 32 bytes");
static_assert(sizeof(Stage) % 16 == 0, "Stage must keep 16-byte TMA alignment");
static_assert(offsetof(Stage, quals) % 16 == 0 && offsetof(Stage, reads) % 16 == 0 &&
                  offsetof(Stage, units) % 16 == 0 && offsetof(Stage, tile) % 16 == 0,
              "TMA destinations must be 16-byte aligned");

namespace {

constexpr int kSlots = 4;                        // max chunk pipeline depth of fgb_submit
constexpr uint64_t kChunkColumnBytes = 96ull << 20;  // default per-column bytes per chunk

struct Slot {
  cudaStream_t stream = nullptr;
  uint8_t* bases = nullptr;
  uint8_t* quals = nullptr;
  uint8_t* packed = nullptr;     // PACK8 transfer column (fgb_submit_pack8)
  uint64_t cap_packed = 0;
  uint8_t* unit_status = nullptr;   // filter epilogue results
  uint32_t* unit_masked = nullptr;
  uint64_t cap_ustat = 0, cap_umask = 0;
  uint8_t* out_depth8 = nullptr; // narrow outputs (FGB_OUT_U8)
  uint8_t* out_errors8 = nullptr;
  uint64_t cap_out8 = 0;
  uint8_t* seq4 = nullptr;       // BAM4 transfer columns (fgb_submit_bam4)
  uint8_t* qraw = nullptr;
  fgb_raw_read* rawreads = nullptr;
  uint64_t cap_seq4 = 0, cap_qraw = 0, cap_rawreads = 0;
  uint8_t* recblob = nullptr;    // RECORDS transfer blob (fgb_submit_ex, FGB_IN_RECORDS)
  uint64_t cap_recblob = 0;
  std::vector<fgb_tile> tile_stage;   // class-sorted copy of a chunk's tiles (host)
  fgb_record_job* recjobs = nullptr; uint64_t cap_recjobs = 0;   // record assembly (K5)
  uint8_t* recout = nullptr; uint64_t cap_recout = 0;
  // strand-combine jobs of fgb_submit_ex (duplex / CODEC callers)
  fgb_duplex_job* djobs = nullptr; uint64_t cap_djobs = 0;
  fgb_codec_job* cjobs = nullptr; uint64_t cap_cjobs = 0;
  uint8_t* c_base = nullptr; uint8_t* c_qual = nullptr; uint16_t* c_depth = nullptr; uint16_t* c_errors = nullptr;
  uint64_t cap_cout = 0;
  uint8_t* c_status = nullptr; uint32_t* c_dis = nullptr; uint32_t* c_dup = nullptr; uint64_t cap_cjobout = 0;
  uint64_t* reads = nullptr;
  fgb_unit* units = nullptr;
  fgb_tile* tiles = nullptr;
  uint8_t* out_base = nullptr;
  uint8_t* out_qual = nullptr;
  uint16_t* out_depth = nullptr;
  uint16_t* out_errors = nullptr;
  uint64_t cap_bytes = 0, cap_reads = 0, cap_units = 0, cap_tiles = 0, cap_out = 0;
};

}  // namespace

struct fgb_handle {
  int device = -1;
  int sm_count = 0;
  fgb_params params{};
  HostTables host_tables{};
  DeviceTables* d_tables = nullptr;
  unsigned long long* d_counters = nullptr;
  uint64_t launches = 0;
  std::string last_error;
  Slot slots[kSlots];
  bool submit_pending = false;
  uint32_t* d_bad = nullptr;                        // BAM4: set by the unpack kernel on a bad raw span
  bool bam4_pending = false;
  uint16_t* d_emax = nullptr;                       // filter: per-depth error-count limit
  double emax_rate = -1.0;                          // the max_base_error_rate d_emax was built for
  int n_slots = 2;                                  // FGB_SUBMIT_SLOTS (1..kSlots)
  uint64_t chunk_bytes = kChunkColumnBytes;         // FGB_SUBMIT_CHUNK_MB
  bool chunk_bytes_set = false;                     // the environment fixed it: no per-batch adjustment
  unsigned long long* d_ostats = nullptr;            // overlap pre-pass counters (device u64[4])
  uint64_t* ostats_host = nullptr;                  // where fgb_wait adds them
  fgb_overlap_run* d_oruns = nullptr; uint64_t cap_oruns = 0;
  uint8_t* d_recstr = nullptr; uint64_t cap_recstr = 0;   // record assembly: the batch's string blob
  fgb_record_job* d_recjobs = nullptr; uint64_t cap_recjobs = 0;   // ... and its per-unit jobs (both uploaded ahead of chunk 0)
  cudaEvent_t ev_recstr = nullptr;                         // ... uploaded on the first chunk's stream
  bool trace = false;                               // FGB_SUBMIT_TRACE=1: per-chunk device timeline printed by fgb_wait
  struct TraceMark { cudaEvent_t ev; const char* what; int chunk; };
  std::vector<TraceMark> trace_ev;                  // device timeline of the last submit
  std::chrono::steady_clock::time_point trace_t0, trace_t1;
  uint8_t* d_dstatus = nullptr; uint64_t cap_dstatus = 0;   // fgb_vote_duplex_device: job status bytes when the caller wants none
  struct UmiBufs {                                   // fgb_umi_assign: device buffers and their page-locked staging
    fgb_umi_key* keys = nullptr; uint8_t* blob = nullptr; fgb::UmiWork* work = nullptr;
    uint64_t* deg = nullptr; uint64_t* off = nullptr; uint32_t* edges = nullptr;
    uint64_t* sbits_in = nullptr; uint64_t* sbits = nullptr; uint32_t* sidx_in = nullptr; uint32_t* sidx = nullptr;
    uint8_t* temp = nullptr;
    uint64_t cap_keys = 0, cap_blob = 0, cap_work = 0, cap_deg = 0, cap_off = 0, cap_edges = 0, cap_sbits_in = 0,
             cap_sbits = 0, cap_sidx_in = 0, cap_sidx = 0, cap_temp = 0;
    fgb_umi_key* h_keys = nullptr; uint8_t* h_blob = nullptr; fgb::UmiWork* h_work = nullptr;
    uint64_t* h_sbits = nullptr; uint32_t* h_sidx = nullptr; uint64_t* h_off = nullptr; uint32_t* h_edges = nullptr;
    uint64_t hcap_keys = 0, hcap_blob = 0, hcap_work = 0, hcap_sbits = 0, hcap_sidx = 0, hcap_off = 0, hcap_edges = 0;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev2 = nullptr, ev3 = nullptr;   // around the count and fill passes
    double timing[4] = {0, 0, 0, 0};                 // fgb_umi_last_timing
  } umi;
  double sort_timing[6] = {0, 0, 0, 0, 0, 0};        // fgb_sort_last_timing
  double filter_timing[6] = {0, 0, 0, 0, 0, 0};      // fgb_filter_last_timing
  std::vector<uint8_t> filter_kept, filter_rejects;  // fgb_filter_records' output streams
  double zipper_timing[6] = {0, 0, 0, 0, 0, 0};      // fgb_zipper_last_timing
  std::vector<uint8_t> zipper_out;                   // fgb_zipper_records' output stream
  struct ScoreBufs {                                 // template scores (dedup_kernels.cuh): own stream, so that they run
    cudaStream_t stream = nullptr;                   // beside fgb_umi_assign; two page-locked chunks alternate
    uint8_t* h_rec[2] = {nullptr, nullptr}; uint64_t* h_off[2] = {nullptr, nullptr};
    uint8_t* d_rec[2] = {nullptr, nullptr}; uint64_t* d_off[2] = {nullptr, nullptr};
    uint64_t cap_rec = 0, cap_off = 0;               // bytes / entries of each of the four chunk buffers
    uint32_t* d_scores = nullptr; uint32_t* h_scores = nullptr; uint64_t cap_scores = 0;
    cudaEvent_t staged[2] = {nullptr, nullptr};      // the chunk's upload has left its page-locked buffers
    std::vector<cudaEvent_t> ev;                     // kernel start / stop per chunk
  } score;
};

namespace {

fgb_status cuda_fail(fgb_handle* h, cudaError_t e, const char* what) {
  if (h) {
    h->last_error = std::string(what) + ": " + cudaGetErrorString(e);
  }
  return FGB_ERR_CUDA;
}

#define FGB_CUDA(h, call)                                   \
  do {                                                      \
    cudaError_t e__ = (call);                               \
    if (e__ != cudaSuccess) return cuda_fail((h), e__, #call); \
  } while (0)

template <class T>
fgb_status ensure(fgb_handle* h, T** p, uint64_t* cap, uint64_t need) {
  if (need <= *cap && *p) return FGB_OK;
  if (*p) { cudaFree(*p); *p = nullptr; *cap = 0; }
  uint64_t n = need + need / 8 + 64;
  cudaError_t e = cudaMalloc(reinterpret_cast<void**>(p), n * sizeof(T));
  if (e != cudaSuccess) { cuda_fail(h, e, "cudaMalloc"); return FGB_ERR_NOMEM; }
  *cap = n;
  return FGB_OK;
}

// The epilogue arguments of the vote kernels with the duplex combine (fgb_vote_duplex_device).
struct DuplexEpilogueArgs {
  const fgb_tile_jobs* tile_jobs;
  const uint32_t* job_index;
  const fgb_duplex_job* jobs;
  fgb_duplex_out out;       // status non-null
};

fgb_status launch_vote(fgb_handle* h, const fgb_batch& b, const fgb_columns& out,
                       cudaStream_t stream, const DuplexEpilogueArgs* dx = nullptr) {
  if (b.n_tiles == 0) return FGB_OK;
  VoteArgsDuplex a{};
  a.bases = b.bases; a.quals = b.quals; a.reads = b.reads; a.units = b.units; a.tiles = b.tiles;
  a.n_tiles = b.n_tiles;
  a.out_base = out.base; a.out_qual = out.qual; a.out_depth = out.depth; a.out_errors = out.errors;
  a.tables = h->d_tables;
  a.counters = h->d_counters;
  a.min_reads = h->params.min_reads;
  a.min_cons_q = h->params.min_consensus_base_quality;
  a.fast_qual = h->host_tables.fast_qual;
  if (dx) {
    a.tile_jobs = dx->tile_jobs; a.job_index = dx->job_index; a.djobs = dx->jobs;
    a.d_base = dx->out.base; a.d_qual = dx->out.qual; a.d_errors = dx->out.errors; a.d_status = dx->out.status;
  }
  const uint64_t max_grid = static_cast<uint64_t>(h->sm_count) * 2u;
  const uint64_t c0 = b.class_tiles[0], c1 = b.class_tiles[1], c2 = b.class_tiles[2];
  const bool sorted = c0 + c1 + c2 == b.n_tiles;
  auto launch = [&](int cls, uint64_t first, uint64_t n) {
    if (!n) return;
    VoteArgsDuplex x = a;
    x.tiles = b.tiles + first;
    x.n_tiles = n;
    const unsigned grid = static_cast<unsigned>(std::min<uint64_t>(n, max_grid));
    if (dx) {
      x.tile_jobs = dx->tile_jobs + first;
      if (cls == 1) vote_kernel_shallow_duplex<<<grid, kThreads, sizeof(VoteSmem) + kShallowSmemBytes, stream>>>(x);
      else if (cls == 2) vote_kernel_deep_duplex<<<grid, kThreads, sizeof(VoteSmem) + kDeepSmemBytes, stream>>>(x);
      else vote_kernel_duplex<<<grid, kThreads, sizeof(VoteSmem), stream>>>(x);
    } else {
      const VoteArgs& v = x;
      if (cls == 1) vote_kernel_shallow<<<grid, kThreads, sizeof(VoteSmem) + kShallowSmemBytes, stream>>>(v);
      else if (cls == 2) vote_kernel_deep<<<grid, kThreads, sizeof(VoteSmem) + kDeepSmemBytes, stream>>>(v);
      else vote_kernel<<<grid, kThreads, sizeof(VoteSmem) + kPileSmemBytes, stream>>>(v);
    }
    h->launches++;
  };
  if (sorted) { launch(0, 0, c0); launch(1, c0, c1); launch(2, c0 + c1, c2); }
  else launch(0, 0, b.n_tiles);
  FGB_CUDA(h, cudaGetLastError());
  return FGB_OK;
}

// The device pointers the vote kernels can use: bulk copies (cp.async.bulk) read bases, quals, reads and units from
// 16-byte aligned addresses, tiles are read as 16-byte words, and the outputs are written 8 positions at a time
// (8-byte words of base / qual, 16-byte words of depth / errors).  Checked before anything is enqueued.
fgb_status check_vote_pointers(fgb_handle* h, const fgb_batch& b, const fgb_columns& out, const char* who) {
  if (b.n_tiles == 0) return FGB_OK;
  const struct { const void* p; uintptr_t align; const char* name; } ptrs[] = {
      {b.bases, 16, "bases"}, {b.quals, 16, "quals"}, {b.reads, 16, "reads"}, {b.units, 16, "units"},
      {b.tiles, 16, "tiles"}, {out.base, 8, "output base"}, {out.qual, 8, "output qual"},
      {out.depth, 16, "output depth"}, {out.errors, 16, "output errors"}};
  for (const auto& x : ptrs) {
    if (reinterpret_cast<uintptr_t>(x.p) % x.align) {
      h->last_error = std::string(who) + ": " + x.name + " is not " + std::to_string(x.align) + "-byte aligned";
      return FGB_ERR_LAYOUT;
    }
  }
  return FGB_OK;
}

}  // namespace

extern "C" {

fgb_status fgb_sort_tiles_by_class(fgb_tile* tiles, uint64_t n_tiles, uint64_t class_tiles[3]) {
  if ((n_tiles && !tiles) || !class_tiles) return FGB_ERR_INVALID_ARG;
  class_tiles[0] = class_tiles[1] = class_tiles[2] = 0;
  std::stable_sort(tiles, tiles + n_tiles, [](const fgb_tile& x, const fgb_tile& y) {
    return ((x.flags & kTileClassMask) >> kTileClassShift) < ((y.flags & kTileClassMask) >> kTileClassShift);
  });
  for (uint64_t i = 0; i < n_tiles; ++i) {
    const uint32_t c = (tiles[i].flags & kTileClassMask) >> kTileClassShift;
    class_tiles[c < 3 ? c : 0]++;
  }
  return FGB_OK;
}

}  // extern "C"

namespace {
}  // namespace

extern "C" {

uint32_t fgb_abi_version(void) { return FGB_ABI_VERSION; }

const char* fgb_strerror(fgb_status s) {
  switch (s) {
    case FGB_OK: return "ok";
    case FGB_ERR_INVALID_ARG: return "invalid argument";
    case FGB_ERR_CUDA: return "CUDA runtime error";
    case FGB_ERR_NO_DEVICE: return "no usable sm_90 CUDA device (this engine has no CPU fallback)";
    case FGB_ERR_LAYOUT: return "batch violates the SoA layout rules";
    case FGB_ERR_UNIT_TOO_LARGE: return "unit exceeds the supported size";
    case FGB_ERR_NOMEM: return "out of memory";
    case FGB_ERR_BUSY: return "a previous fgb_submit has not been waited on";
    case FGB_ERR_MISSING_TAG: return "first record of the group has no UMI tag";
    case FGB_ERR_NOT_ENCODABLE: return "observation outside the PACK8 alphabet";
    default: return "unknown status";
  }
}

size_t fgb_last_error(const fgb_handle* h, char* buf, size_t buf_len) {
  if (!h) return 0;
  if (buf && buf_len) {
    size_t n = std::min(buf_len - 1, h->last_error.size());
    std::memcpy(buf, h->last_error.data(), n);
    buf[n] = 0;
  }
  return h->last_error.size();
}

fgb_status fgb_create(int device, const fgb_params* params, fgb_handle** out) {
  if (!params || !out) return FGB_ERR_INVALID_ARG;
  if (params->error_rate_pre_umi > FGB_MAX_PHRED || params->error_rate_post_umi > FGB_MAX_PHRED ||
      params->min_reads == 0)
    return FGB_ERR_INVALID_ARG;
  *out = nullptr;
  int n_dev = 0;
  if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev <= 0 || device < 0 || device >= n_dev) {
    cudaGetLastError();
    return FGB_ERR_NO_DEVICE;
  }
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return FGB_ERR_NO_DEVICE;
  if (prop.major != 9 || prop.minor != 0) return FGB_ERR_NO_DEVICE;   // kernels are sm_90a only
  fgb_handle* h = new (std::nothrow) fgb_handle();
  if (!h) return FGB_ERR_NOMEM;
  h->device = device;
  h->sm_count = prop.multiProcessorCount;
  if (const char* e = std::getenv("FGB_SUBMIT_SLOTS")) h->n_slots = std::max(1, std::min(kSlots, std::atoi(e)));
  if (const char* e = std::getenv("FGB_SUBMIT_CHUNK_MB"))
    { h->chunk_bytes = static_cast<uint64_t>(std::max(1, std::atoi(e))) << 20; h->chunk_bytes_set = true; }
  if (const char* e = std::getenv("FGB_SUBMIT_TRACE")) h->trace = std::atoi(e) != 0;
  h->params = *params;
  build_host_tables(params->error_rate_pre_umi, params->error_rate_post_umi, &h->host_tables);

  auto fail = [&](cudaError_t e, const char* what) {
    fprintf(stderr, "fgumi_b200: fgb_create: %s: %s\n", what, cudaGetErrorString(e));
    fgb_destroy(h);
    return FGB_ERR_CUDA;
  };
  cudaError_t e;
  if ((e = cudaSetDevice(device)) != cudaSuccess) return fail(e, "cudaSetDevice");
  if ((e = cudaMalloc(&h->d_tables, sizeof(DeviceTables))) != cudaSuccess) return fail(e, "cudaMalloc tables");
  if ((e = cudaMalloc(&h->d_counters, sizeof(unsigned long long) * FGB_NCOUNTERS)) != cudaSuccess)
    return fail(e, "cudaMalloc counters");
  DeviceTables dt;
  std::memset(&dt, 0, sizeof(dt));
  std::memcpy(dt.correct, h->host_tables.correct, sizeof(dt.correct));
  std::memcpy(dt.err_alt, h->host_tables.err_alt, sizeof(dt.err_alt));
  dt.ln_pre = h->host_tables.ln_pre;
  std::memcpy(dt.single_q, h->host_tables.single_q, sizeof(dt.single_q));
  std::memcpy(dt.qt, h->host_tables.qt, sizeof(dt.qt));
  std::memcpy(dt.dfix, h->host_tables.dfix, sizeof(dt.dfix));
  dt.g2fix = h->host_tables.g2fix;
  dt.nmax2 = h->host_tables.nmax2;
  std::memcpy(dt.pair_q, h->host_tables.pair_q, sizeof(dt.pair_q));
  std::memcpy(dt.sumt, h->host_tables.sumt, sizeof(dt.sumt));
  std::memcpy(dt.qt3, h->host_tables.qt3, sizeof(dt.qt3));
  std::memcpy(dt.ugap_bp, h->host_tables.ugap_bp, sizeof(dt.ugap_bp));
  std::memcpy(dt.ugap_q, h->host_tables.ugap_q, sizeof(dt.ugap_q));
  if ((e = cudaMemcpy(h->d_tables, &dt, sizeof(dt), cudaMemcpyHostToDevice)) != cudaSuccess)
    return fail(e, "cudaMemcpy tables");
  if ((e = cudaMemset(h->d_counters, 0, sizeof(unsigned long long) * FGB_NCOUNTERS)) != cudaSuccess)
    return fail(e, "cudaMemset counters");
  if ((e = cudaFuncSetAttribute(vote_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                static_cast<int>(sizeof(VoteSmem) + kPileSmemBytes))) != cudaSuccess)
    return fail(e, "cudaFuncSetAttribute(vote_kernel)");
  if ((e = cudaFuncSetAttribute(vote_kernel_shallow, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                static_cast<int>(sizeof(VoteSmem) + kShallowSmemBytes))) != cudaSuccess)
    return fail(e, "cudaFuncSetAttribute(vote_kernel_shallow)");
  if ((e = cudaFuncSetAttribute(vote_kernel_deep, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                static_cast<int>(sizeof(VoteSmem) + kDeepSmemBytes))) != cudaSuccess)
    return fail(e, "cudaFuncSetAttribute(vote_kernel_deep)");
  if ((e = cudaFuncSetAttribute(vote_kernel_duplex, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                static_cast<int>(sizeof(VoteSmem)))) != cudaSuccess ||
      (e = cudaFuncSetAttribute(vote_kernel_shallow_duplex, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                static_cast<int>(sizeof(VoteSmem) + kShallowSmemBytes))) != cudaSuccess ||
      (e = cudaFuncSetAttribute(vote_kernel_deep_duplex, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                static_cast<int>(sizeof(VoteSmem) + kDeepSmemBytes))) != cudaSuccess)
    return fail(e, "cudaFuncSetAttribute(vote_kernel_*_duplex)");
  for (int s = 0; s < kSlots; ++s)
    if ((e = cudaStreamCreateWithFlags(&h->slots[s].stream, cudaStreamNonBlocking)) != cudaSuccess)
      return fail(e, "cudaStreamCreate");
  *out = h;
  return FGB_OK;
}

void fgb_destroy(fgb_handle* h) {
  if (!h) return;
  if (h->device >= 0) cudaSetDevice(h->device);
  for (int s = 0; s < kSlots; ++s) {
    Slot& sl = h->slots[s];
    if (sl.stream) { cudaStreamSynchronize(sl.stream); cudaStreamDestroy(sl.stream); }
    cudaFree(sl.bases); cudaFree(sl.quals); cudaFree(sl.packed); cudaFree(sl.unit_status); cudaFree(sl.unit_masked); cudaFree(sl.out_depth8); cudaFree(sl.out_errors8); cudaFree(sl.seq4); cudaFree(sl.qraw); cudaFree(sl.rawreads); cudaFree(sl.recblob); cudaFree(sl.djobs); cudaFree(sl.cjobs); cudaFree(sl.c_base); cudaFree(sl.c_qual); cudaFree(sl.c_depth); cudaFree(sl.c_errors); cudaFree(sl.c_status); cudaFree(sl.c_dis); cudaFree(sl.c_dup); cudaFree(sl.recjobs); cudaFree(sl.recout); cudaFree(sl.reads); cudaFree(sl.units);
    cudaFree(sl.tiles); cudaFree(sl.out_base); cudaFree(sl.out_qual); cudaFree(sl.out_depth);
    cudaFree(sl.out_errors);
  }
  cudaFree(h->d_tables);
  cudaFree(h->d_counters);
  cudaFree(h->d_emax);
  cudaFree(h->d_bad);
  cudaFree(h->d_ostats);
  cudaFree(h->d_oruns);
  cudaFree(h->d_recstr); cudaFree(h->d_recjobs);
  cudaFree(h->d_dstatus);
  {
    auto& u = h->umi;
    cudaFree(u.keys); cudaFree(u.blob); cudaFree(u.work); cudaFree(u.deg); cudaFree(u.off); cudaFree(u.edges);
    cudaFree(u.sbits_in); cudaFree(u.sbits); cudaFree(u.sidx_in); cudaFree(u.sidx); cudaFree(u.temp);
    cudaFreeHost(u.h_keys); cudaFreeHost(u.h_blob); cudaFreeHost(u.h_work); cudaFreeHost(u.h_sbits);
    cudaFreeHost(u.h_sidx); cudaFreeHost(u.h_off); cudaFreeHost(u.h_edges);
    for (cudaEvent_t ev : {u.ev0, u.ev1, u.ev2, u.ev3}) if (ev) cudaEventDestroy(ev);
  }
  {
    auto& c = h->score;
    if (c.stream) { cudaStreamSynchronize(c.stream); cudaStreamDestroy(c.stream); }
    for (int b = 0; b < 2; ++b) {
      cudaFreeHost(c.h_rec[b]); cudaFreeHost(c.h_off[b]); cudaFree(c.d_rec[b]); cudaFree(c.d_off[b]);
      if (c.staged[b]) cudaEventDestroy(c.staged[b]);
    }
    cudaFree(c.d_scores); cudaFreeHost(c.h_scores);
    for (cudaEvent_t ev : c.ev) cudaEventDestroy(ev);
  }
  if (h->ev_recstr) cudaEventDestroy(h->ev_recstr);
  delete h;
}

fgb_status fgb_get_tables(const fgb_handle* h, double* correct, double* err_alt, double* ln_pre,
                          uint8_t* single_input_q) {
  if (!h) return FGB_ERR_INVALID_ARG;
  if (correct) std::memcpy(correct, h->host_tables.correct, sizeof(double) * FGB_NTABLE);
  if (err_alt) std::memcpy(err_alt, h->host_tables.err_alt, sizeof(double) * FGB_NTABLE);
  if (ln_pre) *ln_pre = h->host_tables.ln_pre;
  if (single_input_q) std::memcpy(single_input_q, h->host_tables.single_q, FGB_NTABLE);
  return FGB_OK;
}

fgb_status fgb_host_tables(uint8_t pre, uint8_t post, double* correct, double* err_alt,
                           double* ln_pre, uint8_t* single_input_q, uint8_t* qt,
                           uint32_t* fast_qual) {
  if (pre > FGB_MAX_PHRED || post > FGB_MAX_PHRED) return FGB_ERR_INVALID_ARG;
  HostTables t;
  build_host_tables(pre, post, &t);
  if (correct) std::memcpy(correct, t.correct, sizeof(double) * FGB_NTABLE);
  if (err_alt) std::memcpy(err_alt, t.err_alt, sizeof(double) * FGB_NTABLE);
  if (ln_pre) *ln_pre = t.ln_pre;
  if (single_input_q) std::memcpy(single_input_q, t.single_q, FGB_NTABLE);
  if (qt) std::memcpy(qt, t.qt, sizeof(t.qt));
  if (fast_qual) *fast_qual = t.fast_qual;
  return FGB_OK;
}

fgb_status fgb_host_proof_tables(uint8_t pre, uint8_t post, int32_t* dfix, int32_t* g2fix,
                                 uint32_t* nmax2) {
  if (pre > FGB_MAX_PHRED || post > FGB_MAX_PHRED) return FGB_ERR_INVALID_ARG;
  HostTables t;
  build_host_tables(pre, post, &t);
  if (dfix) std::memcpy(dfix, t.dfix, sizeof(t.dfix));
  if (g2fix) *g2fix = t.g2fix;
  if (nmax2) *nmax2 = t.nmax2;
  return FGB_OK;
}

fgb_status fgb_host_unanimous_steps(uint8_t pre, uint8_t post, int32_t* gap_begin, uint8_t* quality,
                                    uint32_t* n_steps, int32_t* guard) {
  if (pre > FGB_MAX_PHRED || post > FGB_MAX_PHRED) return FGB_ERR_INVALID_ARG;
  HostTables t;
  build_host_tables(pre, post, &t);
  if (gap_begin) std::memcpy(gap_begin, t.ugap_bp, sizeof(t.ugap_bp));
  if (quality) std::memcpy(quality, t.ugap_q, sizeof(t.ugap_q));
  if (n_steps) *n_steps = t.ugap_n;
  if (guard) *guard = kUgapGuard;
  return FGB_OK;
}

// ---- planner ------------------------------------------------------------------------------------
uint32_t fgb_tile_capacity_bytes(void) { return kTileCapBytes; }
uint32_t fgb_tile_max_units(void) { return kTileMaxUnits; }
uint32_t fgb_tile_max_reads(void) { return kTileMaxReads; }

#if FGB_PIPE_TRACE
// Diagnostic builds only (scripts/pipe_trace.py): copies the vote kernels' stall counters (vote_kernel.cuh
// g_pipe_trace) to out[kPipeTraceWords] and zeroes them.  Not declared in the public header.
fgb_status fgb_pipe_trace(uint64_t* out) {
  unsigned long long h[kPipeTraceWords];
  if (!out) return FGB_ERR_INVALID_ARG;
  if (cudaDeviceSynchronize() != cudaSuccess || cudaMemcpyFromSymbol(h, g_pipe_trace, sizeof(h)) != cudaSuccess)
    return FGB_ERR_CUDA;
  std::memcpy(out, h, sizeof(h));
  std::memset(h, 0, sizeof(h));
  if (cudaMemcpyToSymbol(g_pipe_trace, h, sizeof(h)) != cudaSuccess) return FGB_ERR_CUDA;
  return FGB_OK;
}
#endif

fgb_status fgb_plan_tiles(const fgb_unit* units, uint64_t n_units, const fgb_read_desc* reads,
                          uint64_t n_reads, fgb_tile* out, uint64_t cap, uint64_t* n_tiles) {
  if (!n_tiles || (n_units && (!units || (!reads && n_reads)))) return FGB_ERR_INVALID_ARG;
  if (n_units >= 0xFFFFFFFFull || n_reads >= 0xFFFFFFFFull) return FGB_ERR_INVALID_ARG;
  if (n_units && units[0].read_begin != 0) return FGB_ERR_LAYOUT;
  uint64_t nt = 0, prev_read_end = 0;
  fgb_status st = plan_tiles_range(units, 0, n_units, reads, n_reads, &prev_read_end, [&](const fgb_tile& t) {
    if (out && nt < cap) out[nt] = t;
    ++nt;
  });
  if (st != FGB_OK) return st;
  *n_tiles = nt;
  return FGB_OK;
}

// Planner for the duplex epilogue: see include/fgumi_b200.h.
constexpr uint64_t kGlueSpanMax = 16;     // a job keeps its units (and those between them) together up to this distance
fgb_status fgb_plan_tiles_jobs(const fgb_unit* units, uint64_t n_units, const fgb_read_desc* reads,
                               uint64_t n_reads, const fgb_duplex_job* jobs, uint64_t n_jobs,
                               fgb_tile* tiles, uint64_t cap, uint64_t* n_tiles, uint64_t class_tiles[3],
                               fgb_tile_jobs* tile_jobs, uint32_t* job_index, uint64_t* n_attached) {
  if (!n_tiles || (n_units && (!units || (!reads && n_reads))) || (n_jobs && !jobs)) return FGB_ERR_INVALID_ARG;
  if (n_units >= 0xFFFFFFFFull || n_reads >= 0xFFFFFFFFull || n_jobs >= 0xFFFFFFFFull) return FGB_ERR_INVALID_ARG;
  if (n_units && units[0].read_begin != 0) return FGB_ERR_LAYOUT;
  try {
    // glue[u]: some job has one unit before u and the other at or after it
    std::vector<int32_t> diff(n_units + 2, 0);
    for (uint64_t j = 0; j < n_jobs; ++j) {
      const uint64_t a = jobs[j].unit_a, b = jobs[j].unit_b;
      if (a >= n_units || b >= n_units) return FGB_ERR_INVALID_ARG;
      const uint64_t lo = std::min(a, b), hi = std::max(a, b);
      if (hi > lo && hi - lo < kGlueSpanMax) { diff[lo + 1]++; diff[hi + 1]--; }   // partners far apart share no tile anyway
    }
    std::vector<uint8_t> glue(n_units + 1, 0);
    int32_t acc = 0;
    for (uint64_t u = 0; u <= n_units; ++u) { acc += diff[u]; glue[u] = acc > 0 ? 1 : 0; }
    diff = std::vector<int32_t>();
    std::vector<fgb_tile> plan;
    uint64_t prev_read_end = 0;
    fgb_status st = plan_tiles_range(units, 0, n_units, reads, n_reads, &prev_read_end,
                                     [&](const fgb_tile& t) { plan.push_back(t); }, glue.data());
    if (st != FGB_OK) return st;
    const uint64_t nt = plan.size();
    *n_tiles = nt;
    if (!tiles || cap < nt) return FGB_OK;                    // sizing call
    if (!class_tiles || (nt && !tile_jobs) || (n_jobs && !job_index)) return FGB_ERR_INVALID_ARG;
    // tiles in class order (stable), as fgb_sort_tiles_by_class leaves them
    std::vector<uint32_t> order(nt);
    for (uint64_t i = 0; i < nt; ++i) order[i] = static_cast<uint32_t>(i);
    auto cls_of = [&](uint32_t i) { const uint32_t c = (plan[i].flags & kTileClassMask) >> kTileClassShift; return c < 3 ? c : 0u; };
    std::stable_sort(order.begin(), order.end(), [&](uint32_t x, uint32_t y) { return cls_of(x) < cls_of(y); });
    class_tiles[0] = class_tiles[1] = class_tiles[2] = 0;
    std::vector<uint32_t> tile_of(n_units);                   // unit -> tile (position in class order)
    for (uint64_t k = 0; k < nt; ++k) {
      const fgb_tile& t = plan[order[k]];
      tiles[k] = t;
      tile_jobs[k] = fgb_tile_jobs{0u, 0u, 0u};
      class_tiles[cls_of(order[k])]++;
      for (uint32_t u = t.unit_begin; u < t.unit_begin + t.n_units; ++u) tile_of[u] = static_cast<uint32_t>(k);
    }
    auto attach_to = [&](uint64_t j) -> int64_t {            // the tile a job runs in, or -1
      const uint32_t ta = tile_of[jobs[j].unit_a];
      if (ta != tile_of[jobs[j].unit_b] || (tiles[ta].flags & kTileFlagDirect)) return -1;
      return ta;
    };
    for (uint64_t j = 0; j < n_jobs; ++j) {
      const int64_t t = attach_to(j);
      if (t < 0 || tile_jobs[t].count == 0xFFFFu) continue;
      tile_jobs[t].count++;
      const uint32_t la = units[jobs[j].unit_a].cons_len, lb = units[jobs[j].unit_b].cons_len;
      const uint32_t items = (std::min(la, lb) + 7u) >> 3;
      tile_jobs[t].max_items = static_cast<uint16_t>(std::max<uint32_t>(tile_jobs[t].max_items, items));
    }
    uint64_t total = 0;
    for (uint64_t k = 0; k < nt; ++k) { tile_jobs[k].begin = static_cast<uint32_t>(total); total += tile_jobs[k].count; }
    std::vector<uint16_t> fill(nt, 0);
    for (uint64_t j = 0; j < n_jobs; ++j) {
      const int64_t t = attach_to(j);
      if (t < 0 || fill[t] == tile_jobs[t].count) continue;
      job_index[tile_jobs[t].begin + fill[t]++] = static_cast<uint32_t>(j);
    }
    if (n_attached) *n_attached = total;
  } catch (const std::bad_alloc&) {
    return FGB_ERR_NOMEM;
  }
  return FGB_OK;
}

// ---- vote ---------------------------------------------------------------------------------------
fgb_status fgb_vote_device(fgb_handle* h, const fgb_batch* in, const fgb_columns* out,
                           void* stream) {
  if (!h || !in || !out) return FGB_ERR_INVALID_ARG;
  if (in->n_tiles && (!in->tiles || !in->units || !out->base || !out->qual || !out->depth ||
                      !out->errors))
    return FGB_ERR_INVALID_ARG;
  fgb_status st = check_vote_pointers(h, *in, *out, "fgb_vote_device");
  if (st != FGB_OK) return st;
  FGB_CUDA(h, cudaSetDevice(h->device));
  return launch_vote(h, *in, *out, static_cast<cudaStream_t>(stream));
}

fgb_status fgb_host_alloc(void** p, size_t bytes) {
  if (!p) return FGB_ERR_INVALID_ARG;
  cudaError_t e = cudaHostAlloc(p, bytes ? bytes : 1, cudaHostAllocDefault);
  if (e != cudaSuccess) { cudaGetLastError(); *p = nullptr; return FGB_ERR_NOMEM; }
  return FGB_OK;
}
void fgb_host_free(void* p) { if (p) cudaFreeHost(p); }
int fgb_host_is_pinned(const void* p) {
  if (!p) return 0;
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return 0; }
  return at.type == cudaMemoryTypeHost ? 1 : 0;
}

}  // extern "C"

namespace {
enum class HostFormat { kBytes, kPack8, kBam4, kRecords };

// emax[d] = largest error count e (<= d) with (double)e / (double)d <= rate, i.e. exactly the
// positions mask_bases keeps (`errors / depth > max_base_error_rate` masks, filter.rs:681-684).
// Built with the same f64 division the reference performs; e -> e/d is monotone, so bisect.
fgb_status ensure_emax(fgb_handle* h, double rate, cudaStream_t s) {
  if (h->d_emax && h->emax_rate == rate) return FGB_OK;
  std::vector<uint16_t> t(65536, 0);
  for (uint32_t d = 1; d < 65536; ++d) {
    uint32_t lo = 0, hi = d;           // invariant: lo passes (0/d = 0 <= rate unless rate < 0)
    if (!(0.0 / static_cast<double>(d) > rate)) {
      while (lo < hi) {
        uint32_t mid = (lo + hi + 1) >> 1;
        if (static_cast<double>(mid) / static_cast<double>(d) > rate) hi = mid - 1; else lo = mid;
      }
      t[d] = static_cast<uint16_t>(lo);
    } else {
      t[d] = 0;                        // negative rate: even zero errors would be masked; the kernel's
    }                                  // `e > emax` cannot express that, fgb_filter_* rejects rate < 0
  }
  if (!h->d_emax) FGB_CUDA(h, cudaMalloc(&h->d_emax, 65536 * sizeof(uint16_t)));
  FGB_CUDA(h, cudaStreamSynchronize(s));   // the table may still be in use by an earlier launch
  FGB_CUDA(h, cudaMemcpy(h->d_emax, t.data(), 65536 * sizeof(uint16_t), cudaMemcpyHostToDevice));
  h->emax_rate = rate;
  return FGB_OK;
}

bool filter_params_ok(const fgb_filter_params* fp) {
  return fp && fp->max_base_error_rate >= 0.0 && fp->max_no_call_fraction >= 0.0 &&
         fp->min_base_quality <= 255 && fp->min_base_quality >= -1;
}

fgb_status launch_filter(fgb_handle* h, const fgb_unit* units, uint64_t u0, uint64_t u1,
                         const fgb_columns& cols, const fgb_filter_params& fp, uint8_t* status,
                         uint32_t* masked, cudaStream_t s) {
  if (u1 <= u0) return FGB_OK;
  FilterArgs a;
  a.units = units; a.unit_begin = u0; a.unit_end = u1;
  a.base = cols.base; a.qual = cols.qual; a.depth = cols.depth; a.errors = cols.errors;
  a.emax = h->d_emax; a.status = status; a.masked = masked; a.counters = h->d_counters;
  a.min_reads = fp.min_reads;
  a.min_base_quality = fp.min_base_quality < 0 ? 0u : static_cast<uint32_t>(fp.min_base_quality);
  a.per_base_tags = fp.per_base_tags;
  a.max_read_error_rate = fp.max_read_error_rate;
  a.min_mean_base_quality = fp.min_mean_base_quality;
  a.max_no_call_fraction = fp.max_no_call_fraction;
  const uint64_t n = u1 - u0;
  const uintptr_t align8 = reinterpret_cast<uintptr_t>(a.base) | reinterpret_cast<uintptr_t>(a.qual);
  const uintptr_t align16 = reinterpret_cast<uintptr_t>(a.depth) | reinterpret_cast<uintptr_t>(a.errors);
  const uint64_t chunks = (n + kFilterChunk - 1) / kFilterChunk;
  if ((align8 & 7u) == 0 && (align16 & 15u) == 0 && chunks <= 0x7FFFFFFFull) {
    filter_simplex_words_kernel<<<static_cast<unsigned>(chunks), 256, 0, s>>>(a);   // 8 positions per thread
  } else {
    const unsigned grid = static_cast<unsigned>(std::min<uint64_t>((n + 7u) / 8u, static_cast<uint64_t>(h->sm_count) * 16u));
    filter_simplex_kernel<<<grid, 256, 0, s>>>(a);
  }
  h->launches++;
  FGB_CUDA(h, cudaGetLastError());
  return FGB_OK;
}

// `padded`: both columns may be read up to the next multiple of 4 bytes past the resident range (the submit path's
// staging buffers; a caller's columns whose sizes are multiples of 4).
fgb_status launch_unpack_bam4(fgb_handle* h, Bam4Args a, cudaStream_t s, bool padded) {
  const uint64_t n = a.read_end - a.read_begin;
  if (n == 0) return FGB_OK;
  if (!h->d_bad) {
    FGB_CUDA(h, cudaMalloc(&h->d_bad, sizeof(uint32_t)));
    FGB_CUDA(h, cudaMemset(h->d_bad, 0, sizeof(uint32_t)));
  }
  a.bad = h->d_bad;
  h->bam4_pending = true;
  const bool aligned = ((reinterpret_cast<uintptr_t>(a.seq4 + (a.raw_lo >> 1)) | reinterpret_cast<uintptr_t>(a.quals_raw + a.raw_lo)) & 3u) == 0;
  if (padded && aligned) {       // flat (read, word) items; window loads guarded to the resident range
    const unsigned grid = static_cast<unsigned>(std::min<uint64_t>((n + kRowChunk - 1) / kRowChunk, static_cast<uint64_t>(h->sm_count) * 8u));
    unpack_bam4_words_kernel<<<grid, 256, 0, s>>>(a);
  } else {                       // one warp per read, byte loads: any alignment, touches nothing but the spans
    const unsigned grid = static_cast<unsigned>(std::min<uint64_t>((n + 7u) / 8u, static_cast<uint64_t>(h->sm_count) * 16u));
    unpack_bam4_kernel<<<grid, 256, 0, s>>>(a);
  }
  h->launches++;
  FGB_CUDA(h, cudaGetLastError());
  return FGB_OK;
}

fgb_status launch_unpack_records(fgb_handle* h, RecordsArgs a, cudaStream_t s) {
  const uint64_t n = a.read_end - a.read_begin;
  if (n == 0) return FGB_OK;
  if (!h->d_bad) {
    FGB_CUDA(h, cudaMalloc(&h->d_bad, sizeof(uint32_t)));
    FGB_CUDA(h, cudaMemset(h->d_bad, 0, sizeof(uint32_t)));
  }
  a.bad = h->d_bad;
  h->bam4_pending = true;
  const unsigned grid = static_cast<unsigned>(std::min<uint64_t>((n + kRowChunk - 1) / kRowChunk, static_cast<uint64_t>(h->sm_count) * 8u));
  unpack_records_kernel<<<grid, 256, 0, s>>>(a);
  h->launches++;
  FGB_CUDA(h, cudaGetLastError());
  return FGB_OK;
}

fgb_status submit_impl(fgb_handle* h, const fgb_batch* in, const fgb_columns* out, HostFormat fmt,
                       const fgb_raw_columns* raw = nullptr, bool narrow = false,
                       const fgb_submit_options* opt = nullptr) {
  if (!h || !in || !out) return FGB_ERR_INVALID_ARG;
  if (h->submit_pending) return FGB_ERR_BUSY;
  if (in->n_tiles == 0) return FGB_OK;
  const fgb_filter_params* fp = opt ? opt->filter : nullptr;
  if (fp) {
    if (!filter_params_ok(fp) || !opt->unit_status) return FGB_ERR_INVALID_ARG;
    FGB_CUDA(h, cudaSetDevice(h->device));
    for (int i = 0; i < kSlots; ++i)     // the table is shared by every slot stream
      if (h->slots[i].stream) FGB_CUDA(h, cudaStreamSynchronize(h->slots[i].stream));
    fgb_status es = ensure_emax(h, fp->max_base_error_rate, h->slots[0].stream);
    if (es != FGB_OK) return es;
  }
  if (narrow) {
    if (!in->units) return FGB_ERR_INVALID_ARG;
    for (uint64_t u = 0; u < in->n_units; ++u)
      if (in->units[u + 1].read_begin - in->units[u].read_begin > 255u) {
        h->last_error = "FGB_OUT_U8 needs every unit to have at most 255 reads";
        return FGB_ERR_INVALID_ARG;
      }
  }
  if (fmt == HostFormat::kBam4 &&
      (!in->reads || !raw || !raw->seq4 || !raw->quals_raw || !raw->raw_reads))
    return FGB_ERR_INVALID_ARG;
  const fgb_record_columns* rec = opt ? opt->records : nullptr;
  if (fmt == HostFormat::kRecords && (!in->reads || !rec || !rec->records || !rec->raw_reads))
    return FGB_ERR_INVALID_ARG;
  const uint64_t n_djobs = opt ? opt->n_duplex_jobs : 0, n_cjobs = opt ? opt->n_codec_jobs : 0;
  if (n_djobs && (!opt->duplex_jobs || !opt->duplex_out || !opt->duplex_out->base || !opt->duplex_out->qual ||
                  !opt->duplex_out->errors))
    return FGB_ERR_INVALID_ARG;
  if (n_cjobs && (!opt->codec_jobs || !opt->codec_out || !opt->codec_params || !opt->codec_out->status ||
                  !opt->codec_out->cols.base || !opt->codec_out->cols.qual || !opt->codec_out->cols.depth ||
                  !opt->codec_out->cols.errors))
    return FGB_ERR_INVALID_ARG;
  if ((n_djobs || n_cjobs) && (narrow || fp || (n_djobs && n_cjobs))) return FGB_ERR_INVALID_ARG;
  const uint64_t n_oruns = (opt && fmt == HostFormat::kRecords) ? opt->n_overlap_runs : 0;
  if (n_oruns && (!opt->overlap_runs || opt->overlap_agreement > 2 || opt->overlap_disagreement > 2)) return FGB_ERR_INVALID_ARG;
  const bool one_piece = n_djobs || n_cjobs || n_oruns;   // a molecule's units are voted before its combine job runs;
                                                          // a pair's two records must be resident together

  const fgb_record_job* rjobs = opt ? opt->rec_jobs : nullptr;
  if (rjobs && (narrow || fp || n_djobs || n_cjobs || !opt->rec_strings || !opt->rec_out ||
                opt->n_rec_string_bytes < static_cast<uint64_t>(opt->rec_prefix_len) + opt->rec_rg_len))
    return FGB_ERR_INVALID_ARG;
  const bool rows_on_device = fmt == HostFormat::kBam4 || fmt == HostFormat::kRecords;
  if (!in->tiles || !in->units || !in->reads || (!rows_on_device && !in->bases) ||
      (fmt == HostFormat::kBytes && !in->quals) ||
      (!rjobs && (!out->base || !out->qual || !out->depth || !out->errors)))
    return FGB_ERR_INVALID_ARG;
  FGB_CUDA(h, cudaSetDevice(h->device));
  h->submit_pending = true;
  // Any early return below leaves copies in flight that target the caller's buffers: drain them and
  // clear the pending flag so the handle stays usable.
  struct Guard {
    fgb_handle* h; bool ok = false;
    ~Guard() {
      if (ok) return;
      for (int i = 0; i < kSlots; ++i) if (h->slots[i].stream) cudaStreamSynchronize(h->slots[i].stream);
      h->submit_pending = false;
    }
  } guard{h};

  const fgb_tile* T = in->tiles;
  uint64_t t0 = 0;
  int chunk = 0;
  // Chunk size: the first upload and the last copy back are not overlapped with anything, so a batch is cut into at
  // least ~8 chunks (a record-level batch of 200 k families is 240 MB per column: 96 MB chunks left a third of the
  // link time exposed); large batches keep the default, below 24 MB the per-chunk launches start to show.
  const uint64_t chunk_bytes = h->chunk_bytes_set ? h->chunk_bytes
                               : std::min<uint64_t>(h->chunk_bytes, std::max<uint64_t>(24ull << 20, in->n_bytes / 8u));
  if (h->trace) {
    for (auto& m : h->trace_ev) cudaEventDestroy(m.ev);
    h->trace_ev.clear();
    h->trace_t0 = std::chrono::steady_clock::now();
  }
  auto mark = [&](cudaStream_t st, const char* what) {
    if (!h->trace) return;
    cudaEvent_t e = nullptr;
    if (cudaEventCreate(&e) == cudaSuccess) { cudaEventRecord(e, st); h->trace_ev.push_back({e, what, chunk}); }
  };
  while (t0 < in->n_tiles) {
    // Grow the chunk tile by tile up to kChunkColumnBytes of column bytes.
    uint64_t t1 = t0;
    const uint64_t byte0 = T[t0].flags & kTileFlagDirect
                               ? (FGB_READ_OFF(in->reads[T[t0].read_begin]) & ~15ull)
                               : T[t0].byte_begin;
    uint64_t byte1 = byte0;
    while (t1 < in->n_tiles) {
      const fgb_tile& tl = T[t1];
      uint64_t end;
      if (tl.flags & kTileFlagDirect) {
        fgb_read_desc last = in->reads[tl.read_begin + tl.n_reads - 1];
        end = (FGB_READ_OFF(last) + FGB_READ_LEN(last) + 15u) & ~15ull;
      } else {
        end = tl.byte_begin + tl.byte_len;
      }
      end = std::max(end, byte1);
      if (!one_piece && t1 > t0 && end - byte0 > chunk_bytes) break;
      byte1 = end;
      ++t1;
    }
    const fgb_tile& first = T[t0];
    const fgb_tile& last = T[t1 - 1];
    const uint64_t u0 = first.unit_begin, u1 = static_cast<uint64_t>(last.unit_begin) + last.n_units;
    const uint64_t r0 = first.read_begin & ~1ull;
    const uint64_t r1 = static_cast<uint64_t>(last.read_begin) + last.n_reads;
    const uint64_t o0 = in->units[u0].out_off, o1 = in->units[u1].out_off;
    const uint64_t nbytes = byte1 - byte0;
    const uint64_t valid_bytes = std::min(byte1, in->n_bytes) - std::min(byte0, in->n_bytes);

    Slot& sl = h->slots[chunk % h->n_slots];
    // In-stream order makes slot reuse safe: chunk c+kSlots queues behind chunk c's D2H.
    fgb_status st;
    uint64_t cap2 = sl.cap_bytes;
    if ((st = ensure(h, &sl.bases, &sl.cap_bytes, nbytes + 16)) != FGB_OK) return st;
    if ((st = ensure(h, &sl.quals, &cap2, nbytes + 16)) != FGB_OK) return st;
    if ((st = ensure(h, &sl.reads, &sl.cap_reads, r1 - r0 + 2)) != FGB_OK) return st;
    if ((st = ensure(h, &sl.units, &sl.cap_units, u1 - u0 + 1)) != FGB_OK) return st;
    if ((st = ensure(h, &sl.tiles, &sl.cap_tiles, t1 - t0)) != FGB_OK) return st;
    uint64_t c1 = sl.cap_out, c2 = sl.cap_out, c3 = sl.cap_out;
    if ((st = ensure(h, &sl.out_base, &sl.cap_out, o1 - o0 + 4)) != FGB_OK) return st;
    if ((st = ensure(h, &sl.out_qual, &c1, o1 - o0 + 4)) != FGB_OK) return st;
    if ((st = ensure(h, &sl.out_depth, &c2, o1 - o0 + 4)) != FGB_OK) return st;
    if ((st = ensure(h, &sl.out_errors, &c3, o1 - o0 + 4)) != FGB_OK) return st;

    cudaStream_t s = sl.stream;
    mark(s, "chunk begins");
    if (rjobs && chunk == 0) {
      // K5's own inputs (string blob, per-unit jobs) travel FIRST: queued behind a chunk's record blob they would
      // hold the assembly of chunk c until the upload of chunk c+1 had passed through the copy engine
      if ((st = ensure(h, &h->d_recstr, &h->cap_recstr, opt->n_rec_string_bytes + 16)) != FGB_OK) return st;
      if ((st = ensure(h, &h->d_recjobs, &h->cap_recjobs, in->n_units + 1)) != FGB_OK) return st;
      FGB_CUDA(h, cudaMemcpyAsync(h->d_recstr, opt->rec_strings, opt->n_rec_string_bytes, cudaMemcpyHostToDevice, s));
      FGB_CUDA(h, cudaMemcpyAsync(h->d_recjobs, rjobs, in->n_units * sizeof(fgb_record_job), cudaMemcpyHostToDevice, s));
      if (!h->ev_recstr) FGB_CUDA(h, cudaEventCreateWithFlags(&h->ev_recstr, cudaEventDisableTiming));
      FGB_CUDA(h, cudaEventRecord(h->ev_recstr, s));
    }
    if (fmt == HostFormat::kPack8) {
      if ((st = ensure(h, &sl.packed, &sl.cap_packed, nbytes + 16)) != FGB_OK) return st;
      FGB_CUDA(h, cudaMemcpyAsync(sl.packed, in->bases + byte0, valid_bytes, cudaMemcpyHostToDevice, s));
      const uint64_t n16 = (valid_bytes + 15u) >> 4;   // byte0 is 16-aligned; slack bytes are in the buffers
      if (n16) {
        const unsigned grid = static_cast<unsigned>(std::min<uint64_t>((n16 + 255u) / 256u,
                                                                       static_cast<uint64_t>(h->sm_count) * 16u));
        unpack8_kernel<<<grid, 256, 0, s>>>(reinterpret_cast<const uint4*>(sl.packed),
                                            reinterpret_cast<uint4*>(sl.bases),
                                            reinterpret_cast<uint4*>(sl.quals), n16);
        h->launches++;
        FGB_CUDA(h, cudaGetLastError());
      }
    } else if (fmt == HostFormat::kBam4) {
      // raw span of this chunk's reads (ascending by construction), origin aligned down to 32 bases
      const uint64_t rf = first.read_begin, rl = r1;           // absolute read range [rf, rl)
      if (rl > rf) {
        const uint64_t a0 = raw->raw_reads[rf].src_off & ~31ull;
        const uint64_t a1 = raw->raw_reads[rl - 1].src_off + raw->raw_reads[rl - 1].raw_len;
        if (a1 < a0 || a1 > raw->n_raw) {
          h->last_error = "fgb_raw_columns: raw spans must ascend with the reads and stay inside the columns";
          return FGB_ERR_LAYOUT;
        }
        const uint64_t nraw = a1 - a0;
        if ((st = ensure(h, &sl.seq4, &sl.cap_seq4, nraw / 2 + 16)) != FGB_OK) return st;
        if ((st = ensure(h, &sl.qraw, &sl.cap_qraw, nraw + 16)) != FGB_OK) return st;
        if ((st = ensure(h, &sl.rawreads, &sl.cap_rawreads, rl - rf + 1)) != FGB_OK) return st;
        FGB_CUDA(h, cudaMemcpyAsync(sl.seq4, raw->seq4 + a0 / 2, (nraw + 1) / 2, cudaMemcpyHostToDevice, s));
        FGB_CUDA(h, cudaMemcpyAsync(sl.qraw, raw->quals_raw + a0, nraw, cudaMemcpyHostToDevice, s));
        FGB_CUDA(h, cudaMemcpyAsync(sl.rawreads, raw->raw_reads + rf, (rl - rf) * sizeof(fgb_raw_read),
                                    cudaMemcpyHostToDevice, s));
      }
      // (the layout descriptors are uploaded below; the unpack launch follows them)
    } else if (fmt == HostFormat::kRecords) {
      // (the record blob of this chunk's reads is uploaded below, once the read range is known)
    } else {
      FGB_CUDA(h, cudaMemcpyAsync(sl.bases, in->bases + byte0, valid_bytes, cudaMemcpyHostToDevice, s));
      FGB_CUDA(h, cudaMemcpyAsync(sl.quals, in->quals + byte0, valid_bytes, cudaMemcpyHostToDevice, s));
    }
    FGB_CUDA(h, cudaMemcpyAsync(sl.reads, in->reads + r0, (r1 - r0) * 8, cudaMemcpyHostToDevice, s));
    FGB_CUDA(h, cudaMemcpyAsync(sl.units, in->units + u0, (u1 - u0 + 1) * sizeof(fgb_unit),
                                cudaMemcpyHostToDevice, s));
    // the chunk's tiles, sorted by class (the kernels do not care about tile order); the copy below is from
    // pageable memory, which the runtime stages before cudaMemcpyAsync returns, so the vector can be reused
    uint64_t chunk_classes[3] = {t1 - t0, 0, 0};
    const fgb_tile* tsrc = T + t0;
    {
      bool mixed = false;
      for (uint64_t t = t0; t < t1 && !mixed; ++t) mixed = (T[t].flags & kTileClassMask) != 0;
      if (mixed) {
        sl.tile_stage.assign(T + t0, T + t1);
        fgb_sort_tiles_by_class(sl.tile_stage.data(), t1 - t0, chunk_classes);
        tsrc = sl.tile_stage.data();
      }
    }
    FGB_CUDA(h, cudaMemcpyAsync(sl.tiles, tsrc, (t1 - t0) * sizeof(fgb_tile),
                                cudaMemcpyHostToDevice, s));
    // Descriptors keep their absolute offsets; the kernel gets base pointers biased by the chunk
    // origin (byte0 / r0 / u0 / o0 keep every TMA source 16-byte aligned).
    fgb_batch db;
    std::memset(&db, 0, sizeof(db));
    db.n_tiles = t1 - t0;
    db.bases = sl.bases - byte0;
    db.quals = sl.quals - byte0;
    db.reads = sl.reads - r0;
    db.units = sl.units - u0;
    db.tiles = sl.tiles;
    db.class_tiles[0] = chunk_classes[0]; db.class_tiles[1] = chunk_classes[1]; db.class_tiles[2] = chunk_classes[2];
    fgb_columns dc;
    dc.base = sl.out_base - o0;
    dc.qual = sl.out_qual - o0;
    dc.depth = sl.out_depth - o0;
    dc.errors = sl.out_errors - o0;
    if (fmt == HostFormat::kBam4 && r1 > first.read_begin) {
      const uint64_t rf = first.read_begin;
      const uint64_t a0 = raw->raw_reads[rf].src_off & ~31ull;
      Bam4Args ua;
      ua.seq4 = sl.seq4 - a0 / 2;
      ua.quals_raw = sl.qraw - a0;
      ua.raw_reads = sl.rawreads - rf;
      ua.reads = db.reads;
      ua.bases = const_cast<uint8_t*>(db.bases);
      ua.quals = const_cast<uint8_t*>(db.quals);
      ua.read_begin = rf; ua.read_end = r1;
      ua.raw_lo = a0;
      ua.raw_hi = raw->raw_reads[r1 - 1].src_off + raw->raw_reads[r1 - 1].raw_len;
      ua.min_q = raw->min_input_base_quality;
      if ((st = launch_unpack_bam4(h, ua, s, true)) != FGB_OK) return st;
    }
    if (fmt == HostFormat::kRecords && r1 > first.read_begin) {
      // blob byte range this chunk's reads touch (a group's records are contiguous, its reads are not in
      // record order), padded for the kernel's aligned window loads
      const uint64_t rf = first.read_begin;
      uint64_t lo = ~0ull, hi = 0;
      for (uint64_t r = rf; r < r1; ++r) {
        const fgb_raw_read& rr = rec->raw_reads[r];
        const uint64_t e = rr.src_off + ((static_cast<uint64_t>(rr.raw_len) + 1u) >> 1) + rr.raw_len;
        lo = std::min(lo, rr.src_off);
        hi = std::max(hi, e);
      }
      for (uint64_t k = 0; k < n_oruns; ++k) {   // runs may touch records that yield no row: those stay resident too
        const fgb_overlap_run& o = opt->overlap_runs[k];
        lo = std::min(lo, std::min(o.seq1_off, o.seq2_off));
        hi = std::max(hi, std::max(o.seq1_off + ((static_cast<uint64_t>(o.l_seq1) + 1u) >> 1) + o.l_seq1,
                                   o.seq2_off + ((static_cast<uint64_t>(o.l_seq2) + 1u) >> 1) + o.l_seq2));
      }
      if (hi > rec->n_bytes || lo > hi) {
        h->last_error = "fgb_record_columns: a sequence / quality span runs past the record blob";
        return FGB_ERR_LAYOUT;
      }
      const uint64_t a0 = (lo > 64u ? lo - 64u : 0u) & ~63ull;
      const uint64_t a1 = std::min(rec->n_bytes, hi + 32u);
      if ((st = ensure(h, &sl.recblob, &sl.cap_recblob, a1 - a0 + 128)) != FGB_OK) return st;
      if ((st = ensure(h, &sl.rawreads, &sl.cap_rawreads, r1 - rf + 1)) != FGB_OK) return st;
      FGB_CUDA(h, cudaMemcpyAsync(sl.recblob, rec->records + a0, a1 - a0, cudaMemcpyHostToDevice, s));
      FGB_CUDA(h, cudaMemcpyAsync(sl.rawreads, rec->raw_reads + rf, (r1 - rf) * sizeof(fgb_raw_read),
                                  cudaMemcpyHostToDevice, s));
      RecordsArgs ua;
      ua.records = sl.recblob - a0;
      ua.raw_reads = sl.rawreads - rf;
      ua.reads = db.reads;
      ua.bases = const_cast<uint8_t*>(db.bases);
      ua.quals = const_cast<uint8_t*>(db.quals);
      ua.read_begin = rf; ua.read_end = r1;
      ua.rec_lo = a0;                            // resident bytes [a0, a1) plus allocation slack behind them;
      ua.rec_hi = a1 + 96u;                      // the kernel wants 16 bytes either side of every span (lo - a0 >= 16:
      ua.min_q = rec->min_input_base_quality;    // a sequence field starts >= 33 bytes into its record)
      if (n_oruns) {
        if (!h->d_ostats) {
          FGB_CUDA(h, cudaMalloc(&h->d_ostats, 4 * sizeof(unsigned long long)));
          FGB_CUDA(h, cudaMemset(h->d_ostats, 0, 4 * sizeof(unsigned long long)));
        }
        if (!h->d_bad) {
          FGB_CUDA(h, cudaMalloc(&h->d_bad, sizeof(uint32_t)));
          FGB_CUDA(h, cudaMemset(h->d_bad, 0, sizeof(uint32_t)));
        }
        if ((st = ensure(h, &h->d_oruns, &h->cap_oruns, n_oruns)) != FGB_OK) return st;
        FGB_CUDA(h, cudaMemcpyAsync(h->d_oruns, opt->overlap_runs, n_oruns * sizeof(fgb_overlap_run), cudaMemcpyHostToDevice, s));
        OverlapArgs oa;
        oa.records = sl.recblob - a0; oa.runs = h->d_oruns; oa.n_runs = n_oruns;
        oa.rec_lo = a0; oa.rec_hi = a1;
        oa.stats = h->d_ostats; oa.bad = h->d_bad;
        oa.agree = opt->overlap_agreement; oa.disagree = opt->overlap_disagreement;
        h->bam4_pending = true;
        h->ostats_host = opt->overlap_stats;
        const unsigned ogrid = static_cast<unsigned>(std::min<uint64_t>((n_oruns + 255u) / 256u, static_cast<uint64_t>(h->sm_count) * 8u));
        overlap_kernel<<<ogrid, 256, 0, s>>>(oa);
        h->launches++;
        FGB_CUDA(h, cudaGetLastError());
      }
      mark(s, "inputs resident");
      if ((st = launch_unpack_records(h, ua, s)) != FGB_OK) return st;
    }
    mark(s, "rows ready");
    if ((st = launch_vote(h, db, dc, s)) != FGB_OK) return st;
    mark(s, "voted");
    if (n_djobs) {
      const fgb_duplex_out* ho = opt->duplex_out;
      const uint64_t nd = opt->n_duplex_out;
      uint64_t c1 = sl.cap_cout, c2 = sl.cap_cout;
      if ((st = ensure(h, &sl.djobs, &sl.cap_djobs, n_djobs)) != FGB_OK) return st;
      if ((st = ensure(h, &sl.c_base, &sl.cap_cout, nd + 16)) != FGB_OK) return st;
      if ((st = ensure(h, &sl.c_qual, &c1, nd + 16)) != FGB_OK) return st;
      if ((st = ensure(h, &sl.c_errors, &c2, nd + 16)) != FGB_OK) return st;
      if ((st = ensure(h, &sl.c_status, &sl.cap_cjobout, n_djobs + 16)) != FGB_OK) return st;
      FGB_CUDA(h, cudaMemcpyAsync(sl.djobs, opt->duplex_jobs, n_djobs * sizeof(fgb_duplex_job), cudaMemcpyHostToDevice, s));
      fgb_batch jb = db;                       // absolute unit indices: same biased pointers as the vote
      fgb_duplex_out dout{sl.c_base, sl.c_qual, sl.c_errors, sl.c_status};
      if ((st = fgb_duplex_combine_device(h, &jb, &dc, sl.djobs, n_djobs, &dout, s)) != FGB_OK) return st;
      FGB_CUDA(h, cudaMemcpyAsync(ho->base, sl.c_base, nd, cudaMemcpyDeviceToHost, s));
      FGB_CUDA(h, cudaMemcpyAsync(ho->qual, sl.c_qual, nd, cudaMemcpyDeviceToHost, s));
      FGB_CUDA(h, cudaMemcpyAsync(ho->errors, sl.c_errors, nd * 2, cudaMemcpyDeviceToHost, s));
      if (ho->status) FGB_CUDA(h, cudaMemcpyAsync(ho->status, sl.c_status, n_djobs, cudaMemcpyDeviceToHost, s));
    }
    if (n_cjobs) {
      const fgb_codec_out* ho = opt->codec_out;
      const uint64_t nc = opt->n_codec_out;
      uint64_t c1 = sl.cap_cout, c2 = sl.cap_cout, c3 = sl.cap_cout;
      if ((st = ensure(h, &sl.cjobs, &sl.cap_cjobs, n_cjobs)) != FGB_OK) return st;
      if ((st = ensure(h, &sl.c_base, &sl.cap_cout, nc + 16)) != FGB_OK) return st;
      if ((st = ensure(h, &sl.c_qual, &c1, nc + 16)) != FGB_OK) return st;
      if ((st = ensure(h, &sl.c_depth, &c2, nc + 16)) != FGB_OK) return st;
      if ((st = ensure(h, &sl.c_errors, &c3, nc + 16)) != FGB_OK) return st;
      uint64_t cj1 = sl.cap_cjobout, cj2 = sl.cap_cjobout;
      if ((st = ensure(h, &sl.c_status, &sl.cap_cjobout, n_cjobs + 16)) != FGB_OK) return st;
      if ((st = ensure(h, &sl.c_dis, &cj1, n_cjobs + 16)) != FGB_OK) return st;
      if ((st = ensure(h, &sl.c_dup, &cj2, n_cjobs + 16)) != FGB_OK) return st;
      FGB_CUDA(h, cudaMemcpyAsync(sl.cjobs, opt->codec_jobs, n_cjobs * sizeof(fgb_codec_job), cudaMemcpyHostToDevice, s));
      fgb_batch jb = db;
      fgb_codec_out cout{};
      cout.cols = fgb_columns{sl.c_base, sl.c_qual, sl.c_depth, sl.c_errors};
      cout.status = sl.c_status; cout.disagreements = sl.c_dis; cout.duplex_bases = sl.c_dup;
      if ((st = fgb_codec_combine_device(h, &jb, &dc, sl.cjobs, n_cjobs, opt->codec_params, &cout, s)) != FGB_OK) return st;
      FGB_CUDA(h, cudaMemcpyAsync(ho->cols.base, sl.c_base, nc, cudaMemcpyDeviceToHost, s));
      FGB_CUDA(h, cudaMemcpyAsync(ho->cols.qual, sl.c_qual, nc, cudaMemcpyDeviceToHost, s));
      FGB_CUDA(h, cudaMemcpyAsync(ho->cols.depth, sl.c_depth, nc * 2, cudaMemcpyDeviceToHost, s));
      FGB_CUDA(h, cudaMemcpyAsync(ho->cols.errors, sl.c_errors, nc * 2, cudaMemcpyDeviceToHost, s));
      FGB_CUDA(h, cudaMemcpyAsync(ho->status, sl.c_status, n_cjobs, cudaMemcpyDeviceToHost, s));
      if (ho->disagreements) FGB_CUDA(h, cudaMemcpyAsync(ho->disagreements, sl.c_dis, n_cjobs * 4, cudaMemcpyDeviceToHost, s));
      if (ho->duplex_bases) FGB_CUDA(h, cudaMemcpyAsync(ho->duplex_bases, sl.c_dup, n_cjobs * 4, cudaMemcpyDeviceToHost, s));
    }
    if (rjobs) {
      // K5: the finished records of this chunk's units, straight into the host's output stream
      if (chunk != 0) FGB_CUDA(h, cudaStreamWaitEvent(s, h->ev_recstr, 0));   // later chunks run on other streams
      const uint64_t b_lo = rjobs[u0].out_off;
      const uint64_t b_hi = u1 < in->n_units ? rjobs[u1].out_off : opt->n_rec_out_bytes;
      if (b_hi < b_lo || b_hi > opt->n_rec_out_bytes) { h->last_error = "record jobs: offsets must ascend"; return FGB_ERR_LAYOUT; }
      if ((st = ensure(h, &sl.recout, &sl.cap_recout, b_hi - b_lo + 16)) != FGB_OK) return st;
      AssembleArgs aa;
      aa.units = db.units; aa.jobs = h->d_recjobs;
      aa.unit_begin = u0; aa.unit_end = u1;
      aa.base = dc.base; aa.qual = dc.qual; aa.depth = dc.depth; aa.errors = dc.errors;
      aa.strings = h->d_recstr; aa.prefix_len = opt->rec_prefix_len; aa.rg_len = opt->rec_rg_len;
      aa.cell_tag[0] = opt->rec_cell_tag[0]; aa.cell_tag[1] = opt->rec_cell_tag[1];
      aa.per_base_tags = opt->rec_per_base_tags; aa.pad = 0;
      aa.out = sl.recout - b_lo;
      const uint64_t nu = u1 - u0;
      const unsigned agrid = static_cast<unsigned>(std::min<uint64_t>((nu + 7u) / 8u, static_cast<uint64_t>(h->sm_count) * 16u));
      assemble_simplex_kernel<<<agrid, 256, 0, s>>>(aa);
      h->launches++;
      FGB_CUDA(h, cudaGetLastError());
      mark(s, "records assembled");
      if (b_hi > b_lo) FGB_CUDA(h, cudaMemcpyAsync(opt->rec_out + b_lo, sl.recout, b_hi - b_lo, cudaMemcpyDeviceToHost, s));
    }
    if (fp) {
      if ((st = ensure(h, &sl.unit_status, &sl.cap_ustat, u1 - u0 + 16)) != FGB_OK) return st;
      if (opt->unit_masked && (st = ensure(h, &sl.unit_masked, &sl.cap_umask, u1 - u0 + 16)) != FGB_OK) return st;
      if ((st = launch_filter(h, db.units, u0, u1, dc, *fp, sl.unit_status,
                              opt->unit_masked ? sl.unit_masked : nullptr, s)) != FGB_OK) return st;
      FGB_CUDA(h, cudaMemcpyAsync(opt->unit_status + u0, sl.unit_status, u1 - u0, cudaMemcpyDeviceToHost, s));
      if (opt->unit_masked)
        FGB_CUDA(h, cudaMemcpyAsync(opt->unit_masked + u0, sl.unit_masked, (u1 - u0) * 4,
                                    cudaMemcpyDeviceToHost, s));
    }
    const uint64_t no = o1 - o0;
    if (!out->base) {                        // record assembly only: nothing else travels back
      mark(s, "results home");
      t0 = t1;
      ++chunk;
      continue;
    }
    FGB_CUDA(h, cudaMemcpyAsync(out->base + o0, sl.out_base, no, cudaMemcpyDeviceToHost, s));
    FGB_CUDA(h, cudaMemcpyAsync(out->qual + o0, sl.out_qual, no, cudaMemcpyDeviceToHost, s));
    if (narrow) {
      uint64_t c8 = sl.cap_out8;
      if ((st = ensure(h, &sl.out_depth8, &sl.cap_out8, no + 16)) != FGB_OK) return st;
      if ((st = ensure(h, &sl.out_errors8, &c8, no + 16)) != FGB_OK) return st;
      const uint64_t n8 = (no + 7u) >> 3;   // output rows are padded to 8 elements
      const unsigned grid = static_cast<unsigned>(std::min<uint64_t>((n8 + 255u) / 256u,
                                                                     static_cast<uint64_t>(h->sm_count) * 16u));
      narrow_u16_kernel<<<grid, 256, 0, s>>>(reinterpret_cast<const uint4*>(sl.out_depth),
                                             reinterpret_cast<const uint4*>(sl.out_errors),
                                             reinterpret_cast<uint2*>(sl.out_depth8),
                                             reinterpret_cast<uint2*>(sl.out_errors8), n8);
      h->launches++;
      FGB_CUDA(h, cudaGetLastError());
      FGB_CUDA(h, cudaMemcpyAsync(reinterpret_cast<uint8_t*>(out->depth) + o0, sl.out_depth8, no,
                                  cudaMemcpyDeviceToHost, s));
      FGB_CUDA(h, cudaMemcpyAsync(reinterpret_cast<uint8_t*>(out->errors) + o0, sl.out_errors8, no,
                                  cudaMemcpyDeviceToHost, s));
    } else {
      FGB_CUDA(h, cudaMemcpyAsync(out->depth + o0, sl.out_depth, no * 2, cudaMemcpyDeviceToHost, s));
      FGB_CUDA(h, cudaMemcpyAsync(out->errors + o0, sl.out_errors, no * 2, cudaMemcpyDeviceToHost, s));
    }
    mark(s, "results home");
    t0 = t1;
    ++chunk;
  }
  if (h->trace) h->trace_t1 = std::chrono::steady_clock::now();
  guard.ok = true;
  return FGB_OK;
}
}  // namespace

extern "C" {

fgb_status fgb_submit(fgb_handle* h, const fgb_batch* in, const fgb_columns* out) {
  return submit_impl(h, in, out, HostFormat::kBytes);
}

fgb_status fgb_submit_pack8(fgb_handle* h, const fgb_batch* in, const fgb_columns* out) {
  return submit_impl(h, in, out, HostFormat::kPack8);
}

fgb_status fgb_submit_bam4(fgb_handle* h, const fgb_batch* in, const fgb_raw_columns* raw,
                           const fgb_columns* out) {
  return submit_impl(h, in, out, HostFormat::kBam4, raw);
}

fgb_status fgb_submit_ex(fgb_handle* h, const fgb_batch* in, const fgb_columns* out,
                         const fgb_submit_options* opt) {
  if (!opt || opt->input_format > FGB_IN_RECORDS || opt->output_format > FGB_OUT_U8) return FGB_ERR_INVALID_ARG;
  const HostFormat f = opt->input_format == FGB_IN_PACK8 ? HostFormat::kPack8
                       : opt->input_format == FGB_IN_BAM4 ? HostFormat::kBam4
                       : opt->input_format == FGB_IN_RECORDS ? HostFormat::kRecords : HostFormat::kBytes;
  return submit_impl(h, in, out, f, opt->raw, opt->output_format == FGB_OUT_U8, opt);
}

fgb_status fgb_filter_simplex_device(fgb_handle* h, const fgb_batch* in, const fgb_columns* cols,
                                     const fgb_filter_params* fp, uint8_t* unit_status,
                                     uint32_t* unit_masked, void* stream) {
  if (!h || !in || !cols || !unit_status || !filter_params_ok(fp)) return FGB_ERR_INVALID_ARG;
  if (in->n_units == 0) return FGB_OK;
  if (!in->units || !cols->base || !cols->qual || !cols->depth || !cols->errors) return FGB_ERR_INVALID_ARG;
  FGB_CUDA(h, cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  fgb_status st = ensure_emax(h, fp->max_base_error_rate, s);
  if (st != FGB_OK) return st;
  return launch_filter(h, in->units, 0, in->n_units, *cols, *fp, unit_status, unit_masked, s);
}

fgb_status fgb_unpack_bam4_device(fgb_handle* h, const fgb_batch* in, const fgb_raw_columns* raw,
                                  uint8_t* bases, uint8_t* quals, void* stream) {
  if (!h || !in || !raw || !bases || !quals || !in->reads || !raw->seq4 || !raw->quals_raw ||
      !raw->raw_reads)
    return FGB_ERR_INVALID_ARG;
  FGB_CUDA(h, cudaSetDevice(h->device));
  Bam4Args ua;
  ua.seq4 = raw->seq4; ua.quals_raw = raw->quals_raw; ua.raw_reads = raw->raw_reads;
  ua.reads = in->reads; ua.bases = bases; ua.quals = quals;
  ua.read_begin = 0; ua.read_end = in->n_reads;
  ua.raw_lo = 0; ua.raw_hi = raw->n_raw;
  ua.min_q = raw->min_input_base_quality;
  return launch_unpack_bam4(h, ua, static_cast<cudaStream_t>(stream),
                            ((raw->n_raw + 1u) / 2u) % 4u == 0 && raw->n_raw % 4u == 0);
}

fgb_status fgb_unpack_records_device(fgb_handle* h, const fgb_batch* in, const fgb_record_columns* rec,
                                     uint8_t* bases, uint8_t* quals, void* stream) {
  if (!h || !in || !rec || !bases || !quals || !in->reads || !rec->records || !rec->raw_reads)
    return FGB_ERR_INVALID_ARG;
  FGB_CUDA(h, cudaSetDevice(h->device));
  RecordsArgs ua;
  ua.records = rec->records; ua.raw_reads = rec->raw_reads;
  ua.reads = in->reads; ua.bases = bases; ua.quals = quals;
  ua.read_begin = 0; ua.read_end = in->n_reads;
  ua.rec_lo = 0; ua.rec_hi = rec->n_bytes;          // the caller pads the device blob by 16 bytes at the end
  ua.min_q = rec->min_input_base_quality;
  return launch_unpack_records(h, ua, static_cast<cudaStream_t>(stream));
}

fgb_status fgb_pack8_encode(const uint8_t* bases, const uint8_t* quals, uint64_t n, uint8_t* out) {
  if (n && (!bases || !quals || !out)) return FGB_ERR_INVALID_ARG;
  static const uint8_t kCode[256] = {   // 0..3 = A,C,G,T; 4 = N; 5 = padding (0); 255 = not encodable
#define X 255
      5, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X,
      X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X,
      X, 0, X, 1, X, X, X, 2, X, X, X, X, X, X, 4, X, X, X, X, X, 3, X, X, X, X, X, X, X, X, X, X, X,
      X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X,
      X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X,
      X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X,
      X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X,
      X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X, X
#undef X
  };
  uint32_t bad = 0;
  for (uint64_t i = 0; i < n; ++i) {
    const uint32_t c = kCode[bases[i]], q = quals[i];
    uint32_t v;
    if (c < 4u) { v = (c << 6) | q; bad |= q > 61u; }
    else if (c == 4u) { v = 0x3Eu; bad |= q != 2u; }
    else if (c == 5u) { v = 0u; bad |= q != 0u; }
    else { v = 0u; bad = 1u; }
    out[i] = static_cast<uint8_t>(v);
  }
  return bad ? FGB_ERR_NOT_ENCODABLE : FGB_OK;
}

fgb_status fgb_wait(fgb_handle* h) {
  if (!h) return FGB_ERR_INVALID_ARG;
  h->submit_pending = false;
  FGB_CUDA(h, cudaSetDevice(h->device));
  for (int s = 0; s < kSlots; ++s) FGB_CUDA(h, cudaStreamSynchronize(h->slots[s].stream));
  if (h->trace && !h->trace_ev.empty()) {     // FGB_SUBMIT_TRACE=1: where the device time of the last submit went
    const double host_ms = std::chrono::duration<double, std::milli>(h->trace_t1 - h->trace_t0).count();
    const double wait_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - h->trace_t1).count();
    std::fprintf(stderr, "fgb submit trace: host side of the submit call %.2f ms, then %.2f ms until the streams drained\n", host_ms, wait_ms);
    for (auto& m : h->trace_ev) {
      float ms = 0.f;
      cudaEventElapsedTime(&ms, h->trace_ev.front().ev, m.ev);
      std::fprintf(stderr, "  chunk %d  %-18s +%8.3f ms\n", m.chunk, m.what, ms);
      }
    for (auto& m : h->trace_ev) cudaEventDestroy(m.ev);
    h->trace_ev.clear();
  }
  if (h->ostats_host) {                // overlap pre-pass counters of the submit that just finished
    unsigned long long v[4] = {0, 0, 0, 0};
    FGB_CUDA(h, cudaMemcpy(v, h->d_ostats, sizeof(v), cudaMemcpyDeviceToHost));
    FGB_CUDA(h, cudaMemset(h->d_ostats, 0, sizeof(v)));
    for (int i = 0; i < 4; ++i) h->ostats_host[i] += v[i];
    h->ostats_host = nullptr;
  }
  if (h->bam4_pending) {               // the unpack kernel validates the raw spans where it reads them
    h->bam4_pending = false;
    uint32_t bad = 0;
    FGB_CUDA(h, cudaMemcpy(&bad, h->d_bad, sizeof(bad), cudaMemcpyDeviceToHost));
    if (bad) {
      FGB_CUDA(h, cudaMemset(h->d_bad, 0, sizeof(uint32_t)));
      h->last_error = "fgb_raw_columns: a raw span is odd-aligned, runs past the columns or is shorter than its row";
      return FGB_ERR_LAYOUT;
    }
  }
  return FGB_OK;
}

// ---- strand combine -----------------------------------------------------------------------------
fgb_status fgb_duplex_combine_device(fgb_handle* h, const fgb_batch* in, const fgb_columns* ss,
                                     const fgb_duplex_job* jobs, uint64_t n_jobs,
                                     const fgb_duplex_out* out, void* stream) {
  if (!h || !in || !ss || !out || (n_jobs && !jobs)) return FGB_ERR_INVALID_ARG;
  if (n_jobs == 0) return FGB_OK;
  FGB_CUDA(h, cudaSetDevice(h->device));
  DuplexArgs a;
  a.bases = in->bases; a.reads = in->reads; a.units = in->units;
  a.ss_base = ss->base; a.ss_qual = ss->qual; a.ss_depth = ss->depth; a.ss_errors = ss->errors;
  a.jobs = jobs; a.n_jobs = n_jobs;
  a.out_base = out->base; a.out_qual = out->qual; a.out_errors = out->errors;
  a.out_status = out->status;
  a.counters = h->d_counters;
  // the word kernel moves 8 elements at a time: byte columns 8-byte aligned, u16 columns 16-byte aligned
  const uintptr_t align8 = reinterpret_cast<uintptr_t>(a.bases) | reinterpret_cast<uintptr_t>(a.ss_base) |
                           reinterpret_cast<uintptr_t>(a.ss_qual) | reinterpret_cast<uintptr_t>(a.out_base) |
                           reinterpret_cast<uintptr_t>(a.out_qual);
  const uintptr_t align16 = reinterpret_cast<uintptr_t>(a.ss_depth) | reinterpret_cast<uintptr_t>(a.out_errors);
  const uint64_t chunks = (n_jobs + kDuplexChunk - 1) / kDuplexChunk;
  if ((align8 & 7u) == 0 && (align16 & 15u) == 0 && chunks <= 0x7FFFFFFFull) {
    // word kernel: 8 positions per thread, a CTA per chunk of consecutive jobs
    duplex_combine_words_kernel<<<static_cast<unsigned>(chunks), kCombineThreads, 0, static_cast<cudaStream_t>(stream)>>>(a);
  } else {
    unsigned grid = static_cast<unsigned>(std::min<uint64_t>((n_jobs + kCombineJobsPerCta - 1) / kCombineJobsPerCta,
                                                             static_cast<uint64_t>(h->sm_count) * 8u));
    duplex_combine_kernel<<<grid, kCombineThreads, 0, static_cast<cudaStream_t>(stream)>>>(a);
  }
  h->launches++;
  FGB_CUDA(h, cudaGetLastError());
  return FGB_OK;
}

fgb_status fgb_vote_duplex_device(fgb_handle* h, const fgb_batch* in, const fgb_columns* ss,
                                  const fgb_duplex_job* jobs, uint64_t n_jobs,
                                  const fgb_tile_jobs* tile_jobs, const uint32_t* job_index,
                                  const fgb_duplex_out* out, void* stream) {
  if (!h || !in || !ss || !out || (n_jobs && !jobs)) return FGB_ERR_INVALID_ARG;
  if (in->n_tiles && (!in->tiles || !in->units || !ss->base || !ss->qual || !ss->depth || !ss->errors))
    return FGB_ERR_INVALID_ARG;
  fgb_status vst = check_vote_pointers(h, *in, *ss, "fgb_vote_duplex_device");
  if (vst != FGB_OK) return vst;
  FGB_CUDA(h, cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // the epilogue moves 8 elements at a time: byte columns 8-byte aligned, u16 columns and job records 16-byte aligned
  // (the batch and the SS columns passed check_vote_pointers; what is left are the pointers only the epilogue uses)
  const uintptr_t align8 = reinterpret_cast<uintptr_t>(out->base) | reinterpret_cast<uintptr_t>(out->qual) |
                           reinterpret_cast<uintptr_t>(tile_jobs);
  const uintptr_t align16 = reinterpret_cast<uintptr_t>(out->errors) | reinterpret_cast<uintptr_t>(jobs);
  const bool fused = n_jobs && in->n_tiles && tile_jobs && job_index && (align8 & 7u) == 0 && (align16 & 15u) == 0;
  if (!fused) {
    fgb_status st = launch_vote(h, *in, *ss, s);
    if (st != FGB_OK || n_jobs == 0) return st;
    return fgb_duplex_combine_device(h, in, ss, jobs, n_jobs, out, stream);
  }
  DuplexEpilogueArgs dx{tile_jobs, job_index, jobs, *out};
  if (!dx.out.status) {
    fgb_status st = ensure(h, &h->d_dstatus, &h->cap_dstatus, n_jobs);
    if (st != FGB_OK) return st;
    dx.out.status = h->d_dstatus;
  }
  FGB_CUDA(h, cudaMemsetAsync(dx.out.status, FGB_DUPLEX_PENDING, n_jobs, s));
  fgb_status st = launch_vote(h, *in, *ss, s, &dx);
  if (st != FGB_OK) return st;
  // what the epilogue left pending: single-strand arms, jobs whose units sit in different tiles, general layouts
  DuplexArgs a;
  a.bases = in->bases; a.reads = in->reads; a.units = in->units;
  a.ss_base = ss->base; a.ss_qual = ss->qual; a.ss_depth = ss->depth; a.ss_errors = ss->errors;
  a.jobs = jobs; a.n_jobs = n_jobs;
  a.out_base = out->base; a.out_qual = out->qual; a.out_errors = out->errors;
  a.out_status = dx.out.status;
  a.counters = h->d_counters;
  const uint64_t groups = (n_jobs + kCombineThreads - 1) / kCombineThreads;
  const unsigned grid = static_cast<unsigned>(std::min<uint64_t>(groups, static_cast<uint64_t>(h->sm_count) * 8u));
  duplex_combine_pending_kernel<<<grid, kCombineThreads, 0, s>>>(a);
  h->launches++;
  FGB_CUDA(h, cudaGetLastError());
  return FGB_OK;
}

// ---- K0z: BGZF members inflated on the device -----------------------------------------------------------
fgb_status fgb_bgzf_inflate_device(fgb_handle* h, const uint8_t* data, const fgb_bgzf_member* members,
                                   uint64_t n_members, uint8_t* out, uint8_t* status, int check_crc,
                                   unsigned long long* n_bad, void* stream) {
  if (!h || (n_members && (!data || !members || !status))) return FGB_ERR_INVALID_ARG;
  if (n_members == 0) return FGB_OK;
  FGB_CUDA(h, cudaSetDevice(h->device));
  InflateArgs a;
  a.in = data; a.members = members; a.n_members = n_members; a.out = out; a.status = status;
  a.check_crc = check_crc ? 1u : 0u; a.n_bad = n_bad;
  const uint64_t blocks = (n_members + kInflateWarps - 1) / kInflateWarps;
  const unsigned grid = static_cast<unsigned>(std::min<uint64_t>(blocks, static_cast<uint64_t>(h->sm_count) * 16u));   // 64 decoders per SM
  bgzf_inflate_kernel<<<grid, kInflateThreads, 0, static_cast<cudaStream_t>(stream)>>>(a);
  h->launches++;
  FGB_CUDA(h, cudaGetLastError());
  return FGB_OK;
}

fgb_status fgb_codec_combine_device(fgb_handle* h, const fgb_batch* in, const fgb_columns* ss,
                                    const fgb_codec_job* jobs, uint64_t n_jobs,
                                    const fgb_codec_params* cp, const fgb_codec_out* out,
                                    void* stream) {
  if (!h || !in || !ss || !out || !cp || (n_jobs && !jobs)) return FGB_ERR_INVALID_ARG;
  if (n_jobs == 0) return FGB_OK;
  if (!out->status || !out->cols.base || !out->cols.qual || !out->cols.depth || !out->cols.errors)
    return FGB_ERR_INVALID_ARG;
  FGB_CUDA(h, cudaSetDevice(h->device));
  CodecArgs a;
  a.units = in->units;
  a.ss_base = ss->base; a.ss_qual = ss->qual; a.ss_depth = ss->depth; a.ss_errors = ss->errors;
  a.jobs = jobs; a.n_jobs = n_jobs;
  a.cp = *cp;
  a.out_base = out->cols.base; a.out_qual = out->cols.qual; a.out_depth = out->cols.depth;
  a.out_errors = out->cols.errors;
  a.status = out->status; a.disagreements = out->disagreements; a.duplex_bases = out->duplex_bases;
  a.counters = h->d_counters;
  const uintptr_t align8 = reinterpret_cast<uintptr_t>(a.ss_base) | reinterpret_cast<uintptr_t>(a.ss_qual) |
                           reinterpret_cast<uintptr_t>(a.out_base) | reinterpret_cast<uintptr_t>(a.out_qual);
  const uintptr_t align16 = reinterpret_cast<uintptr_t>(a.ss_depth) | reinterpret_cast<uintptr_t>(a.ss_errors) |
                            reinterpret_cast<uintptr_t>(a.out_depth) | reinterpret_cast<uintptr_t>(a.out_errors);
  const uint64_t chunks = (n_jobs + kCodecChunk - 1) / kCodecChunk;
  if ((align8 & 7u) == 0 && (align16 & 15u) == 0 && chunks <= 0x7FFFFFFFull) {
    // word kernel: 8 output positions per thread, a CTA per chunk of consecutive jobs
    codec_combine_words_kernel<<<static_cast<unsigned>(chunks), kCombineThreads, 0, static_cast<cudaStream_t>(stream)>>>(a);
  } else {
    unsigned grid = static_cast<unsigned>(std::min<uint64_t>((n_jobs + kCodecJobsPerCta - 1) / kCodecJobsPerCta,
                                                             static_cast<uint64_t>(h->sm_count) * 8u));
    codec_combine_kernel<<<grid, kCombineThreads, 0, static_cast<cudaStream_t>(stream)>>>(a);
  }
  h->launches++;
  FGB_CUDA(h, cudaGetLastError());
  return FGB_OK;
}

// ---- statistics ---------------------------------------------------------------------------------
fgb_status fgb_stats(fgb_handle* h, uint64_t counters[FGB_NCOUNTERS]) {
  if (!h || !counters) return FGB_ERR_INVALID_ARG;
  FGB_CUDA(h, cudaSetDevice(h->device));
  FGB_CUDA(h, cudaDeviceSynchronize());
  FGB_CUDA(h, cudaMemcpy(counters, h->d_counters, sizeof(uint64_t) * FGB_NCOUNTERS,
                         cudaMemcpyDeviceToHost));
  return FGB_OK;
}

fgb_status fgb_stats_device_ptr(fgb_handle* h, uint64_t** dev_counters) {
  if (!h || !dev_counters) return FGB_ERR_INVALID_ARG;
  *dev_counters = reinterpret_cast<uint64_t*>(h->d_counters);
  return FGB_OK;
}

fgb_status fgb_stats_reset(fgb_handle* h) {
  if (!h) return FGB_ERR_INVALID_ARG;
  FGB_CUDA(h, cudaSetDevice(h->device));
  FGB_CUDA(h, cudaDeviceSynchronize());
  FGB_CUDA(h, cudaMemset(h->d_counters, 0, sizeof(unsigned long long) * FGB_NCOUNTERS));
  return FGB_OK;
}

uint64_t fgb_launch_count(const fgb_handle* h) { return h ? h->launches : 0; }
uint32_t fgb_engine_caps(void) { return FGB_CAP_RECORD_ASSEMBLY; }

}  // extern "C"

// ---- UMI assignment (umi_kernels.cuh, host/umi_host.cpp) ----------------------------------------------------------
namespace {

template <class T>
fgb_status ensure_pinned(fgb_handle* h, T** p, uint64_t* cap, uint64_t need) {
  if (need <= *cap && *p) return FGB_OK;
  if (*p) { cudaFreeHost(*p); *p = nullptr; *cap = 0; }
  const uint64_t n = need + need / 8 + 64;
  cudaError_t e = cudaHostAlloc(reinterpret_cast<void**>(p), n * sizeof(T), cudaHostAllocDefault);
  if (e != cudaSuccess) { cuda_fail(h, e, "cudaHostAlloc"); return FGB_ERR_NOMEM; }
  *cap = n;
  return FGB_OK;
}

// Smallest call (unique keys) that takes the enumeration form instead of all-pairs, by k.  Set from the device time
// of the two forms' edge kernels (CUDA events, scripts/bench_umi_assign.py --crossover; DESIGN.md section 9).
// FGB_UMI_ENUM_MIN_KEYS overrides both for that measurement.
uint64_t umi_enum_min_keys(uint32_t k) {
  if (const char* e = std::getenv("FGB_UMI_ENUM_MIN_KEYS")) return std::strtoull(e, nullptr, 10);
  return k <= 1 ? 1000 : 8000;
}

#define FGB_TRY(x) do { fgb_status s__ = (x); if (s__ != FGB_OK) return s__; } while (0)

// Host phase 1 of fgb_umi_assign / fgb_umi_edges: key tables of every call (umi_off is indexed by call_off).
fgb_status umi_prepare_calls(fgb_handle* h, const fgb_umi_options& o, const uint8_t* umis, const uint64_t* umi_off,
                             const uint64_t* call_off, uint64_t n_calls, std::vector<fgb_umi::Call>* calls) {
  calls->assign(n_calls, fgb_umi::Call{});
  std::vector<std::string> err(n_calls);
  fgb_umi::parallel_for(n_calls, o.n_threads, [&](uint64_t c) {
    try {
      err[c] = fgb_umi::prepare(o, umis, umi_off + call_off[c], call_off[c + 1] - call_off[c], &(*calls)[c]);
    } catch (const std::bad_alloc&) {
      err[c] = "out of host memory";
    }
  });
  for (uint64_t c = 0; c < n_calls; ++c)
    if (!err[c].empty()) {
      h->last_error = "fgb_umi_assign: call " + std::to_string(c) + ": " + err[c];
      return err[c] == "out of host memory" ? FGB_ERR_NOMEM : FGB_ERR_INVALID_ARG;
    }
  return FGB_OK;
}

// The device phase: capture lists of every call that can have an edge.  row_base[c] = the call's first CSR row
// (UINT64_MAX: no device work); the CSR is left in h->umi.h_off (rows + 1 entries) / h->umi.h_edges.
fgb_status umi_device_edges(fgb_handle* h, const fgb_umi_options& o, const std::vector<fgb_umi::Call>& calls,
                            std::vector<uint64_t>* row_base_out, float* device_ms) {
  const uint64_t n_calls = calls.size();
  const bool bytes = fgb_umi::uses_bytes(o);
  fgb::UmiCmp cmp{};
  cmp.k = o.edits;
  cmp.directed = o.strategy != FGB_UMI_EDIT;
  cmp.bytes = bytes;
  cmp.reverse = bytes && o.strategy == FGB_UMI_PAIRED;
  cmp.zero_ok = o.edits != 1;
  std::vector<uint64_t>& row_base = *row_base_out;
  row_base.assign(n_calls, UINT64_MAX);
  std::vector<uint64_t> enum_calls;
  std::vector<uint8_t> is_enum(n_calls, 0);
  uint64_t n_rows = 0, n_blob = 0, n_work = 0, n_sorted = 0, max_sorted = 0;
  for (uint64_t c = 0; c < n_calls; ++c) {
    if (!fgb_umi::needs_edges(o, calls[c])) continue;
    const uint64_t nk = calls[c].keys.size();
    if (nk > UINT32_MAX) { h->last_error = "fgb_umi_assign: call " + std::to_string(c) + ": too many unique UMIs"; return FGB_ERR_INVALID_ARG; }
    row_base[c] = n_rows;
    n_rows += nk;
    if (bytes) n_blob += calls[c].bytes.size();
    if (!bytes && o.edits <= 2 && nk >= umi_enum_min_keys(o.edits)) {
      enum_calls.push_back(c);
      is_enum[c] = 1;
      n_sorted += nk;
      max_sorted = std::max(max_sorted, nk);
    } else {
      n_work += (nk + fgb::kUmiThreads - 1) / fgb::kUmiThreads;
    }
  }
  if (device_ms) *device_ms = 0.f;
  if (!n_rows) return FGB_OK;
  auto& B = h->umi;
  std::vector<uint64_t> sorted_base(n_calls, 0);
  FGB_CUDA(h, cudaSetDevice(h->device));
  cudaStream_t st = h->slots[0].stream;
  FGB_TRY(ensure_pinned(h, &B.h_keys, &B.hcap_keys, n_rows));
  FGB_TRY(ensure_pinned(h, &B.h_blob, &B.hcap_blob, n_blob + 1));
  FGB_TRY(ensure_pinned(h, &B.h_work, &B.hcap_work, n_work + 1));
  FGB_TRY(ensure_pinned(h, &B.h_sbits, &B.hcap_sbits, n_sorted + 1));
  FGB_TRY(ensure_pinned(h, &B.h_sidx, &B.hcap_sidx, n_sorted + 1));
  FGB_TRY(ensure(h, &B.keys, &B.cap_keys, n_rows));
  FGB_TRY(ensure(h, &B.blob, &B.cap_blob, n_blob + 1));
  FGB_TRY(ensure(h, &B.work, &B.cap_work, n_work + 1));
  FGB_TRY(ensure(h, &B.deg, &B.cap_deg, n_rows + 1));
  FGB_TRY(ensure(h, &B.off, &B.cap_off, n_rows + 1));
  FGB_TRY(ensure(h, &B.sbits_in, &B.cap_sbits_in, n_sorted + 1));
  FGB_TRY(ensure(h, &B.sbits, &B.cap_sbits, n_sorted + 1));
  FGB_TRY(ensure(h, &B.sidx_in, &B.cap_sidx_in, n_sorted + 1));
  FGB_TRY(ensure(h, &B.sidx, &B.cap_sidx, n_sorted + 1));
  if (!B.ev0) {
    FGB_CUDA(h, cudaEventCreate(&B.ev0));
    FGB_CUDA(h, cudaEventCreate(&B.ev1));
    FGB_CUDA(h, cudaEventCreate(&B.ev2));
    FGB_CUDA(h, cudaEventCreate(&B.ev3));
  }
  // stage the tables (string offsets rebased onto the batch's blob) and the all-pairs work list
  uint64_t w = 0, blob_at = 0, s_at = 0;
  for (uint64_t c = 0; c < n_calls; ++c) {
    if (row_base[c] == UINT64_MAX) continue;
    const auto& cl = calls[c];
    const uint64_t nk = cl.keys.size();
    fgb_umi_key* dst = B.h_keys + row_base[c];
    std::memcpy(dst, cl.keys.data(), nk * sizeof(fgb_umi_key));
    if (bytes) {
      for (uint64_t k = 0; k < nk; ++k) dst[k].str_off += blob_at;
      std::memcpy(B.h_blob + blob_at, cl.bytes.data(), cl.bytes.size());
      blob_at += cl.bytes.size();
    }
    if (is_enum[c]) {
      sorted_base[c] = s_at;
      for (uint64_t k = 0; k < nk; ++k) { B.h_sbits[s_at + k] = cl.keys[k].bits; B.h_sidx[s_at + k] = static_cast<uint32_t>(k); }
      s_at += nk;
    } else {
      for (uint64_t q = 0; q < nk; q += fgb::kUmiThreads)
        B.h_work[w++] = fgb::UmiWork{row_base[c], static_cast<uint32_t>(nk), static_cast<uint32_t>(q)};
    }
  }
  FGB_CUDA(h, cudaMemcpyAsync(B.keys, B.h_keys, n_rows * sizeof(fgb_umi_key), cudaMemcpyHostToDevice, st));
  if (n_blob) FGB_CUDA(h, cudaMemcpyAsync(B.blob, B.h_blob, n_blob, cudaMemcpyHostToDevice, st));
  if (n_work) FGB_CUDA(h, cudaMemcpyAsync(B.work, B.h_work, n_work * sizeof(fgb::UmiWork), cudaMemcpyHostToDevice, st));
  if (n_sorted) {
    FGB_CUDA(h, cudaMemcpyAsync(B.sbits_in, B.h_sbits, n_sorted * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
    FGB_CUDA(h, cudaMemcpyAsync(B.sidx_in, B.h_sidx, n_sorted * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
  }
  size_t temp_sort = 0, temp_scan = 0;
  if (max_sorted)
    FGB_CUDA(h, cub::DeviceRadixSort::SortPairs(nullptr, temp_sort, B.sbits_in, B.sbits, B.sidx_in, B.sidx,
                                                static_cast<int>(max_sorted), 0, 64, st));
  FGB_CUDA(h, cub::DeviceScan::ExclusiveSum(nullptr, temp_scan, B.deg, B.off, static_cast<int>(n_rows + 1), st));
  FGB_TRY(ensure(h, &B.temp, &B.cap_temp, std::max(temp_sort, temp_scan) + 16));
  // count pass (events bracket the device work: sort, count, scan | fill)
  FGB_CUDA(h, cudaEventRecord(B.ev0, st));
  FGB_CUDA(h, cudaMemsetAsync(B.deg + n_rows, 0, sizeof(uint64_t), st));
  if (n_work) {
    fgb::umi_pairs_kernel<false><<<static_cast<unsigned>(n_work), fgb::kUmiThreads, 0, st>>>(
        B.work, B.keys, B.blob, cmp, B.deg, B.off, B.edges);
    h->launches++;
  }
  for (uint64_t c : enum_calls) {
    const uint64_t nk = calls[c].keys.size(), sb = sorted_base[c];
    size_t tb = B.cap_temp;
    FGB_CUDA(h, cub::DeviceRadixSort::SortPairs(B.temp, tb, B.sbits_in + sb, B.sbits + sb, B.sidx_in + sb, B.sidx + sb,
                                                static_cast<int>(nk), 0, 64, st));
    fgb::umi_enum_kernel<false><<<static_cast<unsigned>((nk + fgb::kUmiThreads - 1) / fgb::kUmiThreads), fgb::kUmiThreads, 0, st>>>(
        B.keys + row_base[c], static_cast<uint32_t>(nk), B.sbits + sb, B.sidx + sb, cmp, B.deg + row_base[c], nullptr, nullptr);
    h->launches += 2;
  }
  FGB_CUDA(h, cudaGetLastError());
  {
    size_t tb = B.cap_temp;
    FGB_CUDA(h, cub::DeviceScan::ExclusiveSum(B.temp, tb, B.deg, B.off, static_cast<int>(n_rows + 1), st));
  }
  FGB_CUDA(h, cudaEventRecord(B.ev1, st));
  FGB_TRY(ensure_pinned(h, &B.h_off, &B.hcap_off, n_rows + 1));
  FGB_CUDA(h, cudaMemcpyAsync(B.h_off, B.off, (n_rows + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  FGB_CUDA(h, cudaStreamSynchronize(st));
  const uint64_t n_edges = B.h_off[n_rows];
  FGB_TRY(ensure(h, &B.edges, &B.cap_edges, n_edges + 1));
  FGB_TRY(ensure_pinned(h, &B.h_edges, &B.hcap_edges, n_edges + 1));
  // fill pass
  FGB_CUDA(h, cudaEventRecord(B.ev2, st));
  if (n_work) {
    fgb::umi_pairs_kernel<true><<<static_cast<unsigned>(n_work), fgb::kUmiThreads, 0, st>>>(
        B.work, B.keys, B.blob, cmp, B.deg, B.off, B.edges);
    h->launches++;
  }
  for (uint64_t c : enum_calls) {
    const uint64_t nk = calls[c].keys.size(), sb = sorted_base[c];
    fgb::umi_enum_kernel<true><<<static_cast<unsigned>((nk + fgb::kUmiThreads - 1) / fgb::kUmiThreads), fgb::kUmiThreads, 0, st>>>(
        B.keys + row_base[c], static_cast<uint32_t>(nk), B.sbits + sb, B.sidx + sb, cmp, nullptr, B.off + row_base[c], B.edges);
    h->launches++;
  }
  FGB_CUDA(h, cudaGetLastError());
  FGB_CUDA(h, cudaEventRecord(B.ev3, st));
  if (n_edges) FGB_CUDA(h, cudaMemcpyAsync(B.h_edges, B.edges, n_edges * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  FGB_CUDA(h, cudaStreamSynchronize(st));
  if (device_ms) {
    float a = 0.f, b = 0.f;
    FGB_CUDA(h, cudaEventElapsedTime(&a, B.ev0, B.ev1));
    FGB_CUDA(h, cudaEventElapsedTime(&b, B.ev2, B.ev3));
    *device_ms = a + b;
  }
  return FGB_OK;
}

fgb_status umi_check_layout(fgb_handle* h, const uint64_t* umi_off, uint64_t n_umis, const uint64_t* call_off,
                            uint64_t n_calls, const uint64_t* group_off, uint64_t n_groups) {
  auto layout = [&](const char* what) { h->last_error = std::string("fgb_umi_assign: ") + what; return FGB_ERR_INVALID_ARG; };
  if (group_off[0] != 0 || group_off[n_groups] != n_calls) return layout("group_off must run from 0 to n_calls");
  if (call_off[0] != 0 || call_off[n_calls] != n_umis) return layout("call_off must run from 0 to n_umis");
  for (uint64_t g = 0; g < n_groups; ++g) if (group_off[g + 1] < group_off[g]) return layout("group_off descends");
  for (uint64_t c = 0; c < n_calls; ++c) if (call_off[c + 1] < call_off[c]) return layout("call_off descends");
  for (uint64_t u = 0; u < n_umis; ++u) if (umi_off[u + 1] < umi_off[u]) return layout("umi_off descends");
  return FGB_OK;
}

fgb_status umi_assign_impl(fgb_handle* h, const fgb_umi_options& o, const uint8_t* umis, const uint64_t* umi_off,
                           uint64_t n_umis, const uint64_t* call_off, uint64_t n_calls, const uint64_t* group_off,
                           uint64_t n_groups, uint64_t* ids, uint8_t* kinds, uint64_t* group_mi_count) {
  FGB_TRY(umi_check_layout(h, umi_off, n_umis, call_off, n_calls, group_off, n_groups));
  // 1. unique / count / sort per call on the host threads
  std::vector<fgb_umi::Call> calls;
  const auto t0 = std::chrono::steady_clock::now();
  FGB_TRY(umi_prepare_calls(h, o, umis, umi_off, call_off, n_calls, &calls));
  const auto t1 = std::chrono::steady_clock::now();
  // 2. the device: capture lists of every call that can have an edge
  std::vector<uint64_t> row_base;
  float dev_ms = 0.f;
  FGB_TRY(umi_device_edges(h, o, calls, &row_base, &dev_ms));
  const auto t2 = std::chrono::steady_clock::now();
  auto& B = h->umi;
  // 3. the order-dependent rules per call, in parallel across calls
  fgb_umi::parallel_for(n_calls, o.n_threads, [&](uint64_t c) {
    const bool dev = row_base[c] != UINT64_MAX;
    fgb_umi::resolve(o, calls[c], dev ? B.h_off + row_base[c] : nullptr, dev ? B.h_edges : nullptr,
                     ids + call_off[c], kinds + call_off[c]);
  });
  // 4. numbering across a group's calls: mapped assigners keep one counter, unmapped ones restart at 0
  for (uint64_t g = 0; g < n_groups; ++g) {
    uint64_t base = 0, count = 0;
    for (uint64_t c = group_off[g]; c < group_off[g + 1]; ++c) {
      uint64_t taken = 0;
      for (uint64_t u = call_off[c]; u < call_off[c + 1]; ++u) {
        if (kinds[u] == FGB_MOL_NONE) continue;
        taken = std::max(taken, ids[u] + 1);
        if (o.rules == FGB_UMI_RULES_MAPPED) ids[u] += base;
        count = std::max(count, ids[u] + 1);
      }
      if (o.rules == FGB_UMI_RULES_MAPPED) base += taken;
    }
    group_mi_count[g] = count;
  }
  const auto t3 = std::chrono::steady_clock::now();
  auto ms = [](auto a, auto b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
  B.timing[0] = ms(t0, t1);
  B.timing[1] = ms(t1, t2);
  B.timing[2] = dev_ms;
  B.timing[3] = ms(t2, t3);
  return FGB_OK;
}

}  // namespace

extern "C" {

fgb_status fgb_umi_assign(fgb_handle* h, const fgb_umi_options* opt, const uint8_t* umis, const uint64_t* umi_off,
                          uint64_t n_umis, const uint64_t* call_off, uint64_t n_calls, const uint64_t* group_off,
                          uint64_t n_groups, uint64_t* ids, uint8_t* kinds, uint64_t* group_mi_count) {
  if (!h || !opt || !umi_off || !call_off || !group_off || (n_umis && (!umis || !ids || !kinds)) ||
      (n_groups && !group_mi_count))
    return FGB_ERR_INVALID_ARG;
  const std::string bad = fgb_umi::check_options(*opt);
  if (!bad.empty()) { h->last_error = "fgb_umi_assign: " + bad; return FGB_ERR_INVALID_ARG; }
  if (h->submit_pending) { h->last_error = "fgb_umi_assign: a submit has not been waited on"; return FGB_ERR_BUSY; }
  return fgb::link::guarded(&h->last_error, "fgb_umi_assign", [&] {
    return umi_assign_impl(h, *opt, umis, umi_off, n_umis, call_off, n_calls, group_off, n_groups, ids, kinds,
                           group_mi_count);
  });
}

fgb_status fgb_umi_last_timing(const fgb_handle* h, double ms[4]) {
  if (!h || !ms) return FGB_ERR_INVALID_ARG;
  std::memcpy(ms, h->umi.timing, sizeof(h->umi.timing));
  return FGB_OK;
}

fgb_status fgb_umi_edges(fgb_handle* h, const fgb_umi_options* opt, const uint8_t* umis, const uint64_t* umi_off,
                         uint64_t n_umis, uint64_t* n_keys, uint64_t* edge_off, uint32_t* edges, uint64_t cap,
                         uint64_t* n_edges) {
  if (!h || !opt || !umi_off || !n_keys || !edge_off || !n_edges || (n_umis && !umis)) return FGB_ERR_INVALID_ARG;
  const std::string bad = fgb_umi::check_options(*opt);
  if (!bad.empty()) { h->last_error = "fgb_umi_edges: " + bad; return FGB_ERR_INVALID_ARG; }
  if (h->submit_pending) { h->last_error = "fgb_umi_edges: a submit has not been waited on"; return FGB_ERR_BUSY; }
  // reports as "fgb_umi_assign: ..." like the assignment whose edge phase this is
  return fgb::link::guarded(&h->last_error, "fgb_umi_assign", [&]() -> fgb_status {
    const uint64_t call_off[2] = {0, n_umis}, group_off[2] = {0, 1};
    FGB_TRY(umi_check_layout(h, umi_off, n_umis, call_off, 1, group_off, 1));
    std::vector<fgb_umi::Call> calls;
    FGB_TRY(umi_prepare_calls(h, *opt, umis, umi_off, call_off, 1, &calls));
    std::vector<uint64_t> row_base;
    FGB_TRY(umi_device_edges(h, *opt, calls, &row_base, nullptr));
    const uint64_t nk = calls[0].keys.size();
    *n_keys = nk;
    if (row_base[0] == UINT64_MAX) {   // nothing for the device: no edges
      std::fill(edge_off, edge_off + nk + 1, 0);
      *n_edges = 0;
      return FGB_OK;
    }
    const uint64_t* o = h->umi.h_off + row_base[0];
    for (uint64_t k = 0; k <= nk; ++k) edge_off[k] = o[k] - o[0];
    *n_edges = o[nk] - o[0];
    if (edges && cap >= *n_edges && *n_edges) std::memcpy(edges, h->umi.h_edges + o[0], *n_edges * sizeof(uint32_t));
    return FGB_OK;
  });
}

}  // extern "C"

// ---- the record commands' view of the handle (host/record_link.h) ------------------------------------------------
fgb::link::HandleInfo fgb::link::info(fgb_handle* h, Command c) {
  if (c == Command::kZipper)
    return HandleInfo{h->device, h->sm_count, h->slots[0].stream, h->submit_pending, &h->last_error,
                      h->zipper_timing, &h->zipper_out, nullptr};
  const bool filter = c == Command::kFilter;
  return HandleInfo{h->device, h->sm_count, h->slots[0].stream, h->submit_pending, &h->last_error,
                    filter ? h->filter_timing : h->sort_timing, filter ? &h->filter_kept : nullptr,
                    filter ? &h->filter_rejects : nullptr};
}

// ---- record sort (sort_kernels.cuh; the driver is host/sort_host.cpp) --------------------------------------------
namespace fgb {
namespace sortdev {

namespace {
unsigned blocks(uint32_t n) { return (n + kSortThreads - 1) / kSortThreads; }
}  // namespace

cudaError_t keys(const uint8_t* rec, const uint64_t* off, uint64_t base, uint32_t n, const sortk::Ctx& ctx, int words,
                 uint64_t* keys, uint32_t* size, unsigned long long* and_or, cudaStream_t s) {
  if (!n) return cudaSuccess;
  if (words == 1) sort_key_kernel<1><<<blocks(n), kSortThreads, 0, s>>>(rec, off, base, n, ctx, keys, size, and_or);
  else sort_key_kernel<sortk::kWords><<<blocks(n), kSortThreads, 0, s>>>(rec, off, base, n, ctx, keys, size, and_or);
  return cudaGetLastError();
}

cudaError_t name_keys(const uint8_t* rec, const uint64_t* off, uint64_t base, uint32_t n, bool natural, int name_words,
                      uint64_t* keys, uint32_t* size, unsigned long long* and_or, cudaStream_t s) {
  if (!n) return cudaSuccess;
  sort_name_key_kernel<<<blocks(n), kSortThreads, 0, s>>>(rec, off, base, n, natural, name_words, keys, size, and_or);
  return cudaGetLastError();
}

cudaError_t word_gather(const uint64_t* word, const uint32_t* perm, uint32_t n, uint64_t* dst, cudaStream_t s) {
  if (!n) return cudaSuccess;
  sort_word_gather_kernel<<<blocks(n), kSortThreads, 0, s>>>(word, perm, n, dst, nullptr);
  return cudaGetLastError();
}

cudaError_t iota(uint32_t* v, uint32_t n, cudaStream_t s) {
  if (!n) return cudaSuccess;
  sort_word_gather_kernel<<<blocks(n), kSortThreads, 0, s>>>(nullptr, nullptr, n, nullptr, v);
  return cudaGetLastError();
}

cudaError_t key_rows(const uint64_t* keys, const uint32_t* perm, uint32_t n, int words, uint64_t* rows, cudaStream_t s) {
  if (!n) return cudaSuccess;
  sort_key_rows_kernel<<<blocks(n), kSortThreads, 0, s>>>(keys, perm, n, words, rows);
  return cudaGetLastError();
}

cudaError_t radix_pass(void* temp, size_t* temp_bytes, const uint64_t* kin, uint64_t* kout, const uint32_t* vin,
                       uint32_t* vout, uint32_t n, int begin, int end, cudaStream_t s) {
  return cub::DeviceRadixSort::SortPairs(temp, *temp_bytes, kin, kout, vin, vout, static_cast<int>(n), begin, end, s);
}

cudaError_t out_offsets(void* temp, size_t* temp_bytes, const uint32_t* size, const uint32_t* perm, uint32_t n,
                        uint64_t* out_size, uint64_t* out_off, cudaStream_t s) {
  if (!temp) return cub::DeviceScan::ExclusiveSum(nullptr, *temp_bytes, out_size, out_off, static_cast<int>(n) + 1, s);
  if (n) sort_out_size_kernel<<<blocks(n), kSortThreads, 0, s>>>(size, perm, n, out_size);
  cudaError_t e = cudaMemsetAsync(out_size + n, 0, sizeof(uint64_t), s);
  if (e != cudaSuccess) return e;
  return cub::DeviceScan::ExclusiveSum(temp, *temp_bytes, out_size, out_off, static_cast<int>(n) + 1, s);
}

cudaError_t gather(const uint8_t* rec, const uint64_t* off, uint64_t base, const uint32_t* perm,
                   const uint64_t* out_off, uint32_t n, uint8_t* out, int sm_count, cudaStream_t s) {
  if (!n) return cudaSuccess;
  const uint64_t want = (static_cast<uint64_t>(n) * 32 + kSortThreads - 1) / kSortThreads;   // one warp per record
  const unsigned grid = static_cast<unsigned>(std::min<uint64_t>(want, static_cast<uint64_t>(sm_count) * 16));
  sort_gather_kernel<<<grid, kSortThreads, 0, s>>>(rec, off, base, perm, out_off, n, out);
  return cudaGetLastError();
}

}  // namespace sortdev
}  // namespace fgb

// ---- record filter (filter_records_kernels.cuh; the driver is host/filter_host.cpp) ---------------------------------
namespace fgb {
namespace filterdev {

namespace {
unsigned warp_grid(uint32_t n, int sm_count) {   // one warp per record, at most 16 CTAs per SM (grid-stride)
  const uint64_t want = (static_cast<uint64_t>(n) * 32 + kFilterThreads - 1) / kFilterThreads;
  return static_cast<unsigned>(std::max<uint64_t>(1, std::min<uint64_t>(want, static_cast<uint64_t>(sm_count) * 16)));
}
}  // namespace

cudaError_t pass1(uint8_t* rec, const uint64_t* off, uint64_t base, uint32_t n, const FilterCfg& cfg,
                  const int32_t* ctg_of_ref, const uint64_t* ctg_off, const uint64_t* ctg_len, const uint8_t* genome,
                  uint64_t first, FRec* out, unsigned long long* err, unsigned long long* counters, int sm_count,
                  cudaStream_t s) {
  if (!n) return cudaSuccess;
  filter_pass1_kernel<<<warp_grid(n, sm_count), kFilterThreads, 0, s>>>(rec, off, base, n, cfg, ctg_of_ref, ctg_off,
                                                                       ctg_len, genome, first, out, err, counters);
  return cudaGetLastError();
}

cudaError_t decide(FRec* fr, const uint32_t* order, const uint32_t* tpl, uint32_t n_tpl, bool by_template,
                   unsigned long long* counters, cudaStream_t s) {
  if (!n_tpl) return cudaSuccess;
  filter_decide_kernel<<<(n_tpl + kFilterThreads - 1) / kFilterThreads, kFilterThreads, 0, s>>>(fr, order, tpl, n_tpl,
                                                                                                 by_template, counters);
  return cudaGetLastError();
}

cudaError_t offsets(void* temp, size_t* temp_bytes, const FRec* fr, const uint32_t* order, uint32_t n,
                    bool track_rejects, uint64_t* ks, uint64_t* rs, uint64_t* koff, uint64_t* roff, cudaStream_t s) {
  if (!temp) return cub::DeviceScan::ExclusiveSum(nullptr, *temp_bytes, ks, koff, static_cast<int>(n) + 1, s);
  filter_sizes_kernel<<<(n + kFilterThreads) / kFilterThreads, kFilterThreads, 0, s>>>(fr, order, n, track_rejects, ks,
                                                                                      rs);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  size_t tb = *temp_bytes;
  if ((e = cub::DeviceScan::ExclusiveSum(temp, tb, ks, koff, static_cast<int>(n) + 1, s)) != cudaSuccess) return e;
  tb = *temp_bytes;
  return cub::DeviceScan::ExclusiveSum(temp, tb, rs, roff, static_cast<int>(n) + 1, s);
}

cudaError_t pass2(const uint8_t* rec, const uint64_t* off, uint64_t base, uint32_t n, const FRec* fr,
                  const uint32_t* order, const uint64_t* koff, const uint64_t* roff, bool track_rejects,
                  const uint8_t* genome, uint8_t* kept, uint8_t* rejects, int sm_count, cudaStream_t s) {
  if (!n) return cudaSuccess;
  filter_pass2_kernel<<<warp_grid(n, sm_count), kFilterThreads, 0, s>>>(rec, off, base, n, fr, order, koff, roff,
                                                                       track_rejects, genome, kept, rejects);
  return cudaGetLastError();
}

}  // namespace filterdev
}  // namespace fgb

// ---- template scores (dedup_kernels.cuh; the deduper is host/dedup_host.cpp) ----------------------------------------
namespace fgb {
namespace dedupdev {

namespace {

constexpr uint64_t kScoreStageBytes = 16ull << 20;   // one page-locked chunk of records (two alternate)

// The chunk buffers for `bytes` of records and `entries` offsets, grown (never shrunk) without touching last_error:
// a failure here is reported through the caller's string, since fgb_umi_assign may run on the handle meanwhile.
cudaError_t score_buffers(fgb_handle* h, uint64_t bytes, uint64_t entries, uint64_t n) {
  auto& c = h->score;
  cudaError_t e;
  if (!c.stream && (e = cudaStreamCreateWithFlags(&c.stream, cudaStreamNonBlocking)) != cudaSuccess) return e;
  for (int b = 0; b < 2; ++b)
    if (!c.staged[b] && (e = cudaEventCreateWithFlags(&c.staged[b], cudaEventDisableTiming)) != cudaSuccess) return e;
  if (bytes > c.cap_rec) {
    const uint64_t cap = bytes + bytes / 8 + 64;
    for (int b = 0; b < 2; ++b) {
      cudaFreeHost(c.h_rec[b]); cudaFree(c.d_rec[b]);
      c.h_rec[b] = nullptr; c.d_rec[b] = nullptr;
    }
    c.cap_rec = 0;
    for (int b = 0; b < 2; ++b)
      if ((e = cudaHostAlloc(reinterpret_cast<void**>(&c.h_rec[b]), cap, cudaHostAllocDefault)) != cudaSuccess ||
          (e = cudaMalloc(reinterpret_cast<void**>(&c.d_rec[b]), cap)) != cudaSuccess)
        return e;
    c.cap_rec = cap;
  }
  if (entries > c.cap_off) {
    const uint64_t cap = entries + entries / 8 + 64;
    for (int b = 0; b < 2; ++b) {
      cudaFreeHost(c.h_off[b]); cudaFree(c.d_off[b]);
      c.h_off[b] = nullptr; c.d_off[b] = nullptr;
    }
    c.cap_off = 0;
    for (int b = 0; b < 2; ++b)
      if ((e = cudaHostAlloc(reinterpret_cast<void**>(&c.h_off[b]), cap * 8, cudaHostAllocDefault)) != cudaSuccess ||
          (e = cudaMalloc(reinterpret_cast<void**>(&c.d_off[b]), cap * 8)) != cudaSuccess)
        return e;
    c.cap_off = cap;
  }
  if (n > c.cap_scores) {
    const uint64_t cap = n + n / 8 + 64;
    cudaFree(c.d_scores); cudaFreeHost(c.h_scores);
    c.d_scores = nullptr; c.h_scores = nullptr; c.cap_scores = 0;
    if ((e = cudaMalloc(reinterpret_cast<void**>(&c.d_scores), cap * 4)) != cudaSuccess ||
        (e = cudaHostAlloc(reinterpret_cast<void**>(&c.h_scores), cap * 4, cudaHostAllocDefault)) != cudaSuccess)
      return e;
    c.cap_scores = cap;
  }
  return cudaSuccess;
}

}  // namespace

fgb_status quality_scores(fgb_handle* h, uint64_t n, const uint8_t* const* rec, const uint64_t* len, uint32_t n_threads,
                          uint32_t* scores, float* kernel_ms, std::string* err) {
  *kernel_ms = 0.f;
  if (!n) return FGB_OK;
  auto fail = [&](cudaError_t e, const char* what) {
    *err = std::string("template scores: ") + what + ": " + cudaGetErrorString(e);
    return e == cudaErrorMemoryAllocation ? FGB_ERR_NOMEM : FGB_ERR_CUDA;
  };
  cudaError_t e = cudaSetDevice(h->device);
  if (e != cudaSuccess) return fail(e, "cudaSetDevice");
  // chunks: as many consecutive records as fit one staging buffer (at least one)
  std::vector<uint64_t> chunk{0};
  uint64_t max_bytes = 0, max_n = 0;
  for (uint64_t i = 0; i < n;) {
    uint64_t bytes = len[i], j = i + 1;
    while (j < n && bytes + len[j] <= kScoreStageBytes) bytes += len[j++];
    max_bytes = std::max(max_bytes, bytes);
    max_n = std::max(max_n, j - i);
    chunk.push_back(j);
    i = j;
  }
  const uint64_t n_chunks = chunk.size() - 1;
  if ((e = score_buffers(h, max_bytes + 16, max_n + 1, n)) != cudaSuccess) { cudaGetLastError(); return fail(e, "buffers"); }
  auto& c = h->score;
  while (c.ev.size() < 2 * n_chunks) {
    cudaEvent_t ev;
    if ((e = cudaEventCreate(&ev)) != cudaSuccess) return fail(e, "cudaEventCreate");
    c.ev.push_back(ev);
  }
  const unsigned max_grid = static_cast<unsigned>(std::max(h->sm_count, 1)) * 8;
  for (uint64_t k = 0; k < n_chunks; ++k) {
    const int b = static_cast<int>(k & 1);
    const uint64_t i0 = chunk[k], cnt = chunk[k + 1] - i0;
    if ((e = cudaEventSynchronize(c.staged[b])) != cudaSuccess) return fail(e, "cudaEventSynchronize");
    uint64_t* off = c.h_off[b];
    off[0] = 0;
    for (uint64_t x = 0; x < cnt; ++x) off[x + 1] = off[x] + len[i0 + x];
    const uint64_t t = std::min<uint64_t>(std::max<uint32_t>(n_threads, 1), std::max<uint64_t>(off[cnt] >> 22, 1));
    fgb_umi::parallel_for(t, n_threads, [&](uint64_t w) {
      for (uint64_t x = cnt * w / t, xe = cnt * (w + 1) / t; x < xe; ++x)
        std::memcpy(c.h_rec[b] + off[x], rec[i0 + x], len[i0 + x]);
    });
    if ((e = cudaMemcpyAsync(c.d_rec[b], c.h_rec[b], off[cnt], cudaMemcpyHostToDevice, c.stream)) != cudaSuccess ||
        (e = cudaMemcpyAsync(c.d_off[b], off, (cnt + 1) * 8, cudaMemcpyHostToDevice, c.stream)) != cudaSuccess ||
        (e = cudaEventRecord(c.staged[b], c.stream)) != cudaSuccess)
      return fail(e, "upload");
    const unsigned grid = static_cast<unsigned>(std::min<uint64_t>((cnt + kScoreThreads / 32 - 1) / (kScoreThreads / 32), max_grid));
    if ((e = cudaEventRecord(c.ev[2 * k], c.stream)) != cudaSuccess) return fail(e, "cudaEventRecord");
    dedup_score_kernel<<<grid, kScoreThreads, 0, c.stream>>>(c.d_rec[b], c.d_off[b], static_cast<uint32_t>(cnt),
                                                              c.d_scores + i0);
    if ((e = cudaGetLastError()) != cudaSuccess) return fail(e, "dedup_score_kernel");
    if ((e = cudaEventRecord(c.ev[2 * k + 1], c.stream)) != cudaSuccess) return fail(e, "cudaEventRecord");
  }
  if ((e = cudaMemcpyAsync(c.h_scores, c.d_scores, n * 4, cudaMemcpyDeviceToHost, c.stream)) != cudaSuccess ||
      (e = cudaStreamSynchronize(c.stream)) != cudaSuccess)
    return fail(e, "download");
  std::memcpy(scores, c.h_scores, n * 4);
  for (uint64_t k = 0; k < n_chunks; ++k) {
    float ms = 0.f;
    if ((e = cudaEventElapsedTime(&ms, c.ev[2 * k], c.ev[2 * k + 1])) != cudaSuccess) return fail(e, "cudaEventElapsedTime");
    *kernel_ms += ms;
  }
  return FGB_OK;
}

}  // namespace dedupdev
}  // namespace fgb

extern "C" {

fgb_status fgb_record_quality_scores(fgb_handle* h, const uint8_t* records, const uint64_t* rec_off,
                                     uint64_t n_records, uint32_t* scores) {
  if (!h || (n_records && (!records || !rec_off || !scores))) return FGB_ERR_INVALID_ARG;
  if (h->submit_pending) { h->last_error = "fgb_record_quality_scores: a submit has not been waited on"; return FGB_ERR_BUSY; }
  for (uint64_t i = 0; i < n_records; ++i)
    if (rec_off[i + 1] < rec_off[i] || rec_off[i + 1] - rec_off[i] < 32) {
      h->last_error = "fgb_record_quality_scores: record " + std::to_string(i) + " is shorter than 32 bytes";
      return FGB_ERR_LAYOUT;
    }
  return fgb::link::guarded(&h->last_error, "fgb_record_quality_scores", [&] {
    std::vector<const uint8_t*> rp(n_records);
    std::vector<uint64_t> rl(n_records);
    for (uint64_t i = 0; i < n_records; ++i) { rp[i] = records + rec_off[i]; rl[i] = rec_off[i + 1] - rec_off[i]; }
    float kernel_ms = 0.f;
    std::string err;
    const fgb_status st = fgb::dedupdev::quality_scores(h, n_records, rp.data(), rl.data(), 1, scores, &kernel_ms, &err);
    if (st != FGB_OK) h->last_error = "fgb_record_quality_scores: " + err;
    return st;
  });
}

}  // extern "C"
