// The host-device plumbing of the record commands' drivers (sort_host.cpp, filter_host.cpp, metrics_host.cpp): the handle as a driver
// sees it, the device budget, failure texts, and one call's resources -- its device buffers, the two page-locked
// staging buffers through which each run's bytes cross the link, and its timing events.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cstdint>
#include <cstring>
#include <new>
#include <string>
#include <string_view>
#include <vector>

#include "../../../include/fgumi_b200.h"
#include "umi_host.h"

struct fgb_handle;

namespace fgb {
namespace link {

constexpr uint64_t kStageBytes = 64ull << 20;   // the largest page-locked staging buffer (two alternate)

struct HandleInfo {
  int device;
  int sm_count;
  cudaStream_t stream;
  bool busy;                       // a submit has not been waited on
  std::string* last_error;
  double* timing;                  // the command's six *_last_timing phases
  std::vector<uint8_t>* kept;      // the filter's library-owned output streams (null for the sort)
  std::vector<uint8_t>* rejects;
};
enum class Command { kSort, kFilter, kZipper };   // kZipper: its output stream is `kept`, `rejects` is null
HandleInfo info(fgb_handle* h, Command c);   // defined in capi.cu, which owns the handle

inline double ms_since(std::chrono::steady_clock::time_point t) {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t).count();
}

// The @SQ SN names of the header, in order
inline std::vector<std::string> sq_names(std::string_view text) {
  std::vector<std::string> out;
  size_t p = 0;
  while (p < text.size()) {
    size_t e = text.find('\n', p);
    if (e == std::string_view::npos) e = text.size();
    const std::string_view ln = text.substr(p, e - p);
    if (ln.substr(0, 4) == "@SQ\t") {
      std::string sn;
      for (size_t q = 4; q <= ln.size();) {
        size_t t = ln.find('\t', q);
        if (t == std::string_view::npos) t = ln.size();
        if (ln.substr(q, 3) == "SN:") { sn = std::string(ln.substr(q + 3, t - q - 3)); break; }
        q = t + 1;
      }
      if (!sn.empty() && sn.back() == '\r') sn.pop_back();
      out.push_back(sn);
    }
    p = e + 1;
  }
  return out;
}

// memcpy on n_threads host threads (the staging copies are what bounds the upload and download)
inline void par_copy(uint8_t* dst, const uint8_t* src, uint64_t n, uint32_t n_threads) {
  const uint64_t t = std::min<uint64_t>(std::max<uint32_t>(n_threads, 1), std::max<uint64_t>(n >> 22, 1));
  fgb_umi::parallel_for(t, n_threads, [&](uint64_t w) {
    const uint64_t b = n * w / t, e = n * (w + 1) / t;
    if (e > b) std::memcpy(dst + b, src + b, e - b);
  });
}

// Device bytes a call may use: `requested` when non-zero, else the free memory less an eighth and less another
// eighth of at most 512 MiB.
inline cudaError_t device_budget(uint64_t requested, uint64_t* budget) {
  *budget = requested;
  if (requested) return cudaSuccess;
  size_t free_b = 0, total_b = 0;
  const cudaError_t e = cudaMemGetInfo(&free_b, &total_b);
  if (e == cudaSuccess) *budget = free_b - free_b / 8 - std::min<uint64_t>(free_b / 8, 512ull << 20);
  return e;
}

// A failed CUDA call `what` of entry point `who`: "<who>: <what>: <error>" in last_error, and the status to return.
inline fgb_status fail(std::string* last_error, const char* who, cudaError_t e, const char* what) {
  cudaGetLastError();   // a failed allocation must not surface in the handle's next launch check
  *last_error = std::string(who) + ": " + what + ": " + cudaGetErrorString(e);
  return e == cudaErrorMemoryAllocation ? FGB_ERR_NOMEM : FGB_ERR_CUDA;
}

// f() with an escaping exception turned into *last_error and FGB_ERR_NOMEM: no exception crosses the ABI or leaves a
// std::thread.
template <class F>
fgb_status guarded(std::string* last_error, const char* who, F&& f) {
  try {
    return f();
  } catch (const std::bad_alloc&) {
    *last_error = std::string(who) + ": out of host memory";
  } catch (const std::exception& x) {
    *last_error = std::string(who) + ": " + x.what();
  }
  return FGB_ERR_NOMEM;
}

// Everything one call allocates, freed on every way out.  upload and download move bytes on `stream` through two
// page-locked staging buffers used alternately: the host copy into (out of) one overlaps the transfer out of (into)
// the other, and the event staged_[b] marks the end of the last transfer of buffer b.
class Resources {
 public:
  cudaEvent_t ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};   // the driver's timing events

  Resources(cudaStream_t stream, uint32_t n_threads) : s_(stream), threads_(n_threads) {}
  Resources(const Resources&) = delete;
  Resources& operator=(const Resources&) = delete;
  ~Resources() {
    for (void* p : dev_) cudaFree(p);
    for (auto* s : stage_) if (s) cudaFreeHost(s);
    for (auto e : staged_) if (e) cudaEventDestroy(e);
    for (auto e : ev) if (e) cudaEventDestroy(e);
  }

  template <class T>
  cudaError_t alloc(T** p, uint64_t count) {
    void* q = nullptr;
    const cudaError_t e = cudaMalloc(&q, std::max<uint64_t>(count, 1) * sizeof(T));
    if (e == cudaSuccess) dev_.push_back(q);
    *p = static_cast<T*>(q);
    return e;
  }
  template <class T>
  cudaError_t grow(T** p, uint64_t* cap, uint64_t count) {   // a buffer of at least `count` elements
    if (count <= *cap) return cudaSuccess;
    if (*p) { dev_.erase(std::find(dev_.begin(), dev_.end(), static_cast<void*>(*p))); cudaFree(*p); *p = nullptr; }
    *cap = 0;
    const uint64_t want = count + count / 8 + 64;
    const cudaError_t e = alloc(p, want);
    if (e == cudaSuccess) *cap = want;
    return e;
  }

  // The staging buffers of stage_bytes each (also the transfers' chunk size), their events and the timing events;
  // on failure *what names the CUDA call that failed.
  cudaError_t open(uint64_t stage_bytes, const char** what) {
    stage_bytes_ = stage_bytes;
    cudaError_t e = cudaSuccess;
    *what = "cudaHostAlloc";
    for (int b = 0; b < 2 && e == cudaSuccess; ++b)
      e = cudaHostAlloc(reinterpret_cast<void**>(&stage_[b]), stage_bytes, cudaHostAllocDefault);
    if (e != cudaSuccess) return e;
    *what = "cudaEventCreate";
    for (int b = 0; b < 2 && e == cudaSuccess; ++b) e = cudaEventCreateWithFlags(&staged_[b], cudaEventDisableTiming);
    for (int i = 0; i < 5 && e == cudaSuccess; ++i) e = cudaEventCreate(&ev[i]);
    return e;
  }

  // host -> device; returns once the last chunk is queued (the caller synchronises the stream)
  cudaError_t upload(void* dst_v, const void* src_v, uint64_t n) {
    uint8_t* dst = static_cast<uint8_t*>(dst_v);
    const uint8_t* src = static_cast<const uint8_t*>(src_v);
    for (uint64_t at = 0, k = 0; at < n; at += stage_bytes_, ++k) {
      const int b = static_cast<int>(k & 1);
      const uint64_t len = std::min(stage_bytes_, n - at);
      cudaError_t e = cudaEventSynchronize(staged_[b]);
      if (e != cudaSuccess) return e;
      par_copy(stage_[b], src + at, len, threads_);
      if ((e = cudaMemcpyAsync(dst + at, stage_[b], len, cudaMemcpyHostToDevice, s_)) != cudaSuccess) return e;
      if ((e = cudaEventRecord(staged_[b], s_)) != cudaSuccess) return e;
    }
    return cudaSuccess;
  }

  // device -> host; returns with every byte in dst
  cudaError_t download(void* dst_v, const void* src_v, uint64_t n) {
    uint8_t* dst = static_cast<uint8_t*>(dst_v);
    const uint8_t* src = static_cast<const uint8_t*>(src_v);
    uint64_t prev_at = 0, prev_len = 0;
    int prev = -1;
    for (uint64_t at = 0, k = 0; at < n; at += stage_bytes_, ++k) {
      const int b = static_cast<int>(k & 1);
      const uint64_t len = std::min(stage_bytes_, n - at);
      // stage_[b] needs no wait: its copy-out of chunk k - 2, or of a preceding download, ended on this thread, and
      // the transfer out of it by a preceding upload is ahead of this one on the stream
      cudaError_t e = cudaMemcpyAsync(stage_[b], src + at, len, cudaMemcpyDeviceToHost, s_);
      if (e != cudaSuccess || (e = cudaEventRecord(staged_[b], s_)) != cudaSuccess) return e;
      if (prev >= 0) {
        if ((e = cudaEventSynchronize(staged_[prev])) != cudaSuccess) return e;
        par_copy(dst + prev_at, stage_[prev], prev_len, threads_);
      }
      prev = b; prev_at = at; prev_len = len;
    }
    if (prev >= 0) {
      const cudaError_t e = cudaEventSynchronize(staged_[prev]);
      if (e != cudaSuccess) return e;
      par_copy(dst + prev_at, stage_[prev], prev_len, threads_);
    }
    return cudaSuccess;
  }

 private:
  cudaStream_t s_;
  uint32_t threads_;
  std::vector<void*> dev_;
  uint8_t* stage_[2] = {nullptr, nullptr};
  cudaEvent_t staged_[2] = {nullptr, nullptr};
  uint64_t stage_bytes_ = 0;
};

}  // namespace link
}  // namespace fgb
