// Host half of UMI assignment (fgb_umi_assign): the unique-key table of a call and the order-dependent rules
// applied to the capture lists the device found.  umi_host.cpp; restated in oracle/umi_oracle.py.
#pragma once

#include <cstdint>
#include <string>
#include <string_view>
#include <vector>

#include "../../../include/fgumi_b200.h"

namespace fgb_umi {

struct Call {
  std::vector<std::string_view> umis;   // the call's UMIs after truncation (views into the caller's buffer)
  std::vector<fgb_umi_key> keys;
  std::vector<uint8_t> bytes;           // key strings
  std::vector<uint32_t> key_of;         // per UMI; UINT32_MAX = no key
};

// "" on success, else what is wrong with the options / call.
std::string check_options(const fgb_umi_options& o);
std::string prepare(const fgb_umi_options& o, const uint8_t* umis, const uint64_t* off, uint64_t n, Call* c);
// Does the call need the device (any edge possible)?
bool needs_edges(const fgb_umi_options& o, const Call& c);
// Mapped edit and mapped paired compare bytes; the rest compare BitEncs.
bool uses_bytes(const fgb_umi_options& o);
// ids from 0 as a fresh assigner gives them; edge_off / edges: the call's CSR (may be null when needs_edges
// is false).
void resolve(const fgb_umi_options& o, const Call& c, const uint64_t* edge_off, const uint32_t* edges,
             uint64_t* ids, uint8_t* kinds);

// Runs f(i) for i in [0, n) on up to n_threads threads (contiguous ranges).
template <class F>
void parallel_for(uint64_t n, uint32_t n_threads, F&& f);

}  // namespace fgb_umi

#include <algorithm>
#include <exception>
#include <thread>

template <class F>
void fgb_umi::parallel_for(uint64_t n, uint32_t n_threads, F&& f) {
  const uint64_t t = std::min<uint64_t>(n_threads > 1 ? n_threads : 1, n);
  if (t <= 1) {
    for (uint64_t i = 0; i < n; ++i) f(i);
    return;
  }
  // An exception of a worker (or of creating one) is rethrown on the calling thread after every worker has joined.
  std::vector<std::exception_ptr> errs(t);
  std::vector<std::thread> th;
  std::exception_ptr spawn;
  try {
    th.reserve(t);
    for (uint64_t w = 0; w < t; ++w)
      th.emplace_back([&, w] {
        try {
          for (uint64_t i = n * w / t, e = n * (w + 1) / t; i < e; ++i) f(i);
        } catch (...) {
          errs[w] = std::current_exception();
        }
      });
  } catch (...) {
    spawn = std::current_exception();
  }
  for (auto& x : th) x.join();
  if (spawn) std::rethrow_exception(spawn);
  for (auto& e : errs) if (e) std::rethrow_exception(e);
}
