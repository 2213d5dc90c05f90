// The device half of the metrics collector: launchers of ../metrics_kernels.cuh and the CUB calls, defined in
// ../metrics.cu, called by the host driver in metrics_host.cpp.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

#include "metrics_rules.h"

namespace fgb {
namespace metrics {

constexpr int kSmall = 32;          // sizes 0..31 in the shared histograms
constexpr int kPair = 8;            // (ab, ba) with both below 8 in the shared pair table
constexpr int kCountThreads = 128;
constexpr int kTplThreads = 128;
enum : uint32_t { kCs = 0, kSs = 1, kDs = 2, kDup = 3 };

struct FTpl {                       // one kept template as the family pass reads it
  int32_t ref1, start1, ref2, start2;
  uint8_t strand1, strand2, kind, bucket;
  uint32_t pad;
  uint64_t base;                    // canonical MI number, or (1 << 63) | host dictionary id
};

struct Overflow {                   // a size (kind < kDup) or a pair (kDup) the shared tables do not hold
  uint32_t code;                    // kind << 8 | fraction
  uint32_t a, b;
};

struct Hist {                       // the family pass's global outputs
  unsigned long long* sizes;        // [3][kFractions][kSmall]
  unsigned long long* pairs;        // [kFractions][kPair][kPair]
  unsigned long long* templates;    // [kFractions]
  Overflow* over;
  unsigned long long* n_over;       // entries appended (may exceed cap: the host then fails the call)
  uint64_t cap;
};


// out[t] for the n_tpl templates of a staged run: records rec + off[k] (run-local k), template t's records
// [tpl_first[t], tpl_first[t + 1]), its primary R1 / R2 slots prim[2 t], prim[2 t + 1] (-1: absent)
cudaError_t template_pass(const uint8_t* rec, const uint64_t* off, const uint32_t* tpl_first, const int32_t* prim,
                          uint32_t n_tpl, const IvTable& iv, fgb_metrics_template* out, cudaStream_t s);

// The family pass's scratch for n templates; temp == nullptr sizes the CUB scratch into *temp_bytes.
struct FamilyBufs {
  uint32_t *flag, *gid, *group_start, *perm_a, *perm_b, *key_a, *key_b, *run_start, *counts;   // counts[2]
  uint64_t *base_a, *base_b;
  void* temp;
  size_t temp_bytes;
};
cudaError_t family_temp_bytes(uint32_t n, size_t* bytes);
// Histograms of the n templates t (closed coordinate groups in stream order) added to h.  b.perm_a is left holding the
// templates in (group, base) order, stream order within each, and b.run_start[0 .. b.counts[1]) the DS runs' starts
// in it.  base_bits: the bits the base keys use.
cudaError_t family_pass(const FTpl* t, uint32_t n, int base_bits, FamilyBufs& b, const Hist& h, cudaStream_t s);

}  // namespace metrics
}  // namespace fgb
