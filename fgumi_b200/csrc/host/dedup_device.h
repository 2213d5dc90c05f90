// The device half of the template scores (dedup_kernels.cuh): defined in capi.cu, which owns the handle and compiles
// the kernel; called by fgb_record_quality_scores there and by the deduper's flush in dedup_host.cpp.
#pragma once
#include <cstdint>
#include <string>

#include "../../../include/fgumi_b200.h"

namespace fgb {
namespace dedupdev {

// scores[i] = sum(min(q, 15)) over the quality bytes of record i (rec[i], len[i] bytes, each at least 32), staged
// through the handle's page-locked chunks on n_threads host threads.  Touches only the handle's score state (its own
// stream, buffers and events), so it may run on one thread while another runs fgb_umi_assign on the same handle.
// kernel_ms: the score kernel's time by CUDA events.  On failure *err says why.
fgb_status quality_scores(fgb_handle* h, uint64_t n, const uint8_t* const* rec, const uint64_t* len, uint32_t n_threads,
                          uint32_t* scores, float* kernel_ms, std::string* err);

}  // namespace dedupdev
}  // namespace fgb
