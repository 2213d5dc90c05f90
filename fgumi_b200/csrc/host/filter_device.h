// The device half of fgb_filter_records: launchers of filter_records_kernels.cuh and the CUB scans, defined in
// capi.cu (which owns the handle and compiles the kernels), called by the host driver in filter_host.cpp.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

#include "record_filter.h"

namespace fgb {

struct FilterCfg {                    // the options as pass 1 reads them
  rfilter::Tier cc, ab, ba;
  double min_mean_q, max_no_call;     // min_mean_q < 0: none
  int min_bq;                         // < 0: none
  uint8_t require_ss, reverse_tags, regenerate;   // regenerate: a reference was given
};

enum : uint8_t { kTagsKept = 0, kTagsRemoved = 1, kTagsRegenerated = 2 };
enum : uint8_t { kErrNone = 0, kErrContig = 1, kErrPastEnd = 2, kErrCigar = 3 };   // pass 1's error codes

struct FRec {                         // pass 1's result for one record, read by the decision and pass 2
  uint32_t nm_s, nm_e, uq_s, uq_e, md_s, md_e;   // the first NM / UQ / MD entries, record offsets; s == e: none
  int32_t nm;
  uint32_t uq, md_len;
  uint32_t out_size;                  // the edited record's size
  uint64_t ref0;                      // the alignment's first base in the genome; ~0: no reference span (MD "0")
  uint16_t flags;
  uint8_t action, pass, keep, pad[3];
};

namespace filterdev {

cudaError_t pass1(uint8_t* rec, const uint64_t* off, uint64_t base, uint32_t n, const FilterCfg& cfg,
                  const int32_t* ctg_of_ref, const uint64_t* ctg_off, const uint64_t* ctg_len, const uint8_t* genome,
                  uint64_t first, FRec* out, unsigned long long* err, unsigned long long* counters, int sm_count,
                  cudaStream_t s);
cudaError_t decide(FRec* fr, const uint32_t* order, const uint32_t* tpl, uint32_t n_tpl, bool by_template,
                   unsigned long long* counters, cudaStream_t s);
// koff / roff[0..n]: offsets of each output position's entry in the kept / rejects stream (ks / rs: n + 1 scratch).
// temp == nullptr sizes the scan's scratch.
cudaError_t offsets(void* temp, size_t* temp_bytes, const FRec* fr, const uint32_t* order, uint32_t n,
                    bool track_rejects, uint64_t* ks, uint64_t* rs, uint64_t* koff, uint64_t* roff, cudaStream_t s);
cudaError_t pass2(const uint8_t* rec, const uint64_t* off, uint64_t base, uint32_t n, const FRec* fr,
                  const uint32_t* order, const uint64_t* koff, const uint64_t* roff, bool track_rejects,
                  const uint8_t* genome, uint8_t* kept, uint8_t* rejects, int sm_count, cudaStream_t s);

}  // namespace filterdev
}  // namespace fgb
