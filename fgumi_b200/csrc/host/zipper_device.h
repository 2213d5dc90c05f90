// The device half of fgb_zipper_records: launchers of ../zipper_kernels.cuh and the CUB scan, defined in zipper.cu,
// called by the host driver in zipper_host.cpp.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

#include "zipper_rules.h"

namespace fgb {
namespace zipdev {

// size[p] = 4 + the size of output record p, size[n] = 0 (the exclusive scan's total).  um / mp: the run's unmapped
// and mapped records; uoff / moff: their offsets relative to um / mp.
cudaError_t sizes(const uint8_t* um, const uint64_t* uoff, const uint8_t* mp, const uint64_t* moff,
                  const zip::ZRec* zr, uint32_t n, zip::Sets sets, bool skip_tc, uint64_t* size, int sm_count,
                  cudaStream_t s);
// off[0..n]: the exclusive scan of size[0..n]; temp == nullptr sizes the scan's scratch
cudaError_t offsets(void* temp, size_t* temp_bytes, const uint64_t* size, uint64_t* off, uint32_t n, cudaStream_t s);
// Each output record as [u32 block_size][record] at out + off[p]
cudaError_t write(const uint8_t* um, const uint64_t* uoff, const uint8_t* mp, const uint64_t* moff,
                  const zip::ZRec* zr, uint32_t n, zip::Sets sets, bool skip_tc, const uint64_t* off, uint8_t* out,
                  int sm_count, cudaStream_t s);

}  // namespace zipdev
}  // namespace fgb
