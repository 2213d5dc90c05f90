// Launchers of the zipper's kernels (zipper_kernels.cuh) and its CUB scan; the driver is host/zipper_host.cpp.
#include <cuda_runtime.h>

#include <algorithm>
#include <cub/device/device_scan.cuh>

#include "host/zipper_device.h"
#include "zipper_kernels.cuh"

namespace fgb {
namespace zipdev {

namespace {
unsigned warp_grid(uint32_t n, int sm_count) {   // one warp per record, at most 16 CTAs per SM (grid-stride)
  const uint64_t want = (static_cast<uint64_t>(n) * 32 + kZipperThreads - 1) / kZipperThreads;
  return static_cast<unsigned>(std::max<uint64_t>(1, std::min<uint64_t>(want, static_cast<uint64_t>(sm_count) * 16)));
}
}  // namespace

cudaError_t sizes(const uint8_t* um, const uint64_t* uoff, const uint8_t* mp, const uint64_t* moff,
                  const zip::ZRec* zr, uint32_t n, zip::Sets sets, bool skip_tc, uint64_t* size, int sm_count,
                  cudaStream_t s) {
  cudaError_t e = cudaMemsetAsync(size + n, 0, sizeof(uint64_t), s);
  if (e != cudaSuccess || !n) return e;
  zipper_sizes_kernel<<<warp_grid(n, sm_count), kZipperThreads, 0, s>>>(um, uoff, mp, moff, zr, n, sets, skip_tc, size);
  return cudaGetLastError();
}

cudaError_t offsets(void* temp, size_t* temp_bytes, const uint64_t* size, uint64_t* off, uint32_t n, cudaStream_t s) {
  return cub::DeviceScan::ExclusiveSum(temp, *temp_bytes, size, off, static_cast<int>(n) + 1, s);
}

cudaError_t write(const uint8_t* um, const uint64_t* uoff, const uint8_t* mp, const uint64_t* moff,
                  const zip::ZRec* zr, uint32_t n, zip::Sets sets, bool skip_tc, const uint64_t* off, uint8_t* out,
                  int sm_count, cudaStream_t s) {
  if (!n) return cudaSuccess;
  zipper_write_kernel<<<warp_grid(n, sm_count), kZipperThreads, 0, s>>>(um, uoff, mp, moff, zr, n, sets, skip_tc, off,
                                                                        out);
  return cudaGetLastError();
}

}  // namespace zipdev
}  // namespace fgb
