// Launchers of the metrics collector's kernels (metrics_kernels.cuh) and its CUB scans, selects and radix sorts;
// the driver is host/metrics_host.cpp.
#include <cuda_runtime.h>

#include <algorithm>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <cub/iterator/counting_input_iterator.cuh>

#include "host/metrics_device.h"
#include "metrics_kernels.cuh"

namespace fgb {
namespace metrics {

namespace {
unsigned blocks(uint32_t n, int threads) { return std::max<unsigned>(1, (n + threads - 1) / threads); }
int bits_of(uint64_t v) { int b = 0; while (b < 64 && (v >> b)) ++b; return std::max(b, 1); }
}  // namespace

cudaError_t template_pass(const uint8_t* rec, const uint64_t* off, const uint32_t* tpl_first, const int32_t* prim,
                          uint32_t n_tpl, const IvTable& iv, fgb_metrics_template* out, cudaStream_t s) {
  if (!n_tpl) return cudaSuccess;
  metrics_template_kernel<<<blocks(n_tpl, kTplThreads), kTplThreads, 0, s>>>(rec, off, tpl_first, prim, n_tpl, iv, out);
  return cudaGetLastError();
}

cudaError_t family_temp_bytes(uint32_t n, size_t* bytes) {
  size_t a = 0, b = 0, c = 0, d = 0;
  cub::CountingInputIterator<uint32_t> it(0);
  cudaError_t e;
  if ((e = cub::DeviceScan::InclusiveSum(nullptr, a, static_cast<uint32_t*>(nullptr), static_cast<uint32_t*>(nullptr),
                                         static_cast<int>(n))))
    return e;
  if ((e = cub::DeviceSelect::Flagged(nullptr, b, it, static_cast<uint32_t*>(nullptr), static_cast<uint32_t*>(nullptr),
                                      static_cast<uint32_t*>(nullptr), static_cast<int>(n))))
    return e;
  if ((e = cub::DeviceRadixSort::SortPairs(nullptr, c, static_cast<uint64_t*>(nullptr), static_cast<uint64_t*>(nullptr),
                                           static_cast<uint32_t*>(nullptr), static_cast<uint32_t*>(nullptr),
                                           static_cast<int>(n))))
    return e;
  if ((e = cub::DeviceRadixSort::SortPairs(nullptr, d, static_cast<uint32_t*>(nullptr), static_cast<uint32_t*>(nullptr),
                                           static_cast<uint32_t*>(nullptr), static_cast<uint32_t*>(nullptr),
                                           static_cast<int>(n))))
    return e;
  *bytes = std::max(std::max(a, b), std::max(c, d));
  return cudaSuccess;
}

cudaError_t family_pass(const FTpl* t, uint32_t n, int base_bits, FamilyBufs& b, const Hist& h, cudaStream_t s) {
  if (!n) return cudaSuccess;
  const int ni = static_cast<int>(n);
  cub::CountingInputIterator<uint32_t> it(0);
  size_t tb = b.temp_bytes;
  cudaError_t e;
  metrics_group_flags_kernel<<<blocks(n, 256), 256, 0, s>>>(t, n, b.flag, b.base_a, b.perm_a);
  if ((e = cudaGetLastError())) return e;
  // group ids (1-based) and group starts
  if ((e = cub::DeviceScan::InclusiveSum(b.temp, tb, b.flag, b.gid, ni, s))) return e;
  tb = b.temp_bytes;
  if ((e = cub::DeviceSelect::Flagged(b.temp, tb, it, b.flag, b.group_start, b.counts, ni, s))) return e;
  // stable (group, base) order: by base, then by group
  tb = b.temp_bytes;
  if ((e = cub::DeviceRadixSort::SortPairs(b.temp, tb, b.base_a, b.base_b, b.perm_a, b.perm_b, ni, 0, base_bits, s)))
    return e;
  metrics_gather_kernel<<<blocks(n, 256), 256, 0, s>>>(b.gid, b.perm_b, n, b.key_a);
  if ((e = cudaGetLastError())) return e;
  tb = b.temp_bytes;
  if ((e = cub::DeviceRadixSort::SortPairs(b.temp, tb, b.key_a, b.key_b, b.perm_b, b.perm_a, ni, 0, bits_of(n), s)))
    return e;
  metrics_run_flags_kernel<<<blocks(n, 256), 256, 0, s>>>(t, b.key_b, b.perm_a, n, b.flag);
  if ((e = cudaGetLastError())) return e;
  tb = b.temp_bytes;
  if ((e = cub::DeviceSelect::Flagged(b.temp, tb, it, b.flag, b.run_start, b.counts + 1, ni, s))) return e;
  metrics_ds_kernel<<<blocks(n, kCountThreads), kCountThreads, 0, s>>>(t, b.perm_a, b.run_start, b.counts + 1, n, h);
  if ((e = cudaGetLastError())) return e;
  metrics_cs_kernel<<<blocks(n, kCountThreads), kCountThreads, 0, s>>>(t, b.group_start, b.counts, n, h);
  return cudaGetLastError();
}

}  // namespace metrics
}  // namespace fgb
