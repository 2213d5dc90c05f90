// `fgumi zipper` on the device (driven by host/zipper_host.cpp through the launchers in zipper.cu), one warp per
// output record with the lanes across its bytes:
//   sizes  the record's plan (mate fix, tag layout, AS / XS, tc; host/zipper_rules.h) and its output size, the mate's
//          CIGAR text length by a warp sum of the ops' digit counts;
//   write  the edited record with its block_size word at its scanned offset: fixed fields, name, CIGAR, sequence and
//          qualities copied by lanes, the aux area assembled, reversal and reverse complement done by lanes, MC
//          rendered with each op's place from a warp scan.
// A passed-through unmapped record is copied as it is.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "host/zipper_rules.h"

namespace fgb {

constexpr int kZipperThreads = 256;

namespace zk {

constexpr unsigned kFull = 0xffffffffu;

struct WarpSum {
  __device__ uint32_t operator()(uint32_t v) const { return __reduce_add_sync(kFull, v); }
};
struct WarpPrefix {   // inclusive prefix of v over the lanes; last(): lane 31's
  int lane;
  __device__ uint32_t operator()(uint32_t v) const {
    uint32_t x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t y = __shfl_up_sync(kFull, x, d);
      if (lane >= d) x += y;
    }
    return x;
  }
  __device__ uint32_t last(uint32_t x) const { return __shfl_sync(kFull, x, 31); }
};

}  // namespace zk

__global__ void __launch_bounds__(kZipperThreads) zipper_sizes_kernel(
    const uint8_t* __restrict__ um, const uint64_t* __restrict__ uoff, const uint8_t* __restrict__ mp,
    const uint64_t* __restrict__ moff, const zip::ZRec* __restrict__ zr, uint32_t n, zip::Sets sets, bool skip_tc,
    uint64_t* __restrict__ size) {
  const int lane = threadIdx.x & 31;
  const uint32_t warps = gridDim.x * (blockDim.x / 32);
  for (uint32_t i = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32; i < n; i += warps) {
    const zip::ZRec z = zr[i];
    uint64_t sz;
    if (z.kind == zip::kPass) {
      sz = uoff[z.src + 1] - uoff[z.src];
    } else {
      const zip::Plan p = zip::plan(z, um, uoff, mp, moff, sets, skip_tc, lane, 32, zk::WarpSum{});
      sz = zip::out_size(p, sets);
    }
    if (lane == 0) size[i] = 4 + sz;
  }
}

__global__ void __launch_bounds__(kZipperThreads) zipper_write_kernel(
    const uint8_t* __restrict__ um, const uint64_t* __restrict__ uoff, const uint8_t* __restrict__ mp,
    const uint64_t* __restrict__ moff, const zip::ZRec* __restrict__ zr, uint32_t n, zip::Sets sets, bool skip_tc,
    const uint64_t* __restrict__ off, uint8_t* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const uint32_t warps = gridDim.x * (blockDim.x / 32);
  for (uint32_t i = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32; i < n; i += warps) {
    const zip::ZRec z = zr[i];
    uint8_t* d = out + off[i];
    const uint32_t bs = static_cast<uint32_t>(off[i + 1] - off[i] - 4);
    if (lane < 4) d[lane] = static_cast<uint8_t>(bs >> (8 * lane));
    if (z.kind == zip::kPass) {
      zip::copy(d + 4, um + uoff[z.src], bs, lane, 32);
    } else {
      const zip::Plan p = zip::plan(z, um, uoff, mp, moff, sets, skip_tc, lane, 32, zk::WarpSum{});
      zip::write(d + 4, p, sets, lane, 32, zk::WarpPrefix{lane});
    }
  }
}

}  // namespace fgb
