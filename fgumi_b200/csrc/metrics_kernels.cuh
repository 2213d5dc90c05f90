// Device kernels of `fgumi duplex-metrics` / `simplex-metrics` (driver: host/metrics_host.cpp, launchers: metrics.cu).
//
// Template pass: one thread per template (QNAME run) of a staged run -- the host's template_order has already named
// the run's primary R1 and R2, so what is left per template is two flag tests, two tag walks over R1's aux block, two
// CIGAR walks and a Murmur3 over a ~30-byte name; metrics_rules.h holds that code for the host and the device.
//
// Family pass over the templates of closed coordinate groups (FTpl, in stream order):
//   metrics_group_flags_kernel  1 where a template's ReadInfoKey differs from its predecessor's (then a CUB scan gives
//                               group ids and a CUB select the group starts);
//   two stable CUB radix sorts, by base key then by group id, make each DS family (group, MI base) one contiguous
//   run in stream order; metrics_gather_kernel / metrics_run_flags_kernel find the runs;
//   metrics_ds_kernel           one thread per DS run: templates per (suffix kind, bucket), prefix sums over the 20
//                               fractions, then per fraction the SS sizes (no suffix, /A, /B), the DS size and the
//                               (ab, ba) pair (duplex_metrics.rs:318-356);
//   metrics_cs_kernel           one thread per coordinate group: the CS size and templates per fraction.
// Sizes below kSmall and pairs below kPair are counted in shared memory and added to the global histograms once per
// block; larger ones are appended to an overflow list that the host folds in.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "host/metrics_device.h"

namespace fgb {
namespace metrics {

__global__ void metrics_template_kernel(const uint8_t* __restrict__ rec, const uint64_t* __restrict__ off,
                                        const uint32_t* __restrict__ tpl_first, const int32_t* __restrict__ prim,
                                        uint32_t n_tpl, IvTable iv, fgb_metrics_template* __restrict__ out) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_tpl) return;
  const uint64_t b = tpl_first[t], e = tpl_first[t + 1];
  const int32_t p1 = prim[2 * t], p2 = prim[2 * t + 1];
  template_pass([&](int64_t k) { return rec + off[k]; }, [&](int64_t k) { return off[k + 1] - off[k]; }, e - b,
                p1, p2, iv, out + t);   // out[t].r1 is run-local: the host rebases it
}

__device__ __forceinline__ bool same_key(const FTpl& x, const FTpl& y) {
  return x.ref1 == y.ref1 && x.start1 == y.start1 && x.strand1 == y.strand1 && x.ref2 == y.ref2 &&
         x.start2 == y.start2 && x.strand2 == y.strand2;
}

// flag[i]: template i opens a coordinate group; the first sort's input (base key, stream index)
__global__ void metrics_group_flags_kernel(const FTpl* __restrict__ t, uint32_t n, uint32_t* __restrict__ flag,
                                           uint64_t* __restrict__ base, uint32_t* __restrict__ idx) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  flag[i] = i == 0 || !same_key(t[i], t[i - 1]);
  base[i] = t[i].base;
  idx[i] = i;
}

// gid_by_perm[i] = gid[perm[i]] - 1 (the scan is inclusive): the second sort's keys
__global__ void metrics_gather_kernel(const uint32_t* __restrict__ gid, const uint32_t* __restrict__ perm, uint32_t n,
                                      uint32_t* __restrict__ gid_by_perm) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) gid_by_perm[i] = gid[perm[i]] - 1;
}

__global__ void metrics_run_flags_kernel(const FTpl* __restrict__ t, const uint32_t* __restrict__ sgid,
                                         const uint32_t* __restrict__ perm, uint32_t n, uint32_t* __restrict__ flag) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) flag[i] = i == 0 || sgid[i] != sgid[i - 1] || t[perm[i]].base != t[perm[i - 1]].base;
}

struct SharedHist {
  uint32_t sizes[3][kFractions][kSmall];
  uint32_t pairs[kFractions][kPair][kPair];
  uint32_t templates[kFractions];
};

__device__ __forceinline__ void hist_clear(SharedHist& s) {
  uint32_t* w = &s.sizes[0][0][0];
  for (uint32_t i = threadIdx.x; i < sizeof(SharedHist) / 4; i += blockDim.x) w[i] = 0;
}

__device__ __forceinline__ void hist_flush(const SharedHist& s, const Hist& h) {
  for (uint32_t i = threadIdx.x; i < 3 * kFractions * kSmall; i += blockDim.x) {
    const uint32_t v = (&s.sizes[0][0][0])[i];
    if (v) atomicAdd(h.sizes + i, static_cast<unsigned long long>(v));
  }
  for (uint32_t i = threadIdx.x; i < kFractions * kPair * kPair; i += blockDim.x) {
    const uint32_t v = (&s.pairs[0][0][0])[i];
    if (v) atomicAdd(h.pairs + i, static_cast<unsigned long long>(v));
  }
  for (uint32_t i = threadIdx.x; i < kFractions; i += blockDim.x)
    if (s.templates[i]) atomicAdd(h.templates + i, static_cast<unsigned long long>(s.templates[i]));
}

__device__ __forceinline__ void push_over(const Hist& h, uint32_t kind, uint32_t f, uint32_t a, uint32_t b) {
  const unsigned long long k = atomicAdd(h.n_over, 1ull);
  if (k < h.cap) h.over[k] = Overflow{kind << 8 | f, a, b};
}

__device__ __forceinline__ void add_size(SharedHist& s, const Hist& h, uint32_t kind, uint32_t f, uint32_t size) {
  if (size < kSmall) atomicAdd(&s.sizes[kind][f][size], 1u);
  else push_over(h, kind, f, size, 0);
}

__global__ void __launch_bounds__(kCountThreads) metrics_ds_kernel(const FTpl* __restrict__ t,
                                                                   const uint32_t* __restrict__ perm,
                                                                   const uint32_t* __restrict__ run_start,
                                                                   const uint32_t* __restrict__ n_runs_p, uint32_t n,
                                                                   Hist h) {
  __shared__ SharedHist s;
  __shared__ uint32_t cnt[3][kFractions][kCountThreads];   // this thread's templates per (kind, bucket)
  hist_clear(s);
  const uint32_t me = threadIdx.x;
  for (int k = 0; k < 3; ++k)
    for (int f = 0; f < kFractions; ++f) cnt[k][f][me] = 0;
  __syncthreads();
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x, n_runs = *n_runs_p;
  if (r < n_runs) {
    const uint32_t b = run_start[r], e = r + 1 < n_runs ? run_start[r + 1] : n;
    for (uint32_t i = b; i < e; ++i) {
      const FTpl& x = t[perm[i]];
      ++cnt[x.kind][x.bucket][me];
    }
    uint32_t n0 = 0, na = 0, nb = 0;
    for (uint32_t f = 0; f < kFractions; ++f) {
      n0 += cnt[0][f][me];
      na += cnt[1][f][me];
      nb += cnt[2][f][me];
      if (n0 + na + nb == 0) continue;   // the family is not in this fraction's downsampled group
      if (n0) add_size(s, h, kSs, f, n0);
      if (na) add_size(s, h, kSs, f, na);
      if (nb) add_size(s, h, kSs, f, nb);
      add_size(s, h, kDs, f, na + nb);   // a family without suffixes still counts, with size 0
      const uint32_t ab = na >= nb ? na : nb, ba = na >= nb ? nb : na;
      if (ab < kPair) atomicAdd(&s.pairs[f][ab][ba], 1u);
      else push_over(h, kDup, f, ab, ba);
    }
  }
  __syncthreads();
  hist_flush(s, h);
}

__global__ void __launch_bounds__(kCountThreads) metrics_cs_kernel(const FTpl* __restrict__ t,
                                                                   const uint32_t* __restrict__ group_start,
                                                                   const uint32_t* __restrict__ n_groups_p, uint32_t n,
                                                                   Hist h) {
  __shared__ SharedHist s;
  __shared__ uint32_t cnt[kFractions][kCountThreads];
  hist_clear(s);
  const uint32_t me = threadIdx.x;
  for (int f = 0; f < kFractions; ++f) cnt[f][me] = 0;
  __syncthreads();
  const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x, n_groups = *n_groups_p;
  if (g < n_groups) {
    const uint32_t b = group_start[g], e = g + 1 < n_groups ? group_start[g + 1] : n;
    for (uint32_t i = b; i < e; ++i) ++cnt[t[i].bucket][me];
    uint32_t size = 0;
    for (uint32_t f = 0; f < kFractions; ++f) {
      size += cnt[f][me];
      if (!size) continue;
      add_size(s, h, kCs, f, size);
      atomicAdd(&s.templates[f], size);
    }
  }
  __syncthreads();
  hist_flush(s, h);
}

}  // namespace metrics
}  // namespace fgb
