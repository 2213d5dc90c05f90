// K4 — consensus filter as an epilogue of the vote (SURVEY §8f N2), single-strand reads.
// What `fgumi filter` does to a simplex consensus record, on the columns while they are still in
// HBM: per-base masking (crates/fgumi-consensus/src/filter.rs:655-696 mask_bases), the per-read depth
// and error-rate gates (:453-471 filter_read, fed by the cD / cE values the caller would write,
// caller.rs:322-329) and the no-call / mean-quality gates (commands/filter.rs:909-929).
// One warp per unit; integer work plus one f32 and two f64 divisions per unit.
#pragma once
#include <stdint.h>

#include "../../include/fgumi_b200.h"

namespace fgb {

struct FilterArgs {
  const fgb_unit* units;        // biased like the vote's
  uint64_t unit_begin, unit_end;
  uint8_t* base;                // consensus columns, masked in place
  uint8_t* qual;
  const uint16_t* depth;
  const uint16_t* errors;
  const uint16_t* emax;         // [65536]: largest error count e with (double)e / (double)d <= max_base_error_rate
  uint8_t* status;              // per unit (index u - unit_begin)
  uint32_t* masked;             // per unit newly masked bases, may be null
  unsigned long long* counters; // device counter block (FGB_CTR_FILTER_*)
  uint32_t min_reads;
  uint32_t min_base_quality;    // 0 = none (no quality is below 0)
  uint32_t per_base_tags;       // 0: the record carries no cd/ce arrays -> depth 0 everywhere (filter.rs:677-678)
  double max_read_error_rate;
  double min_mean_base_quality; // < 0 = none
  double max_no_call_fraction;
};

// The read-level gates of one unit from its reductions (filter.rs:453-471, commands/filter.rs:909-929).
__device__ __forceinline__ uint32_t filter_unit_status(const FilterArgs& a, uint32_t L, uint32_t maxd, uint32_t td,
                                                       uint32_t te, uint32_t ncount, uint32_t qsum) {
  uint32_t st = FGB_FILTER_PASS;
  const float ce = td == 0u ? 0.0f : __fdiv_rn(__uint2float_rn(te), __uint2float_rn(td));   // caller.rs:322-329
  if (maxd < a.min_reads) st = FGB_FILTER_INSUFFICIENT_READS;                               // cD
  else if (static_cast<double>(ce) > a.max_read_error_rate) st = FGB_FILTER_EXCESSIVE_ERROR_RATE;
  else {
    const uint32_t non_n = L - ncount;
    const double mean = non_n == 0u ? 0.0 : __ddiv_rn(static_cast<double>(qsum), static_cast<double>(non_n));
    if (a.min_mean_base_quality >= 0.0 && mean < a.min_mean_base_quality) st = FGB_FILTER_LOW_MEAN_QUALITY;
    else if (a.max_no_call_fraction >= 1.0) {
      if (static_cast<double>(ncount) > a.max_no_call_fraction) st = FGB_FILTER_TOO_MANY_NO_CALLS;
    } else if (__ddiv_rn(static_cast<double>(ncount), static_cast<double>(L)) > a.max_no_call_fraction) {
      st = FGB_FILTER_TOO_MANY_NO_CALLS;
    }
  }
  return st;
}

// One unit on one warp, one position per lane and step (any alignment).  Lane 0 returns status and newly masked bases.
__device__ __forceinline__ uint32_t filter_unit_warp(const FilterArgs& a, const fgb_unit& un, uint32_t lane, uint32_t& newly_out) {
  const uint32_t L = un.cons_len;
  uint32_t maxd = 0, td = 0, te = 0, ncount = 0, qsum = 0, newly = 0;
  for (uint32_t p = lane; p < L; p += 32u) {
    const uint64_t o = un.out_off + p;
    uint32_t b = a.base[o], q = a.qual[o];
    const uint32_t d = a.depth[o], e = a.errors[o];
    maxd = d > maxd ? d : maxd; td += d; te += e;
    // the filter reads cd / ce back from the record, where the simplex caller stored them clamped to
    // i16::MAX (vanilla_caller.rs:1410-1412)
    const uint32_t dt = a.per_base_tags ? (d < 32767u ? d : 32767u) : 0u, et = a.per_base_tags ? (e < 32767u ? e : 32767u) : 0u;
    const bool mask = q < a.min_base_quality || dt < a.min_reads || (dt > 0u && et > a.emax[dt]);
    if (mask) {
      newly += (b != 'N');
      b = 'N'; q = 2u;
      a.base[o] = 'N'; a.qual[o] = 2;
    }
    if (b == 'N') ++ncount; else qsum += q;
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const uint32_t m = __shfl_xor_sync(0xFFFFFFFFu, maxd, off);
    maxd = m > maxd ? m : maxd;
    td += __shfl_xor_sync(0xFFFFFFFFu, td, off);
    te += __shfl_xor_sync(0xFFFFFFFFu, te, off);
    ncount += __shfl_xor_sync(0xFFFFFFFFu, ncount, off);
    qsum += __shfl_xor_sync(0xFFFFFFFFu, qsum, off);
    newly += __shfl_xor_sync(0xFFFFFFFFu, newly, off);
  }
  newly_out = newly;
  return filter_unit_status(a, L, maxd, td, te, ncount, qsum);
}

// Fallback kernel: one warp per unit (column pointers that are not aligned for the word kernel).
__global__ void __launch_bounds__(256) filter_simplex_kernel(const FilterArgs a) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint64_t warps = (static_cast<uint64_t>(gridDim.x) * blockDim.x) >> 5;
  unsigned long long pass_cnt = 0, masked_cnt = 0, rec_cnt = 0;
  for (uint64_t u = a.unit_begin + ((static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5);
       u < a.unit_end; u += warps) {
    const fgb_unit un = a.units[u];
    if (un.cons_len == 0) {                     // no consensus read was produced for this unit
      if (lane == 0) { a.status[u - a.unit_begin] = FGB_FILTER_NO_RECORD; if (a.masked) a.masked[u - a.unit_begin] = 0; }
      continue;
    }
    uint32_t newly;
    const uint32_t st = filter_unit_warp(a, un, lane, newly);
    if (lane == 0) {
      a.status[u - a.unit_begin] = static_cast<uint8_t>(st);
      if (a.masked) a.masked[u - a.unit_begin] = newly;
      ++rec_cnt; pass_cnt += (st == FGB_FILTER_PASS); masked_cnt += newly;
    }
  }
  if (lane == 0 && rec_cnt) {
    atomicAdd(a.counters + FGB_CTR_FILTER_RECORDS, rec_cnt);
    atomicAdd(a.counters + FGB_CTR_FILTER_PASSED, pass_cnt);
    atomicAdd(a.counters + FGB_CTR_FILTER_BASES_MASKED, masked_cnt);
  }
}

// ---- K4, word kernel ---------------------------------------------------------------------------------
// Work item = 8 consecutive positions of one unit (one 8-byte word of the base and quality rows, one 16-byte word
// of the depth and error rows); a CTA takes kFilterChunk consecutive units and deals their items to its threads from
// one flat index, so a 150-base unit (19 items) does not leave 13 lanes of a warp idle.  The per-unit reductions are
// folded inside the warp first (items of one unit sit on consecutive lanes: a segmented shuffle reduction) and then
// into shared memory by the first lane of each run.
#ifndef FGB_FILTER_CHUNK
#define FGB_FILTER_CHUNK 256
#endif
constexpr int kFilterChunk = FGB_FILTER_CHUNK;     // 32 .. 256 (power of two): units / jobs whose descriptors are fetched in one round

__global__ void __launch_bounds__(256, 4) filter_simplex_words_kernel(const FilterArgs a) {
  __shared__ unsigned long long s_off[kFilterChunk];
  __shared__ uint32_t s_len[kFilterChunk], s_pref[kFilterChunk + 1], s_general[kFilterChunk];
  __shared__ uint32_t s_maxd[kFilterChunk], s_td[kFilterChunk], s_te[kFilterChunk], s_qs[kFilterChunk], s_nc[kFilterChunk], s_new[kFilterChunk];
  const uint32_t tid = threadIdx.x, lane = tid & 31u;
  const uint64_t u0 = a.unit_begin + static_cast<uint64_t>(blockIdx.x) * kFilterChunk;
  const uint32_t nj = static_cast<uint32_t>(a.unit_end - u0 < kFilterChunk ? a.unit_end - u0 : kFilterChunk);
  __shared__ uint32_t s_wsum[kFilterChunk / 32];
  if (tid < static_cast<uint32_t>(kFilterChunk)) {
    uint32_t items = 0;
    if (tid < nj) {
      const fgb_unit un = a.units[u0 + tid];
      const bool general = (un.out_off & 7ull) != 0ull;
      s_off[tid] = un.out_off; s_len[tid] = un.cons_len; s_general[tid] = general ? 1u : 0u;
      s_maxd[tid] = 0u; s_td[tid] = 0u; s_te[tid] = 0u; s_qs[tid] = 0u; s_nc[tid] = 0u; s_new[tid] = 0u;
      items = general ? 0u : (un.cons_len + 7u) >> 3;
    }
    uint32_t incl = items;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const uint32_t v = __shfl_up_sync(0xFFFFFFFFu, incl, off);
      if (lane >= static_cast<uint32_t>(off)) incl += v;
    }
    s_pref[tid + 1] = incl;                            // within the warp; the warps in front are added below
    if (lane == 31u) s_wsum[tid >> 5] = incl;
  }
  __syncthreads();
  if (kFilterChunk > 32 && tid >= 32u && tid < static_cast<uint32_t>(kFilterChunk)) {
    uint32_t add = 0;
    for (uint32_t w = 0; w < (tid >> 5); ++w) add += s_wsum[w];
    s_pref[tid + 1] += add;
  }
  if (tid == 0) s_pref[0] = 0u;
  __syncthreads();
  const uint32_t total = s_pref[kFilterChunk];
  const uint32_t minq = a.min_base_quality, min_reads = a.min_reads;
  const bool tags = a.per_base_tags != 0u;
  for (uint32_t base = 0; base < total; base += 256u) {        // uniform trip count: the shuffles below need every lane
    const uint32_t it = base + tid;
    uint32_t jl = 0xFFFFFFFFu;
    uint32_t maxd = 0, td = 0, te = 0, qn = 0, newly = 0;       // qn = quality sum | no-call count << 16
    if (it < total) {
      jl = 0;
#pragma unroll
      for (int step = kFilterChunk / 2; step > 0; step >>= 1)
        if (s_pref[jl + step] <= it) jl += step;
      const uint32_t p0 = (it - s_pref[jl]) * 8u;
      const uint32_t L = s_len[jl];
      const uint32_t live = L - p0 < 8u ? L - p0 : 8u;
      const unsigned long long o = s_off[jl] + p0;
      uint2 b2 = *reinterpret_cast<const uint2*>(a.base + o);
      uint2 q2 = *reinterpret_cast<const uint2*>(a.qual + o);
      const uint4 d4 = *reinterpret_cast<const uint4*>(a.depth + o);
      const uint4 e4 = *reinterpret_cast<const uint4*>(a.errors + o);
      uint32_t bw[2] = {b2.x, b2.y}, qw[2] = {q2.x, q2.y};
      const uint32_t dw[4] = {d4.x, d4.y, d4.z, d4.w}, ew[4] = {e4.x, e4.y, e4.z, e4.w};
      uint32_t last_dt = 0xFFFFFFFFu, last_lim = 0u, ncount = 0u, qsum = 0u;
      bool changed = false;
#pragma unroll
      for (uint32_t k = 0; k < 8u; ++k) {
        if (k < live) {
          const uint32_t sh8 = 8u * (k & 3u), sh16 = 16u * (k & 1u);
          uint32_t b = (bw[k >> 2] >> sh8) & 0xFFu, q = (qw[k >> 2] >> sh8) & 0xFFu;
          const uint32_t d = (dw[k >> 1] >> sh16) & 0xFFFFu, e = (ew[k >> 1] >> sh16) & 0xFFFFu;
          maxd = d > maxd ? d : maxd; td += d; te += e;
          // the filter reads cd / ce back from the record, clamped to i16::MAX (vanilla_caller.rs:1410-1412)
          const uint32_t dt = tags ? (d < 32767u ? d : 32767u) : 0u, et = tags ? (e < 32767u ? e : 32767u) : 0u;
          if (dt != last_dt) { last_dt = dt; last_lim = dt ? a.emax[dt] : 0u; }   // neighbours mostly share a depth
          const bool mask = q < minq || dt < min_reads || (dt > 0u && et > last_lim);
          if (mask) {
            newly += (b != 'N');
            b = 'N'; q = 2u;
            bw[k >> 2] = (bw[k >> 2] & ~(0xFFu << sh8)) | (0x4Eu << sh8);
            qw[k >> 2] = (qw[k >> 2] & ~(0xFFu << sh8)) | (0x02u << sh8);
            changed = true;
          }
          if (b == 'N') ++ncount; else qsum += q;
        }
      }
      if (changed) {                             // bytes behind the row's end are written back as they were read
        *reinterpret_cast<uint2*>(a.base + o) = make_uint2(bw[0], bw[1]);
        *reinterpret_cast<uint2*>(a.qual + o) = make_uint2(qw[0], qw[1]);
      }
      qn = qsum | (ncount << 16);
    }
    // segmented reduction over runs of equal jl (items of a unit are on consecutive lanes)
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const uint32_t j2 = __shfl_down_sync(0xFFFFFFFFu, jl, off);
      const uint32_t m2 = __shfl_down_sync(0xFFFFFFFFu, maxd, off);
      const uint32_t t2 = __shfl_down_sync(0xFFFFFFFFu, td, off);
      const uint32_t e2 = __shfl_down_sync(0xFFFFFFFFu, te, off);
      const uint32_t q2 = __shfl_down_sync(0xFFFFFFFFu, qn, off);
      const uint32_t n2 = __shfl_down_sync(0xFFFFFFFFu, newly, off);
      if (lane + off < 32u && j2 == jl) {
        maxd = m2 > maxd ? m2 : maxd; td += t2; te += e2; qn += q2; newly += n2;
      }
    }
    const uint32_t jprev = __shfl_up_sync(0xFFFFFFFFu, jl, 1);
    if (jl != 0xFFFFFFFFu && (lane == 0u || jprev != jl)) {
      atomicMax(&s_maxd[jl], maxd);
      atomicAdd(&s_td[jl], td);
      atomicAdd(&s_te[jl], te);
      atomicAdd(&s_new[jl], newly);
      // (inside one warp the packed word cannot carry: 32 items x 8 positions x Q255 < 65536; across items it could)
      atomicAdd(&s_qs[jl], qn & 0xFFFFu);
      atomicAdd(&s_nc[jl], qn >> 16);
    }
  }
  __syncthreads();
  // units whose rows are not 8-aligned: one warp per unit
  for (uint32_t jl = tid >> 5; jl < nj; jl += 8u) {
    if (s_general[jl] && s_len[jl] != 0u) {
      uint32_t newly;
      const fgb_unit un = a.units[u0 + jl];
      const uint32_t st = filter_unit_warp(a, un, lane, newly);
      if (lane == 0) { s_new[jl] = newly; s_maxd[jl] = 0x80000000u | st; }
    }
  }
  __syncthreads();
  if (tid < static_cast<uint32_t>(kFilterChunk)) {
    unsigned long long rec = 0, pass = 0, msk = 0;
    if (tid < nj) {
      const uint32_t L = s_len[tid];
      uint32_t st, newly = 0;
      if (L == 0u) st = FGB_FILTER_NO_RECORD;
      else {
        newly = s_new[tid];
        st = s_general[tid] ? (s_maxd[tid] & 0xFFu)
                            : filter_unit_status(a, L, s_maxd[tid], s_td[tid], s_te[tid], s_nc[tid], s_qs[tid]);
        rec = 1; pass = st == FGB_FILTER_PASS; msk = newly;
      }
      a.status[u0 + tid - a.unit_begin] = static_cast<uint8_t>(st);
      if (a.masked) a.masked[u0 + tid - a.unit_begin] = newly;
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      rec += __shfl_xor_sync(0xFFFFFFFFu, rec, off);
      pass += __shfl_xor_sync(0xFFFFFFFFu, pass, off);
      msk += __shfl_xor_sync(0xFFFFFFFFu, msk, off);
    }
    if (lane == 0 && rec) {                  // one warp per 32 units of the chunk
      atomicAdd(a.counters + FGB_CTR_FILTER_RECORDS, rec);
      atomicAdd(a.counters + FGB_CTR_FILTER_PASSED, pass);
      atomicAdd(a.counters + FGB_CTR_FILTER_BASES_MASKED, msk);
    }
  }
}

}  // namespace fgb
