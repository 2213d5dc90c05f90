// K2 (duplex) and K3 (CODEC) strand-combine kernels for sm_90a — pure integer/byte work.
//
// Replaces (reference = fgumi 0.2.0, crates/fgumi-consensus/src/):
//   duplex_caller.rs:838-1015   DuplexConsensusCaller::duplex_consensus (methylation disabled)
//   codec_caller.rs:507-520     reverse_complement_ss
//   codec_caller.rs:980-1023    pad_consensus (lowercase 'n', Q0, depth 0, errors 0)
//   codec_caller.rs:1029-1178   build_duplex_consensus_from_padded (+ disagreement gate)
//   codec_caller.rs:1183-1212   mask_consensus_quals_query_based
//   fgumi-dna/src/dna.rs:30-40  complement_base
//
// One warp per job, lanes stride the position axis (coalesced byte/u16 loads and stores); the
// job-level reductions (any-depth, disagreement counts) are warp shuffles.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/fgumi_b200.h"
#include "duplex_word.cuh"

namespace fgb {

constexpr int kCombineThreads = 256;
constexpr int kCombineJobsPerCta = kCombineThreads / 32;
constexpr int kCodecJobsPerCta = kCombineThreads / 32;

struct DuplexArgs {
  const uint8_t* bases;        // source base column (for the exact error recount)
  const uint64_t* reads;
  const fgb_unit* units;
  const uint8_t* ss_base;
  const uint8_t* ss_qual;
  const uint16_t* ss_depth;
  const uint16_t* ss_errors;
  const fgb_duplex_job* jobs;
  uint64_t n_jobs;
  uint8_t* out_base;
  uint8_t* out_qual;
  uint16_t* out_errors;
  uint8_t* out_status;
  unsigned long long* counters;
};

// duplex_caller.rs:783-791
__device__ __forceinline__ uint32_t cap_quality(int32_t s) {
  return s < 2 ? 2u : (s > 93 ? 93u : static_cast<uint32_t>(s));
}

// One job's descriptors, fetched one job ahead of the combine (the loads of job j + stride are in flight while
// job j is combined: two dependent rounds of global-memory latency leave the critical path).
struct DuplexJobRegs {
  fgb_duplex_job job;
  fgb_unit ua, ub;
  uint32_t ra1, rb1;      // read_begin of the units after a and b
};
__device__ __forceinline__ DuplexJobRegs load_duplex_job(const DuplexArgs& a, uint64_t j) {
  DuplexJobRegs r;
  r.job = a.jobs[j];
  r.ua = a.units[r.job.unit_a];
  r.ub = a.units[r.job.unit_b];
  r.ra1 = a.units[r.job.unit_a + 1].read_begin;
  r.rb1 = a.units[r.job.unit_b + 1].read_begin;
  return r;
}

// One job on one warp: every arm of duplex_consensus, any row length, any alignment.  It is the whole of the fallback
// kernel and the redo path of the word kernel below (single-strand arms, rows that are not 8-aligned, more than 255
// pooled source reads).
__device__ __forceinline__ uint8_t duplex_job_warp(const DuplexArgs& a, const DuplexJobRegs& cur, uint32_t lane) {
  const fgb_duplex_job job = cur.job;
  const fgb_unit ua = cur.ua, ub = cur.ub;
  const uint32_t la = ua.cons_len, lb = ub.cons_len;
  const uint32_t len = la < lb ? la : lb;                       // duplex_caller.rs:846-849
  const uint32_t ra0 = ua.read_begin, ra1 = cur.ra1;
  const uint32_t rb0 = ub.read_begin, rb1 = cur.rb1;
  // Word path: 8 positions per lane with byte-parallel arithmetic.  Needs 8-aligned rows (the layout rule
  // for inputs; job.out_off is the caller's) and per-position error counts that fit a byte.
  const bool words = ((ua.out_off | ub.out_off | job.out_off) & 7u) == 0 && (ra1 - ra0) + (rb1 - rb0) <= 255u;
  uint8_t status;
  if (words && len <= 256u) {
    // ---- one block per job (reads up to 256 bases): everything the job needs is requested at once ----
    const uint32_t p0 = lane * 8u;
    const bool active = p0 < len;
    uint2 ab2 = make_uint2(0, 0), bb2 = ab2, aq2 = ab2, bq2 = ab2;
    uint4 ad4 = make_uint4(0, 0, 0, 0), bd4 = ad4;
    if (active) {
      ab2 = *reinterpret_cast<const uint2*>(a.ss_base + ua.out_off + p0);
      bb2 = *reinterpret_cast<const uint2*>(a.ss_base + ub.out_off + p0);
      aq2 = *reinterpret_cast<const uint2*>(a.ss_qual + ua.out_off + p0);
      bq2 = *reinterpret_cast<const uint2*>(a.ss_qual + ub.out_off + p0);
      ad4 = *reinterpret_cast<const uint4*>(a.ss_depth + ua.out_off + p0);
      bd4 = *reinterpret_cast<const uint4*>(a.ss_depth + ub.out_off + p0);
    }
    const uint32_t na = ra1 - ra0, nr = na + (rb1 - rb0);
    // descriptors of the pooled source rows (AB rows then BA rows), one per lane, 32 at a time
    const uint64_t first_desc = lane < nr ? a.reads[lane < na ? ra0 + lane : rb0 + (lane - na)] : 0ull;
    // :852-853 strands with no coverage inside the truncated region are dropped (rows are padded with
    // zero depth, but a longer strand has real depths behind `len`: mask the last word)
    const uint32_t live = active ? (len - p0 < 8u ? len - p0 : 8u) : 0u;
    auto any16 = [&](const uint4& d) {
      const uint32_t w[4] = {d.x, d.y, d.z, d.w};
      uint32_t acc = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t keep = live >= 2u * k + 2u ? 0xFFFFFFFFu : (live == 2u * k + 1u ? 0x0000FFFFu : 0u);
        acc |= w[k] & keep;
      }
      return acc != 0u;
    };
    const bool a_any = __any_sync(0xFFFFFFFFu, any16(ad4));
    const bool b_any = __any_sync(0xFFFFFFFFu, any16(bd4));
    if (a_any && b_any) {
      status = FGB_DUPLEX_BOTH;
      uint32_t ob[2], oq[2], rawb[2], cnt[2] = {0u, 0u};
      const uint32_t abw[2] = {ab2.x, ab2.y}, bbw[2] = {bb2.x, bb2.y};
      const uint32_t aqw[2] = {aq2.x, aq2.y}, bqw[2] = {bq2.x, bq2.y};
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t eq = __vcmpeq4(abw[h], bbw[h]);                    // :912-927, bytewise
        const uint32_t sum = __vminu4(__vaddus4(aqw[h], bqw[h]), 0x5D5D5D5Du);
        const uint32_t dif = __vminu4(__vabsdiffu4(aqw[h], bqw[h]), 0x5D5D5D5Du);
        const uint32_t rq = __vmaxu4((eq & sum) | (~eq & dif), 0x02020202u);   // cap_quality; equal-quality dissent -> 2
        const uint32_t b_wins = ~eq & __vcmpgtu4(bqw[h], aqw[h]);
        rawb[h] = (bbw[h] & b_wins) | (abw[h] & ~b_wins);
        const uint32_t mask = __vcmpeq4(abw[h], 0x4E4E4E4Eu) | __vcmpeq4(bbw[h], 0x4E4E4E4Eu) |
                              __vcmpeq4(rq, 0x02020202u);                 // :930-935
        ob[h] = (0x4E4E4E4Eu & mask) | (rawb[h] & ~mask);
        oq[h] = (0x02020202u & mask) | (rq & ~mask);
      }
      // :943-951 exact error recount against the pooled source reads
      auto recount_word = [&](uint64_t d) {
        const uint32_t rl = static_cast<uint32_t>(d & 0xFFFFu);
        if (active && rl > p0) {
          const uint2 sb = *reinterpret_cast<const uint2*>(a.bases + (d >> 16) + p0);
          const uint32_t cov = rl - p0;                                   // covered positions of this word
          const uint32_t c0 = cov >= 4u ? 0xFFFFFFFFu : ((1u << (8u * cov)) - 1u);
          const uint32_t c1 = cov >= 8u ? 0xFFFFFFFFu : (cov > 4u ? ((1u << (8u * (cov - 4u))) - 1u) : 0u);
          const uint32_t sw[2] = {sb.x, sb.y}, cw[2] = {c0, c1};
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const uint32_t ne = ~__vcmpeq4(sw[h], rawb[h]) & ~__vcmpeq4(sw[h], 0x4E4E4E4Eu) & cw[h];
            cnt[h] += ne & 0x01010101u;
          }
        }
      };
      for (uint32_t c0 = 0; c0 < nr; c0 += 32u) {
        const uint32_t k = c0 + lane;
        const uint64_t mine = c0 == 0 ? first_desc : (k < nr ? a.reads[k < na ? ra0 + k : rb0 + (k - na)] : 0ull);
        const uint32_t m = nr - c0 < 32u ? nr - c0 : 32u;
#pragma unroll 8
        for (uint32_t r = 0; r < m; ++r) recount_word(__shfl_sync(0xFFFFFFFFu, mine, r));
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) cnt[h] &= ~__vcmpeq4(rawb[h], 0x4E4E4E4Eu);   // raw base N: no recount
      if (active) {
        *reinterpret_cast<uint2*>(a.out_base + job.out_off + p0) = make_uint2(ob[0], ob[1]);
        *reinterpret_cast<uint2*>(a.out_qual + job.out_off + p0) = make_uint2(oq[0], oq[1]);
        *reinterpret_cast<uint4*>(a.out_errors + job.out_off + p0) =
            make_uint4(__byte_perm(cnt[0], 0u, 0x4140u), __byte_perm(cnt[0], 0u, 0x4342u),
                       __byte_perm(cnt[1], 0u, 0x4140u), __byte_perm(cnt[1], 0u, 0x4342u));
      }
    } else if (a_any || b_any) {
      // :855-882 single-strand passthrough keeps the FULL length of the surviving strand
      status = a_any ? FGB_DUPLEX_A_ONLY : FGB_DUPLEX_B_ONLY;
      const fgb_unit us = a_any ? ua : ub;
      for (uint32_t i = lane; i < us.cons_len; i += 32) {
        a.out_base[job.out_off + i] = a.ss_base[us.out_off + i];
        a.out_qual[job.out_off + i] = a.ss_qual[us.out_off + i];
        a.out_errors[job.out_off + i] = a.ss_errors[us.out_off + i];
      }
    } else {
      status = FGB_DUPLEX_NONE;
    }
    return status;
  }
  // ---- general path (long reads, unaligned rows, more than 255 pooled source reads) ----
  // :852-853 strands with no coverage inside the truncated region are dropped
  bool a_any = false, b_any = false;
  for (uint32_t i = lane; i < len; i += 32) {
    a_any |= a.ss_depth[ua.out_off + i] > 0;
    b_any |= a.ss_depth[ub.out_off + i] > 0;
  }
  a_any = __any_sync(0xFFFFFFFFu, a_any);
  b_any = __any_sync(0xFFFFFFFFu, b_any);
  if (a_any && b_any) {
    status = FGB_DUPLEX_BOTH;
    if (words) {
      for (uint32_t base0 = 0; base0 < len; base0 += 256u) {
        const uint32_t p0 = base0 + lane * 8u;
        const bool active = p0 < len;
        uint2 ab2 = make_uint2(0, 0), bb2 = ab2, aq2 = ab2, bq2 = ab2;
        if (active) {
          ab2 = *reinterpret_cast<const uint2*>(a.ss_base + ua.out_off + p0);
          bb2 = *reinterpret_cast<const uint2*>(a.ss_base + ub.out_off + p0);
          aq2 = *reinterpret_cast<const uint2*>(a.ss_qual + ua.out_off + p0);
          bq2 = *reinterpret_cast<const uint2*>(a.ss_qual + ub.out_off + p0);
        }
        uint32_t ob[2], oq[2], rawb[2], cnt[2] = {0u, 0u};
        const uint32_t abw[2] = {ab2.x, ab2.y}, bbw[2] = {bb2.x, bb2.y};
        const uint32_t aqw[2] = {aq2.x, aq2.y}, bqw[2] = {bq2.x, bq2.y};
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const uint32_t eq = __vcmpeq4(abw[h], bbw[h]);                    // :912-927, bytewise
          const uint32_t sum = __vminu4(__vaddus4(aqw[h], bqw[h]), 0x5D5D5D5Du);
          const uint32_t dif = __vminu4(__vabsdiffu4(aqw[h], bqw[h]), 0x5D5D5D5Du);
          const uint32_t rq = __vmaxu4((eq & sum) | (~eq & dif), 0x02020202u);   // cap_quality; equal-quality dissent -> 2
          const uint32_t b_wins = ~eq & __vcmpgtu4(bqw[h], aqw[h]);
          rawb[h] = (bbw[h] & b_wins) | (abw[h] & ~b_wins);
          const uint32_t mask = __vcmpeq4(abw[h], 0x4E4E4E4Eu) | __vcmpeq4(bbw[h], 0x4E4E4E4Eu) |
                                __vcmpeq4(rq, 0x02020202u);                 // :930-935
          ob[h] = (0x4E4E4E4Eu & mask) | (rawb[h] & ~mask);
          oq[h] = (0x02020202u & mask) | (rq & ~mask);
        }
        // :943-951 exact error recount against the pooled source reads (AB rows then BA rows)
        // descriptors are fetched 32 at a time, one per lane, and broadcast by shuffle, so the row
        // loads of a chunk are independent of each other (all lanes take part in the shuffles)
        auto recount_word = [&](uint64_t d) {
          const uint32_t rl = static_cast<uint32_t>(d & 0xFFFFu);
          if (active && rl > p0) {
            const uint2 sb = *reinterpret_cast<const uint2*>(a.bases + (d >> 16) + p0);
            const uint32_t cov = rl - p0;                                   // covered positions of this word
            const uint32_t c0 = cov >= 4u ? 0xFFFFFFFFu : ((1u << (8u * cov)) - 1u);
            const uint32_t c1 = cov >= 8u ? 0xFFFFFFFFu : (cov > 4u ? ((1u << (8u * (cov - 4u))) - 1u) : 0u);
            const uint32_t sw[2] = {sb.x, sb.y}, cw[2] = {c0, c1};
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const uint32_t ne = ~__vcmpeq4(sw[h], rawb[h]) & ~__vcmpeq4(sw[h], 0x4E4E4E4Eu) & cw[h];
              cnt[h] += ne & 0x01010101u;
            }
          }
        };
        const uint32_t na = ra1 - ra0, nr = na + (rb1 - rb0);
        for (uint32_t c0 = 0; c0 < nr; c0 += 32u) {
          const uint32_t k = c0 + lane;
          const uint64_t mine = k < nr ? a.reads[k < na ? ra0 + k : rb0 + (k - na)] : 0ull;
          const uint32_t m = nr - c0 < 32u ? nr - c0 : 32u;
#pragma unroll 4
          for (uint32_t r = 0; r < m; ++r) recount_word(__shfl_sync(0xFFFFFFFFu, mine, r));
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) cnt[h] &= ~__vcmpeq4(rawb[h], 0x4E4E4E4Eu);   // raw base N: no recount
        if (active) {
          *reinterpret_cast<uint2*>(a.out_base + job.out_off + p0) = make_uint2(ob[0], ob[1]);
          *reinterpret_cast<uint2*>(a.out_qual + job.out_off + p0) = make_uint2(oq[0], oq[1]);
          *reinterpret_cast<uint4*>(a.out_errors + job.out_off + p0) =
              make_uint4(__byte_perm(cnt[0], 0u, 0x4140u), __byte_perm(cnt[0], 0u, 0x4342u),
                         __byte_perm(cnt[1], 0u, 0x4140u), __byte_perm(cnt[1], 0u, 0x4342u));
        }
      }
    } else {
    for (uint32_t i = lane; i < len; i += 32) {
      uint32_t a_base = a.ss_base[ua.out_off + i], b_base = a.ss_base[ub.out_off + i];
      int32_t a_qual = a.ss_qual[ua.out_off + i], b_qual = a.ss_qual[ub.out_off + i];
      uint32_t raw_base, raw_qual;                               // :912-927
      if (a_base == b_base) { raw_base = a_base; raw_qual = cap_quality(a_qual + b_qual); }
      else if (a_qual > b_qual) { raw_base = a_base; raw_qual = cap_quality(a_qual - b_qual); }
      else if (b_qual > a_qual) { raw_base = b_base; raw_qual = cap_quality(b_qual - a_qual); }
      else { raw_base = a_base; raw_qual = 2u; }
      bool mask = a_base == 'N' || b_base == 'N' || raw_qual == 2u;   // :930-935
      // :943-951 exact error recount against the pooled source reads (AB rows then BA rows)
      int32_t nerr = 0;
      if (raw_base != 'N') {
        for (uint32_t r = ra0; r < ra1; ++r) {
          uint64_t d = a.reads[r];
          if ((d & 0xFFFFu) > i) {
            uint32_t sb = a.bases[(d >> 16) + i];
            nerr += (sb != 'N' && sb != raw_base);
          }
        }
        for (uint32_t r = rb0; r < rb1; ++r) {
          uint64_t d = a.reads[r];
          if ((d & 0xFFFFu) > i) {
            uint32_t sb = a.bases[(d >> 16) + i];
            nerr += (sb != 'N' && sb != raw_base);
          }
        }
      }
      nerr = nerr > 32767 ? 32767 : nerr;
      a.out_base[job.out_off + i] = mask ? 'N' : static_cast<uint8_t>(raw_base);
      a.out_qual[job.out_off + i] = mask ? 2 : static_cast<uint8_t>(raw_qual);
      a.out_errors[job.out_off + i] = static_cast<uint16_t>(nerr);
    }
    }
  } else if (a_any || b_any) {
    // :855-882 single-strand passthrough keeps the FULL length of the surviving strand
    status = a_any ? FGB_DUPLEX_A_ONLY : FGB_DUPLEX_B_ONLY;
    const fgb_unit us = a_any ? ua : ub;
    for (uint32_t i = lane; i < us.cons_len; i += 32) {
      a.out_base[job.out_off + i] = a.ss_base[us.out_off + i];
      a.out_qual[job.out_off + i] = a.ss_qual[us.out_off + i];
      a.out_errors[job.out_off + i] = a.ss_errors[us.out_off + i];
    }
  } else {
    status = FGB_DUPLEX_NONE;
  }
  return status;
}

__global__ void __launch_bounds__(kCombineThreads) duplex_combine_kernel(const DuplexArgs a) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint64_t warp0 = static_cast<uint64_t>(blockIdx.x) * kCombineJobsPerCta + (threadIdx.x >> 5);
  const uint64_t wstride = static_cast<uint64_t>(gridDim.x) * kCombineJobsPerCta;
  uint32_t done = 0;
  DuplexJobRegs nx;
  if (warp0 < a.n_jobs) nx = load_duplex_job(a, warp0);
  for (uint64_t j = warp0; j < a.n_jobs; j += wstride) {
    const DuplexJobRegs cur = nx;
    if (j + wstride < a.n_jobs) nx = load_duplex_job(a, j + wstride);
    const uint8_t status = duplex_job_warp(a, cur, lane);
    if (lane == 0) {
      if (a.out_status) a.out_status[j] = status;
      ++done;
    }
  }
  if (lane == 0 && done) atomicAdd(a.counters + FGB_CTR_COMBINED, static_cast<unsigned long long>(done));
}

// ---- K2, word kernel ---------------------------------------------------------------------------------
// Work item = 8 consecutive positions of one job; a CTA takes kDuplexChunk consecutive jobs and deals their items to
// its threads from one flat index (a 150-base job is 19 items: one job per warp leaves 13 of 32 lanes idle and walks
// the pooled source rows once per warp instead of once per 8 positions of work).  Pass 1 reads the depth words and
// settles each job's arm (:852-882) in shared memory; pass 2 combines the both-strand jobs (:912-951); the rare
// single-strand arms and the layouts the word path does not take are redone by duplex_job_warp.
#ifndef FGB_DUPLEX_CHUNK
#define FGB_DUPLEX_CHUNK 256
#endif
constexpr int kDuplexDescCache = 8;          // row descriptors of a job kept in shared memory (4 + 4 reads per strand fit)
constexpr int kDuplexChunk = FGB_DUPLEX_CHUNK;     // 32, 64, 128 or 256: jobs whose descriptors are fetched in one round
static_assert(kDuplexChunk >= 32 && kDuplexChunk <= kCombineThreads && (kDuplexChunk & (kDuplexChunk - 1)) == 0, "chunk size");

struct DuplexJobSm {
  unsigned long long out_off, a_off, b_off;
  uint32_t len, ra0, na, rb0, nb;
  uint32_t general;       // 1: duplex_job_warp does the whole job
  uint32_t done;          // 1: combined in the vote's epilogue already (duplex_combine_pending_kernel)
  uint32_t pad_;
};

__device__ __forceinline__ uint32_t chunk_job_of(const uint32_t* pref, uint32_t it) {
  uint32_t jl = 0;                        // last job with pref[jl] <= it
#pragma unroll
  for (int step = kDuplexChunk / 2; step > 0; step >>= 1)
    if (pref[jl + step] <= it) jl += step;
  return jl;
}

// `skip_done`: jobs whose status byte is not FGB_DUPLEX_PENDING were combined in the vote kernels' epilogue
// (vote_kernel.cuh duplex_epilogue) and are left alone; a chunk without pending jobs costs one byte load per job.
template <bool SkipDone>
__device__ __forceinline__ void duplex_combine_words_chunk(const DuplexArgs& a, const uint64_t j0, DuplexJobSm* sj,
                                                           uint32_t* s_pref, uint32_t* s_any,
                                                           uint64_t (*s_desc)[kDuplexDescCache]) {
  const uint32_t tid = threadIdx.x, lane = tid & 31u;
  const uint32_t nj = static_cast<uint32_t>(a.n_jobs - j0 < kDuplexChunk ? a.n_jobs - j0 : kDuplexChunk);
  __shared__ uint32_t s_wsum[kDuplexChunk / 32];
  if (tid < kDuplexChunk) {
    uint32_t items = 0;
    bool is_new = false;
    if (tid < nj) {
      DuplexJobSm s;
      s.general = 0u;
      s.done = (SkipDone && a.out_status[j0 + tid] != FGB_DUPLEX_PENDING) ? 1u : 0u;
      if (!s.done) {
        const DuplexJobRegs r = load_duplex_job(a, j0 + tid);
        s.out_off = r.job.out_off; s.a_off = r.ua.out_off; s.b_off = r.ub.out_off;
        s.len = r.ua.cons_len < r.ub.cons_len ? r.ua.cons_len : r.ub.cons_len;       // duplex_caller.rs:846-849
        s.ra0 = r.ua.read_begin; s.na = r.ra1 - r.ua.read_begin;
        s.rb0 = r.ub.read_begin; s.nb = r.rb1 - r.ub.read_begin;
        s.general = (((r.job.out_off | r.ua.out_off | r.ub.out_off) & 7ull) != 0ull ||
                     static_cast<unsigned long long>(s.na) + s.nb > 255ull) ? 1u : 0u;
        items = s.general ? 0u : (s.len + 7u) >> 3;
        if (!s.general) {        // the pooled rows' descriptors (AB rows then BA rows): pass 2 then asks for a word's
          const uint32_t nr = s.na + s.nb;     // SS words and source rows in one round of loads
#pragma unroll
          for (uint32_t k = 0; k < static_cast<uint32_t>(kDuplexDescCache); ++k)
            if (k < nr) s_desc[tid][k] = __ldg(a.reads + (k < s.na ? s.ra0 + k : s.rb0 + (k - s.na)));
        }
      } else {
        s.out_off = s.a_off = s.b_off = 0ull; s.len = s.ra0 = s.na = s.rb0 = s.nb = 0u;
      }
      sj[tid] = s;
      s_any[tid] = 0u;
      is_new = !s.done;
    }
    uint32_t incl = items;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const uint32_t v = __shfl_up_sync(0xFFFFFFFFu, incl, off);
      if (lane >= static_cast<uint32_t>(off)) incl += v;
    }
    s_pref[tid + 1] = incl;                            // within the warp; the warps in front are added below
    if (lane == 31u) s_wsum[tid >> 5] = incl;
    const uint32_t n_new = __popc(__ballot_sync(0xFFFFFFFFu, is_new));
    if (lane == 0 && n_new) atomicAdd(a.counters + FGB_CTR_COMBINED, static_cast<unsigned long long>(n_new));
  }
  __syncthreads();
  if (kDuplexChunk > 32) {
    if (tid >= 32u && tid < kDuplexChunk) {
      uint32_t add = 0;
      for (uint32_t w = 0; w < (tid >> 5); ++w) add += s_wsum[w];
      s_pref[tid + 1] += add;
    }
  }
  if (tid == 0) s_pref[0] = 0u;
  __syncthreads();
  const uint32_t total = s_pref[kDuplexChunk];
  // ---- pass 1: which strands have coverage inside the truncated region (:852-853) ----
  // A strand almost always has depth in its first word: item 0 of every job settles the arm then, and the other
  // depth words are read only for the jobs it leaves open (600 of a 150-base job's 3 016 bytes otherwise).
  bool open_jobs = false;
  if (tid < nj && !sj[tid].general && !sj[tid].done && sj[tid].len > 0u) {
    const uint32_t len = sj[tid].len;
    const uint32_t live = len < 8u ? len : 8u;
    const uint4 ad4 = __ldg(reinterpret_cast<const uint4*>(a.ss_depth + sj[tid].a_off));
    const uint4 bd4 = __ldg(reinterpret_cast<const uint4*>(a.ss_depth + sj[tid].b_off));
    const uint32_t f = (duplex_any_depth(ad4, live) ? 1u : 0u) | (duplex_any_depth(bd4, live) ? 2u : 0u);
    s_any[tid] = f;
    open_jobs = f != 3u && len > 8u;
  }
  if (__syncthreads_or(open_jobs ? 1 : 0)) {
    for (uint32_t it = tid; it < total; it += kCombineThreads) {
      const uint32_t jl = chunk_job_of(s_pref, it);
      const uint32_t p0 = (it - s_pref[jl]) * 8u;
      if (p0 == 0u || s_any[jl] == 3u) continue;
      const uint32_t len = sj[jl].len;
      const uint32_t live = len - p0 < 8u ? len - p0 : 8u;
      const uint4 ad4 = __ldg(reinterpret_cast<const uint4*>(a.ss_depth + sj[jl].a_off + p0));
      const uint4 bd4 = __ldg(reinterpret_cast<const uint4*>(a.ss_depth + sj[jl].b_off + p0));
      const uint32_t f = (duplex_any_depth(ad4, live) ? 1u : 0u) | (duplex_any_depth(bd4, live) ? 2u : 0u);
      if (f & ~s_any[jl]) atomicOr(&s_any[jl], f);
    }
    __syncthreads();
  }
  // ---- pass 2: the both-strand jobs ----
  for (uint32_t it = tid; it < total; it += kCombineThreads) {
    const uint32_t jl = chunk_job_of(s_pref, it);
    if (s_any[jl] != 3u) continue;
    const DuplexJobSm s = sj[jl];
    const uint32_t p0 = (it - s_pref[jl]) * 8u;
    const uint2 ab2 = __ldg(reinterpret_cast<const uint2*>(a.ss_base + s.a_off + p0));
    const uint2 bb2 = __ldg(reinterpret_cast<const uint2*>(a.ss_base + s.b_off + p0));
    const uint2 aq2 = __ldg(reinterpret_cast<const uint2*>(a.ss_qual + s.a_off + p0));
    const uint2 bq2 = __ldg(reinterpret_cast<const uint2*>(a.ss_qual + s.b_off + p0));
    const DuplexWord w = duplex_combine_word(ab2, bb2, aq2, bq2);
    uint32_t cnt[2] = {0u, 0u};
    // :943-951 exact error recount against the pooled source reads (AB rows then BA rows), four rows in flight
    const uint32_t nr = s.na + s.nb;
    for (uint32_t r0 = 0; r0 < nr; r0 += 4u) {
      uint64_t d[4];
      uint2 sb[4];
#pragma unroll
      for (uint32_t k = 0; k < 4u; ++k) {
        const uint32_t r = r0 + k;
        d[k] = r < nr ? (r < static_cast<uint32_t>(kDuplexDescCache)
                             ? s_desc[jl][r] : __ldg(a.reads + (r < s.na ? s.ra0 + r : s.rb0 + (r - s.na)))) : 0ull;
      }
#pragma unroll
      for (uint32_t k = 0; k < 4u; ++k) {
        sb[k] = make_uint2(0x4E4E4E4Eu, 0x4E4E4E4Eu);                   // N: counts nothing
        if (static_cast<uint32_t>(d[k] & 0xFFFFu) > p0) sb[k] = __ldg(reinterpret_cast<const uint2*>(a.bases + (d[k] >> 16) + p0));
      }
#pragma unroll
      for (uint32_t k = 0; k < 4u; ++k) {
        const uint32_t rl = static_cast<uint32_t>(d[k] & 0xFFFFu);
        duplex_recount_row(sb[k], rl > p0 ? rl - p0 : 0u, w.rawb, cnt);     // covered positions of this word
      }
    }
    *reinterpret_cast<uint2*>(a.out_base + s.out_off + p0) = make_uint2(w.ob[0], w.ob[1]);
    *reinterpret_cast<uint2*>(a.out_qual + s.out_off + p0) = make_uint2(w.oq[0], w.oq[1]);
    *reinterpret_cast<uint4*>(a.out_errors + s.out_off + p0) = duplex_errors_word(w.rawb, cnt);
  }
  // ---- the rest: single-strand arms and general layouts, one warp per job ----
  for (uint32_t jl = tid >> 5; jl < nj; jl += kCombineThreads / 32) {
    if (sj[jl].done) continue;
    const uint32_t f = s_any[jl];
    const bool general = sj[jl].general != 0u;
    uint8_t status = f == 3u ? FGB_DUPLEX_BOTH : FGB_DUPLEX_NONE;
    if (general || f == 1u || f == 2u) status = duplex_job_warp(a, load_duplex_job(a, j0 + jl), lane);
    if (lane == 0 && a.out_status) a.out_status[j0 + jl] = status;
  }
}

__global__ void __launch_bounds__(kCombineThreads, 4) duplex_combine_words_kernel(const DuplexArgs a) {
  __shared__ DuplexJobSm sj[kDuplexChunk];
  __shared__ uint32_t s_pref[kDuplexChunk + 1];
  __shared__ uint32_t s_any[kDuplexChunk];
  __shared__ uint64_t s_desc[kDuplexChunk][kDuplexDescCache];
  duplex_combine_words_chunk<false>(a, static_cast<uint64_t>(blockIdx.x) * kDuplexChunk, sj, s_pref, s_any, s_desc);
}

// After a vote with the duplex epilogue: a CTA looks at the status bytes of kCombineThreads jobs (eight chunks) and
// runs the word kernel's body on the chunks that still have pending jobs.
__global__ void __launch_bounds__(kCombineThreads, 4) duplex_combine_pending_kernel(const DuplexArgs a) {
  __shared__ DuplexJobSm sj[kDuplexChunk];
  __shared__ uint32_t s_pref[kDuplexChunk + 1];
  __shared__ uint32_t s_any[kDuplexChunk];
  __shared__ uint64_t s_desc[kDuplexChunk][kDuplexDescCache];
  const uint64_t groups = (a.n_jobs + kCombineThreads - 1) / kCombineThreads;
  for (uint64_t g = blockIdx.x; g < groups; g += gridDim.x) {
    const uint64_t jg = g * kCombineThreads;
    const uint64_t j = jg + threadIdx.x;
    const bool pending = j < a.n_jobs && a.out_status[j] == FGB_DUPLEX_PENDING;
    for (uint32_t c = 0; c < kCombineThreads / kDuplexChunk; ++c) {
      const uint64_t j0 = jg + static_cast<uint64_t>(c) * kDuplexChunk;
      // CTA-uniform verdict on this chunk; the barrier also separates the last chunk's use of sj / s_pref / s_any / s_desc
      const int any = __syncthreads_or(pending && threadIdx.x / kDuplexChunk == c ? 1 : 0);
      if (j0 >= a.n_jobs || !any) continue;
      duplex_combine_words_chunk<true>(a, j0, sj, s_pref, s_any, s_desc);
    }
  }
}

// ---- CODEC ------------------------------------------------------------------------------------
struct CodecArgs {
  const fgb_unit* units;
  const uint8_t* ss_base;
  const uint8_t* ss_qual;
  const uint16_t* ss_depth;
  const uint16_t* ss_errors;
  const fgb_codec_job* jobs;
  uint64_t n_jobs;
  fgb_codec_params cp;
  uint8_t* out_base;
  uint8_t* out_qual;
  uint16_t* out_depth;
  uint16_t* out_errors;
  uint8_t* status;
  uint32_t* disagreements;
  uint32_t* duplex_bases;
  unsigned long long* counters;
};

// fgumi-dna dna.rs:30-40
__device__ __forceinline__ uint32_t complement_base(uint32_t b) {
  switch (b) {
    case 'A': case 'a': return 'T';
    case 'T': case 't': return 'A';
    case 'C': case 'c': return 'G';
    case 'G': case 'g': return 'C';
    default: return b;   // 'N' stays 'N', 'n' stays 'n', anything else unchanged
  }
}

struct SsCol {
  uint32_t base, qual, depth, err;
};

// Column `i` of a single-strand consensus after orientation (reverse_complement_ss) and padding.
__device__ __forceinline__ SsCol padded_column(const CodecArgs& a, const fgb_unit& un, uint32_t i,
                                               uint32_t pad_left, bool rc) {
  SsCol c;
  uint32_t p = i - pad_left;                 // wraps to a huge value when i < pad_left
  if (i >= pad_left && p < un.cons_len) {
    uint32_t s = rc ? un.cons_len - 1u - p : p;
    uint32_t b = a.ss_base[un.out_off + s];
    c.base = rc ? complement_base(b) : b;
    c.qual = a.ss_qual[un.out_off + s];
    c.depth = a.ss_depth[un.out_off + s];
    c.err = a.ss_errors[un.out_off + s];
  } else {                                   // pad_consensus, codec_caller.rs:991-995
    c.base = 'n'; c.qual = 0; c.depth = 0; c.err = 0;
  }
  return c;
}

// One job on one warp, one position per lane and step: the literal restatement of the reference's loops.  It is the
// path for layouts the word kernel below does not take (rows that are not 8-aligned, bases outside A/C/G/T/N/n).
__device__ __forceinline__ void codec_job_scalar(const CodecArgs& a, const fgb_codec_job& job, uint32_t lane,
                                                 uint32_t& n_dup_out, uint32_t& n_dis_out) {
  const fgb_unit ua = a.units[job.unit_a], ub = a.units[job.unit_b];
  const uint32_t len = job.len;
  const uint32_t outer_len = a.cp.outer_bases_length;
  const uint32_t outer_hi = len > outer_len ? len - outer_len : 0u;   // saturating_sub, :1205
  uint32_t n_dup = 0, n_dis = 0;
  for (uint32_t i = lane; i < len; i += 32) {
    SsCol A = padded_column(a, ua, i, job.pad_a_left, job.rc_a != 0);
    SsCol B = padded_column(a, ub, i, job.pad_b_left, job.rc_b != 0);
    const bool a_has = A.base != 'N' && A.base != 'n';           // :1064-1065
    const bool b_has = B.base != 'N' && B.base != 'n';
    uint32_t dbase, dqual, depth, err;
    if (a_has && b_has) {                                        // :1068-1113
      ++n_dup;
      uint32_t raw_base, raw_qual;
      if (A.base == B.base) {
        raw_base = A.base;
        uint32_t s = A.qual + B.qual;
        raw_qual = s > 93u ? 93u : s;
      } else if (A.qual > B.qual) {
        ++n_dis; raw_base = A.base;
        uint32_t d = A.qual - B.qual; raw_qual = d < 2u ? 2u : d;
      } else if (B.qual > A.qual) {
        ++n_dis; raw_base = B.base;
        uint32_t d = B.qual - A.qual; raw_qual = d < 2u ? 2u : d;
      } else {
        ++n_dis; raw_base = A.base; raw_qual = 2u;
      }
      if (raw_qual == 2u) { dbase = 'N'; dqual = 2u; } else { dbase = raw_base; dqual = raw_qual; }
      if (A.base == B.base) err = A.err + B.err;
      else if (A.base == raw_base) err = A.err + (B.depth > B.err ? B.depth - B.err : 0u);
      else err = B.err + (A.depth > A.err ? A.depth - A.err : 0u);
      depth = A.depth + B.depth;
    } else if (a_has) {                                          // :1115-1122
      if (A.qual == 2u) { dbase = 'N'; dqual = 2u; } else { dbase = A.base; dqual = A.qual; }
      depth = A.depth; err = A.err;
    } else if (b_has) {                                          // :1124-1131
      if (B.qual == 2u) { dbase = 'N'; dqual = 2u; } else { dbase = B.base; dqual = B.qual; }
      depth = B.depth; err = B.err;
    } else {                                                     // :1133-1139
      dbase = 'N'; dqual = 2u; depth = 0; err = A.err + B.err;
    }
    if (A.base == 'N' || B.base == 'N') { dbase = 'N'; dqual = 2u; }   // :1145-1149
    // mask_consensus_quals_query_based, :1191-1209
    if ((A.base == 'N' || B.base == 'N') && dbase != 'N') {
      if (a.cp.single_strand_qual >= 0) dqual = static_cast<uint32_t>(a.cp.single_strand_qual);
    }
    if (a.cp.outer_bases_qual >= 0) {
      if (i < outer_len || i >= outer_hi) {
        uint32_t oq = static_cast<uint32_t>(a.cp.outer_bases_qual);
        dqual = dqual < oq ? dqual : oq;
      }
    }
    // final re-orientation, :783-784
    uint32_t oi = job.rc_out ? len - 1u - i : i;
    uint32_t ob = job.rc_out ? complement_base(dbase) : dbase;
    a.out_base[job.out_off + oi] = static_cast<uint8_t>(ob);
    a.out_qual[job.out_off + oi] = static_cast<uint8_t>(dqual);
    a.out_depth[job.out_off + oi] = static_cast<uint16_t>(depth);
    a.out_errors[job.out_off + oi] = static_cast<uint16_t>(err);
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    n_dup += __shfl_xor_sync(0xFFFFFFFFu, n_dup, off);
    n_dis += __shfl_xor_sync(0xFFFFFFFFu, n_dis, off);
  }
  n_dup_out = n_dup;
  n_dis_out = n_dis;
}

// The disagreement gate of one job (:1155-1166) from its two counts.
__device__ __forceinline__ uint8_t codec_gate(const CodecArgs& a, uint32_t n_dup, uint32_t n_dis) {
  uint8_t st = FGB_CODEC_OK;
  if (n_dup > 0) {
    const double rate = static_cast<double>(n_dis) / static_cast<double>(n_dup);
    if (n_dis > a.cp.max_duplex_disagreements) st = FGB_CODEC_HIGH_DISAGREEMENT_COUNT;
    else if (rate > a.cp.max_duplex_disagreement_rate) st = FGB_CODEC_HIGH_DISAGREEMENT_RATE;
  }
  return st;
}

// Fallback kernel: one warp per job, scalar positions (column pointers that are not 16-byte aligned).
__global__ void __launch_bounds__(kCombineThreads) codec_combine_kernel(const CodecArgs a) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint64_t warp0 = static_cast<uint64_t>(blockIdx.x) * kCodecJobsPerCta + (threadIdx.x >> 5);
  const uint64_t wstride = static_cast<uint64_t>(gridDim.x) * kCodecJobsPerCta;
  unsigned long long tot_bases = 0, tot_dis = 0;
  uint32_t done = 0;
  for (uint64_t j = warp0; j < a.n_jobs; j += wstride) {
    const fgb_codec_job job = a.jobs[j];
    uint32_t n_dup, n_dis;
    codec_job_scalar(a, job, lane, n_dup, n_dis);
    if (lane == 0) {
      if (n_dup > 0) { tot_bases += n_dup; tot_dis += n_dis; }
      a.status[j] = codec_gate(a, n_dup, n_dis);
      if (a.disagreements) a.disagreements[j] = n_dis;
      if (a.duplex_bases) a.duplex_bases[j] = n_dup;
      ++done;
    }
  }
  if (lane == 0) {
    if (tot_bases) atomicAdd(a.counters + FGB_CTR_DUPLEX_BASES, tot_bases);
    if (tot_dis) atomicAdd(a.counters + FGB_CTR_DUPLEX_DISAGREE, tot_dis);
    if (done) atomicAdd(a.counters + FGB_CTR_COMBINED, static_cast<unsigned long long>(done));
  }
}

// ---- K3, word kernel ---------------------------------------------------------------------------------
// Work item = 8 consecutive OUTPUT positions of one job; a CTA takes kCodecChunk consecutive jobs and deals their
// items to its threads from one flat index (a 150..300-base job is 19..38 items: dealing whole jobs to warps leaves
// half the lanes idle).  In output coordinates every input strand is a window of 8 consecutive source elements,
// ascending or descending, at an arbitrary offset: orientation (:507-520), padding (:980-1023) and the final
// re-orientation (:783-784) collapse into "fetch the window at a 4-byte-aligned address, funnel-shift, mask what
// lies outside the strand to the pad value, reverse and complement if the strand runs against the output".
// The combine itself (:1029-1152) is byte-parallel on two 32-bit halves (bases, qualities) and four 2 x u16 words
// (depths, errors).  Complementing both strands at once commutes with every comparison the rule makes as long as
// all bases are A/C/G/T/N or the pad 'n'; a job with any other byte is redone by codec_job_scalar.
#ifndef FGB_CODEC_CHUNK
#define FGB_CODEC_CHUNK 256
#endif
constexpr int kCodecChunk = FGB_CODEC_CHUNK;     // 32 .. 256 (power of two): units / jobs whose descriptors are fetched in one round

struct CodecJobSm {
  unsigned long long out_off, a_off, b_off;
  uint32_t len, la, lb;
  int32_t ca, cb;          // source index of output position 0 (ascending: s = c + o; descending: s = c - o)
  uint32_t flags;          // bit 0 strand A descending (= complemented), bit 1 strand B, bit 2 rc_out, bit 3 scalar job
};

__device__ __forceinline__ unsigned long long bytes_below(int n) {     // mask of bytes 0..n-1 of a 64-bit word
  return n <= 0 ? 0ull : (n >= 8 ? ~0ull : ((1ull << (8 * n)) - 1ull));
}

struct Win8 {
  uint32_t b[2], q[2], d[4], e[4];
};

// The window of strand elements that feeds output positions o0 .. o0+7, in output order, pads filled in.
__device__ __forceinline__ Win8 codec_window(const CodecArgs& a, unsigned long long row, uint32_t n, int32_t c,
                                             bool desc, uint32_t o0) {
  Win8 w;
  const int lo = desc ? c - static_cast<int>(o0) - 7 : c + static_cast<int>(o0);
  uint32_t xb[3] = {0u, 0u, 0u}, xq[3] = {0u, 0u, 0u}, yd[5] = {0u, 0u, 0u, 0u, 0u}, ye[5] = {0u, 0u, 0u, 0u, 0u};
  const bool hit = lo < static_cast<int>(n) && lo + 8 > 0;
  if (hit) {
    const uint32_t* rb = reinterpret_cast<const uint32_t*>(a.ss_base + row);
    const uint32_t* rq = reinterpret_cast<const uint32_t*>(a.ss_qual + row);
    const uint32_t* rd = reinterpret_cast<const uint32_t*>(a.ss_depth + row);
    const uint32_t* re = reinterpret_cast<const uint32_t*>(a.ss_errors + row);
    const int w8 = lo >> 2, n8 = static_cast<int>((n + 3u) >> 2);
    const int w16 = lo >> 1, n16 = static_cast<int>((n + 1u) >> 1);
#pragma unroll
    for (int k = 0; k < 3; ++k)
      if (static_cast<unsigned>(w8 + k) < static_cast<unsigned>(n8)) { xb[k] = __ldg(rb + w8 + k); xq[k] = __ldg(rq + w8 + k); }
#pragma unroll
    for (int k = 0; k < 5; ++k)
      if (static_cast<unsigned>(w16 + k) < static_cast<unsigned>(n16)) { yd[k] = __ldg(rd + w16 + k); ye[k] = __ldg(re + w16 + k); }
  }
  const uint32_t s8 = (static_cast<uint32_t>(lo) & 3u) * 8u, s16 = (static_cast<uint32_t>(lo) & 1u) * 16u;
  // valid window bytes: source index lo + k inside [0, n)
  const unsigned long long m = hit ? (bytes_below(static_cast<int>(n) - lo) & ~bytes_below(-lo)) : 0ull;
  const uint32_t m0 = static_cast<uint32_t>(m), m1 = static_cast<uint32_t>(m >> 32);
  uint32_t b0 = (__funnelshift_r(xb[0], xb[1], s8) & m0) | (0x6E6E6E6Eu & ~m0);      // pad_consensus: 'n', Q0, 0, 0
  uint32_t b1 = (__funnelshift_r(xb[1], xb[2], s8) & m1) | (0x6E6E6E6Eu & ~m1);
  uint32_t q0 = __funnelshift_r(xq[0], xq[1], s8) & m0;
  uint32_t q1 = __funnelshift_r(xq[1], xq[2], s8) & m1;
  const uint32_t mm[4] = {__byte_perm(m0, 0u, 0x1100u), __byte_perm(m0, 0u, 0x3322u),
                          __byte_perm(m1, 0u, 0x1100u), __byte_perm(m1, 0u, 0x3322u)};
  uint32_t d[4], e[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    d[k] = __funnelshift_r(yd[k], yd[k + 1], s16) & mm[k];
    e[k] = __funnelshift_r(ye[k], ye[k + 1], s16) & mm[k];
  }
  // descending strands: reverse the eight elements (and complement the bases, reverse_complement_ss)
  const uint32_t sa = desc ? 0x4567u : 0x3210u, sb = desc ? 0x0123u : 0x7654u, sh = desc ? 0x5476u : 0x3210u;
  w.b[0] = __byte_perm(b0, b1, sa); w.b[1] = __byte_perm(b0, b1, sb);
  w.q[0] = __byte_perm(q0, q1, sa); w.q[1] = __byte_perm(q0, q1, sb);
  w.d[0] = __byte_perm(d[0], d[3], sh); w.d[1] = __byte_perm(d[1], d[2], sh);
  w.d[2] = __byte_perm(d[2], d[1], sh); w.d[3] = __byte_perm(d[3], d[0], sh);
  w.e[0] = __byte_perm(e[0], e[3], sh); w.e[1] = __byte_perm(e[1], e[2], sh);
  w.e[2] = __byte_perm(e[2], e[1], sh); w.e[3] = __byte_perm(e[3], e[0], sh);
  return w;
}

__global__ void __launch_bounds__(kCombineThreads) codec_combine_words_kernel(const CodecArgs a) {
  __shared__ CodecJobSm sj[kCodecChunk];
  __shared__ uint32_t s_pref[kCodecChunk + 1];
  __shared__ uint32_t s_dup[kCodecChunk], s_dis[kCodecChunk], s_redo[kCodecChunk];
  const uint32_t tid = threadIdx.x, lane = tid & 31u;
  const uint64_t j0 = static_cast<uint64_t>(blockIdx.x) * kCodecChunk;
  const uint32_t nj = static_cast<uint32_t>(a.n_jobs - j0 < kCodecChunk ? a.n_jobs - j0 : kCodecChunk);
  __shared__ uint32_t s_wsum[kCodecChunk / 32];
  if (tid < static_cast<uint32_t>(kCodecChunk)) {
    uint32_t items = 0;
    if (tid < nj) {
      const fgb_codec_job job = a.jobs[j0 + tid];
      const fgb_unit ua = a.units[job.unit_a], ub = a.units[job.unit_b];
      CodecJobSm s;
      s.out_off = job.out_off; s.a_off = ua.out_off; s.b_off = ub.out_off;
      s.len = job.len; s.la = ua.cons_len; s.lb = ub.cons_len;
      const bool ro = job.rc_out != 0, ra = job.rc_a != 0, rb = job.rc_b != 0;
      const int len = static_cast<int>(job.len), la = static_cast<int>(ua.cons_len), lb = static_cast<int>(ub.cons_len);
      const int pa = static_cast<int>(job.pad_a_left), pb = static_cast<int>(job.pad_b_left);
      // output position o -> padded column i = ro ? len-1-o : o -> strand position p = i - pad -> source s = rc ? l-1-p : p
      s.ca = ro ? (ra ? la - len + pa : len - 1 - pa) : (ra ? la - 1 + pa : -pa);
      s.cb = ro ? (rb ? lb - len + pb : len - 1 - pb) : (rb ? lb - 1 + pb : -pb);
      const bool scalar = ((job.out_off | ua.out_off | ub.out_off) & 7ull) != 0ull || job.len > 0x10000000u ||
                          ua.cons_len > 0x10000000u || ub.cons_len > 0x10000000u ||
                          job.pad_a_left > 0x10000000u || job.pad_b_left > 0x10000000u;
      s.flags = (ra != ro ? 1u : 0u) | (rb != ro ? 2u : 0u) | (ro ? 4u : 0u) | (scalar ? 8u : 0u);
      sj[tid] = s;
      items = scalar ? 0u : (job.len + 7u) >> 3;
      s_dup[tid] = 0u; s_dis[tid] = 0u; s_redo[tid] = scalar ? 1u : 0u;
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
  if (kCodecChunk > 32 && tid >= 32u && tid < static_cast<uint32_t>(kCodecChunk)) {
    uint32_t add = 0;
    for (uint32_t w = 0; w < (tid >> 5); ++w) add += s_wsum[w];
    s_pref[tid + 1] += add;
  }
  if (tid == 0) s_pref[0] = 0u;
  __syncthreads();
  const uint32_t total = s_pref[kCodecChunk];
  const int32_t oqual = a.cp.outer_bases_qual;
  for (uint32_t it = tid; it < total; it += kCombineThreads) {
    uint32_t jl = 0;                      // last job with s_pref[jl] <= it
#pragma unroll
    for (int step = kCodecChunk / 2; step > 0; step >>= 1)
      if (s_pref[jl + step] <= it) jl += step;
    const CodecJobSm s = sj[jl];
    const uint32_t o0 = (it - s_pref[jl]) * 8u;
    const uint32_t live = s.len - o0 < 8u ? s.len - o0 : 8u;
    const unsigned long long lm = bytes_below(static_cast<int>(live));
    const uint32_t lmh[2] = {static_cast<uint32_t>(lm), static_cast<uint32_t>(lm >> 32)};
    Win8 A = codec_window(a, s.a_off, s.la, s.ca, (s.flags & 1u) != 0u, o0);
    Win8 B = codec_window(a, s.b_off, s.lb, s.cb, (s.flags & 2u) != 0u, o0);
    const uint32_t ca_on = (s.flags & 1u) ? 0xFFFFFFFFu : 0u, cb_on = (s.flags & 2u) ? 0xFFFFFFFFu : 0u;
    uint32_t ob[2], oq[2], od[4], oe[4];
    uint32_t unknown = 0u, n_dup = 0u, n_dis = 0u;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      uint32_t ab = A.b[h], bb = B.b[h];
      const uint32_t aq = A.q[h], bq = B.q[h];
      // base classes; complement_base (dna.rs:30-40) on A/C/G/T is an XOR: A^T = 0x15, C^G = 0x04
      const uint32_t a_at = __vcmpeq4(ab, 0x41414141u) | __vcmpeq4(ab, 0x54545454u);
      const uint32_t a_cg = __vcmpeq4(ab, 0x43434343u) | __vcmpeq4(ab, 0x47474747u);
      const uint32_t a_N = __vcmpeq4(ab, 0x4E4E4E4Eu), a_n = __vcmpeq4(ab, 0x6E6E6E6Eu);
      const uint32_t b_at = __vcmpeq4(bb, 0x41414141u) | __vcmpeq4(bb, 0x54545454u);
      const uint32_t b_cg = __vcmpeq4(bb, 0x43434343u) | __vcmpeq4(bb, 0x47474747u);
      const uint32_t b_N = __vcmpeq4(bb, 0x4E4E4E4Eu), b_n = __vcmpeq4(bb, 0x6E6E6E6Eu);
      unknown |= ~(a_at | a_cg | a_N | a_n) | ~(b_at | b_cg | b_N | b_n);
      ab ^= ca_on & ((a_at & 0x15151515u) | (a_cg & 0x04040404u));
      bb ^= cb_on & ((b_at & 0x15151515u) | (b_cg & 0x04040404u));
      const uint32_t a_has = a_at | a_cg, b_has = b_at | b_cg;       // :1064-1065 (given the known classes)
      const uint32_t both = a_has & b_has;
      const uint32_t eqb = __vcmpeq4(ab, bb);
      const uint32_t sum = __vminu4(__vaddus4(aq, bq), 0x5D5D5D5Du);               // :1072-1074
      const uint32_t dif = __vmaxu4(__vabsdiffu4(aq, bq), 0x02020202u);            // :1075-1095
      const uint32_t rq = (eqb & sum) | (~eqb & dif);
      const uint32_t b_wins = ~eqb & __vcmpgtu4(bq, aq);
      const uint32_t raw_base = (bb & b_wins) | (ab & ~b_wins);
      const uint32_t a_only = a_has & ~b_has, b_only = b_has & ~a_has, none = ~(a_has | b_has);
      const uint32_t sq = (both & rq) | (a_only & aq) | (b_only & bq) | (none & 0x02020202u);
      const uint32_t sb = (both & raw_base) | (a_only & ab) | (b_only & bb);
      // :1098-1103, :1115-1139 quality 2 -> N; :1145-1149 an upper-case N on either strand -> (N, 2)
      const uint32_t eitherN = a_N | b_N;
      const uint32_t toN = __vcmpeq4(sq, 0x02020202u) | eitherN | none;
      ob[h] = (0x4E4E4E4Eu & toN) | (sb & ~toN);
      oq[h] = (0x02020202u & eitherN) | (sq & ~eitherN);
      // (mask_consensus_quals_query_based's single-strand rule, :1196-1201, needs an upper-case N on a strand AND a
      //  called base: after :1145-1149 that never holds, so single_strand_qual has no effect -- as in the reference)
      const uint32_t dis = both & ~eqb;
      n_dup += __popc(both & lmh[h] & 0x01010101u);
      n_dis += __popc(dis & lmh[h] & 0x01010101u);
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const uint32_t sel = k ? 0x3322u : 0x1100u;
        const int w = 2 * h + k;
        const uint32_t ah = __byte_perm(a_has, 0u, sel), bh = __byte_perm(b_has, 0u, sel);
        const uint32_t dz = __byte_perm(dis, 0u, sel), bw = __byte_perm(b_wins, 0u, sel);
        const uint32_t ea = A.e[w], eb = B.e[w], da = A.d[w], db = B.d[w];
        const uint32_t simple = __vadd2(ea & (ah | ~bh), eb & (bh | ~ah));          // agree / single strand / neither
        const uint32_t ta = __vadd2(ea, __vsubus2(db, eb));                         // A chosen: :1108
        const uint32_t tb = __vadd2(eb, __vsubus2(da, ea));                         // B chosen: :1111
        oe[w] = (dz & ((bw & tb) | (~bw & ta))) | (~dz & simple);
        od[w] = __vadd2(da & ah, db & bh);
      }
    }
    if (((unknown & lmh[0]) | (unknown & lmh[1])) != 0u) s_redo[jl] = 1u;
    if (oqual >= 0) {                                                // outer bases, :1203-1208, in padded coordinates
      const uint32_t olen = a.cp.outer_bases_length;
      const uint32_t ohi = s.len > olen ? s.len - olen : 0u;
      const uint32_t i_lo = (s.flags & 4u) ? s.len - o0 - live : o0;     // padded columns of this word: [i_lo, i_lo + live)
      if (i_lo < olen || i_lo + live > ohi) {
        const uint32_t cap = static_cast<uint32_t>(oqual) & 0xFFu;
        uint32_t cm[2] = {0u, 0u};
        for (uint32_t k = 0; k < live; ++k) {
          const uint32_t i = (s.flags & 4u) ? s.len - 1u - (o0 + k) : o0 + k;
          if (i < olen || i >= ohi) cm[k >> 2] |= 0xFFu << (8u * (k & 3u));
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) oq[h] = (__vminu4(oq[h], cap * 0x01010101u) & cm[h]) | (oq[h] & ~cm[h]);
      }
    }
    if (n_dup) atomicAdd(&s_dup[jl], n_dup);
    if (n_dis) atomicAdd(&s_dis[jl], n_dis);
    const unsigned long long o = s.out_off + o0;
    if (live == 8u) {
      *reinterpret_cast<uint2*>(a.out_base + o) = make_uint2(ob[0], ob[1]);
      *reinterpret_cast<uint2*>(a.out_qual + o) = make_uint2(oq[0], oq[1]);
      *reinterpret_cast<uint4*>(a.out_depth + o) = make_uint4(od[0], od[1], od[2], od[3]);
      *reinterpret_cast<uint4*>(a.out_errors + o) = make_uint4(oe[0], oe[1], oe[2], oe[3]);
    } else {
      for (uint32_t k = 0; k < live; ++k) {
        a.out_base[o + k] = static_cast<uint8_t>(ob[k >> 2] >> (8u * (k & 3u)));
        a.out_qual[o + k] = static_cast<uint8_t>(oq[k >> 2] >> (8u * (k & 3u)));
        a.out_depth[o + k] = static_cast<uint16_t>(od[k >> 1] >> (16u * (k & 1u)));
        a.out_errors[o + k] = static_cast<uint16_t>(oe[k >> 1] >> (16u * (k & 1u)));
      }
    }
  }
  __syncthreads();
  // jobs the word path could not take: one warp per job, scalar positions (rewrites the job's rows and counts)
  for (uint32_t jl = tid >> 5; jl < nj; jl += kCombineThreads / 32) {
    if (s_redo[jl]) {
      uint32_t n_dup, n_dis;
      codec_job_scalar(a, a.jobs[j0 + jl], lane, n_dup, n_dis);
      if (lane == 0) { s_dup[jl] = n_dup; s_dis[jl] = n_dis; }
    }
  }
  __syncthreads();
  if (tid < static_cast<uint32_t>(kCodecChunk)) {
    unsigned long long tb = 0, td = 0;
    if (tid < nj) {
      const uint32_t n_dup = s_dup[tid], n_dis = s_dis[tid];
      a.status[j0 + tid] = codec_gate(a, n_dup, n_dis);
      if (a.disagreements) a.disagreements[j0 + tid] = n_dis;
      if (a.duplex_bases) a.duplex_bases[j0 + tid] = n_dup;
      if (n_dup) { tb = n_dup; td = n_dis; }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      tb += __shfl_xor_sync(0xFFFFFFFFu, tb, off);
      td += __shfl_xor_sync(0xFFFFFFFFu, td, off);
    }
    if (lane == 0) {                         // one warp per 32 jobs of the chunk
      if (tb) atomicAdd(a.counters + FGB_CTR_DUPLEX_BASES, tb);
      if (td) atomicAdd(a.counters + FGB_CTR_DUPLEX_DISAGREE, td);
      if (tid == 0) atomicAdd(a.counters + FGB_CTR_COMBINED, static_cast<unsigned long long>(nj));
    }
  }
}

}  // namespace fgb
