// The duplex strand combine on one 8-position word, shared by the standalone word kernel (combine_kernels.cuh) and the
// vote kernels' duplex epilogue (vote_kernel.cuh).  Pure byte-parallel integer work.
//
// Replaces (reference = fgumi 0.2.0, crates/fgumi-consensus/src/duplex_caller.rs):
//   :912-927  agreement / disagreement rule (sum capped at 93; higher quality wins with the difference; equal -> Q2)
//   :930-935  N propagation and the Q2 mask
//   :943-951  exact error recount against the pooled source reads (is_error, :797-800)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace fgb {

struct DuplexWord {
  uint32_t ob[2], oq[2];     // final bases / qualities, positions 0-3 and 4-7
  uint32_t rawb[2];          // raw consensus bases (what the recount compares against)
};

__device__ __forceinline__ DuplexWord duplex_combine_word(const uint2 ab2, const uint2 bb2, const uint2 aq2,
                                                          const uint2 bq2) {
  DuplexWord r;
  const uint32_t abw[2] = {ab2.x, ab2.y}, bbw[2] = {bb2.x, bb2.y};
  const uint32_t aqw[2] = {aq2.x, aq2.y}, bqw[2] = {bq2.x, bq2.y};
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const uint32_t eq = __vcmpeq4(abw[h], bbw[h]);                    // :912-927, bytewise
    const uint32_t sum = __vminu4(__vaddus4(aqw[h], bqw[h]), 0x5D5D5D5Du);
    const uint32_t dif = __vminu4(__vabsdiffu4(aqw[h], bqw[h]), 0x5D5D5D5Du);
    const uint32_t rq = __vmaxu4((eq & sum) | (~eq & dif), 0x02020202u);   // cap_quality; equal-quality dissent -> 2
    const uint32_t b_wins = ~eq & __vcmpgtu4(bqw[h], aqw[h]);
    r.rawb[h] = (bbw[h] & b_wins) | (abw[h] & ~b_wins);
    const uint32_t mask = __vcmpeq4(abw[h], 0x4E4E4E4Eu) | __vcmpeq4(bbw[h], 0x4E4E4E4Eu) |
                          __vcmpeq4(rq, 0x02020202u);                 // :930-935
    r.ob[h] = (0x4E4E4E4Eu & mask) | (r.rawb[h] & ~mask);
    r.oq[h] = (0x02020202u & mask) | (rq & ~mask);
  }
  return r;
}

// One source row's word against the raw bases: `cov` = positions of this word the row covers (0..8, more = 8).
__device__ __forceinline__ void duplex_recount_row(const uint2 sb, const uint32_t cov, const uint32_t (&rawb)[2],
                                                   uint32_t (&cnt)[2]) {
  const uint32_t c0 = cov >= 4u ? 0xFFFFFFFFu : ((1u << (8u * cov)) - 1u);
  const uint32_t c1 = cov >= 8u ? 0xFFFFFFFFu : (cov > 4u ? ((1u << (8u * (cov - 4u))) - 1u) : 0u);
  const uint32_t sw[2] = {sb.x, sb.y}, cw[2] = {c0, c1};
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const uint32_t ne = ~__vcmpeq4(sw[h], rawb[h]) & ~__vcmpeq4(sw[h], 0x4E4E4E4Eu) & cw[h];
    cnt[h] += ne & 0x01010101u;
  }
}

// Byte counters -> the eight u16 error counts of the word (a raw base of N counts nothing).
__device__ __forceinline__ uint4 duplex_errors_word(const uint32_t (&rawb)[2], uint32_t (&cnt)[2]) {
#pragma unroll
  for (int h = 0; h < 2; ++h) cnt[h] &= ~__vcmpeq4(rawb[h], 0x4E4E4E4Eu);
  return make_uint4(__byte_perm(cnt[0], 0u, 0x4140u), __byte_perm(cnt[0], 0u, 0x4342u),
                    __byte_perm(cnt[1], 0u, 0x4140u), __byte_perm(cnt[1], 0u, 0x4342u));
}

// Any non-zero depth among the first `live` (1..8) of eight u16 depths (a longer strand has real depths behind the
// truncated length: the last word is masked).  duplex_caller.rs:852-853.
__device__ __forceinline__ bool duplex_any_depth(const uint4& d, const uint32_t live) {
  const uint32_t w[4] = {d.x, d.y, d.z, d.w};
  uint32_t acc = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const uint32_t keep = live >= 2u * k + 2u ? 0xFFFFFFFFu : (live == 2u * k + 1u ? 0x0000FFFFu : 0u);
    acc |= w[k] & keep;
  }
  return acc != 0u;
}

}  // namespace fgb
