// K1 — simplex / single-strand consensus vote for sm_90a.
//
// Replaces (reference = fgumi 0.2.0, crates/fgumi-consensus/src/):
//   vanilla_caller.rs:1260-1358  create_consensus_from_source_reads (position loop, thresholds,
//                                single-read LUT path)
//   base_builder.rs:295-327      ConsensusBaseBuilder::add   (4-lane f64 Kahan likelihoods)
//   base_builder.rs:338-379      try_unanimous_fast_path
//   base_builder.rs:391-458      call (log-sum-exp, argmax / tie -> N, posterior -> phred)
//
// Shape of the kernel (DESIGN.md §3):
//   * persistent CTAs (2 per SM), each walks tiles  t = blockIdx.x, +gridDim.x, ...
//   * warp-specialised: one PRODUCER warp stages tiles (base bytes, qual bytes, read descriptors,
//     unit descriptors) into shared memory with four TMA bulk copies (cp.async.bulk ... mbarrier
//     complete_tx) as soon as a stage's "empty" mbarrier says all eight CONSUMER warps are done
//     with it; consumers never meet at a CTA barrier, so a warp that finishes its share of a tile
//     moves straight on to the next one while HBM streams into the other stage;
//   * FAST PASS: one thread per 8 consecutive positions (one 64-bit word of each row).  Over the depth axis it
//     keeps a SWAR "all reads equal the first read" mask and a SWAR "every quality >= qT(n)" mask;
//     a position that is unanimous over A/C/G/T, covered by every read and passes the quality
//     mask is PROVEN to take the reference's unanimous fast path (sum of per-read likelihood gaps
//     >= n*Dmono[qT] > 23), whose result is the constant (base, phred(ln_pre)) — no f64 needed;
//   * everything else (disagreements, Ns, ragged ends, shallow / low-quality pileups) goes to a
//     warp-private queue in shared memory and is resolved, packed one position per lane, first by
//     the integer "dominant winner" proof (host_tables.cpp) and only then by the literal algorithm:
//     sequential, in-order, 4-lane f64 Kahan accumulation from the host-built tables and the f64
//     call() tail;
//   * results leave as coalesced 8-byte (bases, quals) and 16-byte (depths, errors) stores.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/fgumi_b200.h"
#include "device_math.cuh"
#include "duplex_word.cuh"
#include "fgb_config.h"
#include "host_tables.h"
#include "swar.cuh"

namespace fgb {

struct DeviceTables {
  double correct[FGB_NTABLE];   // adjusted_correct_table, base_builder.rs:265
  double err_alt[FGB_NTABLE];   // adjusted_error_per_alt, base_builder.rs:268
  double ln_pre;                // ln_error_pre_umi, base_builder.rs:277
  uint8_t single_q[96];         // single_input_consensus_quals, vanilla_caller.rs:463-482
  uint8_t qt[kQtEntries];       // fast-path quality threshold by depth; 255 = never
  int32_t dfix[96];             // fixed-point likelihood gaps (host_tables.cpp), INT32_MIN = unusable
  int32_t g2fix;                // dominant-winner threshold, fixed point
  uint32_t nmax2;               // dominant-winner proof valid up to this many observations
  uint8_t pair_q[94 * 94];      // unanimous two-read pileups: quality by (q1, q2); 255 = literal path
  uint16_t sumt[8];             // sum-of-qualities thresholds by depth (host_tables.cpp), 0xFFFF = none
  uint8_t qt3[kQtEntries];      // near-unanimous quality threshold by depth (deep kernel); 255 = never
  int32_t ugap_bp[128];         // unanimous pileups: quality steps by fixed-point gap (host_tables.h ugap_*)
  uint8_t ugap_q[128];
};

struct VoteArgs {
  const uint8_t* bases;
  const uint8_t* quals;
  const uint64_t* reads;
  const fgb_unit* units;
  const fgb_tile* tiles;
  uint64_t n_tiles;
  uint8_t* out_base;
  uint8_t* out_qual;
  uint16_t* out_depth;
  uint16_t* out_errors;
  const DeviceTables* tables;
  unsigned long long* counters;
  uint32_t min_reads;
  uint32_t min_cons_q;
  uint32_t fast_qual;   // ln_prob_to_phred(ln_pre), host-evaluated (base_builder.rs:370)
};

// The kernels with the duplex epilogue (vote_kernel*_duplex, fgb_vote_duplex_device) take these on top.  (A separate
// struct: ptxas' register allocation of the plain kernels is sensitive to the parameter block.)
struct VoteArgsDuplex : VoteArgs {
  const fgb_tile_jobs* tile_jobs;     // per tile of this launch
  const uint32_t* job_index;
  const fgb_duplex_job* djobs;
  uint8_t* d_base;
  uint8_t* d_qual;
  uint16_t* d_errors;
  uint8_t* d_status;                  // preset to FGB_DUPLEX_PENDING; the epilogue writes FGB_DUPLEX_BOTH
};

struct __align__(16) Stage {
  uint8_t bases[kTileCapBytes];
  uint8_t quals[kTileCapBytes];
  uint64_t reads[kTileMaxReads + 2];
  fgb_unit units[kTileMaxUnits + 1];
  fgb_tile tile;
  uint32_t aux[4];   // written by the producer: [0] = 2^32 / items-per-unit + 1 (uniform tiles), [1] = items
};

struct __align__(128) VoteSmem {
  Stage st[kStages];
  double correct[FGB_NTABLE];
  double err_alt[FGB_NTABLE];
  double ln_pre;
  uint64_t full[kStages];
  uint64_t empty[kStages];
  uint32_t queue[kConsumerWarps][kWarpQueueCap];
  uint32_t q_count[kConsumerWarps];
  uint8_t single_q[96];
  uint8_t qt[kQtEntries];
  uint8_t qt3[kQtEntries];
  int32_t dfix[96];
  int32_t g2fix;
  uint32_t nmax2;
  const uint8_t* pair_q;        // DeviceTables::pair_q (global memory, L1-resident)
};

constexpr uint32_t kPairSmemBytes = 94u * 94u;                 // 8836 = 4 * 2209
constexpr uint32_t kUgapSmemOff = (kPairSmemBytes + 15u) & ~15u;   // the unanimous-gap steps follow the pair table
constexpr uint32_t kShallowSmemBytes = kUgapSmemOff + 128u * 4u + 128u;
static_assert(kPairSmemBytes % 4u == 0, "pair table is copied as words");
static_assert(sizeof(VoteSmem) % 16u == 0, "the pair table follows VoteSmem in dynamic shared memory");

// ---- PTX wrappers ------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Blocks until the phase with the given parity completes.  `hint_ns` lets the hardware park the
// thread between probes instead of spinning through issue slots.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, uint32_t hint_ns) {
  uint32_t addr = smem_u32(bar);
  uint32_t done;
  do {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(done)
        : "r"(addr), "r"(parity), "r"(hint_ns)
        : "memory");
  } while (!done);
}
// Non-blocking probe of a phase.
__device__ __forceinline__ bool mbar_test(uint64_t* bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(done)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return done != 0;
}
// TMA 1-D bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP).
__device__ __forceinline__ void tma_load_1d(void* dst, const void* src, uint32_t bytes,
                                            uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
          "r"(smem_u32(dst)),
      "l"(src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// ---- diagnostic builds only (scripts/pipe_trace.py) ----------------------------------------------
// FGB_PIPE_TRACE: clock64 stall breakdown of the stage pipeline, summed over the grid into g_pipe_trace
// (fgb_pipe_trace reads it back).  FGB_PIPE_NOVOTE: the consumers store constant words for their items instead of
// voting -- producer, stage ring and stores unchanged: the kernel's data movement alone.
#ifndef FGB_PIPE_TRACE
#define FGB_PIPE_TRACE 0
#endif
#ifndef FGB_PIPE_NOVOTE
#define FGB_PIPE_NOVOTE 0
#endif
#if FGB_PIPE_TRACE
// [0] CTA cycles (producer lane, prologue to last issue)  [1] producer cycles waiting on `empty`
// [2] consumer-warp cycles  [3] consumer cycles waiting on `full`  [4] voting cycles  [5] fast pass  [6] slow pass
// [7] tiles whose copy had not landed when warp 0 arrived  [8] their issue -> full cycles  [9] tiles  [10] CTAs
constexpr int kPipeTraceWords = 16;
__device__ unsigned long long g_pipe_trace[kPipeTraceWords];
__shared__ long long g_trace_mark[kConsumerWarps];   // per warp: end of the fast pass of the current tile
#endif

// ---- memory-space policy: tiles live in shared memory, oversize units are read from HBM -------
struct ShMem {
  // Plain pointers derived from the extern __shared__ block: nvcc's address-space inference turns
  // these into LDS and is free to batch the independent loads of an unrolled depth loop.
  using addr_t = const uint8_t*;
  using off_t = uint32_t;
  static __device__ __forceinline__ uint32_t ld8(addr_t a) { return *a; }
  static __device__ __forceinline__ uint32_t ld32(addr_t a) {
    return *reinterpret_cast<const uint32_t*>(a);
  }
  static __device__ __forceinline__ uint64_t ld64(addr_t a) {
    return *reinterpret_cast<const uint64_t*>(a);
  }
  // tile-relative byte offset of a read row: 32-bit arithmetic is enough inside a stage
  static __device__ __forceinline__ off_t row_offset(uint64_t d, uint64_t, uint32_t base32) {
    return static_cast<uint32_t>(d >> 16) - base32;
  }
};
struct GlMem {
  using addr_t = const uint8_t*;
  using off_t = uint64_t;
  static __device__ __forceinline__ uint32_t ld8(addr_t a) { return __ldg(a); }
  static __device__ __forceinline__ uint32_t ld32(addr_t a) {
    return __ldg(reinterpret_cast<const uint32_t*>(a));
  }
  static __device__ __forceinline__ uint64_t ld64(addr_t a) {
    return __ldg(reinterpret_cast<const unsigned long long*>(a));
  }
  static __device__ __forceinline__ off_t row_offset(uint64_t d, uint64_t byte_base, uint32_t) {
    return (d >> 16) - byte_base;
  }
};

template <class M>
struct TileView {
  typename M::addr_t bases;   // address of byte `byte_base` of the base column
  typename M::addr_t quals;
  typename M::addr_t reads;   // address of the descriptor of read `read_base`
  uint64_t byte_base;
  uint32_t read_base;
};

__device__ __forceinline__ bool is_acgt_upper(uint32_t b) {
  // 'A'=65 'C'=67 'G'=71 'T'=84 -> bits 1,3,7,20 of a mask indexed by b-64
  uint32_t t = b - 64u;
  return t < 32u && ((0x0010008Au >> t) & 1u);
}
// BASE_TO_INDEX, base_builder.rs:204-215 (case-insensitive A,C,G,T -> 0..3, else 4)
// Branch-free: a compare chain here becomes data-dependent branches, and lanes that split on the
// base do not reconverge before the end of the out-of-line resolver.
__device__ __forceinline__ uint32_t base_to_index(uint32_t b) {
  const uint32_t u = b & 0xDFu;
  const uint32_t x = (u >> 1) & 3u;            // A 0, C 1, T 2, G 3
  return is_acgt_upper(u) ? (x ^ (x >> 1)) : 4u;
}

struct Called {
  uint32_t base, qual, depth, errors;
};

// Certified single-precision evaluation of the call() tail (base_builder.rs:433-457) for a position
// with a unique winner.  With d_b = ll[b] - ll[w] (exact f64 differences, then rounded to f32) the
// posterior error is s / (1 + s), s = sum_b e^(d_b): every term is positive, so there is no
// cancellation and OUR value of s carries < 1e-4 relative error (argument rounding, exp/log
// approximation).  The REFERENCE's value does not: it forms ln_sum by folding `x + exp(-x)` terms
// (phred.rs:148-158, 307-330) and subtracts, which leaves an absolute rounding noise of a few
// ulp(max |ll|) on s -- negligible for s >= 1e-9, a percent at s ~ 1e-12 (reachable with a pre-UMI
// error rate near Q93).  So the tail is evaluated at both ends of the interval that contains the
// reference's s, and the result is accepted only if both ends take the same branch of
// ln_error_prob_two_trials (its `p1 - p2 >= 6` shortcut, phred.rs:238, is a discontinuity) and floor
// to the same quality (phred.rs:126) with 2e-3 phred to spare.  Anything else -- and any non-finite
// likelihood -- is left to the literal f64 tail, which replays the reference's operations exactly.
__device__ __forceinline__ bool tail_phred(float err, float lp, float* x, int* branch) {
  const float p1 = fmaxf(lp, err), p2 = fminf(lp, err);
  const float diff = p1 - p2;
  if (!(fabsf(diff - 6.0f) > 2.0e-3f)) return false;      // too close to the shortcut (or NaN)
  float fin;
  if (diff >= 6.0f) {
    if (p1 == lp) { *branch = 0; *x = 0.0f; return true; }   // ln_pre passes through: phred(ln_pre)
    *branch = 1; fin = err;
  } else {
    *branch = 2; fin = p1 + log1pf(__expf(p2 - p1) - 1.3333334f * __expf(p2));
  }
  *x = fin * -4.3429446f + 0.001f;                         // -10 / ln(10)
  return *x == *x;
}
__device__ __forceinline__ float clamp_floor_phred(float x) {
  return x >= 94.0f ? 93.0f : (x < 2.0f ? 2.0f : floorf(x));
}
__device__ __forceinline__ bool certified_quality(const double (&ll)[4], int mi, double mx, double ln_pre,
                                                  uint32_t fast_qual, uint32_t* q_out) {
  float s = 0.0f;
  double maxabs = fabs(mx);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (i == mi) continue;
    const double d = __dsub_rn(ll[i], mx);
    // a -inf likelihood (quality-0 observation) makes the reference's ln_sum_exp_array return -inf
    // outright (phred.rs:318-320): that quirk, and NaN, belong to the literal tail
    if (!(d <= 0.0) || !(d > -1.0e300)) return false;
    maxabs = fmax(maxabs, fabs(ll[i]));
    if (d > -100.0) s += __expf(static_cast<float>(d));
  }
  if (!(maxabs < 1.0e300)) return false;
  const float lp = static_cast<float>(ln_pre);
  const float noise = static_cast<float>(maxabs * 1.8e-15);   // 8 ulp(max |ll|) on the reference's s
  const float s_hi = (s + noise) * 1.0001f;
  const float s_lo = fmaxf(s - noise, 0.0f) * 0.9999f;
  float x_lo, x_hi;
  int b_lo, b_hi;
  if (!tail_phred(__logf(s_hi) - log1pf(s_hi), lp, &x_lo, &b_lo)) return false;   // more error, lower quality
  const float err_lo = s_lo > 0.0f ? __logf(s_lo) - log1pf(s_lo) : -CUDART_INF_F;
  if (!tail_phred(err_lo, lp, &x_hi, &b_hi)) return false;
  if (b_lo != b_hi) return false;
  if (b_lo == 0) { *q_out = fast_qual; return true; }
  const float qa = clamp_floor_phred(x_lo - 2.0e-3f), qb = clamp_floor_phred(x_hi + 2.0e-3f);
  if (qa != qb) return false;
  *q_out = static_cast<uint32_t>(qa);
  return true;
}

// The same certified evaluation fed by the FIXED-POINT likelihood gaps of the integer pass (sums of
// round(D[q] * 65536), host_tables.cpp): best = the winner's sum, o1..o3 = the sums of the three other bases
// (0 for an unobserved base), each gap within e = 2 * depth + 1 units of the exact one.  Decides the quality of
// a position the dominant-winner proof could not (a shallow or low-quality pileup, a pileup with dissent)
// without the f64 Kahan sums; returns false -- the literal path decides -- when a gap is too small for the
// fixed-point sums to rule out a tie, when the reference's unanimous fast path (gap > 23.0,
// base_builder.rs:338-379) cannot be told from the full call, or when the interval straddles a branch or a
// quality boundary.
__device__ __noinline__ bool certified_from_fixed(int32_t best, int32_t o1, int32_t o2, int32_t o3, uint32_t depth,
                                                     bool unanimous, double ln_pre, uint32_t fast_qual, uint32_t* q_out) {
  const int32_t e = static_cast<int32_t>(2u * depth + 1u);
  const int32_t g1 = best - o1, g2 = best - o2, g3 = best - o3;
  const int32_t gmin = min(g1, min(g2, g3));
  if (gmin <= e + 64) return false;
  if (unanimous) {                                     // all three gaps equal the winner's sum
    const int32_t t23 = 23 * 65536;
    if (gmin - e > t23) { *q_out = fast_qual; return true; }
    if (gmin + e >= t23) return false;
  }
  const float k = -1.0f / 65536.0f;
  float s_hi = __expf(static_cast<float>(g1 - e) * k) + __expf(static_cast<float>(g2 - e) * k) + __expf(static_cast<float>(g3 - e) * k);
  float s_lo = __expf(static_cast<float>(g1 + e) * k) + __expf(static_cast<float>(g2 + e) * k) + __expf(static_cast<float>(g3 + e) * k);
  const float lp = static_cast<float>(ln_pre);
  const float noise = static_cast<float>(depth) * 32.0f * 1.8e-15f;   // 8 ulp(max |ll|) on the reference's s, |ll| <= 32 * depth
  s_hi = (s_hi + noise) * 1.0002f;
  s_lo = fmaxf(s_lo - noise, 0.0f) * 0.9998f;
  float x_lo, x_hi;
  int b_lo, b_hi;
  if (!tail_phred(__logf(s_hi) - log1pf(s_hi), lp, &x_lo, &b_lo)) return false;
  const float err_lo = s_lo > 0.0f ? __logf(s_lo) - log1pf(s_lo) : -CUDART_INF_F;
  if (!tail_phred(err_lo, lp, &x_hi, &b_hi)) return false;
  if (b_lo != b_hi) return false;
  if (b_lo == 0) { *q_out = fast_qual; return true; }
  const float qa = clamp_floor_phred(x_lo - 2.0e-3f), qb = clamp_floor_phred(x_hi + 2.0e-3f);
  if (qa != qb) return false;
  *q_out = static_cast<uint32_t>(qa);
  return true;
}

// The literal per-position algorithm (vanilla_caller.rs:1319-1355 + base_builder.rs:295-458).
//
// Two-read units take a shortcut first: when both reads cover the position, agree on an A/C/G/T base
// and have tabulated qualities, the result is the host-evaluated outcome of the reference's
// add/add/call sequence (host_tables.cpp pair_quality).  Shallow pileups rarely reach the
// dominant-winner gap, so without the table every position of a two-read unit would run the f64
// path.  The shortcut lives here, out of line, so the vote loop's register allocation is untouched.
// Bit 31 of the returned depth flags a result of the f64 algorithm (diagnostic counter).
constexpr uint32_t kLiteralFlag = 0x80000000u;

template <class M>
__device__ __noinline__ Called exact_position(const TileView<M>& tv, const VoteSmem& S,
                                              uint32_t read_begin, uint32_t n_reads,
                                              uint32_t pos, uint32_t min_reads,
                                              uint32_t min_cons_q, uint32_t fast_qual) {
  if (n_reads == 2u) {
    const uint64_t d0 = M::ld64(tv.reads + static_cast<typename M::off_t>(read_begin - tv.read_base) * 8u);
    const uint64_t d1 = M::ld64(tv.reads + static_cast<typename M::off_t>(read_begin - tv.read_base + 1u) * 8u);
    if (pos < (static_cast<uint32_t>(d0) & 0xFFFFu) && pos < (static_cast<uint32_t>(d1) & 0xFFFFu)) {
      const typename M::off_t r0 = static_cast<typename M::off_t>((d0 >> 16) - tv.byte_base) + pos;
      const typename M::off_t r1 = static_cast<typename M::off_t>((d1 >> 16) - tv.byte_base) + pos;
      const uint32_t i0 = base_to_index(M::ld8(tv.bases + r0));
      if (i0 < 4u && i0 == base_to_index(M::ld8(tv.bases + r1))) {
        uint32_t qa = M::ld8(tv.quals + r0), qb = M::ld8(tv.quals + r1);
        qa = qa > FGB_MAX_PHRED ? FGB_MAX_PHRED : qa;
        qb = qb > FGB_MAX_PHRED ? FGB_MAX_PHRED : qb;
        const uint32_t cq = __ldg(S.pair_q + qa * 94u + qb);
        if (cq != 255u) {
          Called o;
          o.depth = 2; o.errors = 0;
          if (2u < min_reads) { o.base = 'N'; o.qual = 0; }                 // vanilla_caller.rs:1345-1349
          else if (cq < min_cons_q) { o.base = 'N'; o.qual = 2; }
          else { o.base = (0x54474341u >> (8u * i0)) & 0xFFu; o.qual = cq; }
          return o;
        }
      }
    }
  }
  double ll[4] = {0.0, 0.0, 0.0, 0.0};   // LN_ONE
  double kc[4] = {0.0, 0.0, 0.0, 0.0};   // Kahan compensations
  uint64_t cnt = 0;                      // 4 x u16 observation counters
  for (uint32_t r = 0; r < n_reads; ++r) {
    uint64_t d = M::ld64(tv.reads + static_cast<typename M::off_t>(read_begin - tv.read_base + r) * 8u);
    uint32_t len = static_cast<uint32_t>(d & 0xFFFFu);
    if (pos < len) {                                          // vanilla_caller.rs:1323
      typename M::off_t row = static_cast<typename M::off_t>((d >> 16) - tv.byte_base) + pos;
      uint32_t b = M::ld8(tv.bases + row);
      uint32_t idx = base_to_index(b);
      if (b != 'N' && idx < 4u) {                             // :1328 and base_builder.rs:300
        uint32_t q = M::ld8(tv.quals + row);
        q = q > FGB_MAX_PHRED ? FGB_MAX_PHRED : q;            // base_builder.rs:307
        double c = S.correct[q];
        double e = S.err_alt[q];
#pragma unroll
        for (int i = 0; i < 4; ++i) {                         // base_builder.rs:312-324
          double v = (static_cast<uint32_t>(i) == idx) ? c : e;
          double y = __dsub_rn(v, kc[i]);
          double t = __dadd_rn(ll[i], y);
          kc[i] = __dsub_rn(__dsub_rn(t, ll[i]), y);
          ll[i] = t;
        }
        cnt += 1ull << (16u * idx);
      }
    }
  }
  uint32_t n0 = cnt & 0xFFFFu, n1 = (cnt >> 16) & 0xFFFFu, n2 = (cnt >> 32) & 0xFFFFu,
           n3 = (cnt >> 48) & 0xFFFFu;
  uint32_t depth = (n0 + n1 + n2 + n3) & 0xFFFFu;             // contributions(): u16 sum
  uint32_t cbase = 'N', cqual = 2;                            // base_builder.rs:392-394
  uint32_t nobs_call = 0;
  uint32_t literal = 0;                                       // set when the f64 tail decided
  if (depth != 0) {
    uint32_t kinds = (n0 != 0) + (n1 != 0) + (n2 != 0) + (n3 != 0);
    bool done = false;
    if (kinds == 1) {                                         // base_builder.rs:338-379
      uint32_t w = n0 ? 0u : n1 ? 1u : n2 ? 2u : 3u;
      double winner = w == 0 ? ll[0] : w == 1 ? ll[1] : w == 2 ? ll[2] : ll[3];
      double loser = w == 0 ? ll[1] : w == 1 ? ll[2] : w == 2 ? ll[3] : ll[0];
      if (__dsub_rn(winner, loser) > 23.0) {
        cbase = (0x54474341u >> (8u * w)) & 0xFFu;
        cqual = fast_qual;
        nobs_call = depth;
        done = true;
      }
    }
    if (!done) {                                              // base_builder.rs:401-457
      // argmax and tie rule first: pure comparisons (the reference evaluates ln_sum before them;
      // the order is immaterial)
      double mx = -CUDART_INF;
      int mi = -1;
      bool tie = false;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        double v = ll[i];
        if (v > mx) { mx = v; mi = i; tie = false; }
        else if (v == mx) { tie = true; }
        else if (v < mx) { if (fabs(__dsub_rn(v, mx)) <= dm::kEps) tie = true; }
      }
      if (!(tie || mi < 0)) {
        uint32_t q;
        if (certified_quality(ll, mi, mx, S.ln_pre, fast_qual, &q)) {
          cqual = q;
        } else {
          double ln_sum = dm::ln_sum_exp_array4(ll);
          double post = __dsub_rn(mx, ln_sum);
          double err = dm::ln_one_minus_exp(post);
          double fin = dm::ln_error_prob_two_trials(S.ln_pre, err);
          cqual = dm::ln_prob_to_phred(fin);
          literal = kLiteralFlag;
        }
        cbase = (0x54474341u >> (8 * mi)) & 0xFFu;
        nobs_call = mi == 0 ? n0 : mi == 1 ? n1 : mi == 2 ? n2 : n3;
      }
    }
  }
  Called out;
  out.depth = depth | literal;
  out.errors = (depth - nobs_call) & 0xFFFFu;                 // vanilla_caller.rs:1341
  if (depth < min_reads) { out.base = 'N'; out.qual = 0; }    // :1345-1346
  else if (cqual < min_cons_q) { out.base = 'N'; out.qual = 2; }  // :1347-1348
  else { out.base = cbase; out.qual = cqual & 0xFFu; }
  return out;
}

struct LocalStats {
  uint32_t positions, exact, nocall;
};

// ---- duplex epilogue -----------------------------------------------------------------------------------------
// Runs on the eight voting warps after a tile's vote (and a barrier among them): the tile's attached duplex jobs,
// both of whose single-strand units this tile has just voted, are combined 8 positions per thread.  The SS words
// come back through L2 (ld.global.cg: they were written by other threads of this CTA a moment ago), the source rows
// for the exact error recount (duplex_caller.rs:943-951) are still in the stage.  Only the both-strand arm of a
// word-path job is taken (every item of a job reaches the same verdict from job-level data); anything else keeps
// its FGB_DUPLEX_PENDING status byte and is done by duplex_combine_pending_kernel after the vote.
__device__ __forceinline__ uint32_t duplex_epilogue(const VoteArgsDuplex& a, const Stage& st, const uint8_t* st_bases,
                                                    const uint8_t* st_reads, const uint32_t base32,
                                                    const uint32_t read_base, const uint32_t jbegin,
                                                    const uint32_t count, const uint32_t M, const uint32_t tid) {
  const uint32_t total = count * M;
  const uint32_t ub0 = st.tile.unit_begin;
  uint32_t done = 0;
  for (uint32_t it = tid; it < total; it += kVoteThreads) {
    const uint32_t jl = it / M, p0 = (it - jl * M) * 8u;
    const uint32_t j = __ldg(a.job_index + jbegin + jl);
    const uint4 jw = __ldg(reinterpret_cast<const uint4*>(a.djobs + j));     // {unit_a, unit_b, out_off}
    const uint32_t la = jw.x - ub0, lb = jw.y - ub0;
    const uint64_t out_off = (static_cast<uint64_t>(jw.w) << 32) | jw.z;
    const fgb_unit ua = st.units[la], ub = st.units[lb];
    const uint32_t len = ua.cons_len < ub.cons_len ? ua.cons_len : ub.cons_len;       // duplex_caller.rs:846-849
    if (p0 >= len) continue;                                   // (an empty job is left pending, too)
    const uint32_t na = st.units[la + 1u].read_begin - ua.read_begin;
    const uint32_t nb = st.units[lb + 1u].read_begin - ub.read_begin;
    if ((out_off & 7ull) != 0ull || na + nb > 255u) continue;  // not a word-path job
    // :852-882 both strands must have coverage inside the truncated region; the first word nearly always shows it
    const uint32_t live0 = len < 8u ? len : 8u;
    const uint4 ad0 = __ldcg(reinterpret_cast<const uint4*>(a.out_depth + ua.out_off));
    const uint4 bd0 = __ldcg(reinterpret_cast<const uint4*>(a.out_depth + ub.out_off));
    if (!(duplex_any_depth(ad0, live0) && duplex_any_depth(bd0, live0))) continue;
    const uint2 ab2 = __ldcg(reinterpret_cast<const uint2*>(a.out_base + ua.out_off + p0));
    const uint2 bb2 = __ldcg(reinterpret_cast<const uint2*>(a.out_base + ub.out_off + p0));
    const uint2 aq2 = __ldcg(reinterpret_cast<const uint2*>(a.out_qual + ua.out_off + p0));
    const uint2 bq2 = __ldcg(reinterpret_cast<const uint2*>(a.out_qual + ub.out_off + p0));
    const DuplexWord w = duplex_combine_word(ab2, bb2, aq2, bq2);
    uint32_t cnt[2] = {0u, 0u};
    const uint32_t ra0 = ua.read_begin - read_base, rb0 = ub.read_begin - read_base;
    const uint32_t nr = na + nb;
    for (uint32_t r0 = 0; r0 < nr; r0 += 4u) {                 // AB rows then BA rows, four in flight
      uint64_t d[4];
      uint2 sb[4];
#pragma unroll
      for (uint32_t k = 0; k < 4u; ++k) {
        const uint32_t r = r0 + k;
        d[k] = r < nr ? *reinterpret_cast<const uint64_t*>(st_reads + 8u * (r < na ? ra0 + r : rb0 + (r - na))) : 0ull;
      }
#pragma unroll
      for (uint32_t k = 0; k < 4u; ++k) {
        sb[k] = make_uint2(0x4E4E4E4Eu, 0x4E4E4E4Eu);          // N: counts nothing
        if (static_cast<uint32_t>(d[k] & 0xFFFFu) > p0)
          sb[k] = *reinterpret_cast<const uint2*>(st_bases + (static_cast<uint32_t>(d[k] >> 16) - base32 + p0));
      }
#pragma unroll
      for (uint32_t k = 0; k < 4u; ++k) {
        const uint32_t rl = static_cast<uint32_t>(d[k] & 0xFFFFu);
        duplex_recount_row(sb[k], rl > p0 ? rl - p0 : 0u, w.rawb, cnt);
      }
    }
    *reinterpret_cast<uint2*>(a.d_base + out_off + p0) = make_uint2(w.ob[0], w.ob[1]);
    *reinterpret_cast<uint2*>(a.d_qual + out_off + p0) = make_uint2(w.oq[0], w.oq[1]);
    *reinterpret_cast<uint4*>(a.d_errors + out_off + p0) = duplex_errors_word(w.rawb, cnt);
    if (p0 == 0u) { a.d_status[j] = FGB_DUPLEX_BOTH; ++done; }
  }
  return done;
}

__device__ __forceinline__ void write_called(const VoteArgs& a, uint64_t o, const Called& c) {
  a.out_base[o] = static_cast<uint8_t>(c.base);
  a.out_qual[o] = static_cast<uint8_t>(c.qual);
  a.out_depth[o] = static_cast<uint16_t>(c.depth);
  a.out_errors[o] = static_cast<uint16_t>(c.errors);
}

// "Dominant winner" evaluation of one position in integers (proof: host_tables.cpp).  Returns true
// and fills `out` when the reference's result is PROVEN to be (winner, phred(ln_pre)) after the
// thresholds of vanilla_caller.rs:1345-1349; returns false when the literal f64 path must decide.
// Cert: try the certified evaluation from the fixed-point gaps before giving a position to the literal path.
// Enabled in the shallow-class kernel only: the call keeps registers live across it, which costs the general
// kernel's item loop a quarter of its speed (measured), and shallow pileups are where the dominant-winner
// proof fails most.
// Quality of a UNANIMOUS pileup from its fixed-point gap through the host-built step table (host_tables.h ugap_*;
// shallow kernel only: the table sits in dynamic shared memory behind the pair table).  `g` is within 2 * depth + 1
// units of the exact gap; the answer stands only if that interval, widened by kUgapGuard, lies inside one step.
__device__ __forceinline__ bool cert_unanimous(const VoteSmem& S, int32_t g, uint32_t depth, uint32_t* q) {
  const int32_t* bp = reinterpret_cast<const int32_t*>(reinterpret_cast<const uint8_t*>(&S) + sizeof(VoteSmem) + kUgapSmemOff);
  const uint8_t* qv = reinterpret_cast<const uint8_t*>(bp + 128);
  const int32_t e = static_cast<int32_t>(2u * depth + 1u) + kUgapGuard;
  const int32_t glo = g - e, ghi = g + e;
  uint32_t k = 0;
#pragma unroll
  for (uint32_t step = 64u; step > 0u; step >>= 1)
    if (bp[k + step] <= glo) k += step;                 // largest k with bp[k] <= glo (entries past the table: INT32_MAX)
  if (bp[k] > glo || bp[k + 1] <= ghi) return false;    // below the first step, or the interval reaches the next one
  *q = qv[k];
  return true;
}

template <class M, bool Cert = false>
__device__ __forceinline__ bool dominant_position(const TileView<M>& tv, const VoteSmem& S,
                                                  uint32_t read_begin, uint32_t n_reads,
                                                  uint32_t pos, uint32_t min_reads,
                                                  uint32_t min_cons_q, uint32_t fast_qual,
                                                  Called& out) {
  if (n_reads > S.nmax2) return false;
  int32_t s0 = 0, s1 = 0, s2 = 0, s3 = 0;
  uint32_t c0 = 0, c1 = 0, c2 = 0, c3 = 0;
  bool usable = true;
  for (uint32_t r = 0; r < n_reads; ++r) {
    uint64_t d = M::ld64(tv.reads + static_cast<typename M::off_t>(read_begin - tv.read_base + r) * 8u);
    uint32_t len = static_cast<uint32_t>(d & 0xFFFFu);
    if (pos < len) {
      typename M::off_t row = static_cast<typename M::off_t>((d >> 16) - tv.byte_base) + pos;
      uint32_t b = M::ld8(tv.bases + row);
      uint32_t idx = base_to_index(b);
      if (b != 'N' && idx < 4u) {
        uint32_t q = M::ld8(tv.quals + row);
        q = q > FGB_MAX_PHRED ? FGB_MAX_PHRED : q;
        int32_t dq = S.dfix[q];
        usable &= (dq != INT32_MIN);
        s0 += idx == 0 ? dq : 0; c0 += idx == 0;
        s1 += idx == 1 ? dq : 0; c1 += idx == 1;
        s2 += idx == 2 ? dq : 0; c2 += idx == 2;
        s3 += idx == 3 ? dq : 0; c3 += idx == 3;
      }
    }
  }
  const uint32_t depth = c0 + c1 + c2 + c3;
  if (depth == 0) {   // base_builder.rs:392-394 then vanilla_caller.rs:1345 (min_reads >= 1)
    out.base = 'N'; out.qual = 0; out.depth = 0; out.errors = 0;
    return true;
  }
  if (!usable) return false;
  // winner over all four lanes (an unobserved base has S = 0) and the runner-up
  int32_t best = s0, second = INT32_MIN;
  uint32_t w = 0, cw = c0;
  auto consider = [&](int32_t sv, uint32_t idx, uint32_t cv) {
    if (sv > best) { second = best; best = sv; w = idx; cw = cv; }
    else if (sv > second) { second = sv; }
  };
  consider(s1, 1u, c1);
  consider(s2, 2u, c2);
  consider(s3, 3u, c3);
  // every fixed-point term is within half a unit of D[q]*65536; two sums of <= depth terms
  uint32_t q = fast_qual;
  if (static_cast<int64_t>(best) - second < static_cast<int64_t>(S.g2fix) + 2 * static_cast<int64_t>(depth) + 1) {
    if (!Cert) return false;
    bool have = false;
    if (depth == cw && depth <= 4u) {
      // unanimous (the three other sums are 0, every gap = best): the step table instead of the float evaluation --
      // the unanimous low-quality cycles at the start of every shallow family come through here
      const int32_t e = static_cast<int32_t>(2u * depth + 1u), t23 = 23 * 65536;
      if (best > e + 64) {
        if (best - e > t23) { q = fast_qual; have = true; }                   // base_builder.rs:338-379
        else if (best + e < t23) have = cert_unanimous(S, best, depth, &q);
      }
    }
    if (!have) {
      const int32_t oa = w == 0 ? s1 : s0, ob = w <= 1 ? s2 : s1, oc = w == 3 ? s2 : s3;   // the three other sums
      if (!certified_from_fixed(best, oa, ob, oc, depth, depth == cw, S.ln_pre, fast_qual, &q)) return false;
    }
  }
  out.depth = depth;
  out.errors = depth - cw;
  if (depth < min_reads) { out.base = 'N'; out.qual = 0; }
  else if (q < min_cons_q) { out.base = 'N'; out.qual = 2; }
  else { out.base = (0x54474341u >> (8u * w)) & 0xFFu; out.qual = q; }
  return true;
}

// high bit of each byte set where the byte of x is zero
__device__ __forceinline__ uint32_t zero_bytes(uint32_t x) {
  return ~(((x & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | x | 0x7F7F7F7Fu);
}
// 0x80 in the low `k` bytes (k = 0..4)
__device__ __forceinline__ uint32_t low_bytes_mask(uint32_t k) {
  return k >= 4u ? 0x80808080u : (0x80808080u & ((1u << (8u * k)) - 1u));
}
// high bit of each byte set where the byte is one of 'A','C','G','T' (0x41,0x43,0x47,0x54)
__device__ __forceinline__ uint32_t acgt_bytes(uint32_t x) {
  uint32_t y = x ^ 0x41414141u;                       // A,C,G,T -> 0x00,0x02,0x06,0x15
  uint32_t in0246 = zero_bytes(y & 0xF9F9F9F9u);      // {0,2,4,6}
  uint32_t is4 = zero_bytes(y ^ 0x04040404u);         // 'E'
  uint32_t isT = zero_bytes(y ^ 0x15151515u);
  return (in0246 & ~is4) | isT;
}

// 0x80 in every byte of `sum` (bytes <= 255) that is >= t (t <= 255)
__device__ __forceinline__ uint32_t bytes_ge(uint32_t sum, uint32_t t) {
  const uint32_t add = (0x100u - t) * 0x00010001u;
  const uint32_t ev = ((sum & 0x00FF00FFu) + add) & 0x01000100u;          // bytes 0, 2 -> bits 8, 24
  const uint32_t od = (((sum >> 8) & 0x00FF00FFu) + add) & 0x01000100u;   // bytes 1, 3
  return (ev >> 1) | (od << 7);
}

// Resolve one undecided position: integer proof first, the literal f64 algorithm otherwise.
template <class M, bool Cert = false>
__device__ __forceinline__ Called resolve_position(const TileView<M>& tv, const VoteSmem& S,
                                                   uint32_t rb, uint32_t n, uint32_t pos,
                                                   const VoteArgs& a, LocalStats& ls) {
  Called c;
  if (!dominant_position<M, Cert>(tv, S, rb, n, pos, a.min_reads, a.min_cons_q, a.fast_qual, c)) {
    c = exact_position<M>(tv, S, rb, n, pos, a.min_reads, a.min_cons_q, a.fast_qual);
    ls.exact += c.depth >> 31;
    c.depth &= ~kLiteralFlag;
  }
  ls.nocall += (c.base == 'N');
  return c;
}

// Resolves a warp's queued positions.  The depth axis is split across a GROUP of lanes (8 lanes
// per position when every queued pileup has <= 8 reads, else the whole warp): each lane classifies
// its reads and looks up their fixed-point likelihood gaps, a __shfl_xor butterfly sums the four
// per-base gap sums and counts over the group, and the group leader applies the dominant-winner
// proof (host_tables.cpp).  Whatever the proof cannot decide runs the literal f64 algorithm.
template <class M, uint32_t G, bool Cert = false>
__device__ __forceinline__ void slow_pass_g(const VoteArgs& a, const VoteSmem& S, const Stage& st,
                                            const TileView<M>& tv, const uint32_t* wqueue, uint32_t qn,
                                            uint32_t lane, LocalStats& ls) {
  constexpr uint32_t per_pass = 32u / G;
  constexpr uint32_t gshift = G == 8u ? 3u : 5u;
  const uint32_t sub = lane & (G - 1u);
  for (uint32_t e0 = 0; e0 < qn; e0 += per_pass) {
    const uint32_t e = e0 + (lane >> gshift);
    const bool valid = e < qn;
    uint32_t u = 0, pos = 0, rb = 0, n = 0;
    uint64_t out_off = 0;
    if (valid) {
      uint32_t ent = wqueue[e];
      u = ent >> 16; pos = ent & 0xFFFFu;
      const fgb_unit un = st.units[u];
      rb = un.read_begin; out_off = un.out_off;
      n = st.units[u + 1].read_begin - rb;
    }
    const bool provable = n <= S.nmax2;
    int32_t s0 = 0, s1 = 0, s2 = 0, s3 = 0;
    uint32_t c01 = 0, c23 = 0;      // 4 x u16 observation counts; bit 31 of c23 = "unusable quality seen"
    if (provable) {
      for (uint32_t r = sub; r < n; r += G) {
        uint64_t d = M::ld64(tv.reads + static_cast<typename M::off_t>(rb - tv.read_base + r) * 8u);
        uint32_t len = static_cast<uint32_t>(d) & 0xFFFFu;
        if (pos < len) {
          typename M::off_t row = static_cast<typename M::off_t>((d >> 16) - tv.byte_base) + pos;
          uint32_t b = M::ld8(tv.bases + row);
          uint32_t q = M::ld8(tv.quals + row);
          if (is_acgt_upper(b & 0xDFu)) {       // A,C,G,T in either case; 'N' and the rest are skipped
            const uint32_t x = (b >> 1) & 3u;   // A 0, C 1, T 2, G 3
            const uint32_t idx = x ^ (x >> 1);  // A 0, C 1, G 2, T 3
            q = q > FGB_MAX_PHRED ? FGB_MAX_PHRED : q;
            int32_t dq = S.dfix[q];
            if (dq == INT32_MIN) { c23 |= 0x80000000u; dq = 0; }
            s0 += idx == 0 ? dq : 0; s1 += idx == 1 ? dq : 0;
            s2 += idx == 2 ? dq : 0; s3 += idx == 3 ? dq : 0;
            c01 += idx == 0 ? 1u : (idx == 1 ? 0x10000u : 0u);
            c23 += idx == 2 ? 1u : (idx == 3 ? 0x10000u : 0u);
          }
        }
      }
    }
    // butterfly over the group (n <= nmax2 <= 1024 keeps every 16-bit count and the flag intact)
#pragma unroll
    for (uint32_t off = G >> 1; off > 0; off >>= 1) {
      s0 += __shfl_xor_sync(0xFFFFFFFFu, s0, off);
      s1 += __shfl_xor_sync(0xFFFFFFFFu, s1, off);
      s2 += __shfl_xor_sync(0xFFFFFFFFu, s2, off);
      s3 += __shfl_xor_sync(0xFFFFFFFFu, s3, off);
      c01 += __shfl_xor_sync(0xFFFFFFFFu, c01, off);
      uint32_t o23 = __shfl_xor_sync(0xFFFFFFFFu, c23, off);
      c23 = ((c23 & 0x7FFFFFFFu) + (o23 & 0x7FFFFFFFu)) | ((c23 | o23) & 0x80000000u);
    }
    if (valid && sub == 0) {
      Called c;
      bool done = false;
      if (provable) {
        const uint32_t c0 = c01 & 0xFFFFu, c1 = c01 >> 16, c2 = c23 & 0xFFFFu, c3 = (c23 >> 16) & 0x7FFFu;
        const uint32_t depth = c0 + c1 + c2 + c3;
        if (depth == 0) {   // base_builder.rs:392-394 then vanilla_caller.rs:1345 (min_reads >= 1)
          c.base = 'N'; c.qual = 0; c.depth = 0; c.errors = 0;
          done = true;
        } else if (!(c23 & 0x80000000u)) {
          int32_t best = s0, second = INT32_MIN;
          uint32_t w = 0, cw = c0;
          if (s1 > best) { second = best; best = s1; w = 1; cw = c1; } else if (s1 > second) second = s1;
          if (s2 > best) { second = best; best = s2; w = 2; cw = c2; } else if (s2 > second) second = s2;
          if (s3 > best) { second = best; best = s3; w = 3; cw = c3; } else if (s3 > second) second = s3;
          // every fixed-point term is within half a unit of D[q]*65536; two sums of <= depth terms
          uint32_t q = a.fast_qual;
          bool proven = static_cast<int64_t>(best) - second >=
                        static_cast<int64_t>(S.g2fix) + 2 * static_cast<int64_t>(depth) + 1;
          if (Cert && !proven) {
            const int32_t oa = w == 0 ? s1 : s0, ob = w <= 1 ? s2 : s1, oc = w == 3 ? s2 : s3;
            proven = certified_from_fixed(best, oa, ob, oc, depth, depth == cw, S.ln_pre, a.fast_qual, &q);
          }
          if (proven) {
            c.depth = depth;
            c.errors = depth - cw;
            if (depth < a.min_reads) { c.base = 'N'; c.qual = 0; }
            else if (q < a.min_cons_q) { c.base = 'N'; c.qual = 2; }
            else { c.base = (0x54474341u >> (8u * w)) & 0xFFu; c.qual = q; }
            done = true;
          }
        }
      }
      if (!done) {
        c = exact_position<M>(tv, S, rb, n, pos, a.min_reads, a.min_cons_q, a.fast_qual);
        ls.exact += c.depth >> 31;
        c.depth &= ~kLiteralFlag;
      }
      ls.nocall += (c.base == 'N');
      write_called(a, out_off + pos, c);
    }
  }
}

// Group width (warp-uniform): 8 lanes per position (each lane strides the depth axis by 8) when no
// queued pileup is deeper than 64 reads -- the planner's shallow-tile hint answers that without
// looking -- else the whole warp per position.
template <class M, bool Cert = false>
__device__ __forceinline__ void slow_pass(const VoteArgs& a, const VoteSmem& S, const Stage& st,
                                          const TileView<M>& tv, const uint32_t* wqueue, uint32_t qn,
                                          uint32_t lane, LocalStats& ls) {
  bool shallow = (st.tile.flags & kTileFlagShallow) != 0;
  if (!shallow) {
    uint32_t nmax = 0;
    for (uint32_t e = lane; e < qn; e += 32) {
      uint32_t u = wqueue[e] >> 16;
      uint32_t n = st.units[u + 1].read_begin - st.units[u].read_begin;
      nmax = n > nmax ? n : nmax;
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      uint32_t o = __shfl_xor_sync(0xFFFFFFFFu, nmax, off);
      nmax = o > nmax ? o : nmax;
    }
    shallow = nmax <= 64u;
  }
  if (shallow && qn < kLaneMinQueue) {
    slow_pass_g<M, 8u, Cert>(a, S, st, tv, wqueue, qn, lane, ls);
  } else if (shallow) {
    // one lane per queued position: with at most 64 reads the depth loop is short, and 32 positions
    // per pass beat splitting each pileup over a group of lanes
    for (uint32_t e = lane; e < qn; e += 32u) {
      const uint32_t ent = wqueue[e];
      const uint32_t u = ent >> 16, pos = ent & 0xFFFFu;
      const fgb_unit un = st.units[u];
      const Called c = resolve_position<M, Cert>(tv, S, un.read_begin, st.units[u + 1].read_begin - un.read_begin,
                                                 pos, a, ls);
      write_called(a, un.out_off + pos, c);
    }
  } else {
    slow_pass_g<M, 32u, Cert>(a, S, st, tv, wqueue, qn, lane, ls);
  }
}

// Votes this warp's share of one tile.  Called by the eight consumer warps; `vt` is the thread's
// rotating slot (0..kVoteThreads-1): it owns items vt, vt+256, ...  An item is 8 consecutive
// positions of one unit: one 64-bit word of every read's base row and quality row.
//
// Regular tiles (planner flag): every read of the tile has the same length L, rows are packed back
// to back at stride round_up(L, 8) and every unit calls L positions.  The read descriptors are then
// redundant for the scan: read r of the tile starts at word (r - tile.read_begin) * m, m = stride/8.
// V = 0: the general kernel; V = 1: the shallow-class kernel (tiles whose units have at most four reads):
// two-read units take the pair table in line.  (A sum-of-qualities proof for three- and four-read units was
// built and measured: the exact threshold -- host_tables.cpp sumt -- has to guard against one very low
// quality among high ones and ends up above what the per-read minimum test already accepts; dropped.)
template <class M, bool Regular, int V = 0>
__device__ __forceinline__ void vote_tile(const VoteArgs& a, VoteSmem& S, const Stage& st,
                                          const TileView<M>& tv, uint32_t vt, uint32_t warp,
                                          uint32_t n_items, LocalStats& ls) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t n_units = st.tile.n_units;
  const uint64_t out0 = st.units[0].out_off;
  const uint32_t min_reads = a.min_reads, min_cons_q = a.min_cons_q, fast_qual = a.fast_qual;
  // regular-tile constants
  const uint32_t reg_len = st.units[0].cons_len;
  const uint32_t reg_tail = reg_len - (((reg_len + 7u) >> 3) - 1u) * 8u;      // positions in a row's last word
  const uint32_t reg_tl_lo = low_bytes_mask(reg_tail), reg_tl_hi = low_bytes_mask(reg_tail > 4u ? reg_tail - 4u : 0u);
  const uint32_t reg_row0 = (st.tile.flags & kTileFlagSkew8) ? 8u : 0u;        // first row inside the stage
  // constant result of a proven position after the thresholds of vanilla_caller.rs:1345-1349
  const bool fast_masked = fast_qual < min_cons_q;
  const uint32_t fq4 = (fast_masked ? 2u : fast_qual) * 0x01010101u;
  // planner hint: every unit of the tile has the same number of items
  const uint32_t uni_m = st.tile.flags >> 8;
  const uint32_t uni_recip = st.aux[0];
  const uint32_t base32 = static_cast<uint32_t>(tv.byte_base);
  uint32_t* const wqueue = S.queue[warp];
  uint32_t* const wcount = &S.q_count[warp];
  // V == 1: the pair table sits in dynamic shared memory right behind VoteSmem (kPairSmemBytes, copied in the
  // kernel prologue); from global memory the eight random lookups per item were what bound depth 2 (each a
  // 32-line gather in L1)
  const uint8_t* const pair_sm = reinterpret_cast<const uint8_t*>(&S) + sizeof(VoteSmem);

  // ---------------- FAST PASS: one thread per 8 positions ----------------
  for (uint32_t item = vt; item < n_items; item += kVoteThreads) {
    uint32_t u;
    if (Regular || uni_m) {
      u = __umulhi(item, uni_recip);            // exact floor(item / uni_m): 2 <= uni_m <= 4096, item*uni_m < 2^32
    } else {                                    // largest u with start(u) <= item
      uint32_t lo = 0, hi = n_units;
      while (hi - lo > 1) {
        uint32_t mid = (lo + hi) >> 1;
        uint32_t start = static_cast<uint32_t>((st.units[mid].out_off - out0) >> 3);
        if (start <= item) lo = mid; else hi = mid;
      }
      u = lo;
    }
    const fgb_unit un = st.units[u];
    const uint32_t rb = un.read_begin;
    const uint32_t n = st.units[u + 1].read_begin - rb;
    const uint32_t cons_len = un.cons_len;
    const uint64_t o = out0 + (static_cast<uint64_t>(item) << 3);
    uint32_t p0, real, rm_lo, rm_hi;
    uint32_t reg_word = 0;                      // regular tiles: word index of read 0's word in the stage
    if (Regular) {
      const uint32_t w = item - u * uni_m;
      const bool last = w + 1u == uni_m;
      p0 = w << 3;
      real = last ? reg_tail : 8u;
      rm_lo = last ? reg_tl_lo : 0x80808080u;
      rm_hi = last ? reg_tl_hi : 0x80808080u;
      reg_word = (rb - st.tile.read_begin) * uni_m + w;
    } else {
      p0 = (item - static_cast<uint32_t>((un.out_off - out0) >> 3)) << 3;
      real = cons_len - p0 < 8u ? cons_len - p0 : 8u;   // positions of this item (>= 1)
      rm_lo = low_bytes_mask(real); rm_hi = low_bytes_mask(real > 4u ? real - 4u : 0u);
    }

    uint32_t wb_lo = 0, wb_hi = 0, wq_lo = 0, wq_hi = 0;   // 8 output bases / quals
    uint4 dep = make_uint4(0, 0, 0, 0), err = make_uint4(0, 0, 0, 0);   // 8 x u16 each
    uint32_t todo_lo = 0, todo_hi = 0;          // positions left for in-place resolution (queue overflow)
    ls.positions += real;

    if (n == 1) {
      // single-read consensus, vanilla_caller.rs:1285-1316
      uint32_t len;
      typename M::off_t row;
      if (Regular) {
        len = reg_len;
        row = reg_row0 + reg_word * 8u;
      } else {
        uint64_t d = M::ld64(tv.reads + static_cast<typename M::off_t>(rb - tv.read_base) * 8u);
        len = static_cast<uint32_t>(d & 0xFFFFu);
        row = static_cast<typename M::off_t>((d >> 16) - tv.byte_base) + p0;
      }
      uint64_t rbw = 0, rqw = 0;
      if (p0 < len) { rbw = M::ld64(tv.bases + row); rqw = M::ld64(tv.quals + row); }
      if (V == 1) {
        // byte-parallel form of the per-position rule: positions of the read (pos < len, pos < cons_len) get the
        // table quality or, below min_consensus_base_quality, (N, 2); depth 1 unless the base is N; positions of the
        // consensus row behind the read's end are (N, 2, 0)
        const uint32_t lim = len < cons_len ? len : cons_len;
        const uint32_t cov = lim > p0 ? lim - p0 : 0u;
        const uint32_t cm_lo = low_bytes_mask(cov), cm_hi = low_bytes_mask(cov > 4u ? cov - 4u : 0u);
        const uint32_t b_lo = static_cast<uint32_t>(rbw), b_hi = static_cast<uint32_t>(rbw >> 32);
        const uint32_t ql = __vminu4(static_cast<uint32_t>(rqw), 0x5F5F5F5Fu);          // `.get(idx).unwrap_or(0)`:
        const uint32_t qh = __vminu4(static_cast<uint32_t>(rqw >> 32), 0x5F5F5F5Fu);    // single_q[94] = [95] = 0
        const uint32_t a_lo = static_cast<uint32_t>(S.single_q[ql & 0xFFu]) | (static_cast<uint32_t>(S.single_q[(ql >> 8) & 0xFFu]) << 8) |
                              (static_cast<uint32_t>(S.single_q[(ql >> 16) & 0xFFu]) << 16) | (static_cast<uint32_t>(S.single_q[ql >> 24]) << 24);
        const uint32_t a_hi = static_cast<uint32_t>(S.single_q[qh & 0xFFu]) | (static_cast<uint32_t>(S.single_q[(qh >> 8) & 0xFFu]) << 8) |
                              (static_cast<uint32_t>(S.single_q[(qh >> 16) & 0xFFu]) << 16) | (static_cast<uint32_t>(S.single_q[qh >> 24]) << 24);
        const uint32_t keep_lo = bytes_ge(a_lo, min_cons_q > 255u ? 255u : min_cons_q) & cm_lo & (min_cons_q > 255u ? 0u : 0xFFFFFFFFu);
        const uint32_t keep_hi = bytes_ge(a_hi, min_cons_q > 255u ? 255u : min_cons_q) & cm_hi & (min_cons_q > 255u ? 0u : 0xFFFFFFFFu);
        const uint32_t kb_lo = spread_msb(keep_lo), kb_hi = spread_msb(keep_hi);
        const uint32_t rb_lo = spread_msb(rm_lo), rb_hi = spread_msb(rm_hi);
        wb_lo = ((b_lo & kb_lo) | (0x4E4E4E4Eu & ~kb_lo)) & rb_lo;
        wb_hi = ((b_hi & kb_hi) | (0x4E4E4E4Eu & ~kb_hi)) & rb_hi;
        wq_lo = ((a_lo & kb_lo) | (0x02020202u & ~kb_lo)) & rb_lo;
        wq_hi = ((a_hi & kb_hi) | (0x02020202u & ~kb_hi)) & rb_hi;
        const uint32_t nn_lo = ~zero_bytes(b_lo ^ 0x4E4E4E4Eu) & 0x80808080u, nn_hi = ~zero_bytes(b_hi ^ 0x4E4E4E4Eu) & 0x80808080u;   // base is not N
        const uint32_t d_lo = spread_msb(nn_lo & cm_lo), d_hi = spread_msb(nn_hi & cm_hi);
        dep = make_uint4(0x00010001u & __byte_perm(d_lo, 0u, 0x1100u), 0x00010001u & __byte_perm(d_lo, 0u, 0x3322u),
                         0x00010001u & __byte_perm(d_hi, 0u, 0x1100u), 0x00010001u & __byte_perm(d_hi, 0u, 0x3322u));
        ls.nocall += __popc(rm_lo & ~(keep_lo & nn_lo)) + __popc(rm_hi & ~(keep_hi & nn_hi));
      } else {      // general / deep kernels: the literal per-position loop (single-read units are the shallow class's)
        uint64_t obw = 0, oqw = 0, odw_lo = 0, odw_hi = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          uint32_t pos = p0 + j;
          if (pos < cons_len) {
            uint32_t b = static_cast<uint32_t>(rbw >> (8 * j)) & 0xFFu;
            uint32_t q = static_cast<uint32_t>(rqw >> (8 * j)) & 0xFFu;
            uint32_t ob = 'N', oq = 2, od = 0;
            if (pos < len) {
              uint32_t adj = q < FGB_NTABLE ? S.single_q[q] : 0u;   // `.get(idx).unwrap_or(0)`
              if (adj >= min_cons_q) { ob = b; oq = adj; }
              od = (b != 'N');
            }
            obw |= static_cast<uint64_t>(ob) << (8 * j);
            oqw |= static_cast<uint64_t>(oq) << (8 * j);
            if (j < 4) odw_lo |= static_cast<uint64_t>(od) << (16 * j);
            else odw_hi |= static_cast<uint64_t>(od) << (16 * (j - 4));
            ls.nocall += (ob == 'N');
          }
        }
        wb_lo = static_cast<uint32_t>(obw); wb_hi = static_cast<uint32_t>(obw >> 32);
        wq_lo = static_cast<uint32_t>(oqw); wq_hi = static_cast<uint32_t>(oqw >> 32);
        dep = make_uint4(static_cast<uint32_t>(odw_lo), static_cast<uint32_t>(odw_lo >> 32),
                         static_cast<uint32_t>(odw_hi), static_cast<uint32_t>(odw_hi >> 32));
      }
    } else if (V == 1 && n == 2u && min_reads <= 2u) {
      // two-read units: where both reads cover the position and agree on an A/C/G/T base, the result is the
      // host-evaluated outcome of the reference's add / add / call sequence (host_tables.cpp pair_quality)
      typename M::off_t ra, rc;
      uint32_t l0, l1;
      if (Regular) {
        ra = reg_row0 + reg_word * 8u; rc = ra + uni_m * 8u; l0 = l1 = reg_len;
      } else {
        typename M::addr_t rd = tv.reads + static_cast<typename M::off_t>(rb - tv.read_base) * 8u;
        const uint64_t d0 = M::ld64(rd), d1 = M::ld64(rd + 8u);
        l0 = static_cast<uint32_t>(d0) & 0xFFFFu; l1 = static_cast<uint32_t>(d1) & 0xFFFFu;
        ra = M::row_offset(d0, tv.byte_base, base32) + (l0 > p0 ? p0 : 0u);
        rc = M::row_offset(d1, tv.byte_base, base32) + (l1 > p0 ? p0 : 0u);
      }
      const uint64_t b0w = M::ld64(tv.bases + ra), b1w = M::ld64(tv.bases + rc);
      const uint64_t q0w = M::ld64(tv.quals + ra), q1w = M::ld64(tv.quals + rc);
      const uint32_t ml = l0 < l1 ? l0 : l1;
      const uint32_t covered = ml > p0 ? ml - p0 : 0u;
      const uint32_t e_lo = zero_bytes(static_cast<uint32_t>(b0w) ^ static_cast<uint32_t>(b1w)) &
                            acgt_bytes(static_cast<uint32_t>(b0w)) & low_bytes_mask(covered) & rm_lo;
      const uint32_t e_hi = zero_bytes(static_cast<uint32_t>(b0w >> 32) ^ static_cast<uint32_t>(b1w >> 32)) &
                            acgt_bytes(static_cast<uint32_t>(b0w >> 32)) &
                            low_bytes_mask(covered > 4u ? covered - 4u : 0u) & rm_hi;
      // byte-parallel: eight table lookups (indices are in range whatever the flags say: qualities are clamped),
      // then the thresholds of vanilla_caller.rs:1345-1349 on the assembled words
      const uint32_t qa_lo = __vminu4(static_cast<uint32_t>(q0w), FGB_MAX_PHRED * 0x01010101u);
      const uint32_t qa_hi = __vminu4(static_cast<uint32_t>(q0w >> 32), FGB_MAX_PHRED * 0x01010101u);
      const uint32_t qb_lo = __vminu4(static_cast<uint32_t>(q1w), FGB_MAX_PHRED * 0x01010101u);
      const uint32_t qb_hi = __vminu4(static_cast<uint32_t>(q1w >> 32), FGB_MAX_PHRED * 0x01010101u);
      auto look4 = [&](uint32_t qa4, uint32_t qb4) {
        const uint32_t c0 = pair_sm[(qa4 & 0xFFu) * 94u + (qb4 & 0xFFu)];
        const uint32_t c1 = pair_sm[((qa4 >> 8) & 0xFFu) * 94u + ((qb4 >> 8) & 0xFFu)];
        const uint32_t c2 = pair_sm[((qa4 >> 16) & 0xFFu) * 94u + ((qb4 >> 16) & 0xFFu)];
        const uint32_t c3 = pair_sm[(qa4 >> 24) * 94u + (qb4 >> 24)];
        return c0 | (c1 << 8) | (c2 << 16) | (c3 << 24);
      };
      const uint32_t cq_lo = look4(qa_lo, qb_lo), cq_hi = look4(qa_hi, qb_hi);
      const uint32_t mq = min_cons_q > 255u ? 255u : min_cons_q;
      const uint32_t ok_lo = e_lo & ~zero_bytes(~cq_lo), ok_hi = e_hi & ~zero_bytes(~cq_hi);    // 255 = literal path
      const uint32_t mk_lo = ok_lo & ~bytes_ge(cq_lo, mq), mk_hi = ok_hi & ~bytes_ge(cq_hi, mq);   // below min_cons_q: (N, 2)
      {
        const uint32_t vb_lo = spread_msb(ok_lo), vb_hi = spread_msb(ok_hi), mb_lo = spread_msb(mk_lo), mb_hi = spread_msb(mk_hi);
        wb_lo = ((static_cast<uint32_t>(b0w) & ~mb_lo) | (0x4E4E4E4Eu & mb_lo)) & vb_lo;
        wb_hi = ((static_cast<uint32_t>(b0w >> 32) & ~mb_hi) | (0x4E4E4E4Eu & mb_hi)) & vb_hi;
        wq_lo = ((cq_lo & ~mb_lo) | (0x02020202u & mb_lo)) & vb_lo;
        wq_hi = ((cq_hi & ~mb_hi) | (0x02020202u & mb_hi)) & vb_hi;
        ls.nocall += __popc(mk_lo) + __popc(mk_hi);
      }
      const uint32_t kb_lo = spread_msb(ok_lo), kb_hi = spread_msb(ok_hi);
      dep.x = 0x00020002u & __byte_perm(kb_lo, 0u, 0x1100u);
      dep.y = 0x00020002u & __byte_perm(kb_lo, 0u, 0x3322u);
      dep.z = 0x00020002u & __byte_perm(kb_hi, 0u, 0x1100u);
      dep.w = 0x00020002u & __byte_perm(kb_hi, 0u, 0x3322u);
      todo_lo = rm_lo & ~ok_lo; todo_hi = rm_hi & ~ok_hi;
      if (todo_lo | todo_hi) {
        const uint32_t cnt = static_cast<uint32_t>(__popc(todo_lo) + __popc(todo_hi));
        uint32_t slot = atomicAdd(wcount, cnt);
        const uint32_t ent = (u << 16) | p0;
        uint32_t keep_lo = 0, keep_hi = 0;
        for (uint32_t t = todo_lo; t; t &= t - 1u, ++slot) {
          if (slot < kWarpQueueCap) wqueue[slot] = ent + ((__ffs(t) - 1) >> 3);
          else keep_lo |= t & (0u - t);
        }
        for (uint32_t t = todo_hi; t; t &= t - 1u, ++slot) {
          if (slot < kWarpQueueCap) wqueue[slot] = ent + 4u + ((__ffs(t) - 1) >> 3);
          else keep_hi |= t & (0u - t);
        }
        todo_lo = keep_lo; todo_hi = keep_hi;
      }
    } else {
      const uint32_t qt = S.qt[n < kQtEntries ? n : kQtEntries - 1];
      const bool fast_ok = (qt <= FGB_MAX_PHRED) && (n >= min_reads) && (n <= 0xFFFFu);
      uint32_t fm_lo = 0, fm_hi = 0, b0_lo = 0, b0_hi = 0;
      if (fast_ok) {
        const uint32_t tsplat = qt * 0x01010101u;
        uint32_t diff_lo = 0, diff_hi = 0, okq_lo = 0x80808080u, okq_hi = 0x80808080u;
        if (Regular) {
          // every read covers the item: walk the rows at a constant stride, no descriptors
          typename M::addr_t pb = tv.bases + reg_row0 + reg_word * 8u;
          const uint32_t step = uni_m * 8u;
          {
            uint64_t w = M::ld64(pb);
            b0_lo = static_cast<uint32_t>(w); b0_hi = static_cast<uint32_t>(w >> 32);
          }
#pragma unroll 4
          for (uint32_t r = 0; r < n; ++r, pb += step) {
            uint64_t wb = M::ld64(pb);
            uint64_t wq = M::ld64(pb + kTileCapBytes);      // quality column sits kTileCapBytes above
            diff_lo |= static_cast<uint32_t>(wb) ^ b0_lo;
            diff_hi |= static_cast<uint32_t>(wb >> 32) ^ b0_hi;
            okq_lo &= (static_cast<uint32_t>(wq) | 0x80808080u) - tsplat;
            okq_hi &= (static_cast<uint32_t>(wq >> 32) | 0x80808080u) - tsplat;
          }
          fm_lo = zero_bytes(diff_lo) & okq_lo & acgt_bytes(b0_lo) & rm_lo;
          fm_hi = zero_bytes(diff_hi) & okq_hi & acgt_bytes(b0_hi) & rm_hi;
        } else {
          typename M::addr_t rd = tv.reads + static_cast<typename M::off_t>(rb - tv.read_base) * 8u;
          uint32_t minlen = 0xFFFFFFFFu;
          {   // reference word: read 0 (if it does not reach p0, minlen vetoes the item anyway)
            uint64_t d = M::ld64(rd);
            uint32_t len = static_cast<uint32_t>(d) & 0xFFFFu;
            uint64_t w = M::ld64(tv.bases + M::row_offset(d, tv.byte_base, base32) + (len > p0 ? p0 : 0u));
            b0_lo = static_cast<uint32_t>(w); b0_hi = static_cast<uint32_t>(w >> 32);
          }
#pragma unroll 4
          for (uint32_t r = 0; r < n; ++r) {
            uint64_t d = M::ld64(rd + r * 8u);
            uint32_t len = static_cast<uint32_t>(d) & 0xFFFFu;
            minlen = len < minlen ? len : minlen;
            // an uncovered read points at its own first word: harmless, minlen already vetoes
            typename M::off_t row = M::row_offset(d, tv.byte_base, base32) + (len > p0 ? p0 : 0u);
            uint64_t wb = M::ld64(tv.bases + row);
            uint64_t wq = M::ld64(tv.quals + row);
            diff_lo |= static_cast<uint32_t>(wb) ^ b0_lo;
            diff_hi |= static_cast<uint32_t>(wb >> 32) ^ b0_hi;
            // byte high bit survives iff q >= qT (no borrows: every minuend byte is >= 0x80 > qT)
            okq_lo &= (static_cast<uint32_t>(wq) | 0x80808080u) - tsplat;
            okq_hi &= (static_cast<uint32_t>(wq >> 32) | 0x80808080u) - tsplat;
          }
          // per-byte verdict: unanimous & quality-proven & A/C/G/T & covered by every read
          const uint32_t covered = minlen > p0 ? minlen - p0 : 0u;
          fm_lo = zero_bytes(diff_lo) & okq_lo & acgt_bytes(b0_lo) & low_bytes_mask(covered) & rm_lo;
          fm_hi = zero_bytes(diff_hi) & okq_hi & acgt_bytes(b0_hi) &
                  low_bytes_mask(covered > 4u ? covered - 4u : 0u) & rm_hi;
        }
      }
      // proven positions: constant quality, depth n, no errors
      const uint32_t fb_lo = (fm_lo >> 7) * 0xFFu, fb_hi = (fm_hi >> 7) * 0xFFu;
      wb_lo = (fast_masked ? 0x4E4E4E4Eu : b0_lo) & fb_lo;
      wb_hi = (fast_masked ? 0x4E4E4E4Eu : b0_hi) & fb_hi;
      wq_lo = fq4 & fb_lo;
      wq_hi = fq4 & fb_hi;
      const uint32_t nn = n | (n << 16);
      // expand byte mask pairs to u16 pairs: bytes (0,1) -> dep.x, (2,3) -> dep.y, ...
      dep.x = nn & __byte_perm(fb_lo, 0u, 0x1100u);
      dep.y = nn & __byte_perm(fb_lo, 0u, 0x3322u);
      dep.z = nn & __byte_perm(fb_hi, 0u, 0x1100u);
      dep.w = nn & __byte_perm(fb_hi, 0u, 0x3322u);
      ls.nocall += fast_masked ? (__popc(fm_lo) + __popc(fm_hi)) : 0;
      todo_lo = rm_lo & ~fm_lo; todo_hi = rm_hi & ~fm_hi;
      if (todo_lo | todo_hi) {
        // undecided positions go to this warp's queue; if it is full they are resolved in place,
        // after the item's words have been stored (below)
        const uint32_t cnt = static_cast<uint32_t>(__popc(todo_lo) + __popc(todo_hi));
        uint32_t slot = atomicAdd(wcount, cnt);
        const uint32_t ent = (u << 16) | p0;
        uint32_t keep_lo = 0, keep_hi = 0;
        for (uint32_t t = todo_lo; t; t &= t - 1u, ++slot) {
          if (slot < kWarpQueueCap) wqueue[slot] = ent + ((__ffs(t) - 1) >> 3);
          else keep_lo |= t & (0u - t);
        }
        for (uint32_t t = todo_hi; t; t &= t - 1u, ++slot) {
          if (slot < kWarpQueueCap) wqueue[slot] = ent + 4u + ((__ffs(t) - 1) >> 3);
          else keep_hi |= t & (0u - t);
        }
        todo_lo = keep_lo; todo_hi = keep_hi;
      }
    }
    *reinterpret_cast<uint2*>(a.out_base + o) = make_uint2(wb_lo, wb_hi);
    *reinterpret_cast<uint2*>(a.out_qual + o) = make_uint2(wq_lo, wq_hi);
    *reinterpret_cast<uint4*>(a.out_depth + o) = dep;
    *reinterpret_cast<uint4*>(a.out_errors + o) = err;
    if (todo_lo | todo_hi) {                    // rare: the warp queue overflowed
      for (uint32_t j = 0; j < 8u; ++j) {
        if ((j < 4u ? todo_lo >> (8u * j) : todo_hi >> (8u * (j - 4u))) & 0x80u) {
          Called c = resolve_position<M, false>(tv, S, rb, n, p0 + j, a, ls);
          write_called(a, o + j, c);
        }
      }
    }
  }
  __syncwarp();

#if FGB_PIPE_TRACE
  if (lane == 0) g_trace_mark[warp] = clock64();
#endif

  // ---------------- SLOW PASS: this warp's undecided positions ----------------
  // (a queued position's word was stored above by a lane of this same warp: program order within
  //  the warp + __syncwarp() orders the byte stores below after it)
  uint32_t qn = *wcount;
  qn = qn < kWarpQueueCap ? qn : kWarpQueueCap;
  if (qn) slow_pass<M, V == 1>(a, S, st, tv, wqueue, qn, lane, ls);
  __syncwarp();
  if (lane == 0) *wcount = 0;
}


// Deep-class tiles (every unit has at least kDeepMin reads): a tile is one to five units, 19 .. 95 items --
// too few to keep 256 threads busy one item each, and every item is a walk over 24 .. 512 rows.  So a GROUP
// of g lanes (g = 2^k, chosen per tile so that items * g fills the CTA) shares an item: lane `sub` walks rows
// sub, sub + g, ..., a __shfl_xor butterfly folds the partial masks, and the group's first lane finishes the
// item exactly as vote_tile does.  Undecided positions are resolved by the warp-wide slow pass.
template <class M, bool Regular>
__device__ __forceinline__ void vote_tile_deep(const VoteArgs& a, VoteSmem& S, const Stage& st,
                                               const TileView<M>& tv, uint32_t tid, uint32_t warp,
                                               uint32_t n_items, LocalStats& ls) {
  const uint32_t lane = tid & 31u;
  const uint32_t n_units = st.tile.n_units;
  const uint64_t out0 = st.units[0].out_off;
  const uint32_t min_reads = a.min_reads, min_cons_q = a.min_cons_q, fast_qual = a.fast_qual;
  const uint32_t reg_len = st.units[0].cons_len;
  const uint32_t reg_row0 = (st.tile.flags & kTileFlagSkew8) ? 8u : 0u;
  const bool fast_masked = fast_qual < min_cons_q;
  const uint32_t fq4 = (fast_masked ? 2u : fast_qual) * 0x01010101u;
  const uint32_t uni_m = st.tile.flags >> 8;
  const uint32_t uni_recip = st.aux[0];
  const uint32_t base32 = static_cast<uint32_t>(tv.byte_base);
  uint32_t* const wqueue = S.queue[warp];
  uint32_t* const wcount = &S.q_count[warp];
  // lanes per item: the largest power of two with n_items * g <= kVoteThreads (at least 1, at most 32)
  uint32_t gs = 0;
  while (gs < 5u && (n_items << (gs + 1u)) <= static_cast<uint32_t>(kVoteThreads)) ++gs;
  const uint32_t g = 1u << gs;
  const uint32_t sub = tid & (g - 1u);
  const uint32_t per_round = static_cast<uint32_t>(kVoteThreads) >> gs;

  // group j of warp w takes item base + j * 8 + w: the items -- and with them the queued positions -- are spread
  // over all eight warps even when a tile has only 19 of them
  const uint32_t in_round = ((lane >> gs) << 3) + warp;
  for (uint32_t base = 0; base < n_items; base += per_round) {
    const uint32_t item_raw = base + in_round;
    const bool valid = item_raw < n_items;                  // idle groups shadow the last item; nothing of theirs is stored
    const uint32_t item = valid ? item_raw : n_items - 1u;
    uint32_t u;
    if (Regular || uni_m) {
      u = __umulhi(item, uni_recip);
    } else {
      uint32_t lo = 0, hi = n_units;
      while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        const uint32_t start = static_cast<uint32_t>((st.units[mid].out_off - out0) >> 3);
        if (start <= item) lo = mid; else hi = mid;
      }
      u = lo;
    }
    const fgb_unit un = st.units[u];
    const uint32_t rb = un.read_begin;
    const uint32_t n = st.units[u + 1].read_begin - rb;
    const uint32_t cons_len = un.cons_len;
    const uint64_t o = out0 + (static_cast<uint64_t>(item) << 3);
    const uint32_t p0 = Regular ? (item - u * uni_m) << 3
                                : (item - static_cast<uint32_t>((un.out_off - out0) >> 3)) << 3;
    const uint32_t real = cons_len - p0 < 8u ? cons_len - p0 : 8u;
    const uint32_t rm_lo = low_bytes_mask(real), rm_hi = low_bytes_mask(real > 4u ? real - 4u : 0u);
    // One quality threshold per unit: the near-unanimous one when the depth has it (it also proves the
    // unanimous positions: it is never below qt[n]), else the unanimous one alone.
    const uint32_t qt_near = S.qt3[n < kQtEntries ? n : kQtEntries - 1];
    const bool near_ok = qt_near <= FGB_MAX_PHRED;
    const uint32_t qt = near_ok ? qt_near : S.qt[n < kQtEntries ? n : kQtEntries - 1];
    const bool fast_ok = (qt <= FGB_MAX_PHRED) && (n >= min_reads) && (n <= 0xFFFFu) && n >= 2u;
    if (n == 1u) {
      // a single-read unit never belongs to a deep tile (planner); kept correct for hand-made tile arrays:
      // the group's first lane applies the single-input rule (vanilla_caller.rs:1285-1316) position by position
      if (valid && sub == 0) {
        const uint64_t d = M::ld64(tv.reads + static_cast<typename M::off_t>(rb - tv.read_base) * 8u);
        const uint32_t len = static_cast<uint32_t>(d & 0xFFFFu);
        for (uint32_t j = 0; j < real; ++j) {
          const uint32_t pos = p0 + j;
          Called c; c.base = 'N'; c.qual = 2; c.depth = 0; c.errors = 0;
          if (pos < len) {
            const typename M::off_t row = static_cast<typename M::off_t>((d >> 16) - tv.byte_base) + pos;
            const uint32_t b = M::ld8(tv.bases + row), q = M::ld8(tv.quals + row);
            const uint32_t adj = q < FGB_NTABLE ? S.single_q[q] : 0u;
            if (adj >= min_cons_q) { c.base = b; c.qual = adj; }
            c.depth = (b != 'N');
          }
          ls.nocall += (c.base == 'N');
          write_called(a, o + j, c);
        }
        ls.positions += real;
      }
      __syncwarp();
      continue;
    }
    uint32_t b0_lo = 0, b0_hi = 0;
    uint32_t diff_lo = 0, diff_hi = 0, okq_lo = 0x80808080u, okq_hi = 0x80808080u, minlen = 0xFFFFFFFFu;
    // rows that differ from read 0 somewhere in the word (rare): per byte, how many rows differ, and whether a
    // differing row holds anything but A/C/G/T there (such an observation is not counted at all, base_builder.rs:300)
    uint32_t cnt_lo = 0, cnt_hi = 0, bad_lo = 0, bad_hi = 0;
    auto dissent = [&](uint32_t wl, uint32_t wh, uint32_t xl, uint32_t xh) {
      const uint32_t ml = ~zero_bytes(xl) & 0x80808080u, mh = ~zero_bytes(xh) & 0x80808080u;
      bad_lo |= ml & ~acgt_bytes(wl); bad_hi |= mh & ~acgt_bytes(wh);
      cnt_lo += ml >> 7; cnt_hi += mh >> 7;
    };
    if (fast_ok) {
      const uint32_t tsplat = qt * 0x01010101u;
      if (Regular) {
        const uint32_t step = uni_m * 8u;
        typename M::addr_t pb = tv.bases + reg_row0 + ((rb - st.tile.read_begin) * uni_m + (p0 >> 3)) * 8u;
        {
          const uint64_t w = M::ld64(pb);
          b0_lo = static_cast<uint32_t>(w); b0_hi = static_cast<uint32_t>(w >> 32);
        }
        pb += sub * step;
        const uint32_t gstep = step << gs;
#pragma unroll 4
        for (uint32_t r = sub; r < n; r += g, pb += gstep) {
          const uint64_t wb = M::ld64(pb);
          const uint64_t wq = M::ld64(pb + kTileCapBytes);
          const uint32_t xl = static_cast<uint32_t>(wb) ^ b0_lo, xh = static_cast<uint32_t>(wb >> 32) ^ b0_hi;
          diff_lo |= xl; diff_hi |= xh;
          if (xl | xh) dissent(static_cast<uint32_t>(wb), static_cast<uint32_t>(wb >> 32), xl, xh);
          okq_lo &= (static_cast<uint32_t>(wq) | 0x80808080u) - tsplat;
          okq_hi &= (static_cast<uint32_t>(wq >> 32) | 0x80808080u) - tsplat;
        }
        minlen = reg_len;
      } else {
        typename M::addr_t rd = tv.reads + static_cast<typename M::off_t>(rb - tv.read_base) * 8u;
        {
          const uint64_t d = M::ld64(rd);
          const uint32_t len = static_cast<uint32_t>(d) & 0xFFFFu;
          const uint64_t w = M::ld64(tv.bases + M::row_offset(d, tv.byte_base, base32) + (len > p0 ? p0 : 0u));
          b0_lo = static_cast<uint32_t>(w); b0_hi = static_cast<uint32_t>(w >> 32);
        }
#pragma unroll 4
        for (uint32_t r = sub; r < n; r += g) {
          const uint64_t d = M::ld64(rd + r * 8u);
          const uint32_t len = static_cast<uint32_t>(d) & 0xFFFFu;
          minlen = len < minlen ? len : minlen;
          const typename M::off_t row = M::row_offset(d, tv.byte_base, base32) + (len > p0 ? p0 : 0u);
          const uint64_t wb = M::ld64(tv.bases + row);
          const uint64_t wq = M::ld64(tv.quals + row);
          const uint32_t xl = static_cast<uint32_t>(wb) ^ b0_lo, xh = static_cast<uint32_t>(wb >> 32) ^ b0_hi;
          diff_lo |= xl; diff_hi |= xh;
          if (xl | xh) dissent(static_cast<uint32_t>(wb), static_cast<uint32_t>(wb >> 32), xl, xh);
          okq_lo &= (static_cast<uint32_t>(wq) | 0x80808080u) - tsplat;
          okq_hi &= (static_cast<uint32_t>(wq >> 32) | 0x80808080u) - tsplat;
        }
      }
    }
    // fold the group (every lane of the warp takes part; groups are aligned runs of g lanes)
    for (uint32_t off = g >> 1; off > 0; off >>= 1) {
      diff_lo |= __shfl_xor_sync(0xFFFFFFFFu, diff_lo, off);
      diff_hi |= __shfl_xor_sync(0xFFFFFFFFu, diff_hi, off);
      okq_lo &= __shfl_xor_sync(0xFFFFFFFFu, okq_lo, off);
      okq_hi &= __shfl_xor_sync(0xFFFFFFFFu, okq_hi, off);
      const uint32_t ml = __shfl_xor_sync(0xFFFFFFFFu, minlen, off);
      minlen = ml < minlen ? ml : minlen;
      if (near_ok) {                                        // warp-uniform per group; byte counters stay below 256 (n < 255)
        cnt_lo += __shfl_xor_sync(0xFFFFFFFFu, cnt_lo, off);
        cnt_hi += __shfl_xor_sync(0xFFFFFFFFu, cnt_hi, off);
        bad_lo |= __shfl_xor_sync(0xFFFFFFFFu, bad_lo, off);
        bad_hi |= __shfl_xor_sync(0xFFFFFFFFu, bad_hi, off);
      }
    }
    if (valid && sub == 0) {
      uint32_t fm_lo = 0, fm_hi = 0;
      uint4 errw = make_uint4(0, 0, 0, 0);
      if (fast_ok) {
        const uint32_t covered = minlen > p0 ? minlen - p0 : 0u;
        const uint32_t base_lo = okq_lo & acgt_bytes(b0_lo) & low_bytes_mask(covered) & rm_lo;
        const uint32_t base_hi = okq_hi & acgt_bytes(b0_hi) & low_bytes_mask(covered > 4u ? covered - 4u : 0u) & rm_hi;
        fm_lo = zero_bytes(diff_lo) & base_lo;
        fm_hi = zero_bytes(diff_hi) & base_hi;
        if (near_ok && (cnt_lo | cnt_hi)) {
          // near-unanimous positions: at most kNearK rows differ, all of them A/C/G/T: the dominant-winner proof
          // holds (host_tables.cpp qt3): read 0's base wins with phred(ln_pre), depth n, errors = the count
          const uint32_t le_lo = ~((cnt_lo | 0x80808080u) - 0x04040404u) & ~cnt_lo & 0x80808080u;   // cnt <= 3
          const uint32_t le_hi = ~((cnt_hi | 0x80808080u) - 0x04040404u) & ~cnt_hi & 0x80808080u;
          const uint32_t nm_lo = base_lo & le_lo & ~bad_lo & ~fm_lo, nm_hi = base_hi & le_hi & ~bad_hi & ~fm_hi;
          const uint32_t el = cnt_lo & spread_msb(nm_lo), eh = cnt_hi & spread_msb(nm_hi);
          errw = make_uint4(__byte_perm(el, 0u, 0x4140u), __byte_perm(el, 0u, 0x4342u),
                            __byte_perm(eh, 0u, 0x4140u), __byte_perm(eh, 0u, 0x4342u));
          fm_lo |= nm_lo; fm_hi |= nm_hi;
        }
      }
      const uint32_t fb_lo = spread_msb(fm_lo), fb_hi = spread_msb(fm_hi);
      const uint32_t wb_lo = (fast_masked ? 0x4E4E4E4Eu : b0_lo) & fb_lo;
      const uint32_t wb_hi = (fast_masked ? 0x4E4E4E4Eu : b0_hi) & fb_hi;
      const uint32_t nn = n | (n << 16);
      uint4 dep;
      dep.x = nn & __byte_perm(fb_lo, 0u, 0x1100u);
      dep.y = nn & __byte_perm(fb_lo, 0u, 0x3322u);
      dep.z = nn & __byte_perm(fb_hi, 0u, 0x1100u);
      dep.w = nn & __byte_perm(fb_hi, 0u, 0x3322u);
      ls.nocall += fast_masked ? (__popc(fm_lo) + __popc(fm_hi)) : 0;
      ls.positions += real;
      *reinterpret_cast<uint2*>(a.out_base + o) = make_uint2(wb_lo, wb_hi);
      *reinterpret_cast<uint2*>(a.out_qual + o) = make_uint2(fq4 & fb_lo, fq4 & fb_hi);
      *reinterpret_cast<uint4*>(a.out_depth + o) = dep;
      *reinterpret_cast<uint4*>(a.out_errors + o) = errw;
      uint32_t todo_lo = rm_lo & ~fm_lo, todo_hi = rm_hi & ~fm_hi;
      if (todo_lo | todo_hi) {
        const uint32_t cnt = static_cast<uint32_t>(__popc(todo_lo) + __popc(todo_hi));
        uint32_t slot = atomicAdd(wcount, cnt);
        const uint32_t ent = (u << 16) | p0;
        uint32_t keep_lo = 0, keep_hi = 0;
        for (uint32_t t = todo_lo; t; t &= t - 1u, ++slot) {
          if (slot < kWarpQueueCap) wqueue[slot] = ent + ((__ffs(t) - 1) >> 3);
          else keep_lo |= t & (0u - t);
        }
        for (uint32_t t = todo_hi; t; t &= t - 1u, ++slot) {
          if (slot < kWarpQueueCap) wqueue[slot] = ent + 4u + ((__ffs(t) - 1) >> 3);
          else keep_hi |= t & (0u - t);
        }
        if (keep_lo | keep_hi) {                             // rare: the warp queue overflowed
          for (uint32_t j = 0; j < 8u; ++j) {
            if ((j < 4u ? keep_lo >> (8u * j) : keep_hi >> (8u * (j - 4u))) & 0x80u) {
              const Called c = resolve_position<M>(tv, S, rb, n, p0 + j, a, ls);
              write_called(a, o + j, c);
            }
          }
        }
      }
    }
    __syncwarp();
  }
  __syncwarp();
  uint32_t qn = *wcount;
  qn = qn < kWarpQueueCap ? qn : kWarpQueueCap;
  if (qn) {
    // eight lanes per queued position (four positions per pass) as long as a lane's share of the rows stays
    // short; the whole warp per position for the oversize units voted from HBM
    if (st.tile.flags & kTileFlagDirect) slow_pass_g<M, 32u>(a, S, st, tv, wqueue, qn, lane, ls);
    else slow_pass_g<M, 8u>(a, S, st, tv, wqueue, qn, lane, ls);
  }
  __syncwarp();
  if (lane == 0) *wcount = 0;
}

// Deep-class tiles, second form (shared-memory tiles of at most kDeepItemsMax items -- every tile the planner
// cuts for this class).  The (item, row) plane of the tile is dealt flat to the 256 voting threads: thread t walks
// rows grp, grp + G, ... of item t mod n_items, G = 256 / n_items.  Lanes of a warp then read CONSECUTIVE words of one
// row (no bank conflicts; the group-of-lanes form above strides over rows), 247 of 256 threads work on a 19-item tile
// (152 with lane groups), and nothing is folded by shuffles: a thread whose partial result is not the identity --
// a dissenting row, a low quality -- merges it into the item's slot in shared memory with an atomic.  One named
// barrier per tile separates the walk from the finish; the finish of item i runs on lane i / 8 of warp i mod 8, so the
// queued positions are spread over all warps.  The slots are double-buffered by tile parity: the finisher resets the
// slot it read, two tiles before its next use.
constexpr uint32_t kDeepItemsMax = 112u;        // >= kTileCapBytes / (8 * kDeepMin) = 106
struct DeepSlots {
  uint32_t diff_lo[kDeepItemsMax], diff_hi[kDeepItemsMax];
  uint32_t okq_lo[kDeepItemsMax], okq_hi[kDeepItemsMax];
  uint32_t cnt_lo[kDeepItemsMax], cnt_hi[kDeepItemsMax];
  uint32_t bad_lo[kDeepItemsMax], bad_hi[kDeepItemsMax];
  uint32_t minlen[kDeepItemsMax];
};
constexpr uint32_t kDeepSmemBytes = 2u * sizeof(DeepSlots);

__device__ __forceinline__ void consumer_barrier() {      // the eight voting warps (the producer warp is not part of it)
  asm volatile("bar.sync 1, %0;" ::"n"(kVoteThreads) : "memory");
}

template <bool Regular>
__device__ __forceinline__ void vote_tile_deep_flat(const VoteArgs& a, VoteSmem& S, DeepSlots& R, const Stage& st,
                                                    const TileView<ShMem>& tv, uint32_t tid, uint32_t warp,
                                                    uint32_t n_items, LocalStats& ls) {
  using M = ShMem;
  const uint32_t lane = tid & 31u;
  const uint32_t n_units = st.tile.n_units;
  const uint64_t out0 = st.units[0].out_off;
  const uint32_t min_reads = a.min_reads, min_cons_q = a.min_cons_q, fast_qual = a.fast_qual;
  const uint32_t reg_len = st.units[0].cons_len;
  const uint32_t reg_row0 = (st.tile.flags & kTileFlagSkew8) ? 8u : 0u;
  const bool fast_masked = fast_qual < min_cons_q;
  const uint32_t fq4 = (fast_masked ? 2u : fast_qual) * 0x01010101u;
  const uint32_t uni_m = st.tile.flags >> 8;
  const uint32_t uni_recip = st.aux[0];
  const uint32_t base32 = static_cast<uint32_t>(tv.byte_base);
  uint32_t* const wqueue = S.queue[warp];
  uint32_t* const wcount = &S.q_count[warp];

  struct Item {
    uint32_t u, rb, n, cons_len, p0, qt;
    bool near_ok, fast_ok;
  };
  auto locate = [&](uint32_t item) {
    Item it;
    if (Regular || uni_m) {
      it.u = __umulhi(item, uni_recip);
    } else {
      uint32_t lo = 0, hi = n_units;
      while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        const uint32_t start = static_cast<uint32_t>((st.units[mid].out_off - out0) >> 3);
        if (start <= item) lo = mid; else hi = mid;
      }
      it.u = lo;
    }
    const fgb_unit un = st.units[it.u];
    it.rb = un.read_begin;
    it.n = st.units[it.u + 1].read_begin - it.rb;
    it.cons_len = un.cons_len;
    it.p0 = Regular ? (item - it.u * uni_m) << 3 : (item - static_cast<uint32_t>((un.out_off - out0) >> 3)) << 3;
    // One quality threshold per unit: the near-unanimous one when the depth has it (it also proves the unanimous
    // positions: it is never below qt[n]), else the unanimous one alone.
    const uint32_t qt_near = S.qt3[it.n < kQtEntries ? it.n : kQtEntries - 1];
    it.near_ok = qt_near <= FGB_MAX_PHRED;
    it.qt = it.near_ok ? qt_near : S.qt[it.n < kQtEntries ? it.n : kQtEntries - 1];
    it.fast_ok = (it.qt <= FGB_MAX_PHRED) && (it.n >= min_reads) && (it.n <= 0xFFFFu) && it.n >= 2u;
    return it;
  };
  // read 0's word of the item: the reference every row is compared with
  auto ref_word = [&](const Item& it, uint32_t& b0_lo, uint32_t& b0_hi) {
    uint64_t w;
    if (Regular) {
      w = M::ld64(tv.bases + reg_row0 + ((it.rb - st.tile.read_begin) * uni_m + (it.p0 >> 3)) * 8u);
    } else {
      const uint64_t d = M::ld64(tv.reads + static_cast<typename M::off_t>(it.rb - tv.read_base) * 8u);
      const uint32_t len = static_cast<uint32_t>(d) & 0xFFFFu;
      w = M::ld64(tv.bases + M::row_offset(d, tv.byte_base, base32) + (len > it.p0 ? it.p0 : 0u));
    }
    b0_lo = static_cast<uint32_t>(w); b0_hi = static_cast<uint32_t>(w >> 32);
  };

  // ---------------- WALK: thread t -> item t mod n_items, rows grp, grp + G, ... ----------------
  const uint32_t G = n_items ? static_cast<uint32_t>(kVoteThreads) / n_items : 0u;   // >= 2 (n_items <= kDeepItemsMax)
  const uint32_t grp = n_items > 1u ? __umulhi(tid, 0xFFFFFFFFu / n_items + 1u) : tid;   // tid / n_items, exact for these sizes
  if (grp < G) {
    const uint32_t item = tid - grp * n_items;
    const Item it = locate(item);
    if (it.fast_ok && grp < it.n) {
      uint32_t b0_lo, b0_hi;
      ref_word(it, b0_lo, b0_hi);
      const uint32_t tsplat = it.qt * 0x01010101u;
      uint32_t diff_lo = 0, diff_hi = 0, okq_lo = 0x80808080u, okq_hi = 0x80808080u, minlen = 0xFFFFFFFFu;
      // rows that differ from read 0 somewhere in the word (rare): per byte, how many rows differ, and whether a
      // differing row holds anything but A/C/G/T there (such an observation is not counted at all, base_builder.rs:300)
      uint32_t cnt_lo = 0, cnt_hi = 0, bad_lo = 0, bad_hi = 0;
      auto dissent = [&](uint32_t wl, uint32_t wh, uint32_t xl, uint32_t xh) {
        const uint32_t ml = ~zero_bytes(xl) & 0x80808080u, mh = ~zero_bytes(xh) & 0x80808080u;
        bad_lo |= ml & ~acgt_bytes(wl); bad_hi |= mh & ~acgt_bytes(wh);
        cnt_lo += ml >> 7; cnt_hi += mh >> 7;
      };
      if (Regular) {
        const uint32_t step = uni_m * 8u;
        typename M::addr_t pb = tv.bases + reg_row0 + ((it.rb - st.tile.read_begin + grp) * uni_m + (it.p0 >> 3)) * 8u;
        const uint32_t gstep = step * G;
#pragma unroll 4
        for (uint32_t r = grp; r < it.n; r += G, pb += gstep) {
          const uint64_t wb = M::ld64(pb);
          const uint64_t wq = M::ld64(pb + kTileCapBytes);
          const uint32_t xl = static_cast<uint32_t>(wb) ^ b0_lo, xh = static_cast<uint32_t>(wb >> 32) ^ b0_hi;
          diff_lo |= xl; diff_hi |= xh;
          if (xl | xh) dissent(static_cast<uint32_t>(wb), static_cast<uint32_t>(wb >> 32), xl, xh);
          okq_lo &= (static_cast<uint32_t>(wq) | 0x80808080u) - tsplat;
          okq_hi &= (static_cast<uint32_t>(wq >> 32) | 0x80808080u) - tsplat;
        }
      } else {
        typename M::addr_t rd = tv.reads + static_cast<typename M::off_t>(it.rb - tv.read_base) * 8u;
#pragma unroll 4
        for (uint32_t r = grp; r < it.n; r += G) {
          const uint64_t d = M::ld64(rd + r * 8u);
          const uint32_t len = static_cast<uint32_t>(d) & 0xFFFFu;
          minlen = len < minlen ? len : minlen;
          const typename M::off_t row = M::row_offset(d, tv.byte_base, base32) + (len > it.p0 ? it.p0 : 0u);
          const uint64_t wb = M::ld64(tv.bases + row);
          const uint64_t wq = M::ld64(tv.quals + row);
          const uint32_t xl = static_cast<uint32_t>(wb) ^ b0_lo, xh = static_cast<uint32_t>(wb >> 32) ^ b0_hi;
          diff_lo |= xl; diff_hi |= xh;
          if (xl | xh) dissent(static_cast<uint32_t>(wb), static_cast<uint32_t>(wb >> 32), xl, xh);
          okq_lo &= (static_cast<uint32_t>(wq) | 0x80808080u) - tsplat;
          okq_hi &= (static_cast<uint32_t>(wq >> 32) | 0x80808080u) - tsplat;
        }
        if (minlen != 0xFFFFFFFFu) atomicMin(&R.minlen[item], minlen);
      }
      // merge what is not the identity (a unanimous, well-covered, high-quality word merges nothing)
      if (diff_lo) atomicOr(&R.diff_lo[item], diff_lo);
      if (diff_hi) atomicOr(&R.diff_hi[item], diff_hi);
      if (okq_lo != 0x80808080u) atomicAnd(&R.okq_lo[item], okq_lo);
      if (okq_hi != 0x80808080u) atomicAnd(&R.okq_hi[item], okq_hi);
      if (cnt_lo) atomicAdd(&R.cnt_lo[item], cnt_lo);        // byte counters: at most n < 255 rows differ
      if (cnt_hi) atomicAdd(&R.cnt_hi[item], cnt_hi);
      if (bad_lo) atomicOr(&R.bad_lo[item], bad_lo);
      if (bad_hi) atomicOr(&R.bad_hi[item], bad_hi);
    }
  }
  consumer_barrier();

  // ---------------- FINISH: item i on lane i / 8 of warp i mod 8 ----------------
  {
    const uint32_t item = (lane << 3) + warp;
    if (item < n_items) {
      const Item it = locate(item);
      const uint32_t real = it.cons_len - it.p0 < 8u ? it.cons_len - it.p0 : 8u;
      const uint32_t rm_lo = low_bytes_mask(real), rm_hi = low_bytes_mask(real > 4u ? real - 4u : 0u);
      const uint64_t o = out0 + (static_cast<uint64_t>(item) << 3);
      const uint32_t n = it.n, rb = it.rb, p0 = it.p0;
      if (n == 1u) {
        // a single-read unit never belongs to a deep tile (planner); kept correct for hand-made tile arrays:
        // the single-input rule (vanilla_caller.rs:1285-1316) position by position
        const uint64_t d = M::ld64(tv.reads + static_cast<typename M::off_t>(rb - tv.read_base) * 8u);
        const uint32_t len = static_cast<uint32_t>(d & 0xFFFFu);
        for (uint32_t j = 0; j < real; ++j) {
          const uint32_t pos = p0 + j;
          Called c; c.base = 'N'; c.qual = 2; c.depth = 0; c.errors = 0;
          if (pos < len) {
            const typename M::off_t row = static_cast<typename M::off_t>((d >> 16) - tv.byte_base) + pos;
            const uint32_t b = M::ld8(tv.bases + row), q = M::ld8(tv.quals + row);
            const uint32_t adj = q < FGB_NTABLE ? S.single_q[q] : 0u;
            if (adj >= min_cons_q) { c.base = b; c.qual = adj; }
            c.depth = (b != 'N');
          }
          ls.nocall += (c.base == 'N');
          write_called(a, o + j, c);
        }
        ls.positions += real;
      } else {
        uint32_t b0_lo = 0, b0_hi = 0;
        uint32_t fm_lo = 0, fm_hi = 0;
        uint4 errw = make_uint4(0, 0, 0, 0);
        if (it.fast_ok) {
          ref_word(it, b0_lo, b0_hi);
          const uint32_t diff_lo = R.diff_lo[item], diff_hi = R.diff_hi[item];
          const uint32_t okq_lo = R.okq_lo[item], okq_hi = R.okq_hi[item];
          const uint32_t cnt_lo = R.cnt_lo[item], cnt_hi = R.cnt_hi[item];
          const uint32_t bad_lo = R.bad_lo[item], bad_hi = R.bad_hi[item];
          const uint32_t minlen = Regular ? reg_len : R.minlen[item];
          // back to the identities for this slot's next tile (two tiles from now, behind another barrier)
          if (diff_lo) R.diff_lo[item] = 0u;
          if (diff_hi) R.diff_hi[item] = 0u;
          if (okq_lo != 0x80808080u) R.okq_lo[item] = 0x80808080u;
          if (okq_hi != 0x80808080u) R.okq_hi[item] = 0x80808080u;
          if (cnt_lo) R.cnt_lo[item] = 0u;
          if (cnt_hi) R.cnt_hi[item] = 0u;
          if (bad_lo) R.bad_lo[item] = 0u;
          if (bad_hi) R.bad_hi[item] = 0u;
          if (!Regular) R.minlen[item] = 0xFFFFFFFFu;
          const uint32_t covered = minlen > p0 ? minlen - p0 : 0u;
          const uint32_t base_lo = okq_lo & acgt_bytes(b0_lo) & low_bytes_mask(covered) & rm_lo;
          const uint32_t base_hi = okq_hi & acgt_bytes(b0_hi) & low_bytes_mask(covered > 4u ? covered - 4u : 0u) & rm_hi;
          fm_lo = zero_bytes(diff_lo) & base_lo;
          fm_hi = zero_bytes(diff_hi) & base_hi;
          if (it.near_ok && (cnt_lo | cnt_hi)) {
            // near-unanimous positions: at most kNearK rows differ, all of them A/C/G/T: the dominant-winner proof
            // holds (host_tables.cpp qt3): read 0's base wins with phred(ln_pre), depth n, errors = the count
            const uint32_t le_lo = ~((cnt_lo | 0x80808080u) - 0x04040404u) & ~cnt_lo & 0x80808080u;   // cnt <= 3
            const uint32_t le_hi = ~((cnt_hi | 0x80808080u) - 0x04040404u) & ~cnt_hi & 0x80808080u;
            const uint32_t nm_lo = base_lo & le_lo & ~bad_lo & ~fm_lo, nm_hi = base_hi & le_hi & ~bad_hi & ~fm_hi;
            const uint32_t el = cnt_lo & spread_msb(nm_lo), eh = cnt_hi & spread_msb(nm_hi);
            errw = make_uint4(__byte_perm(el, 0u, 0x4140u), __byte_perm(el, 0u, 0x4342u),
                              __byte_perm(eh, 0u, 0x4140u), __byte_perm(eh, 0u, 0x4342u));
            fm_lo |= nm_lo; fm_hi |= nm_hi;
          }
        }
        const uint32_t fb_lo = spread_msb(fm_lo), fb_hi = spread_msb(fm_hi);
        const uint32_t wb_lo = (fast_masked ? 0x4E4E4E4Eu : b0_lo) & fb_lo;
        const uint32_t wb_hi = (fast_masked ? 0x4E4E4E4Eu : b0_hi) & fb_hi;
        const uint32_t nn = n | (n << 16);
        uint4 dep;
        dep.x = nn & __byte_perm(fb_lo, 0u, 0x1100u);
        dep.y = nn & __byte_perm(fb_lo, 0u, 0x3322u);
        dep.z = nn & __byte_perm(fb_hi, 0u, 0x1100u);
        dep.w = nn & __byte_perm(fb_hi, 0u, 0x3322u);
        ls.nocall += fast_masked ? (__popc(fm_lo) + __popc(fm_hi)) : 0;
        ls.positions += real;
        *reinterpret_cast<uint2*>(a.out_base + o) = make_uint2(wb_lo, wb_hi);
        *reinterpret_cast<uint2*>(a.out_qual + o) = make_uint2(fq4 & fb_lo, fq4 & fb_hi);
        *reinterpret_cast<uint4*>(a.out_depth + o) = dep;
        *reinterpret_cast<uint4*>(a.out_errors + o) = errw;
        const uint32_t todo_lo = rm_lo & ~fm_lo, todo_hi = rm_hi & ~fm_hi;
        if (todo_lo | todo_hi) {
          const uint32_t cnt = static_cast<uint32_t>(__popc(todo_lo) + __popc(todo_hi));
          uint32_t slot = atomicAdd(wcount, cnt);
          const uint32_t ent = (it.u << 16) | p0;
          uint32_t keep_lo = 0, keep_hi = 0;
          for (uint32_t t = todo_lo; t; t &= t - 1u, ++slot) {
            if (slot < kWarpQueueCap) wqueue[slot] = ent + ((__ffs(t) - 1) >> 3);
            else keep_lo |= t & (0u - t);
          }
          for (uint32_t t = todo_hi; t; t &= t - 1u, ++slot) {
            if (slot < kWarpQueueCap) wqueue[slot] = ent + 4u + ((__ffs(t) - 1) >> 3);
            else keep_hi |= t & (0u - t);
          }
          if (keep_lo | keep_hi) {                             // rare: the warp queue overflowed
            for (uint32_t j = 0; j < 8u; ++j) {
              if ((j < 4u ? keep_lo >> (8u * j) : keep_hi >> (8u * (j - 4u))) & 0x80u) {
                const Called c = resolve_position<M>(tv, S, rb, n, p0 + j, a, ls);
                write_called(a, o + j, c);
              }
            }
          }
        }
      }
    }
  }
  __syncwarp();
  uint32_t qn = *wcount;
  qn = qn < kWarpQueueCap ? qn : kWarpQueueCap;
  if (qn) slow_pass_g<M, 8u>(a, S, st, tv, wqueue, qn, lane, ls);     // eight lanes per queued position
  __syncwarp();
  if (lane == 0) *wcount = 0;
}

#ifndef FGB_DEEP_FLAT_MIN
#define FGB_DEEP_FLAT_MIN 64      // the flat deep form takes single-unit tiles of at least this many reads
#endif

template <int V, bool Fused = false, class Args = VoteArgs>
__device__ __forceinline__ void vote_kernel_body(const Args& a) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  VoteSmem& S = *reinterpret_cast<VoteSmem*>(smem_raw);
  const uint32_t tid = threadIdx.x;
  const uint32_t warp = tid >> 5;

  for (uint32_t i = tid; i < FGB_NTABLE; i += kThreads) {
    S.correct[i] = a.tables->correct[i];
    S.err_alt[i] = a.tables->err_alt[i];
  }
  for (uint32_t i = tid; i < 96; i += kThreads) S.single_q[i] = a.tables->single_q[i];
  for (uint32_t i = tid; i < kQtEntries; i += kThreads) { S.qt[i] = a.tables->qt[i]; S.qt3[i] = a.tables->qt3[i]; }
  for (uint32_t i = tid; i < 96; i += kThreads) S.dfix[i] = a.tables->dfix[i];
  if (tid < kConsumerWarps) S.q_count[tid] = 0;
  if (V == 1) {                                             // the shallow kernel's in-line pair table
    uint32_t* dst = reinterpret_cast<uint32_t*>(smem_raw + sizeof(VoteSmem));
    const uint32_t* src = reinterpret_cast<const uint32_t*>(a.tables->pair_q);
    for (uint32_t i = tid; i < kPairSmemBytes / 4u; i += kThreads) dst[i] = __ldg(src + i);
    int32_t* ub = reinterpret_cast<int32_t*>(smem_raw + sizeof(VoteSmem) + kUgapSmemOff);
    for (uint32_t i = tid; i < 128u; i += kThreads) {
      ub[i] = a.tables->ugap_bp[i];
      reinterpret_cast<uint8_t*>(ub + 128)[i] = a.tables->ugap_q[i];
    }
  }
  if (V == 2) {                                             // the deep kernel's reduction slots: identities
    DeepSlots* R2 = reinterpret_cast<DeepSlots*>(smem_raw + sizeof(VoteSmem));
    for (uint32_t i = tid; i < 2u * kDeepItemsMax; i += kThreads) {
      DeepSlots& R = R2[i / kDeepItemsMax];
      const uint32_t j = i % kDeepItemsMax;
      R.diff_lo[j] = 0u; R.diff_hi[j] = 0u; R.okq_lo[j] = 0x80808080u; R.okq_hi[j] = 0x80808080u;
      R.cnt_lo[j] = 0u; R.cnt_hi[j] = 0u; R.bad_lo[j] = 0u; R.bad_hi[j] = 0u; R.minlen[j] = 0xFFFFFFFFu;
    }
  }
  if (tid == 0) {
    S.ln_pre = a.tables->ln_pre;
    S.g2fix = a.tables->g2fix;
    S.nmax2 = a.tables->nmax2;
    S.pair_q = a.tables->pair_q;
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&S.full[s], 1);                 // producer's arrive.expect_tx
      mbar_init(&S.empty[s], kConsumerWarps);   // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  const uint32_t grid = gridDim.x;
  const uint32_t n_tiles = static_cast<uint32_t>(a.n_tiles);   // < 2^32: fgb_plan_tiles bounds n_units

  if (warp == kConsumerWarps) {
    // ================= PRODUCER WARP: one elected lane drives the TMA pipeline =================
    if ((tid & 31u) == 0) {
      uint32_t k = 0;
      uint64_t n_units_done = 0, n_reads_done = 0;
#if FGB_PIPE_TRACE
      const long long tr_start = clock64();
      long long tr_empty = 0;
#endif
      // No L2 prefetch of the tiles ahead of the ring (cp.async.bulk.prefetch.L2): on the H100 a prefetch one grid
      // round ahead made the general kernel 21 % slower at depth 8 (DESIGN.md section 3).
      for (uint32_t t = blockIdx.x; t < n_tiles; t += grid, ++k) {
        const int s = k % kStages;
        const uint32_t use = k / kStages;
        if (use > 0) {                                          // consumers released the stage
#if FGB_PIPE_TRACE
          const long long tw = clock64();
#endif
          mbar_wait(&S.empty[s], (use - 1u) & 1u, V == 2 ? 1000u : 20000u);   // deep tiles are small: shorter naps
#if FGB_PIPE_TRACE
          tr_empty += clock64() - tw;
#endif
        }
        Stage& st = S.st[s];
        const uint4* gt = reinterpret_cast<const uint4*>(a.tiles + t);
        uint4 t0 = __ldg(gt), t1 = __ldg(gt + 1);
        *reinterpret_cast<uint4*>(&st.tile) = t0;
        *(reinterpret_cast<uint4*>(&st.tile) + 1) = t1;
        uint64_t byte_begin = (static_cast<uint64_t>(t0.y) << 32) | t0.x;
        uint32_t byte_len = t0.z, unit_begin = t0.w, n_units = t1.x, read_begin = t1.y,
                 n_reads = t1.z, flags = t1.w;
        uint32_t units_bytes = (n_units + 1u) * 16u;
        bool direct = (flags & kTileFlagDirect) != 0;
        uint32_t rskew = read_begin & 1u;
        uint32_t rbytes = ((n_reads + rskew + 1u) & ~1u) * 8u;
        uint32_t tx = units_bytes + (direct ? 0u : 2u * byte_len + rbytes);
        const uint32_t uni_m = flags >> 8;     // per-tile constants every consumer lane would otherwise derive
        st.aux[0] = uni_m ? 0xFFFFFFFFu / uni_m + 1u : 0u;
        st.aux[1] = uni_m * n_units;
        n_units_done += n_units; n_reads_done += n_reads;
#if FGB_PIPE_TRACE
        *reinterpret_cast<long long*>(&st.aux[2]) = clock64();   // issue time, read by consumer warp 0
#endif
        mbar_arrive_expect_tx(&S.full[s], tx);
        tma_load_1d(st.units, a.units + unit_begin, units_bytes, &S.full[s]);
        if (!direct) {
          if (byte_len) {
            tma_load_1d(st.bases, a.bases + byte_begin, byte_len, &S.full[s]);
            tma_load_1d(st.quals, a.quals + byte_begin, byte_len, &S.full[s]);
          }
          if (rbytes) tma_load_1d(st.reads, a.reads + (read_begin - rskew), rbytes, &S.full[s]);
        }
      }
      if (n_units_done) atomicAdd(a.counters + FGB_CTR_UNITS, static_cast<unsigned long long>(n_units_done));
      if (n_reads_done) atomicAdd(a.counters + FGB_CTR_INPUT_READS, static_cast<unsigned long long>(n_reads_done));
#if FGB_PIPE_TRACE
      atomicAdd(&g_pipe_trace[0], static_cast<unsigned long long>(clock64() - tr_start));
      atomicAdd(&g_pipe_trace[1], static_cast<unsigned long long>(tr_empty));
      atomicAdd(&g_pipe_trace[10], 1ull);
#endif
    }
    return;
  }

  // ================= CONSUMER WARPS =================
  LocalStats ls = {0, 0, 0};
  uint32_t combined = 0;
  uint32_t k = 0, rot = 0;
#if FGB_PIPE_TRACE
  const long long tr_start = clock64();
  long long tr_full = 0, tr_vote = 0, tr_fast = 0, tr_slow = 0, tr_lat = 0;
  uint32_t tr_late = 0, tr_tiles = 0;
#endif
  for (uint32_t t = blockIdx.x; t < n_tiles; t += grid, ++k) {
    const int s = k % kStages;
#if FGB_PIPE_TRACE
    const long long tw = clock64();
    const bool landed = mbar_test(&S.full[s], (k / kStages) & 1u);
#endif
    mbar_wait(&S.full[s], (k / kStages) & 1u, V == 2 ? 300u : 2000u);
    Stage& st = S.st[s];
#if FGB_PIPE_TRACE
    const long long tv0 = clock64();
    tr_full += tv0 - tw;
    ++tr_tiles;
    if (!landed) { ++tr_late; tr_lat += tv0 - *reinterpret_cast<const long long*>(&st.aux[2]); }
    if ((tid & 31u) == 0) g_trace_mark[warp] = -1;
#endif
    // rotating item assignment: the partial last round of a tile lands on different warps from
    // tile to tile, so every warp does the same work in the long run
    const uint32_t vt = (tid - rot) & (kVoteThreads - 1);
    uint32_t n_items = st.aux[1];
    if (n_items == 0)
      n_items = static_cast<uint32_t>((st.units[st.tile.n_units].out_off - st.units[0].out_off) >> 3);
    if (FGB_PIPE_NOVOTE) {
      const uint64_t out0 = st.units[0].out_off;
      for (uint32_t item = vt; item < n_items; item += kVoteThreads) {
        const uint64_t o = out0 + (static_cast<uint64_t>(item) << 3);
        *reinterpret_cast<uint2*>(a.out_base + o) = make_uint2(0x41414141u, 0x41414141u);
        *reinterpret_cast<uint2*>(a.out_qual + o) = make_uint2(0x1E1E1E1Eu, 0x1E1E1E1Eu);
        *reinterpret_cast<uint4*>(a.out_depth + o) = make_uint4(0, 0, 0, 0);
        *reinterpret_cast<uint4*>(a.out_errors + o) = make_uint4(0, 0, 0, 0);
      }
    } else if (st.tile.flags & kTileFlagDirect) {
      TileView<GlMem> tv;
      tv.bases = a.bases; tv.quals = a.quals;
      tv.reads = reinterpret_cast<const uint8_t*>(a.reads + st.tile.read_begin);
      tv.byte_base = 0; tv.read_base = st.tile.read_begin;
      if (V == 2) vote_tile_deep<GlMem, false>(a, S, st, tv, tid, warp, n_items, ls);
      else vote_tile<GlMem, false, V>(a, S, st, tv, vt, warp, n_items, ls);
    } else {
      TileView<ShMem> tv;
      tv.bases = st.bases; tv.quals = st.quals;
      tv.reads = reinterpret_cast<const uint8_t*>(st.reads) + (st.tile.read_begin & 1u) * 8u;
      tv.byte_base = st.tile.byte_begin; tv.read_base = st.tile.read_begin;
      if (V == 2) {
        // The flat form pays one CTA-wide barrier per tile: it wins only where a tile is one very deep unit (depth 100:
        // 0.49 -> 0.52 of the roofline; at depth 24-50 the lane-group form is 5-20 % faster, profiles/r02_depth_sweep_flat_deep.log)
        if (n_items <= kDeepItemsMax && st.tile.n_units == 1u && st.tile.n_reads >= FGB_DEEP_FLAT_MIN) {   // CTA-uniform
          DeepSlots& R = reinterpret_cast<DeepSlots*>(smem_raw + sizeof(VoteSmem))[k & 1u];
          if (st.tile.flags & kTileFlagRegular) vote_tile_deep_flat<true>(a, S, R, st, tv, tid, warp, n_items, ls);
          else vote_tile_deep_flat<false>(a, S, R, st, tv, tid, warp, n_items, ls);
        } else if (st.tile.flags & kTileFlagRegular) vote_tile_deep<ShMem, true>(a, S, st, tv, tid, warp, n_items, ls);
        else vote_tile_deep<ShMem, false>(a, S, st, tv, tid, warp, n_items, ls);
      } else {
        if (st.tile.flags & kTileFlagRegular) vote_tile<ShMem, true, V>(a, S, st, tv, vt, warp, n_items, ls);
        else vote_tile<ShMem, false, V>(a, S, st, tv, vt, warp, n_items, ls);
      }
      if constexpr (Fused) {
        const uint2 tj = __ldg(reinterpret_cast<const uint2*>(a.tile_jobs + t));   // {begin, count | max_items << 16}
        if (tj.y & 0xFFFFu) {                                  // CTA-uniform
          consumer_barrier();                                  // every SS word of the tile is written
          combined += duplex_epilogue(a, st, st.bases, tv.reads, static_cast<uint32_t>(st.tile.byte_begin),
                                      st.tile.read_begin, tj.x, tj.y & 0xFFFFu, tj.y >> 16, tid);
        }
      }
    }
    rot = (rot + n_items) & (kVoteThreads - 1);
    __syncwarp();
#if FGB_PIPE_TRACE
    {
      const long long tv1 = clock64(), mark = g_trace_mark[warp];
      tr_vote += tv1 - tv0;
      if (mark >= tv0) { tr_fast += mark - tv0; tr_slow += tv1 - mark; }
    }
#endif
    if ((tid & 31u) == 0) mbar_arrive(&S.empty[s]);   // this warp is done with stage s
  }
#if FGB_PIPE_TRACE
  if ((tid & 31u) == 0) {
    atomicAdd(&g_pipe_trace[2], static_cast<unsigned long long>(clock64() - tr_start));
    atomicAdd(&g_pipe_trace[3], static_cast<unsigned long long>(tr_full));
    atomicAdd(&g_pipe_trace[4], static_cast<unsigned long long>(tr_vote));
    atomicAdd(&g_pipe_trace[5], static_cast<unsigned long long>(tr_fast));
    atomicAdd(&g_pipe_trace[6], static_cast<unsigned long long>(tr_slow));
    if (warp == 0) {
      atomicAdd(&g_pipe_trace[7], static_cast<unsigned long long>(tr_late));
      atomicAdd(&g_pipe_trace[8], static_cast<unsigned long long>(tr_lat));
      atomicAdd(&g_pipe_trace[9], static_cast<unsigned long long>(tr_tiles));
    }
  }
#endif

  // ---- counters: warp-reduce, one atomic per warp ----
  uint32_t v0 = ls.positions, v1 = ls.exact, v2 = ls.nocall;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    v0 += __shfl_down_sync(0xFFFFFFFFu, v0, off);
    v1 += __shfl_down_sync(0xFFFFFFFFu, v1, off);
    v2 += __shfl_down_sync(0xFFFFFFFFu, v2, off);
  }
  if ((tid & 31u) == 0) {
    if (v0) atomicAdd(a.counters + FGB_CTR_POSITIONS, static_cast<unsigned long long>(v0));
    if (v1) atomicAdd(a.counters + FGB_CTR_EXACT_POSITIONS, static_cast<unsigned long long>(v1));
    if (v2) atomicAdd(a.counters + FGB_CTR_NOCALL_POSITIONS, static_cast<unsigned long long>(v2));
  }
  if constexpr (Fused) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) combined += __shfl_down_sync(0xFFFFFFFFu, combined, off);
    if ((tid & 31u) == 0 && combined) atomicAdd(a.counters + FGB_CTR_COMBINED, static_cast<unsigned long long>(combined));
  }
}


// Three instantiations, one per tile class (fgb_config.h): the planner cuts class-homogeneous tiles and the
// engine launches each kernel on its own run of the (class-sorted) tile array.  Every one of them is correct
// for any tile; they differ in how the work of a tile is dealt to the threads.  Two CTAs per SM is the design point
// (DESIGN.md section 3); without the minimum-blocks bound ptxas for sm_90a caps them at 72 registers and spills in
// the item loop.
__global__ void __launch_bounds__(kThreads, 2) vote_kernel(const VoteArgs a) { vote_kernel_body<0>(a); }
__global__ void __launch_bounds__(kThreads, 2) vote_kernel_shallow(const VoteArgs a) { vote_kernel_body<1>(a); }
__global__ void __launch_bounds__(kThreads, 2) vote_kernel_deep(const VoteArgs a) { vote_kernel_body<2>(a); }
// The same three with the duplex epilogue (fgb_vote_duplex_device).
__global__ void __launch_bounds__(kThreads, 2) vote_kernel_duplex(const VoteArgsDuplex a) { vote_kernel_body<0, true, VoteArgsDuplex>(a); }
__global__ void __launch_bounds__(kThreads, 2) vote_kernel_shallow_duplex(const VoteArgsDuplex a) { vote_kernel_body<1, true, VoteArgsDuplex>(a); }
__global__ void __launch_bounds__(kThreads, 2) vote_kernel_deep_duplex(const VoteArgsDuplex a) { vote_kernel_body<2, true, VoteArgsDuplex>(a); }

}  // namespace fgb
