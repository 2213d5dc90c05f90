// The per-template rules of `fgumi duplex-metrics` / `simplex-metrics`, written once for the host and the device
// (FGB_HD): the template pass kernel (../metrics_kernels.cuh) runs them one template per thread and
// fgb_host_metrics_templates runs the very same functions on host threads; tests/metrics_oracle.py restates them.
// Citations are relative to the fgumi 0.2.0 source tree:
//   shared_metrics.rs  src/lib/commands/shared_metrics.rs   (process_templates_from_bam, compute_hash_fraction,
//                                                            overlaps_intervals, compute_template_metadata)
//   cigar.rs           crates/fgumi-raw-bam/src/cigar.rs    (unclipped_5prime_from_raw_bam, alignment_end_from_raw)
#pragma once
#include <stdint.h>

#include "../../../include/fgumi_b200.h"
#include "../sort_keys.h"
#include "record_filter.h"

namespace fgb {
namespace metrics {

constexpr int kFractions = 20;

// DOWNSAMPLING_FRACTIONS (shared_metrics.rs:22-26) as the same f64 literals: 0.05 * 3 is not 0.15
FGB_HD double fraction_at(int i) {
  switch (i) {
    case 0: return 0.05; case 1: return 0.10; case 2: return 0.15; case 3: return 0.20; case 4: return 0.25;
    case 5: return 0.30; case 6: return 0.35; case 7: return 0.40; case 8: return 0.45; case 9: return 0.50;
    case 10: return 0.55; case 11: return 0.60; case 12: return 0.65; case 13: return 0.70; case 14: return 0.75;
    case 15: return 0.80; case 16: return 0.85; case 17: return 0.90; case 18: return 0.95; default: return 1.00;
  }
}

// compute_hash_fraction (shared_metrics.rs:129-136): wrapping_abs keeps i32::MIN, whose quotient is just below -1
FGB_HD double hash_fraction(int32_t h) {
  const int32_t a = h == INT32_MIN ? h : (h < 0 ? -h : h);
  return static_cast<double>(a) / 2147483647.0;
}

// The template joins fraction f iff hash_fraction <= f (duplex_metrics.rs:311-312): the first such index, found by the
// same comparisons.  A fraction is at most 1.0, so every template lands in a bucket below 20.
FGB_HD uint32_t bucket_of(int32_t h) {
  const double f = hash_fraction(h);
  for (int i = 0; i < kFractions; ++i)
    if (f <= fraction_at(i)) return static_cast<uint32_t>(i);
  return kFractions;
}

// htsjdk Murmur3.hashUnencodedChars (shared_metrics.rs:141-184) over UTF-16 code units; unit(i) gives unit i
FGB_HD uint32_t mix_k1(uint32_t k1) {
  k1 *= 0xcc9e2d51u;
  k1 = (k1 << 15) | (k1 >> 17);
  return k1 * 0x1b873593u;
}
template <class Unit>
FGB_HD int32_t murmur3_units(Unit&& unit, uint32_t n, uint32_t seed) {
  uint32_t h1 = seed;
  for (uint32_t i = 1; i < n; i += 2) {
    h1 ^= mix_k1(static_cast<uint32_t>(unit(i - 1)) | (static_cast<uint32_t>(unit(i)) << 16));
    h1 = (h1 << 13) | (h1 >> 19);
    h1 = h1 * 5u + 0xe6546b64u;
  }
  if (n & 1) h1 ^= mix_k1(static_cast<uint32_t>(unit(n - 1)));
  h1 ^= 2u * n;
  h1 ^= h1 >> 16;
  h1 *= 0x85ebca6bu;
  h1 ^= h1 >> 13;
  h1 *= 0xc2b2ae35u;
  h1 ^= h1 >> 16;
  return static_cast<int32_t>(h1);
}

// compute_template_metadata (shared_metrics.rs:418-432): "/A" or "/B" stripped off; the base as a number when it is
// a canonical decimal (no leading zero, at most 18 digits), so that equal numbers are equal strings
FGB_HD void parse_mi(const uint8_t* s, uint32_t n, uint8_t* kind, uint8_t* canonical, uint64_t* base) {
  *kind = 0;
  if (n >= 2 && s[n - 2] == '/' && (s[n - 1] == 'A' || s[n - 1] == 'B')) {
    *kind = s[n - 1] == 'A' ? 1 : 2;
    n -= 2;
  }
  uint64_t v = 0;
  bool ok = n >= 1 && n <= 18 && (n == 1 || s[0] != '0');
  for (uint32_t i = 0; ok && i < n; ++i) {
    ok = s[i] >= '0' && s[i] <= '9';
    v = v * 10 + (s[i] - '0');
  }
  *canonical = ok;
  *base = ok ? v : 0;
}

// The interval table as the template pass reads it: for @SQ index s the intervals of its name are
// [sq_begin[s], sq_begin[s + 1]), sorted by start, maxend[k] the largest end of the first k + 1 of them
struct IvTable {
  const uint32_t* sq_begin;
  const int64_t* start;
  const int64_t* maxend;
  uint32_t n_sq;
  uint8_t active;   // intervals were given
};

// overlaps_intervals (shared_metrics.rs:271-289): some interval [s, e) of the contig with start <= e and s < end
FGB_HD bool overlaps(const IvTable& iv, int32_t contig, int64_t start, int64_t end) {
  if (!iv.active) return true;
  if (contig < 0 || static_cast<uint32_t>(contig) >= iv.n_sq) return false;
  uint32_t lo = iv.sq_begin[contig], hi = iv.sq_begin[contig + 1];
  const uint32_t b = lo;
  while (lo < hi) {   // the intervals with s < end are [b, lo)
    const uint32_t mid = (lo + hi) / 2;
    if (iv.start[mid] < end) lo = mid + 1;
    else hi = mid;
  }
  return lo > b && iv.maxend[lo - 1] >= start;
}

FGB_HD bool passes(uint16_t f, bool first) {   // shared_metrics.rs:478-487
  return (f & 0x1) && !(f & 0x4) && !(f & 0x8) && (f & (first ? 0x40 : 0x80)) && !(f & 0x100) && !(f & 0x800);
}

FGB_HD uint32_t ref_len(const uint8_t* r) {   // reference_length_from_raw_bam (cigar.rs:155-176), CIGAR in bounds
  const uint32_t nc = sortk::ld16(r + 12);
  const uint64_t cs = 32 + static_cast<uint64_t>(r[8]);
  uint32_t len = 0;
  for (uint32_t i = 0; i < nc; ++i) {
    const uint32_t op = sortk::ld32(r + cs + 4ull * i);
    if (sortk::consumes_ref(op & 0xF)) len += op >> 4;
  }
  return len;
}

// One template (process_templates_from_bam, shared_metrics.rs:489-597): rec(k) / len(k) give record k of the call,
// whose records passed the layout check; p1 / p2 are the template's primary R1 / R2 slots (template_order, -1:
// absent) and n_recs its record count.  Writes everything but the host's parts (non-ASCII names, MI dictionary).
template <class Rec, class Len>
FGB_HD void template_pass(Rec&& rec, Len&& len, uint64_t n_recs, int64_t p1, int64_t p2, const IvTable& iv,
                          fgb_metrics_template* t) {
  *t = fgb_metrics_template{};
  t->status = FGB_MT_SKIP;
  t->name_ascii = 1;
  if (n_recs < 2) return;
  // the first record in template order passing each filter: only the primary slots can (template.rs order)
  int64_t a = -1, b = -1;
  const int64_t slots[2] = {p1, p2};
  for (int k = 1; k >= 0; --k) {
    if (slots[k] < 0) continue;
    const uint16_t f = sortk::ld16(rec(slots[k]) + 14);
    if (passes(f, true)) a = slots[k];
    if (passes(f, false)) b = slots[k];
  }
  if (a < 0 || b < 0) return;
  const uint8_t* r1 = rec(a);
  const uint8_t* r2 = rec(b);
  const uint64_t n1 = len(a);
  t->r1 = static_cast<uint32_t>(a);
  // MI then RX from R1 (required_z_tag, shared_metrics.rs:609-621): absent, not a Z string or not UTF-8 fails
  const uint32_t aux = static_cast<uint32_t>(32 + r1[8] + 4ull * sortk::ld16(r1 + 12) + (sortk::ld32(r1 + 16) + 1ull) / 2 +
                                             sortk::ld32(r1 + 16));
  const rfilter::TagRef mi = rfilter::find_tag(r1 + aux, n1 - aux, "MI");
  if (mi.type != 'Z') { t->status = FGB_MT_ERR_MI_MISSING; return; }
  t->mi_off = static_cast<uint32_t>(mi.data - r1);
  t->mi_len = mi.count - 1;
  if (!sortk::valid_utf8(mi.data, t->mi_len)) { t->status = FGB_MT_ERR_MI_UTF8; return; }
  const rfilter::TagRef rx = rfilter::find_tag(r1 + aux, n1 - aux, "RX");
  if (rx.type != 'Z') { t->status = FGB_MT_ERR_RX_MISSING; return; }
  t->rx_off = static_cast<uint32_t>(rx.data - r1);
  t->rx_len = rx.count - 1;
  if (!sortk::valid_utf8(rx.data, t->rx_len)) { t->status = FGB_MT_ERR_RX_UTF8; return; }
  parse_mi(mi.data, t->mi_len, &t->mi_kind, &t->mi_canonical, &t->mi_base);
  const int32_t tid1 = static_cast<int32_t>(sortk::ld32(r1)), tid2 = static_cast<int32_t>(sortk::ld32(r2));
  if (tid1 < 0 || tid2 < 0) return;
  if (sortk::ld16(r1 + 12) == 0 || sortk::ld16(r2 + 12) == 0) return;   // no unclipped 5' position
  const uint16_t f1 = sortk::ld16(r1 + 14), f2 = sortk::ld16(r2 + 14);
  const int32_t pos1 = static_cast<int32_t>(sortk::ld32(r1 + 4)), pos2 = static_cast<int32_t>(sortk::ld32(r2 + 4));
  const int32_t s1 = sortk::unclipped_5prime(r1, n1, pos1, f1 & 0x10);
  const int32_t s2 = sortk::unclipped_5prime(r2, len(b), pos2, f2 & 0x10);
  // the insert (shared_metrics.rs:533-547); alignment_end_from_raw is None for pos < 0 or no reference bases
  const int64_t st1 = static_cast<int64_t>(pos1) + 1, st2 = static_cast<int64_t>(pos2) + 1;
  const uint32_t rl1 = ref_len(r1), rl2 = ref_len(r2);
  const bool has_e1 = pos1 >= 0 && rl1, has_e2 = pos2 >= 0 && rl2;
  const int64_t e1 = static_cast<int64_t>(pos1) + rl1, e2 = static_cast<int64_t>(pos2) + rl2;
  int64_t ins_s, ins_e;
  if (tid1 == tid2) {
    ins_s = st1 < st2 ? st1 : st2;
    if (has_e1 && has_e2) ins_e = e1 > e2 ? e1 : e2;
    else ins_e = st1 > st2 ? st1 : st2;
  } else {
    ins_s = st1;
    ins_e = has_e1 ? e1 : st1;
  }
  t->contig = tid1;
  t->ins_start = static_cast<int32_t>(ins_s);
  t->ins_end = static_cast<int32_t>(ins_e);
  const bool r1_first = tid1 < tid2 || (tid1 == tid2 && s1 <= s2);   // ReadInfoKey (shared_metrics.rs:549-568)
  t->ref1 = r1_first ? tid1 : tid2;
  t->start1 = r1_first ? s1 : s2;
  t->strand1 = ((r1_first ? f1 : f2) & 0x10) ? 1 : 0;
  t->ref2 = r1_first ? tid2 : tid1;
  t->start2 = r1_first ? s2 : s1;
  t->strand2 = ((r1_first ? f2 : f1) & 0x10) ? 1 : 0;
  // the read name as UTF-16 code units: bytes below 0x80 are their own units; any other byte leaves it to the host
  const uint32_t nl = r1[8] ? r1[8] - 1u : 0u;
  const uint8_t* nm = r1 + 32;
  for (uint32_t i = 0; i < nl; ++i)
    if (nm[i] >= 0x80) t->name_ascii = 0;
  if (t->name_ascii) t->bucket = static_cast<uint8_t>(bucket_of(murmur3_units([&](uint32_t i) { return nm[i]; }, nl, 42)));
  t->status = overlaps(iv, tid1, ins_s, ins_e) ? FGB_MT_KEPT : FGB_MT_OUTSIDE;
}

}  // namespace metrics
}  // namespace fgb
