// Overlapping-bases pre-pass: co-calls the bases of R1 and R2 that cover the same reference
// position, in place on the raw records, before the UMI vote (so the two mates are not counted as
// independent observations).  Behaviour of fgumi's OverlappingBasesConsensusCaller::call
// (crates/fgumi-consensus/src/overlapping.rs:236-337) and apply_overlapping_consensus (:625-667).
//
// Design: instead of walking two per-base iterators, each read's CIGAR is turned into its aligned
// segments (ref_start, read_start, len) clipped to the pair's common reference window; the two
// sorted segment lists are intersected run by run, and each run is processed on the packed
// 4-bit sequence directly (no decode / re-encode of the whole read).
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

#include "bam.h"

namespace fgb {
namespace overlap {

enum Agreement : uint8_t { kAgreeConsensus = 0, kAgreeMaxQual = 1, kAgreePassThrough = 2 };
enum Disagreement : uint8_t { kDisagreeConsensus = 0, kDisagreeMaskBoth = 1, kDisagreeMaskLower = 2 };

struct Stats {   // CorrectionStats, overlapping.rs:42-77
  uint64_t overlapping_bases = 0, bases_agreeing = 0, bases_disagreeing = 0, bases_corrected = 0;
};

struct Segment { int64_t ref; int64_t read; int64_t len; };   // 1-based ref, 0-based read offset

// One maximal stretch of a pair's overlap: `len` consecutive bases of R1 from read offset o1 against the same
// number of bases of R2 from o2 (record indices within the group).  What call() applies position by position;
// planned on its own when the device applies it (fgb_overlap_run, FGB_IN_RECORDS batches).
struct Run { uint32_t rec1, rec2; uint32_t o1, o2, len; };

// Aligned (M/=/X) runs of a record inside [win_lo, win_hi] (1-based, inclusive), read offsets
// limited to l_seq.
inline void aligned_segments(const bam::View& v, int64_t win_lo, int64_t win_hi, std::vector<Segment>* out) {
  out->clear();
  if (!v.cigar_in_bounds()) return;
  int64_t ref = static_cast<int64_t>(v.pos()) + 1, read = 0;
  const int64_t l_seq = v.l_seq();
  for (uint32_t i = 0; i < v.n_cigar(); ++i) {
    const uint32_t op = v.cigar_op(i);
    const uint32_t k = op & 0xF;
    const int64_t n = op >> 4;
    if (k == 0 || k == 7 || k == 8) {
      int64_t lo = std::max(ref, win_lo), hi = std::min(ref + n - 1, win_hi);
      hi = std::min(hi, ref + (l_seq - read) - 1);        // never past the stored sequence
      if (lo <= hi) out->push_back(Segment{lo, read + (lo - ref), hi - lo + 1});
      ref += n; read += n;
    } else {
      if (bam::consumes_ref(k)) ref += n;
      if (bam::consumes_query(k)) read += n;
    }
    if (ref > win_hi) break;
  }
}

inline uint8_t get_code(const uint8_t* seq, int64_t i) {
  return (i & 1) ? (seq[i >> 1] & 0xF) : (seq[i >> 1] >> 4);
}
inline void set_code(uint8_t* seq, int64_t i, uint8_t code) {
  uint8_t& b = seq[i >> 1];
  b = (i & 1) ? static_cast<uint8_t>((b & 0xF0) | code) : static_cast<uint8_t>((code << 4) | (b & 0x0F));
}

class Caller {
 public:
  Caller(Agreement a, Disagreement d) : agree_(a), disagree_(d) {}
  Stats stats;

  // Returns true when the mates share at least one aligned reference position.
  bool call(uint8_t* r1, size_t n1, uint8_t* r2, size_t n2) {
    bam::View v1(r1, n1), v2(r2, n2);
    if ((v1.flags() | v2.flags()) & bam::kUnmapped) return false;
    if (v1.ref_id() != v2.ref_id()) return false;
    int64_t s1, e1, s2, e2;
    if (!span(v1, &s1, &e1) || !span(v2, &s2, &e2)) return false;
    const int64_t lo = std::max(s1, s2), hi = std::min(e1, e2);
    if (lo > hi) return false;
    aligned_segments(v1, lo, hi, &seg1_);
    aligned_segments(v2, lo, hi, &seg2_);
    uint8_t* seq1 = r1 + v1.seq_off(); uint8_t* q1 = r1 + v1.qual_off();
    uint8_t* seq2 = r2 + v2.seq_off(); uint8_t* q2 = r2 + v2.qual_off();
    bool any = false;
    size_t i = 0, j = 0;
    while (i < seg1_.size() && j < seg2_.size()) {
      const Segment& a = seg1_[i];
      const Segment& b = seg2_[j];
      const int64_t from = std::max(a.ref, b.ref);
      const int64_t to = std::min(a.ref + a.len, b.ref + b.len);   // exclusive
      if (from < to) {
        any = true;
        run(seq1, q1, a.read + (from - a.ref), seq2, q2, b.read + (from - b.ref), to - from);
      }
      if (a.ref + a.len <= b.ref + b.len) ++i; else ++j;
    }
    return any;
  }

  // The runs of one pair, without touching a base (the headers and CIGARs decide them).
  void plan_pair(const uint8_t* r1, size_t n1, const uint8_t* r2, size_t n2, uint32_t i1, uint32_t i2, std::vector<Run>* out) {
    bam::View v1(r1, n1), v2(r2, n2);
    if ((v1.flags() | v2.flags()) & bam::kUnmapped) return;
    if (v1.ref_id() != v2.ref_id()) return;
    int64_t s1, e1, s2, e2;
    if (!span(v1, &s1, &e1) || !span(v2, &s2, &e2)) return;
    const int64_t lo = std::max(s1, s2), hi = std::min(e1, e2);
    if (lo > hi) return;
    aligned_segments(v1, lo, hi, &seg1_);
    aligned_segments(v2, lo, hi, &seg2_);
    size_t i = 0, j = 0;
    while (i < seg1_.size() && j < seg2_.size()) {
      const Segment& a = seg1_[i];
      const Segment& b = seg2_[j];
      const int64_t from = std::max(a.ref, b.ref);
      const int64_t to = std::min(a.ref + a.len, b.ref + b.len);   // exclusive
      if (from < to)
        out->push_back(Run{i1, i2, static_cast<uint32_t>(a.read + (from - a.ref)), static_cast<uint32_t>(b.read + (from - b.ref)),
                           static_cast<uint32_t>(to - from)});
      if (a.ref + a.len <= b.ref + b.len) ++i; else ++j;
    }
  }

  // apply_overlapping_consensus as a PLAN: the runs of every pair of the group, in pair order.
  void plan_group(const uint8_t* records, const uint64_t* off, uint32_t n, std::vector<Run>* out) {
    pair_up(records, off, n);
    for (const auto& p : order_) {
      if (p.idx[0] < 0 || p.idx[1] < 0) continue;
      plan_pair(records + off[p.idx[0]], off[p.idx[0] + 1] - off[p.idx[0]], records + off[p.idx[1]],
                off[p.idx[1] + 1] - off[p.idx[1]], static_cast<uint32_t>(p.idx[0]), static_cast<uint32_t>(p.idx[1]), out);
    }
  }

  // What one position of a run becomes on each side (the rule of run(), without writing or counting):
  // c / q in: the two mates' base codes and qualities; out: side 1 and side 2.
  void position_rule(uint8_t c1, uint8_t c2, uint8_t x, uint8_t y, uint8_t* oc1, uint8_t* oq1, uint8_t* oc2, uint8_t* oq2) const {
    *oc1 = c1; *oq1 = x; *oc2 = c2; *oq2 = y;
    if (c1 == 15 || c2 == 15) return;
    if (c1 == c2) {
      if (agree_ == kAgreePassThrough) return;
      const uint8_t nq = agree_ == kAgreeConsensus ? static_cast<uint8_t>(std::min<unsigned>(unsigned(x) + unsigned(y), 93u)) : std::max(x, y);
      *oq1 = nq; *oq2 = nq;
      return;
    }
    if (disagree_ == kDisagreeConsensus) {
      uint8_t code = 15, q = 2;
      if (x > y) { code = c1; q = std::max<uint8_t>(static_cast<uint8_t>(x - y), 2); }
      else if (y > x) { code = c2; q = std::max<uint8_t>(static_cast<uint8_t>(y - x), 2); }
      *oc1 = code; *oc2 = code; *oq1 = q; *oq2 = q;
    } else if (disagree_ == kDisagreeMaskBoth || x == y) {
      *oc1 = 15; *oc2 = 15; *oq1 = 2; *oq2 = 2;
    } else if (x < y) {
      *oc1 = 15; *oq1 = 2;
    } else {
      *oc2 = 15; *oq2 = 2;
    }
  }
  Agreement agreement() const { return agree_; }
  Disagreement disagreement() const { return disagree_; }

  // The counters one run adds, without writing a base: for runs whose pairs yield no row, so nothing is built from
  // the rewritten bases (the counters still follow the reference, which co-calls every pair of every group).
  void count_run(const uint8_t* seq1, const uint8_t* q1, int64_t o1, const uint8_t* seq2, const uint8_t* q2, int64_t o2,
                 int64_t len) {
    // run<false> only reads through the pointers
    run<false>(const_cast<uint8_t*>(seq1), const_cast<uint8_t*>(q1), o1, const_cast<uint8_t*>(seq2),
               const_cast<uint8_t*>(q2), o2, len);
  }

  // apply_overlapping_consensus: pair primary R1/R2 records of one group by name; the last record
  // seen for a (name, segment) wins, as in the reference's map insertion.
  void apply_group(uint8_t* records, const uint64_t* off, uint32_t n) {
    pair_up(records, off, n);
    for (const auto& p : order_) {
      if (p.idx[0] < 0 || p.idx[1] < 0) continue;
      call(records + off[p.idx[0]], off[p.idx[0] + 1] - off[p.idx[0]],
           records + off[p.idx[1]], off[p.idx[1] + 1] - off[p.idx[1]]);
    }
  }

 private:
  struct Pair { int64_t idx[2]; };

  void pair_up(const uint8_t* records, const uint64_t* off, uint32_t n) {
    pairs_.clear();
    order_.clear();
    for (uint32_t i = 0; i < n; ++i) {
      bam::View v(records + off[i], off[i + 1] - off[i]);
      const uint16_t f = v.flags();
      if (f & (bam::kSecondary | bam::kSupplementary)) continue;
      int slot = (f & bam::kFirst) ? 0 : (f & bam::kLast) ? 1 : -1;
      if (slot < 0) continue;
      std::string name(reinterpret_cast<const char*>(v.b + 32), v.l_read_name() > 1 ? v.l_read_name() - 1 : 0);
      auto it = pairs_.find(name);
      if (it == pairs_.end()) {
        it = pairs_.emplace(std::move(name), order_.size()).first;
        order_.push_back({-1, -1});
      }
      order_[it->second].idx[slot] = static_cast<int64_t>(i);
    }
  }

  static bool span(const bam::View& v, int64_t* s, int64_t* e) {   // cigar.rs:314-335
    if (v.pos() < 0 || !v.cigar_in_bounds()) return false;
    int64_t rl = 0;
    for (uint32_t i = 0; i < v.n_cigar(); ++i) {
      uint32_t op = v.cigar_op(i);
      if (bam::consumes_ref(op & 0xF)) rl += op >> 4;
    }
    if (rl == 0) return false;
    *s = static_cast<int64_t>(v.pos()) + 1;
    *e = static_cast<int64_t>(v.pos()) + rl;
    return true;
  }

  template <bool kWrite = true>
  void run(uint8_t* seq1, uint8_t* q1, int64_t o1, uint8_t* seq2, uint8_t* q2, int64_t o2, int64_t len) {
    for (int64_t k = 0; k < len; ++k, ++o1, ++o2) {
      const uint8_t c1 = get_code(seq1, o1), c2 = get_code(seq2, o2);
      if (c1 == 15 || c2 == 15) continue;          // no-call in either mate: position is skipped
      ++stats.overlapping_bases;
      const uint8_t x = q1[o1], y = q2[o2];
      if (c1 == c2) {
        ++stats.bases_agreeing;
        if (agree_ == kAgreePassThrough) continue;
        const uint8_t nq = agree_ == kAgreeConsensus
                               ? static_cast<uint8_t>(std::min<unsigned>(unsigned(x) + unsigned(y), 93u))
                               : std::max(x, y);
        if constexpr (kWrite) { q1[o1] = nq; q2[o2] = nq; }
        if (nq != x || nq != y) ++stats.bases_corrected;
        continue;
      }
      ++stats.bases_disagreeing;
      if (disagree_ == kDisagreeConsensus) {         // higher quality wins with the difference; tie -> N
        uint8_t code = 15, q = 2;
        if (x > y) { code = c1; q = std::max<uint8_t>(static_cast<uint8_t>(x - y), 2); }
        else if (y > x) { code = c2; q = std::max<uint8_t>(static_cast<uint8_t>(y - x), 2); }
        if constexpr (kWrite) { set_code(seq1, o1, code); set_code(seq2, o2, code); q1[o1] = q; q2[o2] = q; }
        stats.bases_corrected += 2;
      } else if (disagree_ == kDisagreeMaskBoth || x == y) {
        if constexpr (kWrite) { set_code(seq1, o1, 15); set_code(seq2, o2, 15); q1[o1] = 2; q2[o2] = 2; }
        stats.bases_corrected += 2;
      } else if (x < y) {
        if constexpr (kWrite) { set_code(seq1, o1, 15); q1[o1] = 2; }
        ++stats.bases_corrected;
      } else {
        if constexpr (kWrite) { set_code(seq2, o2, 15); q2[o2] = 2; }
        ++stats.bases_corrected;
      }
    }
  }

  Agreement agree_;
  Disagreement disagree_;
  std::vector<Segment> seg1_, seg2_;
  std::unordered_map<std::string, size_t> pairs_;
  std::vector<Pair> order_;
};

}  // namespace overlap
}  // namespace fgb
