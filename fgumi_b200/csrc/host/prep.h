// Shared host-side preparation code of the record-level callers (product code, header-only):
// source-read creation, CIGAR grouping, RX consensus and the SoA batch packer.
//
// Behavioural spec (reference = fgumi 0.2.0, crates/fgumi-consensus/src/):
//   vanilla_caller.rs:47-119    select_most_common_alignment_group
//   vanilla_caller.rs:780-804   find_quality_trim_point
//   vanilla_caller.rs:863-955   create_source_read
//   vanilla_caller.rs:961-1013  filter_source_reads_by_alignment
//   vanilla_caller.rs:1269-1277 consensus length = min_reads-th longest read
//   simple_umi.rs:36-134,236-245  SimpleConsensusCaller / consensus_umis
#pragma once
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <functional>
#include <string>
#include <vector>

#include "../../../include/fgumi_b200.h"
#include "../host_math.h"
#include "../host_tables.h"
#include "bam.h"

namespace fgb {
namespace prep {

using bam::View;

inline size_t round_up(size_t x, size_t m) { return (x + m - 1) / m * m; }

struct PrepOptions {
  uint8_t min_input_base_quality = 10;
  bool trim = false;
};

struct SourceRead {
  uint32_t original_idx = 0;
  uint16_t flags = 0;
  std::vector<uint8_t> bases, quals;
  bam::SimpleCigar cigar;
};

// Host ConsensusBaseBuilder for the RX (UMI) consensus only (simple_umi.rs:36-134): f64, literal.
struct UmiBuilder {
  HostTables t;
  UmiBuilder() { build_host_tables(90, 90, &t); }   // simple_umi.rs:13-19 defaults (90, 90, Q20)
  // One column of characters, all DNA (A/C/G/T/N, any case); returns the called base.
  uint8_t call(const std::vector<uint8_t>& col) const {
    using namespace hostmath;
    {
      // A column whose non-N characters are all the same base calls that base: the only observed base
      // has ll = n * correct against n * err_alt for the others (a gap of >= 5.7 nats per observation),
      // so neither the tie rule nor rounding can change the argmax; all-N columns have depth 0 -> 'N'.
      static const int8_t kIdx[256] = {
#define FGB_R16(v) v, v, v, v, v, v, v, v, v, v, v, v, v, v, v, v
          FGB_R16(-1), FGB_R16(-1), FGB_R16(-1), FGB_R16(-1),
          -1, 0, -1, 1, -1, -1, -1, 2, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, 3, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1,
          -1, 0, -1, 1, -1, -1, -1, 2, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, 3, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1,
          FGB_R16(-1), FGB_R16(-1), FGB_R16(-1), FGB_R16(-1), FGB_R16(-1), FGB_R16(-1), FGB_R16(-1), FGB_R16(-1)
#undef FGB_R16
      };
      int first = -1;
      bool uniform = true;
      for (uint8_t ch : col) {
        const int idx = kIdx[ch];
        if (idx < 0) continue;
        if (first < 0) first = idx;
        else if (idx != first) { uniform = false; break; }
      }
      if (uniform) return first < 0 ? 'N' : static_cast<uint8_t>("ACGT"[first]);
    }
    double ll[4] = {0, 0, 0, 0}, kc[4] = {0, 0, 0, 0};
    uint32_t obs[4] = {0, 0, 0, 0};
    const double c = t.correct[20], e = t.err_alt[20];
    for (uint8_t ch : col) {
      int idx;
      switch (ch) {
        case 'A': case 'a': idx = 0; break;
        case 'C': case 'c': idx = 1; break;
        case 'G': case 'g': idx = 2; break;
        case 'T': case 't': idx = 3; break;
        default: idx = -1;
      }
      if (idx < 0) continue;   // 'N' is ignored by add(), base_builder.rs:300
      for (int i = 0; i < 4; ++i) {   // base_builder.rs:312-324
        double v = i == idx ? c : e;
        double y = v - kc[i];
        double s = ll[i] + y;
        kc[i] = (s - ll[i]) - y;
        ll[i] = s;
      }
      obs[idx]++;
    }
    const uint32_t depth = obs[0] + obs[1] + obs[2] + obs[3];
    if (depth == 0) return 'N';
    int kinds = (obs[0] != 0) + (obs[1] != 0) + (obs[2] != 0) + (obs[3] != 0);
    static const char kB[5] = "ACGT";
    if (kinds == 1) {
      int w = obs[0] ? 0 : obs[1] ? 1 : obs[2] ? 2 : 3;
      if (ll[w] - ll[(w + 1) % 4] > 23.0) return kB[w];
    }
    double mx = kNegInf;
    int mi = -1;
    bool tie = false;
    for (int i = 0; i < 4; ++i) {   // base_builder.rs:413-431
      if (ll[i] > mx) { mx = ll[i]; mi = i; tie = false; }
      else if (ll[i] == mx) tie = true;
      else if (ll[i] < mx && std::fabs(ll[i] - mx) <= DBL_EPSILON) tie = true;
    }
    if (tie || mi < 0) return 'N';
    return kB[mi];
  }
};


// find_quality_trim_point, vanilla_caller.rs:780-804
inline size_t quality_trim_point(const std::vector<uint8_t>& q, uint8_t trim_qual) {
  size_t length = q.size();
  if (trim_qual < 1 || length == 0) return 0;
  int32_t score = 0, max_score = 0;
  size_t trim_point = length;
  for (size_t i = length; i-- > 0;) {
    score += static_cast<int32_t>(trim_qual) - static_cast<int32_t>(q[i]);
    if (score < 0) break;
    if (score > max_score) { max_score = score; trim_point = i; }
  }
  return trim_point;
}


// create_source_read, vanilla_caller.rs:863-955.
// One fused pass: the reference decodes the 4-bit sequence, reverse-complements negative-strand reads,
// masks low qualities, clips and strips trailing Ns in separate sweeps; only the first
// min(read_len - mate_clip, trim_to) oriented positions can survive, so only those are produced, each
// straight from its nibble (a second 16-entry table decodes AND complements) and quality byte.
static const char kFwd[17] = "=ACMGRSVTWYHKDBN";       // sequence.rs nibble codes
static const char kRev[17] = "=TGMCRSVAWYHKDBN";       // ... complemented (A<->T, C<->G, rest unchanged)

// The per-read decisions of create_source_read (vanilla_caller.rs:863-955) WITHOUT decoding the read: the
// length of the SourceRead row after the mate-overlap clip, the optional quality trim and the trailing-N
// strip, 0 when the read yields no source read (no bases, truncated record, missing qualities, fully
// clipped / trimmed / masked).  A position is 'N' when its quality is below min_input_base_quality or its
// base nibble is 15; only those are stripped from the end (:918-927).  The record-level callers use it on
// its own when the device builds the rows (FGB_IN_RECORDS).
// `eff(j, &nib, &q)` may replace the base code and quality of raw position j by what an earlier in-place pass
// would have left there (the overlapping-bases pre-pass applied on the device: only the row's tail is looked at
// here, so the host evaluates the rule for those few positions instead of rewriting the read).
template <class Eff>
inline uint32_t plan_read_len_eff(const PrepOptions& opt, const View& v, size_t mate_clip, Eff&& eff) {
  const bool neg = v.flags() & bam::kReverse;
  const uint8_t min_bq = opt.min_input_base_quality;
  const uint32_t read_len = v.l_seq();
  if (read_len == 0 || v.qual_off() + read_len > v.n) return 0;
  const uint8_t* s = v.b + v.seq_off();
  const uint8_t* q = v.b + v.qual_off();
  bool all_ff = true;
  for (uint32_t i = 0; i < read_len; ++i) if (q[i] != 0xFF) { all_ff = false; break; }
  if (all_ff) return 0;                                      // missing qualities
  size_t trim_to = read_len;
  if (opt.trim) {                                            // needs the oriented qualities as a whole
    static thread_local std::vector<uint8_t> oriented;
    if (neg) oriented.assign(std::reverse_iterator<const uint8_t*>(q + read_len), std::reverse_iterator<const uint8_t*>(q));
    else oriented.assign(q, q + read_len);
    trim_to = quality_trim_point(oriented, min_bq);
  }
  const size_t clip_position = read_len > mate_clip ? read_len - mate_clip : 0;
  size_t final_len = std::min(clip_position, trim_to);
  while (final_len > 0) {                                    // oriented position i is record position j
    const size_t i = final_len - 1, j = neg ? read_len - 1 - i : i;
    uint8_t nib = static_cast<uint8_t>((j & 1) ? (s[j >> 1] & 15u) : (s[j >> 1] >> 4));
    uint8_t qq = q[j];
    eff(j, &nib, &qq);
    if (qq < min_bq || nib == 15u) --final_len; else break;
  }
  return static_cast<uint32_t>(final_len);
}

inline uint32_t plan_read_len(const PrepOptions& opt, const View& v, size_t mate_clip) {
  return plan_read_len_eff(opt, v, mate_clip, [](size_t, uint8_t*, uint8_t*) {});
}

// The per-base half of create_source_read (vanilla_caller.rs:893-916): the first `bound` oriented positions of a read
// whose packed sequence starts at `s` (read_len bases, the qualities (read_len + 1) / 2 bytes later), decoded,
// reverse-complemented when `neg`, and (N, 2) where the quality is below min_bq -- the row the device builds from a
// staged record (FGB_IN_RECORDS).
inline void decode_source_row(const uint8_t* s, uint32_t read_len, bool neg, size_t bound, uint8_t min_bq,
                              uint8_t* __restrict ob, uint8_t* __restrict oq) {
  const uint8_t* q = s + (read_len + 1) / 2;
  // a pair table decodes one packed byte (two bases) per step, complemented and swapped for
  // negative-strand reads; then a (reversed) copy of the qualities and a compare-and-blend pass that
  // the compiler vectorises
  struct PairTables {
    uint16_t fwd[256], rev[256];
    PairTables() {
      for (int b = 0; b < 256; ++b) {
        const uint8_t f[2] = {static_cast<uint8_t>(kFwd[b >> 4]), static_cast<uint8_t>(kFwd[b & 15])};
        const uint8_t r[2] = {static_cast<uint8_t>(kRev[b & 15]), static_cast<uint8_t>(kRev[b >> 4])};
        std::memcpy(&fwd[b], f, 2);
        std::memcpy(&rev[b], r, 2);
      }
    }
  };
  static const PairTables kPairs;
  if (!neg) {
    const size_t n2 = bound >> 1;
    for (size_t k = 0; k < n2; ++k) std::memcpy(ob + 2 * k, &kPairs.fwd[s[k]], 2);
    if (bound & 1) ob[bound - 1] = static_cast<uint8_t>(kFwd[s[bound >> 1] >> 4]);
    std::memcpy(oq, q, bound);
  } else {
    size_t i = 0, j = read_len - 1;                        // oriented position i is record position j
    if (bound > 0 && !(j & 1)) { ob[0] = static_cast<uint8_t>(kRev[s[j >> 1] >> 4]); i = 1; --j; }
    for (; i + 2 <= bound; i += 2, j -= 2) std::memcpy(ob + i, &kPairs.rev[s[j >> 1]], 2);   // j odd: (low, high) nibble
    if (i < bound) ob[i] = static_cast<uint8_t>(kRev[s[j >> 1] & 15]);
    std::reverse_copy(q + (read_len - bound), q + read_len, oq);
  }
  for (size_t i = 0; i < bound; ++i) {
    const bool low = oq[i] < min_bq;
    ob[i] = low ? static_cast<uint8_t>('N') : ob[i];
    oq[i] = low ? static_cast<uint8_t>(2) : oq[i];
  }
}

inline bool make_source_read(const PrepOptions& opt, const View& v, uint32_t idx, size_t mate_clip,
                             std::vector<uint32_t>* ops, SourceRead* sr) {
  const size_t bound = plan_read_len(opt, v, mate_clip);     // only these oriented positions survive
  if (bound == 0) return false;
  const bool neg = v.flags() & bam::kReverse;
  sr->bases.resize(bound);
  sr->quals.resize(bound);
  decode_source_row(v.b + v.seq_off(), v.l_seq(), neg, bound, opt.min_input_base_quality, sr->bases.data(), sr->quals.data());
  const size_t final_len = bound;                            // the trailing Ns are already gone
  bam::cigar_ops(v, ops);
  bam::simplify_cigar(*ops, &sr->cigar);
  if (neg) std::reverse(sr->cigar.begin(), sr->cigar.end());
  bam::truncate_cigar(&sr->cigar, final_len);
  sr->original_idx = idx;
  sr->flags = v.flags();
  return true;
}


// filter_source_reads_by_alignment + select_most_common_alignment_group, vanilla_caller.rs:47-119,961-1013
// over the first `n` elements of `srs`: the kept reads are moved to the front in their original order
// (by swapping, so every element keeps its buffers for reuse) and their number is returned.
inline size_t filter_by_alignment_n(std::vector<SourceRead>* srs, size_t n) {
  if (n < 2) return n;
  static thread_local std::vector<uint32_t> order;
  order.resize(n);
  for (uint32_t i = 0; i < n; ++i) order[i] = i;
  std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) {
    return (*srs)[a].bases.size() > (*srs)[b].bases.size();
  });
  struct Group { const bam::SimpleCigar* cigar; std::vector<uint32_t> members; };
  static thread_local std::vector<Group> groups;
  size_t n_groups = 0;
  for (uint32_t idx : order) {
    const bam::SimpleCigar& cg = (*srs)[idx].cigar;
    bool found = false;
    for (size_t g = 0; g < n_groups; ++g)
      if (bam::is_cigar_prefix(cg, *groups[g].cigar)) { groups[g].members.push_back(idx); found = true; }   // no break (fgbio)
    if (!found) {
      if (n_groups == groups.size()) groups.emplace_back();
      groups[n_groups].cigar = &cg;
      groups[n_groups].members.assign(1, idx);
      ++n_groups;
    }
  }
  // Iterator::max_by keeps the LAST maximum: larger group wins, then the smaller CIGAR
  const Group* best = nullptr;
  for (size_t gi = 0; gi < n_groups; ++gi) {
    const Group& g = groups[gi];
    if (!best) { best = &g; continue; }
    int cmp = g.members.size() < best->members.size() ? -1 : (g.members.size() > best->members.size() ? 1 : 0);
    if (cmp == 0) cmp = bam::cmp_cigar(*best->cigar, *g.cigar);
    if (cmp >= 0) best = &g;
  }
  if (best->members.size() == n) return n;                  // the common case: nothing to drop
  static thread_local std::vector<char> keep;
  keep.assign(n, 0);
  for (uint32_t i : best->members) keep[i] = 1;
  size_t w = 0;
  for (size_t i = 0; i < n; ++i) {
    if (!keep[i]) continue;
    if (w != i) { std::swap((*srs)[w], (*srs)[i]); std::swap(keep[w], keep[i]); }
    ++w;
  }
  return w;
}

// Vector form: drops the minority reads, returns how many were dropped.
inline size_t filter_by_alignment(std::vector<SourceRead>* srs) {
  const size_t n = srs->size();
  const size_t kept = filter_by_alignment_n(srs, n);
  srs->resize(kept);
  return n - kept;
}


// consensus_umis, simple_umi.rs:65-122,236-245.  Returns false for the reference's panics
// (length mismatch, DNA / non-DNA mix).
inline bool consensus_umis(const UmiBuilder& builder, const std::vector<std::string>& umis, std::string* out) {
  out->clear();
  if (umis.empty()) return true;
  if (umis.size() == 1) { *out = umis[0]; return true; }
  const std::string& first = umis[0];
  for (const auto& s : umis) if (s.size() != first.size()) return false;
  auto is_dna = [](uint8_t ch) {
    switch (ch) { case 'A': case 'C': case 'G': case 'T': case 'N':
                  case 'a': case 'c': case 'g': case 't': case 'n': return true; default: return false; }
  };
  std::vector<uint8_t> col(umis.size());
  for (size_t i = 0; i < first.size(); ++i) {
    size_t non_dna = 0;
    for (size_t k = 0; k < umis.size(); ++k) {
      col[k] = static_cast<uint8_t>(umis[k][i]);
      if (!is_dna(col[k])) {
        ++non_dna;
        if (col[k] != static_cast<uint8_t>(first[i])) return false;
      }
    }
    if (non_dna == 0) out->push_back(static_cast<char>(builder.call(col)));
    else if (non_dna == umis.size()) out->push_back(first[i]);
    else return false;
  }
  return true;
}


// Allocator whose resize() leaves new elements uninitialised (the two byte columns are always
// overwritten right after they grow; zero-filling 100 MB per batch first would cost as much as the copy).
template <class T>
struct DefaultInitAlloc : std::allocator<T> {
  template <class U> struct rebind { using other = DefaultInitAlloc<U>; };
  template <class U> void construct(U* p) noexcept { ::new (static_cast<void*>(p)) U; }
  template <class U, class... A> void construct(U* p, A&&... a) { ::new (static_cast<void*>(p)) U(std::forward<A>(a)...); }
};
using ByteColumn = std::vector<uint8_t, DefaultInitAlloc<uint8_t>>;

// The packed SoA batch of include/fgumi_b200.h, grown unit by unit.
struct Packer {
  ByteColumn bases, quals;
  std::vector<uint64_t> reads;
  std::vector<fgb_unit> units;
  uint64_t n_out = 0;
  // Appends one unit (its SourceRead rows); returns the unit index.
  uint32_t add_unit(const std::vector<SourceRead>& srs, size_t min_reads) {
    return add_unit_rows(srs.size(), min_reads, [&](size_t k) -> const SourceRead& { return srs[k]; });
  }
  // ... rows given by pointer (the duplex caller splits one pooled vector into four sub-families)
  uint32_t add_unit(const std::vector<const SourceRead*>& rows, size_t min_reads) {
    return add_unit_rows(rows.size(), min_reads, [&](size_t k) -> const SourceRead& { return *rows[k]; });
  }
  template <class Row>
  uint32_t add_unit_rows(size_t n, size_t min_reads, Row row) {
    fgb_unit u;
    u.out_off = n_out;
    u.read_begin = static_cast<uint32_t>(reads.size());
    static thread_local std::vector<size_t> lens;
    lens.clear();
    size_t total = 0;
    for (size_t k = 0; k < n; ++k) total += round_up(row(k).bases.size(), FGB_READ_ALIGN);
    size_t off = bases.size();
    bases.resize(off + total);                               // one uninitialised growth per unit ...
    quals.resize(off + total);
    for (size_t k = 0; k < n; ++k) {
      const SourceRead& sr = row(k);
      const size_t len = sr.bases.size();
      const size_t padded = round_up(len, FGB_READ_ALIGN);
      reads.push_back(FGB_READ_DESC(off, len));
      std::memcpy(bases.data() + off, sr.bases.data(), len);
      std::memcpy(quals.data() + off, sr.quals.data(), len);
      std::memset(bases.data() + off + len, 0, padded - len); // ... rows and their zero padding written in place
      std::memset(quals.data() + off + len, 0, padded - len);
      off += padded;
      lens.push_back(len);
    }
    std::sort(lens.begin(), lens.end(), std::greater<size_t>());
    u.cons_len = static_cast<uint32_t>(lens[min_reads - 1]);   // vanilla_caller.rs:1269-1277
    units.push_back(u);
    n_out += round_up(u.cons_len, FGB_OUT_ALIGN);
    return static_cast<uint32_t>(units.size() - 1);
  }
  // Seals the batch (sentinel unit, 16-byte column padding, descriptor padding).
  void seal(uint64_t* n_bytes, uint64_t* n_reads) {
    fgb_unit sentinel;
    sentinel.out_off = n_out;
    sentinel.read_begin = static_cast<uint32_t>(reads.size());
    sentinel.cons_len = 0;
    units.push_back(sentinel);
    *n_bytes = bases.size();
    bases.resize(round_up(bases.size() + 1, 16), 0);
    quals.resize(bases.size(), 0);
    *n_reads = reads.size();
    reads.resize(reads.size() + 2, 0);
  }
  void clear() { bases.clear(); quals.clear(); reads.clear(); units.clear(); n_out = 0; }
};

}  // namespace prep
}  // namespace fgb
