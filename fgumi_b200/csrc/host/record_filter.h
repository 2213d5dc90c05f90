// `fgumi filter` applied to one assembled consensus record on the host: the duplex arm
// (crates/fgumi-consensus/src/filter.rs:477-557 filter_duplex_read, :702-806 mask_duplex_bases), the
// single-strand arm for records without aD / bD (filter.rs:453-471, 650-696) and the shared read-level
// gates (src/lib/commands/filter.rs:909-968).  The simplex caller runs its filter on the device columns
// (filter_kernel.cuh); duplex reads carry three depth/error tiers and optional strand-agreement
// strings, which exist only in the assembled record -- so this arm reads the record like the
// reference does.  The tag lookup, the per-base mask predicates and the read gates are FGB_HD: the record-level
// filter (fgb_filter_records, ../filter_records_kernels.cuh) runs the same code per record on the device.
#pragma once
#include <stdint.h>

#include <string.h>

#include <algorithm>
#include <cstring>

#include "../../../include/fgumi_b200.h"
#include "bam.h"

#ifndef FGB_HD
#ifdef __CUDACC__
#define FGB_HD __host__ __device__ __forceinline__
#else
#define FGB_HD inline
#endif
#endif

namespace fgb {
namespace rfilter {

// ---- the rules on the host and the device (FGB_HD): the record-level filter (filter_records_kernels.cuh) runs them
// per record on the device, fgb_filter_record and the duplex caller's fused filter below on the host.

FGB_HD uint16_t ld16(const uint8_t* p) { return static_cast<uint16_t>(p[0] | (p[1] << 8)); }
FGB_HD uint32_t ld32(const uint8_t* p) {
  return static_cast<uint32_t>(p[0]) | (static_cast<uint32_t>(p[1]) << 8) | (static_cast<uint32_t>(p[2]) << 16) |
         (static_cast<uint32_t>(p[3]) << 24);
}

// the complement of reverse_complement_string_tag_in_place (tags.rs:818-836): A / C / G / T in either case to the
// upper-case complement, any other byte unchanged
FGB_HD uint8_t complement(uint8_t b) {
  switch (b) {
    case 'A': case 'a': return 'T';
    case 'T': case 't': return 'A';
    case 'C': case 'c': return 'G';
    case 'G': case 'g': return 'C';
    default: return b;
  }
}

struct TagRef {
  uint8_t type = 0;       // 0 = absent; 'B' arrays carry `sub` and `count`
  uint8_t sub = 0;
  uint32_t count = 0;
  const uint8_t* data = nullptr;
};

FGB_HD size_t fixed_size(uint8_t t) {
  switch (t) {
    case 'A': case 'c': case 'C': return 1;
    case 's': case 'S': return 2;
    case 'i': case 'I': case 'f': return 4;
    default: return 0;
  }
}

// tag_value_size (fields.rs:289-310) of the entry at a + p, p + 3 <= an: its value's bytes, 0 when its type byte is
// unknown, a Z / H string lacks its NUL or a B array its header or element type; *sub / *count: a B array's element
// type and count
FGB_HD size_t value_size(const uint8_t* a, size_t an, size_t p, uint8_t* sub, uint32_t* count) {
  const uint8_t vt = a[p + 2];
  const size_t size = fixed_size(vt);
  if (size) return size;
  if (vt == 'Z' || vt == 'H') {
    size_t z = p + 3;
    while (z < an && a[z]) ++z;
    return z == an ? 0 : z - (p + 3) + 1;
  }
  if (vt != 'B' || an - (p + 3) < 5) return 0;
  const size_t es = fixed_size(a[p + 3]);
  if (!es) return 0;
  *sub = a[p + 3];
  *count = ld32(a + p + 4);
  return 5 + static_cast<size_t>(*count) * es;
}

// bam_fields::find_tag_position semantics for a value lookup: the first occurrence, absent when the walk meets
// malformed data first or the entry's value runs past `an`.  *entry (optional) = the entry's offset in `a` and
// *entry_end its end, when found.
FGB_HD TagRef find_tag(const uint8_t* a, size_t an, const char tag[2], size_t* entry = nullptr,
                       size_t* entry_end = nullptr) {
  TagRef r;
  size_t p = 0;
  while (p + 3 <= an) {
    const uint8_t vt = a[p + 2];
    uint8_t sub = 0;
    uint32_t count = 0;
    const size_t size = value_size(a, an, p, &sub, &count);
    if (!size || p + 3 + size > an) return r;
    if (a[p] == static_cast<uint8_t>(tag[0]) && a[p + 1] == static_cast<uint8_t>(tag[1])) {
      r.type = vt; r.sub = sub; r.count = vt == 'B' ? count : static_cast<uint32_t>(size);
      r.data = a + p + 3 + (vt == 'B' ? 5 : 0);
      if (entry) *entry = p;
      if (entry_end) *entry_end = p + 3 + size;
      return r;
    }
    p += 3 + size;
  }
  return r;
}

FGB_HD bool tag_int(const TagRef& t, int64_t* v) {            // raw-bam tags.rs:118-150: any integer type
  switch (t.type) {
    case 'c': *v = static_cast<int8_t>(t.data[0]); return true;
    case 'C': *v = t.data[0]; return true;
    case 's': *v = static_cast<int16_t>(ld16(t.data)); return true;
    case 'S': *v = ld16(t.data); return true;
    case 'i': *v = static_cast<int32_t>(ld32(t.data)); return true;
    case 'I': *v = ld32(t.data); return true;
    default: return false;
  }
}
FGB_HD bool tag_float(const TagRef& t, float* v) {            // 'f' only
  if (t.type != 'f') return false;
  const uint32_t b = ld32(t.data);
  float f;
  memcpy(&f, &b, 4);
  *v = f;
  return true;
}
FGB_HD uint16_t array_u16(const TagRef& t, size_t i) {        // raw-bam tags.rs:479-497
  if (t.type != 'B' || i >= t.count) return 0;
  switch (t.sub) {
    case 'C': return t.data[i];
    case 'S': return ld16(t.data + 2 * i);
    case 's': { int16_t v = static_cast<int16_t>(ld16(t.data + 2 * i)); return v > 0 ? static_cast<uint16_t>(v) : 0; }
    case 'c': { int8_t v = static_cast<int8_t>(t.data[i]); return v > 0 ? static_cast<uint16_t>(v) : 0; }
    default: return 0;
  }
}

struct Tier {               // FilterThresholds, filter.rs:31-40
  uint64_t min_reads;
  double max_read_error_rate, max_base_error_rate;
};

FGB_HD int filter_read(const uint8_t* aux, size_t an, const Tier& th) {          // filter.rs:453-471
  int64_t depth;
  if (tag_int(find_tag(aux, an, "cD"), &depth)) {
    const int64_t mr = th.min_reads > static_cast<uint64_t>(INT64_MAX) ? INT64_MAX : static_cast<int64_t>(th.min_reads);
    if (depth < mr) return FGB_FILTER_INSUFFICIENT_READS;
  }
  float er;
  if (tag_float(find_tag(aux, an, "cE"), &er) && static_cast<double>(er) > th.max_read_error_rate)
    return FGB_FILTER_EXCESSIVE_ERROR_RATE;
  return FGB_FILTER_PASS;
}

FGB_HD int filter_duplex_read(const uint8_t* aux, size_t an, const Tier& cc, const Tier& ab, const Tier& ba) {
  int r = filter_read(aux, an, cc);                                                // filter.rs:477-557
  if (r != FGB_FILTER_PASS) return r;
  int64_t a_d = 0, b_d = 0;
  bool has_a = tag_int(find_tag(aux, an, "aD"), &a_d) || tag_int(find_tag(aux, an, "aM"), &a_d);
  bool has_b = tag_int(find_tag(aux, an, "bD"), &b_d) || tag_int(find_tag(aux, an, "bM"), &b_d);
  float a_e = 0, b_e = 0;
  const bool has_ae = tag_float(find_tag(aux, an, "aE"), &a_e), has_be = tag_float(find_tag(aux, an, "bE"), &b_e);
  int64_t worst_d, best_d;
  if (has_a && has_b) { if (a_d < b_d) { worst_d = a_d; best_d = b_d; } else { worst_d = b_d; best_d = a_d; } }
  else if (has_a) { worst_d = 0; best_d = a_d; }
  else if (has_b) { worst_d = 0; best_d = b_d; }
  else return FGB_FILTER_PASS;
  float best_e, worst_e;
  if (has_ae && has_be) { if (a_e < b_e) { best_e = a_e; worst_e = b_e; } else { best_e = b_e; worst_e = a_e; } }
  else if (has_ae) best_e = worst_e = a_e;
  else if (has_be) best_e = worst_e = b_e;
  else best_e = worst_e = 0.0f;
  // `(depth as usize) < min_reads`: a negative depth wraps to a huge usize and passes
  if (static_cast<uint64_t>(best_d) < ab.min_reads) return FGB_FILTER_INSUFFICIENT_READS;
  if (static_cast<double>(best_e) > ab.max_read_error_rate) return FGB_FILTER_EXCESSIVE_ERROR_RATE;
  if (static_cast<uint64_t>(worst_d) < ba.min_reads) return FGB_FILTER_INSUFFICIENT_READS;
  if (static_cast<double>(worst_e) > ba.max_read_error_rate) return FGB_FILTER_EXCESSIVE_ERROR_RATE;
  return FGB_FILTER_PASS;
}

// find_tag_type semantics (tags.rs:56-59 over find_tag_position, :13-34): an entry's name is matched before its value
// is sized, so the first entry named `tag` counts even when its type byte is unknown or its value runs past the aux
// data; the walk stops at the first malformed entry before it.  find_tag, which every value lookup goes through,
// reports such an entry as absent.
FGB_HD bool has_tag(const uint8_t* a, size_t an, const char tag[2]) {
  size_t p = 0;
  while (p + 3 <= an) {
    if (a[p] == static_cast<uint8_t>(tag[0]) && a[p + 1] == static_cast<uint8_t>(tag[1])) return true;
    uint8_t sub;
    uint32_t count;
    const size_t size = value_size(a, an, p, &sub, &count);
    if (!size) return false;
    p += 3 + size;
  }
  return false;
}

// is_duplex_consensus (filter.rs:443-446): an aD or bD entry, found as find_tag_type finds it
FGB_HD bool is_duplex(const uint8_t* aux, size_t an) { return has_tag(aux, an, "aD") || has_tag(aux, an, "bD"); }

FGB_HD uint8_t base_code(const uint8_t* rec, size_t so, size_t i) {   // the 4-bit code of base i
  const uint8_t b = rec[so + i / 2];
  return (i & 1) ? (b & 0xF) : (b >> 4);
}
FGB_HD uint8_t get_base(const uint8_t* rec, size_t so, size_t i) {
  return static_cast<uint8_t>("=ACMGRSVTWYHKDBN"[base_code(rec, so, i)]);
}

// Z string or B:C / B:c array (filter.rs:621-639); absent / other types -> false
FGB_HD bool string_or_u8(const TagRef& t, const uint8_t** p, size_t* n) {
  if (t.type == 'Z') { *p = t.data; *n = t.count ? t.count - 1 : 0; return true; }
  if (t.type == 'B' && (t.sub == 'C' || t.sub == 'c')) { *p = t.data; *n = t.count; return true; }
  return false;
}

// mask_bases' per-base predicate (filter.rs:672-684): depth / errors from cd / ce, q the base's quality
FGB_HD bool mask_simplex(uint8_t q, uint16_t depth, uint16_t errors, const Tier& th, int min_bq) {
  return (min_bq >= 0 && q < min_bq) || depth < th.min_reads ||
         (depth > 0 && static_cast<double>(errors) / static_cast<double>(depth) > th.max_base_error_rate);
}

// mask_duplex_bases' per-base predicate (filter.rs:730-800) for a base that is not N: the three tiers, then
// single-strand agreement (x / y: the base of ac / bc at i, 'N' past their end or without them)
FGB_HD bool mask_duplex(uint8_t q, uint16_t a_d, uint16_t b_d, uint16_t a_e, uint16_t b_e, const Tier& cc,
                        const Tier& ab, const Tier& ba, int min_bq, bool require_ss_agreement, uint8_t x, uint8_t y) {
  const uint16_t best_d = a_d > b_d ? a_d : b_d, worst_d = a_d < b_d ? a_d : b_d;
  const double a_r = a_d > 0 ? static_cast<double>(a_e) / static_cast<double>(a_d) : 0.0;
  const double b_r = b_d > 0 ? static_cast<double>(b_e) / static_cast<double>(b_d) : 0.0;
  const double best_r = a_r < b_r ? a_r : b_r, worst_r = a_r > b_r ? a_r : b_r;
  const uint32_t tot_d = static_cast<uint32_t>(a_d) + b_d;
  const double tot_r = tot_d > 0 ? static_cast<double>(static_cast<uint32_t>(a_e) + b_e) / static_cast<double>(tot_d) : 0.0;
  const bool should = (min_bq >= 0 && q < min_bq) || tot_d < cc.min_reads || tot_r > cc.max_base_error_rate ||
                      best_d < ab.min_reads || best_r > ab.max_base_error_rate ||
                      worst_d < ba.min_reads || worst_r > ba.max_base_error_rate;
  return should || (require_ss_agreement && a_d > 0 && b_d > 0 && x != y);
}

// The read-level no-call and mean-quality gates (commands/filter.rs:909-929) from compute_read_stats' counts
FGB_HD int no_call_gate(uint64_t L, uint64_t n_count, uint64_t qsum, double min_mean_q, double max_no_call) {
  const uint64_t non_n = L - n_count;
  const double mean_q = non_n ? static_cast<double>(qsum) / static_cast<double>(non_n) : 0.0;
  if (min_mean_q >= 0.0 && mean_q < min_mean_q) return FGB_FILTER_LOW_MEAN_QUALITY;
  if (max_no_call >= 1.0) {
    if (static_cast<double>(n_count) > max_no_call) return FGB_FILTER_TOO_MANY_NO_CALLS;
  } else {
    const double frac = L ? static_cast<double>(n_count) / static_cast<double>(L) : 0.0;
    if (frac > max_no_call) return FGB_FILTER_TOO_MANY_NO_CALLS;
  }
  return FGB_FILTER_PASS;
}

// ---- host loops over one assembled record (fgb_filter_record, the duplex caller's fused filter) ----

inline void mask_base(uint8_t* rec, size_t so, size_t i) {     // nibble 15 = N
  uint8_t& b = rec[so + i / 2];
  b = (i & 1) ? static_cast<uint8_t>(b | 0x0F) : static_cast<uint8_t>(b | 0xF0);
}

inline uint32_t mask_bases(uint8_t* rec, size_t n, const Tier& th, int min_bq) {   // filter.rs:650-696
  const bam::View v(rec, n);
  const size_t so = v.seq_off(), qo = v.qual_off(), L = v.l_seq(), ao = v.aux_off();
  const uint8_t* aux = rec + ao;
  const size_t an = n - ao;
  const TagRef cd = find_tag(aux, an, "cd"), ce = find_tag(aux, an, "ce");
  uint32_t masked = 0;
  for (size_t i = 0; i < L; ++i) {
    if (mask_simplex(rec[qo + i], array_u16(cd, i), array_u16(ce, i), th, min_bq)) {
      if (get_base(rec, so, i) != 'N') ++masked;
      mask_base(rec, so, i);
      rec[qo + i] = 2;
    }
  }
  return masked;
}

inline uint32_t mask_duplex_bases(uint8_t* rec, size_t n, const Tier& cc, const Tier& ab, const Tier& ba,
                                  int min_bq, bool require_ss_agreement) {          // filter.rs:702-806
  const bam::View v(rec, n);
  const size_t so = v.seq_off(), qo = v.qual_off(), L = v.l_seq(), ao = v.aux_off();
  const uint8_t* aux = rec + ao;
  const size_t an = n - ao;
  const TagRef ad = find_tag(aux, an, "ad"), ae = find_tag(aux, an, "ae");
  const TagRef bd = find_tag(aux, an, "bd"), be = find_tag(aux, an, "be");
  const uint8_t *acp = nullptr, *bcp = nullptr;
  size_t acn = 0, bcn = 0;
  bool has_ac = false, has_bc = false;
  if (require_ss_agreement) {
    has_ac = string_or_u8(find_tag(aux, an, "ac"), &acp, &acn);
    has_bc = string_or_u8(find_tag(aux, an, "bc"), &bcp, &bcn);
  }
  uint32_t masked = 0;
  for (size_t i = 0; i < L; ++i) {
    if (get_base(rec, so, i) == 'N') continue;
    const uint8_t x = (has_ac && i < acn) ? acp[i] : 'N', y = (has_bc && i < bcn) ? bcp[i] : 'N';
    if (mask_duplex(rec[qo + i], array_u16(ad, i), array_u16(bd, i), array_u16(ae, i), array_u16(be, i), cc, ab, ba,
                    min_bq, require_ss_agreement, x, y)) {
      ++masked;
      mask_base(rec, so, i);
      rec[qo + i] = 2;
    }
  }
  return masked;
}

// compute_read_stats + check_no_call_and_quality (filter.rs:565-590, commands/filter.rs:909-929)
inline int no_call_and_quality(const uint8_t* rec, size_t n, double min_mean_q, double max_no_call) {
  const bam::View v(rec, n);
  const size_t so = v.seq_off(), qo = v.qual_off(), L = v.l_seq();
  uint64_t n_count = 0, qsum = 0;
  for (size_t i = 0; i < L; ++i) {
    if (get_base(rec, so, i) == 'N') ++n_count; else qsum += rec[qo + i];
  }
  return no_call_gate(L, n_count, qsum, min_mean_q, max_no_call);
}

// One record through the filter (commands/filter.rs:770-793 masking, :949-968 read-level gates).
inline int filter_record(uint8_t* rec, size_t n, const fgb_duplex_filter_params& p, uint32_t* masked) {
  const Tier cc{p.cc.min_reads, p.cc.max_read_error_rate, p.cc.max_base_error_rate};
  const Tier ab{p.ab_min_reads, p.ab_max_read_error_rate, p.ab_max_base_error_rate};
  const Tier ba{p.ba_min_reads, p.ba_max_read_error_rate, p.ba_max_base_error_rate};
  const bam::View v(rec, n);
  const size_t ao = v.aux_off();
  const bool duplex = is_duplex(rec + ao, n - ao);
  int st;
  if (duplex) {
    *masked = mask_duplex_bases(rec, n, cc, ab, ba, p.cc.min_base_quality, p.require_ss_agreement != 0);
    st = filter_duplex_read(rec + ao, n - ao, cc, ab, ba);
  } else {
    *masked = mask_bases(rec, n, cc, p.cc.min_base_quality);
    st = filter_read(rec + ao, n - ao, cc);
  }
  if (st != FGB_FILTER_PASS) return st;
  return no_call_and_quality(rec, n, p.cc.min_mean_base_quality, p.cc.max_no_call_fraction);
}

}  // namespace rfilter
}  // namespace fgb
