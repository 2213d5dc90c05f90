// Record rules `fgumi group` and `fgumi dedup` share: record checks, the aux walk of their filters (MQ and the UMI in
// one pass), the unclipped 5' end, the pair-orientation split with each template's UMI, and update_string_tag on
// output; then the queue both keep around fgb_umi_assign.  Used by group_host.cpp and dedup_host.cpp; the citations are
// to fgumi 0.2.0 as there.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <map>
#include <numeric>
#include <string>
#include <string_view>
#include <vector>

#include "../../../include/fgumi_b200.h"
#include "bam.h"
#include "umi_host.h"

namespace fgb {
namespace grp {

using bam::View;

constexpr uint64_t kNone = UINT64_MAX;

inline std::string_view read_name(const View& v) {
  const uint32_t l = v.l_read_name();
  return std::string_view(reinterpret_cast<const char*>(v.b + 32), l ? l - 1 : 0);
}

inline bool record_ok(const uint8_t* records, const uint64_t* rec_off, uint64_t i) {
  if (rec_off[i + 1] < rec_off[i] || rec_off[i + 1] - rec_off[i] < 32) return false;
  const View v(records + rec_off[i], rec_off[i + 1] - rec_off[i]);
  return 32 + static_cast<size_t>(v.l_read_name()) <= v.n && v.cigar_in_bounds() && v.aux_off() <= v.n;
}

// tag_value_size (fields.rs:289-310); 0 = unknown type or truncated
inline size_t tag_value_size(uint8_t t, const uint8_t* d, size_t n) {
  switch (t) {
    case 'A': case 'c': case 'C': return 1;
    case 's': case 'S': return 2;
    case 'i': case 'I': case 'f': return 4;
    case 'Z': case 'H': {
      const void* z = std::memchr(d, 0, n);
      return z ? static_cast<const uint8_t*>(z) - d + 1 : 0;
    }
    case 'B': {
      if (n < 5) return 0;
      const uint8_t e = d[0];
      const size_t es = (e == 'c' || e == 'C') ? 1 : (e == 's' || e == 'S') ? 2 : (e == 'i' || e == 'I' || e == 'f') ? 4 : 0;
      return es ? 5 + static_cast<size_t>(bam::rd32(d + 1)) * es : 0;
    }
    default: return 0;
  }
}

// unclipped_5prime_from_raw_bam (cigar.rs:201-228, 470-508): 1-based; 0 for an unmapped read, i32::MAX without CIGAR
inline int32_t unclipped_5prime(const View& v) {
  const uint16_t f = v.flags();
  if (f & bam::kUnmapped) return 0;
  const uint32_t n = v.n_cigar();
  if (n == 0 || !v.cigar_in_bounds()) return INT32_MAX;
  const int32_t pos = v.pos() + 1;
  if (!(f & bam::kReverse)) {
    int32_t clipped = 0;
    for (uint32_t i = 0; i < n; ++i) {
      const uint32_t op = v.cigar_op(i);
      if ((op & 0xF) == 4 || (op & 0xF) == 5) clipped += static_cast<int32_t>(op >> 4);
      else break;
    }
    return pos - clipped;
  }
  int32_t ref_len = 0, trailing = 0;
  bool saw = false;
  for (uint32_t i = 0; i < n; ++i) {
    const uint32_t op = v.cigar_op(i);
    if (bam::consumes_ref(op & 0xF)) { ref_len += static_cast<int32_t>(op >> 4); trailing = 0; saw = true; }
    else if (((op & 0xF) == 4 || (op & 0xF) == 5) && saw) trailing += static_cast<int32_t>(op >> 4);
  }
  return pos + ref_len + trailing - 1;
}

// The filters' one aux walk for the mate's MQ and the UMI (group.rs:157-221, dedup.rs:299-361): the first UMI tag of
// type Z, and MQ of any integer type widened to i64 (a float or string MQ, or a truncated one, is None).  The walk
// stops once it has what it looks for, at an unknown type or at a truncated value.
struct MqUmi {
  bool have_mq = false, have_umi = false;
  int64_t mq = 0;
  const uint8_t* umi = nullptr;
  size_t umi_len = 0;
};

inline MqUmi scan_mq_umi(const View& r, bool check_mq, bool check_umi, const char umi_tag[2]) {
  MqUmi s;
  const uint8_t* a = r.b + r.aux_off();
  const size_t an = r.n - r.aux_off();
  size_t p = 0;
  while (p + 3 <= an) {
    const uint8_t t0 = a[p], t1 = a[p + 1], vt = a[p + 2];
    if (check_umi && t0 == static_cast<uint8_t>(umi_tag[0]) && t1 == static_cast<uint8_t>(umi_tag[1]) && vt == 'Z') {
      const void* z = std::memchr(a + p + 3, 0, an - (p + 3));
      if (!z) break;
      s.umi = a + p + 3;
      s.umi_len = static_cast<const uint8_t*>(z) - s.umi;
      s.have_umi = true;
      p += 3 + s.umi_len + 1;
      if (!check_mq || s.have_mq) break;
      continue;
    }
    if (check_mq && t0 == 'M' && t1 == 'Q') {
      const uint8_t* d = a + p + 3;
      const size_t left = an - (p + 3);
      s.have_mq = true;
      switch (vt) {
        case 'C': if (left >= 1) s.mq = d[0]; else s.have_mq = false; break;
        case 'c': if (left >= 1) s.mq = static_cast<int8_t>(d[0]); else s.have_mq = false; break;
        case 'S': if (left >= 2) s.mq = bam::rd16(d); else s.have_mq = false; break;
        case 's': if (left >= 2) s.mq = static_cast<int16_t>(bam::rd16(d)); else s.have_mq = false; break;
        case 'I': if (left >= 4) s.mq = bam::rd32(d); else s.have_mq = false; break;
        case 'i': if (left >= 4) s.mq = bam::rdi32(d); else s.have_mq = false; break;
        default: s.have_mq = false;
      }
    }
    const size_t size = tag_value_size(vt, a + p + 3, an - (p + 3));
    if (!size) break;
    p += 3 + size;
    if ((!check_umi || s.have_umi) && (!check_mq || s.have_mq)) break;
  }
  return s;
}

// validate_umi (fgumi-umi lib.rs:323-333): -1 for an upper-case N, else the number of ACGT bases (either case)
inline int64_t umi_bases(const uint8_t* umi, size_t len) {
  int64_t bases = 0;
  for (size_t i = 0; i < len; ++i) {
    const uint8_t c = umi[i];
    if (c == 'N') return -1;
    if (c == 'A' || c == 'C' || c == 'G' || c == 'T' || c == 'a' || c == 'c' || c == 'g' || c == 't') ++bases;
  }
  return bases;
}

// build_templates_from_records + Template::from_records (grouper.rs:596-651, template.rs:159-330) for the records
// k in [b, e) of one QNAME run, flags(k) giving each one's flags: appends them to `order` in template order -- R1, R2,
// then the R1 and the R2 supplementary and the R1 and the R2 secondary records, each list reversed (fgbio's prepend
// order; secondary wins over supplementary) -- and sets *r1 / *r2 to the primary reads (-1: absent).  The two-record
// fast path's swap lands on the same order.  Returns "" or the reference's error for a second primary R1 or R2, with
// *dup = that record.  `lists` is scratch.
template <class Flags>
std::string template_order(uint64_t b, uint64_t e, Flags&& flags, std::string_view name, std::vector<uint64_t> lists[4],
                           std::vector<uint64_t>* order, int64_t* r1, int64_t* r2, uint64_t* dup) {
  *r1 = -1;
  *r2 = -1;
  for (int l = 0; l < 4; ++l) lists[l].clear();   // r1 supp, r2 supp, r1 sec, r2 sec
  for (uint64_t k = b; k < e; ++k) {
    const uint16_t f = flags(k);
    const bool is_r1 = !(f & bam::kPaired) || (f & bam::kFirst);
    if (f & bam::kSecondary) { lists[is_r1 ? 2 : 3].push_back(k); continue; }
    if (f & bam::kSupplementary) { lists[is_r1 ? 0 : 1].push_back(k); continue; }
    int64_t& slot = is_r1 ? *r1 : *r2;
    if (slot >= 0) {
      *dup = k;
      return std::string("Multiple non-secondary, non-supplemental ") + (is_r1 ? "R1" : "R2") + " records for read '" +
             std::string(name) + "'";
    }
    slot = static_cast<int64_t>(k);
  }
  if (*r1 >= 0) order->push_back(static_cast<uint64_t>(*r1));
  if (*r2 >= 0) order->push_back(static_cast<uint64_t>(*r2));
  for (int l = 0; l < 4; ++l) order->insert(order->end(), lists[l].rbegin(), lists[l].rend());
  return "";
}

// The calls of one position group and the UMI of each template, as the assigner receives them.
struct Calls {
  std::vector<uint32_t> order;     // templates in call order (the calls concatenated)
  std::vector<uint32_t> call_end;
  std::string umis;                // per `order` entry: its UMI as umi_for_read made it
  std::vector<uint64_t> umi_end;
};

// The orientation split (group.rs:373-422, dedup.rs:543-587): sub-groups in (r1_positive, r2_positive) order, false
// first; paired strategies take the whole group as one call.  Then the UMI of each template (group.rs:440-477,
// dedup.rs:498-529): R1's tag if R1 exists, else R2's, through umi_for_read; "" for every template with no_umi.
// r1(t) / r2(t) give template t's primary reads (nullptr: absent).  Returns "" or why the reference's assignment
// fails: group drops the position group, dedup fails the command.
template <class R1, class R2>
std::string split_and_umis(const fgb_umi_options& umi, bool no_umi, const char umi_tag[2], size_t nt, R1&& r1, R2&& r2,
                           Calls* c) {
  if (umi.strategy != FGB_UMI_PAIRED) {
    std::vector<uint8_t> ori(nt);
    for (size_t t = 0; t < nt; ++t) {
      const View* a = r1(t);
      const View* b = r2(t);
      const bool p1 = !a || !(a->flags() & bam::kReverse);
      const bool p2 = !b || !(b->flags() & bam::kReverse);
      ori[t] = static_cast<uint8_t>(p1 * 2 + p2);
    }
    for (uint8_t o = 0; o < 4; ++o) {
      const size_t before = c->order.size();
      for (size_t t = 0; t < nt; ++t) if (ori[t] == o) c->order.push_back(static_cast<uint32_t>(t));
      if (c->order.size() > before) c->call_end.push_back(static_cast<uint32_t>(c->order.size()));
    }
  } else {
    c->order.resize(nt);
    std::iota(c->order.begin(), c->order.end(), 0u);
    c->call_end.push_back(static_cast<uint32_t>(nt));
  }
  c->umi_end.reserve(nt);
  std::vector<uint8_t> buf;
  for (uint32_t t : c->order) {
    if (!no_umi) {
      const View* a = r1(t);
      const View* b = r2(t);
      const View& v = a ? *a : *b;
      const uint8_t* val = nullptr;
      size_t len = 0;
      if (!bam::find_string_tag(v, umi_tag, &val, &len)) return "No UMI tag found";
      if (!bam::valid_utf8(val, len)) return "Invalid UTF-8 in UMI";
      bool r1_earlier = true;   // is_r1_genomically_earlier_raw (group.rs:268-279, dedup.rs:460-469)
      if (a && b)
        r1_earlier = a->ref_id() != b->ref_id() ? a->ref_id() < b->ref_id() : unclipped_5prime(*a) <= unclipped_5prime(*b);
      buf.resize(2 * len + 2 * umi.edits + 16);
      size_t out_len = 0;
      if (fgb_host_umi_for_read(&umi, val, len, r1_earlier, buf.data(), buf.size(), &out_len) != FGB_OK)
        return "Paired strategy used but UMI did not contain 2 segments: " + std::string(reinterpret_cast<const char*>(val), len);
      c->umis.append(reinterpret_cast<const char*>(buf.data()), out_len);
    }
    c->umi_end.push_back(c->umis.size());
  }
  return "";
}

// update_string_tag (fgumi-raw-bam tags.rs:694-721) on a copy of `rec`, appended to `out`: the first entry of the
// tag (of any type) has its value overwritten when the lengths agree (its type byte is kept), is replaced by a Z
// entry when they differ; a record without the tag gets one appended.
inline void emit_with_tag(const uint8_t* rec, size_t n, const char tag[2], std::string_view val, std::vector<uint8_t>* out) {
  const View v(rec, n);
  const size_t aux = v.aux_off();
  size_t p = aux, start = kNone, end = 0;
  while (aux < n && p + 3 <= n) {
    const size_t size = tag_value_size(rec[p + 2], rec + p + 3, n - (p + 3));
    if (rec[p] == static_cast<uint8_t>(tag[0]) && rec[p + 1] == static_cast<uint8_t>(tag[1])) {
      if (size) { start = p; end = p + 3 + size; }
      break;
    }
    if (!size) break;
    p += 3 + size;
  }
  const uint32_t bs0 = 0;
  const size_t at = out->size();
  out->insert(out->end(), reinterpret_cast<const uint8_t*>(&bs0), reinterpret_cast<const uint8_t*>(&bs0) + 4);
  const uint8_t* vb = reinterpret_cast<const uint8_t*>(val.data());
  const uint8_t z[3] = {static_cast<uint8_t>(tag[0]), static_cast<uint8_t>(tag[1]), 'Z'};
  if (start != kNone && end - start - 4 == val.size()) {
    out->insert(out->end(), rec, rec + n);
    std::memcpy(out->data() + at + 4 + start + 3, vb, val.size());
  } else if (start != kNone) {
    out->insert(out->end(), rec, rec + start);
    out->insert(out->end(), z, z + 3);
    out->insert(out->end(), vb, vb + val.size());
    out->push_back(0);
    out->insert(out->end(), rec + end, rec + n);
  } else {
    out->insert(out->end(), rec, rec + n);
    out->insert(out->end(), z, z + 3);
    out->insert(out->end(), vb, vb + val.size());
    out->push_back(0);
  }
  const uint32_t bs = static_cast<uint32_t>(out->size() - at - 4);
  std::memcpy(out->data() + at, &bs, 4);
}

inline void emit_plain(const uint8_t* rec, size_t n, std::vector<uint8_t>* out) {
  const uint32_t bs = static_cast<uint32_t>(n);
  out->insert(out->end(), reinterpret_cast<const uint8_t*>(&bs), reinterpret_cast<const uint8_t*>(&bs) + 4);
  out->insert(out->end(), rec, rec + n);
}

// The MI string of a molecule: its number plus the run's base, "/A" or "/B" for paired molecules
inline void mi_string(uint8_t kind, uint64_t id, uint64_t base, std::string* mi) {
  *mi = std::to_string(id + base);
  if (kind == FGB_MOL_A) *mi += "/A";
  else if (kind == FGB_MOL_B) *mi += "/B";
}

// MoleculeId::to_vec_index + 1 (lib.rs:112-119), 0 for None, so that None sorts first
inline uint64_t vec_index(uint8_t kind, uint64_t id) {
  return kind == FGB_MOL_NONE ? 0 : kind == FGB_MOL_SINGLE ? id + 1 : 2 * id + (kind == FGB_MOL_B) + 1;
}

// ---- the queue of the grouper and the deduper around fgb_umi_assign ----------------------------------------------

// The device handle of a grouper or deduper (none for FGB_DEVICE_NONE).  The assignment reads none of the consensus
// parameters; fgb_create only wants them valid.
inline fgb_status open_handle(int device, fgb_handle** h) {
  if (device == FGB_DEVICE_NONE) return FGB_OK;
  fgb_params p{};
  p.error_rate_pre_umi = 45;
  p.error_rate_post_umi = 40;
  p.min_consensus_base_quality = 40;
  p.min_reads = 1;
  return fgb_create(device, &p, h);
}

// fgb_*_add_groups up to the queue: the group table and every record it covers checked, then prepare(b, e, &(*prep)[x])
// for the records [b, e) of each position group x on n_threads.  A failure leaves "<who>: ..." in *err.
template <class G, class Prepare>
fgb_status prepare_groups(const char* who, const uint8_t* records, const uint64_t* rec_off, const uint64_t* group_rec,
                          uint64_t n_groups, uint32_t n_threads, Prepare&& prepare, std::vector<G>* prep,
                          std::string* err) {
  for (uint64_t x = 0; x < n_groups; ++x)
    if (group_rec[x + 1] < group_rec[x]) { *err = std::string(who) + ": group_rec descends"; return FGB_ERR_LAYOUT; }
  const uint64_t r0 = n_groups ? group_rec[0] : 0, r1 = n_groups ? group_rec[n_groups] : 0;
  for (uint64_t i = r0; i < r1; ++i)
    if (!record_ok(records, rec_off, i)) {
      *err = std::string(who) + ": record " + std::to_string(i) + " is malformed";
      return FGB_ERR_LAYOUT;
    }
  prep->resize(n_groups);
  std::vector<std::string> why(n_groups);
  fgb_umi::parallel_for(n_groups, n_threads, [&](uint64_t x) {
    why[x] = prepare(group_rec[x], group_rec[x + 1], &(*prep)[x]);
  });
  for (uint64_t x = 0; x < n_groups; ++x)
    if (!why[x].empty()) {
      *err = std::string(who) + ": position group " + std::to_string(x) + ": " + why[x];
      return FGB_ERR_INVALID_ARG;
    }
  return FGB_OK;
}

// The UMI batch of a queue of position groups as fgb_umi_assign takes it: every group's calls and UMIs (its
// Calls c) back to back, group b's first UMI at call_off[group_off[b]].  Built on demand; ready = false whenever
// the queue changes.
struct UmiBatch {
  bool ready = false;
  std::vector<uint8_t> umis;
  std::vector<uint64_t> umi_off, call_off, group_off;

  template <class G>
  void build(const std::vector<G>& queue) {
    if (ready) return;
    umis.clear(); umi_off.assign(1, 0); call_off.assign(1, 0); group_off.assign(1, 0);
    for (const G& gp : queue) {
      const uint64_t base = umis.size();
      umis.insert(umis.end(), gp.c.umis.begin(), gp.c.umis.end());
      for (uint64_t e : gp.c.umi_end) umi_off.push_back(base + e);
      const uint64_t ub = call_off.back();
      for (uint32_t e : gp.c.call_end) call_off.push_back(ub + e);
      group_off.push_back(call_off.size() - 1);
    }
    ready = true;
  }
  uint64_t n_umis() const { return umi_off.size() - 1; }
  uint64_t n_groups() const { return group_off.size() - 1; }

  // fgb_*_pending
  void pending(const uint8_t** u, const uint64_t** uo, uint64_t* nu, const uint64_t** co, uint64_t* nc,
               const uint64_t** go, uint64_t* ng) const {
    *u = umis.data();
    *uo = umi_off.data();
    *nu = n_umis();
    *co = call_off.data();
    *nc = call_off.size() - 1;
    *go = group_off.data();
    *ng = n_groups();
  }

  // fgb_umi_assign on the batch; a failure leaves "<who>: <the handle's error>" in *err
  fgb_status assign(fgb_handle* h, const fgb_umi_options& umi, const char* who, uint64_t* ids, uint8_t* kinds,
                    uint64_t* counts, std::string* err) const {
    const uint8_t no_bytes = 0;   // every UMI empty (no_umi): the ABI still wants a pointer
    const fgb_status st = fgb_umi_assign(h, &umi, umis.empty() ? &no_bytes : umis.data(), umi_off.data(), n_umis(),
                                         call_off.data(), call_off.size() - 1, group_off.data(), n_groups(), ids,
                                         kinds, counts);
    if (st != FGB_OK) {
      std::string e(fgb_last_error(h, nullptr, 0), '\0');
      fgb_last_error(h, &e[0], e.size() + 1);
      *err = std::string(who) + ": " + e;
    }
    return st;
  }
};

// The MI base of each of a flush's ng groups: the counter *next advances by max(id) + 1 = mi_count[b] per group
// (group.rs:1569-1575, dedup.rs:791-797, 1123-1133).  False, with *next unchanged, when it would overflow.
inline bool mi_bases(const uint64_t* mi_count, uint64_t ng, uint64_t* next, std::vector<uint64_t>* base) {
  base->resize(ng);
  uint64_t at = *next;
  for (uint64_t b = 0; b < ng; ++b) {
    (*base)[b] = at;
    if (at + mi_count[b] < at) return false;
    at += mi_count[b];
  }
  *next = at;
  return true;
}

// The groups' output bytes back to back in *out (copied on n_threads), so that the stream is in queue order for any
// thread count; returns the number of records.
template <class O>
uint64_t concat_outputs(const std::vector<O>& outs, uint32_t n_threads, std::vector<uint8_t>* out) {
  const uint64_t ng = outs.size();
  std::vector<uint64_t> at(ng + 1, 0);
  uint64_t recs = 0;
  for (uint64_t b = 0; b < ng; ++b) { at[b + 1] = at[b] + outs[b].bytes.size(); recs += outs[b].n_records; }
  out->resize(at[ng]);
  fgb_umi::parallel_for(ng, n_threads, [&](uint64_t b) {
    if (!outs[b].bytes.empty()) std::memcpy(out->data() + at[b], outs[b].bytes.data(), outs[b].bytes.size());
  });
  return recs;
}

// fgb_*_histogram: *n entries; sizes / counts filled when cap holds them all
inline fgb_status copy_histogram(const std::map<uint64_t, uint64_t>& h, uint64_t* sizes, uint64_t* counts,
                                 uint64_t cap, uint64_t* n) {
  *n = h.size();
  if (cap < h.size()) return FGB_OK;
  if (h.size() && (!sizes || !counts)) return FGB_ERR_INVALID_ARG;
  uint64_t i = 0;
  for (const auto& [s, c] : h) { sizes[i] = s; counts[i] = c; ++i; }
  return FGB_OK;
}

// fgb_*_last_error: the message's length; as much of it as fits in buf, NUL-terminated
inline size_t copy_error(const std::string& e, char* buf, size_t buf_len) {
  if (buf && buf_len) {
    const size_t n = std::min(buf_len - 1, e.size());
    std::memcpy(buf, e.data(), n);
    buf[n] = 0;
  }
  return e.size();
}

// Position grouping of fgb_host_group_by_position and, with include_secondary_supplementary, of
// fgb_host_dedup_group_by_position.  Defined in group_host.cpp.
fgb_status group_by_position(const uint8_t* records, const uint64_t* rec_off, uint64_t n_records,
                             const char* header_text, size_t header_len, const char* cell_tag,
                             bool include_secondary_supplementary, uint8_t* keep, uint64_t* group_begin,
                             uint64_t* n_groups, uint64_t* bad_record);

}  // namespace grp
}  // namespace fgb
