// Host-side BAM record access and consensus-record assembly (product code, header-only).
//
// Behavioural spec (reference = fgumi 0.2.0, crates/):
//   fgumi-raw-bam/src/fields.rs:6-23,240-265,289-310,393-502   record layout, flags, aux walking
//   fgumi-raw-bam/src/sequence.rs:9-35,148-209                 4-bit sequence codec
//   fgumi-raw-bam/src/cigar.rs:50-70,82-101,137-150,294-306,514-573   CIGAR helpers, MC parsing
//   fgumi-raw-bam/src/overlap.rs:15-260                        FR-pair test, mate-overlap clip
//   fgumi-raw-bam/src/noodles_compat.rs:10-55                  simplify_cigar_from_raw
//   fgumi-raw-bam/src/builder.rs:90-230, tags.rs:512-667       UnmappedSamBuilder + tag encoders
//   fgumi-sam/src/clipper.rs:2425-2448                         is_cigar_prefix
//   fgumi-dna/src/dna.rs:30-60                                 reverse_complement
#pragma once
#include <cstdint>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

namespace fgb {
namespace bam {

enum : uint16_t {
  kPaired = 0x1, kProperPair = 0x2, kUnmapped = 0x4, kMateUnmapped = 0x8, kReverse = 0x10,
  kMateReverse = 0x20, kFirst = 0x40, kLast = 0x80, kSecondary = 0x100, kSupplementary = 0x800
};

inline uint16_t rd16(const uint8_t* p) { uint16_t v; std::memcpy(&v, p, 2); return v; }
inline uint32_t rd32(const uint8_t* p) { uint32_t v; std::memcpy(&v, p, 4); return v; }
inline int32_t rdi32(const uint8_t* p) { int32_t v; std::memcpy(&v, p, 4); return v; }

// A borrowed view of one BAM record (no block_size prefix).
struct View {
  const uint8_t* b;
  size_t n;
  View(const uint8_t* p, size_t len) : b(p), n(len) {}
  int32_t ref_id() const { return rdi32(b); }
  int32_t pos() const { return rdi32(b + 4); }
  uint32_t l_read_name() const { return b[8]; }
  uint32_t n_cigar() const { return rd16(b + 12); }
  uint16_t flags() const { return rd16(b + 14); }
  uint32_t l_seq() const { return rd32(b + 16); }
  int32_t mate_ref_id() const { return rdi32(b + 20); }
  int32_t mate_pos() const { return rdi32(b + 24); }
  int32_t tlen() const { return rdi32(b + 28); }
  size_t cigar_off() const { return 32 + l_read_name(); }
  size_t seq_off() const { return cigar_off() + 4 * static_cast<size_t>(n_cigar()); }
  size_t qual_off() const { return seq_off() + (l_seq() + 1) / 2; }
  size_t aux_off() const { return qual_off() + l_seq(); }
  uint32_t cigar_op(uint32_t i) const { return rd32(b + cigar_off() + 4 * i); }
  bool cigar_in_bounds() const { return n_cigar() == 0 || cigar_off() + 4 * static_cast<size_t>(n_cigar()) <= n; }
};

inline bool consumes_query(uint32_t op) { return (0x3C1A7u >> ((op & 0xFu) << 1)) & 1u; }
inline bool consumes_ref(uint32_t op) { return (0x3C1A7u >> ((op & 0xFu) << 1)) & 2u; }

inline void cigar_ops(const View& v, std::vector<uint32_t>* ops) {
  ops->clear();
  if (!v.cigar_in_bounds()) return;
  for (uint32_t i = 0; i < v.n_cigar(); ++i) ops->push_back(v.cigar_op(i));
}

inline int32_t reference_length(const std::vector<uint32_t>& ops) {
  int32_t r = 0;
  for (uint32_t op : ops) if (consumes_ref(op & 0xF)) r += static_cast<int32_t>(op >> 4);
  return r;
}

// 4-bit packed sequence -> ASCII
inline void decode_sequence(const View& v, std::vector<uint8_t>* out) {
  static const char kTab[17] = "=ACMGRSVTWYHKDBN";
  const uint32_t l = v.l_seq();
  out->resize(l);
  const uint8_t* s = v.b + v.seq_off();
  for (uint32_t i = 0; i < l; ++i) {
    uint8_t byte = s[i >> 1];
    (*out)[i] = static_cast<uint8_t>(kTab[(i & 1) ? (byte & 0xF) : (byte >> 4)]);
  }
}

// Locates a Z-type tag; returns false when absent or not a string.
inline bool find_string_tag(const View& v, const char tag[2], const uint8_t** val, size_t* len) {
  size_t off = v.aux_off();
  if (off > v.n) return false;
  const uint8_t* a = v.b + off;
  const size_t an = v.n - off;
  auto fixed = [](uint8_t t) -> size_t {
    switch (t) {
      case 'A': case 'c': case 'C': return 1;
      case 's': case 'S': return 2;
      case 'i': case 'I': case 'f': return 4;
      default: return 0;
    }
  };
  size_t p = 0;
  while (p + 3 <= an) {
    uint8_t vt = a[p + 2];
    if (a[p] == static_cast<uint8_t>(tag[0]) && a[p + 1] == static_cast<uint8_t>(tag[1])) {
      if (vt != 'Z') return false;
      const void* z = std::memchr(a + p + 3, 0, an - (p + 3));
      if (!z) return false;
      *val = a + p + 3;
      *len = static_cast<const uint8_t*>(z) - (a + p + 3);
      return true;
    }
    size_t size = fixed(vt);
    if (!size) {
      if (vt == 'Z' || vt == 'H') {
        const void* z = std::memchr(a + p + 3, 0, an - (p + 3));
        if (!z) return false;
        size = static_cast<const uint8_t*>(z) - (a + p + 3) + 1;
      } else if (vt == 'B') {
        if (an - (p + 3) < 5) return false;
        size_t es = fixed(a[p + 3]);
        if (!es) return false;
        size = 5 + static_cast<size_t>(rd32(a + p + 4)) * es;
      } else {
        return false;
      }
    }
    p += 3 + size;
  }
  return false;
}

// One walk over the aux area for several Z tags at once: want[k] = the two tag letters, val[k] / len[k]
// receive the value of the FIRST occurrence (val[k] = nullptr when absent or not a string), exactly what
// find_string_tag would return for each tag on its own.
inline void find_string_tags(const View& v, const char (*want)[2], int n_want, const uint8_t** val, size_t* len) {
  for (int k = 0; k < n_want; ++k) { val[k] = nullptr; len[k] = 0; }
  size_t off = v.aux_off();
  if (off > v.n) return;
  const uint8_t* a = v.b + off;
  const size_t an = v.n - off;
  auto fixed = [](uint8_t t) -> size_t {
    switch (t) {
      case 'A': case 'c': case 'C': return 1;
      case 's': case 'S': return 2;
      case 'i': case 'I': case 'f': return 4;
      default: return 0;
    }
  };
  uint32_t seen = 0;                   // tags already met (found or found-with-another-type): first occurrence wins
  int left = n_want;
  size_t p = 0;
  while (p + 3 <= an && left > 0) {
    const uint8_t vt = a[p + 2];
    int hit = -1;
    for (int k = 0; k < n_want; ++k)
      if (!(seen & (1u << k)) && a[p] == static_cast<uint8_t>(want[k][0]) && a[p + 1] == static_cast<uint8_t>(want[k][1])) { hit = k; break; }
    size_t size = fixed(vt);
    if (!size) {
      if (vt == 'Z' || vt == 'H') {
        const void* z = std::memchr(a + p + 3, 0, an - (p + 3));
        if (!z) return;
        size = static_cast<const uint8_t*>(z) - (a + p + 3) + 1;
        if (hit >= 0 && vt == 'Z') { val[hit] = a + p + 3; len[hit] = size - 1; }
      } else if (vt == 'B') {
        if (an - (p + 3) < 5) return;
        const size_t es = fixed(a[p + 3]);
        if (!es) return;
        size = 5 + static_cast<size_t>(rd32(a + p + 4)) * es;
      } else {
        return;
      }
    }
    if (hit >= 0) { seen |= 1u << hit; --left; }
    p += 3 + size;
  }
}

// ---- mate-overlap clip (overlap.rs) ----
inline int32_t parse_int(const char* s, size_t a, size_t b) {
  if (a >= b) return 0;
  long long v = 0;
  for (size_t i = a; i < b; ++i) {
    if (s[i] < '0' || s[i] > '9') return 0;
    v = v * 10 + (s[i] - '0');
    if (v > 2147483647LL) return 0;   // str::parse::<i32> fails -> unwrap_or(0)
  }
  return static_cast<int32_t>(v);
}

inline int32_t mc_leading_clips(const char* c, size_t n) {
  int32_t clipped = 0;
  size_t num_start = 0;
  for (size_t i = 0; i < n; ++i) {
    if (c[i] >= '0' && c[i] <= '9') continue;
    int32_t num = parse_int(c, num_start, i);
    if (c[i] == 'S' || c[i] == 'H') { clipped += num; num_start = i + 1; }
    else break;
  }
  return clipped;
}

inline void mc_ref_len_and_trailing(const char* c, size_t n, int32_t* ref_len, int32_t* trailing) {
  *ref_len = 0; *trailing = 0;
  size_t num_start = 0;
  bool saw = false;
  for (size_t i = 0; i < n; ++i) {
    if (c[i] >= '0' && c[i] <= '9') continue;
    int32_t num = parse_int(c, num_start, i);
    num_start = i + 1;
    switch (c[i]) {
      case 'M': case 'D': case 'N': case '=': case 'X': *ref_len += num; *trailing = 0; saw = true; break;
      case 'S': case 'H': if (saw) *trailing += num; break;
      default: break;
    }
  }
}

// std::str::from_utf8 acceptance test (well-formed UTF-8, no surrogates / overlongs)
inline bool valid_utf8(const uint8_t* s, size_t n) {
  size_t i = 0;
  while (i < n) {
    uint8_t c = s[i];
    if (c < 0x80) { ++i; continue; }
    size_t need; uint32_t cp, lo;
    if ((c & 0xE0) == 0xC0) { need = 1; cp = c & 0x1F; lo = 0x80; }
    else if ((c & 0xF0) == 0xE0) { need = 2; cp = c & 0x0F; lo = 0x800; }
    else if ((c & 0xF8) == 0xF0) { need = 3; cp = c & 0x07; lo = 0x10000; }
    else return false;
    for (size_t k = 1; k <= need; ++k) {
      if (i + k >= n) return false;
      uint8_t d = s[i + k];
      if ((d & 0xC0) != 0x80) return false;
      cp = (cp << 6) | (d & 0x3F);
    }
    if (cp < lo || cp > 0x10FFFF || (cp >= 0xD800 && cp <= 0xDFFF)) return false;
    i += need + 1;
  }
  return true;
}

inline bool is_fr_pair(const View& v, const std::vector<uint32_t>& ops) {
  const uint16_t f = v.flags();
  if (!(f & kPaired)) return false;
  if ((f & kUnmapped) || (f & kMateUnmapped)) return false;
  if (v.ref_id() != v.mate_ref_id()) return false;
  const bool rev = f & kReverse, mrev = f & kMateReverse;
  if (rev == mrev) return false;
  const int32_t start = v.pos() + 1, mstart = v.mate_pos() + 1;
  int32_t pos5, neg5;
  if (rev) {
    int32_t rl = reference_length(ops);
    int32_t end = start + (rl - 1 > 0 ? rl - 1 : 0);
    pos5 = mstart; neg5 = end;
  } else {
    pos5 = start; neg5 = start + v.tlen();
  }
  return pos5 < neg5;
}

inline size_t read_pos_at_ref(const std::vector<uint32_t>& ops, int32_t start1, int32_t target,
                              bool at_or_past) {
  int32_t ref_pos = start1;
  size_t read_pos = 0;
  for (uint32_t op : ops) {
    uint32_t t = op & 0xF, ln = op >> 4;
    if (t == 0 || t == 7 || t == 8) {
      for (uint32_t k = 0; k < ln; ++k) {
        ++read_pos;
        if (ref_pos == target) return at_or_past ? read_pos : (read_pos ? read_pos - 1 : 0);
        ++ref_pos;
      }
    } else if (t == 1 || t == 4) {
      read_pos += ln;
    } else if (t == 2 || t == 3) {
      for (uint32_t k = 0; k < ln; ++k) {
        if (ref_pos == target) return 0;
        ++ref_pos;
      }
    }
  }
  return 0;
}

// num_bases_extending_past_mate_raw (overlap.rs:65-136) with the MC value already located
// (mc == nullptr: the record has no MC string tag).
inline size_t num_bases_extending_past_mate_mc(const View& v, const std::vector<uint32_t>& ops, const uint8_t* mc, size_t mcn);

inline size_t num_bases_extending_past_mate(const View& v, const std::vector<uint32_t>& ops) {
  if (!is_fr_pair(v, ops)) return 0;
  const uint8_t* mc; size_t mcn;
  if (!find_string_tag(v, "MC", &mc, &mcn)) return 0;
  return num_bases_extending_past_mate_mc(v, ops, mc, mcn);
}

inline size_t num_bases_extending_past_mate_mc(const View& v, const std::vector<uint32_t>& ops, const uint8_t* mc, size_t mcn) {
  if (!mc || !is_fr_pair(v, ops)) return 0;
  const char* mcs = reinterpret_cast<const char*>(mc);
  if (!valid_utf8(mc, mcn)) return 0;                            // std::str::from_utf8 fails
  const int32_t this_pos = v.pos() + 1, m_pos = v.mate_pos() + 1;
  size_t read_length = 0;
  for (uint32_t op : ops) if (consumes_query(op & 0xF)) read_length += op >> 4;
  if (v.flags() & kReverse) {
    int32_t mate_us = m_pos - mc_leading_clips(mcs, mcn);
    if (this_pos <= mate_us) return read_pos_at_ref(ops, this_pos, mate_us, false);
    size_t lead = 0;
    for (uint32_t op : ops) { uint32_t t = op & 0xF; if (t == 4) lead += op >> 4; else if (t != 5) break; }
    size_t gap = static_cast<size_t>(static_cast<uint32_t>(this_pos - mate_us));
    return lead > gap ? lead - gap : 0;
  }
  int32_t rl = reference_length(ops);
  int32_t aln_end = this_pos + rl - 1;
  int32_t mrl, mtc;
  mc_ref_len_and_trailing(mcs, mcn, &mrl, &mtc);
  int32_t mate_ue = m_pos + mrl + mtc - 1;
  if (aln_end >= mate_ue) {
    size_t past = read_pos_at_ref(ops, this_pos, mate_ue, true);
    return read_length > past ? read_length - past : 0;
  }
  size_t trail = 0;
  for (size_t i = ops.size(); i-- > 0;) { uint32_t t = ops[i] & 0xF; if (t == 4) trail += ops[i] >> 4; else if (t != 5) break; }
  size_t gap = static_cast<size_t>(static_cast<uint32_t>(mate_ue - aln_end));
  return trail > gap ? trail - gap : 0;
}


// ---- virtual CIGAR clipping (cigar.rs:337-841) and ref->query mapping (cigar.rs:412-457) ----
inline uint32_t enc_op(uint32_t type, size_t len) { return (static_cast<uint32_t>(len) << 4) | type; }
inline bool consumes_read(uint32_t t) { return t == 0 || t == 1 || t == 7 || t == 8; }

// Existing leading (from_start) or trailing H then S clips; returns how many ops they span.
inline size_t existing_clips(const std::vector<uint32_t>& ops, bool from_start, size_t* hard, size_t* soft) {
  *hard = 0; *soft = 0;
  size_t skip = 0;
  const size_t n = ops.size();
  auto at = [&](size_t k) { return from_start ? ops[k] : ops[n - 1 - k]; };
  while (skip < n && (at(skip) & 0xF) == 5) { *hard += at(skip) >> 4; ++skip; }
  while (skip < n && (at(skip) & 0xF) == 4) { *soft += at(skip) >> 4; ++skip; }
  return skip;
}

// clip_cigar_ops_raw: returns the clipped ops; *ref_consumed = reference bases removed at the start.
inline std::vector<uint32_t> clip_cigar_ops(const std::vector<uint32_t>& ops, size_t clip_amount,
                                            bool from_start, size_t* ref_consumed) {
  *ref_consumed = 0;
  if (clip_amount == 0 || ops.empty()) return ops;
  const size_t n = ops.size();
  size_t existing = 0;
  for (size_t k = 0; k < n; ++k) {
    uint32_t op = from_start ? ops[k] : ops[n - 1 - k];
    if ((op & 0xF) == 4 || (op & 0xF) == 5) existing += op >> 4; else break;
  }
  size_t hard, soft;
  const size_t skip = existing_clips(ops, from_start, &hard, &soft);
  std::vector<uint32_t> res;
  if (clip_amount <= existing) {   // upgrade_clipping_raw: soft clips become hard, alignment unchanged
    size_t up = std::min(soft, clip_amount > hard ? clip_amount - hard : 0);
    if (from_start) {
      res.push_back(enc_op(5, hard + up));
      if (soft - up > 0) res.push_back(enc_op(4, soft - up));
      res.insert(res.end(), ops.begin() + skip, ops.end());
    } else {
      res.assign(ops.begin(), ops.end() - skip);
      if (soft - up > 0) res.push_back(enc_op(4, soft - up));
      res.push_back(enc_op(5, hard + up));
    }
    return res;
  }
  const size_t want = clip_amount - existing;
  size_t read_clipped = 0, ref_clipped = 0;
  std::vector<uint32_t> new_ops;
  if (from_start) {   // clip_cigar_start_raw
    size_t idx = skip;
    while (idx < n) {
      uint32_t op = ops[idx], t = op & 0xF; size_t ln = op >> 4;
      if (read_clipped == want && new_ops.empty() && t == 2) { ref_clipped += ln; ++idx; continue; }
      if (read_clipped >= want) break;
      bool is_read = consumes_read(t), is_ref = consumes_ref(t);
      if (is_read && ln > want - read_clipped) {
        if (t == 1) read_clipped += ln;
        else {
          size_t rem = want - read_clipped;
          read_clipped += rem;
          if (is_ref) ref_clipped += rem;
          new_ops.push_back(enc_op(t, ln - rem));
        }
      } else {
        if (is_read) read_clipped += ln;
        if (is_ref) ref_clipped += ln;
      }
      ++idx;
    }
    res.push_back(enc_op(5, hard + soft + read_clipped));
    res.insert(res.end(), new_ops.begin(), new_ops.end());
    res.insert(res.end(), ops.begin() + idx, ops.end());
    *ref_consumed = ref_clipped;
    return res;
  }
  // clip_cigar_end_raw
  size_t idx = n - skip;
  while (idx > 0) {
    uint32_t op = ops[idx - 1], t = op & 0xF; size_t ln = op >> 4;
    if (read_clipped == want && new_ops.empty() && t == 2) { --idx; continue; }
    if (read_clipped >= want) break;
    bool is_read = consumes_read(t);
    if (is_read && ln > want - read_clipped) {
      if (t == 1) read_clipped += ln;
      else {
        size_t rem = want - read_clipped;
        read_clipped += rem;
        new_ops.push_back(enc_op(t, ln - rem));
      }
    } else if (is_read) {
      read_clipped += ln;
    }
    --idx;
  }
  res.assign(ops.begin(), ops.begin() + idx);
  res.insert(res.end(), new_ops.rbegin(), new_ops.rend());
  res.push_back(enc_op(5, hard + soft + read_clipped));
  return res;
}

// read_pos_at_ref_pos_raw: 1-based query position at a 1-based reference position; false = None.
inline bool read_pos_at_ref_pos(const std::vector<uint32_t>& ops, size_t alignment_start, size_t ref_pos,
                                bool last_base_if_deleted, size_t* out) {
  if (ref_pos < alignment_start) return false;
  size_t ref_off = 0, q_off = 0;
  for (uint32_t op : ops) {
    uint32_t t = op & 0xF; size_t ln = op >> 4;
    size_t op_ref_start = alignment_start + ref_off;
    if (consumes_ref(t)) {
      size_t op_ref_end = op_ref_start + ln - 1;
      if (ref_pos >= op_ref_start && ref_pos <= op_ref_end && ln > 0) {
        if (consumes_query(t)) { *out = q_off + (ref_pos - op_ref_start) + 1; return true; }
        if (last_base_if_deleted) { *out = q_off > 0 ? q_off : 1; return true; }
        return false;
      }
      ref_off += ln;
    }
    if (consumes_query(t)) q_off += ln;
  }
  return false;
}

// ---- simplified CIGAR ----
using SimpleCigar = std::vector<std::pair<uint8_t, uint32_t>>;   // (kind 0..8, length)

inline void simplify_cigar(const std::vector<uint32_t>& ops, SimpleCigar* out) {
  out->clear();
  for (uint32_t raw : ops) {
    uint32_t t = raw & 0xF, ln = raw >> 4;
    if (t > 8) continue;
    uint8_t kind = (t == 4 || t == 7 || t == 8 || t == 5) ? 0 : static_cast<uint8_t>(t);
    if (!out->empty() && out->back().first == kind) out->back().second += ln;
    else out->emplace_back(kind, ln);
  }
}

inline void truncate_cigar(SimpleCigar* c, size_t query_len) {   // vanilla_caller.rs:816-851
  size_t remaining = query_len, w = 0;                           // in place: elements only shrink
  for (size_t i = 0; i < c->size(); ++i) {
    if (remaining == 0) break;
    auto e = (*c)[i];
    const bool q = e.first == 0 || e.first == 1 || e.first == 4 || e.first == 7 || e.first == 8;
    if (q) {
      const uint32_t take = e.second < remaining ? e.second : static_cast<uint32_t>(remaining);
      (*c)[w++] = {e.first, take};
      remaining -= take;
    } else {
      (*c)[w++] = e;
    }
  }
  c->resize(w);
}

inline bool is_cigar_prefix(const SimpleCigar& a, const SimpleCigar& b) {
  if (a.size() > b.size()) return false;
  size_t last = a.empty() ? 0 : a.size() - 1;
  for (size_t i = 0; i < a.size(); ++i) {
    if (a[i].first != b[i].first) return false;
    if (i == last) { if (a[i].second > b[i].second) return false; }
    else if (a[i].second != b[i].second) return false;
  }
  return true;
}

inline int cmp_cigar(const SimpleCigar& a, const SimpleCigar& b) {   // vanilla_caller.rs:77-105
  size_t n = a.size() < b.size() ? a.size() : b.size();
  for (size_t i = 0; i < n; ++i) {
    if (a[i].second != b[i].second) return a[i].second < b[i].second ? -1 : 1;
    if (a[i].first != b[i].first) return a[i].first < b[i].first ? -1 : 1;
  }
  return a.size() < b.size() ? -1 : (a.size() > b.size() ? 1 : 0);
}

inline uint8_t complement(uint8_t b) {
  switch (b) {
    case 'A': case 'a': return 'T';
    case 'T': case 't': return 'A';
    case 'C': case 'c': return 'G';
    case 'G': case 'g': return 'C';
    default: return b;
  }
}

// ---- record writer (UnmappedSamBuilder + tag encoders) ----
struct Writer {
  std::vector<uint8_t>* out;
  size_t start = 0;   // offset of the block_size word of the record being built
  explicit Writer(std::vector<uint8_t>* o) : out(o) {}
  void put(const void* p, size_t n) { const uint8_t* s = static_cast<const uint8_t*>(p); out->insert(out->end(), s, s + n); }
  template <class T> void le(T v) { put(&v, sizeof(T)); }
  static uint8_t code(uint8_t b) {
    switch (b) {
      case '=': return 0; case 'A': case 'a': return 1; case 'C': case 'c': return 2;
      case 'M': case 'm': return 3; case 'G': case 'g': return 4; case 'R': case 'r': return 5;
      case 'S': case 's': return 6; case 'V': case 'v': return 7; case 'T': case 't': return 8;
      case 'W': case 'w': return 9; case 'Y': case 'y': return 10; case 'H': case 'h': return 11;
      case 'K': case 'k': return 12; case 'D': case 'd': return 13; case 'B': case 'b': return 14;
      default: return 15;
    }
  }
  struct CodeTable { uint8_t t[256]; CodeTable() { for (int b = 0; b < 256; ++b) t[b] = code(static_cast<uint8_t>(b)); } };
  void begin(const std::string& name, uint16_t flag, const uint8_t* bases, const uint8_t* quals, uint32_t l) {
    start = out->size();
    le<uint32_t>(0);                       // block_size, patched in end()
    le<int32_t>(-1); le<int32_t>(-1);
    out->push_back(static_cast<uint8_t>(name.size() + 1));
    out->push_back(0);
    le<uint16_t>(4680); le<uint16_t>(0); le<uint16_t>(flag); le<uint32_t>(l);
    le<int32_t>(-1); le<int32_t>(-1); le<int32_t>(0);
    put(name.data(), name.size());
    out->push_back(0);
    // packed sequence + qualities: sized once, written in place
    static const CodeTable kCodes;
    const size_t o = out->size(), nb = (static_cast<size_t>(l) + 1) / 2;
    out->resize(o + nb + l);
    uint8_t* p = out->data() + o;
    for (uint32_t i = 0; i + 1 < l; i += 2) p[i >> 1] = static_cast<uint8_t>((kCodes.t[bases[i]] << 4) | kCodes.t[bases[i + 1]]);
    if (l & 1) p[l >> 1] = static_cast<uint8_t>(kCodes.t[bases[l - 1]] << 4);
    if (l) std::memcpy(p + nb, quals, l);
  }
  void tag(const char t[2], char type) { out->push_back(t[0]); out->push_back(t[1]); out->push_back(type); }
  void str(const char t[2], const void* v, size_t n) { tag(t, 'Z'); put(v, n); out->push_back(0); }
  void integer(const char t[2], int32_t v) {
    if (v >= -128 && v <= 127) { tag(t, 'c'); out->push_back(static_cast<uint8_t>(static_cast<int8_t>(v))); }
    else if (v >= 0 && v <= 255) { tag(t, 'C'); out->push_back(static_cast<uint8_t>(v)); }
    else if (v >= 0 && v <= 65535) { tag(t, 'S'); le<uint16_t>(static_cast<uint16_t>(v)); }
    else if (v >= -32768 && v <= 32767) { tag(t, 's'); le<int16_t>(static_cast<int16_t>(v)); }
    else { tag(t, 'i'); le<int32_t>(v); }
  }
  void real(const char t[2], float v) { tag(t, 'f'); le<float>(v); }
  uint8_t* grow(size_t n) { const size_t o = out->size(); out->resize(o + n); return out->data() + o; }
  void i16_array(const char t[2], const uint16_t* v, uint32_t n) {   // values clamp to i16::MAX
    tag(t, 'B'); out->push_back('s'); le<uint32_t>(n);
    uint8_t* p = grow(2 * static_cast<size_t>(n));
    for (uint32_t i = 0; i < n; ++i) { const uint16_t x = v[i] > 32767 ? 32767 : v[i]; std::memcpy(p + 2 * i, &x, 2); }
  }
  void i16_array_wrap(const char t[2], const uint16_t* v, uint32_t n) {   // `as i16` (wrapping): same bits
    tag(t, 'B'); out->push_back('s'); le<uint32_t>(n);
    uint8_t* p = grow(2 * static_cast<size_t>(n));
    if (n) std::memcpy(p, v, 2 * static_cast<size_t>(n));
  }
  void phred33(const char t[2], const uint8_t* q, uint32_t n) {
    tag(t, 'Z');
    uint8_t* p = grow(static_cast<size_t>(n) + 1);
    for (uint32_t i = 0; i < n; ++i) p[i] = static_cast<uint8_t>(q[i] > 222 ? 255 : q[i] + 33);
    p[n] = 0;
  }
  void end() {
    uint32_t bs = static_cast<uint32_t>(out->size() - start - 4);
    std::memcpy(out->data() + start, &bs, 4);
  }
};

}  // namespace bam
}  // namespace fgb
