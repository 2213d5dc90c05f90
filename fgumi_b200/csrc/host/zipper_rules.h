// `fgumi zipper`'s per-record rules (src/lib/commands/zipper.rs merge_raw :373-521, Template::fix_mate_info in
// src/lib/template.rs:411-710, the tag editors of crates/fgumi-raw-bam/src/tags.rs) in closed form, compiled for the
// host (fgb_host_zipper_records, zipper_host.cpp) and the device (../zipper_kernels.cuh).
//
// merge_raw edits a mapped record by a sequence of remove_tag / update_*_tag / append calls.  With unique tag names in
// both records (the driver checks that) every append is preceded by the removal of its name, so the edited aux area is:
// the original entries that no step removes, in their original order (MQ / MC edited in place where update_int_tag /
// update_string_tag keep the entry's place), then each name whose last edit was an append, in the order of those
// appends: MQ, MC, ms (the mate fix), the unmapped read's entries in its order, AS, XS, tc.  An appended entry that a
// later step removes is dropped.  tests/zipper_oracle.py replays the calls literally and the tests compare the two.
//
// Every function takes (lane, nl): the device runs it with a warp's 32 lanes, the host with lane 0 of 1.  Control flow
// depends only on the record, so the lanes of a warp stay converged; byte ranges are copied lane-strided.
#pragma once
#include <stdint.h>

#include "record_filter.h"

namespace fgb {
namespace zip {

using rfilter::ld16;
using rfilter::ld32;

constexpr uint32_t kNone = 0xffffffffu;
enum : uint8_t { kMerged = 0, kPass = 1 };                      // a mapped record of a merged template / an unmapped one
enum : uint8_t { kRoleNone = 0, kRolePrim = 1, kRoleSupp = 2 };  // which fix_mate_info arm edits the record

// One output record, built by the host (run-local record indices; kNone = absent)
struct ZRec {
  uint32_t src;            // the mapped record (kMerged) or the unmapped record (kPass)
  uint32_t mate;           // kRolePrim: the other primary; kRoleSupp: the opposite segment's primary
  uint32_t partner;        // the mate's partner: the primary of the record's own segment
  uint32_t umap;           // the unmapped primary of the record's segment (R1 for an unpaired read)
  uint32_t r1, r2;         // the mapped template's primary R1 / R2, for the tc tag
  uint8_t kind, role, mate_is_r1, pad;
};

// The tag lists: n two-byte names each
struct Sets {
  const uint8_t* remove;
  const uint8_t* reverse;
  const uint8_t* revcomp;
  uint32_t n_remove, n_reverse, n_revcomp;
};

FGB_HD bool in_set(const uint8_t* s, uint32_t n, uint8_t a, uint8_t b) {
  for (uint32_t i = 0; i < n; ++i)
    if (s[2 * i] == a && s[2 * i + 1] == b) return true;
  return false;
}
FGB_HD int32_t ldi32(const uint8_t* p) { return static_cast<int32_t>(ld32(p)); }

struct Rec {   // the fixed fields of a record
  const uint8_t* r;
  uint32_t len, co, ao, nc;
  FGB_HD Rec() : r(nullptr), len(0), co(0), ao(0), nc(0) {}
  FGB_HD Rec(const uint8_t* p, uint32_t n) : r(p), len(n) {
    nc = ld16(p + 12);
    const uint32_t L = ld32(p + 16);
    co = 32u + p[8];
    ao = co + 4u * nc + (L + 1) / 2 + L;
  }
  FGB_HD uint16_t flags() const { return ld16(r + 14); }
  FGB_HD int32_t ref() const { return ldi32(r); }
  FGB_HD int32_t pos() const { return ldi32(r + 4); }
  FGB_HD int32_t tlen() const { return ldi32(r + 28); }
  FGB_HD uint8_t mapq() const { return r[9]; }
  FGB_HD uint32_t op(uint32_t k) const { return ld32(r + co + 4u * k); }
};

// The entry named (a, b) in the aux area of `x`: *s / *e its bounds (record offsets); false when absent
FGB_HD bool find(const Rec& x, uint8_t a, uint8_t b, uint32_t* s, uint32_t* e) {
  uint32_t p = x.ao;
  while (p + 3 <= x.len) {
    uint8_t sub;
    uint32_t cnt;
    const uint32_t sz = static_cast<uint32_t>(rfilter::value_size(x.r + x.ao, x.len - x.ao, p - x.ao, &sub, &cnt));
    if (x.r[p] == a && x.r[p + 1] == b) { *s = p; *e = p + 3 + sz; return true; }
    p += 3 + sz;
  }
  return false;
}
FGB_HD uint32_t entry_end(const Rec& x, uint32_t p) {
  uint8_t sub;
  uint32_t cnt;
  return p + 3 + static_cast<uint32_t>(rfilter::value_size(x.r + x.ao, x.len - x.ao, p - x.ao, &sub, &cnt));
}

// find_int_tag (tags.rs:118-151) of the entry at s: an integer of type c C s S i I; false for any other type
FGB_HD bool int_value(const uint8_t* r, uint32_t s, int64_t* v) {
  const uint8_t* d = r + s + 3;
  switch (r[s + 2]) {
    case 'c': *v = static_cast<int8_t>(d[0]); return true;
    case 'C': *v = d[0]; return true;
    case 's': *v = static_cast<int16_t>(ld16(d)); return true;
    case 'S': *v = ld16(d); return true;
    case 'i': *v = ldi32(d); return true;
    case 'I': *v = ld32(d); return true;
    default: return false;
  }
}
// an AS-like tag whose value normalize_int_tag_to_smallest_signed (tags.rs:910-929) rewrites: an integer fitting i32
FGB_HD bool int_i32(const uint8_t* r, uint32_t s, int32_t* v) {
  int64_t w;
  if (!int_value(r, s, &w) || w < INT32_MIN || w > INT32_MAX) return false;
  *v = static_cast<int32_t>(w);
  return true;
}
// append_int_tag (tags.rs:533-553) and append_signed_int_tag (:937-951): the type byte and value size
FGB_HD uint32_t uint_pref_size(int32_t v, uint8_t* t) {
  if (v >= -128 && v <= 127) { *t = 'c'; return 1; }
  if (v >= 0 && v <= 255) { *t = 'C'; return 1; }
  if (v >= 0 && v <= 65535) { *t = 'S'; return 2; }
  if (v >= -32768 && v <= 32767) { *t = 's'; return 2; }
  *t = 'i';
  return 4;
}
FGB_HD uint32_t signed_size(int32_t v, uint8_t* t) {
  if (v >= -128 && v <= 127) { *t = 'c'; return 1; }
  if (v >= -32768 && v <= 32767) { *t = 's'; return 2; }
  *t = 'i';
  return 4;
}

// i32 arithmetic as the reference's release build does it: wrapping
FGB_HD int32_t wadd(int32_t a, int32_t b) { return static_cast<int32_t>(static_cast<uint32_t>(a) + static_cast<uint32_t>(b)); }
FGB_HD int32_t wneg(int32_t a) { return static_cast<int32_t>(0u - static_cast<uint32_t>(a)); }

FGB_HD uint32_t ndigits(uint32_t v) {
  uint32_t d = 1;
  while (v >= 10) { v /= 10; ++d; }
  return d;
}

// reference_length_from_raw_bam: M / D / N / = / X
FGB_HD int32_t ref_len(const Rec& x) {
  uint32_t n = 0;
  for (uint32_t k = 0; k < x.nc; ++k) {
    const uint32_t o = x.op(k), t = o & 0xF;
    if (t == 0 || t == 2 || t == 3 || t == 7 || t == 8) n += o >> 4;
  }
  return static_cast<int32_t>(n);
}

// compute_insert_size_raw (template.rs:714-746)
FGB_HD int32_t insert_size(const Rec& a, const Rec& b) {
  if ((a.flags() & 4) || (b.flags() & 4) || a.ref() != b.ref()) return 0;
  const int32_t p1 = wadd(a.pos(), 1), p2 = wadd(b.pos(), 1);
  const int32_t f1 = (a.flags() & 0x10) ? wadd(wadd(p1, ref_len(a)), -1) : p1;
  const int32_t f2 = (b.flags() & 0x10) ? wadd(wadd(p2, ref_len(b)), -1) : p2;
  return wadd(wadd(f2, wneg(f1)), f2 >= f1 ? 1 : -1);
}

// unclipped_5prime_from_raw_bam (cigar.rs:201-228): 1-based; 0 unmapped, i32::MAX without a CIGAR
FGB_HD int32_t unclipped_5prime(const Rec& x) {
  const uint16_t f = x.flags();
  if (f & 4) return 0;
  if (x.nc == 0) return INT32_MAX;
  const int32_t pos = wadd(x.pos(), 1);
  if (!(f & 0x10)) {
    uint32_t clipped = 0;
    for (uint32_t k = 0; k < x.nc; ++k) {
      const uint32_t o = x.op(k);
      if ((o & 0xF) == 4 || (o & 0xF) == 5) clipped += o >> 4;
      else break;
    }
    return wadd(pos, wneg(static_cast<int32_t>(clipped)));
  }
  uint32_t rl = 0, trailing = 0;
  bool saw = false;
  for (uint32_t k = 0; k < x.nc; ++k) {
    const uint32_t o = x.op(k), t = o & 0xF;
    if (t == 0 || t == 2 || t == 3 || t == 7 || t == 8) { rl += o >> 4; trailing = 0; saw = true; }
    else if ((t == 4 || t == 5) && saw) trailing += o >> 4;
  }
  return wadd(pos, static_cast<int32_t>(rl + trailing - 1u));
}

// A primary read's ref, pos and TLEN after the pair arm of fix_mate_info (template.rs:421-456), `partner` being the
// other primary (partner.r == nullptr: absent, untouched); x_is_r1 orders compute_insert_size_raw's arguments
struct Fixed {
  int32_t ref, pos, tlen;
};
FGB_HD Fixed fixed_primary(const Rec& x, const Rec& partner, bool x_is_r1) {
  Fixed f{x.ref(), x.pos(), x.tlen()};
  if (!partner.r) return f;
  const bool xu = x.flags() & 4, pu = partner.flags() & 4;
  if (!xu && !pu) f.tlen = x_is_r1 ? insert_size(x, partner) : wneg(insert_size(partner, x));
  else f.tlen = 0;
  if (xu && pu) { f.ref = -1; f.pos = -1; }
  else if (xu) { f.ref = partner.ref(); f.pos = partner.pos(); }
  return f;
}

// The mate's CIGAR as text (cigar_to_string_from_raw, cigar.rs:115-129): its length, the ops' digit counts summed
// across the lanes
template <class Sum>
FGB_HD uint32_t cigar_text_len(const Rec& m, int lane, int nl, Sum&& sum) {
  uint32_t n = 0;
  for (uint32_t k = lane; k < m.nc; k += nl) n += ndigits(m.op(k) >> 4) + 1;
  return sum(n);
}

// Everything the aux layout of one merged record depends on
struct Plan {
  Rec x, u;                    // the mapped record and the unmapped primary of its segment (u.r == nullptr: none)
  uint8_t mq_mode, mc_mode;    // 0 untouched, 1 update_*_tag, 2 remove_tag
  bool mq_inplace, ms_set, has_pg, as_norm, xs_norm, tc, rev;
  int32_t mq_val, ms_val, as_val, xs_val;
  int32_t tc_ref1, tc_pos1, tc_neg1, tc_ref2, tc_pos2, tc_neg2;
  uint32_t mq_s, mq_e, mc_s, mc_e;   // the original MQ / MC entries (s == e: absent)
  uint32_t mc_len;             // the MC text's length
  Rec mate;                    // the mate whose CIGAR MC takes
  // the record's fixed fields after the edits
  int32_t ref, pos, mref, mpos, tlen;
  uint16_t flags;
};

// copied(N): the unmapped read's entry N goes to this record (merge_raw :434-445)
FGB_HD bool copied(const Plan& p, const Sets& s, uint8_t a, uint8_t b) {
  if (!p.u.r) return false;
  if (a == 'P' && b == 'G' && p.has_pg) return false;
  if (in_set(s.remove, s.n_remove, a, b)) return false;
  uint32_t us, ue;
  return find(p.u, a, b, &us, &ue);
}

// Pass 1's plan of output record z.  um / mp: the unmapped and mapped records of the run; uoff / moff: their offsets
// (relative to the buffers' starts).
template <class Sum>
FGB_HD Plan plan(const ZRec& z, const uint8_t* um, const uint64_t* uoff, const uint8_t* mp, const uint64_t* moff,
                 const Sets& s, bool skip_tc, int lane, int nl, Sum&& sum) {
  auto mrec = [&](uint32_t i) { return Rec(mp + moff[i], static_cast<uint32_t>(moff[i + 1] - moff[i])); };
  Plan p{};
  p.x = mrec(z.src);
  p.u = z.umap == kNone ? Rec() : Rec(um + uoff[z.umap], static_cast<uint32_t>(uoff[z.umap + 1] - uoff[z.umap]));
  const Rec& x = p.x;
  const uint16_t f0 = x.flags();
  p.flags = f0;
  p.ref = x.ref(); p.pos = x.pos(); p.mref = ldi32(x.r + 20); p.mpos = ldi32(x.r + 24); p.tlen = x.tlen();
  p.rev = f0 & 0x10;
  if (z.role != kRoleNone) {
    // set_mate_info_* (template.rs:549-693) and the supplementary arms (:458-544)
    const Rec m = mrec(z.mate);
    const Rec part = z.partner == kNone ? Rec() : mrec(z.partner);
    const Fixed mf = fixed_primary(m, part, z.mate_is_r1);
    const uint16_t mfl = m.flags();
    const bool mu = mfl & 4;
    p.mref = mf.ref; p.mpos = mf.pos;
    p.flags = static_cast<uint16_t>((p.flags & ~0x28) | ((mfl & 0x10) ? 0x20 : 0) | (mu ? 0x08 : 0));
    p.mq_val = m.mapq();
    if (z.role == kRolePrim) {
      const Fixed xf = fixed_primary(x, m, !z.mate_is_r1);
      p.ref = xf.ref; p.pos = xf.pos; p.tlen = xf.tlen;
      p.mq_mode = mu ? 2 : 1;
      p.mc_mode = mu ? 2 : (m.nc ? 1 : 2);
    } else {
      p.tlen = wneg(mf.tlen);
      p.mq_mode = 1;
      p.mc_mode = (m.nc && !mu) ? 1 : 2;
    }
    p.mate = m;
    if (p.mc_mode == 1) p.mc_len = cigar_text_len(m, lane, nl, sum);
    uint32_t as, ae;
    if (find(m, 'A', 'S', &as, &ae) && int_i32(m.r, as, &p.ms_val)) p.ms_set = true;
  }
  if (p.u.r) p.flags = static_cast<uint16_t>((p.flags & ~0x200) | (p.u.flags() & 0x200));   // merge_raw :495-506
  find(x, 'M', 'Q', &p.mq_s, &p.mq_e);
  find(x, 'M', 'C', &p.mc_s, &p.mc_e);
  p.mq_inplace = p.mq_mode == 1 && p.mq_e - p.mq_s == 7 && (x.r[p.mq_s + 2] == 'i' || x.r[p.mq_s + 2] == 'I');
  uint32_t t0, t1;
  p.has_pg = find(x, 'P', 'G', &t0, &t1) && !in_set(s.remove, s.n_remove, 'P', 'G');
  // AS / XS as step 5 finds them: the unmapped read's copy, else the mapped record's own unless removed
  for (int k = 0; k < 2; ++k) {
    const uint8_t b = k ? 'X' : 'A';
    bool norm = false;
    int32_t v = 0;
    uint32_t es, ee;
    if (copied(p, s, b, 'S')) { find(p.u, b, 'S', &es, &ee); norm = int_i32(p.u.r, es, &v); }
    else if (!in_set(s.remove, s.n_remove, b, 'S') && find(x, b, 'S', &es, &ee)) norm = int_i32(x.r, es, &v);
    if (k) { p.xs_norm = norm; p.xs_val = v; } else { p.as_norm = norm; p.as_val = v; }
  }
  // add_template_coordinate_tags_raw (zipper.rs:259-332)
  if (!skip_tc && (f0 & 0x900)) {
    const Rec q1 = z.r1 == kNone ? Rec() : mrec(z.r1), q2 = z.r2 == kNone ? Rec() : mrec(z.r2);
    const bool h1 = q1.r && !(q1.flags() & 4), h2 = q2.r && !(q2.flags() & 4);
    if (h1 || h2) {
      p.tc = true;
      const int32_t t1 = h1 ? q1.ref() : 0, p1 = h1 ? unclipped_5prime(q1) : 0, n1 = h1 ? (q1.flags() & 0x10) != 0 : 0;
      const int32_t t2 = h2 ? q2.ref() : 0, p2 = h2 ? unclipped_5prime(q2) : 0, n2 = h2 ? (q2.flags() & 0x10) != 0 : 0;
      // the earlier by (ref, pos) first; a single mapped primary fills both halves
      const bool first1 = h1 && (!h2 || t1 < t2 || (t1 == t2 && p1 <= p2));
      const bool second1 = h1 && !(h2 && first1);
      p.tc_ref1 = first1 ? t1 : t2; p.tc_pos1 = first1 ? p1 : p2; p.tc_neg1 = first1 ? n1 : n2;
      p.tc_ref2 = second1 ? t1 : t2; p.tc_pos2 = second1 ? p1 : p2; p.tc_neg2 = second1 ? n1 : n2;
    }
  }
  return p;
}

// Does the original entry (a, b) of the mapped record survive every step?
FGB_HD bool survives(const Plan& p, const Sets& s, uint8_t a, uint8_t b) {
  if (a == 'M' && b == 'Q' && (p.mq_mode == 2 || (p.mq_mode == 1 && !p.mq_inplace))) return false;
  if (a == 'M' && b == 'C' && p.mc_mode == 2) return false;
  if (a == 'm' && b == 's' && p.ms_set) return false;
  if (in_set(s.remove, s.n_remove, a, b) || copied(p, s, a, b)) return false;
  if (a == 'A' && b == 'S' && p.as_norm) return false;
  if (a == 'X' && b == 'S' && p.xs_norm) return false;
  if (a == 't' && b == 'c' && p.tc) return false;
  return true;
}
// Is the unmapped read's entry (a, b) in the output?
FGB_HD bool u_kept(const Plan& p, const Sets& s, uint8_t a, uint8_t b) {
  if (!copied(p, s, a, b)) return false;
  if (a == 'A' && b == 'S' && p.as_norm) return false;
  if (a == 'X' && b == 'S' && p.xs_norm) return false;
  if (a == 't' && b == 'c' && p.tc) return false;
  return true;
}
FGB_HD bool mq_appended(const Plan& p, const Sets& s) {
  return p.mq_mode == 1 && !p.mq_inplace && !in_set(s.remove, s.n_remove, 'M', 'Q') && !copied(p, s, 'M', 'Q');
}
FGB_HD bool mc_appended(const Plan& p, const Sets& s) {
  return p.mc_mode == 1 && p.mc_s == p.mc_e && !in_set(s.remove, s.n_remove, 'M', 'C') && !copied(p, s, 'M', 'C');
}
FGB_HD bool ms_appended(const Plan& p, const Sets& s) {
  return p.ms_set && !in_set(s.remove, s.n_remove, 'm', 's') && !copied(p, s, 'm', 's');
}
// The size of the original MC entry after update_string_tag: in place at the same value length, else spliced as Z
FGB_HD uint32_t mc_entry_size(const Plan& p) {
  return p.mc_e - p.mc_s - 4 == p.mc_len ? p.mc_e - p.mc_s : 4 + p.mc_len;
}

// The edited record's size (no block_size word)
FGB_HD uint32_t out_size(const Plan& p, const Sets& s) {
  const Rec& x = p.x;
  uint32_t n = x.ao;
  for (uint32_t q = x.ao; q < x.len;) {
    const uint32_t e = entry_end(x, q);
    if (survives(p, s, x.r[q], x.r[q + 1])) n += (q == p.mc_s && p.mc_mode == 1) ? mc_entry_size(p) : e - q;
    q = e;
  }
  uint8_t t;
  if (mq_appended(p, s)) n += 3 + uint_pref_size(p.mq_val, &t);
  if (mc_appended(p, s)) n += 4 + p.mc_len;
  if (ms_appended(p, s)) n += 3 + signed_size(p.ms_val, &t);
  if (p.u.r)
    for (uint32_t q = p.u.ao; q < p.u.len;) {
      const uint32_t e = entry_end(p.u, q);
      if (u_kept(p, s, p.u.r[q], p.u.r[q + 1])) n += e - q;
      q = e;
    }
  if (p.as_norm) n += 3 + signed_size(p.as_val, &t);
  if (p.xs_norm) n += 3 + signed_size(p.xs_val, &t);
  if (p.tc) n += 3 + 5 + 24;
  return n;
}

FGB_HD void copy(uint8_t* d, const uint8_t* s, uint32_t n, int lane, int nl) {
  for (uint32_t j = lane; j < n; j += nl) d[j] = s[j];
}
FGB_HD void put_int(uint8_t* d, uint8_t a, uint8_t b, uint8_t t, uint32_t sz, int32_t v, int lane) {
  if (lane == 0) {
    d[0] = a; d[1] = b; d[2] = t;
    for (uint32_t k = 0; k < sz; ++k) d[3 + k] = static_cast<uint8_t>(static_cast<uint32_t>(v) >> (8 * k));
  }
}

// The mate's CIGAR text at d (mc_len bytes).  prefix(n) returns the inclusive prefix of n over the lanes (n for nl 1);
// lane nl - 1's is the lanes' total.
template <class Prefix>
FGB_HD void write_cigar(uint8_t* d, const Rec& m, int lane, int nl, Prefix&& prefix) {
  uint32_t base = 0;
  for (uint32_t k0 = 0; k0 < m.nc; k0 += nl) {
    const uint32_t k = k0 + lane;
    uint32_t op = 0, nd = 0;
    if (k < m.nc) { op = m.op(k); nd = ndigits(op >> 4); }
    const uint32_t piece = k < m.nc ? nd + 1 : 0;
    const uint32_t incl = prefix(piece);
    const uint32_t tot = prefix.last(incl);
    const uint32_t at = base + incl - piece;
    if (k < m.nc) {
      uint32_t v = op >> 4;
      for (uint32_t j = nd; j > 0; --j) { d[at + j - 1] = static_cast<uint8_t>('0' + v % 10); v /= 10; }
      d[at + nd] = static_cast<uint8_t>("MIDNSHP=X"[op & 0xF]);
    }
    base += tot;
  }
}

// An unmapped entry [q, e) of u copied to d, reversed or reverse-complemented on a reverse-strand record
// (reverse_tag_in_place_raw_by_type / revcomp_tag_in_place_raw_by_type, zipper.rs:540-581; tags.rs:754-836)
FGB_HD void copy_u_entry(uint8_t* d, const Plan& p, const Sets& s, uint32_t q, uint32_t e, int lane, int nl) {
  const uint8_t* src = p.u.r + q;
  const uint32_t n = e - q;
  const uint8_t a = src[0], b = src[1], t = src[2];
  const bool rv = p.rev && in_set(s.reverse, s.n_reverse, a, b);
  const bool rc = p.rev && !rv && in_set(s.revcomp, s.n_revcomp, a, b);
  if ((rv || rc) && t == 'Z') {
    const uint32_t m = n - 4;   // the value without its NUL
    copy(d, src, 3, lane, nl);
    for (uint32_t j = lane; j < m; j += nl) {
      const uint8_t c = src[3 + m - 1 - j];
      d[3 + j] = rc ? rfilter::complement(c) : c;
    }
    if (lane == 0) d[n - 1] = 0;
  } else if ((rv || rc) && t == 'B') {
    const uint32_t es = static_cast<uint32_t>(rfilter::fixed_size(src[3])), cnt = ld32(src + 4);
    copy(d, src, 8, lane, nl);
    for (uint32_t j = lane; j < cnt * es; j += nl) {
      const uint32_t k = j / es, x = j % es;
      d[8 + j] = src[8 + (cnt - 1 - k) * es + x];
    }
  } else {
    copy(d, src, n, lane, nl);
  }
}

// Pass 2: the edited record at d (out_size bytes)
template <class Prefix>
FGB_HD void write(uint8_t* d, const Plan& p, const Sets& s, int lane, int nl, Prefix&& prefix) {
  const Rec& x = p.x;
  for (uint32_t j = lane; j < 32; j += nl) {   // the fixed fields, each byte from the edited value or the record
    const uint32_t f = j >> 2;
    const int32_t v = f == 0 ? p.ref : f == 1 ? p.pos : f == 5 ? p.mref : f == 6 ? p.mpos : f == 7 ? p.tlen
                      : f == 3 ? static_cast<int32_t>((static_cast<uint32_t>(p.flags) << 16) | ld16(x.r + 12))
                               : ldi32(x.r + (j & ~3u));
    d[j] = static_cast<uint8_t>(static_cast<uint32_t>(v) >> (8 * (j & 3)));
  }
  copy(d + 32, x.r + 32, x.ao - 32, lane, nl);
  uint32_t w = x.ao;
  for (uint32_t q = x.ao; q < x.len;) {
    const uint32_t e = entry_end(x, q);
    const uint8_t a = x.r[q], b = x.r[q + 1];
    if (survives(p, s, a, b)) {
      if (a == 'M' && b == 'Q' && p.mq_inplace) {
        put_int(d + w, 'M', 'Q', x.r[q + 2], 4, p.mq_val, lane);
        w += 7;
      } else if (q == p.mc_s && p.mc_mode == 1) {
        const bool same = e - q - 4 == p.mc_len;
        if (lane == 0) { d[w] = 'M'; d[w + 1] = 'C'; d[w + 2] = same ? x.r[q + 2] : 'Z'; d[w + 3 + p.mc_len] = same ? x.r[e - 1] : 0; }
        write_cigar(d + w + 3, p.mate, lane, nl, prefix);
        w += 4 + p.mc_len;
      } else {
        copy(d + w, x.r + q, e - q, lane, nl);
        w += e - q;
      }
    }
    q = e;
  }
  uint8_t t;
  uint32_t sz;
  if (mq_appended(p, s)) { sz = uint_pref_size(p.mq_val, &t); put_int(d + w, 'M', 'Q', t, sz, p.mq_val, lane); w += 3 + sz; }
  if (mc_appended(p, s)) {
    if (lane == 0) { d[w] = 'M'; d[w + 1] = 'C'; d[w + 2] = 'Z'; d[w + 3 + p.mc_len] = 0; }
    write_cigar(d + w + 3, p.mate, lane, nl, prefix);
    w += 4 + p.mc_len;
  }
  if (ms_appended(p, s)) { sz = signed_size(p.ms_val, &t); put_int(d + w, 'm', 's', t, sz, p.ms_val, lane); w += 3 + sz; }
  if (p.u.r)
    for (uint32_t q = p.u.ao; q < p.u.len;) {
      const uint32_t e = entry_end(p.u, q);
      if (u_kept(p, s, p.u.r[q], p.u.r[q + 1])) { copy_u_entry(d + w, p, s, q, e, lane, nl); w += e - q; }
      q = e;
    }
  if (p.as_norm) { sz = signed_size(p.as_val, &t); put_int(d + w, 'A', 'S', t, sz, p.as_val, lane); w += 3 + sz; }
  if (p.xs_norm) { sz = signed_size(p.xs_val, &t); put_int(d + w, 'X', 'S', t, sz, p.xs_val, lane); w += 3 + sz; }
  if (p.tc && lane == 0) {
    d[w] = 't'; d[w + 1] = 'c'; d[w + 2] = 'B'; d[w + 3] = 'i';
    d[w + 4] = 6; d[w + 5] = 0; d[w + 6] = 0; d[w + 7] = 0;
    auto st32 = [&](uint32_t at, int32_t v) {
      for (int j = 0; j < 4; ++j) d[at + j] = static_cast<uint8_t>(static_cast<uint32_t>(v) >> (8 * j));
    };
    st32(w + 8, p.tc_ref1); st32(w + 12, p.tc_pos1); st32(w + 16, p.tc_neg1);
    st32(w + 20, p.tc_ref2); st32(w + 24, p.tc_pos2); st32(w + 28, p.tc_neg2);
  }
}

}  // namespace zip
}  // namespace fgb
