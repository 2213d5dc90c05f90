// Sort keys of `fgumi sort` (coordinate, template-coordinate and queryname) from raw BAM records, written once for the
// host and the device (FGB_HD): the key kernels (sort_kernels.cuh) run one record per thread, fgb_host_sort_keys,
// fgb_host_sort_name_key and fgb_host_sort_verify run the very same functions on host threads, and the CPU tests
// compare both with oracle/sort_oracle.py (queryname: tests/queryname_oracle.py).  Citations are relative to the
// fgumi 0.2.0 source tree:
//   inline_buffer.rs  src/lib/sort/inline_buffer.rs         (PackedCoordinateKey, TemplateKey, core_cmp)
//   raw.rs            src/lib/sort/raw.rs                   (LibraryLookup, extract_template_key_inline)
//   tags.rs           crates/fgumi-raw-bam/src/tags.rs      (parse_mi_bytes, extract_template_aux_tags)
//   fields.rs         crates/fgumi-raw-bam/src/fields.rs    (tag_value_size, aux_data_slice)
//   cigar.rs          crates/fgumi-raw-bam/src/cigar.rs     (unclipped_5prime_raw, mate_unclipped_5prime)
//
// Every byte read is checked against the record's length.  Only a record shorter than its 32-byte fixed part is an
// error; everything else takes the reference's soft handling so that the keys match: a read name that runs past the
// record hashes as empty, a CIGAR that runs past it leaves pos unchanged, and aux problems end the scan.  Integer
// arithmetic on positions wraps as the reference's release build does.
//
// The one deliberate deviation: the reference hashes the read name and the cell barcode with ahash, whose output
// depends on the CPU features it was built for; here both are 64-bit FNV-1a over the bytes (DESIGN.md section 10).
#pragma once
#include <stdint.h>

#ifndef FGB_HD
#ifdef __CUDACC__
#define FGB_HD __host__ __device__ __forceinline__
#else
#define FGB_HD inline
#endif
#endif

namespace fgb {
namespace sortk {

enum : uint32_t { kCoordinate = 0, kTemplateCoordinate = 1, kQueryname = 2, kQuerynameNatural = 3 };
constexpr int kWords = 5;   // primary, secondary, cb_hash, tertiary, name_hash_upper
constexpr int kNameWordsMax = 64;   // queryname: a 254-byte name encodes to at most 2 * 254 + 1 bytes (natural)
constexpr int32_t kI32Max = 2147483647;

// What the key functions need beyond the record: the header's RG -> library table (IDs sorted bytewise, so a
// lookup is a binary search) and the cell tag.
struct Ctx {
  const uint8_t* rg_bytes;   // RG IDs back to back
  const uint32_t* rg_off;    // n_rg + 1 offsets into rg_bytes
  const uint32_t* rg_lib;    // library ordinal of each RG
  uint32_t n_rg;
  uint32_t order;            // kCoordinate / kTemplateCoordinate
  uint8_t cell[2];
  uint8_t has_cell;
  uint8_t reserved;
};

FGB_HD uint16_t ld16(const uint8_t* p) { return static_cast<uint16_t>(p[0] | (p[1] << 8)); }
FGB_HD uint32_t ld32(const uint8_t* p) {
  return static_cast<uint32_t>(p[0]) | (static_cast<uint32_t>(p[1]) << 8) | (static_cast<uint32_t>(p[2]) << 16) |
         (static_cast<uint32_t>(p[3]) << 24);
}

// 64-bit FNV-1a (the deviation above; oracle/sort_oracle.py fnv1a64)
FGB_HD uint64_t fnv1a64(const uint8_t* p, uint64_t n) {
  uint64_t h = 0xcbf29ce484222325ull;
  for (uint64_t i = 0; i < n; ++i) { h ^= p[i]; h *= 0x100000001b3ull; }
  return h;
}

// std::str::from_utf8 acceptance: well-formed UTF-8, no surrogates, no overlong forms
FGB_HD bool valid_utf8(const uint8_t* s, uint64_t n) {
  uint64_t i = 0;
  while (i < n) {
    const uint8_t c = s[i];
    if (c < 0x80) { ++i; continue; }
    uint32_t need, cp, lo;
    if ((c & 0xE0) == 0xC0) { need = 1; cp = c & 0x1F; lo = 0x80; }
    else if ((c & 0xF0) == 0xE0) { need = 2; cp = c & 0x0F; lo = 0x800; }
    else if ((c & 0xF8) == 0xF0) { need = 3; cp = c & 0x07; lo = 0x10000; }
    else return false;
    for (uint32_t k = 1; k <= need; ++k) {
      if (i + k >= n) return false;
      const uint8_t d = s[i + k];
      if ((d & 0xC0) != 0x80) return false;
      cp = (cp << 6) | (d & 0x3F);
    }
    if (cp < lo || cp > 0x10FFFF || (cp >= 0xD800 && cp <= 0xDFFF)) return false;
    i += need + 1;
  }
  return true;
}

// extract_coordinate_key_inline (inline_buffer.rs:423-436) with PackedCoordinateKey::new (:66-78): the unmapped flag
// is not looked at, only tid < 0 sorts last.
FGB_HD uint64_t coordinate_key(const uint8_t* r) {
  const int32_t tid = static_cast<int32_t>(ld32(r)), pos = static_cast<int32_t>(ld32(r + 4));
  if (tid < 0) return ~0ull;
  const uint64_t rev = (ld16(r + 14) & 0x10) ? 1 : 0;
  return (static_cast<uint64_t>(static_cast<uint32_t>(tid)) << 34) |
         ((static_cast<uint64_t>(static_cast<int64_t>(pos)) + 1) << 1) | rev;
}

FGB_HD bool consumes_ref(uint32_t t) { return t == 0 || t == 2 || t == 3 || t == 7 || t == 8; }

// unclipped_5prime_raw (cigar.rs:237-255, 470-508): 0-based, in the basis of `pos`; pos unchanged without a CIGAR or
// when the CIGAR runs past the record
FGB_HD int32_t unclipped_5prime(const uint8_t* r, uint64_t n, int32_t pos, bool reverse) {
  const uint32_t nc = ld16(r + 12);
  if (nc == 0) return pos;
  const uint64_t cs = 32 + static_cast<uint64_t>(r[8]);
  if (cs + 4ull * nc > n) return pos;
  if (!reverse) {
    uint32_t clipped = 0;
    for (uint32_t i = 0; i < nc; ++i) {
      const uint32_t op = ld32(r + cs + 4ull * i), t = op & 0xF;
      if (t == 4 || t == 5) clipped += op >> 4;
      else break;
    }
    return static_cast<int32_t>(static_cast<uint32_t>(pos) - clipped);
  }
  uint32_t ref_len = 0, trailing = 0;
  bool saw = false;
  for (uint32_t i = 0; i < nc; ++i) {
    const uint32_t op = ld32(r + cs + 4ull * i), t = op & 0xF;
    if (consumes_ref(t)) { ref_len += op >> 4; trailing = 0; saw = true; }
    else if ((t == 4 || t == 5) && saw) trailing += op >> 4;
  }
  return static_cast<int32_t>(static_cast<uint32_t>(pos) + ref_len + trailing - 1u);
}

FGB_HD bool is_digit(uint8_t c) { return c >= '0' && c <= '9'; }

// cigar[a..b].parse::<i32>().unwrap_or(0) on a run of ASCII digits: 0 when empty or past i32::MAX
FGB_HD uint32_t parse_num(const uint8_t* s, uint32_t a, uint32_t b) {
  if (a >= b) return 0;
  uint64_t v = 0;
  for (uint32_t i = a; i < b; ++i) {
    v = v * 10 + (s[i] - '0');
    if (v > 2147483647ull) return 0;
  }
  return static_cast<uint32_t>(v);
}

// mate_unclipped_5prime (cigar.rs:263-269) over unclipped_other_start / unclipped_other_end (:294-306) and the MC
// parsers parse_leading_clips / parse_ref_len_and_trailing_clips (:514-573); 0-based like mate_pos
FGB_HD int32_t mate_unclipped_5prime(int32_t mate_pos, bool mate_reverse, const uint8_t* mc, uint32_t n) {
  uint32_t num_start = 0;
  if (!mate_reverse) {
    uint32_t clipped = 0;
    for (uint32_t i = 0; i < n; ++i) {
      if (is_digit(mc[i])) continue;
      const uint32_t num = parse_num(mc, num_start, i);
      if (mc[i] == 'S' || mc[i] == 'H') { clipped += num; num_start = i + 1; }
      else break;
    }
    return static_cast<int32_t>(static_cast<uint32_t>(mate_pos) - clipped);
  }
  uint32_t ref_len = 0, trailing = 0;
  bool saw = false;
  for (uint32_t i = 0; i < n; ++i) {
    const uint8_t c = mc[i];
    if (is_digit(c)) continue;
    const uint32_t num = parse_num(mc, num_start, i);
    num_start = i + 1;
    if (c == 'M' || c == 'D' || c == 'N' || c == '=' || c == 'X') { ref_len += num; trailing = 0; saw = true; }
    else if ((c == 'S' || c == 'H') && saw) trailing += num;
  }
  return static_cast<int32_t>(static_cast<uint32_t>(mate_pos) + ref_len + trailing - 1u);
}

// TAG_FIXED_SIZES (fields.rs:269-280)
FGB_HD uint32_t fixed_size(uint8_t t) {
  switch (t) {
    case 'A': case 'c': case 'C': return 1;
    case 's': case 'S': return 2;
    case 'i': case 'I': case 'f': return 4;
    default: return 0;
  }
}

// The first NUL in [p, p + n): its index, or n when there is none
FGB_HD uint64_t find_nul(const uint8_t* p, uint64_t n) {
  uint64_t i = 0;
  while (i < n && p[i]) ++i;
  return i;
}

// tag_value_size (fields.rs:289-310): false = None.  Fixed sizes are returned whether or not the value fits, as there.
FGB_HD bool tag_value_size(uint8_t t, const uint8_t* d, uint64_t left, uint64_t* size) {
  const uint32_t f = fixed_size(t);
  if (f) { *size = f; return true; }
  if (t == 'Z' || t == 'H') {
    const uint64_t z = find_nul(d, left);
    if (z == left) return false;
    *size = z + 1;
    return true;
  }
  if (t == 'B') {
    if (left < 5) return false;
    const uint32_t es = fixed_size(d[0]);
    if (!es) return false;
    *size = 5 + static_cast<uint64_t>(ld32(d + 1)) * es;
    return true;
  }
  return false;
}

// parse_mi_bytes (tags.rs:184-212) with the caller's unwrap_or((0, true))
FGB_HD void parse_mi(const uint8_t* s, uint64_t n, uint64_t* mi, bool* is_a) {
  *mi = 0;
  *is_a = true;
  if (n == 0) return;
  uint64_t num = n;
  bool a = true;
  if (n >= 2 && s[n - 2] == '/') { num = n - 2; a = s[n - 1] != 'B'; }
  if (num == 0) return;
  uint64_t v = 0;
  for (uint64_t i = 0; i < num; ++i) {
    if (!is_digit(s[i])) return;
    const uint64_t d = s[i] - '0';
    v = v > (~0ull - d) / 10 ? ~0ull : v * 10 + d;   // saturating_mul(10).saturating_add(d)
  }
  *mi = v;
  *is_a = a;
}

struct Aux {
  uint64_t mi;
  bool mi_a, has_rg, has_cell, has_mc;
  const uint8_t* rg; uint64_t rg_len;
  const uint8_t* cell; uint64_t cell_len;
  const uint8_t* mc; uint64_t mc_len;
};

// extract_template_aux_tags (tags.rs:299-377): one pass for MI (Z or any integer type), RG, the cell tag and MC, which
// ends early once every wanted tag has been met; a later entry of a tag replaces an earlier one until then.
FGB_HD Aux template_aux(const uint8_t* r, uint64_t n, const Ctx& c) {
  Aux x;
  x.mi = 0; x.mi_a = true; x.has_rg = x.has_cell = x.has_mc = false;
  x.rg = x.cell = x.mc = r; x.rg_len = x.cell_len = x.mc_len = 0;
  // aux_data_slice (fields.rs:449-483): empty when the offset runs past the record
  const uint64_t off = 32 + static_cast<uint64_t>(r[8]) + 4ull * ld16(r + 12) + (static_cast<uint64_t>(ld32(r + 16)) + 1) / 2 +
                       ld32(r + 16);
  if (off > n) return x;
  const uint8_t* a = r + off;
  const uint64_t an = n - off;
  const uint32_t target = c.has_cell ? 0xF : 0xB;
  uint32_t found = 0;
  uint64_t p = 0;
  while (p + 3 <= an) {
    const uint8_t t0 = a[p], t1 = a[p + 1], vt = a[p + 2];
    const uint8_t* d = a + p + 3;
    const uint64_t left = an - (p + 3);
    uint64_t size = 0;
    if (t0 == 'M' && t1 == 'I') {
      if (vt == 'Z') {
        const uint64_t z = find_nul(d, left);
        if (z == left) break;
        parse_mi(d, z, &x.mi, &x.mi_a);
        p += 3 + z + 1;
      } else {
        // extract_int_value (tags.rs:127-151): the value must fit; a negative one is ignored
        bool has = false;
        int64_t v = 0;
        switch (vt) {
          case 'c': if (left >= 1) { v = static_cast<int8_t>(d[0]); has = true; } break;
          case 'C': if (left >= 1) { v = d[0]; has = true; } break;
          case 's': if (left >= 2) { v = static_cast<int16_t>(ld16(d)); has = true; } break;
          case 'S': if (left >= 2) { v = ld16(d); has = true; } break;
          case 'i': if (left >= 4) { v = static_cast<int32_t>(ld32(d)); has = true; } break;
          case 'I': if (left >= 4) { v = ld32(d); has = true; } break;
          default: break;
        }
        if (has && v >= 0) { x.mi = static_cast<uint64_t>(v); x.mi_a = true; }
        if (!tag_value_size(vt, d, left, &size)) break;
        p += 3 + size;
      }
      found |= 1;
      if ((found & target) == target) return x;
      continue;
    }
    if (vt == 'Z') {
      const uint64_t z = find_nul(d, left);
      if (z == left) break;
      if (t0 == 'R' && t1 == 'G') { x.rg = d; x.rg_len = z; x.has_rg = true; found |= 2; }
      if (c.has_cell && t0 == c.cell[0] && t1 == c.cell[1]) { x.cell = d; x.cell_len = z; x.has_cell = true; found |= 4; }
      if (t0 == 'M' && t1 == 'C') {
        x.has_mc = valid_utf8(d, z);   // from_utf8(value).ok(): a non-UTF-8 MC counts as absent
        x.mc = d; x.mc_len = z;
        found |= 8;
      }
      if ((found & target) == target) return x;
      p += 3 + z + 1;
      continue;
    }
    if (!tag_value_size(vt, d, left, &size)) break;
    p += 3 + size;
  }
  return x;
}

// LibraryLookup::ordinal_from_rg (raw.rs:307-312): 0 for no RG or an RG the header does not declare
FGB_HD uint32_t library_ordinal(const Ctx& c, const uint8_t* rg, uint64_t len) {
  uint32_t lo = 0, hi = c.n_rg;
  while (lo < hi) {
    const uint32_t mid = lo + (hi - lo) / 2;
    const uint8_t* s = c.rg_bytes + c.rg_off[mid];
    const uint64_t sl = c.rg_off[mid + 1] - c.rg_off[mid];
    int cmp = 0;
    const uint64_t m = sl < len ? sl : len;
    for (uint64_t i = 0; i < m && !cmp; ++i) cmp = s[i] < rg[i] ? -1 : s[i] > rg[i] ? 1 : 0;
    if (!cmp) cmp = sl < len ? -1 : sl > len ? 1 : 0;
    if (cmp == 0) return c.rg_lib[mid];
    if (cmp < 0) lo = mid + 1;
    else hi = mid;
  }
  return 0;
}

// TemplateKey::new (inline_buffer.rs:478-520), truncations included
FGB_HD void pack_template(int32_t tid1, int32_t pos1, bool neg1, int32_t tid2, int32_t pos2, bool neg2, uint64_t cb_hash,
                          uint32_t library, uint64_t mi, bool mi_a, uint64_t name_hash, bool is_upper, uint64_t k[kWords]) {
  const uint64_t t1 = tid1 == kI32Max ? 0xFFFFull : static_cast<uint64_t>(tid1 < 0 ? 0 : tid1) & 0xFFFF;
  const uint64_t t2 = tid2 == kI32Max ? 0xFFFFull : static_cast<uint64_t>(tid2 < 0 ? 0 : tid2) & 0xFFFF;
  const uint64_t p1 = static_cast<uint32_t>(pos1) ^ 0x80000000u, p2 = static_cast<uint32_t>(pos2) ^ 0x80000000u;
  k[0] = (t1 << 48) | (t2 << 32) | p1;
  k[1] = (p2 << 32) | (static_cast<uint64_t>(!neg1) << 1) | static_cast<uint64_t>(!neg2);
  k[2] = cb_hash;
  k[3] = ((static_cast<uint64_t>(library) & 0xFFFF) << 48) | ((mi & 0xFFFFFFFFFFFFull) << 1) | static_cast<uint64_t>(!mi_a);
  k[4] = (name_hash << 1) | static_cast<uint64_t>(is_upper);
}

// extract_template_key_inline (raw.rs:2917-3013)
FGB_HD void template_key(const uint8_t* r, uint64_t n, const Ctx& c, uint64_t k[kWords]) {
  const Aux x = template_aux(r, n, c);
  const uint32_t library = x.has_rg ? library_ordinal(c, x.rg, x.rg_len) : 0;
  const uint64_t cb_hash = x.has_cell ? fnv1a64(x.cell, x.cell_len) : 0;
  const int32_t tid = static_cast<int32_t>(ld32(r)), pos = static_cast<int32_t>(ld32(r + 4));
  const int32_t mate_tid = static_cast<int32_t>(ld32(r + 20)), mate_pos = static_cast<int32_t>(ld32(r + 24));
  const uint16_t flag = ld16(r + 14);
  const bool unmapped = flag & 0x4, mate_unmapped = flag & 0x8, reverse = flag & 0x10, mate_reverse = flag & 0x20;
  const bool paired = flag & 0x1;
  const uint64_t name_len = r[8] ? r[8] - 1u : 0;   // without the NUL; empty when it runs past the record
  const uint64_t name_hash = fnv1a64(r + 32, name_len > 0 && 32 + name_len <= n ? name_len : 0);
  const bool mate_mapped = paired && !mate_unmapped;
  const int32_t mate_unclipped = mate_mapped && x.has_mc
      ? mate_unclipped_5prime(mate_pos, mate_reverse, x.mc, static_cast<uint32_t>(x.mc_len)) : mate_pos;
  if (unmapped) {
    if (mate_mapped) {   // the mate's position, always "upper"
      pack_template(mate_tid, mate_unclipped, mate_reverse, kI32Max, kI32Max, false, cb_hash, library, x.mi, x.mi_a,
                    name_hash, true, k);
      return;
    }
    // TemplateKey::unmapped (inline_buffer.rs:524-532)
    k[0] = ~0ull; k[1] = ~0ull; k[2] = cb_hash; k[3] = 0;
    k[4] = (name_hash << 1) | ((flag & 0x80) ? 1u : 0u);
    return;
  }
  const int32_t this_pos = unclipped_5prime(r, n, pos, reverse);
  if (mate_mapped) {
    const bool is_upper = tid > mate_tid || (tid == mate_tid && (this_pos > mate_unclipped ||
                                                                 (this_pos == mate_unclipped && reverse)));
    if (is_upper)
      pack_template(mate_tid, mate_unclipped, mate_reverse, tid, this_pos, reverse, cb_hash, library, x.mi, x.mi_a,
                    name_hash, true, k);
    else
      pack_template(tid, this_pos, reverse, mate_tid, mate_unclipped, mate_reverse, cb_hash, library, x.mi, x.mi_a,
                    name_hash, false, k);
    return;
  }
  pack_template(tid, this_pos, reverse, kI32Max, kI32Max, false, cb_hash, library, x.mi, x.mi_a, name_hash, false, k);
}

// The key of one record (n bytes, no block_size prefix): false for a record shorter than its fixed part.  The
// coordinate key is word 0; the other words are 0.
FGB_HD bool record_key(const uint8_t* r, uint64_t n, const Ctx& c, uint64_t k[kWords]) {
  for (int w = 0; w < kWords; ++w) k[w] = 0;
  if (n < 32) return false;
  if (c.order == kCoordinate) k[0] = coordinate_key(r);
  else template_key(r, n, c, k);
  return true;
}

// ---- queryname (keys.rs:338-363, 446-456, 495-628; natural_compare_nul in crates/fgumi-raw-bam/src/sort.rs:181-238) --
// The key of a record is a byte string E, zero-padded to W big-endian words, then one word
// (len(E) << 16) | queryname_flag_order(flag).  Comparing the W + 1 words in order is exactly the reference comparator
// (DESIGN.md section 10 has the argument):
//   lexicographic: E = the name bytes, embedded NULs included;
//   natural:       E = the name cut at its first NUL, each maximal run of ASCII digits replaced by 0x30, the count of
//                  its significant digits (leading zeros stripped) and those digits; other bytes copied.

// queryname_flag_order (keys.rs:361-363): R1 / R2, then secondary, then supplementary
FGB_HD uint32_t queryname_flag_order(uint16_t f) {
  return ((f & 0xc0u) << 8) | ((f & 0x100u) << 3) | ((f & 0x800u) >> 3);
}

// extract_raw_name_and_flags (keys.rs:450-456): bam[32 .. 32 + l_read_name - 1] when that fits the record, else empty
FGB_HD uint32_t name_length(const uint8_t* r, uint64_t n) {
  const uint32_t l = r[8] ? r[8] - 1u : 0;
  return l > 0 && 32 + static_cast<uint64_t>(l) <= n ? l : 0;
}

// The name words W of a record whose l_read_name byte is `lrn`: E has at most lrn - 1 bytes (natural: 2 (lrn - 1) + 1,
// every other byte a one-digit run).  A run uses the largest W of its records.
FGB_HD uint32_t name_words(uint8_t lrn, bool natural) {
  const uint32_t l = lrn ? lrn - 1u : 0;
  const uint32_t e = natural && l ? 2 * l + 1 : l;
  return (e + 7) / 8;
}

// E one byte at a time, read straight from the record (no copy of the name): next() is the next byte, or -1 after the
// last; `len` counts the bytes returned.
struct NameEncoder {
  const uint8_t* s;
  uint32_t n, i, run_end, len;
  uint8_t phase;   // natural: 0 between tokens, 1 the count byte is next, 2 digits [i, run_end) are next
  bool natural;

  FGB_HD void init(const uint8_t* r, uint64_t rn, bool nat) {
    s = r + 32;
    n = name_length(r, rn);
    if (nat) n = static_cast<uint32_t>(find_nul(s, n));   // natural_compare_nul stops at the first NUL
    i = run_end = len = 0;
    phase = 0;
    natural = nat;
  }
  FGB_HD void init_empty() { s = nullptr; n = i = run_end = len = 0; phase = 0; natural = false; }

  FGB_HD int next() {
    if (phase == 2) {
      if (i < run_end) { ++len; return s[i++]; }
      phase = 0;
    }
    if (phase == 1) { phase = 2; ++len; return static_cast<int>(run_end - i); }
    if (i >= n) return -1;
    const uint8_t c = s[i];
    ++len;
    if (!natural || !is_digit(c)) { ++i; return c; }
    uint32_t e = i;
    while (e < n && is_digit(s[e])) ++e;
    while (i < e && s[i] == '0') ++i;
    run_end = e;
    phase = 1;
    return 0x30;
  }

  // the next big-endian word of E, zero-padded past its end
  FGB_HD uint64_t word() {
    uint64_t w = 0;
    for (int b = 0; b < 8; ++b) {
      const int c = next();
      w = (w << 8) | static_cast<uint64_t>(c < 0 ? 0 : c);
    }
    return w;
  }
};

// The last key word, once all W name words have been taken from `e`
FGB_HD uint64_t name_last_word(const NameEncoder& e, const uint8_t* r) {
  return (static_cast<uint64_t>(e.len) << 16) | queryname_flag_order(ld16(r + 14));
}

// The reference comparator on two records (the host merge and --verify): the lexicographic byte compare of
// RawQuerynameLexKey::cmp (keys.rs:624-628) or natural_compare_nul, then the flag order.  Negative, 0 or positive.
FGB_HD int nul_at(const uint8_t* s, uint32_t n, uint32_t p) { return p < n ? s[p] : 0; }

FGB_HD int natural_compare_nul(const uint8_t* a, uint32_t na, const uint8_t* b, uint32_t nb) {
  // sort.rs:181-238 over names cut at their first NUL; index n reads as the terminating NUL
  uint32_t pa = 0, pb = 0;
  while (nul_at(a, na, pa) && nul_at(b, nb, pb)) {
    const int ca = nul_at(a, na, pa), cb = nul_at(b, nb, pb);
    if (!is_digit(static_cast<uint8_t>(ca)) || !is_digit(static_cast<uint8_t>(cb))) {
      if (ca != cb) return ca - cb;
      ++pa; ++pb;
    } else {
      while (nul_at(a, na, pa) == '0') ++pa;
      while (nul_at(b, nb, pb) == '0') ++pb;
      while (is_digit(static_cast<uint8_t>(nul_at(a, na, pa))) && nul_at(a, na, pa) == nul_at(b, nb, pb)) { ++pa; ++pb; }
      const bool a_digit = is_digit(static_cast<uint8_t>(nul_at(a, na, pa)));
      const bool b_digit = is_digit(static_cast<uint8_t>(nul_at(b, nb, pb)));
      const int diff = nul_at(a, na, pa) - nul_at(b, nb, pb);
      if (a_digit && b_digit) { ++pa; ++pb; }
      while (is_digit(static_cast<uint8_t>(nul_at(a, na, pa))) && is_digit(static_cast<uint8_t>(nul_at(b, nb, pb)))) {
        ++pa; ++pb;
      }
      if (is_digit(static_cast<uint8_t>(nul_at(a, na, pa)))) return 1;
      if (is_digit(static_cast<uint8_t>(nul_at(b, nb, pb)))) return -1;
      if (diff) return diff;
    }
  }
  if (nul_at(a, na, pa)) return 1;
  if (nul_at(b, nb, pb)) return -1;
  return 0;
}

FGB_HD int queryname_cmp(const uint8_t* a, uint64_t na, const uint8_t* b, uint64_t nb, bool natural) {
  uint32_t la = name_length(a, na), lb = name_length(b, nb);
  int c = 0;
  if (natural) {
    la = static_cast<uint32_t>(find_nul(a + 32, la));
    lb = static_cast<uint32_t>(find_nul(b + 32, lb));
    c = natural_compare_nul(a + 32, la, b + 32, lb);
  } else {
    const uint32_t m = la < lb ? la : lb;
    for (uint32_t i = 0; i < m && !c; ++i) c = static_cast<int>(a[32 + i]) - static_cast<int>(b[32 + i]);
    if (!c) c = la < lb ? -1 : la > lb ? 1 : 0;
  }
  if (c) return c;
  const uint32_t fa = queryname_flag_order(ld16(a + 14)), fb = queryname_flag_order(ld16(b + 14));
  return fa < fb ? -1 : fa > fb ? 1 : 0;
}

}  // namespace sortk
}  // namespace fgb
