// `fgumi filter --ref` on the device (driven by host/filter_host.cpp through the launchers in capi.cu), one warp per
// record with the lanes across its bases:
//   pass 1    per-base tag reversal, masking, the NM / UQ / MD-length walk over the resident reference and the read
//             gates, in place on the uploaded records; an error code with the first bad record by atomicMin;
//   decision  one thread per template: each record's kept / rejected flag;
//   pass 2    each edited record with its block_size word written into its slot of the kept or the rejects stream.
// The rules themselves (tag lookup, per-base mask predicates, read gates) are host/record_filter.h, shared with the
// host filter.  Citations: alignment_tags.rs = crates/fgumi-sam/src/alignment_tags.rs, tags.rs =
// crates/fgumi-raw-bam/src/tags.rs, tag_reversal.rs = src/lib/tag_reversal.rs.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "host/filter_device.h"
#include "host/record_filter.h"

namespace fgb {

constexpr int kFilterThreads = 256;

namespace frk {

constexpr unsigned kFull = 0xffffffffu;

__device__ __forceinline__ uint32_t warp_sum(uint32_t v) { return __reduce_add_sync(kFull, v); }
__device__ __forceinline__ uint8_t lower(uint8_t c) { return (c >= 'A' && c <= 'Z') ? c + 32 : c; }
__device__ __forceinline__ uint32_t ndigits(uint32_t v) {
  uint32_t d = 1;
  while (v >= 10) { v /= 10; ++d; }
  return d;
}
__device__ __forceinline__ void put_digits(uint8_t* dst, uint32_t v, uint32_t nd) {
  for (uint32_t k = nd; k > 0; --k) { dst[k - 1] = static_cast<uint8_t>('0' + v % 10); v /= 10; }
}
// append_int_tag's smallest type (tags.rs:533-553): 1, 2 or 4 value bytes and the type byte
__device__ __forceinline__ uint32_t int_size(int32_t v, uint8_t* type) {
  if (v >= -128 && v <= 127) { *type = 'c'; return 1; }
  if (v >= 0 && v <= 255) { *type = 'C'; return 1; }
  if (v >= 0 && v <= 65535) { *type = 'S'; return 2; }
  if (v >= -32768 && v < 0) { *type = 's'; return 2; }
  *type = 'i';
  return 4;
}
__device__ __forceinline__ void warp_copy(uint8_t* dst, const uint8_t* src, uint64_t n, int lane) {
  for (uint64_t j = lane; j < n; j += 32) dst[j] = src[j];
}
using rfilter::complement;   // reverse_complement_string_tag_in_place

// reverse_per_base_tags_raw (tag_reversal.rs:27-66) on a reverse-strand record's aux area: the B arrays and Z strings
// cd ce ad ae bd be aq bq reversed element by element, the Z strings ac bc reverse-complemented
__device__ void reverse_tags(uint8_t* aux, uint64_t an, int lane) {
  const char* kRev = "cdceadaebdbeaqbqacbc";
  for (int t = 0; t < 10; ++t) {
    const rfilter::TagRef r = rfilter::find_tag(aux, an, kRev + 2 * t);
    uint8_t* d = const_cast<uint8_t*>(r.data);
    if (t < 8 && r.type == 'B') {
      const uint32_t es = static_cast<uint32_t>(rfilter::fixed_size(r.sub));
      for (uint32_t k = lane; k < r.count / 2; k += 32) {
        uint8_t* a = d + static_cast<uint64_t>(k) * es;
        uint8_t* b = d + static_cast<uint64_t>(r.count - 1 - k) * es;
        for (uint32_t x = 0; x < es; ++x) { const uint8_t v = a[x]; a[x] = b[x]; b[x] = v; }
      }
    } else if (r.type == 'Z') {
      const uint32_t m = r.count - 1;   // without the NUL
      const bool rc = t >= 8;
      for (uint32_t k = lane; k < (m + 1) / 2; k += 32) {
        const uint32_t j = m - 1 - k;
        const uint8_t a = d[k], b = d[j];
        d[k] = rc ? complement(b) : b;
        d[j] = rc ? complement(a) : a;
      }
    }
    __syncwarp();
  }
}

struct Walk {
  int32_t nm;
  uint32_t uq, md_len;
  bool bad;
};

// regenerate_alignment_tags_raw's CIGAR walk (alignment_tags.rs:323-411) with the lanes across the bases of each
// M / = / X op: the mismatches of 32 bases by ballot, each mismatch's preceding match run from the ballot (or the run
// carried in from the bases before), the MD pieces' offsets by a warp scan.  W: write the MD text to `md`.  `ref` is
// the reference from the alignment start.  bad: an op consumes more bases than l_seq.
template <bool W>
__device__ Walk md_walk(const uint8_t* r, uint32_t nc, uint64_t co, uint64_t so, uint64_t qo, uint32_t L,
                        const uint8_t* __restrict__ ref, uint8_t* md, int lane) {
  Walk w{0, 0, 0, false};
  uint32_t run = 0, seq_pos = 0;
  uint64_t ref_off = 0;
  for (uint32_t k = 0; k < nc; ++k) {
    const uint32_t op = rfilter::ld32(r + co + 4ull * k), t = op & 0xF, len = op >> 4;
    if (t == 0 || t == 7 || t == 8) {
      if (static_cast<uint64_t>(seq_pos) + len > L) { w.bad = true; return w; }
      for (uint32_t c = 0; c < len; c += 32) {
        const uint32_t i = c + lane;
        bool mis = false;
        uint8_t rb = 0;
        uint32_t q = 0;
        if (i < len) {
          const uint32_t sp = seq_pos + i;
          const uint8_t code = rfilter::base_code(r, so, sp);
          rb = ref[ref_off + i];
          mis = code == 15 || lower(static_cast<uint8_t>("=ACMGRSVTWYHKDBN"[code])) != lower(rb);
          if (mis) q = r[qo + sp];
        }
        const unsigned m = __ballot_sync(kFull, mis);
        uint32_t piece = 0, my_run = 0;
        if (mis) {
          const unsigned below = m & ((1u << lane) - 1u);
          my_run = below ? static_cast<uint32_t>(lane - (31 - __clz(below)) - 1) : run + lane;
          piece = ndigits(my_run) + 1;
        }
        uint32_t x = piece;   // inclusive scan of the pieces
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const uint32_t y = __shfl_up_sync(kFull, x, d);
          if (lane >= d) x += y;
        }
        if (W && mis) {
          put_digits(md + w.md_len + x - piece, my_run, piece - 1);
          md[w.md_len + x - 1] = rb;
        }
        w.md_len += __shfl_sync(kFull, x, 31);
        w.nm += __popc(m);
        w.uq += warp_sum(q);
        const uint32_t n_act = len - c < 32 ? len - c : 32;
        run = m ? (n_act - 1) - static_cast<uint32_t>(31 - __clz(m)) : run + n_act;
      }
      seq_pos += len;
      ref_off += len;
    } else if (t == 1) {
      if (static_cast<uint64_t>(seq_pos) + len > L) { w.bad = true; return w; }
      w.nm += static_cast<int32_t>(len);
      seq_pos += len;
    } else if (t == 2) {
      w.nm += static_cast<int32_t>(len);
      const uint32_t d = ndigits(run);
      if (W) {
        if (lane == 0) { put_digits(md + w.md_len, run, d); md[w.md_len + d] = '^'; }
        for (uint32_t j = lane; j < len; j += 32) md[w.md_len + d + 1 + j] = ref[ref_off + j];
      }
      w.md_len += d + 1 + len;
      run = 0;
      ref_off += len;
    } else if (t == 4) {
      if (static_cast<uint64_t>(seq_pos) + len > L) { w.bad = true; return w; }
      seq_pos += len;
    } else if (t == 3) {
      ref_off += len;
    }
  }
  const uint32_t d = ndigits(run);
  if (W && lane == 0) put_digits(md + w.md_len, run, d);
  w.md_len += d;
  return w;
}

}  // namespace frk

// Pass 1: records [off[i] - base, off[i + 1] - base) of `rec` (the host has checked their fixed fields, ref_id and
// position), edited in place by tag reversal and masking.  ctg_of_ref maps the header's @SQ index to a FASTA contig
// (-1: absent); ctg_off / ctg_len place the contigs in `genome`.  err: min of (first + i) << 8 | kErr*.
// counters[0] += bases masked.
__global__ void __launch_bounds__(kFilterThreads) filter_pass1_kernel(
    uint8_t* __restrict__ rec, const uint64_t* __restrict__ off, uint64_t base, uint32_t n, FilterCfg cfg,
    const int32_t* __restrict__ ctg_of_ref, const uint64_t* __restrict__ ctg_off, const uint64_t* __restrict__ ctg_len,
    const uint8_t* __restrict__ genome, uint64_t first, FRec* __restrict__ out, unsigned long long* err,
    unsigned long long* counters) {
  const int lane = threadIdx.x & 31;
  const uint32_t warps = gridDim.x * (blockDim.x / 32);
  for (uint32_t i = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32; i < n; i += warps) {
    uint8_t* r = rec + (off[i] - base);
    const uint64_t len = off[i + 1] - off[i];
    const uint32_t nc = rfilter::ld16(r + 12), L = rfilter::ld32(r + 16);
    const uint16_t flags = rfilter::ld16(r + 14);
    const uint64_t co = 32 + r[8], so = co + 4ull * nc, qo = so + (L + 1ull) / 2, ao = qo + L;
    uint8_t* aux = r + ao;
    const uint64_t an = len - ao;
    FRec f{};
    f.flags = flags;
    f.out_size = static_cast<uint32_t>(len);
    f.ref0 = ~0ull;
    if (cfg.reverse_tags && (flags & 0x10)) frk::reverse_tags(aux, an, lane);
    // masking (filter.rs:650-806) and, on the masked bases, compute_read_stats (filter.rs:565-590)
    const bool duplex = rfilter::is_duplex(aux, an);
    const rfilter::TagRef t0 = rfilter::find_tag(aux, an, duplex ? "ad" : "cd");
    const rfilter::TagRef t1 = rfilter::find_tag(aux, an, duplex ? "ae" : "ce");
    rfilter::TagRef t2, t3;
    const uint8_t *acp = nullptr, *bcp = nullptr;
    size_t acn = 0, bcn = 0;
    bool has_ac = false, has_bc = false;
    if (duplex) {
      t2 = rfilter::find_tag(aux, an, "bd");
      t3 = rfilter::find_tag(aux, an, "be");
      if (cfg.require_ss) {
        has_ac = rfilter::string_or_u8(rfilter::find_tag(aux, an, "ac"), &acp, &acn);
        has_bc = rfilter::string_or_u8(rfilter::find_tag(aux, an, "bc"), &bcp, &bcn);
      }
    }
    uint32_t masked = 0, n_count = 0;
    uint64_t qsum = 0;
    for (uint32_t j = lane; 2 * j < L; j += 32) {   // one sequence byte (two bases) per lane
      uint8_t sb = r[so + j];
      for (uint32_t h = 0; h < 2 && 2 * j + h < L; ++h) {
        const uint32_t b = 2 * j + h;
        const uint8_t code = h ? (sb & 0xF) : (sb >> 4);
        bool m;
        if (duplex) {
          const uint8_t x = (has_ac && b < acn) ? acp[b] : 'N', y = (has_bc && b < bcn) ? bcp[b] : 'N';
          m = code != 15 && rfilter::mask_duplex(r[qo + b], rfilter::array_u16(t0, b), rfilter::array_u16(t2, b),
                                                 rfilter::array_u16(t1, b), rfilter::array_u16(t3, b), cfg.cc, cfg.ab,
                                                 cfg.ba, cfg.min_bq, cfg.require_ss != 0, x, y);
        } else {
          m = rfilter::mask_simplex(r[qo + b], rfilter::array_u16(t0, b), rfilter::array_u16(t1, b), cfg.cc, cfg.min_bq);
        }
        if (m) {
          if (code != 15) ++masked;
          sb = h ? (sb | 0x0F) : (sb | 0xF0);
          r[qo + b] = 2;
        }
        if (m || code == 15) ++n_count;
        else qsum += r[qo + b];
      }
      r[so + j] = sb;
    }
    masked = frk::warp_sum(masked);
    n_count = frk::warp_sum(n_count);
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) qsum += __shfl_xor_sync(frk::kFull, qsum, s);
    __syncwarp();
    // regenerate_alignment_tags_raw (alignment_tags.rs:254-420)
    uint8_t e = kErrNone;
    if (cfg.regenerate) {
      size_t s0 = 0, e0 = 0;
      if (rfilter::find_tag(aux, an, "NM", &s0, &e0).type) { f.nm_s = ao + s0; f.nm_e = ao + e0; }
      if (rfilter::find_tag(aux, an, "UQ", &s0, &e0).type) { f.uq_s = ao + s0; f.uq_e = ao + e0; }
      if (rfilter::find_tag(aux, an, "MD", &s0, &e0).type) { f.md_s = ao + s0; f.md_e = ao + e0; }
      const int32_t ref_id = static_cast<int32_t>(rfilter::ld32(r));
      if (flags & 0x4) {
        f.action = kTagsRemoved;
        f.out_size -= (f.nm_e - f.nm_s) + (f.uq_e - f.uq_s) + (f.md_e - f.md_s);
      } else if (ref_id >= 0) {
        f.action = kTagsRegenerated;
        uint64_t span = 0;
        for (uint32_t k = lane; k < nc; k += 32) {
          const uint32_t op = rfilter::ld32(r + co + 4ull * k), t = op & 0xF;
          if (t == 0 || t == 2 || t == 3 || t == 7 || t == 8) span += op >> 4;
        }
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) span += __shfl_xor_sync(frk::kFull, span, s);
        if (span == 0) {
          f.md_len = 1;
        } else {
          const int32_t c = ctg_of_ref[ref_id];
          const uint64_t pos = static_cast<uint32_t>(rfilter::ld32(r + 4));
          if (c < 0) e = kErrContig;
          else if (pos + span > ctg_len[c]) e = kErrPastEnd;   // fetch_slice (reference.rs:291-318)
          else {
            f.ref0 = ctg_off[c] + pos;
            const frk::Walk w = frk::md_walk<false>(r, nc, co, so, qo, L, genome + f.ref0, nullptr, lane);
            if (w.bad) e = kErrCigar;
            f.nm = w.nm;
            f.uq = w.uq > 0x7fffffffu ? 0x7fffffffu : w.uq;
            f.md_len = w.md_len;
          }
        }
        // update_int_tag (tags.rs:729-750) for NM and UQ, then update_string_tag (:694-721) for MD
        uint8_t ty;
        if (!(f.nm_e - f.nm_s == 7 && (r[f.nm_s + 2] == 'i' || r[f.nm_s + 2] == 'I')))
          f.out_size += 3 + frk::int_size(f.nm, &ty) - (f.nm_e - f.nm_s);
        if (!(f.uq_e - f.uq_s == 7 && (r[f.uq_s + 2] == 'i' || r[f.uq_s + 2] == 'I')))
          f.out_size += 3 + frk::int_size(static_cast<int32_t>(f.uq), &ty) - (f.uq_e - f.uq_s);
        f.out_size += 4 + f.md_len - (f.md_e - f.md_s);
      }
    }
    if (lane == 0) {
      if (e != kErrNone) {
        atomicMin(err, ((first + i) << 8) | e);
      } else {
        int st = duplex ? rfilter::filter_duplex_read(aux, an, cfg.cc, cfg.ab, cfg.ba)
                        : rfilter::filter_read(aux, an, cfg.cc);
        if (st == FGB_FILTER_PASS) st = rfilter::no_call_gate(L, n_count, qsum, cfg.min_mean_q, cfg.max_no_call);
        f.pass = st == FGB_FILTER_PASS;
        if (masked) atomicAdd(counters, static_cast<unsigned long long>(masked));
      }
      out[i] = f;
    }
  }
}

// Template decision (commands/filter.rs:641-692, template_passes in crates/fgumi-consensus/src/filter.rs:371-395):
// template t holds output positions [tpl[t], tpl[t + 1]) of `order`.  By template: it passes when it has a primary
// record and all its primary records pass; a primary record follows it, a secondary or supplementary one is kept
// when it passes too.  Otherwise each record stands alone.  counters[1] += records kept.
__global__ void __launch_bounds__(kFilterThreads) filter_decide_kernel(FRec* __restrict__ fr,
                                                                      const uint32_t* __restrict__ order,
                                                                      const uint32_t* __restrict__ tpl, uint32_t n_tpl,
                                                                      bool by_template, unsigned long long* counters) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t kept = 0;
  if (t < n_tpl) {
    const uint32_t b = tpl[t], e = tpl[t + 1];
    bool has_primary = false, all_pass = true;
    for (uint32_t p = b; p < e; ++p) {
      const FRec& f = fr[order[p]];
      if (!(f.flags & 0x900)) { has_primary = true; all_pass = all_pass && f.pass; }
    }
    const bool tpass = has_primary && all_pass;
    for (uint32_t p = b; p < e; ++p) {
      FRec& f = fr[order[p]];
      const bool primary = !(f.flags & 0x900);
      f.keep = by_template ? (primary ? tpass : tpass && f.pass) : f.pass;
      kept += f.keep;
    }
  }
  kept = frk::warp_sum(kept);
  if ((threadIdx.x & 31) == 0 && kept) atomicAdd(counters + 1, static_cast<unsigned long long>(kept));
}

// Entry sizes in output order: ks[p] / rs[p] = 4 + out_size of the record at position p when it goes to the kept /
// rejects stream, else 0; ks[n] = rs[n] = 0 (the exclusive scans' totals).
__global__ void __launch_bounds__(kFilterThreads) filter_sizes_kernel(const FRec* __restrict__ fr,
                                                                     const uint32_t* __restrict__ order, uint32_t n,
                                                                     bool track_rejects, uint64_t* __restrict__ ks,
                                                                     uint64_t* __restrict__ rs) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p > n) return;
  uint64_t k = 0, j = 0;
  if (p < n) {
    const FRec& f = fr[order[p]];
    if (f.keep) k = 4ull + f.out_size;
    else if (track_rejects) j = 4ull + f.out_size;
  }
  ks[p] = k;
  rs[p] = j;
}

// Pass 2: the record at output position p written at kept + koff[p] or rejects + roff[p] as [u32 block_size][record],
// the tag edits where the reference's editor puts them: an NM / UQ entry of type i / I overwritten in place, any
// other removed and the tag appended in its smallest type; MD overwritten in place when its length is unchanged
// (keeping the entry's type byte), else spliced in place as Z, or appended; appended tags in the order NM, UQ, MD.
// Unmapped records lose their first NM, UQ and MD entries.
__global__ void __launch_bounds__(kFilterThreads) filter_pass2_kernel(
    const uint8_t* __restrict__ rec, const uint64_t* __restrict__ off, uint64_t base, uint32_t n,
    const FRec* __restrict__ fr, const uint32_t* __restrict__ order, const uint64_t* __restrict__ koff,
    const uint64_t* __restrict__ roff, bool track_rejects, const uint8_t* __restrict__ genome, uint8_t* kept,
    uint8_t* rejects) {
  const int lane = threadIdx.x & 31;
  const uint32_t warps = gridDim.x * (blockDim.x / 32);
  for (uint32_t p = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32; p < n; p += warps) {
    const uint32_t i = order[p];
    const FRec f = fr[i];
    if (!f.keep && !track_rejects) continue;
    uint8_t* dst = f.keep ? kept + koff[p] : rejects + roff[p];
    const uint8_t* r = rec + (off[i] - base);
    const uint64_t len = off[i + 1] - off[i];
    if (lane < 4) dst[lane] = static_cast<uint8_t>(f.out_size >> (8 * lane));
    uint8_t* o = dst + 4;
    if (f.action == kTagsKept) { frk::warp_copy(o, r, len, lane); continue; }
    const uint32_t nc = rfilter::ld16(r + 12), L = rfilter::ld32(r + 16);
    const uint64_t co = 32 + r[8], so = co + 4ull * nc, qo = so + (L + 1ull) / 2;
    const bool regen = f.action == kTagsRegenerated;
    const bool nm_in = regen && f.nm_e - f.nm_s == 7 && (r[f.nm_s + 2] == 'i' || r[f.nm_s + 2] == 'I');
    const bool uq_in = regen && f.uq_e - f.uq_s == 7 && (r[f.uq_s + 2] == 'i' || r[f.uq_s + 2] == 'I');
    auto write_md = [&](uint64_t at) {   // the MD value (f.md_len bytes) at o + at
      if (f.ref0 == ~0ull) { if (lane == 0) o[at] = '0'; }
      else frk::md_walk<true>(r, nc, co, so, qo, L, genome + f.ref0, o + at, lane);
    };
    auto write_int = [&](uint64_t at, const char* tag, int32_t v) {   // append_int_tag; returns the entry's size
      uint8_t ty;
      const uint32_t sz = frk::int_size(v, &ty);
      if (lane == 0) {
        o[at] = tag[0]; o[at + 1] = tag[1]; o[at + 2] = ty;
        for (uint32_t x = 0; x < sz; ++x) o[at + 3 + x] = static_cast<uint8_t>(static_cast<uint32_t>(v) >> (8 * x));
      }
      return 3 + sz;
    };
    // the edited entries in record order (an absent one has s == e and is skipped)
    uint64_t src = 0, w = 0;
    uint32_t done = 0;
    for (int k = 0; k < 3; ++k) {
      int which = -1;
      uint32_t s = 0xffffffffu, e = 0;
      if (!(done & 1) && f.nm_s != f.nm_e && f.nm_s < s) { which = 0; s = f.nm_s; e = f.nm_e; }
      if (!(done & 2) && f.uq_s != f.uq_e && f.uq_s < s) { which = 1; s = f.uq_s; e = f.uq_e; }
      if (!(done & 4) && f.md_s != f.md_e && f.md_s < s) { which = 2; s = f.md_s; e = f.md_e; }
      if (which < 0) break;
      done |= 1u << which;
      frk::warp_copy(o + w, r + src, s - src, lane);
      w += s - src;
      src = e;
      if (!regen) continue;                                  // remove_tag
      if (which == 2) {                                      // MD: same length in place, else spliced as Z
        const bool same = e - s - 4 == f.md_len;
        if (lane == 0) { o[w] = 'M'; o[w + 1] = 'D'; o[w + 2] = same ? r[s + 2] : 'Z'; }
        write_md(w + 3);
        if (lane == 0) o[w + 3 + f.md_len] = same ? r[s + 3 + f.md_len] : 0;   // update_string_tag keeps that byte
        w += 4 + f.md_len;
      } else if ((which == 0 && nm_in) || (which == 1 && uq_in)) {   // a 4-byte integer: overwritten in place
        const uint32_t v = which == 0 ? static_cast<uint32_t>(f.nm) : f.uq;
        if (lane < 3) o[w + lane] = r[s + lane];
        if (lane >= 3 && lane < 7) o[w + lane] = static_cast<uint8_t>(v >> (8 * (lane - 3)));
        w += 7;
      }
    }
    frk::warp_copy(o + w, r + src, len - src, lane);
    w += len - src;
    if (regen) {
      if (!nm_in) w += write_int(w, "NM", f.nm);
      if (!uq_in) w += write_int(w, "UQ", static_cast<int32_t>(f.uq));
      if (f.md_s == f.md_e) {
        if (lane == 0) { o[w] = 'M'; o[w + 1] = 'D'; o[w + 2] = 'Z'; }
        write_md(w + 3);
        if (lane == 0) o[w + 3 + f.md_len] = 0;
      }
    }
  }
}

}  // namespace fgb
