// UMI graph edges for fgb_umi_assign (include/fgumi_b200.h).  Per unique key of a call, the device emits its capture
// list as CSR, ascending: edit gets undirected edges, adjacency and paired only the edges that satisfy the count
// rule count[j] <= count[i] / 2 + 1 (assigner.rs:1193-1247), so the host's BFS reads the lists as they are.
//
// Two comparators (umi_accept):
//   2-bit  one u64 BitEnc per key: a position differs when either of its two bits does -> popcount.  Adjacency
//          (both rule families), unmapped edit, unmapped paired.  The unmapped rules' edge set is what
//          discover_edges_parallel_k returns (parallel_assigner.rs:180-242): distance exactly 1 for k = 1, 0..=k
//          otherwise, and an edge (a, b), a < b, only where b is the last key of its BitEnc (FGB_UMI_KEY_LAST).
//   bytes  byte Hamming on keys of equal length, optionally against the query's reversed paired form as well
//          (matches_paired, assigner.rs:1773-1783).  Mapped edit and mapped paired.
// Two forms, selected by the host from the call's size and k (capi.cu, umi_enum_min_keys):
//   all-pairs   umi_pairs_kernel: many calls per launch, one CTA per 128 queries of a call, the call's keys
//               staged through shared memory in tiles; a count pass, a scan, a fill pass.
//   enumeration umi_enum_kernel (2-bit, k <= 2): the call's BitEncs radix-sorted (CUB), each thread generates
//               its key's variants (3L for distance 1, 9L(L-1)/2 for distance 2) and binary-searches them.
#pragma once

#include <cstdint>

#include "../../include/fgumi_b200.h"

namespace fgb {

struct UmiCmp {
  uint32_t k;
  uint8_t directed;   // adjacency / paired: count rule
  uint8_t bytes;      // bytes comparator
  uint8_t reverse;    // bytes: also the query's reversed paired form
  uint8_t zero_ok;    // 2-bit: distance 0 (a duplicate BitEnc) counts unless k == 1
};

struct UmiWork {      // one CTA of the all-pairs form
  uint64_t key_base;  // first key of the call in the batch's key array (and CSR row)
  uint32_t n_keys;
  uint32_t q_begin;   // first query (local) of this CTA
};

struct UmiQuery {     // the query key's fields the comparators read, in registers
  uint64_t bits, str_off;
  uint32_t str_len, count, dash, len, flags;
};

__device__ __forceinline__ UmiQuery umi_query(const fgb_umi_key* k) {
  return UmiQuery{k->bits, k->str_off, k->str_len, k->count, k->dash, k->len, k->flags};
}

constexpr int kUmiThreads = 128;
constexpr int kUmiTile = 128;

__device__ __forceinline__ uint32_t umi_hamming2(uint64_t a, uint64_t b) {
  const uint64_t d = a ^ b;
  return __popcll(((d & 0xAAAAAAAAAAAAAAAAull) >> 1) | (d & 0x5555555555555555ull));
}

// Byte t of the reversed paired form "second-first" of s (dash at `dash`).
__device__ __forceinline__ uint8_t umi_rev_byte(const uint8_t* s, uint32_t len, uint32_t dash, uint32_t t) {
  const uint32_t b = len - dash - 1;   // length of the second part
  return t < b ? s[dash + 1 + t] : (t == b ? static_cast<uint8_t>('-') : s[t - b - 1]);
}

__device__ __forceinline__ bool umi_accept(const UmiQuery& qi, const fgb_umi_key& kj, uint32_t i, uint32_t j,
                                           const uint8_t* blob, const UmiCmp& p) {
  if (i == j) return false;
  if (p.bytes) {
    if (qi.str_len != kj.str_len) return false;
    const uint8_t* a = blob + qi.str_off;
    const uint8_t* b = blob + kj.str_off;
    uint32_t d = 0;
    for (uint32_t t = 0; t < qi.str_len && d <= p.k; ++t) d += a[t] != b[t];
    bool ok = d <= p.k;
    if (!ok && p.reverse) {
      d = 0;
      for (uint32_t t = 0; t < qi.str_len && d <= p.k; ++t) d += umi_rev_byte(a, qi.str_len, qi.dash, t) != b[t];
      ok = d <= p.k;
    }
    if (!ok) return false;
  } else {
    if (qi.len != kj.len) return false;
    const uint32_t d = umi_hamming2(qi.bits, kj.bits);
    if (d > p.k || (d == 0 && !p.zero_ok)) return false;
    if (!(i < j ? (kj.flags & FGB_UMI_KEY_LAST) : (qi.flags & FGB_UMI_KEY_LAST))) return false;
  }
  return !p.directed || kj.count <= qi.count / 2u + 1u;
}

// kFill = false: deg[row] = capture-list length; true: the lists at off[row].
template <bool kFill>
__global__ void __maxnreg__(64) umi_pairs_kernel(const UmiWork* __restrict__ work,
                                                               const fgb_umi_key* __restrict__ keys,
                                                               const uint8_t* __restrict__ blob, UmiCmp p,
                                                               uint64_t* __restrict__ deg,
                                                               const uint64_t* __restrict__ off,
                                                               uint32_t* __restrict__ edges) {
  __shared__ fgb_umi_key tile[kUmiTile];
  const UmiWork w = work[blockIdx.x];
  const uint32_t i = w.q_begin + threadIdx.x;
  const bool live = i < w.n_keys;
  UmiQuery qi{};
  if (live) qi = umi_query(keys + w.key_base + i);
  uint32_t n = 0;
  uint64_t out = 0;
  if (kFill && live) out = off[w.key_base + i];
  for (uint32_t t0 = 0; t0 < w.n_keys; t0 += kUmiTile) {
    const uint32_t m = min(static_cast<uint32_t>(kUmiTile), w.n_keys - t0);
    __syncthreads();
    for (uint32_t x = threadIdx.x; x < m; x += kUmiThreads) tile[x] = keys[w.key_base + t0 + x];
    __syncthreads();
    if (!live) continue;
    for (uint32_t x = 0; x < m; ++x) {
      if (umi_accept(qi, tile[x], i, t0 + x, blob, p)) {
        if (kFill) edges[out + n] = t0 + x;
        ++n;
      }
    }
  }
  if (!kFill && live) deg[w.key_base + i] = n;
}

// Keys of the sorted call whose BitEnc is v, through the comparator: appended to row[n..] (fill pass) and counted.
template <bool kFill>
__device__ __forceinline__ uint32_t umi_probe(uint64_t v, const UmiQuery& qi, uint32_t i,
                                              const fgb_umi_key* __restrict__ keys, uint32_t n_keys,
                                              const uint64_t* __restrict__ sorted_bits,
                                              const uint32_t* __restrict__ sorted_idx, const UmiCmp& p,
                                              uint32_t* __restrict__ row, uint32_t n) {
  uint32_t lo = 0, hi = n_keys;   // first sorted_bits >= v
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (sorted_bits[mid] < v) lo = mid + 1; else hi = mid;
  }
  for (; lo < n_keys && sorted_bits[lo] == v; ++lo) {
    const uint32_t j = sorted_idx[lo];
    if (umi_accept(qi, keys[j], i, j, nullptr, p)) {
      if (kFill) row[n] = j;
      ++n;
    }
  }
  return n;
}

// One call, thread per query.  sorted_bits / sorted_idx: the call's BitEncs and local indices sorted by BitEnc.
template <bool kFill>
__global__ void __maxnreg__(64) umi_enum_kernel(const fgb_umi_key* __restrict__ keys, uint32_t n_keys,
                                                              const uint64_t* __restrict__ sorted_bits,
                                                              const uint32_t* __restrict__ sorted_idx, UmiCmp p,
                                                              uint64_t* __restrict__ deg,
                                                              const uint64_t* __restrict__ off,
                                                              uint32_t* __restrict__ edges) {
  const uint32_t i = blockIdx.x * kUmiThreads + threadIdx.x;
  if (i >= n_keys) return;
  const UmiQuery qi = umi_query(keys + i);
  uint32_t* row = kFill ? edges + off[i] : nullptr;
  uint32_t n = 0;
  if (p.zero_ok) n = umi_probe<kFill>(qi.bits, qi, i, keys, n_keys, sorted_bits, sorted_idx, p, row, n);
  for (uint32_t a = 0; a < qi.len && p.k >= 1; ++a)
    for (uint64_t s = 1; s < 4; ++s) {
      const uint64_t va = qi.bits ^ (s << (2 * a));
      n = umi_probe<kFill>(va, qi, i, keys, n_keys, sorted_bits, sorted_idx, p, row, n);
      if (p.k >= 2)
        for (uint32_t b = a + 1; b < qi.len; ++b)
          for (uint64_t r = 1; r < 4; ++r)
            n = umi_probe<kFill>(va ^ (r << (2 * b)), qi, i, keys, n_keys, sorted_bits, sorted_idx, p, row, n);
    }
  if (!kFill) {
    deg[i] = n;
    return;
  }
  for (uint32_t x = 1; x < n; ++x) {   // the list in ascending order (lists are short: at most 1 + 3L + 9L(L-1)/2)
    const uint32_t v = row[x];
    uint32_t y = x;
    for (; y > 0 && row[y - 1] > v; --y) row[y] = row[y - 1];
    row[y] = v;
  }
}

}  // namespace fgb
