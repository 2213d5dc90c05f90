// `fgumi sort` on the device: the key kernels, the word gather between LSD passes and the record gather.  The stable
// sort itself is CUB's radix sort, one pass per key word that varies (driven by host/sort_host.cpp through the
// launchers in capi.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "sort_keys.h"

namespace fgb {

constexpr int kSortThreads = 256;

// One record per thread: its key words (W = 1: coordinate, W = 5: template-coordinate) as SoA (word w of record i at
// keys[w * n + i]), its size, and the AND / OR of every word over the run (and_or[2w] / and_or[2w + 1]), from which
// the host skips constant words and narrows the others to their varying bits.  Records are [base + off[i], base + off[i + 1]) of `rec` minus `base`; the host
// has checked that each holds its 32-byte fixed part.
template <int W>
__global__ void __launch_bounds__(kSortThreads) sort_key_kernel(const uint8_t* __restrict__ rec,
                                                                const uint64_t* __restrict__ off, uint64_t base,
                                                                uint32_t n, sortk::Ctx ctx,
                                                                uint64_t* __restrict__ keys,
                                                                uint32_t* __restrict__ size,
                                                                unsigned long long* __restrict__ and_or) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  uint64_t k[sortk::kWords];
  uint64_t a[W], o[W];
  if (i < n) {
    const uint64_t b = off[i], e = off[i + 1];
    if (W == 1) k[0] = sortk::coordinate_key(rec + (b - base));   // the coordinate order's one word
    else sortk::template_key(rec + (b - base), e - b, ctx, k);
    size[i] = static_cast<uint32_t>(e - b);
#pragma unroll
    for (int w = 0; w < W; ++w) { keys[static_cast<uint64_t>(w) * n + i] = k[w]; a[w] = k[w]; o[w] = k[w]; }
  } else {
#pragma unroll
    for (int w = 0; w < W; ++w) { a[w] = ~0ull; o[w] = 0; }
  }
#pragma unroll
  for (int w = 0; w < W; ++w) {
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
      a[w] &= __shfl_xor_sync(0xffffffffu, a[w], s);
      o[w] |= __shfl_xor_sync(0xffffffffu, o[w], s);
    }
  }
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int w = 0; w < W; ++w) {
      atomicAnd(and_or + 2 * w, static_cast<unsigned long long>(a[w]));
      atomicOr(and_or + 2 * w + 1, static_cast<unsigned long long>(o[w]));
    }
  }
}

// Queryname order, one record per thread: its W name words and its last word (sort_keys.h NameEncoder) as SoA
// (keys[w * n + i], w = 0..W), its size, and the AND / OR of each of the W + 1 words over the run, as sort_key_kernel.
// The encoder streams the name from the record into one word at a time; the host has chosen W for the run's longest
// name, so every thread runs the same W + 1 steps and the warp reductions stay converged.
__global__ void __launch_bounds__(kSortThreads) sort_name_key_kernel(const uint8_t* __restrict__ rec,
                                                                     const uint64_t* __restrict__ off, uint64_t base,
                                                                     uint32_t n, bool natural, int W,
                                                                     uint64_t* __restrict__ keys,
                                                                     uint32_t* __restrict__ size,
                                                                     unsigned long long* __restrict__ and_or) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = i < n;
  const uint8_t* r = nullptr;
  sortk::NameEncoder enc;
  if (live) {
    const uint64_t b = off[i], e = off[i + 1];
    r = rec + (b - base);
    enc.init(r, e - b, natural);
    size[i] = static_cast<uint32_t>(e - b);
  } else {
    enc.init_empty();
  }
  for (int w = 0; w <= W; ++w) {
    uint64_t a = ~0ull, o = 0;
    if (live) {
      const uint64_t k = w < W ? enc.word() : sortk::name_last_word(enc, r);
      keys[static_cast<uint64_t>(w) * n + i] = k;
      a = o = k;
    }
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
      a &= __shfl_xor_sync(0xffffffffu, a, s);
      o |= __shfl_xor_sync(0xffffffffu, o, s);
    }
    if ((threadIdx.x & 31) == 0) {
      atomicAnd(and_or + 2 * w, static_cast<unsigned long long>(a));
      atomicOr(and_or + 2 * w + 1, static_cast<unsigned long long>(o));
    }
  }
}

// Between LSD passes: the next word in the current order (dst[i] = word[perm[i]]); also iota (perm == nullptr).
__global__ void __launch_bounds__(kSortThreads) sort_word_gather_kernel(const uint64_t* __restrict__ word,
                                                                        const uint32_t* __restrict__ perm,
                                                                        uint32_t n, uint64_t* __restrict__ dst,
                                                                        uint32_t* __restrict__ iota) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (iota) iota[i] = i;
  else dst[i] = word[perm[i]];
}

// Several runs: the keys in sorted order, row-major (rows[i * W + w] = word w of record perm[i]), which the host merge
// then reads front to back.
__global__ void __launch_bounds__(kSortThreads) sort_key_rows_kernel(const uint64_t* __restrict__ keys,
                                                                     const uint32_t* __restrict__ perm, uint32_t n,
                                                                     int words, uint64_t* __restrict__ rows) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t j = perm[i];
  for (int w = 0; w < words; ++w) rows[static_cast<uint64_t>(i) * words + w] = keys[static_cast<uint64_t>(w) * n + j];
}

// The output size of each record in sorted order: 4 (block_size) + its length; the host scans it into offsets.
__global__ void __launch_bounds__(kSortThreads) sort_out_size_kernel(const uint32_t* __restrict__ size,
                                                                     const uint32_t* __restrict__ perm, uint32_t n,
                                                                     uint64_t* __restrict__ out_size) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out_size[i] = 4ull + size[perm[i]];
}

// One warp per output record: [u32 block_size][record] at out + out_off[i] from record perm[i].  Output words wholly
// inside the record's span are written as aligned u32 (each assembled from two aligned source words with a funnel
// shift); the bytes at either end are written one by one, since the neighbouring records' warps own the rest of those
// words.  The source may be read up to 4 bytes past a record: the host pads the run's record buffer.
__global__ void __launch_bounds__(kSortThreads) sort_gather_kernel(const uint8_t* __restrict__ rec,
                                                                   const uint64_t* __restrict__ off, uint64_t base,
                                                                   const uint32_t* __restrict__ perm,
                                                                   const uint64_t* __restrict__ out_off, uint32_t n,
                                                                   uint8_t* __restrict__ out) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warps = (static_cast<uint64_t>(gridDim.x) * blockDim.x) >> 5;
  for (uint64_t i = (static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
    const uint32_t j = perm[i];
    const uint64_t s0 = off[j] - base, len = off[j + 1] - off[j];
    const uint64_t d0 = out_off[i], d1 = d0 + 4 + len;
    auto byte_at = [&](uint64_t x) -> uint8_t {   // the output byte at address x in [d0, d1)
      const uint64_t q = x - d0;
      return q < 4 ? static_cast<uint8_t>(len >> (8 * q)) : rec[s0 + q - 4];
    };
    const uint64_t wa = (d0 + 4 + 3) & ~3ull, we = d1 & ~3ull;   // aligned words wholly inside the record's bytes
    if (wa >= we) {
      for (uint64_t x = d0 + lane; x < d1; x += 32) out[x] = byte_at(x);
      continue;
    }
    for (uint64_t x = d0 + lane; x < wa; x += 32) out[x] = byte_at(x);
    for (uint64_t x = we + lane; x < d1; x += 32) out[x] = byte_at(x);
    const uint64_t sa = s0 + (wa - d0 - 4);                      // source address of the first aligned output word
    const uint32_t* src = reinterpret_cast<const uint32_t*>(rec + (sa & ~3ull));
    const uint32_t sh = static_cast<uint32_t>(sa & 3) * 8;
    uint32_t* dst = reinterpret_cast<uint32_t*>(out + wa);
    const uint64_t nw = (we - wa) >> 2;
    for (uint64_t w = lane; w < nw; w += 32) dst[w] = __funnelshift_r(__ldg(src + w), __ldg(src + w + 1), sh);
  }
}

}  // namespace fgb
