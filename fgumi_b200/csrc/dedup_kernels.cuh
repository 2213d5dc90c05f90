// Template scores of `fgumi dedup` (score_template, dedup.rs:230-249): per record the sum of its quality bytes capped
// at 15.  It is the one step of dedup that reads every quality byte, so it runs on the device while the host builds
// the UMI key tables.  One warp per record, grid-stride over records: byte loads up to the first 16-byte boundary of
// the quality slice, then uint4 loads, each word capped with __vminu4 and summed with __dp4a, the tail byte by byte,
// then a warp reduction.  Reads of up to 65 535 bases (and longer) need no special case: the warp strides the slice.
#pragma once
#include <cstdint>

namespace fgb {

constexpr int kScoreThreads = 256;   // 8 warps, one record each per step

// rec: the chunk's records back to back; off[0..n]: their offsets (no block_size prefix); every record is >= 32 bytes
// (checked on the host).  scores[i] for record i.
__global__ void __launch_bounds__(kScoreThreads) dedup_score_kernel(const uint8_t* __restrict__ rec,
                                                                    const uint64_t* __restrict__ off, uint32_t n,
                                                                    uint32_t* __restrict__ scores) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warps = static_cast<uint64_t>(gridDim.x) * (kScoreThreads / 32);
  for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * (kScoreThreads / 32) + (threadIdx.x >> 5); i < n; i += warps) {
    const uint64_t o = off[i], len = off[i + 1] - o;
    const uint8_t* r = rec + o;
    // qual_offset: 32 + l_read_name + 4 n_cigar + (l_seq + 1) / 2 (every lane reads the same fixed fields)
    const uint32_t l_read_name = r[8];
    const uint32_t n_cigar = static_cast<uint32_t>(r[12]) | (static_cast<uint32_t>(r[13]) << 8);
    const uint32_t l_seq = static_cast<uint32_t>(r[16]) | (static_cast<uint32_t>(r[17]) << 8) |
                           (static_cast<uint32_t>(r[18]) << 16) | (static_cast<uint32_t>(r[19]) << 24);
    const uint64_t qo = 32ull + l_read_name + 4ull * n_cigar + (static_cast<uint64_t>(l_seq) + 1) / 2;
    const uint64_t m = qo >= len ? 0 : min(static_cast<uint64_t>(l_seq), len - qo);   // clamped at the record's end
    const uint8_t* q = r + qo;
    uint32_t acc = 0;
    const uint64_t head = min(m, static_cast<uint64_t>((16 - (reinterpret_cast<uintptr_t>(q) & 15)) & 15));
    if (lane < head) acc += min(static_cast<uint32_t>(q[lane]), 15u);
    const uint4* body = reinterpret_cast<const uint4*>(q + head);
    const uint64_t words = (m - head) >> 4;
    for (uint64_t w = lane; w < words; w += 32) {
      const uint4 v = __ldg(body + w);
      acc = __dp4a(__vminu4(v.x, 0x0F0F0F0Fu), 0x01010101u, acc);
      acc = __dp4a(__vminu4(v.y, 0x0F0F0F0Fu), 0x01010101u, acc);
      acc = __dp4a(__vminu4(v.z, 0x0F0F0F0Fu), 0x01010101u, acc);
      acc = __dp4a(__vminu4(v.w, 0x0F0F0F0Fu), 0x01010101u, acc);
    }
    const uint64_t tail_at = head + (words << 4);
    if (tail_at + lane < m) acc += min(static_cast<uint32_t>(q[tail_at + lane]), 15u);
    acc = __reduce_add_sync(0xFFFFFFFFu, acc);
    if (lane == 0) scores[i] = acc;
  }
}

}  // namespace fgb
