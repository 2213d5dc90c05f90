// The device half of fgb_sort_records: launchers of sort_kernels.cuh and CUB, defined in capi.cu (which owns the
// handle and compiles the kernels), called by the host driver in sort_host.cpp.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

#include "../sort_keys.h"

namespace fgb {
namespace sortdev {

// Key words (SoA, `words` of them: 1 for coordinate, 5 for template-coordinate), record sizes and the AND / OR of each
// word over the run, which `and_or` must hold as (~0, 0) pairs on entry.
cudaError_t keys(const uint8_t* rec, const uint64_t* off, uint64_t base, uint32_t n, const sortk::Ctx& ctx, int words,
                 uint64_t* keys, uint32_t* size, unsigned long long* and_or, cudaStream_t s);
// Queryname order: name_words + 1 key words (SoA), sizes and AND / OR as keys()
cudaError_t name_keys(const uint8_t* rec, const uint64_t* off, uint64_t base, uint32_t n, bool natural, int name_words,
                      uint64_t* keys, uint32_t* size, unsigned long long* and_or, cudaStream_t s);
// dst[i] = word[perm[i]]
cudaError_t word_gather(const uint64_t* word, const uint32_t* perm, uint32_t n, uint64_t* dst, cudaStream_t s);
cudaError_t iota(uint32_t* v, uint32_t n, cudaStream_t s);
// rows[i * words + w] = keys[w * n + perm[i]]: a run's keys in sorted order for the host merge
cudaError_t key_rows(const uint64_t* keys, const uint32_t* perm, uint32_t n, int words, uint64_t* rows, cudaStream_t s);
// One stable LSD pass over bits [begin, end) of the keys (CUB DeviceRadixSort::SortPairs); temp == nullptr sizes it.
cudaError_t radix_pass(void* temp, size_t* temp_bytes, const uint64_t* kin, uint64_t* kout, const uint32_t* vin,
                       uint32_t* vout, uint32_t n, int begin, int end, cudaStream_t s);
// out_off[0..n]: offsets of the [u32 block_size][record] entries of the records in perm order; out_size (n + 1) is
// scratch.  temp == nullptr sizes it.
cudaError_t out_offsets(void* temp, size_t* temp_bytes, const uint32_t* size, const uint32_t* perm, uint32_t n,
                        uint64_t* out_size, uint64_t* out_off, cudaStream_t s);
cudaError_t gather(const uint8_t* rec, const uint64_t* off, uint64_t base, const uint32_t* perm,
                   const uint64_t* out_off, uint32_t n, uint8_t* out, int sm_count, cudaStream_t s);

}  // namespace sortdev
}  // namespace fgb
