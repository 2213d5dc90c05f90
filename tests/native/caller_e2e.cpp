// Test harness (not product code): the product's record-level callers end to end on the CPU -- host prep,
// flush, record assembly, filter -- with tests/native/mock_engine.cpp standing in for the GPU engine.
// usage: caller_e2e <groups file> <threads> <variant> <output file>
// variant 0: plain, 1: with the filter stage, 2: simplex with min_reads = 2.  Prints the count and every statistic.
// Built and driven by tests/test_caller_planning.py::test_callers_end_to_end_on_a_mock_engine.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../include/fgumi_b200.h"

int main(int argc, char** argv) {
  if (argc < 5) return 2;
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  const int threads = std::atoi(argv[2]), variant = std::atoi(argv[3]);
  uint32_t mode = 0, n_groups = 0;
  if (std::fread(&mode, 4, 1, f) != 1 || std::fread(&n_groups, 4, 1, f) != 1) return 2;
  std::vector<uint8_t> blob; std::vector<uint64_t> off{0}, grp{0};
  for (uint32_t g = 0; g < n_groups; ++g) {
    uint32_t nr = 0;
    if (std::fread(&nr, 4, 1, f) != 1) return 2;
    for (uint32_t r = 0; r < nr; ++r) {
      uint32_t n = 0;
      if (std::fread(&n, 4, 1, f) != 1) return 2;
      const size_t o = blob.size(); blob.resize(o + n);
      if (n && std::fread(blob.data() + o, 1, n, f) != n) return 2;
      off.push_back(blob.size());
    }
    grp.push_back(off.size() - 1);
  }
  std::fclose(f);
  fgb_caller_options o; std::memset(&o, 0, sizeof(o));
  o.mode = static_cast<uint8_t>(mode); o.error_rate_pre_umi = 45; o.error_rate_post_umi = 40; o.min_input_base_quality = 10;
  o.min_consensus_base_quality = 2; o.produce_per_base_tags = 1; o.min_reads = 1; o.min_xy_reads = 1; o.min_yx_reads = 0;
  o.tag[0] = 'M'; o.tag[1] = 'I'; o.cell_tag[0] = 'C'; o.cell_tag[1] = 'B';
  o.read_name_prefix = mode == 2 ? "codec" : "fgumi"; o.read_group_id = mode == 2 ? "RG1" : "A";
  o.min_duplex_length = 1; o.n_threads = static_cast<uint32_t>(threads);
  o.consensus_call_overlapping_bases = mode == 0 ? 1 : 0;
  o.zero_copy_records = 1;                       // used when the mock engine reports page-locked memory (FGB_MOCK_PINNED)
  o.codec.single_strand_qual = -1; o.codec.outer_bases_qual = -1; o.codec.outer_bases_length = 5;
  o.codec.max_duplex_disagreements = 0xFFFFFFFFu; o.codec.max_duplex_disagreement_rate = 1.0;
  if (variant == 2) o.min_reads = 2;             // simplex, every group one pair: a batch the group rules reject whole
  if (variant == 1 && mode == 0) {
    o.filter_enabled = 1;
    o.filter.min_reads = 1; o.filter.max_read_error_rate = 0.2; o.filter.max_base_error_rate = 0.3;
    o.filter.min_base_quality = 10; o.filter.min_mean_base_quality = -1.0; o.filter.max_no_call_fraction = 0.5;
  }
  if (variant == 1 && mode == 1) {
    o.filter_enabled = 1; o.min_reads = 1; o.min_xy_reads = 1; o.min_yx_reads = 1;
    fgb_duplex_filter_params& d = o.duplex_filter;
    d.cc.min_reads = 3; d.ab_min_reads = 2; d.ba_min_reads = 1;
    d.cc.max_read_error_rate = 0.05; d.ab_max_read_error_rate = 0.05; d.ba_max_read_error_rate = 0.1;
    d.cc.max_base_error_rate = 0.2; d.ab_max_base_error_rate = 0.1; d.ba_max_base_error_rate = 0.3;
    d.cc.min_base_quality = 20; d.cc.min_mean_base_quality = -1.0; d.cc.max_no_call_fraction = 0.3;
  }
  fgb_caller* c = nullptr;
  if (fgb_caller_create(0, &o, &c) != FGB_OK) return 3;
  FILE* out = std::fopen(argv[4], "wb");
  if (!out) return 2;
  unsigned long long total = 0;
  for (int rep = 0; rep < 2; ++rep) {                 // two flushes: buffers that outlive a flush are reused
    if (fgb_caller_add_groups(c, blob.data(), off.data(), grp.data(), n_groups) != FGB_OK) return 4;
    const uint8_t* data; uint64_t len, count;
    fgb_status st = fgb_caller_flush(c, &data, &len, &count);
    if (st != FGB_OK) { char buf[256]; fgb_caller_last_error(c, buf, sizeof buf); std::fprintf(stderr, "flush: %d %s\n", st, buf); return 5; }
    if (rep == 0) { if (len && std::fwrite(data, 1, len, out) != len) return 2; }
    total += count;
  }
  std::fclose(out);
  uint64_t stats[FGB_NSTATS];
  fgb_caller_stats(c, stats);
  std::printf("ok count %llu", total);
  for (int i = 0; i < FGB_NSTATS; ++i) std::printf(" %llu", (unsigned long long)stats[i]);
  std::printf("\n");
  fgb_caller_destroy(c);
  return 0;
}
