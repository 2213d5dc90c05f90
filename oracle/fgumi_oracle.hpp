// TEST INFRASTRUCTURE — NOT PRODUCT CODE.
//
// CPU restatement ("oracle") of the fgumi 0.2.0 (@4271c26e) UMI-consensus hot path.
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
// load this.  The product (fgumi_b200/) never includes, links or calls anything in oracle/.
//
// The reference is Rust and cannot be compiled in this image (no rustc/cargo), so this is a
// line-by-line restatement in C++17, f64 throughout, glibc libm for exp/log/log1p/expm1 (the
// same libm Rust's std calls on x86_64-unknown-linux-gnu).  Build with -ffp-contract=off: Rust
// never contracts a*b+c into an FMA.
//
// Parity pinning: every known-answer test the reference holds for this path (SURVEY.md §8c) is
// reproduced in tests/test_oracle_kat.py.  Record-level byte parity against the Rust binary is
// "parity unpinned" (the reference has no golden outputs and cannot be run here); see DESIGN.md.
//
// All `file:line` citations are relative to the fgumi 0.2.0 source tree.
#pragma once
#include <cstddef>
#include <cstdint>
#include <vector>

namespace fgoracle {

// ---- phred.rs ------------------------------------------------------------------------------
constexpr uint8_t MIN_PHRED = 2;        // fgumi-dna/src/lib.rs:26
constexpr uint8_t MAX_PHRED = 93;       // phred.rs:28
constexpr uint8_t NO_CALL_BASE = 'N';   // fgumi-dna/src/lib.rs:20
constexpr uint8_t NO_CALL_BASE_LOWER = 'n';  // fgumi-dna/src/lib.rs:23

double phred_to_ln_error_prob(uint8_t phred);          // phred.rs:66-68
double phred_to_ln_correct_prob(uint8_t phred);        // phred.rs:89-92
uint8_t ln_prob_to_phred(double ln_prob);              // phred.rs:119-135
double log1pexp(double x);                             // phred.rs:148-158
double ln_one_minus_exp(double x);                     // phred.rs:168-182
double ln_a_minus_b(double a, double b);               // phred.rs:188-198
double ln_error_prob_two_trials(double p1, double p2); // phred.rs:231-251
double ln_sum_exp(double a, double b);                 // phred.rs:274-285
double ln_sum_exp_array(const double* v, size_t n);    // phred.rs:307-330
inline double ln_not(double x) { return ln_one_minus_exp(x); }  // phred.rs:343-345

// ---- base_builder.rs -----------------------------------------------------------------------
// ConsensusBaseBuilder (base_builder.rs:225-485).
class ConsensusBaseBuilder {
 public:
  ConsensusBaseBuilder(uint8_t error_rate_pre_umi, uint8_t error_rate_post_umi);  // :252-278
  void reset();                               // :281-285
  void add(uint8_t base, uint8_t qual);       // :295-327
  void call(uint8_t* base, uint8_t* qual) const;  // :391-458
  uint16_t contributions() const;             // :464-466
  uint16_t observations_for_base(uint8_t base) const;  // :476-479

  double likelihoods[4];
  double compensations[4];
  uint16_t observations[4];
  double adjusted_correct_table[94];
  double adjusted_error_per_alt[94];
  double ln_error_pre_umi;

 private:
  bool try_unanimous_fast_path(uint8_t* base, uint8_t* qual) const;  // :338-379
};

// ---- vanilla_caller.rs ---------------------------------------------------------------------
struct VanillaOptions {            // VanillaUmiConsensusOptions, vanilla_caller.rs:284-341
  uint8_t error_rate_pre_umi = 45;
  uint8_t error_rate_post_umi = 40;
  uint8_t min_input_base_quality = 10;
  size_t min_reads = 2;
  bool produce_per_base_tags = true;
  bool trim = false;
  uint8_t min_consensus_base_quality = 40;
};

// compute_single_input_consensus_quals, vanilla_caller.rs:463-482
std::vector<uint8_t> compute_single_input_consensus_quals(uint8_t pre, uint8_t post);

// One already-prepared SourceRead row (vanilla_caller.rs:129-146: bases/quals only).
struct SourceRow {
  const uint8_t* bases;
  const uint8_t* quals;
  size_t len;
};

struct ConsensusColumns {   // ConsensusResult, vanilla_caller.rs:32
  std::vector<uint8_t> bases, quals;
  std::vector<uint16_t> depths, errors;
};

// create_consensus_from_source_reads, vanilla_caller.rs:1260-1358.  `builder` and
// `single_input_quals` are the caller's cached members (vanilla_caller.rs:420-454).
// Returns false for the `bail!` on empty input (:1264-1266).
bool create_consensus_from_source_reads(const SourceRow* reads, size_t n_reads,
                                        const VanillaOptions& opt, ConsensusBaseBuilder& builder,
                                        const std::vector<uint8_t>& single_input_quals,
                                        ConsensusColumns* out);

// ---- duplex_caller.rs ----------------------------------------------------------------------
// The (Some(a), Some(b)) arm of DuplexConsensusCaller::duplex_consensus, duplex_caller.rs:883-970,
// with methylation disabled (MethylationMode::Disabled, lib.rs:41-45).  `len` = min(len_a,len_b)
// (:846-849).  When `source` is non-null errors follow the exact branch (:943-951), else the
// approximate branch (:952-967).
void duplex_combine(const uint8_t* a_bases, const uint8_t* a_quals, const uint16_t* a_depths,
                    const uint16_t* a_errors, const uint8_t* b_bases, const uint8_t* b_quals,
                    const uint16_t* b_depths, const uint16_t* b_errors, size_t len,
                    const SourceRow* source, size_t n_source, uint8_t* out_bases,
                    uint8_t* out_quals, uint16_t* out_errors);

// All four arms of duplex_consensus (duplex_caller.rs:838-1015): returns 0 = both strands combined
// (output length min(la, lb)), 1 = AB only (B has no depth inside the truncated region; output is
// A at its FULL length, :855-868), 2 = BA only (:869-882), 3 = neither (:1013).  *out_len gets the
// output length.  out_* must hold max(la, lb) elements.
int duplex_consensus_arms(const uint8_t* a_bases, const uint8_t* a_quals, const uint16_t* a_depths,
                          const uint16_t* a_errors, size_t la, const uint8_t* b_bases,
                          const uint8_t* b_quals, const uint16_t* b_depths,
                          const uint16_t* b_errors, size_t lb, const SourceRow* source,
                          size_t n_source, uint8_t* out_bases, uint8_t* out_quals,
                          uint16_t* out_errors, size_t* out_len);

// ---- codec_caller.rs -----------------------------------------------------------------------
struct CodecCombineResult {
  size_t duplex_bases_count = 0;     // codec_caller.rs:1046
  size_t duplex_disagreements = 0;   // codec_caller.rs:1045
};
// build_duplex_consensus_from_padded position loop, codec_caller.rs:1048-1152 (gate at
// :1155-1166 is left to the caller, which gets the two counters back).
CodecCombineResult codec_combine_padded(const uint8_t* a_bases, const uint8_t* a_quals,
                                        const uint16_t* a_depths, const uint16_t* a_errors,
                                        const uint8_t* b_bases, const uint8_t* b_quals,
                                        const uint16_t* b_depths, const uint16_t* b_errors,
                                        size_t len, uint8_t* out_bases, uint8_t* out_quals,
                                        uint16_t* out_depths, uint16_t* out_errors);

// mask_consensus_quals_query_based, codec_caller.rs:1183-1212.  ss_qual/outer_qual < 0 = None.
void codec_mask_quals(const uint8_t* cons_bases, uint8_t* cons_quals, size_t len,
                      const uint8_t* padded_r1_bases, const uint8_t* padded_r2_bases,
                      int ss_qual, int outer_qual, size_t outer_len);

// fgumi-dna/src/dna.rs:30-40 complement_base and :58-60 reverse_complement
uint8_t complement_base(uint8_t b);

// One single-strand consensus (codec_caller.rs SingleStrandConsensus: bases/quals/depths/errors).
struct SsColumns {
  std::vector<uint8_t> bases, quals;
  std::vector<uint16_t> depths, errors;
};
// reverse_complement_ss, codec_caller.rs:507-520
SsColumns reverse_complement_ss(const SsColumns& ss);
// pad_consensus, codec_caller.rs:980-1023
SsColumns pad_consensus(const SsColumns& ss, size_t new_length, bool pad_left);

struct CodecJobResult {
  SsColumns consensus;            // after masking and final re-orientation
  size_t duplex_bases_count = 0;
  size_t duplex_disagreements = 0;
  int status = 0;                 // 0 ok, 1 "High duplex disagreement" (:1160), 2 "... rate" (:1163)
};
// The orient/pad/combine/mask/re-orient tail of consensus_reads_raw, codec_caller.rs:721-784.
CodecJobResult codec_job(const SsColumns& ss_r1, const SsColumns& ss_r2, bool r1_is_negative,
                         bool r2_is_negative, size_t consensus_length, int ss_qual, int outer_qual,
                         size_t outer_len, size_t max_duplex_disagreements,
                         double max_duplex_disagreement_rate);

}  // namespace fgoracle
