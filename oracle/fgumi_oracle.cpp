// TEST INFRASTRUCTURE — NOT PRODUCT CODE.  See fgumi_oracle.hpp for the rules.
// CPU restatement of fgumi-consensus {phred,base_builder,vanilla_caller,duplex_caller,
// codec_caller}.rs hot loops.  Citations are relative to fgumi 0.2.0's crates/fgumi-consensus/src/.
#include "fgumi_oracle.hpp"

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <functional>
#include <limits>

namespace fgoracle {

namespace {
const double LN_10 = 2.302585092994046;            // std::f64::consts::LN_10
const double LN_TWO = 0.6931471805599453;          // phred.rs:16
const double LN_FOUR_THIRDS = 0.2876820724517809;  // phred.rs:19
const double PHRED_PRECISION = 0.001;              // phred.rs:31
const double NEG_INF = -std::numeric_limits<double>::infinity();
}  // namespace

// phred.rs:66-68   `-f64::from(phred) * LN_10 / 10.0`
double phred_to_ln_error_prob(uint8_t phred) { return -static_cast<double>(phred) * LN_10 / 10.0; }

// phred.rs:89-92
double phred_to_ln_correct_prob(uint8_t phred) {
  return ln_one_minus_exp(phred_to_ln_error_prob(phred));
}

// phred.rs:119-135
uint8_t ln_prob_to_phred(double ln_prob) {
  const double MAX_PHRED_AS_LN_ERROR = -static_cast<double>(MAX_PHRED) * LN_10 / 10.0;  // :34
  if (ln_prob < MAX_PHRED_AS_LN_ERROR) return MAX_PHRED;
  double phred = std::floor(-10.0 * ln_prob / LN_10 + PHRED_PRECISION);
  // f64::clamp keeps NaN, and Rust's saturating `NaN as u8` is 0 (reachable: a Q0 observation
  // makes correct[0] = -inf and the Kahan compensation NaN)
  if (std::isnan(phred)) return 0;
  if (phred < static_cast<double>(MIN_PHRED)) phred = MIN_PHRED;
  if (phred > static_cast<double>(MAX_PHRED)) phred = MAX_PHRED;
  return static_cast<uint8_t>(phred);
}

// phred.rs:148-158
double log1pexp(double x) {
  if (x <= -37.0) return std::exp(x);
  if (x <= 18.0) return std::log1p(std::exp(x));
  if (x <= 33.3) return x + std::exp(-x);
  return x;
}

// phred.rs:168-182
double ln_one_minus_exp(double x) {
  if (x >= 0.0) return NEG_INF;
  if (x >= -LN_TWO) return std::log(-std::expm1(x));
  return std::log1p(-std::exp(x));
}

// phred.rs:188-198
double ln_a_minus_b(double a, double b) {
  if (std::isinf(b) && b < 0.0) return a;
  if (std::fabs(a - b) < DBL_EPSILON) return NEG_INF;
  return a + ln_one_minus_exp(b - a);
}

// phred.rs:231-251
double ln_error_prob_two_trials(double ln_p1, double ln_p2) {
  if (ln_p1 < ln_p2) std::swap(ln_p1, ln_p2);
  if (ln_p1 - ln_p2 >= 6.0) return ln_p1;
  double term1 = ln_sum_exp(ln_p1, ln_p2);
  double term2 = LN_FOUR_THIRDS + ln_p1 + ln_p2;
  return ln_a_minus_b(term1, term2);
}

// phred.rs:274-285
double ln_sum_exp(double ln_a, double ln_b) {
  if (std::isinf(ln_a) && ln_a < 0.0) return ln_b;
  if (std::isinf(ln_b) && ln_b < 0.0) return ln_a;
  if (ln_b < ln_a) std::swap(ln_a, ln_b);
  return ln_a + log1pexp(ln_b - ln_a);
}

// phred.rs:307-330
double ln_sum_exp_array(const double* values, size_t n) {
  if (n == 0) return NEG_INF;
  double min_value = std::numeric_limits<double>::infinity();
  size_t min_index = 0;
  for (size_t i = 0; i < n; ++i) {
    if (values[i] < min_value) {
      min_index = i;
      min_value = values[i];
    }
  }
  if (std::isinf(min_value)) return min_value;
  double sum = min_value;
  for (size_t i = 0; i < n; ++i) {
    if (i != min_index) sum = ln_sum_exp(sum, values[i]);
  }
  return sum;
}

// ---- base_builder.rs -----------------------------------------------------------------------
namespace {
const uint8_t DNA_BASES[4] = {'A', 'C', 'G', 'T'};  // base_builder.rs:199
// BASE_TO_INDEX, base_builder.rs:204-215
inline uint8_t base_to_index(uint8_t b) {
  switch (b) {
    case 'A': case 'a': return 0;
    case 'C': case 'c': return 1;
    case 'G': case 'g': return 2;
    case 'T': case 't': return 3;
    default: return 255;
  }
}
}  // namespace

// base_builder.rs:252-278
ConsensusBaseBuilder::ConsensusBaseBuilder(uint8_t pre, uint8_t post) {
  double ln_error_post = phred_to_ln_error_prob(post);
  const double ln3 = std::log(3.0);  // `3.0_f64.ln()`
  for (int q = 0; q <= MAX_PHRED; ++q) {
    double ln_error_seq = phred_to_ln_error_prob(static_cast<uint8_t>(q));
    double adjusted_error = ln_error_prob_two_trials(ln_error_post, ln_error_seq);
    adjusted_correct_table[q] = ln_not(adjusted_error);
    adjusted_error_per_alt[q] = adjusted_error - ln3;
  }
  ln_error_pre_umi = phred_to_ln_error_prob(pre);
  reset();
}

// base_builder.rs:281-285
void ConsensusBaseBuilder::reset() {
  for (int i = 0; i < 4; ++i) {
    likelihoods[i] = 0.0;  // LN_ONE
    compensations[i] = 0.0;
    observations[i] = 0;
  }
}

// base_builder.rs:295-327.  wide::f64x4 lane ops == four independent scalar IEEE ops.
void ConsensusBaseBuilder::add(uint8_t base, uint8_t qual) {
  uint8_t matching_idx = base_to_index(base);
  if (matching_idx == 255) return;
  size_t qual_idx = std::min<uint8_t>(qual, MAX_PHRED);
  double ln_correct = adjusted_correct_table[qual_idx];
  double ln_error_per_base = adjusted_error_per_alt[qual_idx];
  for (int i = 0; i < 4; ++i) {
    double value = (i == matching_idx) ? ln_correct : ln_error_per_base;
    double y = value - compensations[i];
    double t = likelihoods[i] + y;
    compensations[i] = (t - likelihoods[i]) - y;
    likelihoods[i] = t;
  }
  observations[matching_idx] = static_cast<uint16_t>(observations[matching_idx] + 1);
}

// base_builder.rs:338-379
bool ConsensusBaseBuilder::try_unanimous_fast_path(uint8_t* base, uint8_t* qual) const {
  int observed_base_idx = -1;
  int num_bases_observed = 0;
  for (int i = 0; i < 4; ++i) {
    if (observations[i] > 0) {
      ++num_bases_observed;
      observed_base_idx = i;
      if (num_bases_observed > 1) return false;
    }
  }
  if (observed_base_idx < 0) return false;
  const double FAST_PATH_THRESHOLD = 23.0;
  double winner_ll = likelihoods[observed_base_idx];
  double loser_ll = likelihoods[(observed_base_idx + 1) % 4];
  if (winner_ll - loser_ll > FAST_PATH_THRESHOLD) {
    *base = DNA_BASES[observed_base_idx];
    *qual = ln_prob_to_phred(ln_error_pre_umi);
    return true;
  }
  return false;
}

// base_builder.rs:391-458
void ConsensusBaseBuilder::call(uint8_t* base, uint8_t* qual) const {
  if (contributions() == 0) {
    *base = NO_CALL_BASE;
    *qual = MIN_PHRED;
    return;
  }
  if (try_unanimous_fast_path(base, qual)) return;

  double ln_sum = ln_sum_exp_array(likelihoods, 4);

  double max_likelihood = NEG_INF;
  int max_index = -1;
  bool tie = false;
  for (int i = 0; i < 4; ++i) {
    double ll = likelihoods[i];
    if (ll > max_likelihood) {          // Some(Ordering::Greater)
      max_likelihood = ll;
      max_index = i;
      tie = false;
    } else if (ll == max_likelihood) {  // Some(Ordering::Equal)
      tie = true;
    } else if (ll < max_likelihood) {   // Some(Ordering::Less)
      // approx 0.5.1 abs_diff_eq!: |a-b| <= epsilon
      if (std::fabs(ll - max_likelihood) <= DBL_EPSILON) tie = true;
    }                                   // None (NaN): nothing
  }
  if (tie || max_index < 0) {
    *base = NO_CALL_BASE;
    *qual = MIN_PHRED;
    return;
  }
  double ln_posterior = max_likelihood - ln_sum;                         // ln_normalize
  double ln_consensus_error = ln_not(ln_posterior);
  double ln_final_error = ln_error_prob_two_trials(ln_error_pre_umi, ln_consensus_error);
  *base = DNA_BASES[max_index];
  *qual = ln_prob_to_phred(ln_final_error);
}

uint16_t ConsensusBaseBuilder::contributions() const {
  return static_cast<uint16_t>(observations[0] + observations[1] + observations[2] +
                               observations[3]);
}

uint16_t ConsensusBaseBuilder::observations_for_base(uint8_t base) const {
  uint8_t idx = base_to_index(base);
  return idx == 255 ? 0 : observations[idx];
}

// ---- vanilla_caller.rs ---------------------------------------------------------------------
// vanilla_caller.rs:463-494
std::vector<uint8_t> compute_single_input_consensus_quals(uint8_t pre, uint8_t post) {
  uint8_t labeling_error_phred = std::min(pre, post);
  double ln_prob_labeling = phred_to_ln_error_prob(labeling_error_phred);
  std::vector<uint8_t> out;
  out.reserve(MAX_PHRED + 1);
  for (int q = 0; q <= MAX_PHRED; ++q) {
    double ln_prob_seq = phred_to_ln_error_prob(static_cast<uint8_t>(q));
    uint8_t adjusted = ln_prob_to_phred(ln_error_prob_two_trials(ln_prob_seq, ln_prob_labeling));
    out.push_back(std::min(adjusted, MAX_PHRED));
  }
  return out;
}

// vanilla_caller.rs:1260-1358
bool create_consensus_from_source_reads(const SourceRow* reads, size_t n_reads,
                                        const VanillaOptions& opt, ConsensusBaseBuilder& builder,
                                        const std::vector<uint8_t>& single_input_quals,
                                        ConsensusColumns* out) {
  if (n_reads == 0) return false;  // :1264-1266 bail!
  std::vector<size_t> lengths(n_reads);
  for (size_t i = 0; i < n_reads; ++i) lengths[i] = reads[i].len;
  std::sort(lengths.begin(), lengths.end(), std::greater<size_t>());
  const size_t min_reads = opt.min_reads;
  const size_t consensus_len = lengths[min_reads - 1];  // :1277

  out->bases.clear(); out->quals.clear(); out->depths.clear(); out->errors.clear();
  out->bases.reserve(consensus_len); out->quals.reserve(consensus_len);
  out->depths.reserve(consensus_len); out->errors.reserve(consensus_len);

  if (n_reads == 1) {  // :1285-1316
    const SourceRow& sr = reads[0];
    for (size_t pos = 0; pos < consensus_len; ++pos) {
      uint8_t raw_base = sr.bases[pos];
      size_t raw_qual_idx = sr.quals[pos];
      uint8_t adjusted_qual =
          raw_qual_idx < single_input_quals.size() ? single_input_quals[raw_qual_idx] : 0;
      if (adjusted_qual < opt.min_consensus_base_quality) {
        out->bases.push_back(NO_CALL_BASE);
        out->quals.push_back(MIN_PHRED);
      } else {
        out->bases.push_back(raw_base);
        out->quals.push_back(adjusted_qual);
      }
      out->depths.push_back(raw_base != NO_CALL_BASE ? 1 : 0);
      out->errors.push_back(0);
    }
    return true;
  }

  for (size_t pos = 0; pos < consensus_len; ++pos) {  // :1319-1355
    builder.reset();
    for (size_t r = 0; r < n_reads; ++r) {
      const SourceRow& sr = reads[r];
      if (pos < sr.len) {
        uint8_t base = sr.bases[pos];
        uint8_t qual = sr.quals[pos];
        if (base != NO_CALL_BASE) builder.add(base, qual);
      }
    }
    uint8_t base, qual;
    builder.call(&base, &qual);
    uint16_t depth = builder.contributions();
    out->depths.push_back(depth);
    uint16_t error_count = static_cast<uint16_t>(depth - builder.observations_for_base(base));
    out->errors.push_back(error_count);
    if (static_cast<size_t>(depth) < min_reads) {
      out->bases.push_back(NO_CALL_BASE);
      out->quals.push_back(0);  // NotEnoughReadsQual
    } else if (qual < opt.min_consensus_base_quality) {
      out->bases.push_back(NO_CALL_BASE);
      out->quals.push_back(MIN_PHRED);  // TooLowQualityQual
    } else {
      out->bases.push_back(base);
      out->quals.push_back(qual);
    }
  }
  return true;
}

// ---- duplex_caller.rs ----------------------------------------------------------------------
namespace {
// duplex_caller.rs:783-791
inline uint8_t cap_quality(int32_t score) {
  if (score < MIN_PHRED) return MIN_PHRED;
  if (score > MAX_PHRED) return MAX_PHRED;
  return static_cast<uint8_t>(score);
}
// duplex_caller.rs:797-800
inline bool is_error(uint8_t source_base, uint8_t consensus_base) {
  return source_base != 'N' && consensus_base != 'N' && source_base != consensus_base;
}
}  // namespace

// duplex_caller.rs:890-970 (both-strands arm; methylation disabled ⇒ is_conversion_artifact=false)
void duplex_combine(const uint8_t* a_bases, const uint8_t* a_quals, const uint16_t* a_depths,
                    const uint16_t* a_errors, const uint8_t* b_bases, const uint8_t* b_quals,
                    const uint16_t* b_depths, const uint16_t* b_errors, size_t len,
                    const SourceRow* source, size_t n_source, uint8_t* out_bases,
                    uint8_t* out_quals, uint16_t* out_errors) {
  const uint8_t NO_CALL = 'N';
  const uint8_t NO_CALL_QUAL = MIN_PHRED;
  for (size_t i = 0; i < len; ++i) {
    uint8_t a_base = a_bases[i], b_base = b_bases[i];
    int32_t a_qual = a_quals[i], b_qual = b_quals[i];
    uint8_t raw_base, raw_qual;
    if (a_base == b_base) {
      raw_base = a_base; raw_qual = cap_quality(a_qual + b_qual);
    } else if (a_qual > b_qual) {
      raw_base = a_base; raw_qual = cap_quality(a_qual - b_qual);
    } else if (b_qual > a_qual) {
      raw_base = b_base; raw_qual = cap_quality(b_qual - a_qual);
    } else {
      raw_base = a_base; raw_qual = NO_CALL_QUAL;
    }
    if (a_base == NO_CALL || b_base == NO_CALL || raw_qual == NO_CALL_QUAL) {
      out_bases[i] = NO_CALL; out_quals[i] = NO_CALL_QUAL;
    } else {
      out_bases[i] = raw_base; out_quals[i] = raw_qual;
    }
    uint16_t error_count;
    if (source != nullptr) {  // :943-951
      int32_t num_errors = 0;
      for (size_t s = 0; s < n_source; ++s)
        if (source[s].len > i && is_error(source[s].bases[i], raw_base)) ++num_errors;
      error_count = static_cast<uint16_t>(std::clamp<int32_t>(num_errors, 0, INT16_MAX));
    } else {                  // :952-967
      int32_t a_err = a_errors[i], b_err = b_errors[i];
      int32_t a_dep = a_depths[i], b_dep = b_depths[i];
      int32_t err;
      if (a_base == b_base) err = a_err + b_err;
      else if (raw_base == a_base) err = a_err + (b_dep - b_err);
      else err = b_err + (a_dep - a_err);
      error_count = static_cast<uint16_t>(std::clamp<int32_t>(err, 0, INT16_MAX));
    }
    out_errors[i] = error_count;
  }
}

// duplex_caller.rs:838-1015
int duplex_consensus_arms(const uint8_t* a_bases, const uint8_t* a_quals, const uint16_t* a_depths,
                          const uint16_t* a_errors, size_t la, const uint8_t* b_bases,
                          const uint8_t* b_quals, const uint16_t* b_depths,
                          const uint16_t* b_errors, size_t lb, const SourceRow* source,
                          size_t n_source, uint8_t* out_bases, uint8_t* out_quals,
                          uint16_t* out_errors, size_t* out_len) {
  size_t len = std::min(la, lb);                                        // :846-849
  bool a_any = false, b_any = false;                                    // :852-853
  for (size_t i = 0; i < len; ++i) { a_any |= a_depths[i] > 0; b_any |= b_depths[i] > 0; }
  if (a_any && !b_any) {                                                // :855-868
    std::copy(a_bases, a_bases + la, out_bases);
    std::copy(a_quals, a_quals + la, out_quals);
    std::copy(a_errors, a_errors + la, out_errors);
    *out_len = la;
    return 1;
  }
  if (!a_any && b_any) {                                                // :869-882
    std::copy(b_bases, b_bases + lb, out_bases);
    std::copy(b_quals, b_quals + lb, out_quals);
    std::copy(b_errors, b_errors + lb, out_errors);
    *out_len = lb;
    return 2;
  }
  if (!a_any && !b_any) { *out_len = 0; return 3; }                     // :1013
  duplex_combine(a_bases, a_quals, a_depths, a_errors, b_bases, b_quals, b_depths, b_errors, len,
                 source, n_source, out_bases, out_quals, out_errors);
  *out_len = len;
  return 0;
}

// ---- codec_caller.rs -----------------------------------------------------------------------
// codec_caller.rs:1048-1152
CodecCombineResult codec_combine_padded(const uint8_t* a_bases, const uint8_t* a_quals,
                                        const uint16_t* a_depths, const uint16_t* a_errors,
                                        const uint8_t* b_bases, const uint8_t* b_quals,
                                        const uint16_t* b_depths, const uint16_t* b_errors,
                                        size_t len, uint8_t* out_bases, uint8_t* out_quals,
                                        uint16_t* out_depths, uint16_t* out_errors) {
  CodecCombineResult res;
  auto sat_sub16 = [](uint16_t x, uint16_t y) -> uint16_t { return x > y ? x - y : 0; };
  auto sat_sub8 = [](uint8_t x, uint8_t y) -> uint8_t { return x > y ? x - y : 0; };
  for (size_t p = 0; p < len; ++p) {
    uint8_t ba = a_bases[p], qa = a_quals[p];
    uint16_t da = a_depths[p], ea = a_errors[p];
    uint8_t bb = b_bases[p], qb = b_quals[p];
    uint16_t db = b_depths[p], eb = b_errors[p];
    bool a_has = ba != NO_CALL_BASE && ba != NO_CALL_BASE_LOWER;
    bool b_has = bb != NO_CALL_BASE && bb != NO_CALL_BASE_LOWER;
    uint8_t dbase, dqual;
    uint16_t depth, error;
    if (a_has && b_has) {
      ++res.duplex_bases_count;
      uint8_t raw_base, raw_qual;
      if (ba == bb) {
        raw_base = ba;
        raw_qual = static_cast<uint8_t>(std::min<uint16_t>(93, uint16_t(qa) + uint16_t(qb)));
      } else if (qa > qb) {
        ++res.duplex_disagreements;
        raw_base = ba; raw_qual = std::max<uint8_t>(MIN_PHRED, sat_sub8(qa, qb));
      } else if (qb > qa) {
        ++res.duplex_disagreements;
        raw_base = bb; raw_qual = std::max<uint8_t>(MIN_PHRED, sat_sub8(qb, qa));
      } else {
        ++res.duplex_disagreements;
        raw_base = ba; raw_qual = MIN_PHRED;
      }
      if (raw_qual == MIN_PHRED) { dbase = NO_CALL_BASE; dqual = MIN_PHRED; }
      else { dbase = raw_base; dqual = raw_qual; }
      uint16_t derr;
      // Rust u16 `+` would panic on overflow in debug / wrap in release; depths here are tiny.
      if (ba == bb) derr = static_cast<uint16_t>(ea + eb);
      else if (ba == raw_base) derr = static_cast<uint16_t>(ea + sat_sub16(db, eb));
      else derr = static_cast<uint16_t>(eb + sat_sub16(da, ea));
      depth = static_cast<uint16_t>(da + db);
      error = derr;
    } else if (a_has) {
      if (qa == MIN_PHRED) { dbase = NO_CALL_BASE; dqual = MIN_PHRED; }
      else { dbase = ba; dqual = qa; }
      depth = da; error = ea;
    } else if (b_has) {
      if (qb == MIN_PHRED) { dbase = NO_CALL_BASE; dqual = MIN_PHRED; }
      else { dbase = bb; dqual = qb; }
      depth = db; error = eb;
    } else {
      dbase = NO_CALL_BASE; dqual = MIN_PHRED; depth = 0;
      error = static_cast<uint16_t>(ea + eb);
    }
    if (ba == NO_CALL_BASE || bb == NO_CALL_BASE) { dbase = NO_CALL_BASE; dqual = MIN_PHRED; }
    out_bases[p] = dbase; out_quals[p] = dqual; out_depths[p] = depth; out_errors[p] = error;
  }
  return res;
}

// codec_caller.rs:1183-1212
void codec_mask_quals(const uint8_t* cons_bases, uint8_t* cons_quals, size_t len,
                      const uint8_t* padded_r1_bases, const uint8_t* padded_r2_bases,
                      int ss_qual, int outer_qual, size_t outer_len) {
  for (size_t idx = 0; idx < len; ++idx) {
    bool a_is_n = padded_r1_bases[idx] == NO_CALL_BASE;
    bool b_is_n = padded_r2_bases[idx] == NO_CALL_BASE;
    if ((a_is_n || b_is_n) && cons_bases[idx] != NO_CALL_BASE) {
      if (ss_qual >= 0) cons_quals[idx] = static_cast<uint8_t>(ss_qual);
    }
    if (outer_qual >= 0) {
      size_t hi = len > outer_len ? len - outer_len : 0;  // saturating_sub
      if (idx < outer_len || idx >= hi)
        cons_quals[idx] = std::min<uint8_t>(cons_quals[idx], static_cast<uint8_t>(outer_qual));
    }
  }
}

// fgumi-dna/src/dna.rs:30-40
uint8_t complement_base(uint8_t b) {
  switch (b) {
    case 'A': case 'a': return 'T';
    case 'T': case 't': return 'A';
    case 'C': case 'c': return 'G';
    case 'G': case 'g': return 'C';
    default: return b;   // 'N' -> 'N', 'n' -> 'n', anything else unchanged
  }
}

// codec_caller.rs:507-520
SsColumns reverse_complement_ss(const SsColumns& ss) {
  SsColumns o;
  size_t n = ss.bases.size();
  o.bases.resize(n); o.quals.resize(n); o.depths.resize(n); o.errors.resize(n);
  for (size_t i = 0; i < n; ++i) {
    o.bases[i] = complement_base(ss.bases[n - 1 - i]);   // dna.rs:58-60
    o.quals[i] = ss.quals[n - 1 - i];
    o.depths[i] = ss.depths[n - 1 - i];
    o.errors[i] = ss.errors[n - 1 - i];
  }
  return o;
}

// codec_caller.rs:980-1023
SsColumns pad_consensus(const SsColumns& ss, size_t new_length, bool pad_left) {
  size_t cur = ss.bases.size();
  if (new_length <= cur) return ss;
  size_t pad = new_length - cur;
  SsColumns o;
  auto build = [&](auto& dst, const auto& src, auto fill) {
    dst.reserve(new_length);
    if (pad_left) dst.insert(dst.end(), pad, fill);
    dst.insert(dst.end(), src.begin(), src.end());
    if (!pad_left) dst.insert(dst.end(), pad, fill);
  };
  build(o.bases, ss.bases, NO_CALL_BASE_LOWER);
  build(o.quals, ss.quals, uint8_t(0));
  build(o.depths, ss.depths, uint16_t(0));
  build(o.errors, ss.errors, uint16_t(0));
  return o;
}

// codec_caller.rs:721-784 (orient, pad, combine with the gate of :1155-1166, mask, re-orient)
CodecJobResult codec_job(const SsColumns& ss_r1, const SsColumns& ss_r2, bool r1_is_negative,
                         bool r2_is_negative, size_t consensus_length, int ss_qual, int outer_qual,
                         size_t outer_len, size_t max_duplex_disagreements,
                         double max_duplex_disagreement_rate) {
  CodecJobResult res;
  SsColumns r1o = r1_is_negative ? reverse_complement_ss(ss_r1) : ss_r1;   // :746-750
  SsColumns r2o = r1_is_negative ? ss_r2 : reverse_complement_ss(ss_r2);
  SsColumns p1 = pad_consensus(r1o, consensus_length, r1_is_negative);     // :752-753
  SsColumns p2 = pad_consensus(r2o, consensus_length, r2_is_negative);
  size_t len = p1.bases.size();
  SsColumns c;
  c.bases.resize(len); c.quals.resize(len); c.depths.resize(len); c.errors.resize(len);
  CodecCombineResult cr = codec_combine_padded(p1.bases.data(), p1.quals.data(), p1.depths.data(),
                                               p1.errors.data(), p2.bases.data(), p2.quals.data(),
                                               p2.depths.data(), p2.errors.data(), len,
                                               c.bases.data(), c.quals.data(), c.depths.data(),
                                               c.errors.data());
  res.duplex_bases_count = cr.duplex_bases_count;
  res.duplex_disagreements = cr.duplex_disagreements;
  if (cr.duplex_bases_count > 0) {   // :1155-1166
    double rate = static_cast<double>(cr.duplex_disagreements) /
                  static_cast<double>(cr.duplex_bases_count);
    if (cr.duplex_disagreements > max_duplex_disagreements) res.status = 1;
    else if (rate > max_duplex_disagreement_rate) res.status = 2;
  }
  codec_mask_quals(c.bases.data(), c.quals.data(), len, p1.bases.data(), p2.bases.data(), ss_qual,
                   outer_qual, outer_len);                                  // :756
  res.consensus = r1_is_negative ? reverse_complement_ss(c) : c;            // :757-758
  return res;
}

}  // namespace fgoracle
