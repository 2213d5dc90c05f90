// f64 log-space helpers evaluated on the device for positions that leave the integer fast path.
//
// Behavioural spec: fgumi 0.2.0, crates/fgumi-consensus/src/phred.rs (cited per function).
// Add/sub/mul/div are IEEE-754 correctly rounded on sm_90a exactly as on the host, so the Kahan
// likelihood sums, the tie test and the threshold compares are bit-identical to the reference's.
// exp/log/log1p/expm1 come from CUDA's libdevice (<= 1-2 ulp) rather than glibc; their results only
// reach the output through floor(x + 0.001), so a difference needs x within ~1e-15 of an integer
// boundary (DESIGN.md "numerics").
#pragma once
#include <math_constants.h>
#include <stdint.h>

namespace fgb {
namespace dm {

__device__ constexpr double kLn10 = 2.302585092994046;            // f64::consts::LN_10
__device__ constexpr double kLn2 = 0.6931471805599453;            // phred.rs:16
__device__ constexpr double kLnFourThirds = 0.2876820724517809;   // phred.rs:19
__device__ constexpr double kEps = 2.220446049250313e-16;         // f64::EPSILON
__device__ constexpr double kMaxPhredAsLnError = -93.0 * 2.302585092994046 / 10.0;  // phred.rs:34

// phred.rs:119-135
__device__ __forceinline__ uint32_t ln_prob_to_phred(double ln_prob) {
  if (ln_prob < kMaxPhredAsLnError) return 93u;
  double phred = floor(__dadd_rn(__ddiv_rn(__dmul_rn(-10.0, ln_prob), kLn10), 0.001));
  if (isnan(phred)) return 0u;   // Rust: NaN.clamp(..) is NaN and `NaN as u8` saturates to 0
  phred = phred < 2.0 ? 2.0 : phred;
  phred = phred > 93.0 ? 93.0 : phred;
  return (uint32_t)phred;
}

// phred.rs:148-158
__device__ __forceinline__ double log1pexp(double x) {
  if (x <= -37.0) return exp(x);
  if (x <= 18.0) return log1p(exp(x));
  if (x <= 33.3) return x + exp(-x);
  return x;
}

// phred.rs:168-182
__device__ __forceinline__ double ln_one_minus_exp(double x) {
  if (x >= 0.0) return -CUDART_INF;
  if (x >= -kLn2) return log(-expm1(x));
  return log1p(-exp(x));
}

// phred.rs:274-285
__device__ __forceinline__ double ln_sum_exp(double a, double b) {
  if (isinf(a) && a < 0.0) return b;
  if (isinf(b) && b < 0.0) return a;
  if (b < a) { double t = a; a = b; b = t; }
  return a + log1pexp(b - a);
}

// phred.rs:188-198
__device__ __forceinline__ double ln_a_minus_b(double a, double b) {
  if (isinf(b) && b < 0.0) return a;
  if (fabs(a - b) < kEps) return -CUDART_INF;
  return a + ln_one_minus_exp(b - a);
}

// phred.rs:231-251
__device__ __forceinline__ double ln_error_prob_two_trials(double p1, double p2) {
  if (p1 < p2) { double t = p1; p1 = p2; p2 = t; }
  if (p1 - p2 >= 6.0) return p1;
  double term1 = ln_sum_exp(p1, p2);
  double term2 = __dadd_rn(__dadd_rn(kLnFourThirds, p1), p2);
  return ln_a_minus_b(term1, term2);
}

// phred.rs:307-330 specialised to the four likelihoods
__device__ __forceinline__ double ln_sum_exp_array4(const double (&v)[4]) {
  double min_value = CUDART_INF;
  int min_index = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i)
    if (v[i] < min_value) { min_index = i; min_value = v[i]; }
  if (isinf(min_value)) return min_value;
  double sum = min_value;
#pragma unroll
  for (int i = 0; i < 4; ++i)
    if (i != min_index) sum = ln_sum_exp(sum, v[i]);
  return sum;
}

}  // namespace dm
}  // namespace fgb
