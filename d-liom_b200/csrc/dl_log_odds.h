// ProbabilityToLogOddsInteger (C/mapping/submaps.h:37-53) as a table of float thresholds, built on the host.
//
// The reference evaluates std::log (glibc logf) per pixel. The device never calls a log: on [kMinProbability, kMaxProbability]
// the reference's integer is a monotone step function of the probability, so the host finds, by bisection over the float bit
// patterns, the first probability at which it reaches 2, 3, ..., 255, and the device counts the thresholds at or below a value.
// tests/cpp/log_odds_table_check.cc compares the table with log_odds_integer() for every float of [0.1f, 0.9f].
// Host code only (glibc logf); compile without contraction, as the rest of the library.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

namespace dl {

constexpr float kMinProbability = 0.1f;                  // probability_values.h
constexpr float kMaxProbability = 1.f - kMinProbability;
constexpr int kLogOddsThresholds = 256;                  // 254 steps, padded with +inf to a power of two

// Logit(probability) (submaps.h:37-39); the call goes through a volatile pointer so that glibc evaluates every log, never the
// compiler's constant folding.
inline float logit(float probability) {
  float (*volatile glibc_logf)(float) = ::logf;
  return glibc_logf(probability / (1.f - probability));
}

// ProbabilityToLogOddsInteger in the reference's expression order: ((Logit(p) - kMinLogOdds) * 254.f) / (kMaxLogOdds -
// kMinLogOdds), rounded half away from zero, plus 1. Defined for p in [kMinProbability, kMaxProbability].
inline int log_odds_integer(float probability) {
  const float min_log_odds = logit(kMinProbability);
  const float max_log_odds = logit(kMaxProbability);
  return (int)lroundf((logit(probability) - min_log_odds) * 254.f / (max_log_odds - min_log_odds)) + 1;
}

inline float float_of_bits(uint32_t b) {
  float f;
  std::memcpy(&f, &b, sizeof(f));
  return f;
}
inline uint32_t bits_of_float(float f) {
  uint32_t b;
  std::memcpy(&b, &f, sizeof(b));
  return b;
}

// thresholds[k] (k < 254) = the least float p in [kMinProbability, kMaxProbability] with log_odds_integer(p) >= k + 2;
// +inf where no such p exists, and in the two padding entries. Then, for every p of that range,
// log_odds_integer(p) == 1 + #{k : thresholds[k] <= p}.
inline void build_log_odds_thresholds(float* thresholds) {
  const uint32_t first = bits_of_float(kMinProbability), last = bits_of_float(kMaxProbability);
  for (int k = 0; k < kLogOddsThresholds; ++k) {
    const int want = k + 2;
    thresholds[k] = INFINITY;
    if (k >= 254 || log_odds_integer(float_of_bits(last)) < want) continue;
    uint32_t lo = first, hi = last;  // log_odds_integer(hi) >= want
    while (lo < hi) {
      const uint32_t mid = lo + (hi - lo) / 2;
      if (log_odds_integer(float_of_bits(mid)) >= want) hi = mid;
      else lo = mid + 1;
    }
    thresholds[k] = float_of_bits(lo);
  }
}

// 1 + the number of thresholds at or below p: the device side's lookup, also usable on the host.
#ifdef __CUDACC__
__host__ __device__
#endif
inline int log_odds_integer_from_table(const float* thresholds, float p) {
  int pos = 0;
  for (int step = kLogOddsThresholds / 2; step > 0; step >>= 1)
    if (thresholds[pos + step - 1] <= p) pos += step;
  return 1 + pos;
}

}  // namespace dl
