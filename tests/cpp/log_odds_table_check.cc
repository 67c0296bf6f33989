// Host-side check of dl::build_log_odds_thresholds (d-liom_b200/csrc/dl_log_odds.h), the table the texture kernel reads instead of
// a device log: for EVERY float p in [kMinProbability, kMaxProbability], 1 + #{thresholds <= p} must equal a direct statement of
// ProbabilityToLogOddsInteger (C/mapping/submaps.h:37-53) with glibc logf. Prints "n=<floats> bad=<mismatches> steps=<distinct
// values>"; exit status 1 on a mismatch.
#include <cmath>
#include <cstdio>
#include <cstring>

#include "../../d-liom_b200/csrc/dl_log_odds.h"

namespace {
float (*volatile glibc_logf)(float) = ::logf;
float Logit(float probability) { return glibc_logf(probability / (1.f - probability)); }
}  // namespace

int main() {
  const float kMinProbability = 0.1f, kMaxProbability = 1.f - kMinProbability;
  const float kMaxLogOdds = Logit(kMaxProbability), kMinLogOdds = Logit(kMinProbability);
  float table[dl::kLogOddsThresholds];
  dl::build_log_odds_thresholds(table);
  long n = 0, bad = 0;
  int steps = 0, last = -1;
  for (float p = kMinProbability; p <= kMaxProbability; p = nextafterf(p, 2.f)) {
    const int want = (int)lroundf((Logit(p) - kMinLogOdds) * 254.f / (kMaxLogOdds - kMinLogOdds)) + 1;
    const int got = dl::log_odds_integer_from_table(table, p);
    if (got != want && bad < 10) printf("p=%.9g want %d got %d\n", p, want, got);
    bad += got != want;
    steps += want != last;
    last = want;
    ++n;
  }
  printf("n=%ld bad=%ld steps=%d\n", n, bad, steps);
  return bad != 0;
}
