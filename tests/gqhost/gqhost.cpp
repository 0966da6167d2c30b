// gqhost.cpp — the generated quantities of a user model header (include/dhmc_models.h) evaluated on the CPU: the checker of
// dhmc_generated and of the summary's generated rows (tests/test_generated_quantities.py).  The header's formulas are
// compiled for the host with the CPU oracle's flags (no implicit FMA), so that they equal the device's bit for bit.
#include "../../include/dhmc_models.h"

#ifndef DHMC_USER_GENERATED
#error "gqhost: the model header declares no generated quantities (DHMC_USER_GENERATED)"
#endif

extern "C" int orc_user_ngq(int D) { return dhmc_user_ngq(D); }

// out [n][G] ← g(theta [n][D]), every point with the parameter block params
extern "C" void orc_user_generated(const double* theta, long long n, int D, const double* params, double* out) {
  const int G = dhmc_user_ngq(D);
  for (long long i = 0; i < n; ++i)
    for (int k = 0; k < G; ++k) out[i * G + k] = dhmc_user_generated(k, D, theta + i * D, params);
}
