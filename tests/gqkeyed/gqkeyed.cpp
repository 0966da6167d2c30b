// gqkeyed.cpp — the generated quantities of a user model header (include/dhmc_models.h) evaluated on the CPU with a key per
// point: the checker of dhmc_generated_keyed and of the summary's random rows (tests/test_posterior_predictive.py).  It
// compiles for either quantity signature: random quantities (DHMC_USER_GENERATED_RNG) draw from dhmc_math.h's Philox
// streams, keyed as on the device; deterministic ones ignore the key.  The header's formulas are compiled for the host with
// the CPU oracle's flags (no implicit FMA), so that they equal the device's bit for bit.
#include "../../include/dhmc_models.h"

#ifndef DHMC_USER_GENERATED
#error "gqkeyed: the model header declares no generated quantities (DHMC_USER_GENERATED)"
#endif

#ifdef DHMC_USER_GENERATED_RNG
#define GQKEYED_EVAL(k, D, q, params, rng) dhmc_user_generated(k, D, q, params, rng)
#define GQKEYED_RANDOM 1
#else
#define GQKEYED_EVAL(k, D, q, params, rng) ((void)(rng), dhmc_user_generated(k, D, q, params))
#define GQKEYED_RANDOM 0
#endif

extern "C" int orc_user_ngq(int D) { return dhmc_user_ngq(D); }

// 1 when the quantities are random, else 0
extern "C" int orc_user_random(void) { return GQKEYED_RANDOM; }

// out [n][G] ← g(theta [n][D]) with point i keyed by (seed, chain[i]) and transition[i], every point with the parameter
// block params
extern "C" void orc_user_generated_keyed(const double* theta, long long n, int D, const double* params, unsigned long long seed,
                                         const long long* chain, const unsigned* transition, double* out) {
  const int G = dhmc_user_ngq(D);
  for (long long i = 0; i < n; ++i) {
    dhmc_gq_rng rng;
    rng.key = dm_make_key(seed, (uint64_t)chain[i]);
    rng.t = transition[i];
    for (int k = 0; k < G; ++k) out[i * G + k] = GQKEYED_EVAL(k, D, theta + i * D, params, &rng);
  }
}

// the streams themselves: out [n] ← dhmc_gq_normal (normal != 0) or dhmc_gq_uniform of key i at index index[i]
extern "C" void orc_gq_numbers(unsigned long long seed, const long long* chain, const unsigned* transition, const unsigned* index,
                               long long n, int normal, double* out) {
  for (long long i = 0; i < n; ++i) {
    dhmc_gq_rng rng;
    rng.key = dm_make_key(seed, (uint64_t)chain[i]);
    rng.t = transition[i];
    out[i] = normal ? dhmc_gq_normal(&rng, index[i]) : dhmc_gq_uniform(&rng, index[i]);
  }
}
