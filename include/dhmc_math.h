/* dhmc_math.h — deterministic scalar math + counter-based RNG shared by the
 * sm_90a kernels (dynamichmc.jl_b200/csrc) and the CPU oracle (oracle/).
 *
 * Why this header exists: the parity gate (SURVEY.md §8d) wants the INTEGER
 * decisions of the NUTS tree (depth, termination, steps, accept bits) bit-exact
 * between the CUDA path and the CPU restatement.  That is only possible if every
 * floating-point value feeding a comparison is produced by the same sequence of
 * IEEE-754 operations on both sides.  libm (glibc) and libdevice differ in the
 * last ulp, so exp/log/log1p/sincos are written here once, using only
 * + - * / sqrt fma and integer bit operations, all of which are correctly
 * rounded on x86-64 and on sm_90a.  Build rules: g++ -ffp-contract=off -mfma,
 * nvcc -fmad=false.  fma() is used explicitly where a fused operation is wanted.
 *
 * The RNG is Philox-4x32-10 (Salmon et al. 2011), keyed by the user seed and
 * countered by (chain, transition, stream, index); it replaces Julia's
 * Xoshiro/ziggurat stream at the reference call sites
 *   randn  : src/hamiltonian.jl:124 (rand_p)
 *   UInt32 : src/trees.jl:23        (Directions)
 *   randexp: src/NUTS.jl:44         (rand_bool_logprob)
 *   rand   : src/mcmc.jl:108        (random_position)
 * Stream parity with Julia is unpinned by the reference's tests (SURVEY §8c ii).
 */
#ifndef DHMC_MATH_H
#define DHMC_MATH_H

#include <stdint.h>
#include <math.h>
#include <string.h>

#if defined(__CUDACC__)
#define DHMC_HD __host__ __device__ __forceinline__
#else
#define DHMC_HD static inline
#endif
/* heavy transcendental bodies: optionally out of line on the device (code size).  Each out-of-line function dm_f has a
 * force-inlined twin dm_f_inl with the same body, for the call sites on a kernel's serial path (the tree's merges and
 * the momentum draw of the diagonal-metric kernels, csrc/device_backend.cuh): there a call costs its latency, keeps
 * independent evaluations from overlapping and pushes the values live across it to the stack.  Both twins perform the
 * same operations, so they return the same bits. */
#if defined(__CUDACC__) && defined(DHMC_NOINLINE_MATH)
#define DHMC_HDH static __host__ __device__ __noinline__
#else
#define DHMC_HDH DHMC_HD
#endif

/* ------------------------------------------------------------------ bits */
DHMC_HD uint64_t dm_bits(double x) {
#if defined(__CUDA_ARCH__)
  return (uint64_t)__double_as_longlong(x);
#else
  uint64_t u; memcpy(&u, &x, 8); return u;
#endif
}
DHMC_HD double dm_from_bits(uint64_t u) {
#if defined(__CUDA_ARCH__)
  return __longlong_as_double((long long)u);
#else
  double x; memcpy(&x, &u, 8); return x;
#endif
}
DHMC_HD double dm_inf(void) { return dm_from_bits(0x7FF0000000000000ull); }
DHMC_HD double dm_nan(void) { return dm_from_bits(0x7FF8000000000000ull); }
DHMC_HD int dm_isfinite(double x) {
  return ((dm_bits(x) >> 52) & 0x7FF) != 0x7FF;
}
DHMC_HD int dm_isnan(double x) { return x != x; }
DHMC_HD double dm_fma(double a, double b, double c) {
#if defined(__CUDA_ARCH__)
  return __fma_rn(a, b, c);
#else
  return __builtin_fma(a, b, c);
#endif
}
DHMC_HD double dm_sqrt(double x) {
#if defined(__CUDA_ARCH__)
  return __dsqrt_rn(x);
#else
  return __builtin_sqrt(x);
#endif
}
DHMC_HD double dm_floor(double x) {
#if defined(__CUDA_ARCH__)
  return floor(x);
#else
  return __builtin_floor(x);
#endif
}
DHMC_HD double dm_fabs(double x) {
  return dm_from_bits(dm_bits(x) & 0x7FFFFFFFFFFFFFFFull);
}
/* Julia's min/max propagate NaN (Base.min); used at NUTS.jl:79,86. */
DHMC_HD double dm_min_nan(double a, double b) {
  if (a != a) return a;
  if (b != b) return b;
  return a < b ? a : b;
}
DHMC_HD double dm_max_nan(double a, double b) {
  if (a != a) return a;
  if (b != b) return b;
  return a > b ? a : b;
}
/* 2^k for -1022 <= k <= 1023 */
DHMC_HD double dm_pow2i(int k) {
  return dm_from_bits((uint64_t)(k + 1023) << 52);
}

/* Blocked dot product Σ_j a[j·sa]·b[j] (what a BLAS does, with a FIXED blocking): sequential fused
 * multiply-adds within chunks of DHMC_DOT_CHUNK elements, the chunk sums added in increasing order,
 * ((s₀ + s₁) + s₂) + …; n <= 64 is one plain sequential chain.  The chunks are independent accumulation
 * chains — the unit the tensor-core paths (mma.sync.m8n8k4.f64 = four sequential FMAs) spread over warps.
 * Used for η = Xβ of the logistic model and for the Symmetric metric's M⁻¹p (hamiltonian.jl:110). */
#define DHMC_DOT_CHUNK 64
DHMC_HD double dm_blocked_dot(const double* a, size_t sa, const double* b, int n) {
  double tot = 0.0;
  for (int j0 = 0; j0 < n; j0 += DHMC_DOT_CHUNK) {
    const int j1 = j0 + DHMC_DOT_CHUNK < n ? j0 + DHMC_DOT_CHUNK : n;
    double sacc = 0.0;
    for (int j = j0; j < j1; ++j) sacc = dm_fma(a[(size_t)j * sa], b[j], sacc);
    tot = j0 == 0 ? sacc : tot + sacc;
  }
  return tot;
}

/* ------------------------------------------------------------------- exp */
#define DM_LN2_HI 6.93147180369123816490e-01 /* 0x3FE62E42FEE00000 */
#define DM_LN2_LO 1.90821492927058770002e-10 /* 0x3DEA39EF35793C76 */
#define DM_INVLN2 1.44269504088896338700e+00

DHMC_HDH double dm_exp(double x) {
  if (x != x) return x;
  if (x > 709.782712893384) return dm_inf();
  if (x < -745.1332191019412) return 0.0;
  double kd = dm_floor(x * DM_INVLN2 + 0.5);
  double hi = x - kd * DM_LN2_HI; /* kd*LN2_HI exact: 21 trailing zero bits */
  double lo = kd * DM_LN2_LO;
  double r = hi - lo; /* |r| <= ~0.3466 */
  /* Taylor to r^13: truncation < 4e-18 relative */
  double p = 1.0 / 6227020800.0;
  p = dm_fma(p, r, 1.0 / 479001600.0);
  p = dm_fma(p, r, 1.0 / 39916800.0);
  p = dm_fma(p, r, 1.0 / 3628800.0);
  p = dm_fma(p, r, 1.0 / 362880.0);
  p = dm_fma(p, r, 1.0 / 40320.0);
  p = dm_fma(p, r, 1.0 / 5040.0);
  p = dm_fma(p, r, 1.0 / 720.0);
  p = dm_fma(p, r, 1.0 / 120.0);
  p = dm_fma(p, r, 1.0 / 24.0);
  p = dm_fma(p, r, 1.0 / 6.0);
  p = dm_fma(p, r, 0.5);
  /* exp(r) = 1 + r + r^2 * p */
  double y = 1.0 + dm_fma(r * r, p, r);
  int k = (int)kd;
  int k1 = k / 2, k2 = k - k1;
  return (y * dm_pow2i(k1)) * dm_pow2i(k2);
}

/* ------------------------------------------------------------------- log */
DHMC_HD double dm_log_inl(double x) {
  if (x != x) return x;
  if (x < 0.0) return dm_nan();
  if (x == 0.0) return -dm_inf();
  if (!dm_isfinite(x)) return x;
  int e = 0;
  uint64_t b = dm_bits(x);
  if ((b >> 52) == 0) { /* subnormal */
    x = x * 18014398509481984.0; /* 2^54 */
    b = dm_bits(x);
    e = -54;
  }
  e += (int)(b >> 52) - 1023;
  uint64_t m = b & 0x000FFFFFFFFFFFFFull;
  double xm;
  if (m >= 0x0006A09E667F3BCDull) { /* mantissa >= sqrt(2): use [sqrt2/2,1) */
    xm = dm_from_bits(0x3FE0000000000000ull | m);
    e += 1;
  } else {
    xm = dm_from_bits(0x3FF0000000000000ull | m);
  }
  double f = xm - 1.0; /* exact */
  double s = f / (2.0 + f);
  double z = s * s; /* <= 0.02944 */
  /* log(1+f) = 2 atanh(s) = 2s + s*R, R = sum_{n>=1} 2/(2n+1) z^n, 11 terms */
  double R = 2.0 / 23.0;
  R = dm_fma(R, z, 2.0 / 21.0);
  R = dm_fma(R, z, 2.0 / 19.0);
  R = dm_fma(R, z, 2.0 / 17.0);
  R = dm_fma(R, z, 2.0 / 15.0);
  R = dm_fma(R, z, 2.0 / 13.0);
  R = dm_fma(R, z, 2.0 / 11.0);
  R = dm_fma(R, z, 2.0 / 9.0);
  R = dm_fma(R, z, 2.0 / 7.0);
  R = dm_fma(R, z, 2.0 / 5.0);
  R = dm_fma(R, z, 2.0 / 3.0);
  R = R * z;
  /* 2s = f - s*f  =>  log(1+f) = f - s*(f - R) */
  double dk = (double)e;
  return dk * DM_LN2_HI + (f + (dk * DM_LN2_LO - s * (f - R)));
}
DHMC_HDH double dm_log(double x) { return dm_log_inl(x); }

/* log1p via Kahan's correction; |error| a few ulp, deterministic. */
DHMC_HD double dm_log1p(double x) {
  double u = 1.0 + x;
  if (u == 1.0) return x;
  if (!dm_isfinite(u)) return dm_log(u);
  return dm_log(u) * (x / (u - 1.0));
}

/* x^y for x > 0 (DualAveraging: m^(-kappa), src/stepsize.jl:154) */
DHMC_HD double dm_pow(double x, double y) { return dm_exp(y * dm_log(x)); }

/* softplus(-d) = log(1 + exp(-d)) for d >= 0 — the only transcendental on the tree's
 * per-merge critical path (logaddexp of log weights / acceptance sums).  Table driven, no
 * division: exp(-d) = 2^k * T[j] * exp(r) with |r| <= ln2/128, then log(u), u = 1 + t in
 * (1,2), = logc[i] + log1p(u*invc[i] - 1) over 128 intervals, plus the rounding error of u.
 * Absolute error ~1e-16 (it is always ADDED to max(a,b)); deterministic like the rest. */
#include "dhmc_tables.h"
static const double dm_h_exp2[64] = DM_TAB_EXP2_INIT;
static const double dm_h_invc[128] = DM_TAB_INVC_INIT;
static const double dm_h_logc[128] = DM_TAB_LOGC_INIT;
#if defined(__CUDACC__)
static __constant__ double dm_d_exp2[64] = DM_TAB_EXP2_INIT;
static __constant__ double dm_d_invc[128] = DM_TAB_INVC_INIT;
static __constant__ double dm_d_logc[128] = DM_TAB_LOGC_INIT;
#endif
#if defined(__CUDA_ARCH__)
#define DM_TAB(name, i) dm_d_##name[i]
#else
#define DM_TAB(name, i) dm_h_##name[i]
#endif
/* Body shared by the two entry points below: TE(j), TI(i), TL(i) read the exp2 / invc / logc tables;
 * *t_out receives exp(-d) (it is a by-product: the logistic model's σ(η) reuses it). */
#define DM_SOFTPLUS_NEG_BODY(TE, TI, TL)                                                        \
  if (d != d) { *t_out = d; return d; }                                                         \
  if (d == 0.0) { *t_out = 1.0; return DM_LN2; }                                                \
  if (d > 745.2) { *t_out = 0.0; return 0.0; }                                                  \
  const double x = -d;                                                                          \
  const double kd = dm_floor(x * DM_64_INVLN2 + 0.5);                                           \
  const int n = (int)kd;                                                                        \
  double r = dm_fma(kd, -DM_LN2_64_HI, x);        /* kd * HI is exact */                        \
  r = dm_fma(kd, -DM_LN2_64_LO, r);               /* |r| <= ln2/128 */                          \
  const int j = n & 63, k = n >> 6;               /* n = 64 k + j, 0 <= j < 64 */               \
  double p = 1.0 / 120.0;                                                                       \
  p = dm_fma(p, r, 1.0 / 24.0);                                                                 \
  p = dm_fma(p, r, 1.0 / 6.0);                                                                  \
  p = dm_fma(p, r, 0.5);                                                                        \
  p = dm_fma(p * r, r, r);                        /* expm1(r) */                                \
  const double tj = TE(j);                                                                      \
  const double y = dm_fma(tj, p, tj);             /* 2^(j/64) e^r */                            \
  const int k1 = k / 2, k2 = k - k1;                                                            \
  const double t = (y * dm_pow2i(k1)) * dm_pow2i(k2);   /* exp(-d) */                           \
  *t_out = t;                                                                                   \
  if (d > 36.7368005696771) return t;             /* 1 + t == 1: log1p(t) = t */                \
  const double u = 1.0 + t;                                                                     \
  if (u >= 2.0) return DM_LN2;                                                                  \
  const int i = (int)((dm_bits(u) >> 45) & 127u);                                               \
  const double ic = TI(i);                                                                      \
  const double rr = dm_fma(u, ic, -1.0);          /* |rr| <~ 2^-8 */                            \
  double q = -1.0 / 6.0;                                                                        \
  q = dm_fma(q, rr, 1.0 / 5.0);                                                                 \
  q = dm_fma(q, rr, -1.0 / 4.0);                                                                \
  q = dm_fma(q, rr, 1.0 / 3.0);                                                                 \
  q = dm_fma(q, rr, -0.5);                                                                      \
  q = dm_fma(q * rr, rr, rr);                     /* log1p(rr) */                               \
  const double c = t - (u - 1.0);                 /* rounding error of u, exact */              \
  return TL(i) + dm_fma(c, ic, q);

#define DM_TE_DEFAULT(j) DM_TAB(exp2, j)
#define DM_TI_DEFAULT(i) DM_TAB(invc, i)
#define DM_TL_DEFAULT(i) DM_TAB(logc, i)
/* softplus(-d) and exp(-d); tables from constant memory on the device (uniform indices: one access) */
DHMC_HD double dm_softplus_neg_exp_inl(double d, double* t_out) {
  DM_SOFTPLUS_NEG_BODY(DM_TE_DEFAULT, DM_TI_DEFAULT, DM_TL_DEFAULT)
}
DHMC_HDH double dm_softplus_neg_exp(double d, double* t_out) { return dm_softplus_neg_exp_inl(d, t_out); }
DHMC_HD double dm_softplus_neg(double d) {
  double t;
  return dm_softplus_neg_exp(d, &t);
}
/* Same arithmetic with the tables behind a pointer, [exp2 (64) | invc (128) | logc (128)] — for code whose
 * lanes look up DIFFERENT entries (a copy in shared memory avoids the serialised constant-cache accesses). */
#define DM_TABS_DOUBLES 320
#define DM_TE_PTR(j) tabs[j]
#define DM_TI_PTR(i) tabs[64 + (i)]
#define DM_TL_PTR(i) tabs[192 + (i)]
DHMC_HD double dm_softplus_neg_exp_tabs(double d, double* t_out, const double* tabs) {
  DM_SOFTPLUS_NEG_BODY(DM_TE_PTR, DM_TI_PTR, DM_TL_PTR)
}
/* the default tables as one array in the layout above (host side: static data; device: constant memory) */
DHMC_HD double dm_tabs_entry(int i) {
  return i < 64 ? DM_TAB(exp2, i) : i < 192 ? DM_TAB(invc, i - 64) : DM_TAB(logc, i - 192);
}

/* log(exp(a)+exp(b)), LogExpFunctions.logaddexp semantics
 * (call sites src/trees.jl:145, src/NUTS.jl:70): equal arguments (incl. both
 * -Inf) give a + log(2); otherwise max + log1pexp(-|a-b|).  SFX selects the
 * out-of-line softplus (empty) or its inlined twin (_inl). */
#define DM_LOGADDEXP_BODY(SFX)                                                  \
  double d = (a == b) ? 0.0 : dm_fabs(a - b);                                   \
  double mx = dm_max_nan(a, b);                                                 \
  double t;                                                                     \
  return mx + dm_softplus_neg_exp##SFX(d, &t);
DHMC_HD double dm_logaddexp(double a, double b) { DM_LOGADDEXP_BODY() }
DHMC_HD double dm_logaddexp_inl(double a, double b) { DM_LOGADDEXP_BODY(_inl) }

/* log(1+exp(x)) (logistic-regression likelihood) */
DHMC_HD double dm_log1pexp(double x) {
  if (x < -36.7368005696771) return dm_exp(x);
  if (x <= 18.021826694558577) return dm_log1p(dm_exp(x));
  if (x <= 33.23111882352963) return x + dm_exp(-x);
  return x;
}

/* -------------------------------------------------- sin/cos of 2*pi*u */
#define DM_PIO4 7.85398163397448309616e-01
/* u in [0,1): returns cos(2 pi u), sin(2 pi u); octant reduction is exact. */
DHMC_HD void dm_sincos2pi_inl(double u, double* sn, double* cs) {
  double a = 8.0 * u;
  double jf = dm_floor(a);
  int j = ((int)jf) & 7;
  double f = a - jf; /* exact, [0,1) */
  if (j & 1) f = 1.0 - f; /* exact */
  double x = f * DM_PIO4;
  double z = x * x;
  /* sin x = x + x*z*S(z), Taylor to x^19 */
  double S = 1.0 / 121645100408832000.0;  /* 1/19! */
  S = dm_fma(S, z, -1.0 / 355687428096000.0); /* -1/17! */
  S = dm_fma(S, z, 1.0 / 1307674368000.0);
  S = dm_fma(S, z, -1.0 / 6227020800.0);
  S = dm_fma(S, z, 1.0 / 39916800.0);
  S = dm_fma(S, z, -1.0 / 362880.0);
  S = dm_fma(S, z, 1.0 / 5040.0);
  S = dm_fma(S, z, -1.0 / 120.0);
  S = dm_fma(S, z, 1.0 / 6.0);
  double s = dm_fma(-(x * z), S, x);
  /* cos x = 1 - z/2 + z^2*C(z), Taylor to x^20 */
  double C = 1.0 / 2432902008176640000.0; /* 1/20! */
  C = dm_fma(C, z, -1.0 / 6402373705728000.0); /* -1/18! */
  C = dm_fma(C, z, 1.0 / 20922789888000.0);
  C = dm_fma(C, z, -1.0 / 87178291200.0);
  C = dm_fma(C, z, 1.0 / 479001600.0);
  C = dm_fma(C, z, -1.0 / 3628800.0);
  C = dm_fma(C, z, 1.0 / 40320.0);
  C = dm_fma(C, z, -1.0 / 720.0);
  C = dm_fma(C, z, 1.0 / 24.0);
  double c = dm_fma(z * z, C, dm_fma(-0.5, z, 1.0));
  double ss, cc;
  switch (j) {
    case 0: cc = c;  ss = s;  break;
    case 1: cc = s;  ss = c;  break;
    case 2: cc = -s; ss = c;  break;
    case 3: cc = -c; ss = s;  break;
    case 4: cc = -c; ss = -s; break;
    case 5: cc = -s; ss = -c; break;
    case 6: cc = s;  ss = -c; break;
    default: cc = c; ss = -s; break;
  }
  *sn = ss; *cs = cc;
}
DHMC_HDH void dm_sincos2pi(double u, double* sn, double* cs) { dm_sincos2pi_inl(u, sn, cs); }

/* ------------------------------------------------------- Philox-4x32-10 */
typedef struct { uint32_t v[4]; } dm_u32x4;

DHMC_HD uint32_t dm_mulhi32(uint32_t a, uint32_t b) {
#if defined(__CUDA_ARCH__)
  return __umulhi(a, b);
#else
  return (uint32_t)(((uint64_t)a * (uint64_t)b) >> 32);
#endif
}

DHMC_HD dm_u32x4 dm_philox4x32_10_inl(uint32_t c0, uint32_t c1, uint32_t c2,
                                      uint32_t c3, uint32_t k0, uint32_t k1) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u;
  const uint32_t W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0 = dm_mulhi32(M0, c0), lo0 = M0 * c0;
    uint32_t hi1 = dm_mulhi32(M1, c2), lo1 = M1 * c2;
    uint32_t n0 = hi1 ^ c1 ^ k0;
    uint32_t n2 = hi0 ^ c3 ^ k1;
    c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
    k0 += W0; k1 += W1;
  }
  dm_u32x4 o;
  o.v[0] = c0; o.v[1] = c1; o.v[2] = c2; o.v[3] = c3;
  return o;
}
DHMC_HDH dm_u32x4 dm_philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2,
                                   uint32_t c3, uint32_t k0, uint32_t k1) {
  return dm_philox4x32_10_inl(c0, c1, c2, c3, k0, k1);
}

/* RNG streams: one Philox block = (idx, transition, chain_lo, stream|chain_hi) */
enum {
  DHMC_STREAM_Q0 = 0,      /* random_position, mcmc.jl:108 */
  DHMC_STREAM_PSEARCH = 1, /* momentum of the step-size search, mcmc.jl:138 */
  DHMC_STREAM_P = 2,       /* rand_p per transition, NUTS.jl:233 */
  DHMC_STREAM_DIR = 3,     /* Directions per transition, NUTS.jl:233 */
  DHMC_STREAM_EXP = 4,     /* randexp draws in merge order, NUTS.jl:44 */
  DHMC_STREAM_GQ_U = 5,    /* uniforms of random generated quantities (dhmc_gq_uniform); the sampler never reads it */
  DHMC_STREAM_GQ_N = 6     /* normals of random generated quantities (dhmc_gq_normal); the sampler never reads it */
};

typedef struct {
  uint32_t k0, k1;       /* seed */
  uint32_t chain_lo;     /* global chain id, low 32 bits */
  uint32_t chain_hi24;   /* global chain id, bits 32..55 */
} dm_rng_key;

DHMC_HD dm_rng_key dm_make_key(uint64_t seed, uint64_t chain) {
  dm_rng_key k;
  k.k0 = (uint32_t)seed; k.k1 = (uint32_t)(seed >> 32);
  k.chain_lo = (uint32_t)chain;
  k.chain_hi24 = (uint32_t)((chain >> 32) & 0xFFFFFFu);
  return k;
}
/* The composites below come in the same two forms: SFX empty calls the out-of-line bodies, SFX = _inl their twins. */
#define DM_RNG_BLOCK_BODY(SFX)                                                  \
  return dm_philox4x32_10##SFX(idx, t, k.chain_lo, (stream << 24) | k.chain_hi24, k.k0, k.k1);
DHMC_HD dm_u32x4 dm_rng_block(dm_rng_key k, uint32_t stream, uint32_t t,
                               uint32_t idx) { DM_RNG_BLOCK_BODY() }
DHMC_HD dm_u32x4 dm_rng_block_inl(dm_rng_key k, uint32_t stream, uint32_t t,
                                   uint32_t idx) { DM_RNG_BLOCK_BODY(_inl) }
/* 52-bit uniform strictly inside (0,1): (n + 1/2) * 2^-52, exact */
DHMC_HD double dm_u01(uint32_t a, uint32_t b) {
  uint64_t n = ((uint64_t)a << 20) | (uint64_t)(b >> 12);
  return ((double)n + 0.5) * 2.220446049250313e-16;
}
/* Standard normals for elements (2j, 2j+1) of a D-vector: Box-Muller. */
DHMC_HD void dm_normal_pair(dm_rng_key k, uint32_t stream, uint32_t t,
                            uint32_t j, double* z0, double* z1) {
  dm_u32x4 r = dm_rng_block(k, stream, t, j);
  double u1 = dm_u01(r.v[0], r.v[1]);
  double u2 = dm_u01(r.v[2], r.v[3]);
  double rad = dm_sqrt(-2.0 * dm_log(u1));
  double sn, cs;
  dm_sincos2pi(u2, &sn, &cs);
  *z0 = rad * cs; *z1 = rad * sn;
}
/* n independent pairs at once, z0[h], z1[h] for pair j[h]: each pair takes exactly the operations of dm_normal_pair (inlined
 * bodies), but the Philox blocks, the logs and the sin/cos of all pairs are evaluated stage by stage, so that the n
 * dependency chains can overlap instead of running one after the other. */
DHMC_HD void dm_normal_pairs_inl(dm_rng_key k, uint32_t stream, uint32_t t, const uint32_t* j, int n,
                                 double* z0, double* z1) {
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
  for (int h = 0; h < n; ++h) {
    dm_u32x4 r = dm_rng_block_inl(k, stream, t, j[h]);
    z0[h] = dm_u01(r.v[0], r.v[1]);                                          /* u1 */
    z1[h] = dm_u01(r.v[2], r.v[3]);                                          /* u2 */
  }
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
  for (int h = 0; h < n; ++h) z0[h] = dm_sqrt(-2.0 * dm_log_inl(z0[h]));     /* rad */
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
  for (int h = 0; h < n; ++h) {
    double sn, cs;
    dm_sincos2pi_inl(z1[h], &sn, &cs);
    const double rad = z0[h];
    z0[h] = rad * cs; z1[h] = rad * sn;
  }
}
DHMC_HD double dm_normal_elem(dm_rng_key k, uint32_t stream, uint32_t t,
                              uint32_t i) {
  double z0, z1;
  dm_normal_pair(k, stream, t, i >> 1, &z0, &z1);
  return (i & 1u) ? z1 : z0;
}
/* Uniform (0,1) for element i (two per block). */
DHMC_HD double dm_uniform_elem(dm_rng_key k, uint32_t stream, uint32_t t,
                               uint32_t i) {
  dm_u32x4 r = dm_rng_block(k, stream, t, i >> 1);
  return (i & 1u) ? dm_u01(r.v[2], r.v[3]) : dm_u01(r.v[0], r.v[1]);
}
/* The j-th randexp of transition t: -log(u). */
DHMC_HD double dm_randexp(dm_rng_key k, uint32_t t, uint32_t j) {
  dm_u32x4 r = dm_rng_block(k, DHMC_STREAM_EXP, t, j >> 1);
  double u = (j & 1u) ? dm_u01(r.v[2], r.v[3]) : dm_u01(r.v[0], r.v[1]);
  return -dm_log(u);
}
DHMC_HD uint32_t dm_rand_directions(dm_rng_key k, uint32_t t) {
  return dm_rng_block(k, DHMC_STREAM_DIR, t, 0).v[0];
}

/* Random numbers of random generated quantities (include/dhmc_models.h, DHMC_USER_GENERATED_RNG): the key of one draw is
 * (seed, global chain id) and the transition counter t of the transition that produced it.  uniform(i) and normal(i) are
 * pure functions of (key, t, i): every quantity of a draw that asks for index i gets the same number, different indices
 * are independent, uniforms and normals come from different streams (no shared bits), and neither stream is read by the
 * sampler.  Host and device give the same bits. */
typedef struct {
  dm_rng_key key;
  uint32_t t;
} dhmc_gq_rng;
DHMC_HD double dhmc_gq_uniform(const dhmc_gq_rng* r, uint32_t i) { return dm_uniform_elem(r->key, DHMC_STREAM_GQ_U, r->t, i); }
DHMC_HD double dhmc_gq_normal(const dhmc_gq_rng* r, uint32_t i) { return dm_normal_elem(r->key, DHMC_STREAM_GQ_N, r->t, i); }

#endif /* DHMC_MATH_H */
