// family_tu.cu — instantiates the kernels of ONE log-density family (and one part of it) per
// translation unit so that the library builds in parallel: nvcc -DDHMC_TU_FAM=<0..3> -DDHMC_TU_PART=<0, 1, 3>
// (kernels.cuh: kernel_ptr).
// The host side (dhmc_b200.cu) reaches the kernels through dhmc_family_kernel_<fam>_<part>().
#include "kernels.cuh"

#ifndef DHMC_TU_FAM
#error "compile with -DDHMC_TU_FAM=<family id> -DDHMC_TU_PART=<part>"
#endif
#define DHMC_CAT3(a, b, c) a##b##_##c
#define DHMC_TU_NAME(f, p) DHMC_CAT3(dhmc_family_kernel_, f, p)

__attribute__((visibility("hidden"))) const void* DHMC_TU_NAME(DHMC_TU_FAM, DHMC_TU_PART)(int W, int epl, int kernel, int dense) {
  return dhmc::family_kernel_ptr<DHMC_TU_FAM, DHMC_TU_PART>(W, epl, (dhmc::KernelId)kernel, dense != 0);
}

// USER family (include/dhmc_models.h): `make user USER_HEADER=…` compiles this file with -DDHMC_TU_FAM=4 and
// -DDHMC_USER_MODEL_HEADER='"…"'; the host side reaches the two parts through weak references.
#if DHMC_TU_FAM == 4
#ifndef DHMC_HAVE_USER_FAMILY
#error "family 4 is the USER family: compile with -DDHMC_USER_MODEL_HEADER='\"/path/to/model.h\"'"
#endif
#if DHMC_TU_PART == 0
extern "C" __attribute__((visibility("hidden"))) const void* dhmc_user_family_kernel_0(int W, int epl, int kernel, int dense) {
  return dhmc::family_kernel_ptr<DHMC_FAMILY_USER, 0>(W, epl, (dhmc::KernelId)kernel, dense != 0);
}
extern "C" __attribute__((visibility("hidden"))) const char* dhmc_user_family_name_str(void) { return DHMC_USER_NAME; }
extern "C" __attribute__((visibility("hidden"))) int dhmc_user_family_min_dim(void) { return DHMC_USER_MIN_DIM; }
#ifdef DHMC_USER_GENERATED
// Generated quantities at given points (dhmc_generated): one CTA of T threads (the handle's chain width) per point, thread
// tid writing quantities k = tid + e·T.  theta [n_problems][n][D], out [n_problems][n][G]; the points of local problem j
// read the parameter block of problem first + j (problems null: the handle's one problem).  Random quantities
// (DHMC_USER_GENERATED_RNG) take point pt's key from chain [pt] and transition [pt] under `seed`; deterministic ones
// ignore the keys (null).
namespace dhmc {
__global__ void k_generated(const double* theta, long long n, long long n_problems, int D, int ng, const double* mparams,
                            const ProblemDesc* problems, long long first, const long long* chain, const unsigned* transition,
                            unsigned long long seed, double* out) {
  for (long long pt = blockIdx.x; pt < n * n_problems; pt += gridDim.x) {
    const double* params = mparams + (problems ? problems[first + pt / n].mparams : 0);
    const double* q = theta + (size_t)pt * D;
#ifdef DHMC_USER_GENERATED_RNG
    dhmc_gq_rng rng;
    rng.key = dm_make_key(seed, (uint64_t)chain[pt]);
    rng.t = transition[pt];
    for (int k = threadIdx.x; k < ng; k += blockDim.x) out[(size_t)pt * ng + k] = dhmc_user_generated(k, D, q, params, &rng);
#else
    (void)chain; (void)transition; (void)seed;
    for (int k = threadIdx.x; k < ng; k += blockDim.x) out[(size_t)pt * ng + k] = dhmc_user_generated(k, D, q, params);
#endif
  }
}
}  // namespace dhmc
extern "C" __attribute__((visibility("hidden"))) int dhmc_user_family_ngq(int D) { return dhmc_user_ngq(D); }
#ifdef DHMC_USER_GENERATED_RNG
extern "C" __attribute__((visibility("hidden"))) int dhmc_user_family_random(void) { return 1; }
#else
extern "C" __attribute__((visibility("hidden"))) int dhmc_user_family_random(void) { return 0; }
#endif
extern "C" __attribute__((visibility("hidden"))) int dhmc_user_family_generated(const double* theta, long long n, long long n_problems,
                                                                                int D, int ng, const double* mparams, const void* problems,
                                                                                long long first, const long long* chain,
                                                                                const unsigned* transition, unsigned long long seed,
                                                                                double* out, int T, int grid, cudaStream_t stream) {
  dhmc::k_generated<<<grid, T, 0, stream>>>(theta, n, n_problems, D, ng, mparams, (const dhmc::ProblemDesc*)problems, first, chain,
                                            transition, seed, out);
  return (int)cudaGetLastError();
}
#endif
#elif DHMC_TU_PART == 3
extern "C" __attribute__((visibility("hidden"))) const void* dhmc_user_family_kernel_3(int W, int epl, int kernel, int dense) {
  return dhmc::family_kernel_ptr<DHMC_FAMILY_USER, 3>(W, epl, (dhmc::KernelId)kernel, dense != 0);
}
#endif
#endif
