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
#elif DHMC_TU_PART == 3
extern "C" __attribute__((visibility("hidden"))) const void* dhmc_user_family_kernel_3(int W, int epl, int kernel, int dense) {
  return dhmc::family_kernel_ptr<DHMC_FAMILY_USER, 3>(W, epl, (dhmc::KernelId)kernel, dense != 0);
}
#endif
#endif
