// dmma_order_probe.cu — which summation order does mma.sync.m8n8k4.f64 use on sm_90a?
//
// Round-2 preparation (DESIGN.md §7, item (i)): the cooperative logistic likelihood is a
// [rows × p]·[p × 8 chains] product, the shape of the FP64 tensor-core MMA.  To keep the oracle
// bit-exact it has to restate the instruction's accumulation order, so this probe compares the
// instruction against candidate orders on adversarial random inputs and reports the match counts.
//
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O2 -fmad=false -o dmma_order_probe dmma_order_probe.cu
// Run: ./dmma_order_probe [trials]
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

// One warp: D[8x8] = A[8x4] · B[4x8] + C[8x8].  Fragment layout (PTX ISA, m8n8k4 .f64):
// A: lane holds A[lane>>2][lane&3]; B: lane holds B[lane&3][lane>>2];
// C/D: lane holds rows lane>>2, columns 2·(lane&3) and 2·(lane&3)+1.
__global__ void k_dmma(const double* A, const double* B, const double* C, double* D, int n) {
  const int lane = threadIdx.x & 31;
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (w >= n) return;
  const double a = A[(size_t)w * 32 + (lane >> 2) * 4 + (lane & 3)];
  const double b = B[(size_t)w * 32 + (lane & 3) * 8 + (lane >> 2)];
  const int r = lane >> 2, c0 = 2 * (lane & 3);
  double c_0 = C[(size_t)w * 64 + r * 8 + c0], c_1 = C[(size_t)w * 64 + r * 8 + c0 + 1];
  double d0, d1;
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%4,%5};"
               : "=d"(d0), "=d"(d1)
               : "d"(a), "d"(b), "d"(c_0), "d"(c_1));
  D[(size_t)w * 64 + r * 8 + c0] = d0;
  D[(size_t)w * 64 + r * 8 + c0 + 1] = d1;
}

static uint64_t s_state = 0x9E3779B97F4A7C15ull;
static uint64_t rnd() {
  s_state ^= s_state << 7; s_state ^= s_state >> 9;
  return s_state * 0x2545F4914F6CDD1Dull;
}
// random double with an exponent spread that makes the order of additions visible
static double rnd_double() {
  const double m = 1.0 + (double)(rnd() >> 11) * (1.0 / 9007199254740992.0);
  const int e = (int)(rnd() % 61) - 30;
  return ((rnd() & 1) ? -m : m) * std::ldexp(1.0, e);
}

int main(int argc, char** argv) {
  const int n = argc > 1 ? std::atoi(argv[1]) : 20000;
  std::vector<double> A((size_t)n * 32), B((size_t)n * 32), C((size_t)n * 64), D((size_t)n * 64);
  for (auto& v : A) v = rnd_double();
  for (auto& v : B) v = rnd_double();
  for (auto& v : C) v = rnd_double();
  double *dA, *dB, *dC, *dD;
  cudaMalloc(&dA, A.size() * 8); cudaMalloc(&dB, B.size() * 8);
  cudaMalloc(&dC, C.size() * 8); cudaMalloc(&dD, D.size() * 8);
  cudaMemcpy(dA, A.data(), A.size() * 8, cudaMemcpyHostToDevice);
  cudaMemcpy(dB, B.data(), B.size() * 8, cudaMemcpyHostToDevice);
  cudaMemcpy(dC, C.data(), C.size() * 8, cudaMemcpyHostToDevice);
  k_dmma<<<(n * 32 + 127) / 128, 128>>>(dA, dB, dC, dD, n);
  if (cudaMemcpy(D.data(), dD, D.size() * 8, cudaMemcpyDeviceToHost) != cudaSuccess) {
    std::printf("CUDA error: %s\n", cudaGetErrorString(cudaGetLastError()));
    return 1;
  }
  const char* names[] = {"sequential fma k=0..3 onto c", "sequential fma k=3..0 onto c",
                         "pairwise: fma(a0,b0,a1*b1)+fma(a2,b2,a3*b3), then + c",
                         "exact sum rounded once (float128)", "separately rounded mul/add k=0..3"};
  long match[5] = {0, 0, 0, 0, 0}, total = 0;
  for (int w = 0; w < n; ++w)
    for (int i = 0; i < 8; ++i)
      for (int j = 0; j < 8; ++j) {
        const double* a = &A[(size_t)w * 32 + i * 4];
        double b[4];
        for (int k = 0; k < 4; ++k) b[k] = B[(size_t)w * 32 + k * 8 + j];
        const double c = C[(size_t)w * 64 + i * 8 + j], d = D[(size_t)w * 64 + i * 8 + j];
        double r0 = c, r1 = c;
        for (int k = 0; k < 4; ++k) r0 = std::fma(a[k], b[k], r0);
        for (int k = 3; k >= 0; --k) r1 = std::fma(a[k], b[k], r1);
        const double r2 = (std::fma(a[0], b[0], a[1] * b[1]) + std::fma(a[2], b[2], a[3] * b[3])) + c;
        __float128 q = (__float128)c;
        for (int k = 0; k < 4; ++k) q += (__float128)a[k] * (__float128)b[k];
        const double r3 = (double)q;
        double r4 = c;
        for (int k = 0; k < 4; ++k) { volatile double pr = a[k] * b[k]; r4 = r4 + pr; }
        const double cand[5] = {r0, r1, r2, r3, r4};
        for (int m = 0; m < 5; ++m) match[m] += (cand[m] == d);
        ++total;
      }
  std::printf("mma.sync.m8n8k4.f64 on %d random 8x8x4 problems (%ld outputs)\n", n, total);
  for (int m = 0; m < 5; ++m) std::printf("  %-58s %ld / %ld\n", names[m], match[m], total);
  return 0;
}
