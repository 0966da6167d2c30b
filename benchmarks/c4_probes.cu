// c4_probes.cu — round-2 hardware probes behind the C4 (logistic regression) kernel design.
//
//   1. FP64 tensor-core rate and latency on sm_90a for mma.sync .f64 shapes m8n8k4 / m16n8k4 /
//      m16n8k8 / m16n8k16, next to the plain DFMA rate (is DMMA worth it, which shape, how many
//      independent accumulator chains per warp hide the latency);
//   2. the same m8n8k4 stream with its A fragment fetched from shared memory per instruction
//      (conflict-free stride ≡ 4 mod 16 doubles), the inner loop of the likelihood round;
//   3. L2 → SM delivery when every SM sweeps the same 20 MB design matrix with cp.async.bulk
//      (mbarrier complete_tx ring), all SMs in step vs. skewed starts vs. cluster-2 multicast.
//
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o c4_probes c4_probes.cu
// Run: ./c4_probes (one CTA per SM of device 0)
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

static int g_sms = 0;   // SMs of device 0: one CTA each

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { std::printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); std::exit(1); } } while (0)

// ------------------------------------------------------------------ 1. MMA / FMA rate
template <int SHAPE>   // 0: m8n8k4, 1: m16n8k4, 2: m16n8k8, 3: m16n8k16, 9: DFMA (one warp-wide FMA)
struct Mma {
  static constexpr int NA = SHAPE == 0 ? 1 : SHAPE == 1 ? 2 : SHAPE == 2 ? 4 : SHAPE == 3 ? 8 : 1;
  static constexpr int NB = SHAPE == 0 ? 1 : SHAPE == 1 ? 1 : SHAPE == 2 ? 2 : SHAPE == 3 ? 4 : 1;
  static constexpr int NC = SHAPE == 0 ? 2 : SHAPE == 9 ? 1 : 4;
  static constexpr int FMAS = SHAPE == 0 ? 256 : SHAPE == 1 ? 512 : SHAPE == 2 ? 1024 : SHAPE == 3 ? 2048 : 32;
  __device__ static __forceinline__ void run(double (&c)[NC], const double (&a)[NA], const double (&b)[NB]) {
    if constexpr (SHAPE == 0)
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                   : "+d"(c[0]), "+d"(c[1]) : "d"(a[0]), "d"(b[0]));
    else if constexpr (SHAPE == 1)
      asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                   : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a[0]), "d"(a[1]), "d"(b[0]));
    else if constexpr (SHAPE == 2)
      asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                   : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                   : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
    else if constexpr (SHAPE == 3)
      asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, {%0,%1,%2,%3};"
                   : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                   : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
                     "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
    else
      asm volatile("fma.rn.f64 %0, %1, %2, %0;" : "+d"(c[0]) : "d"(a[0]), "d"(b[0]));
  }
};

template <int SHAPE, int CH>
__global__ void __launch_bounds__(1024, 1) k_rate(double* sink, long long* cycles, int iters) {
  using M = Mma<SHAPE>;
  double a[M::NA], b[M::NB], c[CH][M::NC];
  for (int i = 0; i < M::NA; ++i) a[i] = 1.0 + 1e-9 * (threadIdx.x + i);
  for (int i = 0; i < M::NB; ++i) b[i] = 1.0 - 1e-9 * (threadIdx.x + i);
  for (int ch = 0; ch < CH; ++ch)
    for (int i = 0; i < M::NC; ++i) c[ch][i] = (double)(ch + i);
  __syncthreads();
  const long long t0 = clock64();
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int ch = 0; ch < CH; ++ch) M::run(c[ch], a, b);
  }
  const long long t1 = clock64();
  double s = 0;
  for (int ch = 0; ch < CH; ++ch)
    for (int i = 0; i < M::NC; ++i) s += c[ch][i];
  if (s == 12345.678) sink[0] = s;
  if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

template <int SHAPE, int CH>
static void rate(const char* name, int warps, double* sink, long long* dcyc) {
  const int iters = 4096;
  k_rate<SHAPE, CH><<<g_sms, 32 * warps>>>(sink, dcyc, 64);
  CK(cudaDeviceSynchronize());
  k_rate<SHAPE, CH><<<g_sms, 32 * warps>>>(sink, dcyc, iters);
  CK(cudaDeviceSynchronize());
  std::vector<long long> cyc(g_sms);
  CK(cudaMemcpy(cyc.data(), dcyc, g_sms * sizeof(long long), cudaMemcpyDeviceToHost));
  double mean = 0;
  for (auto v : cyc) mean += (double)v;
  mean /= g_sms;
  const double per_instr_warp = mean / ((double)iters * CH);                 // cycles between a warp's issues
  const double per_smsp = mean / ((double)iters * CH * ((warps + 3) / 4));   // cycles per instruction per SMSP
  const double fma_per_clk_sm = (double)Mma<SHAPE>::FMAS * iters * CH * warps / mean;
  std::printf("rate %-9s warps/SM %2d chains/warp %d : %7.2f clk/instr/warp  %6.2f clk/instr/SMSP  %7.1f FMA/clk/SM\n",
              name, warps, CH, per_instr_warp, per_smsp, fma_per_clk_sm);
}

// ------------------------------------------------------------------ 2. m8n8k4 fed from shared memory
// A fragment = tile[(k0 + lane&3) * XS + row0 + (lane>>2)]: the phase-2 access of the likelihood round;
// B fragment constant.  CH accumulator chains = CH different row blocks of the same k-step.
template <int CH>
__global__ void __launch_bounds__(512, 1) k_rate_lds(double* sink, long long* cycles, int iters) {
  extern __shared__ double tile[];
  constexpr int XS = 260;                   // ≡ 4 mod 16
  constexpr int ROWS = 64;
  for (int i = threadIdx.x; i < ROWS * XS; i += blockDim.x) tile[i] = 1.0 + 1e-9 * i;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int fr = lane >> 2, fk = lane & 3;
  double c[CH][2];
  for (int ch = 0; ch < CH; ++ch) { c[ch][0] = ch; c[ch][1] = -ch; }
  const double b = 1.0 - 1e-9 * lane;
  const long long t0 = clock64();
  for (int it = 0; it < iters; ++it) {
    const double* base = tile + ((it & 15) * 4 + fk) * XS + fr + (warp & 1) * 8;
#pragma unroll
    for (int ch = 0; ch < CH; ++ch) {
      const double a = base[ch * 16];
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                   : "+d"(c[ch][0]), "+d"(c[ch][1]) : "d"(a), "d"(b));
    }
  }
  const long long t1 = clock64();
  double s = 0;
  for (int ch = 0; ch < CH; ++ch) s += c[ch][0] + c[ch][1];
  if (s == 12345.678) sink[0] = s;
  if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}
template <int CH>
static void rate_lds(int warps, double* sink, long long* dcyc) {
  const int iters = 4096;
  const size_t smem = 64 * 260 * sizeof(double);
  CK(cudaFuncSetAttribute(k_rate_lds<CH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_rate_lds<CH><<<g_sms, 32 * warps, smem>>>(sink, dcyc, 64);
  CK(cudaDeviceSynchronize());
  k_rate_lds<CH><<<g_sms, 32 * warps, smem>>>(sink, dcyc, iters);
  CK(cudaDeviceSynchronize());
  std::vector<long long> cyc(g_sms);
  CK(cudaMemcpy(cyc.data(), dcyc, g_sms * sizeof(long long), cudaMemcpyDeviceToHost));
  double mean = 0;
  for (auto v : cyc) mean += (double)v;
  mean /= g_sms;
  std::printf("rate m8n8k4+LDS.64 warps/SM %2d chains/warp %d : %6.2f clk/instr/SMSP  %7.1f FMA/clk/SM\n", warps, CH,
              mean / ((double)iters * CH * ((warps + 3) / 4)), 256.0 * iters * CH * warps / mean);
}

// ------------------------------------------------------------------ 3. L2 → SM sweep with cp.async.bulk
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n.reg .pred p;\nWAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\nbra WAIT_%=;\nDONE_%=:\n}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void bulk_g2s_mc(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint16_t mask) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)), "h"(mask) : "memory");
}

constexpr int kStages = 4;
constexpr int kTileBytes = 32768;
// every CTA sweeps buf[0 .. bytes) `sweeps` times, starting at tile (skew · blockIdx) mod ntiles
__global__ void __launch_bounds__(256, 1) k_sweep(const char* buf, size_t bytes, int sweeps, int skew, double* sink,
                                                  long long* cycles) {
  extern __shared__ __align__(128) unsigned char sm[];
  uint64_t* full = reinterpret_cast<uint64_t*>(sm);
  uint64_t* empty = full + kStages;
  unsigned char* tiles = sm + 128;
  const int ntiles = (int)(bytes / kTileBytes);
  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, blockDim.x / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int total = ntiles * sweeps;
  const int start = (int)(((long long)skew * blockIdx.x) % ntiles);
  const long long t0 = clock64();
  double acc = 0;
  if (threadIdx.x == 0) {   // producer and consumer roles interleaved in one thread for the issue, all threads consume
    for (int t = 0; t < kStages && t < total; ++t) {
      mbar_expect_tx(full + t, kTileBytes);
      bulk_g2s(tiles + (size_t)t * kTileBytes, buf + (size_t)((start + t) % ntiles) * kTileBytes, kTileBytes, full + t);
    }
  }
  for (int t = 0; t < total; ++t) {
    const int s = t % kStages;
    const uint32_t ph = (uint32_t)((t / kStages) & 1);
    mbar_wait(full + s, ph);
    const double* d = reinterpret_cast<const double*>(tiles + (size_t)s * kTileBytes);
    acc += d[threadIdx.x];                               // touch the tile
    __syncwarp();
    if ((threadIdx.x & 31) == 0) mbar_arrive(empty + s);
    if (threadIdx.x == 0 && t + kStages < total) {
      mbar_wait(empty + s, ph);
      mbar_expect_tx(full + s, kTileBytes);
      bulk_g2s(tiles + (size_t)s * kTileBytes, buf + (size_t)((start + t + kStages) % ntiles) * kTileBytes, kTileBytes, full + s);
    }
  }
  const long long t1 = clock64();
  if (acc == 12345.678) sink[0] = acc;
  if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

// cluster of 2: each CTA fetches half of every tile and multicasts it to both
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(256, 1)
k_sweep_mc(const char* buf, size_t bytes, int sweeps, int skew, double* sink, long long* cycles) {
  extern __shared__ __align__(128) unsigned char sm[];
  uint64_t* full = reinterpret_cast<uint64_t*>(sm);
  uint64_t* empty = full + kStages;      // counts the warps of BOTH CTAs (remote arrives)
  unsigned char* tiles = sm + 128;
  uint32_t rank;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
  const int ntiles = (int)(bytes / kTileBytes);
  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, 2 * (blockDim.x / 32)); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  asm volatile("barrier.cluster.arrive.release.aligned;\nbarrier.cluster.wait.acquire.aligned;" ::: "memory");
  const int total = ntiles * sweeps;
  const int start = (int)(((long long)skew * (blockIdx.x / 2)) % ntiles);
  const int half = kTileBytes / 2;
  const long long t0 = clock64();
  double acc = 0;
  auto issue = [&](int t) {
    const int s = t % kStages;
    mbar_expect_tx(full + s, kTileBytes);   // both halves land in this CTA's stage
    bulk_g2s_mc(tiles + (size_t)s * kTileBytes + rank * half,
                buf + (size_t)((start + t) % ntiles) * kTileBytes + rank * half, half, full + s, (uint16_t)3);
  };
  if (threadIdx.x == 0)
    for (int t = 0; t < kStages && t < total; ++t) issue(t);
  for (int t = 0; t < total; ++t) {
    const int s = t % kStages;
    const uint32_t ph = (uint32_t)((t / kStages) & 1);
    mbar_wait(full + s, ph);
    const double* d = reinterpret_cast<const double*>(tiles + (size_t)s * kTileBytes);
    acc += d[threadIdx.x];
    __syncwarp();
    if ((threadIdx.x & 31) == 0) {
      // release the stage in both CTAs: the peer's producer writes into OUR stage as well
      const uint32_t local = smem_u32(empty + s);
#pragma unroll
      for (uint32_t r = 0; r < 2; ++r) {
        uint32_t remote;
        asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local), "r"(r));
        asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
      }
    }
    if (threadIdx.x == 0 && t + kStages < total) {
      mbar_wait(empty + s, ph);
      issue(t + kStages);
    }
  }
  const long long t1 = clock64();
  asm volatile("barrier.cluster.arrive.release.aligned;\nbarrier.cluster.wait.acquire.aligned;" ::: "memory");
  if (acc == 12345.678) sink[0] = acc;
  if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

static void sweep(const char* buf, size_t bytes, int sweeps, int skew, bool mc, double* sink, long long* dcyc) {
  const size_t smem = 128 + (size_t)kStages * kTileBytes;
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  float ms = 0;
  for (int rep = 0; rep < 2; ++rep) {
    CK(cudaEventRecord(e0));
    if (mc) {
      CK(cudaFuncSetAttribute(k_sweep_mc, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      k_sweep_mc<<<g_sms, 256, smem>>>(buf, bytes, sweeps, skew, sink, dcyc);
    } else {
      CK(cudaFuncSetAttribute(k_sweep, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      k_sweep<<<g_sms, 256, smem>>>(buf, bytes, sweeps, skew, sink, dcyc);
    }
    CK(cudaEventRecord(e1));
    CK(cudaDeviceSynchronize());
    CK(cudaEventElapsedTime(&ms, e0, e1));
  }
  const double tb = (double)g_sms * (double)bytes * sweeps / (ms * 1e-3) / 1e12;
  std::printf("sweep %-9s buf %5.1f MB x%d skew %4d : %8.3f ms  %6.2f TB/s delivered to the SMs (%5.1f GB/s per SM)\n",
              mc ? "cluster2" : "unicast", bytes / 1e6, sweeps, skew, ms, tb, tb * 1e3 / g_sms);
}

int main() {
  double* sink; long long* dcyc;
  CK(cudaDeviceGetAttribute(&g_sms, cudaDevAttrMultiProcessorCount, 0));
  CK(cudaMalloc(&sink, 8)); CK(cudaMalloc(&dcyc, g_sms * sizeof(long long)));
  int clk = 0;
  CK(cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0));
  std::printf("SM clock (max) %d kHz\n", clk);
  std::printf("--- FP64 rates: FMA/clk/SM, 64 = the nominal DFMA rate\n");
  rate<9, 8>("dfma", 4, sink, dcyc);  rate<9, 8>("dfma", 8, sink, dcyc);  rate<9, 8>("dfma", 16, sink, dcyc);
  rate<0, 1>("m8n8k4", 1, sink, dcyc);      // latency
  rate<0, 1>("m8n8k4", 4, sink, dcyc);
  rate<0, 2>("m8n8k4", 4, sink, dcyc);  rate<0, 4>("m8n8k4", 4, sink, dcyc);  rate<0, 8>("m8n8k4", 4, sink, dcyc);
  rate<0, 1>("m8n8k4", 8, sink, dcyc);  rate<0, 2>("m8n8k4", 8, sink, dcyc);  rate<0, 4>("m8n8k4", 8, sink, dcyc);
  rate<0, 1>("m8n8k4", 16, sink, dcyc); rate<0, 2>("m8n8k4", 16, sink, dcyc); rate<0, 4>("m8n8k4", 16, sink, dcyc);
  rate<1, 1>("m16n8k4", 1, sink, dcyc); rate<1, 4>("m16n8k4", 4, sink, dcyc); rate<1, 2>("m16n8k4", 16, sink, dcyc);
  rate<2, 1>("m16n8k8", 1, sink, dcyc); rate<2, 4>("m16n8k8", 4, sink, dcyc); rate<2, 2>("m16n8k8", 16, sink, dcyc);
  rate<3, 1>("m16n8k16", 1, sink, dcyc); rate<3, 4>("m16n8k16", 4, sink, dcyc); rate<3, 2>("m16n8k16", 16, sink, dcyc);
  std::printf("--- m8n8k4 with the A fragment from shared memory\n");
  rate_lds<1>(16, sink, dcyc); rate_lds<2>(16, sink, dcyc); rate_lds<4>(16, sink, dcyc); rate_lds<4>(8, sink, dcyc);
  std::printf("--- L2 -> SM sweeps (cp.async.bulk, 4 x 32 KB ring per SM, %d CTAs)\n", g_sms);
  const size_t bytes = (size_t)20480000 / kTileBytes * kTileBytes;     // X: 10 000 x 256 doubles
  char* buf;
  CK(cudaMalloc(&buf, 2 * bytes));
  CK(cudaMemset(buf, 1, 2 * bytes));
  sweep(buf, bytes, 8, 0, false, sink, dcyc);
  sweep(buf, bytes, 8, 1, false, sink, dcyc);
  sweep(buf, bytes, 8, 37, false, sink, dcyc);
  sweep(buf, 2 * bytes, 4, 37, false, sink, dcyc);
  sweep(buf, bytes, 8, 0, true, sink, dcyc);
  sweep(buf, bytes, 8, 37, true, sink, dcyc);
  return 0;
}
