// device_backend.cuh — sm_90a vector backend of the NUTS state machine.
//
// One chain = one chain group of T = 32·W threads (= one CTA; packed chain groups of the
// logistic family put 8 groups in a CTA, see coop_core_tma).  Element i of
// every D-vector belongs to thread (i mod T), register slot e = i div T, so a
// vector is EPL doubles per thread, HBM accesses of a chain row are fully
// coalesced, shared-memory slot accesses are conflict-free, and — because the
// owner of an element never changes — slot traffic needs NO synchronisation:
// the only cross-thread communication is the scalar all-reduce below.
//
// The current phase point (q, p, ∇ℓ), the metric diagonal and the running
// momentum sum ρ of the incoming subtree live in registers for the whole run of
// a chain; the tree's other vectors live in "slots": the first n_sm in shared
// memory, the rest in a per-CTA global scratch arena that stays L2-resident.
//
// Replaces (reference, tpapp/DynamicHMC.jl v3.6.0):
//   leapfrog hamiltonian.jl:273-282, evaluate_ℓ :202-217, logdensity :251-256,
//   kinetic_energy :103, calculate_p♯ :110, rand_p :124,
//   combine_turn_statistics NUTS.jl:132-139 (the six dot products),
//   sample_M⁻¹(Diagonal) mcmc.jl:209 (streaming form).
#pragma once
#include <cuda_runtime.h>

#include <type_traits>

#include "../../include/dhmc_models.h"
#include "nuts_machine.cuh"

namespace dhmc {

constexpr int kRedWidth = 8;   // values per cross-warp exchange row
constexpr int kMaxWarps = 8;   // T <= 256

struct SmemLayout {
  int red_off;    // doubles: [2][kMaxWarps][kRedWidth], or with rg > 1 reduction groups [2][W][rg · kRedWidth]
  int ctl_off;    // bytes from base: Entry[W][levels]
  int misc_off;   // bytes: int[4]
  int top_off;    // bytes: TopState[W] (transition-level scalars, one copy per warp)
  int tab_off;    // bytes: double*[ntab] base address of every slot (shared or global)
  int xs_off;     // bytes: staging vector for the dense mat-vec (dense metric only)
  int slots_off;  // bytes
  size_t total;   // bytes
};
// stride = doubles per slot (a slot of the dense metric holds a (p, p♯) pair), xs = doubles of staging
// levels = stack entries per warp (max_depth + 1), ntab = entries of the slot-address table (>= n_slots); kernels for
// max_depth <= 12 use the compile-time standard values.  rg = groups of kRedWidth values that one all-reduce carries
// (DeviceBackend::kFused: the leapfrog's sums and every merge check of a leaf)
constexpr int kStdLevels = 13, kStdTab = 64;
__host__ __device__ inline size_t red_half_doubles(int W, int rg) { return rg > 1 ? (size_t)W * kRedWidth * rg : (size_t)kMaxWarps * kRedWidth; }
__host__ __device__ inline SmemLayout smem_layout(int W, int n_sm, size_t stride, size_t xs = 0, int levels = kStdLevels, int ntab = kStdTab,
                                                  int rg = 1) {
  SmemLayout L;
  size_t off = 0;
  L.red_off = 0;
  off += sizeof(double) * 2 * red_half_doubles(W, rg);
  L.ctl_off = (int)off;
  off += sizeof(Entry) * (size_t)W * (size_t)levels;
  off = (off + 15) & ~(size_t)15;
  L.misc_off = (int)off;
  off += 16;
  L.top_off = (int)off;
  off += ((sizeof(TopState) + 15) & ~(size_t)15) * (size_t)W;
  L.tab_off = (int)off;
  off += sizeof(double*) * (size_t)ntab;
  L.xs_off = (int)off;
  off += sizeof(double) * xs;
  L.slots_off = (int)off;
  off += sizeof(double) * stride * (size_t)n_sm;
  L.total = off;
  return L;
}

// ---- packed chain groups (logistic family): one likelihood round of the whole CTA on the FP64 tensor cores ----
// Every warp of the CTA calls this the same number of times: a warp with a chain calls it from eval_model
// (active, its β already published), a warp that has run out of chains attends from coop_finish until all
// warps are done, so the CTA barriers below always see all 32·G threads.
// mma.sync.m8n8k4.f64 (SASS DMMA.8x8x4) computes fma(a3,b3, fma(a2,b2, fma(a1,b1, fma(a0,b0, c))))
// (benchmarks/dmma_order_probe.cu), i.e. the model's own sequential order, so the results are those of the
// one-chain-per-CTA FMA loops (eval_model) bit for bit; test_logistic_packed_groups_equal_one_chain_per_cta
// holds the kernels to it.  On the H100 the DMMA pipe has twice the DFMA rate (data sheet) with 1/8 of the
// instructions.
//
// One pass over the design matrix per gradient.  X is kept in HBM/L2 as zero-padded row blocks
// [32 rows][XS] (XS ≡ 4 mod 16 doubles: every fragment load below is bank-conflict free); one elected
// thread streams the blocks through a two-stage shared-memory ring with cp.async.bulk (SASS UBLKCP)
// completing on an mbarrier, consumers release a stage through a second mbarrier.  Per block:
//   P1  four 8-row tiles × four chunks of 64 coefficients spread over all warps: chunk sums of
//       η[8 obs × 8 chains] += X[8 × 4] · β[4 × 8] (η is a blocked dot product, dhmc_logit_eta: the chunks are
//       independent chains of 16 dependent DMMAs, so P1 is bound by the tensor pipe, not by DMMA latency);
//   E   warp g = chain g, lane = row: η from the chunk sums, ll term into the lane's canonical Σ ll partial,
//       residual y − σ(η) → shared tile [chain][32]; rows ≥ N give residual 0;
//   P2  all warps, ⌈D/8⌉ coefficient tiles split over the warps:
//       (Xᵀr)[8 coeff × 8 chains] += Xᵀ[8 × 4 obs] · r[4 obs × 8] — accumulators live in registers for the round.
// Zero padding (rows ≥ N, columns ≥ D) only ever adds fma(0, 0, acc) = acc.
constexpr int kTmaRows = 32;                 // rows of X per block
constexpr int kTmaStages = 2;
constexpr int kTmaPieces = 8;                // bulk copies per block (4 rows each: 16-byte multiples)
constexpr int kTmaBS = 260;                  // row pitch of β [chain][·]            (≡ 4 mod 16)
constexpr int kTmaES = 36;                   // row pitch of the η / residual tiles  (≡ 4 mod 16)
__host__ __device__ inline int tma_xs(int D) { int w = (D + 7) & ~7; while ((w & 15) != 4) ++w; return w; }
__host__ __device__ inline size_t tma_stage_doubles(int D) { return (size_t)kTmaRows * tma_xs(D); }
// CTA-shared area behind the per-group blocks: [0,32) flags, [64,96) mbarriers full[2] empty[2],
// [128, …) β, η tile, residual tile, math tables (lanes look up different entries), ring
__host__ __device__ inline size_t tma_beta_off() { return 128; }
__host__ __device__ inline size_t tma_eta_off(int G) { return tma_beta_off() + sizeof(double) * (size_t)G * kTmaBS; }
constexpr int kTmaChunks = 256 / DHMC_LOGIT_CHUNK;     // η chunk sums per row (dim <= 256)
// η area: kTmaChunks partial tiles [chain][kTmaES], then the residual tile; after the round the first G·64 doubles
// hand the per-thread Σ ll partials back
__host__ __device__ inline size_t tma_tabs_off(int G) { return tma_eta_off(G) + sizeof(double) * (kTmaChunks + 1) * (size_t)G * kTmaES; }   // math tables, DM_TABS_DOUBLES
__host__ __device__ inline size_t tma_y_off(int G) { return tma_tabs_off(G) + sizeof(double) * DM_TABS_DOUBLES; }             // pooled-metric GEMM: M⁻¹·[8 vectors] result [chain][kTmaBS]
__host__ __device__ inline size_t tma_ring_off(int G) { return (tma_y_off(G) + sizeof(double) * (size_t)G * kTmaBS + 127) & ~(size_t)127; }
__host__ __device__ inline size_t tma_smem_bytes(int G, int D) { return tma_ring_off(G) + sizeof(double) * kTmaStages * tma_stage_doubles(D); }

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
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
// the same with an L2 eviction policy: the design matrix is re-read by every SM for every gradient (evict_last keeps it
// resident while the per-chain metrics stream past), a chain's metric block is read once per mat-vec (evict_first)
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ void bulk_g2s_hint(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint64_t policy) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy) : "memory");
}
__device__ __forceinline__ double lds64(uint32_t addr) {
  double v;
  asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts64(uint32_t addr, double v) {
  asm volatile("st.shared.f64 [%0], %1;" ::"r"(addr), "d"(v) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void dmma_8x8x4(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

// One chunk (up to 16 k-steps = four groups of four) of D[8 × 8] += A[8 × 4] · B[4 × 8] for TWO row tiles that share
// the B fragments: A from shared addresses ap / ap2 (+32 bytes per k-step), B from bp (+32 bytes per k-step).
// Two fragment sets in ping-pong; every statement is a volatile asm, so the order below is the issue order and the
// loads run one group ahead of the DMMAs that consume them.
__device__ __forceinline__ void mma_chunk_2tiles(uint32_t ap, uint32_t ap2, uint32_t bp, int ngr,
                                                 double& c0, double& c1, double& d0, double& d1) {
  double fa[2][4], fa2[2][4], fb[2][4];
#define DHMC_P1_LOAD(set, g)                                                                   \
  _Pragma("unroll") for (int u = 0; u < 4; ++u) {                                              \
    fa[set][u] = lds64(ap + 128 * (g) + 32 * u); fa2[set][u] = lds64(ap2 + 128 * (g) + 32 * u); \
    fb[set][u] = lds64(bp + 128 * (g) + 32 * u);                                               \
  }
#define DHMC_P1_MMA(set)                                                                       \
  _Pragma("unroll") for (int u = 0; u < 4; ++u) {                                              \
    dmma_8x8x4(c0, c1, fa[set][u], fb[set][u]); dmma_8x8x4(d0, d1, fa2[set][u], fb[set][u]);   \
  }
  DHMC_P1_LOAD(0, 0)
  if (ngr > 1) { DHMC_P1_LOAD(1, 1) }
  DHMC_P1_MMA(0)
  if (ngr > 2) { DHMC_P1_LOAD(0, 2) }
  if (ngr > 1) { DHMC_P1_MMA(1) }
  if (ngr > 3) { DHMC_P1_LOAD(1, 3) }
  if (ngr > 2) { DHMC_P1_MMA(0) }
  if (ngr > 3) { DHMC_P1_MMA(1) }
#undef DHMC_P1_LOAD
#undef DHMC_P1_MMA
}

// ---- the Symmetric metric's mat-vec p♯ = M⁻¹p (hamiltonian.jl:110,117) of a packed CTA on the FP64 tensor cores ----
// Inside the tree all chains of a CTA need M⁻¹·(their own vector) at the same point of the leapfrog step, so the CTA does
// them one after the other with all its MMA warps: chain c's padded matrix Mp_c [⌈D/32⌉·32][XS] (per-chain metric, as in the
// reference: this is a GEMV, the MMA's n-dimension carries the same vector eight times) streams through the likelihood's
// TMA ring in blocks of 32 rows; per block the 8 MMA warps run the P1 scheme (4 row tiles × 4 chunks of 64 columns, the
// blocked dot product dm_blocked_dot), the chunk sums of all rows are collected in shared memory and added in order when
// the chain's last block is done.  x is published in the β area [chain][kTmaBS] and y handed back in place.
// Returns false when no warp of the CTA is active any more.
template <int G>
__device__ __noinline__ bool coop_matvec_tma(bool active, long chain, int tid, int grp, int ctid, int D,
                                             const double* __restrict__ Mp, unsigned char* shared, uint32_t& ring_n) {
  constexpr int NT = 32 * G;
  constexpr int NW = G;
  constexpr int MW = 8;
  int* cb_flags = reinterpret_cast<int*>(shared);
  int* cb_chain = reinterpret_cast<int*>(shared + 32);        // [G] chain index of every group (metric lookup)
  uint64_t* full = reinterpret_cast<uint64_t*>(shared + 64);
  uint64_t* empty = full + kTmaStages;
  const uint32_t sh = smem_u32(shared);
  const uint32_t beta_a = sh + (uint32_t)tma_beta_off();
  const uint32_t part_a = sh + (uint32_t)tma_eta_off(G);      // chunk sums [chunk][256 rows] (the idle η / residual tiles)
  const uint32_t ring_a = sh + (uint32_t)tma_ring_off(G);
  double* ring = reinterpret_cast<double*>(shared + tma_ring_off(G));
  const int lane = ctid & 31, wq = ctid >> 5;
  const int fr = lane >> 2, fk = lane & 3;
  if (tid == 0) { cb_flags[grp] = active ? 1 : 0; cb_chain[grp] = (int)chain; }
  __syncthreads();
  unsigned amask = 0;
#pragma unroll
  for (int gg = 0; gg < G; ++gg)
    if (cb_flags[gg]) amask |= 1u << gg;
  if (amask == 0) return false;
  const int XS = tma_xs(D);
  const int nbc = (D + kTmaRows - 1) / kTmaRows;              // row blocks per chain
  const int rows_pad = nbc * kTmaRows;
  const int ng = (D + 15) >> 4, nch = (D + DHMC_DOT_CHUNK - 1) / DHMC_DOT_CHUNK;
  const int nact = __popc(amask);
  const int nblk = nact * nbc;
  const uint32_t stage_bytes = (uint32_t)(sizeof(double) * kTmaRows * XS);
  const bool producer = (wq == NW - 1) && (lane == 0);
  const uint32_t n0 = ring_n;
  const uint64_t pol = l2_policy_evict_first();
  auto nth_chain = [&](int ci) { unsigned m = amask; for (int i = 0; i < ci; ++i) m &= m - 1; return __ffs((int)m) - 1; };
  auto issue = [&](int b) {
    const uint32_t n = n0 + (uint32_t)b;
    const int s = (int)(n & 1u);
    const int c = nth_chain(b / nbc), kb = b % nbc;
    mbar_wait(empty + s, ((n >> 1) & 1u) ^ 1u);
    mbar_expect_tx(full + s, stage_bytes);
    const uint32_t piece = stage_bytes / kTmaPieces;
    char* dst = reinterpret_cast<char*>(ring + (size_t)s * kTmaRows * XS);
    const char* src = reinterpret_cast<const char*>(Mp + ((size_t)cb_chain[c] * rows_pad + (size_t)kb * kTmaRows) * XS);
#pragma unroll
    for (int pc = 0; pc < kTmaPieces; ++pc) bulk_g2s_hint(dst + (size_t)pc * piece, src + (size_t)pc * piece, piece, full + s, pol);
  };
  if (producer) {
    fence_proxy_async();
    issue(0);
    if (nblk > 1) issue(1);
  }
  __syncwarp();
  const int pc1 = wq & 3, mp = (wq >> 2) & 1;
  const int g0 = 4 * pc1, g1 = (4 * pc1 + 4 < ng) ? 4 * pc1 + 4 : ng;
  const uint32_t p1_a = (uint32_t)(sizeof(double) * ((16 * mp + fr) * XS + fk)) + 128 * g0;
  int b = 0;
  for (int ci = 0; ci < nact; ++ci) {
    const int c = nth_chain(ci);
    const uint32_t bp = beta_a + (uint32_t)(sizeof(double) * (c * kTmaBS + fk)) + 128 * g0;    // x_c[k] for every n: broadcast
    for (int kb = 0; kb < nbc; ++kb, ++b) {
      const uint32_t n = n0 + (uint32_t)b;
      const int s = (int)(n & 1u);
      mbar_wait(full + s, (n >> 1) & 1u);
      if (wq < MW && g0 < g1) {
        const uint32_t ap = ring_a + (uint32_t)s * stage_bytes + p1_a;
        double c0 = 0.0, c1 = 0.0, d0 = 0.0, d1 = 0.0;
        mma_chunk_2tiles(ap, ap + (uint32_t)(sizeof(double) * 8 * XS), bp, g1 - g0, c0, c1, d0, d1);
        if (fk == 0) {                        // columns n = 0 (all eight columns hold the same dot products)
          const uint32_t pa = part_a + (uint32_t)(sizeof(double) * (pc1 * 256 + kb * kTmaRows + 16 * mp + fr));
          sts64(pa, c0);
          sts64(pa + 64, d0);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(empty + s);
      if (producer && b + 2 < nblk) issue(b + 2);
      __syncwarp();
    }
    __syncthreads();                          // all chunk sums of chain c are in place
    for (int i = ctid; i < D; i += NT) {
      const uint32_t pa = part_a + (uint32_t)(sizeof(double) * i);
      double y = lds64(pa);
      for (int cc = 1; cc < nch; ++cc) y = y + lds64(pa + (uint32_t)(sizeof(double) * 256 * cc));
      sts64(beta_a + (uint32_t)(sizeof(double) * (c * kTmaBS + i)), y);     // y_c replaces x_c
    }
    __syncthreads();
  }
  ring_n = n0 + (uint32_t)nblk;
  return true;
}

// ---- the same product when the eight chains of the CTA SHARE their metric (DHMC_METRIC_SYMMETRIC_POOLED, not reference
// semantics): M⁻¹·[x₀ … x₇] is a true GEMM — the metric streams through the ring ONCE per product (not once per chain), and
// the MMA's n-dimension carries the eight chains' vectors exactly as in the likelihood's P1.  Per 32-row block: P1 (chunk
// sums of two row tiles per warp) → barrier → 256 lanes add the chunk sums in order → y [chain][row].
template <int G>
__device__ __noinline__ bool coop_matmul_pooled_tma(bool active, long chain, int tid, int grp, int ctid, int D,
                                                    const double* __restrict__ Mp, unsigned char* shared, uint32_t& ring_n) {
  constexpr int NT = 32 * G;
  constexpr int NW = G;
  constexpr int MW = 8;
  int* cb_flags = reinterpret_cast<int*>(shared);
  int* cb_chain = reinterpret_cast<int*>(shared + 32);
  uint64_t* full = reinterpret_cast<uint64_t*>(shared + 64);
  uint64_t* empty = full + kTmaStages;
  const uint32_t sh = smem_u32(shared);
  const uint32_t beta_a = sh + (uint32_t)tma_beta_off();
  const uint32_t part_a = sh + (uint32_t)tma_eta_off(G);      // chunk sums [chunk][chain][kTmaES] of the current block
  const uint32_t y_a = sh + (uint32_t)tma_y_off(G);
  const uint32_t ring_a = sh + (uint32_t)tma_ring_off(G);
  double* ring = reinterpret_cast<double*>(shared + tma_ring_off(G));
  const int lane = ctid & 31, wq = ctid >> 5;
  const int fr = lane >> 2, fk = lane & 3;
  if (tid == 0) { cb_flags[grp] = active ? 1 : 0; cb_chain[grp] = (int)chain; }
  __syncthreads();
  unsigned amask = 0;
#pragma unroll
  for (int gg = 0; gg < G; ++gg)
    if (cb_flags[gg]) amask |= 1u << gg;
  if (amask == 0) return false;
  const int XS = tma_xs(D);
  const int nblk = (D + kTmaRows - 1) / kTmaRows;
  const int ng = (D + 15) >> 4, nch = (D + DHMC_DOT_CHUNK - 1) / DHMC_DOT_CHUNK;
  const uint32_t stage_bytes = (uint32_t)(sizeof(double) * kTmaRows * XS);
  const bool producer = (wq == NW - 1) && (lane == 0);
  const uint32_t n0 = ring_n;
  const uint64_t pol = l2_policy_evict_first();
  const double* Mg = Mp + (size_t)cb_chain[__ffs((int)amask) - 1] * (size_t)nblk * kTmaRows * XS;   // the group's metric (any active member's copy)
  auto issue = [&](int b) {
    const uint32_t n = n0 + (uint32_t)b;
    const int s = (int)(n & 1u);
    mbar_wait(empty + s, ((n >> 1) & 1u) ^ 1u);
    mbar_expect_tx(full + s, stage_bytes);
    const uint32_t piece = stage_bytes / kTmaPieces;
    char* dst = reinterpret_cast<char*>(ring + (size_t)s * kTmaRows * XS);
    const char* src = reinterpret_cast<const char*>(Mg + (size_t)b * kTmaRows * XS);
#pragma unroll
    for (int pc = 0; pc < kTmaPieces; ++pc) bulk_g2s_hint(dst + (size_t)pc * piece, src + (size_t)pc * piece, piece, full + s, pol);
  };
  if (producer) {
    fence_proxy_async();
    issue(0);
    if (nblk > 1) issue(1);
  }
  __syncwarp();
  const int pc1 = wq & 3, mp = (wq >> 2) & 1;
  const int g0 = 4 * pc1, g1 = (4 * pc1 + 4 < ng) ? 4 * pc1 + 4 : ng;
  const uint32_t p1_a = (uint32_t)(sizeof(double) * ((16 * mp + fr) * XS + fk)) + 128 * g0;
  const uint32_t p1_b = beta_a + (uint32_t)(sizeof(double) * (fr * kTmaBS + fk)) + 128 * g0;     // B[k][n] = x of chain n
  for (int b = 0; b < nblk; ++b) {
    const uint32_t n = n0 + (uint32_t)b;
    const int s = (int)(n & 1u);
    mbar_wait(full + s, (n >> 1) & 1u);
    if (wq < MW && g0 < g1) {
      const uint32_t ap = ring_a + (uint32_t)s * stage_bytes + p1_a;
      double c0 = 0.0, c1 = 0.0, d0 = 0.0, d1 = 0.0;
      mma_chunk_2tiles(ap, ap + (uint32_t)(sizeof(double) * 8 * XS), p1_b, g1 - g0, c0, c1, d0, d1);
      const uint32_t ea = part_a + (uint32_t)(sizeof(double) * (pc1 * G * kTmaES + 16 * mp + fr));
      sts64(ea + (uint32_t)(sizeof(double) * (2 * fk) * kTmaES), c0);
      sts64(ea + (uint32_t)(sizeof(double) * (2 * fk + 1) * kTmaES), c1);
      sts64(ea + (uint32_t)(sizeof(double) * ((2 * fk) * kTmaES + 8)), d0);
      sts64(ea + (uint32_t)(sizeof(double) * ((2 * fk + 1) * kTmaES + 8)), d1);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(empty + s);
    if (producer && b + 2 < nblk) issue(b + 2);
    __syncwarp();
    __syncthreads();                          // the chunk sums of this block are in place
    for (int idx = ctid; idx < G * kTmaRows; idx += NT) {
      const int gg = idx / kTmaRows, r = idx % kTmaRows, i = b * kTmaRows + r;
      if (i < D) {
        const uint32_t pa = part_a + (uint32_t)(sizeof(double) * (gg * kTmaES + r));
        double y = lds64(pa);
        for (int cc = 1; cc < nch; ++cc) y = y + lds64(pa + (uint32_t)(sizeof(double) * cc * G * kTmaES));
        sts64(y_a + (uint32_t)(sizeof(double) * (gg * kTmaBS + i)), y);
      }
    }
    __syncthreads();                          // … and consumed: the next block may overwrite them
  }
  ring_n = n0 + (uint32_t)nblk;
  return true;
}

// lXp: padded row blocks of X, [nblk·32][XS]; shared: the CTA-shared area (layout above);
// ring_n: blocks streamed so far (same in all threads).  Returns false when no warp is active any more;
// otherwise true with this lane's partial Σ ll in *sll_out.
template <int G>
__device__ __noinline__ bool coop_core_tma(double* sll_out, bool active, int tid, int grp, int ctid, int D, int lN,
                                           const double* __restrict__ lXp, const double* __restrict__ ly,
                                           unsigned char* shared, uint32_t& ring_n) {
  static_assert(G == 8, "the n-dimension of the MMA is the chain");
  constexpr int NW = G;                     // warps of the CTA, one per chain
  constexpr int MW = 8;                     // warps that issue DMMAs (two per sub-partition saturate the pipe; more only add
                                            // shared-memory traffic: operands are reused across a warp's tiles)
  constexpr int JT = 32 / MW;               // coefficient tiles per MMA warp in P2 (D <= 256)
  int* cb_flags = reinterpret_cast<int*>(shared);
  uint64_t* full = reinterpret_cast<uint64_t*>(shared + 64);
  uint64_t* empty = full + kTmaStages;
  // shared-state-space addresses: every access below is an explicit ld/st.shared (the pointers reach this
  // function as generic addresses; generic loads would be resolved per access and are slower)
  const uint32_t sh = smem_u32(shared);
  const uint32_t beta_a = sh + (uint32_t)tma_beta_off();
  const uint32_t eta_a = sh + (uint32_t)tma_eta_off(G);                       // η chunk sums [chunk][chain][kTmaES]
  const uint32_t res_a = eta_a + (uint32_t)(sizeof(double) * kTmaChunks * G * kTmaES);   // residuals [chain][kTmaES]
  const uint32_t ring_a = sh + (uint32_t)tma_ring_off(G);
  const double* tabs = reinterpret_cast<const double*>(shared + tma_tabs_off(G));
  double* ring = reinterpret_cast<double*>(shared + tma_ring_off(G));
  const int lane = ctid & 31, wq = ctid >> 5;
  const int fr = lane >> 2, fk = lane & 3;  // fragment row / k index of this lane
  if (tid == 0) cb_flags[grp] = active ? 1 : 0;
  __syncthreads();                          // β and flags are published; the ring (last round's Xᵀr) is free
  unsigned amask = 0;
#pragma unroll
  for (int gg = 0; gg < G; ++gg)
    if (cb_flags[gg]) amask |= 1u << gg;
  if (amask == 0) return false;

  const int XS = tma_xs(D);
  const int nblk = (lN + kTmaRows - 1) / kTmaRows;
  const int ng = (D + 15) >> 4;             // groups of four k-steps of P1 (all chunks)
  const int nch = (D + DHMC_LOGIT_CHUNK - 1) / DHMC_LOGIT_CHUNK;   // η chunks (dhmc_logit_eta)
  const uint32_t stage_bytes = (uint32_t)(sizeof(double) * kTmaRows * XS);
  const bool producer = (wq == NW - 1) && (lane == 0);
  const uint32_t n0 = ring_n;
  const uint64_t pol = l2_policy_evict_last();
  auto issue = [&](int b) {                 // block b of this round -> stage (n0 + b) % 2
    const uint32_t n = n0 + (uint32_t)b;
    const int s = (int)(n & 1u);
    mbar_wait(empty + s, ((n >> 1) & 1u) ^ 1u);             // everyone is done with the stage's previous block
    mbar_expect_tx(full + s, stage_bytes);
    // a single bulk copy is paced by its own latency (~20 B/clk measured): kTmaPieces of them run concurrently
    const uint32_t piece = stage_bytes / kTmaPieces;
    double* dst = ring + (size_t)s * kTmaRows * XS;
    const double* src = lXp + (size_t)b * kTmaRows * XS;
#pragma unroll
    for (int pc = 0; pc < kTmaPieces; ++pc)
      bulk_g2s_hint(reinterpret_cast<char*>(dst) + (size_t)pc * piece, reinterpret_cast<const char*>(src) + (size_t)pc * piece, piece, full + s, pol);
  };
  if (producer) {
    fence_proxy_async();                    // generic writes to the ring (Xᵀr hand-back) precede the async writes
    issue(0);
    if (nblk > 1) issue(1);
  }
  __syncwarp();
  double acc[JT][2];
#pragma unroll
  for (int q = 0; q < JT; ++q) { acc[q][0] = 0.0; acc[q][1] = 0.0; }
  double sl = 0.0;                          // E: this lane's Σ ll partial (thread `lane` of chain wq)
  // P1 work of an MMA warp: chunk c = wq & 3, row tiles 2·(wq >> 2) and 2·(wq >> 2) + 1 (they share the β fragments)
  const int pc1 = wq & 3, mp = (wq >> 2) & 1;
  const uint32_t p1_a = (uint32_t)(sizeof(double) * ((16 * mp + fr) * XS + fk));     // A fragment of P1 within a stage (second tile: + 8 rows)
  const uint32_t p1_b = beta_a + (uint32_t)(sizeof(double) * (fr * kTmaBS + fk));     // B fragment of P1
  const uint32_t p2_b = res_a + (uint32_t)(sizeof(double) * (fr * kTmaES + fk));      // B fragment of P2
  const uint32_t p2_a = (uint32_t)(sizeof(double) * (fk * XS + 8 * wq + fr));         // A fragment of P2 within a stage

  for (int b = 0; b < nblk; ++b) {
    const uint32_t n = n0 + (uint32_t)b;
    const int s = (int)(n & 1u);
    const uint32_t par = (n >> 1) & 1u;
    const uint32_t xt = ring_a + (uint32_t)s * stage_bytes;
    // ---- P1: chunk sums of η for rows 8·mt … 8·mt+7: D[8 obs × 8 chains] += X[8 × 4] · β[4 × 8], a dependent
    // chain of up to 16 DMMAs per chunk (26 clk each), fragments fetched one group of four k-steps ahead;
    // k-steps beyond ⌈D/4⌉ hit the zero padding of X and β (16·⌈D/16⌉ <= XS)
    mbar_wait(full + s, par);
    if (wq < MW) {
      const int g0 = 4 * pc1, g1 = (4 * pc1 + 4 < ng) ? 4 * pc1 + 4 : ng;    // k-step groups of this chunk
      if (g0 < g1) {
        const uint32_t ap = xt + p1_a + 128 * g0;
        double c0 = 0.0, c1 = 0.0, d0 = 0.0, d1 = 0.0;
        mma_chunk_2tiles(ap, ap + (uint32_t)(sizeof(double) * 8 * XS), p1_b + 128 * g0, g1 - g0, c0, c1, d0, d1);
        const uint32_t ea = eta_a + (uint32_t)(sizeof(double) * (pc1 * G * kTmaES + 16 * mp + fr));
        sts64(ea + (uint32_t)(sizeof(double) * (2 * fk) * kTmaES), c0);
        sts64(ea + (uint32_t)(sizeof(double) * (2 * fk + 1) * kTmaES), c1);
        sts64(ea + (uint32_t)(sizeof(double) * ((2 * fk) * kTmaES + 8)), d0);
        sts64(ea + (uint32_t)(sizeof(double) * ((2 * fk + 1) * kTmaES + 8)), d1);
      }
    }
    __syncthreads();
    // ---- E: warp gg evaluates chain gg, lane = row: η = ((s₀ + s₁) + s₂) + s₃, ll term into this lane's
    // canonical partial (thread (n mod 32) of the chain sums n, n+32, … in increasing n), residual -> shared tile
    {
      const int gg = wq, r = lane;
      const int nrow = b * kTmaRows + r;
      const uint32_t ea = eta_a + (uint32_t)(sizeof(double) * (gg * kTmaES + r));
      double eta = lds64(ea);
      for (int c = 1; c < nch; ++c) eta = eta + lds64(ea + (uint32_t)(sizeof(double) * c * G * kTmaES));
      double rv = 0.0;                      // rows >= N contribute fma(x, 0, acc) = acc
      if (nrow < lN) {
        double llv;
        dhmc_logit_ll_resid_tabs(__ldg(ly + nrow), eta, &llv, &rv, tabs);
        sl = sl + llv;
      }
      sts64(res_a + (uint32_t)(sizeof(double) * (gg * kTmaES + r)), rv);
    }
    __syncthreads();
    // ---- P2: (Xᵀr) += Xᵀ[coefficients × rows of the block] · r; operands one k-step ahead
    if (wq < MW) {
      const uint32_t ap = xt + p2_a;
      uint32_t jo[JT];                      // column offset of this warp's coefficient tiles (tiles beyond D are not touched)
#pragma unroll
      for (int q = 0; q < JT; ++q) jo[q] = (wq + q * MW) * 8 < D ? (uint32_t)(sizeof(double) * 8 * MW * q) : 0xffffffffu;
      double bv[2], av[2][JT];              // ping-pong operand sets, one k-step ahead (volatile asm keeps the order)
      bv[0] = lds64(p2_b);
#pragma unroll
      for (int q = 0; q < JT; ++q) av[0][q] = jo[q] != 0xffffffffu ? lds64(ap + jo[q]) : 0.0;
#pragma unroll
      for (int ks = 0; ks < kTmaRows / 4; ++ks) {
        const int cur = ks & 1, nxt = cur ^ 1;
        if (ks + 1 < kTmaRows / 4) {
          bv[nxt] = lds64(p2_b + 32 * (ks + 1));
#pragma unroll
          for (int q = 0; q < JT; ++q)
            av[nxt][q] = jo[q] != 0xffffffffu ? lds64(ap + (uint32_t)(sizeof(double) * 4 * (ks + 1) * XS) + jo[q]) : 0.0;
        }
#pragma unroll
        for (int q = 0; q < JT; ++q)
          if (jo[q] != 0xffffffffu) dmma_8x8x4(acc[q][0], acc[q][1], av[cur][q], bv[cur]);
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(empty + s);
    if (producer && b + 2 < nblk) issue(b + 2);
    __syncwarp();
  }
  ring_n = n0 + (uint32_t)nblk;
  __syncthreads();                          // every warp is done with the ring and the tiles: hand Xᵀr and Σ ll back
#pragma unroll
  for (int q = 0; q < JT; ++q) {
    const int j = (wq + q * MW) * 8 + fr;
    if (wq < MW && j < D) {
      sts64(ring_a + (uint32_t)(sizeof(double) * ((2 * fk) * XS + j)), acc[q][0]);        // cb_grad [chain][XS]
      sts64(ring_a + (uint32_t)(sizeof(double) * ((2 * fk + 1) * XS + j)), acc[q][1]);
    }
  }
  sts64(eta_a + (uint32_t)(sizeof(double) * (wq * 32 + lane)), sl);   // [chain][32]
  __syncthreads();
  const double sll = active ? lds64(eta_a + (uint32_t)(sizeof(double) * (grp * 32 + tid))) : 0.0;
  *sll_out = sll;
  return true;
}

// DENSE = Symmetric M⁻¹ per chain (hamiltonian.jl:73): p♯ = M⁻¹p is a D×D mat-vec
// streamed from HBM, kept in registers next to p and stored with it — a momentum
// slot holds the pair (p, p♯), so the state machine's bookkeeping is unchanged.
//
// PACK > 1 ("packed chain groups", logistic family, one warp per chain): a CTA holds PACK
// independent chains.  Everything except the likelihood is private to the chain's warp; the
// likelihood is evaluated by the whole CTA for all PACK chains at once on the FP64 tensor cores
// (coop_round), so every element of X is read once per PACK gradients instead of once per
// gradient — the family is bound by L2 traffic on X otherwise.  The per-chain arithmetic
// and its order are unchanged (η_n sequential in j, (Xᵀr)_j sequential in n, Σ ll lane-strided).
template <int EPL, int FAM, int WARPS, bool DENSE = false, int PACK = 1, bool DEEP = false>
struct DeviceBackend {
  static constexpr bool kDeep = DEEP;     // max_depth > 12: the slot pool spills past its register word (nuts_machine.cuh)
  static_assert(PACK == 1 || (WARPS == 1 && FAM == DHMC_FAMILY_LOGISTIC), "packed groups: one warp per chain, logistic family");
  static constexpr int G = PACK;
  int grp, ctid;                            // warp (= chain group) within the CTA, thread within the CTA
  double* cb_beta; double* cb_grad;         // CTA-shared exchange area: β [chain][kTmaBS], Xᵀr [chain][tma_xs(D)]
  unsigned char* cb_shared;                 // its base (layout of tma_smem_bytes)
  uint32_t ring_n;                          // blocks of X streamed through the ring so far (uniform over the CTA)
  const double* lXp;                        // zero-padded row blocks of X, [⌈N/32⌉·32][tma_xs(D)]
  const double* Mp;                         // Symmetric metric: padded M⁻¹ of all chains, [chain][⌈D/32⌉·32][tma_xs(D)]
  // geometry: T = 32·WARPS threads per chain, compile-time so that strides fold
  static constexpr int W = WARPS;
  static constexpr int T = 32 * WARPS;
  static constexpr bool kDense = DENSE;
  static constexpr size_t vstride = (size_t)T * EPL;                    // doubles per vector
  static constexpr size_t stride = DENSE ? 2 * vstride : vstride;      // doubles per slot
  int tid, lane, warp, D;
  long chain;            // local chain index
  // registers
  double q[EPL], p[EPL], g[EPL], minv[EPL], rhoL[EPL];
  double ps[DENSE ? EPL : 1];      // p♯ of the current point (dense metric)
  double lq;
  // dense metric: this chain's M⁻¹ (symmetric, [D][D]), Wᵀ (column-major lower W), co-moment
  // accumulator (transposed lower) and the shared-memory staging vector
  const double* Mrow; const double* Wt; double* covt; double* xs;
  double* mean_out;      // pooled Symmetric stage: where this chain's window mean goes (else null)
  // logistic regression: X [N][D], Xᵀ [D][lLd], y [N], residual scratch (per CTA [N]; packed groups [N][G])
  const double* lX; const double* lXt; const double* ly; double* lr; int lN; int lLd;   // lLd: leading dimension of Xᵀ
  // memory
  double* red; int red_buf;
  Entry* ctl;
  TopState* tops;
  double* sm_slots; double* gl_slots; int n_sm;
  const double* mparams;
  int n_slots;

  // Per-element values that stay the same for the whole run of a chain and are cheap to recompute: the element index
  // tid + e·T (and the lane-derived offsets of the reductions), the 1/√M⁻¹ of the momentum draw, the model's
  // parameters.  Left alone, the compiler hoists them out of the transition and leaf loops and keeps them live across
  // the whole tree build, where they crowd the state vectors (q, p, ∇ℓ, M⁻¹, ρ) out of the register budget into local
  // memory.  pin() passes its input through an empty volatile asm, so that what is computed from it stays inside the
  // loop that uses it.  With one element per thread the registers suffice and the recomputation would only cost time,
  // so pin() is the identity there; packed chain groups keep their own register allocation (their time goes to the
  // cooperative likelihood rounds).
  static constexpr bool kPinInvariants = EPL >= 2 && PACK == 1;
  template <class V> __device__ __forceinline__ static V pin(V v) {
    if constexpr (kPinInvariants) {
      if constexpr (std::is_pointer_v<V>) asm volatile("" : "+l"(v));
      else if constexpr (std::is_same_v<V, double>) asm volatile("" : "+d"(v));
      else asm volatile("" : "+r"(v));
    }
    return v;
  }

  __device__ __forceinline__ bool valid(int e) const { return tid + e * T < D; }
  // slot base addresses are tabulated once per CTA in shared memory: one LDS.64 instead of a
  // 64-bit select + multiply-add at every access
  double** slot_tab; int n_tab;
  __device__ __forceinline__ void build_slot_table() {
    for (int s = tid; s < n_tab; s += T)
      slot_tab[s] = s < n_sm ? sm_slots + (size_t)s * stride : gl_slots + (size_t)(s - n_sm) * stride;
    group_sync();
  }
  __device__ __forceinline__ double* slot(int s) const { return slot_tab[s] + tid; }

  // ---- scalar all-reduce of N <= 8 values in the canonical order (DESIGN.md).
  // Intra-warp: shuffle reduce-scatter with xor offsets 16, 8, 4, 2, 1 — at each
  // stage a lane keeps half of its values and sends the other half, so N values
  // cost about N + 3 shuffles instead of 5 N; every value still sees the same
  // pairwise tree (lane l with l^16, then ^8, ...).  The lane that ends up with
  // value `idx` publishes it to shared memory; all threads then read the W x N
  // partials and combine warps with a pairwise tree (offsets 32, 64, ...).
  template <int CW, int OFF>
  __device__ __forceinline__ void rs_stage(double* w, int& idx) const {
    if constexpr (CW >= 2) {
      constexpr int H = CW / 2;
      const bool upper = (lane & OFF) != 0;
#pragma unroll
      for (int j = 0; j < H; ++j) {
        const double send = upper ? w[j] : w[j + H];
        const double recv = __shfl_xor_sync(0xffffffffu, send, OFF);
        const double keep = upper ? w[j + H] : w[j];
        w[j] = keep + recv;
      }
      idx = idx * 2 + (upper ? 1 : 0);
    } else {
      w[0] = w[0] + __shfl_xor_sync(0xffffffffu, w[0], OFF);
    }
  }
  // the pairwise tree over the warps' partials b[0], b[S], b[2S], … (offsets 32, 64, … of the canonical order)
  template <int S>
  __device__ __forceinline__ static double warp_sum(const double* b) { return warp_sum(b, S); }
  __device__ __forceinline__ static double warp_sum(const double* b, int S) {
    if (W == 1) return b[0];
    if (W == 2) return b[0] + b[S];
    if (W == 4) return (b[0] + b[S]) + (b[2 * S] + b[3 * S]);
    return ((b[0] + b[S]) + (b[2 * S] + b[3 * S])) + ((b[4 * S] + b[5 * S]) + (b[6 * S] + b[7 * S]));
  }
  __device__ __forceinline__ int red_half() const {
    if constexpr (kFused) return red_half_n;
    else return kMaxWarps * kRedWidth;
  }
  // the intra-warp part: returns which of the N values this lane ends up with (its warp's partial in *out)
  template <int N>
  __device__ __forceinline__ int warp_scatter(const double (&v)[N], double* out) const {
    constexpr int P = N <= 1 ? 1 : N <= 2 ? 2 : N <= 4 ? 4 : 8;
    static_assert(N <= kRedWidth, "at most 8 values per reduction");
    double w[P];
#pragma unroll
    for (int j = 0; j < P; ++j) w[j] = j < N ? v[j] : 0.0;
    int idx = 0;
    rs_stage<P, 16>(w, idx);
    rs_stage<(P >= 2 ? P / 2 : 1), 8>(w, idx);
    rs_stage<(P >= 4 ? P / 4 : 1), 4>(w, idx);
    rs_stage<1, 2>(w, idx);
    rs_stage<1, 1>(w, idx);
    *out = w[0];
    return idx;
  }
  template <int N>
  __device__ __forceinline__ void reduce(double (&v)[N]) {
#if defined(DHMC_PHASE_CLOCKS)
    const bool ph_leaf_red = ph_cur == kPhLfElem || ph_cur == kPhMcElem;   // the reductions of a leaf are profiled
    if (ph_leaf_red) phase_mark(ph_cur + 1);
#endif
    double w0;
    const int idx = warp_scatter(v, &w0);
    double* buf = red + red_buf * red_half();
    red_buf ^= 1;
    buf[warp * kRedWidth + idx] = w0;
    group_sync();
#pragma unroll
    for (int n = 0; n < N; ++n) v[n] = warp_sum<kRedWidth>(buf + n);
#if defined(DHMC_PHASE_CLOCKS)
    if (ph_leaf_red) phase_mark(kPhCtrl);
#endif
  }

  // ---- one all-reduce per leaf (diagonal metric, one chain per CTA).  The machine tells leapfrog() which merges the new
  // leaf may need: its ctz(k) stack merges (top entry first) and, on the last leaf of an adjacent tree, the doubling-level
  // check against the whole tree.  Their dot products depend only on the new p and on slots fixed before the leaf, so the
  // leapfrog computes them all right after its own elementwise pass (ρ chained speculatively, as merge_check would) and
  // ONE all-reduce carries everything: group 0 = the leapfrog's sums plus the leaf-leaf merge's two products in columns
  // kLeafCol, kLeafCol + 1; group j + (no stack merge ? 1 : 0) = the six products of merge j.  merge_check(j, …) then only
  // reads the sums; those of merges the control never reaches are dropped.  Every value keeps its per-thread order and
  // its pairwise tree (warp_scatter / warp_sum), so the sums are those of one merge_check at a time.  User models keep
  // one reduction per check: with the merges inlined behind their model code the C2-shaped user kernel ran slower.
  static constexpr bool kFused = !DENSE && PACK == 1 && FAM != DHMC_FAMILY_USER;
  static constexpr bool kLeafMerges = true;   // the interface (nuts_machine.cuh); kernels without kFused check one merge at a time
  static constexpr int kLeafCol = 6;
  int red_half_n, red_row;                  // kFused: doubles per buffer half / per warp row (rg · kRedWidth)
  int m_sp, m_c, m_dbl;                     // merges of the current leaf: stack height, stack merges, doubling check
  int m_shift;                              // group of merge j = j + m_shift
  const double* m_buf;                      // the buffer half that holds their sums

  template <int N>
  __device__ __forceinline__ void reduce_leaf(double (&v)[N]) {
    if constexpr (kFused) {
      if (m_c > 0 || m_dbl) { reduce_fused(v); return; }
    }
    reduce(v);
  }
  template <int N>
  __device__ __forceinline__ void reduce_fused(double (&v)[N]) {
    static_assert(N <= kLeafCol, "group 0 holds the leapfrog's sums and two merge products");
    DHMC_PHASE(*this, kPhMcElem);
    double* buf = red + red_buf * red_half_n;
    red_buf ^= 1;
    double* row = buf + warp * red_row;
    {
      double g0[kRedWidth];
#pragma unroll
      for (int n = 0; n < kLeafCol; ++n) g0[n] = n < N ? v[n] : 0.0;
      g0[kLeafCol] = 0.0; g0[kLeafCol + 1] = 0.0;
      if (m_c > 0) {                        // merge 0: two single leaves (see merge_check)
        const double* pEf = slot(ctl[m_sp - 1].sfirst);
#pragma unroll
        for (int e = 0; e < EPL; ++e) {
          const double Ef = pEf[e * T];
          const double A = Ef + p[e];
          const double mEf = minv[e] * Ef, mLl = minv[e] * p[e];
          g0[kLeafCol] = g0[kLeafCol] + mEf * A;
          g0[kLeafCol + 1] = g0[kLeafCol + 1] + mLl * A;
          rhoL[e] = A;
        }
      }
      double w0;
      const int idx = warp_scatter(g0, &w0);
      row[idx] = w0;
    }
    m_shift = m_c > 0 ? 0 : 1;
    const int nm = m_c + m_dbl;
    for (int j = 1 - m_shift; j < nm; ++j) {
      int sEf, sEl, sEr, sLf;
      bool lleaf = false;
      if (j < m_c) {                        // stack merge j: E = the entry below, L = the subtree of merges 0…j-1
        const Entry& E = ctl[m_sp - 1 - j];
        sEf = E.sfirst; sEl = E.slast; sEr = E.srho;
        sLf = ctl[m_sp - j].sfirst;
      } else {                              // the doubling check: E = the whole tree so far, L = this adjacent tree
        const TopState& S = top();
        sEf = S.s_op; sEl = S.s_near; sEr = S.s_rhot;
        lleaf = m_c == 0;
        sLf = lleaf ? sEf : ctl[m_sp - m_c].sfirst;
      }
      const double* pEf = slot(sEf);
      const double* pEl = slot(sEl);
      const double* pEr = slot(sEr);
      const double* pLf = slot(sLf);
      double d[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
      for (int e = 0; e < EPL; ++e) {
        const double Ef = pEf[e * T], El = pEl[e * T], Er = pEr[e * T];
        const double Lf = lleaf ? p[e] : pLf[e * T];
        const double Lr = lleaf ? p[e] : rhoL[e];
        const double A = Er + Lf, Bv = El + Lr, R = Er + Lr;
        const double mEf = minv[e] * Ef, mLf = minv[e] * Lf, mEl = minv[e] * El, mLl = minv[e] * p[e];
        d[0] = d[0] + mEf * A;  d[1] = d[1] + mLf * A;
        d[2] = d[2] + mEl * Bv; d[3] = d[3] + mLl * Bv;
        d[4] = d[4] + mEf * R;  d[5] = d[5] + mLl * R;
        rhoL[e] = R;
      }
      double w0;
      const int idx = warp_scatter(d, &w0);
      row[(j + m_shift) * kRedWidth + idx] = w0;
    }
    DHMC_PHASE(*this, kPhLfRed);
    group_sync();
#pragma unroll
    for (int n = 0; n < N; ++n) v[n] = warp_sum(buf + n, red_row);
    m_buf = buf;
    DHMC_PHASE(*this, kPhCtrl);
  }

#if defined(DHMC_PHASE_CLOCKS)
  unsigned long long* ph_acc;               // this CTA's kPhCount counters
  long long ph_t;                           // clock64() at the last mark
  int ph_cur;                               // the phase that time since the last mark belongs to
  __device__ __forceinline__ void phase_mark(int ph) {
    if (ctid == 0) {
      const long long t = clock64();
      atomicAdd(ph_acc + ph_cur, (unsigned long long)(t - ph_t));
      ph_t = t; ph_cur = ph;
    }
  }
  __device__ __forceinline__ void phase_leaf() { if (ctid == 0) atomicAdd(ph_acc + kPhLeaves, 1ull); }
#endif

  // ---- lane-parallel scalar math: all threads of a chain hold the same scalars,
  // so independent transcendental evaluations are spread over lanes and shared
  // by shuffle instead of being evaluated one after the other by every lane.
  // The kFused kernels inline the softplus here and the Box–Muller math in draw() (dhmc_math.h, the _inl twins): the one
  // runs on the serial path between a leaf's reduction and the next leapfrog, the other at the head of every transition.
  __device__ __forceinline__ void logaddexp2(double a0, double b0, double a1, double b1,
                                             double* r0, double* r1) const {
    const bool odd = (lane & 1) != 0;
    const double a = odd ? a1 : a0, b = odd ? b1 : b0;
    double r;
    if constexpr (kFused) r = dm_logaddexp_inl(a, b);
    else r = dm_logaddexp(a, b);
    *r0 = __shfl_sync(0xffffffffu, r, 0);
    *r1 = __shfl_sync(0xffffffffu, r, 1);
  }
  // randexp draws j = base..base+31 of a transition are generated by the 32 lanes at once
  double rexp_cache;
  uint32_t rexp_base, rexp_t;
  __device__ __forceinline__ double randexp(dm_rng_key key, uint32_t t, uint32_t j) {
    const uint32_t base = j & ~31u;
    if (base != rexp_base || t != rexp_t) {
      rexp_cache = dm_randexp(key, t, base + (uint32_t)lane);   // out of line: once per 32 draws, and inlined it spills more
      rexp_base = base; rexp_t = t;
    }
    return __shfl_sync(0xffffffffu, rexp_cache, (int)(j & 31u));
  }

  // ---- interface used by NutsMachine ----
  __device__ __forceinline__ TopState& top() const { return *tops; }
  __device__ __forceinline__ void top_sync() const { __syncwarp(); }
  __device__ __forceinline__ int reserved_first() const { return n_slots - 2; }   // the two highest slots: Welford mean / M2
  __device__ __forceinline__ double cur_lq() const { return lq; }
  __device__ __forceinline__ void set_cur_lq(double v) { lq = v; }

#define DHMC_ST(name, src)                                   \
  __device__ __forceinline__ void name(int s) {              \
    double* d = slot(s);                                     \
    _Pragma("unroll") for (int e = 0; e < EPL; ++e) d[e * T] = src[e]; \
  }
#define DHMC_LD(name, dst)                                   \
  __device__ __forceinline__ void name(int s) {              \
    const double* d = slot(s);                               \
    _Pragma("unroll") for (int e = 0; e < EPL; ++e) dst[e] = d[e * T]; \
  }
  DHMC_ST(st_q, q) DHMC_ST(st_g, g) DHMC_ST(st_rho, rhoL)
  DHMC_LD(ld_q, q) DHMC_LD(ld_g, g)
#undef DHMC_ST
#undef DHMC_LD
  __device__ __forceinline__ void st_p(int s) {
    double* d = slot(s);
#pragma unroll
    for (int e = 0; e < EPL; ++e) {
      d[e * T] = p[e];
      if constexpr (DENSE) d[vstride + e * T] = ps[e];
    }
  }
  __device__ __forceinline__ void ld_p(int s) {
    const double* d = slot(s);
#pragma unroll
    for (int e = 0; e < EPL; ++e) {
      p[e] = d[e * T];
      if constexpr (DENSE) ps[e] = d[vstride + e * T];
    }
  }

  __device__ __forceinline__ void swap_cur(int sq, int sp, int sg) {
    double* dq = slot(sq); double* dp = slot(sp); double* dg = slot(sg);
#pragma unroll
    for (int e = 0; e < EPL; ++e) {
      double a = dq[e * T]; dq[e * T] = q[e]; q[e] = a;
      double b = dp[e * T]; dp[e * T] = p[e]; p[e] = b;
      if constexpr (DENSE) { double b2 = dp[vstride + e * T]; dp[vstride + e * T] = ps[e]; ps[e] = b2; }
      double c = dg[e * T]; dg[e * T] = g[e]; g[e] = c;
    }
  }
  // ρ of a leaf is its momentum; merge_check reads p directly for leaves and
  // writes the combined ρ into rhoL (dead if the merge turns), so these are no-ops.
  __device__ __forceinline__ void rho_from_p() {}
  __device__ __forceinline__ void rho_commit() {}

  __device__ __forceinline__ void put_entry(int j, const Entry& e) {
    __syncwarp();
    if (lane == 0) ctl[j] = e;
    __syncwarp();
  }
  // stack entries: the register-tight kernels read an entry's fields from shared memory where they are used, instead
  // of holding a copy of all of them across merge_check
  __device__ __forceinline__ std::conditional_t<kPinInvariants, const Entry&, Entry> get_entry(int j) const { return ctl[j]; }

  // all threads of the chain: the warp, or the CTA
  __device__ __forceinline__ void group_sync() const {
    if constexpr (W == 1) __syncwarp();
    else __syncthreads();
  }
  // y = M⁻¹ x for this chain (Symmetric M⁻¹ * v, hamiltonian.jl:110): x is staged in shared
  // memory, every thread accumulates its own rows as a blocked dot product over j (dm_blocked_dot:
  // sequential FMAs within chunks of 64, chunk sums added in order — the oracle's order, and the order of the
  // tensor-core version coop_matvec_tma); row j of M is read coalesced (M is symmetric).
  __device__ __forceinline__ void matvec(const double (&x)[EPL], double (&y)[EPL]) {
#pragma unroll
    for (int e = 0; e < EPL; ++e) xs[tid + e * T] = x[e];
    group_sync();
    double acc[EPL];
#pragma unroll
    for (int e = 0; e < EPL; ++e) acc[e] = 0.0;
    const double* row = Mrow + tid;
    for (int j0 = 0; j0 < D; j0 += DHMC_DOT_CHUNK) {
      const int j1 = j0 + DHMC_DOT_CHUNK < D ? j0 + DHMC_DOT_CHUNK : D;
      double sacc[EPL];
#pragma unroll
      for (int e = 0; e < EPL; ++e) sacc[e] = 0.0;
#pragma unroll 4
      for (int j = j0; j < j1; ++j, row += D) {
        const double xj = xs[j];
#pragma unroll
        for (int e = 0; e < EPL; ++e)
          if (tid + e * T < D) sacc[e] = dm_fma(__ldg(row + e * T), xj, sacc[e]);
      }
#pragma unroll
      for (int e = 0; e < EPL; ++e) acc[e] = j0 == 0 ? sacc[e] : acc[e] + sacc[e];
    }
#pragma unroll
    for (int e = 0; e < EPL; ++e) y[e] = acc[e];
    group_sync();
  }
  // y = W z with lower-triangular W stored transposed (hamiltonian.jl:124, :73)
  __device__ __forceinline__ void trmv(const double (&z)[EPL], double (&y)[EPL]) {
#pragma unroll
    for (int e = 0; e < EPL; ++e) xs[tid + e * T] = z[e];
    group_sync();
    double acc[EPL];
#pragma unroll
    for (int e = 0; e < EPL; ++e) acc[e] = 0.0;
    const double* col = Wt + tid;
    for (int j = 0; j < D; ++j, col += D) {
      const double zj = xs[j];
#pragma unroll
      for (int e = 0; e < EPL; ++e) {
        const int i = tid + e * T;
        if (i < D && j <= i) acc[e] = acc[e] + __ldg(col + e * T) * zj;
      }
    }
#pragma unroll
    for (int e = 0; e < EPL; ++e) y[e] = acc[e];
    group_sync();
  }

  // rand_p — hamiltonian.jl:124: W * randn(D), W = Diagonal(sqrt.(inv.(diag M⁻¹))) (:80)
  __device__ __forceinline__ void draw(dm_rng_key key, uint32_t stream, uint32_t t,
                                       const double* p_override) {
    if (p_override) {
#pragma unroll
      for (int e = 0; e < EPL; ++e) {
        const int i = tid + e * T;
        p[e] = i < D ? p_override[(size_t)chain * D + i] : 0.0;
      }
      if constexpr (DENSE) matvec(p, ps);
      return;
    }
    if constexpr (DENSE) {
      double z[EPL];
#pragma unroll
      for (int e = 0; e < EPL; ++e) {
        const int i = tid + e * T;
        z[e] = i < D ? dm_normal_elem(key, stream, t, (uint32_t)i) : 0.0;
      }
      trmv(z, p);
      matvec(p, ps);
      return;
    }
    if constexpr (EPL >= 2) {
      // Elements (2j, 2j+1) share one Philox block / Box-Muller pair and sit in adjacent
      // lanes (T is even).  The even lane evaluates the pairs of even register slots, the
      // odd lane those of odd slots, and the halves are exchanged by one shuffle.
      const int odd = lane & 1;
      uint32_t jp[EPL / 2];                       // the pair of register slots e, e + 1 that this lane evaluates
#pragma unroll
      for (int e = 0; e < EPL; e += 2) jp[e / 2] = (uint32_t)(((tid & ~1) + (e + odd) * T) >> 1);
      // the kFused kernels evaluate the EPL / 2 pairs of this lane stage by stage, so that their chains overlap
      double zp0[EPL / 2], zp1[EPL / 2];
      if constexpr (kFused) dm_normal_pairs_inl(key, stream, t, jp, EPL / 2, zp0, zp1);
#pragma unroll
      for (int e = 0; e < EPL; e += 2) {
        double z0, z1;
        if constexpr (kFused) { z0 = zp0[e / 2]; z1 = zp1[e / 2]; }
        else dm_normal_pair(key, stream, t, jp[e / 2], &z0, &z1);
        const double recv = __shfl_xor_sync(0xffffffffu, odd ? z0 : z1, 1);
        const double ze = odd ? recv : z0;        // element tid + e*T
        const double zo = odd ? z1 : recv;        // element tid + (e+1)*T
        p[e] = (tid + e * T < D) ? dm_sqrt(1.0 / pin(minv[e])) * ze : 0.0;
        p[e + 1] = (tid + (e + 1) * T < D) ? dm_sqrt(1.0 / pin(minv[e + 1])) * zo : 0.0;
      }
    } else {
#pragma unroll
      for (int e = 0; e < EPL; ++e) {
        const int i = tid + e * T;
        p[e] = i < D ? dm_sqrt(1.0 / pin(minv[e])) * dm_normal_elem(key, stream, t, (uint32_t)i) : 0.0;
      }
    }
  }
  __device__ __forceinline__ void draw_momentum(dm_rng_key key, uint32_t t, const double* po) {
    draw(key, DHMC_STREAM_P, t, po);
  }
  __device__ __forceinline__ void draw_search_momentum(dm_rng_key key, const double* po) {
    draw(key, DHMC_STREAM_PSEARCH, 0, po);
  }

  __device__ __forceinline__ double kinetic_partial() const {
    double acc = 0.0;
#pragma unroll
    for (int e = 0; e < EPL; ++e) {
      if constexpr (DENSE) {
        acc = acc + p[e] * ps[e];
      } else {
        double psv = minv[e] * p[e];
        acc = acc + p[e] * psv;
      }
    }
    return acc;
  }
  __device__ __forceinline__ static double hamiltonian_logdensity(double l, double ksum) {
    if (!dm_isfinite(l)) return -dm_inf();          // hamiltonian.jl:253
    double K = ksum / 2.0;                          // :103
    return l - (dm_isfinite(K) ? K : dm_inf());     // :255
  }
  // logdensity(H, z) for the current point — hamiltonian.jl:251-256
  __device__ __forceinline__ double phase_logdensity() {
    double r[1] = {kinetic_partial()};
    reduce(r);
    return hamiltonian_logdensity(lq, r[0]);
  }

  // evaluate_ℓ sanitising — hamiltonian.jl:205-211 (non-strict)
  __device__ __forceinline__ static double sanitise(double l, bool gbad) {
    if ((dm_isfinite(l) && !gbad) || l == -dm_inf()) return l;
    return -dm_inf();
  }

  // ---- packed chain groups: one likelihood round of the whole CTA (coop_core_tma above) ----
  // Returns false (attendants only) when every warp of the CTA is done.
  __device__ __forceinline__ bool coop_round(bool active, double& sum_ll, double (&xtr)[EPL]) {
    static_assert(PACK > 1, "packed groups only");
    if (active) {
#pragma unroll
      for (int e = 0; e < EPL; ++e) {
        const int i = tid + e * T;
        if (i < D) cb_beta[(size_t)grp * kTmaBS + i] = q[e];      // [chain][coefficient]
      }
    }
    double sll = 0.0;
    if (!coop_core_tma<G>(&sll, active, tid, grp, ctid, D, lN, lXp, ly, cb_shared, ring_n))
      return false;                      // explicit flag (uniform over the CTA), not a property of the data
    sum_ll = sll;
    if (active) {
#pragma unroll
      for (int e = 0; e < EPL; ++e) {
        const int i = tid + e * T;
        xtr[e] = i < D ? cb_grad[(size_t)grp * tma_xs(D) + i] : 0.0;
      }
    }
    return true;
  }
  // packed groups, Symmetric metric: y = M⁻¹x of all chains of the CTA (coop_matvec_tma)
  static constexpr bool kCoopMatvec = DENSE && PACK > 1;
  int pooled;                               // the dense metric is shared by the CTA's 8 chains (DHMC_METRIC_SYMMETRIC_POOLED)
  __device__ __forceinline__ bool coop_matvec_call(bool act) {
    if (pooled) return coop_matmul_pooled_tma<G>(act, chain, tid, grp, ctid, D, Mp, cb_shared, ring_n);
    return coop_matvec_tma<G>(act, chain, tid, grp, ctid, D, Mp, cb_shared, ring_n);
  }
  __device__ __forceinline__ void coop_matvec(const double (&x)[EPL], double (&y)[EPL]) {
#pragma unroll
    for (int e = 0; e < EPL; ++e) {
      const int i = tid + e * T;
      if (i < D) cb_beta[(size_t)grp * kTmaBS + i] = x[e];
    }
    coop_matvec_call(true);
    const double* yb = pooled ? reinterpret_cast<const double*>(cb_shared + tma_y_off(G)) : cb_beta;
#pragma unroll
    for (int e = 0; e < EPL; ++e) {
      const int i = tid + e * T;
      y[e] = i < D ? yb[(size_t)grp * kTmaBS + i] : 0.0;
    }
  }
  // a warp without further chains keeps attending the CTA's cooperative calls, in the order a leapfrog step makes
  // them (M⁻¹pₘ, likelihood, M⁻¹p′ with the cooperative mat-vec; the likelihood alone otherwise)
  __device__ __forceinline__ void coop_finish() {
    if constexpr (PACK > 1) {
      double dummy_ll = 0.0;
      double dummy[EPL];
      if constexpr (kCoopMatvec) {
        while (coop_matvec_call(false)) {
          coop_round(false, dummy_ll, dummy);
          coop_matvec_call(false);
        }
      } else {
        while (coop_round(false, dummy_ll, dummy)) {}
      }
    }
  }

#ifdef DHMC_HAVE_USER_FAMILY
  // USER family (include/dhmc_models.h, "the model header contract"): the chain's whole position is staged in shared
  // memory so that an element's formulas may look at any other element, the K sums run through the canonical
  // reduction, then every thread evaluates the gradient of its own elements.  Same flag / sanitising conventions as the
  // shipped families below.
  __device__ __forceinline__ void eval_user(bool with_p, double h, double qbad_in, double* ksum, int* flags) {
    constexpr int K = DHMC_USER_NSUMS, M = DHMC_USER_NSCALARS;
#pragma unroll
    for (int e = 0; e < EPL; ++e) xs[tid + e * T] = q[e];
    group_sync();
    double r1[K + 1];
#pragma unroll
    for (int k = 0; k < K; ++k) r1[k] = 0.0;
    r1[K] = qbad_in;
#if DHMC_USER_NSUMS > 0
#pragma unroll
    for (int e = 0; e < EPL; ++e) {
      const int i = tid + e * T;
      if (i < D) {
        double t[K];
        dhmc_user_terms(i, D, xs, mparams, t);
#pragma unroll
        for (int k = 0; k < K; ++k) r1[k] = r1[k] + t[k];
      }
    }
#endif
    reduce(r1);
    double S[K + M > 0 ? K + M : 1];
    S[0] = 0.0;
#pragma unroll
    for (int k = 0; k < K; ++k) S[k] = r1[k];
#if DHMC_USER_NSCALARS > 0
    dhmc_user_prepare(D, xs, S, mparams);
#endif
    double r2[2] = {0.0, 0.0};                     // Σ p·p♯, bad ∇ℓ
#pragma unroll
    for (int e = 0; e < EPL; ++e) {
      const int i = tid + e * T;
      double ge = 0.0;
      if (i < D) {
        ge = dhmc_user_grad(i, D, xs, S, mparams);
        if (!dm_isfinite(ge)) r2[1] = 1.0;
      }
      g[e] = ge;
      if (with_p) {
        p[e] = p[e] + h * ge;
        if constexpr (!DENSE) {
          double psv = minv[e] * p[e];
          r2[0] = r2[0] + p[e] * psv;
        }
      }
    }
    double l = dhmc_user_logdensity(D, xs, S, mparams);
    reduce(r2);
    if (!((dm_isfinite(l) && r2[1] == 0.0) || l == -dm_inf())) *flags |= 4;
    l = sanitise(l, r2[1] != 0.0);
    if (r1[K] != 0.0) { *flags |= 1; l = -dm_inf(); }
    if (r2[1] != 0.0) *flags |= 2;
    lq = l;
    *ksum = r2[0];
    group_sync();                                  // the staging vector is rewritten by the next evaluation / mat-vec
  }
#endif

  // Model evaluation at the current q: fills g, sets lq (sanitised).  If
  // `with_p`, also performs the second momentum half-step p += h·∇ℓ(q′) and
  // returns Σ p·(M⁻¹p) through *ksum (fused into the same reductions).
  // flags bit0: non-finite q (reference throws, hamiltonian.jl:203), bit1: bad gradient,
  // bit2: ℓq was replaced by −Inf (what `strict` turns into an error, :212-215).
  __device__ __forceinline__ void eval_model(bool with_p, double h, double qbad_in, double* ksum,
                                             int* flags) {
    if constexpr (FAM == DHMC_FAMILY_LOGISTIC && PACK > 1) {
      double r[5] = {0.0, 0.0, qbad_in, 0.0, 0.0};   // Σ ll, Σ β², bad q, bad ∇ℓ, Σ p·p♯
      double acc[EPL];
      coop_round(true, r[0], acc);
#pragma unroll
      for (int e = 0; e < EPL; ++e) {
        const int i = tid + e * T;
        double ge = 0.0;
        if (i < D) {
          ge = dhmc_logit_grad(acc[e], q[e]);
          if (!dm_isfinite(ge)) r[3] = 1.0;
        }
        r[1] = r[1] + q[e] * q[e];
        g[e] = ge;
        if (with_p) {
          p[e] = p[e] + h * ge;
          if constexpr (!DENSE) {
            double psv = minv[e] * p[e];
            r[4] = r[4] + p[e] * psv;
          }
        }
      }
      reduce(r);
      double l = dhmc_logit_lq(r[0], r[1]);
      if (!((dm_isfinite(l) && r[3] == 0.0) || l == -dm_inf())) *flags |= 4;
      l = sanitise(l, r[3] != 0.0);
      if (r[2] != 0.0) { *flags |= 1; l = -dm_inf(); }
      if (r[3] != 0.0) *flags |= 2;
      lq = l;
      *ksum = r[4];
    } else if (FAM == DHMC_FAMILY_LOGISTIC) {
      // η = Xβ: β is staged in shared memory, thread t handles rows n = t, t+T, …
      // (Xᵀ read coalesced over n); residuals go to the per-CTA scratch, then every
      // thread accumulates its own gradient elements over n = 0..N-1 (X read coalesced over j).
#pragma unroll
      for (int e = 0; e < EPL; ++e) xs[tid + e * T] = q[e];
      group_sync();
      double r[5] = {0.0, 0.0, qbad_in, 0.0, 0.0};   // Σ ll, Σ β², bad q, bad ∇ℓ, Σ p·p♯
      for (int n0 = tid; n0 < lN; n0 += 4 * T) {     // four rows per pass for ILP
        double eta[4] = {0.0, 0.0, 0.0, 0.0};
        const double* col = lXt + n0;
        for (int j0 = 0; j0 < D; j0 += DHMC_LOGIT_CHUNK) {      // blocked dot product: dhmc_logit_eta
          const int j1 = j0 + DHMC_LOGIT_CHUNK < D ? j0 + DHMC_LOGIT_CHUNK : D;
          double sacc[4] = {0.0, 0.0, 0.0, 0.0};
          for (int j = j0; j < j1; ++j, col += lLd) {
            const double bj = xs[j];
#pragma unroll
            for (int u = 0; u < 4; ++u)
              if (n0 + u * T < lN) sacc[u] = dhmc_logit_mac(sacc[u], __ldg(col + u * T), bj);
          }
#pragma unroll
          for (int u = 0; u < 4; ++u) eta[u] = j0 == 0 ? sacc[u] : eta[u] + sacc[u];
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int n = n0 + u * T;
          if (n < lN) {
            const double yn = __ldg(ly + n);
            double llv, rv;
            dhmc_logit_ll_resid(yn, eta[u], &llv, &rv);
            r[0] = r[0] + llv;
            lr[n] = rv;
          }
        }
      }
      group_sync();
      double acc[EPL];
#pragma unroll
      for (int e = 0; e < EPL; ++e) acc[e] = 0.0;
      const double* row = lX + tid;
      for (int n = 0; n < lN; ++n, row += D) {
        const double rn = lr[n];
#pragma unroll
        for (int e = 0; e < EPL; ++e)
          if (tid + e * T < D) acc[e] = dhmc_logit_mac(acc[e], __ldg(row + e * T), rn);
      }
      group_sync();
#pragma unroll
      for (int e = 0; e < EPL; ++e) {
        const int i = tid + e * T;
        double ge = 0.0;
        if (i < D) {
          ge = dhmc_logit_grad(acc[e], q[e]);
          if (!dm_isfinite(ge)) r[3] = 1.0;
        }
        r[1] = r[1] + q[e] * q[e];
        g[e] = ge;
        if (with_p) {
          p[e] = p[e] + h * ge;
          if constexpr (!DENSE) {
            double psv = minv[e] * p[e];
            r[4] = r[4] + p[e] * psv;
          }
        }
      }
      reduce_leaf(r);
      double l = dhmc_logit_lq(r[0], r[1]);
      if (!((dm_isfinite(l) && r[3] == 0.0) || l == -dm_inf())) *flags |= 4;
      l = sanitise(l, r[3] != 0.0);
      if (r[2] != 0.0) { *flags |= 1; l = -dm_inf(); }
      if (r[3] != 0.0) *flags |= 2;
      lq = l;
      *ksum = r[4];
#ifdef DHMC_HAVE_USER_FAMILY
    } else if constexpr (FAM == DHMC_FAMILY_USER) {
      eval_user(with_p, h, qbad_in, ksum, flags);
#endif
    } else if (FAM == DHMC_FAMILY_FUNNEL) {
      double r1[3] = {0.0, 0.0, qbad_in};
#pragma unroll
      for (int e = 0; e < EPL; ++e) {
        const int i = tid + e * T;
        r1[0] = r1[0] + dhmc_funnel_term(i, q[e]);
        if (i == 0) r1[1] = q[e];
      }
      reduce(r1);
      const double S = r1[0], v = r1[1];
      const double ev = dm_exp(-v);
      double r2[2] = {0.0, 0.0};
#pragma unroll
      for (int e = 0; e < EPL; ++e) {
        const int i = tid + e * T;
        double ge = 0.0;
        if (i < D) {
          ge = dhmc_funnel_grad(i, q[e], v, ev, S, D);
          if (!dm_isfinite(ge)) r2[1] = 1.0;
        }
        g[e] = ge;
        if (with_p) {
          p[e] = p[e] + h * ge;
          if constexpr (!DENSE) {
            double psv = minv[e] * p[e];
            r2[0] = r2[0] + p[e] * psv;
          }
        }
      }
      reduce_leaf(r2);
      double l = dhmc_funnel_lq(v, ev, S, D);
      if (!((dm_isfinite(l) && r2[1] == 0.0) || l == -dm_inf())) *flags |= 4;
      l = sanitise(l, r2[1] != 0.0);
      if (r1[2] != 0.0) { *flags |= 1; l = -dm_inf(); }
      if (r2[1] != 0.0) *flags |= 2;
      lq = l;
      *ksum = r2[0];
    } else {
      double r[4] = {0.0, 0.0, qbad_in, 0.0};   // Σ term, Σ p·p♯, bad q, bad ∇ℓ
#pragma unroll
      for (int e = 0; e < EPL; ++e) {
        const int i = tid + e * T;
        double ge;
        if (FAM == DHMC_FAMILY_STD_NORMAL) {
          r[0] = r[0] + dhmc_std_term(q[e]);
          ge = dhmc_std_grad(q[e]);
        } else {
          double mu = 0.0, pr = 0.0;
          if (i < D) { mu = __ldg(mparams + i); pr = __ldg(mparams + D + i); }
          const double tt = dhmc_diag_scaled(q[e], mu, pr);
          r[0] = r[0] + dhmc_diag_term(q[e], mu, tt);
          ge = dhmc_diag_grad(tt);
        }
        if (i < D && !dm_isfinite(ge)) r[3] = 1.0;
        g[e] = ge;
        if (with_p) {
          p[e] = p[e] + h * ge;
          if constexpr (!DENSE) {
            double psv = minv[e] * p[e];
            r[1] = r[1] + p[e] * psv;
          }
        }
      }
      reduce_leaf(r);
      double l = (FAM == DHMC_FAMILY_STD_NORMAL) ? dhmc_std_lq(r[0]) : dhmc_diag_lq(r[0]);
      if (!((dm_isfinite(l) && r[3] == 0.0) || l == -dm_inf())) *flags |= 4;
      l = sanitise(l, r[3] != 0.0);
      if (r[2] != 0.0) { *flags |= 1; l = -dm_inf(); }
      if (r[3] != 0.0) *flags |= 2;
      lq = l;
      *ksum = r[1];
    }
  }

  // leapfrog(H, z, ϵ) — hamiltonian.jl:273-282, then logdensity(H, z′).
  // sp, nc, dbl: the merges the new leaf may need (see reduce_fused); dense and packed backends check them one at a time
  __device__ __forceinline__ double leapfrog(double eps, int* flags, int sp = 0, int nc = 0, bool dbl = false) {
    DHMC_PHASE(*this, kPhLfElem);
    if constexpr (kFused) { m_sp = sp; m_c = nc; m_dbl = dbl ? 1 : 0; }
    tid = pin(tid); lane = pin(lane); warp = pin(warp); mparams = pin(mparams);
    const double h = eps / 2;
    double qbad = 0.0;
    if constexpr (DENSE) {
      double vel[EPL];
#pragma unroll
      for (int e = 0; e < EPL; ++e) p[e] = p[e] + h * g[e];       // pₘ                        :277
      if constexpr (kCoopMatvec) coop_matvec(p, vel); else matvec(p, vel);   // ∇kinetic_energy = M⁻¹ pₘ  :117
#pragma unroll
      for (int e = 0; e < EPL; ++e) {
        q[e] = q[e] + eps * vel[e];                               // q′                        :278
        if (!dm_isfinite(q[e])) qbad = 1.0;
      }
      double ksum;
      eval_model(true, h, qbad, &ksum, flags);                    // Q′, p′                    :279-280
      if constexpr (kCoopMatvec) coop_matvec(p, ps); else matvec(p, ps);     // p♯′ = M⁻¹ p′ (K and turn statistics)
      double r[1] = {kinetic_partial()};
      reduce(r);
      return hamiltonian_logdensity(lq, r[0]);
    } else {
#pragma unroll
      for (int e = 0; e < EPL; ++e) {
        p[e] = p[e] + h * g[e];                 // pₘ = p + ϵ/2 * ∇ℓq        :277
        const double vel = minv[e] * p[e];      // ∇kinetic_energy = M⁻¹ pₘ  :117
        q[e] = q[e] + eps * vel;                // q′ = q + ϵ * (…)           :278
        if (!dm_isfinite(q[e])) qbad = 1.0;
      }
      double ksum;
      eval_model(true, h, qbad, &ksum, flags);  // Q′ = evaluate_ℓ; p′ = pₘ + ϵ/2 ∇ℓq′  :279-280
      if constexpr (kFused) { m_c = 0; m_dbl = 0; }
      return hamiltonian_logdensity(lq, ksum);
    }
  }

  // The six dot products of combine_turn_statistics (NUTS.jl:130-139) in build
  // order; leaves the combined ρ in rhoL.  Returns true when turning.
  // j: the merge's place among those of the current leaf (reduce_fused).
  __device__ __forceinline__ bool merge_check(int j, int sEf, int sEl, int sEr, int sLf, bool L_leaf) {
    if constexpr (kFused) {                 // the sums came with the leapfrog's all-reduce
      const int g = j + m_shift;
      if (g == 0)
        return warp_sum(m_buf + kLeafCol, red_row) < 0 || warp_sum(m_buf + kLeafCol + 1, red_row) < 0;
      const double* bg = m_buf + g * kRedWidth;
      double d[6];
#pragma unroll
      for (int n = 0; n < 6; ++n) d[n] = warp_sum(bg + n, red_row);
      return d[0] < 0 || d[1] < 0 || d[2] < 0 || d[3] < 0 || d[4] < 0 || d[5] < 0;
    }
    DHMC_PHASE(*this, kPhMcElem);
    if constexpr (DENSE) {
      // p♯ of the four edge momenta come from the slots (stored next to p); ρ slots hold ρ only
      const double* pEf = slot(sEf);
      const double* pEl = slot(sEl);
      const double* pEr = slot(sEr);
      const double* pLf = L_leaf ? pEf : slot(sLf);
      double d[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
      for (int e = 0; e < EPL; ++e) {
        const double Ef = pEf[e * T], El = pEl[e * T], Er = pEr[e * T];
        const double sEfv = pEf[vstride + e * T], sElv = pEl[vstride + e * T];
        const double Lf = L_leaf ? p[e] : pLf[e * T];
        const double sLfv = L_leaf ? ps[e] : pLf[vstride + e * T];
        const double Lr = L_leaf ? p[e] : rhoL[e];
        const double A = Er + Lf, Bv = El + Lr, R = Er + Lr;
        d[0] = d[0] + sEfv * A;  d[1] = d[1] + sLfv * A;
        d[2] = d[2] + sElv * Bv; d[3] = d[3] + ps[e] * Bv;
        d[4] = d[4] + sEfv * R;  d[5] = d[5] + ps[e] * R;
        rhoL[e] = R;
      }
      reduce(d);
      return d[0] < 0 || d[1] < 0 || d[2] < 0 || d[3] < 0 || d[4] < 0 || d[5] < 0;
    }
    const double* pEf = slot(sEf);
    const bool e_leaf = (sEl == sEf);
    if (e_leaf && L_leaf) {
      // two single leaves (half of all merges): E.first = E.last = E.ρ = p_E and
      // L.first = L.last = L.ρ = p, so the three candidate sums coincide and the six
      // dot products collapse to two — the very same floating-point operations.
      double d[2] = {0.0, 0.0};
#pragma unroll
      for (int e = 0; e < EPL; ++e) {
        const double Ef = pEf[e * T];
        const double A = Ef + p[e];
        const double mEf = minv[e] * Ef, mLl = minv[e] * p[e];
        d[0] = d[0] + mEf * A;
        d[1] = d[1] + mLl * A;
        rhoL[e] = A;
      }
      reduce(d);
      return d[0] < 0 || d[1] < 0;
    }
    const double* pEl = slot(sEl);
    const double* pEr = slot(sEr);
    double d[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    if (!L_leaf) {
      const double* pLf = slot(sLf);
#pragma unroll
      for (int e = 0; e < EPL; ++e) {
        const double Ef = pEf[e * T], El = pEl[e * T], Er = pEr[e * T], Lf = pLf[e * T];
        const double Lr = rhoL[e];
        const double A = Er + Lf, Bv = El + Lr, R = Er + Lr;
        const double mEf = minv[e] * Ef, mLf = minv[e] * Lf, mEl = minv[e] * El, mLl = minv[e] * p[e];
        d[0] = d[0] + mEf * A;  d[1] = d[1] + mLf * A;
        d[2] = d[2] + mEl * Bv; d[3] = d[3] + mLl * Bv;
        d[4] = d[4] + mEf * R;  d[5] = d[5] + mLl * R;
        rhoL[e] = R;
      }
    } else {
      // whole tree so far (three distinct vectors) against a single new leaf: only at depth 0
#pragma unroll
      for (int e = 0; e < EPL; ++e) {
        const double Ef = pEf[e * T];
        const double El = e_leaf ? Ef : pEl[e * T];
        const double Er = e_leaf ? Ef : pEr[e * T];
        const double Lf = p[e], Lr = p[e];
        const double A = Er + Lf, Bv = El + Lr, R = Er + Lr;
        const double mEf = minv[e] * Ef, mLf = minv[e] * Lf, mEl = minv[e] * El, mLl = minv[e] * p[e];
        d[0] = d[0] + mEf * A;  d[1] = d[1] + mLf * A;
        d[2] = d[2] + mEl * Bv; d[3] = d[3] + mLl * Bv;
        d[4] = d[4] + mEf * R;  d[5] = d[5] + mLl * R;
        rhoL[e] = R;
      }
    }
    reduce(d);
    return d[0] < 0 || d[1] < 0 || d[2] < 0 || d[3] < 0 || d[4] < 0 || d[5] < 0;
  }

  // streaming window statistics — sample_M⁻¹, mcmc.jl:209 (Diagonal) / :211 (Symmetric)
  __device__ __forceinline__ void metric_reset(int kind) {
    double* m = slot(n_slots - 1); double* sv = slot(n_slots - 2);
#pragma unroll
    for (int e = 0; e < EPL; ++e) { m[e * T] = 0.0; sv[e * T] = 0.0; }
    if (kind == DHMC_METRIC_SYMMETRIC) {
      for (int j = 0; j < D; ++j) {
#pragma unroll
        for (int e = 0; e < EPL; ++e) if (tid + e * T < D) covt[(size_t)j * D + tid + e * T] = 0.0;
      }
    }
  }
  __device__ __forceinline__ void metric_push(int kind, int n) {
    double* m = slot(n_slots - 1); double* sv = slot(n_slots - 2);
    const double dn = (double)n;
    double dl[EPL];
#pragma unroll
    for (int e = 0; e < EPL; ++e) {
      const double mean = m[e * T];
      const double dlt = q[e] - mean;
      const double mean1 = mean + dlt / dn;
      m[e * T] = mean1;
      dl[e] = dlt;
      if (kind == DHMC_METRIC_DIAGONAL) sv[e * T] = sv[e * T] + dlt * (q[e] - mean1);
      else xs[tid + e * T] = q[e] - mean1;
    }
    if (kind == DHMC_METRIC_SYMMETRIC) {
      // co-moments C[i][j] += δ_i (x_j − mean′_j), j ≤ i, stored transposed (coalesced over i)
      group_sync();
      double* col = covt + tid;
      for (int j = 0; j < D; ++j, col += D) {
        const double yj = xs[j];
#pragma unroll
        for (int e = 0; e < EPL; ++e) {
          const int i = tid + e * T;
          if (i < D && j <= i) col[e * T] = col[e * T] + dl[e] * yj;
        }
      }
      group_sync();
    }
  }
  __device__ __forceinline__ void metric_finish(int kind, int n) {
    if (kind != DHMC_METRIC_DIAGONAL) {         // Symmetric: finished by k_cov_finish / k_cov_pool + k_dense_factor
      if (mean_out) {                           // pooled stage: the group merge needs every chain's window mean
        const double* m = slot(n_slots - 1);
#pragma unroll
        for (int e = 0; e < EPL; ++e) if (valid(e)) mean_out[tid + e * T] = m[e * T];
      }
      return;
    }
    const double* sv = slot(n_slots - 2);
    const double dn1 = (double)(n - 1);
#pragma unroll
    for (int e = 0; e < EPL; ++e) minv[e] = valid(e) ? sv[e * T] / dn1 : 1.0;
  }
};

}  // namespace dhmc
