// leafsim.cpp — host simulation of the NUTS state machine (dynamichmc.jl_b200/csrc/nuts_machine.cuh) against a backend
// with the GPU's leaf-merge interface (kLeafMerges: leapfrog() is told which merges the new leaf may need, merge_check(j, …)
// hands out merge j's result), for `-m "not gpu"` tests (tests/test_slot_roles_host.py).  The backend evaluates a leaf's
// merges together with its leapfrog, as DeviceBackend's one all-reduce per leaf does, and audits the slot pool: reads of
// turn-check operands at slot index >= n_sm (off chip on the device) and live vectors sharing a slot.  Standard normal
// target, unit metric.  Test harness only: not linked into the library.
#include <cstring>
#include <set>
#include <vector>

#include "../../dynamichmc.jl_b200/csrc/nuts_machine.cuh"
#include "../../include/dhmc_models.h"

using vec = std::vector<double>;
using namespace dhmc;

namespace {

template <class F>
double canon_sum(int T, int D, F term) {          // the canonical reduction order (DESIGN.md §3)
  std::vector<double> part(T);
  for (int v = 0; v < T; ++v) {
    double acc = 0.0;
    for (int i = v; i < D; i += T) acc = acc + term(i);
    part[v] = acc;
  }
  for (int base = 0; base < T; base += 32)
    for (int off = 16; off >= 1; off >>= 1)
      for (int v = base; v < base + off; ++v) part[v] = part[v] + part[v + off];
  for (int off = 32; off < T; off <<= 1)
    for (int v = 0; v < T; v += 2 * off) part[v] = part[v] + part[v + off];
  return part[0];
}

struct LeafBackend {
  static constexpr bool kLeafMerges = true;
  static constexpr bool kDeep = true;             // exercise the spill words of the slot pool as well
  int D, T, reserved, n_sm;
  vec q, p, g, rhoL, Rnew;
  double lq = 0;
  std::vector<vec> slots;
  Entry entries[kMaxLevels + 2];
  TopState top_;
  long merge_reads = 0, offchip_reads = 0, slot_clashes = 0;
  std::vector<char> m_turn;                       // the current leaf's merges: turning?, combined ρ
  std::vector<vec> m_rho;

  LeafBackend(int D_, int T_, int nslots, int nsm)
      : D(D_), T(T_), reserved(nslots - kWelfordSlots), n_sm(nsm), q(D_), p(D_), g(D_), rhoL(D_), Rnew(D_),
        slots(nslots, vec(D_)) {}

  TopState& top() { return top_; }
  void top_sync() {}
  int reserved_first() const { return reserved; }  // the two highest slots, as on the device
  double cur_lq() const { return lq; }
  void set_cur_lq(double v) { lq = v; }
  void st_q(int s) { slots[s] = q; }
  void st_p(int s) { slots[s] = p; }
  void st_g(int s) { slots[s] = g; }
  void st_rho(int s) { slots[s] = rhoL; }
  void ld_q(int s) { q = slots[s]; }
  void ld_p(int s) { p = slots[s]; }
  void ld_g(int s) { g = slots[s]; }
  void swap_cur(int sq, int sp, int sg) { q.swap(slots[sq]); p.swap(slots[sp]); g.swap(slots[sg]); }
  void rho_from_p() { rhoL = p; }
  void rho_commit() { rhoL = Rnew; }
  void logaddexp2(double a0, double b0, double a1, double b1, double* r0, double* r1) {
    *r0 = dm_logaddexp(a0, b0); *r1 = dm_logaddexp(a1, b1);
  }
  double randexp(dm_rng_key key, uint32_t t, uint32_t j) { return dm_randexp(key, t, j); }
  void put_entry(int j, const Entry& e) {
    entries[j] = e;
    // every slot held by the stack entries 0…j and by the whole tree: a distinct, unreserved slot of the pool
    std::vector<int> live = {top_.s_oq, top_.s_og, top_.s_zq, top_.s_zg, top_.s_op, top_.s_near, top_.s_rhot};
    for (int i = 0; i <= j; ++i) {
      const Entry& x = entries[i];
      live.insert(live.end(), {x.sfirst, x.szq, x.szg});
      if (!x.leaf) live.insert(live.end(), {x.slast, x.srho});
    }
    std::set<int> seen;
    for (int s : live)
      if (s < 0 || s >= (int)slots.size() || s == reserved || s == reserved + 1 || !seen.insert(s).second) ++slot_clashes;
  }
  Entry get_entry(int j) const { return entries[j]; }
  void draw_momentum(dm_rng_key key, uint32_t t, const double*) {
    for (int i = 0; i < D; ++i) p[i] = dm_sqrt(1.0 / 1.0) * dm_normal_elem(key, DHMC_STREAM_P, t, (uint32_t)i);
  }
  void draw_search_momentum(dm_rng_key key, const double*) {
    for (int i = 0; i < D; ++i) p[i] = dm_sqrt(1.0 / 1.0) * dm_normal_elem(key, DHMC_STREAM_PSEARCH, 0, (uint32_t)i);
  }
  double phase_logdensity() const {
    if (!dm_isfinite(lq)) return -dm_inf();
    const double K = canon_sum(T, D, [&](int i) { double ps = 1.0 * p[i]; return p[i] * ps; }) / 2.0;
    return lq - (dm_isfinite(K) ? K : dm_inf());
  }
  double eval_model(bool* gbad) {
    const double s = canon_sum(T, D, [&](int i) { return dhmc_std_term(q[i]); });
    bool bad = false;
    for (int i = 0; i < D; ++i) { g[i] = dhmc_std_grad(q[i]); bad = bad || !dm_isfinite(g[i]); }
    *gbad = bad;
    const double l = dhmc_std_lq(s);
    return (dm_isfinite(l) && !bad) || l == -dm_inf() ? l : -dm_inf();
  }
  // the leaf's c stack merges (top entry first), then with dbl the doubling-level check, evaluated with the leapfrog
  double leapfrog(double eps, int* flags, int sp = 0, int c = 0, bool dbl = false) {
    const double h = eps / 2;
    for (int i = 0; i < D; ++i) p[i] = p[i] + h * g[i];
    bool qbad = false;
    for (int i = 0; i < D; ++i) { q[i] = q[i] + eps * (1.0 * p[i]); qbad = qbad || !dm_isfinite(q[i]); }
    bool gbad;
    lq = eval_model(&gbad);
    if (qbad) { *flags |= 1; lq = -dm_inf(); }
    for (int i = 0; i < D; ++i) p[i] = p[i] + h * g[i];
    const double H = phase_logdensity();
    const int nm = c + (dbl ? 1 : 0);
    m_turn.assign(nm, 0);
    m_rho.assign(nm, vec());
    rhoL = p;
    for (int j = 0; j < nm; ++j) {
      const bool stack = j < c;
      const int sEf = stack ? entries[sp - 1 - j].sfirst : top_.s_op;
      const int sEl = stack ? entries[sp - 1 - j].slast : top_.s_near;
      const int sEr = stack ? entries[sp - 1 - j].srho : top_.s_rhot;
      const bool lleaf = j == 0;
      m_turn[j] = turn_check(sEf, sEl, sEr, lleaf ? -1 : entries[sp - j].sfirst, lleaf);
      m_rho[j] = Rnew;
      rhoL = Rnew;
    }
    return H;
  }
  bool merge_check(int j, int, int, int, int, bool) {
    Rnew = m_rho[j];
    return m_turn[j];
  }
  void count_read(int s) { ++merge_reads; if (s >= n_sm) ++offchip_reads; }
  // the six dot products of combine_turn_statistics in build order (device_backend.cuh); the slot reads are those of the
  // device: p_E alone for two leaves, else E.first, E.last, E.ρ and, for an inner L, L.first
  bool turn_check(int sEf, int sEl, int sEr, int sLf, bool L_leaf) {
    count_read(sEf);
    if (!(L_leaf && sEl == sEf)) {
      count_read(sEl); count_read(sEr);
      if (!L_leaf) count_read(sLf);
    }
    const vec& Ef = slots[sEf]; const vec& El = slots[sEl]; const vec& Er = slots[sEr];
    const vec& Lf = L_leaf ? p : slots[sLf];
    const vec& Lr = L_leaf ? p : rhoL;
    vec A(D), Bv(D);
    for (int i = 0; i < D; ++i) { A[i] = Er[i] + Lf[i]; Bv[i] = El[i] + Lr[i]; Rnew[i] = Er[i] + Lr[i]; }
    auto dot = [&](const vec& a, const vec& r) { return canon_sum(T, D, [&](int i) { double ps = 1.0 * a[i]; return ps * r[i]; }); };
    return dot(Ef, A) < 0 || dot(Lf, A) < 0 || dot(El, Bv) < 0 || dot(p, Bv) < 0 || dot(Ef, Rnew) < 0 || dot(p, Rnew) < 0;
  }
  void metric_reset(int) {}
  void metric_push(int, int) {}
  void metric_finish(int, int) {}
};

struct Sink {
  LeafBackend& b; double* post; dhmc_tree_stats* stats;
  void operator()(int n, const dhmc_tree_stats& ts, double) {
    if (post) std::memcpy(post + (size_t)n * b.D, b.q.data(), sizeof(double) * b.D);
    if (stats) stats[n] = ts;
  }
};

}  // namespace

extern "C" {

// N transitions of a std-normal chain from q with step size eps (unit metric, no adaptation), T threads per chain, the
// first n_sm slots on chip.  post [N][D] / stats [N] may be null; counts: [0] turn-check operand reads, [1] those at slot
// index >= n_sm, [2] live slots found shared or outside the pool, [3] leapfrog steps.  Returns the chain status bits.
int ls_run(int D, int T, int max_depth, int n_sm, uint64_t seed, uint64_t chain, int N, double eps, const double* q,
           double* post, dhmc_tree_stats* stats, long* counts) {
  const int ns = slots_needed(max_depth);
  LeafBackend b(D, T, ns, n_sm);
  b.q.assign(q, q + D);
  bool gbad;
  b.lq = b.eval_model(&gbad);
  NutsMachine<LeafBackend> m(b, dm_make_key(seed, chain), max_depth, -1000.0, ns);
  static_assert(NutsMachine<LeafBackend>::kLeafMerges, "the leaf-merge interface");
  AdaptConfig cfg{};
  cfg.metric = DHMC_METRIC_NOTHING;
  Sink sink{b, post, stats};
  m.run(0, N, eps, cfg, nullptr, nullptr, sink);
  counts[0] = b.merge_reads; counts[1] = b.offchip_reads; counts[2] = b.slot_clashes; counts[3] = m.steps_out;
  return m.status;
}

}  // extern "C"
