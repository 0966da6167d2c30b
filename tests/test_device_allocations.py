"""Every device allocation of the C ABI may fail, and a handle survives it.  The fault-injection build of the library
(csrc/Makefile `faults`: -DDHMC_ALLOC_FAULTS) fails the k-th next device allocation on request and counts the live ones.
For every allocation of every call of a scenario, the failed call returns DHMC_ENOMEM and frees its temporaries: it holds
no more device allocations than the successful call leaves (grow-only scratch and the dense-metric arrays it allocated
before the failure stay with the handle, for the repeat to use).  The same call repeated then holds exactly as many as the
successful call, and the rest of the scenario gives draws, statistics and summaries bit-identical to a handle that never
saw a failure (sums that the device folds with floating-point atomics, whose order differs between any two runs, to
1e-12).  dhmc_destroy leaves no allocation behind."""
import ctypes as C
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAULTS_LIB = os.path.join(ROOT, "dynamichmc.jl_b200", "csrc", "build", "libdhmc_b200_faults.so")


def _faults_lib(pkg):
    lib = pkg._lib.lib(FAULTS_LIB)
    lib.dhmc_test_fail_alloc.argtypes = [C.c_int64]
    lib.dhmc_test_fail_alloc.restype = None
    lib.dhmc_test_live_allocations.argtypes = []
    lib.dhmc_test_live_allocations.restype = C.c_int64
    return lib


def _bits(a):
    """The bytes of an output; tree statistics without their padding field."""
    if a.dtype.names:
        return tuple(a[f].tobytes() for f in a.dtype.names if f != "pad")
    return a.tobytes()


class Run:
    """One handle of the fault-injection library driven through a scenario; `out` collects what its calls return."""

    def __init__(self, pkg, lib, **cfg):
        self.L, self.lib, self.h, self.out, self.approx = pkg._lib, lib, C.c_void_p(), {}, {}
        self.cfg = pkg._lib.Config(device=0, max_depth=10, threads_per_chain=0, min_delta=-1000.0, ctas_per_sm=0,
                                   reserved=0, chain_offset=0, **cfg)
        self.B, self.D = cfg["n_chains"], cfg["dim"]

    def p(self, a):
        return self.L.ptr(a)

    def stats(self, n):
        return np.zeros((self.B, n), dtype=self.L.tree_stats_dtype)


def _create(r):
    return r.lib.dhmc_create(C.byref(r.cfg), C.byref(r.h))


def _random_position(r):
    return r.lib.dhmc_random_position(r.h)


def _stepsize(eps):
    return lambda r: r.lib.dhmc_set_stepsize(r.h, r.p(np.array([eps])), 1)


def _set_problems(blocks, K):
    def step(r):
        pr = np.concatenate(blocks)
        return r.lib.dhmc_set_problems(r.h, r.p(pr), C.c_size_t(blocks[0].size), C.c_int64(len(blocks)), C.c_int64(K))
    return step


def _mcmc(N, name="mcmc"):
    def step(r):
        post, st, ld = np.empty((r.B, N, r.D)), r.stats(N), np.empty((r.B, N))
        rc = r.lib.dhmc_mcmc(r.h, C.c_int32(N), r.p(post), r.p(st), r.p(ld))
        r.out[name] = (post, st, ld)
        return rc
    return step


def _warmup(N, metric, name):
    def step(r):
        post, st, eps, ld = np.empty((r.B, N, r.D)), r.stats(N), np.empty((r.B, N)), np.empty((r.B, N))
        da = C.byref(r.L.DualAveragingC(0.8, 0.05, 0.75, 10, 0))
        rc = r.lib.dhmc_warmup_stage(r.h, C.c_int32(N), C.c_int32(metric), da, C.c_double(0.05), r.p(post), r.p(st),
                                     r.p(eps), r.p(ld))
        r.out[name] = (post, st, eps, ld)
        return rc
    return step


def _state(r):
    q, lq, g, minv, eps, p = (np.empty((r.B, r.D)), np.empty(r.B), np.empty((r.B, r.D)), np.empty((r.B, r.D)),
                              np.empty(r.B), np.empty((r.B, r.D)))
    rc = r.lib.dhmc_get_state(r.h, r.p(q), r.p(lq), r.p(g), r.p(minv), r.p(eps), r.p(p))
    r.out["state"] = (q, lq, g, minv, eps, p)
    return rc


def _logistic_block(N, D, seed):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(N, D)) / np.sqrt(D)
    y = (rng.uniform(size=N) < 0.5) * 1.0
    return np.concatenate([[float(N)], X.ravel(), y])


def _diag_normal_blocks(D, P, seed):
    rng = np.random.default_rng(seed)
    return [np.concatenate([rng.normal(size=D), rng.uniform(0.5, 2.0, D)]) for _ in range(P)]


def _sample_tree(r):
    """One tree from a given momentum and given directions (their scratch: tmp_bd, tmp_dir)."""
    rng = np.random.default_rng(7)
    p, dirs, st = rng.normal(size=(r.B, r.D)), rng.integers(0, 2 ** 31, r.B, dtype=np.uint32), r.stats(1)
    rc = r.lib.dhmc_sample_tree(r.h, r.p(p), r.p(dirs), r.p(st))
    r.out["tree"] = (st,)
    return rc


def _phase(r):
    phase = np.empty(r.B)
    rc = r.lib.dhmc_phase_logdensity(r.h, r.p(phase))
    r.out["phase"] = (phase,)
    return rc


def _summary_histogram(N, nbins):
    def step(r):
        P = r.out_P
        R = r.D
        ref = np.zeros((P, R))
        lo, hi = np.full((P, R), -4.0), np.full((P, R), 4.0)
        rec = np.empty((P, R, r.L.SUMMARY_FIELDS))
        cnt = np.empty((P, R, nbins + 2), dtype=np.int64)
        st, ld = r.stats(N), np.empty((r.B, N))
        rc = r.lib.dhmc_mcmc_summary_histogram(r.h, N, 1, r.p(ref), r.p(lo), r.p(hi), nbins, r.p(rec), r.p(cnt), r.p(st),
                                               r.p(ld))
        exact = [r.L.SUMMARY_CHAINS, r.L.SUMMARY_NKEEP, r.L.SUMMARY_BELOW]
        r.out["summary"] = (np.ascontiguousarray(rec[..., exact]), cnt, st, ld)
        r.approx["summary"] = (np.delete(rec, exact, axis=-1),)
        return rc
    return step


def _diagnostics(N):
    """dhmc_mcmc_dev into device arrays, then the device reductions over them."""
    def sample(r):
        import torch
        r.draws = torch.empty(r.B * N * r.D, dtype=torch.float64, device="cuda")
        r.stats_dev = torch.empty(r.B * N * r.L.tree_stats_dtype.itemsize, dtype=torch.uint8, device="cuda")
        return r.lib.dhmc_mcmc_dev(r.h, C.c_int32(N), C.c_void_p(r.draws.data_ptr()), C.c_void_p(r.stats_dev.data_ptr()), None)

    def tree_summary(r):
        depth, term, acc, steps, ebfmi = (np.empty(33, np.int64), np.empty(3, np.int64), np.empty(1), np.empty(1, np.int64),
                                          np.empty(r.B))
        rc = r.lib.dhmc_tree_summary_dev(r.h, C.c_void_p(r.stats_dev.data_ptr()), C.c_int32(N), r.p(depth), r.p(term),
                                         r.p(acc), r.p(steps), r.p(ebfmi))
        r.out["tree_summary"] = (depth, term, steps, ebfmi)
        r.approx["tree_summary"] = (acc,)
        return rc

    def ess_rhat(r):
        rhat, ess = np.empty((r.out_P, r.D)), np.empty((r.out_P, r.D))
        rc = r.lib.dhmc_ess_rhat_problems_dev(r.h, C.c_void_p(r.draws.data_ptr()), C.c_int32(N), C.c_int32(0), r.p(rhat),
                                              r.p(ess))
        r.approx["ess_rhat"] = (rhat, ess)
        return rc

    def acceptance_quantiles(r):
        probs, q = np.array([0.1, 0.5, 0.9]), np.empty(3)
        rc = r.lib.dhmc_acceptance_quantiles_dev(r.h, C.c_void_p(r.stats_dev.data_ptr()), C.c_int32(N), r.p(probs),
                                                 C.c_int32(3), r.p(q))
        r.out["acceptance_quantiles"] = (q,)
        return rc

    def download(r):
        r.out["draws"] = (r.draws.cpu().numpy(), r.stats_dev.cpu().numpy().view(r.L.tree_stats_dtype))
        return 0

    return [sample, tree_summary, ess_rhat, acceptance_quantiles, download]


def _scenarios():
    D_LOG, D_DN = 12, 3
    logistic = [_logistic_block(40, D_LOG, 1), _logistic_block(40, D_LOG, 2)]
    dn = _diag_normal_blocks(D_DN, 2, 3)
    eye = np.eye(D_DN).ravel()
    return {
        # packed chain groups (automatic layout, dim <= 256): the batch installer's arrays and the residual scratch
        "logistic_batch": (dict(family=3, dim=D_LOG, n_chains=16, seed=11),
                           [_create, _set_problems(logistic, 8), _random_position, _stepsize(0.05), _mcmc(3), _state]),
        # ensure_dense, the diagonal → dense re-plan (dhmc_set_metric_dense), a Symmetric stage on the dense kernels, the
        # dense → diagonal re-plan (dhmc_set_metric)
        "dense_metric": (dict(family=1, dim=D_DN, n_chains=16, seed=12),
                         [_create, _set_problems(dn, 8), _random_position, _stepsize(0.3),
                          lambda r: r.lib.dhmc_set_metric_dense(r.h, r.p(eye), 1), _warmup(20, 2, "symmetric"),
                          lambda r: r.lib.dhmc_set_metric(r.h, r.p(np.ones(D_DN)), 1), _mcmc(4), _state]),
        "pooled_warmup": (dict(family=1, dim=D_DN, n_chains=16, seed=13),
                          [_create, _set_problems(dn, 8), _random_position, _stepsize(0.3),
                           lambda r: r.lib.dhmc_set_metric_dense(r.h, r.p(eye), 1), _warmup(20, 3, "pooled"), _mcmc(4),
                           _state]),
        "staged_mcmc": (dict(family=0, dim=5, n_chains=16, seed=14),
                        [_create, _random_position, _stepsize(0.4), _sample_tree, _phase, _mcmc(6), _mcmc(3, "again"), _state]),
        "summary_histogram": (dict(family=1, dim=D_DN, n_chains=16, seed=15),
                              [_create, _set_problems(dn, 8), _random_position, _stepsize(0.3), _summary_histogram(8, 16),
                               _state]),
        "diagnostics": (dict(family=1, dim=D_DN, n_chains=16, seed=16),
                        [_create, _set_problems(dn, 8), _random_position, _stepsize(0.3)] + _diagnostics(8)),
    }


def _run_steps(r, steps):
    for i, step in enumerate(steps):
        rc = step(r)
        assert rc == 0, (i, rc, r.lib.dhmc_last_error(r.h if r.h.value else None))


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(_scenarios()))
def test_every_failed_allocation_leaves_a_usable_handle(pkg, name):
    lib = _faults_lib(pkg)
    cfg, steps = _scenarios()[name]
    P = 2 if name != "staged_mcmc" else 1

    runs = []

    def fresh():
        r = Run(pkg, lib, **cfg)
        r.out_P = P
        runs.append(r)
        return r

    def finish(r):
        lib.dhmc_destroy(r.h)
        r.h = C.c_void_p()
        assert lib.dhmc_test_live_allocations() == 0
        return {k: [_bits(a) for a in v] for k, v in r.out.items()}, r.approx

    def same(got, want):
        (g_exact, g_approx), (w_exact, w_approx) = got, want
        assert g_exact.keys() == w_exact.keys() and g_approx.keys() == w_approx.keys()
        bad = [k for k in w_exact if g_exact[k] != w_exact[k]]
        for k in w_approx:
            for g, w in zip(g_approx[k], w_approx[k]):
                scale = np.abs(w[np.isfinite(w)]).max(initial=0.0)
                if not (np.array_equal(np.isnan(g), np.isnan(w)) and np.allclose(g, w, rtol=1e-12, atol=1e-12 * scale, equal_nan=True)):
                    bad.append(k)
        assert not bad, bad
        return True

    assert lib.dhmc_test_live_allocations() == 0
    try:
        ref, ref_live = fresh(), []
        for step in steps:                           # live allocations after each call of the run without failures
            _run_steps(ref, [step])
            ref_live.append(lib.dhmc_test_live_allocations())
        expect = finish(ref)
        failures = 0
        for i, step in enumerate(steps):
            for k in range(1, 100):
                r = fresh()
                _run_steps(r, steps[:i])
                lib.dhmc_test_fail_alloc(k)
                rc = step(r)
                lib.dhmc_test_fail_alloc(0)
                if rc == 0:                # the call makes fewer than k allocations
                    finish(r)
                    break
                failures += 1
                err = lib.dhmc_last_error(r.h if r.h.value else None).decode()
                assert rc == pkg._lib.DHMC_ENOMEM, (i, k, rc, err)
                # what the call allocated before the failure is freed, or kept by the handle as the successful call keeps it
                assert lib.dhmc_test_live_allocations() <= ref_live[i], (i, k, err)
                _run_steps(r, [step])
                assert lib.dhmc_test_live_allocations() == ref_live[i], (i, k, err)
                _run_steps(r, steps[i + 1:])
                assert same(finish(r), expect), (i, k, err)
            else:
                pytest.fail(f"step {i} still fails at its 99th allocation")
        assert failures >= 1
    finally:
        lib.dhmc_test_fail_alloc(0)
        for r in runs:
            if r.h.value:
                lib.dhmc_destroy(r.h)
