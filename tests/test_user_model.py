"""User models — the device counterpart of handing the reference an arbitrary LogDensityProblems object
(`logdensity_and_gradient`, call site src/hamiltonian.jl:204): a header of scalar formulas (include/dhmc_models.h, "the
model header contract"; examples in include/models/) compiled into its own build of the library as family 4.

CPU part: the oracle built from the same header — (i) Neal's funnel written as a user model reproduces the shipped FUNNEL
family bit for bit (values, trees, whole warm-ups), which pins the user-model evaluation order to a shipped one; (ii) the
example models' ℓ, ∇ℓ against numpy closed forms and finite differences; (iii) the user-model library builds for sm_90a,
exports the whole C ABI and reports its model, while the stock library refuses family 4.
GPU part (-m gpu): the CUDA path of a user model against that oracle, bit for bit, and against the shipped family."""
import ctypes as C
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODELS = os.path.join(ROOT, "include", "models")
INT_FIELDS = ("depth", "left", "right", "steps", "directions")


def _hdr(name):
    return os.path.join(MODELS, name + ".h")


# ------------------------------------------------------------------ numpy forms of the example models
def rosenbrock_np(q, a, b):
    u = q[1:] - q[:-1] ** 2
    w = a - q[:-1]
    l = -float(np.sum(b * u * u + w * w))
    g = np.zeros_like(q)
    g[:-1] += 4 * b * q[:-1] * u + 2 * w
    g[1:] -= 2 * b * u
    return l, g


def eight_schools_np(q, y, sigma):
    mu, lt, eta = q[0], q[1], q[2:]
    tau = np.exp(lt)
    r = (y - mu - tau * eta) / sigma
    l = -0.5 * np.sum(r * r) - 0.5 * np.sum(eta * eta) - mu * mu / 50 - np.log1p(tau * tau / 25) + lt
    g = np.empty_like(q)
    g[0] = np.sum(r / sigma) - mu / 25
    g[1] = tau * np.sum(r * eta / sigma) - 2 * tau * tau / (25 + tau * tau) + 1
    g[2:] = tau * r / sigma - eta
    return float(l), g


SCHOOLS_Y = np.array([28.0, 8, -3, 7, -1, 1, 18, 12])
SCHOOLS_S = np.array([15.0, 10, 16, 11, 9, 11, 10, 18])


def _fd_grad(f, q, h=1e-6):
    g = np.empty_like(q)
    for i in range(q.size):
        e = np.zeros_like(q); e[i] = h
        g[i] = (f(q + e)[0] - f(q - e)[0]) / (2 * h)
    return g


# ------------------------------------------------------------------ CPU: the oracle with a user model
@pytest.mark.parametrize("D,T", [(2, 32), (10, 32), (77, 64), (300, 128)])
def test_funnel_as_user_model_equals_shipped_family_in_the_oracle(po, D, T):
    rng = np.random.default_rng(D)
    with po.user_model(_hdr("funnel_user")) as lib:
        assert lib.orc_user_family_name().decode() == "funnel_user"
        for _ in range(5):
            q = rng.normal(size=D) * 1.5
            lu, gu = po.logdensity_and_gradient(po.FAMILY_USER, q, None, T)
            lf, gf = po.logdensity_and_gradient(po.FAMILY_FUNNEL, q, None, T)
            assert lu == lf and np.array_equal(gu, gf)
        q = rng.normal(size=D)
        for t in range(3):
            a = po.sample_tree(po.FAMILY_USER, q, 0.2, 7, 3, t, T=T)
            b = po.sample_tree(po.FAMILY_FUNNEL, q, 0.2, 7, 3, t, T=T)
            for f in INT_FIELDS:
                assert a["stats"][f] == b["stats"][f]
            assert np.array_equal(a["q"], b["q"]) and a["lq"] == b["lq"]
            q = a["q"]
    assert po.lib().orc_user_family_name().decode() == ""         # back on the stock oracle


@pytest.mark.parametrize("D,T", [(1, 32), (100, 32), (1000, 128)])
def test_std_normal_as_user_model_equals_shipped_family_in_the_oracle(po, D, T):
    rng = np.random.default_rng(D)
    st = po.default_warmup_stages(init_steps=25, middle_steps=20, doubling_stages=1, terminating_steps=20)
    with po.user_model(_hdr("std_normal_user")):
        q = rng.normal(size=D)
        assert po.logdensity_and_gradient(po.FAMILY_USER, q, None, T)[0] == po.logdensity_and_gradient(po.FAMILY_STD_NORMAL, q, None, T)[0]
        a = po.mcmc_with_warmup(po.FAMILY_USER, D, 8, 3, 1, stages=st, T=T, welford=True, keep_warmup=True)
        b = po.mcmc_with_warmup(po.FAMILY_STD_NORMAL, D, 8, 3, 1, stages=st, T=T, welford=True, keep_warmup=True)
    assert np.array_equal(a["posterior_matrix"], b["posterior_matrix"]) and a["eps"] == b["eps"]
    for f in INT_FIELDS:
        assert np.array_equal(a["warmup_stats"][f], b["warmup_stats"][f])


def test_funnel_as_user_model_whole_warmup_in_the_oracle(po):
    D, N = 10, 25
    st = po.default_warmup_stages(init_steps=30, middle_steps=20, doubling_stages=2, terminating_steps=20)
    with po.user_model(_hdr("funnel_user")):
        a = po.mcmc_with_warmup(po.FAMILY_USER, D, N, 11, 2, stages=st, welford=True, keep_warmup=True)
        b = po.mcmc_with_warmup(po.FAMILY_FUNNEL, D, N, 11, 2, stages=st, welford=True, keep_warmup=True)
    assert np.array_equal(a["posterior_matrix"], b["posterior_matrix"]) and a["eps"] == b["eps"]
    assert np.array_equal(a["minv"], b["minv"])
    for f in INT_FIELDS:
        assert np.array_equal(a["warmup_stats"][f], b["warmup_stats"][f])


@pytest.mark.parametrize("D,T", [(2, 32), (5, 32), (64, 32), (129, 64), (1000, 128)])
def test_rosenbrock_oracle_values(po, D, T):
    rng = np.random.default_rng(40 + D)
    a, b = 1.0, 5.0
    with po.user_model(_hdr("rosenbrock")):
        for _ in range(4):
            q = rng.normal(size=D)
            l, g = po.logdensity_and_gradient(po.FAMILY_USER, q, np.array([a, b]), T)
            ln, gn = rosenbrock_np(q, a, b)
            assert l == pytest.approx(ln, rel=1e-12)
            np.testing.assert_allclose(g, gn, rtol=1e-11, atol=1e-11)
            if D <= 64:
                np.testing.assert_allclose(g, _fd_grad(lambda x: rosenbrock_np(x, a, b), q), rtol=2e-5, atol=2e-5)


def test_eight_schools_oracle_values(po):
    rng = np.random.default_rng(8)
    pr = np.concatenate([SCHOOLS_Y, SCHOOLS_S])
    with po.user_model(_hdr("eight_schools")):
        for _ in range(6):
            q = rng.normal(size=10)
            l, g = po.logdensity_and_gradient(po.FAMILY_USER, q, pr, 32)
            ln, gn = eight_schools_np(q, SCHOOLS_Y, SCHOOLS_S)
            assert l == pytest.approx(ln, rel=1e-12)
            np.testing.assert_allclose(g, gn, rtol=1e-11, atol=1e-12)
            np.testing.assert_allclose(g, _fd_grad(lambda x: eight_schools_np(x, SCHOOLS_Y, SCHOOLS_S), q), rtol=1e-5, atol=1e-5)
        # a short run: finite draws, plausible posterior for mu (sampling error only loosely bounded here)
        st = po.default_warmup_stages(init_steps=40, middle_steps=25, doubling_stages=2, terminating_steps=30)
        o = po.mcmc_with_warmup(po.FAMILY_USER, 10, 300, 5, 0, stages=st, params=pr, welford=True)
    assert np.all(np.isfinite(o["posterior_matrix"]))
    assert -5 < o["posterior_matrix"][:, 0].mean() < 15


def test_model_without_sums_oracle_values(po):
    """DHMC_USER_NSUMS 0 (ℓ straight from the position): the 2-d banana, against the direct formula and finite differences."""
    s_, b = 3.0, 0.1

    def f(q):
        u = q[1] + b * q[0] ** 2 - b * s_ * s_
        return -0.5 * (q[0] ** 2 / s_ ** 2 + u * u), np.array([-q[0] / s_ ** 2 - 2 * b * q[0] * u, -u])
    rng = np.random.default_rng(0)
    with po.user_model(_hdr("banana2d")):
        for _ in range(6):
            q = rng.normal(size=2) * 2
            l, g = po.logdensity_and_gradient(po.FAMILY_USER, q, np.array([s_, b]), 32)
            assert l == pytest.approx(f(q)[0], rel=1e-13, abs=1e-15) and np.allclose(g, f(q)[1], rtol=1e-12, atol=1e-14)
            np.testing.assert_allclose(g, _fd_grad(f, q), rtol=1e-5, atol=1e-6)
        o = po.mcmc_with_warmup(po.FAMILY_USER, 2, 200, 1, 0, params=np.array([s_, b]))
    assert np.all(np.isfinite(o["posterior_matrix"])) and o["tree_statistics"]["depth"].max() <= 10


# ------------------------------------------------------------------ CPU: the user-model build of the library
def test_user_library_builds_and_reports_its_model(pkg):
    """nvcc cross-compiles the model for sm_90a (no GPU needed); the result carries the whole C ABI plus the model."""
    so = pkg.compile_user_model(_hdr("rosenbrock"), deep=True)        # the build __graft_entry__.build() prepares
    lib = pkg._lib.lib(so)
    for name in pkg._lib.EXPORTS:
        assert hasattr(lib, name), name
    buf = C.create_string_buffer(64)
    assert lib.dhmc_user_family_name(buf, C.c_size_t(64)) == pkg._lib.DHMC_OK and buf.value == b"rosenbrock"
    small = C.create_string_buffer(5)
    assert lib.dhmc_user_family_name(small, C.c_size_t(5)) == pkg._lib.DHMC_OK and small.value == b"rose"
    assert pkg.compile_user_model(_hdr("rosenbrock"), deep=True) == so          # cached by content hash
    ℓ = pkg.UserLogDensity(_hdr("rosenbrock"), 12, params=[1.0, 5.0], cpu=lambda q: rosenbrock_np(q, 1.0, 5.0), deep=True)
    assert ℓ.model_name() == "rosenbrock" and ℓ.dimension() == 12 and ℓ.capabilities() == 1
    assert ℓ.logdensity_and_gradient(np.zeros(12))[0] == -11.0
    stock = pkg._lib.lib()
    assert stock.dhmc_user_family_name(buf, C.c_size_t(64)) == pkg._lib.DHMC_EARG
    # which kernel families each library carries (weak references to the per-family translation units, resolved at link
    # time): the stock library the four shipped ones, the user-model library family 4 only
    def available(so):
        out = []
        for fam in range(6):
            v = C.c_int32(-1)
            assert so.dhmc_family_available(C.c_int32(fam), C.byref(v)) == pkg._lib.DHMC_OK
            out.append(v.value)
        return out
    assert available(stock) == [1, 1, 1, 1, 0, 0]
    assert available(lib) == [0, 0, 0, 0, 1, 0]
    cfg = pkg._lib.Config(device=0, family=pkg._lib.FAMILY_STD_NORMAL, dim=4, n_chains=2, chain_offset=0, seed=1, max_depth=10,
                          threads_per_chain=0, min_delta=-1000.0, ctas_per_sm=0, reserved=0)
    h = C.c_void_p()
    assert lib.dhmc_create(C.byref(cfg), C.byref(h)) == pkg._lib.DHMC_EARG
    assert b"family not built into this library" in lib.dhmc_last_error(None)


def test_stock_library_refuses_the_user_family(pkg):
    """dhmc_create(family = USER) on a library without a model: ArgumentError before any CUDA call."""
    cfg = pkg._lib.Config(device=0, family=pkg._lib.FAMILY_USER, dim=4, n_chains=2, chain_offset=0, seed=1, max_depth=10,
                          threads_per_chain=0, min_delta=-1000.0, ctas_per_sm=0, reserved=0)
    h = C.c_void_p()
    lib = pkg._lib.lib()
    assert lib.dhmc_create(C.byref(cfg), C.byref(h)) == pkg._lib.DHMC_EARG
    assert b"without a user model" in lib.dhmc_last_error(None)
    with pytest.raises(pkg.ArgumentError):
        pkg.compile_user_model(os.path.join(MODELS, "no_such_model.h"))


def test_user_library_enforces_min_dim(pkg):
    so = pkg.compile_user_model(_hdr("rosenbrock"), deep=True)
    cfg = pkg._lib.Config(device=0, family=pkg._lib.FAMILY_USER, dim=1, n_chains=2, chain_offset=0, seed=1, max_depth=10,
                          threads_per_chain=0, min_delta=-1000.0, ctas_per_sm=0, reserved=0)
    h = C.c_void_p()
    lib = pkg._lib.lib(so)
    assert lib.dhmc_create(C.byref(cfg), C.byref(h)) == pkg._lib.DHMC_EARG
    assert b"DHMC_USER_MIN_DIM" in lib.dhmc_last_error(None)


# ------------------------------------------------------------------ GPU: the CUDA path of a user model
@pytest.mark.gpu
def test_funnel_as_user_model_equals_shipped_family_on_device(pkg):
    """Same seed, same stages: the user-model build of Neal's funnel and the shipped FUNNEL kernels give identical chains."""
    D, K, N, seed = 10, 96, 20, 31
    stages = pkg.default_warmup_stages(init_steps=30, middle_steps=20, doubling_stages=2, terminating_steps=20)
    ra = pkg.mcmc_keep_warmup(seed, pkg.UserLogDensity(_hdr("funnel_user"), D), N, chains=K, warmup_stages=stages)
    rb = pkg.mcmc_keep_warmup(seed, pkg.Funnel(D), N, chains=K, warmup_stages=stages)
    assert ra["engine"].layout() == rb["engine"].layout()
    for k in range(K):
        a, b = ra["inference"][k], rb["inference"][k]
        assert np.array_equal(a["posterior_matrix"], b["posterior_matrix"]) and a["ϵ"] == b["ϵ"]
        assert np.array_equal(a["κ"].minv, b["κ"].minv) and np.array_equal(a["logdensities"], b["logdensities"])
        for f in INT_FIELDS:
            assert np.array_equal(a["tree_statistics"][f], b["tree_statistics"][f])
    ra["engine"].close(); rb["engine"].close()


@pytest.mark.gpu
@pytest.mark.parametrize("D,K", [(100, 40), (1000, 16)])
def test_std_normal_as_user_model_equals_shipped_family_on_device(pkg, D, K):
    """The model bench.py times as `user_model`: identical chains to the shipped STD_NORMAL kernels (same layout)."""
    stages = pkg.default_warmup_stages(init_steps=25, middle_steps=20, doubling_stages=1, terminating_steps=20)
    ra = pkg.mcmc_keep_warmup(17, pkg.UserLogDensity(_hdr("std_normal_user"), D), 6, chains=K, warmup_stages=stages)
    rb = pkg.mcmc_keep_warmup(17, pkg.StandardNormal(D), 6, chains=K, warmup_stages=stages)
    assert ra["engine"].layout() == rb["engine"].layout()
    for k in range(K):
        a, b = ra["inference"][k], rb["inference"][k]
        assert np.array_equal(a["posterior_matrix"], b["posterior_matrix"]) and a["ϵ"] == b["ϵ"]
        for f in INT_FIELDS:
            assert np.array_equal(a["tree_statistics"][f], b["tree_statistics"][f])
    ra["engine"].close(); rb["engine"].close()


def _user_cases(pkg):
    rng = np.random.default_rng(2)
    cases = [("rosenbrock", D, np.array([1.0, 5.0])) for D in (2, 37, 300, 1000)]
    cases.append(("eight_schools", 10, np.concatenate([SCHOOLS_Y, SCHOOLS_S])))
    J = 500
    cases.append(("eight_schools", J + 2, np.concatenate([rng.normal(size=J) * 10, rng.uniform(5, 20, J)])))
    return cases


@pytest.mark.gpu
def test_user_models_leapfrog_and_trees_match_oracle(pkg, po):
    rng = np.random.default_rng(17)
    for name, D, pr in _user_cases(pkg):
        K = 12
        ℓ = pkg.UserLogDensity(_hdr(name), D, params=pr, deep=(name == "rosenbrock"))
        eng = pkg.Engine(ℓ, chains=K, seed=77)
        T, _ = eng.layout()
        q, p = rng.normal(size=(K, D)) * 0.5, rng.normal(size=(K, D))
        minv = rng.uniform(0.5, 2, (K, D))
        eps = np.exp(rng.uniform(np.log(0.005), np.log(0.1), K))
        eng.set_metric(minv); eng.set_position(q); eng.set_momentum(p); eng.set_stepsize(eps)
        with po.user_model(_hdr(name)):
            st0 = eng.get_state(("lq", "grad"))
            for k in range(K):
                l, g = po.logdensity_and_gradient(po.FAMILY_USER, q[k], pr, T)
                assert st0["lq"][k] == l and np.array_equal(st0["grad"][k], g), (name, D, k)
            eng.leapfrog(2, 1)
            st = eng.get_state()
            for k in range(K):
                qo, p_o, go, lqo = po.leapfrog(po.FAMILY_USER, q[k], p[k], eps[k], minv=minv[k], params=pr, T=T, n_steps=2)
                np.testing.assert_allclose(st["q"][k], qo, rtol=1e-10, atol=0)
                assert np.array_equal(st["q"][k], qo) and np.array_equal(st["p"][k], p_o)
                assert np.array_equal(st["grad"][k], go) and st["lq"][k] == lqo
            eng.set_position(q)
            for t in range(2):
                stats = eng.sample_tree()
                s2 = eng.get_state(("q", "lq", "grad"))
                for k in range(K):
                    o = po.sample_tree(po.FAMILY_USER, q[k], eps[k], 77, k, t, minv=minv[k], params=pr, T=T)
                    for f in INT_FIELDS:
                        assert o["stats"][f] == stats[k][f], (name, D, f, k, t)
                    assert o["stats"]["pi"] == stats[k]["pi"] and o["stats"]["acceptance_rate"] == stats[k]["acceptance_rate"]
                    assert np.array_equal(s2["q"][k], o["q"]) and np.array_equal(s2["grad"][k], o["g"]) and s2["lq"][k] == o["lq"]
                q = s2["q"]
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("M", ["Diagonal", "Symmetric"])
def test_user_model_full_warmup_matches_oracle(pkg, po, M):
    """mcmc_with_warmup of the hierarchical example (diagonal and Symmetric metric windows) and a deep-tree run."""
    pr = np.concatenate([SCHOOLS_Y, SCHOOLS_S])
    ℓ = pkg.UserLogDensity(_hdr("eight_schools"), 10, params=pr)
    K, N, seed = 16, 25, 404
    stages = pkg.default_warmup_stages(M=getattr(pkg, M), init_steps=30, middle_steps=25, doubling_stages=2, terminating_steps=20)
    r = pkg.mcmc_keep_warmup(seed, ℓ, N, chains=K, warmup_stages=stages)
    T, _ = r["engine"].layout()
    ostages = po.default_warmup_stages(init_steps=30, middle_steps=25, doubling_stages=2, terminating_steps=20,
                                       M=po.METRIC_SYMMETRIC if M == "Symmetric" else po.METRIC_DIAGONAL)
    with po.user_model(_hdr("eight_schools")):
        for k in range(0, K, 5):
            o = po.mcmc_with_warmup(po.FAMILY_USER, 10, N, seed, k, stages=ostages, params=pr, T=T, welford=True, keep_warmup=True)
            w = np.concatenate([s["results"]["tree_statistics"][k] for s in r["warmup"] if s["results"]])
            for f in INT_FIELDS:
                assert np.array_equal(w[f], o["warmup_stats"][f]), f
            res = r["inference"][k]
            assert res["ϵ"] == o["eps"] and np.array_equal(res["κ"].minv, o["minv"])
            assert np.array_equal(res["posterior_matrix"].T, o["posterior_matrix"])
    r["engine"].close()
    if M == "Diagonal":      # max_depth > 12: the deep kernel instantiations of the user family
        eng = pkg.Engine(pkg.UserLogDensity(_hdr("rosenbrock"), 3, params=[1.0, 5.0], deep=True), chains=6, seed=9, algorithm=pkg.NUTS(max_depth=15))
        T, _ = eng.layout()
        rng = np.random.default_rng(1)
        q = rng.normal(size=(6, 3)) * 0.3
        eps = np.full(6, 3e-4)
        eng.set_position(q); eng.set_stepsize(eps)
        stats = eng.sample_tree()
        newq = eng.get_state(("q",))["q"]
        with po.user_model(_hdr("rosenbrock")):
            for k in range(6):
                o = po.sample_tree(po.FAMILY_USER, q[k], eps[k], 9, k, 0, params=np.array([1.0, 5.0]), T=T, max_depth=15)
                for f in INT_FIELDS:
                    assert o["stats"][f] == stats[k][f]
                assert np.array_equal(newq[k], o["q"])
        eng.close()


@pytest.mark.gpu
def test_dense_mvnormal_user_model_on_device(pkg, po):
    """The reference's sample-correctness target family (test/sample-correctness_tests.jl: `multivariate_normal(μ, L)` with
    `default_warmup_stages(; M = Symmetric)`) on the device through include/models/mvnormal_dense.h — the third isolated
    ill-conditioned case (:43-49), 64 chains: sampled chains equal the oracle built from the same header, and the pooled
    draws have the target's mean / covariance and R̂ within the reference's thresholds (CPU counterpart with all cases:
    tests/test_oracle_sample_correctness.py)."""
    import test_oracle_sample_correctness as sc
    mu, L, D = np.array(sc.ILL3_MU), np.diag(sc.ILL3_D) @ sc._mat(sc.ILL3_C), 10
    Sigma = L @ L.T
    P = np.linalg.inv(Sigma); P = 0.5 * (P + P.T)
    params = np.concatenate([mu, P.ravel()])
    K, N, seed = 64, 200, 77
    ℓ = pkg.UserLogDensity(_hdr("mvnormal_dense"), D, params=params)
    r = pkg.mcmc_keep_warmup(seed, ℓ, N, chains=K, warmup_stages=pkg.default_warmup_stages(M=pkg.Symmetric))
    T, _ = r["engine"].layout()
    res = r["inference"]
    ostages = po.default_warmup_stages(M=po.METRIC_SYMMETRIC)
    with po.user_model(_hdr("mvnormal_dense")):
        for k in (0, 31, 63):
            o = po.mcmc_with_warmup(po.FAMILY_USER, D, N, seed, k, stages=ostages, params=params, T=T, welford=True)
            assert res[k]["ϵ"] == o["eps"] and np.array_equal(res[k]["κ"].minv, o["minv"])
            assert np.array_equal(res[k]["posterior_matrix"].T, o["posterior_matrix"])
            for f in INT_FIELDS:
                assert np.array_equal(res[k]["tree_statistics"][f], o["tree_statistics"][f])
    draws = np.stack([res[k]["posterior_matrix"].T for k in range(K)])      # [chain, draw, parameter]
    er = pkg.diagnostics.ess_rhat(draws)
    Z, sd = draws.reshape(-1, D), np.sqrt(np.diag(Sigma))
    assert er["rhat"].max() <= 1.02 and (er["ess"] / (K * N)).min() >= 0.35
    assert np.max(np.abs(Z.mean(0) - mu) / sd) < 0.1
    assert np.max(np.abs(np.cov(Z.T) - Sigma) / np.outer(sd, sd)) < 0.15
    r["engine"].close()


@pytest.mark.gpu
def test_check_gradient_on_device(pkg):
    """diagnostics.check_gradient: ∇ℓ of a user model against central differences of its ℓ, both evaluated by the device."""
    rng = np.random.default_rng(4)
    r = pkg.diagnostics.check_gradient(pkg.UserLogDensity(_hdr("rosenbrock"), 9, params=[1.0, 5.0], deep=True), rng.normal(size=9) * 0.7)
    assert r["max_abs_err"] < 1e-5
    q = rng.normal(size=10)
    r = pkg.diagnostics.check_gradient(pkg.UserLogDensity(_hdr("eight_schools"), 10, params=np.concatenate([SCHOOLS_Y, SCHOOLS_S])), q)
    assert r["max_abs_err"] < 1e-5
    ln, gn = eight_schools_np(q, SCHOOLS_Y, SCHOOLS_S)
    assert r["lq"] == pytest.approx(ln, rel=1e-12) and np.allclose(r["grad"], gn, rtol=1e-10, atol=1e-12)
