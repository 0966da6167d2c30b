"""-m gpu: the CUDA path, called through the C ABI, against the oracle.

Bar (BASELINE.json north_star): integer tree decisions bit-exact; θ/p after a
leapfrog step within 1e-10 relative (we observe bit-equality because both sides
use the same canonical reduction order and deterministic math)."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

INT_FIELDS = ("depth", "left", "right", "steps", "directions")
RTOL = 1e-10


def _engine(pkg, ℓ, K, seed=5, **kw):
    return pkg.Engine(ℓ, chains=K, seed=seed, **kw)


def _models(pkg, rng, D):
    return [(pkg.StandardNormal(D), 0, None),
            (pkg.DiagNormal(rng.normal(size=D), rng.uniform(0.2, 5, D)), 1, True),
            (pkg.Funnel(D), 2, None)]


@pytest.mark.parametrize("D", [2, 3, 10, 100, 200, 500, 1000, 2000, 3000, 5000, 8192])
def test_leapfrog_matches_oracle(pkg, po, D):
    rng = np.random.default_rng(D)
    K = 8
    for ℓ, fam, hasp in _models(pkg, rng, D):
        eng = _engine(pkg, ℓ, K)
        T, _ = eng.layout()
        q, p = rng.normal(size=(K, D)), rng.normal(size=(K, D))
        minv = rng.uniform(0.5, 2, (K, D))
        eps = rng.uniform(0.01, 0.2, K)
        eng.set_metric(minv); eng.set_position(q); eng.set_momentum(p); eng.set_stepsize(eps)
        params = ℓ.params() if hasp else None
        H = eng.phase_logdensity()
        for sign, n in ((1, 1), (-1, 3)):
            eng.leapfrog(n, sign)
            st = eng.get_state()
            for k in range(K):
                qo, p_o, go, lqo = po.leapfrog(fam, q[k], p[k], sign * eps[k], minv=minv[k], params=params, T=T, n_steps=n)
                np.testing.assert_allclose(st["q"][k], qo, rtol=RTOL, atol=0)
                np.testing.assert_allclose(st["p"][k], p_o, rtol=RTOL, atol=0)
                assert np.array_equal(st["q"][k], qo) and np.array_equal(st["p"][k], p_o)
                assert np.array_equal(st["grad"][k], go) and st["lq"][k] == lqo
            q, p = st["q"], st["p"]
        lq0 = [po.logdensity_and_gradient(fam, qq, params, T)[0] for qq in q]
        H1 = eng.phase_logdensity()
        for k in range(K):
            assert H1[k] == po.phase_logdensity(minv[k], lq0[k], p[k], T)
        eng.close()


@pytest.mark.parametrize("D,K", [(2, 64), (10, 96), (100, 48), (256, 16), (1000, 12), (2000, 6), (3000, 4), (6000, 3)])
def test_sample_tree_matches_oracle(pkg, po, D, K):
    rng = np.random.default_rng(1000 + D)
    for ℓ, fam, hasp in _models(pkg, rng, D):
        eng = _engine(pkg, ℓ, K, seed=77)
        T, _ = eng.layout()
        q = rng.normal(size=(K, D))
        minv = rng.uniform(0.3, 3, (K, D))
        eps = np.exp(rng.uniform(np.log(0.01), np.log(1.2), K))
        eng.set_metric(minv); eng.set_position(q); eng.set_stepsize(eps)
        params = ℓ.params() if hasp else None
        for t in range(3):
            stats = eng.sample_tree()
            st = eng.get_state(("q", "lq", "grad"))
            for k in range(K):
                o = po.sample_tree(fam, q[k], eps[k], 77, k, t, minv=minv[k], params=params, T=T)
                for f in INT_FIELDS:
                    assert o["stats"][f] == stats[k][f], (f, k, t, o["stats"], stats[k])
                assert o["stats"]["pi"] == stats[k]["pi"]
                assert o["stats"]["acceptance_rate"] == stats[k]["acceptance_rate"]
                np.testing.assert_allclose(st["q"][k], o["q"], rtol=RTOL, atol=0)
                assert np.array_equal(st["q"][k], o["q"]) and np.array_equal(st["grad"][k], o["g"])
                assert st["lq"][k] == o["lq"]
            q = st["q"]
        eng.close()


def test_sample_tree_overrides_and_exits(pkg, po):
    """p= / directions= keywords (NUTS.jl:232-233); every tree exit is hit."""
    rng = np.random.default_rng(3)
    D, K = 20, 128
    ℓ = pkg.StandardNormal(D)
    seen = dict(div=0, turn=0, maxd=0)
    for max_depth, min_delta in ((3, -1000.0), (10, -0.02), (10, -1000.0)):
        eng = _engine(pkg, ℓ, K, algorithm=pkg.NUTS(max_depth=max_depth, min_Δ=min_delta))
        T, _ = eng.layout()
        q, p = rng.normal(size=(K, D)), rng.normal(size=(K, D))
        dirs = rng.integers(0, 2 ** 32, K, dtype=np.uint64).astype(np.uint32)
        eps = np.exp(rng.uniform(np.log(0.02), np.log(1.0), K))
        eng.set_position(q); eng.set_stepsize(eps)
        stats = eng.sample_tree(p=p, directions=dirs)
        newq = eng.get_state(("q",))["q"]
        for k in range(K):
            o = po.sample_tree(0, q[k], eps[k], 5, k, 0, T=T, p=p[k], directions=int(dirs[k]),
                               max_depth=max_depth, min_delta=min_delta)
            for f in INT_FIELDS:
                assert o["stats"][f] == stats[k][f]
            assert np.array_equal(newq[k], o["q"])
            s = stats[k]
            seen["div"] += int(s["left"] == s["right"])
            seen["maxd"] += int((s["left"], s["right"]) == (1, 0))
            seen["turn"] += int(s["left"] < s["right"] or (s["left"] > s["right"] and (s["left"], s["right"]) != (1, 0)))
        eng.close()
    assert min(seen.values()) > 3, seen


def test_mcmc_draws_and_layout(pkg, po):
    """mcmc (mcmc.jl:366-381): [D, N, B] output, logdensities, RNG counter continuity."""
    D, K, N = 50, 40, 6
    rng = np.random.default_rng(8)
    ℓ = pkg.DiagNormal(rng.normal(size=D), rng.uniform(0.5, 2, D))
    eng = _engine(pkg, ℓ, K, seed=9)
    T, _ = eng.layout()
    eng.random_position()
    q0 = eng.get_state(("q",))["q"]
    eng.set_stepsize(0.3)
    a = eng.mcmc(4)
    b = eng.mcmc(N - 4)                       # continues the same chains (counter 4, 5)
    assert eng.transition_count == N
    post = np.concatenate([a["posterior_matrix"], b["posterior_matrix"]], axis=1)
    stats = np.concatenate([a["tree_statistics"], b["tree_statistics"]], axis=1)
    logd = np.concatenate([a["logdensities"], b["logdensities"]], axis=1)
    assert eng.last_total_steps() == int(b["tree_statistics"]["steps"].sum())
    for k in range(0, K, 7):
        assert np.array_equal(q0[k], po.random_position(9, k, D))
        q = q0[k]
        for n in range(N):
            o = po.sample_tree(1, q, 0.3, 9, k, n, params=ℓ.params(), T=T)
            for f in INT_FIELDS:
                assert o["stats"][f] == stats[k, n][f]
            assert np.array_equal(post[k, n], o["q"]) and logd[k, n] == o["lq"]
            q = o["q"]
    eng.close()


@pytest.mark.parametrize("fam,D", [(0, 100), (1, 40), (2, 10)])
def test_full_warmup_matches_oracle(pkg, po, fam, D):
    """mcmc_with_warmup through the host mirror vs the oracle with the streaming
    (Welford) window variance: identical chains."""
    rng = np.random.default_rng(21)
    ℓ = [pkg.StandardNormal(D), pkg.DiagNormal(rng.normal(size=D), np.logspace(-1, 1, D)), pkg.Funnel(D)][fam]
    K, N, seed = 24, 30, 4242
    stages = pkg.default_warmup_stages(init_steps=30, middle_steps=20, doubling_stages=2, terminating_steps=20)
    r = pkg.mcmc_keep_warmup(seed, ℓ, N, chains=K, warmup_stages=stages)
    T, _ = r["engine"].layout()
    res = r["inference"]
    ostages = po.default_warmup_stages(init_steps=30, middle_steps=20, doubling_stages=2, terminating_steps=20)
    params = ℓ.params() if fam == 1 else None
    for k in range(0, K, 5):
        o = po.mcmc_with_warmup(fam, D, N, seed, k, stages=ostages, params=params, T=T, welford=True,
                                keep_warmup=True)
        w = np.concatenate([s["results"]["tree_statistics"][k] for s in r["warmup"] if s["results"]])
        for f in INT_FIELDS:
            assert np.array_equal(w[f], o["warmup_stats"][f]), f
        weps = np.concatenate([s["results"]["ϵs"][k] for s in r["warmup"] if s["results"]])
        assert np.array_equal(weps, o["warmup_eps"])
        assert res[k]["ϵ"] == o["eps"] and np.array_equal(res[k]["κ"].minv, o["minv"])
        assert np.array_equal(res[k]["posterior_matrix"].T, o["posterior_matrix"])
        for f in INT_FIELDS:
            assert np.array_equal(res[k]["tree_statistics"][f], o["tree_statistics"][f])
    r["engine"].close()


def test_c1_exact_config_matches_oracle(pkg, po):
    """BASELINE.json configs[0] verbatim on the device: 100-dim standard MvNormal, 4 chains, the default warm-up (900
    transitions, diagonal metric windows) and 1000 draws — every chain equals the oracle (integers, ϵ, metric, draws), and
    the pooled posterior has the N(0, I) moments within sampling error (test_mcmc.jl:18-26 style)."""
    D, K, N, seed = 100, 4, 1000, 1
    r = pkg.mcmc_keep_warmup(seed, pkg.StandardNormal(D), N, chains=K)
    T, _ = r["engine"].layout()
    for k in range(K):
        o = po.mcmc_with_warmup(po.FAMILY_STD_NORMAL, D, N, seed, k, T=T, welford=True, keep_warmup=True)
        w = np.concatenate([s["results"]["tree_statistics"][k] for s in r["warmup"] if s["results"]])
        assert w.size == 900
        for f in INT_FIELDS:
            assert np.array_equal(w[f], o["warmup_stats"][f]), f
        res = r["inference"][k]
        assert res["ϵ"] == o["eps"] and np.array_equal(res["κ"].minv, o["minv"])
        assert np.array_equal(res["posterior_matrix"].T, o["posterior_matrix"])
        for f in INT_FIELDS:
            assert np.array_equal(res["tree_statistics"][f], o["tree_statistics"][f])
    pooled = pkg.pool_posterior_matrices(r["inference"])            # [D, N·K]
    assert np.abs(pooled.mean(axis=1)).max() < 0.12 and np.abs(pooled.var(axis=1) - 1).max() < 0.25
    r["engine"].close()


def _c5_model(pkg, D=1000):
    """BASELINE.json configs[4]: MvNormal with σᵢ² = 10^{4(i−1)/(D−1)} (κ = 10⁴), SURVEY.md §8d."""
    return pkg.DiagNormal(np.zeros(D), 10.0 ** (4.0 * np.arange(D) / (D - 1)))


def test_c5_shape_full_default_warmup_matches_oracle(pkg, po):
    """C5 at its exact shape: D = 1000, κ = 10⁴, the FULL default warm-up (search + 75 + 25…400 with diagonal metric
    windows + 50 = 900 transitions, mcmc.jl:415-425) and draws; the chains are the LAST ones of a 65 536-chain shard
    (global ids 65 512 … 65 535 through chain_offset, i.e. the same RNG keys): warm-up statistics, step sizes, adapted
    metric and draws must equal the oracle's."""
    ℓ = _c5_model(pkg)
    K, N, seed, off = 24, 10, 2026, 65536 - 24
    r = pkg.mcmc_keep_warmup(seed, ℓ, N, chains=K, chain_offset=off)
    T, _ = r["engine"].layout()
    params = ℓ.params()
    for k in (0, 11, K - 1):
        o = po.mcmc_with_warmup(po.FAMILY_DIAG_NORMAL, 1000, N, seed, off + k, params=params, T=T, welford=True, keep_warmup=True)
        w = np.concatenate([s["results"]["tree_statistics"][k] for s in r["warmup"] if s["results"]])
        assert w.size == 900
        for f in INT_FIELDS:
            assert np.array_equal(w[f], o["warmup_stats"][f]), f
        weps = np.concatenate([s["results"]["ϵs"][k] for s in r["warmup"] if s["results"]])
        assert np.array_equal(weps, o["warmup_eps"])
        res = r["inference"][k]
        assert res["ϵ"] == o["eps"] and np.array_equal(res["κ"].minv, o["minv"])
        np.testing.assert_allclose(res["posterior_matrix"].T, o["posterior_matrix"], rtol=RTOL, atol=0)
        assert np.array_equal(res["posterior_matrix"].T, o["posterior_matrix"])
        for f in INT_FIELDS:
            assert np.array_equal(res["tree_statistics"][f], o["tree_statistics"][f])
    r["engine"].close()


def test_c5_last_chain_of_a_65536_chain_handle(pkg, po):
    """The same model on a full-size handle (65 536 chains, 2.1 GB of state): the last chain (index arithmetic at scale)
    after the step-size search, a dual-averaging stage and a diagonal metric window equals the oracle."""
    ℓ = _c5_model(pkg)
    K, N, seed = 65536, 4, 77
    stages = (pkg.InitialStepsizeSearch(), pkg.TuningNUTS(20, pkg.DualAveraging()),
              pkg.TuningNUTS(20, pkg.DualAveraging(), pkg.Diagonal), pkg.TuningNUTS(20, pkg.DualAveraging()))
    r = pkg.mcmc_keep_warmup(seed, ℓ, N, chains=K, warmup_stages=stages, keep_warmup=False)
    T, _ = r["engine"].layout()
    ostages = po.default_warmup_stages(init_steps=20, middle_steps=20, doubling_stages=1, terminating_steps=20)
    for k in (0, 40000, K - 1):
        o = po.mcmc_with_warmup(po.FAMILY_DIAG_NORMAL, 1000, N, seed, k, stages=ostages, params=ℓ.params(), T=T, welford=True)
        res = r["inference"][k]
        assert res["ϵ"] == o["eps"] and np.array_equal(res["κ"].minv, o["minv"])
        assert np.array_equal(res["posterior_matrix"].T, o["posterior_matrix"])
        for f in INT_FIELDS:
            assert np.array_equal(res["tree_statistics"][f], o["tree_statistics"][f])
    r["engine"].close()


def test_c3_shape_funnel_262144_chains(pkg, po):
    """C3 at its exact shape: Neal's funnel D = 10 on a 262 144-chain handle (ragged tree depths, one warp per chain).
    Sampled chain ids against the oracle, and the device-side depth histogram / termination counts
    (dhmc_tree_summary_dev) against the host-side counts of the very same statistics."""
    import ctypes as C
    ℓ = pkg.Funnel(10)
    K, N, seed = 262144, 6, 9
    eng = pkg.Engine(ℓ, chains=K, seed=seed)
    T, _ = eng.layout()
    eng.random_position(); eng.find_initial_stepsize()
    eng.warmup_stage(pkg.TuningNUTS(30, pkg.DualAveraging()))
    eng.warmup_stage(pkg.TuningNUTS(25, pkg.DualAveraging(), pkg.Diagonal))
    eng.warmup_stage(pkg.TuningNUTS(20, pkg.DualAveraging()))
    out = eng.mcmc(N)
    st = eng.get_state(("minv", "eps"))
    ostages = [(po.STAGE_SEARCH, 0, po.METRIC_NOTHING, 0), (po.STAGE_TUNING, 30, po.METRIC_NOTHING, 1),
               (po.STAGE_TUNING, 25, po.METRIC_DIAGONAL, 1), (po.STAGE_TUNING, 20, po.METRIC_NOTHING, 1)]
    for k in (0, 1, 31, 4097, 131071, 200003, K - 1):
        o = po.mcmc_with_warmup(po.FAMILY_FUNNEL, 10, N, seed, k, stages=ostages, T=T, welford=True)
        assert st["eps"][k] == o["eps"] and np.array_equal(st["minv"][k], o["minv"])
        assert np.array_equal(out["posterior_matrix"][k], o["posterior_matrix"])
        for f in INT_FIELDS:
            assert np.array_equal(out["tree_statistics"][k][f], o["tree_statistics"][f])
    # device-side summary of a device-resident statistics buffer == host-side counts of the same records
    import torch
    dstats = torch.empty((K, N, 56), dtype=torch.uint8, device="cuda")
    eng.mcmc_dev(N, 0, dstats.data_ptr(), 0)
    host = dstats.cpu().numpy().view(pkg._lib.tree_stats_dtype).reshape(K, N)
    summ = eng.tree_summary_dev(dstats.data_ptr(), N, ebfmi=False)
    depth_counts = np.bincount(host["depth"].ravel(), minlength=len(summ["depth_counts"]))
    assert depth_counts.tolist()[:len(summ["depth_counts"])] == summ["depth_counts"] and depth_counts.sum() == K * N
    div = int(np.sum(host["left"] == host["right"]))
    mx = int(np.sum((host["left"] == 1) & (host["right"] == 0)))
    assert summ["termination_counts"] == dict(max_depth=mx, divergence=div, turning=K * N - div - mx)
    assert summ["steps"] == int(host["steps"].sum())
    assert len(summ["depth_counts"]) >= 5                      # ragged: several depths occur
    eng.close()


def test_initial_stepsize_search(pkg, po):
    D, K = 30, 64
    rng = np.random.default_rng(12)
    ℓ = pkg.DiagNormal(np.zeros(D), np.logspace(-2, 2, D))
    eng = _engine(pkg, ℓ, K, seed=31)
    T, _ = eng.layout()
    q = rng.normal(size=(K, D)) * np.sqrt(ℓ.sigma2)
    eng.set_position(q)
    eng.find_initial_stepsize()
    eps = eng.get_state(("eps",))["eps"]
    for k in range(K):
        p = po.normals(31, k, 1, 0, D)          # DHMC_STREAM_PSEARCH
        assert eps[k] == po.find_initial_stepsize(1, q[k], p, params=ℓ.params(), T=T)
    with pytest.raises(pkg.ArgumentError):     # mcmc.jl:137
        eng.find_initial_stepsize()
    eng.close()


def test_error_conventions(pkg):
    D, K = 5, 8
    eng = _engine(pkg, pkg.StandardNormal(D), K)
    q = np.zeros((K, D))
    q[3, 2] = np.nan
    with pytest.raises(pkg.DynamicHMCError) as e:     # hamiltonian.jl:203 via mcmc.jl:131
        eng.set_position(q)
    st = e.value.debug_information["chain_status"]
    assert st[3] != 0 and np.count_nonzero(st) == 1
    with pytest.raises(pkg.ArgumentError):
        eng.mcmc(3)                                    # no step size yet
    with pytest.raises(pkg.ArgumentError):
        eng.set_stepsize(-1.0)                         # stepsize.jl:135
    eng.close()
    with pytest.raises(pkg.ArgumentError):
        pkg.Engine(pkg.StandardNormal(9000), chains=2)  # dim too large for this build (dim <= 8192)
    # funnel with a huge step: divergent first leaf, chain stays put, others unaffected
    eng = _engine(pkg, pkg.Funnel(10), K)
    q = np.zeros((K, 10)); q[:, 0] = -8.0; q[:, 1:] = 5.0
    eng.set_position(q); eng.set_stepsize(50.0)
    stats = eng.sample_tree()
    assert np.all(stats["left"] == stats["right"]) and np.all(stats["depth"] == 0) and np.all(stats["steps"] == 1)
    assert np.array_equal(eng.get_state(("q",))["q"], q)
    eng.close()


def test_sharding_invariance(pkg):
    """§8e: the Philox key is the GLOBAL chain id, so a shard (chain_offset) reproduces
    the corresponding chains of the full run bit for bit — independent of #GPUs."""
    D, K, N = 64, 256, 5
    ℓ = pkg.StandardNormal(D)
    full = _engine(pkg, ℓ, K, seed=3)
    full.random_position(); full.set_stepsize(0.4)
    a = full.mcmc(N)
    full.close()
    for off, n in ((0, 32), (100, 50), (250, 6)):
        sh = pkg.Engine(ℓ, chains=n, seed=3, chain_offset=off)
        sh.random_position(); sh.set_stepsize(0.4)
        b = sh.mcmc(N)
        sh.close()
        assert np.array_equal(a["posterior_matrix"][off:off + n], b["posterior_matrix"])
        assert np.array_equal(a["tree_statistics"][off:off + n], b["tree_statistics"])


def test_layout_independence_within_tolerance(pkg):
    """Different threads_per_chain = different (documented) summation order: results
    agree to rounding for a single leapfrog (1e-10 bar), not necessarily bit for bit."""
    D, K = 200, 16
    rng = np.random.default_rng(2)
    q, p = rng.normal(size=(K, D)), rng.normal(size=(K, D))
    out = []
    for T in (32, 64, 128):
        eng = pkg.Engine(pkg.StandardNormal(D), chains=K, threads_per_chain=T)
        assert eng.layout()[0] == T
        eng.set_position(q); eng.set_momentum(p); eng.set_stepsize(0.1)
        eng.leapfrog(5, 1)
        out.append(eng.get_state(("q", "p", "lq")))
        eng.close()
    for o in out[1:]:
        np.testing.assert_allclose(o["q"], out[0]["q"], rtol=1e-12)
        np.testing.assert_allclose(o["lq"], out[0]["lq"], rtol=1e-12)


def test_chunked_host_output_pipeline(pkg):
    """Large host outputs are produced chunk by chunk (k_nuts per chain range, D2H on a
    second stream).  The result must equal un-chunked shards of the same global chains."""
    D, K, N = 64, 8192, 8          # 33.5 MB of draws -> chunked path
    ℓ = pkg.StandardNormal(D)
    full = _engine(pkg, ℓ, K, seed=13)
    full.random_position(); full.set_stepsize(0.45)
    a = full.mcmc(N)
    assert full.last_total_steps() == int(a["tree_statistics"]["steps"].sum())
    st = full.get_state(("q",))
    assert np.array_equal(st["q"], a["posterior_matrix"][:, -1, :])
    full.close()
    for off, n in ((0, 100), (1000, 64), (8100, 92)):
        sh = pkg.Engine(ℓ, chains=n, seed=13, chain_offset=off)
        sh.random_position(); sh.set_stepsize(0.45)
        b = sh.mcmc(N)
        sh.close()
        assert np.array_equal(a["posterior_matrix"][off:off + n], b["posterior_matrix"])
        assert np.array_equal(a["tree_statistics"][off:off + n], b["tree_statistics"])
        assert np.array_equal(a["logdensities"][off:off + n], b["logdensities"])


# --------------------------------------------------------------- Symmetric (dense) metric
def _spd(rng, D):
    A = rng.normal(size=(D, D))
    return A @ A.T / D + np.diag(rng.uniform(0.5, 2.0, D))


@pytest.mark.parametrize("D", [3, 10, 40, 100, 256, 400, 700, 1100])
def test_dense_metric_leapfrog_and_tree_match_oracle(pkg, po, D):
    """GaussianKineticEnergy(Symmetric M⁻¹) (hamiltonian.jl:73): W = cholesky(inv(M⁻¹)).L on
    device, p♯ = M⁻¹p mat-vec, rand_p = W·randn — against the oracle, bit for bit."""
    rng = np.random.default_rng(500 + D)
    K = 6
    ℓ = pkg.DiagNormal(rng.normal(size=D), rng.uniform(0.3, 3, D))
    eng = _engine(pkg, ℓ, K, seed=21)
    T, _ = eng.layout()
    Minv = np.stack([_spd(rng, D) for _ in range(K)])
    q, p = rng.normal(size=(K, D)), rng.normal(size=(K, D))
    eps = rng.uniform(0.02, 0.2, K)
    eng.set_metric_dense(Minv)
    assert eng.metric_is_dense() and np.array_equal(eng.get_metric_dense(), Minv)
    eng.set_position(q); eng.set_momentum(p); eng.set_stepsize(eps)
    H = eng.phase_logdensity()
    lq0 = [po.logdensity_and_gradient(1, q[k], ℓ.params(), T)[0] for k in range(K)]
    for k in range(K):
        assert H[k] == po.phase_logdensity(Minv[k], lq0[k], p[k], T)
    eng.leapfrog(3, 1)
    st = eng.get_state(("q", "p", "grad", "lq"))
    for k in range(K):
        qo, p_o, go, lqo = po.leapfrog(1, q[k], p[k], eps[k], minv=Minv[k], params=ℓ.params(), T=T, n_steps=3)
        np.testing.assert_allclose(st["q"][k], qo, rtol=RTOL, atol=0)
        assert np.array_equal(st["q"][k], qo) and np.array_equal(st["p"][k], p_o) and st["lq"][k] == lqo
    eng.set_position(q)
    for t in range(2):
        stats = eng.sample_tree()
        new = eng.get_state(("q",))["q"]
        for k in range(K):
            o = po.sample_tree(1, q[k], eps[k], 21, k, t, minv=Minv[k], params=ℓ.params(), T=T)
            for f in INT_FIELDS:
                assert o["stats"][f] == stats[k][f], (f, k, t)
            assert o["stats"]["acceptance_rate"] == stats[k]["acceptance_rate"]
            assert np.array_equal(new[k], o["q"])
        q = new
    # switching back to a diagonal metric works
    eng.set_metric(np.ones(D))
    assert not eng.metric_is_dense()
    eng.sample_tree()
    eng.close()


def test_large_dims_full_warmup_matches_oracle(pkg, po):
    """dim above 2048 (16 / 32 elements per thread) and a Symmetric metric above dim 512 through the whole default warm-up
    (shortened) — bit-equal warm-up statistics, adapted metric, step size and draws."""
    rng = np.random.default_rng(4242)
    for D, M, code in ((2500, pkg.Diagonal, po.METRIC_DIAGONAL), (640, pkg.Symmetric, po.METRIC_SYMMETRIC)):
        ℓ = pkg.DiagNormal(rng.normal(size=D), np.logspace(-0.5, 0.5, D))
        K, N, seed = 4, 6, 31
        kw = dict(init_steps=25, middle_steps=20, doubling_stages=1, terminating_steps=20)
        r = pkg.mcmc_keep_warmup(seed, ℓ, N, chains=K, warmup_stages=pkg.default_warmup_stages(M=M, **kw))
        T, _ = r["engine"].layout()
        res = r["inference"]
        for k in (0, K - 1):
            o = po.mcmc_with_warmup(1, D, N, seed, k, stages=po.default_warmup_stages(M=code, **kw), params=ℓ.params(), T=T,
                                    welford=True, keep_warmup=True)
            w = np.concatenate([s["results"]["tree_statistics"][k] for s in r["warmup"] if s["results"]])
            for f in INT_FIELDS:
                assert np.array_equal(w[f], o["warmup_stats"][f]), (D, f)
            assert np.array_equal(res[k]["κ"].minv, o["minv"]) and res[k]["ϵ"] == o["eps"]
            assert np.array_equal(res[k]["posterior_matrix"].T, o["posterior_matrix"])
        r["engine"].close()


def test_dense_metric_not_positive_definite(pkg):
    D, K = 4, 3
    eng = _engine(pkg, pkg.StandardNormal(D), K)
    M = np.stack([np.eye(D)] * K)
    M[1] = -np.eye(D)
    with pytest.raises(pkg.DynamicHMCError) as e:          # PosDefException in the reference
        eng.set_metric_dense(M)
    st = e.value.debug_information["chain_status"]
    assert st[1] & 16 and st[0] == 0 and st[2] == 0
    eng.close()


@pytest.mark.parametrize("D", [8, 50])
def test_full_warmup_symmetric_matches_oracle(pkg, po, D):
    """default_warmup_stages(; M = Symmetric) (mcmc.jl:415-425): covariance window, shrinkage,
    dense factorisation — vs the oracle with streaming co-moments."""
    rng = np.random.default_rng(77)
    ℓ = pkg.DiagNormal(rng.normal(size=D), np.logspace(-1, 1, D))
    K, N, seed = 10, 20, 99
    stages = pkg.default_warmup_stages(M=pkg.Symmetric, init_steps=30, middle_steps=25, doubling_stages=2,
                                       terminating_steps=20)
    r = pkg.mcmc_keep_warmup(seed, ℓ, N, chains=K, warmup_stages=stages)
    T, _ = r["engine"].layout()
    res = r["inference"]
    ostages = po.default_warmup_stages(init_steps=30, middle_steps=25, doubling_stages=2, terminating_steps=20,
                                       M=po.METRIC_SYMMETRIC)
    for k in range(0, K, 3):
        o = po.mcmc_with_warmup(1, D, N, seed, k, stages=ostages, params=ℓ.params(), T=T, welford=True,
                                keep_warmup=True)
        w = np.concatenate([s["results"]["tree_statistics"][k] for s in r["warmup"] if s["results"]])
        for f in INT_FIELDS:
            assert np.array_equal(w[f], o["warmup_stats"][f]), f
        assert res[k]["κ"].dense and np.array_equal(res[k]["κ"].minv, o["minv"])
        assert res[k]["ϵ"] == o["eps"]
        assert np.array_equal(res[k]["posterior_matrix"].T, o["posterior_matrix"])
    r["engine"].close()


# --------------------------------------------------------------- logistic regression family
@pytest.mark.parametrize("N,p", [(50, 3), (333, 40), (1000, 100), (2000, 256), (600, 400)])
def test_logistic_regression_matches_oracle(pkg, po, N, p):
    rng = np.random.default_rng(N + p)
    X = rng.normal(size=(N, p)) / np.sqrt(p)
    y = (rng.uniform(size=N) < 1 / (1 + np.exp(-X @ rng.normal(size=p)))).astype(float)
    ℓ = pkg.LogisticRegression(X, y)
    K = 5
    eng = _engine(pkg, ℓ, K, seed=8)
    T, _ = eng.layout()
    params = po.logistic_params(X, y)
    q = rng.normal(size=(K, p)) * 0.3
    pm = rng.normal(size=(K, p))
    eps = rng.uniform(0.01, 0.08, K)
    eng.set_position(q); eng.set_momentum(pm); eng.set_stepsize(eps)
    st = eng.get_state(("lq", "grad"))
    for k in range(K):
        lq, g = po.logdensity_and_gradient(po.FAMILY_LOGISTIC, q[k], params, T)
        assert st["lq"][k] == lq and np.array_equal(st["grad"][k], g)
    eng.leapfrog(2, 1)
    st = eng.get_state(("q", "p", "lq"))
    for k in range(K):
        qo, p_o, go, lqo = po.leapfrog(po.FAMILY_LOGISTIC, q[k], pm[k], eps[k], params=params, T=T, n_steps=2)
        np.testing.assert_allclose(st["q"][k], qo, rtol=RTOL, atol=0)
        assert np.array_equal(st["q"][k], qo) and np.array_equal(st["p"][k], p_o) and st["lq"][k] == lqo
    eng.set_position(q)
    stats = eng.sample_tree()
    new = eng.get_state(("q",))["q"]
    for k in range(K):
        o = po.sample_tree(po.FAMILY_LOGISTIC, q[k], eps[k], 8, k, 0, params=params, T=T)
        for f in INT_FIELDS:
            assert o["stats"][f] == stats[k][f]
        assert np.array_equal(new[k], o["q"])
    eng.close()


def test_logistic_dense_warmup_matches_oracle(pkg, po):
    """C4 in miniature: logistic regression, default_warmup_stages(; M = Symmetric)."""
    ℓ, _ = pkg.LogisticRegression.synthetic(N=400, p=12, seed=7)
    K, N, seed = 6, 15, 5
    stages = pkg.default_warmup_stages(M=pkg.Symmetric, init_steps=25, middle_steps=25, doubling_stages=2,
                                       terminating_steps=20)
    r = pkg.mcmc_keep_warmup(seed, ℓ, N, chains=K, warmup_stages=stages)
    T, _ = r["engine"].layout()
    params = po.logistic_params(ℓ.X, ℓ.y)
    ostages = po.default_warmup_stages(init_steps=25, middle_steps=25, doubling_stages=2, terminating_steps=20,
                                       M=po.METRIC_SYMMETRIC)
    for k in (0, 3, 5):
        o = po.mcmc_with_warmup(po.FAMILY_LOGISTIC, 12, N, seed, k, stages=ostages, params=params, T=T,
                                welford=True)
        res = r["inference"][k]
        assert res["κ"].dense and np.array_equal(res["κ"].minv, o["minv"]) and res["ϵ"] == o["eps"]
        assert np.array_equal(res["posterior_matrix"].T, o["posterior_matrix"])
        for f in INT_FIELDS:
            assert np.array_equal(res["tree_statistics"][f], o["tree_statistics"][f])
    r["engine"].close()


@pytest.mark.parametrize("M", ["Diagonal", "Symmetric"])
@pytest.mark.parametrize("N,p,K", [(300, 20, 21), (1100, 130, 9), (2000, 256, 16), (999, 255, 11), (1037, 77, 19), (31, 5, 8),
                                   (700, 200, 10), (640, 256, 9)])
def test_logistic_packed_groups_equal_one_chain_per_cta(pkg, N, p, K, M):
    """Packed chain groups (8 chains per CTA sharing every pass over X on the FP64 tensor cores, the default for
    dim <= 256) against one chain per CTA with the same threads per chain, whose likelihood is plain FMA loops.
    mma.sync.m8n8k4.f64 accumulates as sequential FMAs (benchmarks/dmma_order_probe.cu) and the per-chain arithmetic
    and its order are the same, so everything is bit-identical: the likelihood rounds and, with a Symmetric metric,
    the cooperative M⁻¹p — odd dimensions, a ragged last row block, a ragged last CTA and warps that run out of
    chains early and only attend the cooperative rounds."""
    ℓ, _ = pkg.LogisticRegression.synthetic(N=N, p=p, seed=N + p)
    stages = pkg.default_warmup_stages(M=getattr(pkg, M), init_steps=20, middle_steps=20, doubling_stages=1,
                                       terminating_steps=20)
    out = []
    T = None
    for packed in (True, False):      # an explicit threads_per_chain selects one chain per CTA
        r = pkg.mcmc_keep_warmup(77, ℓ, 12, chains=K, warmup_stages=stages,
                                 engine_opts=None if packed else dict(threads_per_chain=T))
        T = r["engine"].layout()[0] if packed else T
        assert r["engine"].layout()[0] == T
        out.append(r)
    for k in range(K):
        a, b = out[0]["inference"][k], out[1]["inference"][k]
        assert a["ϵ"] == b["ϵ"] and np.array_equal(a["κ"].minv, b["κ"].minv)
        assert np.array_equal(a["posterior_matrix"], b["posterior_matrix"])
        assert np.array_equal(a["logdensities"], b["logdensities"])
        for f in INT_FIELDS:
            assert np.array_equal(a["tree_statistics"][f], b["tree_statistics"][f])
    for r in out:
        r["engine"].close()


@pytest.mark.parametrize("family", ["diag_normal", "logistic", "logistic256"])
def test_pooled_symmetric_metric_matches_oracle(pkg, po, family):
    """The optional exchange of SURVEY §8e (NOT reference semantics, off by default): TuningNUTS(N, M = SymmetricPooled) ends
    the window with ONE dense metric per group of 8 consecutive global chains, estimated from the group's pooled draws.  The
    oracle implements the same option (mcmc_with_warmup_pooled); draws, integers, step sizes and the shared metric must be
    equal — one chain per CTA (diag_normal) and the packed tensor-core kernels, whose M⁻¹·[8 vectors] is then a true GEMM."""
    rng = np.random.default_rng(4)
    if family == "diag_normal":
        D = 24
        ℓ = pkg.DiagNormal(rng.normal(size=D), rng.uniform(0.3, 3, D)); fam, params = po.FAMILY_DIAG_NORMAL, ℓ.params()
    else:
        N_, D = (500, 20) if family == "logistic" else (900, 256)
        ℓ, _ = pkg.LogisticRegression.synthetic(N=N_, p=D, seed=11); fam, params = po.FAMILY_LOGISTIC, po.logistic_params(ℓ.X, ℓ.y)
    K, N, seed, off = 24, 4, 2026, 40
    stages = (pkg.InitialStepsizeSearch(), pkg.TuningNUTS(22, pkg.DualAveraging()),
              pkg.TuningNUTS(28, pkg.DualAveraging(), pkg.SymmetricPooled), pkg.TuningNUTS(20, pkg.DualAveraging()))
    r = pkg.mcmc_keep_warmup(seed, ℓ, N, chains=K, warmup_stages=stages, chain_offset=off, keep_warmup=False)
    T, _ = r["engine"].layout()
    ostages = [(po.STAGE_SEARCH, 0, 0, 0), (po.STAGE_TUNING, 22, 0, 1), (po.STAGE_TUNING, 28, po.METRIC_SYMMETRIC_POOLED, 1),
               (po.STAGE_TUNING, 20, 0, 1)]
    for g in range(K // 8):
        o = po.mcmc_with_warmup_pooled(fam, D, N, seed, off + 8 * g, ostages, params=params, T=T)
        for c in range(8):
            res = r["inference"][8 * g + c]
            assert res["κ"].dense and np.array_equal(res["κ"].minv, o["minv"]) and res["ϵ"] == o["eps"][c]
            assert np.array_equal(res["posterior_matrix"].T, o["posterior_matrix"][c])
            for f in INT_FIELDS:
                assert np.array_equal(res["tree_statistics"][f], o["tree_statistics"][c][f])
    r["engine"].close()


def test_c4_shape_matches_oracle(pkg, po):
    """BASELINE.json configs[3] at its exact shape — logistic regression N = 10 000, p = 256, per-chain dense
    (Symmetric) metric — against the oracle: warm-up with a Symmetric stage (so M⁻¹, W and ϵ are the adapted ones),
    then draws; chains 0, 5 and the last one of a handle whose chain count is not a multiple of the CTA's 8.
    Integers bit-exact, positions / metric / step size bit-equal (tolerance bar: 1e-10 relative)."""
    ℓ, _ = pkg.LogisticRegression.synthetic(N=10000, p=256, seed=7)
    K, N, seed = 13, 3, 2026
    stages = (pkg.InitialStepsizeSearch(), pkg.TuningNUTS(20, pkg.DualAveraging()),
              pkg.TuningNUTS(20, pkg.DualAveraging(), pkg.Symmetric), pkg.TuningNUTS(20, pkg.DualAveraging()))
    r = pkg.mcmc_keep_warmup(seed, ℓ, N, chains=K, warmup_stages=stages)
    T, _ = r["engine"].layout()
    params = po.logistic_params(ℓ.X, ℓ.y)
    ostages = po.default_warmup_stages(init_steps=20, middle_steps=20, doubling_stages=1, terminating_steps=20,
                                       M=po.METRIC_SYMMETRIC)
    for k in (0, 5, K - 1):
        o = po.mcmc_with_warmup(po.FAMILY_LOGISTIC, 256, N, seed, k, stages=ostages, params=params, T=T, welford=True)
        res = r["inference"][k]
        assert res["κ"].dense
        np.testing.assert_allclose(res["κ"].minv, o["minv"], rtol=RTOL, atol=0)
        np.testing.assert_allclose(res["posterior_matrix"].T, o["posterior_matrix"], rtol=RTOL, atol=0)
        assert np.array_equal(res["κ"].minv, o["minv"]) and res["ϵ"] == o["eps"]
        assert np.array_equal(res["posterior_matrix"].T, o["posterior_matrix"])
        for f in INT_FIELDS:
            assert np.array_equal(res["tree_statistics"][f], o["tree_statistics"][f])
    r["engine"].close()


@pytest.mark.parametrize("D,max_depth,eps_lo,eps_hi", [(3, 15, 2e-4, 4e-4), (2, 20, 4e-4, 3e-3), (40, 32, 2e-4, 6e-4)])
def test_deep_trees_match_oracle(pkg, po, D, max_depth, eps_lo, eps_hi):
    """max_depth beyond 12 (reference limit: 0 < max_depth ≤ 32, NUTS.jl:190, trees.jl:10): the slot pool spills past its
    64-slot register word.  Tiny step sizes make the trees 11-15 doublings deep — some end at max_depth, some by a U-turn
    deep in the tree — and every integer and the new position must still equal the recursive oracle's."""
    rng = np.random.default_rng(max_depth)
    K = 6
    ℓ = pkg.StandardNormal(D)
    eng = _engine(pkg, ℓ, K, seed=31, algorithm=pkg.NUTS(max_depth=max_depth))
    T, _ = eng.layout()
    q = rng.normal(size=(K, D))
    eps = np.exp(rng.uniform(np.log(eps_lo), np.log(eps_hi), K))
    eng.set_position(q); eng.set_stepsize(eps)
    depths = []
    for t in range(2):
        stats = eng.sample_tree()
        st = eng.get_state(("q", "grad"))
        for k in range(K):
            o = po.sample_tree(po.FAMILY_STD_NORMAL, q[k], eps[k], 31, k, t, T=T, max_depth=max_depth)
            for f in INT_FIELDS:
                assert o["stats"][f] == stats[k][f], (f, k, t, o["stats"], stats[k])
            assert o["stats"]["pi"] == stats[k]["pi"] and o["stats"]["acceptance_rate"] == stats[k]["acceptance_rate"]
            assert np.array_equal(st["q"][k], o["q"]) and np.array_equal(st["grad"][k], o["g"])
            depths.append(int(stats[k]["depth"]))
        q = st["q"]
    assert max(depths) >= min(13, max_depth)        # the spill words of the slot pool were really used
    eng.close()


@pytest.mark.parametrize("direct", ["0", "1"])
def test_thinned_draws_into_page_locked_buffers(pkg, monkeypatch, direct):
    """§8f-3: dhmc_mcmc_thinned keeps every thin-th transition; with page-locked output buffers (dhmc_host_alloc) the
    draws are either staged and copied (default while they fit in HBM) or written by the sampling kernel straight into
    the host buffer (DHMC_DIRECT=1 — the route taken when they do not fit).  Both must equal the plain mcmc call."""
    monkeypatch.setenv("DHMC_DIRECT", direct)
    D, K, N, thin = 130, 200, 12, 3
    rng = np.random.default_rng(8)
    ℓ = pkg.DiagNormal(rng.normal(size=D), rng.uniform(0.5, 2, D))
    outs = []
    for mode in ("plain", "thinned"):
        eng = pkg.Engine(ℓ, chains=K, seed=99)
        eng.random_position(); eng.find_initial_stepsize()
        eng.warmup_stage(pkg.TuningNUTS(30, pkg.DualAveraging()))
        if mode == "plain":
            outs.append(eng.mcmc(N))
        else:
            bufs = dict(posterior_matrix=eng.host_alloc((K, N // thin, D)),
                        tree_statistics=eng.host_alloc((K, N // thin), dtype=pkg._lib.tree_stats_dtype),
                        logdensities=eng.host_alloc((K, N // thin)))
            r = eng.mcmc_thinned(N, thin, out=bufs)
            outs.append({k: np.array(v) for k, v in r.items()})
        eng.close()
    a, b = outs
    assert np.array_equal(a["posterior_matrix"][:, thin - 1::thin], b["posterior_matrix"])
    assert np.array_equal(a["logdensities"][:, thin - 1::thin], b["logdensities"])
    for f in INT_FIELDS:
        assert np.array_equal(a["tree_statistics"][f][:, thin - 1::thin], b["tree_statistics"][f])


def test_device_ess_rhat_and_acceptance_quantiles(pkg):
    """§8f-2: split-R̂ / ESS across chains and the acceptance-rate quantiles reduced on the GPU from device-resident draws
    and statistics, against the numpy mirror (diagnostics.ess_rhat) resp. numpy quantiles of the same records."""
    import torch
    D, K, N = 37, 512, 120
    rng = np.random.default_rng(3)
    ℓ = pkg.DiagNormal(rng.normal(size=D), rng.uniform(0.3, 4, D))
    eng = pkg.Engine(ℓ, chains=K, seed=17)
    eng.random_position(); eng.find_initial_stepsize()
    eng.warmup_stage(pkg.TuningNUTS(60, pkg.DualAveraging()))
    draws = torch.empty((K, N, D), dtype=torch.float64, device="cuda")
    stats = torch.empty((K, N, 56), dtype=torch.uint8, device="cuda")
    eng.mcmc_dev(N, draws.data_ptr(), stats.data_ptr(), 0)
    dev = eng.ess_rhat_dev(draws.data_ptr(), N, max_lag=40)
    ref = pkg.diagnostics.ess_rhat(draws.cpu().numpy(), max_lag=40)
    np.testing.assert_allclose(dev["rhat"], ref["rhat"], rtol=1e-9)
    np.testing.assert_allclose(dev["ess"], ref["ess"], rtol=1e-7)
    assert np.all(dev["rhat"] < 1.02) and np.all(dev["ess"] > 0.2 * K * N)        # the bar of sample-correctness_utilities.jl:107-110
    a = stats.cpu().numpy().view(pkg._lib.tree_stats_dtype).reshape(K, N)["acceptance_rate"].ravel()
    q = eng.acceptance_quantiles_dev(stats.data_ptr(), N)
    np.testing.assert_allclose(q, np.quantile(a, pkg.diagnostics.ACCEPTANCE_QUANTILES), atol=5e-4)
    eng.close()


# --------------------------------------------------------------- trajectory diagnostics (diagnostics.jl:139-216)
def test_trajectory_diagnostics_match_oracle(pkg, po):
    D = 37
    rng = np.random.default_rng(12)
    mu, sigma2 = rng.normal(size=D), rng.uniform(0.3, 4, D)
    ℓ = pkg.DiagNormal(mu, sigma2)
    params = ℓ.params()                      # [μ, 1/σ²]
    minv = rng.uniform(0.5, 2, D)
    κ = pkg.GaussianKineticEnergy(minv)
    q = rng.normal(size=D)
    ps = rng.normal(size=(4, D))
    log2eps = [-6, -3, -1, 0, 1]
    A = pkg.diagnostics.explore_log_acceptance_ratios(ℓ, q, log2eps, κ=κ, ps=ps)
    assert A.shape == (5, 4)
    T = 32 if D <= 128 else 64
    for i, l2 in enumerate(log2eps):
        for j in range(4):
            assert A[i, j] == po.local_log_acceptance_ratio(po.FAMILY_DIAG_NORMAL, q, ps[j], 2.0 ** l2, minv=minv,
                                                            params=params, T=T)
    assert pkg.diagnostics.explore_log_acceptance_ratios(ℓ, q, [-2.0], κ=κ, N=7, seed=3).shape == (1, 7)
    traj = pkg.diagnostics.leapfrog_trajectory(ℓ, q, 0.11, range(-3, 5), κ=κ, p=ps[0])
    assert [t["position"] for t in traj] == list(range(-3, 5)) and traj[3]["Δ"] == 0.0
    lq0, _ = po.logdensity_and_gradient(po.FAMILY_DIAG_NORMAL, q, params, T)
    π0 = po.phase_logdensity(minv, lq0, ps[0], T)
    for t in traj:
        i = t["position"]
        if i == 0:
            assert np.array_equal(t["z"]["q"], q) and t["z"]["lq"] == lq0
            continue
        qo, p_o, _, lqo = po.leapfrog(po.FAMILY_DIAG_NORMAL, q, ps[0], 0.11 if i > 0 else -0.11, minv=minv,
                                     params=params, T=T, n_steps=abs(i))
        assert np.array_equal(t["z"]["q"], qo) and np.array_equal(t["z"]["p"], p_o) and t["z"]["lq"] == lqo
        assert t["Δ"] == po.phase_logdensity(minv, lqo, p_o, T) - π0
    with pytest.raises(pkg.ArgumentError):
        pkg.diagnostics.leapfrog_trajectory(ℓ, q, 0.1, range(1, 4), κ=κ)


# --------------------------------------------------------------- full-size properties (BASELINE configs[1])
def test_full_size_properties_c2(pkg):
    """65 536 chains × D=1000 (config C2): size-independent properties the domain offers —
    leapfrog reversibility, energy error of the integrator, tree-statistics invariants,
    and agreement of a shard with the full run."""
    D, K = 1000, 65536
    ℓ = pkg.StandardNormal(D)
    eng = _engine(pkg, ℓ, K, seed=2026)
    eng.random_position()
    q0 = eng.get_state(("q",))["q"]
    rng = np.random.default_rng(0)
    p0 = rng.normal(size=(K, D))
    eng.set_momentum(p0)
    eng.set_stepsize(0.05)
    H0 = eng.phase_logdensity()
    eng.leapfrog(8, 1)
    H1 = eng.phase_logdensity()
    assert np.max(np.abs(H1 - H0)) < 0.5                      # test_hamiltonian.jl:118-141
    eng.leapfrog(8, -1)
    st = eng.get_state(("q", "p"))
    assert np.max(np.abs(st["q"] - q0)) < 1e-9 and np.max(np.abs(st["p"] - p0)) < 1e-9   # :143-177
    eng.set_stepsize(0.28)
    q_before = st["q"]
    out = eng.mcmc(1)
    ts = out["tree_statistics"][:, 0]
    # the chunk-pipelined upload path (dhmc_mcmc_from) gives the same transition
    eng2 = _engine(pkg, ℓ, K, seed=2026)
    eng2.set_stepsize(0.28)
    out2 = eng2.mcmc_from(q_before, 1)
    eng2.close()
    assert np.array_equal(out2["posterior_matrix"], out["posterior_matrix"])
    assert np.array_equal(out2["tree_statistics"], out["tree_statistics"])
    del out2
    assert np.all(ts["depth"] >= 0) and np.all(ts["depth"] <= 10)
    assert np.all(ts["steps"] >= 1) and np.all(ts["steps"] <= 2 ** (ts["depth"] + 1) - 1)
    assert np.all(ts["steps"] >= 2 ** ts["depth"] - 1)
    assert np.all((ts["acceptance_rate"] >= 0) & (ts["acceptance_rate"] <= 1))
    maxd = (ts["left"] == 1) & (ts["right"] == 0)
    assert np.all(ts["depth"][maxd] == 10)
    assert eng.last_total_steps() == int(ts["steps"].sum())
    assert np.all(np.isfinite(out["logdensities"])) and np.all(eng.chain_status() == 0)
    lq = -0.5 * np.einsum("kd,kd->k", out["posterior_matrix"][:, 0], out["posterior_matrix"][:, 0])
    np.testing.assert_allclose(out["logdensities"][:, 0], lq, rtol=1e-12)
    eng.close()
    # a 64-chain shard at offset 40 000 reproduces those chains bit for bit
    sh = pkg.Engine(ℓ, chains=64, seed=2026, chain_offset=40000)
    sh.random_position(); sh.set_momentum(p0[40000:40064]); sh.set_stepsize(0.05)
    sh.leapfrog(8, 1); sh.leapfrog(8, -1)
    sh.set_stepsize(0.28)
    b = sh.mcmc(1)
    sh.close()
    assert np.array_equal(b["posterior_matrix"], out["posterior_matrix"][40000:40064])
    assert np.array_equal(b["tree_statistics"], out["tree_statistics"][40000:40064])


def test_checkpoint_and_resume(pkg):
    """mcmc_keep_warmup / mcmc_steps surface (mcmc.jl:335-351, :521-532): (Q, κ, ϵ, RNG counter)
    is a complete checkpoint — a fresh handle restored from it continues the same chains."""
    D, K = 30, 50
    ℓ = pkg.DiagNormal(np.zeros(D), np.linspace(0.5, 4, D))
    a = _engine(pkg, ℓ, K, seed=5)
    a.random_position(); a.find_initial_stepsize()
    a.warmup_stage(pkg.TuningNUTS(40, pkg.DualAveraging(), pkg.Diagonal))
    ck = a.get_state(("q", "minv", "eps"))
    t = a.transition_count
    ref = a.mcmc(6)
    a.close()
    b = _engine(pkg, ℓ, K, seed=5)
    b.set_metric(ck["minv"]); b.set_position(ck["q"]); b.set_stepsize(ck["eps"])
    b.transition_count = t
    first = b.mcmc(2)
    second = b.mcmc(4)
    b.close()
    got = np.concatenate([first["posterior_matrix"], second["posterior_matrix"]], axis=1)
    assert np.array_equal(got, ref["posterior_matrix"])


@pytest.mark.parametrize("M", ["Diagonal", "Symmetric"])
def test_checkpoint_file_round_trip(pkg, tmp_path, M):
    """Engine.save_checkpoint / load_checkpoint: a fresh handle restored from the file continues the same chains (diagonal
    and Symmetric κ)."""
    D, K = 12, 40
    ℓ = pkg.DiagNormal(np.zeros(D), np.linspace(0.5, 4, D))
    a = _engine(pkg, ℓ, K, seed=5)
    a.random_position(); a.find_initial_stepsize()
    a.warmup_stage(pkg.TuningNUTS(40, pkg.DualAveraging(), getattr(pkg, M)))
    path = str(tmp_path / "ck.npz")
    a.save_checkpoint(path)
    ref = a.mcmc(5)
    a.close()
    b = _engine(pkg, ℓ, K, seed=5)
    b.load_checkpoint(path)
    got = b.mcmc(5)
    b.close()
    assert np.array_equal(got["posterior_matrix"], ref["posterior_matrix"])
    assert np.array_equal(got["tree_statistics"], ref["tree_statistics"])


def test_many_chains_per_cta_single_transition(pkg, po):
    """Regression: with more chains than resident CTAs and N = 1, every chain must use its own
    randexp stream (the 32-wide batch is per chain)."""
    D, K = 16, 20000
    eng = _engine(pkg, pkg.StandardNormal(D), K, seed=4)
    T, _ = eng.layout()
    eng.random_position(); eng.set_stepsize(0.3)
    q0 = eng.get_state(("q",))["q"]
    stats = eng.sample_tree()
    q1 = eng.get_state(("q",))["q"]
    for k in list(range(0, K, 997)) + [K - 1]:
        o = po.sample_tree(0, q0[k], 0.3, 4, k, 0, T=T)
        for f in INT_FIELDS:
            assert o["stats"][f] == stats[k][f]
        assert o["stats"]["pi"] == stats[k]["pi"] and np.array_equal(q1[k], o["q"])
    eng.close()


def test_mcmc_from_host_positions(pkg):
    """dhmc_mcmc_from = set_position + mcmc, pipelined; same results, strict initial check."""
    D, K, N = 64, 8192, 8
    ℓ = pkg.StandardNormal(D)
    rng = np.random.default_rng(1)
    q = rng.normal(size=(K, D))
    a = _engine(pkg, ℓ, K, seed=6)
    a.set_position(q); a.set_stepsize(0.4)
    ra = a.mcmc(N)
    a.close()
    b = _engine(pkg, ℓ, K, seed=6)
    b.set_stepsize(0.4)
    rb = b.mcmc_from(q, N)
    assert np.array_equal(ra["posterior_matrix"], rb["posterior_matrix"])
    assert np.array_equal(ra["tree_statistics"], rb["tree_statistics"])
    q[77, 3] = np.inf
    with pytest.raises(pkg.DynamicHMCError) as e:
        b.mcmc_from(q, 1)
    assert e.value.debug_information["chain_status"][77] & 1
    b.close()


def test_stepwise_sampling_equals_mcmc(pkg):
    """mcmc_steps / mcmc_next_step (mcmc.jl:335-351): N single transitions from the returned positions are the N draws of
    one mcmc call (same RNG counter, ℓ and ∇ℓ re-evaluated from the uploaded positions)."""
    D, K, N = 30, 200, 4
    ℓ = pkg.DiagNormal(np.linspace(-1, 1, D), np.logspace(-1, 1, D))
    stages = pkg.default_warmup_stages(init_steps=25, middle_steps=20, doubling_stages=1, terminating_steps=20)
    ra = pkg.mcmc_keep_warmup(8, ℓ, N, chains=K, warmup_stages=stages)
    rb = pkg.mcmc_keep_warmup(8, ℓ, 0, chains=K, warmup_stages=stages)
    steps = pkg.mcmc_steps(rb["engine"])
    Q = steps.Q
    for n in range(N):
        Q, stats = pkg.mcmc_next_step(steps, Q)
        for k in (0, 57, K - 1):
            assert np.array_equal(Q[k], ra["inference"][k]["posterior_matrix"][:, n])
            assert stats[k] == ra["inference"][k]["tree_statistics"][n]
    ra["engine"].close(); rb["engine"].close()


# --------------------------------------------------------------- reference integration tests (test/test_mcmc.jl)
def _rhat(x):
    """split-R̂ per parameter; x: [draw, chain, param] (stack_posterior_matrices layout)."""
    n = x.shape[0] // 2
    y = np.concatenate([x[:n], x[n:2 * n]], axis=1)
    W = y.var(0, ddof=1).mean(0)
    B = n * y.mean(0).var(0, ddof=1)
    return np.sqrt(((n - 1) / n * W + B / n) / W)


def test_mcmc_with_warmup_normal_moments(pkg):
    """test_mcmc.jl:18-26 with the full default warm-up, 64 chains at once."""
    D, N, K = 5, 2000, 64
    ℓ = pkg.DiagNormal(np.ones(D), np.ones(D))
    res = pkg.mcmc_with_warmup(123, ℓ, N, chains=K)
    Z = pkg.pool_posterior_matrices(res)                      # [param, draw ⊗ chain]
    assert Z.shape == (D, N * K)
    assert np.max(np.abs(Z.mean(1) - 1)) < 0.04 and np.max(np.abs(Z.std(1, ddof=1) - 1)) < 0.04
    S = pkg.stack_posterior_matrices(res)                     # [draw, chain, param], test_mcmc.jl:74-80
    assert S.shape == (N, K, D)
    assert np.all(_rhat(S) < 1.02)                            # sample-correctness_utilities.jl:107-110
    for k in (0, K - 1):
        r = res[k]
        assert r["posterior_matrix"].shape == (D, N)
        assert r["tree_statistics"]["acceptance_rate"].mean() >= 0.7
        assert 0.5 <= r["ϵ"] <= 2
        lq = np.array([ℓ.logdensity_and_gradient(q)[0] for q in r["posterior_matrix"].T[:20]])
        np.testing.assert_allclose(r["logdensities"][:20], lq, rtol=1e-12)
    accs = np.mean([res[k]["tree_statistics"]["acceptance_rate"].mean() for k in range(K)])
    assert accs >= 0.8


def test_fixed_stepsize_and_skipped_search(pkg):
    """test_mcmc.jl:28-48"""
    D, N, K = 5, 1000, 32
    ℓ = pkg.DiagNormal(np.ones(D), np.ones(D))
    res = pkg.mcmc_with_warmup(5, ℓ, N, chains=K, initialization={"ϵ": 1.0},
                               warmup_stages=pkg.fixed_stepsize_warmup_stages())
    assert all(res[k]["ϵ"] == 1.0 for k in range(K))
    Z = pkg.pool_posterior_matrices(res)
    assert np.max(np.abs(Z.mean(1) - 1)) < 0.05
    res = pkg.mcmc_with_warmup(6, ℓ, N, chains=K, initialization=dict(ϵ=1.0),
                               warmup_stages=pkg.default_warmup_stages(stepsize_search=None))
    assert all(0.5 <= res[k]["ϵ"] <= 2 for k in range(K))
    with pytest.raises(pkg.ArgumentError):              # search refuses a user-supplied ϵ, mcmc.jl:137
        pkg.mcmc_with_warmup(6, ℓ, 10, chains=4, initialization={"ϵ": 1.0})


def test_200_dim_never_reaches_max_depth(pkg):
    """test_mcmc.jl:60-72: N(0, I₂₀₀), max_depth 12, 20 chains × 1000 draws."""
    res = pkg.mcmc_with_warmup(11, pkg.StandardNormal(200), 1000, chains=20, algorithm=pkg.NUTS(max_depth=12))
    for k in range(20):
        ts = res[k]["tree_statistics"]
        assert not np.any((ts["left"] == 1) & (ts["right"] == 0)) and ts["depth"].max() < 12


def test_funnel_sample_correctness(pkg):
    """sample-correctness_tests.jl:112-118 (funnel): R̂ and marginal of v across many chains.
    The raw funnel's neck makes v mix slowly for NUTS with 1000 draws (the reference tests a
    mixed/transformed funnel with 10 000 draws), hence the looser bound on v."""
    res = pkg.mcmc_with_warmup(3, pkg.Funnel(5), 1000, chains=256)
    S = pkg.stack_posterior_matrices(res)
    rh = _rhat(S)
    assert rh[0] < 1.4 and np.all(rh[1:] < 1.2), rh
    v = S[:, :, 0]
    # v ~ N(0, 3) exactly, but NUTS under-explores the neck of the raw funnel: the known upward bias
    # of E[v] (≈ +1 at this chain length, identical in the oracle) — check the biased range.
    assert -0.5 < v.mean() < 1.8 and 2.0 < v.std() < 3.4, (v.mean(), v.std())


def test_diagnostics_host_and_device(pkg):
    """Diagnostics.EBFMI / summarize_tree_statistics (diagnostics.jl): numpy mirror on returned
    statistics vs the device-side reduction over a device-resident statistics buffer."""
    import torch
    D, K, N = 20, 300, 64
    eng = _engine(pkg, pkg.Funnel(D), K, seed=17)
    eng.random_position(); eng.set_stepsize(0.2)
    stats_dev = torch.empty((K, N, 56), dtype=torch.uint8, device="cuda")
    eng.mcmc_dev(N, 0, stats_dev.data_ptr(), 0)
    dev = eng.tree_summary_dev(stats_dev.data_ptr(), N)
    host = np.frombuffer(stats_dev.cpu().numpy().tobytes(), dtype=pkg._lib.tree_stats_dtype).reshape(K, N)
    eng.close()
    summ = pkg.diagnostics.summarize_tree_statistics(host)
    assert dev["N"] == summ.N == K * N
    assert dev["a_mean"] == pytest.approx(summ.a_mean, rel=1e-12)
    assert dev["termination_counts"] == summ.termination_counts and dev["depth_counts"] == summ.depth_counts
    assert dev["steps"] == int(host["steps"].sum())
    eb = np.array([pkg.diagnostics.EBFMI(host[k]) for k in range(K)])
    np.testing.assert_allclose(dev["EBFMI"], eb, rtol=1e-10)
    assert len(summ.a_quantiles) == 5 and sum(summ.termination_counts.values()) == K * N


def test_one_dimensional_problem(pkg, po):
    """dimension(ℓ) = 1 (the reference's variance-5e8 / 5e-8 univariate targets, sample-correctness_tests.jl:48-60)."""
    K = 40
    for var in (5e8, 5e-8, 1.0):
        ℓ = pkg.DiagNormal(np.array([0.3]), np.array([var]))
        eng = _engine(pkg, ℓ, K, seed=2)
        T, _ = eng.layout()
        q = np.random.default_rng(1).normal(size=(K, 1)) * np.sqrt(var)
        eng.set_position(q); eng.set_metric(np.array([var])); eng.set_stepsize(0.7)
        stats = eng.sample_tree()
        new = eng.get_state(("q",))["q"]
        for k in range(0, K, 7):
            o = po.sample_tree(1, q[k], 0.7, 2, k, 0, minv=np.array([var]), params=ℓ.params(), T=T)
            for f in INT_FIELDS:
                assert o["stats"][f] == stats[k][f]
            assert np.array_equal(new[k], o["q"])
        eng.close()
    res = pkg.mcmc_with_warmup(7, pkg.DiagNormal(np.array([1.0]), np.array([5e8])), 500, chains=32)
    Z = pkg.pool_posterior_matrices(res)
    assert abs(Z.std() / np.sqrt(5e8) - 1) < 0.1
