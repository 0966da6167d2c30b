"""Problem batches (dhmc_set_problems): P posteriors of one family and dimension on one handle, global chain g sampling
problem g // K.  The definition of correctness needs no oracle: chains [p·K, (p+1)·K) of a batch equal, bit for bit, a
handle that holds problem p alone with chain_offset = p·K.  The CPU tests check the host-side validation and the
per-problem views of the results."""
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODELS = os.path.join(ROOT, "include", "models")
INT_FIELDS = ("depth", "left", "right", "steps", "directions")


def _stages(pkg, M="Diagonal"):
    return pkg.default_warmup_stages(M=getattr(pkg, M), init_steps=20, middle_steps=20, doubling_stages=1,
                                     terminating_steps=20)


def _logistic_batch(pkg, N, p, P, seed=0):
    return [pkg.LogisticRegression.synthetic(N=N, p=p, seed=seed + 31 * i)[0] for i in range(P)]


def _diag_batch(pkg, D, P, seed=0):
    rng = np.random.default_rng(seed)
    return [pkg.DiagNormal(rng.normal(size=D) * 3, rng.uniform(0.3, 3, D)) for _ in range(P)]


def _assert_same_chain(a, b):
    """a, b: the reference's per-chain NamedTuples (Results[k])."""
    assert a["ϵ"] == b["ϵ"]
    assert np.array_equal(a["κ"].minv, b["κ"].minv)
    assert np.array_equal(a["posterior_matrix"], b["posterior_matrix"])
    assert np.array_equal(a["logdensities"], b["logdensities"])
    for f in INT_FIELDS:
        assert np.array_equal(a["tree_statistics"][f], b["tree_statistics"][f]), f
    for f in ("pi", "acceptance_rate"):
        assert np.array_equal(a["tree_statistics"][f], b["tree_statistics"][f]), f


def _batch_equals_separate(pkg, problems, K, N, stages, seed=77, engine_opts=None, algorithm=None):
    batch = pkg.ProblemBatch(problems, K)
    r = pkg.mcmc_keep_warmup(seed, batch, N, warmup_stages=stages, engine_opts=engine_opts, algorithm=algorithm)
    assert len(r["inference"]) == len(problems) * K
    per = pkg.results_by_problem(r["inference"], batch)
    layout = r["engine"].layout()
    r["engine"].close()
    for p, ℓ in enumerate(problems):
        s = pkg.mcmc_keep_warmup(seed, ℓ, N, chains=K, chain_offset=p * K, warmup_stages=stages, engine_opts=engine_opts,
                                 algorithm=algorithm)
        assert s["engine"].layout() == layout
        s["engine"].close()
        assert len(per[p]) == K
        for k in range(K):
            _assert_same_chain(per[p][k], s["inference"][k])
    return layout


# --------------------------------------------------------------- CPU: host-side validation and views
def test_problem_batch_validation(pkg):
    rng = np.random.default_rng(0)
    d = _diag_batch(pkg, 7, 3)
    b = pkg.ProblemBatch(d, 4)
    assert (b.family, b.dimension(), b.n_problems, b.chains, b.block_size) == (pkg._lib.FAMILY_DIAG_NORMAL, 7, 3, 12, 14)
    assert b.library_path is None
    assert np.array_equal(b.params(), np.concatenate([x.params() for x in d]))
    assert [b.problem_chains(p) for p in range(3)] == [(0, 4), (4, 8), (8, 12)]
    assert [b.problem_chains(p, chain_offset=6, chains=4) for p in range(3)] == [(0, 0), (0, 2), (2, 4)]
    with pytest.raises(pkg.ArgumentError):
        pkg.ProblemBatch([], 4)
    with pytest.raises(pkg.ArgumentError):
        pkg.ProblemBatch(d, 0)
    with pytest.raises(pkg.ArgumentError, match="dimension"):
        pkg.ProblemBatch(d + _diag_batch(pkg, 8, 1), 4)
    with pytest.raises(pkg.ArgumentError, match="family"):
        pkg.ProblemBatch([d[0], pkg.LogisticRegression(rng.normal(size=(5, 7)), np.ones(5))], 4)
    for ℓ in (pkg.StandardNormal(7), pkg.Funnel(7)):
        with pytest.raises(pkg.ArgumentError, match="no parameters"):
            pkg.ProblemBatch([ℓ, ℓ], 4)
    lg = [pkg.LogisticRegression(rng.normal(size=(n, 5)), np.ones(n)) for n in (30, 30, 31)]
    assert pkg.ProblemBatch(lg[:2], 8).block_size == 1 + 30 * 5 + 30
    with pytest.raises(pkg.ArgumentError, match="same N"):
        pkg.ProblemBatch(lg, 8)

    class FakeUser(pkg.api.DeviceLogDensity):        # user models: same library required (no build needed to check it)
        family = pkg._lib.FAMILY_USER

        def __init__(self, lib, pr):
            self.D, self.library_path, self._p = 4, lib, np.asarray(pr, float)

        def params(self):
            return self._p

    assert pkg.ProblemBatch([FakeUser("a.so", [1, 2]), FakeUser("a.so", [3, 4])], 2).library_path == "a.so"
    with pytest.raises(pkg.ArgumentError, match="library"):
        pkg.ProblemBatch([FakeUser("a.so", [1, 2]), FakeUser("b.so", [3, 4])], 2)
    with pytest.raises(pkg.ArgumentError, match="same length"):
        pkg.ProblemBatch([FakeUser("a.so", [1, 2]), FakeUser("a.so", [3, 4, 5])], 2)


def test_results_by_problem_views(pkg):
    P, K, N, D = 4, 3, 5, 2
    B = P * K
    post = np.arange(B * N * D, dtype=float).reshape(B, N, D)
    stats = np.zeros((B, N), dtype=pkg._lib.tree_stats_dtype)
    stats["depth"] = np.arange(B)[:, None]
    logd = np.arange(B * N, dtype=float).reshape(B, N)
    minv = np.arange(B * D, dtype=float).reshape(B, D)
    eps = np.arange(B, dtype=float) / 10
    res = pkg.Results(post, stats, logd, minv, eps)
    batch = pkg.ProblemBatch(_diag_batch(pkg, D, P), K)
    per = pkg.results_by_problem(res, batch)
    assert [len(r) for r in per] == [K] * P
    for p in range(P):
        for k in range(K):
            g = p * K + k
            assert np.array_equal(per[p][k]["posterior_matrix"], post[g].T)
            assert per[p][k]["tree_statistics"]["depth"][0] == g and per[p][k]["ϵ"] == eps[g]
            assert np.array_equal(per[p][k]["κ"].minv, minv[g])
    assert np.shares_memory(per[2]._post, post)                   # zero-copy
    # a shard that starts in the middle of problem 1 and ends in problem 2
    shard = pkg.Results(post[4:8], stats[4:8], logd[4:8], minv[4:8], eps[4:8])
    per = pkg.results_by_problem(shard, batch, chain_offset=4)
    assert [len(r) for r in per] == [0, 2, 2, 0]
    assert per[1][0]["tree_statistics"]["depth"][0] == 4 and per[2][1]["tree_statistics"]["depth"][0] == 7


# --------------------------------------------------------------- GPU: batch = separate handles, bit for bit
@pytest.mark.gpu
def test_diag_normal_batch_equals_separate_handles(pkg):
    _batch_equals_separate(pkg, _diag_batch(pkg, 37, 5, seed=1), K=6, N=12, stages=_stages(pkg))


@pytest.mark.gpu
@pytest.mark.parametrize("M", ["Diagonal", "Symmetric"])
@pytest.mark.parametrize("N,p", [(300, 20), (900, 256)])
def test_logistic_packed_batch_equals_separate_handles(pkg, N, p, M):
    """Packed chain groups: a CTA takes 8 consecutive chains of one problem and its tensor-core rounds read that problem's X."""
    layout = _batch_equals_separate(pkg, _logistic_batch(pkg, N, p, 3, seed=N + p), K=16, N=8, stages=_stages(pkg, M))
    assert layout[0] == 32                                          # one warp per chain: the packed kernels ran


@pytest.mark.gpu
def test_logistic_one_chain_per_cta_batch_with_problems_mid_cta(pkg):
    """threads_per_chain=32: one chain per CTA, no 8-alignment — with K = 5 problems start anywhere."""
    _batch_equals_separate(pkg, _logistic_batch(pkg, 300, 20, 3, seed=5), K=5, N=8, stages=_stages(pkg),
                           engine_opts=dict(threads_per_chain=32))


@pytest.mark.gpu
def test_deep_tree_batch_equals_separate_handles(pkg):
    """max_depth > 12: the deep kernels read the problem's block too."""
    _batch_equals_separate(pkg, _diag_batch(pkg, 6, 3, seed=2), K=4, N=6, stages=_stages(pkg),
                           algorithm=pkg.NUTS(max_depth=15))


def _eight_schools(pkg, P):
    rng = np.random.default_rng(8)
    y0 = np.array([28.0, 8, -3, 7, -1, 1, 18, 12])
    s0 = np.array([15.0, 10, 16, 11, 9, 11, 10, 18])
    return [pkg.UserLogDensity(os.path.join(MODELS, "eight_schools.h"), 10,
                               params=np.concatenate([y0 + rng.normal(size=8) * 5, s0 * rng.uniform(0.7, 1.3, 8)]))
            for _ in range(P)]


@pytest.mark.gpu
def test_user_model_batch_equals_separate_handles(pkg):
    """Eight schools with different (y, σ) per problem: eval_user reads the problem's params."""
    _batch_equals_separate(pkg, _eight_schools(pkg, 3), K=6, N=10, stages=_stages(pkg))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["diag_normal", "logistic", "user"])
def test_light_kernels_batch_equal_separate_handles(pkg, kind):
    """k_eval (set_position), k_leapfrog and k_phase from set positions, momenta and step sizes."""
    P, K = 3, 8
    problems = {"diag_normal": lambda: _diag_batch(pkg, 37, P, seed=3),
                "logistic": lambda: _logistic_batch(pkg, 300, 20, P, seed=9),
                "user": lambda: _eight_schools(pkg, P)}[kind]()
    D = problems[0].dimension()
    rng = np.random.default_rng(4)
    q, mom = rng.normal(size=(P * K, D)) * 0.3, rng.normal(size=(P * K, D))
    minv, eps = rng.uniform(0.5, 2, (P * K, D)), rng.uniform(0.01, 0.05, P * K)

    def run(ℓ, sl, off):
        eng = pkg.Engine(ℓ, chains=sl.stop - sl.start, seed=3, chain_offset=off)
        eng.set_metric(minv[sl]); eng.set_position(q[sl]); eng.set_momentum(mom[sl]); eng.set_stepsize(eps[sl])
        out = [eng.get_state(("q", "lq", "grad")), eng.phase_logdensity()]
        eng.leapfrog(3, 1)
        out += [eng.get_state(("q", "p", "lq", "grad")), eng.phase_logdensity()]
        eng.close()
        return out

    full = run(pkg.ProblemBatch(problems, K), slice(0, P * K), 0)
    for p in range(P):
        sep = run(problems[p], slice(p * K, (p + 1) * K), p * K)
        for a, b in zip(full, sep):
            if isinstance(a, dict):
                for f in b:
                    assert np.array_equal(a[f][p * K:(p + 1) * K], b[f]), f
            else:
                assert np.array_equal(a[p * K:(p + 1) * K], b)


# --------------------------------------------------------------- GPU: against the oracle
@pytest.mark.gpu
@pytest.mark.parametrize("family", ["diag_normal", "logistic"])
def test_batch_matches_oracle(pkg, po, family):
    P, K, N, seed = 3, 8, 10, 515
    if family == "diag_normal":
        problems, fam, D = _diag_batch(pkg, 12, P, seed=6), po.FAMILY_DIAG_NORMAL, 12
        params = [ℓ.params() for ℓ in problems]
    else:
        problems, fam, D = _logistic_batch(pkg, 200, 16, P, seed=6), po.FAMILY_LOGISTIC, 16
        params = [po.logistic_params(ℓ.X, ℓ.y) for ℓ in problems]
    kw = dict(init_steps=20, middle_steps=20, doubling_stages=1, terminating_steps=20)
    r = pkg.mcmc_keep_warmup(seed, pkg.ProblemBatch(problems, K), N, warmup_stages=pkg.default_warmup_stages(**kw))
    T, _ = r["engine"].layout()
    r["engine"].close()
    ostages = po.default_warmup_stages(**kw)
    for g in range(0, P * K, 3):
        o = po.mcmc_with_warmup(fam, D, N, seed, g, stages=ostages, params=params[g // K], T=T, welford=True)
        res = r["inference"][g]
        assert res["ϵ"] == o["eps"] and np.array_equal(res["κ"].minv, o["minv"])
        assert np.array_equal(res["posterior_matrix"].T, o["posterior_matrix"])
        for f in INT_FIELDS:
            assert np.array_equal(res["tree_statistics"][f], o["tree_statistics"][f])


# --------------------------------------------------------------- GPU: shards and chunks
def _short_run(pkg, ℓ, chains, off, seed=21, N=6, eps=0.05, **kw):
    eng = pkg.Engine(ℓ, chains=chains, seed=seed, chain_offset=off, **kw)
    eng.random_position(); eng.set_stepsize(eps)
    out = eng.mcmc(N)
    eng.close()
    return out


@pytest.mark.gpu
def test_batch_shards_equal_slices_of_the_full_run(pkg):
    # one chain per CTA: a shard that starts in the middle of a problem
    batch = pkg.ProblemBatch(_diag_batch(pkg, 20, 4, seed=7), 6)
    full = _short_run(pkg, batch, 24, 0, eps=0.3)
    for off, n in ((9, 10), (0, 6), (20, 4)):
        sh = _short_run(pkg, batch, n, off, eps=0.3)
        for f in ("posterior_matrix", "tree_statistics", "logdensities"):
            assert np.array_equal(full[f][off:off + n], sh[f]), (off, f)
    # packed groups: 8-aligned shards
    batch = pkg.ProblemBatch(_logistic_batch(pkg, 300, 20, 4, seed=8), 16)
    full = _short_run(pkg, batch, 64, 0)
    for off, n in ((24, 24), (48, 16)):
        sh = _short_run(pkg, batch, n, off)
        for f in ("posterior_matrix", "tree_statistics", "logdensities"):
            assert np.array_equal(full[f][off:off + n], sh[f]), (off, f)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["diag_normal", "logistic_packed"])
def test_chunked_mcmc_from_on_a_batch(pkg, monkeypatch, kind):
    """dhmc_mcmc_from cut into chain chunks (DHMC_E2E_CHUNKS forces the chunking at this size); packed batches cut on
    multiples of 8 chains, so no CTA group straddles a chunk (80 chains in 3 chunks: 0/24/48/80 — chain-granular cuts would
    fall at 26 and 53, inside groups).  Equal to the single-launch call."""
    if kind == "diag_normal":
        batch, B = pkg.ProblemBatch(_diag_batch(pkg, 20, 5, seed=9), 7), 35
    else:
        batch, B = pkg.ProblemBatch(_logistic_batch(pkg, 300, 20, 5, seed=10), 16), 80
    outs = []
    for chunks in ("1", "3"):
        monkeypatch.setenv("DHMC_E2E_CHUNKS", chunks)
        eng = pkg.Engine(batch, chains=B, seed=5)
        eng.random_position(); eng.set_stepsize(0.05)
        q = eng.get_state(("q",))["q"]
        outs.append(eng.mcmc_from(q, 6))
        eng.close()
    for f in ("posterior_matrix", "tree_statistics", "logdensities"):
        assert np.array_equal(outs[0][f], outs[1][f]), f


# --------------------------------------------------------------- GPU: pooled metric
@pytest.mark.gpu
def test_pooled_metric_batch_equals_separate_pooled_handles(pkg):
    stages = (pkg.InitialStepsizeSearch(), pkg.TuningNUTS(22, pkg.DualAveraging()),
              pkg.TuningNUTS(28, pkg.DualAveraging(), pkg.SymmetricPooled), pkg.TuningNUTS(20, pkg.DualAveraging()))
    _batch_equals_separate(pkg, _logistic_batch(pkg, 300, 20, 2, seed=12), K=16, N=6, stages=stages)


# --------------------------------------------------------------- GPU: per-problem diagnostics
@pytest.mark.gpu
def test_per_problem_ess_rhat(pkg):
    import torch
    P, K, D, N = 4, 64, 5, 200
    problems = [pkg.DiagNormal(np.full(D, 10.0 * p), np.ones(D)) for p in range(P)]
    batch = pkg.ProblemBatch(problems, K)
    eng = pkg.Engine(batch, chains=P * K, seed=19)
    eng.random_position(); eng.find_initial_stepsize()
    eng.warmup_stage(pkg.TuningNUTS(150, pkg.DualAveraging()))
    draws = torch.empty((P * K, N, D), dtype=torch.float64, device="cuda")
    eng.mcmc_dev(N, draws.data_ptr(), 0, 0)
    per = eng.ess_rhat_problems_dev(draws.data_ptr(), N, max_lag=40)
    host = draws.cpu().numpy()
    assert per["rhat"].shape == (P, D) and per["ess"].shape == (P, D)
    for p in range(P):
        ref = pkg.diagnostics.ess_rhat(host[p * K:(p + 1) * K], max_lag=40)
        np.testing.assert_allclose(per["rhat"][p], ref["rhat"], rtol=1e-10)
        np.testing.assert_allclose(per["ess"][p], ref["ess"], rtol=1e-7)
    assert np.all(per["rhat"] < 1.01)
    pooled = eng.ess_rhat_dev(draws.data_ptr(), N, max_lag=40)
    assert np.all(pooled["rhat"] > 5)                   # the pooled R̂ mixes problems 10 apart: meaningless for a batch
    eng.close()
    # a shard from the middle of problem 1 to the middle of problem 2: problems 0 and 3 have no local chain
    eng = pkg.Engine(batch, chains=K, seed=19, chain_offset=K + K // 2)
    eng.random_position(); eng.set_stepsize(0.5)
    eng.mcmc_dev(N, draws.data_ptr(), 0, 0)
    per = eng.ess_rhat_problems_dev(draws.data_ptr(), N, max_lag=40)
    host = draws[:K].cpu().numpy()
    assert np.all(np.isnan(per["rhat"][[0, 3]])) and np.all(np.isnan(per["ess"][[0, 3]]))
    for p, sl in ((1, slice(0, K // 2)), (2, slice(K // 2, K))):
        np.testing.assert_allclose(per["rhat"][p], pkg.diagnostics.ess_rhat(host[sl], max_lag=40)["rhat"], rtol=1e-10)
    eng.close()


# --------------------------------------------------------------- GPU: argument errors keep the previous problem
def _run_and_compare(pkg, eng, batch, chains, seed, **kw):
    eng.random_position(); eng.set_stepsize(0.05)
    a = eng.mcmc(4)
    ref = _short_run(pkg, batch, chains, 0, seed=seed, N=4, **kw)
    for f in ("posterior_matrix", "tree_statistics", "logdensities"):
        assert np.array_equal(a[f], ref[f]), f


@pytest.mark.gpu
def test_argument_errors_keep_the_previous_problem(pkg):
    import ctypes as C
    L = pkg._lib
    # DIAG_NORMAL: a wrong block length, and P·K that does not cover the handle's chains — then a run straight away
    batch = pkg.ProblemBatch(_diag_batch(pkg, 10, 3, seed=13), 8)
    eng = pkg.Engine(batch, chains=24, seed=21)
    pr = batch.params()
    with pytest.raises(pkg.ArgumentError, match="mu"):
        eng._ck(eng._lib.dhmc_set_problems(eng._h, L.ptr(pr), C.c_size_t(19), C.c_int64(3), C.c_int64(8)))
    with pytest.raises(pkg.ArgumentError, match="beyond"):
        eng._set_problem(pkg.ProblemBatch(_diag_batch(pkg, 10, 2, seed=14), 8))
    with pytest.raises(pkg.ArgumentError, match="beyond"):
        eng._set_problem(pkg.ProblemBatch(_diag_batch(pkg, 10, 3, seed=14), 7))
    _run_and_compare(pkg, eng, batch, 24, 21)
    eng.close()
    # the pooled metric needs chains_per_problem % 8 == 0: its groups of 8 chains would straddle problems
    eng = pkg.Engine(pkg.ProblemBatch(_diag_batch(pkg, 10, 4, seed=14), 6), chains=24, seed=21)
    eng.random_position(); eng.find_initial_stepsize()
    with pytest.raises(pkg.ArgumentError, match="multiple of 8"):
        eng.warmup_stage(pkg.TuningNUTS(20, pkg.DualAveraging(), pkg.SymmetricPooled))
    eng.close()
    # LOGISTIC packed: unequal N (only reachable through the C ABI: ProblemBatch refuses it) and K % 8 != 0
    problems = _logistic_batch(pkg, 200, 12, 2, seed=15)
    batch = pkg.ProblemBatch(problems, 16)
    eng = pkg.Engine(batch, chains=32, seed=22)
    pr = batch.params().copy()
    pr[batch.block_size] = 199.0                       # problem 1 claims N = 199 with a block of the same length
    with pytest.raises(pkg.ArgumentError, match="same N"):
        eng._ck(eng._lib.dhmc_set_problems(eng._h, L.ptr(pr), C.c_size_t(batch.block_size), C.c_int64(2), C.c_int64(16)))
    with pytest.raises(pkg.ArgumentError, match="threads_per_chain=32"):
        eng._set_problem(pkg.ProblemBatch(_logistic_batch(pkg, 200, 12, 3, seed=16), 12))
    _run_and_compare(pkg, eng, batch, 32, 22)
    eng.close()
    # FUNNEL has no parameters: the C ABI refuses a batch as well
    eng = pkg.Engine(pkg.Funnel(6), chains=8, seed=23)
    blk = np.zeros(4)
    with pytest.raises(pkg.ArgumentError, match="no parameters"):
        eng._ck(eng._lib.dhmc_set_problems(eng._h, L.ptr(blk), C.c_size_t(2), C.c_int64(2), C.c_int64(4)))
    _run_and_compare(pkg, eng, pkg.Funnel(6), 8, 23)
    eng.close()
