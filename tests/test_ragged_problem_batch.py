"""Ragged problem batches (dhmc_set_problems_ragged): P posteriors whose parameter blocks differ in length — logistic
regressions with their own number of observations each — on one handle.  Correctness is that of every batch: chains
[p·K, (p+1)·K) equal, bit for bit, a handle that holds problem p alone with chain_offset = p·K.  The CPU tests check the
host-side validation and the per-problem views of the results."""
import ctypes as C
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODELS = os.path.join(ROOT, "include", "models")
INT_FIELDS = ("depth", "left", "right", "steps", "directions")


def _stages(pkg, M="Diagonal"):
    return pkg.default_warmup_stages(M=getattr(pkg, M), init_steps=20, middle_steps=20, doubling_stages=1,
                                     terminating_steps=20)


def _ragged_logistic(pkg, Ns, p, seed=0):
    return [pkg.LogisticRegression.synthetic(N=n, p=p, seed=seed + 31 * i)[0] for i, n in enumerate(Ns)]


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


def _batch_equals_separate(pkg, problems, K, N, stages, seed=77, engine_opts=None, algorithm=None, packed=False, single=None):
    """Runs the ragged batch, then problem p alone (or single[p], the same posterior as another object) with
    chain_offset = p·K, and compares every chain.  packed: assert that the handle ran packed chain groups — only those
    refuse a chains_per_problem that is not a multiple of 8."""
    batch = pkg.RaggedProblemBatch(problems, K)
    r = pkg.mcmc_keep_warmup(seed, batch, N, warmup_stages=stages, engine_opts=engine_opts, algorithm=algorithm)
    assert len(r["inference"]) == len(problems) * K
    per = pkg.results_by_problem(r["inference"], batch)
    layout = r["engine"].layout()
    if packed:
        with pytest.raises(pkg.ArgumentError, match="threads_per_chain=32"):
            r["engine"]._set_problem(pkg.RaggedProblemBatch(problems, K + 1))
    r["engine"].close()
    for p, ℓ in enumerate(single or problems):
        s = pkg.mcmc_keep_warmup(seed, ℓ, N, chains=K, chain_offset=p * K, warmup_stages=stages, engine_opts=engine_opts,
                                 algorithm=algorithm)
        assert s["engine"].layout() == layout
        s["engine"].close()
        assert len(per[p]) == K
        for k in range(K):
            _assert_same_chain(per[p][k], s["inference"][k])
    return layout


# --------------------------------------------------------------- CPU: host-side validation and views
def test_ragged_problem_batch_validation(pkg):
    rng = np.random.default_rng(0)
    lg = [pkg.LogisticRegression(rng.normal(size=(n, 5)), np.ones(n)) for n in (30, 7, 31)]
    b = pkg.RaggedProblemBatch(lg, 8)
    assert isinstance(b, pkg.ProblemBatch)
    assert (b.family, b.dimension(), b.n_problems, b.chains) == (pkg._lib.FAMILY_LOGISTIC, 5, 3, 24)
    sizes = [1 + n * 5 + n for n in (30, 7, 31)]
    assert b.block_offsets.dtype == np.dtype(C.c_size_t)
    assert b.block_offsets.tolist() == [0, sizes[0], sizes[0] + sizes[1], sum(sizes)]
    assert np.array_equal(b.params(), np.concatenate([x.params() for x in lg]))
    for p in range(3):
        assert np.array_equal(b.params()[b.block_offsets[p]:b.block_offsets[p + 1]], lg[p].params())
    assert [b.problem_chains(p) for p in range(3)] == [(0, 8), (8, 16), (16, 24)]
    # equal N is the general form's special case
    eq = pkg.RaggedProblemBatch(lg[:1] * 2, 4)
    assert eq.block_offsets.tolist() == [0, sizes[0], 2 * sizes[0]]
    assert np.array_equal(eq.params(), pkg.ProblemBatch(lg[:1] * 2, 4).params())
    # ProblemBatch itself keeps refusing unequal N
    with pytest.raises(pkg.ArgumentError, match="same N"):
        pkg.ProblemBatch(lg, 8)
    with pytest.raises(pkg.ArgumentError):
        pkg.RaggedProblemBatch([], 4)
    with pytest.raises(pkg.ArgumentError):
        pkg.RaggedProblemBatch(lg, 0)
    d = _diag_batch(pkg, 5, 2)
    with pytest.raises(pkg.ArgumentError, match="dimension"):
        pkg.RaggedProblemBatch(lg + [pkg.LogisticRegression(rng.normal(size=(9, 6)), np.ones(9))], 8)
    with pytest.raises(pkg.ArgumentError, match="family"):
        pkg.RaggedProblemBatch(lg + d, 8)
    for ℓ in (pkg.StandardNormal(5), pkg.Funnel(5)):
        with pytest.raises(pkg.ArgumentError, match="no parameters"):
            pkg.RaggedProblemBatch([ℓ, ℓ], 4)

    class FakeUser(pkg.api.DeviceLogDensity):        # user models: same library required (no build needed to check it)
        family = pkg._lib.FAMILY_USER

        def __init__(self, lib, pr):
            self.D, self.library_path, self._p = 4, lib, np.asarray(pr, float)

        def params(self):
            return self._p

    u = pkg.RaggedProblemBatch([FakeUser("a.so", [1, 2]), FakeUser("a.so", [3, 4, 5])], 2)
    assert u.library_path == "a.so" and u.block_offsets.tolist() == [0, 2, 5]
    with pytest.raises(pkg.ArgumentError, match="library"):
        pkg.RaggedProblemBatch([FakeUser("a.so", [1, 2]), FakeUser("b.so", [3, 4, 5])], 2)
    with pytest.raises(pkg.ArgumentError, match="non-empty"):
        pkg.RaggedProblemBatch([FakeUser("a.so", [1, 2]), FakeUser("a.so", [])], 2)


def test_ragged_entry_point_refuses_a_null_handle(pkg):
    """Like every entry point: a null handle is an argument error, answered without touching CUDA."""
    lib = pkg._lib.lib()
    pr, off = np.zeros(4), np.array([0, 2, 4], dtype=np.dtype(C.c_size_t))
    assert lib.dhmc_set_problems_ragged(None, pkg._lib.ptr(pr), pkg._lib.ptr(off), C.c_int64(2), C.c_int64(4)) == \
        pkg._lib.DHMC_EARG


def test_results_by_problem_on_a_ragged_batch(pkg):
    P, K, N, D = 3, 4, 5, 3
    B = P * K
    post = np.arange(B * N * D, dtype=float).reshape(B, N, D)
    stats = np.zeros((B, N), dtype=pkg._lib.tree_stats_dtype)
    stats["depth"] = np.arange(B)[:, None]
    logd = np.arange(B * N, dtype=float).reshape(B, N)
    minv = np.arange(B * D, dtype=float).reshape(B, D)
    eps = np.arange(B, dtype=float) / 10
    res = pkg.Results(post, stats, logd, minv, eps)
    rng = np.random.default_rng(1)
    batch = pkg.RaggedProblemBatch([pkg.LogisticRegression(rng.normal(size=(n, D)), np.ones(n)) for n in (4, 40, 9)], K)
    per = pkg.results_by_problem(res, batch)
    assert [len(r) for r in per] == [K] * P
    for p in range(P):
        for k in range(K):
            g = p * K + k
            assert np.array_equal(per[p][k]["posterior_matrix"], post[g].T)
            assert per[p][k]["tree_statistics"]["depth"][0] == g and per[p][k]["ϵ"] == eps[g]
            assert np.array_equal(per[p][k]["κ"].minv, minv[g])
    assert np.shares_memory(per[1]._post, post)                   # zero-copy
    # a shard that starts in the middle of problem 0 and ends in the middle of problem 2
    shard = pkg.Results(post[2:10], stats[2:10], logd[2:10], minv[2:10], eps[2:10])
    per = pkg.results_by_problem(shard, batch, chain_offset=2)
    assert [len(r) for r in per] == [2, 4, 2]
    assert per[0][0]["tree_statistics"]["depth"][0] == 2 and per[2][1]["tree_statistics"]["depth"][0] == 9


# --------------------------------------------------------------- GPU: batch = separate handles, bit for bit
@pytest.mark.gpu
@pytest.mark.parametrize("M", ["Diagonal", "Symmetric"])
@pytest.mark.parametrize("p,Ns", [(20, (1, 31, 32, 33, 64, 300)), (256, (33, 900))])
def test_logistic_packed_ragged_batch_equals_separate_handles(pkg, p, Ns, M):
    """Packed chain groups: the 8 warps of a CTA run one problem, and its tensor-core rounds stream that problem's
    ⌈N_p/32⌉ row blocks — N_p straddles the 32-row block edges."""
    layout = _batch_equals_separate(pkg, _ragged_logistic(pkg, Ns, p, seed=p), K=16, N=8, stages=_stages(pkg, M),
                                    packed=True)
    assert layout[0] == 32                                          # one warp per chain


@pytest.mark.gpu
def test_logistic_one_chain_per_cta_ragged_batch_with_problems_mid_cta(pkg):
    """threads_per_chain=32: one chain per CTA and K = 5, so problems start anywhere; the largest N sits in the middle,
    so a residual scratch strided by anything but the largest N would overlap the next CTA's."""
    _batch_equals_separate(pkg, _ragged_logistic(pkg, (40, 300, 77), 20, seed=5), K=5, N=8, stages=_stages(pkg),
                           engine_opts=dict(threads_per_chain=32))


@pytest.mark.gpu
def test_deep_tree_ragged_batch_equals_separate_handles(pkg):
    """max_depth > 12: the deep kernels read the problem's descriptor through the same load_chain."""
    _batch_equals_separate(pkg, _ragged_logistic(pkg, (30, 90, 55), 8, seed=2), K=4, N=6, stages=_stages(pkg),
                           algorithm=pkg.NUTS(max_depth=15))


def _eight_schools_padded(pkg, P):
    """Eight schools [y(8), σ(8)] per problem, each followed by a different number of zeros: a wrong block offset reads
    another problem's data or the zeros (σ = 0)."""
    rng = np.random.default_rng(8)
    y0 = np.array([28.0, 8, -3, 7, -1, 1, 18, 12])
    s0 = np.array([15.0, 10, 16, 11, 9, 11, 10, 18])
    return [pkg.UserLogDensity(os.path.join(MODELS, "eight_schools.h"), 10,
                               params=np.concatenate([y0 + rng.normal(size=8) * 5, s0 * rng.uniform(0.7, 1.3, 8),
                                                      np.zeros(3 * p + 1)]))
            for p in range(P)]


@pytest.mark.gpu
def test_user_model_ragged_batch_equals_separate_handles(pkg):
    _batch_equals_separate(pkg, _eight_schools_padded(pkg, 3), K=6, N=10, stages=_stages(pkg))


@pytest.mark.gpu
@pytest.mark.parametrize("tpc", [0, 32])
def test_light_kernels_ragged_batch_equal_separate_handles(pkg, tpc):
    """k_eval (set_position), k_leapfrog and k_phase from set positions, momenta and step sizes; tpc = 0 is the packed
    handle (whose light kernels run one chain per CTA with the largest-N scratch stride), 32 one chain per CTA."""
    P, K = 4, 8
    problems = _ragged_logistic(pkg, (300, 17, 64, 129), 20, seed=9)
    D = problems[0].dimension()
    rng = np.random.default_rng(4)
    q, mom = rng.normal(size=(P * K, D)) * 0.3, rng.normal(size=(P * K, D))
    minv, eps = rng.uniform(0.5, 2, (P * K, D)), rng.uniform(0.01, 0.05, P * K)

    def run(ℓ, sl, off):
        eng = pkg.Engine(ℓ, chains=sl.stop - sl.start, seed=3, chain_offset=off, threads_per_chain=tpc)
        eng.set_metric(minv[sl]); eng.set_position(q[sl]); eng.set_momentum(mom[sl]); eng.set_stepsize(eps[sl])
        out = [eng.get_state(("q", "lq", "grad")), eng.phase_logdensity()]
        eng.leapfrog(3, 1)
        out += [eng.get_state(("q", "p", "lq", "grad")), eng.phase_logdensity()]
        eng.close()
        return out

    full = run(pkg.RaggedProblemBatch(problems, K), slice(0, P * K), 0)
    for p in range(P):
        sep = run(problems[p], slice(p * K, (p + 1) * K), p * K)
        for a, b in zip(full, sep):
            if isinstance(a, dict):
                for f in b:
                    assert np.array_equal(a[f][p * K:(p + 1) * K], b[f]), f
            else:
                assert np.array_equal(a[p * K:(p + 1) * K], b)


@pytest.mark.gpu
def test_pooled_metric_ragged_batch_equals_separate_pooled_handles(pkg):
    stages = (pkg.InitialStepsizeSearch(), pkg.TuningNUTS(22, pkg.DualAveraging()),
              pkg.TuningNUTS(28, pkg.DualAveraging(), pkg.SymmetricPooled), pkg.TuningNUTS(20, pkg.DualAveraging()))
    _batch_equals_separate(pkg, _ragged_logistic(pkg, (300, 45), 20, seed=12), K=16, N=6, stages=stages, packed=True)


@pytest.mark.gpu
@pytest.mark.parametrize("tpc", [0, 32])
def test_equal_n_ragged_batch_equals_the_problem_batch(pkg, tpc):
    problems = _ragged_logistic(pkg, (200, 200, 200), 16, seed=3)
    out = []
    for batch in (pkg.ProblemBatch(problems, 8), pkg.RaggedProblemBatch(problems, 8)):
        r = pkg.mcmc_keep_warmup(31, batch, 8, warmup_stages=_stages(pkg), engine_opts=dict(threads_per_chain=tpc))
        r["engine"].close()
        out.append(r["inference"])
    for k in range(len(out[0])):
        _assert_same_chain(out[0][k], out[1][k])


# --------------------------------------------------------------- GPU: against the oracle
@pytest.mark.gpu
def test_ragged_batch_matches_oracle(pkg, po):
    P, K, N, seed, D = 3, 8, 10, 515, 16
    problems = _ragged_logistic(pkg, (70, 200, 33), D, seed=6)
    params = [po.logistic_params(ℓ.X, ℓ.y) for ℓ in problems]
    kw = dict(init_steps=20, middle_steps=20, doubling_stages=1, terminating_steps=20)
    r = pkg.mcmc_keep_warmup(seed, pkg.RaggedProblemBatch(problems, K), N, warmup_stages=pkg.default_warmup_stages(**kw))
    T, _ = r["engine"].layout()
    r["engine"].close()
    ostages = po.default_warmup_stages(**kw)
    for g in (0, 5, 9, 14, 16, 23):
        o = po.mcmc_with_warmup(po.FAMILY_LOGISTIC, D, N, seed, g, stages=ostages, params=params[g // K], T=T, welford=True)
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
def test_ragged_batch_shards_equal_slices_of_the_full_run(pkg):
    problems = _ragged_logistic(pkg, (300, 40, 129, 77), 20, seed=8)
    # packed groups: 8-aligned shards
    batch = pkg.RaggedProblemBatch(problems, 16)
    full = _short_run(pkg, batch, 64, 0)
    for off, n in ((24, 24), (48, 16)):
        sh = _short_run(pkg, batch, n, off)
        for f in ("posterior_matrix", "tree_statistics", "logdensities"):
            assert np.array_equal(full[f][off:off + n], sh[f]), (off, f)
    # one chain per CTA: shards that start in the middle of a problem
    batch = pkg.RaggedProblemBatch(problems, 6)
    full = _short_run(pkg, batch, 24, 0, threads_per_chain=32)
    for off, n in ((9, 10), (3, 6), (20, 4)):
        sh = _short_run(pkg, batch, n, off, threads_per_chain=32)
        for f in ("posterior_matrix", "tree_statistics", "logdensities"):
            assert np.array_equal(full[f][off:off + n], sh[f]), (off, f)


@pytest.mark.gpu
def test_chunked_mcmc_from_on_a_ragged_packed_batch(pkg, monkeypatch):
    """dhmc_mcmc_from cut into 3 chain chunks (DHMC_E2E_CHUNKS) on multiples of 8 chains equals the single launch."""
    batch, B = pkg.RaggedProblemBatch(_ragged_logistic(pkg, (300, 20, 77, 160, 33), 20, seed=10), 16), 80
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


# --------------------------------------------------------------- GPU: per-problem diagnostics
@pytest.mark.gpu
def test_per_problem_ess_rhat_on_a_ragged_batch(pkg):
    import torch
    P, K, D, N = 3, 32, 6, 200
    batch = pkg.RaggedProblemBatch(_ragged_logistic(pkg, (50, 400, 120), D, seed=17), K)
    eng = pkg.Engine(batch, chains=P * K, seed=19)
    eng.random_position(); eng.find_initial_stepsize()
    eng.warmup_stage(pkg.TuningNUTS(150, pkg.DualAveraging()))
    draws = torch.empty((P * K, N, D), dtype=torch.float64, device="cuda")
    eng.mcmc_dev(N, draws.data_ptr(), 0, 0)
    per = eng.ess_rhat_problems_dev(draws.data_ptr(), N, max_lag=40)
    host = draws.cpu().numpy()
    eng.close()
    assert per["rhat"].shape == (P, D) and per["ess"].shape == (P, D)
    for p in range(P):
        ref = pkg.diagnostics.ess_rhat(host[p * K:(p + 1) * K], max_lag=40)
        np.testing.assert_allclose(per["rhat"][p], ref["rhat"], rtol=1e-10)
        np.testing.assert_allclose(per["ess"][p], ref["ess"], rtol=1e-7)


# --------------------------------------------------------------- GPU: argument errors keep the previous problem
def _run_and_compare(pkg, eng, batch, chains, seed, **kw):
    eng.random_position(); eng.set_stepsize(0.05)
    a = eng.mcmc(4)
    ref = _short_run(pkg, batch, chains, 0, seed=seed, N=4, **kw)
    for f in ("posterior_matrix", "tree_statistics", "logdensities"):
        assert np.array_equal(a[f], ref[f]), f


@pytest.mark.gpu
def test_ragged_argument_errors_keep_the_previous_problem(pkg):
    L = pkg._lib
    batch = pkg.RaggedProblemBatch(_ragged_logistic(pkg, (120, 200), 12, seed=15), 16)
    eng = pkg.Engine(batch, chains=32, seed=22)
    pr, off = batch.params(), batch.block_offsets

    def call(params, offsets):
        eng._ck(eng._lib.dhmc_set_problems_ragged(eng._h, L.ptr(params), L.ptr(offsets), C.c_int64(2), C.c_int64(16)))

    bad = off.copy(); bad[0] = 1
    with pytest.raises(pkg.ArgumentError, match=r"block_offsets\[0\]"):
        call(pr, bad)
    bad = off.copy(); bad[1] = 0
    with pytest.raises(pkg.ArgumentError, match="strictly increase"):
        call(pr, bad)
    bad = off.copy(); bad[2] -= 1                     # the offsets end before the array does
    with pytest.raises(pkg.ArgumentError, match="disagrees with its N"):
        call(pr, bad)
    p2 = pr.copy(); p2[off[1]] = 199.0                # problem 1 claims N = 199 with a block of 200 rows
    with pytest.raises(pkg.ArgumentError, match="disagrees with its N"):
        call(p2, off)
    p2 = pr.copy(); p2[off[1]] = 200.5
    with pytest.raises(pkg.ArgumentError, match="integer"):
        call(p2, off)
    p2 = pr.copy(); p2[off[2] - 1] = 1.5              # the last y of problem 1
    with pytest.raises(pkg.ArgumentError, match="0 <= y <= 1"):
        call(p2, off)
    with pytest.raises(pkg.ArgumentError, match="threads_per_chain=32"):
        eng._set_problem(pkg.RaggedProblemBatch(_ragged_logistic(pkg, (50, 70, 90), 12, seed=16), 12))
    _run_and_compare(pkg, eng, batch, 32, 22)
    eng.close()
    # FUNNEL has no parameters: the ragged entry point refuses a batch as well
    eng = pkg.Engine(pkg.Funnel(6), chains=8, seed=23)
    blk, offs = np.zeros(4), np.array([0, 2, 4], dtype=np.dtype(C.c_size_t))
    with pytest.raises(pkg.ArgumentError, match="no parameters"):
        eng._ck(eng._lib.dhmc_set_problems_ragged(eng._h, L.ptr(blk), L.ptr(offs), C.c_int64(2), C.c_int64(4)))
    _run_and_compare(pkg, eng, pkg.Funnel(6), 8, 23)
    eng.close()
