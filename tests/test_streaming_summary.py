"""Streaming posterior summary: sampling that folds its kept draws into per-(problem, parameter) statistics on the device
(dhmc_mcmc_summary, include/dhmc.h; DESIGN.md §4.4) instead of returning them.

CPU: the numpy mirror (diagnostics.summary_from_draws / merge_summaries / finish_summary) against the definitions evaluated
in exact rational arithmetic; the C record merge and finish against the mirror; the argument checks.
GPU: for every k_nuts flavour a summary call changes nothing about sampling (bit-identical state, statistics and transition
count to mcmc from the same checkpoint) and equals the mirror on the draws mcmc returned; R̂ equals
dhmc_ess_rhat_problems_dev; shards merge into the one-handle summary; SBC ranks of a 1 024-problem batch are uniform; a
chain that halts is left out."""
import math
import os
import zlib
from fractions import Fraction

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROSENBROCK = os.path.join(ROOT, "include", "models", "rosenbrock.h")
STATS = ("mean", "sd", "mcse", "ess", "rhat")
# Rounding bound of a float64 summary against the exact one, relative to the statistic (the mean: to |mean| + sd).  The sums
# run over at most a few thousand terms, each with relative error ≤ 2⁻⁵³; the device adds its terms in atomic order.
RTOL = 1e-9


# ------------------------------------------------------------------ exact reference, from the definitions in include/dhmc.h
def _exact(draws, cpp, thin, ref, off, P, completed=None):
    x = np.asarray(draws, float)[:, thin - 1::thin]
    K, nk, D = x.shape
    n = nk // 2
    prob = (off + np.arange(K)) // cpp if cpp else np.zeros(K, int)
    ok = np.ones(K, bool) if completed is None else np.asarray(completed, bool)
    out = {k: np.full((P, D), np.nan) for k in STATS}
    out["rank"] = np.full((P, D), 0 if ref is not None else -1, np.int64)
    out["draws"] = np.zeros((P, D), np.int64)
    for p in range(P):
        idx = [k for k in range(K) if prob[k] == p and ok[k]]
        M = len(idx)
        out["draws"][p] = nk * M
        if ref is not None:
            out["rank"][p] = [sum(int(x[k, j, d] < ref[p, d]) for k in idx for j in range(nk)) for d in range(D)]
        if M == 0:
            continue
        for d in range(D):
            seqs = [[Fraction(float(v)) for v in x[k, h * n:(h + 1) * n, d]] for k in idx for h in (0, 1)]
            m = len(seqs)
            mu_s = [sum(s) / n for s in seqs]
            allx = [v for s in seqs for v in s]
            mean = sum(allx) / len(allx)
            var = sum((v - mean) ** 2 for v in allx) / (len(allx) - 1)
            W = sum(sum((v - mu) ** 2 for v in s) / (n - 1) for s, mu in zip(seqs, mu_s)) / m
            mbar = sum(mu_s) / m
            var_plus = Fraction(n - 1, n) * W + sum((mu - mbar) ** 2 for mu in mu_s) / (m - 1)
            out["mean"][p, d] = float(mean)
            out["sd"][p, d] = math.sqrt(var)
            out["rhat"][p, d] = math.sqrt(var_plus / W) if W > 0 else np.nan
            if M >= 2:
                mu_c = [(mu_s[2 * i] + mu_s[2 * i + 1]) / 2 for i in range(M)]
                var_c = sum((mu - mbar) ** 2 for mu in mu_c) / (M - 1) / M
                out["mcse"][p, d] = math.sqrt(var_c)
                if var_plus > 0:
                    out["ess"][p, d] = float(var / var_c) if var_c > 0 else np.inf
    return out


def _close(got, want, ctx=""):
    """float statistics within RTOL (NaN where NaN), ranks and draw counts exactly"""
    for k in ("rank", "draws"):
        assert np.array_equal(got[k], want[k]), (ctx, k, got[k], want[k])
    for k in STATS:
        g, w = np.asarray(got[k], float), np.asarray(want[k], float)
        assert np.array_equal(np.isnan(g), np.isnan(w)), (ctx, k, g, w)
        scale = np.abs(w) + (np.nan_to_num(np.asarray(want["sd"], float)) if k == "mean" else 0.0)
        ok = np.isnan(w) | (g == w) | (np.abs(g - w) <= RTOL * scale)
        assert np.all(ok), (ctx, k, g[~ok], w[~ok])


def _synthetic(rng, K, N, D, offset=0.0, spread=1.0):
    x = offset + spread * rng.normal(size=(K, N, D))
    return x + 0.3 * spread * rng.normal(size=(K, 1, D))          # chain-level offsets: R̂ > 1, finite batch-means ESS


EDGE_CASES = {
    # name: (K, N, D, thin, chains_per_problem, chain_offset, P, offset, spread)
    "odd_n_keep": (6, 9, 3, 1, 0, 0, 1, 0.0, 1.0),
    "thin_3": (5, 30, 4, 3, 0, 0, 1, 0.0, 1.0),
    "n_keep_4": (4, 4, 2, 1, 0, 0, 1, 0.0, 1.0),
    "d_33": (3, 10, 33, 2, 0, 0, 1, 0.0, 1.0),
    "large_offset": (4, 12, 3, 1, 0, 0, 1, 1e8, 1e-3),
    "one_chain_per_problem": (5, 8, 2, 1, 1, 0, 5, 0.0, 1.0),
    "shard_inside_a_problem": (7, 10, 3, 2, 3, 4, 6, 0.0, 1.0),   # global chains 4…10 of problems of 3: problem 1 from its
}                                                                    # middle, problems 0, 4, 5 without a local chain


@pytest.mark.parametrize("case", list(EDGE_CASES))
def test_mirror_matches_exact_definitions(pkg, case):
    K, N, D, thin, cpp, off, P, offset, spread = EDGE_CASES[case]
    rng = np.random.default_rng(zlib.crc32(case.encode()))
    x = _synthetic(rng, K, N, D, offset, spread)
    ref = offset + spread * rng.normal(size=(P, D))
    rec = pkg.diagnostics.summary_from_draws(x, cpp, thin, ref, off, n_problems=P)
    _close(pkg.diagnostics.finish_summary(rec), _exact(x, cpp, thin, ref, off, P), case)
    rec = pkg.diagnostics.summary_from_draws(x, cpp, thin, None, off, n_problems=P)
    got = pkg.diagnostics.finish_summary(rec)
    assert np.all(got["rank"] == -1)


def test_constant_parameter_and_one_chain(pkg):
    """a parameter constant at one value has var⁺ = 0: R̂ and ESS are NaN, sd and mcse 0; one chain: mcse and ESS NaN"""
    d = pkg.diagnostics
    rng = np.random.default_rng(3)
    x = rng.normal(size=(4, 10, 3))
    x[:, :, 1] = 2.5
    out = d.finish_summary(d.summary_from_draws(x))
    assert np.isnan(out["rhat"][0, 1]) and np.isnan(out["ess"][0, 1])
    assert out["sd"][0, 1] == 0 and out["mcse"][0, 1] == 0 and out["mean"][0, 1] == 2.5
    assert np.all(np.isfinite(out["rhat"][0, [0, 2]])) and np.all(np.isfinite(out["ess"][0, [0, 2]]))
    one = d.finish_summary(d.summary_from_draws(x[:1]))
    assert np.all(np.isnan(one["mcse"])) and np.all(np.isnan(one["ess"])) and np.all(np.isfinite(one["sd"][0, [0, 2]]))


def test_left_out_chains_and_empty_problems(pkg):
    rng = np.random.default_rng(4)
    x = _synthetic(rng, 8, 10, 2)
    done = np.array([1, 1, 0, 1, 0, 0, 1, 1], bool)               # problem 1 (chains 2, 3) keeps one chain, problem 2 none
    ref = rng.normal(size=(4, 2))
    rec = pkg.diagnostics.summary_from_draws(x, 2, 1, ref, 0, completed=done)
    out = pkg.diagnostics.finish_summary(rec)
    _close(out, _exact(x, 2, 1, ref, 0, 4, completed=done))
    assert np.all(np.isnan(out["mean"][2])) and np.all(out["rank"][2] == 0) and np.all(out["draws"][2] == 0)
    assert np.all(out["draws"][1] == 10) and np.all(np.isnan(out["mcse"][1]))


def _records_of_split(pkg, x, cpp, thin, ref, P, cuts):
    bounds = [0, *cuts, x.shape[0]]
    return [pkg.diagnostics.summary_from_draws(x[a:b], cpp, thin, ref, a, n_problems=P) for a, b in zip(bounds, bounds[1:])]


@pytest.mark.parametrize("cuts", [(5,), (1, 2, 9), (3, 6, 7, 10), (4,)], ids=lambda c: "-".join(map(str, c)))
def test_merge_of_any_split_equals_the_whole(pkg, cuts):
    """shards cut anywhere, inside problems too, merge (numpy and C) into the record of all chains"""
    rng = np.random.default_rng(sum(cuts))
    K, N, D, cpp, P = 12, 16, 5, 3, 4
    x = _synthetic(rng, K, N, D, offset=50.0)
    ref = 50.0 + rng.normal(size=(P, D))
    whole = pkg.diagnostics.summary_from_draws(x, cpp, 2, ref, 0, n_problems=P)
    parts = _records_of_split(pkg, x, cpp, 2, ref, P, cuts)
    merged = pkg.diagnostics.merge_summaries(*parts)
    L = pkg._lib
    exact_fields = (L.SUMMARY_CHAINS, L.SUMMARY_NKEEP, L.SUMMARY_BELOW)
    assert np.array_equal(merged[..., exact_fields], whole[..., exact_fields])
    assert np.allclose(merged, whole, rtol=1e-12, atol=1e-12 * np.abs(whole).max())
    _close(pkg.diagnostics.finish_summary(merged), pkg.diagnostics.finish_summary(whole))
    lib = L.lib()
    acc = np.ascontiguousarray(parts[0])
    for r in parts[1:]:
        assert lib.dhmc_summary_merge(L.ptr(acc), L.ptr(np.ascontiguousarray(r)), D, P) == 0
    assert np.array_equal(acc[..., exact_fields], whole[..., exact_fields])
    assert np.allclose(acc, merged, rtol=1e-13, atol=1e-13 * np.abs(whole).max())


def _c_finish(pkg, rec):
    L = pkg._lib
    P, D = rec.shape[:2]
    out = {k: np.empty((P, D)) for k in STATS}
    out.update(rank=np.empty((P, D), np.int64), draws=np.empty((P, D), np.int64))
    rc = L.lib().dhmc_summary_finish(L.ptr(np.ascontiguousarray(rec)), D, P, *(L.ptr(out[k]) for k in (*STATS, "rank", "draws")))
    assert rc == 0
    return out


@pytest.mark.parametrize("case", ["odd_n_keep", "large_offset", "one_chain_per_problem", "shard_inside_a_problem"])
def test_c_finish_matches_mirror(pkg, case):
    K, N, D, thin, cpp, off, P, offset, spread = EDGE_CASES[case]
    rng = np.random.default_rng(7)
    x = _synthetic(rng, K, N, D, offset, spread)
    for ref in (offset + spread * rng.normal(size=(P, D)), None):
        rec = pkg.diagnostics.summary_from_draws(x, cpp, thin, ref, off, n_problems=P)
        _close(_c_finish(pkg, rec), pkg.diagnostics.finish_summary(rec), case)


def test_argument_checks_without_gpu(pkg):
    L = pkg._lib
    lib = L.lib()
    rec = np.zeros((2, 3, L.SUMMARY_FIELDS))
    other = rec.copy()
    rec[..., L.SUMMARY_CHAINS], rec[..., L.SUMMARY_NKEEP] = 2, 10
    other[..., L.SUMMARY_CHAINS], other[..., L.SUMMARY_NKEEP] = 1, 12
    before = rec.copy()
    assert lib.dhmc_summary_merge(L.ptr(rec), L.ptr(other), 3, 2) == L.DHMC_EARG        # different n_keep
    assert np.array_equal(rec, before)                                                  # nothing written
    assert lib.dhmc_summary_merge(None, L.ptr(other), 3, 2) == L.DHMC_EARG
    assert lib.dhmc_summary_finish(None, 3, 2, *([None] * 7)) == L.DHMC_EARG
    assert lib.dhmc_summary_finish(L.ptr(rec), 0, 2, *([None] * 7)) == L.DHMC_EARG
    assert lib.dhmc_mcmc_summary(None, 10, 1, None, L.ptr(rec), None, None) == L.DHMC_EARG
    with pytest.raises(pkg.ArgumentError):
        pkg.diagnostics.merge_summaries(rec, other)
    # the Python checks run before the library is called (an Engine shell without a handle)
    eng = object.__new__(pkg.Engine)
    eng.K, eng.D, eng.ℓ, eng._h, eng._lib = 4, 3, pkg.StandardNormal(3), None, lib
    for kw in (dict(N=10, thin=0), dict(N=10, thin=3), dict(N=3), dict(N=0), dict(N=12, thin=4),
               dict(N=10, reference=np.zeros((3, 1))), dict(N=10, reference=np.zeros((2, 3)))):
        with pytest.raises(pkg.ArgumentError):
            eng.mcmc_summary(**kw)
    with pytest.raises(pkg.ArgumentError):
        pkg.diagnostics.summary_from_draws(np.zeros((2, 6, 3)), thin=2)                  # 3 kept draws
    with pytest.raises(pkg.ArgumentError):
        pkg.diagnostics.summary_from_draws(np.zeros((2, 8, 3)), 2, 1, np.zeros((3, 2)))  # reference of the wrong width


# ------------------------------------------------------------------ GPU
def _same_bits(a, b):
    return np.asarray(a).tobytes() == np.asarray(b).tobytes()


def _drop_in(pkg, eng, N, thin=1, reference=None, cpp=0, P=1, ctx=""):
    """mcmc from a checkpoint, then mcmc_summary from the same checkpoint: same final state, statistics and transition
    count bit for bit; the summary equals the mirror on mcmc's draws.  Returns the summary."""
    ck = eng.checkpoint()
    t0 = eng.transition_count
    run = eng.mcmc(N)
    s1, t1 = eng.get_state(("q", "lq", "grad", "eps")), eng.transition_count
    eng.restore(ck)
    summ = eng.mcmc_summary(N, thin=thin, reference=reference, stats=True)
    s2, t2 = eng.get_state(("q", "lq", "grad", "eps")), eng.transition_count
    assert t1 == t2 == t0 + N, ctx
    for f in s1:
        assert _same_bits(s1[f], s2[f]), (ctx, f)
    assert _same_bits(run["tree_statistics"][:, thin - 1::thin], summ["tree_statistics"]), ctx
    assert _same_bits(run["logdensities"][:, thin - 1::thin], summ["logdensities"]), ctx
    rec = pkg.diagnostics.summary_from_draws(run["posterior_matrix"], cpp, thin, reference, 0, n_problems=P)
    _close(summ, pkg.diagnostics.finish_summary(rec), ctx)
    assert summ["record"].shape == (P, eng.D, pkg._lib.SUMMARY_FIELDS)
    return summ


def _engine(pkg, ℓ, K, eps, seed=31, **kw):
    eng = pkg.Engine(ℓ, chains=K, seed=seed, **kw)
    eng.random_position()
    eng.set_stepsize(eps)
    return eng


@pytest.mark.gpu
def test_drop_in_std_normal_dim_1000(pkg):
    """the one-chain-per-CTA kernels with the fused all-reduce (the C2 layout), one problem"""
    eng = _engine(pkg, pkg.StandardNormal(1000), 384, 0.05)
    try:
        _drop_in(pkg, eng, 8, ctx="std1000")
    finally:
        eng.close()


def _diag_batch(pkg, P, D, K, seed=5):
    rng = np.random.default_rng(seed)
    return pkg.ProblemBatch([pkg.DiagNormal(rng.normal(size=D), rng.uniform(0.5, 2.0, D)) for _ in range(P)], K)


@pytest.mark.gpu
def test_drop_in_diag_batch_thinned_with_reference(pkg):
    batch = _diag_batch(pkg, 12, 6, 4)
    ref = np.random.default_rng(1).normal(size=(12, 6))
    eng = _engine(pkg, batch, batch.chains, 0.4)
    try:
        s = _drop_in(pkg, eng, 60, thin=10, reference=ref, cpp=4, P=12, ctx="diag-batch")
        assert np.all(s["draws"] == 6 * 4) and np.all((s["rank"] >= 0) & (s["rank"] <= 24))
    finally:
        eng.close()


def _logistic(pkg, rng, N, p):
    X = rng.normal(size=(N, p)) / np.sqrt(p)
    return pkg.LogisticRegression(X, (rng.uniform(size=N) < 0.5).astype(float))


@pytest.mark.gpu
@pytest.mark.parametrize("ragged", [False, True], ids=["batch", "ragged"])
def test_drop_in_packed_logistic(pkg, ragged):
    """packed groups of 8 chains per CTA (one warp per chain, tensor-core likelihood)"""
    rng = np.random.default_rng(9)
    probs = [_logistic(pkg, rng, int(rng.integers(20, 90)) if ragged else 50, 24) for _ in range(4)]
    batch = (pkg.RaggedProblemBatch if ragged else pkg.ProblemBatch)(probs, 8)
    ref = rng.normal(size=(4, 24))
    eng = _engine(pkg, batch, batch.chains, 0.1)
    try:
        _drop_in(pkg, eng, 10, thin=2, reference=ref, cpp=8, P=4, ctx="logistic")
    finally:
        eng.close()


@pytest.mark.gpu
def test_drop_in_deep_twin(pkg):
    eng = _engine(pkg, pkg.StandardNormal(40), 64, 0.02, algorithm=pkg.NUTS(max_depth=14))
    try:
        _drop_in(pkg, eng, 6, ctx="deep")
    finally:
        eng.close()


@pytest.mark.gpu
def test_drop_in_symmetric_metric(pkg):
    D = 12
    rng = np.random.default_rng(2)
    A = rng.normal(size=(D, D)) / np.sqrt(D)
    eng = _engine(pkg, pkg.DiagNormal(rng.normal(size=D), rng.uniform(0.5, 2.0, D)), 96, 0.3)
    try:
        eng.set_metric_dense(A @ A.T + np.eye(D))
        assert eng.metric_is_dense()
        _drop_in(pkg, eng, 9, reference=rng.normal(size=(1, D)), ctx="dense")
    finally:
        eng.close()


@pytest.mark.gpu
def test_drop_in_user_model(pkg):
    ℓ = pkg.UserLogDensity(ROSENBROCK, 6, params=[1.0, 0.5], deep=True)   # __graft_entry__.build() compiles it
    eng = _engine(pkg, ℓ, 64, 0.02)
    try:
        _drop_in(pkg, eng, 8, ctx="rosenbrock")
    finally:
        eng.close()


@pytest.mark.gpu
def test_rhat_equals_ess_rhat_problems_dev(pkg):
    import torch
    batch = _diag_batch(pkg, 10, 5, 6, seed=8)
    N = 40
    eng = _engine(pkg, batch, batch.chains, 0.5)
    try:
        ck = eng.checkpoint()
        buf = torch.empty((batch.chains, N, 5), dtype=torch.float64, device="cuda")
        eng.mcmc_dev(N, buf.data_ptr())
        torch.cuda.synchronize()
        want = eng.ess_rhat_problems_dev(buf.data_ptr(), N)["rhat"]
        eng.restore(ck)
        got = eng.mcmc_summary(N)["rhat"]
    finally:
        eng.close()
    assert np.all(np.isfinite(want)) and np.allclose(got, want, rtol=RTOL, atol=0)


@pytest.mark.gpu
def test_shards_merge_into_the_one_handle_summary(pkg):
    """two handles on one GPU split a batch at a chain offset inside a problem; the merged records give the one-handle
    summary"""
    batch = _diag_batch(pkg, 6, 7, 4, seed=12)
    ref = np.random.default_rng(3).normal(size=(6, 7))
    N, thin, cut = 24, 2, 10                                      # chains 8, 9 | 10, 11 of problem 2
    outs = []
    for off, K in ((0, batch.chains), (0, cut), (cut, batch.chains - cut)):
        eng = _engine(pkg, batch, K, 0.45, chain_offset=off)
        try:
            outs.append(eng.mcmc_summary(N, thin=thin, reference=ref))
        finally:
            eng.close()
    whole, a, b = outs
    L = pkg._lib
    rec = a["record"].copy()
    assert L.lib().dhmc_summary_merge(L.ptr(rec), L.ptr(b["record"]), 7, 6) == 0
    merged = pkg.diagnostics.finish_summary(rec)
    _close(merged, whole, "shards")
    _close(pkg.diagnostics.finish_summary(pkg.diagnostics.merge_summaries(a["record"], b["record"])), whole, "shards-numpy")
    assert np.array_equal(a["draws"][2] + b["draws"][2], whole["draws"][2]) and np.all(a["draws"][3:] == 0)


def _rank_histogram(rank, draws, bins):
    """counts of ranks 0 … draws in `bins` groups of consecutive values, and the counts a uniform rank expects (the groups
    hold ⌊(draws + 1)/bins⌋ or one more values)"""
    values = np.bincount(np.arange(draws + 1) * bins // (draws + 1), minlength=bins)
    hist = np.bincount(np.ravel(rank) * bins // (draws + 1), minlength=bins)
    return hist, values / (draws + 1) * hist.sum()


@pytest.mark.gpu
def test_sbc_ranks_are_uniform(pkg):
    """simulation-based calibration end to end: 1 024 Gaussian posteriors, each reference drawn from its own posterior, so
    every rank is uniform on {0, …, draws}"""
    from scipy import stats
    P, D, K = 1024, 4, 4
    rng = np.random.default_rng(20261017)
    mu, s2 = rng.normal(size=(P, D)), rng.uniform(0.3, 3.0, size=(P, D))
    batch = pkg.ProblemBatch([pkg.DiagNormal(mu[p], s2[p]) for p in range(P)], K)
    ref = mu + np.sqrt(s2) * rng.normal(size=(P, D))
    out = pkg.summarize_with_warmup(77, batch, 400, thin=10, reference=ref)
    assert np.all(out["draws"] == 40 * K)
    hist, expected = _rank_histogram(out["rank"], 40 * K, 16)
    p_value = stats.chisquare(hist, expected).pvalue
    assert p_value > 1e-4, (hist, p_value)
    assert np.all(np.isfinite(out["rhat"])) and np.median(np.abs(out["rhat"] - 1)) < 0.05


@pytest.mark.gpu
def test_argument_checks_before_launch(pkg):
    eng = _engine(pkg, pkg.StandardNormal(3), 8, 0.5)
    try:
        L = pkg._lib
        rec = np.zeros((1, 3, L.SUMMARY_FIELDS))
        t0, n0 = eng.transition_count, eng.kernel_launches()
        for N, thin, r in ((10, 0, rec), (10, 3, rec), (3, 1, rec), (0, 1, rec), (12, 4, rec), (10, 1, None)):
            assert eng._lib.dhmc_mcmc_summary(eng._h, N, thin, None, L.ptr(r), None, None) == L.DHMC_EARG, (N, thin)
        assert eng.transition_count == t0 and eng.kernel_launches() == n0
    finally:
        eng.close()


@pytest.mark.gpu
def test_halted_chain_is_left_out(pkg):
    """min_Δ = −Inf: chain 3's first leaf lands where q² overflows, is not divergent, and the next leapfrog would start
    from ℓ = −∞ (hamiltonian.jl:276): the chain stops with DHMC_CHAIN_LEAPFROG_NONFINITE.  The summary call raises the
    ArgumentError mcmc raises, reports the same status words, and leaves the chain out of its problem's statistics."""
    K, D, N = 16, 4, 8
    rng = np.random.default_rng(90)
    q = rng.normal(size=(K, D))
    q[3] = [1.5e153, 0, 0, 0]
    eps = np.full(K, 0.4)
    eps[3] = 5.0
    eng = pkg.Engine(pkg.DiagNormal(np.zeros(D), np.ones(D)), chains=K, seed=5, algorithm=pkg.NUTS(min_Δ=-np.inf))
    try:
        eng.set_position(q)
        eng.set_stepsize(eps)
        ck = eng.checkpoint()
        L = pkg._lib
        post, st, ld = np.empty((K, N, D)), np.zeros((K, N), dtype=L.tree_stats_dtype), np.empty((K, N))
        rc = eng._lib.dhmc_mcmc(eng._h, N, L.ptr(post), L.ptr(st), L.ptr(ld))
        status = eng.chain_status()
        msg = eng._lib.dhmc_last_error(eng._h).decode()
        assert rc == L.DHMC_ENUMERIC and status[3] == L.DHMC_CHAIN_LEAPFROG_NONFINITE and np.all(np.delete(status, 3) == 0)
        eng.restore(ck)
        with pytest.raises(pkg.ArgumentError, match="leapfrog called from non-finite log density") as e:
            eng.mcmc_summary(N, reference=np.zeros((1, D)))
        assert eng._lib.dhmc_last_error(eng._h).decode() == msg
        assert np.array_equal(e.value.debug_information["chain_status"], status)
        summ = e.value.debug_information["summary"]
        assert np.all(summ["record"][..., L.SUMMARY_CHAINS] == K - 1) and np.all(summ["draws"] == N * (K - 1))
        rec = pkg.diagnostics.summary_from_draws(post, 0, 1, np.zeros((1, D)), completed=status == 0)
        _close(summ, pkg.diagnostics.finish_summary(rec), "halted")
    finally:
        eng.close()
