"""Streaming quantiles: per-(problem, parameter) histograms of the kept draws on a grid the caller fixes, folded on the device
by the streaming summary (dhmc_mcmc_summary_histogram, include/dhmc.h; DESIGN.md §4.4), and the bracketed type-7 quantiles
read from them (dhmc_histogram_quantiles).

CPU: the numpy mirror's bin rule (diagnostics.histogram_from_draws) against the rule evaluated in plain Python on edge
values; diagnostics.histogram_quantiles brackets np.quantile on ties, single bins, tails, α = 0 and 1; the C quantiles equal
the mirror bit for bit, and at the grid (0, 1, 4096) the placement dhmc_acceptance_quantiles_dev used before it shared the
helper; argument checks; quantile_grid's placeholders; histograms of shards add up.
GPU: for every k_nuts flavour the histogram call is a drop-in for mcmc (bit-identical state, statistics and transition
count) whose counts equal the mirror on mcmc's draws as integers; a chain that halts after keeping draws is left out while
its chain group is reused; shards on one grid add up; end to end on 64 Gaussian posteriors with the pilot grid; argument
checks before launch."""
import math
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROSENBROCK = os.path.join(ROOT, "include", "models", "rosenbrock.h")
WALL = os.path.join(ROOT, "include", "models", "walled_normal.h")
STATS = ("mean", "sd", "mcse", "ess", "rhat")
RTOL = 1e-9            # the record against the mirror, as tests/test_streaming_summary.py
PROBS = (0.0, 0.05, 0.25, 0.5, 0.75, 0.95, 1.0)


def _slack(lo, hi):
    """the rounding of the edges the bracket guarantee allows: a few ulps of max(|lo|, |hi|)"""
    return 4 * np.spacing(np.maximum(np.abs(lo), np.abs(hi)))


def _plain_bin(theta, lo, hi, nbins):
    """the bin rule of include/dhmc.h in plain Python floats"""
    inv_w = nbins / (hi - lo)
    t = (theta - lo) * inv_w
    if t < 0:
        return 0
    if not t < nbins:
        return nbins + 1
    return 1 + int(t)


def _counts_of(pkg, x, lo, hi, bins):
    """counts [1, 1, bins + 2] of the values x (one chain, one parameter)"""
    x = np.asarray(x, float)
    return pkg.diagnostics.histogram_from_draws(x.reshape(1, -1, 1), [[lo]], [[hi]], bins)


# ------------------------------------------------------------------ CPU: the mirror
GRIDS = {"seven_bins": (-1.0, 2.0, 7), "one_bin": (-0.5, 0.25, 1), "narrow": (1.0, 1.0 + 2.0 ** -40, 64),
         "wide": (-1e300, 1e300, 4096), "offset": (1e8, 1e8 + 3.0, 256)}


@pytest.mark.parametrize("grid", list(GRIDS))
def test_bin_rule_matches_plain_python(pkg, grid):
    lo, hi, nb = GRIDS[grid]
    w = (hi - lo) / nb
    edges = [lo + k * w for k in range(nb)] + [hi]
    vals = [lo, hi, np.nextafter(hi, -np.inf), np.nextafter(lo, -np.inf), np.nextafter(lo, np.inf), np.inf, -np.inf,
            np.nan, 0.5 * (lo + hi), lo - 1e3 * w, hi + 1e3 * w]
    vals += edges[:64] + [np.nextafter(e, -np.inf) for e in edges[:64]]
    vals += list(np.random.default_rng(nb).uniform(lo - w, hi + w, 200))
    got = _counts_of(pkg, vals, lo, hi, nb)[0, 0]
    want = np.bincount([_plain_bin(float(v), lo, hi, nb) for v in vals], minlength=nb + 2)
    assert np.array_equal(got, want), grid
    assert got[0] >= 3 and got[-1] >= 4                      # below lo (−∞ too), at or above hi (+∞ and NaN too)


def _samples():
    rng = np.random.default_rng(11)
    return {
        "ties": (np.repeat([0.1, 0.3, 0.3, 0.7, 0.9], 9), 0.0, 1.0, 16),
        "one_bin": (0.51 + 0.001 * rng.uniform(size=40), 0.0, 1.0, 8),
        "both_tails": (rng.normal(size=500), -1.0, 1.0, 32),
        "normal": (rng.normal(size=2000), -6.0, 6.0, 256),
        "constant": (np.full(12, 2.0), 1.0, 3.0, 4),
        "on_edges": (np.linspace(-1.0, 0.75, 8), -1.0, 1.0, 8),
    }


@pytest.mark.parametrize("case", list(_samples()))
def test_quantiles_bracket_the_exact_quantile(pkg, case):
    x, lo, hi, nb = _samples()[case]
    counts = _counts_of(pkg, x, lo, hi, nb)
    q, q_lo, q_hi = (a[0, 0] for a in pkg.diagnostics.histogram_quantiles(counts, [[lo]], [[hi]], PROBS))
    s = _slack(lo, hi)
    tails = 0
    for i, a in enumerate(PROBS):
        exact = np.quantile(x, a, method="linear")
        assert q_lo[i] - s <= exact <= q_hi[i] + s, (case, a, q_lo[i], exact, q_hi[i])
        if np.isnan(q[i]):
            assert np.isinf(q_lo[i]) or np.isinf(q_hi[i]), (case, a)
            tails += 1
        else:
            assert q_lo[i] <= q[i] <= q_hi[i], (case, a)
            assert np.isfinite(q_lo[i]) and np.isfinite(q_hi[i])
    if case == "both_tails":                               # α = 0 and 1 need a tail bin: q NaN, that side infinite
        assert tails >= 2 and q_lo[0] == -np.inf and q_hi[-1] == np.inf and np.isnan(q[0]) and np.isnan(q[-1])
    else:
        assert tails == 0


def test_empty_histogram_gives_nan(pkg):
    q = pkg.diagnostics.histogram_quantiles(np.zeros((2, 3, 6), np.int64), np.zeros((2, 3)), np.ones((2, 3)), PROBS)
    assert all(np.all(np.isnan(a)) for a in q)


def _c_quantiles(pkg, counts, lo, hi, probs):
    L = pkg._lib
    c = np.ascontiguousarray(counts, np.int64)
    P, D, nb2 = c.shape
    probs = np.ascontiguousarray(probs, float)
    out = [np.full((P, D, probs.size), 7.0) for _ in range(3)]
    rc = L.lib().dhmc_histogram_quantiles(L.ptr(c), L.ptr(np.ascontiguousarray(lo, float)), L.ptr(np.ascontiguousarray(hi, float)),
                                          nb2 - 2, D, P, L.ptr(probs), probs.size, *(L.ptr(a) for a in out))
    return rc, out


def _same_values(a, b):
    """bit for bit where a value is a number, NaN at the same places"""
    a, b = np.asarray(a, float), np.asarray(b, float)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.where(na, 0.0, a).tobytes() == np.where(nb, 0.0, b).tobytes()


@pytest.mark.parametrize("nb", [1, 5, 64, 4096])
def test_c_quantiles_equal_the_mirror(pkg, nb):
    rng = np.random.default_rng(nb)
    P, D = 3, 5
    lo = rng.normal(size=(P, D)) * 10.0 ** rng.integers(-3, 4, (P, D)).astype(float)
    hi = lo + rng.uniform(0.01, 5.0, (P, D))
    counts = rng.integers(0, 4, (P, D, nb + 2)) * (rng.uniform(size=(P, D, nb + 2)) < 0.3)
    counts[0, 0] = 0                                                        # empty
    counts[0, 1] = 0
    counts[0, 1, nb // 2 + 1] = 9                                           # everything in one bin
    counts[1, 0, 0] += 50                                                   # heavy lower tail
    counts[1, 1, -1] += 50                                                  # heavy upper tail
    probs = np.array([0.0, 1e-3, 0.05, 0.3, 0.5, 0.95, 1.0])
    rc, got = _c_quantiles(pkg, counts, lo, hi, probs)
    assert rc == 0
    want = pkg.diagnostics.histogram_quantiles(counts, lo, hi, probs)
    for g, w, name in zip(got, want, ("q", "q_lo", "q_hi")):
        assert _same_values(g, w), (nb, name)


def test_acceptance_placement_is_the_shared_helper(pkg):
    """dhmc_acceptance_quantiles_dev now reads its quantiles through the helper of dhmc_histogram_quantiles on the grid
    (0, 1, 4096) with empty tails; its former placement ((b + (r − C + 0.5)/c_b) / 4096, Julia's type 7 over it) is
    reproduced here and must agree bit for bit"""
    BINS = 4096
    rng = np.random.default_rng(5)
    for trial in range(4):
        hist = rng.integers(0, 3, BINS) * (rng.uniform(size=BINS) < 0.05)
        hist[rng.integers(0, BINS)] += 1
        tot = int(hist.sum())

        def order_stat(j):
            cum = 0
            for b in range(BINS):
                if j < cum + hist[b]:
                    return (b + ((j - cum) + 0.5) / hist[b]) / BINS
                cum += int(hist[b])
            return 1.0

        probs = np.array([0.0, 0.05, 0.25, 0.5, 0.75, 0.95, 1.0, rng.uniform()])
        want = []
        for a in probs:
            pos = a * float(tot - 1)
            j = int(pos)
            g = pos - j
            x = order_stat(j)
            want.append(x + g * (order_stat(j + 1) - x) if g > 0 else x)
        counts = np.zeros((1, 1, BINS + 2), np.int64)
        counts[0, 0, 1:-1] = hist
        rc, (q, _, _) = _c_quantiles(pkg, counts, [[0.0]], [[1.0]], probs)
        assert rc == 0 and np.array(want).tobytes() == q[0, 0].tobytes(), trial


def test_argument_checks_without_gpu(pkg):
    L = pkg._lib
    lib = L.lib()
    good = (np.zeros((2, 3, 10), np.int64), np.zeros((2, 3)), np.ones((2, 3)), np.array([0.5]))

    def call(counts=None, lo=None, hi=None, nb=8, probs=None, D=3, P=2, ptr_counts=True):
        c, l, h, p = (good[0] if counts is None else counts), (good[1] if lo is None else lo), \
            (good[2] if hi is None else hi), (good[3] if probs is None else probs)
        out = np.empty((p.size, D * P))
        return lib.dhmc_histogram_quantiles(L.ptr(c) if ptr_counts else None, L.ptr(np.ascontiguousarray(l, float)),
                                            L.ptr(np.ascontiguousarray(h, float)), nb, D, P, L.ptr(np.asarray(p, float)),
                                            p.size, L.ptr(out), None, None)

    assert call() == 0
    bad_lo = good[1].copy(); bad_lo[1, 2] = np.nan
    bad_hi = good[2].copy(); bad_hi[0, 1] = np.inf
    eq_hi = good[2].copy(); eq_hi[1, 0] = 0.0
    neg = good[0].copy(); neg[1, 1, 3] = -1
    for kw in (dict(nb=0), dict(nb=4097), dict(lo=bad_lo), dict(hi=bad_hi), dict(hi=eq_hi), dict(hi=-good[2]),
               dict(lo=np.full((2, 3), -1e308), hi=np.full((2, 3), 1e308)),           # hi − lo overflows
               dict(hi=np.full((2, 3), 1e-320)),                                      # nbins / (hi − lo) overflows
               dict(probs=np.array([0.5, 1.5])), dict(probs=np.array([-0.1])), dict(probs=np.array([np.nan])),
               dict(counts=neg), dict(ptr_counts=False), dict(D=0)):
        assert call(**kw) == L.DHMC_EARG, kw
    rec = np.zeros((2, 3, L.SUMMARY_FIELDS))
    assert lib.dhmc_mcmc_summary_histogram(None, 10, 1, None, L.ptr(good[1]), L.ptr(good[2]), 8, L.ptr(rec),
                                           L.ptr(good[0]), None, None) == L.DHMC_EARG
    d = pkg.diagnostics
    for lo, hi, nb in ((good[1], good[2], 0), (good[1], good[2], 4097), (bad_lo, good[2], 8), (good[1], eq_hi, 8)):
        with pytest.raises(pkg.ArgumentError):
            d.check_grid(lo, hi, nb)
    with pytest.raises(pkg.ArgumentError):
        d.histogram_quantiles(good[0], good[1], good[2], [1.5])
    with pytest.raises(pkg.ArgumentError):
        d.histogram_quantiles(neg, good[1], good[2], [0.5])
    with pytest.raises(pkg.ArgumentError):
        d.histogram_from_draws(np.zeros((2, 8, 3)), good[1], good[2], 8, thin=3)
    x = np.random.default_rng(0).normal(size=(2, 8, 3))                  # an integral float bin count is the integer
    assert np.array_equal(d.histogram_from_draws(x, good[1], good[2], 8.0), d.histogram_from_draws(x, good[1], good[2], 8))
    # the Python checks run before the library is called (an Engine shell without a handle)
    eng = object.__new__(pkg.Engine)
    eng.K, eng.D, eng.ℓ, eng._h, eng._lib = 4, 3, pkg.StandardNormal(3), None, lib
    lo, hi = np.zeros((1, 3)), np.ones((1, 3))
    for kw in (dict(quantiles=[0.5]), dict(quantiles=[1.5], grid=(lo, hi)), dict(quantiles=[0.5], grid=(lo, hi), bins=0),
               dict(quantiles=[0.5], grid=(hi, lo)), dict(quantiles=[0.5], grid=(np.zeros((2, 3)), np.ones((2, 3)))),
               dict(grid=(lo, hi))):
        with pytest.raises(pkg.ArgumentError):
            eng.mcmc_summary(10, **kw)


def test_quantile_grid_placeholders(pkg):
    d = pkg.diagnostics
    mean = np.array([[0.5, 2.0, np.nan, 3.0, 1e305, -4.0, 7.0]])
    sd = np.array([[2.0, 0.0, np.nan, np.inf, 1e308, np.nan, 1e-300]])
    lo, hi = d.quantile_grid(dict(mean=mean, sd=sd))
    assert lo[0, 0] == 0.5 - 12.0 and hi[0, 0] == 0.5 + 12.0
    assert (lo[0, 1], hi[0, 1]) == (0.0, 4.0)                               # sd = 0: (c − max(1, |c|), c + max(1, |c|))
    assert (lo[0, 2], hi[0, 2]) == (-1.0, 1.0)                              # no chain
    assert (lo[0, 3], hi[0, 3]) == (0.0, 6.0)                               # sd not finite
    assert (lo[0, 4], hi[0, 4]) == (-1.0, 1.0)                              # mean ± 6 sd overflows; |mean| > 1e300
    assert (lo[0, 5], hi[0, 5]) == (-8.0, 0.0)
    assert (lo[0, 6], hi[0, 6]) == (0.0, 14.0)                              # mean ± 6 sd rounds to lo = hi
    for nb in (1, 256, 4096):
        d.check_grid(lo, hi, nb)
    # from a record: the same rule on finish_summary(record)
    rng = np.random.default_rng(2)
    x = rng.normal(size=(4, 12, 3))
    rec = d.summary_from_draws(x)
    s = d.finish_summary(rec)
    lo2, hi2 = d.quantile_grid(rec, width=3.0)
    assert np.array_equal(lo2, s["mean"] - 3.0 * s["sd"]) and np.array_equal(hi2, s["mean"] + 3.0 * s["sd"])


@pytest.mark.parametrize("cuts", [(5,), (1, 2, 9), (3, 6, 7, 10), (4,)], ids=lambda c: "-".join(map(str, c)))
def test_histograms_of_any_split_add_up(pkg, cuts):
    rng = np.random.default_rng(sum(cuts))
    K, N, D, cpp, P, thin, nb = 12, 16, 5, 3, 4, 2, 12
    x = rng.normal(size=(K, N, D)) * 2.0
    lo, hi = np.full((P, D), -1.5), np.full((P, D), 1.5)
    whole = pkg.diagnostics.histogram_from_draws(x, lo, hi, nb, cpp, thin)
    bounds = [0, *cuts, K]
    parts = [pkg.diagnostics.histogram_from_draws(x[a:b], lo, hi, nb, cpp, thin, a) for a, b in zip(bounds, bounds[1:])]
    assert np.array_equal(sum(parts), whole)
    assert np.all(whole.sum(axis=2) == (N // thin) * cpp) and whole[..., 0].sum() > 0 and whole[..., -1].sum() > 0
    done = rng.uniform(size=K) < 0.7
    rec = pkg.diagnostics.finish_summary(pkg.diagnostics.summary_from_draws(x, cpp, thin, None, 0, n_problems=P, completed=done))
    h = pkg.diagnostics.histogram_from_draws(x, lo, hi, nb, cpp, thin, completed=done)
    assert np.array_equal(h.sum(axis=2), rec["draws"])                     # Σ over bins = the summary's draws


# ------------------------------------------------------------------ GPU
def _same_bits(a, b):
    return np.asarray(a).tobytes() == np.asarray(b).tobytes()


def _close(got, want, ctx=""):
    """summary statistics within RTOL (NaN where NaN), ranks and draw counts exactly (as test_streaming_summary.py)"""
    for k in ("rank", "draws"):
        assert np.array_equal(got[k], want[k]), (ctx, k)
    for k in STATS:
        g, w = np.asarray(got[k], float), np.asarray(want[k], float)
        assert np.array_equal(np.isnan(g), np.isnan(w)), (ctx, k)
        scale = np.abs(w) + (np.nan_to_num(np.asarray(want["sd"], float)) if k == "mean" else 0.0)
        ok = np.isnan(w) | (g == w) | (np.abs(g - w) <= RTOL * scale)
        assert np.all(ok), (ctx, k, g[~ok], w[~ok])


def _narrow_grid(draws, cpp, P, thin):
    """per (problem, parameter) the 30 % and 70 % points of its kept draws: both tails receive draws"""
    x = np.asarray(draws)[:, thin - 1::thin]
    K, _, D = x.shape
    prob = np.arange(K) // cpp if cpp else np.zeros(K, int)
    lo, hi = np.empty((P, D)), np.empty((P, D))
    for p in range(P):
        v = x[prob == p].reshape(-1, D)
        lo[p], hi[p] = np.quantile(v, 0.3, axis=0), np.quantile(v, 0.7, axis=0)
        hi[p] = np.maximum(hi[p], lo[p] + 1e-9 * (1.0 + np.abs(lo[p])))
    return lo, hi


def _drop_in(pkg, eng, N, thin=1, reference=None, cpp=0, P=1, bins=16, ctx=""):
    """mcmc from a checkpoint, then the summary with histograms from the same checkpoint: same final state, statistics,
    log densities and transition count bit for bit; the histogram equals the mirror on mcmc's draws as integers and the
    record the summary mirror"""
    ck = eng.checkpoint()
    t0 = eng.transition_count
    run = eng.mcmc(N)
    s1, t1 = eng.get_state(("q", "lq", "grad", "eps")), eng.transition_count
    lo, hi = _narrow_grid(run["posterior_matrix"], cpp, P, thin)
    eng.restore(ck)
    summ = eng.mcmc_summary(N, thin=thin, reference=reference, stats=True, quantiles=(0.05, 0.5, 0.95), grid=(lo, hi),
                            bins=bins)
    s2, t2 = eng.get_state(("q", "lq", "grad", "eps")), eng.transition_count
    assert t1 == t2 == t0 + N, ctx
    for f in s1:
        assert _same_bits(s1[f], s2[f]), (ctx, f)
    assert _same_bits(run["tree_statistics"][:, thin - 1::thin], summ["tree_statistics"]), ctx
    assert _same_bits(run["logdensities"][:, thin - 1::thin], summ["logdensities"]), ctx
    d = pkg.diagnostics
    want = d.histogram_from_draws(run["posterior_matrix"], lo, hi, bins, cpp, thin, 0, P)
    assert summ["histogram"].dtype == np.int64 and summ["histogram"].shape == (P, eng.D, bins + 2), ctx
    assert np.array_equal(summ["histogram"], want), ctx
    assert np.array_equal(summ["histogram"].sum(axis=2), summ["draws"]), ctx
    assert np.all(want[..., 0] > 0) and np.all(want[..., -1] > 0), ctx          # both tails received draws
    rec = d.summary_from_draws(run["posterior_matrix"], cpp, thin, reference, 0, n_problems=P)
    _close(summ, d.finish_summary(rec), ctx)
    q = d.histogram_quantiles(want, lo, hi, summ["probs"])
    for a, k in zip(q, ("quantile", "quantile_lo", "quantile_hi")):
        assert _same_bits(np.nan_to_num(a), np.nan_to_num(summ[k])), (ctx, k)
    return summ


def _engine(pkg, ℓ, K, eps, seed=31, **kw):
    eng = pkg.Engine(ℓ, chains=K, seed=seed, **kw)
    eng.random_position()
    eng.set_stepsize(eps)
    return eng


@pytest.mark.gpu
def test_drop_in_std_normal_dim_1000(pkg):
    eng = _engine(pkg, pkg.StandardNormal(1000), 384, 0.05)
    try:
        _drop_in(pkg, eng, 8, bins=256, ctx="std1000")
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
        _drop_in(pkg, eng, 60, thin=10, reference=ref, cpp=4, P=12, bins=5, ctx="diag-batch")
    finally:
        eng.close()


def _logistic(pkg, rng, N, p):
    X = rng.normal(size=(N, p)) / np.sqrt(p)
    return pkg.LogisticRegression(X, (rng.uniform(size=N) < 0.5).astype(float))


@pytest.mark.gpu
@pytest.mark.parametrize("ragged", [False, True], ids=["batch", "ragged"])
def test_drop_in_packed_logistic(pkg, ragged):
    rng = np.random.default_rng(9)
    probs = [_logistic(pkg, rng, int(rng.integers(20, 90)) if ragged else 50, 24) for _ in range(4)]
    batch = (pkg.RaggedProblemBatch if ragged else pkg.ProblemBatch)(probs, 8)
    ref = rng.normal(size=(4, 24))
    eng = _engine(pkg, batch, batch.chains, 0.1)
    try:
        _drop_in(pkg, eng, 10, thin=2, reference=ref, cpp=8, P=4, bins=7, ctx="logistic")
    finally:
        eng.close()


@pytest.mark.gpu
def test_drop_in_deep_twin(pkg):
    eng = _engine(pkg, pkg.StandardNormal(40), 64, 0.02, algorithm=pkg.NUTS(max_depth=14))
    try:
        _drop_in(pkg, eng, 6, bins=1, ctx="deep")
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
        _drop_in(pkg, eng, 9, reference=rng.normal(size=(1, D)), bins=64, ctx="dense")
    finally:
        eng.close()


@pytest.mark.gpu
def test_drop_in_user_model(pkg):
    ℓ = pkg.UserLogDensity(ROSENBROCK, 6, params=[1.0, 0.5], deep=True)   # __graft_entry__.build() compiles it
    eng = _engine(pkg, ℓ, 64, 0.02)
    try:
        _drop_in(pkg, eng, 8, bins=4096, ctx="rosenbrock")
    finally:
        eng.close()


@pytest.mark.gpu
def test_halted_chain_is_left_out_after_keeping_draws(pkg):
    """walled normal, mode 0 (ℓ = −∞ beyond q₀ = a), min_Δ = −∞: a leaf beyond the wall is not divergent and the next
    leapfrog from it halts the chain with DHMC_CHAIN_LEAPFROG_NONFINITE.  One CTA per SM keeps many chains per resident
    chain group, so chains that halted after keeping draws hand their group's staging histogram to later chains.  The
    histogram is the mirror's over the chains with status 0."""
    L = pkg._lib
    K, D, N, a = 2048, 2, 24, -2.8
    rng = np.random.default_rng(17)
    q = rng.normal(size=(K, D))
    q[:, 0] = np.abs(q[:, 0]) + 0.25                                        # every chain starts inside the wall
    eng = pkg.Engine(pkg.UserLogDensity(WALL, D, params=[a, 0.0], deep=True), chains=K, seed=23,
                     algorithm=pkg.NUTS(min_Δ=-np.inf), ctas_per_sm=1)
    try:
        import torch
        # resident chain groups: grid·G with grid ≤ ctas_per_sm · SMs, and G = 1 (one chain per CTA; only logistic handles
        # pack chains).  Every group therefore runs at least two chains on average.
        T, _ = eng.layout()
        groups = torch.cuda.get_device_properties(0).multi_processor_count
        assert T >= 32 and K >= 2 * groups, (K, groups)
        eng.set_position(q)
        eng.set_stepsize(0.7)
        ck = eng.checkpoint()
        post, ld = np.empty((K, N, D)), np.empty((K, N))
        st = np.zeros((K, N), dtype=L.tree_stats_dtype)
        st.view(np.uint8)[...] = 0xA5                                       # sentinel: rows mcmc never wrote keep it
        sentinel = st[0, 0].tobytes()
        rc = eng._lib.dhmc_mcmc(eng._h, N, L.ptr(post), L.ptr(st), L.ptr(ld))
        status = eng.chain_status()
        assert rc == L.DHMC_ENUMERIC and set(np.unique(status)) == {0, L.DHMC_CHAIN_LEAPFROG_NONFINITE}
        written = np.array([[st[k, n].tobytes() != sentinel for n in range(N)] for k in range(K)])
        halted = status == L.DHMC_CHAIN_LEAPFROG_NONFINITE
        kept_before_halt = written[halted].sum(axis=1)
        assert np.all(written[~halted]) and np.any(kept_before_halt >= 2), kept_before_halt   # the precondition
        # chains leave the queue in index order: a chain that halted after keeping draws with more than `groups` chains
        # queued behind it hands its group, staging histogram included, to a later chain
        early = np.flatnonzero(halted)[kept_before_halt >= 2]
        assert np.any(early < K - 2 * groups), early
        assert np.count_nonzero(~halted) >= K // 4
        lo, hi = np.full((1, D), -1.0), np.full((1, D), 1.0)
        eng.restore(ck)
        with pytest.raises(pkg.ArgumentError, match="leapfrog called from non-finite log density") as e:
            eng.mcmc_summary(N, quantiles=(0.5,), grid=(lo, hi), bins=32)
        assert np.array_equal(e.value.debug_information["chain_status"], status)
        summ = e.value.debug_information["summary"]
        want = pkg.diagnostics.histogram_from_draws(post, lo, hi, 32, completed=status == 0)
        assert np.array_equal(summ["histogram"], want)
        assert np.all(summ["histogram"].sum(axis=2) == N * np.count_nonzero(status == 0))
    finally:
        eng.close()


@pytest.mark.gpu
def test_shard_histograms_add_up_to_the_one_handle_histogram(pkg):
    batch = _diag_batch(pkg, 6, 7, 4, seed=12)
    rng = np.random.default_rng(3)
    lo = rng.normal(size=(6, 7)) - 0.5
    hi = lo + 1.0
    N, thin, cut = 24, 2, 10                                      # chains 8, 9 | 10, 11 of problem 2
    outs = []
    for off, K in ((0, batch.chains), (0, cut), (cut, batch.chains - cut)):
        eng = _engine(pkg, batch, K, 0.45, chain_offset=off)
        try:
            outs.append(eng.mcmc_summary(N, thin=thin, quantiles=(0.1, 0.9), grid=(lo, hi), bins=24))
        finally:
            eng.close()
    whole, a, b = outs
    assert np.array_equal(a["histogram"] + b["histogram"], whole["histogram"])
    assert np.all(a["histogram"][3:] == 0) and np.all(b["histogram"][:2] == 0)
    assert whole["histogram"][..., 0].sum() > 0 and whole["histogram"][..., -1].sum() > 0
    q = pkg.diagnostics.histogram_quantiles(a["histogram"] + b["histogram"], lo, hi, (0.1, 0.9))
    assert _same_bits(np.nan_to_num(q[0]), np.nan_to_num(whole["quantile"]))


@pytest.mark.gpu
def test_end_to_end_quantiles_of_gaussian_posteriors(pkg):
    """64 DiagNormal posteriors, the pilot grid: almost no mass in the tails, and the known μ + σΦ⁻¹(α) within one bin
    width plus 5 quantile-MCSEs (√(α(1 − α)/ESS)/φ(z_α) in units of σ, ESS the summary's, at most the draws)"""
    from scipy import stats
    P, D, K, N = 64, 4, 16, 400
    rng = np.random.default_rng(20261018)
    mu, s2 = rng.normal(size=(P, D)) * 3.0, rng.uniform(0.3, 3.0, size=(P, D))
    batch = pkg.ProblemBatch([pkg.DiagNormal(mu[p], s2[p]) for p in range(P)], K)
    probs = (0.05, 0.5, 0.95)
    out = pkg.summarize_with_warmup(78, batch, N, quantiles=probs)
    h = out["histogram"]
    assert np.all(h.sum(axis=2) == N * K) and np.all(out["draws"] == N * K)
    assert (h[..., 0].sum() + h[..., -1].sum()) / h.sum() <= 1e-3
    lo, hi = out["grid"]
    width = (hi - lo) / 256
    sigma = np.sqrt(s2)
    ess = np.minimum(np.nan_to_num(out["ess"], nan=1.0), N * K)
    for i, a in enumerate(probs):
        z = stats.norm.ppf(a)
        truth = mu + sigma * z
        mcse = sigma * math.sqrt(a * (1 - a)) / stats.norm.pdf(z) / np.sqrt(ess)
        err = np.abs(out["quantile"][..., i] - truth)
        assert np.all(err <= width + 5 * mcse), (a, np.max(err / (width + 5 * mcse)))
        assert np.all(out["quantile_lo"][..., i] <= out["quantile"][..., i])
        assert np.all(out["quantile"][..., i] <= out["quantile_hi"][..., i])


@pytest.mark.gpu
def test_argument_checks_before_launch(pkg):
    eng = _engine(pkg, pkg.StandardNormal(3), 8, 0.5)
    try:
        L = pkg._lib
        rec = np.zeros((1, 3, L.SUMMARY_FIELDS))
        lo, hi = np.zeros((1, 3)), np.ones((1, 3))
        counts = np.zeros((1, 3, 10), np.int64)
        nan_lo = lo.copy(); nan_lo[0, 1] = np.nan
        inf_hi = hi.copy(); inf_hi[0, 2] = np.inf
        t0, n0 = eng.transition_count, eng.kernel_launches()
        for l, h, nb, c in ((lo, hi, 0, counts), (lo, hi, 4097, counts), (hi, lo, 8, counts), (lo, lo, 8, counts),
                            (nan_lo, hi, 8, counts), (lo, inf_hi, 8, counts), (lo, hi, 8, None)):
            assert eng._lib.dhmc_mcmc_summary_histogram(eng._h, 10, 1, None, L.ptr(l), L.ptr(h), nb, L.ptr(rec), L.ptr(c),
                                                        None, None) == L.DHMC_EARG, nb
        assert eng._lib.dhmc_mcmc_summary_histogram(eng._h, 10, 3, None, L.ptr(lo), L.ptr(hi), 8, L.ptr(rec), L.ptr(counts),
                                                    None, None) == L.DHMC_EARG
        assert eng.transition_count == t0 and eng.kernel_launches() == n0
        assert np.all(counts == 0)
    finally:
        eng.close()
