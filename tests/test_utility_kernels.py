"""The on-device diagnostics (k_tree_summary, k_pilot_mean + k_ess_rhat, k_acceptance_hist, and the host code that finishes
their results) and the warm-up metric estimate (the streaming co-moments of metric_push / metric_finish, then k_cov_finish
or k_cov_pool) against references written here from the definitions, in exact or long-double arithmetic.

The diagnostics are fed synthetic device buffers (draws [K, N, D], tree statistics [K, N]) built to hit the inputs where
such reductions go wrong: odd N, tiny n, the tails of the 32-parameter warp tiles, constant parameters, a large common
offset, chains that disagree, depth 32, step sums above 2³², gaps in the acceptance sample.  No sampling is needed.

The metric estimate is checked on real warm-up windows: the M⁻¹ a window leaves must be regularize_M⁻¹ of the exact
covariance of the window draws the call returns (mcmc.jl:209-221), within a stated rounding bound."""
import math
from collections import Counter
from fractions import Fraction

import numpy as np
import pytest

U = 2.0 ** -53                      # unit roundoff of binary64
NAN = float("nan")


# ====================================================================== references
def lag_cap(n, max_lag):
    """L = clamp(max_lag or 64, 1, n − 2)"""
    return max(1, min(max_lag if max_lag > 0 else 64, n - 2))


def _geyer_ess(rho, L, m, n):
    """τ = −1 + 2 Σ (ρ̂₂ₖ + ρ̂₂ₖ₊₁) over the pairs with 2k + 1 ≤ L while the pair is positive, each pair capped by the one
    before it (the initial monotone sequence); τ ≥ 1 / log10(m·n); ESS = m·n / τ"""
    tau, prev = 0, None
    for t in range(0, L, 2):
        pair = rho[t] + rho[t + 1]
        if not pair > 0:
            break
        if prev is not None and pair > prev:
            pair = prev
        prev = pair
        tau += 2 * pair
    tau -= 1
    cap = 1 / math.log10(m * n)
    return m * n / (float(tau) if tau >= cap else cap)


def ess_rhat_exact(x, max_lag=0):
    """Split-R̂ and ESS per parameter of draws x [K, N, D] in rational arithmetic (only the final square root, the cap
    and the division are rounded), straight from the definition of include/dhmc.h:
      - sequences: the first n and the next n draws of every chain, n = ⌊N/2⌋ (an odd N drops the last draw), m = 2K;
      - biased autocovariances acovₜ = Σᵢ (xᵢ − x̄)(xᵢ₊ₜ − x̄) / n;
      - W = mean over the sequences of acov₀ · n / (n − 1), var⁺ = (n − 1)/n · W + var(sequence means), R̂ = √(var⁺/W);
      - ρ̂ₜ = 1 − (W − mean acovₜ) / var⁺ for t = 0 … L, L = clamp(max_lag or 64, 1, n − 2);
      - Geyer's initial monotone sequence with the cap τ ≥ 1/log10(m·n) (_geyer_ess);
      - var⁺ = 0 (every sequence constant at one value): ESS = NaN, as MCMCDiagnosticTools.
    Where this differs from MCMCDiagnosticTools.ess_rhat, on purpose and in the library too: ρ̂₀ is not set to 1, the lag
    cap defaults to 64, and the draws are not rank-normalised."""
    x = np.asarray(x, float)
    K, N, D = x.shape
    n, m = N // 2, 2 * K
    L = lag_cap(n, max_lag)
    rhat, ess = np.empty(D), np.empty(D)
    for d in range(D):
        seqs = [[Fraction(v) for v in x[c, h * n:(h + 1) * n, d]] for c in range(K) for h in (0, 1)]
        means = [sum(s) / n for s in seqs]
        acov = [[sum((s[i] - mu) * (s[i + t] - mu) for i in range(n - t)) / n for t in range(L + 1)]
                for s, mu in zip(seqs, means)]
        W = sum(a[0] for a in acov) / m * n / (n - 1)
        gm = sum(means) / m
        vp = (n - 1) * W / n + (sum((mu - gm) ** 2 for mu in means) / (m - 1) if m > 1 else 0)
        rhat[d] = math.sqrt(vp / W) if W else (math.inf if vp else NAN)
        if vp == 0:
            ess[d] = NAN
            continue
        rho = [1 - (W - sum(a[t] for a in acov) / m) / vp for t in range(L + 1)]
        ess[d] = _geyer_ess(rho, L, m, n)
    return rhat, ess


def _mean_long(col):
    """x₁ + (x − x₁) summed exactly (math.fsum) and rounded once, divided in long double: the mean of a float64 column
    to within u·|mean − x₁| (a constant column gets its value exactly)"""
    x0 = float(col[0])
    s = math.fsum(list(map(float, col)) + [-x0] * len(col))
    return np.longdouble(x0) + np.longdouble(s) / len(col)


def ess_rhat_long(x, max_lag=0):
    """ess_rhat_exact in long double (means by math.fsum), vectorised for the large shapes"""
    x = np.asarray(x, float)
    K, N, D = x.shape
    n, m = N // 2, 2 * K
    L = lag_cap(n, max_lag)
    seq = np.stack([x[:, :n], x[:, n:2 * n]], axis=1).reshape(m, n, D)
    mu = np.array([[_mean_long(seq[j, :, d]) for d in range(D)] for j in range(m)], dtype=np.longdouble)
    xc = seq.astype(np.longdouble) - mu[:, None, :]
    acov = np.stack([(xc[:, :n - t] * xc[:, t:]).sum(axis=1) / n for t in range(L + 1)])      # [L + 1, m, D]
    W = acov[0].sum(axis=0) / m * n / (n - 1)
    dm = mu - mu[0]
    vp = (n - 1) * W / n + (((dm - dm.sum(axis=0) / m) ** 2).sum(axis=0) / (m - 1) if m > 1 else 0)
    rho = 1 - (W - acov.sum(axis=1) / m) / np.where(vp > 0, vp, 1)
    rhat, ess = np.empty(D), np.empty(D)
    for d in range(D):
        rhat[d] = float(np.sqrt(vp[d] / W[d])) if W[d] else (math.inf if vp[d] else NAN)
        ess[d] = _geyer_ess(list(rho[:, d]), L, m, n) if vp[d] > 0 else NAN
    return rhat, ess


def ess_rhat_ref(x, max_lag=0):
    """exact where that is cheap, long double otherwise"""
    K, N, D = np.shape(x)
    return (ess_rhat_exact if K * N * D * (lag_cap(N // 2, max_lag) + 1) <= 30000 else ess_rhat_long)(x, max_lag)


def ebfmi_exact(pis):
    """EBFMI (diagnostics.jl:29-32): mean(abs2, diff(πs)) / var(πs), exact; NaN for fewer than 2 records and for a
    constant π (0 / 0)"""
    p = [Fraction(float(v)) for v in pis]
    N = len(p)
    if N < 2:
        return NAN
    mean = sum(p) / N
    var = sum((v - mean) ** 2 for v in p) / (N - 1)
    if var == 0:
        return NAN
    return float(sum((b - a) ** 2 for a, b in zip(p, p[1:])) / (N - 1) / var)


def count_terminations_ref(left, right):
    """diagnostics.jl:65-81: REACHED_MAX_DEPTH is InvalidTree(1, 0); is_divergent is left == right (trees.jl:187);
    every other termination is turning"""
    c = Counter()
    for l, r in zip(left, right):
        c["max_depth" if (l, r) == (1, 0) else "divergence" if l == r else "turning"] += 1
    return dict(max_depth=c["max_depth"], divergence=c["divergence"], turning=c["turning"])


def count_depths_ref(depth):
    """diagnostics.jl:87-94: counts of depth 0 … 32, trailing zeros dropped"""
    c = [0] * 33
    for d in depth:
        c[int(d)] += 1
    while c and c[-1] == 0:
        c.pop()
    return c


def quantile7_exact(values, p):
    """Julia's quantile (type 7), exact: x₍ⱼ₎ + γ (x₍ⱼ₊₁₎ − x₍ⱼ₎) at (n − 1)·p = j + γ of the sorted sample"""
    xs = sorted(Fraction(float(v)) for v in values)
    h = Fraction(p) * (len(xs) - 1)
    j = math.floor(h)
    g = h - j
    return xs[j] + g * (xs[j + 1] - xs[j]) if g else xs[j]


def cov_long(X):
    """cov(X; dims = 1) of a window [n, D] in long double (column means by math.fsum): the covariance and the means"""
    n, D = X.shape
    mu = np.array([_mean_long(X[:, d]) for d in range(D)], dtype=np.longdouble)
    Xc = X.astype(np.longdouble) - mu
    return (Xc.T @ Xc) / (n - 1), mu


def cov_exact(X):
    n, D = X.shape
    F = [[Fraction(float(v)) for v in row] for row in X]
    mu = [sum(F[i][d] for i in range(n)) / n for d in range(D)]
    return [[sum((F[k][i] - mu[i]) * (F[k][j] - mu[j]) for k in range(n)) / (n - 1) for j in range(D)] for i in range(D)]


def regularize(S, lam):
    """regularize_M⁻¹(Symmetric(S), λ) = (1 − λ) S + λ Diagonal(diag(S)) (mcmc.jl:218-221), in S's arithmetic"""
    R = (1 - lam) * S
    R[np.diag_indices(S.shape[0])] = np.diag(S)
    return R


def metric_bound(S, mu, n):
    """the rounding bound of a window estimate: n·u·((|x̄ᵢ| + σᵢ)(|x̄ⱼ| + σⱼ) − |x̄ᵢ||x̄ⱼ|) = n·u·(|x̄ᵢ|σⱼ + σᵢ|x̄ⱼ| + σᵢσⱼ).
    A streaming (Welford) estimate errs by rounding of the running means (~u·|x̄|) times the centred draws (~σ), so no
    |x̄ᵢ||x̄ⱼ| term belongs in it; that term is the error of a one-pass Σxx − n·x̄x̄, which the bound must not admit."""
    a, s = np.abs(mu), np.sqrt(np.maximum(np.diag(S), 0))
    return (n * U * (np.outer(a, s) + np.outer(s, a) + np.outer(s, s))).astype(float)


# ====================================================================== synthetic inputs
KINDS = ("iid", "ar0.95", "ar0.995", "ar-0.7", "constant", "chain_constants", "offset1e8", "far_means")


def _ar1(rng, K, N, rho):
    e = rng.normal(size=(K, N))
    x = np.empty((K, N))
    x[:, 0] = e[:, 0] / math.sqrt(1 - rho * rho)             # stationary start
    for i in range(1, N):
        x[:, i] = rho * x[:, i - 1] + e[:, i]
    return x


def synthetic_draws(K, N, D, seed):
    """[K, N, D]; parameter d is of kind KINDS[d % 8]"""
    rng = np.random.default_rng(seed)
    x = np.empty((K, N, D))
    for d in range(D):
        kind = KINDS[d % len(KINDS)]
        if kind == "iid":
            x[:, :, d] = rng.normal(size=(K, N))
        elif kind.startswith("ar"):
            x[:, :, d] = _ar1(rng, K, N, float(kind[2:]))
        elif kind == "constant":                              # a value whose naive mean is not the value (0.1·3 / 3 ≠ 0.1)
            x[:, :, d] = 0.1
        elif kind == "chain_constants":
            x[:, :, d] = (0.1 * (1 + np.arange(K)))[:, None]
        elif kind == "offset1e8":
            x[:, :, d] = 1e8 + rng.normal(size=(K, N))
        else:                                                 # chains around means 50 apart: R̂ ≫ 1
            x[:, :, d] = 50.0 * np.arange(K)[:, None] + rng.normal(size=(K, N))
    return x


def ess_tolerance(x):
    """element-wise relative tolerance of the device's R̂ and ESS for each parameter of x [K, N, D]: 1e-9 for data of
    scale ~1, widened by √n·u·|mean| / sd for data far from 0 (the device's sequence means carry a rounding of u·|mean|,
    which the variance of the means, spread ~ sd/√n, sees relatively)"""
    n = x.shape[1] // 2
    mean = np.abs(x.mean(axis=(0, 1)))
    sd = x.std(axis=(0, 1))
    with np.errstate(divide="ignore", invalid="ignore"):
        cond = np.where(sd > 0, mean / sd, 0.0)
    return 1e-9 + 16 * U * math.sqrt(n) * cond


def ebfmi_tolerance(pis):
    """relative tolerance of the device's EBFMI per chain of pis [B, N]: 1e-12, plus 4·(u·|mean| / sd)² — the device's
    mean of π carries a rounding of u·|mean|, which adds its square to each centred square"""
    B, N = pis.shape
    if N < 2:
        return np.full(B, 1e-12)
    mean, sd = np.abs(pis.mean(axis=1)), pis.std(axis=1, ddof=1)
    with np.errstate(divide="ignore", invalid="ignore"):
        return 1e-12 + 4 * np.where(sd > 0, (U * mean / sd) ** 2, 0.0)


def assert_close_nan(dev, ref, rtol, what):
    """same NaN / ±inf pattern, finite entries within rtol (element-wise)"""
    dev, ref = np.asarray(dev, float), np.asarray(ref, float)
    rtol = np.broadcast_to(rtol, ref.shape)
    assert np.array_equal(np.isnan(dev), np.isnan(ref)), (what, "NaN pattern", dev, ref)
    fin = np.isfinite(ref)
    assert np.array_equal(dev[~fin & ~np.isnan(ref)], ref[~fin & ~np.isnan(ref)]), (what, "inf", dev, ref)
    err = np.abs(dev[fin] - ref[fin]) / np.maximum(np.abs(ref[fin]), 1e-300)
    bad = err > rtol[fin]
    assert not bad.any(), (what, np.flatnonzero(fin)[bad], dev[fin][bad], ref[fin][bad], err[bad])


def tree_stats(pkg, B, N, seed):
    """[B, N] records: depth 0 … 32 (all of them when B·N ≥ 33), the three termination classes with turning on both
    sides (left < right and left > right), steps up to 2³² − 1, acceptance rates with exact 0 and 1; chain 0 has a
    constant π (a value whose naive mean is not itself), chain 1 π = 1e9 + N(0, 1)"""
    rng = np.random.default_rng(seed)
    s = np.zeros((B, N), dtype=pkg._lib.tree_stats_dtype)
    total = B * N
    depth = rng.integers(0, 33, total)
    depth[:min(33, total)] = np.arange(min(33, total))
    s["depth"] = depth.reshape(B, N)
    cls = rng.integers(0, 4, total)
    left, right = rng.integers(0, 2 ** 40, total), rng.integers(0, 2 ** 40, total)
    left = np.where(cls == 0, 1, left); right = np.where(cls == 0, 0, right)                         # REACHED_MAX_DEPTH
    right = np.where(cls == 1, left, right)                                                           # divergent
    lo, hi = np.minimum(left, right), np.maximum(left, right) + 2
    left = np.where(cls == 2, lo, np.where(cls == 3, hi, left))                                       # turning, left < right
    right = np.where(cls == 2, hi, np.where(cls == 3, lo, right))                                     # turning, left > right
    s["left"], s["right"] = left.reshape(B, N), right.reshape(B, N)
    s["steps"] = rng.integers(0, 2 ** 32, (B, N))
    a = rng.uniform(size=total)
    a[rng.uniform(size=total) < 0.1] = 1.0
    a[rng.uniform(size=total) < 0.05] = 0.0
    s["acceptance_rate"] = a.reshape(B, N)
    s["pi"] = rng.normal(-40.0, 3.0, (B, N))
    s["pi"][0] = 0.1
    if B > 1:
        s["pi"][1] = 1e9 + rng.normal(size=N)
    return s


def _device(arr):
    import torch
    return torch.from_numpy(np.ascontiguousarray(arr)).cuda()


def _device_stats(s):
    import torch
    return torch.from_numpy(np.ascontiguousarray(s).view(np.uint8).reshape(s.shape + (s.dtype.itemsize,)).copy()).cuda()


# ====================================================================== CPU: the references agree with each other
def test_long_double_references_match_the_exact_ones():
    """within 1e-14, plus 2⁻⁶⁰·|mean|/sd for data far from 0 (long-double centring) — far inside the GPU tolerances"""
    for K, N, D, lag in ((1, 4, 8, 0), (2, 7, 8, 1), (3, 9, 16, 0), (2, 12, 8, 3), (2, 13, 8, 100)):
        x = synthetic_draws(K, N, D, seed=K * 100 + N)
        ex, ln = ess_rhat_exact(x, lag), ess_rhat_long(x, lag)
        with np.errstate(divide="ignore", invalid="ignore"):
            cond = np.nan_to_num(np.abs(x.mean(axis=(0, 1))) / x.std(axis=(0, 1)), posinf=0.0)
        for e, l in zip(ex, ln):
            assert_close_nan(l, e, 1e-14 + 2.0 ** -60 * cond, (K, N, D, lag))
    rng = np.random.default_rng(4)
    for X in (rng.normal(size=(7, 3)), 1e3 + 1e-3 * rng.normal(size=(20, 4)), np.full((5, 2), 0.1)):
        S, _ = cov_long(X)
        E = np.array([[float(v) for v in row] for row in cov_exact(X)])
        np.testing.assert_allclose(S.astype(float), E, rtol=1e-15, atol=1e-300)


def test_ess_rhat_reference_on_edge_inputs():
    """a constant parameter has R̂ = ESS = NaN; chains at different constants have W = 0, R̂ = ∞ and ρ̂ₜ = 1 at every
    lag, so τ = 4·(number of pairs) − 1; an anticorrelated chain hits the cap"""
    K, N = 3, 12
    x = synthetic_draws(K, N, 8, seed=9)
    rhat, ess = ess_rhat_exact(x)
    c = KINDS.index("constant"), KINDS.index("chain_constants"), KINDS.index("ar-0.7")
    assert math.isnan(rhat[c[0]]) and math.isnan(ess[c[0]])
    n, m = N // 2, 2 * K
    L = lag_cap(n, 0)
    assert rhat[c[1]] == math.inf and ess[c[1]] == m * n / (4 * ((L + 1) // 2) - 1)
    x = _ar1(np.random.default_rng(1), 4, 400, -0.7)[:, :, None]
    _, e = ess_rhat_long(x)
    assert e[0] == pytest.approx(8 * 200 * math.log10(8 * 200), rel=1e-12)


def test_diagnostics_mirror_matches_the_references(pkg):
    """diagnostics.ess_rhat and diagnostics.EBFMI (the numpy mirror of the device) against the references on the edge
    inputs"""
    for K, N, D, lag in ((1, 4, 8, 0), (2, 5, 8, 1), (3, 7, 8, 0), (2, 40, 16, 1000), (4, 129, 8, 0)):
        x = synthetic_draws(K, N, D, seed=7 + N)
        r = pkg.diagnostics.ess_rhat(x, max_lag=lag)
        rhat, ess = ess_rhat_ref(x, lag)
        tol = ess_tolerance(x)
        assert_close_nan(r["rhat"], rhat, tol, ("rhat", K, N, D))
        assert_close_nan(r["ess"], ess, tol, ("ess", K, N, D))
    s = tree_stats(pkg, 3, 33, seed=2)
    for N in (1, 2, 3, 33):
        for c in range(3):
            got, ref = pkg.diagnostics.EBFMI(s[c, :N]), ebfmi_exact(s["pi"][c, :N])
            assert (math.isnan(got) and math.isnan(ref)) or got == pytest.approx(ref, rel=1e-12), (N, c, got, ref)


# ====================================================================== GPU: split-R̂ and ESS
ESS_SHAPES = [      # (K, N, D, max_lag): N with odd values, max_lag 0 / 1 / n − 2 / far above n, D at the warp-tile tails
    (1, 4, 1, 0), (2, 5, 31, 1), (3, 7, 32, 0), (1, 129, 33, 62), (2, 129, 33, 1000), (4099, 5, 33, 0),
    (4099, 4, 1, 1), (3, 129, 257, 62), (4, 1000, 33, 0), (2, 1000, 257, 1), (3, 1000, 32, 5000),
]


@pytest.mark.gpu
@pytest.mark.parametrize("K,N,D,max_lag", ESS_SHAPES)
def test_ess_rhat_matches_the_exact_reference(pkg, K, N, D, max_lag):
    x = synthetic_draws(K, N, D, seed=K * 7919 + N * 31 + D)
    eng = pkg.Engine(pkg.StandardNormal(D), chains=K, seed=1)
    try:
        buf = _device(x)                 # bound to a name: the tensor must outlive the call that reads it
        dev = eng.ess_rhat_dev(buf.data_ptr(), N, max_lag=max_lag)
    finally:
        eng.close()
    rhat, ess = ess_rhat_ref(x, max_lag)
    tol = ess_tolerance(x)
    assert_close_nan(dev["ess"], ess, tol, "ess")
    assert_close_nan(dev["rhat"], rhat, tol, "rhat")


@pytest.mark.gpu
@pytest.mark.parametrize("P,K,off,B", [(4, 3, 4, 5), (4, 5, 7, 9)])
def test_ess_rhat_per_problem_on_a_shard(pkg, P, K, off, B):
    """a shard that starts inside a problem (chain_offset not a multiple of K) and problems without a local chain (NaN)"""
    D, N = 33, 129
    rng = np.random.default_rng(P * K + off)
    batch = pkg.ProblemBatch([pkg.DiagNormal(rng.normal(size=D), rng.uniform(0.5, 2, D)) for _ in range(P)], K)
    x = synthetic_draws(B, N, D, seed=off)
    eng = pkg.Engine(batch, chains=B, seed=1, chain_offset=off)
    try:
        buf = _device(x)
        dev = eng.ess_rhat_problems_dev(buf.data_ptr(), N)
    finally:
        eng.close()
    empty = 0
    for p in range(P):
        lo, hi = batch.problem_chains(p, off, B)
        if lo == hi:
            empty += 1
            assert np.isnan(dev["rhat"][p]).all() and np.isnan(dev["ess"][p]).all(), p
            continue
        rhat, ess = ess_rhat_ref(x[lo:hi])
        tol = ess_tolerance(x[lo:hi])
        assert_close_nan(dev["ess"][p], ess, tol, ("ess", p))
        assert_close_nan(dev["rhat"][p], rhat, tol, ("rhat", p))
    assert empty >= 1


# ====================================================================== GPU: tree summary
@pytest.mark.gpu
@pytest.mark.parametrize("B,N", [(5, 1), (5, 2), (5, 3), (7, 33), (3, 1000), (70000, 2)])
def test_tree_summary_matches_the_exact_reference(pkg, B, N):
    """counts and the step sum exact; the acceptance sum within (B·N)·u·2 relative; EBFMI within ebfmi_tolerance (NaN
    for N = 1 and for a constant π)"""
    s = tree_stats(pkg, B, N, seed=B + N)
    eng = pkg.Engine(pkg.StandardNormal(1), chains=B, seed=1)
    try:
        buf = _device_stats(s)
        dev = eng.tree_summary_dev(buf.data_ptr(), N)
    finally:
        eng.close()
    assert dev["depth_counts"] == count_depths_ref(s["depth"].ravel())
    assert dev["termination_counts"] == count_terminations_ref(s["left"].ravel(), s["right"].ravel())
    steps = sum(int(v) for v in s["steps"].ravel())
    assert dev["steps"] == steps and (B * N < 2 or steps > 2 ** 32)
    acc = math.fsum(s["acceptance_rate"].ravel())
    assert abs(dev["a_mean"] * B * N - acc) <= 2 * (B * N + 64) * U * acc
    eb = np.array([ebfmi_exact(s["pi"][c]) for c in range(B)])
    assert_close_nan(dev["EBFMI"], eb, ebfmi_tolerance(s["pi"]), "EBFMI")
    if N > 1:
        assert math.isnan(dev["EBFMI"][0]) and np.isfinite(dev["EBFMI"][1])


# ====================================================================== GPU: acceptance quantiles
PROBS = (0.0, 0.05, 0.25, 0.5, 0.75, 0.95, 1.0)
QUANTILE_SAMPLES = {
    "zero_one": [0.0, 1.0],
    "wide_gaps": [0.03, 0.5, 0.51, 0.97, 0.2],
    "all_equal": [0.37] * 10,
    "exact_0_and_1": [0.0, 0.0, 0.0, 1.0, 1.0, 0.5, 1.0],
    "nan_records": [NAN, 0.2, NAN, 0.9, 1.0, NAN],
    "single": [0.42],
    "clamped_ones": list(np.random.default_rng(5).uniform(0.6, 1.0, 300)) + [1.0] * 700,
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(QUANTILE_SAMPLES))
def test_acceptance_quantiles_within_one_bin_of_type7(pkg, name):
    vals = np.array(QUANTILE_SAMPLES[name])
    B = 5 if vals.size % 5 == 0 else 1
    s = np.zeros((B, vals.size // B), dtype=pkg._lib.tree_stats_dtype)
    s["acceptance_rate"] = vals.reshape(B, -1)
    eng = pkg.Engine(pkg.StandardNormal(1), chains=B, seed=1)
    try:
        buf = _device_stats(s)
        q = eng.acceptance_quantiles_dev(buf.data_ptr(), vals.size // B, PROBS)
    finally:
        eng.close()
    finite = vals[~np.isnan(vals)]
    for p, got in zip(PROBS, q):
        ref = quantile7_exact(finite, p)
        assert abs(Fraction(float(got)) - ref) <= Fraction(1, 4096), (name, p, float(got), float(ref))


@pytest.mark.gpu
def test_acceptance_quantiles_of_no_rate_are_nan(pkg):
    s = np.zeros((1, 3), dtype=pkg._lib.tree_stats_dtype)
    s["acceptance_rate"] = NAN
    eng = pkg.Engine(pkg.StandardNormal(1), chains=1, seed=1)
    try:
        buf = _device_stats(s)
        q = eng.acceptance_quantiles_dev(buf.data_ptr(), 3, PROBS)
    finally:
        eng.close()
    assert np.isnan(q).all()


# ====================================================================== metric estimation
# TuningNUTS takes windows of N ≥ 20 (mcmc.jl:191), so 20 and 21 are the smallest windows there are.
METRIC_BOUND = 1.0      # |M̂⁻¹ᵢⱼ − M⁻¹ᵢⱼ| ≤ METRIC_BOUND · n·u·(|x̄ᵢ|σⱼ + σᵢ|x̄ⱼ| + σᵢσⱼ)  (metric_bound)
CALIBRATION_MARGIN = 0.5   # the oracle (bit-identical to the device) stays below half of it on the calibration windows


def _target(D, kind):
    """'offset': DIAG_NORMAL with mean 1e3 and sd 1e-3 in every coordinate; 'unit': means N(0, 1), sd 0.5 … 2"""
    rng = np.random.default_rng(D)
    if kind == "offset":
        mu, sd = np.full(D, 1e3), np.full(D, 1e-3)
    else:
        mu, sd = rng.normal(size=D), rng.uniform(0.5, 2.0, D)
    return mu, sd


def _reference_metric(X, M, lam):
    """(reference M⁻¹, bound) of one window X [n, D] (a pooled group: its 8·n draws)"""
    S, mu = cov_long(X)
    bound = METRIC_BOUND * metric_bound(S, mu, X.shape[0])
    if M == "Diagonal":
        return np.diag(S).astype(float), np.diag(bound)                   # var, mcmc.jl:209; regularize is the identity
    return regularize(S, np.longdouble(lam)).astype(float), bound


def test_metric_bound_is_calibrated_on_the_oracle(po):
    """The bound of the GPU metric tests on the oracle, whose streaming estimate is bit-identical to the device's: it holds
    with a margin; an estimate with a wrong divisor or a recurrence on the stale mean exceeds it, and so does a one-pass
    Σxx − n·x̄x̄ on the target far from 0 (on the other, centred target a one-pass estimate is as accurate as any)."""
    for kind in ("offset", "unit"):
        for D, n in ((2, 20), (5, 25), (33, 21)):
            rng = np.random.default_rng(D + n)
            mu, sd = (np.full(D, 1e3), np.full(D, 1e-3)) if kind == "offset" else (rng.normal(size=D), rng.uniform(0.5, 2, D))
            params = np.concatenate([mu, 1 / sd ** 2])
            q0 = mu + sd * rng.normal(size=D)
            for code, M in ((po.METRIC_DIAGONAL, "Diagonal"), (po.METRIC_SYMMETRIC, "Symmetric")):
                o = po.mcmc_with_warmup(po.FAMILY_DIAG_NORMAL, D, 1, 5, 3, stages=[(po.STAGE_TUNING, n, code, 1)],
                                        params=params, T=32, q0=q0, minv0=sd ** 2, eps0=0.5, welford=True, keep_warmup=True)
                X = o["warmup_posterior"]
                ref, bound = _reference_metric(X, M, 5.0 / n)
                assert np.all(np.abs(o["minv"] - ref) <= CALIBRATION_MARGIN * bound), (kind, D, n, M)
                # what a wrong finish would give
                assert np.any(np.abs(o["minv"] * (n - 1) / n - ref) > bound), (kind, D, n, M, "divisor n")
            # a recurrence on the stale mean: C += δᵢ δⱼ instead of δᵢ (xⱼ − x̄′ⱼ)
            m_, C = np.zeros(D), np.zeros((D, D))
            for i, x in enumerate(X, 1):
                dl = x - m_
                m_ = m_ + dl / i
                C += np.outer(dl, dl)
            ref, bound = _reference_metric(X, "Symmetric", 5.0 / n)
            assert np.any(np.abs(regularize(C / (n - 1), 5.0 / n) - ref) > bound), (kind, D, n, "stale mean")
            if kind == "offset":    # one pass: Σ xxᵀ − n x̄x̄ᵀ in binary64
                naive = (X.T @ X - n * np.outer(X.mean(axis=0), X.mean(axis=0))) / (n - 1)
                assert np.any(np.abs(regularize(naive, 5.0 / n) - ref) > bound), (kind, D, n, "one pass")


def _window_minv(eng, M):
    return eng.get_metric_dense() if M != "Diagonal" else eng.get_state(("minv",))["minv"]


METRIC_CASES = [    # (metric, window n, D, λ (None: the default 5/n), target)
    ("Diagonal", 20, 1, None, "offset"), ("Diagonal", 21, 2, None, "unit"), ("Diagonal", 25, 33, None, "offset"),
    ("Diagonal", 20, 129, None, "unit"), ("Diagonal", 21, 257, None, "offset"), ("Diagonal", 25, 513, None, "offset"),
    ("Symmetric", 20, 1, 0.0, "offset"), ("Symmetric", 21, 2, None, "unit"), ("Symmetric", 25, 2, 0.0, "offset"),
    ("Symmetric", 20, 33, None, "offset"), ("Symmetric", 21, 33, 1.0, "unit"), ("Symmetric", 25, 129, 1.0, "offset"),
    ("Symmetric", 20, 257, None, "unit"), ("Symmetric", 25, 513, None, "offset"), ("Symmetric", 21, 513, 1.0, "unit"),
    ("SymmetricPooled", 20, 1, None, "offset"), ("SymmetricPooled", 25, 2, 0.0, "unit"),
    ("SymmetricPooled", 21, 33, 1.0, "offset"), ("SymmetricPooled", 20, 129, None, "offset"),
    ("SymmetricPooled", 25, 257, None, "unit"), ("SymmetricPooled", 20, 513, 1.0, "offset"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("M,n,D,lam,target", METRIC_CASES, ids=lambda v: str(v))
def test_window_metric_is_the_regularized_covariance_of_the_window(pkg, M, n, D, lam, target):
    """M⁻¹ after warmup_stage(TuningNUTS(n, DualAveraging(), M, λ)) against regularize_M⁻¹(cov(window), λ) (Symmetric),
    var(window) (Diagonal), or the covariance of the group's 8·n concatenated draws (pooled), element-wise within
    METRIC_BOUND · n·u·(|x̄ᵢ|σⱼ + σᵢ|x̄ⱼ| + σᵢσⱼ) (n: the draws the estimate is taken over)"""
    mu, sd = _target(D, target)
    K = 16 if M == "SymmetricPooled" else 3
    lam = 5.0 / n if lam is None else lam
    rng = np.random.default_rng(n * D)
    eng = pkg.Engine(pkg.DiagNormal(mu, sd ** 2), chains=K, seed=11)
    try:
        eng.set_metric(sd ** 2)
        eng.set_position(mu + sd * rng.normal(size=(K, D)))
        eng.set_stepsize(0.5)
        X = eng.warmup_stage(pkg.TuningNUTS(n, pkg.DualAveraging(), M, lam), keep=True)["posterior_matrix"]
        got = _window_minv(eng, M)
    finally:
        eng.close()
    assert np.all(X.std(axis=1) > 0), "the window did not move"
    groups = [(range(g, g + 8), X[g:g + 8].reshape(8 * n, D)) for g in range(0, K, 8)] if M == "SymmetricPooled" \
        else [((k,), X[k]) for k in range(K)]
    for chains, W in groups:
        ref, bound = _reference_metric(W, M, lam)
        for k in chains:
            err = np.abs(got[k] - ref)
            assert np.all(err <= bound), (k, float((err / bound).max()))


@pytest.mark.gpu
def test_window_metric_is_bit_identical_to_the_oracle(pkg, po):
    """one window of each metric kind, equal bit for bit to the oracle's streaming estimate"""
    D, n, seed = 5, 25, 3
    rng = np.random.default_rng(0)
    mu, sd = rng.normal(size=D), rng.uniform(0.5, 2, D)
    ℓ = pkg.DiagNormal(mu, sd ** 2)
    q = mu + sd * rng.normal(size=(3, D))
    for M, code in (("Diagonal", po.METRIC_DIAGONAL), ("Symmetric", po.METRIC_SYMMETRIC)):
        eng = pkg.Engine(ℓ, chains=3, seed=seed)
        try:
            T, _ = eng.layout()
            eng.set_metric(sd ** 2); eng.set_position(q); eng.set_stepsize(0.5)
            X = eng.warmup_stage(pkg.TuningNUTS(n, pkg.DualAveraging(), M), keep=True)["posterior_matrix"]
            got = _window_minv(eng, M)
        finally:
            eng.close()
        for k in range(3):
            o = po.mcmc_with_warmup(po.FAMILY_DIAG_NORMAL, D, 1, seed, k, stages=[(po.STAGE_TUNING, n, code, 1)],
                                    params=ℓ.params(), T=T, q0=q[k], minv0=sd ** 2, eps0=0.5, welford=True, keep_warmup=True)
            assert np.array_equal(X[k], o["warmup_posterior"]) and np.array_equal(got[k], o["minv"]), (M, k)
    stages = [(po.STAGE_SEARCH, 0, 0, 0), (po.STAGE_TUNING, n, po.METRIC_SYMMETRIC_POOLED, 1)]
    eng = pkg.Engine(ℓ, chains=8, seed=seed)
    try:
        T, _ = eng.layout()
        eng.random_position(); eng.find_initial_stepsize()
        eng.warmup_stage(pkg.TuningNUTS(n, pkg.DualAveraging(), pkg.SymmetricPooled))
        got = eng.get_metric_dense()
    finally:
        eng.close()
    o = po.mcmc_with_warmup_pooled(po.FAMILY_DIAG_NORMAL, D, 1, seed, 0, stages, params=ℓ.params(), T=T)
    for k in range(8):
        assert np.array_equal(got[k], o["minv"]), k
