"""Host-side mirror of DynamicHMC.Diagnostics (src/diagnostics.jl) over the returned
tree-statistics arrays, plus access to the device-side reduction (dhmc_tree_summary_dev)
that avoids shipping 56 B × N × chains of statistics to the host (SURVEY.md §8f item 2)."""
from dataclasses import dataclass

import numpy as np

ACCEPTANCE_QUANTILES = [0.05, 0.25, 0.5, 0.75, 0.95]      # diagnostics.jl:35


def EBFMI(tree_statistics):
    """diagnostics.jl:29-32: mean(abs2, diff(πs)) / var(πs) for one chain's statistics.  The variance is taken of
    πs − π₁, so a constant π gives 0 / 0 = NaN (as the device reduction does), not 0 over a rounding residue."""
    pis = np.asarray(tree_statistics["pi"], float)
    if pis.size < 2:
        return float("nan")
    with np.errstate(invalid="ignore", divide="ignore"):
        return float(np.mean(np.diff(pis) ** 2) / np.var(pis - pis[0], ddof=1))


def count_terminations(tree_statistics):
    """diagnostics.jl:65-81"""
    l, r = np.asarray(tree_statistics["left"]), np.asarray(tree_statistics["right"])
    maxd = (l == 1) & (r == 0)
    div = (l == r)
    return dict(max_depth=int(maxd.sum()), divergence=int(div.sum()), turning=int((~maxd & ~div).sum()))


def count_depths(tree_statistics):
    """diagnostics.jl:88-94 (first element is depth 0, trailing zeros dropped)"""
    c = np.bincount(np.asarray(tree_statistics["depth"]).ravel(), minlength=33)
    nz = np.nonzero(c)[0]
    return c[: nz[-1] + 1].tolist() if nz.size else []


@dataclass
class TreeStatisticsSummary:
    """diagnostics.jl:44-57"""
    N: int
    a_mean: float
    a_quantiles: list
    termination_counts: dict
    depth_counts: list


def summarize_tree_statistics(tree_statistics):
    """diagnostics.jl:100-106"""
    a = np.asarray(tree_statistics["acceptance_rate"], float).ravel()
    return TreeStatisticsSummary(int(a.size), float(a.mean()),
                                 [float(v) for v in np.quantile(a, ACCEPTANCE_QUANTILES)],
                                 count_terminations(tree_statistics), count_depths(tree_statistics))


# ------------------------------------------------------------------ trajectory diagnostics
# These drive the device path itself (dhmc_leapfrog / dhmc_phase_logdensity); there is no host
# re-implementation of the integrator here.
def _rand_ps(κ, D, N, seed):
    """rand_p(rng, κ) hamiltonian.jl:124 for the default `ps` (host RNG: the reference draws
    them from the caller's rng, so there is nothing to be bit-compatible with)."""
    z = np.random.default_rng(seed).normal(size=(N, D))
    if κ is None:
        return z
    minv = np.asarray(κ.minv, float)
    if κ.dense:
        W = np.linalg.cholesky(np.linalg.inv(minv))          # hamiltonian.jl:73
        return z @ W.T
    return z / np.sqrt(minv)


def explore_log_acceptance_ratios(ℓ, q, log2ϵs, κ=None, N=20, ps=None, seed=0, device=0):
    """diagnostics.jl:139-147.  From the position `q`, the uncapped log acceptance ratio
    `logdensity(H, leapfrog(H, z, ϵ)) − logdensity(H, z)` (stepsize.jl:83-85) for every
    ϵ = 2^log2ϵ and every momentum in `ps` (N random ones by default).  Returns the matrix
    [len(log2ϵs), len(ps)]; every (ϵ, p) pair is one chain of a single device pass."""
    from . import api
    q = np.asarray(q, float)
    D = q.size
    ps = _rand_ps(κ, D, N, seed) if ps is None else np.asarray(ps, float).reshape(-1, D)
    eps = 2.0 ** np.asarray(log2ϵs, float).reshape(-1)
    E, P = eps.size, ps.shape[0]
    eng = api.Engine(ℓ, chains=E * P, seed=seed, device=device)
    try:
        if κ is not None:
            eng.set_kinetic_energy(κ)
        eng.set_position(np.broadcast_to(q, (E * P, D)))
        eng.set_momentum(np.tile(ps, (E, 1)))                # chain e·P + j = (ϵ_e, p_j)
        eng.set_stepsize(np.repeat(eps, P))
        h0 = eng.phase_logdensity()
        eng.leapfrog(1, 1)
        h1 = eng.phase_logdensity()
    finally:
        eng.close()
    return (h1 - h0).reshape(E, P)


def leapfrog_trajectory(ℓ, q, ϵ, positions, κ=None, p=None, seed=0, device=0):
    """diagnostics.jl:200-216.  Leapfrog trajectory visiting `positions` (a range containing 0)
    relative to `q` with stepsize ϵ, tracked in each direction up to the first non-finite log
    density.  Returns a list of dicts (z = (q, p, ℓq), position, Δ) ordered by position, where
    Δ is the log density + kinetic energy relative to position 0."""
    from . import api
    lo, hi = positions[0], positions[-1]
    api._argcheck(lo <= 0 <= hi, "0 ∈ positions")
    q = np.asarray(q, float)
    D = q.size
    p = _rand_ps(κ, D, 1, seed)[0] if p is None else np.asarray(p, float)
    eng = api.Engine(ℓ, chains=1, seed=seed, device=device)
    out = {}
    try:
        if κ is not None:
            eng.set_kinetic_energy(κ)
        eng.set_stepsize(float(ϵ))
        for sgn, last in ((+1, hi), (-1, -lo)):
            eng.set_position(q[None, :])
            eng.set_momentum(p[None, :])
            st = eng.get_state(("q", "p", "lq"))
            π0 = eng.phase_logdensity()[0]
            out[0] = dict(z=dict(q=st["q"][0], p=st["p"][0], lq=float(st["lq"][0])), position=0, Δ=0.0)
            for i in range(1, last + 1):
                if not np.isfinite(st["lq"][0]):            # iterate(::LeapfrogTrajectory), diagnostics.jl:176-186
                    break
                eng.leapfrog(1, sgn)
                st = eng.get_state(("q", "p", "lq"))
                out[sgn * i] = dict(z=dict(q=st["q"][0], p=st["p"][0], lq=float(st["lq"][0])),
                                    position=sgn * i, Δ=float(eng.phase_logdensity()[0] - π0))
    finally:
        eng.close()
    return [out[i] for i in sorted(out)]


def check_gradient(ℓ, q, h=1e-6, device=0):
    """∇ℓ of a device log density against central finite differences of its ℓ — both evaluated ON THE DEVICE (the first
    thing to run on a new user model header, include/dhmc_models.h): 2·D + 1 chains of one engine hold q and q ± h·eᵢ.
    Returns dict(grad=[D], fd=[D], max_abs_err, max_rel_err, lq).  (The reference leaves this to the user's AD backend.)"""
    from . import api
    q = np.asarray(q, float).ravel()
    D = q.size
    Q = np.repeat(q[None, :], 2 * D + 1, axis=0)
    for i in range(D):
        Q[1 + 2 * i, i] += h
        Q[2 + 2 * i, i] -= h
    eng = api.Engine(ℓ, chains=2 * D + 1, seed=0, device=device)
    try:
        eng.set_position(Q)                                     # strict evaluate_ℓ at every point (hamiltonian.jl:202-217)
        st = eng.get_state(("lq", "grad"))
    finally:
        eng.close()
    lq = np.asarray(st["lq"], float)
    fd = (lq[1::2] - lq[2::2]) / (2 * h)
    g = np.asarray(st["grad"][0], float)
    err = np.abs(g - fd)
    return dict(grad=g, fd=fd, lq=float(lq[0]), max_abs_err=float(err.max()),
                max_rel_err=float((err / np.maximum(np.abs(fd), 1e-300)).max()))


def ess_rhat(draws, max_lag=0):
    """Numpy mirror of dhmc_ess_rhat_dev (include/dhmc.h): split-R̂ and ESS per parameter of `draws` [chains, N, D].
    Every chain is split in two halves (m = 2·chains sequences of n = N // 2 draws); W = mean within-sequence variance,
    var⁺ = (n−1)/n·W + var(sequence means); ρ̂_t = 1 − (W − mean_c acov_c(t)) / var⁺ with the biased autocovariance;
    τ = −1 + 2 Σ (ρ̂_2k + ρ̂_2k+1) over Geyer's initial monotone sequence; ESS = m·n / τ.  The quantities the reference's
    correctness tests take from MCMCDiagnosticTools.ess_rhat (test/sample-correctness_utilities.jl:40-43).  A sequence's
    mean is x₁ + mean(x − x₁), so constant sequences centre to exact zeros; a parameter whose sequences are all constant
    at one value (var⁺ = 0) gets R̂ = ESS = NaN, as in MCMCDiagnosticTools."""
    x = np.asarray(draws, float)
    K, N, D = x.shape
    n = N // 2
    L = max_lag if max_lag > 0 else 64
    L = max(1, min(L, n - 2))
    seq = np.stack([x[:, :n], x[:, n:2 * n]], axis=1).reshape(2 * K, n, D)     # sequence 2c = first half of chain c, 2c+1 = second
    m = 2 * K
    mu = seq[:, 0] + (seq - seq[:, :1]).mean(axis=1)          # [m, D]
    xc = seq - mu[:, None, :]
    acov = np.stack([(xc[:, : n - t] * xc[:, t:]).sum(axis=1) / n for t in range(L + 1)])   # [L+1, m, D]
    mean_var = acov[0].mean(axis=0) * n / (n - 1.0)
    var_plus = mean_var * (n - 1.0) / n + ((mu - mu[0]).var(axis=0, ddof=1) if m > 1 else 0.0)
    with np.errstate(invalid="ignore", divide="ignore"):
        rhat = np.sqrt(var_plus / mean_var)
        rho = 1.0 - (mean_var[None] - acov.mean(axis=1)) / var_plus[None]                  # [L+1, D]
    ess = np.full(D, np.nan)
    for d in np.flatnonzero(var_plus > 0):
        tau, prev = 0.0, np.inf
        for t in range(0, L, 2):
            pair = rho[t, d] + rho[t + 1, d]
            if not pair > 0:
                break
            pair = min(pair, prev)
            prev = pair
            tau += 2 * pair
        tau -= 1.0
        tau = max(tau, 1.0 / np.log10(m * n))
        ess[d] = m * n / tau
    return dict(rhat=rhat, ess=ess)
