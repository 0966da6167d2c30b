"""Host-side mirror of DynamicHMC.Diagnostics (src/diagnostics.jl) over the returned
tree-statistics arrays, plus access to the device-side reduction (dhmc_tree_summary_dev)
that avoids shipping 56 B × N × chains of statistics to the host (SURVEY.md §8f item 2)."""
from dataclasses import dataclass

import numpy as np

from . import _lib as L

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


# ------------------------------------------------------------------ streaming posterior summary
# Numpy mirror of dhmc_mcmc_summary / dhmc_summary_merge / dhmc_summary_finish (include/dhmc.h, DESIGN.md §4.4): the
# definitions the tests check the device against, and the merge path for shards gathered with torch.distributed.  A record
# is [P, D, SUMMARY_FIELDS] (numpy order; the C ABI's column-major [F, D, P]) of mergeable quantities.
def summary_from_draws(draws, chains_per_problem=0, thin=1, reference=None, chain_offset=0, n_problems=None,
                       completed=None):
    """The record dhmc_mcmc_summary folds on the device, from draws [K, N, D] of all N transitions (every thin-th is kept).
    Chain k of this shard is global chain chain_offset + k and samples problem (chain_offset + k) // chains_per_problem
    (chains_per_problem = 0: one problem).  `reference` [P, D] adds the rank counts; `completed` [K] (bool) leaves the
    chains that failed out.  P defaults to reference's rows, else to the problems the shard reaches."""
    from .api import _argcheck
    x = np.asarray(draws, float)
    _argcheck(x.ndim == 3, "draws: [chains, N, D]")
    K, N, D = x.shape
    _argcheck(thin >= 1 and N % thin == 0 and N // thin >= 4, "thin ≥ 1, N a multiple of thin, N / thin ≥ 4")
    x = x[:, thin - 1::thin]
    n_keep = x.shape[1]
    n = n_keep // 2
    cpp = int(chains_per_problem or 0)
    if reference is not None:
        reference = np.asarray(reference, float)
        _argcheck(reference.ndim == 2 and reference.shape[1] == D, "reference: [P, D]")
    if cpp:
        P = int(n_problems if n_problems is not None else
                reference.shape[0] if reference is not None else -(-(chain_offset + K) // cpp))
        prob = (chain_offset + np.arange(K)) // cpp
    else:
        P, prob = 1, np.zeros(K, dtype=np.int64)
    _argcheck(reference is None or reference.shape[0] == P, "reference: [P, D]")
    ok = np.ones(K, bool) if completed is None else np.asarray(completed, bool)
    rec = np.zeros((P, D, L.SUMMARY_FIELDS))
    rec[..., L.SUMMARY_NKEEP] = n_keep
    rec[..., L.SUMMARY_BELOW] = np.nan if reference is None else 0.0
    for p in range(P):
        idx = np.flatnonzero((prob == p) & ok)
        M = idx.size
        rec[p, :, L.SUMMARY_CHAINS] = M
        if M == 0:
            continue
        s = x[idx[0], 0]                                                  # shift: everything below is relative to one draw,
        seq = np.stack([x[idx, :n], x[idx, n:2 * n]], axis=1) - s         # so a large common offset cancels exactly [M, 2, n, D]
        mu = seq.mean(axis=2)                                             # [M, 2, D] sequence means
        mbar = mu.mean(axis=(0, 1))
        muc = 0.5 * (mu[:, 0] + mu[:, 1])                                 # chain means over 2n draws
        rec[p, :, L.SUMMARY_MEAN] = s + mbar
        rec[p, :, L.SUMMARY_SS_SEQ] = ((mu - mbar) ** 2).sum(axis=(0, 1))
        rec[p, :, L.SUMMARY_M2] = ((seq - mu[:, :, None]) ** 2).sum(axis=(0, 1, 2))
        rec[p, :, L.SUMMARY_SS_CHAIN] = ((muc - mbar) ** 2).sum(axis=0)
        if reference is not None:
            rec[p, :, L.SUMMARY_BELOW] = (x[idx] < reference[p]).sum(axis=(0, 1))
    return rec


def merge_summaries(*records):
    """dhmc_summary_merge over any number of records of the same [P, D]: the record of all their chains (Chan, Golub and
    LeVeque's pairwise update of means and centred sums of squares; counts add)."""
    from .api import _argcheck
    out = np.array(records[0], float, copy=True)
    for r in records[1:]:
        r = np.asarray(r, float)
        _argcheck(r.shape == out.shape, "records of the same [P, D]")
        ma, mb = out[..., L.SUMMARY_CHAINS], r[..., L.SUMMARY_CHAINS]
        both = (ma > 0) & (mb > 0)
        _argcheck(np.all(out[..., L.SUMMARY_NKEEP][both] == r[..., L.SUMMARY_NKEEP][both]),
                  "records of runs with the same number of kept draws per chain")
        below = out[..., L.SUMMARY_BELOW] + r[..., L.SUMMARY_BELOW]
        take = (ma == 0) & (mb > 0)
        out[take] = r[take]
        M = ma + mb
        with np.errstate(invalid="ignore", divide="ignore"):
            delta = r[..., L.SUMMARY_MEAN] - out[..., L.SUMMARY_MEAN]
            mean = out[..., L.SUMMARY_MEAN] + delta * (mb / M)
            ss = out[..., L.SUMMARY_SS_SEQ] + r[..., L.SUMMARY_SS_SEQ] + delta * delta * (2.0 * ma * mb / M)
            ssc = out[..., L.SUMMARY_SS_CHAIN] + r[..., L.SUMMARY_SS_CHAIN] + delta * delta * (ma * mb / M)
        out[..., L.SUMMARY_MEAN] = np.where(both, mean, out[..., L.SUMMARY_MEAN])
        out[..., L.SUMMARY_SS_SEQ] = np.where(both, ss, out[..., L.SUMMARY_SS_SEQ])
        out[..., L.SUMMARY_SS_CHAIN] = np.where(both, ssc, out[..., L.SUMMARY_SS_CHAIN])
        out[..., L.SUMMARY_M2] = np.where(both, out[..., L.SUMMARY_M2] + r[..., L.SUMMARY_M2], out[..., L.SUMMARY_M2])
        out[..., L.SUMMARY_CHAINS] = np.where(both, M, out[..., L.SUMMARY_CHAINS])
        out[..., L.SUMMARY_BELOW] = below
    return out


def finish_summary(record):
    """dhmc_summary_finish: mean, sd, mcse, ess, rhat [P, D] (float), rank and draws [P, D] (int64; rank −1 without a
    reference) from a record.  Definitions in include/dhmc.h; ess is a between-chain batch-means estimate, not the Geyer
    ESS of ess_rhat."""
    r = np.asarray(record, float)
    M = r[..., L.SUMMARY_CHAINS]
    m, n = 2.0 * M, np.floor(r[..., L.SUMMARY_NKEEP] / 2.0)
    ss, m2 = r[..., L.SUMMARY_SS_SEQ], r[..., L.SUMMARY_M2]
    none = M == 0
    with np.errstate(invalid="ignore", divide="ignore"):
        var = (m2 + n * ss) / (m * n - 1.0)
        W = m2 / (m * (n - 1.0))
        var_plus = (n - 1.0) / n * W + ss / (m - 1.0)
        var_c = r[..., L.SUMMARY_SS_CHAIN] / (M - 1.0) / M
        out = dict(mean=np.where(none, np.nan, r[..., L.SUMMARY_MEAN]), sd=np.where(none, np.nan, np.sqrt(var)),
                   rhat=np.where(none, np.nan, np.sqrt(var_plus / W)),
                   mcse=np.where(M >= 2, np.sqrt(var_c), np.nan),
                   ess=np.where((M >= 2) & (var_plus > 0), var / var_c, np.nan))
    below = r[..., L.SUMMARY_BELOW]
    out["rank"] = np.where(np.isnan(below), -1, np.nan_to_num(below)).astype(np.int64)
    out["draws"] = (r[..., L.SUMMARY_NKEEP] * M).astype(np.int64)
    return out


# ------------------------------------------------------------------ streaming quantiles
# Numpy mirror of dhmc_mcmc_summary_histogram's bin counts and of dhmc_histogram_quantiles (include/dhmc.h, DESIGN.md §4.4):
# the same IEEE operations in the same order, so counts agree as integers and quantiles bit for bit.  Counts are
# [P, D, bins + 2] int64 (numpy order; the C ABI's column-major [bins + 2, D, P]); bin 0 is below lo, bin bins + 1 at or
# above hi (and NaN).
MAX_BINS = 4096


def check_grid(lo, hi, bins, shape=None):
    """(lo, hi) as float arrays [P, D] after the checks of the C ABI: 1 ≤ bins ≤ 4096 and, per cell, finite lo < hi with
    hi − lo and bins / (hi − lo) finite."""
    from .api import _argcheck
    lo, hi = np.ascontiguousarray(lo, float), np.ascontiguousarray(hi, float)
    _argcheck(lo.ndim == 2 and lo.shape == hi.shape and (shape is None or lo.shape == tuple(shape)),
              f"grid: lo and hi of shape [P, D]{'' if shape is None else ' = ' + str(tuple(shape))}")
    _argcheck(int(bins) == bins and 1 <= bins <= MAX_BINS, f"bins: 1 … {MAX_BINS}")
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        w = hi - lo
        ok = np.isfinite(lo) & np.isfinite(hi) & (lo < hi) & np.isfinite(w) & np.isfinite(float(bins) / w)
    _argcheck(bool(np.all(ok)), "grid: finite lo < hi with hi − lo and bins / (hi − lo) finite in every cell")
    return lo, hi


def histogram_from_draws(draws, lo, hi, bins, chains_per_problem=0, thin=1, chain_offset=0, n_problems=None,
                         completed=None):
    """The bin counts [P, D, bins + 2] dhmc_mcmc_summary_histogram folds on the device, from draws [K, N, D] of all N
    transitions (every thin-th is kept), on the grid lo, hi [P, D].  Chains and problems as summary_from_draws; `completed`
    [K] (bool) leaves the chains that failed out.  P is the grid's number of rows."""
    from .api import _argcheck
    x = np.asarray(draws, float)
    _argcheck(x.ndim == 3, "draws: [chains, N, D]")
    K, N, D = x.shape
    _argcheck(thin >= 1 and N % thin == 0 and N // thin >= 4, "thin ≥ 1, N a multiple of thin, N / thin ≥ 4")
    lo, hi = check_grid(lo, hi, bins)
    bins = int(bins)
    P = lo.shape[0]
    _argcheck(lo.shape[1] == D and (n_problems is None or n_problems == P), "grid: [P, D]")
    x = x[:, thin - 1::thin]
    cpp = int(chains_per_problem or 0)
    prob = (chain_offset + np.arange(K)) // cpp if cpp else np.zeros(K, dtype=np.int64)
    ok = np.ones(K, bool) if completed is None else np.asarray(completed, bool)
    inv_w = float(bins) / (hi - lo)
    cells = bins + 2
    counts = np.zeros((P, D, cells), np.int64)
    for p in range(P):
        xs = x[(prob == p) & ok]                                            # [M, n_keep, D]
        with np.errstate(invalid="ignore", over="ignore"):
            t = (xs - lo[p]) * inv_w[p]                                     # rounded apart, as on the device
            inside = (t >= 0.0) & (t < bins)
        k = np.where(t < 0.0, 0, bins + 1)
        k[inside] = 1 + t[inside].astype(np.int64)
        flat = (k + cells * np.arange(D)).ravel()
        counts[p] = np.bincount(flat, minlength=D * cells).reshape(D, cells)
    return counts


def histogram_quantiles(counts, lo, hi, probs):
    """dhmc_histogram_quantiles: (q, q_lo, q_hi), each [P, D, len(probs)], of counts [P, D, bins + 2] on the grid lo, hi
    [P, D].  q is the type-7 quantile of the in-bin placements of the order statistics (NaN when one lies in a tail bin);
    the exact type-7 quantile of the counted values lies in [q_lo, q_hi] up to the rounding of the edges."""
    from .api import _argcheck
    c = np.asarray(counts)
    _argcheck(c.ndim == 3 and c.shape[2] >= 3 and np.issubdtype(c.dtype, np.integer) and np.all(c >= 0),
              "counts: [P, D, bins + 2] of non-negative integers")
    nb = c.shape[2] - 2
    lo, hi = check_grid(lo, hi, nb, c.shape[:2])
    probs = np.atleast_1d(np.asarray(probs, float))
    _argcheck(probs.ndim == 1 and np.all((probs >= 0.0) & (probs <= 1.0)), "0 ≤ p ≤ 1")
    cum = np.cumsum(c.astype(np.int64), axis=-1)
    n = cum[..., -1]
    w = (hi - lo) / float(nb)

    def edge(k):
        return np.where(k < nb, lo + k.astype(float) * w, hi)

    def bin_of(r):                                                          # the first bin k with r < C_k
        return (cum <= r[..., None]).sum(axis=-1)

    def place(r, k):
        kk = np.clip(k, 1, nb)
        below = np.take_along_axis(cum, (kk - 1)[..., None], -1)[..., 0]
        ck = np.take_along_axis(cum, kk[..., None], -1)[..., 0] - below
        with np.errstate(invalid="ignore", divide="ignore"):
            x = edge(kk - 1) + ((r - below).astype(float) + 0.5) / ck.astype(float) * (edge(kk) - edge(kk - 1))
        return np.where((k == 0) | (k == nb + 1), np.nan, x)

    shape = (*c.shape[:2], probs.size)
    q, q_lo, q_hi = np.empty(shape), np.empty(shape), np.empty(shape)
    empty = n == 0
    for i, alpha in enumerate(probs):
        pos = alpha * np.maximum(n - 1, 0).astype(float)
        j = pos.astype(np.int64)
        gamma = pos - j.astype(float)
        kj = bin_of(j)
        kh = np.where(gamma > 0.0, bin_of(j + 1), kj)
        xj = place(j, kj)
        with np.errstate(invalid="ignore"):
            qi = np.where(gamma > 0.0, xj + gamma * (place(j + 1, kh) - xj), xj)
        q[..., i] = np.where(empty, np.nan, qi)
        q_lo[..., i] = np.where(empty, np.nan, np.where(kj == 0, -np.inf, edge(np.maximum(kj - 1, 0))))
        q_hi[..., i] = np.where(empty, np.nan, np.where(kh == nb + 1, np.inf, edge(np.minimum(kh, nb))))
    return q, q_lo, q_hi


def quantile_grid(summary, width=6.0):
    """The pilot grid of summarize_with_warmup: lo, hi [P, D] = mean ∓ width·sd per (problem, parameter), from a summary
    (the dict of Engine.mcmc_summary / finish_summary) or a record [P, D, SUMMARY_FIELDS] (merged pilot records of shards
    give every rank the same grid).  A cell whose mean ± width·sd is not a valid grid (sd = 0, sd not finite, no chain)
    gets (c − s, c + s): c the mean (0 where it is not finite or |mean| > 1e300), s = max(1, |c|)."""
    s = summary if isinstance(summary, dict) else finish_summary(summary)
    mean, sd = np.asarray(s["mean"], float), np.asarray(s["sd"], float)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        lo, hi = mean - width * sd, mean + width * sd
        w = hi - lo
        ok = np.isfinite(lo) & np.isfinite(hi) & (lo < hi) & np.isfinite(w) & np.isfinite(float(MAX_BINS) / w)
    c = np.where(np.isfinite(mean) & (np.abs(mean) <= 1e300), mean, 0.0)
    half = np.maximum(1.0, np.abs(c))
    return np.where(ok, lo, c - half), np.where(ok, hi, c + half)
