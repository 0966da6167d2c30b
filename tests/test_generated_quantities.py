"""Generated quantities of user models (include/dhmc_models.h): functions of each draw that the streaming summary reports
beside the parameters, and dhmc_generated(_dev), which evaluates them at given points (include/dhmc.h).

The example is include/models/eight_schools_gq.h: eight_schools.h (θ = (μ, log τ, η₁…η_J)) with G = J + 1 quantities,
τ = exp(q₁) and the centred effects θ_j = q₀ + τ·q_{j+1} (j = 1 … J).  tests/gqhost is their host evaluator, compiled from the same
header with the oracle's flags.

CPU: the host evaluator against numpy; G = 0 for the stock library and for models without the part; the summary mirror
on [θ, g(θ)] against the exact definitions; the Python argument checks and the reference extension; the sm_90a SASS of
the stock and Rosenbrock libraries is that of the libraries without generated quantities.
GPU: dhmc_generated(_dev) equals the host evaluator bit for bit; sampling is untouched by the part; the summary's D + G
rows are a drop-in for mcmc plus the mirror (thinned batch with a reference, ragged batch, deep twin, Symmetric metric);
shards merge; a halted chain is left out of the generated rows; bracketed quantiles of τ and θ_j end to end."""
import ctypes as C
import hashlib
import json
import math
import os
import subprocess
import zlib
from fractions import Fraction

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODELS = os.path.join(ROOT, "include", "models")
GQ = os.path.join(MODELS, "eight_schools_gq.h")
PLAIN = os.path.join(MODELS, "eight_schools.h")
ROSENBROCK = os.path.join(MODELS, "rosenbrock.h")
GQHOST = os.path.join(ROOT, "tests", "gqhost", "build", "libgqhost_eight_schools_gq.so")   # __graft_entry__.build()
CUDA_BIN = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin")
STATS = ("mean", "sd", "mcse", "ess", "rhat")
RTOL = 1e-9             # the record against the mirror, as tests/test_streaming_summary.py
Y0 = np.array([28.0, 8, -3, 7, -1, 1, 18, 12])
S0 = np.array([15.0, 10, 16, 11, 9, 11, 10, 18])


# ------------------------------------------------------------------ host evaluator
def _host():
    lib = C.CDLL(GQHOST)
    lib.orc_user_ngq.argtypes = [C.c_int]
    lib.orc_user_generated.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_void_p, C.c_void_p]
    return lib


def host_generated(theta, params):
    """g(θ) [..., G] of points θ [..., D] of one problem (parameter block `params`), on the CPU"""
    th = np.ascontiguousarray(theta, float)
    D = th.shape[-1]
    lib = _host()
    G = lib.orc_user_ngq(D)
    out = np.empty(th.shape[:-1] + (G,))
    pr = np.ascontiguousarray(params, float)
    lib.orc_user_generated(th.ctypes.data, th.size // D, D, pr.ctypes.data, out.ctypes.data)
    return out


def _schools_np(q):
    tau = np.exp(q[..., 1])
    return np.concatenate([tau[..., None], q[..., :1] + tau[..., None] * q[..., 2:]], axis=-1)


def test_host_evaluator_matches_numpy():
    rng = np.random.default_rng(1)
    for J in (1, 8, 33):
        q = rng.normal(size=(50, J + 2)) * np.r_[5.0, 1.0, np.ones(J)]
        got = host_generated(q, np.concatenate([rng.normal(size=J), rng.uniform(5, 20, J)]))
        want = _schools_np(q)
        assert got.shape == (50, J + 1)
        # τ to 1e-15 relative; θ_j = μ + τη_j to 1e-15 of the size of its terms (the sum may cancel)
        scale = np.concatenate([want[:, :1], np.abs(q[:, :1]) + np.abs(want[:, :1] * q[:, 2:])], axis=1)
        assert np.all(np.abs(got - want) <= 1e-15 * scale), np.max(np.abs(got - want) / scale)


# ------------------------------------------------------------------ G per library, without a GPU
def test_generated_count_per_library(pkg):
    L = pkg._lib
    G = C.c_int32(-1)
    assert L.lib().dhmc_user_generated_count(10, C.byref(G)) == L.DHMC_EARG      # the stock library: no user model
    assert L.lib().dhmc_generated_count(None, C.byref(G)) == L.DHMC_EARG
    assert pkg.UserLogDensity(ROSENBROCK, 6, deep=True).generated_count() == 0
    assert pkg.UserLogDensity(PLAIN, 10).generated_count() == 0
    assert pkg.UserLogDensity(GQ, 10, deep=True).generated_count() == 9
    assert pkg.UserLogDensity(GQ, 3, deep=True).generated_count() == 2
    assert "dhmc_generated" in L.EXPORTS and "dhmc_generated_dev" in L.EXPORTS


# ------------------------------------------------------------------ exact reference (test_streaming_summary.py's definitions)
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
    """statistics within RTOL (NaN where NaN), ranks and draw counts exactly"""
    for k in ("rank", "draws"):
        assert np.array_equal(got[k], want[k]), (ctx, k, got[k], want[k])
    for k in STATS:
        g, w = np.asarray(got[k], float), np.asarray(want[k], float)
        assert np.array_equal(np.isnan(g), np.isnan(w)), (ctx, k, g, w)
        scale = np.abs(w) + (np.nan_to_num(np.asarray(want["sd"], float)) if k == "mean" else 0.0)
        ok = np.isnan(w) | (g == w) | (np.abs(g - w) <= RTOL * scale)
        assert np.all(ok), (ctx, k, g[~ok], w[~ok])


# the edge cases of test_streaming_summary.py, with D ≥ 3 (eight schools) and log τ kept near 0 (exp of the large offset
# would overflow); the centred θ_j then carry the large offset
EDGE_CASES = {
    # name: (K, N, D, thin, chains_per_problem, chain_offset, P, offset, spread)
    "odd_n_keep": (6, 9, 3, 1, 0, 0, 1, 0.0, 1.0),
    "thin_3": (5, 30, 4, 3, 0, 0, 1, 0.0, 1.0),
    "n_keep_4": (4, 4, 3, 1, 0, 0, 1, 0.0, 1.0),
    "d_33": (3, 10, 33, 2, 0, 0, 1, 0.0, 1.0),
    "large_offset": (4, 12, 3, 1, 0, 0, 1, 1e8, 1e-3),
    "one_chain_per_problem": (5, 8, 3, 1, 1, 0, 5, 0.0, 1.0),
    "shard_inside_a_problem": (7, 10, 3, 2, 3, 4, 6, 0.0, 1.0),
}


@pytest.mark.parametrize("case", list(EDGE_CASES))
def test_mirror_on_generated_rows_matches_exact_definitions(pkg, case):
    K, N, D, thin, cpp, off, P, offset, spread = EDGE_CASES[case]
    rng = np.random.default_rng(zlib.crc32(case.encode()))
    x = offset + spread * rng.normal(size=(K, N, D)) + 0.3 * spread * rng.normal(size=(K, 1, D))
    x[..., 1] = spread * rng.normal(size=(K, N))
    pr = np.concatenate([Y0[:D - 2], S0[:D - 2]])
    xr = np.concatenate([x, host_generated(x, pr)], axis=2)                # [θ, g(θ)]: R = D + G = 2D − 1 rows
    assert xr.shape[2] == 2 * D - 1
    ref = offset + spread * rng.normal(size=(P, D))
    ref[:, 1] = 0.0
    ref = np.concatenate([ref, host_generated(ref, pr)], axis=1)
    d = pkg.diagnostics
    _close(d.finish_summary(d.summary_from_draws(xr, cpp, thin, ref, off, n_problems=P)), _exact(xr, cpp, thin, ref, off, P), case)
    lo, hi = ref - 0.5 * spread, ref + 0.5 * spread
    h = d.histogram_from_draws(xr, lo, hi, 8, cpp, thin, off, P)
    assert h.shape == (P, 2 * D - 1, 10) and np.array_equal(h.sum(axis=2), _exact(xr, cpp, thin, ref, off, P)["draws"])


# ------------------------------------------------------------------ Python checks, without a GPU
class _FakeLib:
    """the real library, with dhmc_generated answered by the host evaluator and the summary calls recorded (an Engine
    shell without a handle: the Python layer's arguments, not the device, are under test)"""

    def __init__(self, real, params, P, D, R):
        self.real, self.params, self.P, self.D, self.R, self.calls = real, params, P, D, R, []

    def __getattr__(self, name):
        return getattr(self.real, name)

    @staticmethod
    def _arr(ptr, n):
        return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_double)), (n,)).copy()

    def dhmc_generated(self, h, theta, n, first, n_problems, out):
        th = self._arr(theta, n * n_problems * self.D).reshape(n_problems, n, self.D)
        g = np.stack([host_generated(th[j], self.params[first + j]) for j in range(n_problems)])
        C.memmove(out, g.ctypes.data, g.nbytes)
        self.calls.append(("generated", n, first, n_problems))
        return 0

    def dhmc_mcmc_summary(self, h, N, thin, ref, record, st, ld):
        self.calls.append(("summary", None if ref is None else self._arr(ref, self.P * self.R).reshape(self.P, self.R)))
        return 0


def _shell(pkg, P, D=10, G=9):
    pr = [np.concatenate([Y0 + p, S0]) for p in range(P)]
    ℓs = [pkg.UserLogDensity(GQ, D, params=pr[p], deep=True) for p in range(P)]
    eng = object.__new__(pkg.Engine)
    eng.K, eng.D, eng._h, eng.chain_offset = 2 * P, D, None, 0
    eng.ℓ = pkg.ProblemBatch(ℓs, 2) if P > 1 else ℓs[0]
    eng._G = G
    eng._lib = _FakeLib(pkg._lib.lib(ℓs[0].library_path), pr, P, D, D + G)
    return eng


def test_python_argument_checks_without_gpu(pkg):
    P, D, G = 3, 10, 9
    eng = _shell(pkg, P)
    rng = np.random.default_rng(5)
    ref = rng.normal(size=(P, D))
    out = eng.mcmc_summary(8, reference=ref)
    assert out["mean"].shape == (P, D + G) and out["record"].shape == (P, D + G, pkg._lib.SUMMARY_FIELDS)
    (kind, n, first, n_problems), (_, sent) = eng._lib.calls
    assert (kind, n, first, n_problems) == ("generated", 1, 0, P)           # one device call for the P references
    want = np.concatenate([ref, np.stack([host_generated(ref[p], eng._lib.params[p]) for p in range(P)])], axis=1)
    assert sent.tobytes() == want.tobytes()                                  # [P, D] is extended with g(reference)
    eng._lib.calls.clear()
    full = rng.normal(size=(P, D + G))
    eng.mcmc_summary(8, reference=full)
    assert len(eng._lib.calls) == 1 and eng._lib.calls[0][1].tobytes() == full.tobytes()   # [P, D + G] as given
    for bad in (rng.normal(size=(P, D - 1)), rng.normal(size=(P, D + 1)), rng.normal(size=(P + 1, D)),
                rng.normal(size=(P, D + G + 1)), rng.normal(size=(D,))):
        with pytest.raises(pkg.ArgumentError, match="reference"):
            eng.mcmc_summary(8, reference=bad)
    lo, hi = np.zeros((P, D)), np.ones((P, D))
    with pytest.raises(pkg.ArgumentError, match="grid"):                     # the grid covers all R rows
        eng.mcmc_summary(8, quantiles=[0.5], grid=(lo, hi))
    # generated: the posterior layout of mcmc (whole problems: one call), one point per problem, one problem
    eng._lib.calls.clear()
    post = rng.normal(size=(2 * P, 5, D))
    g = eng.generated(post)
    assert eng._lib.calls == [("generated", 10, 0, P)] and g.shape == (2 * P, 5, G)
    for k in range(2 * P):
        assert g[k].tobytes() == host_generated(post[k], eng._lib.params[k // 2]).tobytes()
    assert eng.generated(post[0, 0], problem=2).tobytes() == host_generated(post[0, 0], eng._lib.params[2]).tobytes()
    for bad, kw in ((rng.normal(size=(P, D + 1)), {}), (rng.normal(size=(P + 1, D)), {}), (post[:3], {}),
                    (post[0, 0], dict(problem=P)), (post[0, 0], dict(problem=-1))):
        with pytest.raises(pkg.ArgumentError):
            eng.generated(bad, **kw)
    # a model without the part: no generated rows, and generated is refused before the library is called
    plain = _shell(pkg, 1, G=0)
    plain._lib.calls.clear()
    with pytest.raises(pkg.ArgumentError, match="no generated quantities"):
        plain.generated(np.zeros(D))
    with pytest.raises(pkg.ArgumentError, match="reference"):
        plain.mcmc_summary(8, reference=np.zeros((1, D + G)))
    assert plain._lib.calls == []


# ------------------------------------------------------------------ SASS of the libraries without generated quantities
def _sass_sha(so):
    out = subprocess.run([os.path.join(CUDA_BIN, "cuobjdump"), "-sass", so], check=True, capture_output=True, text=True).stdout
    body = "\n".join(l for l in out.splitlines() if not l.startswith("Fatbin") and "code for sm_" not in l)
    return hashlib.sha256(body.encode()).hexdigest()


def test_sass_of_libraries_without_generated_quantities_is_unchanged(pkg):
    """The part is compiled only into a library whose model declares it: the sm_90a code of the stock library and of the
    (deep) Rosenbrock library is byte for byte that of the build before generated quantities existed (CUDA 12.9 nvcc,
    csrc/Makefile flags; tests/golden/sass_without_generated_quantities.json)."""
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "sass_without_generated_quantities.json")))
    ver = subprocess.run([os.path.join(CUDA_BIN, "nvcc"), "--version"], check=True, capture_output=True, text=True).stdout
    if golden["nvcc"] not in ver:
        pytest.skip(f"the golden SASS digests are of nvcc {golden['nvcc']}")
    assert _sass_sha(pkg._lib.LIB_PATH) == golden["libdhmc_b200.so"]
    assert _sass_sha(pkg.compile_user_model(ROSENBROCK, deep=True)) == golden["rosenbrock-deep"]


# ------------------------------------------------------------------ GPU
def _schools(pkg, P, header=GQ, ragged=False, seed=8):
    """P eight-schools problems with their own (y, σ); build() compiles eight_schools_gq.h with the deep kernels"""
    rng = np.random.default_rng(seed)
    return [pkg.UserLogDensity(header, 10, deep=header == GQ,
                               params=np.concatenate([Y0 + rng.normal(size=8) * 5, S0 * rng.uniform(0.7, 1.3, 8)] +
                                                     ([np.zeros(3 * p + 1)] if ragged else [])))
            for p in range(P)]


def _engine(pkg, ℓ, K, eps, seed=31, **kw):
    eng = pkg.Engine(ℓ, chains=K, seed=seed, **kw)
    eng.random_position()
    eng.set_stepsize(eps)
    return eng


def _same_bits(a, b):
    return np.asarray(a).tobytes() == np.asarray(b).tobytes()


def _host_of_draws(post, problems, cpp, off=0):
    """[K, N, G]: g of every draw of chain k with the parameter block of its problem"""
    return np.stack([host_generated(post[k], problems[(off + k) // cpp if cpp else 0].params()) for k in range(post.shape[0])])


@pytest.mark.gpu
def test_generated_equals_host_evaluator(pkg):
    import torch
    probs = _schools(pkg, 3)
    batch = pkg.ProblemBatch(probs, 4)
    eng = _engine(pkg, batch, batch.chains, 0.2)
    try:
        assert eng.generated_count == 9
        post = eng.mcmc(12)["posterior_matrix"]                               # [K, N, D] = column-major [D, N, K]
        want = _host_of_draws(post, probs, 4)
        got = eng.generated(post)
        assert _same_bits(got, want)
        dev = torch.from_numpy(post).cuda()
        out = torch.empty((12, 12, 9), dtype=torch.float64, device="cuda")
        n0 = eng.kernel_launches()
        eng._ck(eng._lib.dhmc_generated_dev(eng._h, C.c_void_p(dev.data_ptr()), 4 * 12, 0, 3, C.c_void_p(out.data_ptr())))
        assert eng.kernel_launches() == n0 + 1 and _same_bits(out.cpu().numpy(), want)
        # one problem of the batch, and the per-problem references [D, P] (n = 1)
        assert _same_bits(eng.generated(post[4:8], problem=1), want[4:8])
        ref = post[::4, 0]
        assert _same_bits(eng.generated(ref), np.stack([host_generated(ref[p], probs[p].params()) for p in range(3)]))
        # checks before anything runs
        L = pkg._lib
        n0 = eng.kernel_launches()
        o = np.empty(9 * 4)
        for n, first, npr, th, ot in ((1, 0, 4, post, o), (1, -1, 1, post, o), (1, 3, 1, post, o), (0, 0, 1, post, o),
                                      (1, 0, 1, None, o), (1, 0, 1, post, None)):
            assert eng._lib.dhmc_generated(eng._h, L.ptr(th), n, first, npr, L.ptr(ot)) == L.DHMC_EARG, (n, first, npr)
        assert eng.kernel_launches() == n0
    finally:
        eng.close()
    eng = _engine(pkg, pkg.StandardNormal(4), 8, 0.5)
    try:
        assert eng.generated_count == 0
        o = np.empty(4)
        assert eng._lib.dhmc_generated(eng._h, pkg._lib.ptr(np.zeros(4)), 1, 0, 1, pkg._lib.ptr(o)) == pkg._lib.DHMC_EARG
    finally:
        eng.close()


@pytest.mark.gpu
def test_sampling_is_untouched_by_generated_quantities(pkg):
    """the eight_schools_gq and eight_schools libraries: bit-identical draws, statistics, final state and transition counts
    from one seed, with mcmc and with the summary (whose parameter rows need no generated quantity)"""
    outs = []
    for hdr in (GQ, PLAIN):
        probs = _schools(pkg, 3, header=hdr)
        batch = pkg.ProblemBatch(probs, 8)
        eng = _engine(pkg, batch, batch.chains, 0.25, seed=44)
        try:
            ck = eng.checkpoint()
            run = eng.mcmc(20)
            st = eng.get_state(("q", "lq", "grad", "eps"))
            t = eng.transition_count
            eng.restore(ck)
            summ = eng.mcmc_summary(20, thin=2, stats=True)
            outs.append((run, st, t, eng.get_state(("q", "lq", "grad", "eps")), eng.transition_count, summ))
        finally:
            eng.close()
    (ra, sa, ta, sa2, ta2, ma), (rb, sb, tb, sb2, tb2, mb) = outs
    for f in ("posterior_matrix", "tree_statistics", "logdensities"):
        assert _same_bits(ra[f], rb[f]), f
    for f in sa:
        assert _same_bits(sa[f], sb[f]) and _same_bits(sa2[f], sb2[f]) and _same_bits(sa[f], sa2[f]), f
    assert ta == tb == ta2 == tb2
    assert _same_bits(ma["tree_statistics"], mb["tree_statistics"]) and _same_bits(ma["logdensities"], mb["logdensities"])
    assert ma["mean"].shape == (3, 19) and mb["mean"].shape == (3, 10)
    assert np.array_equal(ma["draws"][:, :10], mb["draws"])


def _narrow_grid(x, cpp, P, thin):
    x = np.asarray(x)[:, thin - 1::thin]
    K, _, R = x.shape
    prob = np.arange(K) // cpp if cpp else np.zeros(K, int)
    lo, hi = np.empty((P, R)), np.empty((P, R))
    for p in range(P):
        v = x[prob == p].reshape(-1, R)
        lo[p], hi[p] = np.quantile(v, 0.3, axis=0), np.quantile(v, 0.7, axis=0)
        hi[p] = np.maximum(hi[p], lo[p] + 1e-9 * (1.0 + np.abs(lo[p])))
    return lo, hi


def _drop_in(pkg, eng, problems, N, thin=1, reference=None, cpp=0, P=1, bins=None, ctx=""):
    """mcmc from a checkpoint, then mcmc_summary from the same checkpoint: same state, statistics and transition count bit
    for bit; all R = D + G rows equal the mirror on [θ, g(θ)], and with `bins` the histogram of every row equals the
    mirror's as integers"""
    ck = eng.checkpoint()
    t0 = eng.transition_count
    run = eng.mcmc(N)
    s1, t1 = eng.get_state(("q", "lq", "grad", "eps")), eng.transition_count
    post = run["posterior_matrix"]
    xr = np.concatenate([post, _host_of_draws(post, problems, cpp)], axis=2)
    R = xr.shape[2]
    kw = {}
    if bins:
        lo, hi = _narrow_grid(xr, cpp, P, thin)
        kw = dict(quantiles=(0.05, 0.5, 0.95), grid=(lo, hi), bins=bins)
    eng.restore(ck)
    summ = eng.mcmc_summary(N, thin=thin, reference=reference, stats=True, **kw)
    s2, t2 = eng.get_state(("q", "lq", "grad", "eps")), eng.transition_count
    assert t1 == t2 == t0 + N, ctx
    for f in s1:
        assert _same_bits(s1[f], s2[f]), (ctx, f)
    assert _same_bits(run["tree_statistics"][:, thin - 1::thin], summ["tree_statistics"]), ctx
    assert _same_bits(run["logdensities"][:, thin - 1::thin], summ["logdensities"]), ctx
    d = pkg.diagnostics
    ref = None
    if reference is not None:
        ref = np.asarray(reference, float)
        if ref.shape[1] == eng.D:
            ref = np.concatenate([ref, np.stack([host_generated(ref[p], problems[p].params()) for p in range(P)])], axis=1)
    assert summ["record"].shape == (P, R, pkg._lib.SUMMARY_FIELDS), ctx
    _close(summ, d.finish_summary(d.summary_from_draws(xr, cpp, thin, ref, 0, n_problems=P)), ctx)
    if bins:
        want = d.histogram_from_draws(xr, lo, hi, bins, cpp, thin, 0, P)
        assert summ["histogram"].shape == (P, R, bins + 2) and np.array_equal(summ["histogram"], want), ctx
        assert np.all(want[..., 0] > 0) and np.all(want[..., -1] > 0), ctx
    return summ


@pytest.mark.gpu
def test_drop_in_thinned_batch_with_reference(pkg):
    probs = _schools(pkg, 5)
    batch = pkg.ProblemBatch(probs, 4)
    eng = _engine(pkg, batch, batch.chains, 0.2)
    rng = np.random.default_rng(1)
    ref = rng.normal(size=(5, 10))
    try:
        s = _drop_in(pkg, eng, probs, 40, thin=5, reference=ref, cpp=4, P=5, ctx="batch-ref")
        assert np.all(s["draws"] == 8 * 4) and np.all((s["rank"] >= 0) & (s["rank"] <= 32))
        full = np.concatenate([ref, rng.normal(size=(5, 9))], axis=1)           # [P, D + G] taken as given
        _drop_in(pkg, eng, probs, 40, thin=5, reference=full, cpp=4, P=5, bins=16, ctx="batch-ref-full")
    finally:
        eng.close()


@pytest.mark.gpu
def test_drop_in_ragged_batch(pkg):
    probs = _schools(pkg, 4, ragged=True)
    batch = pkg.RaggedProblemBatch(probs, 6)
    eng = _engine(pkg, batch, batch.chains, 0.2)
    try:
        _drop_in(pkg, eng, probs, 16, thin=2, reference=np.zeros((4, 10)), cpp=6, P=4, bins=24, ctx="ragged")
    finally:
        eng.close()


@pytest.mark.gpu
def test_drop_in_deep_twin(pkg):
    probs = _schools(pkg, 1)
    eng = _engine(pkg, probs[0], 64, 0.05, algorithm=pkg.NUTS(max_depth=14))
    try:
        _drop_in(pkg, eng, probs, 8, bins=5, ctx="deep")
    finally:
        eng.close()


@pytest.mark.gpu
def test_drop_in_symmetric_metric(pkg):
    probs = _schools(pkg, 1)
    rng = np.random.default_rng(2)
    A = rng.normal(size=(10, 10)) / np.sqrt(10)
    eng = _engine(pkg, probs[0], 96, 0.2)
    try:
        eng.set_metric_dense(0.3 * (A @ A.T) + np.eye(10))
        assert eng.metric_is_dense()
        _drop_in(pkg, eng, probs, 9, reference=rng.normal(size=(1, 10)), bins=64, ctx="dense")
    finally:
        eng.close()


@pytest.mark.gpu
def test_shards_merge_on_all_rows(pkg):
    """two handles split a batch inside a problem; merged records give the one-handle summary on all D + G rows, and the
    generated rows' histograms add up"""
    probs = _schools(pkg, 4, seed=12)
    batch = pkg.ProblemBatch(probs, 4)
    rng = np.random.default_rng(3)
    ref = rng.normal(size=(4, 10))
    lo = np.concatenate([np.full((4, 10), -2.0), np.zeros((4, 1)), np.full((4, 8), -10.0)], axis=1)
    hi = np.concatenate([np.full((4, 10), 2.0), np.full((4, 1), 15.0), np.full((4, 8), 25.0)], axis=1)
    N, thin, cut = 24, 2, 6                                       # chains 4, 5 | 6, 7 of problem 1
    outs = []
    for off, K in ((0, batch.chains), (0, cut), (cut, batch.chains - cut)):
        eng = _engine(pkg, batch, K, 0.2, chain_offset=off)
        try:
            outs.append(eng.mcmc_summary(N, thin=thin, reference=ref, quantiles=(0.1, 0.9), grid=(lo, hi), bins=24))
        finally:
            eng.close()
    whole, a, b = outs
    L = pkg._lib
    rec = a["record"].copy()
    assert rec.shape == (4, 19, L.SUMMARY_FIELDS)
    assert L.lib().dhmc_summary_merge(L.ptr(rec), L.ptr(b["record"]), 19, 4) == 0
    _close(pkg.diagnostics.finish_summary(rec), whole, "shards")
    assert np.array_equal(a["histogram"] + b["histogram"], whole["histogram"])
    assert np.all(a["histogram"][2:] == 0) and np.all(b["histogram"][:1] == 0)
    assert np.all(whole["histogram"][:, 10:].sum(axis=2) == whole["draws"][:, 10:])


@pytest.mark.gpu
def test_halted_chain_is_left_out_of_generated_rows(pkg):
    """min_Δ = −∞: chain 3 starts with η₃ = 1.5e153 (η₃² is finite) and step 5; its first leaf lands where η² overflows, is
    not divergent, and the next leapfrog would start from ℓ = −∞: the chain stops with DHMC_CHAIN_LEAPFROG_NONFINITE (the
    oracle's tree from this start halts, seed 5, chain 3, transition 0).  The generated rows leave it out as the parameter
    rows do."""
    K, D, N = 16, 10, 8
    probs = _schools(pkg, 1)
    rng = np.random.default_rng(90)
    q = rng.normal(size=(K, D)) * 0.5
    q[3] = 0.0
    q[3, 4] = 1.5e153
    eps = np.full(K, 0.2)
    eps[3] = 5.0
    eng = pkg.Engine(probs[0], chains=K, seed=5, algorithm=pkg.NUTS(min_Δ=-np.inf))
    try:
        eng.set_position(q)
        eng.set_stepsize(eps)
        ck = eng.checkpoint()
        L = pkg._lib
        post, st, ld = np.empty((K, N, D)), np.zeros((K, N), dtype=L.tree_stats_dtype), np.empty((K, N))
        rc = eng._lib.dhmc_mcmc(eng._h, N, L.ptr(post), L.ptr(st), L.ptr(ld))
        status = eng.chain_status()
        assert rc == L.DHMC_ENUMERIC and status[3] == L.DHMC_CHAIN_LEAPFROG_NONFINITE and np.all(np.delete(status, 3) == 0)
        ref = np.zeros((1, D))
        eng.restore(ck)
        xr = np.concatenate([post, _host_of_draws(post, probs, 0)], axis=2)
        lo, hi = _narrow_grid(xr[status == 0], 0, 1, 1)
        with pytest.raises(pkg.ArgumentError, match="leapfrog called from non-finite log density") as e:
            eng.mcmc_summary(N, reference=ref, quantiles=(0.5,), grid=(lo, hi), bins=16)
        summ = e.value.debug_information["summary"]
        assert np.all(summ["record"][..., L.SUMMARY_CHAINS] == K - 1) and np.all(summ["draws"] == N * (K - 1))
        refr = np.concatenate([ref, host_generated(ref, probs[0].params())], axis=1)
        d = pkg.diagnostics
        _close(summ, d.finish_summary(d.summary_from_draws(xr, 0, 1, refr, completed=status == 0)), "halted")
        assert np.array_equal(summ["histogram"], d.histogram_from_draws(xr, lo, hi, 16, completed=status == 0))
    finally:
        eng.close()


@pytest.mark.gpu
def test_end_to_end_quantiles_of_tau_and_school_effects(pkg):
    """summarize_with_warmup on 64 eight-schools problems: the pilot grid covers the generated rows too, and τ and every
    θ_j get finite brackets around their quantiles"""
    probs = _schools(pkg, 64, seed=21)
    batch = pkg.ProblemBatch(probs, 8)
    out = pkg.summarize_with_warmup(79, batch, 400, quantiles=(0.05, 0.5, 0.95))
    assert out["quantile"].shape == (64, 19, 3) and out["grid"][0].shape == (64, 19)
    g = slice(10, 19)
    for k in ("quantile", "quantile_lo", "quantile_hi"):
        assert np.all(np.isfinite(out[k][:, g])), k
    assert np.all(out["quantile_lo"][:, g] <= out["quantile"][:, g]) and np.all(out["quantile"][:, g] <= out["quantile_hi"][:, g])
    assert np.all(out["quantile"][:, 10] > 0)                                        # τ
    assert np.all(out["histogram"][:, g].sum(axis=2) == out["draws"][:, g]) and np.all(out["draws"] == 400 * 8)
