"""Random generated quantities (include/dhmc_models.h DHMC_USER_GENERATED_RNG): posterior predictive replicates drawn on
the device from Philox streams of their own, keyed like the draws, and summarized like any other generated row.

The example is include/models/eight_schools_ppc.h: eight schools (θ = (μ, log τ, η₁…η_J), D = J + 2) with G = 2J + 4 rows,
τ, θ_j = μ + τη_j, the replicates y_rep_j = θ_j + σ_j·normal(j − 1) and three p-value indicators (max, min, χ²) that
re-derive y_rep from the same indices.  tests/gqkeyed is the keyed host evaluator, compiled from the same header.

CPU: the streams against an independent numpy Philox4x32-10 + Box–Muller and KS tests; the indicator rows against numpy;
the flag per library; the Python argument checks; the per-function sm_90a SASS of the deterministic eight_schools_gq
library is the parent's except k_generated.
GPU: dhmc_generated_keyed(_dev) equals the host evaluator bit for bit; sampling is untouched; the summary's rows are a
drop-in for mcmc plus the keyed host evaluator plus the mirror; a halted chain is left out; end to end on eight schools."""
import ctypes as C
import hashlib
import json
import math
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODELS = os.path.join(ROOT, "include", "models")
PPC = os.path.join(MODELS, "eight_schools_ppc.h")
GQ = os.path.join(MODELS, "eight_schools_gq.h")
PLAIN = os.path.join(MODELS, "eight_schools.h")
GQKEYED = os.path.join(ROOT, "tests", "gqkeyed", "build", "libgqkeyed_{}.so")   # __graft_entry__.build()
CUDA_BIN = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin")
STATS = ("mean", "sd", "mcse", "ess", "rhat")
RTOL = 1e-9
Y0 = np.array([28.0, 8, -3, 7, -1, 1, 18, 12])
S0 = np.array([15.0, 10, 16, 11, 9, 11, 10, 18])
STREAM_GQ_U, STREAM_GQ_N, STREAM_P = 5, 6, 2


# ------------------------------------------------------------------ keyed host evaluator
def _host(name="eight_schools_ppc"):
    lib = C.CDLL(GQKEYED.format(name))
    lib.orc_user_ngq.argtypes = [C.c_int]
    lib.orc_user_generated_keyed.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_void_p, C.c_ulonglong, C.c_void_p,
                                             C.c_void_p, C.c_void_p]
    lib.orc_gq_numbers.argtypes = [C.c_ulonglong, C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong, C.c_int, C.c_void_p]
    return lib


def host_keyed(theta, params, seed, chain, trans, name="eight_schools_ppc"):
    """g(θ) [..., G] of points θ [..., D] of one problem, point i keyed by (seed, chain[i]) and trans[i]"""
    th = np.ascontiguousarray(theta, float)
    D = th.shape[-1]
    lib = _host(name)
    G = lib.orc_user_ngq(D)
    out = np.empty(th.shape[:-1] + (G,))
    ch = np.ascontiguousarray(np.broadcast_to(chain, th.shape[:-1]), np.int64)
    tr = np.ascontiguousarray(np.broadcast_to(trans, th.shape[:-1]), np.uint32)
    pr = np.ascontiguousarray(params, float)
    lib.orc_user_generated_keyed(th.ctypes.data, th.size // D, D, pr.ctypes.data, seed, ch.ctypes.data, tr.ctypes.data,
                                 out.ctypes.data)
    return out


def host_numbers(seed, chain, trans, index, normal):
    ch, tr, ix = (np.ascontiguousarray(a, t) for a, t in ((chain, np.int64), (trans, np.uint32), (index, np.uint32)))
    out = np.empty(ch.size)
    _host().orc_gq_numbers(seed, ch.ctypes.data, tr.ctypes.data, ix.ctypes.data, ch.size, int(normal), out.ctypes.data)
    return out


# ------------------------------------------------------------------ numpy restatement of the streams (include/dhmc_math.h)
def _philox(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 on uint64 arrays holding 32-bit words"""
    M0, M1, W0, W1, m32 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85, 0xFFFFFFFF
    c0, c1, c2, c3 = (np.asarray(c, np.uint64) & m32 for c in (c0, c1, c2, c3))
    k0, k1 = np.uint64(k0), np.uint64(k1)
    for _ in range(10):
        p0, p1 = np.uint64(M0) * c0, np.uint64(M1) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & np.uint64(m32), (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & np.uint64(m32)
        k0, k1 = (k0 + np.uint64(W0)) & np.uint64(m32), (k1 + np.uint64(W1)) & np.uint64(m32)
    return c0, c1, c2, c3


def _u01(a, b):
    return ((a << np.uint64(20)) | (b >> np.uint64(12))).astype(np.float64) * 2.0 ** -52 + 2.0 ** -53


def np_numbers(seed, chain, trans, index, stream):
    """(uniform(i), normal(i)) of stream `stream` at keys (seed, chain, trans) and indices i, as dhmc_math.h defines them"""
    chain, index = np.asarray(chain, np.uint64), np.asarray(index, np.uint64)
    v = _philox(index >> np.uint64(1), trans, chain & np.uint64(0xFFFFFFFF),
                (np.uint64(stream) << np.uint64(24)) | ((chain >> np.uint64(32)) & np.uint64(0xFFFFFF)),
                seed & 0xFFFFFFFF, seed >> 32)
    odd = (index & np.uint64(1)) == 1
    u = np.where(odd, _u01(v[2], v[3]), _u01(v[0], v[1]))
    u1, u2 = _u01(v[0], v[1]), _u01(v[2], v[3])
    rad = np.sqrt(-2.0 * np.log(u1))
    z = np.where(odd, rad * np.sin(2 * np.pi * u2), rad * np.cos(2 * np.pi * u2))
    return u, z


def _keys(n, seed):
    rng = np.random.default_rng(seed)
    return (rng.integers(0, 2 ** 56, n, dtype=np.int64), rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32),
            rng.integers(0, 64, n).astype(np.uint32))


def test_streams_match_numpy_philox():
    seed = 0x1234_5678_9ABC_DEF0
    chain, trans, idx = _keys(5000, 1)
    u_np, _ = np_numbers(seed, chain, trans, idx, STREAM_GQ_U)
    _, z_np = np_numbers(seed, chain, trans, idx, STREAM_GQ_N)
    u = host_numbers(seed, chain, trans, idx, False)
    z = host_numbers(seed, chain, trans, idx, True)
    assert np.array_equal(u, u_np)                                         # exact: Philox and the 52-bit uniform
    assert np.all(np.abs(z - z_np) <= 1e-13 * (1.0 + np.abs(z_np)))       # Box–Muller: the library's log and sin/cos


def test_replicates_are_the_stream_normals():
    """(y_rep_j − θ_j)/σ_j of the keyed evaluator is normal(j − 1) of stream 6 at the draw's key"""
    J, D = 8, 10
    seed = 77
    rng = np.random.default_rng(2)
    n = 400
    chain = rng.integers(0, 2 ** 40, n)
    trans = rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32)
    q0 = np.zeros((n, D))
    q0[:, 1] = rng.normal(size=n)
    g0 = host_keyed(q0, np.concatenate([Y0, np.ones(J)]), seed, chain, trans)       # θ = 0, σ = 1: y_rep = normal exactly
    assert g0.shape == (n, 2 * J + 4) and np.all(g0[:, 1:J + 1] == 0.0)
    idx = np.tile(np.arange(J, dtype=np.uint32), n)
    ch, tr = np.repeat(chain, J), np.repeat(trans, J)
    z = host_numbers(seed, ch, tr, idx, True).reshape(n, J)
    assert np.array_equal(g0[:, J + 1:2 * J + 1], z)
    _, z_np = np_numbers(seed, ch, tr, idx, STREAM_GQ_N)
    assert np.all(np.abs(z - z_np.reshape(n, J)) <= 1e-13 * (1.0 + np.abs(z)))
    # general θ, σ: (y_rep − θ)/σ is the same normal up to the rounding of θ + σz
    q = rng.normal(size=(n, D)) * np.r_[5.0, 1.0, np.ones(J)]
    sig = S0 * rng.uniform(0.5, 2, J)
    g = host_keyed(q, np.concatenate([Y0, sig]), seed, chain, trans)
    th, rep = g[:, 1:J + 1], g[:, J + 1:2 * J + 1]
    assert np.all(np.abs((rep - th) / sig - z) <= 1e-14 * (np.abs(th) + np.abs(rep)) / sig + 1e-15)


def test_stream_distributions():
    """≥ 10⁵ keys, fixed seeds: normals pass a KS test against N(0, 1), uniforms against U(0, 1); they differ from the
    sampler's momentum normals (stream 2) at the same key, and uniforms and normals of one key are uncorrelated"""
    from scipy import stats
    for s in (3, 4):
        chain, trans, idx = _keys(100_000, s)
        z = host_numbers(11 + s, chain, trans, idx, True)
        u = host_numbers(11 + s, chain, trans, idx, False)
        assert stats.kstest(z, "norm").pvalue > 1e-3
        assert stats.kstest(u, "uniform").pvalue > 1e-3
        assert np.all((u > 0) & (u < 1))
        assert abs(np.corrcoef(u, z)[0, 1]) < 0.02
        assert abs(np.corrcoef(z[::2], z[1::2])[0, 1]) < 0.02


def test_normals_differ_from_momentum_stream(po):
    D = 16
    for seed, chain, t in ((1, 0, 0), (5, 3, 7), (2 ** 40 + 1, 2 ** 33 + 5, 2 ** 31)):
        mom = po.normals(seed, chain, STREAM_P, t, D)
        z = host_numbers(seed, np.full(D, chain), np.full(D, t), np.arange(D), True)
        assert np.all(mom != z)
        _, z_np = np_numbers(seed, np.full(D, chain), np.full(D, t), np.arange(D), STREAM_P)
        assert np.all(np.abs(mom - z_np) <= 1e-13 * (1.0 + np.abs(mom)))      # the restatement reads stream 2 too


def _indicators(th, rep, y, sig):
    """the three p-value indicators of eight_schools_ppc.h in numpy, summed in the header's order"""
    chi_rep = chi_y = 0.0
    for j in range(len(y)):
        zr, zy = (rep[j] - th[j]) / sig[j], (y[j] - th[j]) / sig[j]
        chi_rep, chi_y = chi_rep + zr * zr, chi_y + zy * zy
    return [float(np.max(rep) >= np.max(y)), float(np.min(rep) <= np.min(y)), float(chi_rep >= chi_y)]


def test_indicator_rows_match_numpy():
    rng = np.random.default_rng(6)
    for J in (1, 3, 8):
        D, n = J + 2, 300
        q = rng.normal(size=(n, D)) * np.r_[5.0, 1.0, np.ones(J)]
        y, sig = rng.normal(size=J) * 10, rng.uniform(5, 20, J)
        g = host_keyed(q, np.concatenate([y, sig]), 9, rng.integers(0, 1000, n), rng.integers(0, 10 ** 6, n))
        assert g.shape == (n, 2 * J + 4)
        want = np.array([_indicators(g[i, 1:J + 1], g[i, J + 1:2 * J + 1], y, sig) for i in range(n)])
        assert np.array_equal(g[:, 2 * J + 1:], want)
        assert 0 < want.mean() < 1
        # τ and θ_j are eight_schools_gq's, bit for bit
        gq = host_keyed(q, np.concatenate([y, sig]), 9, 0, 0, name="eight_schools_gq")
        assert np.array_equal(g[:, :J + 1], gq)


# ------------------------------------------------------------------ flags per library, without a GPU
def test_generated_random_per_library(pkg):
    L = pkg._lib
    r = C.c_int32(-1)
    assert L.lib().dhmc_user_generated_random(C.byref(r)) == L.DHMC_EARG           # the stock library: no user model
    assert L.lib().dhmc_generated_random(None, C.byref(r)) == L.DHMC_EARG
    assert pkg.UserLogDensity(PLAIN, 10).generated_random() == 0
    assert pkg.UserLogDensity(GQ, 10, deep=True).generated_random() == 0
    ppc = pkg.UserLogDensity(PPC, 10, deep=True)
    assert ppc.generated_random() == 1 and ppc.generated_count() == 20
    for name in ("dhmc_generated_random", "dhmc_user_generated_random", "dhmc_generated_keyed", "dhmc_generated_keyed_dev"):
        assert name in L.EXPORTS and hasattr(L.lib(ppc.library_path), name), name


# ------------------------------------------------------------------ Python checks, without a GPU
class _FakeLib:
    """the real library, with dhmc_generated_keyed answered by the keyed host evaluator and the other calls recorded (an
    Engine shell without a handle: the Python layer's arguments, not the device, are under test)"""

    def __init__(self, real, params, P, D, R, seed):
        self.real, self.params, self.P, self.D, self.R, self.seed, self.calls = real, params, P, D, R, seed, []

    def __getattr__(self, name):
        return getattr(self.real, name)

    @staticmethod
    def _arr(ptr, n, t=C.c_double):
        return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(t)), (n,)).copy()

    def dhmc_generated(self, h, theta, n, first, n_problems, out):
        self.calls.append(("generated",))
        return 2

    def dhmc_generated_keyed(self, h, theta, n, first, n_problems, chain, trans, out):
        m = n * n_problems
        th = self._arr(theta, m * self.D).reshape(n_problems, n, self.D)
        ch, tr = self._arr(chain, m, C.c_int64).reshape(n_problems, n), self._arr(trans, m, C.c_uint32).reshape(n_problems, n)
        g = np.stack([host_keyed(th[j], self.params[first + j], self.seed, ch[j], tr[j]) for j in range(n_problems)])
        C.memmove(out, g.ctypes.data, g.nbytes)
        self.calls.append(("keyed", n, first, n_problems))
        return 0

    def dhmc_mcmc_summary(self, h, N, thin, ref, record, st, ld):
        self.calls.append(("summary", None if ref is None else self._arr(ref, self.P * self.R).reshape(self.P, self.R)))
        return 0


def _shell(pkg, P, D=10, seed=3):
    pr = [np.concatenate([Y0 + p, S0]) for p in range(P)]
    ℓs = [pkg.UserLogDensity(PPC, D, params=pr[p], deep=True) for p in range(P)]
    eng = object.__new__(pkg.Engine)
    eng.K, eng.D, eng._h, eng.chain_offset = 2 * P, D, None, 0
    eng.ℓ = pkg.ProblemBatch(ℓs, 2) if P > 1 else ℓs[0]
    eng._G, eng._GR = 2 * D, 1
    eng._lib = _FakeLib(pkg._lib.lib(ℓs[0].library_path), pr, P, D, 3 * D, seed)
    return eng


def test_python_argument_checks_without_gpu(pkg):
    P, D, G, seed = 3, 10, 20, 3
    eng = _shell(pkg, P, seed=seed)
    assert eng.generated_random == 1
    rng = np.random.default_rng(5)
    post = rng.normal(size=(2 * P, 5, D))
    # keys are required, and their shapes and ranges are checked, before the library is called
    for kw in ({}, dict(keys=(0,)), dict(keys=(np.zeros(3, int), 0)), dict(keys=(np.zeros((2 * P, 4), int), 0)),
               dict(keys=(-1, 0)), dict(keys=(2 ** 56, 0)), dict(keys=(0, 2 ** 32)), dict(keys=(0.5, 0)),
               dict(keys=(0, np.full(5, -1)))):
        with pytest.raises(pkg.ArgumentError, match="keys"):
            eng.generated(post, **kw)
    assert eng._lib.calls == []
    # draw_keys: the posterior_matrix layout of a thinned call started at t0
    ch, tr = eng.draw_keys(2 ** 32 - 3, 15, thin=3)
    assert ch.shape == tr.shape == (2 * P, 5) and tr.dtype == np.uint32
    assert np.array_equal(ch, np.repeat(np.arange(2 * P)[:, None], 5, axis=1))
    assert np.array_equal(tr[0], [(2 ** 32 - 3 + 3 * (j + 1) - 1) % 2 ** 32 for j in range(5)])
    g = eng.generated(post, keys=(ch, tr))
    assert eng._lib.calls == [("keyed", 10, 0, P)] and g.shape == (2 * P, 5, G)
    for k in range(2 * P):
        assert g[k].tobytes() == host_keyed(post[k], eng._lib.params[k // 2], seed, ch[k], tr[k]).tobytes()
    # broadcasting keys: one chain id and one transition for the points of one problem
    one = eng.generated(post[0], problem=1, keys=(7, 9))
    assert one.tobytes() == host_keyed(post[0], eng._lib.params[1], seed, 7, 9).tobytes()
    # the summary: a [P, D] reference is refused (g(reference) is random), [P, D + G] is taken as given
    eng._lib.calls.clear()
    with pytest.raises(pkg.ArgumentError, match="reference"):
        eng.mcmc_summary(8, reference=rng.normal(size=(P, D)))
    assert eng._lib.calls == []
    full = rng.normal(size=(P, D + G))
    out = eng.mcmc_summary(8, reference=full)
    assert out["mean"].shape == (P, D + G)
    assert len(eng._lib.calls) == 1 and eng._lib.calls[0][1].tobytes() == full.tobytes()
    assert not any(c[0] == "generated" for c in eng._lib.calls)


# ------------------------------------------------------------------ per-function SASS of eight_schools_gq
def _sass_functions(so):
    """{function name: SHA-256 of its sm_90a SASS}, the cuobjdump listing split at its function headers (a name that
    occurs in several object files is numbered)"""
    out = subprocess.run([os.path.join(CUDA_BIN, "cuobjdump"), "-sass", so], check=True, capture_output=True, text=True).stdout
    funcs, name, body = {}, None, []

    def close():
        if name is not None:
            key, i = name, 1
            while key in funcs:
                i += 1
                key = f"{name}#{i}"
            funcs[key] = hashlib.sha256("\n".join(body).encode()).hexdigest()
    for line in out.splitlines():
        s = line.strip()
        if s.startswith("Function : "):
            close()
            name, body = s[len("Function : "):], []
        elif name is not None and not line.startswith("Fatbin") and "code for sm_" not in line:
            body.append(line)
    close()
    return funcs


def test_sass_of_deterministic_generated_quantities_is_unchanged(pkg):
    """Random quantities are compiled only into a library whose model declares them: in eight_schools_gq (deterministic
    quantities) every function but k_generated, which takes the optional keys, has the sm_90a SASS of the build before
    random quantities existed (CUDA 12.9 nvcc, csrc/Makefile flags; tests/golden/sass_without_random_generated.json)."""
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "sass_without_random_generated.json")))
    ver = subprocess.run([os.path.join(CUDA_BIN, "nvcc"), "--version"], check=True, capture_output=True, text=True).stdout
    if golden["nvcc"] not in ver:
        pytest.skip(f"the golden SASS digests are of nvcc {golden['nvcc']}")
    got = _sass_functions(pkg.compile_user_model(GQ, deep=True))
    want = golden["eight_schools_gq-deep"]
    keep = lambda f: {k: v for k, v in f.items() if "k_generated" not in k}          # noqa: E731
    assert len(keep(want)) > 100 and any("k_generated" in k for k in got)
    assert keep(got) == keep(want)


# ------------------------------------------------------------------ GPU
def _schools(pkg, P, header=PPC, ragged=False, seed=8):
    rng = np.random.default_rng(seed)
    return [pkg.UserLogDensity(header, 10, deep=header != PLAIN,
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


def _host_of_draws(post, problems, cpp, seed, keys, off=0):
    """[K, N, G]: g of every draw of chain k with the parameter block of its problem and the draw's key"""
    ch, tr = keys
    return np.stack([host_keyed(post[k], problems[(off + k) // cpp if cpp else 0].params(), seed, ch[k], tr[k])
                     for k in range(post.shape[0])])


@pytest.mark.gpu
def test_keyed_generated_equals_host_evaluator(pkg):
    import torch
    probs = _schools(pkg, 3)
    batch = pkg.ProblemBatch(probs, 4)
    seed = 31
    eng = _engine(pkg, batch, batch.chains, 0.2, seed=seed)
    L = pkg._lib
    try:
        assert eng.generated_count == 20 and eng.generated_random == 1
        t0 = eng.transition_count
        post = eng.mcmc(12)["posterior_matrix"]
        keys = eng.draw_keys(t0, 12)
        want = _host_of_draws(post, probs, 4, seed, keys)
        assert _same_bits(eng.generated(post, keys=keys), want)
        dev = torch.from_numpy(post).cuda()
        kc, kt = torch.from_numpy(keys[0]).cuda(), torch.from_numpy(keys[1].view(np.int32)).cuda()
        out = torch.empty((12, 12, 20), dtype=torch.float64, device="cuda")
        n0 = eng.kernel_launches()
        eng._ck(eng._lib.dhmc_generated_keyed_dev(eng._h, C.c_void_p(dev.data_ptr()), 4 * 12, 0, 3, C.c_void_p(kc.data_ptr()),
                                                  C.c_void_p(kt.data_ptr()), C.c_void_p(out.data_ptr())))
        assert eng.kernel_launches() == n0 + 1 and _same_bits(out.cpu().numpy(), want)
        # dhmc_generated refuses the random model, keyed calls refuse NULL keys and chain ids outside [0, 2^56): no launch
        o = np.empty(20 * 48)
        ch, tr = keys[0].copy(), keys[1].copy()
        assert eng._lib.dhmc_generated(eng._h, L.ptr(post), 48, 0, 1, L.ptr(o)) == L.DHMC_EARG
        assert "dhmc_generated_keyed" in eng._lib.dhmc_last_error(eng._h).decode()
        for c_, t_ in ((None, tr), (ch, None)):
            assert eng._lib.dhmc_generated_keyed(eng._h, L.ptr(post), 48, 0, 1, L.ptr(c_), L.ptr(t_), L.ptr(o)) == L.DHMC_EARG
        for bad in (-1, 2 ** 56):
            ch2 = ch.copy()
            ch2[1, 3] = bad
            assert eng._lib.dhmc_generated_keyed(eng._h, L.ptr(post), 48, 0, 1, L.ptr(ch2), L.ptr(tr), L.ptr(o)) == L.DHMC_EARG
        assert eng.kernel_launches() == n0 + 1
    finally:
        eng.close()
    # the deterministic model: τ and θ_j are the ppc rows; keys are ignored, the keyed call is dhmc_generated bit for bit
    gq = pkg.ProblemBatch(_schools(pkg, 3, header=GQ), 4)
    eng = _engine(pkg, gq, gq.chains, 0.2, seed=seed)
    try:
        assert eng.generated_random == 0
        plain = eng.generated(post)
        assert _same_bits(plain, want[..., :9])
        assert _same_bits(eng.generated(post, keys=(np.arange(12)[:, None] + 5, 3)), plain)
    finally:
        eng.close()


@pytest.mark.gpu
def test_sampling_is_untouched_by_random_quantities(pkg):
    """the eight_schools_ppc and eight_schools libraries: bit-identical draws, statistics, final state and transition
    counts from one seed, with mcmc and with the summary"""
    outs = []
    for hdr in (PPC, PLAIN):
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
    assert ma["mean"].shape == (3, 30) and mb["mean"].shape == (3, 10)


def _close(got, want, ctx=""):
    for k in ("rank", "draws"):
        assert np.array_equal(got[k], want[k]), (ctx, k, got[k], want[k])
    for k in STATS:
        g, w = np.asarray(got[k], float), np.asarray(want[k], float)
        assert np.array_equal(np.isnan(g), np.isnan(w)), (ctx, k, g, w)
        scale = np.abs(w) + (np.nan_to_num(np.asarray(want["sd"], float)) if k == "mean" else 0.0)
        ok = np.isnan(w) | (g == w) | (np.abs(g - w) <= RTOL * scale)
        assert np.all(ok), (ctx, k, g[~ok], w[~ok])


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


def _drop_in(pkg, eng, problems, N, seed, thin=1, reference=None, cpp=0, P=1, bins=None, ctx=""):
    """mcmc_thinned from a checkpoint, then mcmc_summary from the same checkpoint: same state, statistics and transition
    count bit for bit; all R = D + G rows equal the mirror on [θ, g(θ; key)] with the keyed host evaluator at
    t = t0 + (j + 1)·thin − 1, and with `bins` the histogram of every row equals the mirror's as integers"""
    ck = eng.checkpoint()
    t0 = eng.transition_count
    run = eng.mcmc_thinned(N, thin=thin)
    s1, t1 = eng.get_state(("q", "lq", "grad", "eps")), eng.transition_count
    post = run["posterior_matrix"]
    xr = np.concatenate([post, _host_of_draws(post, problems, cpp, seed, eng.draw_keys(t0, N, thin))], axis=2)
    R = xr.shape[2]
    kw = {}
    if bins:
        lo, hi = _narrow_grid(xr, cpp, P, 1)
        kw = dict(quantiles=(0.05, 0.5, 0.95), grid=(lo, hi), bins=bins)
    eng.restore(ck)
    summ = eng.mcmc_summary(N, thin=thin, reference=reference, stats=True, **kw)
    s2, t2 = eng.get_state(("q", "lq", "grad", "eps")), eng.transition_count
    assert t1 == t2 == t0 + N, ctx
    for f in s1:
        assert _same_bits(s1[f], s2[f]), (ctx, f)
    assert _same_bits(run["tree_statistics"], summ["tree_statistics"]), ctx
    d = pkg.diagnostics
    assert summ["record"].shape == (P, R, pkg._lib.SUMMARY_FIELDS), ctx
    ref = None if reference is None else np.asarray(reference, float)
    _close(summ, d.finish_summary(d.summary_from_draws(xr, cpp, 1, ref, 0, n_problems=P)), ctx)
    if bins:
        want = d.histogram_from_draws(xr, lo, hi, bins, cpp, 1, 0, P)
        assert summ["histogram"].shape == (P, R, bins + 2) and np.array_equal(summ["histogram"], want), ctx
    return summ, xr


@pytest.mark.gpu
def test_drop_in_thinned_batch_with_reference(pkg):
    probs = _schools(pkg, 5)
    batch = pkg.ProblemBatch(probs, 4)
    eng = _engine(pkg, batch, batch.chains, 0.2, seed=31)
    rng = np.random.default_rng(1)
    ref = np.concatenate([rng.normal(size=(5, 10)), rng.normal(size=(5, 20)) * 10], axis=1)
    ref[:, -3:] = 0.5                                                      # an indicator's rank: the draws equal to 0
    ref[0, 12] = np.nan                                                    # a NaN cell counts nothing
    try:
        s, xr = _drop_in(pkg, eng, probs, 40, 31, thin=5, reference=ref, cpp=4, P=5, bins=16, ctx="batch-ref")
        assert np.all(s["draws"] == 8 * 4) and s["rank"][0, 12] == 0
        assert np.all(s["rank"][:, -3:] == (xr[..., -3:].reshape(5, -1, 3) == 0).sum(axis=1))
        with pytest.raises(pkg.ArgumentError, match="reference"):
            eng.mcmc_summary(40, thin=5, reference=ref[:, :10])
    finally:
        eng.close()


@pytest.mark.gpu
def test_drop_in_ragged_batch(pkg):
    probs = _schools(pkg, 4, ragged=True)
    batch = pkg.RaggedProblemBatch(probs, 6)
    eng = _engine(pkg, batch, batch.chains, 0.2, seed=32)
    try:
        _drop_in(pkg, eng, probs, 16, 32, thin=2, reference=np.zeros((4, 30)), cpp=6, P=4, bins=24, ctx="ragged")
    finally:
        eng.close()


@pytest.mark.gpu
def test_drop_in_deep_twin(pkg):
    probs = _schools(pkg, 1)
    eng = _engine(pkg, probs[0], 64, 0.05, seed=33, algorithm=pkg.NUTS(max_depth=14))
    try:
        eng.mcmc(3)                                                        # t0 > 0
        _drop_in(pkg, eng, probs, 8, 33, bins=5, ctx="deep")
    finally:
        eng.close()


@pytest.mark.gpu
def test_drop_in_symmetric_metric(pkg):
    probs = _schools(pkg, 1)
    rng = np.random.default_rng(2)
    A = rng.normal(size=(10, 10)) / np.sqrt(10)
    eng = _engine(pkg, probs[0], 96, 0.2, seed=34)
    try:
        eng.set_metric_dense(0.3 * (A @ A.T) + np.eye(10))
        assert eng.metric_is_dense()
        _drop_in(pkg, eng, probs, 9, 34, reference=rng.normal(size=(1, 30)), bins=64, ctx="dense")
    finally:
        eng.close()


@pytest.mark.gpu
def test_shards_merge_on_random_rows(pkg):
    """two handles split a batch inside a problem; the random rows of each shard are keyed by global chain ids, so the
    merged records give the one-handle summary and the histograms add up exactly"""
    probs = _schools(pkg, 4, seed=12)
    batch = pkg.ProblemBatch(probs, 4)
    rng = np.random.default_rng(3)
    ref = rng.normal(size=(4, 30))
    lo = np.concatenate([np.full((4, 10), -2.0), np.zeros((4, 1)), np.full((4, 16), -40.0), np.full((4, 3), -0.5)], axis=1)
    hi = np.concatenate([np.full((4, 10), 2.0), np.full((4, 1), 15.0), np.full((4, 16), 60.0), np.full((4, 3), 1.5)], axis=1)
    N, thin, cut = 24, 2, 6
    outs = []
    for off, K in ((0, batch.chains), (0, cut), (cut, batch.chains - cut)):
        eng = _engine(pkg, batch, K, 0.2, seed=35, chain_offset=off)
        try:
            outs.append(eng.mcmc_summary(N, thin=thin, reference=ref, quantiles=(0.1, 0.9), grid=(lo, hi), bins=24))
        finally:
            eng.close()
    whole, a, b = outs
    L = pkg._lib
    rec = a["record"].copy()
    assert rec.shape == (4, 30, L.SUMMARY_FIELDS)
    assert L.lib().dhmc_summary_merge(L.ptr(rec), L.ptr(b["record"]), 30, 4) == 0
    _close(pkg.diagnostics.finish_summary(rec), whole, "shards")
    assert np.array_equal(a["histogram"] + b["histogram"], whole["histogram"])
    assert np.all(whole["histogram"][:, 10:].sum(axis=2) == whole["draws"][:, 10:])


@pytest.mark.gpu
def test_halted_chain_is_left_out_of_random_rows(pkg):
    """the halting start of tests/test_generated_quantities.py (seed 5, chain 3 stops with DHMC_CHAIN_LEAPFROG_NONFINITE):
    the random rows leave the chain out as the parameter rows do"""
    K, D, N, seed = 16, 10, 8, 5
    probs = _schools(pkg, 1)
    rng = np.random.default_rng(90)
    q = rng.normal(size=(K, D)) * 0.5
    q[3] = 0.0
    q[3, 4] = 1.5e153
    eps = np.full(K, 0.2)
    eps[3] = 5.0
    eng = pkg.Engine(probs[0], chains=K, seed=seed, algorithm=pkg.NUTS(min_Δ=-np.inf))
    try:
        eng.set_position(q)
        eng.set_stepsize(eps)
        ck = eng.checkpoint()
        t0 = eng.transition_count
        L = pkg._lib
        post, st, ld = np.empty((K, N, D)), np.zeros((K, N), dtype=L.tree_stats_dtype), np.empty((K, N))
        rc = eng._lib.dhmc_mcmc(eng._h, N, L.ptr(post), L.ptr(st), L.ptr(ld))
        status = eng.chain_status()
        assert rc == L.DHMC_ENUMERIC and status[3] == L.DHMC_CHAIN_LEAPFROG_NONFINITE and np.all(np.delete(status, 3) == 0)
        eng.restore(ck)
        xr = np.concatenate([post, _host_of_draws(post, probs, 0, seed, eng.draw_keys(t0, N))], axis=2)
        ref = np.zeros((1, 3 * D))
        lo, hi = _narrow_grid(xr[status == 0], 0, 1, 1)
        with pytest.raises(pkg.ArgumentError, match="leapfrog called from non-finite log density") as e:
            eng.mcmc_summary(N, reference=ref, quantiles=(0.5,), grid=(lo, hi), bins=16)
        summ = e.value.debug_information["summary"]
        assert np.all(summ["record"][..., L.SUMMARY_CHAINS] == K - 1) and np.all(summ["draws"] == N * (K - 1))
        d = pkg.diagnostics
        _close(summ, d.finish_summary(d.summary_from_draws(xr, 0, 1, ref, completed=status == 0)), "halted")
        assert np.array_equal(summ["histogram"], d.histogram_from_draws(xr, lo, hi, 16, completed=status == 0))
    finally:
        eng.close()


@pytest.mark.gpu
def test_end_to_end_posterior_predictive_check(pkg):
    """eight schools, 64 chains, N = 2 000 after the warm-up: var(y_rep_j) = var(θ_j) + σ_j² within 5 %, the replicate
    means are the θ_j means within 4 MCSE, and the three p-values are means of 0/1 rows with MCSEs"""
    J = 8
    ℓ = pkg.UserLogDensity(PPC, J + 2, params=np.concatenate([Y0, S0]), deep=True)
    out = pkg.summarize_with_warmup(17, ℓ, 2000, chains=64)
    assert out["mean"].shape == (1, 30) and np.all(out["draws"] == 2000 * 64)
    th, rep, pv = slice(11, 11 + J), slice(11 + J, 11 + 2 * J), slice(11 + 2 * J, 30)
    var_rep, var_th = out["sd"][0, rep] ** 2, out["sd"][0, th] ** 2
    assert np.all(np.abs(var_rep / (var_th + S0 ** 2) - 1) < 0.05), var_rep / (var_th + S0 ** 2)
    assert np.all(np.abs(out["mean"][0, rep] - out["mean"][0, th]) < 4 * out["mcse"][0, rep]), (out["mean"][0, rep], out["mean"][0, th])
    p = out["mean"][0, pv]
    assert np.all((p >= 0) & (p <= 1)) and np.all(np.isfinite(out["mcse"][0, pv])) and np.all(out["mcse"][0, pv] > 0)
    assert np.all((p > 0.02) & (p < 0.98)), p                              # eight schools fits: no extreme p-value
