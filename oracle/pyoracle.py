"""ctypes wrapper over oracle/liboracle.so — the CPU restatement of the
DynamicHMC.jl sampler path (oracle/oracle.hpp).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline / --impl reference leg, never by the product package.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

FAMILY_STD_NORMAL, FAMILY_DIAG_NORMAL, FAMILY_FUNNEL, FAMILY_LOGISTIC, FAMILY_USER = 0, 1, 2, 3, 4
STAGE_NOTHING, STAGE_SEARCH, STAGE_TUNING = 0, 1, 2
METRIC_NOTHING, METRIC_DIAGONAL, METRIC_SYMMETRIC = 0, 1, 2

tree_stats_dtype = np.dtype(
    [("pi", "<f8"), ("depth", "<i8"), ("left", "<i8"), ("right", "<i8"),
     ("acceptance_rate", "<f8"), ("steps", "<i8"), ("directions", "<u4"), ("pad", "<u4")])
assert tree_stats_dtype.itemsize == 56


class OracleError(RuntimeError):
    """status 2 = DynamicHMCError, 1 = ArgumentError in the reference."""

    def __init__(self, status, msg):
        super().__init__(f"[{status}] {msg}")
        self.status = status


class DummyOut(C.Structure):
    _fields_ = [("valid", C.c_int), ("inv_left", C.c_long), ("inv_right", C.c_long),
                ("zeta_lo", C.c_long), ("zeta_hi", C.c_long), ("n_lp", C.c_int),
                ("lp", C.c_double * 4096), ("omega", C.c_double), ("tau_flag", C.c_int),
                ("tau_lo", C.c_long), ("tau_hi", C.c_long), ("z_last", C.c_long),
                ("i_last", C.c_long), ("v_a", C.c_double), ("v_steps", C.c_long),
                ("n_visited", C.c_int), ("visited", C.c_long * 4096),
                ("adjacency_ok", C.c_int), ("depth", C.c_int)]


def build(force=False):
    so = os.path.join(_HERE, "liboracle.so")
    srcs = [os.path.join(_HERE, f) for f in ("oracle_capi.cpp", "oracle.hpp")] + [
        os.path.join(_HERE, "..", "include", f) for f in ("dhmc_math.h", "dhmc_models.h")]
    stale = (not os.path.exists(so)) or any(
        os.path.exists(s) and os.path.getmtime(s) > os.path.getmtime(so) for s in srcs)
    if force or stale:
        subprocess.check_call(["make", "-C", _HERE, "-B", "liboracle.so"],
                              stdout=subprocess.DEVNULL)
    return so


def _load(path):
    so = C.CDLL(path)
    so.orc_last_error.restype = C.c_char_p
    so.orc_user_family_name.restype = C.c_char_p
    so.orc_randexp.restype = C.c_double
    so.orc_directions.restype = C.c_uint32
    so.orc_canon_dot.restype = C.c_double
    so.orc_logdensity_and_gradient.restype = C.c_double
    so.orc_kinetic_energy.restype = C.c_double
    so.orc_phase_logdensity.restype = C.c_double
    so.orc_acceptance_rate.restype = C.c_double
    so.orc_local_log_acceptance_ratio.restype = C.c_double
    return so


def lib():
    global _LIB
    if _LIB is None:
        _LIB = _load(build())
    return _LIB


def build_user(header, force=False):
    """liboracle with the user model `header` compiled in as family 4 (oracle/Makefile `user`): the checker of a
    user-model library.  Built under oracle/_user/ (git-ignored); returns the path."""
    header = os.path.abspath(header)
    name = os.path.splitext(os.path.basename(header))[0]
    out_dir = os.path.join(_HERE, "_user")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, f"liboracle_user_{name}.so")
    srcs = [header] + [os.path.join(_HERE, f) for f in ("oracle_capi.cpp", "oracle.hpp")] + [
        os.path.join(_HERE, "..", "include", f) for f in ("dhmc_math.h", "dhmc_models.h")]
    if force or not os.path.exists(so) or any(os.path.getmtime(x) > os.path.getmtime(so) for x in srcs):
        subprocess.check_call(["make", "-C", _HERE, "-B", "user", f"USER_HEADER={header}", f"USER_LIB={so}"],
                              stdout=subprocess.DEVNULL)
    return so


class user_model:
    """`with pyoracle.user_model(header): …` — every oracle call inside the block goes to the oracle library that has the
    user model compiled in (family FAMILY_USER; the shipped families are there too)."""
    _cache = {}

    def __init__(self, header):
        self.path = build_user(header)

    def __enter__(self):
        global _LIB
        self.prev = _LIB
        if self.path not in user_model._cache:
            user_model._cache[self.path] = _load(self.path)
        _LIB = user_model._cache[self.path]
        return _LIB

    def __exit__(self, *exc):
        global _LIB
        _LIB = self.prev


def _check(status):
    if status != 0:
        raise OracleError(status, lib().orc_last_error().decode())


def _d(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class _metric:
    """Pass `minv` ([D] diagonal or [D, D] Symmetric) and flip the library's dense mode."""

    def __init__(self, minv, D):
        if minv is None:
            minv = np.ones(D)
        self.a = _d(minv)
        self.dense = self.a.ndim == 2
        if self.dense:
            assert self.a.shape == (D, D)

    def __enter__(self):
        lib().orc_set_dense(C.c_int(int(self.dense)))
        return self.a

    def __exit__(self, *exc):
        lib().orc_set_dense(C.c_int(0))


def dense_factor(minv):
    minv = _d(minv)
    D = minv.shape[0]
    W = np.empty((D, D))
    st = lib().orc_dense_factor(C.c_int(D), _p(minv), _p(W))
    if st != 0:
        raise OracleError(st, "PosDefException")
    return W


def seed_dense_factor(minv, W):
    """Let the following calls of this thread that take exactly this Symmetric M⁻¹ use W = cholesky(inv(M⁻¹)).L instead of
    factorising M⁻¹ (O(D³)) themselves.  W must be what dense_factor(minv) returns."""
    minv, W = _d(minv), _d(W)
    D = minv.shape[0]
    assert minv.shape == W.shape == (D, D)
    lib().orc_seed_dense_factor(C.c_int(D), _p(minv), _p(W))


def rand_p(seed, chain, stream, t, minv):
    D = np.asarray(minv).shape[0]
    out = np.empty(D)
    with _metric(minv, D) as m:
        lib().orc_rand_p(C.c_uint64(seed), C.c_uint64(chain), C.c_uint32(stream), C.c_uint32(t),
                         C.c_int(D), _p(m), _p(out))
    return out


def logistic_params(X, y):
    """params vector of the LOGISTIC family: [N, X row-major, y]"""
    X, y = _d(X), _d(y)
    return np.concatenate([[float(X.shape[0])], X.ravel(), y])


def _params(family, D, params):
    if family == FAMILY_DIAG_NORMAL:
        params = _d(params)
        assert params.size == 2 * D
        return params
    if family == FAMILY_LOGISTIC:
        params = _d(params)
        N = int(params[0])
        assert params.size == 1 + N * D + N
        lib().orc_set_logistic_n(C.c_int(N))
        return params
    if family == FAMILY_USER:
        params = _d(params if params is not None else np.zeros(0))
        lib().orc_set_user_nparams(C.c_int(params.size))
        return params if params.size else np.zeros(1)
    return np.zeros(1)


# ---------------------------------------------------------------- math
_FN = {"exp": 0, "log": 1, "log1p": 2, "logaddexp": 3, "pow": 4, "log1pexp": 5,
       "sin2pi": 6, "cos2pi": 7, "softplus_neg": 8}


def math(fn, x, y=None):
    x = _d(x).ravel()
    y = _d(y).ravel() if y is not None else np.zeros_like(x)
    out = np.empty_like(x)
    lib().orc_math(_FN[fn], C.c_int(x.size), _p(x), _p(y), _p(out))
    return out


def philox(ctr, key):
    ctr = np.ascontiguousarray(ctr, dtype=np.uint32)
    key = np.ascontiguousarray(key, dtype=np.uint32)
    out = np.empty(4, dtype=np.uint32)
    lib().orc_philox(_p(ctr), _p(key), _p(out))
    return out


def normals(seed, chain, stream, t, D):
    out = np.empty(D)
    lib().orc_normals(C.c_uint64(seed), C.c_uint64(chain), C.c_uint32(stream), C.c_uint32(t),
                      C.c_int(D), _p(out))
    return out


def random_position(seed, chain, D):
    out = np.empty(D)
    lib().orc_random_position(C.c_uint64(seed), C.c_uint64(chain), C.c_int(D), _p(out))
    return out


def randexp(seed, chain, t, j):
    return lib().orc_randexp(C.c_uint64(seed), C.c_uint64(chain), C.c_uint32(t), C.c_uint32(j))


def directions(seed, chain, t):
    return int(lib().orc_directions(C.c_uint64(seed), C.c_uint64(chain), C.c_uint32(t)))


def canon_dot(T, a, b):
    a, b = _d(a), _d(b)
    return lib().orc_canon_dot(C.c_int(T), C.c_int(a.size), _p(a), _p(b))


def next_directions(flags, n):
    out = np.empty(n, dtype=np.int32)
    lib().orc_next_directions(C.c_uint32(flags), C.c_int(n), _p(out))
    return [bool(v) for v in out]


# ------------------------------------------------------------ dummy trees
def _dummy_result(o, sample):
    r = dict(valid=bool(o.valid), invalid=(o.inv_left, o.inv_right),
             zeta=(range(o.zeta_lo, o.zeta_hi + 1), np.array(o.lp[:o.n_lp])),
             omega=o.omega, tau=(bool(o.tau_flag), range(o.tau_lo, o.tau_hi + 1)),
             z_last=o.z_last, i_last=o.i_last, v=(o.v_a, o.v_steps),
             visited=list(o.visited[:o.n_visited]), adjacency_ok=bool(o.adjacency_ok))
    if sample:
        r["termination"] = (o.inv_left, o.inv_right)
        r["depth"] = o.depth
    return r


def _la(xs):
    a = np.ascontiguousarray(list(xs), dtype=np.int64)
    return a, a.size


def dummy_adjacent_tree(z, i, depth, is_forward, turning=(), divergent=()):
    t, nt = _la(turning)
    d, nd = _la(divergent)
    o = DummyOut()
    _check(lib().orc_dummy_adjacent_tree(C.c_long(z), C.c_long(i), C.c_int(depth),
                                         C.c_int(int(is_forward)), _p(t), C.c_int(nt), _p(d),
                                         C.c_int(nd), C.byref(o)))
    return _dummy_result(o, False)


def dummy_sample_trajectory(z, max_depth, flags, turning=(), divergent=()):
    t, nt = _la(turning)
    d, nd = _la(divergent)
    o = DummyOut()
    _check(lib().orc_dummy_sample_trajectory(C.c_long(z), C.c_int(max_depth), C.c_uint32(flags),
                                             _p(t), C.c_int(nt), _p(d), C.c_int(nd), C.byref(o)))
    return _dummy_result(o, True)


# ------------------------------------------------------------ hamiltonian
def logdensity_and_gradient(family, q, params=None, T=32):
    q = _d(q)
    D = q.size
    g = np.empty(D)
    pr = _params(family, D, params)
    lq = lib().orc_logdensity_and_gradient(C.c_int(family), C.c_int(D), _p(pr), C.c_int(T), _p(q),
                                           _p(g))
    return lq, g


def evaluate_l(family, q, params=None, T=32, strict=False):
    q = _d(q)
    D = q.size
    g = np.empty(D)
    lq = C.c_double()
    pr = _params(family, D, params)
    _check(lib().orc_evaluate_l(C.c_int(family), C.c_int(D), _p(pr), C.c_int(T), _p(q),
                                C.c_int(int(strict)), C.byref(lq), _p(g)))
    return lq.value, g


def kinetic_energy(minv, p, T=32):
    p = _d(p)
    with _metric(minv, p.size) as m:
        return lib().orc_kinetic_energy(C.c_int(p.size), C.c_int(T), _p(m), _p(p))


def phase_logdensity(minv, lq, p, T=32):
    p = _d(p)
    with _metric(minv, p.size) as m:
        return lib().orc_phase_logdensity(C.c_int(p.size), C.c_int(T), _p(m), C.c_double(lq), _p(p))


def leapfrog(family, q, p, eps, minv=None, params=None, T=32, n_steps=1):
    q, p = _d(q).copy(), _d(p).copy()
    D = q.size
    g = np.empty(D)
    lq = C.c_double()
    pr = _params(family, D, params)
    with _metric(minv, D) as m:
        _check(lib().orc_leapfrog(C.c_int(family), C.c_int(D), _p(pr), C.c_int(T), _p(m), _p(q),
                                  _p(p), _p(g), C.byref(lq), C.c_double(eps), C.c_int(n_steps)))
    return q, p, g, lq.value


# ------------------------------------------------------------------ NUTS
def combine_turn_statistics(x5, y5, T=32):
    """x5, y5: arrays [5, D] = (p₋, p♯₋, p₊, p♯₊, ρ).  Returns (turning, ρ)."""
    x5, y5 = _d(x5), _d(y5)
    D = x5.shape[1]
    rho = np.empty(D)
    turning = lib().orc_combine_turn_statistics(C.c_int(D), C.c_int(T), _p(x5), _p(y5), _p(rho))
    return bool(turning), (None if turning else rho)


def acceptance_rate(deltas, is_initial):
    deltas = _d(deltas)
    ii = np.ascontiguousarray(is_initial, dtype=np.int32)
    return lib().orc_acceptance_rate(C.c_int(deltas.size), _p(deltas), _p(ii))


def rand_bool_logprob(seed, chain, t, j, logprob):
    consumed = C.c_int()
    b = lib().orc_rand_bool_logprob(C.c_uint64(seed), C.c_uint64(chain), C.c_uint32(t),
                                    C.c_uint32(j), C.c_double(logprob), C.byref(consumed))
    return bool(b), consumed.value


def sample_tree(family, q, eps, seed, chain, t, minv=None, params=None, T=32, max_depth=10,
                min_delta=-1000.0, p=None, directions=None, always_divergent=False):
    q = _d(q)
    D = q.size
    pr = _params(family, D, params)
    q1, g1 = np.empty(D), np.empty(D)
    lq1 = C.c_double()
    stats = np.zeros(1, dtype=tree_stats_dtype)
    trace = np.zeros(1 << 14, dtype=np.int32)
    ntrace = C.c_int()
    pp = None if p is None else _d(p)
    dd = None if directions is None else np.array([directions], dtype=np.uint32)
    with _metric(minv, D) as m:
        _check(lib().orc_sample_tree(
            C.c_int(family), C.c_int(D), _p(pr), C.c_int(T), _p(m), C.c_int(max_depth),
            C.c_double(min_delta), C.c_int(int(always_divergent)), C.c_uint64(seed), C.c_uint64(chain),
            C.c_uint32(t), _p(q), C.c_double(eps), _p(pp), _p(dd), _p(q1), C.byref(lq1), _p(g1),
            _p(stats), _p(trace), C.c_int(trace.size), C.byref(ntrace)))
    return dict(q=q1, lq=lq1.value, g=g1, stats=stats[0], accept_trace=trace[:ntrace.value].copy())


# -------------------------------------------------------------- stepsize
def search_params_check(initial_eps=0.1, log_threshold=np.log(0.8), maxiter=400):
    _check(lib().orc_search_params_check(C.c_double(initial_eps), C.c_double(log_threshold),
                                         C.c_int(maxiter)))


def find_initial_stepsize_affine(c, d, initial_eps=0.1, log_threshold=np.log(0.8), maxiter=400):
    eps = C.c_double()
    _check(lib().orc_find_initial_stepsize_affine(C.c_double(c), C.c_double(d),
                                                  C.c_double(initial_eps),
                                                  C.c_double(log_threshold), C.c_int(maxiter),
                                                  C.byref(eps)))
    return eps.value


def find_initial_stepsize(family, q, p, minv=None, params=None, T=32, initial_eps=0.1,
                          log_threshold=np.log(0.8), maxiter=400):
    q, p = _d(q), _d(p)
    D = q.size
    pr = _params(family, D, params)
    eps = C.c_double()
    with _metric(minv, D) as m:
        _check(lib().orc_find_initial_stepsize(C.c_int(family), C.c_int(D), _p(pr), C.c_int(T),
                                               _p(m), _p(q), _p(p), C.c_double(initial_eps),
                                               C.c_double(log_threshold), C.c_int(maxiter),
                                               C.byref(eps)))
    return eps.value


def local_log_acceptance_ratio(family, q, p, eps, minv=None, params=None, T=32):
    q, p = _d(q), _d(p)
    D = q.size
    pr = _params(family, D, params)
    with _metric(minv, D) as m:
        return lib().orc_local_log_acceptance_ratio(C.c_int(family), C.c_int(D), _p(pr), C.c_int(T),
                                                    _p(m), _p(q), _p(p), C.c_double(eps))


def da_init(eps):
    s = np.empty(5)
    _check(lib().orc_da_init(C.c_double(eps), _p(s)))
    return s


def da_adapt(state, a, delta=0.8, gamma=0.05, kappa=0.75, t0=10):
    s = _d(state).copy()
    _check(lib().orc_da_adapt(C.c_double(delta), C.c_double(gamma), C.c_double(kappa),
                              C.c_int(t0), _p(s), C.c_double(a)))
    return s


# ------------------------------------------------------------------ mcmc
def default_warmup_stages(init_steps=75, middle_steps=25, doubling_stages=5, terminating_steps=50,
                          search=True, dual_averaging=True, M=METRIC_DIAGONAL):
    """(kind, N, metric, dual_averaging) tuples mirroring mcmc.jl:415-425."""
    st = []
    if search:
        st.append((STAGE_SEARCH, 0, METRIC_NOTHING, 0))
    if dual_averaging:
        st.append((STAGE_TUNING, init_steps, METRIC_NOTHING, 1))
    for i in range(doubling_stages):
        st.append((STAGE_TUNING, middle_steps * 2 ** i, M, int(dual_averaging)))
    if dual_averaging:
        st.append((STAGE_TUNING, terminating_steps, METRIC_NOTHING, 1))
    return st


METRIC_SYMMETRIC_POOLED = 3     # not in the reference: one dense metric per group of 8 chains (SURVEY §8e "optional exchange")


def mcmc_with_warmup_pooled(family, D, N, seed, chain0, stages, params=None, T=32, max_depth=10, min_delta=-1000.0,
                            da=(0.8, 0.05, 0.75, 10), search=(0.1, float(np.log(0.8)), 400)):
    """The chain group [chain0, chain0 + 8) with pooled Symmetric stages: dict of posterior [8, N, D], tree_statistics [8, N],
    logdensities [8, N], eps [8], minv [D, D] (the shared final metric)."""
    (kind, stN, metric, da_on), ns = _stage_arrays(stages)
    pr = _params(family, D, params)
    post = np.empty((8, N, D)); stats = np.zeros((8, N), dtype=tree_stats_dtype); logd = np.empty((8, N))
    minv = np.empty(D * D); eps = np.empty(8)
    _check(lib().orc_mcmc_with_warmup_pooled(
        C.c_int(family), C.c_int(D), _p(pr), C.c_int(T), C.c_int(max_depth), C.c_double(min_delta), C.c_uint64(seed),
        C.c_uint64(chain0), C.c_int(N), C.c_int(ns), _p(kind), _p(stN), _p(metric), _p(da_on), _p(_d(da)), _p(_d(search)),
        _p(post), _p(stats), _p(logd), _p(minv), _p(eps)))
    return dict(posterior_matrix=post, tree_statistics=stats, logdensities=logd, eps=eps, minv=minv.reshape(D, D))


def _stage_arrays(stages):
    arr = np.array(stages, dtype=np.int32).reshape(-1, 4) if len(stages) else np.zeros((0, 4), np.int32)
    cols = [np.ascontiguousarray(arr[:, k]) for k in range(4)]
    return cols, arr.shape[0]


def mcmc_with_warmup(family, D, N, seed, chain, stages=None, params=None, T=32, max_depth=10,
                     min_delta=-1000.0, q0=None, minv0=None, eps0=None, welford=False,
                     da=(0.8, 0.05, 0.75, 10), search=(0.1, float(np.log(0.8)), 400),
                     keep_warmup=False):
    stages = default_warmup_stages() if stages is None else stages
    (kind, stN, metric, da_on), ns = _stage_arrays(stages)
    pr = _params(family, D, params)
    post = np.empty((N, D))
    stats = np.zeros(N, dtype=tree_stats_dtype)
    logd = np.empty(N)
    m0 = None if minv0 is None else _d(minv0)
    dense_in = m0 is not None and m0.ndim == 2
    dense_out = dense_in or any(s[0] == STAGE_TUNING and s[2] == METRIC_SYMMETRIC for s in stages)
    for s_ in stages:
        if s_[0] == STAGE_TUNING and s_[2] == METRIC_SYMMETRIC:
            dense_out = True
        elif s_[0] == STAGE_TUNING and s_[2] == METRIC_DIAGONAL:
            dense_out = False
    minv = np.empty(D * D if (dense_out or dense_in) else D)
    eps = C.c_double()
    nw = int(sum(s[1] for s in stages if s[0] == STAGE_TUNING))
    post_w = np.empty((nw, D)) if keep_warmup else None
    stats_w = np.zeros(nw, dtype=tree_stats_dtype) if keep_warmup else None
    eps_w = np.empty(nw) if keep_warmup else None
    qf = np.empty(D)
    da4, s3 = _d(da), _d(search)
    q0a = None if q0 is None else _d(q0)
    m0a = m0
    e0 = None if eps0 is None else C.byref(C.c_double(eps0))
    lib().orc_set_dense(C.c_int(int(dense_in)))
    try:
        _mcmc_call = lib().orc_mcmc_with_warmup
    finally:
        pass
    _check(_mcmc_call(
        C.c_int(family), C.c_int(D), _p(pr), C.c_int(T), C.c_int(max_depth), C.c_double(min_delta),
        C.c_uint64(seed), C.c_uint64(chain), C.c_int(N), C.c_int(ns), _p(kind), _p(stN),
        _p(metric), _p(da_on), _p(da4), _p(s3), _p(q0a), _p(m0a), e0, C.c_int(int(welford)),
        _p(post), _p(stats), _p(logd), _p(minv), C.byref(eps), _p(post_w), _p(stats_w), _p(eps_w),
        _p(qf)))
    lib().orc_set_dense(C.c_int(0))
    minv = minv.reshape(D, D) if dense_out else minv[:D]
    out = dict(posterior_matrix=post, tree_statistics=stats, logdensities=logd, minv=minv,
               eps=eps.value, q_final=qf)
    if keep_warmup:
        out.update(warmup_posterior=post_w, warmup_stats=stats_w, warmup_eps=eps_w)
    return out


def bench_mcmc(family, D, n_chains, n_threads, N, stages=(), params=None, T=32, max_depth=10,
               min_delta=-1000.0, seed=2026, minv0=None, eps0=None):
    (kind, stN, metric, da_on), ns = _stage_arrays(list(stages))
    pr = _params(family, D, params)
    m0a = None if minv0 is None else _d(minv0)
    e0 = None if eps0 is None else C.byref(C.c_double(eps0))
    steps = C.c_int64()
    secs = C.c_double()
    st = lib().orc_bench_mcmc(C.c_int(family), C.c_int(D), _p(pr), C.c_int(T), C.c_int(max_depth),
                              C.c_double(min_delta), C.c_uint64(seed), C.c_int(n_chains),
                              C.c_int(n_threads), C.c_int(N), C.c_int(ns), _p(kind), _p(stN),
                              _p(metric), _p(da_on), _p(m0a), e0, C.byref(steps), C.byref(secs),
                              None)
    if st != 0:
        raise OracleError(st, "a chain failed in orc_bench_mcmc")
    return steps.value, secs.value
