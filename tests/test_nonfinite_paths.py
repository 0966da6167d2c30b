"""Trees, step-size searches and warm-ups that meet ℓ = −∞, NaN and overflow, against the oracle.

Every finite path is held to the oracle elsewhere; here ℓ or ∇ℓ turn non-finite inside a tree, a search or a warm-up:
evaluate_ℓ (hamiltonian.jl:202-217) sanitises NaN / +∞ / a bad gradient to −∞ (or raises when strict), logdensity
(:251-256) maps a non-finite ℓ to −∞, leapfrog refuses to start from a non-finite ℓ (:276, ArgumentError), a leaf is
divergent when Δ < min_Δ (NUTS.jl:148-159) and the search's ratio is −∞ or NaN beyond a wall (stepsize.jl:75-85).  The
device restates these branches in every model arm, in the user-model path and in the packed tensor-core round of the
logistic family, whose 8 chains share one CTA: a chain that meets NaN or ∞ there must leave the other seven alone.

The walled normal (include/models/walled_normal.h) is a standard normal for q₀ ≥ a; beyond the wall its `mode` chooses
what a model without a transform returns there (ℓ = −∞, NaN, +∞, or a finite ℓ with a NaN / ±∞ gradient element).

GPU checks compare with the oracle bit for bit — the five integers of the tree statistics, π, the acceptance rate, q, ∇ℓ
and ℓ, NaN equal to NaN — fail on exactly the chains where the oracle raises (with the reference's exception), and
assert that the branch they are about was reached."""
import contextlib
import ctypes as C
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WALL = os.path.join(ROOT, "include", "models", "walled_normal.h")
INT_FIELDS = ("depth", "left", "right", "steps", "directions")
SEED = 20261017
STD, DIAG, FUNNEL, LOGISTIC, USER = 0, 1, 2, 3, 4
NONFINITE_Q, SEARCH_FAILED, BAD_INITIAL, LEAPFROG_NONFINITE = 4, 2, 1, 64     # include/dhmc.h DHMC_CHAIN_*
MODES = range(7)


# ------------------------------------------------------------------ the wall model on the CPU
def _wall_direct(po, q, a, mode):
    """ℓ, ∇ℓ of walled_normal.h written out (Σ q² in the canonical order of a 32-thread chain)."""
    q = np.asarray(q, float)
    lq, g = -0.5 * po.canon_dot(32, q, q), -q.copy()
    if q[0] >= a:
        return lq, g
    lq = {0: -np.inf, 1: -np.inf, 2: np.nan, 3: np.inf}.get(mode, lq)
    g[0] = {1: np.nan, 4: np.nan, 5: np.inf, 6: -np.inf}.get(mode, g[0])
    return lq, g


# evaluate_ℓ, hamiltonian.jl:202-217, for each mode beyond the wall: (non-strict ℓ, strict outcome)
#   ℓ finite and ∇ℓ finite, or ℓ == −∞ (whatever ∇ℓ is)  -> accepted as is, strict too
#   otherwise, non-strict                                  -> ℓ replaced by −∞
#   otherwise, strict: ℓ finite (so ∇ℓ is bad)             -> "Gradient has non-finite elements."
#                      ℓ NaN or +∞                         -> "Invalid log posterior."
EVALUATE_TABLE = {0: (-np.inf, None), 1: (-np.inf, None), 2: (-np.inf, "Invalid log posterior"),
                  3: (-np.inf, "Invalid log posterior"), 4: (-np.inf, "Gradient has non-finite"),
                  5: (-np.inf, "Gradient has non-finite"), 6: (-np.inf, "Gradient has non-finite")}


def test_wall_model_oracle_values_and_evaluate_table(po):
    rng = np.random.default_rng(1)
    with po.user_model(WALL):
        for mode in MODES:
            for D in (1, 2, 5, 40):
                a = float(rng.normal())
                for side in (+1, -1):
                    q = rng.normal(size=D)
                    q[0] = a + side * abs(rng.normal()) + (0.0 if side > 0 else -1e-3)
                    pr = np.array([a, float(mode)])
                    lq, g = po.logdensity_and_gradient(USER, q, pr)
                    lq_d, g_d = _wall_direct(po, q, a, mode)
                    assert np.array_equal([lq], [lq_d], equal_nan=True) and np.array_equal(g, g_d, equal_nan=True), \
                        (mode, D, side)
                    l_ns, g_ns = po.evaluate_l(USER, q, pr)
                    assert np.array_equal(g_ns, g_d, equal_nan=True)
                    if side > 0:
                        assert l_ns == lq_d and po.evaluate_l(USER, q, pr, strict=True)[0] == lq_d
                        continue
                    want_l, want_err = EVALUATE_TABLE[mode]
                    assert l_ns == want_l, mode
                    if want_err is None:
                        assert po.evaluate_l(USER, q, pr, strict=True)[0] == want_l
                    else:
                        with pytest.raises(po.OracleError, match=want_err) as e:
                            po.evaluate_l(USER, q, pr, strict=True)
                        assert e.value.status == 2
            q = np.array([2.0, 0.5])
            assert po.evaluate_l(USER, q, np.array([2.0, float(mode)]), strict=True)[0] == -0.5 * 4.25   # on the wall: inside


# ------------------------------------------------------------------ GPU helpers
def _same(a, b):
    return np.array_equal(np.asarray(a, float), np.asarray(b, float), equal_nan=True)


def _same_stats(o, d, ctx):
    for f in INT_FIELDS:
        assert o[f] == d[f], (ctx, f, o, d)
    assert _same(o["pi"], d["pi"]) and _same(o["acceptance_rate"], d["acceptance_rate"]), (ctx, o, d)


def _oracle_bit(po, e):
    """the device status bit of an oracle exception"""
    msg = str(e)
    if e.status == 1 and "leapfrog called from non-finite log density" in msg:
        return LEAPFROG_NONFINITE
    if "Position vector has non-finite elements" in msg:
        return NONFINITE_Q
    raise AssertionError(f"unexpected oracle failure {msg}")


def _expect_failure(pkg, eng, rc, bits):
    """the call failed iff some chain failed, with the reference's exception"""
    if not np.any(bits):
        assert rc == 0, eng._lib.dhmc_last_error(eng._h).decode()
        return
    exc = pkg.ArgumentError if np.any(bits == LEAPFROG_NONFINITE) else pkg.DynamicHMCError
    with pytest.raises(exc):
        eng._ck(rc)


@contextlib.contextmanager
def _engine(pkg, ℓ, K, **kw):
    eng = pkg.Engine(ℓ, chains=K, seed=SEED, **kw)
    try:
        yield eng
    finally:
        eng.close()


def _wall(pkg, D, a, mode):
    return pkg.UserLogDensity(WALL, D, params=[a, float(mode)], deep=True)   # __graft_entry__.build() compiles it deep


def _tree_call(pkg, po, eng, fam, params, minv, max_depth, min_delta, t=0):
    """one dhmc_sample_tree on every chain against po.sample_tree: returns (oracle result or exception bit per chain,
    device stats).  A chain the oracle fails must carry exactly that status bit; a halted chain (leapfrog from ℓ = −∞) keeps
    its state; every other chain equals the oracle."""
    L = pkg._lib
    K, D = eng.K, eng.D
    T, _ = eng.layout()
    st0 = eng.get_state(("q", "lq", "grad", "eps"))
    stats = np.zeros(K, dtype=L.tree_stats_dtype)
    rc = eng._lib.dhmc_sample_tree(eng._h, None, None, L.ptr(stats))
    status = eng.chain_status()
    st1 = eng.get_state(("q", "lq", "grad"))
    res, bits = [], np.zeros(K, np.int32)
    for k in range(K):
        m = minv if minv is None or np.ndim(minv) == 2 else minv[k]
        try:
            o = po.sample_tree(fam, st0["q"][k], st0["eps"][k], SEED, k, t, minv=m, params=params, T=T,
                               max_depth=max_depth, min_delta=min_delta)
        except po.OracleError as e:
            bits[k] = _oracle_bit(po, e)
            res.append(bits[k])
            assert status[k] == bits[k], (k, status[k], str(e))
            if bits[k] == LEAPFROG_NONFINITE:
                assert _same(st1["q"][k], st0["q"][k]) and _same(st1["grad"][k], st0["grad"][k]) and \
                    _same(st1["lq"][k], st0["lq"][k]), k
            continue
        res.append(o)
        assert status[k] == 0, (k, status[k])
        _same_stats(o["stats"], stats[k], k)
        assert _same(o["q"], st1["q"][k]) and _same(o["g"], st1["grad"][k]) and _same(o["lq"], st1["lq"][k]), k
    _expect_failure(pkg, eng, rc, bits)
    return res, stats


# ------------------------------------------------------------------ evaluation and leapfrog
@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_wall_evaluation_and_leapfrog(pkg, po, mode):
    """set_position flags DHMC_CHAIN_BAD_INITIAL exactly where the oracle's strict evaluate_ℓ raises; a leapfrog into the
    wall gives the oracle's sanitised ℓ and its ∇ℓ; a second leapfrog from there halts the chain (ArgumentError) where the
    oracle raises it, and leaves it as it was."""
    rng = np.random.default_rng(10 + mode)
    K, D, a = 16, 3, 0.25
    pr = np.array([a, float(mode)])
    q = rng.normal(size=(K, D))
    q[:, 0] = a + np.where(np.arange(K) % 2 == 0, 1, -1) * rng.uniform(0.01, 1.0, K)   # odd chains beyond the wall
    with po.user_model(WALL), _engine(pkg, _wall(pkg, D, a, mode), K) as eng:
        raises = np.zeros(K, bool)
        for k in range(K):
            try:
                po.evaluate_l(USER, q[k], pr, strict=True)
            except po.OracleError:
                raises[k] = True
        assert raises.any() == (mode >= 2)
        rc = eng._lib.dhmc_set_position(eng._h, pkg._lib.ptr(np.ascontiguousarray(q)))
        assert np.array_equal((eng.chain_status() & BAD_INITIAL) != 0, raises)
        if raises.any():
            with pytest.raises(pkg.DynamicHMCError):
                eng._ck(rc)
        # from in front of the wall, momenta towards it: one step lands beyond it on the odd chains
        q[:, 0] = a + 0.2
        p = rng.normal(size=(K, D))
        p[:, 0] = np.where(np.arange(K) % 2 == 0, 0.3, -3.0)
        eng.set_position(q)
        eng.set_momentum(p)
        eng.set_stepsize(0.5)
        eng.leapfrog(1)
        st = eng.get_state(("q", "p", "lq", "grad"))
        beyond = st["q"][:, 0] < a
        assert np.array_equal(beyond, np.arange(K) % 2 == 1)
        T, _ = eng.layout()
        for k in range(K):
            oq, op, og, ol = po.leapfrog(USER, q[k], p[k], 0.5, params=pr, T=T)
            assert _same(oq, st["q"][k]) and _same(op, st["p"][k]) and _same(og, st["grad"][k]) and _same(ol, st["lq"][k]), k
            assert (ol == -np.inf) == beyond[k] and (mode not in (1, 4, 5, 6) or not beyond[k] or not np.isfinite(og[0]))
        # the next leapfrog starts from ℓ = −∞ on the odd chains: hamiltonian.jl:276
        rc = eng._lib.dhmc_leapfrog(eng._h, 1, 1)
        status = eng.chain_status()
        st2 = eng.get_state(("q", "p", "lq", "grad"))
        bits = np.zeros(K, np.int32)
        for k in range(K):
            try:
                oq, op, og, ol = po.leapfrog(USER, st["q"][k], st["p"][k], 0.5, params=pr, T=T)
            except po.OracleError as e:
                bits[k] = _oracle_bit(po, e)
                for f in ("q", "p", "lq", "grad"):
                    assert _same(st2[f][k], st[f][k]), (k, f)
                continue
            assert _same(oq, st2["q"][k]) and _same(op, st2["p"][k]) and _same(og, st2["grad"][k]) and \
                _same(ol, st2["lq"][k]), k
        assert np.array_equal(bits, np.where(beyond, LEAPFROG_NONFINITE, 0)) and np.array_equal(status, bits)
        _expect_failure(pkg, eng, rc, bits)


# ------------------------------------------------------------------ trees across the wall
def _wall_starts(rng, K, D, a):
    """chains started close to the wall on its inside (q₀ − a in [0.005, 0.6]), momenta drawn by the sampler; chains
    3 and 11 start beyond it (ℓ(q₀) = −∞ is accepted by a strict evaluation in modes 0 and 1 only)"""
    q = rng.normal(size=(K, D))
    q[:, 0] = a + np.exp(rng.uniform(np.log(0.005), np.log(0.6), K))
    return q


def _tree_coverage(res, stats, q0, qs):
    first, deep, before = 0, 0, 0
    for k, o in enumerate(res):
        if not isinstance(o, dict):
            continue
        s = o["stats"]
        if s["left"] == s["right"]:
            first += s["depth"] == 0
            deep += s["depth"] >= 3
            before += s["depth"] >= 1 and not np.array_equal(qs[k], q0[k])
    return first, deep, before


@pytest.mark.gpu
@pytest.mark.parametrize("D", [2, 40, 300, 1000, 3000])
@pytest.mark.parametrize("dense", [False, True], ids=["diagonal", "symmetric"])
def test_trees_across_the_wall(pkg, po, D, dense):
    """two trees per chain at step sizes from 0.02 to 1 in every wall mode whose start a strict evaluation accepts.
    Coverage over the modes: trees divergent at their first leaf, wall divergences at depth ≥ 3 (inside a subtree),
    and divergent trees that had selected a proposal before reaching the wall (the chain moved).  Symmetric at D = 3000
    (the dense kernels with 8 warps per chain) runs one mode at larger steps: the oracle's dense trees cost O(D²) per
    leaf and its factorisation of M⁻¹ O(D³), so there it checks first-leaf divergences and the halted chains only."""
    rng = np.random.default_rng(D + 7 * dense)
    K, a = 24, -0.3
    cover = np.zeros(3, int)
    halted = 0
    small = dense and D == 3000
    modes = MODES if D <= 300 else (0,) if small else (0, 1, 4)
    lo_eps = 0.3 if small else 0.02
    if dense:
        A = rng.normal(size=(D, D)) / np.sqrt(D)
        M = np.eye(D) + 0.2 * (A @ A.T)
        M = (M + M.T) / 2
    with po.user_model(WALL):
        if dense:
            po.seed_dense_factor(M, po.dense_factor(M))
        for mode in modes:
            q = _wall_starts(rng, K, D, a)
            if mode in (0, 1):
                q[[3, 11], 0] = a - 0.1
            eps = np.exp(rng.uniform(np.log(lo_eps), np.log(1.0), K))
            pr = np.array([a, float(mode)])
            with _engine(pkg, _wall(pkg, D, a, mode), K) as eng:
                if dense:
                    eng.set_metric_dense(M)
                eng.set_position(q)
                eng.set_stepsize(eps)
                for t in range(2):
                    qb = eng.get_state(("q",))["q"]
                    res, stats = _tree_call(pkg, po, eng, USER, pr, M if dense else None, 10, -1000.0, t=t)
                    qa = eng.get_state(("q",))["q"]
                    cover += _tree_coverage(res, stats, qb, qa)
                    halted += sum(1 for o in res if not isinstance(o, dict))
                    if t == 0 and mode in (0, 1):
                        assert res[3] == LEAPFROG_NONFINITE and res[11] == LEAPFROG_NONFINITE
    assert (cover[0] >= 1 if small else np.all(cover >= 1)), cover
    assert halted >= 4


@pytest.mark.gpu
def test_deep_trees_into_the_wall(pkg, po):
    """max_depth = 15 (the deep kernels, slot pool past its register word): tiny steps reach the wall only after
    thousands of leaves, so the divergence ends a subtree at depth > 12."""
    K, D, a = 8, 2, -0.3
    rng = np.random.default_rng(15)
    q = rng.normal(size=(K, D))
    q[:, 0] = a + rng.uniform(0.05, 0.3, K)
    with po.user_model(WALL), _engine(pkg, _wall(pkg, D, a, 0), K, algorithm=pkg.NUTS(max_depth=15)) as eng:
        eng.set_position(q)
        eng.set_stepsize(np.full(K, 2e-4))
        res, stats = _tree_call(pkg, po, eng, USER, np.array([a, 0.0]), None, 15, -1000.0)
    div = [o["stats"]["depth"] for o in res if isinstance(o, dict) and o["stats"]["left"] == o["stats"]["right"]]
    assert len(div) >= 2 and max(div) > 12, div


# ------------------------------------------------------------------ step-size search
@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_search_across_the_wall(pkg, po, mode):
    """initial_ϵ = 4 from just inside the wall: the first trial leapfrogs land beyond it (ratio −∞), the search halves
    until one stays inside.  ϵ equals the oracle's on every chain; SEARCH_FAILED is set exactly where the oracle raises
    (a start at ℓ = −∞ beyond the wall: "Starting point has non-finite density")."""
    rng = np.random.default_rng(40 + mode)
    K, D, a = 16, 5, 0.0
    pr = np.array([a, float(mode)])
    q = rng.normal(size=(K, D))
    q[:, 0] = a + rng.uniform(0.001, 0.2, K)
    if mode in (0, 1):
        q[[2, 9], 0] = a - 0.5
    search = pkg.InitialStepsizeSearch(initial_ϵ=4.0)
    with po.user_model(WALL), _engine(pkg, _wall(pkg, D, a, mode), K) as eng:
        eng.set_position(q)
        T, _ = eng.layout()
        rc = eng._lib.dhmc_find_initial_stepsize(eng._h, C.c_double(4.0), C.c_double(search.log_threshold),
                                                 C.c_int32(search.maxiter_crossing))
        status = eng.chain_status()
        eps = eng.get_state(("eps",))["eps"]
        if mode in (0, 1):
            with pytest.raises(pkg.DynamicHMCError):
                eng._ck(rc)
        else:
            assert rc == 0
        failed, beyond = np.zeros(K, bool), 0
        for k in range(K):
            p0 = po.rand_p(SEED, k, 1, 0, np.ones(D))
            if q[k, 0] >= a:                   # (the oracle's ratio function does not return from a start at ℓ = −∞)
                beyond += po.local_log_acceptance_ratio(USER, q[k], p0, 4.0, params=pr, T=T) == -np.inf
            try:
                e = po.find_initial_stepsize(USER, q[k], p0, params=pr, T=T, initial_eps=4.0)
            except po.OracleError:
                failed[k] = True
                assert status[k] == SEARCH_FAILED and np.isnan(eps[k]), (k, status[k])
                continue
            assert status[k] == 0 and eps[k] == e, (k, eps[k], e)
    assert beyond >= 4
    assert np.array_equal(np.nonzero(failed)[0], [2, 9] if mode in (0, 1) else [])


# ------------------------------------------------------------------ warm-up
@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["diagonal", "symmetric"])
def test_warmup_with_wall_divergences(pkg, po, metric):
    """search + dual averaging + a metric window + dual averaging, Welford, on the walled normal with the wall at the
    mode: about half of every chain's draws would lie beyond it, so wall divergences are frequent in every stage."""
    K, D, a, n = 8, 4, 0.0, 30
    rng = np.random.default_rng(50)
    q = rng.normal(size=(K, D))
    q[:, 0] = np.abs(q[:, 0]) + 0.05
    M = pkg.Diagonal if metric == "diagonal" else pkg.Symmetric
    code = po.METRIC_DIAGONAL if metric == "diagonal" else po.METRIC_SYMMETRIC
    stages = [(po.STAGE_SEARCH, 0, po.METRIC_NOTHING, 0), (po.STAGE_TUNING, n, po.METRIC_NOTHING, 1),
              (po.STAGE_TUNING, n, code, 1), (po.STAGE_TUNING, n, po.METRIC_NOTHING, 1)]
    pr = np.array([a, 1.0])
    with po.user_model(WALL), _engine(pkg, _wall(pkg, D, a, 1), K) as eng:
        T, _ = eng.layout()
        eng.set_position(q)
        eng.find_initial_stepsize()
        ws = [eng.warmup_stage(pkg.TuningNUTS(n, pkg.DualAveraging(), m), keep=True) for m in (None, M, None)]
        out = eng.mcmc(n)
        ck = eng.checkpoint()
    div = 0
    for k in range(K):
        with po.user_model(WALL):
            o = po.mcmc_with_warmup(USER, D, n, SEED, k, stages=stages, params=pr, T=T, q0=q[k], welford=True,
                                    keep_warmup=True)
        wst = np.concatenate([w["tree_statistics"][k] for w in ws])
        for f in INT_FIELDS:
            assert np.array_equal(wst[f], o["warmup_stats"][f]), (k, f)
        assert _same(wst["acceptance_rate"], o["warmup_stats"]["acceptance_rate"]), k
        assert _same(np.concatenate([w["posterior_matrix"][k] for w in ws]), o["warmup_posterior"]), k
        for i in range(n):
            _same_stats(o["tree_statistics"][i], out["tree_statistics"][k, i], (k, i))
        assert _same(out["posterior_matrix"][k], o["posterior_matrix"]) and _same(out["logdensities"][k], o["logdensities"])
        assert ck["eps"][k] == o["eps"] and _same(ck["minv"][k], o["minv"]), k
        div += int(np.sum(wst["left"] == wst["right"]))
    assert div >= K * 3 * n // 10, div


# ------------------------------------------------------------------ shipped families at overflow
def _shipped_trees(pkg, po, ℓ, fam, params, q, eps, tpc=0, min_delta=-1000.0, t_max=2):
    K = q.shape[0]
    out = []
    with _engine(pkg, ℓ, K, threads_per_chain=tpc, algorithm=pkg.NUTS(min_Δ=min_delta)) as eng:
        raises = np.zeros(K, bool)
        for k in range(K):
            try:
                po.evaluate_l(fam, q[k], params, T=eng.layout()[0], strict=True)
            except po.OracleError:
                raises[k] = True
        rc = eng._lib.dhmc_set_position(eng._h, pkg._lib.ptr(np.ascontiguousarray(q)))
        assert not raises.any() and rc == 0
        eng.set_stepsize(eps)
        for t in range(t_max):
            res, stats = _tree_call(pkg, po, eng, fam, params, None, 10, min_delta, t=t)
            out.append((res, stats, eng.get_state(("q", "lq", "grad"))))
    return out


@pytest.mark.gpu
def test_funnel_and_diag_normal_at_overflow(pkg, po):
    """the funnel with v in ±[709, 745] (exp(−v) overflows, or is subnormal) and DIAG_NORMAL with |q_i| or
    prec·(q − μ) near overflow: starts a strict evaluation accepts; chains whose first leapfrog starts from ℓ = −∞ halt
    where the oracle raises, the others equal it."""
    rng = np.random.default_rng(60)
    K, D = 32, 6
    q = rng.normal(size=(K, D))
    q[:, 0] = np.where(np.arange(K) % 2 == 0, 1, -1) * rng.uniform(709.0, 745.0, K)
    for k in range(K):                          # keep the starts a strict evaluation accepts
        try:
            po.evaluate_l(FUNNEL, q[k], strict=True)
        except po.OracleError:
            q[k, 0] = 700.0 * np.sign(q[k, 0])
    eps = np.exp(rng.uniform(np.log(0.01), np.log(0.5), K))
    runs = _shipped_trees(pkg, po, pkg.Funnel(D), FUNNEL, None, q, eps)
    halted = sum(1 for res, _, _ in runs for o in res if not isinstance(o, dict))
    assert halted >= 2 and sum(1 for o in runs[0][0] if isinstance(o, dict)) >= 4
    mu, prec = rng.normal(size=D), np.exp(rng.uniform(np.log(0.5), np.log(2.0), D))
    q = rng.normal(size=(K, D))
    big = rng.integers(D, size=K)
    q[np.arange(K), big] = np.where(np.arange(K) % 2, 1, -1) * np.exp(rng.uniform(np.log(1e153), np.log(3e154), K))
    ℓ = pkg.DiagNormal(mu, 1.0 / prec)
    params = ℓ.params()                         # [μ, 1/σ²]
    for k in range(K):
        try:
            po.evaluate_l(DIAG, q[k], params, strict=True)
        except po.OracleError:
            q[k, big[k]] = 1e153
    runs = _shipped_trees(pkg, po, ℓ, DIAG, params, q, eps)
    halted = sum(1 for res, _, _ in runs for o in res if not isinstance(o, dict))
    assert halted >= 2
    # prec·(q − μ) overflows: one coordinate with precision 1e300 and |q − μ| from 1e3 to 1e10.  Beyond ≈ 1.8e8 the
    # product is ±∞ (gradient ∓∞); beyond ≈ 1.3e4 already the term (q − μ)·prec·(q − μ) is.  Either way ℓ(q₀) = −∞, which
    # a strict evaluation accepts, and exactly those chains halt at their first leapfrog.
    prec2 = prec.copy()
    prec2[2] = 1e300
    ℓ2 = pkg.DiagNormal(mu, 1.0 / prec2)
    params2 = ℓ2.params()
    q = rng.normal(size=(K, D))
    q[:, 2] = mu[2] + np.where(np.arange(K) % 2, 1, -1) * np.exp(rng.uniform(np.log(1e3), np.log(1e10), K))
    q[:4, 2] = mu[2] + rng.normal(size=4)           # and some chains where everything is finite
    with np.errstate(over="ignore"):
        overflow = ~np.isfinite(params2[D + 2] * (q[:, 2] - mu[2]))
    minus_inf = np.array([po.evaluate_l(DIAG, q[k], params2, strict=True)[0] == -np.inf for k in range(K)])
    assert overflow.sum() >= 4 and np.all(minus_inf[overflow]) and not minus_inf.all()
    runs = _shipped_trees(pkg, po, ℓ2, DIAG, params2, q, eps)
    halted = [k for k, o in enumerate(runs[0][0]) if not isinstance(o, dict)]
    assert np.array_equal(np.nonzero(minus_inf)[0], halted), (np.nonzero(minus_inf)[0], halted)


OVERFLOW_AT = 1.5          # |q_j| beyond which a scaled row's product x_j·q_j overflows


def _scaled_logistic(rng, N, p):
    """N − 3 ordinary rows and three scaled ones, s = floatmax / 1.5, so that η leaves the finite range where the normal
    prior (std 1) sends the chains:
      row 0:  s·e₀,  y = 1  →  η = +∞ for q₀ > 1.5: limit ll = 0;  q₀ < 0: ll ≈ −1e308 or −∞ (a wall)
      row 1: −s·e₀,  y = 0  →  η = −∞ for q₀ > 1.5: limit ll = 0
      row 2:  s·(e₁ − e_{p−1}),  y = 1  →  η = +∞ for q₁ > 1.5; once q_{p−1} > 1.5 too, η stays +∞ where both non-zeros
              share a 64-coefficient chunk of the blocked dot product (p ≤ 64: the fused multiply-add adds a finite
              exact product to +∞) and is NaN (chunk sums ∞ − ∞) where they do not (p = 256)"""
    sc = np.finfo(np.float64).max / OVERFLOW_AT
    X = rng.normal(size=(N, p)) / np.sqrt(p)
    y = (rng.uniform(size=N) < 0.5).astype(float)
    X[:3] = 0.0
    X[0, 0], y[0] = sc, 1.0
    X[1, 0], y[1] = -sc, 0.0
    X[2, 1], X[2, p - 1], y[2] = sc, -sc, 1.0
    return X, y


def _eta(X, q):
    """η of the three scaled rows as the model computes it (dm_blocked_dot): fused multiply-adds in order within each
    64-coefficient chunk — an accumulator that reached ±∞ stays there, since the exact product added to it is finite —
    then the chunk sums added in order, where ∞ − ∞ = NaN"""
    from fractions import Fraction
    big = Fraction(np.finfo(np.float64).max) + Fraction(2) ** 970          # rounds to ±∞ from here on
    out = []
    for r in range(3):
        tot = None
        for c0 in range(0, X.shape[1], 64):
            acc = 0.0
            for j in np.nonzero(X[r, c0:c0 + 64])[0] + c0:
                if np.isfinite(acc):
                    e = Fraction(float(X[r, j])) * Fraction(float(q[j])) + Fraction(acc)
                    acc = float(np.sign(e)) * np.inf if abs(e) >= big else float(e)
            with np.errstate(invalid="ignore"):
                tot = acc if tot is None else tot + acc
        out.append(tot)
    return np.array(out)


@pytest.mark.gpu
@pytest.mark.parametrize("p", [5, 33, 256])
def test_logistic_with_overflowing_rows(pkg, po, p):
    """η = ±∞ with the outcome its sign predicts (ll = 0, residual 0: ℓ and ∇ℓ stay finite and trees go on through those
    points), η = ±∞ against the outcome (ℓ = −∞) and, at p = 256, η = NaN (∞ − ∞).  One chain per CTA (threads_per_chain = 32) and
    packed groups of 8 (automatic layout, the tensor-core likelihood round) give the same trees, the same ℓ and ∇ℓ at the
    end points, and both equal the oracle.  Chains 3 and 11 start where η = −∞ meets y = 1, so ℓ(q₀) = −∞ (accepted by a
    strict evaluation) and they halt at their first leapfrog — inside a packed CTA the other seven chains go on.  A
    leapfrog into the NaN region compares the sanitised ℓ and the NaN gradient with the oracle's."""
    rng = np.random.default_rng(70 + p)
    X, y = _scaled_logistic(rng, 40, p)
    ℓ = pkg.LogisticRegression(X, y)
    params = po.logistic_params(X, y)
    K = 16
    q = rng.normal(size=(K, p)) * 0.3
    q[:, 0] = rng.uniform(1.6, 3.0, K)                  # rows 0, 1: η = ±∞ with the predicted outcome
    q[:, 1] = rng.uniform(1.6, 3.0, K)                  # row 2: η = +∞ …
    q[:, p - 1] = rng.uniform(-1.0, 1.2, K)             # … until q_{p−1} passes 1.5
    q[[3, 11], 0] = -2.5                                # row 0: η = −∞ with y = 1, ℓ(q₀) = −∞
    for k in range(K):
        lq0 = po.evaluate_l(LOGISTIC, q[k], params, strict=True)[0]
        assert (lq0 == -np.inf) == (k in (3, 11)), (k, lq0)
        assert not np.all(np.isfinite(_eta(X, q[k])))
    eps = np.exp(rng.uniform(np.log(0.05), np.log(0.3), K))
    pm = rng.normal(size=(K, p)) * 0.1
    pm[:, p - 1] = np.where(np.arange(K) % 2 == 0, 6.0, -1.0)
    # the automatic layout packs 8 chains per CTA: such a handle refuses a batch of 4 chains per problem
    with pytest.raises(pkg.ArgumentError, match="packed chain groups"):
        pkg.Engine(pkg.ProblemBatch([ℓ, ℓ], chains_per_problem=4), chains=8, seed=SEED)
    runs = {}
    for tpc in (32, 0):
        runs[tpc] = []
        with _engine(pkg, ℓ, K, threads_per_chain=tpc) as eng:
            eng.set_position(q)
            eng.set_stepsize(eps)
            for t in range(2):
                q_before = eng.get_state(("q",))["q"]
                res, stats = _tree_call(pkg, po, eng, LOGISTIC, params, None, 10, -1000.0, t=t)
                runs[tpc].append((res, stats, q_before, eng.get_state(("q", "lq", "grad"))))
            # a leapfrog from the start: momenta that carry q_{p−1} past 1.5 (row 2: η = NaN) on the even chains
            eng.set_position(q)
            eng.set_momentum(pm)
            eng.set_stepsize(0.5)
            rc = eng._lib.dhmc_leapfrog(eng._h, 1, 1)
            status = eng.chain_status()
            st = eng.get_state(("q", "p", "lq", "grad"))
            T, _ = eng.layout()
            nan_eta = 0
            for k in range(K):
                try:
                    oq, op, og, ol = po.leapfrog(LOGISTIC, q[k], pm[k], 0.5, params=params, T=T)
                except po.OracleError as e:
                    assert k in (3, 11) and _oracle_bit(po, e) == LEAPFROG_NONFINITE and status[k] == LEAPFROG_NONFINITE
                    continue
                assert status[k] == 0, k
                assert _same(oq, st["q"][k]) and _same(op, st["p"][k]) and _same(og, st["grad"][k]) and \
                    _same(ol, st["lq"][k]), k
                if np.isnan(_eta(X, oq)[2]):
                    nan_eta += 1
                    assert ol == -np.inf
            assert (nan_eta >= 3) if p > 64 else (nan_eta == 0), nan_eta
            with pytest.raises(pkg.ArgumentError):
                eng._ck(rc)
    moved_through, finite_at_overflow = 0, 0
    for (ra, sa, q0a, qa), (rb, sb, q0b, qb) in zip(runs[32], runs[0]):
        for f in INT_FIELDS + ("pi", "acceptance_rate"):
            assert _same(sa[f], sb[f]), f
        for f in ("q", "lq", "grad"):
            assert _same(qa[f], qb[f]), f
        assert [k for k, o in enumerate(ra) if not isinstance(o, dict)] == [3, 11]
        for k, o in enumerate(ra):
            if not isinstance(o, dict):
                continue
            eta0, eta1 = _eta(X, q0a[k]), _eta(X, qa["q"][k])
            if o["stats"]["depth"] >= 1 and not np.array_equal(qa["q"][k], q0a[k]) and not np.all(np.isfinite(eta0)):
                moved_through += 1
            if not np.all(np.isfinite(eta1)) and np.isfinite(qa["lq"][k]) and np.all(np.isfinite(qa["grad"][k])):
                finite_at_overflow += 1
    assert moved_through >= 6 and finite_at_overflow >= 6, (moved_through, finite_at_overflow)


# ------------------------------------------------------------------ chain isolation
def _isolation_problem(rng, p=5):
    X = rng.normal(size=(60, p)) / np.sqrt(p)
    y = (rng.uniform(size=60) < 0.5).astype(float)
    return X, y


@pytest.mark.gpu
@pytest.mark.parametrize("tpc", [0, 32], ids=["packed", "one_per_cta"])
def test_chain_isolation(pkg, po, tpc):
    """chains 2 and 5 of a CTA's 8 get ϵ = 1e300: their first leapfrog overflows q.  NONFINITE_Q is set on exactly those
    chains (the oracle raises there), the call fails, and every other chain equals the oracle — sample_tree, mcmc,
    leapfrog; in the step-size search the two chains get M⁻¹ = 1e308 (a trial step overflows) instead."""
    rng = np.random.default_rng(80)
    X, y = _isolation_problem(rng)
    ℓ, params = pkg.LogisticRegression(X, y), po.logistic_params(X, y)
    K, D, bad = 16, 5, np.array([2, 5, 10, 13])
    q = rng.normal(size=(K, D)) * 0.5
    eps = np.exp(rng.uniform(np.log(0.05), np.log(0.3), K))
    eps[bad] = 1e300
    with _engine(pkg, ℓ, K, threads_per_chain=tpc) as eng:
        T, _ = eng.layout()
        eng.set_position(q)
        eng.set_stepsize(eps)
        res, _ = _tree_call(pkg, po, eng, LOGISTIC, params, None, 10, -1000.0)
        assert np.array_equal([k for k, o in enumerate(res) if not isinstance(o, dict)], bad)
        # mcmc: 3 transitions from the current state, transition counter back at 0 (the oracle's chains start there)
        eng.transition_count = 0
        st0 = eng.get_state(("q",))
        L = pkg._lib
        post, stats, ld = np.empty((K, 3, D)), np.zeros((K, 3), dtype=L.tree_stats_dtype), np.empty((K, 3))
        rc = eng._lib.dhmc_mcmc(eng._h, 3, L.ptr(post), L.ptr(stats), L.ptr(ld))
        status = eng.chain_status()
        for k in range(K):
            if k in bad:
                assert status[k] & NONFINITE_Q, k
                continue
            assert status[k] == 0
            o = po.mcmc_with_warmup(LOGISTIC, D, 3, SEED, k, stages=[], params=params, T=T, q0=st0["q"][k], eps0=eps[k])
            for n in range(3):
                _same_stats(o["tree_statistics"][n], stats[k, n], (k, n))
            assert _same(o["posterior_matrix"], post[k]) and _same(o["logdensities"], ld[k]), k
        with pytest.raises(pkg.DynamicHMCError):
            eng._ck(rc)
        # leapfrog (k_leapfrog runs one chain per CTA in every layout)
        eng.set_position(q)
        p = rng.normal(size=(K, D))
        eng.set_momentum(p)
        rc = eng._lib.dhmc_leapfrog(eng._h, 1, 1)
        status = eng.chain_status()
        st = eng.get_state(("q", "p", "lq", "grad"))
        for k in range(K):
            try:
                oq, op, og, ol = po.leapfrog(LOGISTIC, q[k], p[k], eps[k], params=params, T=T)
            except po.OracleError as e:
                assert k in bad and _oracle_bit(po, e) == NONFINITE_Q and status[k] == NONFINITE_Q
                continue
            assert k not in bad and status[k] == 0
            assert _same(oq, st["q"][k]) and _same(op, st["p"][k]) and _same(og, st["grad"][k]) and _same(ol, st["lq"][k])
        with pytest.raises(pkg.DynamicHMCError):
            eng._ck(rc)
    # the step-size search
    minv = np.ones((K, D))
    minv[bad] = 1e308
    with _engine(pkg, ℓ, K, threads_per_chain=tpc) as eng:
        eng.set_metric(minv)
        eng.set_position(q)
        rc = eng._lib.dhmc_find_initial_stepsize(eng._h, C.c_double(100.0), C.c_double(np.log(0.8)), C.c_int32(400))
        status = eng.chain_status()
        e_dev = eng.get_state(("eps",))["eps"]
        for k in range(K):
            p0 = po.rand_p(SEED, k, 1, 0, minv[k])
            try:
                e = po.find_initial_stepsize(LOGISTIC, q[k], p0, minv=minv[k], params=params, T=T, initial_eps=100.0)
            except po.OracleError as err:
                assert k in bad and _oracle_bit(po, err) == NONFINITE_Q and status[k] & NONFINITE_Q, (k, status[k])
                continue
            assert k not in bad and status[k] == 0 and e_dev[k] == e, k
        with pytest.raises(pkg.DynamicHMCError):
            eng._ck(rc)


# ------------------------------------------------------------------ leapfrog from a non-finite log density
@pytest.mark.gpu
@pytest.mark.parametrize("tpc", [0, 32], ids=["auto", "one_per_cta"])
def test_leapfrog_from_nonfinite_density_halts_only_that_chain(pkg, po, tpc):
    """the two ways a tree reaches leapfrog's @argcheck isfinite(Q.ℓq) (hamiltonian.jl:276): (1) min_Δ = −Inf, so a leaf
    at ℓ = −∞ is not divergent and the next leapfrog starts from it (DIAG_NORMAL, q₀ = (1.5e153, 0, 0, 0), ϵ = 5: the first
    leaf lands where q² overflows);
    (2) ℓ(q₀) = −∞ accepted by a strict evaluation with a given step size (q₀² overflows; the funnel at v ≈ −745).  The
    call raises ArgumentError, the halted chains keep their state, every other chain equals the oracle — in a tree and in
    mcmc."""
    rng = np.random.default_rng(90)
    K, D = 16, 4
    params = np.concatenate([np.zeros(D), np.ones(D)])
    q = rng.normal(size=(K, D))
    q[3] = [1.5e153, 0, 0, 0]
    q[12] = [2e154, 0.5, 0, 0]
    ℓ = pkg.DiagNormal(np.zeros(D), np.ones(D))
    eps = np.full(K, 0.4)
    eps[3] = 5.0
    for min_delta in (-np.inf, -1000.0):
        with _engine(pkg, ℓ, K, threads_per_chain=tpc, algorithm=pkg.NUTS(min_Δ=min_delta)) as eng:
            eng.set_position(q)
            eng.set_stepsize(eps)
            res, _ = _tree_call(pkg, po, eng, DIAG, params, None, 10, min_delta)
            halted = [k for k, o in enumerate(res) if not isinstance(o, dict)]
            assert halted == ([3, 12] if min_delta == -np.inf else [12]), halted
            # mcmc: the halted chains stop, the others run on (transition counter back at 0, where the oracle's chains start)
            eng.transition_count = 0
            st0 = eng.get_state(("q", "lq", "grad"))
            L = pkg._lib
            post, stats, ld = np.empty((K, 3, D)), np.zeros((K, 3), dtype=L.tree_stats_dtype), np.empty((K, 3))
            rc = eng._lib.dhmc_mcmc(eng._h, 3, L.ptr(post), L.ptr(stats), L.ptr(ld))
            status = eng.chain_status()
            st1 = eng.get_state(("q", "lq", "grad"))
            T, _ = eng.layout()
            for k in range(K):
                try:
                    o = po.mcmc_with_warmup(DIAG, D, 3, SEED, k, stages=[], params=params, T=T, q0=st0["q"][k],
                                            eps0=eps[k], min_delta=min_delta)
                except po.OracleError as e:
                    assert _oracle_bit(po, e) == LEAPFROG_NONFINITE and status[k] == LEAPFROG_NONFINITE, k
                    assert k in halted
                    for f in ("q", "lq", "grad"):
                        assert _same(st1[f][k], st0[f][k]), (k, f)
                    continue
                assert status[k] == 0, k
                for n in range(3):
                    _same_stats(o["tree_statistics"][n], stats[k, n], (k, n))
                assert _same(o["posterior_matrix"], post[k]) and _same(o["logdensities"], ld[k])
            with pytest.raises(pkg.ArgumentError, match="leapfrog called from non-finite log density"):
                eng._ck(rc)
    # the funnel's neck: exp(−v) overflows at v ≈ −745 and ℓ = −∞ is accepted
    Df = 5
    qf = rng.normal(size=(8, Df))
    for k in (1, 6):
        for v in np.linspace(-745.0, -709.0, 400):
            qf[k, 0] = v
            try:
                if po.evaluate_l(FUNNEL, qf[k], strict=True)[0] == -np.inf:
                    break
            except po.OracleError:
                pass
        assert po.evaluate_l(FUNNEL, qf[k], strict=True)[0] == -np.inf
    with _engine(pkg, pkg.Funnel(Df), 8, threads_per_chain=tpc) as eng:
        eng.set_position(qf)
        eng.set_stepsize(0.3)
        res, _ = _tree_call(pkg, po, eng, FUNNEL, None, None, 10, -1000.0)
        assert [k for k, o in enumerate(res) if not isinstance(o, dict)] == [1, 6]


def test_logistic_likelihood_at_overflowing_eta(po):
    """When η = xᵀβ overflows, a row's ll = yη − log(1 + e^η) is its limit: 0 for the outcome the sign predicts (y = 1 at
    η = +∞, y = 0 at η = −∞), −∞ for any other y; a NaN η stays NaN (ℓ is then sanitised to −∞ by evaluate_ℓ).  The
    formula itself would give ∞ − ∞ or 0·∞ = NaN, i.e. a wall where the density is finite.  Finite η keep their values."""
    rng = np.random.default_rng(3)
    p = 4
    sc = np.finfo(np.float64).max / OVERFLOW_AT
    X0 = rng.normal(size=(12, p)) / 2
    y0 = (rng.uniform(size=12) < 0.5).astype(float)
    for y_row, q0, want in ((1.0, 2.0, "finite"), (0.0, 2.0, "-inf"), (0.5, 2.0, "-inf"),
                            (0.0, -2.0, "finite"), (1.0, -2.0, "-inf"), (0.5, -2.0, "-inf")):
        X = np.vstack([X0, sc * np.eye(p)[:1]])
        y = np.append(y0, y_row)
        q = rng.normal(size=p) * 0.3
        q[0] = q0
        lq, g = po.logdensity_and_gradient(LOGISTIC, q, po.logistic_params(X, y))
        lq_ref, g_ref = po.logdensity_and_gradient(LOGISTIC, q, po.logistic_params(X0, y0))   # the row's limit is 0
        if want == "finite":
            assert np.isclose(lq, lq_ref, rtol=1e-13, atol=0) and np.allclose(g, g_ref, rtol=1e-13, atol=1e-13)
        else:
            assert lq == -np.inf, (y_row, q0, lq)
    # ∞ − ∞: two overflowing products in different 64-coefficient chunks (in one chunk the fused multiply-add keeps +∞)
    p2 = 128
    X = np.zeros((2, p2))
    X[0, 1], X[0, 100] = sc, -sc
    X[1, 1], X[1, 2] = sc, -sc
    q = np.zeros(p2)
    q[[1, 2, 100]] = 2.0
    assert np.isnan(po.logdensity_and_gradient(LOGISTIC, q, po.logistic_params(X[:1], np.array([1.0])))[0])
    assert po.logdensity_and_gradient(LOGISTIC, q, po.logistic_params(X[1:], np.array([1.0])))[0] == -6.0
    # finite η: bit for bit the formula y·η − (max(η, 0) + log(1 + e^{−|η|}))
    for eta, yv in ((3.0, 1.0), (-7.5, 0.0), (1e300, 1.0), (-1e300, 0.3), (0.0, 0.5)):
        X = np.array([[eta, 0.0]])
        lq, _ = po.logdensity_and_gradient(LOGISTIC, np.array([1.0, 0.0]), po.logistic_params(X, np.array([yv])))
        sp = po.math("softplus_neg", [abs(eta)])[0]
        assert lq == (yv * eta - (max(eta, 0.0) + sp)) - 0.5 * 1.0, (eta, yv)
