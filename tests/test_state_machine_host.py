"""The product's flattened NUTS state machine (nuts_machine.cuh, compiled for the
host by tests/hostsim) against the recursive oracle: integers bit-exact, floats
bit-exact (same canonical reduction, same deterministic math, same RNG)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim"))
import pyhostsim as hs  # noqa: E402

INT_FIELDS = ("depth", "left", "right", "steps", "directions")


def _same_stats(a, b):
    for f in INT_FIELDS:
        assert a[f] == b[f], (f, a, b)
    assert a["pi"] == b["pi"] or (np.isnan(a["pi"]) and np.isnan(b["pi"]))
    assert a["acceptance_rate"] == b["acceptance_rate"]


def _problem(rng, family, D):
    if family == 1:
        return np.concatenate([rng.normal(size=D), rng.uniform(0.2, 5.0, D)])
    if family == 3:
        N = int(rng.integers(20, 80))
        X = rng.normal(size=(N, D)) / np.sqrt(D)
        y = (rng.uniform(size=N) < 0.5).astype(float)
        return np.concatenate([[float(N)], X.ravel(), y])
    return None


@pytest.mark.parametrize("family", [0, 1, 2, 3])
def test_single_transitions_match_oracle(po, family):
    rng = np.random.default_rng(100 + family)
    seen_depths, seen_div, seen_turn_sub, seen_max = set(), 0, 0, 0
    for trial in range(250):
        D = int(rng.choice([2, 3, 10, 33, 100]))
        T = int(rng.choice([32, 64, 128])) if D > 32 else 32
        params = _problem(rng, family, D)
        minv = rng.uniform(0.3, 3.0, D) if trial % 2 else np.ones(D)
        q = rng.normal(size=D)
        eps = float(np.exp(rng.uniform(np.log(0.005), np.log(1.5))))
        max_depth = int(rng.choice([1, 2, 3, 5, 8, 10]))
        min_delta = -1000.0 if trial % 5 else -0.05     # force "divergences" sometimes
        seed, chain, t = int(rng.integers(1 << 40)), int(rng.integers(1 << 20)), int(rng.integers(1000))
        o = po.sample_tree(family, q, eps, seed, chain, t, minv=minv, params=params, T=T,
                           max_depth=max_depth, min_delta=min_delta)
        h = hs.run(family, q, eps, seed, chain, t0=t, N=1, minv=minv, params=params, T=T,
                   max_depth=max_depth, min_delta=min_delta)
        _same_stats(o["stats"], h["tree_statistics"][0])
        assert np.array_equal(o["q"], h["q"]) and np.array_equal(o["g"], h["g"]) and o["lq"] == h["lq"]
        s = o["stats"]
        seen_depths.add(int(s["depth"]))
        seen_div += int(s["left"] == s["right"])
        seen_turn_sub += int(s["left"] != s["right"] and abs(s["right"] - s["left"]) + 1 < 2 ** s["depth"])
        seen_max += int((s["left"], s["right"]) == (1, 0))
    # the sweep must actually exercise every exit of the tree
    assert len(seen_depths) >= 5 and seen_div > 5 and seen_turn_sub > 5 and seen_max > 5


def test_overrides_p_and_directions(po):
    rng = np.random.default_rng(7)
    D = 20
    for flags in (0, 0xFFFFFFFF, 0b101, 0b110101, 0xAAAAAAAA):
        q, p = rng.normal(size=D), rng.normal(size=D)
        o = po.sample_tree(0, q, 0.2, 1, 2, 3, p=p, directions=flags, T=32)
        h = hs.run(0, q, 0.2, 1, 2, t0=3, p=p, directions=flags, T=32)
        _same_stats(o["stats"], h["tree_statistics"][0])
        assert o["stats"]["directions"] == flags
        assert np.array_equal(o["q"], h["q"])


def test_always_divergent_equivalent(po):
    # huge step on the funnel: first leaf diverges -> depth 0, steps 1, rate from Δ
    q = np.zeros(10)
    q[0] = -8.0
    q[1:] = 5.0
    o = po.sample_tree(2, q, 50.0, 1, 0, 0)
    h = hs.run(2, q, 50.0, 1, 0)
    _same_stats(o["stats"], h["tree_statistics"][0])
    assert o["stats"]["depth"] == 0 and o["stats"]["steps"] == 1
    assert o["stats"]["left"] == o["stats"]["right"]
    assert np.array_equal(h["q"], q)


@pytest.mark.parametrize("family,D,T", [(0, 100, 32), (1, 50, 64), (2, 10, 32)])
def test_full_warmup_matches_oracle_welford(po, family, D, T):
    # Same stages, Welford metric on both sides => identical chains, bit for bit.
    rng = np.random.default_rng(5)
    params = _problem(rng, family, D)
    seed, chain = 77, 3
    stages = po.default_warmup_stages(init_steps=30, middle_steps=20, doubling_stages=2,
                                      terminating_steps=20)
    o = po.mcmc_with_warmup(family, D, 40, seed, chain, stages=stages, params=params, T=T,
                            welford=True, keep_warmup=True)
    # drive the host simulation through the same stage sequence
    q0 = po.random_position(seed, chain, D)
    eps, st = hs.find_initial_stepsize(family, q0, seed, chain, params=params, T=T)
    assert st == 0
    q, minv, t = q0, np.ones(D), 0
    wstats = []
    for kind, N, metric, da_on in stages[1:]:
        r = hs.run(family, q, eps, seed, chain, t0=t, N=N, minv=minv, params=params, T=T,
                   adapt=(0.8, 0.05, 0.75, 10) if da_on else None, metric=metric)
        q, minv, eps, t = r["q"], r["minv"], r["eps"], t + N
        wstats.append(r["tree_statistics"])
        assert r["status"] == 0
    wstats = np.concatenate(wstats)
    for f in INT_FIELDS:
        assert np.array_equal(wstats[f], o["warmup_stats"][f]), f
    assert np.array_equal(wstats["acceptance_rate"], o["warmup_stats"]["acceptance_rate"])
    assert eps == o["eps"] and np.array_equal(minv, o["minv"])
    r = hs.run(family, q, eps, seed, chain, t0=t, N=40, minv=minv, params=params, T=T)
    assert np.array_equal(r["posterior_matrix"], o["posterior_matrix"])
    assert np.array_equal(r["logdensities"], o["logdensities"])
    for f in INT_FIELDS + ("pi", "acceptance_rate"):
        assert np.array_equal(r["tree_statistics"][f], o["tree_statistics"][f]), f


def test_initial_stepsize_matches_oracle(po):
    rng = np.random.default_rng(11)
    for family in (0, 1, 2):
        for _ in range(20):
            D = int(rng.choice([5, 10, 64]))
            params = _problem(rng, family, D)
            minv = rng.uniform(0.3, 3, D)
            q, p = rng.normal(size=D), rng.normal(size=D)
            e_o = po.find_initial_stepsize(family, q, p, minv=minv, params=params, T=32)
            e_h, st = hs.find_initial_stepsize(family, q, 1, 0, minv=minv, params=params, T=32, p=p)
            assert st == 0 and e_o == e_h


def test_slot_pool_is_large_enough():
    # max_depth 12 must fit the 64-slot pool of this build
    assert hs.lib().hs_slots_needed(12) <= 64
    rng = np.random.default_rng(3)
    q = rng.normal(size=4)
    r = hs.run(0, q, 1e-3, 9, 9, max_depth=12, N=2)      # tiny ϵ: never turns, reaches depth 12
    assert np.all(r["tree_statistics"]["depth"] == 12)
    assert np.all(r["tree_statistics"]["steps"] == 2 ** 12 - 1)


# ---- the flattened machine on the reference's DummyTrajectory (test/test_trees.jl) ----
def test_dummy_sampled_tree_known_answer():
    """test_trees.jl:156-165: sample_trajectory(…, 0, 3, Directions(0b101))."""
    r = hs.dummy_sample_trajectory(0, 3, 0b101)
    assert r["visited"] == [1, -1, -2, 2, 3, 4, 5]
    assert r["termination"] == (1, 0) and r["depth"] == 3 and r["steps"] == 7


@pytest.mark.parametrize("kw,z", [(dict(), 0), (dict(turning=[1, 2]), 3), (dict(divergent=[10, 11]), 3),
                                  (dict(divergent=[10, 11, 12], turning=[-3, -2]), 3),
                                  (dict(turning=[5, 6, 7]), 0), (dict(divergent=[5, 6, 7]), 0),
                                  (dict(turning=[-1, -2, -3, -4]), 0)])
def test_flattened_tree_matches_reference_recursion_exhaustively(po, kw, z):
    """Every direction word up to depth 6 (the sets of test_trees.jl:238-262 and :126-142): visited
    order, depth, termination code (incl. the unsorted backward turning span) and step count of the
    flattened explicit-stack tree equal those of the reference-style recursion."""
    for depth in range(1, 7):
        for flags in range(2 ** depth):
            o = po.dummy_sample_trajectory(z, depth, flags, **kw)
            h = hs.dummy_sample_trajectory(z, depth, flags, **kw)
            assert h["visited"] == o["visited"], (depth, flags)
            assert h["depth"] == o["depth"] and h["termination"] == o["termination"], (depth, flags, h, o)
            assert h["steps"] == o["v"][1]


# ---- property-based sweep (hypothesis): flattened machine == recursive oracle on arbitrary inputs ----
from hypothesis import given, settings, strategies as st  # noqa: E402


@settings(max_examples=150, deadline=None)
@given(family=st.sampled_from([0, 1, 2, 3]), D=st.integers(2, 70), T=st.sampled_from([32, 64]),
       logeps=st.floats(-6.0, 1.0), max_depth=st.integers(1, 9), seed=st.integers(0, 2 ** 40),
       chain=st.integers(0, 2 ** 30), t=st.integers(0, 5000), dirs=st.one_of(st.none(), st.integers(0, 2 ** 32 - 1)),
       min_delta=st.sampled_from([-1000.0, -1.0, -0.01]))
def test_hypothesis_single_transition(po, family, D, T, logeps, max_depth, seed, chain, t, dirs, min_delta):
    rng = np.random.default_rng(seed % (2 ** 32))
    params = _problem(rng, family, D)
    minv = np.exp(rng.uniform(-2, 2, D))
    q = rng.normal(size=D)
    eps = float(np.exp(logeps))
    try:
        o = po.sample_tree(family, q, eps, seed, chain, t, minv=minv, params=params, T=T, max_depth=max_depth,
                           min_delta=min_delta, directions=dirs)
    except po.OracleError:
        return      # non-finite position: the reference throws (hamiltonian.jl:203); the device flags the chain
    h = hs.run(family, q, eps, seed, chain, t0=t, N=1, minv=minv, params=params, T=T, max_depth=max_depth,
               min_delta=min_delta, directions=dirs)
    _same_stats(o["stats"], h["tree_statistics"][0])
    assert np.array_equal(o["q"], h["q"]) and o["lq"] == h["lq"]


# ---- leapfrog's @argcheck isfinite(Q.ℓq) (hamiltonian.jl:276): a leapfrog never starts from ℓ = −∞ ----
LEAPFROG_NONFINITE = 64     # DHMC_CHAIN_LEAPFROG_NONFINITE, include/dhmc.h


def _raises_leapfrog_argcheck(po, fn):
    try:
        fn()
    except po.OracleError as e:
        assert e.status == 1 and "leapfrog called from non-finite log density" in str(e), e
        return True
    return False


def test_leapfrog_from_nonfinite_density_halts_the_chain(po):
    """The two ways a tree reaches a leapfrog from ℓ = −∞, where the reference raises ArgumentError and the machine used
    to go on with status 0: (1) min_Δ = −Inf: from q₀ = 1e153 the first leaf lands where q² overflows, ℓ = −∞ there, Δ = −∞
    is not below min_Δ, so the leaf is not divergent and the next leapfrog starts from it; (2) a strict evaluation accepts
    ℓ(q₀) = −∞ (q₀² overflows), and the first leapfrog starts from q₀.  The machine flags the chain and stops it, also when
    the call asked for more transitions.  (That the chain then keeps its stored state is the kernels' part: k_nuts and
    k_leapfrog do not write a halted chain back, which the GPU tests check.)"""
    D = 4
    params = np.concatenate([np.zeros(D), np.ones(D)])
    for q, eps, min_delta in ((np.array([1e153, 0, 0, 0.]), 5.0, -np.inf), (np.array([2e154, 0, 0, 0.]), 0.5, -1000.0)):
        po.evaluate_l(1, q, params, strict=True)            # accepted: ℓ(q₀) is finite, or −∞
        assert _raises_leapfrog_argcheck(po, lambda: po.sample_tree(1, q, eps, 1, 0, 0, params=params, min_delta=min_delta))
        for N in (1, 3):
            h = hs.run(1, q, eps, 1, 0, N=N, params=params, min_delta=min_delta)
            assert h["status"] == LEAPFROG_NONFINITE
            assert np.all(h["tree_statistics"]["steps"] == 0)     # it halts in its first transition: nothing recorded


def test_near_overflow_starts_match_oracle():
    """Random starts near overflow that a strict evaluation accepts: DIAG_NORMAL with one |q_i| in [1e153, 1e155] (q²
    overflows beyond 1.34e154) and the funnel with v in ±[700, 746] (exp(−v) overflows or is subnormal).  Where the
    oracle raises the leapfrog ArgumentError the machine flags exactly that; everywhere else the
    tree equals the oracle's bit for bit with status 0."""
    import pyoracle as po
    rng = np.random.default_rng(2)
    seen = {1: [0, 0], 2: [0, 0]}
    for family in (1, 2):
        for trial in range(250):
            D = int(rng.choice([2, 4, 10]))
            q = rng.normal(size=D)
            if family == 1:
                params = np.concatenate([rng.normal(size=D), rng.uniform(0.5, 2, D)])
                q[rng.integers(D)] = rng.choice([-1, 1]) * np.exp(rng.uniform(np.log(1e153), np.log(1e155)))
            else:
                params = None
                q[0] = rng.uniform(-746, -700) if trial % 2 else rng.uniform(700, 746)
                q[1:] *= np.exp(rng.uniform(-5, 5))
            try:
                po.evaluate_l(family, q, params, strict=True)
            except po.OracleError:
                continue
            eps = float(np.exp(rng.uniform(-3, 1)))
            h = hs.run(family, q, eps, 1, trial, params=params)
            out = {}
            if _raises_leapfrog_argcheck(po, lambda: out.update(po.sample_tree(family, q, eps, 1, trial, 0, params=params))):
                assert h["status"] == LEAPFROG_NONFINITE, (family, trial)
                seen[family][0] += 1
            else:
                assert h["status"] == 0, (family, trial)
                _same_stats(out["stats"], h["tree_statistics"][0])
                assert np.array_equal(out["q"], h["q"]) and np.array_equal(out["g"], h["g"]) and out["lq"] == h["lq"]
                seen[family][1] += 1
    assert all(a >= 20 and b >= 20 for a, b in seen.values()), seen
