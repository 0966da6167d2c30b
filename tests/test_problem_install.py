"""dhmc_set_problem installs one problem through the installer of problem batches.  A handle that was given one problem,
then a batch, then another problem samples exactly as a fresh handle of each; a block that dhmc_set_problem refuses
leaves the previous problem in effect."""
import ctypes as C
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STD_NORMAL_USER = os.path.join(ROOT, "include", "models", "std_normal_user.h")


def _run(eng, eps):
    eng.random_position(); eng.set_stepsize(eps)
    return eng.mcmc(4)


def _assert_same(a, b):
    for f in ("posterior_matrix", "tree_statistics", "logdensities"):
        assert np.array_equal(a[f], b[f]), f


def _fresh_run(pkg, ℓ, chains, seed, eps, **kw):
    eng = pkg.Engine(ℓ, chains=chains, seed=seed, **kw)
    out = _run(eng, eps)
    eng.close()
    return out


def _single_batch_single(pkg, first, batch, last, chains, seed, eps, **kw):
    """One handle: `first`, then `batch` (a run), then `last` (a run from transition 0); each run equals a fresh handle's."""
    eng = pkg.Engine(first, chains=chains, seed=seed, **kw)
    eng._set_problem(batch)
    _assert_same(_run(eng, eps), _fresh_run(pkg, batch, chains, seed, eps, **kw))
    eng.transition_count = 0
    eng._set_problem(last)
    _assert_same(_run(eng, eps), _fresh_run(pkg, last, chains, seed, eps, **kw))
    eng.close()


def _logistic(pkg, N, seed, p=12):
    return pkg.LogisticRegression.synthetic(N=N, p=p, seed=seed)[0]


@pytest.mark.gpu
@pytest.mark.parametrize("threads_per_chain", [0, 32])
def test_logistic_single_batch_single(pkg, threads_per_chain):
    """Packed chain groups (automatic layout) and one chain per CTA; the last problem has an N of its own."""
    batch = pkg.ProblemBatch([_logistic(pkg, 60, 2), _logistic(pkg, 60, 3)], 8)
    _single_batch_single(pkg, _logistic(pkg, 100, 1), batch, _logistic(pkg, 57, 4), 16, 41, 0.05,
                         threads_per_chain=threads_per_chain)


@pytest.mark.gpu
def test_diag_normal_single_batch_single(pkg):
    rng = np.random.default_rng(5)
    diag = [pkg.DiagNormal(rng.normal(size=9) * 3, rng.uniform(0.3, 3, 9)) for _ in range(4)]
    _single_batch_single(pkg, diag[0], pkg.ProblemBatch(diag[1:3], 8), diag[3], 16, 42, 0.3)


@pytest.mark.gpu
def test_user_model_without_parameters_single_batch_single(pkg):
    """An empty parameter block before and after a batch of one-value blocks."""
    user = lambda pr: pkg.UserLogDensity(STD_NORMAL_USER, 5, params=pr)      # noqa: E731
    _single_batch_single(pkg, user([]), pkg.ProblemBatch([user([1.0]), user([2.0])], 8), user([]), 16, 43, 0.3)


@pytest.mark.gpu
def test_set_problem_refuses_a_logistic_n_that_is_not_an_integer_in_range(pkg):
    """N = NaN, -1, 2.5 (with the length of N = 2) and 2^31; after each refusal the handle samples the previous problem,
    in step with a handle that never saw the refused blocks."""
    L = pkg._lib
    prev = _logistic(pkg, 80, 5)
    eng = pkg.Engine(prev, chains=16, seed=44)
    ref = pkg.Engine(prev, chains=16, seed=44)
    blocks = []
    for v in (np.nan, -1.0, 2.0 ** 31):
        b = prev.params().copy(); b[0] = v
        blocks.append(b)
    b = _logistic(pkg, 2, 6).params().copy(); b[0] = 2.5
    blocks.append(b)
    for b in blocks:
        with pytest.raises(pkg.ArgumentError, match="integer"):
            eng._ck(eng._lib.dhmc_set_problem(eng._h, L.ptr(b), C.c_size_t(b.size)))
        _assert_same(_run(eng, 0.05), _run(ref, 0.05))
    eng.close()
    ref.close()
