"""Deterministic math + RNG shared by oracle and device (include/dhmc_math.h)."""
import numpy as np
import pytest

mp = pytest.importorskip("mpmath")


def _max_ulp(got, ref):
    worst = 0.0
    for g, r in zip(got, ref):
        r64 = float(r)
        if r64 == 0 or not np.isfinite(r64):
            continue
        worst = max(worst, float(abs((mp.mpf(float(g)) - r) / np.spacing(abs(r64)))))
    return worst


def test_exp_log_accuracy(po):
    mp.mp.prec = 200
    rng = np.random.default_rng(0)
    x = np.concatenate([rng.uniform(-700, 700, 4000), rng.uniform(-1, 1, 4000)])
    assert _max_ulp(po.math("exp", x), [mp.exp(mp.mpf(float(v))) for v in x]) < 1.5
    x = np.concatenate([np.exp(rng.uniform(-700, 700, 4000)), rng.uniform(0.5, 2, 4000),
                        [5e-324, 1e-310, 2.3e-308]])
    assert _max_ulp(po.math("log", x), [mp.log(mp.mpf(float(v))) for v in x]) < 1.5
    x = rng.uniform(-0.9, 5, 4000)
    assert _max_ulp(po.math("log1p", x), [mp.log1p(mp.mpf(float(v))) for v in x]) < 4
    u = rng.uniform(0, 1, 4000)
    assert _max_ulp(po.math("sin2pi", u), [mp.sin(2 * mp.pi * mp.mpf(float(v))) for v in u]) < 3
    assert _max_ulp(po.math("cos2pi", u), [mp.cos(2 * mp.pi * mp.mpf(float(v))) for v in u]) < 3


def test_exp_at_underflow_and_overflow(po):
    """dm_exp where the funnel's exp(−v) and the logistic link leave the normal range.  On [−745.14, −708.4] the result
    is subnormal (or rounds to 0), and the error is bounded in units of the subnormal spacing 2⁻¹⁰⁷⁴: below 1 everywhere
    (one of the two neighbours of the true value), and within 0.5 + 2⁻⁷ below 2⁻¹⁰³⁰, where the polynomial's relative
    error is worth less than 2⁻⁸ spacings — one rounding into the subnormal range, no double rounding.  Near
    log(floatmax) = 709.7827… the result is within 1.5 ulp, and +Inf exactly where the true value rounds past floatmax."""
    mp.mp.prec = 200
    rng = np.random.default_rng(1)
    sub = 2.0 ** -1074
    x = np.concatenate([rng.uniform(-745.14, -708.4, 6000), rng.uniform(-745.14, -744.0, 1000),
                        [-745.1332191019412, -745.13321910194122, -745.1332191019411, -708.3964185322641,
                         -708.39641853226408, -744.44007192138126, -745.14]])
    got = po.math("exp", x)
    ref = [mp.exp(mp.mpf(float(v))) for v in x]
    err = np.array([float(abs(mp.mpf(float(g)) - r) / sub) for g, r in zip(got, ref)])
    deep = np.array([r < mp.mpf(2) ** -1030 for r in ref])
    assert np.all(got >= 0)
    assert err.max() < 1.0, x[np.argmax(err)]
    assert deep.sum() > 2000 and err[deep].max() <= 0.5 + 2 ** -7, x[deep][np.argmax(err[deep])]
    assert np.any(got == 0.0) and np.any(got == sub)        # the two ends: rounds to 0, to the smallest subnormal
    fmax = np.finfo(np.float64).max
    x = np.concatenate([rng.uniform(709.0, 709.782712893384, 3000), np.nextafter(709.782712893384, 0) - np.arange(50) * 1e-13,
                        [709.782712893384, np.nextafter(709.782712893384, np.inf), 709.79]])
    got = po.math("exp", x)
    for g, v in zip(got, x):
        ref = mp.exp(mp.mpf(float(v)))
        if ref >= mp.mpf(fmax) + mp.mpf(2) ** 970:                # rounds to +Inf in binary64 (half an ulp of floatmax)
            assert g == np.inf, v
        else:
            assert np.isfinite(g) and abs(mp.mpf(float(g)) - ref) / np.spacing(float(ref)) < 1.5, v


def test_softplus_table_accuracy(po):
    """dm_softplus_neg(d) = log(1 + exp(-d)): table-driven, absolute error ~1e-16 (it is always
    added to max(a, b) inside logaddexp)."""
    mp.mp.prec = 200
    rng = np.random.default_rng(5)
    d = np.concatenate([rng.uniform(0, 40, 6000), np.exp(rng.uniform(-40, 3, 2000)),
                        [0.0, 36.7368005696771, 36.74, 50.0, 700.0, 745.0, 746.0]])
    got = po.math("softplus_neg", d)
    ref = np.array([float(mp.log1p(mp.exp(-mp.mpf(float(v))))) for v in d])
    assert np.max(np.abs(got - ref)) < 2.3e-16
    assert po.math("softplus_neg", [np.inf])[0] == 0.0 and np.isnan(po.math("softplus_neg", [np.nan])[0])


def test_special_values(po):
    inf, nan = np.inf, np.nan
    e = po.math("exp", [-inf, inf, 710.0, -746.0, 0.0])
    assert list(e) == [0.0, inf, inf, 0.0, 1.0]
    assert np.isnan(po.math("exp", [nan])[0])
    l = po.math("log", [0.0, inf, 1.0])
    assert list(l) == [-inf, inf, 0.0]
    assert np.isnan(po.math("log", [-1.0])[0])
    la = po.math("logaddexp", [-inf, -inf, 0.0, 1.0], [-inf, 1.0, -inf, 1.0])
    assert la[0] == -inf and la[1] == 1.0 and la[2] == 0.0
    assert abs(la[3] - (1.0 + np.log(2.0))) < 1e-15
    # agrees with numpy to absolute 1e-15 on a broad range
    rng = np.random.default_rng(1)
    a, b = rng.uniform(-60, 10, 2000), rng.uniform(-60, 10, 2000)
    assert np.max(np.abs(po.math("logaddexp", a, b) - np.logaddexp(a, b))) < 5e-15


def test_philox_known_answers(po):
    # Random123 kat_vectors, philox4x32-10
    assert [hex(v) for v in po.philox([0, 0, 0, 0], [0, 0])] == \
        ['0x6627e8d5', '0xe169c58d', '0xbc57ac4c', '0x9b00dbd8']
    assert [hex(v) for v in po.philox([0xffffffff] * 4, [0xffffffff] * 2)] == \
        ['0x408f276d', '0x41c83b0e', '0xa20bc7c6', '0x6d5451fd']
    assert [hex(v) for v in po.philox([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344],
                                      [0xa4093822, 0x299f31d0])] == \
        ['0xd16cfe09', '0x94fdcceb', '0x5001e420', '0x24126ea1']


def test_rng_distributions(po):
    z = po.normals(7, 3, 2, 5, 100000)
    assert abs(z.mean()) < 0.015 and abs(z.std() - 1) < 0.01
    assert abs(np.mean(z ** 4) - 3) < 0.1
    # distinct (chain, t, stream) give distinct streams; same inputs are reproducible
    assert np.array_equal(z, po.normals(7, 3, 2, 5, 100000))
    assert not np.array_equal(z[:100], po.normals(7, 4, 2, 5, 100))
    assert not np.array_equal(z[:100], po.normals(7, 3, 2, 6, 100))
    q = po.random_position(1, 0, 50000)
    assert q.min() > -2 and q.max() < 2 and abs(q.mean()) < 0.03
    e = np.array([po.randexp(1, 2, 3, j) for j in range(20000)])
    assert e.min() > 0 and abs(e.mean() - 1) < 0.03


def test_canonical_reduction_width(po):
    rng = np.random.default_rng(3)
    a, b = rng.normal(size=1000), rng.normal(size=1000)
    ref = float(np.dot(a, b))
    for T in (0, 32, 64, 128, 256):
        assert abs(po.canon_dot(T, a, b) - ref) < 1e-12
    # explicit restatement of the canonical order for T = 64: lane-strided partials,
    # per-warp pairwise tree with offsets 16,8,4,2,1, then warps with offsets 32,...
    T = 64
    part = np.zeros(T)
    for v in range(T):
        acc = 0.0
        for i in range(v, 1000, T):
            acc = acc + a[i] * b[i]
        part[v] = acc
    for base in range(0, T, 32):
        off = 16
        while off >= 1:
            for v in range(base, base + off):
                part[v] = part[v] + part[v + off]
            off //= 2
    part[0] = part[0] + part[32]
    assert po.canon_dot(T, a, b) == part[0]


def test_logaddexp_at_logexpfunctions_branch_points(po):
    """LogExpFunctions.logaddexp(x, y) = max + log1pexp(-|x - y|), and its Float64 log1pexp switches formulas at
    x0 ≈ -745.13 (exp underflows), x1 ≈ -36.74 (log1p(e) == e), x2 ≈ 18.02 and x3 ≈ 33.23 (SURVEY.md §8c-i).  The package is
    not vendored with the reference, so these are pinned against an 80-digit evaluation: the engine's table-driven
    logaddexp must agree with the true value to a few ulp ON BOTH SIDES of every branch point (any branch of the Julia
    implementation is itself accurate to ~1 ulp there, so this bounds the engine-vs-Julia difference)."""
    import mpmath
    mpmath.mp.dps = 80
    pts = []
    for c in (-745.1332191019412, -36.7368005696771, 18.021826694558577, 33.23111882352963, 0.0, -1e-300, -0.6931471805599453):
        for k in (-3, -1, 0, 1, 3):
            pts.append(float(np.nextafter(c, np.inf)) if k > 0 else float(np.nextafter(c, -np.inf)) if k < 0 else c)
            pts.append(c + k * 1e-9)
    pts = np.array(sorted(set(pts)))
    for base in (0.0, 3.5, -120.25, 1e6):
        a = np.full(pts.size, base); b = base + pts          # b - a = the branch-point argument
        got = po.math("logaddexp", a, b)
        for ai, bi, gi in zip(a, b, got):
            true = mpmath.log(mpmath.exp(mpmath.mpf(ai)) + mpmath.exp(mpmath.mpf(bi))) if max(ai, bi) < 700 else \
                mpmath.mpf(max(ai, bi)) + mpmath.log1p(mpmath.exp(-abs(mpmath.mpf(ai) - mpmath.mpf(bi))))
            err = abs(mpmath.mpf(float(gi)) - true)
            ulp = np.spacing(abs(float(true))) if float(true) != 0 else 5e-324
            assert err <= 4 * ulp + mpmath.mpf(2.3e-16), (ai, bi, gi, float(true))
