"""Every NUTS template-kernel instantiation the library ships, against the oracle.

The host picks one instantiation of k_nuts, k_search, k_leapfrog, k_eval and k_phase per handle from the family, the
layout (warps per chain W, elements per thread EPL), the packing of 8 logistic chains per CTA (G = 8), max_depth > 12
(the deep twins, DP) and the metric kind (DN).  CASES below is a table of handles, each (family, D, threads_per_chain,
max_depth, B); `launched(case)` restates the host's choice and names the instantiations the case runs.

CPU (after __graft_entry__.build()): the entry functions in the sm_90a code of libdhmc_b200.so and of the Rosenbrock
user-model library must all be claimed by a case (or listed in UNREACHABLE with a reason), every claimed name must exist,
and the deep cases' step sizes must make the oracle's trees deeper than 12.

GPU: every case, first with a diagonal and then with a Symmetric metric, bit-equal to the oracle through every kernel:
k_eval (set / random position), k_search (initial step-size search), k_phase, k_leapfrog (forwards, then backwards),
k_nuts (two trees, then on a fresh handle a warm-up window and draws)."""
import contextlib
import os
import re
import subprocess
import zlib
from typing import NamedTuple

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dynamichmc.jl_b200", "csrc")
ROSENBROCK = os.path.join(ROOT, "include", "models", "rosenbrock.h")
ROSENBROCK_PARAMS = np.array([1.0, 0.5])
CUDA_BIN = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin")   # csrc/Makefile: NVCC ?= /usr/local/cuda/bin/nvcc

STD, DIAG, FUNNEL, LOGISTIC, USER = 0, 1, 2, 3, 4      # include/dhmc.h DHMC_FAMILY_*
FAMILY_NAMES = {STD: "std", DIAG: "diag", FUNNEL: "funnel", LOGISTIC: "logistic", USER: "rosenbrock"}
TEMPLATE_KERNELS = ("k_nuts", "k_search", "k_leapfrog", "k_eval", "k_phase")
HEAVY = ("k_nuts", "k_search")
# the host's utility kernels (dhmc_b200.cu): not templates of a layout, checked by the suite's other tests
UTILITY_KERNELS = ("k_dense_factor", "k_cov_finish", "k_cov_pool", "k_pad_metric", "k_pad_rows", "k_transpose",
                   "k_tree_summary", "k_pilot_mean", "k_ess_rhat", "k_acceptance_hist", "k_broadcast", "k_broadcast_mat",
                   "k_fill")
# shipped instantiations no handle can launch: {name: reason}
UNREACHABLE = {}

K_PACK = 8                  # kernels.cuh: kPack
DEEP_ABOVE = 12             # dhmc_b200.cu:608: max_depth > 12 selects the deep twins
DEEP_DEPTH = 14
LOGISTIC_N = 33             # observations of the logistic cases: one full 32-row block and a ragged one
DENSE_MAX_DIM = 4097        # the Symmetric phase runs up to here: (8, 32)'s dense kernels at the smallest dim of that layout
DENSE_PER_CHAIN_MAX_DIM = 256   # up to here every chain has its own M⁻¹; above, all share one block-diagonal M⁻¹
DENSE_BLOCK = 16
DENSE_WINDOW_MAX_DIM = 513  # up to here the warm-up window of the dense phase estimates a new Symmetric M⁻¹
DRAWS_MAX_DIM_DENSE = 2048  # above, the dense phase stops after the trees (the oracle's mat-vec is O(D²) per leapfrog)
SEED = 2027
N_WINDOW, N_DRAWS = 20, 2
INT_FIELDS = ("depth", "left", "right", "steps", "directions")


# ------------------------------------------------------------------ restatement of the host's kernel choice
def layout_supported(W, epl):
    """kernels.cuh:387-392"""
    return epl in {1: (1, 2, 4, 8), 2: (4, 8), 4: (4, 8), 8: (4, 8, 16, 32)}.get(W, ())


def choose_layout(D, req_T):
    """dhmc_b200.cu:531-551 -> (T, EPL); (0, 0) when no layout fits"""
    if req_T:
        W = req_T // 32
        e = -(-D // req_T)
        e = next((v for v in (1, 2, 4, 8, 16, 32) if e <= v), 0)
        if e and not layout_supported(W, e):
            e = 4 if e < 4 and layout_supported(W, 4) else 8 if e < 8 and layout_supported(W, 8) else 0
        return req_T, e
    for bound, T, e in ((32, 32, 1), (64, 32, 2), (128, 32, 4), (256, 64, 4), (512, 128, 4), (1024, 128, 8),
                        (2048, 256, 8), (4096, 256, 16), (8192, 256, 32)):
        if D <= bound:
            return T, e
    return 0, 0


def handle_layout(family, D, req_T, max_depth):
    """dhmc_create, dhmc_b200.cu:603-612 -> (T, EPL, G): logistic regression with the automatic layout, dim <= 256 and
    max_depth <= 12 packs 8 chains per CTA, one warp each (8 elements per lane above dim 128)"""
    T, e = choose_layout(D, req_T)
    if family == LOGISTIC and req_T == 0 and D <= 32 * K_PACK and max_depth <= DEEP_ABOVE:
        return (32, 8, K_PACK) if D > 128 else (T, e, K_PACK)
    return T, e, 1


def kernel_part(kernel, deep, G):
    """dhmc_b200.cu:437-441; launch() passes G = 1 for the light kernels (:491)"""
    if kernel in HEAVY and deep:
        return 3
    return 1 if kernel in HEAVY and G > 1 else 0


def kernel_name(kernel, EPL, family, W, dense, part):
    """kernel_ptr, kernels.cuh:402-443: the demangled instantiation, or None where kernel_ptr returns nullptr"""
    DN = "true" if dense else "false"
    if part == 3:
        return f"dhmc::{kernel}<{EPL}, {family}, {W}, {DN}, 1, true>" if kernel in HEAVY else None
    if part == 1:
        ok = family == LOGISTIC and W == 1 and kernel in HEAVY
        return f"dhmc::{kernel}<{EPL}, {family}, {W}, {DN}, {K_PACK}, false>" if ok else None
    if kernel == "k_eval":                    # one instantiation for both metrics (the dense switch falls through)
        return f"dhmc::k_eval<{EPL}, {family}, {W}>"
    if kernel in HEAVY:
        return f"dhmc::{kernel}<{EPL}, {family}, {W}, {DN}, 1, false>"
    return f"dhmc::{kernel}<{EPL}, {family}, {W}, {DN}>"


class Case(NamedTuple):
    family: int
    D: int
    T: int = 0              # threads_per_chain (0: the automatic layout)
    max_depth: int = 10
    B: int = 0              # chains (0: by dimension)

    @property
    def K(self):
        if self.B:
            return self.B
        if self.deep:           # trees of 8 191 - 16 383 leapfrog steps in the oracle
            return 2 if self.D <= 257 else 1
        return 3 if self.D <= 257 else 2 if self.D <= 1025 else 1

    @property
    def deep(self):
        return self.max_depth > DEEP_ABOVE

    @property
    def dense(self):
        return self.D <= DENSE_MAX_DIM

    def layout(self):
        return handle_layout(self.family, self.D, self.T, self.max_depth)

    def __str__(self):
        return f"{FAMILY_NAMES[self.family]}-D{self.D}-T{self.T}-md{self.max_depth}-B{self.K}"


def launched(case):
    """the instantiations the case's handles launch: every kernel, diagonal and (if the case has a dense phase) Symmetric"""
    T, EPL, G = case.layout()
    names = set()
    for dense in (False, True) if case.dense else (False,):
        for k in TEMPLATE_KERNELS:
            n = kernel_name(k, EPL, case.family, T // 32, dense, kernel_part(k, case.deep, G))
            assert n is not None, (case, k, dense)
            names.add(n)
    return names


# (D, threads_per_chain) reaching each of the twelve layouts at its smallest dim (lower bound + 1: only the first lanes'
# last element is live), D odd wherever the layout allows
LAYOUT_CASES = [(2, 0), (33, 0), (97, 0), (129, 32), (129, 0), (257, 64), (257, 0), (513, 0), (769, 256), (1025, 0),
                (2049, 0), (4097, 0)]


def _cases():
    cases = []
    for fam in (STD, DIAG, FUNNEL, LOGISTIC, USER):
        for D, T in LAYOUT_CASES:
            if fam == DIAG and D == 2:
                D = 1
            for md in (10, DEEP_DEPTH):
                # logistic, dim <= 256: the automatic layout packs 8 chains per CTA; an explicit threads_per_chain keeps
                # one chain per CTA at the layout the automatic choice would give
                t = choose_layout(D, 0)[0] if fam == LOGISTIC and T == 0 and D <= 256 and md <= DEEP_ABOVE else T
                cases.append(Case(fam, D, t, md))
    cases += [Case(LOGISTIC, p, 0, 10, 8) for p in (1, 33, 97, 129)]     # packed chain groups, one per lane count
    cases.append(Case(STD, 8192, 0, 10, 1))                              # fully populated (8, 32)
    cases.append(Case(STD, 2, 0, 10, 2200))                              # more chains than light_grid = 16 · 132 SMs
    return cases


CASES = _cases()


# ------------------------------------------------------------------ what ships
def _entry_functions(so):
    """demangled __global__ entry functions of the sm_90a code in `so`"""
    out = subprocess.run([os.path.join(CUDA_BIN, "cuobjdump"), "-symbols", so], check=True, capture_output=True,
                         text=True).stdout
    mangled = sorted({ln.split()[-1] for ln in out.splitlines() if "STO_ENTRY" in ln})
    dem = subprocess.run([os.path.join(CUDA_BIN, "cu++filt")], input="\n".join(mangled) + "\n", check=True,
                         capture_output=True, text=True).stdout.split("\n")
    names = set()
    for d in dem[:len(mangled)]:
        d = re.sub(r"\(int\)", "", d)
        d = d.replace("(bool)0", "false").replace("(bool)1", "true")
        m = re.fullmatch(r"void (dhmc::k_\w+<[^<>()]*>)\(dhmc::KArgs\)|(k_\w+)\([^()]*\)", d)
        assert m, f"{so}: entry function of an unknown form: {d}"     # every entry is classified, none is dropped
        names.add(m.group(1) or m.group(2))
    assert len(names) == len(mangled), so
    return names


def _shipped(pkg):
    stock = _entry_functions(os.path.join(CSRC, "libdhmc_b200.so"))
    user = _entry_functions(pkg.compile_user_model(ROSENBROCK, deep=True))    # the build __graft_entry__.build() prepares
    out = {}
    for lib, names in (("stock", stock), ("rosenbrock", user)):
        util = {n for n in names if n in UTILITY_KERNELS}
        tmpl = names - util
        assert util == set(UTILITY_KERNELS), (lib, util ^ set(UTILITY_KERNELS))
        assert all(re.match(r"dhmc::(%s)<" % "|".join(TEMPLATE_KERNELS), n) for n in tmpl), (lib, tmpl)
        out[lib] = tmpl
    return out


def test_every_shipped_instantiation_is_claimed_by_a_case(pkg):
    shipped = _shipped(pkg)
    every = shipped["stock"] | shipped["rosenbrock"]
    claimed = {}
    for c in CASES:
        for n in launched(c):
            claimed.setdefault(n, []).append(str(c))
    missing = sorted(n for n in claimed if n not in every)
    assert not missing, f"claimed by a case but not in the libraries: {missing}"
    assert not set(UNREACHABLE) - every, "UNREACHABLE lists names that do not ship"
    orphans = sorted(every - set(claimed) - set(UNREACHABLE))
    assert not orphans, f"{len(orphans)} shipped instantiation(s) no case launches: {orphans}"
    family = lambda n: int(n.split("<")[1].split(",")[1])      # noqa: E731
    assert {family(n) for n in shipped["rosenbrock"]} == {USER}
    assert {family(n) for n in shipped["stock"]} == {STD, DIAG, FUNNEL, LOGISTIC}
    print(f"\n{len(every)} shipped template-kernel instantiations ({len(shipped['stock'])} in libdhmc_b200.so, "
          f"{len(shipped['rosenbrock'])} in the Rosenbrock library); {len(every & set(claimed))} launched by the "
          f"{len(CASES)} cases, {len(UNREACHABLE)} unreachable")


def test_layout_rules_agree_with_the_shipped_layouts(pkg):
    """The restated layout choice only yields supported layouts, reaches each one, and these are exactly the (W, EPL)
    pairs the libraries instantiate for every family (family_kernel_ptr)."""
    supported = {(W, e) for W in (1, 2, 4, 8) for e in (1, 2, 4, 8, 16, 32) if layout_supported(W, e)}
    reached = set()
    for T in (0, 32, 64, 128, 256):
        for D in range(1, 8194):
            t, e = choose_layout(D, T)
            if e == 0:
                assert D > 32 * (T or 256) or (T == 32 and D > 256) or (T == 64 and D > 512) or (T == 128 and D > 1024), (D, T)
                continue
            assert (t // 32, e) in supported and t * e >= D, (D, T, t, e)
            reached.add((t // 32, e))
    assert reached == supported
    shipped = _shipped(pkg)
    for fam in (STD, DIAG, FUNNEL, LOGISTIC, USER):
        lib = shipped["rosenbrock" if fam == USER else "stock"]
        pat = re.compile(r"dhmc::k_leapfrog<(\d+), %d, (\d+), false>" % fam)
        got = {(int(m.group(2)), int(m.group(1))) for n in lib for m in [pat.match(n)] if m}
        assert got == supported, (fam, got ^ supported)
    for c in CASES:
        T, e, G = c.layout()
        assert layout_supported(T // 32, e) and T * e >= c.D and (G == 1 or T == 32), c


# ------------------------------------------------------------------ case inputs (shared by the CPU and GPU tests)
def _spd(rng, n):
    A = rng.normal(size=(n, n))
    return 0.3 * (A @ A.T) / n + np.diag(rng.uniform(0.7, 1.3, n))


def block_diagonal_metric(po, D, seed=0):
    """(M⁻¹, W): a block-diagonal SPD M⁻¹ with 16 x 16 blocks and W = cholesky(inv(M⁻¹)).L assembled from the blocks'
    factors.  Every product and sum dense_factor forms across two blocks is an exact zero, so the assembled W is what
    dense_factor(M⁻¹) returns (test_block_diagonal_factor_is_the_blockwise_factor), at O(D·16²) instead of O(D³)."""
    rng = np.random.default_rng(7000 + D + seed)
    M, W = np.zeros((D, D)), np.zeros((D, D))
    for a in range(0, D, DENSE_BLOCK):
        b = min(D, a + DENSE_BLOCK)
        M[a:b, a:b] = _spd(rng, b - a)
        W[a:b, a:b] = po.dense_factor(M[a:b, a:b])
    return M, W


DEEP_EPS = {STD: 5e-4, DIAG: 5e-4, FUNNEL: 5e-4, LOGISTIC: 4e-4, USER: 1.5e-4}   # trees of depth 13 (dims 1, 2: a tenth;
                                                                                 # a Symmetric M⁻¹: 0.7)
MODERATE_EPS = {STD: 0.3, DIAG: 0.3, FUNNEL: 0.2, LOGISTIC: 0.3, USER: 0.1}


class Inputs(NamedTuple):
    params: object          # the oracle's parameter block (None: the family has none)
    model_args: tuple
    q: np.ndarray           # [K, D]
    p: np.ndarray
    minv: np.ndarray        # diagonal M⁻¹ [K, D]
    Minv: object            # Symmetric M⁻¹: [K, D, D] (one per chain) or [D, D] (shared), None without a dense phase
    W: object               # the factor of a shared M⁻¹ (seeded into the oracle), else None
    eps_tree: np.ndarray    # ϵ of the leapfrog / tree checks, per metric kind
    eps_tree_dense: np.ndarray
    eps_warm: np.ndarray    # initial ϵ of the warm-up window


def case_inputs(po, case):
    rng = np.random.default_rng(zlib.crc32(str(case).encode()))
    D, K, fam = case.D, case.K, case.family
    params, model_args, scale = None, (), 1.0
    base = np.ones(D)
    if fam == DIAG:
        mu, s2 = rng.normal(size=D), rng.uniform(0.5, 2.0, D)
        params, model_args, base = np.concatenate([mu, 1.0 / s2]), (mu, s2), s2     # DiagNormal.params()
    elif fam == LOGISTIC:
        X = rng.normal(size=(LOGISTIC_N, D)) / np.sqrt(D)
        y = (rng.uniform(size=LOGISTIC_N) < 0.5).astype(float)
        params, model_args = po.logistic_params(X, y), (X, y)
    elif fam == USER:
        params, scale = ROSENBROCK_PARAMS, 0.3
    q = rng.normal(size=(K, D)) * scale
    p = rng.normal(size=(K, D))
    minv = base * rng.uniform(0.8, 1.25, (K, D))
    Minv = W = None
    if case.dense:
        if D <= DENSE_PER_CHAIN_MAX_DIM:
            Minv = np.stack([_spd(rng, D) for _ in range(K)])
        else:
            Minv, W = block_diagonal_metric(po, D)
    jitter = rng.uniform(0.9, 1.0, K)
    deep_eps = DEEP_EPS[fam] * jitter * (0.1 if D <= 2 else 1.0)
    mod_eps = MODERATE_EPS[fam] * jitter
    eps_tree = deep_eps if case.deep else mod_eps
    eps_tree_dense = 0.7 * deep_eps if case.deep and D <= DENSE_PER_CHAIN_MAX_DIM else mod_eps
    return Inputs(params, model_args, q, p, minv, Minv, W, eps_tree, eps_tree_dense, mod_eps)


def chain_metric(inp, k, dense):
    if not dense:
        return inp.minv[k]
    return inp.Minv if inp.Minv.ndim == 2 else inp.Minv[k]


@contextlib.contextmanager
def oracle_for(po, case):
    with po.user_model(ROSENBROCK) if case.family == USER else contextlib.nullcontext():
        yield


def seed_factor(po, inp, dense):
    """a shared M⁻¹: hand the oracle its factor before every call that takes it (another M⁻¹ may have replaced it)"""
    if dense and inp.W is not None:
        po.seed_dense_factor(inp.Minv, inp.W)


# ------------------------------------------------------------------ CPU: the oracle side of the cases
def test_block_diagonal_factor_is_the_blockwise_factor(po):
    for D in (16, 70, 257):
        M, W = block_diagonal_metric(po, D, seed=1)
        assert np.array_equal(po.dense_factor(M), W), D


def test_deep_cases_grow_trees_past_depth_12(po):
    """The deep cases' step sizes make chain 0's first tree deeper than 12 (so the slot pool's spill words are used); the
    oracle equals the device bit for bit, so this holds on the device too.  Dense deep cells above dim 256 use moderate
    step sizes (their trees are shallow)."""
    for case in CASES:
        if not case.deep:
            continue
        inp = case_inputs(po, case)
        T = case.layout()[0]
        with oracle_for(po, case):
            for dense in (False, True) if case.dense and case.D <= DENSE_PER_CHAIN_MAX_DIM else (False,):
                eps = (inp.eps_tree_dense if dense else inp.eps_tree)[0]
                o = po.sample_tree(case.family, inp.q[0], eps, SEED, 0, 0, minv=chain_metric(inp, 0, dense),
                                   params=inp.params, T=T, max_depth=case.max_depth)
                assert o["stats"]["depth"] > DEEP_ABOVE, (str(case), dense, o["stats"])


def test_oracle_warmup_takes_a_1x1_symmetric_metric_as_dense(po):
    """A Symmetric M⁻¹ handed to the oracle's mcmc_with_warmup is dense at every dim: at dim 1 it has the length of a
    diagonal one, and the kind comes from the caller, not from the length.  With no warm-up stage the first draw is
    sample_tree's from the same state.  (Taken as diagonal, W = √(1/m) and cholesky(inv(m)) differ in the last bit for
    some m: 3 of these 40.)"""
    M2 = block_diagonal_metric(po, 2, seed=2)[0]
    for M in [np.array([[m]]) for m in np.linspace(0.3, 3.0, 40)] + [M2]:
        D = M.shape[0]
        params = np.concatenate([np.zeros(D), np.full(D, 1.5)])
        q0 = np.linspace(-0.7, 0.4, D)
        o = po.mcmc_with_warmup(DIAG, D, 1, SEED, 1, stages=[], params=params, q0=q0, minv0=M, eps0=0.3)
        t = po.sample_tree(DIAG, q0, 0.3, SEED, 1, 0, minv=M, params=params)
        assert np.array_equal(o["posterior_matrix"][0], t["q"]) and np.array_equal(o["minv"], M), M
        _same_stats(o["tree_statistics"][0], t["stats"], M)


# ------------------------------------------------------------------ GPU
def _model(pkg, case, inp):
    fam, D = case.family, case.D
    if fam == STD:
        return pkg.StandardNormal(D)
    if fam == DIAG:
        return pkg.DiagNormal(*inp.model_args)
    if fam == FUNNEL:
        return pkg.Funnel(D)
    if fam == LOGISTIC:
        return pkg.LogisticRegression(*inp.model_args)
    return pkg.UserLogDensity(ROSENBROCK, D, params=ROSENBROCK_PARAMS, deep=True)


@contextlib.contextmanager
def _engine(pkg, ℓ, case):
    """the case's handle, released however the check ends"""
    eng = pkg.Engine(ℓ, chains=case.K, seed=SEED, algorithm=pkg.NUTS(max_depth=case.max_depth), threads_per_chain=case.T)
    try:
        T, EPL, _ = case.layout()
        assert eng.layout() == (T, EPL), (str(case), eng.layout())
        yield eng
    finally:
        eng.close()


def _assert_packing(pkg, ℓ, case):
    """layout() does not tell packed from one-chain-per-CTA logistic handles; a problem batch does: a packed handle refuses
    one whose chains_per_problem is not a multiple of 8 (dhmc_b200.cu:766-768)"""
    G = case.layout()[2]
    try:
        eng = pkg.Engine(pkg.ProblemBatch([ℓ, ℓ], chains_per_problem=4), chains=8, seed=SEED,
                         algorithm=pkg.NUTS(max_depth=case.max_depth), threads_per_chain=case.T)
    except pkg.ArgumentError as e:
        assert G == K_PACK and "packed chain groups" in str(e), (str(case), str(e))
    else:
        eng.close()
        assert G == 1, str(case)


def _set_metric(eng, inp, dense):
    if dense:
        eng.set_metric_dense(inp.Minv)
        assert eng.metric_is_dense()
    else:
        eng.set_metric(inp.minv)


def _same_stats(a, b, ctx):
    for f in INT_FIELDS + ("pi", "acceptance_rate"):
        assert a[f] == b[f], (ctx, f, a, b)


def _fine_grained(pkg, po, case, inp, ℓ, dense):
    fam, K, D, T = case.family, case.K, case.D, case.layout()[0]
    with _engine(pkg, ℓ, case) as eng:
        _set_metric(eng, inp, dense)
        # k_eval: random_position, then set_position
        eng.random_position()
        st = eng.get_state(("q", "lq", "grad"))
        for k in range(K):
            qr = po.random_position(SEED, k, D)
            lq, g = po.logdensity_and_gradient(fam, qr, inp.params, T)
            assert np.array_equal(st["q"][k], qr) and st["lq"][k] == lq and np.array_equal(st["grad"][k], g), (k, "random")
        eng.set_position(inp.q)
        st = eng.get_state(("q", "lq", "grad"))
        lq0 = []
        for k in range(K):
            lq, g = po.logdensity_and_gradient(fam, inp.q[k], inp.params, T)
            assert st["lq"][k] == lq and np.array_equal(st["grad"][k], g), (k, "set")
            lq0.append(lq)
        # k_search: the momentum is drawn from stream 1 (the search) at transition 0
        eng.find_initial_stepsize()
        eps = eng.get_state(("eps",))["eps"]
        for k in range(K):
            seed_factor(po, inp, dense)
            m = chain_metric(inp, k, dense)
            p0 = po.rand_p(SEED, k, 1, 0, m)
            assert eps[k] == po.find_initial_stepsize(fam, inp.q[k], p0, minv=m, params=inp.params, T=T), (k, "search")
        # k_phase
        e = inp.eps_tree_dense if dense else inp.eps_tree
        eng.set_stepsize(e)
        eng.set_momentum(inp.p)
        H = eng.phase_logdensity()
        for k in range(K):
            seed_factor(po, inp, dense)
            assert H[k] == po.phase_logdensity(chain_metric(inp, k, dense), lq0[k], inp.p[k], T), (k, "phase")
        # k_leapfrog: two steps forwards, one backwards
        q, p = inp.q, inp.p
        for n, sign in ((2, 1), (1, -1)):
            eng.leapfrog(n, sign)
            st = eng.get_state(("q", "p", "grad", "lq"))
            for k in range(K):
                seed_factor(po, inp, dense)
                qo, po_, go, lqo = po.leapfrog(fam, q[k], p[k], sign * e[k], minv=chain_metric(inp, k, dense),
                                               params=inp.params, T=T, n_steps=n)
                assert (np.array_equal(st["q"][k], qo) and np.array_equal(st["p"][k], po_) and np.array_equal(st["grad"][k], go)
                        and st["lq"][k] == lqo), (k, n, sign)
            q, p = st["q"], st["p"]
        # k_nuts: two transitions from the set positions
        eng.set_position(inp.q)
        t0 = eng.transition_count
        q = inp.q
        depths = []
        for t in range(2):
            stats = eng.sample_tree()
            st = eng.get_state(("q", "lq", "grad"))
            for k in range(K):
                seed_factor(po, inp, dense)
                o = po.sample_tree(fam, q[k], e[k], SEED, k, t0 + t, minv=chain_metric(inp, k, dense), params=inp.params, T=T,
                                   max_depth=case.max_depth)
                _same_stats(o["stats"], stats[k], (k, t))
                assert np.array_equal(st["q"][k], o["q"]) and np.array_equal(st["grad"][k], o["g"]) and st["lq"][k] == o["lq"], (k, t)
                depths.append(int(stats[k]["depth"]))
            q = st["q"]
        if case.deep and (not dense or D <= DENSE_PER_CHAIN_MAX_DIM):
            assert max(depths) > DEEP_ABOVE, depths          # the slot pool's spill words were used


def _window_then_draws(pkg, po, case, inp, ℓ, dense):
    """a fresh handle: one TuningNUTS window with dual averaging, then draws — bit-equal to the oracle's chain with the
    same initial position, metric and step size"""
    fam, K, D, T = case.family, case.K, case.D, case.layout()[0]
    if not dense:
        M, code = pkg.Diagonal, po.METRIC_DIAGONAL
    elif D <= DENSE_WINDOW_MAX_DIM:
        M, code = pkg.Symmetric, po.METRIC_SYMMETRIC
    else:                        # the window keeps the given M⁻¹ (the oracle's factorisation of a new one is O(D³))
        M, code = None, po.METRIC_NOTHING
    with _engine(pkg, ℓ, case) as eng:
        _set_metric(eng, inp, dense)
        eng.set_position(inp.q)
        eng.set_stepsize(inp.eps_warm)
        w = eng.warmup_stage(pkg.TuningNUTS(N_WINDOW, pkg.DualAveraging(), M), keep=True)
        out = eng.mcmc(N_DRAWS)
        ck = eng.checkpoint()
    assert ck["dense"] == dense
    for k in range(K):
        seed_factor(po, inp, dense)
        o = po.mcmc_with_warmup(fam, D, N_DRAWS, SEED, k, stages=[(po.STAGE_TUNING, N_WINDOW, code, 1)], params=inp.params,
                                T=T, max_depth=case.max_depth, q0=inp.q[k], minv0=chain_metric(inp, k, dense),
                                eps0=inp.eps_warm[k], welford=True, keep_warmup=True)
        for f in INT_FIELDS:
            assert np.array_equal(w["tree_statistics"][k][f], o["warmup_stats"][f]), (k, f)
        assert np.array_equal(w["posterior_matrix"][k], o["warmup_posterior"]) and np.array_equal(w["ϵs"][k], o["warmup_eps"]), k
        for n in range(N_DRAWS):
            _same_stats(o["tree_statistics"][n], out["tree_statistics"][k, n], (k, n))
        assert np.array_equal(out["posterior_matrix"][k], o["posterior_matrix"]), k
        assert np.array_equal(out["logdensities"][k], o["logdensities"]), k
        assert ck["eps"][k] == o["eps"] and np.array_equal(ck["minv"][k], o["minv"]), k


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=str)
def test_case_matches_oracle(pkg, po, case):
    inp = case_inputs(po, case)
    ℓ = _model(pkg, case, inp)
    if case.family == LOGISTIC:
        _assert_packing(pkg, ℓ, case)
    with oracle_for(po, case):
        for dense in (False, True) if case.dense else (False,):
            _fine_grained(pkg, po, case, inp, ℓ, dense)
            if not dense or case.D <= DRAWS_MAX_DIM_DENSE:
                _window_then_draws(pkg, po, case, inp, ℓ, dense)
