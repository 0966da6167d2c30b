"""Host-side mirror of the DynamicHMC.jl sampler API over the C ABI.

Names, argument meaning and error behaviour follow the reference
(src/mcmc.jl, src/NUTS.jl, src/stepsize.jl, src/hamiltonian.jl); the numeric
work happens in libdhmc_b200.so for `chains` independent chains at once.  The
reference's toolchain (Julia) is absent from this image, so this Python layer
plays the role of the Julia shim shown in INTEGRATION.md / julia/B200HMC.jl.

    results = mcmc_with_warmup(seed, ℓ, N; chains=K, initialization=..., warmup_stages=...,
                               algorithm=NUTS())
returns a `Results` whose `[k]` is the reference's NamedTuple for chain k
(posterior_matrix [D, N], tree_statistics [N], logdensities [N], κ, ϵ).
"""
import ctypes as C
import hashlib
import math
import os
import subprocess
import unicodedata
from dataclasses import dataclass, field
from typing import Optional, Sequence

import numpy as np

from . import _lib as L


# ------------------------------------------------------------------ errors
class DynamicHMCError(Exception):
    """src/utilities.jl:17-27 — numerical failure; `debug_information` carries chain ids."""

    def __init__(self, message, **debug_information):
        super().__init__(message)
        self.message = message
        self.debug_information = debug_information


class ArgumentError(ValueError):
    """Julia's ArgumentError raised by @argcheck in the reference.  A per-chain one (leapfrog from a non-finite log
    density, hamiltonian.jl:276) carries the chain status words in `debug_information`, as DynamicHMCError does."""

    def __init__(self, message, **debug_information):
        super().__init__(message)
        self.debug_information = debug_information


def _argcheck(cond, msg):
    if not cond:
        raise ArgumentError(msg)


# ------------------------------------------------------------------ log densities
# DeviceLogDensity types: the LogDensityProblems objects whose ℓ, ∇ℓ exist as
# device code (hamiltonian.jl:204 is the only call site).  Each also evaluates on
# the CPU through numpy so that the same object can be handed to other samplers.
class DeviceLogDensity:
    family = -1

    def dimension(self):
        return self.D

    def capabilities(self):
        return 1  # LogDensityOrder{1}

    def params(self):
        return np.zeros(0)


@dataclass
class StandardNormal(DeviceLogDensity):
    D: int
    family = L.FAMILY_STD_NORMAL

    def logdensity_and_gradient(self, q):
        q = np.asarray(q, float)
        return -0.5 * float(q @ q), -q


@dataclass
class DiagNormal(DeviceLogDensity):
    """N(μ, Diagonal(σ²))"""
    mu: np.ndarray
    sigma2: np.ndarray
    family = L.FAMILY_DIAG_NORMAL

    def __post_init__(self):
        self.mu = np.ascontiguousarray(self.mu, float)
        self.sigma2 = np.ascontiguousarray(self.sigma2, float)
        _argcheck(self.mu.shape == self.sigma2.shape and self.mu.ndim == 1, "mu, sigma2: same length")
        self.D = self.mu.size

    def params(self):
        return np.concatenate([self.mu, 1.0 / self.sigma2])

    def logdensity_and_gradient(self, q):
        d = np.asarray(q, float) - self.mu
        t = d / self.sigma2
        return -0.5 * float(d @ t), -t


@dataclass
class Funnel(DeviceLogDensity):
    """Neal's funnel θ = (v, x₁…x_{D-1}) (SURVEY.md §8d C3)."""
    D: int = 10
    family = L.FAMILY_FUNNEL

    def logdensity_and_gradient(self, q):
        q = np.asarray(q, float)
        v, x = q[0], q[1:]
        S = float(x @ x)
        ev = math.exp(-v)
        g = np.empty_like(q)
        g[0] = -v / 9 + 0.5 * ev * S - 0.5 * (self.D - 1)
        g[1:] = -ev * x
        return -v * v / 18 - 0.5 * ev * S - 0.5 * (self.D - 1) * v, g


@dataclass
class LogisticRegression(DeviceLogDensity):
    """ℓ(β) = Σ[yᵢ xᵢᵀβ − log1pexp(xᵢᵀβ)] − ½‖β‖²  (SURVEY.md §8d C4); X is [N, p], y ∈ {0,1}ᴺ."""
    X: np.ndarray
    y: np.ndarray
    family = L.FAMILY_LOGISTIC

    def __post_init__(self):
        self.X = np.ascontiguousarray(self.X, float)
        self.y = np.ascontiguousarray(self.y, float)
        _argcheck(self.X.ndim == 2 and self.y.shape == (self.X.shape[0],), "X: [N, p], y: [N]")
        _argcheck(bool(np.all((self.y >= 0.0) & (self.y <= 1.0))), "0 ≤ y ≤ 1 (Bernoulli responses)")
        self.D = self.X.shape[1]

    def params(self):
        return np.concatenate([[float(self.X.shape[0])], self.X.ravel(), self.y])

    def logdensity_and_gradient(self, q):
        q = np.asarray(q, float)
        eta = self.X @ q
        ll = self.y * eta - np.logaddexp(0.0, eta)
        r = self.y - 1.0 / (1.0 + np.exp(-eta))
        return float(ll.sum() - 0.5 * q @ q), self.X.T @ r - q

    @staticmethod
    def synthetic(N=10000, p=256, seed=7):
        """The C4 data set: Xᵢⱼ ~ N(0,1)/√p, β* ~ N(0,I), yᵢ ~ Bernoulli(σ(xᵢᵀβ*))."""
        rng = np.random.default_rng(seed)
        X = rng.normal(size=(N, p)) / np.sqrt(p)
        beta = rng.normal(size=p)
        y = (rng.uniform(size=N) < 1.0 / (1.0 + np.exp(-(X @ beta)))).astype(float)
        return LogisticRegression(X, y), beta


# ------------------------------------------------------------------ user models
# The reference accepts ANY LogDensityProblems object; its only use of it is logdensity_and_gradient at hamiltonian.jl:204.
# On the device the counterpart is a header of scalar formulas (include/dhmc_models.h, "the model header contract";
# examples in include/models/) that is compiled — nvcc, sm_90a, same flags as the shipped families — into its own copy of
# the library, where it is family DHMC_FAMILY_USER.
_CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc")


def compile_user_model(header, out_dir=None, force=False, jobs=2, deep=False):
    """Build (or reuse) the library that carries the model in `header` as family FAMILY_USER; returns its path.
    `deep=True` also compiles the kernels for NUTS(max_depth > 12) (up to the reference's limit 32; twice the build time).

    The build is keyed by the header's content and the library sources' modification times, lives under
    csrc/user_models/<name>-<hash>/ (in-tree, so that it travels with the package) unless `out_dir` is given, and needs nvcc
    plus the object files of the stock library (`__graft_entry__.build()`); it takes a few minutes of CPU time."""
    header = os.path.abspath(header)
    if not os.path.exists(header):
        raise ArgumentError(f"user model header {header} does not exist")
    name = os.path.splitext(os.path.basename(header))[0]
    srcs = [os.path.join(_CSRC, f) for f in ("family_tu.cu", "kernels.cuh", "device_backend.cuh", "nuts_machine.cuh",
                                            "dhmc_b200.cu")]
    srcs += [os.path.join(_CSRC, "..", "..", "include", f) for f in ("dhmc.h", "dhmc_math.h", "dhmc_models.h", "dhmc_tables.h")]
    hsh = hashlib.sha256(open(header, "rb").read())
    for f in srcs:
        hsh.update(open(f, "rb").read())
    tag = f"{name}-{hsh.hexdigest()[:12]}" + ("-deep" if deep else "")
    out_dir = os.path.abspath(out_dir or os.path.join(_CSRC, "user_models", tag))
    so = os.path.join(out_dir, f"libdhmc_user_{name}.so")
    if force or not os.path.exists(so):
        import fcntl
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, ".lock"), "w") as lock:        # several ranks / test workers may ask for the same model
            fcntl.flock(lock, fcntl.LOCK_EX)
            if force or not os.path.exists(so):
                tmp = so + ".tmp%d" % os.getpid()                       # linked under a private name, published by rename
                cmd = ["make", "-C", _CSRC, f"-j{jobs}", "user", f"USER_HEADER={header}", f"USER_LIB={tmp}",
                       f"USER_BUILD={os.path.join(out_dir, 'build')}", "USER_PARTS=" + ("0 3" if deep else "0")]
                r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
                if r.returncode != 0 or not os.path.exists(tmp):
                    raise RuntimeError(f"user model build failed ({' '.join(cmd)}):\n{r.stdout[-4000:]}")
                os.replace(tmp, so)
                for f in os.listdir(os.path.join(out_dir, "build")):   # keep the ptxas logs, drop the objects (they are in the .so)
                    if f.endswith(".o"):
                        os.remove(os.path.join(out_dir, "build", f))
    return so


class UserLogDensity(DeviceLogDensity):
    """ℓ given as a model header (the device-side LogDensityProblems object).  `params` is the block of doubles the
    header's formulas receive; `cpu` optionally is a callable q ↦ (ℓ(q), ∇ℓ(q)) so that the object also answers
    logdensity_and_gradient on the host (like the shipped families' numpy forms).  `library` may name a prebuilt library;
    `deep=True` builds the kernels for NUTS(max_depth > 12) as well."""
    family = L.FAMILY_USER

    def __init__(self, header, D, params=(), cpu=None, library=None, deep=False):
        self.header, self.D = os.path.abspath(header), int(D)
        self._params = np.ascontiguousarray(params, float).ravel()
        self._cpu = cpu
        self.library_path = library or compile_user_model(self.header, deep=deep)

    @classmethod
    def from_source(cls, source, name, D, params=(), **kw):
        """The model given as the TEXT of its header (e.g. generated by the caller): written to
        csrc/user_models/src/<name>-<hash>.h and handled like a header file."""
        _argcheck(name.isidentifier(), "name: a valid identifier (it becomes a file name)")
        src_dir = os.path.join(_CSRC, "user_models", "src")
        os.makedirs(src_dir, exist_ok=True)
        path = os.path.join(src_dir, f"{name}-{hashlib.sha256(source.encode()).hexdigest()[:12]}.h")
        if not os.path.exists(path):
            tmp = path + ".tmp%d" % os.getpid()
            with open(tmp, "w") as f:
                f.write(source)
            os.replace(tmp, path)
        return cls(path, D, params=params, **kw)

    def params(self):
        return self._params

    def model_name(self):
        buf = C.create_string_buffer(128)
        rc = L.lib(self.library_path).dhmc_user_family_name(buf, C.c_size_t(128))
        _argcheck(rc == L.DHMC_OK, f"{self.library_path} carries no user model")
        return buf.value.decode()

    def logdensity_and_gradient(self, q):
        if self._cpu is None:
            raise NotImplementedError("this UserLogDensity was created without a host-side `cpu` callable")
        return self._cpu(np.asarray(q, float))


# ------------------------------------------------------------------ problem batches
class ProblemBatch:
    """Many posteriors on one handle (dhmc_set_problems): `problems` are P log densities of one family and dimension whose
    parameter blocks have equal length (logistic regression: the same N), each sampled by `chains_per_problem` chains.
    Global chain g samples problem g // chains_per_problem, and those chains are bit-identical to a handle that holds
    problem p alone with chain_offset = p·chains_per_problem — for simulation-based calibration, bootstrap or
    cross-validation refits and one fit per unit, which need many posteriors and only a few chains each.  Validated on
    the host; hand it to Engine / mcmc_with_warmup in place of ℓ."""

    def __init__(self, problems, chains_per_problem):
        blocks = self._check_problems(problems, chains_per_problem)
        if self.family == L.FAMILY_LOGISTIC:
            _argcheck(all(b[0] == blocks[0][0] for b in blocks), "every logistic problem of a batch has the same N")
        _argcheck(all(b.size == blocks[0].size for b in blocks), "every problem of a batch has a parameter block of the same length")
        _argcheck(blocks[0].size >= 1, "the problems have empty parameter blocks")
        self.block_size = blocks[0].size
        self._params = np.concatenate(blocks)

    def _check_problems(self, problems, chains_per_problem):
        """the checks every batch shares (family, dimension, library, chain count); returns the parameter blocks"""
        problems = list(problems)
        _argcheck(len(problems) >= 1, "a batch needs at least one problem")
        _argcheck(all(isinstance(x, DeviceLogDensity) for x in problems), "problems: DeviceLogDensity objects")
        self.chains_per_problem = int(chains_per_problem)
        _argcheck(self.chains_per_problem >= 1, "chains_per_problem ≥ 1")
        first = problems[0]
        self.family, self.D = first.family, int(first.dimension())
        _argcheck(all(x.family == self.family for x in problems), "every problem of a batch has the same family")
        _argcheck(all(int(x.dimension()) == self.D for x in problems), "every problem of a batch has the same dimension")
        _argcheck(self.family not in (L.FAMILY_STD_NORMAL, L.FAMILY_FUNNEL),
                  "this family has no parameters: a batch of it would be one problem")
        self.library_path = getattr(first, "library_path", None)
        _argcheck(all(getattr(x, "library_path", None) == self.library_path for x in problems),
                  "every problem of a batch lives in the same user-model library")
        self.problems = problems
        return [np.ascontiguousarray(x.params(), float).ravel() for x in problems]

    @property
    def n_problems(self):
        return len(self.problems)

    @property
    def chains(self):
        """chains of the whole batch: n_problems · chains_per_problem"""
        return self.n_problems * self.chains_per_problem

    def dimension(self):
        return self.D

    def capabilities(self):
        return min(x.capabilities() for x in self.problems)

    def params(self):
        """the P blocks back to back, [P · block_size]"""
        return self._params

    def problem_chains(self, p, chain_offset=0, chains=None):
        """local chain range [lo, hi) of problem p on a handle with `chains` chains from global id `chain_offset`"""
        chains = self.chains - chain_offset if chains is None else chains
        K = self.chains_per_problem
        lo, hi = max(p * K - chain_offset, 0), min((p + 1) * K - chain_offset, chains)
        return lo, max(lo, hi)


class RaggedProblemBatch(ProblemBatch):
    """A ProblemBatch whose parameter blocks may differ in length (dhmc_set_problems_ragged): logistic regressions with
    their own number of observations each — one fit per hospital, school or customer, or the folds of a k-fold split.
    Each problem's data take device memory of their own size, and a packed CTA streams only its problem's rows, where
    padding every problem to the largest N would cost max N / mean N of the useful work.  A user model's formulas do not
    receive the length of their block: a model that needs it stores it in the block.  Problems of equal length are
    accepted too and sample exactly as the ProblemBatch of the same problems.  Problem p's block is
    params()[block_offsets[p]:block_offsets[p + 1]] (block_offsets: [P + 1], size_t)."""

    def __init__(self, problems, chains_per_problem):
        blocks = self._check_problems(problems, chains_per_problem)
        _argcheck(all(b.size >= 1 for b in blocks), "every problem of a batch needs a non-empty parameter block")
        self.block_size = None
        self.block_offsets = np.zeros(len(blocks) + 1, dtype=np.dtype(C.c_size_t))
        np.cumsum([b.size for b in blocks], out=self.block_offsets[1:])
        self._params = np.concatenate(blocks)


# ------------------------------------------------------------------ algorithm structs
@dataclass
class NUTS:
    """src/NUTS.jl:178-195"""
    max_depth: int = 10
    min_Δ: float = -1000.0

    def __post_init__(self):
        _argcheck(0 < self.max_depth <= 32, "0 < max_depth ≤ MAX_DIRECTIONS_DEPTH")
        _argcheck(self.min_Δ < 0, "min_Δ < 0")


@dataclass
class DualAveraging:
    """src/stepsize.jl:98-118"""
    δ: float = 0.8
    γ: float = 0.05
    κ: float = 0.75
    t0: int = 10

    def __post_init__(self):
        _argcheck(0 < self.δ < 1, "0 < δ < 1")
        _argcheck(self.γ > 0, "γ > 0")
        _argcheck(0.5 < self.κ <= 1, "0.5 < κ ≤ 1")
        _argcheck(self.t0 >= 0, "t₀ ≥ 0")


class FixedStepsize:
    """src/stepsize.jl:181-189"""


@dataclass
class InitialStepsizeSearch:
    """src/stepsize.jl:23-36"""
    initial_ϵ: float = 0.1
    log_threshold: float = math.log(0.8)
    maxiter_crossing: int = 400

    def __post_init__(self):
        _argcheck(math.isfinite(self.log_threshold) and self.log_threshold < 0, "isfinite(log_threshold) && log_threshold < 0")
        _argcheck(math.isfinite(self.initial_ϵ) and 0 < self.initial_ϵ, "isfinite(initial_ϵ) && 0 < initial_ϵ")
        _argcheck(self.maxiter_crossing >= 50, "maxiter_crossing ≥ 50")


Diagonal = "Diagonal"
Symmetric = "Symmetric"
SymmetricPooled = "SymmetricPooled"      # NOT in the reference: one dense metric per group of 8 chains (dhmc.h, DHMC_METRIC_SYMMETRIC_POOLED)


@dataclass
class TuningNUTS:
    """src/mcmc.jl:178-195 — M ∈ {None, Diagonal, Symmetric}"""
    N: int
    stepsize_adaptation: object = field(default_factory=DualAveraging)
    M: Optional[str] = None
    λ: Optional[float] = None

    def __post_init__(self):
        _argcheck(self.N >= 20, "N ≥ 20")
        if self.λ is None:
            self.λ = 5.0 / self.N
        _argcheck(self.λ >= 0, "λ ≥ 0")
        _argcheck(self.M in (None, Diagonal, Symmetric, SymmetricPooled), "M <: Union{Nothing,Diagonal,Symmetric}")


def default_warmup_stages(stepsize_search=InitialStepsizeSearch(), M=Diagonal,
                          stepsize_adaptation=DualAveraging(), init_steps=75, middle_steps=25,
                          doubling_stages=5, terminating_steps=50):
    """src/mcmc.jl:415-425"""
    return (stepsize_search, TuningNUTS(init_steps, stepsize_adaptation),
            *(TuningNUTS(middle_steps * 2 ** i, stepsize_adaptation, M) for i in range(doubling_stages)),
            TuningNUTS(terminating_steps, stepsize_adaptation))


def fixed_stepsize_warmup_stages(M=Diagonal, middle_steps=25, doubling_stages=5):
    """src/mcmc.jl:436-440"""
    return tuple(TuningNUTS(middle_steps * 2 ** i, FixedStepsize(), M) for i in range(doubling_stages))


@dataclass
class GaussianKineticEnergy:
    """src/hamiltonian.jl:56-87.  Diagonal M⁻¹ (:80): `minv` is [D] (all chains) or one row
    per chain.  Symmetric M⁻¹ (:73, `dense=True`): `minv` is [D, D] (all chains) or [K, D, D]."""
    minv: np.ndarray
    dense: bool = False

    @staticmethod
    def identity(N, m=1.0):
        return GaussianKineticEnergy(np.full(N, float(m)))

    @staticmethod
    def symmetric(Minv):
        return GaussianKineticEnergy(np.ascontiguousarray(Minv, float), dense=True)


# ------------------------------------------------------------------ engine
class Engine:
    """Owns a dhmc_handle: K chains of one problem (or of a ProblemBatch) on one GPU."""

    def __init__(self, ℓ: DeviceLogDensity, chains: int, seed: int = 0, algorithm: NUTS = None,
                 device: int = 0, chain_offset: int = 0, threads_per_chain: int = 0,
                 ctas_per_sm: int = 0):
        algorithm = algorithm or NUTS()
        _argcheck(ℓ.capabilities() >= 1, "capabilities(ℓ) ≥ LogDensityOrder(1)")   # hamiltonian.jl:146
        self.ℓ, self.K, self.D, self.algorithm = ℓ, int(chains), int(ℓ.dimension()), algorithm
        self._lib = L.lib(getattr(ℓ, "library_path", None))     # a user model lives in its own build of the library
        cfg = L.Config(device=device, family=ℓ.family, dim=self.D, n_chains=self.K,
                       chain_offset=chain_offset, seed=seed, max_depth=algorithm.max_depth,
                       threads_per_chain=threads_per_chain, min_delta=algorithm.min_Δ,
                       ctas_per_sm=ctas_per_sm, reserved=0)
        h = C.c_void_p()
        rc = self._lib.dhmc_create(C.byref(cfg), C.byref(h))
        if rc != L.DHMC_OK:
            msg = self._lib.dhmc_last_error(None).decode()
            if rc == L.DHMC_EARG:
                raise ArgumentError(msg)
            raise RuntimeError(f"dhmc_create failed [{rc}]: {msg}")
        self._h = h
        self._set_problem(ℓ)

    def _set_problem(self, ℓ):
        """dhmc_set_problem, or dhmc_set_problems(_ragged) for a (Ragged)ProblemBatch.  On an error the handle keeps its previous problem."""
        if self.ℓ is not ℓ:                              # replacing the problem of an existing handle
            _argcheck(ℓ.family == self.ℓ.family and int(ℓ.dimension()) == self.D, "same family and dimension as the handle")
            _argcheck(getattr(ℓ, "library_path", None) == getattr(self.ℓ, "library_path", None),
                      "a user model of the handle's own library")
        pr = np.ascontiguousarray(ℓ.params(), float)
        if isinstance(ℓ, RaggedProblemBatch):
            self._ck(self._lib.dhmc_set_problems_ragged(self._h, L.ptr(pr), L.ptr(ℓ.block_offsets), C.c_int64(ℓ.n_problems),
                                                        C.c_int64(ℓ.chains_per_problem)))
        elif isinstance(ℓ, ProblemBatch):
            self._ck(self._lib.dhmc_set_problems(self._h, L.ptr(pr), C.c_size_t(ℓ.block_size), C.c_int64(ℓ.n_problems),
                                                 C.c_int64(ℓ.chains_per_problem)))
        else:
            self._ck(self._lib.dhmc_set_problem(self._h, L.ptr(pr) if pr.size else None, C.c_size_t(pr.size)))
        self.ℓ = ℓ

    # -- plumbing
    def _ck(self, rc):
        if rc == L.DHMC_OK:
            return
        msg = self._lib.dhmc_last_error(self._h).decode()
        if rc == L.DHMC_EARG:
            raise ArgumentError(msg)
        if rc == L.DHMC_ENUMERIC:
            st = self.chain_status()
            # leapfrog's @argcheck isfinite(Q.ℓq) (hamiltonian.jl:276) is an ArgumentError in the reference; a chain whose
            # strict initial evaluation failed, or that met a non-finite position first, has failed with DynamicHMCError
            # before it got there
            halted = (st & L.DHMC_CHAIN_LEAPFROG_NONFINITE) != 0
            if np.any(halted & ((st & (L.DHMC_CHAIN_BAD_INITIAL | L.DHMC_CHAIN_NONFINITE_Q)) == 0)):
                raise ArgumentError(msg, chain_status=st)
            raise DynamicHMCError(msg, chain_status=st)
        raise RuntimeError(f"libdhmc_b200 error [{rc}]: {msg}")

    def close(self):
        if getattr(self, "_h", None):
            self.host_free_all()
            self._lib.dhmc_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def layout(self):
        t, e = C.c_int32(), C.c_int32()
        self._ck(self._lib.dhmc_get_layout(self._h, C.byref(t), C.byref(e)))
        return t.value, e.value

    def _kd(self, a, name):
        a = np.ascontiguousarray(a, float)
        _argcheck(a.shape == (self.K, self.D), f"{name}: expected [D, K] column-major = numpy ({self.K}, {self.D})")
        return a

    # -- state
    def set_position(self, q):
        q = self._kd(q, "q")
        self._ck(self._lib.dhmc_set_position(self._h, L.ptr(q)))

    def random_position(self):
        self._ck(self._lib.dhmc_random_position(self._h))

    def set_metric(self, minv=None):
        if minv is None:
            self._ck(self._lib.dhmc_set_metric(self._h, None, 0))
            return
        minv = np.ascontiguousarray(minv, float)
        if minv.ndim == 1:
            _argcheck(minv.size == self.D, "dimension(ℓ) == size(κ, 1)")            # hamiltonian.jl:147
            self._ck(self._lib.dhmc_set_metric(self._h, L.ptr(minv), 1))
        else:
            self._ck(self._lib.dhmc_set_metric(self._h, L.ptr(self._kd(minv, "minv")), 0))

    def set_metric_dense(self, Minv):
        """κ = GaussianKineticEnergy(Symmetric(M⁻¹)) — hamiltonian.jl:73."""
        M = np.ascontiguousarray(Minv, float)
        if M.ndim == 2:
            _argcheck(M.shape == (self.D, self.D), "dimension(ℓ) == size(κ, 1)")
            self._ck(self._lib.dhmc_set_metric_dense(self._h, L.ptr(M), 1))
        else:
            _argcheck(M.shape == (self.K, self.D, self.D), "M⁻¹: [D, D] or one matrix per chain")
            self._ck(self._lib.dhmc_set_metric_dense(self._h, L.ptr(M), 0))

    def set_kinetic_energy(self, κ: "GaussianKineticEnergy"):
        if κ.dense:
            self.set_metric_dense(κ.minv)
        else:
            self.set_metric(κ.minv)

    def metric_is_dense(self):
        v = C.c_int32()
        self._ck(self._lib.dhmc_metric_is_dense(self._h, C.byref(v)))
        return bool(v.value)

    def get_metric_dense(self):
        out = np.empty((self.K, self.D, self.D))
        self._ck(self._lib.dhmc_get_metric_dense(self._h, L.ptr(out)))
        return out

    def set_stepsize(self, eps):
        e = np.ascontiguousarray(eps, float).reshape(-1)
        if e.size == 1:
            self._ck(self._lib.dhmc_set_stepsize(self._h, L.ptr(e), 1))
        else:
            _argcheck(e.size == self.K, "one ϵ per chain")
            self._ck(self._lib.dhmc_set_stepsize(self._h, L.ptr(e), 0))

    def set_momentum(self, p):
        self._ck(self._lib.dhmc_set_momentum(self._h, L.ptr(self._kd(p, "p"))))

    def get_state(self, fields=("q", "lq", "grad", "minv", "eps", "p")):
        K, D = self.K, self.D
        out = {}
        shapes = dict(q=(K, D), lq=(K,), grad=(K, D), minv=(K, D), eps=(K,), p=(K, D))
        for f in fields:
            out[f] = np.empty(shapes[f])
        args = [L.ptr(out[f]) if f in out else None for f in ("q", "lq", "grad", "minv", "eps", "p")]
        self._ck(self._lib.dhmc_get_state(self._h, *args))
        return out

    def chain_status(self):
        st = np.zeros(self.K, dtype=np.int32)
        self._lib.dhmc_chain_status(self._h, L.ptr(st))
        return st

    @property
    def transition_count(self):
        t = C.c_uint32()
        self._ck(self._lib.dhmc_get_transition_count(self._h, C.byref(t)))
        return t.value

    @transition_count.setter
    def transition_count(self, t):
        self._ck(self._lib.dhmc_set_transition_count(self._h, C.c_uint32(t)))

    # -- checkpoint / resume: WarmupState(Q, κ, ϵ) (mcmc.jl:72-79) + the RNG counter is everything a fresh handle needs
    def checkpoint(self):
        """dict(q [K, D], minv ([K, D] diagonal or [K, D, D] Symmetric), dense, eps [K], transition_count, K, D)."""
        st = self.get_state(("q", "minv", "eps"))
        dense = self.metric_is_dense()
        return dict(q=st["q"], eps=st["eps"], dense=bool(dense), minv=self.get_metric_dense() if dense else st["minv"],
                    transition_count=int(self.transition_count), K=self.K, D=self.D)

    def restore(self, ck):
        """Continue the chains of `ck` (from `checkpoint()` / `load_checkpoint`) on this handle: same seed and chain_offset
        give the same draws as the handle that was checkpointed (the Philox counter is (chain, transition, …))."""
        _argcheck(int(ck["K"]) == self.K and int(ck["D"]) == self.D, "checkpoint of a different shape (chains, dimension)")
        if bool(ck["dense"]):
            self.set_metric_dense(ck["minv"])
        else:
            self.set_metric(ck["minv"])
        self.set_position(ck["q"])
        self.set_stepsize(ck["eps"])
        self.transition_count = int(ck["transition_count"])

    def save_checkpoint(self, path):
        np.savez(path, **self.checkpoint())

    def load_checkpoint(self, path):
        with np.load(path) as f:
            self.restore({k: f[k] for k in f.files})

    # -- fine-grained path
    def leapfrog(self, n_steps=1, sign=1):
        self._ck(self._lib.dhmc_leapfrog(self._h, C.c_int32(n_steps), C.c_int32(sign)))

    def phase_logdensity(self):
        out = np.empty(self.K)
        self._ck(self._lib.dhmc_phase_logdensity(self._h, L.ptr(out)))
        return out

    def sample_tree(self, p=None, directions=None):
        stats = np.zeros(self.K, dtype=L.tree_stats_dtype)
        pp = None if p is None else self._kd(p, "p")
        dd = None if directions is None else np.ascontiguousarray(directions, dtype=np.uint32)
        self._ck(self._lib.dhmc_sample_tree(self._h, L.ptr(pp), L.ptr(dd), L.ptr(stats)))
        return stats

    # -- coarse path
    def find_initial_stepsize(self, search: InitialStepsizeSearch = None):
        s = search or InitialStepsizeSearch()
        self._ck(self._lib.dhmc_find_initial_stepsize(self._h, C.c_double(s.initial_ϵ),
                                                      C.c_double(s.log_threshold),
                                                      C.c_int32(s.maxiter_crossing)))

    def warmup_stage(self, stage: TuningNUTS, keep=False):
        K, D, N = self.K, self.D, stage.N
        post = np.empty((K, N, D)) if keep else None
        stats = np.zeros((K, N), dtype=L.tree_stats_dtype) if keep else None
        eps = np.empty((K, N)) if keep else None
        ld = np.empty((K, N)) if keep else None
        da = None
        if isinstance(stage.stepsize_adaptation, DualAveraging):
            a = stage.stepsize_adaptation
            da = C.byref(L.DualAveragingC(a.δ, a.γ, a.κ, a.t0, 0))
        metric = {Diagonal: L.METRIC_DIAGONAL, Symmetric: L.METRIC_SYMMETRIC,
                  SymmetricPooled: L.METRIC_SYMMETRIC_POOLED}.get(stage.M, L.METRIC_NOTHING)
        self._ck(self._lib.dhmc_warmup_stage(self._h, C.c_int32(N), C.c_int32(metric), da,
                                             C.c_double(stage.λ), L.ptr(post), L.ptr(stats),
                                             L.ptr(eps), L.ptr(ld)))
        if keep:
            return {"posterior_matrix": post, "tree_statistics": stats, "ϵs": eps, "eps_used": eps,
                    "logdensities": ld}
        return None

    def mcmc(self, N, keep_draws=True):
        K, D = self.K, self.D
        post = np.empty((K, N, D)) if keep_draws else None
        stats = np.zeros((K, N), dtype=L.tree_stats_dtype)
        ld = np.empty((K, N))
        self._ck(self._lib.dhmc_mcmc(self._h, C.c_int32(N), L.ptr(post), L.ptr(stats), L.ptr(ld)))
        return dict(posterior_matrix=post, tree_statistics=stats, logdensities=ld)

    def mcmc_from(self, q, N, out=None):
        """mcmc starting from host positions q ([K, D]); upload, evaluate_ℓ, sampling and
        download are pipelined by chain chunks.  `out` may hold preallocated (pinned) arrays."""
        K, D = self.K, self.D
        q = self._kd(q, "q")
        out = out or {}
        post = out.get("posterior_matrix", None)
        post = np.empty((K, N, D)) if post is None else post
        stats = out.get("tree_statistics", None)
        stats = np.zeros((K, N), dtype=L.tree_stats_dtype) if stats is None else stats
        ld = out.get("logdensities", None)
        ld = np.empty((K, N)) if ld is None else ld
        self._ck(self._lib.dhmc_mcmc_from(self._h, L.ptr(q), C.c_int32(N), L.ptr(post), L.ptr(stats), L.ptr(ld)))
        return dict(posterior_matrix=post, tree_statistics=stats, logdensities=ld)

    def mcmc_thinned(self, N, thin=1, q=None, out=None):
        """N transitions, every `thin`-th kept (dhmc_mcmc_thinned).  `out` may hold preallocated arrays; page-locked
        ones (host_alloc) are written by the sampling kernel directly, so the kept draws need not fit in HBM."""
        _argcheck(thin >= 1 and N % thin == 0, "thin ≥ 1 and N a multiple of thin")
        K, D, n = self.K, self.D, N // thin
        out = out or {}
        post = out.get("posterior_matrix", None)
        post = np.empty((K, n, D)) if post is None else post
        stats = out.get("tree_statistics", None)
        stats = np.zeros((K, n), dtype=L.tree_stats_dtype) if stats is None else stats
        ld = out.get("logdensities", None)
        ld = np.empty((K, n)) if ld is None else ld
        qq = None if q is None else self._kd(q, "q")
        self._ck(self._lib.dhmc_mcmc_thinned(self._h, L.ptr(qq), C.c_int32(N), C.c_int32(thin), L.ptr(post),
                                             L.ptr(stats), L.ptr(ld)))
        return dict(posterior_matrix=post, tree_statistics=stats, logdensities=ld)

    def mcmc_summary(self, N, thin=1, reference=None, stats=False, quantiles=None, grid=None, bins=256):
        """N transitions as mcmc (same draws, same final state and transition count), every thin-th kept and folded on the
        device into per-(problem, parameter) statistics instead of being returned (dhmc_mcmc_summary, DESIGN §4.4).
        `reference` [P, D] adds the SBC rank of each reference value among its problem's kept draws.  Returns a dict of
        [P, D] arrays — mean, sd, mcse, ess (between-chain batch means, not the Geyer ESS), rhat (split-R̂), rank (−1
        without a reference), draws — plus `record` [P, D, SUMMARY_FIELDS], the mergeable form (diagnostics.merge_summaries,
        dhmc_summary_merge), and with stats=True the kept transitions' tree_statistics and logdensities [K, N // thin].
        A chain that fails is left out of its problem's statistics; the call raises as mcmc does, and the exception's
        debug_information["summary"] holds the summary of the other chains.

        `quantiles` (probabilities in [0, 1]) with `grid` = (lo, hi), each [P, D], also counts the kept draws into `bins`
        equal bins between lo and hi plus one tail bin on each side (dhmc_mcmc_summary_histogram) and adds `quantile`,
        `quantile_lo`, `quantile_hi` [P, D, len(quantiles)] (the exact quantile of the kept draws lies in [quantile_lo,
        quantile_hi]; diagnostics.histogram_quantiles), `histogram` [P, D, bins + 2] (exact counts: those of shards on one
        grid add up), `grid` and `probs`."""
        from . import diagnostics
        _argcheck(N >= 1 and thin >= 1 and N % thin == 0, "N ≥ 1, thin ≥ 1 and N a multiple of thin")
        _argcheck(N // thin >= 4, "at least 4 kept draws per chain (N / thin ≥ 4)")
        P = self.ℓ.n_problems if isinstance(self.ℓ, ProblemBatch) else 1
        ref = None
        if reference is not None:
            ref = np.ascontiguousarray(reference, float)
            _argcheck(ref.shape == (P, self.D), f"reference: [P, D] = ({P}, {self.D})")
        _argcheck(quantiles is not None or grid is None, "grid without quantiles")
        counts = None
        if quantiles is not None:
            probs = np.ascontiguousarray(np.atleast_1d(np.asarray(quantiles, float)))
            _argcheck(probs.ndim == 1 and probs.size >= 1 and np.all((probs >= 0.0) & (probs <= 1.0)),
                      "quantiles: probabilities in [0, 1]")
            _argcheck(grid is not None and len(grid) == 2, "quantiles need grid = (lo, hi), each [P, D]")
            lo, hi = diagnostics.check_grid(grid[0], grid[1], bins, (P, self.D))
            bins = int(bins)
            counts = np.zeros((P, self.D, bins + 2), np.int64)
        record = np.zeros((P, self.D, L.SUMMARY_FIELDS))
        n = N // thin
        st = np.zeros((self.K, n), dtype=L.tree_stats_dtype) if stats else None
        ld = np.empty((self.K, n)) if stats else None
        if counts is None:
            rc = self._lib.dhmc_mcmc_summary(self._h, N, thin, L.ptr(ref), L.ptr(record), L.ptr(st), L.ptr(ld))
        else:
            rc = self._lib.dhmc_mcmc_summary_histogram(self._h, N, thin, L.ptr(ref), L.ptr(lo), L.ptr(hi), bins,
                                                       L.ptr(record), L.ptr(counts), L.ptr(st), L.ptr(ld))
        if rc not in (L.DHMC_OK, L.DHMC_ENUMERIC):
            self._ck(rc)
        out = self.summary_finish(record)
        out["record"] = record
        if counts is not None:
            shape = (P, self.D, probs.size)
            q, q_lo, q_hi = np.empty(shape), np.empty(shape), np.empty(shape)
            self._ck(self._lib.dhmc_histogram_quantiles(L.ptr(counts), L.ptr(lo), L.ptr(hi), bins, self.D, P, L.ptr(probs),
                                                        probs.size, L.ptr(q), L.ptr(q_lo), L.ptr(q_hi)))
            out.update(quantile=q, quantile_lo=q_lo, quantile_hi=q_hi, histogram=counts, grid=(lo, hi), probs=probs)
        if stats:
            out.update(tree_statistics=st, logdensities=ld)
        try:
            self._ck(rc)
        except (ArgumentError, DynamicHMCError) as e:
            e.debug_information["summary"] = out
            raise
        return out

    def summary_finish(self, record):
        """dhmc_summary_finish of a record [P, D, SUMMARY_FIELDS] → mean, sd, mcse, ess, rhat, rank, draws [P, D]."""
        rec = np.ascontiguousarray(record, float)
        P, D = rec.shape[:2]
        _argcheck(rec.shape == (P, D, L.SUMMARY_FIELDS), "record: [P, D, SUMMARY_FIELDS]")
        out = {k: np.empty((P, D)) for k in ("mean", "sd", "mcse", "ess", "rhat")}
        out.update(rank=np.empty((P, D), np.int64), draws=np.empty((P, D), np.int64))
        self._ck(self._lib.dhmc_summary_finish(L.ptr(rec), D, P, *(L.ptr(out[k]) for k in
                                                                      ("mean", "sd", "mcse", "ess", "rhat", "rank", "draws"))))
        return out

    def host_alloc(self, shape, dtype=np.float64):
        """Page-locked, device-mapped numpy array on the NUMA node of this engine's GPU (dhmc_host_alloc).
        Freed with the engine (or host_free)."""
        dt = np.dtype(dtype)
        nbytes = int(np.prod(shape)) * dt.itemsize
        p, node = C.c_void_p(), C.c_int32(-1)
        self._ck(self._lib.dhmc_host_alloc(self._h, C.c_size_t(max(nbytes, 1)), C.byref(p), C.byref(node)))
        buf = (C.c_char * max(nbytes, 1)).from_address(p.value)
        a = np.frombuffer(buf, dtype=dt, count=int(np.prod(shape))).reshape(shape)
        self._host_allocs = getattr(self, "_host_allocs", [])
        self._host_allocs.append(p.value)
        self.numa_node = node.value
        return a

    def host_free_all(self):
        for p in getattr(self, "_host_allocs", []):
            self._lib.dhmc_host_free(self._h, C.c_void_p(p))
        self._host_allocs = []

    # -- multi-GPU (include/dhmc.h, "multi-GPU"): one all-gather of draws at the end
    @staticmethod
    def comm_unique_id():
        lib = L.lib()
        buf = (C.c_char * L.COMM_ID_BYTES)()
        rc = lib.dhmc_comm_unique_id(buf)
        if rc != L.DHMC_OK:
            raise RuntimeError(f"dhmc_comm_unique_id failed [{rc}]: {lib.dhmc_last_error(None).decode()}")
        return bytes(buf)

    def comm_init(self, nranks, rank, unique_id: bytes):
        _argcheck(len(unique_id) == L.COMM_ID_BYTES, "128-byte ncclUniqueId")
        self._ck(self._lib.dhmc_comm_init(self._h, C.c_int32(nranks), C.c_int32(rank), C.c_char_p(unique_id)))

    def allgather_dev(self, send_ptr, recv_ptr, count):
        self._ck(self._lib.dhmc_allgather_dev(self._h, C.c_void_p(send_ptr), C.c_void_p(recv_ptr), C.c_size_t(count)))
        v = C.c_double()
        self._ck(self._lib.dhmc_last_comm_ms(self._h, C.byref(v)))
        return v.value

    def allgather_positions_dev(self, recv_ptr):
        self._ck(self._lib.dhmc_allgather_positions_dev(self._h, C.c_void_p(recv_ptr)))
        v = C.c_double()
        self._ck(self._lib.dhmc_last_comm_ms(self._h, C.byref(v)))
        return v.value

    def mcmc_dev(self, N, posterior_ptr=0, stats_ptr=0, logdens_ptr=0):
        """Device-pointer variant: draws stay in HBM (e.g. torch tensors' data_ptr())."""
        self._ck(self._lib.dhmc_mcmc_dev(self._h, C.c_int32(N), C.c_void_p(posterior_ptr or None),
                                         C.c_void_p(stats_ptr or None), C.c_void_p(logdens_ptr or None)))

    def tree_summary_dev(self, stats_ptr, N, ebfmi=True):
        """Diagnostics reduced on the GPU from a DEVICE statistics buffer [K, N] (dhmc_mcmc_dev)."""
        depth = np.zeros(33, dtype=np.int64)
        term = np.zeros(3, dtype=np.int64)
        acc, steps = C.c_double(), C.c_int64()
        eb = np.empty(self.K) if ebfmi else None
        self._ck(self._lib.dhmc_tree_summary_dev(self._h, C.c_void_p(stats_ptr), C.c_int32(N), L.ptr(depth), L.ptr(term),
                                                 C.byref(acc), C.byref(steps), L.ptr(eb)))
        nz = np.nonzero(depth)[0]
        return dict(N=self.K * N, a_mean=acc.value / (self.K * N), steps=steps.value,
                    termination_counts=dict(max_depth=int(term[0]), divergence=int(term[1]), turning=int(term[2])),
                    depth_counts=depth[: nz[-1] + 1].tolist() if nz.size else [], EBFMI=eb)

    def ess_rhat_dev(self, draws_ptr, N, max_lag=0):
        """split-R̂ and ESS per parameter from a DEVICE draws buffer [K, N, D] (dhmc_ess_rhat_dev)."""
        rhat, ess = np.empty(self.D), np.empty(self.D)
        self._ck(self._lib.dhmc_ess_rhat_dev(self._h, C.c_void_p(draws_ptr), C.c_int32(N), C.c_int32(max_lag),
                                             L.ptr(rhat), L.ptr(ess)))
        return dict(rhat=rhat, ess=ess)

    def ess_rhat_problems_dev(self, draws_ptr, N, max_lag=0):
        """split-R̂ and ESS per (problem, parameter) of a ProblemBatch, each over its problem's local chains, from a DEVICE
        draws buffer [K, N, D] (dhmc_ess_rhat_problems_dev) → rhat, ess [P, D]; NaN for a problem without local chains."""
        _argcheck(isinstance(self.ℓ, ProblemBatch), "the engine holds no ProblemBatch")
        P = self.ℓ.n_problems
        rhat, ess = np.empty((P, self.D)), np.empty((P, self.D))
        self._ck(self._lib.dhmc_ess_rhat_problems_dev(self._h, C.c_void_p(draws_ptr), C.c_int32(N), C.c_int32(max_lag),
                                                      L.ptr(rhat), L.ptr(ess)))
        return dict(rhat=rhat, ess=ess)

    def acceptance_quantiles_dev(self, stats_ptr, N, probs=(0.05, 0.25, 0.5, 0.75, 0.95)):
        """a_quantiles of summarize_tree_statistics (diagnostics.jl:35) from a DEVICE statistics buffer."""
        pr = np.ascontiguousarray(probs, float)
        out = np.empty(pr.size)
        self._ck(self._lib.dhmc_acceptance_quantiles_dev(self._h, C.c_void_p(stats_ptr), C.c_int32(N), L.ptr(pr),
                                                         C.c_int32(pr.size), L.ptr(out)))
        return out

    # -- measurement hooks
    def last_total_steps(self):
        v = C.c_int64()
        self._ck(self._lib.dhmc_last_total_steps(self._h, C.byref(v)))
        return v.value

    def last_kernel_ms(self):
        v = C.c_double()
        self._ck(self._lib.dhmc_last_kernel_ms(self._h, C.byref(v)))
        return v.value

    def kernel_launches(self):
        v = C.c_int64()
        self._ck(self._lib.dhmc_kernel_launches(self._h, C.byref(v)))
        return v.value


# ------------------------------------------------------------------ results
class Results(Sequence):
    """results[k] is the reference's NamedTuple for chain k; the [D, N, K]
    column-major buffer is shared (zero-copy views)."""

    def __init__(self, post, stats, logd, minv, eps):
        self._post, self._stats, self._logd, self._minv, self._eps = post, stats, logd, minv, eps

    def __len__(self):
        return self._post.shape[0]

    def __getitem__(self, k):
        # NB: string keys, not keywords — Python NFKC-normalises identifiers (ϵ → ε)
        return {"posterior_matrix": self._post[k].T,        # [D, N] view, mcmc.jl:230
                "tree_statistics": self._stats[k], "logdensities": self._logd[k],
                "κ": GaussianKineticEnergy(self._minv[k], dense=self._minv[k].ndim == 2), "ϵ": float(self._eps[k]),
                "eps": float(self._eps[k])}


def results_by_problem(results: Results, batch: ProblemBatch, chain_offset=0):
    """The Results of a ProblemBatch run split per problem: element p holds problem p's local chains (zero-copy views;
    empty for a problem with no chain on this handle).  `chain_offset` is the handle's (a shard of the batch)."""
    B = len(results)
    out = []
    for p in range(batch.n_problems):
        lo, hi = batch.problem_chains(p, chain_offset, B)
        out.append(Results(results._post[lo:hi], results._stats[lo:hi], results._logd[lo:hi], results._minv[lo:hi],
                           results._eps[lo:hi]))
    return out


def stack_posterior_matrices(results: Results):
    """[draw, chain, parameter] view — src/mcmc.jl:602-604"""
    return results._post.transpose(1, 0, 2)


def pool_posterior_matrices(results: Results):
    """[parameter, draw ⊗ chain] — src/mcmc.jl:614-616"""
    K, N, D = results._post.shape
    return results._post.reshape(K * N, D).T


# ------------------------------------------------------------------ drivers
def _initialize(engine: Engine, initialization):
    """initialize_warmup_state — src/mcmc.jl:129-132"""
    # keys may arrive as keywords (NFKC-normalised by Python: ϵ → ε) or as strings
    init = {unicodedata.normalize("NFKC", k): v for k, v in dict(initialization or {}).items()}
    init = {{"ε": "ϵ", "eps": "ϵ", "kappa": "κ"}.get(k, k): v for k, v in init.items()}
    unknown = set(init) - {"q", "κ", "ϵ"}
    _argcheck(not unknown, f"unknown initialization fields {unknown}")
    if init.get("κ") is not None:
        engine.set_kinetic_energy(init["κ"])
    if init.get("q") is not None:
        q = np.asarray(init["q"], float)
        if q.ndim == 1:
            q = np.broadcast_to(q, (engine.K, engine.D))
        engine.set_position(q)
    else:
        engine.random_position()
    if init.get("ϵ") is not None:
        engine.set_stepsize(init["ϵ"])


def _report(reporter, message, **kw):
    """The reporter hook (src/reporting.jl; `report(reporter, …)` call sites mcmc.jl:279,378): the reference reports per
    transition, this engine once per batch of transitions between two library calls.  `reporter` is None
    (NoProgressReport) or a callable `reporter(message, **fields)`; a failing reporter never aborts sampling."""
    if reporter is None:
        return
    try:
        reporter(message, **kw)
    except Exception:
        pass


def _default_chains(ℓ, chains, chain_offset):
    if chains is not None:
        return chains
    return ℓ.chains - chain_offset if isinstance(ℓ, ProblemBatch) else 1


def _warm_up(seed, ℓ, chains, initialization, warmup_stages, algorithm, keep_warmup, device, chain_offset, engine_opts,
             reporter):
    """the warm-up half of mcmc_keep_warmup: a new Engine taken through every stage → (engine, per-stage results)"""
    stages = default_warmup_stages() if warmup_stages is None else warmup_stages
    eng = Engine(ℓ, chains, seed=seed, algorithm=algorithm, device=device, chain_offset=chain_offset,
                 **(engine_opts or {}))
    _initialize(eng, initialization)
    warm = []
    for i, stage in enumerate(stages):                       # _warmup fold, mcmc.jl:450-457
        if stage is None:                                    # no-op stage, mcmc.jl:99-101
            warm.append(dict(stage=None, results=None))
        elif isinstance(stage, InitialStepsizeSearch):
            eng.find_initial_stepsize(stage)
            warm.append(dict(stage=stage, results=None))
        elif isinstance(stage, TuningNUTS):
            warm.append(dict(stage=stage, results=eng.warmup_stage(stage, keep=keep_warmup)))
        else:
            raise ArgumentError(f"unknown warmup stage {stage!r}")
        _report(reporter, "warmup stage finished", stage=i + 1, of=len(stages), kind=type(stage).__name__,
                transitions=getattr(stage, "N", 0), chains=chains)
    return eng, warm


def mcmc_keep_warmup(seed, ℓ, N, chains=None, initialization=None, warmup_stages=None,
                     algorithm=None, keep_warmup=True, device=0, chain_offset=0, engine_opts=None, reporter=None):
    """src/mcmc.jl:521-532 for `chains` chains at once (default 1; for a ProblemBatch every chain of the batch from
    chain_offset on)."""
    chains = _default_chains(ℓ, chains, chain_offset)
    eng, warm = _warm_up(seed, ℓ, chains, initialization, warmup_stages, algorithm, keep_warmup, device, chain_offset,
                         engine_opts, reporter)
    inf = eng.mcmc(N)
    _report(reporter, "inference finished", transitions=N, chains=chains)
    st = eng.get_state(("minv", "eps"))
    minv = eng.get_metric_dense() if eng.metric_is_dense() else st["minv"]
    results = Results(inf["posterior_matrix"], inf["tree_statistics"], inf["logdensities"],
                      minv, st["eps"])
    return dict(warmup=warm, inference=results, engine=eng)


def mcmc_with_warmup(seed, ℓ, N, chains=None, initialization=None, warmup_stages=None, algorithm=None,
                     device=0, chain_offset=0, engine_opts=None, reporter=None):
    """src/mcmc.jl:575-584 for `chains` chains at once → Results (a ProblemBatch: results_by_problem splits them)."""
    r = mcmc_keep_warmup(seed, ℓ, N, chains=chains, initialization=initialization,
                         warmup_stages=warmup_stages, algorithm=algorithm, keep_warmup=False,
                         device=device, chain_offset=chain_offset, engine_opts=engine_opts, reporter=reporter)
    r["engine"].close()
    return r["inference"]


def summarize_with_warmup(seed, ℓ, N, thin=1, reference=None, chains=None, initialization=None, warmup_stages=None,
                          algorithm=None, device=0, chain_offset=0, engine_opts=None, reporter=None, quantiles=None,
                          grid=None, bins=256):
    """mcmc_with_warmup ending in Engine.mcmc_summary instead of Results: the warm-up, then N transitions whose every
    thin-th draw is folded on the device into per-(problem, parameter) mean, sd, mcse, ess, rhat and — with a reference
    [P, D] — SBC ranks.  Memory and traffic do not grow with N: simulation-based calibration over a ProblemBatch of
    thousands of data sets is one call.  Returns the dict of Engine.mcmc_summary.

    `quantiles` adds bracketed quantiles on `bins` bins of `grid` = (lo, hi) [P, D] (Engine.mcmc_summary).  Without a grid,
    a pilot fixes it: after the warm-up, mcmc_summary(max(4, N // 10)) runs as a last warm-up step and the grid is
    diagnostics.quantile_grid of its summary, mean ± 6·sd per (problem, parameter).  The pilot's transitions come before
    the N transitions of the summary (the chains go on from where the pilot left them)."""
    from . import diagnostics
    chains = _default_chains(ℓ, chains, chain_offset)
    eng, _ = _warm_up(seed, ℓ, chains, initialization, warmup_stages, algorithm, False, device, chain_offset,
                      engine_opts, reporter)
    try:
        if quantiles is not None and grid is None:
            n_pilot = max(4, N // 10)
            grid = diagnostics.quantile_grid(eng.mcmc_summary(n_pilot))
            _report(reporter, "quantile grid pilot finished", transitions=n_pilot, chains=chains)
        out = eng.mcmc_summary(N, thin=thin, reference=reference, quantiles=quantiles, grid=grid, bins=bins)
        _report(reporter, "inference finished", transitions=N, chains=chains)
    finally:
        eng.close()
    return out


class MCMCSteps:
    """src/mcmc.jl:335-346 — the sampler frozen at the adapted (κ, ϵ) of a finished warm-up, for stepwise sampling:
        r = mcmc_keep_warmup(seed, ℓ, 0, chains=K); steps = mcmc_steps(r["engine"]); Q = steps.Q
        Q, stats = mcmc_next_step(steps, Q)
    `Q` is the [K, D] matrix of positions (the reference's EvaluatedLogDensity per chain; ℓ and ∇ℓ are re-evaluated
    strictly on upload, hamiltonian.jl:202-217)."""

    def __init__(self, engine: Engine):
        self.engine = engine

    @property
    def Q(self):
        return self.engine.get_state(("q",))["q"]


def mcmc_steps(engine: Engine) -> MCMCSteps:
    """mcmc_steps(sampling_logdensity, warmup_state) — src/mcmc.jl:335-346; the warm-up state lives in the engine."""
    return MCMCSteps(engine)


def mcmc_next_step(steps: MCMCSteps, Q):
    """One NUTS transition of every chain from the positions Q → (Q′, tree_statistics [K]) — src/mcmc.jl:348-351."""
    out = steps.engine.mcmc_from(np.asarray(Q, float), 1)
    return out["posterior_matrix"][:, 0, :], out["tree_statistics"][:, 0]
