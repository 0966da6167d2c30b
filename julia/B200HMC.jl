# B200HMC.jl — the Julia side of the drop-in boundary (NOT executed in this image: Julia is not
# installed here; the Python mirror dynamichmc.jl_b200/api.py binds the very same C entry points
# through ctypes and is what the tests exercise; tests/test_cabi_exports.py checks every ccall below
# against include/dhmc.h: argument counts, and that chain_status is always called with its K).
#
# Usage next to the real package:
#     using DynamicHMC, B200HMC
#     ℓ = B200HMC.StandardNormal(1000)                  # a DeviceLogDensity
#     results = B200HMC.mcmc_with_warmup(2026, ℓ, 10; chains = 65_536)     # draws are D·N·chains·8 B on the host (5.2 GB here)
#     results[k].posterior_matrix, results[k].tree_statistics, results[k].κ, results[k].ϵ
# `results[k]` has the fields of DynamicHMC.mcmc_with_warmup's NamedTuple (src/mcmc.jl:575-584), so
# stack_posterior_matrices / pool_posterior_matrices (src/mcmc.jl:602-617) and DynamicHMC.Diagnostics
# work unchanged.  mcmc_keep_warmup / mcmc_steps / mcmc_next_step mirror src/mcmc.jl:521-532, 335-351.
module B200HMC

using DynamicHMC: DynamicHMC, NUTS, DualAveraging, FixedStepsize, InitialStepsizeSearch,
                  TuningNUTS, GaussianKineticEnergy, TreeStatisticsNUTS, DynamicHMCError,
                  default_warmup_stages, NoProgressReport
using LinearAlgebra: Diagonal, Symmetric
import LogDensityProblems

const LIB = get(ENV, "DHMC_B200_LIB", "libdhmc_b200.so")

# ---- include/dhmc.h --------------------------------------------------------
struct Config                     # dhmc_config
    device::Int32; family::Int32; dim::Int64; n_chains::Int64; chain_offset::Int64
    seed::UInt64; max_depth::Int32; threads_per_chain::Int32; min_delta::Float64
    ctas_per_sm::Int32; reserved::Int32
end
struct DualAveragingC             # dhmc_dual_averaging
    delta::Float64; gamma::Float64; kappa::Float64; t0::Int32; pad::Int32
end
# TreeStatisticsNUTS is isbits with the layout of dhmc_tree_stats (56 bytes), so the
# output buffer is a Matrix{TreeStatisticsNUTS} passed as Ptr{Cvoid}.
@assert sizeof(TreeStatisticsNUTS) == 56

const OK, EARG, ENUMERIC = 0, 1, 2
const CHAIN_BAD_INITIAL, CHAIN_NONFINITE_Q, CHAIN_LEAPFROG_NONFINITE = Int32(1), Int32(4), Int32(64)   # per-chain status bits

mutable struct Handle
    ptr::Ptr{Cvoid}
    D::Int; K::Int
    function Handle(cfg::Config)
        out = Ref{Ptr{Cvoid}}(C_NULL)
        rc = ccall((:dhmc_create, LIB), Cint, (Ref{Config}, Ref{Ptr{Cvoid}}), cfg, out)
        rc == OK || _throw(rc, C_NULL, 0)
        h = new(out[], cfg.dim, cfg.n_chains)
        finalizer(h -> ccall((:dhmc_destroy, LIB), Cint, (Ptr{Cvoid},), h.ptr), h)
    end
end

function chain_status(ptr::Ptr{Cvoid}, K::Integer)
    st = Vector{Int32}(undef, K)
    K > 0 && ccall((:dhmc_chain_status, LIB), Cint, (Ptr{Cvoid}, Ptr{Int32}), ptr, st)
    st
end
# status codes -> the reference's exceptions (utilities.jl:17-27; @argcheck sites → ArgumentError)
function _throw(rc, ptr, K)
    msg = unsafe_string(ccall((:dhmc_last_error, LIB), Cstring, (Ptr{Cvoid},), ptr))
    rc == EARG && throw(ArgumentError(msg))
    if rc == ENUMERIC
        status = ptr == C_NULL ? Int32[] : chain_status(ptr, K)
        # leapfrog's @argcheck isfinite(Q.ℓq) (hamiltonian.jl:276) is an ArgumentError; a chain whose strict initial
        # evaluation failed or that met a non-finite position first has failed with DynamicHMCError before it got there
        halted = findall(s -> (s & CHAIN_LEAPFROG_NONFINITE) != 0 && (s & (CHAIN_BAD_INITIAL | CHAIN_NONFINITE_Q)) == 0,
                         status)
        isempty(halted) || throw(ArgumentError("$msg (chains $halted)"))
        throw(DynamicHMCError(msg, (; failed_chains = findall(!iszero, status), status)))
    end
    error("libdhmc_b200 error [$rc]: $msg")
end
_ck(h::Handle, rc) = rc == OK ? nothing : _throw(rc, h.ptr, h.K)

# ---- device log densities (LogDensityProblems API on the CPU side too) ------
abstract type DeviceLogDensity end
struct StandardNormal <: DeviceLogDensity; D::Int; end
struct DiagNormal <: DeviceLogDensity; μ::Vector{Float64}; σ²::Vector{Float64}; end
struct Funnel <: DeviceLogDensity; D::Int; end
"Logistic regression with a N(0, I) prior: X is N×p, 0 ≤ y ≤ 1 (include/dhmc_models.h, LOGISTIC)."
struct LogisticRegression <: DeviceLogDensity
    X::Matrix{Float64}; y::Vector{Float64}
    function LogisticRegression(X, y)
        size(X, 1) == length(y) || throw(ArgumentError("X: [N, p], y: [N]"))
        all(v -> 0 ≤ v ≤ 1, y) || throw(ArgumentError("0 ≤ y ≤ 1 (Bernoulli responses)"))
        new(X, y)
    end
end
"""
The user's own ℓ as device code: a model header (include/dhmc_models.h, "the model header contract"; examples in
include/models/) compiled into its own build of the library, where it is family 4 (USER).  `params` is the block of doubles
the header's formulas receive; `cpu` optionally is `q -> (ℓ(q), ∇ℓ(q))` for host-side use of the same object.
A user-model library carries the USER family only, and `LIB` is a per-module constant, so such a model is run through a copy
of this module bound to its library:

    lib = B200HMC.compile_user_model("include/models/rosenbrock.h")       # make user USER_HEADER=… (nvcc, sm_90a)
    M = B200HMC.bind_user_library(lib)                                     # a copy of B200HMC with LIB = lib
    results = M.mcmc_with_warmup(2026, M.UserModel(100, [1.0, 5.0]), 100; chains = 65_536)
"""
struct UserModel{F} <: DeviceLogDensity
    D::Int; params::Vector{Float64}; cpu::F
end
UserModel(D::Integer, params = Float64[]; cpu = nothing) = UserModel(Int(D), Vector{Float64}(params), cpu)
family(::StandardNormal) = Int32(0); family(::DiagNormal) = Int32(1); family(::Funnel) = Int32(2)
family(::LogisticRegression) = Int32(3); family(::UserModel) = Int32(4)
params(::DeviceLogDensity) = Float64[]
params(ℓ::UserModel) = ℓ.params
LogDensityProblems.dimension(ℓ::UserModel) = ℓ.D
LogDensityProblems.logdensity_and_gradient(ℓ::UserModel, q) =
    ℓ.cpu === nothing ? error("this UserModel was created without a host-side `cpu` function") : ℓ.cpu(q)
"DHMC_USER_NAME of the model compiled into LIB (dhmc_user_family_name); `nothing` for the stock library."
function user_family_name()
    buf = zeros(UInt8, 128)
    rc = ccall((:dhmc_user_family_name, LIB), Cint, (Ptr{UInt8}, Csize_t), buf, length(buf))
    rc == OK ? unsafe_string(pointer(buf)) : nothing
end
"Whether LIB carries the kernels of `family` (dhmc_family_available): the stock library 0…3, a user-model library 4."
family_available(fam::Integer) = (v = Ref{Int32}(0);
    ccall((:dhmc_family_available, LIB), Cint, (Int32, Ref{Int32}), fam, v) == OK && v[] != 0)
"Build the library that carries the model in `header` (csrc/Makefile target `user`); returns its path."
function compile_user_model(header::AbstractString; csrc = joinpath(@__DIR__, "..", "dynamichmc.jl_b200", "csrc"),
                            out_dir = joinpath(csrc, "user_models", splitext(basename(header))[1]), deep::Bool = false)
    so = joinpath(abspath(out_dir), "libdhmc_user_" * splitext(basename(header))[1] * ".so")
    mkpath(out_dir)
    parts = deep ? "0 3" : "0"                    # "0 3": also the kernels for NUTS(max_depth > 12)
    run(`make -C $csrc -j2 user USER_HEADER=$(abspath(header)) USER_LIB=$so USER_BUILD=$(joinpath(abspath(out_dir), "build")) USER_PARTS=$parts`)
    so
end
"A copy of this module whose ccalls go to the user-model library `path`."
function bind_user_library(path::AbstractString; name = Symbol("B200HMC_", replace(splitext(basename(path))[1], r"\W" => "_")))
    withenv("DHMC_B200_LIB" => abspath(path)) do
        outer = Module(name)
        Base.include(outer, @__FILE__)            # evaluates `module B200HMC … end` again, with LIB = path
        getfield(outer, :B200HMC)
    end
end
"""
Many posteriors on one handle (dhmc_set_problems): `problems` share family and dimension and have parameter blocks of equal
length (logistic regression: the same N); global chain g samples problem g ÷ K.  Built by
`mcmc_with_warmup(seed, problems, N; chains_per_problem = K)`.
"""
struct ProblemBatch <: DeviceLogDensity
    problems::Vector{DeviceLogDensity}; K::Int
    function ProblemBatch(problems::AbstractVector, K::Integer)
        isempty(problems) && throw(ArgumentError("a batch needs at least one problem"))
        K ≥ 1 || throw(ArgumentError("chains_per_problem ≥ 1"))
        f, D = family(first(problems)), LogDensityProblems.dimension(first(problems))
        all(ℓ -> family(ℓ) == f && LogDensityProblems.dimension(ℓ) == D, problems) ||
            throw(ArgumentError("every problem of a batch has the same family and dimension"))
        all(ℓ -> length(params(ℓ)) == length(params(first(problems))), problems) ||
            throw(ArgumentError("every problem of a batch has a parameter block of the same length (logistic: the same N)"))
        new(collect(DeviceLogDensity, problems), Int(K))
    end
end
"""
A problem batch whose parameter blocks may differ in length (dhmc_set_problems_ragged): logistic regressions with their own
number of observations each.  Each problem's data take device memory of their own size.  `mcmc_with_warmup(seed, problems, N;
chains_per_problem = K)` builds one when the blocks differ in length.
"""
struct RaggedProblemBatch <: DeviceLogDensity
    problems::Vector{DeviceLogDensity}; K::Int
    function RaggedProblemBatch(problems::AbstractVector, K::Integer)
        isempty(problems) && throw(ArgumentError("a batch needs at least one problem"))
        K ≥ 1 || throw(ArgumentError("chains_per_problem ≥ 1"))
        f, D = family(first(problems)), LogDensityProblems.dimension(first(problems))
        all(ℓ -> family(ℓ) == f && LogDensityProblems.dimension(ℓ) == D, problems) ||
            throw(ArgumentError("every problem of a batch has the same family and dimension"))
        all(ℓ -> !isempty(params(ℓ)), problems) || throw(ArgumentError("every problem of a batch needs a non-empty parameter block"))
        new(collect(DeviceLogDensity, problems), Int(K))
    end
end
const AnyProblemBatch = Union{ProblemBatch,RaggedProblemBatch}
family(b::AnyProblemBatch) = family(first(b.problems))
params(b::AnyProblemBatch) = reduce(vcat, params.(b.problems))
LogDensityProblems.dimension(b::AnyProblemBatch) = LogDensityProblems.dimension(first(b.problems))
"Offsets of the blocks of a ragged batch in `params(b)`, [P + 1] (block p is params(b)[offsets[p]+1:offsets[p+1]])."
block_offsets(b::RaggedProblemBatch) = Csize_t.(cumsum(vcat(0, length.(params.(b.problems)))))
params(ℓ::DiagNormal) = vcat(ℓ.μ, 1 ./ ℓ.σ²)
params(ℓ::LogisticRegression) = vcat(Float64(size(ℓ.X, 1)), vec(permutedims(ℓ.X)), ℓ.y)   # [N, X row-major, y]
LogDensityProblems.capabilities(::Type{<:DeviceLogDensity}) = LogDensityProblems.LogDensityOrder{1}()
LogDensityProblems.dimension(ℓ::Union{StandardNormal,Funnel}) = ℓ.D
LogDensityProblems.dimension(ℓ::DiagNormal) = length(ℓ.μ)
LogDensityProblems.dimension(ℓ::LogisticRegression) = size(ℓ.X, 2)
function LogDensityProblems.logdensity_and_gradient(ℓ::LogisticRegression, β)
    η = ℓ.X * β
    sum(ℓ.y .* η .- log1p.(exp.(η))) - sum(abs2, β) / 2, ℓ.X' * (ℓ.y .- 1 ./ (1 .+ exp.(-η))) .- β
end
LogDensityProblems.logdensity_and_gradient(::StandardNormal, q) = (-sum(abs2, q) / 2, -q)
function LogDensityProblems.logdensity_and_gradient(ℓ::DiagNormal, q)
    t = (q .- ℓ.μ) ./ ℓ.σ²
    -sum((q .- ℓ.μ) .* t) / 2, -t
end
function LogDensityProblems.logdensity_and_gradient(ℓ::Funnel, q)
    v, x = q[1], @view q[2:end]; S = sum(abs2, x); ev = exp(-v); n = ℓ.D - 1
    -v^2 / 18 - ev * S / 2 - n * v / 2, vcat(-v / 9 + ev * S / 2 - n / 2, -ev .* x)
end

# ---- state accessors ---------------------------------------------------------
metric_is_dense(h::Handle) = (v = Ref{Int32}(0);
    _ck(h, ccall((:dhmc_metric_is_dense, LIB), Cint, (Ptr{Cvoid}, Ref{Int32}), h.ptr, v)); v[] != 0)
"κ of every chain: GaussianKineticEnergy(Diagonal(m⁻¹)) or, after a TuningNUTS{Symmetric} stage, GaussianKineticEnergy(Symmetric(M⁻¹))."
function kinetic_energies(h::Handle)
    if metric_is_dense(h)
        M = Array{Float64}(undef, h.D, h.D, h.K)
        _ck(h, ccall((:dhmc_get_metric_dense, LIB), Cint, (Ptr{Cvoid}, Ptr{Float64}), h.ptr, M))
        return [GaussianKineticEnergy(Symmetric(M[:, :, k])) for k in 1:h.K]
    end
    minv = Matrix{Float64}(undef, h.D, h.K)
    _ck(h, ccall((:dhmc_get_state, LIB), Cint,
                 (Ptr{Cvoid}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}),
                 h.ptr, C_NULL, C_NULL, C_NULL, minv, C_NULL, C_NULL))
    [GaussianKineticEnergy(Diagonal(minv[:, k])) for k in 1:h.K]
end
function stepsizes(h::Handle)
    ϵ = Vector{Float64}(undef, h.K)
    _ck(h, ccall((:dhmc_get_state, LIB), Cint,
                 (Ptr{Cvoid}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}),
                 h.ptr, C_NULL, C_NULL, C_NULL, C_NULL, ϵ, C_NULL))
    ϵ
end
function positions(h::Handle)
    q = Matrix{Float64}(undef, h.D, h.K)
    _ck(h, ccall((:dhmc_get_state, LIB), Cint,
                 (Ptr{Cvoid}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}),
                 h.ptr, q, C_NULL, C_NULL, C_NULL, C_NULL, C_NULL))
    q
end

# ---- initialize_warmup_state — src/mcmc.jl:129-132 ---------------------------
function _initialize(seed, ℓ::DeviceLogDensity, chains, initialization, algorithm, device, chain_offset)
    D = LogDensityProblems.dimension(ℓ)
    h = Handle(Config(device, family(ℓ), D, chains, chain_offset, seed, algorithm.max_depth, 0,
                      algorithm.min_Δ, 0, 0))
    p = params(ℓ)
    if ℓ isa RaggedProblemBatch
        _ck(h, ccall((:dhmc_set_problems_ragged, LIB), Cint, (Ptr{Cvoid}, Ptr{Float64}, Ptr{Csize_t}, Int64, Int64),
                     h.ptr, p, block_offsets(ℓ), length(ℓ.problems), ℓ.K))
    elseif ℓ isa ProblemBatch
        _ck(h, ccall((:dhmc_set_problems, LIB), Cint, (Ptr{Cvoid}, Ptr{Float64}, Csize_t, Int64, Int64),
                     h.ptr, p, length(p) ÷ length(ℓ.problems), length(ℓ.problems), ℓ.K))
    else
        _ck(h, ccall((:dhmc_set_problem, LIB), Cint, (Ptr{Cvoid}, Ptr{Float64}, Csize_t), h.ptr, p, length(p)))
    end
    init = NamedTuple(initialization)
    if haskey(init, :κ)
        M⁻¹ = init.κ.M⁻¹
        if M⁻¹ isa Diagonal
            m = Matrix{Float64}(repeat(Vector(M⁻¹.diag), 1, chains))
            _ck(h, ccall((:dhmc_set_metric, LIB), Cint, (Ptr{Cvoid}, Ptr{Float64}, Cint), h.ptr, m, 0))
        else
            set_metric_dense!(h, M⁻¹)
        end
    end
    if haskey(init, :q)
        q = Matrix{Float64}(repeat(init.q, 1, chains))            # [D, K] column-major
        _ck(h, ccall((:dhmc_set_position, LIB), Cint, (Ptr{Cvoid}, Ptr{Float64}), h.ptr, q))
    else
        _ck(h, ccall((:dhmc_random_position, LIB), Cint, (Ptr{Cvoid},), h.ptr))
    end
    haskey(init, :ϵ) &&
        _ck(h, ccall((:dhmc_set_stepsize, LIB), Cint, (Ptr{Cvoid}, Ref{Float64}, Cint), h.ptr, Float64(init.ϵ), 1))
    h
end

# one `report` per batch of transitions (the reference reports per transition, mcmc.jl:279,378)
_report(::NoProgressReport, args...; kw...) = nothing
_report(reporter, msg; kw...) = try DynamicHMC.report(reporter, msg; kw...) catch; nothing end

function _mcmc(h::Handle, N::Integer)                             # mcmc — src/mcmc.jl:366-381
    posterior = Array{Float64}(undef, h.D, N, h.K)                # [D, N, K]: results[k] is a view
    stats = Matrix{TreeStatisticsNUTS}(undef, N, h.K)
    logd = Matrix{Float64}(undef, N, h.K)
    _ck(h, ccall((:dhmc_mcmc, LIB), Cint, (Ptr{Cvoid}, Int32, Ptr{Float64}, Ptr{Cvoid}, Ptr{Float64}),
                 h.ptr, N, posterior, stats, logd))
    posterior, stats, logd
end

"N transitions of every chain, every `thin`-th kept (dhmc_mcmc_thinned; output contract of `mcmc`, src/mcmc.jl:366-381, with
N ÷ thin draws): what a many-chain run uses instead of keeping D·N·K doubles.  Returns (posterior [D, N÷thin, K], stats, logd)."
function mcmc_thinned(h::Handle, N::Integer, thin::Integer)
    n = N ÷ thin
    posterior = Array{Float64}(undef, h.D, n, h.K)
    stats = Matrix{TreeStatisticsNUTS}(undef, n, h.K)
    logd = Matrix{Float64}(undef, n, h.K)
    _ck(h, ccall((:dhmc_mcmc_thinned, LIB), Cint, (Ptr{Cvoid}, Ptr{Float64}, Int32, Int32, Ptr{Float64}, Ptr{Cvoid}, Ptr{Float64}),
                 h.ptr, C_NULL, N, thin, posterior, stats, logd))
    posterior, stats, logd
end

# ---- mcmc_keep_warmup(rng, ℓ, N; …) — src/mcmc.jl:521-532 ---------------------
"Returns, per chain, `(; initial_warmup_state, warmup, final_warmup_state, inference)` plus the handle (`sampling_logdensity`)."
function mcmc_keep_warmup(seed::Integer, ℓ::DeviceLogDensity, N::Integer; chains::Integer = 1,
                          initialization = (), warmup_stages = default_warmup_stages(),
                          algorithm = NUTS(), reporter = NoProgressReport(), device = 0, chain_offset = 0)
    h = _initialize(seed, ℓ, chains, initialization, algorithm, device, chain_offset)
    q₀ = positions(h)
    warmup = []
    for stage in warmup_stages                                   # _warmup fold — src/mcmc.jl:450-457
        res = warmup!(h, stage; keep = true)
        _report(reporter, "warmup stage finished"; stage = string(typeof(stage)))
        push!(warmup, (; stage, results = res, warmup_state = (; Q = positions(h), κ = kinetic_energies(h), ϵ = stepsizes(h))))
    end
    posterior, stats, logd = _mcmc(h, N)
    _report(reporter, "inference finished"; N)
    κ, ϵ = kinetic_energies(h), stepsizes(h)
    inference = [(; posterior_matrix = view(posterior, :, :, k), tree_statistics = view(stats, :, k),
                    logdensities = view(logd, :, k)) for k in 1:chains]
    (; initial_warmup_state = (; Q = q₀), warmup, final_warmup_state = (; Q = positions(h), κ, ϵ), inference,
       sampling_logdensity = h)
end

# ---- mcmc_with_warmup(rng, ℓ, N; …) for `chains` chains — src/mcmc.jl:575-584 --
function mcmc_with_warmup(seed::Integer, ℓ::DeviceLogDensity, N::Integer; kwargs...)
    r = mcmc_keep_warmup(seed, ℓ, N; kwargs...)
    (; κ, ϵ) = r.final_warmup_state
    [(; r.inference[k]..., κ = κ[k], ϵ = ϵ[k]) for k in eachindex(r.inference)]
end

# ---- problem batches: P posteriors, K chains each, one handle (dhmc_set_problems, _ragged) ----------------------------
"""The results of P problems on one handle: element p is the vector of its K chains' NamedTuples (as `mcmc_with_warmup`).
Problems whose parameter blocks differ in length (logistic regressions with different numbers of observations) form a
RaggedProblemBatch, others a ProblemBatch."""
function mcmc_with_warmup(seed::Integer, problems::AbstractVector{<:DeviceLogDensity}, N::Integer; chains_per_problem::Integer,
                          kwargs...)
    ragged = !isempty(problems) && any(ℓ -> length(params(ℓ)) != length(params(first(problems))), problems)
    b = ragged ? RaggedProblemBatch(problems, chains_per_problem) : ProblemBatch(problems, chains_per_problem)
    r = mcmc_with_warmup(seed, b, N; chains = length(problems) * b.K, kwargs...)
    [r[(p - 1) * b.K + 1:p * b.K] for p in eachindex(problems)]
end
"split-R̂ and ESS per (parameter, problem) of a batch handle's DEVICE draws [D, N, chains] (dhmc_ess_rhat_problems_dev): [D, P]."
function ess_rhat_problems(h::Handle, draws_dev::Ptr{Float64}, N::Integer, P::Integer; max_lag::Integer = 0)
    rhat, ess = Matrix{Float64}(undef, h.D, P), Matrix{Float64}(undef, h.D, P)
    _ck(h, ccall((:dhmc_ess_rhat_problems_dev, LIB), Cint, (Ptr{Cvoid}, Ptr{Float64}, Int32, Int32, Ptr{Float64}, Ptr{Float64}),
                 h.ptr, draws_dev, N, max_lag, rhat, ess))
    (; rhat, ess)
end

# ---- streaming posterior summary (dhmc_mcmc_summary, include/dhmc.h; DESIGN.md §4.4) ----------------------------------
const SUMMARY_FIELDS = 7
"""N transitions at the adapted (κ, ϵ), every `thin`-th folded on the device into per-(parameter, problem) statistics; no draw
is returned.  `reference` [D, P] adds the SBC ranks.  Returns the mergeable record [SUMMARY_FIELDS, D, P] (merge shards with
`summary_merge!`, finish with `summary_finish`)."""
function mcmc_summary(h::Handle, N::Integer, P::Integer; thin::Integer = 1, reference = nothing)
    record = Array{Float64}(undef, SUMMARY_FIELDS, h.D, P)
    ref = reference === nothing ? C_NULL : convert(Matrix{Float64}, reference)
    _ck(h, ccall((:dhmc_mcmc_summary, LIB), Cint, (Ptr{Cvoid}, Int32, Int32, Ptr{Float64}, Ptr{Float64}, Ptr{Cvoid}, Ptr{Float64}),
                 h.ptr, N, thin, ref, record, C_NULL, C_NULL))
    record
end
"record ← record ⊕ other (dhmc_summary_merge): the record of the chains of both"
function summary_merge!(record::Array{Float64,3}, other::Array{Float64,3})
    rc = ccall((:dhmc_summary_merge, LIB), Cint, (Ptr{Float64}, Ptr{Float64}, Int64, Int64),
               record, other, size(record, 2), size(record, 3))
    rc == 0 || throw(ArgumentError("records of different shapes or kept-draw counts"))
    record
end
"mean, sd, mcse, ess (batch means), rhat (split-R̂), rank (−1 without a reference), draws: [D, P] each (dhmc_summary_finish)"
function summary_finish(record::Array{Float64,3})
    D, P = size(record, 2), size(record, 3)
    mean, sd, mcse, ess, rhat = (Matrix{Float64}(undef, D, P) for _ in 1:5)
    rank, draws = Matrix{Int64}(undef, D, P), Matrix{Int64}(undef, D, P)
    rc = ccall((:dhmc_summary_finish, LIB), Cint,
               (Ptr{Float64}, Int64, Int64, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Int64}, Ptr{Int64}),
               record, D, P, mean, sd, mcse, ess, rhat, rank, draws)
    rc == 0 || throw(ArgumentError("summary record"))
    (; mean, sd, mcse, ess, rhat, rank, draws)
end
"""`mcmc_summary` that also counts the kept draws into `nbins` bins of the grid `lo`, `hi` [D, P] plus a tail bin on each side
(dhmc_mcmc_summary_histogram) and returns `(; record, counts, q, q_lo, q_hi)`: counts [nbins + 2, D, P] (shards on one grid
add), and the bracketed quantiles [length(quantiles), D, P] of `histogram_quantiles`."""
function mcmc_summary(h::Handle, N::Integer, P::Integer, lo::AbstractMatrix, hi::AbstractMatrix; quantiles,
                      nbins::Integer = 256, thin::Integer = 1, reference = nothing)
    record = Array{Float64}(undef, SUMMARY_FIELDS, h.D, P)
    counts = zeros(Int64, nbins + 2, h.D, P)
    lo, hi = convert(Matrix{Float64}, lo), convert(Matrix{Float64}, hi)
    ref = reference === nothing ? C_NULL : convert(Matrix{Float64}, reference)
    _ck(h, ccall((:dhmc_mcmc_summary_histogram, LIB), Cint,
                 (Ptr{Cvoid}, Int32, Int32, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Int32, Ptr{Float64}, Ptr{Int64}, Ptr{Cvoid}, Ptr{Float64}),
                 h.ptr, N, thin, ref, lo, hi, nbins, record, counts, C_NULL, C_NULL))
    (; record, counts, histogram_quantiles(counts, lo, hi, quantiles)...)
end
"""q, q_lo, q_hi [length(probs), D, P] of counts [nbins + 2, D, P] on the grid lo, hi [D, P] (dhmc_histogram_quantiles):
the exact type-7 quantile of the counted draws lies in [q_lo, q_hi]; q is NaN when it needs a tail bin."""
function histogram_quantiles(counts::Array{Int64,3}, lo::Matrix{Float64}, hi::Matrix{Float64}, probs)
    nb, D, P = size(counts, 1) - 2, size(counts, 2), size(counts, 3)
    p = convert(Vector{Float64}, collect(probs))
    q, q_lo, q_hi = (Array{Float64}(undef, length(p), D, P) for _ in 1:3)
    rc = ccall((:dhmc_histogram_quantiles, LIB), Cint,
               (Ptr{Int64}, Ptr{Float64}, Ptr{Float64}, Int32, Int64, Int64, Ptr{Float64}, Int32, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}),
               counts, lo, hi, nb, D, P, p, length(p), q, q_lo, q_hi)
    rc == 0 || throw(ArgumentError("histogram quantiles: probabilities in [0, 1] and a valid grid"))
    (; q, q_lo, q_hi)
end

# ---- mcmc_steps / mcmc_next_step — src/mcmc.jl:335-351: stepwise sampling at the adapted (κ, ϵ) -----
struct MCMCSteps; h::Handle; end
mcmc_steps(h::Handle) = MCMCSteps(h)
"One transition of every chain from the positions `Q` ([D, K]); returns (Q′, tree_statistics)."
function mcmc_next_step(s::MCMCSteps, Q::AbstractMatrix{Float64})
    h = s.h
    post = Array{Float64}(undef, h.D, 1, h.K); stats = Matrix{TreeStatisticsNUTS}(undef, 1, h.K)
    logd = Matrix{Float64}(undef, 1, h.K)
    _ck(h, ccall((:dhmc_mcmc_from, LIB), Cint, (Ptr{Cvoid}, Ptr{Float64}, Int32, Ptr{Float64}, Ptr{Cvoid}, Ptr{Float64}),
                 h.ptr, Matrix{Float64}(Q), 1, post, stats, logd))
    reshape(post, h.D, h.K), vec(stats)
end

# GaussianKineticEnergy(Symmetric M⁻¹) — src/hamiltonian.jl:73 (W is computed on the device)
set_metric_dense!(h::Handle, M⁻¹::AbstractMatrix) =
    _ck(h, ccall((:dhmc_set_metric_dense, LIB), Cint, (Ptr{Cvoid}, Ptr{Float64}, Cint), h.ptr, Matrix{Float64}(M⁻¹), 1))

warmup!(h::Handle, ::Nothing; keep = false) = nothing            # src/mcmc.jl:99-101
function warmup!(h::Handle, s::InitialStepsizeSearch; keep = false)   # src/mcmc.jl:134-148
    _ck(h, ccall((:dhmc_find_initial_stepsize, LIB), Cint, (Ptr{Cvoid}, Float64, Float64, Int32),
                 h.ptr, s.initial_ϵ, s.log_threshold, s.maxiter_crossing))
    nothing
end
function warmup!(h::Handle, t::TuningNUTS{M}; keep = false) where {M}   # src/mcmc.jl:258-286
    metric = M === Nothing ? 0 : M <: Diagonal ? 1 : 2            # DHMC_METRIC_NOTHING/_DIAGONAL/_SYMMETRIC
    a = t.stepsize_adaptation
    da = a isa DualAveraging ? Ref(DualAveragingC(a.δ, a.γ, a.κ, a.t₀, 0)) : C_NULL
    post = keep ? Array{Float64}(undef, h.D, t.N, h.K) : C_NULL
    stats = keep ? Matrix{TreeStatisticsNUTS}(undef, t.N, h.K) : C_NULL
    ϵs = keep ? Matrix{Float64}(undef, t.N, h.K) : C_NULL
    logd = keep ? Matrix{Float64}(undef, t.N, h.K) : C_NULL
    _ck(h, ccall((:dhmc_warmup_stage, LIB), Cint,
                 (Ptr{Cvoid}, Int32, Int32, Ptr{Cvoid}, Float64, Ptr{Float64}, Ptr{Cvoid}, Ptr{Float64}, Ptr{Float64}),
                 h.ptr, t.N, metric, da, t.λ, post, stats, ϵs, logd))
    keep ? (; posterior_matrix = post, tree_statistics = stats, ϵs, logdensities = logd) : nothing
end

# ---- fine-grained path used by julia/parity.jl ---------------------------------
"sample_tree with injected momenta `p` ([D, K]) and direction words (NUTS.jl:232-233 keywords)."
function sample_tree!(h::Handle, p::Matrix{Float64}, directions::Vector{UInt32})
    stats = Vector{TreeStatisticsNUTS}(undef, h.K)
    _ck(h, ccall((:dhmc_sample_tree, LIB), Cint, (Ptr{Cvoid}, Ptr{Float64}, Ptr{UInt32}, Ptr{Cvoid}), h.ptr, p, directions, stats))
    positions(h), stats
end
set_position!(h::Handle, q::Matrix{Float64}) = _ck(h, ccall((:dhmc_set_position, LIB), Cint, (Ptr{Cvoid}, Ptr{Float64}), h.ptr, q))
set_stepsize!(h::Handle, ϵ::Vector{Float64}) = _ck(h, ccall((:dhmc_set_stepsize, LIB), Cint, (Ptr{Cvoid}, Ptr{Float64}, Cint), h.ptr, ϵ, 0))
set_transition_count!(h::Handle, t::Integer) = _ck(h, ccall((:dhmc_set_transition_count, LIB), Cint, (Ptr{Cvoid}, UInt32), h.ptr, t))

# ---- multi-GPU: one rank (process) per GPU, one all-gather at the end (include/dhmc.h "multi-GPU") -----
comm_unique_id() = (id = zeros(UInt8, 128);
    ccall((:dhmc_comm_unique_id, LIB), Cint, (Ptr{UInt8},), id) == OK || error("dhmc_comm_unique_id failed"); id)
comm_init!(h::Handle, nranks, rank, id::Vector{UInt8}) =
    _ck(h, ccall((:dhmc_comm_init, LIB), Cint, (Ptr{Cvoid}, Int32, Int32, Ptr{UInt8}), h.ptr, nranks, rank, id))

end # module
