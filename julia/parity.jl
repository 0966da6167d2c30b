# parity.jl — pin the CUDA engine against the REAL DynamicHMC.jl (run where Julia + DynamicHMC are installed; a GPU is
# needed only for the device half).  Not executed in the build image (no Julia there): it exists so that a maintainer can
# close the "parity unpinned" items of SURVEY.md §8c — Julia's Random stream, LogExpFunctions.logaddexp, BLAS dot order.
#
# What it does, per device family (standard / diagonal MvNormal, funnel, logistic regression):
#   1. draws momenta p and direction words with Julia's own RNG and INJECTS them into both sides through the keywords the
#      reference provides for exactly this purpose: `sample_tree(rng, alg, H, Q, ϵ; p = p, directions = d)` (NUTS.jl:232-233)
#      and `dhmc_sample_tree(h, p, directions, stats)`;
#   2. feeds the reference the engine's `randexp` stream: `PhiloxExp <: AbstractRNG` restates the counter-based stream of
#      include/dhmc_math.h (Philox-4x32-10 keyed by (seed), countered by (chain, transition, stream = EXP, index), u ∈ (0,1),
#      randexp = −dm_log(u)), so every `rand_bool_logprob` (NUTS.jl:43-45) sees the same exponential variate on both sides;
#   3. compares TreeStatisticsNUTS field by field (integers must be EQUAL: depth, termination.left/right, steps, directions;
#      π and acceptance_rate within 1e-10 relative) and the new position (1e-10 relative);
#   4. writes tests/golden/julia_<family>.json in the fixture format of tests/golden/ so that `pytest -m "not gpu"` re-checks
#      the ORACLE against these reference-generated vectors (tests/test_golden_vectors.py::test_julia_fixtures_when_present).
#
# Usage:  julia --project julia/parity.jl [--device]   (without --device only the fixtures are written)
using DynamicHMC, LogDensityProblems, Random, LinearAlgebra
using DynamicHMC: Hamiltonian, evaluate_ℓ, sample_tree, NUTS, GaussianKineticEnergy, Directions
import JSON
include(joinpath(@__DIR__, "B200HMC.jl"))

# ------------------------------------------------------------------ include/dhmc_math.h, restated
const M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
mulhi(a::UInt32, b::UInt32) = UInt32((UInt64(a) * UInt64(b)) >> 32)
function philox4x32_10(c0::UInt32, c1::UInt32, c2::UInt32, c3::UInt32, k0::UInt32, k1::UInt32)
    for _ in 1:10
        hi0, lo0 = mulhi(M0, c0), M0 * c0
        hi1, lo1 = mulhi(M1, c2), M1 * c2
        c0, c1, c2, c3 = hi1 ⊻ c1 ⊻ k0, lo1, hi0 ⊻ c3 ⊻ k1, lo0
        k0 += W0; k1 += W1
    end
    (c0, c1, c2, c3)
end
const STREAM_EXP = UInt32(4)
rng_block(seed::UInt64, chain::UInt64, stream::UInt32, t::UInt32, idx::UInt32) =
    philox4x32_10(idx, t, UInt32(chain & 0xffffffff), (stream << 24) | UInt32((chain >> 32) & 0xffffff),
                  UInt32(seed & 0xffffffff), UInt32(seed >> 32))
u01(a::UInt32, b::UInt32) = (Float64((UInt64(a) << 20) | UInt64(b >> 12)) + 0.5) * 2.220446049250313e-16
const LN2_HI, LN2_LO = 6.93147180369123816490e-01, 1.90821492927058770002e-10
function dm_log(x::Float64)            # bit-for-bit dm_log of include/dhmc_math.h (only + − × ÷ fma: no libm)
    x != x && return x; x < 0 && return NaN; x == 0 && return -Inf; isfinite(x) || return x
    e = 0; b = reinterpret(UInt64, x)
    if (b >> 52) == 0
        x *= 18014398509481984.0; b = reinterpret(UInt64, x); e = -54
    end
    e += Int(b >> 52) - 1023
    m = b & 0x000FFFFFFFFFFFFF
    if m >= 0x0006A09E667F3BCD
        xm = reinterpret(Float64, 0x3FE0000000000000 | m); e += 1
    else
        xm = reinterpret(Float64, 0x3FF0000000000000 | m)
    end
    f = xm - 1.0; s = f / (2.0 + f); z = s * s
    R = 2.0 / 23.0
    for c in (2.0 / 21.0, 2.0 / 19.0, 2.0 / 17.0, 2.0 / 15.0, 2.0 / 13.0, 2.0 / 11.0, 2.0 / 9.0, 2.0 / 7.0, 2.0 / 5.0, 2.0 / 3.0)
        R = fma(R, z, c)
    end
    R *= z
    dk = Float64(e)
    dk * LN2_HI + (f + (dk * LN2_LO - s * (f - R)))
end
"the j-th randexp of transition t of a chain (dm_randexp)"
function dm_randexp(seed::UInt64, chain::UInt64, t::UInt32, j::UInt32)
    r = rng_block(seed, chain, STREAM_EXP, t, j >> 1)
    u = isodd(j) ? u01(r[3], r[4]) : u01(r[1], r[2])
    -dm_log(u)
end
"An RNG that serves ONLY randexp, from the engine's stream; anything else is an error (p and directions are injected)."
mutable struct PhiloxExp <: AbstractRNG
    seed::UInt64; chain::UInt64; t::UInt32; j::UInt32
end
Random.randexp(r::PhiloxExp, ::Type{Float64} = Float64) = (v = dm_randexp(r.seed, r.chain, r.t, r.j); r.j += UInt32(1); v)
Random.rand(::PhiloxExp, args...) = error("PhiloxExp serves randexp only: inject p= and directions=")

# ------------------------------------------------------------------ harness
relerr(a, b) = maximum(abs.(a .- b) ./ max.(abs.(b), floatmin(Float64)))
function stats_dict(s)
    Dict("pi" => s.π, "depth" => s.depth, "left" => s.termination.left, "right" => s.termination.right,
         "acceptance_rate" => s.acceptance_rate, "steps" => s.steps, "directions" => Int(s.directions.flags))
end

function run_family(name, ℓ, D; K = 8, transitions = 3, seed = UInt64(2026), device = false)
    rng = Random.Xoshiro(hash(name))
    q0 = randn(rng, D, K); ϵ = exp.(log(0.02) .+ (log(0.6) - log(0.02)) .* rand(rng, K))
    κ = GaussianKineticEnergy(D)
    H = Hamiltonian(κ, ℓ)
    h = device ? B200HMC._initialize(seed, ℓ, K, (q = q0[:, 1],), NUTS(), 0, 0) : nothing
    if device
        B200HMC.set_position!(h, q0); B200HMC.set_stepsize!(h, ϵ)
    end
    cases = []
    q = copy(q0)
    for t in 0:transitions-1
        P = randn(rng, D, K); dirs = rand(rng, UInt32, K)
        device && B200HMC.set_transition_count!(h, t)
        qd, sd = device ? B200HMC.sample_tree!(h, P, dirs) : (nothing, nothing)
        for k in 1:K
            Q = evaluate_ℓ(ℓ, q[:, k]; strict = true)
            r = PhiloxExp(seed, UInt64(k - 1), UInt32(t), UInt32(0))
            Q′, s = sample_tree(r, NUTS(), H, Q, ϵ[k]; p = P[:, k], directions = Directions(dirs[k]))
            push!(cases, Dict("chain" => k - 1, "t" => t, "q" => q[:, k], "eps" => ϵ[k], "p" => P[:, k],
                              "directions" => Int(dirs[k]), "q_new" => Q′.q, "stats" => stats_dict(s), "n_randexp" => Int(r.j)))
            if device
                d = sd[k]
                @assert (d.depth, d.termination.left, d.termination.right, d.steps, d.directions.flags) ==
                        (s.depth, s.termination.left, s.termination.right, s.steps, s.directions.flags) "integer mismatch: $name chain $k t $t"
                @assert relerr(qd[:, k], Q′.q) ≤ 1e-10 && abs(d.π - s.π) ≤ 1e-10 * max(1, abs(s.π))
            end
            q[:, k] = Q′.q
        end
    end
    out = joinpath(@__DIR__, "..", "tests", "golden", "julia_$name.json")
    open(out, "w") do io
        JSON.print(io, Dict("family" => name, "dim" => D, "seed" => Int(seed), "params" => B200HMC.params(ℓ), "generator" => "julia/parity.jl (real DynamicHMC.jl " *
                            string(pkgversion(DynamicHMC)) * ")", "cases" => cases))
    end
    println("$name: $(length(cases)) cases written to $out", device ? "; device == reference on all integers" : "")
end

device = "--device" in ARGS
run_family("std_normal", B200HMC.StandardNormal(50), 50; device)
run_family("diag_normal", B200HMC.DiagNormal(collect(range(-1, 1; length = 30)), exp.(range(-2, 2; length = 30))), 30; device)
run_family("funnel", B200HMC.Funnel(10), 10; device)
let rng = Random.Xoshiro(7), N = 400, p = 12
    X = randn(rng, N, p) ./ sqrt(p); β = randn(rng, p)
    y = Float64.(rand(rng, N) .< 1 ./ (1 .+ exp.(-(X * β))))
    run_family("logistic", B200HMC.LogisticRegression(X, y), p; device)
end
