"""dynamichmc.jl_b200 — H100-native many-chain NUTS engine behind the
DynamicHMC.jl sampler API.  The numeric path is libdhmc_b200.so (hand-written
sm_90a CUDA, csrc/); this package is the thin host mirror of the reference's
interface over its C ABI.  There is no CPU fallback."""
from . import _lib, diagnostics, parallel
from .api import (ArgumentError, DiagNormal, Diagonal, DualAveraging, DynamicHMCError, Engine,
                  FixedStepsize, Funnel, GaussianKineticEnergy, InitialStepsizeSearch, LogisticRegression, NUTS,
                  MCMCSteps, ProblemBatch, RaggedProblemBatch, Results, StandardNormal, Symmetric, SymmetricPooled, TuningNUTS, UserLogDensity, compile_user_model,
                  default_warmup_stages,
                  fixed_stepsize_warmup_stages, mcmc_keep_warmup, mcmc_next_step, mcmc_steps, mcmc_with_warmup,
                  pool_posterior_matrices, results_by_problem, stack_posterior_matrices)
