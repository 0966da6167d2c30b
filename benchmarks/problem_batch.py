"""Problem batches (dhmc_set_problems, DESIGN.md §4.3): many posteriors on one handle against one handle per posterior.

  (a) SBC shape: P DIAG_NORMAL problems (default 1 024, D = 100), 8 chains each, default warm-up + 1 000 draws (kept on the
      device), as ONE batched handle against P sequential single-problem handles (wall time; all P unless --seq-budget
      stops the sequential side early, which the output then says);
  (b) C4 shape: logistic regression N = 10 000, p = 256, 32 768 chains split into P ∈ {1, 2, 4, 16} problems (a different
      X per problem), after a short step-size warm-up, leapfrog steps / s of the sampling kernel; plus the same chains as one plain problem (no batch: the
      warps of a packed CTA fetch chains on their own) — the P = 1 batch runs the same trees, so the two rates differ only
      by the lock-step group fetch of a batch.  The cases run --c4-repeats times, interleaved, and each case reports the
      range of its rates (the run-to-run spread the differences must exceed).
Prints one JSON line with the GPU name and its power limit read in the same run.

    python benchmarks/problem_batch.py [--problems 1024] [--seq-budget S] [--c4-repeats 3] [--skip-sbc] [--skip-c4]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    import torch
    info = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=20).stdout.strip()
        info["power_limit_w"] = float(out.splitlines()[0])
    except Exception:
        pass
    return info


def sbc(pkg, P, K, D, N, seq_budget):
    import torch
    rng = np.random.default_rng(1)
    problems = [pkg.DiagNormal(rng.normal(size=D), rng.uniform(0.5, 2.0, D)) for _ in range(P)]
    stages = pkg.default_warmup_stages()

    def run(ℓ, chains, off, draws):
        eng = pkg.Engine(ℓ, chains=chains, seed=2026, chain_offset=off)
        eng.random_position(); eng.find_initial_stepsize()
        for st in stages[1:]:
            eng.warmup_stage(st)
        eng.mcmc_dev(N, draws.data_ptr(), 0, 0)
        eng.close()

    draws = torch.empty((P * K, N, D), dtype=torch.float64, device="cuda")
    run(pkg.ProblemBatch(problems[:2], K), 2 * K, 0, draws)          # load the library, first-touch the buffers
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    run(pkg.ProblemBatch(problems, K), P * K, 0, draws)
    torch.cuda.synchronize()
    batched = time.perf_counter() - t0
    del draws
    one = torch.empty((K, N, D), dtype=torch.float64, device="cuda")
    done, t0 = 0, time.perf_counter()
    for p in range(P):
        run(problems[p], K, p * K, one)
        done += 1
        if time.perf_counter() - t0 > seq_budget:
            break
    torch.cuda.synchronize()
    seq = time.perf_counter() - t0
    per_handle = seq / done
    return {"problems": P, "chains_per_problem": K, "dim": D, "draws": N, "warmup": "default_warmup_stages()",
            "batched_s": batched, "sequential_handles_run": done, "sequential_s": seq, "sequential_s_per_handle": per_handle,
            "sequential_s_all": per_handle * P if done < P else seq,
            "sequential_s_all_is": "measured" if done == P else f"extrapolated from {done} of {P} handles",
            "speedup": (per_handle * P) / batched}


def c4(pkg, chains, Ps, steps, n, warm, repeats):
    X0 = [pkg.LogisticRegression.synthetic(N=10000, p=256, seed=7 + i)[0] for i in range(max(Ps))]
    out = []

    def rate(ℓ, label, P):
        import torch
        eng = pkg.Engine(ℓ, chains=chains, seed=2026)
        eng.random_position(); eng.find_initial_stepsize()
        eng.warmup_stage(pkg.TuningNUTS(warm, pkg.DualAveraging()))   # trees of typical depth, not the first step's
        draws = torch.empty((chains, n, 256), dtype=torch.float64, device="cuda")
        eng.mcmc_dev(n, draws.data_ptr(), 0, 0)                     # warm
        st, ms = 0, 0.0
        for _ in range(steps):
            eng.mcmc_dev(n, draws.data_ptr(), 0, 0)
            st += eng.last_total_steps(); ms += eng.last_kernel_ms()
        eng.close()
        return st / (ms * 1e-3), st

    cases = [("one problem, no batch (independent warp fetch)", 1, lambda: X0[0])]
    cases += [(f"batch of {P}", P, lambda P=P: pkg.ProblemBatch(X0[:P], chains // P)) for P in Ps]
    rates = {label: [] for label, _, _ in cases}
    steps_of = {}
    for _ in range(repeats):                                         # interleaved: drifts of the card hit every case alike
        for label, P, make in cases:
            r, st = rate(make(), label, P)
            rates[label].append(r)
            steps_of[label] = st
    for label, P, _ in cases:
        v = rates[label]
        out.append({"case": label, "problems": P, "chains": chains, "leapfrog_steps": steps_of[label],
                    "leapfrog_steps_per_s": v, "min": min(v), "max": max(v), "median": float(np.median(v))})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--problems", type=int, default=1024)
    ap.add_argument("--chains-per-problem", type=int, default=8)
    ap.add_argument("--dim", type=int, default=100)
    ap.add_argument("--draws", type=int, default=1000)
    ap.add_argument("--seq-budget", type=float, default=float("inf"), help="stop the sequential handles of (a) after S seconds")
    ap.add_argument("--c4-chains", type=int, default=32768)
    ap.add_argument("--c4-steps", type=int, default=2)
    ap.add_argument("--c4-draws", type=int, default=2)
    ap.add_argument("--c4-warm", type=int, default=20, help="transitions of the step-size warm-up before timing")
    ap.add_argument("--c4-repeats", type=int, default=3)
    ap.add_argument("--skip-sbc", action="store_true")
    ap.add_argument("--skip-c4", action="store_true")
    args = ap.parse_args()
    from __graft_entry__ import load_package
    pkg = load_package()
    line = gpu_info()
    if not args.skip_sbc:
        line["sbc"] = sbc(pkg, args.problems, args.chains_per_problem, args.dim, args.draws, args.seq_budget)
    if not args.skip_c4:
        line["c4"] = c4(pkg, args.c4_chains, (1, 2, 4, 16), args.c4_steps, args.c4_draws, args.c4_warm, args.c4_repeats)
    line["power_limit_w_after"] = gpu_info()["power_limit_w"]
    print(json.dumps(line))


if __name__ == "__main__":
    main()
