"""Streaming posterior summary (dhmc_mcmc_summary, DESIGN.md §4.4) against keeping the draws.

  (a) SBC shape of benchmarks/problem_batch.py: P = 1 024 DIAG_NORMAL problems, D = 100, 8 chains each, default warm-up,
      then N = 1 000 draws either kept on the device and reduced by dhmc_ess_rhat_problems_dev, or folded into the summary.
      Wall time of the sampling call (+ diagnostics) and the device memory in use when it returns (handle, scratch and the
      draws buffer: everything is grow-only until the handle closes, so this is the run's high-water mark).
  (b) SBC at 16 384 problems (same shape, thin = 10, references drawn from each posterior): the draws would take
      16 384·8·1 000·100·8 B = 105 GB, so it runs as a summary only.
  (c) C2 shape (65 536 chains, D = 1 000, search + 50 dual-averaging transitions) at N = 100: mcmc_dev without outputs,
      the summary (one problem: every chain's chain-end atomics land on the same D accumulators; thin = 1 and thin = 10,
      which folds a tenth of the draws with the same atomics), and the draws brought to
      the host through the e2e pipeline (mcmc_from with page-locked buffers, 50 two-draw calls).  Leapfrog steps / s of the
      sampling kernel (device events) and wall time; the cases alternate --repeats times.
Prints one JSON line with the GPU name and its power limit read in the same run.

    python benchmarks/streaming_summary.py [--skip-sbc] [--skip-big] [--skip-c2] [--repeats 2]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))
from problem_batch import gpu_info  # noqa: E402


def _used_bytes():
    import torch
    free, total = torch.cuda.mem_get_info()
    return total - free


def _warmed(pkg, ℓ, chains, stages, seed=2026):
    eng = pkg.Engine(ℓ, chains=chains, seed=seed)
    eng.random_position()
    eng.find_initial_stepsize()
    for st in stages:
        eng.warmup_stage(st)
    return eng


def sbc(pkg, P, K, D, N):
    import torch
    rng = np.random.default_rng(1)
    batch = pkg.ProblemBatch([pkg.DiagNormal(rng.normal(size=D), rng.uniform(0.5, 2.0, D)) for _ in range(P)], K)
    stages = pkg.default_warmup_stages()[1:]
    out = {"problems": P, "chains_per_problem": K, "dim": D, "draws": N, "warmup": "default_warmup_stages()"}
    for case in ("draws kept on the device + dhmc_ess_rhat_problems_dev", "summary"):
        torch.cuda.synchronize()
        base = _used_bytes()
        eng = _warmed(pkg, batch, P * K, stages)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if case == "summary":
            eng.mcmc_summary(N)
        else:
            draws = torch.empty((P * K, N, D), dtype=torch.float64, device="cuda")
            eng.mcmc_dev(N, draws.data_ptr())
            eng.ess_rhat_problems_dev(draws.data_ptr(), N)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        used = _used_bytes() - base
        kernel_s = eng.last_kernel_ms() * 1e-3
        eng.close()
        if case != "summary":
            del draws
        out[case] = {"wall_s": wall, "sampling_kernel_s": kernel_s, "device_bytes_in_use": used}
    return out


def sbc_big(pkg, P, K, D, N, thin):
    import torch
    rng = np.random.default_rng(2)
    mu, s2 = rng.normal(size=(P, D)), rng.uniform(0.5, 2.0, (P, D))
    batch = pkg.ProblemBatch([pkg.DiagNormal(mu[p], s2[p]) for p in range(P)], K)
    ref = mu + np.sqrt(s2) * rng.normal(size=(P, D))
    torch.cuda.synchronize()
    base = _used_bytes()
    eng = _warmed(pkg, batch, P * K, pkg.default_warmup_stages()[1:])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    s = eng.mcmc_summary(N, thin=thin, reference=ref)
    wall = time.perf_counter() - t0
    used = _used_bytes() - base
    kernel_s = eng.last_kernel_ms() * 1e-3
    eng.close()
    draws = (N // thin) * K
    hist = np.bincount(s["rank"].ravel() * 20 // (draws + 1), minlength=20)       # 20 groups of consecutive rank values
    expected = np.bincount(np.arange(draws + 1) * 20 // (draws + 1), minlength=20) / (draws + 1) * hist.sum()
    from scipy import stats
    return {"problems": P, "chains_per_problem": K, "dim": D, "transitions": N, "thin": thin,
            "draws_if_kept_bytes": P * K * N * D * 8, "wall_s": wall, "sampling_kernel_s": kernel_s,
            "device_bytes_in_use": used, "rank_hist_20_groups": hist.tolist(), "rank_chi2_pvalue": float(stats.chisquare(hist, expected).pvalue),
            "rhat_max": float(np.nanmax(s["rhat"]))}


def c2(pkg, chains, D, N, repeats):
    import torch
    eng = _warmed(pkg, pkg.StandardNormal(D), chains, [pkg.TuningNUTS(50, pkg.DualAveraging())])
    ck = eng.checkpoint()
    n = 2
    q_host = eng.host_alloc((chains, D))
    outs = dict(posterior_matrix=eng.host_alloc((chains, n, D)),
                tree_statistics=eng.host_alloc((chains, n), dtype=pkg._lib.tree_stats_dtype),
                logdensities=eng.host_alloc((chains, n)))

    def run(case):
        eng.restore(ck)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        steps, ms = 0, 0.0
        if case == "mcmc_dev, no outputs":
            eng.mcmc_dev(N)
            steps, ms = eng.last_total_steps(), eng.last_kernel_ms()
        elif case.startswith("summary"):
            eng.mcmc_summary(N, thin=10 if "thin" in case else 1)
            steps, ms = eng.last_total_steps(), eng.last_kernel_ms()
        else:
            q_host[...] = ck["q"]
            for _ in range(N // n):
                eng.mcmc_from(q_host, n, out=outs)
                q_host[...] = outs["posterior_matrix"][:, -1]
                steps += eng.last_total_steps(); ms += eng.last_kernel_ms()
        torch.cuda.synchronize()
        return {"wall_s": time.perf_counter() - t0, "kernel_s": ms * 1e-3, "leapfrog_steps": steps,
                "leapfrog_steps_per_s": steps / (ms * 1e-3)}

    # thin = 10 folds a tenth of the draws with the same chain-end atomics: the two summary rates separate the costs
    cases = ("mcmc_dev, no outputs", "summary", "summary, thin = 10", "host draws through the e2e pipeline (mcmc_from, 2 draws per call)")
    runs = {c: [] for c in cases}
    for c in cases:                                                  # warm every path once
        run(c)
    for _ in range(repeats):
        for c in cases:
            runs[c].append(run(c))
    eng.close()
    out = {"chains": chains, "dim": D, "transitions": N, "warmup": "search + 50 dual-averaging transitions"}
    for c in cases:
        r = [x["leapfrog_steps_per_s"] for x in runs[c]]
        out[c] = {"runs": runs[c], "leapfrog_steps_per_s_min": min(r), "leapfrog_steps_per_s_max": max(r)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-sbc", action="store_true")
    ap.add_argument("--skip-big", action="store_true")
    ap.add_argument("--skip-c2", action="store_true")
    ap.add_argument("--big-problems", type=int, default=16384)
    ap.add_argument("--c2-chains", type=int, default=65536)
    ap.add_argument("--repeats", type=int, default=2)
    args = ap.parse_args()
    from __graft_entry__ import load_package
    pkg = load_package()
    line = gpu_info()
    if not args.skip_sbc:
        line["sbc_1024"] = sbc(pkg, 1024, 8, 100, 1000)
    if not args.skip_big:
        line["sbc_big"] = sbc_big(pkg, args.big_problems, 8, 100, 1000, 10)
    if not args.skip_c2:
        line["c2_n100"] = c2(pkg, args.c2_chains, 1000, 100, args.repeats)
    line["power_limit_w_after"] = gpu_info()["power_limit_w"]
    print(json.dumps(line))


if __name__ == "__main__":
    main()
