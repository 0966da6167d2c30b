"""Ragged problem batches (dhmc_set_problems_ragged, DESIGN.md §4.3): "one fit per unit" — P logistic regressions whose
number of observations N_p differs from problem to problem — on one handle, against the equal-N workaround.

Shape: P = 512 problems, p = 32 coefficients, K = 8 chains each; N_p log-uniform on [32, 4096) (fixed seed), X and y drawn
like LogisticRegression.synthetic; default warm-up, then --draws transitions kept on the device (mcmc_dev).  Three cases,
interleaved over --repeats runs, each reporting the range of its figures:
  (a) the ragged batch in the given order;
  (b) the same ragged batch with the problems sorted by decreasing N_p — whether it beats (a) shows whether the lock-step
      group queue suffers a tail on ragged work;
  (c) the equal-N workaround: a ProblemBatch with every problem zero-padded to max N_p (same ∇ℓ, ℓ shifted by a constant).
Per case: wall time of the whole fit (handle creation to the last draw on the device), leapfrog steps / s of the sampling
kernel (last_total_steps / last_kernel_ms), useful observation rows / s (Σ over chains of leapfrog steps × N_p of the
chain's own problem over the sampling kernel's time: padding rows do not count) and the logistic device bytes computed
from the shapes (X, Xᵀ, y, padded X).  Prints one JSON line with the GPU name and its power limit read in the same run.

    python benchmarks/ragged_batch.py [--problems 512] [--draws 1000] [--repeats 3]
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


def units(pkg, P, p, seed):
    """P logistic regressions with N_p log-uniform on [32, 4096), data as LogisticRegression.synthetic."""
    rng = np.random.default_rng(seed)
    Ns = np.floor(np.exp(rng.uniform(np.log(32), np.log(4096), P))).astype(int)
    Ns = np.clip(Ns, 32, 4095)
    return [pkg.LogisticRegression.synthetic(N=int(n), p=p, seed=seed + 1 + i)[0] for i, n in enumerate(Ns)]


def padded(pkg, ℓ, n_max):
    """the equal-N workaround: zero rows of X (and y = 0) up to n_max — ∇ℓ unchanged, ℓ shifted by a constant"""
    N = ℓ.X.shape[0]
    X = np.zeros((n_max, ℓ.X.shape[1])); X[:N] = ℓ.X
    y = np.zeros(n_max); y[:N] = ℓ.y
    return pkg.LogisticRegression(X, y)


def tma_xs(D):
    w = (D + 7) & ~7
    while (w & 15) != 4:
        w += 1
    return w


def device_bytes(Ns, D, packed=True):
    """X [N][D], Xᵀ [D][ld], y [N] and (packed chain groups) padded X [⌈N/32⌉·32][tma_xs(D)] of every problem"""
    Ns = np.asarray(Ns, dtype=np.int64)
    ld = (Ns + 1) & ~1
    rows = (Ns + 31) // 32 * 32
    return int(8 * (Ns * D + ld * D + Ns + (rows * tma_xs(D) if packed else 0)).sum())


def fit(pkg, batch, chains, draws_n, D):
    import torch
    draws = torch.empty((chains, draws_n, D), dtype=torch.float64, device="cuda")
    stats = torch.empty((chains, draws_n, pkg._lib.tree_stats_dtype.itemsize), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    eng = pkg.Engine(batch, chains=chains, seed=2026)
    eng.random_position(); eng.find_initial_stepsize()
    for st in pkg.default_warmup_stages()[1:]:
        eng.warmup_stage(st)
    eng.mcmc_dev(draws_n, draws.data_ptr(), stats.data_ptr(), 0)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    steps, ms = eng.last_total_steps(), eng.last_kernel_ms()
    eng.close()
    st = stats.cpu().numpy().reshape(-1).view(pkg._lib.tree_stats_dtype).reshape(chains, draws_n)
    return wall, steps, ms, st["steps"].sum(axis=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--problems", type=int, default=512)
    ap.add_argument("--chains-per-problem", type=int, default=8)
    ap.add_argument("--dim", type=int, default=32)
    ap.add_argument("--draws", type=int, default=1000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--seed", type=int, default=11)
    args = ap.parse_args()
    from __graft_entry__ import load_package
    pkg = load_package()
    line = gpu_info()
    P, K, D = args.problems, args.chains_per_problem, args.dim
    probs = units(pkg, P, D, args.seed)
    Ns = np.array([ℓ.X.shape[0] for ℓ in probs])
    order = np.argsort(-Ns, kind="stable")
    n_max = int(Ns.max())
    cases = [("(a) ragged, given order", lambda: pkg.RaggedProblemBatch(probs, K), Ns),
             ("(b) ragged, largest N first", lambda: pkg.RaggedProblemBatch([probs[i] for i in order], K), Ns[order]),
             ("(c) equal-N workaround, zero-padded to max N", lambda: pkg.ProblemBatch([padded(pkg, ℓ, n_max) for ℓ in probs], K),
              Ns)]
    fit(pkg, pkg.RaggedProblemBatch(probs[:8], K), 8 * K, 10, D)      # load the library and the kernels
    res = {label: [] for label, _, _ in cases}
    for _ in range(args.repeats):                                    # interleaved: drifts of the card hit every case alike
        for label, make, n_of_problem in cases:
            wall, steps, ms, chain_steps = fit(pkg, make(), P * K, args.draws, D)
            useful = float((chain_steps * np.repeat(n_of_problem, K)).sum())
            res[label].append(dict(wall_s=wall, steps_per_s=steps / (ms * 1e-3), useful_rows_per_s=useful / (ms * 1e-3),
                                   kernel_ms=ms, leapfrog_steps=steps))
            print(json.dumps({"case": label, **res[label][-1]}), file=sys.stderr, flush=True)   # progress
    out = []
    for label, _, _ in cases:
        runs = res[label]
        row = {"case": label,
               "device_bytes": device_bytes([n_max] * P if label.startswith("(c)") else Ns, D)}
        for k in ("wall_s", "steps_per_s", "useful_rows_per_s"):
            v = [r[k] for r in runs]
            row[k] = {"min": min(v), "max": max(v), "median": float(np.median(v))}
        row["leapfrog_steps"] = [r["leapfrog_steps"] for r in runs]
        out.append(row)
    line.update(problems=P, chains_per_problem=K, dim=D, draws=args.draws, warmup="default_warmup_stages()",
                N_min=int(Ns.min()), N_max=n_max, N_mean=float(Ns.mean()), N_sum=int(Ns.sum()),
                draws_note="as specified" if args.draws == 1000 else f"reduced to {args.draws} draws (default 1000)",
                cases=out)
    line["power_limit_w_after"] = gpu_info()["power_limit_w"]
    print(json.dumps(line))


if __name__ == "__main__":
    main()
