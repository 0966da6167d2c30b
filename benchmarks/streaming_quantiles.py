"""Streaming quantiles (dhmc_mcmc_summary_histogram, DESIGN.md §4.4) against the plain streaming summary.

  (a) C2 shape (65 536 chains, D = 1 000, search + 50 dual-averaging transitions) at N = 100: the summary and the summary
      with 256-bin histograms on the grid (−6, 6) of every parameter, at thin = 1 and thin = 10, run alternately
      --repeats times.  Leapfrog steps / s of the sampling kernel (device events) and wall time including the finish (the
      record, and with histograms their download and the quantiles).  Thin = 10 keeps the chain-end fold (one staging
      read and the histogram atomics of one 65 536-chain problem) and does a tenth of the per-draw staging updates, so the
      two differences separate the costs.  An accuracy line for α = 0.05, 0.5, 0.95: max over d of |q − Φ⁻¹(α)| and the
      mean bracket width.
  (b) SBC at 16 384 problems (D = 100, 8 chains each, default warm-up, N = 1 000, thin = 10, the shape of
      benchmarks/streaming_summary.py), the summary with quantiles at 64 and at 256 bins on a grid of ±6 posterior sd:
      wall time of the sampling call and device memory in use when it returns.
Prints one JSON line with the GPU name and its power limit read in the same run.

    python benchmarks/streaming_quantiles.py [--skip-c2] [--skip-sbc] [--repeats 2]
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
from streaming_summary import _used_bytes, _warmed  # noqa: E402

PROBS = (0.05, 0.5, 0.95)


def c2(pkg, chains, D, N, repeats, bins):
    import torch
    from scipy import stats
    eng = _warmed(pkg, pkg.StandardNormal(D), chains, [pkg.TuningNUTS(50, pkg.DualAveraging())])
    ck = eng.checkpoint()
    grid = (np.full((1, D), -6.0), np.full((1, D), 6.0))
    last = {}

    def run(case):
        thin = 10 if "thin = 10" in case else 1
        kw = dict(quantiles=PROBS, grid=grid, bins=bins) if "histogram" in case else {}
        eng.restore(ck)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = eng.mcmc_summary(N, thin=thin, **kw)
        wall = time.perf_counter() - t0
        steps, ms = eng.last_total_steps(), eng.last_kernel_ms()
        last[case] = out
        return {"wall_s": wall, "kernel_s": ms * 1e-3, "leapfrog_steps": steps, "leapfrog_steps_per_s": steps / (ms * 1e-3)}

    cases = ("summary, thin = 1", f"summary + {bins}-bin histogram, thin = 1", "summary, thin = 10",
             f"summary + {bins}-bin histogram, thin = 10")
    runs = {c: [] for c in cases}
    for c in cases:                                                  # warm every path once
        run(c)
    for _ in range(repeats):
        for c in cases:
            runs[c].append(run(c))
    eng.close()
    out = {"chains": chains, "dim": D, "transitions": N, "bins": bins, "grid": "(-6, 6)",
           "warmup": "search + 50 dual-averaging transitions"}
    for c in cases:
        r = [x["leapfrog_steps_per_s"] for x in runs[c]]
        k = [x["kernel_s"] for x in runs[c]]
        w = [x["wall_s"] for x in runs[c]]
        out[c] = {"runs": runs[c], "leapfrog_steps_per_s_min": min(r), "leapfrog_steps_per_s_max": max(r),
                  "kernel_s_min": min(k), "wall_s_min": min(w)}
    for thin in (1, 10):                                             # measured differences, same transitions and draws
        plain, hist = out[f"summary, thin = {thin}"], out[f"summary + {bins}-bin histogram, thin = {thin}"]
        out[f"histogram cost, thin = {thin}"] = {"kernel_s_min_difference": hist["kernel_s_min"] - plain["kernel_s_min"],
                                                 "wall_s_min_difference": hist["wall_s_min"] - plain["wall_s_min"]}
    for thin in (1, 10):
        s = last[f"summary + {bins}-bin histogram, thin = {thin}"]
        acc = {}
        for i, a in enumerate(PROBS):
            q, lo, hi = s["quantile"][0, :, i], s["quantile_lo"][0, :, i], s["quantile_hi"][0, :, i]
            acc[str(a)] = {"max_abs_error": float(np.max(np.abs(q - stats.norm.ppf(a)))),
                           "mean_bracket_width": float(np.mean(hi - lo))}
        out[f"accuracy, thin = {thin}"] = {"draws_per_parameter": int(s["draws"][0, 0]),
                                           "tail_count": int(s["histogram"][..., [0, -1]].sum()), "quantiles": acc}
    return out


def sbc_quantiles(pkg, P, K, D, N, thin, bins_list):
    import torch
    rng = np.random.default_rng(2)
    mu, s2 = rng.normal(size=(P, D)), rng.uniform(0.5, 2.0, (P, D))
    batch = pkg.ProblemBatch([pkg.DiagNormal(mu[p], s2[p]) for p in range(P)], K)
    grid = (mu - 6.0 * np.sqrt(s2), mu + 6.0 * np.sqrt(s2))
    out = {"problems": P, "chains_per_problem": K, "dim": D, "transitions": N, "thin": thin,
           "grid": "posterior mean ± 6 sd", "warmup": "default_warmup_stages()"}
    for bins in bins_list:
        torch.cuda.synchronize()
        base = _used_bytes()
        eng = _warmed(pkg, batch, P * K, pkg.default_warmup_stages()[1:])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        s = eng.mcmc_summary(N, thin=thin, quantiles=PROBS, grid=grid, bins=bins)
        wall = time.perf_counter() - t0
        used = _used_bytes() - base
        kernel_s = eng.last_kernel_ms() * 1e-3
        eng.close()
        z = (s["quantile"][..., 1] - mu) / np.sqrt(s2)
        out[f"{bins} bins"] = {"wall_s": wall, "sampling_kernel_s": kernel_s, "device_bytes_in_use": used,
                               "median_z_abs_mean": float(np.mean(np.abs(z))),
                               "tail_fraction": float(s["histogram"][..., [0, -1]].sum() / s["histogram"].sum())}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-c2", action="store_true")
    ap.add_argument("--skip-sbc", action="store_true")
    ap.add_argument("--c2-chains", type=int, default=65536)
    ap.add_argument("--sbc-problems", type=int, default=16384)
    ap.add_argument("--repeats", type=int, default=2)
    args = ap.parse_args()
    from __graft_entry__ import load_package
    pkg = load_package()
    line = gpu_info()
    if not args.skip_c2:
        line["c2_n100"] = c2(pkg, args.c2_chains, 1000, 100, args.repeats, 256)
    if not args.skip_sbc:
        line["sbc_big_quantiles"] = sbc_quantiles(pkg, args.sbc_problems, 8, 100, 1000, 10, (64, 256))
    line["power_limit_w_after"] = gpu_info()["power_limit_w"]
    print(json.dumps(line))


if __name__ == "__main__":
    main()
