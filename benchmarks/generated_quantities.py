"""Generated quantities (include/dhmc_models.h, DESIGN.md §4.4): what the per-draw evaluation and its fold cost.

  (a) SBC shape: 16 384 eight-schools problems (J = 8, D = 10), 8 chains each, default warm-up, then the streaming summary
      of N = 1 000 transitions at thin = 10 — once with the eight_schools_gq library (D + G = 19 rows: the 10 coordinates
      and τ, θ₁…θ₈) and once with the eight_schools library (10 rows).  Both handles are warmed up from one seed, so they
      take the same transitions (sampling is bit-identical); the calls alternate from one checkpoint each, --repeats times.
      Sampling-kernel time (device events), wall time of the call, and the device memory the handle and its summary arena
      hold.
  (b) dhmc_generated_dev over a kept-draws buffer of that shape, [D, 100, 131 072] on the device: points / s (wall time
      around calls that end in a device synchronise).
Prints one JSON line with the GPU name and its power limit read in the same run.

    python benchmarks/generated_quantities.py [--problems 16384] [--repeats 3]
"""
import argparse
import ctypes as C
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

MODELS = os.path.join(ROOT, "include", "models")
Y0 = np.array([28.0, 8, -3, 7, -1, 1, 18, 12])
S0 = np.array([15.0, 10, 16, 11, 9, 11, 10, 18])


def _batch(pkg, header, P, K, deep):
    rng = np.random.default_rng(3)
    lib = pkg.compile_user_model(header, deep=deep)
    return pkg.ProblemBatch([pkg.UserLogDensity(header, 10, library=lib, params=np.concatenate(
        [Y0 + rng.normal(size=8) * 5, S0 * rng.uniform(0.7, 1.3, 8)])) for _ in range(P)], K)


def summary(pkg, P, K, N, thin, repeats):
    import torch
    libs = {"eight_schools_gq": (os.path.join(MODELS, "eight_schools_gq.h"), True),
            "eight_schools": (os.path.join(MODELS, "eight_schools.h"), False)}
    engs, out = {}, {"problems": P, "chains_per_problem": K, "dim": 10, "transitions": N, "thin": thin,
                     "warmup": "default_warmup_stages()"}
    for name, (hdr, deep) in libs.items():
        torch.cuda.synchronize()
        base = _used_bytes()
        eng = _warmed(pkg, _batch(pkg, hdr, P, K, deep), P * K, pkg.default_warmup_stages()[1:])
        ck = eng.checkpoint()
        s = eng.mcmc_summary(N, thin=thin)                            # grows the arena; warms the path
        torch.cuda.synchronize()
        out[name] = {"rows": int(s["mean"].shape[1]), "device_bytes_handle_and_arena": _used_bytes() - base, "runs": []}
        engs[name] = (eng, ck)
    for _ in range(repeats):
        for name, (eng, ck) in engs.items():
            eng.restore(ck)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            eng.mcmc_summary(N, thin=thin)
            wall = time.perf_counter() - t0
            out[name]["runs"].append({"wall_s": wall, "sampling_kernel_s": eng.last_kernel_ms() * 1e-3,
                                      "leapfrog_steps": eng.last_total_steps()})
    for name in engs:
        r = out[name]["runs"]
        out[name]["sampling_kernel_s_min"] = min(x["sampling_kernel_s"] for x in r)
        out[name]["wall_s_min"] = min(x["wall_s"] for x in r)
    same = {x["leapfrog_steps"] for name in engs for x in out[name]["runs"]}
    out["same_transitions"] = len(same) == 1
    for name, (eng, _) in engs.items():
        eng.close()
    return out


def generated_dev(pkg, P, K, n_keep, repeats):
    import torch
    ℓ = _batch(pkg, os.path.join(MODELS, "eight_schools_gq.h"), P, K, True)
    eng = pkg.Engine(ℓ, chains=P * K, seed=1)
    try:
        G = eng.generated_count
        theta = torch.randn((P * K, n_keep, 10), dtype=torch.float64, device="cuda")    # column-major [D, n_keep, B]
        out = torch.empty((P * K, n_keep, G), dtype=torch.float64, device="cuda")
        args = (eng._h, C.c_void_p(theta.data_ptr()), K * n_keep, 0, P, C.c_void_p(out.data_ptr()))
        eng._ck(eng._lib.dhmc_generated_dev(*args))                    # warm
        times = []
        for _ in range(repeats):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            eng._ck(eng._lib.dhmc_generated_dev(*args))                # ends in a stream synchronise
            times.append(time.perf_counter() - t0)
        pts = P * K * n_keep
        return {"points": pts, "dim": 10, "generated": G, "wall_s": times, "points_per_s_max": pts / min(times),
                "bytes_per_point": 8 * (10 + G)}
    finally:
        eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--problems", type=int, default=16384)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--skip-summary", action="store_true")
    args = ap.parse_args()
    from __graft_entry__ import load_package
    pkg = load_package()
    line = gpu_info()
    if not args.skip_summary:
        line["sbc_summary"] = summary(pkg, args.problems, 8, 1000, 10, args.repeats)
    line["generated_dev"] = generated_dev(pkg, args.problems, 8, 100, 5)
    line["power_limit_w_after"] = gpu_info()["power_limit_w"]
    print(json.dumps(line))


if __name__ == "__main__":
    main()
