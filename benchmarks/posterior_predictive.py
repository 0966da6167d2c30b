"""Random generated quantities (posterior predictive replicates; include/dhmc_models.h, DESIGN.md §4.4): what they cost.

  (a) SBC shape of benchmarks/generated_quantities.py: 16 384 eight-schools problems (J = 8, D = 10), 8 chains each,
      default warm-up, then the streaming summary of N = 1 000 transitions at thin = 10 — with the eight_schools_ppc
      library (D + G = 30 rows: the coordinates, τ, θ_j, y_rep_j and three p-value indicators), the eight_schools_gq
      library (19 rows) and the eight_schools library (10 rows).  The handles are warmed up from one seed, so they take
      the same transitions (sampling is bit-identical; the leapfrog step counts are compared); the calls alternate from
      one checkpoint each, --repeats times.  Sampling-kernel time (device events) and wall time of the call.
  (b) plain sampling (dhmc_mcmc without outputs) with the ppc and gq libraries, alternated from one checkpoint each, for the
      k_nuts instantiations ptxas allocates differently that eight schools runs (benchmarks/posterior_predictive_ptxas.md).
  (c) dhmc_generated_keyed_dev over [10, 100, 131 072] points with their keys on the device: points / s (wall time
      around calls that end in a device synchronise).
Prints one JSON line with the GPU name and its power limit read in the same run.

    python benchmarks/posterior_predictive.py [--problems 16384] [--repeats 3]
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
from generated_quantities import _batch  # noqa: E402
from problem_batch import gpu_info  # noqa: E402
from streaming_summary import _used_bytes, _warmed  # noqa: E402

MODELS = os.path.join(ROOT, "include", "models")


def summary(pkg, P, K, N, thin, repeats):
    import torch
    libs = {"eight_schools_ppc": (os.path.join(MODELS, "eight_schools_ppc.h"), True),
            "eight_schools_gq": (os.path.join(MODELS, "eight_schools_gq.h"), True),
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
    assert len(same) == 1, f"the libraries took different transitions: leapfrog steps {sorted(same)}"
    out["same_transitions"] = True
    for name, (eng, _) in engs.items():
        eng.close()
    return out


def plain_sampling(pkg, P, K, N, repeats):
    """plain sampling (dhmc_mcmc, no outputs, no summary) with the ppc and gq libraries, whose k_nuts instantiations ptxas
    allocates differently (benchmarks/posterior_predictive_ptxas.md): the kernel eight schools runs (32 threads per chain,
    one element per thread) and its deep twin (max_depth 14)"""
    out = {"problems": P, "chains_per_problem": K, "dim": 10, "transitions": N}
    for label, kw in (("k_nuts<1, 4, 1, false, 1, false>", dict(threads_per_chain=32)),
                      ("k_nuts<1, 4, 1, false, 1, true>", dict(threads_per_chain=32, algorithm=pkg.NUTS(max_depth=14)))):
        engs, res = {}, {}
        for name in ("eight_schools_ppc", "eight_schools_gq"):
            eng = pkg.Engine(_batch(pkg, os.path.join(MODELS, name + ".h"), P, K, True), chains=P * K, seed=5, **kw)
            eng.random_position()
            eng.set_stepsize(0.3)
            eng._ck(eng._lib.dhmc_mcmc(eng._h, 20, None, None, None))          # warm
            engs[name], res[name] = (eng, eng.checkpoint()), []
        for _ in range(repeats):
            for name, (eng, ck) in engs.items():
                eng.restore(ck)
                eng._ck(eng._lib.dhmc_mcmc(eng._h, N, None, None, None))
                res[name].append((eng.last_kernel_ms() * 1e-3, eng.last_total_steps()))
        steps = {s for r in res.values() for _, s in r}
        assert len(steps) == 1, f"{label}: different transitions {sorted(steps)}"
        out[label] = {name: {"sampling_kernel_s": [t for t, _ in r], "leapfrog_steps": r[0][1]} for name, r in res.items()}
        for eng, _ in engs.values():
            eng.close()
    return out


def generated_keyed_dev(pkg, P, K, n_keep, repeats):
    import torch
    ℓ = _batch(pkg, os.path.join(MODELS, "eight_schools_ppc.h"), P, K, True)
    eng = pkg.Engine(ℓ, chains=P * K, seed=1)
    try:
        G = eng.generated_count
        theta = torch.randn((P * K, n_keep, 10), dtype=torch.float64, device="cuda")    # column-major [D, n_keep, B]
        out = torch.empty((P * K, n_keep, G), dtype=torch.float64, device="cuda")
        ch, tr = eng.draw_keys(0, n_keep * 10, thin=10)
        chain = torch.from_numpy(ch).cuda()
        trans = torch.from_numpy(tr.view(np.int32)).cuda()
        args = (eng._h, C.c_void_p(theta.data_ptr()), K * n_keep, 0, P, C.c_void_p(chain.data_ptr()),
                C.c_void_p(trans.data_ptr()), C.c_void_p(out.data_ptr()))
        eng._ck(eng._lib.dhmc_generated_keyed_dev(*args))              # warm
        times = []
        for _ in range(repeats):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            eng._ck(eng._lib.dhmc_generated_keyed_dev(*args))          # ends in a stream synchronise
            times.append(time.perf_counter() - t0)
        pts = P * K * n_keep
        return {"points": pts, "dim": 10, "generated": G, "wall_s": times, "points_per_s_max": pts / min(times),
                "bytes_per_point": 8 * (10 + G) + 12}
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
    line["plain_sampling"] = plain_sampling(pkg, 2048, 8, 400, args.repeats)
    line["generated_keyed_dev"] = generated_keyed_dev(pkg, args.problems, 8, 100, 5)
    line["power_limit_w_after"] = gpu_info()["power_limit_w"]
    print(json.dumps(line))


if __name__ == "__main__":
    main()
