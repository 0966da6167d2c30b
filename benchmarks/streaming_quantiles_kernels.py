"""Leapfrog-steps/s of the five k_nuts instantiations whose spills the quantile histograms changed
(benchmarks/streaming_quantiles_ptxas.md), in plain sampling (mcmc_dev, no summary).  Run it once per build and alternate
the builds in one call to compare them:

    python benchmarks/streaming_quantiles_kernels.py [PACKAGE_ROOT]

PACKAGE_ROOT is a checkout whose library is built (default: this one).  Prints a JSON line with the GPU name and its
power limit, then one line per case as it finishes.  Each case pins the layout with threads_per_chain, so the handle runs exactly the named instantiation
(tests/test_kernel_coverage.py handle_layout restates the host's choice)."""
import importlib.util
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from problem_batch import gpu_info  # noqa: E402

# name: (family, D, threads_per_chain, max_depth, dense, chains)
CASES = {
    "k_nuts<8, 0, 8, true, 1, false>": ("std", 1500, 256, 10, True, 128),
    "k_nuts<32, 1, 8, true, 1, false>": ("diag", 5000, 256, 10, True, 16),
    "k_nuts<32, 2, 8, true, 1, false>": ("funnel", 5000, 256, 10, True, 16),
    "k_nuts<32, 3, 8, true, 1, false>": ("logistic", 5000, 256, 10, True, 16),
    "k_nuts<4, 2, 8, false, 1, true>": ("funnel", 1000, 256, 14, False, 1024),
    "k_nuts<8, 2, 4, true, 1, true>": ("funnel", 1000, 128, 14, True, 512),
    "k_nuts<8, 3, 4, true, 1, true>": ("logistic", 1000, 128, 14, True, 512),
}


def load(root):
    pkg_dir = os.path.join(root, "dynamichmc.jl_b200")
    spec = importlib.util.spec_from_file_location("dynamichmc_jl_b200", os.path.join(pkg_dir, "__init__.py"),
                                                  submodule_search_locations=[pkg_dir])
    mod = importlib.util.module_from_spec(spec)
    sys.modules[spec.name] = mod
    spec.loader.exec_module(mod)
    return mod


def rate(pkg, fam, D, T, md, dense, K, calls=2, N=6):
    ℓ = {"std": lambda: pkg.StandardNormal(D), "funnel": lambda: pkg.Funnel(D),
         "diag": lambda: pkg.DiagNormal(np.zeros(D), np.linspace(0.5, 2.0, D)),
         "logistic": lambda: pkg.LogisticRegression.synthetic(N=400, p=D, seed=3)[0]}[fam]()
    eng = pkg.Engine(ℓ, chains=K, seed=11, algorithm=pkg.NUTS(max_depth=md), threads_per_chain=T)
    try:
        eng.random_position()
        eng.find_initial_stepsize()
        if dense:
            eng.set_metric_dense(np.eye(D))
        eng.mcmc_dev(N)                                        # warm-up call
        out = []
        for _ in range(calls):
            eng.mcmc_dev(N)
            out.append(eng.last_total_steps() / (eng.last_kernel_ms() * 1e-3))
        return {"layout": list(eng.layout()), "leapfrog_steps_per_s": out}
    finally:
        eng.close()


def main():
    root = os.path.abspath(sys.argv[1] if len(sys.argv) > 1 else os.path.dirname(HERE))
    pkg = load(root)
    line = gpu_info()
    line["root"] = root
    print(json.dumps(line), flush=True)
    for name, case in CASES.items():
        print(json.dumps({"kernel": name, **rate(pkg, *case)}), flush=True)


if __name__ == "__main__":
    main()
