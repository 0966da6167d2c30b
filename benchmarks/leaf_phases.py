"""Where a leaf of the NUTS tree spends its cycles: the bench's C2 workload (1000-dim standard normal, diagonal per-chain M⁻¹)
on the library built with -DDHMC_PHASE_CLOCKS, whose k_nuts lets thread 0 of every CTA add clock64() deltas per phase
(nuts_machine.cuh, kPh*).  Prints SM cycles per leaf by phase, summed over all CTAs and divided by the leaves they built.

    python benchmarks/leaf_phases.py [--chains 16384] [--draws 4] [--json OUT]

The profiled library is built with `make -C dynamichmc.jl_b200/csrc prof` (into csrc/build_prof/, apart from the shipped
library) unless it is already there.  The numbers are thread 0's view: time it waits at a barrier for the other warps of its
chain is charged to the phase that holds the barrier.  The clock reads and counter updates add a few instructions per
phase, so the profiled kernel is a little slower than the shipped one; compare profiles with each other, not with bench.py."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dynamichmc.jl_b200", "csrc")
PHASES = ["leapfrog elementwise", "leapfrog all-reduce", "merge checks: slot loads + arithmetic", "merge checks: all-reduce",
          "scalar control", "push stores", "transition level (draw, doubling, output)"]


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--chains", type=int, default=16384)
    ap.add_argument("--draws", type=int, default=4)
    ap.add_argument("--adapt-steps", type=int, default=60, help="dual-averaging warm-up transitions (bench.py's C2 default)")
    ap.add_argument("--lib", default=os.path.join(CSRC, "build_prof", "libdhmc_b200_prof.so"))
    ap.add_argument("--json", default=None, help="also write the table as JSON here")
    args = ap.parse_args()
    if not os.path.exists(args.lib):
        subprocess.check_call(["make", "-C", CSRC, "-j%d" % max(1, min(10, os.cpu_count() or 1)), "prof",
                               "PROF_BUILD=" + os.path.dirname(os.path.abspath(args.lib))])
    os.environ["DHMC_B200_LIB"] = os.path.abspath(args.lib)
    sys.path.insert(0, ROOT)
    import __graft_entry__ as entry
    pkg = entry.load_package()
    so = pkg._lib.lib()
    if not hasattr(so, "dhmc_phase_clocks"):
        sys.exit(f"{args.lib} is not a -DDHMC_PHASE_CLOCKS build")
    so.dhmc_phase_clocks.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.c_int]

    eng = pkg.Engine(pkg.StandardNormal(1000), chains=args.chains, seed=2026)
    counters = (C.c_uint64 * (len(PHASES) + 1))()
    eng.random_position()
    eng.find_initial_stepsize()
    eng.warmup_stage(pkg.TuningNUTS(args.adapt_steps, pkg.DualAveraging()))
    eng.mcmc(1, keep_draws=False)                                   # a sampling call as warm-up of the measured one
    assert so.dhmc_phase_clocks(eng._h, counters, 1) == 0           # start from zero
    eng.mcmc(args.draws, keep_draws=False)
    steps = eng.last_total_steps()
    assert so.dhmc_phase_clocks(eng._h, counters, 0) == 0
    eng.close()

    cyc, leaves = [int(counters[k]) for k in range(len(PHASES))], int(counters[len(PHASES)])
    total = sum(cyc)
    rows = [dict(phase=name, cycles_per_leaf=c / leaves, share=c / total) for name, c in zip(PHASES, cyc)]
    print(f"C2 shape: D=1000, {args.chains} chains, {args.draws} draws after {args.adapt_steps} dual-averaging transitions; "
          f"{leaves} leaves ({steps} leapfrog steps reported)")
    print("| phase | cycles per leaf | share |")
    print("|---|---|---|")
    for r in rows:
        print(f"| {r['phase']} | {r['cycles_per_leaf']:.0f} | {100 * r['share']:.1f} % |")
    print(f"| total | {total / leaves:.0f} | |")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(chains=args.chains, draws=args.draws, leaves=leaves, steps=steps, rows=rows,
                           cycles_per_leaf=total / leaves), f, indent=1)


if __name__ == "__main__":
    main()
