"""The C-ABI library loads without a GPU and exports every symbol include/dhmc.h declares."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "dhmc.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(dhmc_[a-z_]+)\s*\(", src)))


def test_header_symbols_are_exported(pkg):
    lib = pkg._lib.lib()
    names = _declared()
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), f"{n} declared in dhmc.h but not exported"
    assert sorted(pkg._lib.EXPORTS) == names


def test_struct_layouts_match_header(pkg):
    assert pkg._lib.tree_stats_dtype.itemsize == 56          # TreeStatisticsNUTS, NUTS.jl:208-221
    assert ctypes.sizeof(pkg._lib.Config) == 64
    assert ctypes.sizeof(pkg._lib.DualAveragingC) == 32


def test_argument_checks_without_gpu(pkg):
    # @argcheck mirrors run before any CUDA call
    with pytest.raises(pkg.ArgumentError):
        pkg.NUTS(max_depth=0)
    with pytest.raises(pkg.ArgumentError):
        pkg.NUTS(min_Δ=1.0)
    with pytest.raises(pkg.ArgumentError):
        pkg.DualAveraging(δ=1.5)
    with pytest.raises(pkg.ArgumentError):
        pkg.InitialStepsizeSearch(maxiter_crossing=2)
    with pytest.raises(pkg.ArgumentError):
        pkg.TuningNUTS(10)
    st = pkg.default_warmup_stages()
    assert isinstance(st[0], pkg.InitialStepsizeSearch)
    assert [s.N for s in st[1:]] == [75, 25, 50, 100, 200, 400, 50]
    assert [s.M for s in st[1:]] == [None] + [pkg.Diagonal] * 5 + [None]
    assert [s.N for s in pkg.fixed_stepsize_warmup_stages()] == [25, 50, 100, 200, 400]


def test_fails_loudly_without_cuda(pkg):
    import torch
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        pkg.Engine(pkg.StandardNormal(10), chains=4)


def test_device_models_match_oracle_models(pkg, po):
    import numpy as np
    rng = np.random.default_rng(0)
    q = rng.normal(size=10)
    for ℓ, fam, params in ((pkg.StandardNormal(10), 0, None),
                           (pkg.DiagNormal(rng.normal(size=10), rng.uniform(0.5, 2, 10)), 1, "p"),
                           (pkg.Funnel(10), 2, None),
                           (pkg.LogisticRegression(rng.normal(size=(30, 10)), (rng.uniform(size=30) < 0.5) * 1.0), 3, "p")):
        pr = ℓ.params() if params else None
        lq, g = po.logdensity_and_gradient(fam, q, pr)
        lq2, g2 = ℓ.logdensity_and_gradient(q)
        assert lq == pytest.approx(lq2, rel=1e-13) and np.allclose(g, g2, rtol=1e-13)


def _split_top_level(argstr):
    out, depth, cur = [], 0, ""
    for ch in argstr:
        if ch in "([{":
            depth += 1
        elif ch in ")]}":
            depth -= 1
        if ch == "," and depth == 0:
            out.append(cur)
            cur = ""
        else:
            cur += ch
    if cur.strip():
        out.append(cur)
    return out


def _call_sites(text, start=0):
    """(name, n_args, has_star) for every `dhmc_xxx(` call in Python source text."""
    for m in re.finditer(r"\.(dhmc_[a-z_]+)\(", text):
        i, depth = m.end(), 1
        while depth:
            depth += {"(": 1, ")": -1}.get(text[i], 0)
            i += 1
        args = _split_top_level(text[m.end():i - 1])
        yield m.group(1), len(args), any(a.strip().startswith("*") for a in args)


def test_python_call_sites_pass_the_declared_number_of_arguments():
    """ctypes does not check arity for undeclared argtypes: every call of the C ABI from the host
    mirror must pass exactly as many arguments as the prototype in include/dhmc.h has."""
    src = open(os.path.join(ROOT, "include", "dhmc.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    protos = {}
    for m in re.finditer(r"\b(dhmc_[a-z_]+)\s*\(([^;{]*?)\)\s*;", src, flags=re.S):
        params = [p for p in _split_top_level(m.group(2)) if p.strip() and p.strip() != "void"]
        protos[m.group(1)] = len(params)
    assert len(protos) >= 20
    seen = set()
    for rel in ("dynamichmc.jl_b200/api.py", "dynamichmc.jl_b200/_lib.py", "dynamichmc.jl_b200/parallel.py",
                "dynamichmc.jl_b200/diagnostics.py", "bench.py", "__graft_entry__.py"):
        text = open(os.path.join(ROOT, rel)).read()
        for name, n, star in _call_sites(text):
            if name not in protos:
                continue
            seen.add(name)
            if not star:                                   # get_state(*args) is checked at run time
                assert n == protos[name], f"{rel}: {name} called with {n} arguments, prototype has {protos[name]}"
    assert len(seen) >= 20


def test_julia_shim_ccall_signatures_match_the_header():
    """julia/B200HMC.jl cannot be executed in this image; at least its ccall type tuples must have
    the arity of the prototypes they bind (and every argument list must match its type tuple)."""
    src = open(os.path.join(ROOT, "include", "dhmc.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    protos = {}
    for m in re.finditer(r"\b(dhmc_[a-z_]+)\s*\(([^;{]*?)\)\s*;", src, flags=re.S):
        protos[m.group(1)] = len([p for p in _split_top_level(m.group(2)) if p.strip() and p.strip() != "void"])
    jl = open(os.path.join(ROOT, "julia", "B200HMC.jl")).read()
    jl = re.sub(r"#[^\n]*", "", jl)                        # drop comments
    n = 0
    for m in re.finditer(r"ccall\(\(:(dhmc_[a-z_]+),\s*LIB\)\s*,", jl):
        i, depth = m.end(), 1
        while depth:
            depth += {"(": 1, ")": -1}.get(jl[i], 0)
            i += 1
        parts = _split_top_level(jl[m.end():i - 1])        # [rettype, (argtypes...), args...]
        types = parts[1].strip()
        assert types.startswith("(") and types.endswith(")"), (m.group(1), types)
        ntypes = len([t for t in _split_top_level(types[1:-1]) if t.strip()])
        assert m.group(1) in protos, f"{m.group(1)} is not declared in dhmc.h"
        assert ntypes == protos[m.group(1)], f"{m.group(1)}: {ntypes} ccall types, prototype has {protos[m.group(1)]}"
        assert len(parts) - 2 == ntypes, f"{m.group(1)}: {len(parts) - 2} arguments for {ntypes} types"
        n += 1
    assert n >= 10


def test_julia_shim_passes_the_chain_count_to_chain_status():
    """Round-1 defect: `_throw` called chain_status(ptr) with a default K = 0, so failed_chains was always empty.
    Every call (and the definition) must carry the chain count, and the error path must forward it."""
    jl = open(os.path.join(ROOT, "julia", "B200HMC.jl")).read()
    jl = re.sub(r"#[^\n]*", "", jl)
    calls = re.findall(r"chain_status\(([^()]*)\)", jl)
    assert len(calls) >= 2
    for c in calls:
        assert len(_split_top_level(c)) == 2, f"chain_status({c}): expected (ptr, K)"
    assert "K = 0" not in jl and re.search(r"_ck\(h::Handle, rc\).*h\.K", jl)
    # the dense metric is returned as Symmetric(M⁻¹) when the handle is dense, the reference API surface is present
    for needle in ("dhmc_metric_is_dense", "dhmc_get_metric_dense", "Symmetric(M", "function mcmc_keep_warmup", "mcmc_steps(",
                   "function mcmc_next_step", "reporter"):
        assert needle in jl, needle


def test_chain_status_bits_match_header(pkg):
    """The status bits the Python and Julia shims map to exceptions are the header's."""
    src = open(os.path.join(ROOT, "include", "dhmc.h")).read()
    bits = {m.group(1): int(m.group(2)) for m in re.finditer(r"\b(DHMC_CHAIN_[A-Z_]+)\s*=\s*(\d+)", src)}
    assert bits["DHMC_CHAIN_NONFINITE_Q"] == pkg._lib.DHMC_CHAIN_NONFINITE_Q
    assert bits["DHMC_CHAIN_BAD_INITIAL"] == pkg._lib.DHMC_CHAIN_BAD_INITIAL
    assert bits["DHMC_CHAIN_LEAPFROG_NONFINITE"] == pkg._lib.DHMC_CHAIN_LEAPFROG_NONFINITE
    assert sorted(bits.values()) == [1 << i for i in range(len(bits))]      # distinct single bits
    jl = open(os.path.join(ROOT, "julia", "B200HMC.jl")).read()
    m = re.search(r"const CHAIN_BAD_INITIAL, CHAIN_NONFINITE_Q, CHAIN_LEAPFROG_NONFINITE = "
                  r"Int32\((\d+)\), Int32\((\d+)\), Int32\((\d+)\)", jl)
    assert m and tuple(int(g) for g in m.groups()) == (bits["DHMC_CHAIN_BAD_INITIAL"], bits["DHMC_CHAIN_NONFINITE_Q"],
                                                        bits["DHMC_CHAIN_LEAPFROG_NONFINITE"])
