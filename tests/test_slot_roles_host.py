"""The NUTS state machine (nuts_machine.cuh) with the GPU's leaf-merge interface and slot roles, on the host
(tests/leafsim/leafsim.cpp): a backend that evaluates a leaf's merges together with its leapfrog, as the device's one
all-reduce per leaf does, builds the same trees bit for bit as the plain host simulation (tests/hostsim), which checks one
merge at a time; trees of the full max_depth never hand one slot to two live vectors; and at the dim-1000 layout the momenta
and ρ that the turn checks read stay in the on-chip slots while the proposals go to the arena."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "hostsim"))
import pyhostsim as hs  # noqa: E402


@pytest.fixture(scope="module")
def leafsim(tmp_path_factory):
    cxx = os.environ.get("CXX") or shutil.which("g++")
    if not cxx:
        pytest.skip("no C++ compiler")
    so = str(tmp_path_factory.mktemp("leafsim") / "libleafsim.so")
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-mfma", "-mavx2", "-x", "c++", "-shared",
                           "-o", so, os.path.join(HERE, "leafsim", "leafsim.cpp")])
    return C.CDLL(so)


def run(lib, q, eps, seed, chain, N=1, T=128, max_depth=10, n_sm=8):
    q = np.ascontiguousarray(q, dtype=np.float64)
    post = np.empty((N, q.size))
    stats = np.zeros(N, dtype=hs.tree_stats_dtype)
    c = np.zeros(4, dtype=np.int64)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    status = lib.ls_run(C.c_int(q.size), C.c_int(T), C.c_int(max_depth), C.c_int(n_sm), C.c_uint64(seed), C.c_uint64(chain),
                        C.c_int(N), C.c_double(eps), p(q), p(post), p(stats), p(c))
    return dict(status=status, posterior_matrix=post, tree_statistics=stats, merge_reads=int(c[0]),
                offchip_reads=int(c[1]), slot_clashes=int(c[2]), steps=int(c[3]))


@pytest.mark.parametrize("D,T,eps", [(40, 32, 0.3), (300, 128, 0.25), (1000, 128, 0.28)])
def test_leaf_merges_build_the_same_trees(leafsim, D, T, eps):
    for chain in range(3):
        q = np.random.default_rng(chain).standard_normal(D)
        a = run(leafsim, q, eps, 11, chain, N=6, T=T)
        b = hs.run(0, q, eps, 11, chain, N=6, T=T)            # FAMILY_STD_NORMAL, unit metric, fixed step size
        assert a["status"] == b["status"] == 0
        assert a["tree_statistics"].tobytes() == b["tree_statistics"].tobytes()
        assert a["posterior_matrix"].tobytes() == b["posterior_matrix"].tobytes()


@pytest.mark.parametrize("max_depth", [10, 12, 14])
@pytest.mark.parametrize("n_sm", [8, 3])
def test_max_depth_tree_shares_no_slot(leafsim, max_depth, n_sm):
    # a step size far below the U-turn scale: every transition builds all max_depth doublings
    q = np.random.default_rng(max_depth).standard_normal(8)
    r = run(leafsim, q, 1e-5, 7, 3, N=2, T=32, max_depth=max_depth, n_sm=n_sm)
    assert r["status"] == 0
    assert r["steps"] == 2 * (2 ** max_depth - 1)
    assert r["slot_clashes"] == 0


def test_merge_operands_stay_on_chip_at_dim_1000(leafsim):
    # the bench's C2 shape: D = 1000 over 128 threads, 8 slots in shared memory, ϵ near its adapted value
    reads = offchip = 0
    for chain in range(4):
        q = np.random.default_rng(chain).standard_normal(1000)
        r = run(leafsim, q, 0.28, 2026, chain, N=10)
        assert r["status"] == 0 and r["slot_clashes"] == 0
        reads += r["merge_reads"]
        offchip += r["offchip_reads"]
    # proposals taken from the low end as well put about a third of these reads off chip
    assert reads > 0 and offchip / reads < 0.15
