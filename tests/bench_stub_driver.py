"""TEST INFRASTRUCTURE — runs bench.py's b200 arm end to end on a machine WITHOUT a GPU: torch's CUDA entry points and the
engine are replaced by stand-ins that return plausible counters, so that the orchestration of the arm (argument parsing,
the timed loops, the auxiliary legs, the reductions and the one JSON line on stdout) is exercised by the CPU suite
(tests/test_bench_contract.py).  Numbers printed under it mean nothing."""
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

torch.cuda.is_available = lambda: True
torch.cuda.set_device = lambda *_a, **_k: None
torch.cuda.synchronize = lambda *_a, **_k: None
torch.cuda.get_device_properties = lambda *_a, **_k: types.SimpleNamespace(name="stub", multi_processor_count=132,
                                                                           L2_cache_size=50 << 20)
_empty, _tensor = torch.empty, torch.tensor
torch.empty = lambda *a, device=None, **k: _empty(*a, **k)
torch.tensor = lambda *a, device=None, **k: _tensor(*a, **k)

import __graft_entry__ as entry  # noqa: E402

pkg = entry.load_package()


class StubEngine:
    launches = 0

    def __init__(self, ℓ, chains, **kw):
        self.K, self.D = int(chains), int(ℓ.dimension())

    def layout(self):
        return 128, 8

    def random_position(self): pass
    def find_initial_stepsize(self, *a): pass
    def warmup_stage(self, *a, **k): pass
    def leapfrog(self, *a): pass
    def close(self): pass

    def last_total_steps(self):
        return 15 * self.K

    def last_kernel_ms(self):
        return 1.25

    def kernel_launches(self):
        StubEngine.launches += 1
        return StubEngine.launches

    def get_state(self, fields):
        return {"eps": np.full(self.K, 0.28), "q": np.zeros((self.K, self.D))}

    def mcmc_dev(self, *a): pass

    def mcmc_from(self, q, n, out=None):
        return out

    def host_alloc(self, shape, dtype=np.float64):
        return np.zeros(shape, dtype=dtype)

    def tree_summary_dev(self, ptr, n, ebfmi=True):
        return dict(N=self.K * n, a_mean=0.84, steps=15 * self.K * n, termination_counts=dict(max_depth=0, divergence=0, turning=self.K * n),
                    depth_counts=[0, 0, 0, 0, self.K * n], EBFMI=None)


pkg.Engine = StubEngine
sys.argv = ["bench.py"] + sys.argv[1:]
import importlib.util  # noqa: E402

spec = importlib.util.spec_from_file_location("bench", os.path.join(ROOT, "bench.py"))
bench = importlib.util.module_from_spec(spec)
spec.loader.exec_module(bench)
bench.main()
