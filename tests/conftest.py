import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))


def pytest_addoption(parser):
    parser.addoption("--dry-engine", action="store_true", default=False,
                     help="run the Python of selected -m gpu tests without a GPU: the engine is replaced by an oracle-backed "
                          "stand-in (tests/dryrun_engine.py) — checks the test code, proves nothing about the CUDA path")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")


@pytest.fixture(scope="session")
def po():
    import pyoracle
    pyoracle.lib()
    return pyoracle


@pytest.fixture(scope="session")
def pkg(request):
    from __graft_entry__ import load_package
    p = load_package()
    if request.config.getoption("--dry-engine"):
        import pyoracle
        from dryrun_engine import DryRunEngine
        make = lambda ℓ, chains, **kw: DryRunEngine(pyoracle, p, ℓ, chains, **kw)      # noqa: E731
        sys.modules[p.__name__ + ".api"].Engine = make
        p.Engine = make
    return p
