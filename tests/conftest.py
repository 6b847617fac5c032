import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    """The CPU oracle (test infrastructure).  Built on demand; the C restatement only needs gcc."""
    from oracle import pyoracle
    pyoracle.build()
    return pyoracle


@pytest.fixture(scope="session")
def ctx():
    """GPU context of the product.  No fallback: a missing .so or GPU is an error for -m gpu tests."""
    import lumixengine_b200 as lb
    c = lb.Context(0)
    yield c
    c.close()


# The reference's own code (oracle/_ref/libref_lumix.so) has broken static teardown on Linux (its jobs::shutdown()
# crashes too, SURVEY.md §8c): a process that loaded it can segfault inside exit().  When it was loaded, leave
# with os._exit once pytest has printed everything, keeping pytest's own exit status.
_exit_status = [0]


def pytest_sessionfinish(session, exitstatus):
    _exit_status[0] = int(exitstatus)


@pytest.hookimpl(trylast=True)
def pytest_unconfigure(config):
    mod = sys.modules.get("oracle.pyoracle")
    if (mod is not None and getattr(mod, "_ref", None) is not None) or os.environ.get("LB200_ENGINE_SHIM_LOADED") == "1":
        sys.stdout.flush()
        sys.stderr.flush()
        os._exit(_exit_status[0])
