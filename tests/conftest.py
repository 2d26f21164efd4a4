import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


@pytest.fixture(scope="session")
def O():
    """The CPU oracle (test infrastructure).  Built on demand: gcc only, seconds."""
    from oracle import oracle
    oracle.build()
    return oracle


@pytest.fixture(scope="session")
def ref(O):
    """The real reference functions (oracle/_ref), skipped where the library was neither built nor shipped."""
    r = O.ref_fns()
    if r is None:
        pytest.skip("oracle/_ref/libedyn_ref.so not available (needs /root/reference at build time)")
    return r


@pytest.fixture(scope="session")
def E():
    import edyn_b200
    return edyn_b200


def gpu_available():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.fixture(scope="session")
def gpu(E):
    """Hard requirement for -m gpu tests: the CUDA library must load and a device must exist.  No fallback."""
    from edyn_b200 import _lib
    assert os.path.exists(_lib.LIB_PATH), "edyn_b200/libb2d.so missing: run __graft_entry__.build()"
    if os.environ.get("B2D_EMU") == "1" and "libb2d_emu" in _lib.LIB_PATH:
        return True         # development: the -m gpu tests against the CPU emulation of tests/emu (B2D_LIB points at it)
    assert gpu_available(), "no CUDA device visible"
    return True
