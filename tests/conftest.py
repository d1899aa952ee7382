import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "tools"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def _built():
    import util
    need = [util.HOSTSIM_SO, os.path.join(ROOT, "fluent-bit_b200", "libflbgpu.so")]
    if not all(os.path.exists(p) for p in need):
        import __graft_entry__ as g
        g.build()


@pytest.fixture(scope="session", autouse=True)
def built():
    _built()


@pytest.fixture(scope="session")
def sim_lib():
    """The CPU emulation of the device code (tests/hostsim) -- test infrastructure only."""
    import util
    return util.pkg.load(util.HOSTSIM_SO)


@pytest.fixture(scope="session")
def gpu_lib():
    """The product library on a real GPU."""
    import util
    return util.pkg.load()


@pytest.fixture
def ref_available():
    import util
    if not util.have_ref_results():
        pytest.skip("oracle/_ref/libflbref.so is not built and no stored reference results cover this test")
    return True
