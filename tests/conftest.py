import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")

# The CUDA extension is built in-tree (git-ignored).  A fresh checkout has no .so yet: build it once (nvcc
# cross-compiles for sm_90a without a GPU) so that the host-side tests can load the C ABI.
_LIB = os.path.join(ROOT, "rendernet_b200", "librendernet_b200.so")
if not os.path.exists(_LIB):
    import subprocess
    subprocess.run(["make", "-C", os.path.join(ROOT, "rendernet_b200", "csrc"), "-j4"], check=True,
                   stdout=subprocess.DEVNULL)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN
