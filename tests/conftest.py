import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="session", autouse=True)
def _built():
    """Make sure the checker (oracle) and the product library exist; both are cheap no-ops when
    the prebuilt files travelled with the snapshot."""
    import subprocess
    if not os.path.exists(os.path.join(ROOT, "oracle", "liboracle.so")):
        subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "oracle"),
                        os.path.join(ROOT, "oracle", "liboracle.so")], check=True)
    if not os.path.exists(os.path.join(ROOT, "retinanet-examples_b200", "libodtk_b200.so")):
        subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "retinanet-examples_b200", "csrc")], check=True)
