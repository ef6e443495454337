import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


def _have_gpu() -> bool:
    try:
        import bodywork_mlops_demo_b200 as b2
        return b2.native.device_count() > 0
    except Exception:
        return False


@pytest.fixture(scope="session")
def ctx():
    """One device context shared by the GPU tests (fails loudly if the extension is missing)."""
    import bodywork_mlops_demo_b200 as b2
    c = b2.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="session")
def c_client(tmp_path_factory):
    """tests/c_client/fit_client.c built with gcc against include/b2gram.h and the in-tree libb2gram.so."""
    import shutil
    import subprocess
    import bodywork_mlops_demo_b200 as b2
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    lib_dir = os.path.dirname(b2.native.lib_path())
    exe = str(tmp_path_factory.mktemp("c_client") / "fit_client")
    cmd = [gcc, "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-O2", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "c_client", "fit_client.c"), "-o", exe, "-L", lib_dir, "-lb2gram", "-lm",
           "-Wl,-rpath," + lib_dir]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    assert proc.returncode == 0, proc.stderr
    return exe
