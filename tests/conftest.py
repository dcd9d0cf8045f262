import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu)")


def pytest_sessionstart(session):
    """A fresh checkout has no built artefacts (they are git-ignored): build them once, the way
    __graft_entry__.build() does, instead of failing every test on import.  The PRODUCT still
    fails loudly when its library is missing; this is only the test session helping itself."""
    import shutil
    import subprocess
    so = os.path.join(ROOT, "manatee_b200", "libmanatee_gpu.so")
    if not os.path.exists(so) and shutil.which("nvcc") and shutil.which("make"):
        subprocess.run(["make", "-C", os.path.join(ROOT, "manatee_b200", "csrc")], check=False,
                       stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)


@pytest.fixture(scope="session")
def oracle():
    import oracle as O
    O.build()
    return O


@pytest.fixture(scope="session")
def native():
    """libmanatee_gpu.so must be built and loadable; GPU tests fail loudly otherwise."""
    from manatee_b200 import _native
    return _native.lib()


@pytest.fixture(scope="session")
def emul_so(tmp_path_factory):
    """libmanatee_gpu_emul.so (tests/emul/make_emul_lib.py): the whole library compiled for the CPU
    SIMT emulator, built once per session; child pytest processes inherit it through MTZ_EMUL_SO.
    Test infrastructure only -- the product never loads it."""
    import shutil
    import subprocess
    pre = os.environ.get("MTZ_EMUL_SO")
    if pre and os.path.exists(pre):
        return pre
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    so = os.path.join(str(tmp_path_factory.mktemp("emul_lib")), "libmanatee_gpu_emul.so")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "emul", "make_emul_lib.py"), so],
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert r.returncode == 0, r.stderr
    os.environ["MTZ_EMUL_SO"] = so
    return so
