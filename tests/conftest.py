import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a machine that has one)")
    # built artefacts are not in git: build them once if this is a fresh checkout
    pkg = os.path.join(ROOT, "plink_ng_b200")
    if not (os.path.exists(os.path.join(pkg, "libpl2gpu.so")) and os.path.exists(os.path.join(pkg, "plink2_b200"))):
        import subprocess

        subprocess.run(["make", "-C", os.path.join(pkg, "csrc")], check=True, stdout=subprocess.DEVNULL)


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


def _have_gpu():
    try:
        import plink_ng_b200 as p

        return p.lib.pl2gpu_device_count() > 0
    except Exception:
        return False


@pytest.fixture(scope="session")
def gpu_ctx():
    import plink_ng_b200 as p

    if p.lib.pl2gpu_device_count() <= 0:
        pytest.fail("no CUDA device visible: -m gpu tests need an H100 (there is no CPU fallback)")
    ctx = p.GpuContext(0)
    yield ctx
    ctx.close()
