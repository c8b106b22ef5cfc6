import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on the GPU box)")


@pytest.fixture(scope="session")
def pc():
    import pkgload
    return pkgload.load()


@pytest.fixture(scope="session")
def oracle():
    from oracle import orc
    orc.lib()
    return orc


@pytest.fixture(scope="session")
def hostcheck_path():
    """tests/host_emul/libpcgpu_hostcheck.so: the kernel bodies compiled for the host (unit-test harness)."""
    import subprocess
    d = os.path.join(ROOT, "tests", "host_emul")
    subprocess.check_call(["make", "-s", "-C", d])
    return os.path.join(d, "libpcgpu_hostcheck.so")


@pytest.fixture(scope="session")
def gpu_engine(pc):
    """The product library on cuda:0.  Fails loudly (no fallback) if the CUDA build or the device is missing."""
    eng = pc.Engine(0)
    yield eng
    eng.close()


@pytest.fixture(params=["small", "buckets"])
def msm_path(request, monkeypatch):
    """MSMs of <= 4096 terms take the one-launch path (csrc/msm_small.cuh); PCGPU_MSM_SMALL=0 sends them through the bucket
    pipeline instead, so the small-n cases keep covering both."""
    monkeypatch.setenv("PCGPU_MSM_SMALL", "1" if request.param == "small" else "0")
    return request.param
