"""G2 multi-scalar multiplication (<E::G2 as VariableBaseMSM>::msm_bigint) and pcgpu_g2_fixed_base_mul on BLS12-381 and BN254:
the Fq2 field layer, the small one-launch path and the bucket pipeline (raw bases, no pair rounds), on the host-emulated
kernels and on the device.  Case bodies: tests/g2_cases.py."""
import pytest

from oracle import pyref
from tests import g2_cases as gc
from tests import util


@pytest.fixture(scope="module")
def emul(pc, hostcheck_path):
    e = pc.Engine(0, lib_path=hostcheck_path)
    yield e
    e.close()


@pytest.mark.parametrize("cname", gc.PAIRING)
def test_emul_fq2_ops(emul, cname):
    gc.fq2_ops_case(emul, cname)


@pytest.mark.parametrize("cname", gc.PAIRING)
def test_emul_generator_kats(emul, pc, cname, msm_path):
    gc.generator_kat_case(emul, pc, cname, msm_path)


@pytest.mark.parametrize("cname", gc.PAIRING)
def test_emul_edges(emul, pc, cname, msm_path):
    gc.edge_case(emul, pc, cname, msm_path)


@pytest.mark.parametrize("cname", gc.PAIRING)
def test_emul_random_bases_vs_pyref(emul, pc, cname, msm_path):
    gc.random_vs_pyref_case(emul, pc, cname, 300, msm_path)


@pytest.mark.parametrize("cname", gc.PAIRING)
def test_emul_trapdoor(emul, pc, cname, monkeypatch):
    monkeypatch.setenv("PCGPU_MSM_SMALL", "0")
    gc.trapdoor_case(emul, pc, cname, 3000, "buckets")
    gc.trapdoor_case(emul, pc, cname, 2500, "buckets", skewed=True, seed=4)


@pytest.mark.parametrize("cname", gc.PAIRING)
def test_emul_g2_ids_rejected(emul, pc, cname):
    gc.g2_id_rejected_case(emul, pc, cname)


# ---- device ------------------------------------------------------------------------------------------------------------
_KEYED = {}


def _keyed(eng, pc, cname, n):
    """2^20 + 1 trapdoor bases per curve, built once (pcgpu_g2_fixed_base_mul, 256 of them checked against pyref)"""
    if cname not in _KEYED:
        ks = gc.fr_ints(util.rand_fr(cname, n, seed=11, mont=False))
        _KEYED[cname] = (ks, gc.trapdoor_bases(eng, pc, cname, ks, sample=256, seed=11))
    return _KEYED[cname]


@pytest.mark.gpu
@pytest.mark.parametrize("cname", gc.PAIRING)
def test_gpu_fq2_ops_and_kats(gpu_engine, pc, cname, monkeypatch):
    gc.fq2_ops_case(gpu_engine, cname, n=4096)
    for path in ("small", "buckets"):
        monkeypatch.setenv("PCGPU_MSM_SMALL", "1" if path == "small" else "0")
        gc.generator_kat_case(gpu_engine, pc, cname, path)
        gc.edge_case(gpu_engine, pc, cname, path)
    gc.g2_id_rejected_case(gpu_engine, pc, cname)


@pytest.mark.gpu
@pytest.mark.parametrize("cname", gc.PAIRING)
def test_gpu_random_bases_vs_pyref(gpu_engine, pc, cname, monkeypatch):
    for path in ("small", "buckets"):
        monkeypatch.setenv("PCGPU_MSM_SMALL", "1" if path == "small" else "0")
        gc.random_vs_pyref_case(gpu_engine, pc, cname, 1 << 10, path)


@pytest.mark.gpu
@pytest.mark.parametrize("cname", gc.PAIRING)
def test_gpu_trapdoor_sizes(gpu_engine, pc, cname):
    keyed = _keyed(gpu_engine, pc, cname, (1 << 20) + 1)
    for lg in (10, 12, 16, 18, 20):
        for n in (1 << lg, (1 << lg) + 1):
            path = "small" if n <= gc.SMALL_MAX_N else "buckets"
            gc.trapdoor_case(gpu_engine, pc, cname, n, path, keyed=keyed, seed=lg)
            gc.trapdoor_case(gpu_engine, pc, cname, n, path, keyed=keyed, skewed=True, seed=lg + 1)


@pytest.mark.gpu
@pytest.mark.parametrize("cname", gc.PAIRING)
def test_gpu_fixed_base_mul_2_21(gpu_engine, pc, cname):
    ks = gc.fr_ints(util.rand_fr(cname, 1 << 21, seed=12, mont=False))
    ks[5] = 0
    out = gc.trapdoor_bases(gpu_engine, pc, cname, ks, sample=256, seed=12)
    assert not out[5].any()
    assert gc.from_limbs(cname, out[7]) == pyref.G2(cname).mul(ks[7], gc.generator(cname))
