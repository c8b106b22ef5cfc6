"""poly-commit_b200 -- H100-native compute engine for the prover hot path of arkworks-rs/poly-commit.

The product is the C-ABI shared library ``libpcgpu.so`` (CUDA, sm_90a; sources in ``csrc/``,
interface in ``include/pcgpu.h``).  This package is the thin ctypes binding plus a host-side mirror of
the reference's operator interface for the path (``kzg10.KZG10.commit/open``, ``msm_bigint`` ...).

There is no CPU fallback: importing works anywhere, but creating an ``Engine`` raises unless the CUDA
library is present AND an sm_90 device is usable.
"""
from .binding import (Engine, Srs, BrakedownCode, MlpcKey, G2Prepared, HyraxState, PcgpuError, CURVES, BLS12_381, BN254, PALLAS, BLS12_381_G2, BN254_G2,
                      SCALARS_MONT, DEVICE_PTRS, SRS_PRECOMPUTE, NTT_INVERSE, SRS_COMB, library_path, fq_limbs, affine_limbs)

__all__ = ["Engine", "Srs", "BrakedownCode", "MlpcKey", "G2Prepared", "HyraxState", "PcgpuError", "CURVES", "BLS12_381", "BN254", "PALLAS", "BLS12_381_G2",
           "BN254_G2", "SCALARS_MONT", "DEVICE_PTRS", "SRS_PRECOMPUTE", "NTT_INVERSE", "SRS_COMB", "library_path", "fq_limbs",
           "affine_limbs"]
