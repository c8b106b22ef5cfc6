// Kernel + host-template instantiations, one translation unit per (curve, group):
//   nvcc -DPCGPU_UNIT_CURVE=Bls12381 -DPCGPU_UNIT_GROUP=1 ... (build.py).  Group 0 defines every group (host emulation).
//   1 pipeline host logic + digit / plan kernels   2 small MSM   3 SRS + MSM / KZG entry points   4 Fr, NTT, hashes
//   5 IPA + wire   6 pair-round kernels   8 XYZZ accumulate   9 bucket reduction
//   G2 of the pairing curves (BLS12-381, BN254) only: 10 pipeline host logic, small MSM, G2 / MultilinearPC entry points
//   11 G2 XYZZ accumulate   12 G2 bucket reduction
//   the pairing curves only: 13 the pairing (Miller loops plain and over prepared G2 lines, G2 line preparation, final
//   exponentiations, Fq12 diagnostics)
#include "impl.cuh"

#ifndef PCGPU_UNIT_CURVE
#error "compile with -DPCGPU_UNIT_CURVE=<Bls12381|Bn254|Pallas> -DPCGPU_UNIT_GROUP=<0..13>"
#endif
#define PCGPU_UC PCGPU_UNIT_CURVE
#define PCGPU_DEF_OR_EXTERN(GROUP, MACRO) PCGPU_DEF_OR_EXTERN_##GROUP(MACRO)
#define PCGPU_CAT_(a, b) a##b
#define PCGPU_CAT(a, b) PCGPU_CAT_(a, b)
#define PCGPU_PAIRING_Bls12381 1
#define PCGPU_PAIRING_Bn254 1
#define PCGPU_UG2 PCGPU_CAT(PCGPU_UC, G2)   // the curve's G2 group type (Bls12381G2, Bn254G2)

#if PCGPU_UNIT_GROUP == 0
PCGPU_INSTANTIATE(PCGPU_UC, )
#if PCGPU_CAT(PCGPU_PAIRING_, PCGPU_UNIT_CURVE)
PCGPU_INSTANTIATE_G2(PCGPU_UG2, )
PCGPU_INST_PAIRING(PCGPU_UC, )
#endif
#elif PCGPU_UNIT_GROUP == 13
#if !PCGPU_CAT(PCGPU_PAIRING_, PCGPU_UNIT_CURVE)
#error "group 13 (the pairing) exists for the pairing curves only"
#endif
PCGPU_INST_PAIRING(PCGPU_UC, )
#elif PCGPU_UNIT_GROUP >= 10
#if !PCGPU_CAT(PCGPU_PAIRING_, PCGPU_UNIT_CURVE)
#error "groups 10-12 (G2) exist for the pairing curves only"
#endif
#if PCGPU_UNIT_GROUP == 10
PCGPU_INST_PIPE(PCGPU_UG2, ) PCGPU_INST_SMALL(PCGPU_UG2, ) PCGPU_INST_G2(PCGPU_UG2, )
#else
PCGPU_INST_PIPE(PCGPU_UG2, extern)
#endif
#if PCGPU_UNIT_GROUP == 11
PCGPU_INST_ACC(PCGPU_UG2, )
#else
PCGPU_INST_ACC(PCGPU_UG2, extern)
#endif
#if PCGPU_UNIT_GROUP == 12
PCGPU_INST_REDUCE(PCGPU_UG2, )
#else
PCGPU_INST_REDUCE(PCGPU_UG2, extern)
#endif
#else
// the helpers other groups call are declared extern everywhere except in their own unit
#if PCGPU_UNIT_GROUP == 1
PCGPU_INST_PIPE(PCGPU_UC, )
#else
PCGPU_INST_PIPE(PCGPU_UC, extern)
#endif
#if PCGPU_UNIT_GROUP == 2
PCGPU_INST_SMALL(PCGPU_UC, )
#else
PCGPU_INST_SMALL(PCGPU_UC, extern)
#endif
#if PCGPU_UNIT_GROUP == 6
PCGPU_INST_PAIR1(PCGPU_UC, )
#else
PCGPU_INST_PAIR1(PCGPU_UC, extern)
#endif
#if PCGPU_UNIT_GROUP == 8
PCGPU_INST_ACC(PCGPU_UC, )
#else
PCGPU_INST_ACC(PCGPU_UC, extern)
#endif
#if PCGPU_UNIT_GROUP == 9
PCGPU_INST_REDUCE(PCGPU_UC, )
#else
PCGPU_INST_REDUCE(PCGPU_UC, extern)
#endif
#if PCGPU_UNIT_GROUP == 3
PCGPU_INST_SRS(PCGPU_UC, )
#endif
#if PCGPU_UNIT_GROUP == 4
PCGPU_INST_FR(PCGPU_UC, )
#endif
#if PCGPU_UNIT_GROUP == 5
PCGPU_INST_IPA(PCGPU_UC, )
#endif
#endif
