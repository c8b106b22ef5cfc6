#!/usr/bin/env python3
"""Builds poly-commit_b200/libpcgpu.so: nvcc, sm_90a (H100) only, one translation unit per (curve, kernel group) in parallel.
No GPU is needed to build (nvcc cross-compiles).  Re-builds only when a source or this script (architecture, flags) is newer than the library."""
import concurrent.futures
import glob
import os
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libpcgpu.so")
CURVES = ["Bls12381", "Bn254", "Pallas"]
GROUPS = [6, 8, 9, 5, 2, 3, 1, 4]   # inst_unit.cu groups, heaviest first (see the list at the top of that file)
PAIRING_CURVES = ["Bls12381", "Bn254"]
G2_GROUPS = [11, 12, 10]           # G2 point kernels and entry points: the pairing curves only
PAIRING_GROUPS = [13]              # Miller loops and final exponentiations: the pairing curves only
# heaviest first so the thread pool keeps every core busy to the end
UNITS = [("inst_unit", c, g) for g in PAIRING_GROUPS + G2_GROUPS[:1] for c in PAIRING_CURVES] + \
    [("inst_unit", c, g) for g in GROUPS for c in CURVES] + \
    [("inst_unit", c, g) for g in G2_GROUPS[1:] for c in PAIRING_CURVES] + [("api", None, None)]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + ["-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC"]


def _newest_source():
    srcs = glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh")) + \
        glob.glob(os.path.join(CSRC, "*.hpp")) + [os.path.join(HERE, "..", "include", "pcgpu.h"), os.path.abspath(__file__)]
    return max(os.path.getmtime(s) for s in srcs)


def _compile(unit, extra):
    src, curve, group = unit
    name = src if curve is None else f"{src}_{curve.lower()}_{group}"
    out = os.path.join(OBJ, name + ".o")
    defs = [] if curve is None else [f"-DPCGPU_UNIT_CURVE={curve}", f"-DPCGPU_UNIT_GROUP={group}"]
    cmd = ["nvcc"] + NVCC_FLAGS + defs + extra + ["-c", os.path.join(CSRC, src + ".cu"), "-o", out]
    t0 = time.time()
    r = subprocess.run(cmd, capture_output=True, text=True)
    return name, r.returncode, r.stdout + r.stderr + f"[build] {name}: {time.time() - t0:.0f} s\n", out


def build(force=False, verbose=False, extra=()):
    if not force and os.path.exists(LIB) and os.path.getmtime(LIB) >= _newest_source():
        return LIB
    os.makedirs(OBJ, exist_ok=True)
    extra = list(extra) + (["-Xptxas", "-v"] if verbose else [])
    with concurrent.futures.ThreadPoolExecutor(max_workers=max(2, min(len(UNITS), os.cpu_count() or 4))) as ex:
        results = list(ex.map(lambda u: _compile(u, extra), UNITS))
    objs = []
    for unit, rc, log, out in results:
        if verbose or rc:
            sys.stderr.write(log)
        elif os.environ.get("PCGPU_BUILD_TIMES"):
            sys.stderr.write(log.splitlines()[-1] + "\n")
        if rc:
            raise RuntimeError(f"nvcc failed on {unit}.cu")
        objs.append(out)
    # link next to the target and rename: a reader (or a snapshot of the tree) never sees a half-written library
    subprocess.check_call(["nvcc", "-shared", "-o", LIB + ".tmp"] + objs + ARCH)
    os.replace(LIB + ".tmp", LIB)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
