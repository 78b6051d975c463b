"""Build the CUDA library in-tree: astroz_b200/libastroz_b200.so (sm_90a only).

    python -m astroz_b200.build [--force]

nvcc cross-compiles without a GPU; the built .so sits next to the sources it was built from.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libastroz_b200.so")
SOURCES = ["az_kernels.cu", "az_ingest.cu", "az_pairs.cu", "az_capi.cu"]
HEADERS = ["az_math.cuh", "az_device.cuh", "az_kernels.cuh", "az_ingest.cuh", "az_pairs.cuh", "az_elements.hpp", "az_tables.hpp",
           os.path.join("..", "..", "include", "astroz_b200.h")]
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [*GENCODE, "-O3", "-std=c++17", "-lineinfo",
              "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr"]
# Device element initialisation (K5) runs the host builders' arithmetic (az_elements.hpp) without FMA contraction, as the
# host compiler does: the 12-hour resonance polynomials for e > 0.65 cancel terms of 1e5 down to 1e2, so a contracted
# evaluation moved their coefficients by ~1e-12 and a device-initialised Molniya orbit by 4e-4 km after 30 years.
SOURCE_FLAGS = {"az_ingest.cu": ["-fmad=false"]}


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: the CUDA library cannot be built (there is no CPU fallback)")


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build_variant(out: str, defines: list[str]) -> str:
    """Measurement builds (tools/variant_sweep.sh): the same sources with extra -D flags, linked to `out`."""
    nvcc = _nvcc()
    objs = []
    for src in SOURCES:
        obj = out + "." + src.replace(".cu", ".o")
        cmd = [nvcc, *NVCC_FLAGS, *SOURCE_FLAGS.get(src, []), *[f"-D{d}" for d in defines], "-c", os.path.join(CSRC, src),
               "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        objs.append(obj)
    r = subprocess.run([nvcc, "-shared", "-o", out, *objs, *GENCODE, "-cudart", "static"],
                       capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return out


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    nvcc = _nvcc()
    objs = []
    for src in SOURCES:
        obj = os.path.join(CSRC, src.replace(".cu", ".o"))
        cmd = [nvcc, *NVCC_FLAGS, *SOURCE_FLAGS.get(src, []), "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            print(r.stderr)
        objs.append(obj)
    cmd = [nvcc, "-shared", "-o", LIB, *objs, *GENCODE, "-cudart", "static"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    if "--variant" in sys.argv:   # python -m astroz_b200.build --variant lib_x.so AZ_K2_LANES=1 AZ_DEFAULT_K2_BLOCKS=5
        i = sys.argv.index("--variant")
        print(build_variant(sys.argv[i + 1], sys.argv[i + 2:]))
    else:
        print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
