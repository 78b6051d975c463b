"""The Python side of the C ABI is read from include/astroz_b200.h (astroz_b200/_abi.py): the ctypes signatures match the
header's arity for every export, and the descriptor layouts and constants equal what the C compiler makes of the
header."""
import ctypes as C
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def built():
    from astroz_b200 import build

    return build.build()


def test_lib_binds_every_export_with_the_header_arity(built):
    header = open(os.path.join(ROOT, "include", "astroz_b200.h")).read()
    out = subprocess.run(["nm", "-D", "--defined-only", built], capture_output=True, text=True, check=True).stdout
    exported = sorted({ln.split()[-1] for ln in out.splitlines() if "astroz_cuda_" in ln})
    from astroz_b200 import _lib

    L = _lib.lib()
    bound = sorted(k for k in vars(L) if k.startswith("astroz_cuda_"))   # CDLL caches every symbol it has looked up
    assert bound == exported
    stripped = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    for name in bound:
        cargs = re.search(r"\b" + name + r"\s*\(([^;{]*?)\)\s*;", stripped, flags=re.S).group(1).strip()
        assert len(getattr(L, name).argtypes) == (0 if cargs in ("", "void") else cargs.count(",") + 1), name


def c_abi(include_dir: str, structs, defines, tmp_path) -> dict:
    """What the C compiler makes of the header in include_dir: {struct: sizeof, "struct.field": offsetof, define: value}
    for structs = {struct: [field, ...]} and the define names"""
    body = []
    for s, fields in structs.items():
        body.append(f'printf("{s} %zu\\n", sizeof({s}));')
        body += [f'printf("{s}.{f} %zu\\n", offsetof({s}, {f}));' for f in fields]
    body += [f'printf("{d} %lld\\n", (long long)({d}));' for d in defines]
    src, exe = tmp_path / "abi.c", tmp_path / "abi"
    src.write_text("#include <stddef.h>\n#include <stdio.h>\n#include \"astroz_b200.h\"\nint main(void) {\n"
                   + "\n".join(body) + "\nreturn 0;\n}\n")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I", include_dir, str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout
    return {k: int(v) for k, v in (ln.split() for ln in out.splitlines())}


def test_python_abi_matches_the_c_compiler(tmp_path):
    """The ctypes descriptor, the impulse dtype and the Python constants agree with the C compiler's reading of the
    header: sizeof / offsetof of every field of both typedef structs and the value of every ASTROZ_* define."""
    from astroz_b200 import _abi, _lib, fit
    from astroz_b200 import numerical as P
    from astroz_b200.constellation import Layout, OutputMode

    header = open(os.path.join(ROOT, "include", "astroz_b200.h")).read()
    assert set(re.findall(r"typedef struct \{[^}]*\}\s*(\w+)\s*;", header)) == {"astroz_force_model_t",
                                                                               "astroz_impulse_t"}
    defines = sorted(set(re.findall(r"^#define\s+(ASTROZ_\w+)[ \t]+\S", header, flags=re.M)))
    model, imp = P._ForceModelC, P.IMPULSE_DTYPE
    py = {"astroz_force_model_t": C.sizeof(model), "astroz_impulse_t": imp.itemsize,
          **{"astroz_force_model_t." + f: getattr(model, f).offset for f, _ in model._fields_},
          **{"astroz_impulse_t." + f: imp.fields[f][1] for f in imp.names}, **_abi.DEFINES}
    c = c_abi(os.path.join(ROOT, "include"), {"astroz_force_model_t": [f for f, _ in model._fields_],
                                              "astroz_impulse_t": list(imp.names)}, defines, tmp_path)
    assert py == c
    public = {
        "OK": _lib.OK, "WGS84": _lib.WGS84, "WGS72": _lib.WGS72, "MODE_TEME": OutputMode.teme,
        "MODE_ECEF": OutputMode.ecef, "MODE_GEODETIC": OutputMode.geodetic,
        "LAYOUT_SATELLITE_MAJOR": Layout.satelliteMajor, "LAYOUT_TIME_MAJOR": Layout.timeMajor,
        "FORCE_J2": P.FORCE_J2, "FORCE_DRAG": P.FORCE_DRAG, "INTEGRATOR_RK4": P.INTEGRATORS["rk4"],
        "INTEGRATOR_DP87": P.INTEGRATORS["dp87"], "NUMERICAL_OK": P.OK, "NUMERICAL_STOPPED": P.STOPPED,
        "NUMERICAL_SUBSTEP_LIMIT": P.SUBSTEP_LIMIT, "NUMERICAL_NON_FINITE": P.NON_FINITE,
        "MODEL_TWO_BODY": P.TwoBody.kind, "MODEL_J2": P.J2.kind, "MODEL_J3": P.J3.kind, "MODEL_J4": P.J4.kind,
        "MODEL_DRAG": P.Drag.kind, "MODEL_IMPROVED_DRAG": P.ImprovedDrag.kind, "MODEL_SRP": P.SolarRadiationPressure.kind,
        "MODEL_THIRD_BODY": P.ThirdBody.kind, "MODEL_PER_STATE_C": P._PER_STATE["c"],
        "MODEL_PER_STATE_AREA": P._PER_STATE["area"], "MODEL_PER_STATE_MASS": P._PER_STATE["mass"],
        "MODEL_POS_TABLE": P._POS_TABLE, "MAX_MODELS": P.MAX_MODELS, "IMPULSE_ABSOLUTE": P.Absolute.kind,
        "IMPULSE_PROGRADE": P.Prograde.kind, "IMPULSE_PHASE": P.Phase.kind, "IMPULSE_PLANE_CHANGE": P.PlaneChange.kind,
        "MANEUVER_ABNORMAL": P.ABNORMAL, "MANEUVER_TRUNCATED": P.TRUNCATED, "FIT_CONVERGED": fit.CONVERGED,
        "FIT_ITERATION_LIMIT": fit.ITERATION_LIMIT, "FIT_INIT_FAILED": fit.INIT_FAILED,
        "FIT_DEEP_SPACE": fit.DEEP_SPACE, "FIT_TOO_FEW_OBSERVATIONS": fit.TOO_FEW_OBSERVATIONS}
    assert {k: c["ASTROZ_" + k] for k in public} == public
    errors = {"OK": "ok", "BAD_TLE_LENGTH": "badTleLength", "BAD_CHECKSUM": "badChecksum",
              "DEEP_SPACE": "deepSpaceNotSupported", "INVALID_ECC": "invalidEccentricity", "DECAYED": "satelliteDecayed",
              "VALUE_ERROR": "valueError", "ALLOC_FAILED": "allocFailed", "NULL_POINTER": "nullPointer",
              "NOT_INITIALIZED": "notInitialized", "UNKNOWN": "unknown", "CUDA_ERROR": "cudaError",
              "NO_DEVICE": "noCudaDevice"}
    assert _lib.ERROR_NAMES == {c["ASTROZ_" + k]: v for k, v in errors.items()}
    assert _lib.SGP4_ERROR == {c["ASTROZ_INVALID_ECC"]: 1, c["ASTROZ_DEEP_SPACE"]: 3, c["ASTROZ_ALLOC_FAILED"]: 4,
                               c["ASTROZ_DECAYED"]: 6}
