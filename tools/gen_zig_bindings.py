#!/usr/bin/env python
"""Generate zig/src/c_api/cuda.zig from include/astroz_b200.h (CPU tool).

    python tools/gen_zig_bindings.py [--check]

One `pub extern fn` per exported symbol, types mapped from the C declaration, plus the hand-written error mapping.
tests/test_cabi_cpu.py runs this with --check so the committed Zig file can never drift from the header.
"""
from __future__ import annotations

import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from astroz_b200._abi import declarations, structs  # noqa: E402

OUT = os.path.join(ROOT, "zig", "src", "c_api", "cuda.zig")

RET = {"int32_t": "i32", "uint32_t": "u32", "void": "void", "const char *": "[*:0]const u8", "void *": "?*anyopaque"}


def zig_type(ctype: str, name: str) -> str:
    t = " ".join(ctype.split())
    arr = re.search(r"\[(\d+)\]$", name)
    if arr:   # double pos[3], float ms[3]
        base = {"double": "f64", "float": "f32"}[t]
        return f"*[{arr.group(1)}]{base}"
    table = {
        "const char *const *": "[*]const [*:0]const u8",
        "const char *": "[*]const u8" if name == "text" else "[*:0]const u8",
        "const double *": "?[*]const f64",
        "double *": "?[*]f64",
        "double **": "?[*]?[*]f64",
        "const uint8_t *": "?[*]const u8",
        "uint8_t *": "?[*]u8",
        "const uint32_t *": "?[*]const u32",
        "uint32_t *": "?[*]u32",
        "int32_t *": "?[*]i32",
        "const uint64_t *": "?[*]const u64",
        "uint64_t *": "?[*]u64" if name in ("steps", "d_steps", "n_samples", "d_n_samples", "counts", "d_counts")
        else "*u64",
        "void *": "?*anyopaque",
        "void *const *": "?[*]const ?*anyopaque",
        "astroz_constellation_t": "Handle",
        "astroz_sgp4_t": "Handle",
        "astroz_constellation_t *": "*Handle",
        "const astroz_force_model_t *": "?[*]const astroz_force_model_t",
        "const astroz_impulse_t *": "?[*]const astroz_impulse_t",
        "astroz_sgp4_t *": "*Handle",
        "uint32_t": "u32", "int32_t": "i32", "size_t": "usize", "double": "f64",
    }
    if t not in table:
        raise SystemExit(f"gen_zig_bindings: no Zig mapping for C type '{t}' (parameter {name})")
    return table[t]


FIELD = {"int32_t": "i32", "uint32_t": "u32", "double": "f64", "const double *": "?[*]const f64"}


def zig_field(ctype: str, name: str) -> str:
    arr = re.search(r"\[(\d+)\]$", name)
    base = FIELD[" ".join(ctype.split())]
    return f"[{arr.group(1)}]{base}" if arr else base


def render() -> str:
    out = [
        "//! CUDA propagation library bindings -- GENERATED from include/astroz_b200.h by tools/gen_zig_bindings.py.",
        "//! Drop this file in as src/c_api/cuda.zig of ATTron/astroz (next to src/c_api/sgp4.zig); INTEGRATION.md has",
        "//! the build.zig wiring and zig/src/Constellation.device.zig the device branch of Constellation.zig.",
        "//! Error codes are err.Code values (src/c_api/error.zig:3-19) extended with cudaError = -200, noCudaDevice = -201.",
        "//! Uncompiled here: the build image has no Zig toolchain (DESIGN.md section 1).",
        "",
        "pub const Handle = ?*anyopaque;",
        "",
    ]
    for name, fields in structs():
        out.append(f"pub const {name} = extern struct {{")
        out += [f"    {f.split('[')[0]}: {zig_field(t, f)}," for t, f in fields]
        out += ["};", ""]
    for ret, name, args in declarations():
        zargs = ", ".join(f"{n.split('[')[0]}: {zig_type(t, n)}" for t, n in args)
        out.append(f"pub extern fn {name}({zargs}) {RET[ret]};")
    out += [
        "",
        "/// C API code -> the error set of the kernel-level boundary it replaces (src/simdKernels.zig:30-37)",
        "pub fn toError(rc: i32) ?@import(\"../Sgp4.zig\").Error {",
        "    return switch (rc) {",
        "        0 => null,",
        "        -12 => error.SatelliteDecayed,",
        "        -11 => error.InvalidEccentricity,",
        "        -10 => error.DeepSpaceNotSupported,",
        "        else => error.OutOfMemory, // -100 alloc, -200 CUDA, -201 no device: no CPU fallback is attempted",
        "    };",
        "}",
        "",
    ]
    return "\n".join(out)


def main() -> None:
    text = render()
    if "--check" in sys.argv:
        cur = open(OUT).read() if os.path.exists(OUT) else ""
        if cur != text:
            raise SystemExit("zig/src/c_api/cuda.zig is out of date: run python tools/gen_zig_bindings.py")
        return
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    with open(OUT, "w") as f:
        f.write(text)
    print(f"wrote {OUT}")


if __name__ == "__main__":
    main()
