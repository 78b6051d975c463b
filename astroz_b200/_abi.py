"""The C ABI of libastroz_b200.so as include/astroz_b200.h states it.

The header is the one statement of the ABI.  This module reads its function declarations, its `typedef struct` blocks
and its integer `#define ASTROZ_*` constants, and maps C types to ctypes.  The ctypes binding (_lib), the constants and
descriptor layouts of the wrappers, and tools/gen_zig_bindings.py (the Zig binding) are built from what it reads, so
none of them restates the header.
"""
from __future__ import annotations

import ctypes as C
import os
import re

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "astroz_b200.h")


def _uncommented(header: str) -> str:
    if not os.path.exists(header):
        raise ImportError(f"{header} is missing: astroz_b200 reads its C ABI (signatures, constants, structs) from it")
    with open(header) as f:
        return re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)


def declarations(header: str = HEADER):
    """Every `astroz_cuda_*` function of the header, as (return type, name, [(ctype, parameter)])"""
    text = re.sub(r"#[^\n]*", "", _uncommented(header))
    for m in re.finditer(r"([\w \*]+?)\b(astroz_cuda_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", text, flags=re.S):
        ret = " ".join(m.group(1).split())
        ret = ret if not ret.endswith("*") else ret[:-1].strip() + " *"
        args = []
        raw = " ".join(m.group(3).split())
        if raw and raw != "void":
            for a in raw.split(","):
                a = a.strip()
                mm = re.match(r"(.*?)(\w+(?:\[\d+\])?)$", a)
                ctype, name = mm.group(1).strip(), mm.group(2)
                args.append((ctype, name))
        yield ret, m.group(2), args


def structs(header: str = HEADER):
    """`typedef struct { <type> <name>; ... } name;` blocks of the header, as (name, [(ctype, field)])"""
    text = _uncommented(header)
    for m in re.finditer(r"typedef struct \{([^}]*)\}\s*(\w+)\s*;", text):
        fields = []
        for decl in m.group(1).split(";"):
            decl = " ".join(decl.split())
            if decl:
                mm = re.match(r"(.*?)(\w+(?:\[\d+\])?)$", decl)
                fields.append((mm.group(1).strip(), mm.group(2)))
        yield m.group(2), fields


def defines(header: str = HEADER) -> dict[str, int]:
    """The integer `#define ASTROZ_*` constants of the header, written 0, (-20) or 1u"""
    pattern = r"^#define\s+(ASTROZ_\w+)\s+\(?\s*(-?\d+)u?\s*\)?[ \t]*$"
    return {m.group(1): int(m.group(2)) for m in re.finditer(pattern, _uncommented(header), flags=re.M)}


DEFINES = defines()

_SCALARS = {"int32_t": C.c_int32, "uint32_t": C.c_uint32, "size_t": C.c_size_t, "double": C.c_double}
_RETURNS = {"void": None, "void *": C.c_void_p, "const char *": C.c_char_p}
_HANDLES = ("astroz_constellation_t", "astroz_sgp4_t")


def _scalar(ctype: str, where: str):
    if ctype not in _SCALARS:
        raise TypeError(f"astroz_b200: no ctypes mapping for C type '{ctype}' ({where})")
    return _SCALARS[ctype]


def restype(ctype: str, function: str):
    return _RETURNS[ctype] if ctype in _RETURNS else _scalar(ctype, f"return value of {function}")


def argtype(ctype: str, name: str, function: str):
    """A C string is c_char_p; every other pointer, array or handle parameter is c_void_p, which takes what the wrappers
    pass: ctypes pointers and arrays, byref(...), integer addresses and None."""
    if ctype == "const char *":
        return C.c_char_p
    if ctype.endswith("*") or name.endswith("]") or ctype in _HANDLES:
        return C.c_void_p
    return _scalar(ctype, f"parameter {name} of {function}")


def structure(name: str) -> type[C.Structure]:
    """The ctypes Structure of the header's `typedef struct {...} name;`: pointer fields are c_void_p"""
    def field(ctype, decl):
        base, _, count = decl.partition("[")
        t = C.c_void_p if ctype.endswith("*") else _scalar(ctype, f"field {base} of {name}")
        return base, (t * int(count[:-1]) if count else t)

    return type(name, (C.Structure,), {"_fields_": [field(t, f) for t, f in dict(structs())[name]]})
