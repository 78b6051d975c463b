"""ctypes binding of libastroz_b200.so (include/astroz_b200.h).

The CUDA library is the only propagation path.  If it has not been built, or no CUDA device is
visible when a propagation is requested, this module raises -- it never falls back to a CPU path.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import _abi
from ._abi import DEFINES as D

_HERE = os.path.dirname(os.path.abspath(__file__))
# ASTROZ_B200_LIB points measurement tools at an alternative build of the SAME library (tools/variant_sweep.sh);
# there is no other implementation to fall back to
LIB_PATH = os.environ.get("ASTROZ_B200_LIB") or os.path.join(_HERE, "libastroz_b200.so")

OK = D["ASTROZ_OK"]
# the reference's error names (src/c_api/error.zig:3-19, + the CUDA codes)
ERROR_NAMES = {
    D["ASTROZ_OK"]: "ok", D["ASTROZ_BAD_TLE_LENGTH"]: "badTleLength", D["ASTROZ_BAD_CHECKSUM"]: "badChecksum",
    D["ASTROZ_DEEP_SPACE"]: "deepSpaceNotSupported", D["ASTROZ_INVALID_ECC"]: "invalidEccentricity",
    D["ASTROZ_DECAYED"]: "satelliteDecayed", D["ASTROZ_VALUE_ERROR"]: "valueError",
    D["ASTROZ_ALLOC_FAILED"]: "allocFailed", D["ASTROZ_NULL_POINTER"]: "nullPointer",
    D["ASTROZ_NOT_INITIALIZED"]: "notInitialized", D["ASTROZ_UNKNOWN"]: "unknown", D["ASTROZ_CUDA_ERROR"]: "cudaError",
    D["ASTROZ_NO_DEVICE"]: "noCudaDevice",
}
# python-sgp4 error numbers (bindings/python/src/shared.zig:40-47)
SGP4_ERROR = {D["ASTROZ_INVALID_ECC"]: 1, D["ASTROZ_DEEP_SPACE"]: 3, D["ASTROZ_ALLOC_FAILED"]: 4,
              D["ASTROZ_DECAYED"]: 6}

WGS84, WGS72 = D["ASTROZ_WGS84"], D["ASTROZ_WGS72"]

# every function the header declares, as (return type, name, [(ctype, parameter)]): lib() binds exactly these
_DECLARATIONS = list(_abi.declarations())
EXPORTS = [name for _, name, _ in _DECLARATIONS]


class AstrozCudaError(RuntimeError):
    def __init__(self, code: int, detail: str = ""):
        self.code = code
        name = ERROR_NAMES.get(code, "unknown")
        super().__init__(f"astroz_b200: {name} ({code})" + (f": {detail}" if detail else ""))


_lib = None


def lib() -> C.CDLL:
    """Load the CUDA library; loud failure if it is missing (no CPU fallback exists)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -m astroz_b200.build` "
            "(astroz_b200 has no CPU propagation path)")
    L = C.CDLL(LIB_PATH)
    for ret, name, args in _DECLARATIONS:
        fn = getattr(L, name)  # AttributeError here = header/library mismatch: fail loudly
        fn.restype = _abi.restype(ret, name)
        fn.argtypes = [_abi.argtype(t, a, name) for t, a in args]
    _lib = L
    return L


def check(code: int) -> None:
    if code != OK:
        detail = lib().astroz_cuda_last_error().decode(errors="replace") if code <= D["ASTROZ_CUDA_ERROR"] else ""
        raise AstrozCudaError(code, detail)


def dptr(a: np.ndarray):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def as_f64(x) -> np.ndarray:
    return np.ascontiguousarray(np.atleast_1d(np.asarray(x, dtype=np.float64)))


class _PinnedPool:
    """Recycles cudaMallocHost blocks: page-locking is expensive (tens of ms per call, and cudaFreeHost
    synchronises the device), while the python-sgp4 style API returns freshly allocated arrays on every
    call.  Blocks whose arrays were garbage-collected are kept (up to ASTROZ_PINNED_POOL_MB, default 4096)
    and handed out again for requests of a similar size."""

    def __init__(self):
        self.free: list[tuple[int, int]] = []   # (nbytes, ptr)
        self.held = 0
        self.cap = int(os.environ.get("ASTROZ_PINNED_POOL_MB", "4096")) << 20

    def get(self, nbytes: int) -> tuple[int, int]:
        best = None
        for i, (sz, _) in enumerate(self.free):
            if sz >= nbytes and sz <= nbytes + (nbytes >> 2) + 4096 and (best is None or sz < self.free[best][0]):
                best = i
        if best is not None:
            sz, ptr = self.free.pop(best)
            self.held -= sz
            return sz, ptr
        ptr = lib().astroz_cuda_host_alloc(nbytes)
        if not ptr and self.free:       # make room and retry once
            self.trim(0)
            ptr = lib().astroz_cuda_host_alloc(nbytes)
        if not ptr:
            raise AstrozCudaError(D["ASTROZ_ALLOC_FAILED"], "cudaMallocHost failed")
        return nbytes, ptr

    def put(self, nbytes: int, ptr: int) -> None:
        if nbytes > self.cap:
            lib().astroz_cuda_host_free(ptr)
            return
        self.free.append((nbytes, ptr))
        self.held += nbytes
        self.trim(self.cap)

    def trim(self, limit: int) -> None:
        while self.free and self.held > limit:
            sz, ptr = self.free.pop(0)
            self.held -= sz
            lib().astroz_cuda_host_free(ptr)


_POOL = _PinnedPool()


class _PinnedBlock:
    """One cudaMallocHost block exposed through the array interface; returned to the pool when the last
    ndarray viewing it is collected."""

    def __init__(self, nbytes: int):
        nbytes = max(int(nbytes), 8)
        self.nbytes, self.ptr = _POOL.get(nbytes)
        self.__array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (self.ptr, False), "version": 3}

    def __del__(self):
        if getattr(self, "ptr", None):
            try:
                _POOL.put(self.nbytes, self.ptr)
            except Exception:
                pass
            self.ptr = None


def pinned_empty(shape, dtype=np.float64) -> np.ndarray:
    """np.empty in page-locked host memory, so device->host copies run at full PCIe rate."""
    dtype = np.dtype(dtype)
    shape = tuple(int(x) for x in shape)
    n = int(np.prod(shape)) if shape else 1
    block = _PinnedBlock(n * dtype.itemsize)
    return np.asarray(block)[: n * dtype.itemsize].view(dtype).reshape(shape)


def host_register(a: np.ndarray) -> None:
    """Page-lock a caller-owned array in place (cudaHostRegister) so results reach it by direct DMA; undo with
    host_unregister before the array is freed."""
    check(lib().astroz_cuda_host_register(C.c_void_p(a.ctypes.data), a.nbytes))


def host_unregister(a: np.ndarray) -> None:
    check(lib().astroz_cuda_host_unregister(C.c_void_p(a.ctypes.data)))


def device_count() -> int:
    return int(lib().astroz_cuda_device_count())


def require_device() -> None:
    if device_count() <= 0:
        raise AstrozCudaError(D["ASTROZ_NO_DEVICE"],
                              "no CUDA device visible; astroz_b200 has no CPU propagation path")
