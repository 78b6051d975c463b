"""ctypes binding of libastroz_b200.so (include/astroz_b200.h).

The CUDA library is the only propagation path.  If it has not been built, or no CUDA device is
visible when a propagation is requested, this module raises -- it never falls back to a CPU path.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# ASTROZ_B200_LIB points measurement tools at an alternative build of the SAME library (tools/variant_sweep.sh);
# there is no other implementation to fall back to
LIB_PATH = os.environ.get("ASTROZ_B200_LIB") or os.path.join(_HERE, "libastroz_b200.so")

OK = 0
ERROR_NAMES = {
    0: "ok", -1: "badTleLength", -2: "badChecksum", -10: "deepSpaceNotSupported", -11: "invalidEccentricity",
    -12: "satelliteDecayed", -20: "valueError", -100: "allocFailed", -101: "nullPointer", -102: "notInitialized",
    -999: "unknown", -200: "cudaError", -201: "noCudaDevice",
}
# python-sgp4 error numbers (bindings/python/src/shared.zig:40-47)
SGP4_ERROR = {-11: 1, -10: 3, -100: 4, -12: 6}

MODE_TEME, MODE_ECEF, MODE_GEODETIC = 0, 1, 2
LAYOUT_SATELLITE_MAJOR, LAYOUT_TIME_MAJOR = 0, 1
WGS84, WGS72 = 0, 1


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
    dp = C.POINTER(C.c_double)
    vp = C.c_void_p
    u32, i32 = C.c_uint32, C.c_int32
    sig = {
        "astroz_cuda_version": (u32, []),
        "astroz_cuda_device_count": (i32, []),
        "astroz_cuda_last_error": (C.c_char_p, []),
        "astroz_cuda_host_alloc": (vp, [C.c_size_t]),
        "astroz_cuda_host_free": (None, [vp]),
        "astroz_cuda_host_register": (i32, [vp, C.c_size_t]),
        "astroz_cuda_host_unregister": (i32, [vp]),
        "astroz_cuda_constellation_create": (i32, [C.POINTER(C.c_char_p), C.POINTER(C.c_char_p), u32, i32, i32,
                                                   C.POINTER(vp)]),
        "astroz_cuda_constellation_create_from_text": (i32, [C.c_char_p, C.c_size_t, i32, i32, C.POINTER(vp)]),
        "astroz_cuda_constellation_create_from_elements": (i32, [dp, dp, dp, dp, dp, dp, dp, dp, u32, i32, i32,
                                                                 C.POINTER(vp)]),
        "astroz_cuda_constellation_create_from_elements_device": (i32, [vp, vp, vp, vp, vp, vp, vp, vp, u32, i32, i32,
                                                                        C.POINTER(vp)]),
        "astroz_cuda_constellation_free": (None, [vp]),
        "astroz_cuda_constellation_counts": (i32, [vp, C.POINTER(u32), C.POINTER(u32), C.POINTER(u32)]),
        "astroz_cuda_constellation_epochs": (i32, [vp, dp]),
        "astroz_cuda_constellation_classes": (i32, [vp, C.POINTER(i32)]),
        "astroz_cuda_constellation_get_reference_epoch": (i32, [vp, dp]),
        "astroz_cuda_constellation_set_reference_epoch": (i32, [vp, C.c_double]),
        "astroz_cuda_constellation_propagate": (i32, [vp, dp, dp, u32, dp, dp, i32, i32]),
        "astroz_cuda_constellation_propagate_device": (i32, [vp, dp, dp, u32, vp, vp, vp, i32, i32, u32, u32, vp]),
        "astroz_cuda_constellation_propagate_gather": (i32, [vp, dp, dp, u32, C.POINTER(vp), C.POINTER(vp), u32, vp, vp,
                                                             u32, u32, vp]),
        "astroz_cuda_constellation_propagate_device_f32": (i32, [vp, dp, dp, u32, vp, vp, i32, vp]),
        "astroz_cuda_constellation_propagate_pairs": (i32, [vp, vp, dp, dp, u32, i32, dp, dp, vp]),
        "astroz_cuda_constellation_propagate_pairs_device": (i32, [vp, vp, vp, vp, u32, i32, vp, vp, vp, vp]),
        "astroz_cuda_constellation_reset_carry": (i32, [vp]),
        "astroz_cuda_constellation_synchronize": (i32, [vp]),
        "astroz_cuda_constellation_last_kernel_ms": (i32, [vp, C.POINTER(C.c_float)]),
        "astroz_cuda_constellation_set_timing": (i32, [vp, i32]),
        "astroz_cuda_constellation_host_block": (i32, [vp, u32, i32, C.POINTER(vp)]),
        "astroz_cuda_sgp4_propagate_into": (i32, [vp, dp, u32, dp, dp, dp, i32, C.c_double, i32, vp, u32]),
        "astroz_cuda_sgp4_propagate_into_device": (i32, [vp, dp, u32, dp, vp, vp, i32, C.c_double, i32, vp, u32, vp]),
        "astroz_cuda_sdp4_propagate_into": (i32, [vp, dp, dp, u32, dp, dp, i32, i32, u32, u32]),
        "astroz_cuda_sdp4_propagate_into_device": (i32, [vp, dp, dp, u32, vp, vp, i32, i32, u32, u32, vp]),
        "astroz_cuda_sgp4_screen": (i32, [vp, dp, u32, dp, u32, C.c_double, C.c_double, dp, C.POINTER(u32)]),
        "astroz_cuda_constellation_coarse_screen_device": (i32, [vp, vp, u32, u32, i32, C.c_double, vp, vp, vp, u32,
                                                                 C.POINTER(C.c_uint64)]),
        "astroz_cuda_sgp4_screen_all": (i32, [vp, dp, u32, dp, C.c_double, C.POINTER(u32), C.POINTER(u32), u32,
                                              C.POINTER(C.c_uint64)]),
        "astroz_cuda_sgp4_init": (i32, [C.c_char_p, C.c_char_p, i32, i32, C.POINTER(vp)]),
        "astroz_cuda_sgp4_free": (None, [vp]),
        "astroz_cuda_sgp4_is_deep_space": (i32, [vp]),
        "astroz_cuda_sgp4_epoch": (i32, [vp, dp]),
        "astroz_cuda_sgp4_elements": (i32, [vp, dp]),
        "astroz_cuda_sgp4_propagate": (i32, [vp, C.c_double, dp, dp]),
        "astroz_cuda_sgp4_propagate_batch": (i32, [vp, dp, dp, u32]),
        "astroz_cuda_sgp4_array": (i32, [vp, dp, dp, C.c_double, dp, u32]),
        "astroz_cuda_constellation_devices": (i32, [vp, C.POINTER(i32), C.POINTER(i32), C.POINTER(u32)]),
        "astroz_cuda_constellation_propagate_replicated": (i32, [vp, dp, dp, u32, i32, C.POINTER(vp), C.POINTER(vp)]),
        "astroz_cuda_numerical_times": (i32, [C.c_double, C.c_double, C.c_double, vp, C.POINTER(C.c_uint64)]),
        "astroz_cuda_propagate_numerical": (i32, [vp, u32, C.c_double, C.c_double, C.c_double, C.c_double, i32, dp, dp,
                                                  vp, vp, vp, i32, C.c_double, C.c_double, i32, vp, vp, vp]),
        "astroz_cuda_propagate_numerical_device": (i32, [vp, u32, C.c_double, C.c_double, C.c_double, C.c_double, i32,
                                                         dp, dp, vp, vp, vp, i32, C.c_double, C.c_double, i32, vp, vp,
                                                         vp, vp]),
        "astroz_cuda_propagate_numerical_models": (i32, [vp, u32, C.c_double, C.c_double, C.c_double, vp, u32, i32,
                                                         C.c_double, C.c_double, i32, vp, vp, vp]),
        "astroz_cuda_propagate_numerical_models_device": (i32, [vp, u32, C.c_double, C.c_double, C.c_double, vp, u32,
                                                                i32, C.c_double, C.c_double, i32, vp, vp, vp, vp]),
        "astroz_cuda_propagate_maneuvers": (i32, [vp, u32, C.c_double, C.c_double, C.c_double, C.c_double, vp, vp,
                                                  u32, vp, u32, i32, C.c_double, C.c_double, u32, i32, vp, vp, vp, vp,
                                                  vp]),
        "astroz_cuda_propagate_maneuvers_device": (i32, [vp, u32, C.c_double, C.c_double, C.c_double, C.c_double, vp,
                                                         vp, u32, vp, u32, i32, C.c_double, C.c_double, u32, i32, vp, vp,
                                                         vp, vp, vp, vp]),
        "astroz_cuda_fit_elements": (i32, [vp, u32, i32, vp, vp, vp, vp, vp, u32, C.c_double, C.c_double, i32, u32,
                                           i32, vp, vp, vp, vp]),
        "astroz_cuda_fit_elements_device": (i32, [vp, u32, i32, vp, vp, vp, vp, vp, C.c_double, C.c_double, i32, u32,
                                                  i32, vp, vp, vp, vp, vp]),
        "astroz_cuda_fit_elements_mixed": (i32, [vp, u32, i32, vp, vp, vp, vp, vp, u32, C.c_double, C.c_double, i32,
                                                 u32, i32, vp, vp, vp, vp]),
        "astroz_cuda_fit_elements_mixed_device": (i32, [vp, u32, i32, vp, vp, vp, vp, vp, C.c_double, C.c_double, i32,
                                                        u32, i32, vp, vp, vp, vp, vp]),
        "astroz_cuda_parse_tle": (i32, [C.c_char_p, C.c_char_p, dp]),
        "astroz_cuda_fp64_peak": (i32, [i32, dp]),
        "astroz_cuda_fp64_pipe_peak": (i32, [i32, dp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)  # AttributeError here = header/library mismatch: fail loudly
        fn.restype = res
        fn.argtypes = args
    _lib = L
    return L


EXPORTS = [
    "astroz_cuda_version", "astroz_cuda_device_count", "astroz_cuda_last_error", "astroz_cuda_host_alloc",
    "astroz_cuda_host_free", "astroz_cuda_constellation_create", "astroz_cuda_constellation_create_from_text",
    "astroz_cuda_constellation_create_from_elements", "astroz_cuda_constellation_create_from_elements_device",
    "astroz_cuda_constellation_free",
    "astroz_cuda_constellation_counts", "astroz_cuda_constellation_epochs",
    "astroz_cuda_constellation_classes", "astroz_cuda_constellation_get_reference_epoch",
    "astroz_cuda_constellation_set_reference_epoch", "astroz_cuda_constellation_propagate",
    "astroz_cuda_constellation_propagate_device", "astroz_cuda_constellation_propagate_gather",
    "astroz_cuda_constellation_propagate_device_f32", "astroz_cuda_constellation_reset_carry",
    "astroz_cuda_constellation_synchronize", "astroz_cuda_constellation_last_kernel_ms",
    "astroz_cuda_sgp4_propagate_into", "astroz_cuda_sgp4_propagate_into_device", "astroz_cuda_sdp4_propagate_into",
    "astroz_cuda_sdp4_propagate_into_device", "astroz_cuda_sgp4_screen",
    "astroz_cuda_constellation_coarse_screen_device", "astroz_cuda_sgp4_screen_all", "astroz_cuda_sgp4_init",
    "astroz_cuda_sgp4_free", "astroz_cuda_sgp4_is_deep_space", "astroz_cuda_sgp4_epoch", "astroz_cuda_sgp4_elements",
    "astroz_cuda_sgp4_propagate", "astroz_cuda_sgp4_propagate_batch", "astroz_cuda_sgp4_array",
    "astroz_cuda_fp64_peak", "astroz_cuda_fp64_pipe_peak", "astroz_cuda_constellation_devices",
    "astroz_cuda_constellation_propagate_replicated", "astroz_cuda_host_register", "astroz_cuda_host_unregister",
    "astroz_cuda_constellation_set_timing", "astroz_cuda_constellation_host_block",
    "astroz_cuda_constellation_propagate_pairs", "astroz_cuda_constellation_propagate_pairs_device",
    "astroz_cuda_numerical_times", "astroz_cuda_propagate_numerical", "astroz_cuda_propagate_numerical_device",
    "astroz_cuda_propagate_numerical_models", "astroz_cuda_propagate_numerical_models_device",
    "astroz_cuda_propagate_maneuvers", "astroz_cuda_propagate_maneuvers_device",
    "astroz_cuda_fit_elements", "astroz_cuda_fit_elements_device", "astroz_cuda_fit_elements_mixed",
    "astroz_cuda_fit_elements_mixed_device", "astroz_cuda_parse_tle",
]


def check(code: int) -> None:
    if code != OK:
        detail = lib().astroz_cuda_last_error().decode(errors="replace") if code <= -200 else ""
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
            raise AstrozCudaError(-100, "cudaMallocHost failed")
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
        raise AstrozCudaError(-201, "no CUDA device visible; astroz_b200 has no CPU propagation path")
