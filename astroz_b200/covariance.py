"""Carry a fitted element set's covariance to state covariances at any time, on the device (K10,
astroz_b200/csrc/az_covariance.cu).

    from astroz_b200.covariance import propagate_covariance, RTN
    fit = fit_observations(...)                           # FitResult with covariance and deep_space
    res = propagate_covariance(fit, sat, jd, fr, frame=RTN)
    res.state, res.matrix(i), res.status

For each (satellite, time) query: the nominal TEME state of the fit's model, the Jacobian J of that state with respect
to the fit's variables (the forward differences the fit itself forms), and Sigma = J P J^T in TEME or in the RTN frame
of the nominal state.  P is the fit's formal covariance, or any positive semi-definite 7 x 7 matrix in the same
variables: a B* variance added where the fit held B*, an inflated P, an a-priori covariance.  The linear model is the
fit's: far from the data the along-track error grows curved and Sigma underestimates it (DESIGN §3, K10).

Deep-space rows fitted with B* free: SDP4's drag barely moves those orbits, so their B* Jacobian column is rounding
noise and the fit's B* variance is huge; Sigma is then dominated by their product.  Zero the B* row and column of P for
such rows, or put in a B* variance of your own.

A module of its own rather than part of fit.py: it consumes a fit's output (or any covariance in the fit's variables)
and is used where fits are not run, at screening and tasking time.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from ._abi import DEFINES as D
from ._lib import WGS72, check, lib

OK, INIT_FAILED, CELL_FAILED = D["ASTROZ_COV_OK"], D["ASTROZ_COV_INIT_FAILED"], D["ASTROZ_COV_CELL_FAILED"]
STATUS_NAMES = {OK: "ok", INIT_FAILED: "a set cannot be built under the row's model",
                CELL_FAILED: "a deep-space cell failed (decay, eccentricity)"}
TEME, RTN = D["ASTROZ_COV_FRAME_TEME"], D["ASTROZ_COV_FRAME_RTN"]
_WORDS = D["ASTROZ_STATE_COVARIANCE_WORDS"]
_P_WORDS = D["ASTROZ_FIT_COVARIANCE_WORDS"]
_TRIU6 = np.triu_indices(6)
_TRIU7 = np.triu_indices(7)


@dataclass
class CovarianceResult:
    state: np.ndarray            # (m, 6) nominal TEME state [km, km/s]
    covariance: np.ndarray       # (m, 21) upper triangle of Sigma, row by row, in the requested frame
    jacobian: np.ndarray | None  # (m, 6, 7) d(state) / d(fit variables) in the requested frame, or None
    status: np.ndarray           # (m,) uint8 ASTROZ_COV_*

    def matrix(self, i: int) -> np.ndarray:
        """The 6 x 6 Sigma of query i [km^2, km^2/s, km^2/s^2]"""
        S = np.zeros((6, 6))
        S[_TRIU6] = self.covariance[i]
        return S + np.triu(S, 1).T


def _covariance_words(cov, n: int) -> np.ndarray:
    c = np.asarray(cov, dtype=np.float64)
    if c.shape == (n, 7, 7):
        c = c[:, _TRIU7[0], _TRIU7[1]]
    if c.shape != (n, _P_WORDS):
        raise ValueError(f"covariance must be (n, {_P_WORDS}) upper-triangle words or (n, 7, 7) matrices, n = {n}")
    return np.ascontiguousarray(c)


def propagate_covariance(source, sat, jd, fr, *, covariance=None, model=None, frame: int = TEME,
                         jacobian: bool = False, grav: int = WGS72, device: int = 0) -> CovarianceResult:
    """State covariance of m queries (astroz_cuda_propagate_covariance).

    source: a FitResult (elements, covariance and deep_space are taken from it; covariance= or model= override them)
    or an (8, n) array of element columns with covariance= (n, 28) words or (n, 7, 7) matrices in the fit's variables
    and model= (n,) 0 / 1 or bool (1: the deep-space equinoctial variables; default all 0).  Query i: satellite sat[i]
    at jd[i] + fr[i] (jd and fr broadcast to sat), in any order; results come back in that order."""
    if hasattr(source, "elements") and hasattr(source, "deep_space"):
        el = np.ascontiguousarray(source.elements, dtype=np.float64)
        covariance = source.covariance if covariance is None else covariance
        model = source.deep_space if model is None else model
        if covariance is None:
            raise ValueError("this FitResult has no covariance (fit_observations returns one)")
    else:
        el = np.ascontiguousarray(source, dtype=np.float64)
        if el.ndim != 2 or el.shape[0] != 8:
            raise ValueError("source must be a FitResult or an (8, n) array of element columns")
        if covariance is None:
            raise ValueError("covariance= is required with an element array")
    n = el.shape[1]
    cov = _covariance_words(covariance, n)
    md = None
    if model is not None:
        mm = np.asarray(model).reshape(-1)
        if len(mm) != n or (mm.size and (mm.min() < 0 or mm.max() > 1)):
            raise ValueError("model must hold n values, 0 (near-earth) or 1 (deep space)")
        md = np.ascontiguousarray(mm.astype(np.uint8))
    sat = np.asarray(sat).reshape(-1)
    if sat.size and (not np.issubdtype(sat.dtype, np.integer) or sat.min() < 0 or sat.max() >= n):
        raise ValueError("sat must hold satellite indices in [0, n)")
    m = len(sat)
    jd_ = np.broadcast_to(np.asarray(jd, dtype=np.float64), (m,))
    fr_ = np.broadcast_to(np.asarray(fr, dtype=np.float64), (m,))
    order = np.argsort(sat, kind="stable")
    offsets = np.searchsorted(sat[order], np.arange(n + 1)).astype(np.uint32)
    jd_s, fr_s = np.ascontiguousarray(jd_[order]), np.ascontiguousarray(fr_[order])
    st, sig, stat = np.zeros((m, 6)), np.zeros((m, _WORDS)), np.zeros(m, dtype=np.uint8)
    jac = np.zeros((m, 6, 7)) if jacobian else None
    vp = lambda a: None if a is None or a.size == 0 else C.c_void_p(a.ctypes.data)  # noqa: E731
    check(lib().astroz_cuda_propagate_covariance(vp(el), n, int(grav), vp(cov), vp(md), vp(offsets), vp(jd_s),
                                                 vp(fr_s), m, int(frame), int(device), vp(st), vp(sig), vp(jac),
                                                 vp(stat)))
    out = CovarianceResult(np.empty_like(st), np.empty_like(sig), None if jac is None else np.empty_like(jac),
                           np.empty_like(stat))
    out.state[order], out.covariance[order], out.status[order] = st, sig, stat
    if jac is not None:
        out.jacobian[order] = jac
    return out


def propagate_covariance_device(elements, covariance, model, offsets, jd, fr, state, state_covariance, jacobian,
                                status, *, frame: int = TEME, grav: int = WGS72, stream: int = 0) -> None:
    """`propagate_covariance` with torch CUDA tensors on one device, queries grouped by satellite: elements (8, n)
    float64, covariance (n, 28) float64, model (n,) uint8 or None, offsets (n + 1,) int32 (offsets[0] = 0, non-
    decreasing, offsets[n] = m), jd / fr (m,) float64; state (m, 6) float64 or None, state_covariance (m, 21) float64,
    jacobian (m, 6, 7) float64 or None and status (m,) uint8 receive the results.  Two launches on `stream` (a raw
    cudaStream_t value, 0 = the default stream), one when model is None."""
    import torch

    n = int(elements.shape[1]) if elements.dim() == 2 and elements.shape[0] == 8 else -1
    if n < 0 or elements.dtype != torch.float64 or not elements.is_cuda:
        raise ValueError("elements must be a CUDA float64 tensor of shape (8, n)")
    m = int(jd.numel())
    tensors = [("elements", elements, 8 * n, torch.float64), ("covariance", covariance, _P_WORDS * n, torch.float64),
               ("model", model, n, torch.uint8), ("offsets", offsets, n + 1, torch.int32),
               ("jd", jd, m, torch.float64), ("fr", fr, m, torch.float64), ("state", state, 6 * m, torch.float64),
               ("state_covariance", state_covariance, _WORDS * m, torch.float64),
               ("jacobian", jacobian, 42 * m, torch.float64), ("status", status, m, torch.uint8)]
    for name, t, size, dtype in tensors:
        if t is None and name in ("model", "state", "jacobian"):
            continue
        if not isinstance(t, torch.Tensor) or t.dtype != dtype or not t.is_contiguous() or int(t.numel()) != size \
                or t.device != elements.device:
            raise ValueError(f"{name} must be a contiguous {dtype} tensor of {size} elements on {elements.device}")
    ptr = lambda t: None if t is None else C.c_void_p(t.data_ptr())  # noqa: E731
    check(lib().astroz_cuda_propagate_covariance_device(
        ptr(elements), n, int(grav), ptr(covariance), ptr(model), ptr(offsets), ptr(jd), ptr(fr), m, int(frame),
        int(elements.device.index), ptr(state), ptr(state_covariance), ptr(jacobian), ptr(status),
        C.c_void_p(stream) if stream else None))
