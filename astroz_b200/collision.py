"""Assess candidate conjunctions on the device: time of closest approach, miss, relative state and the 2-D probability of
collision from both objects' fitted covariances (K11, astroz_b200/csrc/az_conjunction.cu).

    from astroz_b200.collision import conjunctions
    fit = fit_observations(...)                                   # FitResult with covariance and deep_space
    res = conjunctions(fit, primary, secondary, jd, fr, window_min=2.0, hbr_km=0.02)
    res.tca_jd, res.tca_fr, res.miss_km, res.pc, res.c2, res.status

Candidates are inputs: pairs of catalogue rows with a guess time and a half window, from any screen, a conjunction
message or the caller's own logic; this module does not search for encounters.  For each candidate the TCA is the local
minimum of the range inside the window, each object's state covariance comes from K10 (astroz_b200.covariance) at the
TCA, and Pc is the short-encounter 2-D integral over the combined hard-body disk in the encounter plane, with the two
objects' errors taken as uncorrelated.  For slow encounters (GEO pairs) the short-encounter assumption fails and Pc is
not the collision probability.

`monte_carlo` (K14) makes no such assumption: it draws both objects' element sets from their covariances, finds each
drawn pair's own TCA with the same search and counts the draws that come within the hard-body radius.

    mc = monte_carlo(fit, primary, secondary, jd, fr, window_min=30.0, hbr_km=0.02, samples=10**7, seed=1)
    mc.pc, mc.interval(), mc.hits, mc.failed

`importance_sampling` (K15) moves the same draws onto the linearised collision point and weights each by its exact
likelihood ratio, which reaches the Pc values of 1e-5 to 1e-10 that plain sampling cannot afford.

    r = importance_sampling(fit, primary, secondary, jd, fr, window_min=2.0, hbr_km=0.02, samples=10**6, seed=1)
    r.pc, r.std_error, r.interval(), r.kind
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from ._abi import DEFINES as D
from ._lib import WGS72, check, lib
from .covariance import RTN, TEME, _covariance_words  # noqa: F401  (frames re-exported for callers)

OK, INIT_FAILED, CELL_FAILED = D["ASTROZ_CONJ_OK"], D["ASTROZ_CONJ_INIT_FAILED"], D["ASTROZ_CONJ_CELL_FAILED"]
WINDOW_EDGE, NO_PLANE, BAD_PAIR = D["ASTROZ_CONJ_WINDOW_EDGE"], D["ASTROZ_CONJ_NO_PLANE"], D["ASTROZ_CONJ_BAD_PAIR"]
STATUS_NAMES = {OK: "ok", INIT_FAILED: "a set cannot be built under the row's model",
                CELL_FAILED: "a deep-space cell failed (decay, eccentricity)",
                WINDOW_EDGE: "no minimum inside the window: the nearer window end",
                NO_PLANE: "zero relative velocity: no encounter plane", BAD_PAIR: "bad row pair"}
_WORDS = D["ASTROZ_CONJ_RECORD_WORDS"]
_SIG = D["ASTROZ_STATE_COVARIANCE_WORDS"]


def _catalogue(source, covariance, model):
    """(elements (8, n), covariance words (n, 28), model bytes (n,) or None) of a FitResult or an element array"""
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
    return el, cov, md


def _rows(primary, secondary, n):
    """the candidates' row indices as uint32 arrays, checked against n"""
    rows = []
    for name, a in (("primary", primary), ("secondary", secondary)):
        a = np.asarray(a).reshape(-1)
        if a.size and (not np.issubdtype(a.dtype, np.integer) or a.min() < 0 or a.max() >= n):
            raise ValueError(f"{name} must hold row indices in [0, n)")
        rows.append(np.ascontiguousarray(a.astype(np.uint32)))
    pr, se = rows
    if len(pr) != len(se):
        raise ValueError("primary and secondary must have the same length")
    return pr, se


@dataclass
class ConjunctionResult:
    record: np.ndarray                   # (m, 13) the raw record words (astroz_b200.h, K11)
    tca_jd: np.ndarray                   # (m,) the TCA as jd + fr: jd as given ...
    tca_fr: np.ndarray                   # (m,) ... and fr + dt_tca / 1440
    states: np.ndarray | None            # (m, 2, 6) TEME states of primary and secondary at the TCA, or None
    state_covariance: np.ndarray | None  # (m, 2, 21) each object's Sigma words at the TCA, or None
    status: np.ndarray                   # (m,) uint8 ASTROZ_CONJ_*

    dt_tca_min = property(lambda self: self.record[:, 0])
    miss_km = property(lambda self: self.record[:, 1])
    rel_speed_km_s = property(lambda self: self.record[:, 2])
    rel_position_rtn = property(lambda self: self.record[:, 3:6])   # secondary - primary, primary's RTN [km]
    rel_velocity_rtn = property(lambda self: self.record[:, 6:9])   # [km/s]
    pc = property(lambda self: self.record[:, 12])

    @property
    def c2(self) -> np.ndarray:
        """(m, 2, 2) combined position covariance in the encounter plane [km^2]"""
        xx, xy, yy = self.record[:, 9], self.record[:, 10], self.record[:, 11]
        return np.stack([np.stack([xx, xy], -1), np.stack([xy, yy], -1)], -2)


def conjunctions(source, primary, secondary, jd, fr, *, window_min, hbr_km, covariance=None, model=None,
                 frame: int = TEME, states: bool = False, grav: int = WGS72, device: int = 0) -> ConjunctionResult:
    """Assess m candidate conjunctions (astroz_cuda_conjunction).

    source: a FitResult (elements, covariance and deep_space are taken from it; covariance= or model= override them)
    or an (8, n) array of element columns with covariance= (n, 28) words or (n, 7, 7) matrices in the fit's variables
    and model= (n,) 0 / 1 or bool.  Candidate i: rows primary[i] != secondary[i] around jd[i] + fr[i], half window
    window_min [min] and combined hard-body radius hbr_km [km] (jd, fr, window_min and hbr_km broadcast to primary).
    frame chooses TEME or each object's own RTN for state_covariance; states=True also returns both TEME states."""
    el, cov, md = _catalogue(source, covariance, model)
    n = el.shape[1]
    pr, se = _rows(primary, secondary, n)
    m = len(pr)
    f64 = lambda a: np.ascontiguousarray(np.broadcast_to(np.asarray(a, dtype=np.float64), (m,)))  # noqa: E731
    jd_, fr_, w_, r_ = f64(jd), f64(fr), f64(window_min), f64(hbr_km)
    rec, stat = np.zeros((m, _WORDS)), np.zeros(m, dtype=np.uint8)
    st = np.zeros((m, 2, 6)) if states else None
    sig = np.zeros((m, 2, _SIG))
    vp = lambda a: None if a is None or a.size == 0 else C.c_void_p(a.ctypes.data)  # noqa: E731
    check(lib().astroz_cuda_conjunction(vp(el), n, int(grav), vp(cov), vp(md), vp(pr), vp(se), vp(jd_), vp(fr_),
                                        vp(w_), vp(r_), m, int(frame), int(device), vp(rec), vp(st), vp(sig),
                                        vp(stat)))
    return ConjunctionResult(rec, jd_.copy(), fr_ + rec[:, 0] / 1440.0, st, sig, stat)


def conjunctions_device(elements, covariance, model, primary, secondary, jd, fr, window_min, hbr_km, record, states,
                        state_covariance, status, *, frame: int = TEME, grav: int = WGS72, stream: int = 0) -> None:
    """`conjunctions` with torch CUDA tensors on one device: elements (8, n) float64, covariance (n, 28) float64, model
    (n,) uint8 or None, primary / secondary (m,) int32, jd / fr / window_min / hbr_km (m,) float64; record (m, 13)
    float64, states (m, 2, 6) float64 or None, state_covariance (m, 2, 21) float64 or None and status (m,) uint8
    receive the results.  Two launches on `stream` (a raw cudaStream_t value, 0 = the default stream).  Rows are not
    checked here: a bad pair gets status BAD_PAIR."""
    import torch

    n = int(elements.shape[1]) if elements.dim() == 2 and elements.shape[0] == 8 else -1
    if n < 0 or elements.dtype != torch.float64 or not elements.is_cuda:
        raise ValueError("elements must be a CUDA float64 tensor of shape (8, n)")
    m = int(primary.numel())
    tensors = [("elements", elements, 8 * n, torch.float64), ("covariance", covariance, 28 * n, torch.float64),
               ("model", model, n, torch.uint8), ("primary", primary, m, torch.int32),
               ("secondary", secondary, m, torch.int32), ("jd", jd, m, torch.float64), ("fr", fr, m, torch.float64),
               ("window_min", window_min, m, torch.float64), ("hbr_km", hbr_km, m, torch.float64),
               ("record", record, _WORDS * m, torch.float64), ("states", states, 12 * m, torch.float64),
               ("state_covariance", state_covariance, 2 * _SIG * m, torch.float64), ("status", status, m, torch.uint8)]
    for name, t, size, dtype in tensors:
        if t is None and name in ("model", "states", "state_covariance"):
            continue
        if not isinstance(t, torch.Tensor) or t.dtype != dtype or not t.is_contiguous() or int(t.numel()) != size \
                or t.device != elements.device:
            raise ValueError(f"{name} must be a contiguous {dtype} tensor of {size} elements on {elements.device}")
    ptr = lambda t: None if t is None else C.c_void_p(t.data_ptr())  # noqa: E731
    check(lib().astroz_cuda_conjunction_device(
        ptr(elements), n, int(grav), ptr(covariance), ptr(model), ptr(primary), ptr(secondary), ptr(jd), ptr(fr),
        ptr(window_min), ptr(hbr_km), m, int(frame), int(elements.device.index), ptr(record), ptr(states),
        ptr(state_covariance), ptr(status), C.c_void_p(stream) if stream else None))


# ---- Monte Carlo from epoch (K14, astroz_b200/csrc/az_conjunction_mc.cu) ----------------------------------------------
NOT_PSD = D["ASTROZ_CONJ_NOT_PSD"]
STATUS_NAMES[NOT_PSD] = "a covariance is not positive semidefinite"
_MC_COUNT = D["ASTROZ_CONJ_MC_COUNT_WORDS"]
_MC_SAMPLE = D["ASTROZ_CONJ_MC_SAMPLE_WORDS"]


@dataclass
class MonteCarloResult:
    hits: np.ndarray                  # (m,) uint64: samples whose miss at their TCA is below the radius
    edge: np.ndarray                  # (m,) uint64: samples whose search ended at a window end (scored all the same)
    failed: np.ndarray                # (m,) uint64: samples with a set that cannot be built or a failed cell
    samples: np.ndarray               # (m,) uint64: samples drawn
    status: np.ndarray                # (m,) uint8 ASTROZ_CONJ_*: OK, INIT_FAILED, NOT_PSD
    sample_dt: np.ndarray | None      # (m, record) dt_tca [min] of samples first .. first + record - 1 (NaN: none)
    sample_miss: np.ndarray | None    # (m, record) miss [km]

    @property
    def valid(self) -> np.ndarray:
        """samples scored: samples - failed, 0 for a candidate that is not OK"""
        v = self.samples.astype(np.float64) - self.failed.astype(np.float64)
        return np.where(self.status == OK, v, 0.0)

    @property
    def pc(self) -> np.ndarray:
        """hits / (samples - failed), NaN where no sample was scored"""
        v = self.valid
        with np.errstate(divide="ignore", invalid="ignore"):
            return np.where(v > 0, self.hits.astype(np.float64) / v, np.nan)

    def interval(self, z: float = 1.96) -> tuple[np.ndarray, np.ndarray]:
        """The Wilson score interval (lo, hi) of Pc at z standard errors: sensible at 0 hits, NaN with no sample"""
        n = self.valid
        with np.errstate(divide="ignore", invalid="ignore"):
            p = self.hits.astype(np.float64) / n
            d = 1.0 + z * z / n
            c = (p + z * z / (2.0 * n)) / d
            h = z * np.sqrt(p * (1.0 - p) / n + z * z / (4.0 * n * n)) / d
        bad = ~(n > 0)
        return np.where(bad, np.nan, np.maximum(c - h, 0.0)), np.where(bad, np.nan, np.minimum(c + h, 1.0))


def monte_carlo(source, primary, secondary, jd, fr, *, window_min, hbr_km, samples, seed=0, first=0, record: int = 0,
                covariance=None, model=None, grav: int = WGS72, device: int = 0) -> MonteCarloResult:
    """Monte Carlo collision probability of m candidate conjunctions (astroz_cuda_conjunction_mc).

    source, primary, secondary, jd, fr, window_min, hbr_km, covariance and model are those of `conjunctions`.  Each
    candidate draws samples k in [first, first + samples) of both objects' element sets from their covariances
    (Philox4x32-10 keyed by seed), finds each drawn pair's TCA in the window and counts the draws whose miss is below
    hbr_km.  samples, seed and first broadcast to primary.  record > 0 also returns the dt_tca and miss of the first
    `record` samples.  The draws depend on (seed, k) alone, so counts over [0, 2N) are those over [0, N) plus those
    over [N, 2N): extend a run by calling again with first = N and adding the counts (there is no adaptive stopping).
    Equal seeds give equal draws; pass different seeds for independent estimates."""
    el, cov, md = _catalogue(source, covariance, model)
    n = el.shape[1]
    pr, se = _rows(primary, secondary, n)
    m = len(pr)
    record = int(record)
    if record < 0:
        raise ValueError("record must be >= 0")
    f64 = lambda a: np.ascontiguousarray(np.broadcast_to(np.asarray(a, dtype=np.float64), (m,)))  # noqa: E731

    def u64(a, name):
        a = np.asarray(a)
        if a.size and (not np.issubdtype(a.dtype, np.integer) or a.min() < 0):
            raise ValueError(f"{name} must hold integers >= 0")
        return np.ascontiguousarray(np.broadcast_to(a.astype(np.uint64), (m,)))

    jd_, fr_, w_, r_ = f64(jd), f64(fr), f64(window_min), f64(hbr_km)
    ns, fi, sd = u64(samples, "samples"), u64(first, "first"), u64(seed, "seed")
    counts, stat = np.zeros((m, _MC_COUNT), np.uint64), np.zeros(m, dtype=np.uint8)
    out = np.zeros((m, record, _MC_SAMPLE)) if record else None
    vp = lambda a: None if a is None or a.size == 0 else C.c_void_p(a.ctypes.data)  # noqa: E731
    check(lib().astroz_cuda_conjunction_mc(vp(el), n, int(grav), vp(cov), vp(md), vp(pr), vp(se), vp(jd_), vp(fr_),
                                           vp(w_), vp(r_), vp(ns), vp(fi), vp(sd), m, record, int(device),
                                           vp(counts), vp(out), vp(stat)))
    return MonteCarloResult(counts[:, 0], counts[:, 1], counts[:, 2], ns.copy(), stat,
                            None if out is None else out[:, :, 0], None if out is None else out[:, :, 1])


def monte_carlo_scratch_bytes(m: int) -> int:
    """The scratch of monte_carlo_device for m candidates"""
    b = C.c_uint64(0)
    check(lib().astroz_cuda_conjunction_mc_scratch_bytes(int(m), C.byref(b)))
    return int(b.value)


def monte_carlo_device(elements, covariance, model, primary, secondary, jd, fr, window_min, hbr_km, samples, first,
                       seed, counts, sample_out, status, scratch, *, grav: int = WGS72, stream: int = 0) -> None:
    """`monte_carlo` with torch CUDA tensors on one device: elements (8, n) float64, covariance (n, 28) float64, model
    (n,) uint8 or None, primary / secondary (m,) int32, jd / fr / window_min / hbr_km (m,) float64, samples (m,)
    int64, first / seed (m,) int64 or None (0); counts (m, 3) int64 (hits, edge, failed), sample_out (m, record, 2)
    float64 or None and status (m,) uint8 receive the results; scratch a uint8 tensor of at least
    monte_carlo_scratch_bytes(m) bytes.  The launches go on `stream` (a raw cudaStream_t value, 0 = the default
    stream).  Rows are not checked here: a bad pair gets status BAD_PAIR."""
    import torch

    n = int(elements.shape[1]) if elements.dim() == 2 and elements.shape[0] == 8 else -1
    if n < 0 or elements.dtype != torch.float64 or not elements.is_cuda:
        raise ValueError("elements must be a CUDA float64 tensor of shape (8, n)")
    m = int(primary.numel())
    record = int(sample_out.shape[1]) if sample_out is not None and sample_out.dim() == 3 else 0
    tensors = [("elements", elements, 8 * n, torch.float64), ("covariance", covariance, 28 * n, torch.float64),
               ("model", model, n, torch.uint8), ("primary", primary, m, torch.int32),
               ("secondary", secondary, m, torch.int32), ("jd", jd, m, torch.float64), ("fr", fr, m, torch.float64),
               ("window_min", window_min, m, torch.float64), ("hbr_km", hbr_km, m, torch.float64),
               ("samples", samples, m, torch.int64), ("first", first, m, torch.int64), ("seed", seed, m, torch.int64),
               ("counts", counts, _MC_COUNT * m, torch.int64),
               ("sample_out", sample_out, _MC_SAMPLE * record * m, torch.float64), ("status", status, m, torch.uint8)]
    for name, t, size, dtype in tensors:
        if t is None and name in ("model", "first", "seed", "sample_out"):
            continue
        if not isinstance(t, torch.Tensor) or t.dtype != dtype or not t.is_contiguous() or int(t.numel()) != size \
                or t.device != elements.device:
            raise ValueError(f"{name} must be a contiguous {dtype} tensor of {size} elements on {elements.device}")
    if not isinstance(scratch, torch.Tensor) or not scratch.is_contiguous() or scratch.device != elements.device \
            or scratch.numel() * scratch.element_size() < monte_carlo_scratch_bytes(m):
        raise ValueError(f"scratch must be a contiguous tensor of monte_carlo_scratch_bytes({m}) bytes on "
                         f"{elements.device}")
    ptr = lambda t: None if t is None else C.c_void_p(t.data_ptr())  # noqa: E731
    check(lib().astroz_cuda_conjunction_mc_device(
        ptr(elements), n, int(grav), ptr(covariance), ptr(model), ptr(primary), ptr(secondary), ptr(jd), ptr(fr),
        ptr(window_min), ptr(hbr_km), ptr(samples), ptr(first), ptr(seed), m, record, int(elements.device.index),
        ptr(counts), ptr(sample_out), ptr(status), ptr(scratch), C.c_void_p(stream) if stream else None))


# ---- importance sampling (K15, astroz_b200/csrc/az_conjunction_is.cu) --------------------------------------------------
LINEAR, GIVEN, PLAIN = D["ASTROZ_CONJ_IS_LINEAR"], D["ASTROZ_CONJ_IS_GIVEN"], D["ASTROZ_CONJ_IS_PLAIN"]
_IS_COUNT = D["ASTROZ_CONJ_IS_COUNT_WORDS"]
_IS_PROPOSAL = D["ASTROZ_CONJ_IS_PROPOSAL_WORDS"]
_IS_SAMPLE = D["ASTROZ_CONJ_IS_SAMPLE_WORDS"]


def _u256(words) -> list[int]:
    """(m, 4) uint64 words, least significant first -> m Python integers"""
    w = np.asarray(words, dtype=np.uint64).reshape(-1, 4)
    return [sum(int(x) << (64 * q) for q, x in enumerate(row)) for row in w]


@dataclass
class ImportanceResult:
    counts: np.ndarray                # (m, 12) uint64: hits, edge, failed, overflow, V_hit[4], V2_hit[4]
    samples: np.ndarray               # (m,) uint64: samples drawn
    shift: np.ndarray                 # (m, 14) the shift c (primary's 7 normals, then the secondary's)
    log_scale: np.ndarray             # (m,) l0 = -|c|^2 / 2
    kind: np.ndarray                  # (m,) uint8 LINEAR, GIVEN or PLAIN
    status: np.ndarray                # (m,) uint8 ASTROZ_CONJ_*: OK, INIT_FAILED, NOT_PSD
    sample_dt: np.ndarray | None      # (m, record) dt_tca [min] (NaN: none)
    sample_miss: np.ndarray | None    # (m, record) miss [km]
    sample_log_weight: np.ndarray | None   # (m, record) log w

    hits = property(lambda self: self.counts[:, 0])
    edge = property(lambda self: self.counts[:, 1])
    failed = property(lambda self: self.counts[:, 2])
    overflow = property(lambda self: self.counts[:, 3])

    def _sums(self):
        """(e^l0 V_hit 2^-128 / N, e^2l0 V2_hit 2^-128 / N) per candidate from the words through Python integers"""
        v, v2 = _u256(self.counts[:, 4:8]), _u256(self.counts[:, 8:12])
        m1, m2 = np.zeros(len(v)), np.zeros(len(v))
        for i, (a, b) in enumerate(zip(v, v2)):
            n = int(self.samples[i])
            if n == 0 or self.status[i] != OK:
                m1[i] = m2[i] = np.nan
                continue
            l0 = float(self.log_scale[i])
            m1[i] = np.exp(l0) * float(a) * 2.0 ** -128 / n
            m2[i] = np.exp(2 * l0) * float(b) * 2.0 ** -128 / n
        return m1, m2

    @property
    def pc(self) -> np.ndarray:
        """(1 / N) sum over hits of w: unbiased for P(hit) (a failed draw counts as a non-hit); NaN with no sample"""
        return self._sums()[0]

    @property
    def std_error(self) -> np.ndarray:
        """the standard error of pc: sqrt((mean of w^2 over hits - pc^2) / (N - 1))"""
        m1, m2 = self._sums()
        n = self.samples.astype(np.float64)
        with np.errstate(divide="ignore", invalid="ignore"):
            return np.sqrt(np.maximum(m2 - m1 * m1, 0.0) / np.maximum(n - 1.0, 1.0))

    def interval(self, z: float = 1.96) -> tuple[np.ndarray, np.ndarray]:
        """The normal-approximation interval (lo, hi) of Pc at z standard errors, lo clipped at 0; NaN with no hit"""
        p, s = self.pc, self.std_error
        bad = ~(self.hits > 0) | np.isnan(p)
        return np.where(bad, np.nan, np.maximum(p - z * s, 0.0)), np.where(bad, np.nan, p + z * s)

    @property
    def proposal_hit_fraction(self) -> np.ndarray:
        """hits / N: the share of the proposal's draws that hit"""
        n = self.samples.astype(np.float64)
        with np.errstate(divide="ignore", invalid="ignore"):
            return np.where(n > 0, self.hits.astype(np.float64) / n, np.nan)

    def combine(self, other: "ImportanceResult") -> "ImportanceResult":
        """The result over both runs' samples: the words added exactly.  Both must be the same candidates with the same
        shift, drawn over disjoint sample ranges (first = N for the second run of N samples)."""
        if self.counts.shape != other.counts.shape or not np.array_equal(self.shift, other.shift):
            raise ValueError("combine needs the same candidates with the same shifts")
        counts = self.counts.copy()
        counts[:, :4] = self.counts[:, :4] + other.counts[:, :4]
        for lo in (4, 8):
            tot = [a + b for a, b in zip(_u256(self.counts[:, lo:lo + 4]), _u256(other.counts[:, lo:lo + 4]))]
            counts[:, lo:lo + 4] = np.array([[(t >> (64 * q)) & (2 ** 64 - 1) for q in range(4)] for t in tot],
                                            dtype=np.uint64).reshape(-1, 4)
        return ImportanceResult(counts, self.samples + other.samples, self.shift.copy(), self.log_scale.copy(),
                                self.kind.copy(), self.status.copy(), None, None, None)


def importance_sampling(source, primary, secondary, jd, fr, *, window_min, hbr_km, samples, seed=0, first=0,
                        record: int = 0, shift=None, covariance=None, model=None, grav: int = WGS72,
                        device: int = 0) -> ImportanceResult:
    """Importance-sampled collision probability of m candidate conjunctions (astroz_cuda_conjunction_is).

    The arguments are those of `monte_carlo`, plus shift: None (the linear shift onto the collision point from the
    nominal assessment) or (m, 14) / (14,) given shifts of the normals.  Each draw of `monte_carlo` is moved by the
    shift and weighted by its exact likelihood ratio, so pc = (1 / N) sum over hits of w is unbiased whatever the shift;
    a failed draw counts as a non-hit, so where draws fail pc estimates monte_carlo's pc times (1 - P(failed)).  Extend
    a run with first = N and `combine`."""
    el, cov, md = _catalogue(source, covariance, model)
    n = el.shape[1]
    pr, se = _rows(primary, secondary, n)
    m = len(pr)
    record = int(record)
    if record < 0:
        raise ValueError("record must be >= 0")
    f64 = lambda a: np.ascontiguousarray(np.broadcast_to(np.asarray(a, dtype=np.float64), (m,)))  # noqa: E731

    def u64(a, name):
        a = np.asarray(a)
        if a.size and (not np.issubdtype(a.dtype, np.integer) or a.min() < 0):
            raise ValueError(f"{name} must hold integers >= 0")
        return np.ascontiguousarray(np.broadcast_to(a.astype(np.uint64), (m,)))

    jd_, fr_, w_, r_ = f64(jd), f64(fr), f64(window_min), f64(hbr_km)
    ns, fi, sd = u64(samples, "samples"), u64(first, "first"), u64(seed, "seed")
    sh = None if shift is None else np.ascontiguousarray(
        np.broadcast_to(np.asarray(shift, dtype=np.float64), (m, _IS_PROPOSAL - 1)))
    counts, stat = np.zeros((m, _IS_COUNT), np.uint64), np.zeros(m, dtype=np.uint8)
    prop, kind = np.zeros((m, _IS_PROPOSAL)), np.zeros(m, dtype=np.uint8)
    out = np.zeros((m, record, _IS_SAMPLE)) if record else None
    vp = lambda a: None if a is None or a.size == 0 else C.c_void_p(a.ctypes.data)  # noqa: E731
    check(lib().astroz_cuda_conjunction_is(vp(el), n, int(grav), vp(cov), vp(md), vp(pr), vp(se), vp(jd_), vp(fr_),
                                           vp(w_), vp(r_), vp(ns), vp(fi), vp(sd), vp(sh), m, record, int(device),
                                           vp(counts), vp(prop), vp(kind), vp(out), vp(stat)))
    return ImportanceResult(counts, ns.copy(), prop[:, :-1], prop[:, -1], kind, stat,
                            *((None,) * 3 if out is None else (out[:, :, 0], out[:, :, 1], out[:, :, 2])))


def importance_sampling_scratch_bytes(m: int) -> int:
    """The scratch of importance_sampling_device for m candidates"""
    b = C.c_uint64(0)
    check(lib().astroz_cuda_conjunction_is_scratch_bytes(int(m), C.byref(b)))
    return int(b.value)


def importance_sampling_device(elements, covariance, model, primary, secondary, jd, fr, window_min, hbr_km, samples,
                               first, seed, shift, counts, proposal, proposal_kind, sample_out, status, scratch, *,
                               grav: int = WGS72, stream: int = 0) -> None:
    """`importance_sampling` with torch CUDA tensors on one device: the inputs of `monte_carlo_device`, shift (m, 14)
    float64 or None (linear); counts (m, 12) int64, proposal (m, 15) float64 or None, proposal_kind (m,) uint8 or None,
    sample_out (m, record, 3) float64 or None and status (m,) uint8 receive the results; scratch a uint8 tensor of at
    least importance_sampling_scratch_bytes(m) bytes.  The launches go on `stream` (a raw cudaStream_t value, 0 = the
    default stream).  Rows are not checked here: a bad pair gets status BAD_PAIR."""
    import torch

    n = int(elements.shape[1]) if elements.dim() == 2 and elements.shape[0] == 8 else -1
    if n < 0 or elements.dtype != torch.float64 or not elements.is_cuda:
        raise ValueError("elements must be a CUDA float64 tensor of shape (8, n)")
    m = int(primary.numel())
    record = int(sample_out.shape[1]) if sample_out is not None and sample_out.dim() == 3 else 0
    tensors = [("elements", elements, 8 * n, torch.float64), ("covariance", covariance, 28 * n, torch.float64),
               ("model", model, n, torch.uint8), ("primary", primary, m, torch.int32),
               ("secondary", secondary, m, torch.int32), ("jd", jd, m, torch.float64), ("fr", fr, m, torch.float64),
               ("window_min", window_min, m, torch.float64), ("hbr_km", hbr_km, m, torch.float64),
               ("samples", samples, m, torch.int64), ("first", first, m, torch.int64), ("seed", seed, m, torch.int64),
               ("shift", shift, (_IS_PROPOSAL - 1) * m, torch.float64), ("counts", counts, _IS_COUNT * m, torch.int64),
               ("proposal", proposal, _IS_PROPOSAL * m, torch.float64), ("proposal_kind", proposal_kind, m, torch.uint8),
               ("sample_out", sample_out, _IS_SAMPLE * record * m, torch.float64), ("status", status, m, torch.uint8)]
    for name, t, size, dtype in tensors:
        if t is None and name in ("model", "first", "seed", "shift", "proposal", "proposal_kind", "sample_out"):
            continue
        if not isinstance(t, torch.Tensor) or t.dtype != dtype or not t.is_contiguous() or int(t.numel()) != size \
                or t.device != elements.device:
            raise ValueError(f"{name} must be a contiguous {dtype} tensor of {size} elements on {elements.device}")
    if not isinstance(scratch, torch.Tensor) or not scratch.is_contiguous() or scratch.device != elements.device \
            or scratch.numel() * scratch.element_size() < importance_sampling_scratch_bytes(m):
        raise ValueError(f"scratch must be a contiguous tensor of importance_sampling_scratch_bytes({m}) bytes on "
                         f"{elements.device}")
    ptr = lambda t: None if t is None else C.c_void_p(t.data_ptr())  # noqa: E731
    check(lib().astroz_cuda_conjunction_is_device(
        ptr(elements), n, int(grav), ptr(covariance), ptr(model), ptr(primary), ptr(secondary), ptr(jd), ptr(fr),
        ptr(window_min), ptr(hbr_km), ptr(samples), ptr(first), ptr(seed), ptr(shift), m, record,
        int(elements.device.index), ptr(counts), ptr(proposal), ptr(proposal_kind), ptr(sample_out), ptr(status),
        ptr(scratch), C.c_void_p(stream) if stream else None))


# ---- manoeuvre trials and the avoidance planner (K16, astroz_b200/csrc/az_avoid.cu) -----------------------------------
CONVERSION_FAILED, BAD_TRIAL = D["ASTROZ_CONJ_CONVERSION_FAILED"], D["ASTROZ_CONJ_BAD_TRIAL"]
STATUS_NAMES[CONVERSION_FAILED] = "the post-burn state could not be converted to an element set"
STATUS_NAMES[BAD_TRIAL] = "bad trial: candidate index or burn not before the window"


@dataclass
class ManeuverResult(ConjunctionResult):
    elements: np.ndarray = None          # (t, 8) the post-burn set (epoch, n, e, i, node, w, M, B*)
    covariance: np.ndarray = None        # (t, 28) P' words in the fit's variables
    residual: np.ndarray = None          # (t, 2) conversion residuals [km, km/s]
    model: np.ndarray = None             # (t,) uint8 the primary's model byte

    def catalogue_rows(self):
        """(elements (8, t), covariance words (t, 28), model (t,)): the new rows, ready to append to the catalogue"""
        return np.ascontiguousarray(self.elements.T), self.covariance.copy(), self.model.copy()


def maneuver_trials(source, primary, secondary, jd, fr, *, window_min, hbr_km, candidate, burn_jd, burn_fr, dv_rtn,
                    dv_sigma=None, covariance=None, model=None, grav: int = WGS72, device: int = 0) -> ManeuverResult:
    """Reassess candidates after trial burns of their primary (astroz_cuda_conjunction_maneuver).

    source, primary, secondary, jd, fr, window_min, hbr_km, covariance and model are those of `conjunctions`; the
    primary is the object that burns.  Trial k burns candidate[k]'s primary at burn_jd[k] + burn_fr[k] (before the
    window) by dv_rtn[k] (3,) [km/s] in its RTN frame, with execution sigmas dv_sigma[k] (3,) [km/s] or None; candidate,
    burn_jd, burn_fr, dv_rtn and dv_sigma broadcast to the longest of them.  Each trial's post-burn set keeps the
    primary's epoch; a zero burn copies the primary's row, so its record is conjunctions' record of the nominal pair.
    The returned rows (catalogue_rows) are ordinary catalogue rows for every other call of this module.  P' inherits the
    quantisation of the forward-difference B* columns of J and J' (about 1e-4 km per unit B* in LEO): on rows with B*
    free and a large B* variance its phase entries are good to some 20 % of sqrt(P'_jj P'_kk) (a few cm along track at
    the burn); rows with B* held are not affected (astroz_b200.h, K16)."""
    el, cov, md = _catalogue(source, covariance, model)
    n = el.shape[1]
    pr, se = _rows(primary, secondary, n)
    m = len(pr)
    f64 = lambda a, k: np.ascontiguousarray(np.broadcast_to(np.asarray(a, dtype=np.float64), (k,)))  # noqa: E731
    jd_, fr_, w_, r_ = f64(jd, m), f64(fr, m), f64(window_min, m), f64(hbr_km, m)
    ca = np.asarray(candidate).reshape(-1) if np.ndim(candidate) else np.asarray([candidate])
    if ca.size and (not np.issubdtype(ca.dtype, np.integer) or ca.min() < 0 or ca.max() >= m):
        raise ValueError("candidate must hold candidate indices in [0, m)")
    dv = np.asarray(dv_rtn, dtype=np.float64)
    sg = None if dv_sigma is None else np.asarray(dv_sigma, dtype=np.float64)
    t = max(len(ca), np.size(burn_jd), np.size(burn_fr), dv.size // 3 if dv.ndim > 1 else 1,
            1 if sg is None or sg.ndim < 2 else len(sg))
    ca = np.ascontiguousarray(np.broadcast_to(ca.astype(np.uint32), (t,)))
    bj, bf = f64(burn_jd, t), f64(burn_fr, t)
    dv = np.ascontiguousarray(np.broadcast_to(dv, (t, 3)))
    sg = None if sg is None else np.ascontiguousarray(np.broadcast_to(sg, (t, 3)))
    rec, stat = np.zeros((t, _WORDS)), np.zeros(t, dtype=np.uint8)
    ne, nc, res = np.zeros((t, 8)), np.zeros((t, 28)), np.zeros((t, 2))
    vp = lambda a: None if a is None or a.size == 0 else C.c_void_p(a.ctypes.data)  # noqa: E731
    check(lib().astroz_cuda_conjunction_maneuver(vp(el), n, int(grav), vp(cov), vp(md), vp(pr), vp(se), vp(jd_),
                                                 vp(fr_), vp(w_), vp(r_), m, vp(ca), vp(bj), vp(bf), vp(dv), vp(sg), t,
                                                 int(device), vp(rec), vp(ne), vp(nc), vp(res), vp(stat)))
    mdl = np.zeros(t, np.uint8) if md is None else md[pr[ca]]
    return ManeuverResult(rec, jd_[ca], fr_[ca] + rec[:, 0] / 1440.0, None, None, stat, ne, nc, res, mdl)


def maneuver_trials_scratch_bytes(t: int) -> int:
    """The scratch of maneuver_trials_device for t trials"""
    b = C.c_uint64(0)
    check(lib().astroz_cuda_conjunction_maneuver_scratch_bytes(int(t), C.byref(b)))
    return int(b.value)


def maneuver_trials_device(elements, covariance, model, primary, secondary, jd, fr, window_min, hbr_km, candidate,
                           burn_jd, burn_fr, dv_rtn, dv_sigma, record, new_elements, new_covariance, residual, status,
                           scratch, *, grav: int = WGS72, stream: int = 0) -> None:
    """`maneuver_trials` with torch CUDA tensors on one device: the catalogue and candidates of `conjunctions_device`,
    candidate (t,) int32, burn_jd / burn_fr (t,) float64, dv_rtn (t, 3) float64, dv_sigma (t, 3) float64 or None;
    record (t, 13) float64, new_elements (t, 8) / new_covariance (t, 28) / residual (t, 2) float64 or None and status
    (t,) uint8 receive the results; scratch a uint8 tensor of at least maneuver_trials_scratch_bytes(t) bytes.  The
    launches go on `stream` (a raw cudaStream_t value, 0 = the default stream).  Nothing is checked here: a bad
    candidate index or burn time gets BAD_TRIAL, a bad pair BAD_PAIR."""
    import torch

    n = int(elements.shape[1]) if elements.dim() == 2 and elements.shape[0] == 8 else -1
    if n < 0 or elements.dtype != torch.float64 or not elements.is_cuda:
        raise ValueError("elements must be a CUDA float64 tensor of shape (8, n)")
    m, t = int(primary.numel()), int(candidate.numel())
    tensors = [("elements", elements, 8 * n, torch.float64), ("covariance", covariance, 28 * n, torch.float64),
               ("model", model, n, torch.uint8), ("primary", primary, m, torch.int32),
               ("secondary", secondary, m, torch.int32), ("jd", jd, m, torch.float64), ("fr", fr, m, torch.float64),
               ("window_min", window_min, m, torch.float64), ("hbr_km", hbr_km, m, torch.float64),
               ("candidate", candidate, t, torch.int32), ("burn_jd", burn_jd, t, torch.float64),
               ("burn_fr", burn_fr, t, torch.float64), ("dv_rtn", dv_rtn, 3 * t, torch.float64),
               ("dv_sigma", dv_sigma, 3 * t, torch.float64), ("record", record, _WORDS * t, torch.float64),
               ("new_elements", new_elements, 8 * t, torch.float64),
               ("new_covariance", new_covariance, 28 * t, torch.float64), ("residual", residual, 2 * t, torch.float64),
               ("status", status, t, torch.uint8)]
    for name, x, size, dtype in tensors:
        if x is None and name in ("model", "dv_sigma", "new_elements", "new_covariance", "residual"):
            continue
        if not isinstance(x, torch.Tensor) or x.dtype != dtype or not x.is_contiguous() or int(x.numel()) != size \
                or x.device != elements.device:
            raise ValueError(f"{name} must be a contiguous {dtype} tensor of {size} elements on {elements.device}")
    if not isinstance(scratch, torch.Tensor) or not scratch.is_contiguous() or scratch.device != elements.device \
            or scratch.numel() * scratch.element_size() < maneuver_trials_scratch_bytes(t):
        raise ValueError(f"scratch must be a contiguous tensor of maneuver_trials_scratch_bytes({t}) bytes on "
                         f"{elements.device}")
    ptr = lambda x: None if x is None else C.c_void_p(x.data_ptr())  # noqa: E731
    check(lib().astroz_cuda_conjunction_maneuver_device(
        ptr(elements), n, int(grav), ptr(covariance), ptr(model), ptr(primary), ptr(secondary), ptr(jd), ptr(fr),
        ptr(window_min), ptr(hbr_km), m, ptr(candidate), ptr(burn_jd), ptr(burn_fr), ptr(dv_rtn), ptr(dv_sigma), t,
        int(elements.device.index), ptr(record), ptr(new_elements), ptr(new_covariance), ptr(residual), ptr(status),
        ptr(scratch), C.c_void_p(stream) if stream else None))


NOT_FOUND = 255   # AvoidanceResult.status of a (candidate, lead, sign) where no step up to dv_max_kms is feasible


@dataclass
class AvoidanceResult:
    dv_kms: np.ndarray         # (m, L, 2) the least |dv| found along -direction (0) and +direction (1); NaN: none
    record: np.ndarray         # (m, L, 2, 13) the trial's record at that dv (zeros where NaN)
    status: np.ndarray         # (m, L, 2) its status: OK, or NOT_FOUND where dv_kms is NaN
    ladder_kms: np.ndarray     # (ladder,) the round-0 magnitudes
    pc: np.ndarray             # (m, L, 2, ladder) round 0's Pc (NaN where the trial's status is not OK)
    pc_nominal: np.ndarray     # (m,) the zero burn's Pc without execution error (NaN where it is not OK)
    burn_jd: np.ndarray        # (m, L) the burn times: guess - lead, as jd ...
    burn_fr: np.ndarray        # (m, L) ... and fr


def _feasible(rec, st, pc_max):
    """OK and Pc <= pc_max.  A WINDOW_EDGE record is taken at a window end, not at a TCA, so its Pc says nothing about
    the encounter: a burn that moves the TCA out of the window is never feasible."""
    return (st == OK) & (rec[..., 12] <= pc_max)


def _avoidance(run, m, jd, fr, lead_min, direction, pc_max, dv_max_kms, ladder, rounds, dv_sigma):
    """The planner over run(candidate, burn_jd, burn_fr, dv_rtn, dv_sigma (t, 3) or None) -> (record (t, 13),
    status (t,))"""
    lead = np.atleast_1d(np.asarray(lead_min, dtype=np.float64))
    u = np.asarray(direction, dtype=np.float64).reshape(3)
    if not np.isclose(np.linalg.norm(u), 1.0):
        raise ValueError("direction must be a unit RTN vector")
    if not (dv_max_kms > 0) or int(ladder) < 1 or int(rounds) < 0:
        raise ValueError("dv_max_kms must be > 0, ladder >= 1 and rounds >= 0")
    ladder, Lr = int(ladder), len(lead)
    steps = dv_max_kms * 2.0 ** (np.arange(ladder) - (ladder - 1))   # geometric: dv_max / 2^(ladder-1) .. dv_max
    bj = np.broadcast_to(jd[:, None], (m, Lr))
    bf = fr[:, None] - lead[None, :] / 1440.0
    sgn = np.array([-1.0, 1.0])
    sg = None if dv_sigma is None else np.asarray(dv_sigma, dtype=np.float64).reshape(3)
    sig = lambda t, zero=0: None if sg is None else np.r_[np.tile(sg, (t, 1)), np.zeros((zero, 3))]  # noqa: E731
    # round 0: every (candidate, lead, sign, step), plus one zero burn per candidate without execution error
    ci, li, si, ki = (a.reshape(-1) for a in np.meshgrid(np.arange(m), np.arange(Lr), np.arange(2), np.arange(ladder),
                                                           indexing="ij"))
    nt = len(ci)
    cand = np.r_[ci, np.arange(m)]
    bjd = np.r_[bj[ci, li], jd]
    bfr = np.r_[bf[ci, li], fr - lead.max() / 1440.0]
    dv = np.r_[(sgn[si] * steps[ki])[:, None] * u[None, :], np.zeros((m, 3))]
    rec, st = run(cand, bjd, bfr, dv, sig(nt, m))
    rec0, st0 = rec[:nt].reshape(m, Lr, 2, ladder, -1), st[:nt].reshape(m, Lr, 2, ladder)
    pc_tab = np.where(st0 == OK, rec0[..., 12], np.nan)
    feas = _feasible(rec0, st0, pc_max)
    first = np.where(feas.any(-1), feas.argmax(-1), -1)
    hi = np.where(first >= 0, steps[np.maximum(first, 0)], np.nan)
    lo = np.where(first > 0, steps[np.maximum(first - 1, 0)], 0.0)
    idx = np.maximum(first, 0)[..., None, None]
    best_rec = np.where((first >= 0)[..., None], np.take_along_axis(rec0, idx, axis=3)[:, :, :, 0], 0.0)
    best_st = np.where(first >= 0, np.take_along_axis(st0, idx[..., 0], axis=3)[..., 0], NOT_FOUND).astype(np.uint8)
    # the nominal already meets the target: dv = 0 (no burn, so no execution error either)
    zero_ok = _feasible(rec[nt:], st[nt:], pc_max)[:, None, None]
    first = np.where(zero_ok, -1, first)
    hi = np.where(zero_ok, 0.0, hi)
    best_rec = np.where(zero_ok[..., None], rec[nt:][:, None, None], best_rec)
    best_st = np.where(zero_ok, st[nt:][:, None, None], best_st).astype(np.uint8)
    for _ in range(rounds):
        open_ = np.argwhere(first >= 0)
        if len(open_) == 0:
            break
        c, l, s = open_.T
        mid = 0.5 * (lo[c, l, s] + hi[c, l, s])
        r, q = run(c, bj[c, l], bf[c, l], (sgn[s] * mid)[:, None] * u[None, :], sig(len(c)))
        ok = _feasible(r, q, pc_max)
        hi[c[ok], l[ok], s[ok]] = mid[ok]
        best_rec[c[ok], l[ok], s[ok]] = r[ok]
        best_st[c[ok], l[ok], s[ok]] = q[ok]
        lo[c[~ok], l[~ok], s[~ok]] = mid[~ok]
    pc_nominal = np.where(st[nt:] == OK, rec[nt:, 12], np.nan)
    return AvoidanceResult(hi, best_rec, best_st, steps, pc_tab, pc_nominal, np.array(bj), bf)


def avoidance(source, primary, secondary, jd, fr, *, window_min, hbr_km, lead_min, direction=(0.0, 1.0, 0.0), pc_max,
              dv_max_kms, ladder: int = 32, rounds: int = 20, dv_sigma=None, covariance=None, model=None,
              grav: int = WGS72, device: int = 0) -> AvoidanceResult:
    """The least |dv| along +-direction (a unit RTN vector) that brings each candidate's Pc to pc_max or below.

    For each candidate, each lead in lead_min (burn = guess - lead minutes; each must come before the window) and
    each sign, round 0 is one batched maneuver_trials call over a geometric ladder of `ladder` magnitudes up to
    dv_max_kms (each step twice the one below it), plus the zero burn.  A trial is feasible when its status is OK and
    its Pc <= pc_max.  WINDOW_EDGE is not feasible: its record is taken at a window end, not at a TCA, so a burn that
    moves the encounter out of the window (along-track drift is about 3 dv t) is rejected however low that Pc is; give
    window_min room for the shift the burns cause.  The first feasible step is bracketed against the step below it (or
    0), and
    `rounds` bisection rounds follow, each one batched call over all open brackets; the upper end always stays feasible,
    so dv_kms meets the target and dv_kms (1 - 2 * 2^-rounds) of the bracket does not, to the ladder's resolution.
    Pc(|dv|) need not be monotone: a burn can first move the miss towards the covariance's centre and raise Pc.  The
    result is the least feasible dv at the ladder's resolution: a feasible interval narrower than one ladder step below
    the first feasible step can be missed.  dv_kms is NaN where no step up to dv_max_kms works.  The whole round-0 table
    is returned as pc (NaN where a trial is not OK).  pc_nominal is the zero burn's Pc, without execution error (no burn,
    no execution error); where it already meets pc_max, dv_kms is 0 and the record is the nominal's.  dv_sigma (3,)
    [km/s] is the execution error of every burn.  Where no step is feasible, dv_kms is NaN and status NOT_FOUND."""
    el, cov, md = _catalogue(source, covariance, model)
    n = el.shape[1]
    pr, se = _rows(primary, secondary, n)
    m = len(pr)
    jd_ = np.ascontiguousarray(np.broadcast_to(np.asarray(jd, dtype=np.float64), (m,)))
    fr_ = np.ascontiguousarray(np.broadcast_to(np.asarray(fr, dtype=np.float64), (m,)))

    def run(cand, bjd, bfr, dv, sg):
        r = maneuver_trials(el, pr, se, jd_, fr_, window_min=window_min, hbr_km=hbr_km, candidate=cand, burn_jd=bjd,
                            burn_fr=bfr, dv_rtn=dv, dv_sigma=sg, covariance=cov, model=md, grav=grav, device=device)
        return r.record, r.status

    return _avoidance(run, m, jd_, fr_, lead_min, direction, pc_max, dv_max_kms, ladder, rounds, dv_sigma)
