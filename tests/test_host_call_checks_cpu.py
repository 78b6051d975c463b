"""The input checks of the whole-batch calls of the C ABI and of their _device twins, one table row per refusal.

Each row asserts the return code, the astroz_cuda_last_error() text and that no output word was written.  A
null-pointer refusal or a no-op leaves the last error as it was.  Valid input on a machine without a GPU is
ASTROZ_NO_DEVICE with every output untouched, which shows that every value check runs before the device lookup.  The
device twins are only ever given host arrays: each row refuses, or stops at the device lookup, before any is read.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from astroz_b200 import _abi
from astroz_b200._abi import DEFINES as D

OK, VE, NP, ND = D["ASTROZ_OK"], D["ASTROZ_VALUE_ERROR"], D["ASTROZ_NULL_POINTER"], D["ASTROZ_NO_DEVICE"]
PARAMS = {name: [p for _, p in args] for _, name, args in _abi.declarations()}

# set before every call: the text a null-pointer refusal or a no-op must leave in place
UNCHANGED = "the chi-square quantile needs k >= 1 and p in (0, 1)"
NO_DEVICE = "no CUDA device available (this library has no CPU propagation path)"
GRAV = "grav must be ASTROZ_WGS72 or ASTROZ_WGS84"
DECREASING = "offsets must be non-decreasing"
FIRST = "offsets[0] must be 0"
EMPTY = "a track has no observation"
END_N = "offsets[n] must equal the observation count m"
END_T = "offsets[t] must equal the observation count m"
ELEMENTS = "elements must be finite"
COVARIANCE = "covariance words must be finite"
MODEL = "a model byte is not 0 (near-earth) or 1 (deep space)"
FRAME = "frame must be ASTROZ_COV_FRAME_TEME or ASTROZ_COV_FRAME_RTN"
USED = "a track has no used residual"


def out(shape, dtype=np.float64):
    return np.full(shape, 7, dtype)


def observations():
    """A TEME state, two radar measurements and an optical one, from two stations."""
    kind = np.array([0, 2, 2, 3], np.uint8)
    value = np.zeros((4, 6))
    value[0] = [7000.0, 0.0, 0.0, 0.0, 7.5, 0.0]
    value[1:3, :4] = [1000.0, 0.5, 0.3, 0.0]
    value[3, :2] = [1.0, 0.2]
    sigma = np.full((4, 6), np.inf)
    sigma[0] = [1.0, 1.0, 1.0, 1e-3, 1e-3, 1e-3]
    sigma[1:3, :4] = [0.1, 1e-4, 1e-4, 1e-3]
    sigma[3, :2] = [1e-5, 1e-5]
    return dict(jd=np.full(4, 2460000.5), fr=np.linspace(0.1, 0.2, 4), kind=kind, value=value, sigma=sigma,
                station=np.array([0, 0, 1, 1], np.uint32), m=4,
                stations=np.array([[10.0, 20.0, 0.1], [-30.0, 140.0, 0.5]]), k=2)


def elements(n):
    col = np.array([2460000.5, 15.5, 1e-3, 51.6, 10.0, 20.0, 30.0, 1e-4])
    return np.ascontiguousarray(np.tile(col[:, None], (1, n)))


def covariance(n):
    return np.ascontiguousarray(np.tile(np.eye(7)[np.triu_indices(7)], (n, 1)))


def fit_scene():
    return dict(elements=elements(2), n=2, grav=1, offsets=np.array([0, 2, 4], np.uint32), jd=np.full(4, 2460000.5),
                fr=np.linspace(0.1, 0.2, 4), pos=np.full((4, 3), 7000.0), vel=np.full((4, 3), 1.0), m=4,
                pos_sigma=1.0, vel_sigma=1e-3, fit_bstar=1, max_iter=10, device=0, fitted=out((8, 2)),
                rms=out((2, 2)), iterations=out(2, np.uint32), status=out(2, np.uint8))


def fit_obs_scene():
    return dict(elements=elements(2), n=2, grav=1, offsets=np.array([0, 2, 4], np.uint32), **observations(),
                fit_bstar=1, max_iter=10, device=0, fitted=out((8, 2)), wrms=out(2), n_residuals=out(2, np.uint32),
                covariance=out((2, 28)), iterations=out(2, np.uint32), status=out(2, np.uint8),
                model=out(2, np.uint8))


def observe_scene():
    return dict(states=np.full((4, 6), 1000.0), **observations(), device=0, values=out((4, 6)))


def cov_scene():
    return dict(elements=elements(2), n=2, grav=1, covariance=covariance(2), model=np.zeros(2, np.uint8),
                offsets=np.array([0, 1, 3], np.uint32), jd=np.full(3, 2460000.5), fr=np.linspace(0.1, 0.2, 3), m=3,
                frame=0, device=0, state=out((3, 6)), state_covariance=out((3, 21)), jacobian=out((3, 42)),
                status=out(3, np.uint8))


def conj_scene():
    return dict(elements=elements(3), n=3, grav=1, covariance=covariance(3), model=np.zeros(3, np.uint8),
                primary=np.array([0, 1], np.uint32), secondary=np.array([1, 2], np.uint32), jd=np.full(2, 2460000.5),
                fr=np.array([0.1, 0.2]), window_min=np.ones(2), hbr_km=np.full(2, 0.01), m=2, frame=0, device=0,
                record=out((2, 13)), states=out((2, 2, 6)), state_covariance=out((2, 2, 21)),
                status=out(2, np.uint8))


def corr_scene():
    return dict(elements=elements(2), n=2, grav=1, covariance=covariance(2), model=np.zeros(2, np.uint8),
                offsets=np.array([0, 2, 4], np.uint32), t=2, **observations(), gate_probability=0.999, best=4,
                device=0, scratch=out(64, np.uint8), rows=out((2, 4), np.uint32), d2=out((2, 4)),
                used=out(2, np.uint32), n_gate=out(2, np.uint32), n_failed=out(2, np.uint32), status=out(2, np.uint8),
                row_status=out(2, np.uint8))


def iod_scene():
    return dict(offsets=np.array([0, 2, 4], np.uint32), t=2, **observations(), bstar=np.full(2, 1e-4), grav=1,
                device=0, scratch=out(64, np.uint8), elements=out((8, 2)), state=out((2, 6)), wrms=out(2),
                method=out(2, np.uint8), candidates=out(2, np.uint32), conv=out((2, 2)), deep_space=out(2, np.uint8),
                status=out(2, np.uint8))


def lambert_scene():
    return dict(r1=np.full((2, 3), 7000.0), r2=np.full((2, 3), -7000.0), tof=np.full(2, 3000.0),
                normal=np.tile([0.0, 0.0, 1.0], (2, 1)), n=2, mu=398600.4418, max_revs=1, device=0, v1=out((6, 3)),
                v2=out((6, 3)), status=out(6, np.uint8), iterations=out(6, np.uint8))


OUTPUTS = {"fitted", "rms", "iterations", "status", "wrms", "n_residuals", "model", "values", "state",
           "state_covariance", "jacobian", "record", "states", "scratch", "rows", "d2", "used", "n_gate", "n_failed",
           "row_status", "elements", "method", "candidates", "conv", "deep_space", "v1", "v2"}


def is_output(call, p):
    """covariance and model are outputs of the observation fits and inputs elsewhere; elements the other way round"""
    base = call.removesuffix("_device")
    if p in ("covariance", "model"):
        return base.startswith("astroz_cuda_fit_observations")
    if p == "elements":
        return base == "astroz_cuda_initial_orbits"
    return p in OUTPUTS


def set_(**kw):
    return lambda a: a.update(kw)


def edit(name, index, value):
    def f(a):
        a[name] = a[name].copy()
        a[name][index] = value
    return f


def offsets(*o):
    return set_(offsets=np.array(o, np.uint32))


def no_observations(a):
    a.update(offsets=np.zeros(len(a["offsets"]), np.uint32), m=0, jd=None, fr=None, kind=None, value=None,
             sigma=None, station=None, pos=None, vel=None, states=None)


def long_track(a):   # 257 TEME states in the first track, one in the second
    m = 258
    a.update(offsets=np.array([0, 257, 258], np.uint32), m=m, jd=np.full(m, 2460000.5), fr=np.linspace(0.1, 0.2, m),
             kind=np.zeros(m, np.uint8), value=np.tile(observations()["value"][0], (m, 1)),
             sigma=np.tile(observations()["sigma"][0], (m, 1)), station=np.zeros(m, np.uint32))


def no_used_residual(a):
    a["sigma"] = a["sigma"].copy()
    a["sigma"][0:2] = np.inf


def nulls(*names):
    return [(f"{p} NULL", set_(**{p: None}), NP, UNCHANGED) for p in names]


def obs_value_rows(sigma=True):
    rows = [("stations NULL with k > 0", set_(stations=None), NP, UNCHANGED),
            ("a station not finite", edit("stations", (0, 1), np.nan), VE, "stations must be finite"),
            ("a station latitude", edit("stations", (1, 0), 91.0), VE, "a station latitude is outside [-90, 90] deg"),
            ("a time not finite", edit("jd", 1, np.inf), VE, "observation times must be finite"),
            ("an unknown kind", edit("kind", 0, 4), VE, "unknown observation kind"),
            ("station NULL for a radar measurement", set_(station=None), NP, UNCHANGED),
            ("a station index", edit("station", 1, 2), VE, "a station index is not below the station count k")]
    if sigma:
        rows += [("sigma <= 0", edit("sigma", (1, 0), 0.0), VE, "sigma must be > 0 (+inf: component not used)"),
                 ("a used value not finite", edit("value", (1, 0), np.nan), VE,
                  "a used observation value is not finite"),
                 ("an azimuth without its elevation",
                  lambda a: (edit("value", (1, 2), np.nan)(a), edit("sigma", (1, 2), np.inf)(a)), VE,
                  "a used azimuth or right ascension needs a finite elevation or declination")]
    return rows


def track_offset_rows(limit):
    return [("offsets NULL", set_(offsets=None), NP, UNCHANGED),
            ("offsets[0] != 0", offsets(1, 2, 4), VE, FIRST),
            ("offsets decreasing", offsets(0, 3, 2), VE, DECREASING),
            ("an empty track", offsets(0, 0, 4), VE, EMPTY),
            ("a track too long", long_track, VE, f"a track is longer than {limit} observations"),
            ("offsets[t] != m", offsets(0, 2, 3), VE, END_T)]


VALID = [("valid", set_(), ND, NO_DEVICE)]

FIT_SCALARS = [("device < 0", set_(device=-1), VE, "an element fit runs on one device: pass its ordinal"),
               ("grav", set_(grav=7), VE, GRAV),
               ("pos_sigma 0", set_(pos_sigma=0.0), VE, "pos_sigma and vel_sigma must be finite and > 0"),
               ("vel_sigma nan", set_(vel_sigma=np.nan), VE, "pos_sigma and vel_sigma must be finite and > 0"),
               ("max_iter 0", set_(max_iter=0), VE, "max_iter must be at least 1"),
               ("n = 0", set_(n=0, elements=None, offsets=None), OK, UNCHANGED)]
FIT_HOST = FIT_SCALARS + nulls("elements", "offsets", "fitted", "rms", "iterations", "status") + nulls(
    "jd", "fr", "pos") + [
    ("offsets decreasing", offsets(0, 3, 2), VE, DECREASING),
    ("offsets[n] != m", offsets(0, 2, 3), VE, END_N),
    ("an element not finite", edit("elements", (2, 1), np.nan), VE, "elements and observations must be finite"),
    ("a time not finite", edit("fr", 3, np.inf), VE, "elements and observations must be finite"),
    ("a position not finite", edit("pos", (1, 2), np.nan), VE, "elements and observations must be finite"),
    ("a velocity not finite", edit("vel", (3, 0), np.nan), VE, "elements and observations must be finite"),
    ("vel NULL", set_(vel=None), ND, NO_DEVICE),
    ("offsets[0] != 0 is accepted", offsets(1, 2, 4), ND, NO_DEVICE),
    ("m = 0 with NULL observation arrays", no_observations, ND, NO_DEVICE)] + VALID
FIT_DEVICE = FIT_SCALARS + nulls("elements", "offsets", "jd", "fr", "pos", "fitted", "rms", "iterations",
                                 "status") + [("vel NULL", set_(vel=None), ND, NO_DEVICE)] + VALID

FIT_OBS_SCALARS = [("device < 0", set_(device=-1), VE, "an element fit runs on one device: pass its ordinal"),
                   ("grav", set_(grav=7), VE, GRAV),
                   ("max_iter 0", set_(max_iter=0), VE, "max_iter must be at least 1"),
                   ("n = 0", set_(n=0, elements=None, offsets=None), OK, UNCHANGED)]
FIT_OBS_HOST = FIT_OBS_SCALARS + nulls("elements", "offsets", "fitted", "wrms", "n_residuals", "covariance",
                                       "iterations", "status", "model") + nulls(
    "jd", "fr", "value", "sigma", "kind") + [
    ("offsets decreasing", offsets(0, 3, 2), VE, DECREASING),
    ("offsets[n] != m", offsets(0, 2, 3), VE, END_N),
    ("an element not finite", edit("elements", (0, 1), np.inf), VE, ELEMENTS)] + obs_value_rows() + [
    ("offsets[0] != 0 is accepted", offsets(1, 2, 4), ND, NO_DEVICE),
    ("m = 0 with NULL observation arrays", no_observations, ND, NO_DEVICE),
    ("k = 0 without radar or optical measurements",
     lambda a: a.update(kind=np.zeros(4, np.uint8), stations=None, k=0, station=None), ND, NO_DEVICE)] + VALID
FIT_OBS_DEVICE = FIT_OBS_SCALARS + nulls("elements", "offsets", "jd", "fr", "value", "sigma", "kind", "fitted",
                                         "wrms", "n_residuals", "covariance", "iterations", "status", "model") + [
    ("station and stations NULL", set_(station=None, stations=None), ND, NO_DEVICE)] + VALID

OBSERVE_DEVICE = [("device < 0", set_(device=-1), VE, "observe runs on one device: pass its ordinal"),
                  ("m = 0", set_(m=0, states=None), OK, UNCHANGED)] + nulls("states", "jd", "fr", "kind",
                                                                            "values") + VALID
OBSERVE_HOST = OBSERVE_DEVICE[:-1] + obs_value_rows(sigma=False) + [
    ("a NaN value is not read", edit("value", (1, 0), np.nan), ND, NO_DEVICE)] + VALID

COV_SCALARS = [("device < 0", set_(device=-1), VE, "covariance propagation runs on one device: pass its ordinal"),
               ("grav", set_(grav=-1), VE, GRAV),
               ("frame", set_(frame=2), VE, FRAME)]
COV_HOST = COV_SCALARS + [("offsets NULL", set_(offsets=None), NP, UNCHANGED)] + nulls(
    "elements", "covariance", "jd", "fr", "state_covariance", "status") + [
    ("offsets[0] != 0", offsets(1, 1, 3), VE, FIRST),
    ("offsets decreasing", offsets(0, 2, 1), VE, DECREASING),
    ("offsets[n] != m", offsets(0, 1, 2), VE, "offsets[n] must equal the query count m"),
    ("an element not finite", edit("elements", (7, 0), np.nan), VE, ELEMENTS),
    ("a covariance word not finite", edit("covariance", (1, 5), np.inf), VE, COVARIANCE),
    ("a time not finite", edit("jd", 2, np.nan), VE, "query times must be finite"),
    ("a model byte", edit("model", 1, 2), VE, MODEL),
    ("a model byte with m = 0", lambda a: (no_observations(a), edit("model", 1, 2)(a)), VE, MODEL),
    ("m = 0", no_observations, OK, UNCHANGED),
    ("state, jacobian and model NULL", set_(state=None, jacobian=None, model=None), ND, NO_DEVICE)] + VALID
COV_DEVICE = COV_SCALARS + [("m = 0", set_(m=0, jd=None), OK, UNCHANGED),
                            ("n = 0", set_(n=0, elements=None), OK, UNCHANGED)] + nulls(
    "elements", "covariance", "offsets", "jd", "fr", "state_covariance", "status") + [
    ("state, jacobian and model NULL", set_(state=None, jacobian=None, model=None), ND, NO_DEVICE)] + VALID

CONJ_SCALARS = [("device < 0", set_(device=-1), VE, "conjunction assessment runs on one device: pass its ordinal"),
                ("grav", set_(grav=8), VE, GRAV),
                ("frame", set_(frame=-1), VE, FRAME),
                ("m = 0", set_(m=0, primary=None, record=None), OK, UNCHANGED)]
CONJ_HOST = CONJ_SCALARS + nulls("elements", "covariance", "primary", "secondary", "jd", "fr", "window_min", "hbr_km",
                                 "record", "status") + [
    ("a primary row outside", edit("primary", 0, 3), VE, "a candidate's row is outside the catalogue"),
    ("a secondary row outside", edit("secondary", 1, 9), VE, "a candidate's row is outside the catalogue"),
    ("a row with itself", edit("secondary", 1, 1), VE, "a candidate pairs a row with itself"),
    ("a half window 0", edit("window_min", 0, 0.0), VE, "half windows must be finite and > 0 minutes"),
    ("a half window inf", edit("window_min", 1, np.inf), VE, "half windows must be finite and > 0 minutes"),
    ("a radius < 0", edit("hbr_km", 0, -1.0), VE, "hard-body radii must be finite and >= 0 km"),
    ("a radius nan", edit("hbr_km", 1, np.nan), VE, "hard-body radii must be finite and >= 0 km"),
    ("an element not finite", edit("elements", (3, 2), np.nan), VE, ELEMENTS),
    ("a covariance word not finite", edit("covariance", (2, 27), np.nan), VE, COVARIANCE),
    ("a time not finite", edit("fr", 0, np.inf), VE, "guess times must be finite"),
    ("a model byte", edit("model", 2, 9), VE, MODEL),
    ("states, state_covariance and model NULL", set_(states=None, state_covariance=None, model=None), ND,
     NO_DEVICE)] + VALID
CONJ_DEVICE = CONJ_SCALARS + nulls("elements", "covariance", "primary", "secondary", "jd", "fr", "window_min",
                                   "hbr_km", "record", "status") + [
    ("states, state_covariance and model NULL", set_(states=None, state_covariance=None, model=None), ND,
     NO_DEVICE)] + VALID

CORR_SCALARS = [("device < 0", set_(device=-1), VE, "track correlation runs on one device: pass its ordinal"),
                ("grav", set_(grav=9), VE, GRAV),
                ("best 0", set_(best=0), VE, "best must be in [1, ASTROZ_CORR_MAX_BEST]"),
                ("best 9", set_(best=9), VE, "best must be in [1, ASTROZ_CORR_MAX_BEST]"),
                ("gate 0", set_(gate_probability=0.0), VE, "gate_probability must be in (0, 1)"),
                ("gate 1", set_(gate_probability=1.0), VE, "gate_probability must be in (0, 1)"),
                ("n = t = 0", set_(n=0, t=0, offsets=np.zeros(1, np.uint32), m=0), OK, UNCHANGED)]
CORR_HOST = CORR_SCALARS + nulls("elements", "row_status", "rows", "d2", "used", "n_gate", "n_failed", "status",
                                 "jd", "fr", "kind", "value", "sigma") + track_offset_rows(
    "ASTROZ_CORR_MAX_TRACK") + obs_value_rows() + [
    ("a track with no used residual", no_used_residual, VE, USED),
    ("an element not finite", edit("elements", (1, 1), np.nan), VE, ELEMENTS),
    ("a covariance word not finite", edit("covariance", (0, 0), np.inf), VE, COVARIANCE),
    ("a model byte", edit("model", 0, 2), VE, MODEL),
    ("covariance, model, station and stations NULL",
     lambda a: a.update(covariance=None, model=None, kind=np.zeros(4, np.uint8), station=None, stations=None, k=0),
     ND, NO_DEVICE)] + VALID
CORR_DEVICE = CORR_SCALARS + nulls("elements", "row_status", "offsets", "scratch", "jd", "fr", "kind", "value",
                                   "sigma", "rows", "d2", "used", "n_gate", "n_failed", "status") + [
    ("covariance, model, station and stations NULL", set_(covariance=None, model=None, station=None, stations=None),
     ND, NO_DEVICE)] + VALID

IOD_SCALARS = [("device < 0", set_(device=-1), VE,
                "initial orbit determination runs on one device: pass its ordinal"),
               ("grav", set_(grav=2), VE, GRAV),
               ("t = 0", set_(t=0, offsets=np.zeros(1, np.uint32), m=0), OK, UNCHANGED)]
IOD_HOST = IOD_SCALARS + nulls("elements", "state", "wrms", "method", "candidates", "conv", "deep_space", "status",
                               "jd", "fr", "kind", "value", "sigma") + track_offset_rows(
    "ASTROZ_IOD_MAX_TRACK") + obs_value_rows() + [
    ("a track with no used residual", no_used_residual, VE, USED),
    ("a bstar not finite", edit("bstar", 1, np.nan), VE, "bstar must be finite"),
    ("bstar, station and stations NULL",
     lambda a: a.update(bstar=None, kind=np.zeros(4, np.uint8), station=None, stations=None, k=0), ND,
     NO_DEVICE)] + VALID
IOD_DEVICE = IOD_SCALARS + nulls("offsets", "jd", "fr", "kind", "value", "sigma", "scratch", "elements", "state",
                                 "wrms", "method", "candidates", "conv", "deep_space", "status") + [
    ("bstar, station and stations NULL", set_(bstar=None, station=None, stations=None), ND, NO_DEVICE)] + VALID

LAMBERT_SCALARS = [("device < 0", set_(device=-1), VE, "a Lambert call runs on one device: pass its ordinal"),
                   ("mu 0", set_(mu=0.0), VE, "mu must be finite and > 0"),
                   ("mu nan", set_(mu=np.nan), VE, "mu must be finite and > 0"),
                   ("max_revs 128", set_(max_revs=128), VE, "max_revs must be at most 127"),
                   ("n = 0", set_(n=0, r1=None, v1=None), OK, UNCHANGED)]
LAMBERT_HOST = LAMBERT_SCALARS + nulls("r1", "r2", "tof", "v1", "v2", "status") + [
    ("r1 not finite", edit("r1", (1, 1), np.nan), VE, "r1, r2, tof and normal must be finite"),
    ("r2 not finite", edit("r2", (0, 2), np.inf), VE, "r1, r2, tof and normal must be finite"),
    ("tof not finite", edit("tof", 1, np.nan), VE, "r1, r2, tof and normal must be finite"),
    ("normal not finite", edit("normal", (0, 0), np.nan), VE, "r1, r2, tof and normal must be finite"),
    ("normal and iterations NULL", set_(normal=None, iterations=None), ND, NO_DEVICE)] + VALID
LAMBERT_DEVICE = LAMBERT_SCALARS + nulls("r1", "r2", "tof", "v1", "v2", "status") + [
    ("a NaN tof is not read", edit("tof", 1, np.nan), ND, NO_DEVICE),
    ("normal and iterations NULL", set_(normal=None, iterations=None), ND, NO_DEVICE)] + VALID

TABLE = {
    "astroz_cuda_fit_elements": (fit_scene, FIT_HOST),
    "astroz_cuda_fit_elements_mixed": (fit_scene, FIT_HOST),
    "astroz_cuda_fit_elements_device": (fit_scene, FIT_DEVICE),
    "astroz_cuda_fit_elements_mixed_device": (fit_scene, FIT_DEVICE),
    "astroz_cuda_fit_observations": (fit_obs_scene, FIT_OBS_HOST),
    "astroz_cuda_fit_observations_mixed": (fit_obs_scene, FIT_OBS_HOST),
    "astroz_cuda_fit_observations_device": (fit_obs_scene, FIT_OBS_DEVICE),
    "astroz_cuda_fit_observations_mixed_device": (fit_obs_scene, FIT_OBS_DEVICE),
    "astroz_cuda_observe": (observe_scene, OBSERVE_HOST),
    "astroz_cuda_observe_device": (observe_scene, OBSERVE_DEVICE),
    "astroz_cuda_propagate_covariance": (cov_scene, COV_HOST),
    "astroz_cuda_propagate_covariance_device": (cov_scene, COV_DEVICE),
    "astroz_cuda_conjunction": (conj_scene, CONJ_HOST),
    "astroz_cuda_conjunction_device": (conj_scene, CONJ_DEVICE),
    "astroz_cuda_correlate": (corr_scene, CORR_HOST),
    "astroz_cuda_correlate_device": (corr_scene, CORR_DEVICE),
    "astroz_cuda_initial_orbits": (iod_scene, IOD_HOST),
    "astroz_cuda_initial_orbits_device": (iod_scene, IOD_DEVICE),
    "astroz_cuda_lambert": (lambert_scene, LAMBERT_HOST),
    "astroz_cuda_lambert_device": (lambert_scene, LAMBERT_DEVICE),
}
CASES = [pytest.param(call, change, rc, text, id=f"{call.removeprefix('astroz_cuda_')}: {label}")
         for call, (_, rows) in TABLE.items() for label, change, rc, text in rows]


def argument(call, p, a):
    """The table's argument for parameter p: host names, a device twin's d_ names mapped to them, no stream."""
    if p == "stream":
        return None
    name = p.removeprefix("d_") if call.endswith("_device") else p
    v = a[name]
    return C.c_void_p(v.ctypes.data) if isinstance(v, np.ndarray) else v


@pytest.mark.parametrize("call,change,rc,text", CASES)
def test_whole_batch_call_checks(call, change, rc, text):
    from astroz_b200._lib import lib

    L = lib()
    if rc == ND and L.astroz_cuda_device_count() > 0:
        pytest.skip("a device is visible: the call would run")
    scene, _ = TABLE[call]
    a = scene()
    change(a)
    outputs = {p: a[p].tobytes() for p in a if is_output(call, p) and isinstance(a[p], np.ndarray)}
    x = C.c_double(5.0)
    assert L.astroz_cuda_chi2_quantile(0, 0.5, C.byref(x)) == VE
    got = getattr(L, call)(*[argument(call, p, a) for p in PARAMS[call]])
    assert (got, L.astroz_cuda_last_error().decode()) == (rc, text)
    assert {p: a[p].tobytes() for p in outputs} == outputs


def test_every_whole_batch_call_is_in_the_table():
    host = ["fit_elements", "fit_elements_mixed", "fit_observations", "fit_observations_mixed", "observe",
            "propagate_covariance", "conjunction", "correlate", "initial_orbits", "lambert"]
    names = {f"astroz_cuda_{h}{s}" for h in host for s in ("", "_device")}
    assert names == set(TABLE) and names <= set(PARAMS)
    for call, (scene, _) in TABLE.items():
        a = scene()
        assert all(p == "stream" or (p.removeprefix("d_") if call.endswith("_device") else p) in a
                   for p in PARAMS[call]), call
