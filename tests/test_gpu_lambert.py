"""K9 Lambert on the H100: the device solver against the scalar C statement (tests/lambert_oracle), closure of its
outputs, host vs device calls, batch independence, and porkchop grids against the pairs path, lambert_batch, a CPU brute
force over the oracle's SGP4/SDP4 states, and the Hohmann transfer."""
import math

import numpy as np
import pytest

from tests import lambert_oracle as L
from tests.test_lambert_cpu import closure, random_problems

pytestmark = pytest.mark.gpu

MU = 398600.5
MU72 = 398600.8
OK, NO_SOLUTION, STATE_FAILED = 0, 1, 4


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def _clear_of_tmin(r1, r2, tof, normal, max_revs, margin=1e-5):
    """Problems whose tof is at least `margin` relative away from T_min(M) of every M <= max_revs (near T_min the two
    branches form a double root; the CPU tests cover the boundary)."""
    keep = np.ones(len(tof), dtype=bool)
    for i in range(len(tof)):
        g = L.geometry(r1[i], r2[i], tof[i], MU, normal[i])
        if g is None:
            continue
        lam, T = g
        for M in range(1, min(max_revs, int(T / math.pi)) + 1):
            if abs(T / L.t_min(lam, M) - 1) < margin:
                keep[i] = False
                break
    return r1[keep], r2[keep], tof[keep], normal[keep]


@pytest.fixture(scope="module")
def problems():
    rng = np.random.default_rng(2026)
    return _clear_of_tmin(*random_problems(rng, 100_000, 10), 10)


def test_device_matches_the_statement_and_closes(problems):
    from astroz_b200.lambert import lambert_batch

    r1, r2, tof, normal = problems
    assert len(tof) > 99_000
    v1, v2, st, it = lambert_batch(r1, r2, tof, MU, max_revs=10, normal=normal)
    w1, w2, wst, wit = L.solve(r1, r2, tof, MU, max_revs=10, normal=normal, threads=8)
    assert np.array_equal(st, wst)
    assert np.abs(v1 - w1).max() <= 1e-9 and np.abs(v2 - w2).max() <= 1e-9
    assert np.sum(st == OK) > 250_000   # 292,840 for this seed: multi-revolution slots of both branches
    assert closure(r1[:4000], r2[:4000], tof[:4000], v1[:4000], v2[:4000], st[:4000], MU) > 8000


def test_host_and_device_calls_are_byte_identical_over_pageable_and_pinned(problems):
    import torch

    from astroz_b200 import pinned_empty
    from astroz_b200.lambert import lambert_batch, lambert_batch_device

    r1, r2, tof, normal = (a[:20_000] for a in problems)
    host = lambert_batch(r1, r2, tof, MU, max_revs=4, normal=normal)
    pins = []
    for a in (r1, r2, tof, normal):
        p = pinned_empty(a.shape)
        p[...] = a
        pins.append(p)
    pinned = lambert_batch(*pins[:3], MU, max_revs=4, normal=pins[3])
    dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (r1, r2, tof, normal)]
    n, S = len(tof), 9
    out = [torch.zeros((n, S, 3), dtype=torch.float64, device="cuda") for _ in range(2)]
    st, it = (torch.zeros((n, S), dtype=torch.uint8, device="cuda") for _ in range(2))
    lambert_batch_device(dev[0], dev[1], dev[2], out[0], out[1], st, MU, iterations=it, normal=dev[3], max_revs=4)
    torch.cuda.synchronize()
    device = (out[0].cpu().numpy(), out[1].cpu().numpy(), st.cpu().numpy(), it.cpu().numpy())
    for a, b, c in zip(host, pinned, device):
        assert np.array_equal(_bits(a), _bits(b)) and np.array_equal(_bits(a), _bits(c))


def test_a_problems_bytes_do_not_depend_on_the_batch(problems):
    from astroz_b200.lambert import lambert_batch

    r1, r2, tof, normal = (a[:5000] for a in problems)
    full = lambert_batch(r1, r2, tof, MU, max_revs=3, normal=normal)
    perm = np.random.default_rng(1).permutation(len(tof))
    dup = np.concatenate([perm, perm[:777]])
    shuffled = lambert_batch(r1[dup], r2[dup], tof[dup], MU, max_revs=3, normal=normal[dup])
    for a, b in zip(full, shuffled):
        assert np.array_equal(_bits(a[dup]), _bits(b))
    for i in (0, 17, 4999):
        alone = lambert_batch(r1[i:i + 1], r2[i:i + 1], tof[i:i + 1], MU, max_revs=3, normal=normal[i:i + 1])
        for a, b in zip(full, alone):
            assert np.array_equal(_bits(a[i:i + 1]), _bits(b))


def _catalog():
    """A small mixed catalogue: config-2 near-earth objects with GEO, Molniya and GPS-like objects, and one object low
    and draggy enough to decay during the grid."""
    from astroz_b200 import synth

    tles = synth.mixed_catalog(64, n_geo=6, n_molniya=4, n_gps=2)
    a = 6378.135 + 190.0
    tles.append(synth.tle_lines(99999, 24, 127.0, 51.6, 10.0, 0.001, 0.0, 0.0, 86400 / (2 * math.pi) *
                                math.sqrt(MU72 / a ** 3), 0.5))
    return tles


def _grid(n_dep, n_arr, days):
    jd0 = 2460437.5   # 2024-05-06 00:00 UTC
    dep_fr = np.arange(n_dep) * (0.5 / n_dep)
    arr_fr = 0.2 + np.arange(n_arr) * (days / n_arr)
    return np.full(n_dep, jd0), dep_fr, np.full(n_arr, jd0), arr_fr


def test_constellation_porkchop_equals_pairs_then_porkchop_device_over_chunks():
    import torch

    from astroz_b200 import Constellation
    from astroz_b200.lambert import porkchop_device

    tles = _catalog()
    c = Constellation(tles, device=0)
    rng = np.random.default_rng(5)
    P, Dn, An = 700, 96, 96   # ~166 KB of grid per pair: several chunks
    chaser, target = rng.integers(0, len(tles), P), rng.integers(0, len(tles), P)
    dep_jd, dep_fr, arr_jd, arr_fr = _grid(Dn, An, 1.0)
    dv, slot, st = c.porkchop(chaser, target, dep_jd, dep_fr, arr_jd, arr_fr, max_revs=2)
    assert dv.shape == (P, Dn, An, 2)

    def states(rows, jd, fr):
        k = len(jd)
        sat = torch.tensor(np.repeat(rows, k).astype(np.int32), device="cuda")
        tj = torch.tensor(np.tile(jd, len(rows)), device="cuda")
        tf = torch.tensor(np.tile(fr, len(rows)), device="cuda")
        pos = torch.zeros((len(rows) * k, 3), dtype=torch.float64, device="cuda")
        vel, s = torch.zeros_like(pos), torch.zeros(len(rows) * k, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()   # the handle's stream does not wait for torch's
        c.propagate_pairs_device(sat, tj, tf, pos, vel, s)
        c.synchronize()
        return torch.cat([pos, vel], 1).reshape(len(rows), k, 6).contiguous(), s.reshape(len(rows), k)

    ds, dst = states(chaser, dep_jd, dep_fr)
    as_, ast = states(target, arr_jd, arr_fr)
    t = [torch.tensor(a, device="cuda") for a in (dep_jd, dep_fr, arr_jd, arr_fr)]
    ddv = torch.zeros((P, Dn, An, 2), dtype=torch.float64, device="cuda")
    dslot, dstat = (torch.zeros((P, Dn, An), dtype=torch.uint8, device="cuda") for _ in range(2))
    porkchop_device(ds, dst, as_, ast, *t, MU72, ddv, dslot, dstat, max_revs=2)
    torch.cuda.synchronize()
    assert np.array_equal(_bits(dv), _bits(ddv.cpu().numpy()))
    assert np.array_equal(slot, dslot.cpu().numpy()) and np.array_equal(st, dstat.cpu().numpy())
    assert np.sum(st == OK) > 0.5 * st.size


def test_every_porkchop_cell_is_the_best_slot_of_lambert_batch():
    from astroz_b200 import Constellation
    from astroz_b200.lambert import lambert_batch

    tles = _catalog()
    c = Constellation(tles, device=0)
    rng = np.random.default_rng(8)
    P, Dn, An = 12, 8, 10
    chaser, target = rng.integers(0, len(tles), P), rng.integers(0, len(tles), P)
    dep_jd, dep_fr, arr_jd, arr_fr = _grid(Dn, An, 1.5)
    dv, slot, st = c.porkchop(chaser, target, dep_jd, dep_fr, arr_jd, arr_fr, max_revs=3)
    pc, vc, sc = c.propagate_pairs(np.repeat(chaser, Dn), np.tile(dep_jd, P), np.tile(dep_fr, P))
    pt, vt, stt = c.propagate_pairs(np.repeat(target, An), np.tile(arr_jd, P), np.tile(arr_fr, P))
    pc, vc, sc = pc.reshape(P, Dn, 3), vc.reshape(P, Dn, 3), sc.reshape(P, Dn)
    pt, vt, stt = pt.reshape(P, An, 3), vt.reshape(P, An, 3), stt.reshape(P, An)
    p, d, a = (x.ravel() for x in np.meshgrid(np.arange(P), np.arange(Dn), np.arange(An), indexing="ij"))
    tof = ((arr_jd[a] - dep_jd[d]) + (arr_fr[a] - dep_fr[d])) * 86400.0
    v1, v2, s_all, _ = lambert_batch(pc[p, d], pt[p, a], tof, MU72, max_revs=3, normal=np.cross(pc[p, d], vc[p, d]))
    cost = np.linalg.norm(v1 - vc[p, d][:, None], axis=2) + np.linalg.norm(vt[p, a][:, None] - v2, axis=2)
    cost[s_all != OK] = np.inf
    failed = (sc[p, d] != 0) | (stt[p, a] != 0)
    best = np.argmin(cost, axis=1)
    has = np.isfinite(cost.min(axis=1))
    want_st = np.where(failed, STATE_FAILED, np.where(has, OK, s_all[:, 0]))
    assert np.array_equal(st.ravel(), want_st)
    sel = has & ~failed
    assert np.array_equal(slot.ravel()[sel], best[sel])
    got = dv.reshape(-1, 2)
    assert np.abs(got[sel].sum(axis=1) - cost[sel].min(axis=1)).max() < 1e-12
    assert not np.any(got[~sel]) and not np.any(slot.ravel()[~sel])


def test_porkchop_against_a_cpu_brute_force_over_the_oracles_states():
    from astroz_b200 import Constellation
    from oracle import oracle as orc

    tles = _catalog()
    c = Constellation(tles, device=0)
    klass = np.asarray(c.classes)
    geo = int(np.flatnonzero(klass == 2)[0])       # irez 1: GEO
    molniya = int(np.flatnonzero(klass == 3)[0])   # irez 2: Molniya
    leo = [int(i) for i in np.flatnonzero(klass == 0)[:3]]
    decayed = len(tles) - 1
    chaser = np.array([leo[0], leo[1], leo[2], leo[0], leo[1]])
    target = np.array([geo, molniya, decayed, leo[1], leo[2]])
    Dn, An = 6, 9
    dep_jd, dep_fr, arr_jd, arr_fr = _grid(Dn, An, 5.0)
    arr_fr[0] = dep_fr[2]      # tof = 0 and tof < 0 cells
    dv, slot, st = c.porkchop(chaser, target, dep_jd, dep_fr, arr_jd, arr_fr, max_revs=2)
    pd, vd, ed, _ = orc.constellation_propagate(tles, dep_jd, dep_fr)
    pa, va, ea, _ = orc.constellation_propagate(tles, arr_jd, arr_fr)
    # a near-earth cell below one earth radius is stored and flagged decayed by the pairs path (the oracle's grid
    # stores it without a flag): both are a failed endpoint
    ed = ed.astype(bool) | (np.linalg.norm(pd, axis=2) < 6378.135)
    ea = ea.astype(bool) | (np.linalg.norm(pa, axis=2) < 6378.135)
    P = len(chaser)
    for p in range(P):
        for d in range(Dn):
            for a in range(An):
                if ed[chaser[p], d] or ea[target[p], a]:
                    assert st[p, d, a] == STATE_FAILED
                    continue
                tof = ((arr_jd[a] - dep_jd[d]) + (arr_fr[a] - dep_fr[d])) * 86400.0
                rc, vc, rt, vt = pd[chaser[p], d], vd[chaser[p], d], pa[target[p], a], va[target[p], a]
                v1, v2, s_all, _ = L.solve(rc, rt, tof, MU72, max_revs=2, normal=np.cross(rc, vc))
                ok = np.flatnonzero(s_all[0] == OK)
                if not len(ok):
                    assert st[p, d, a] == s_all[0, 0] and not np.any(dv[p, d, a])
                    continue
                cost = np.linalg.norm(v1[0, ok] - vc, axis=1) + np.linalg.norm(vt - v2[0, ok], axis=1)
                assert st[p, d, a] == OK and slot[p, d, a] == ok[np.argmin(cost)]
                assert abs(dv[p, d, a].sum() - cost.min()) < 1e-6
    assert np.any(st == STATE_FAILED) and np.any(st[:, 2:, 0] == NO_SOLUTION)
    assert np.sum(st == OK) > P * Dn * An // 2


def test_porkchop_minimum_between_coplanar_circular_orbits_is_the_hohmann_transfer():
    import torch

    from astroz_b200.lambert import porkchop_device

    ra, rb = 7000.0, 8000.0
    na, nb = math.sqrt(MU / ra ** 3), math.sqrt(MU / rb ** 3)
    at = (ra + rb) / 2
    t_h = math.pi * math.sqrt(at ** 3 / MU)
    hohmann = (math.sqrt(MU / ra) * (math.sqrt(2 * rb / (ra + rb)) - 1) +
               math.sqrt(MU / rb) * (1 - math.sqrt(2 * ra / (ra + rb))))
    Dn, An = 41, 81
    dep_t = np.linspace(-200.0, 200.0, Dn)
    arr_t = t_h + np.linspace(-0.1, 0.1, An) * t_h
    phase = math.pi - nb * t_h + 3e-3   # the target passes the chaser's antipode near t_h (exactly there is degenerate)

    def circ(r, n, th):
        return np.stack([r * np.cos(th), r * np.sin(th), np.zeros_like(th), -r * n * np.sin(th), r * n * np.cos(th),
                         np.zeros_like(th)], axis=1)

    dep = circ(ra, na, na * dep_t)[None]
    arr = circ(rb, nb, phase + nb * arr_t)[None]
    to = lambda a: torch.tensor(np.ascontiguousarray(a), device="cuda")  # noqa: E731
    dv = torch.zeros((1, Dn, An, 2), dtype=torch.float64, device="cuda")
    slot, st = (torch.zeros((1, Dn, An), dtype=torch.uint8, device="cuda") for _ in range(2))
    porkchop_device(to(dep), None, to(arr), None, to(np.zeros(Dn)), to(dep_t / 86400.0), to(np.zeros(An)),
                    to(arr_t / 86400.0), MU, dv, slot, st)
    torch.cuda.synchronize()
    st, total = st.cpu().numpy(), dv.sum(-1).cpu().numpy()
    assert np.mean(st == OK) > 0.99
    best = total[st == OK].min()
    assert abs(best - hohmann) < 0.01 * hohmann, (best, hohmann)


def test_constellation_porkchop_refuses_rows_outside_the_catalog():
    from astroz_b200 import AstrozCudaError, Constellation

    tles = _catalog()
    c = Constellation(tles, device=0)
    jd, fr, ajd, afr = _grid(2, 2, 1.0)
    with pytest.raises(AstrozCudaError, match="valueError"):
        c.porkchop([0], [len(tles)], jd, fr, ajd, afr)
    with pytest.raises(AstrozCudaError, match="valueError"):
        c.porkchop([0], [1], jd, fr, ajd, afr, mu=-1.0)
