// az_pairs.cuh -- per-query cores of K6, the (satellite, time) pairs path: query i propagates catalog row sat[i] to
// its own epoch jd[i] + fr[i] (what a loop of Satrec.sgp4(jd, fr) calls does one launch at a time,
// bindings/python/src/satrec.zig:169-201).  __host__ __device__, so tests/host_emul runs the same arithmetic on the CPU.
//
// Every value a query produces is a function of (sat, jd, fr) and the handle's tables alone: one query per thread, the
// single-cell form of the cores (the K1 grid chooses its Kepler / drag-rotation series per thread over 2-3 epochs, so a
// shape that puts several queries in one thread would let neighbouring queries change each other's low bits).
#pragma once

#include "az_device.cuh"
#include "az_elements.hpp"

namespace az {

constexpr uint8_t kCellBadSatellite = 3;  // ASTROZ_CELL_BAD_SATELLITE: sat[i] is not a catalog row

// The time model and the GMST below are written in add_rn / sub_rn / mul_rn (az_math.cuh): they must reproduce, bit for
// bit, the expressions the grid path evaluates on the host (upload_time_axis, julian_to_gmst).

// Near-earth minutes since epoch: the grid's tbase[t] + toff[s], tbase = ((jd + fr) - referenceEpochJd) * 1440
// (src/Constellation.zig:425), toff[s] = (referenceEpochJd - epoch[s]) * 1440 from the handle's table.
AZ_HD double pairs_tsince_near(double jdFull, double refJd, double toff) {
    return add_rn(mul_rn(sub_rn(jdFull, refJd), 1440.0), toff);
}
// Deep space: ((jd + fr) - epoch) * 1440 (src/Constellation.zig:465).
AZ_HD double pairs_tsince_deep(double jdFull, double epochJd) { return mul_rn(sub_rn(jdFull, epochJd), 1440.0); }

// julian_to_gmst (src/WorldCoordinateSystem.zig:146-154) operation by operation, uncontracted, so the angle equals the
// host's to the bit; its sine and cosine come from the library's own reduction (sincos_full, 4e-16).
AZ_HD double pairs_gmst(double jd) {
    const double d = sub_rn(jd, 2451545.0);
    const double t = d / 36525.0;
    const double t2 = mul_rn(t, t);
    double gmst = add_rn(280.46061837, mul_rn(360.98564736629, d));
    gmst = add_rn(gmst, mul_rn(mul_rn(0.000387933, t), t));
    gmst = sub_rn(gmst, mul_rn(t2, t) / 38710000.0);
    gmst = detail::wrap(gmst, 360.0);
    if (gmst < 0) gmst = add_rn(gmst, 360.0);
    return mul_rn(gmst, detail::kDeg);
}

// TEME -> the output frame of the query's own epoch: the grid's epilogues (pure GMST rotation, no omega x r).
template <int kMode, bool kVel>
AZ_HD void pairs_frame(double jdFull, CellOut &o) {
    if (kMode != 0) {
        double sg, cg;
        sincos_full(pairs_gmst(jdFull), sg, cg);
        eci_to_ecef(o.rx, o.ry, sg, cg);
        if (kVel) eci_to_ecef(o.vx, o.vy, sg, cg);
        if (kMode == 2) ecef_to_geodetic(o.rx, o.ry, o.rz);
    }
}

// One near-earth query.  col(i) = column i of the query's satellite; returns the status byte (DECAYED diagnostic only:
// the state is always stored, like the grid).
template <int kMode, bool kVel, typename ColFn>
AZ_HD uint8_t pairs_sgp4_query(ColFn col, double jdFull, double refJd, double toff, const GravConsts &g, CellOut &o) {
    const double ts[1] = {pairs_tsince_near(jdFull, refJd, toff)};
    CellOut o1[1];
    sgp4_cell<1>(col, ts, g, o1);
    o = o1[0];
    const uint8_t st = (o.mrt < 1.0) ? 1 : 0;
    pairs_frame<kMode, kVel>(jdFull, o);
    return st;
}

// One deep-space cell at tsince ts [min] into o (TEME), its ASTROZ_CELL_* code returned.  lattice = this satellite's
// [2][nodes] resonance checkpoints (K2a); the state is taken at the node below |tsince| and stepped on from there,
// exactly as K2 does (so the result does not depend on the lattice's extent).
AZ_HD int pairs_sdp4_at(const Sdp4Sat &e, const double2 *lattice, int nodes, double ts, const GravConsts &g,
                        CellOut &o) {
    double xli = e.xlamo, xni = e.no, atime = 0.0;
    if (e.irez != 0) {
        const int node = resonance_node(ts);
        const int have = node < nodes - 1 ? node : nodes - 1;
        const double2 st = lattice[(ts > 0.0 ? 0 : 1) * nodes + have];
        const double delt = ts > 0.0 ? kStepp : -kStepp;
        xli = st.x;
        xni = st.y;
        atime = delt * (double)have;
        for (int j = have; j < node; ++j) resonance_step(e, xli, xni, atime, delt);  // beyond the lattice
    }
    return sdp4_cell(e, ts, xli, xni, atime, g, o);
}

// One deep-space query at its own epoch jd + fr, in the output frame of kMode.  A failing cell is zero-filled; returns
// its ASTROZ_CELL_* code.
template <int kMode, bool kVel>
AZ_HD uint8_t pairs_sdp4_query(const Sdp4Sat &e, const double2 *lattice, int nodes, double jdFull, const GravConsts &g,
                               CellOut &o) {
    const int st = pairs_sdp4_at(e, lattice, nodes, pairs_tsince_deep(jdFull, e.epochJd), g, o);
    if (st != 0) {
        o.rx = o.ry = o.rz = o.vx = o.vy = o.vz = 0.0;
    } else {
        pairs_frame<kMode, kVel>(jdFull, o);
    }
    return (uint8_t)st;
}

}  // namespace az
