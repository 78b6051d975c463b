// TEST INFRASTRUCTURE ONLY: runs the product's __host__ __device__ per-cell cores (az_device.cuh) on the
// CPU with the product's own host tables, so the kernel arithmetic can be checked against the oracle in
// a container without a GPU.  Not part of the shipped library; nothing in astroz_b200/ references it.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <vector>

#include "az_tables.hpp"

using namespace az;  // (az::* names do not collide with CUDA math: rsqrt_nr, div_nr)

static int g_lanes = 1;
extern "C" void emul_set_lanes(int lanes) { g_lanes = lanes; }

extern "C" int emul_constellation_propagate(const char *const *l1, const char *const *l2, uint32_t n, int grav,
                                            const double *jd, const double *fr, uint32_t nt, double *pos, double *vel,
                                            uint8_t *status) {
    CatalogTables cat;
    int rc = build_catalog(l1, l2, n, grav, cat);
    if (rc != kOk) return rc;
    const GravConsts g = grav_consts(cat.grav);
    std::vector<double> jdFull(nt), tbase(nt);
    for (uint32_t t = 0; t < nt; ++t) {
        jdFull[t] = jd[t] + fr[t];
        tbase[t] = (jdFull[t] - cat.referenceEpochJd) * 1440.0;
    }
    for (uint32_t s = 0; s < cat.nSgp4; ++s) {
        const double *tile = cat.sgp4Tiles.data() + (size_t)(s / kTileSats) * kSgp4TileDoubles;
        const int sl = s % kTileSats;
        auto col = [&](int i) { return tile[i * kTileSats + sl]; };
        const double toff = (cat.referenceEpochJd - cat.sgp4Epoch[s]) * 1440.0;
        const uint32_t orig = cat.sgp4Orig[s];
        if (g_lanes == 3) {
            // the shipped near-earth shape: runs of 96 epochs, a thread owning epochs tw + lane, + 32, + 64 (clamped at
            // the end of the axis), so the speculative-path flags are ANDed over exactly the cells the kernel groups
            for (uint32_t tw = 0; tw < nt; tw += 96) {
                for (uint32_t lane = 0; lane < 32; ++lane) {
                    double ts[3];
                    for (int k = 0; k < 3; ++k) ts[k] = tbase[std::min(tw + 32u * k + lane, nt - 1)] + toff;
                    CellOut o3[3];
                    sgp4_cell<3>(col, ts, g, o3);
                    for (int k = 0; k < 3; ++k) {
                        const uint32_t tk = tw + 32u * k + lane;
                        if (tk >= nt) continue;
                        double *p = pos + ((size_t)orig * nt + tk) * 3, *v = vel + ((size_t)orig * nt + tk) * 3;
                        p[0] = o3[k].rx; p[1] = o3[k].ry; p[2] = o3[k].rz;
                        v[0] = o3[k].vx; v[1] = o3[k].vy; v[2] = o3[k].vz;
                        if (status) status[(size_t)orig * nt + tk] = o3[k].mrt < 1.0 ? 1 : 0;
                    }
                }
            }
            continue;
        }
        for (uint32_t t = 0; t < nt; t += g_lanes) {
            CellOut oo[2];
            if (g_lanes == 2) {  // the kernel's 2-epochs-per-thread path (second lane clamped at the end)
                const uint32_t tb = t + 1 < nt ? t + 1 : nt - 1;
                const double ts[2] = {tbase[t] + toff, tbase[tb] + toff};
                sgp4_cell<2>(col, ts, g, oo);
            } else {
                CellOut o1[1];
                const double ts[1] = {tbase[t] + toff};
                sgp4_cell<1>(col, ts, g, o1);
                oo[0] = o1[0];
            }
            for (int k = 0; k < g_lanes && t + k < nt; ++k) {
                const CellOut &o = oo[k];
                double *p = pos + ((size_t)orig * nt + t + k) * 3, *v = vel + ((size_t)orig * nt + t + k) * 3;
                p[0] = o.rx; p[1] = o.ry; p[2] = o.rz; v[0] = o.vx; v[1] = o.vy; v[2] = o.vz;
                if (status) status[(size_t)orig * nt + t + k] = o.mrt < 1.0 ? 1 : 0;
            }
        }
    }
    const int dsLanes = g_lanes == 2 ? 2 : 1;  // the deep-space grid ships one epoch per thread
    for (uint32_t s = 0; s < cat.nSdp4; ++s) {
        const Sdp4Sat &e = cat.sdp4[s];
        const uint32_t orig = cat.sdp4Orig[s];
        for (uint32_t t = 0; t < nt; t += dsLanes) {
            double ts[2], xli[2], xni[2], atime[2];
            for (int k = 0; k < 2; ++k) {  // the kernel's lattice walk, from node 0 (no lattice cache on the host)
                const uint32_t tk = t + k < nt ? t + k : nt - 1;
                ts[k] = (jdFull[tk] - e.epochJd) * 1440.0;
                xli[k] = e.xlamo; xni[k] = e.no; atime[k] = 0.0;
                if (e.irez != 0) {
                    const int node = resonance_node(ts[k]);
                    const double delt = ts[k] > 0.0 ? kStepp : -kStepp;
                    for (int j = 0; j < node; ++j) resonance_step(e, xli[k], xni[k], atime[k], delt);
                }
            }
            CellOut oo[2];
            int st[2] = {0, 0};
            if (dsLanes == 2) {  // the two-epochs-per-thread form of the core
                sdp4_cell_n<2>(e, ts, xli, xni, atime, g, oo, st);
            } else {
                st[0] = sdp4_cell(e, ts[0], xli[0], xni[0], atime[0], g, oo[0]);
            }
            for (int k = 0; k < dsLanes && t + k < nt; ++k) {
                const CellOut &o = oo[k];
                double *p = pos + ((size_t)orig * nt + t + k) * 3, *v = vel + ((size_t)orig * nt + t + k) * 3;
                if (st[k] != 0) { p[0] = p[1] = p[2] = v[0] = v[1] = v[2] = 0.0; }
                else { p[0] = o.rx; p[1] = o.ry; p[2] = o.rz; v[0] = o.vx; v[1] = o.vy; v[2] = o.vz; }
                if (status) status[(size_t)orig * nt + t + k] = (uint8_t)st[k];
            }
        }
    }
    return 0;
}

// The quantities that pick a core's series path, per (satellite, epoch), from the product's host tables: lets a fixture
// prove which path it reaches.  Near-earth rows: [0] tho, the drag angle sgp4_cell rotates by (0 when isimp is set);
// [1] ecco - tempe before the 1e-6 floor; [2] the Newton loop's first step (e sin E) / (1 - e cos E) before the +-0.95
// clamp; [3] -1.  Deep-space rows: [0..2] 0, [3] irez.  ecco[n] and inclo[n] (rad) per satellite.
extern "C" int emul_regimes(const char *const *l1, const char *const *l2, uint32_t n, int grav, const double *jd,
                            const double *fr, uint32_t nt, double *out, double *ecco, double *inclo) {
    CatalogTables cat;
    int rc = build_catalog(l1, l2, n, grav, cat);
    if (rc != kOk) return rc;
    for (uint32_t s = 0; s < cat.nSgp4; ++s) {
        const double *tile = cat.sgp4Tiles.data() + (size_t)(s / kTileSats) * kSgp4TileDoubles;
        const int sl = s % kTileSats;
        auto col = [&](int i) { return tile[i * kTileSats + sl]; };
        const uint32_t orig = cat.sgp4Orig[s];
        ecco[orig] = col(kEcco);
        inclo[orig] = std::atan2(col(kSinio), col(kCosio));
        for (uint32_t k = 0; k < nt; ++k) {
            // sgp4_cell's secular and drag update, one lane
            const double t = ((jd[k] + fr[k]) - cat.referenceEpochJd) * 1440.0 +
                             (cat.referenceEpochJd - cat.sgp4Epoch[s]) * 1440.0;
            const double t2 = t * t, t3 = t2 * t, t4 = t3 * t;
            const double xmdf = fma(col(kMdot), t, col(kMo));
            double argpm = fma(col(kArgpdot), t, col(kArgpo)), mm = xmdf, tho = 0.0;
            double tempa = fma(-col(kCc1), t, 1.0), tempe = col(kBc4) * t, templ = col(kT2cof) * t2;
            if (col(kIsimp) == 0.0) {
                double sm, cm, sd, cd;
                sincos_full(xmdf, sm, cm);
                const double dm = fma(col(kEta), cm, 1.0);
                tho = fma(col(kOmgcof), t, col(kXmcof) * (dm * dm * dm - col(kDelmo)));
                mm = xmdf + tho;
                argpm -= tho;
                sincos_full(tho, sd, cd);
                tempa = tempa - col(kD2) * t2 - col(kD3) * t3 - col(kD4) * t4;
                tempe = fma(col(kBc5), fma(sm, cd, cm * sd) - col(kSinmao), tempe);
                templ = templ + col(kT3cof) * t3 + t4 * fma(t, col(kT5cof), col(kT4cof));
            }
            const double am = col(kAbase) * tempa * tempa;
            const double emRaw = col(kEcco) - tempe;
            const double em = floor_at(emRaw, kHiEmFloor, AZK(emFloor));
            mm = fma(col(kNo), templ, mm);
            // kepler_posvel's prologue and the general loop's first step
            const double ya = rsqrt_nr1(am), temp = ya * ya * rcp_fast(fma(-em, em, 1.0));
            double sw, cw, su, cu;
            sincos_full(argpm, sw, cw);
            const double axnl = em * cw, aynl = fma(em, sw, temp * col(kAycof));
            sincos_full(mm + argpm + temp * col(kXlcof) * axnl, su, cu);
            const double esine = fma(axnl, su, -(aynl * cu)), ecose = fma(axnl, cu, aynl * su);
            double *o = out + ((size_t)orig * nt + k) * 4;
            o[0] = tho;
            o[1] = emRaw;
            o[2] = esine * rcp_fast(1.0 - ecose);
            o[3] = -1.0;
        }
    }
    for (uint32_t s = 0; s < cat.nSdp4; ++s) {
        const Sdp4Sat &e = cat.sdp4[s];
        const uint32_t orig = cat.sdp4Orig[s];
        ecco[orig] = e.ecco;
        inclo[orig] = e.inclo;
        for (uint32_t k = 0; k < nt; ++k) {
            double *o = out + ((size_t)orig * nt + k) * 4;
            o[0] = o[1] = o[2] = 0.0;
            o[3] = (double)e.irez;
        }
    }
    return 0;
}

extern "C" void emul_sincos(const double *x, int n, double *s, double *c) {
    for (int i = 0; i < n; ++i) sincos_full(x[i], s[i], c[i]);
}

extern "C" void emul_ecef_to_geodetic(const double *ecef, int n, double *lla) {
    for (int i = 0; i < n; ++i) {
        double x = ecef[3 * i], y = ecef[3 * i + 1], z = ecef[3 * i + 2];
        ecef_to_geodetic(x, y, z);
        lla[3 * i] = x; lla[3 * i + 1] = y; lla[3 * i + 2] = z;
    }
}
