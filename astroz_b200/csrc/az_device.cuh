// az_device.cuh -- device-side data layout and the per-cell propagation cores (sm_90a, fp64).
//
// Replaces src/Sgp4Batch.zig (BatchElements :15-75, propagateBatchDirect :113-157) and the shared
// src/Sgp4.zig keplerAndPosVel (:646-750) of the reference.  One *cell* = one (satellite, epoch) pair.
#pragma once

#include "az_math.cuh"

namespace az {

// ---- HBM layout of the near-earth element table ----------------------------------------------------
// Satellite-major tiles: tile k holds satellites [8k, 8k+8) as a [kSgp4Cols][8] block of doubles
// (2,496 contiguous bytes): SoA inside the tile, so one cp.async.bulk (TMA) lands the whole tile in
// shared memory and every column chunk is a 64-byte, 128-bit-aligned run.  Only values the kernel
// reads are stored (the reference's 40-column BatchElements(8) carries 4 splatted constants and a
// host-only epoch column, src/Sgp4Batch.zig:21-24,71-73); bstar is folded into cc4/cc5 on the host.
constexpr int kTileSats = 8;
enum Sgp4Col : int {
    kMo, kMdot, kArgpo, kArgpdot, kNodeo, kNodedot, kXnodcf, kCc1, kBc4, kT2cof,
    kOmgcof, kEta, kXmcof, kDelmo, kD2, kD3, kD4, kBc5, kSinmao, kT3cof, kT4cof, kT5cof,
    kAbase, kEcco, kNo, kAycof, kXlcof, kCon41, kX1mth2, kX7thm1, kSinio, kCosio, kIsimp,
    // products of the inclination terms with the literal factors of the short-period block (src/Sgp4.zig:722-740),
    // folded once per satellite instead of once per cell
    kMrtA, kMrtB, kDsuK, kNodeK, kDincK, kRvK,
    kSgp4Cols
};
constexpr int kSgp4TileDoubles = kSgp4Cols * kTileSats;
constexpr int kSgp4TileBytes = kSgp4TileDoubles * 8;
static_assert(kSgp4TileBytes % 16 == 0, "TMA bulk copies move multiples of 16 bytes");

struct GravConsts {  // per-model scalars (kernel parameter -> constant bank)
    double j2, radiusEarthKm, vkmpersec, j3oj2, xke, halfJ2;
};

struct CellOut {
    double rx, ry, rz, vx, vy, vz;
    double mrt;  // radius in earth radii after short-period terms (decay diagnostic)
};

// ---- Kepler solve + short-period terms + orientation -> r, v  (src/Sgp4.zig:646-750) ---------------
// Written over kN independent cells of ONE satellite (kN epochs per thread): every statement is a
// fully unrolled lane loop, so the per-satellite operands are fetched once for kN cells and the
// scheduler interleaves kN dependency chains (ILP) on the half-rate fp64 pipe.
// Differences from the reference's SIMD formulation, none of which changes the value beyond rounding:
//   * no mod-2pi anywhere: every angle goes straight into a range-reducing sincos;
//   * ONE full sincos for the whole Kepler solve: each Newton step is applied to (sin E, cos E) as a
//     rotation by the step (9-op series below 0.05 rad); the loop stops when Newton's residual
//     (e/2) delta^2 is below 1e-15 rad (the reference stops at |delta| < 1e-12);
//   * no atan2: (sinu, cosu) is already a unit vector, the J2 short-period angle is applied as a
//     rotation, and so is the inclination correction (sinio/cosio are per-satellite constants);
//   * sqrt(pl) = sqrt(am)*betal, 1/pl and am^-1.5 come from the two rsqrt seeds already needed.
#define AZ_LANES _Pragma("unroll") for (int k = 0; k < kN; ++k)

struct SatAngles {  // inclination-dependent per-satellite (SGP4) or per-cell (SDP4) terms
    double sinio, cosio, aycof, xlcof, x1mth2;
    double mrtA, mrtB, dsuK, nodeK, dincK, rvK;  // -1.5 con41, 0.5 x1mth2, -0.25 x7thm1, 1.5 cosio, 1.5 cosio sinio, 1.5 con41
    AZ_HD void fold(double con41, double x7thm1) {
        mrtA = -1.5 * con41;
        mrtB = 0.5 * x1mth2;
        dsuK = -0.25 * x7thm1;
        nodeK = 1.5 * cosio;
        dincK = nodeK * sinio;
        rvK = 1.5 * con41;
    }
};

template <int kN>
AZ_HD void rotate_small_n(const double (&s0)[kN], const double (&c0)[kN], const double (&d)[kN], double (&s)[kN],
                          double (&c)[kN]) {
    // The micro series is evaluated unconditionally, as straight-line code the scheduler can interleave with its
    // surroundings; the general evaluation overwrites it in a cold branch (never taken for physical orbits) that keeps
    // the identity exact.
    bool big = false;
    AZ_LANES {
        double sd, cd;
        sincos_micro(d[k], sd, cd);
        rotate(s0[k], c0[k], sd, cd, s[k], c[k]);
        big |= abs_gt(d[k], kHiMicro);
    }
    if (big) {
        AZ_LANES {
            double sd, cd;
            sincos_full(d[k], sd, cd);
            rotate(s0[k], c0[k], sd, cd, s[k], c[k]);
        }
    }
}

#ifndef AZ_KEP_SERIES
#define AZ_KEP_SERIES 1
#endif
template <int kN>
AZ_HD void kepler_posvel(const double (&am)[kN], const double (&em)[kN], const double (&mm)[kN],
                         const double (&argpm)[kN], const double (&nodem)[kN], const SatAngles (&sa)[kN],
                         const GravConsts &g, CellOut (&o)[kN]) {
    double ya[kN], inv_am[kN], axnl[kN], aynl[kN], s[kN], c[kN], eps[kN];
    AZ_LANES {
        // am^-1/2 to 1.5e-12 (one Newton step on the device seed): it scales only J2/J3-sized terms (1/am, am^-3/2, 1/pl), and sqrt(am) below comes out of a
        // Heron correction that squares the error
        ya[k] = rsqrt_nr1(am[k]);
        inv_am[k] = ya[k] * ya[k];
        // 1 / (am (1 - em^2)); only scales the 1e-3-sized J3 terms, so the 1e-12 reciprocal is ample
        const double temp = inv_am[k] * rcp_fast(fma(-em[k], em[k], 1.0));
        double sw, cw;
        sincos_full(argpm[k], sw, cw);
        axnl[k] = em[k] * cw;
        aynl[k] = fma(em[k], sw, temp * sa[k].aycof);
        const double u = mm[k] + argpm[k] + temp * sa[k].xlcof * axnl[k];  // xl - nodem, src/Sgp4.zig:680-682
        sincos_full(u, s[k], c[k]);
        eps[k] = 0.0;
    }
    // Hot path, straight-line: for an orbit with e below ~2e-3 (most of any catalog) Newton's first step is a "micro"
    // rotation (|delta| <= 2e-3) and the second is below 1e-8 rad, where the first-order update is exact to 5e-17 and
    // the solve is finished.  Both steps are evaluated speculatively, without the loop's control flow, so the scheduler
    // interleaves them with the prologue and the short-period block; the flags are checked once, and any other orbit
    // (or a lane that needs the +-0.95 clamp) runs the general loop below from the same starting point instead.
    bool spec = true;
    double s2[kN], c2[kN];
    // e sin E and e cos E at the solution, handed to the short-period block below
    double esineF[kN], ecoseF[kN];
    {
        double d1[kN], s1[kN], c1[kN];
        AZ_LANES {
            const double esine = fma(axnl[k], s[k], -(aynl[k] * c[k]));
            const double ecose = fma(axnl[k], c[k], aynl[k] * s[k]);
#if AZ_KEP_SERIES
            // 1 / (1 - x) = 1 + x + x^2 to x^3 <= 8e-9 for |x| = |e cos E| <= 2e-3 (checked): d1 is off by 1.6e-11 rad at
            // most, which the second step -- an exact Newton step from wherever the first one landed -- takes out
            d1[k] = esine * fma(ecose, ecose + 1.0, 1.0);
            spec &= !abs_gt(ecose, kHiMicro);
#else
            d1[k] = esine * rcp_fast(1.0 - ecose);
#endif
            spec &= !abs_gt(d1[k], kHiMicro);
            double sd, cd;
            sincos_micro(d1[k], sd, cd);
            rotate(s[k], c[k], sd, cd, s1[k], c1[k]);
        }
        AZ_LANES {
            // (reusing the first step's 1 / (1 - e cos E) here would save five instructions, but it moves the result by
            // e * d1 * d2 ~ 1e-14 rad = 6e-10 km at geostationary radius, outside the reference's own 1e-10 km
            // layout-equivalence bound, src/Constellation.zig:869, once two launch shapes solve the same cell differently)
            const double esine = fma(axnl[k], s1[k], -(aynl[k] * c1[k]));
            const double ecose = fma(axnl[k], c1[k], aynl[k] * s1[k]);
#if AZ_KEP_SERIES
            const double d = (esine - d1[k]) * fma(ecose, ecose + 1.0, 1.0);  // |d| < 1e-8: the 8e-9 of the series is 8e-17 rad
#else
            const double d = (esine - d1[k]) * rcp_fast(1.0 - ecose);
#endif
            spec &= abs_lt(d, kHiLinear);
            s2[k] = fma(c1[k], d, s1[k]);
            c2[k] = fma(-s1[k], d, c1[k]);
            // the same first-order step carries (e sin E, e cos E) along: exact to e d^2 / 2 < 1e-19
            esineF[k] = fma(ecose, d, esine);
            ecoseF[k] = fma(-esine, d, ecose);
        }
    }
    if (spec) {
        AZ_LANES {
            s[k] = s2[k];
            c[k] = c2[k];
        }
    } else
#pragma unroll 1
    for (int it = 0; it < 10; ++it) {  // src/Sgp4.zig:687-694
        double delta[kN];
        bool big = false, done = true, linear = true, micro = true;
        AZ_LANES {
            const double esine = fma(axnl[k], s[k], -(aynl[k] * c[k]));
            const double ecose = fma(axnl[k], c[k], aynl[k] * s[k]);
            double d = (esine - eps[k]) * rcp_fast(1.0 - ecose);
            d = clamp_abs(d, kHiClamp, AZK(clamp));
            eps[k] += d;
            delta[k] = d;
            big |= abs_gt(d, kHiTiny);
            micro &= !abs_gt(d, kHiMicro);
            linear &= abs_lt(d, kHiLinear);
            // Newton's residual after this step is ~ (e/2) delta^2 (f'' = e sin E); it is bounded through the exponent
            // fields, |d| < 2^(xd-1022) and em < 2^(xe-1022): em d^2 < 2^-49 (1.8e-15 rad) whenever 2 xd + xe <= 3017
            done &= 2 * expo(d) + expo(em[k]) <= 3017;
        }
        if (linear) {  // |delta| < 1e-8: first-order update is exact to 5e-17 and the solve is finished
            AZ_LANES {
                const double sn = fma(c[k], delta[k], s[k]);
                c[k] = fma(-s[k], delta[k], c[k]);
                s[k] = sn;
            }
            break;
        }
        if (micro) {  // |delta| < 2e-3: the usual first step of a near-circular orbit (delta ~ e)
            AZ_LANES {
                double sd, cd;
                sincos_micro(delta[k], sd, cd);
                const double sn = fma(s[k], cd, c[k] * sd);
                c[k] = fma(c[k], cd, -(s[k] * sd));
                s[k] = sn;
            }
        } else if (!big) {
            AZ_LANES {
                double sd, cd;
                sincos_tiny(delta[k], sd, cd);
                const double sn = fma(s[k], cd, c[k] * sd);
                c[k] = fma(c[k], cd, -(s[k] * sd));
                s[k] = sn;
            }
        } else {
            AZ_LANES {
                double sd, cd;
                sincos_full(delta[k], sd, cd);
                const double sn = fma(s[k], cd, c[k] * sd);
                c[k] = fma(c[k], cd, -(s[k] * sd));
                s[k] = sn;
            }
        }
        if (done) break;
    }
    if (!spec) {
        AZ_LANES {
            ecoseF[k] = fma(axnl[k], c[k], aynl[k] * s[k]);
            esineF[k] = fma(axnl[k], s[k], -(aynl[k] * c[k]));
        }
    }

    double sinu[kN], cosu[kN], dsu[kN], dinc[kN], xnode[kN], mrt[kN], mvt[kN], rvdot[kN];
    AZ_LANES {
        const double ecose = ecoseF[k], esine = esineF[k];
        const double omel2 = 1.0 - fma(axnl[k], axnl[k], aynl[k] * aynl[k]);
        const double yb = rsqrt_nr1(omel2);  // 1.5e-12: betal is Heron-corrected, 1/pl scales J2-sized terms only
        const double betal = sqrt_from_rsqrt(omel2, yb);
        // a / r = 1 / (1 - e cos E).  (Starting this reciprocal from the solver's last 1 / (1 - e cos E), one Newton step
        // instead of four FMAs, gained nothing on its own and lost time together with the carried e sin E / e cos E above.)
        const double omec = 1.0 - ecose;
        const double rl = am[k] * omec;
        const double aor = rcp(omec);
        // sqrt(am) / rl = (a / r) am^-1/2; the 1.5e-12 of ya is 1e-11 km/s on the velocity
        const double q = aor * ya[k];
        const double rdotl = esine * q;
        const double rvdotl = betal * q;  // sqrt(pl) / rl
        const double est = esine * rcp_fast(1.0 + betal);  // multiplies e-sized terms only
        sinu[k] = aor * (s[k] - aynl[k] - axnl[k] * est);
        cosu[k] = aor * (c[k] - axnl[k] + aynl[k] * est);
        const double sin2u = 2.0 * sinu[k] * cosu[k];
        const double cos2u = fma(-2.0 * sinu[k], sinu[k], 1.0);

        const double ipl = inv_am[k] * (yb * yb);  // 1 / pl
        const double temp1 = g.halfJ2 * ipl;
        const double temp2 = temp1 * ipl;
        const double w = inv_am[k] * ya[k];  // nm / xke = am^-3/2
        mrt[k] = fma(rl, fma(temp2 * betal, sa[k].mrtA, 1.0), temp1 * sa[k].mrtB * cos2u);
        dsu[k] = temp2 * sa[k].dsuK * sin2u;
        xnode[k] = fma(temp2 * sa[k].nodeK, sin2u, nodem[k]);
        dinc[k] = temp2 * sa[k].dincK * cos2u;
        const double wt1 = w * temp1;
        mvt[k] = fma(-wt1 * sa[k].x1mth2, sin2u, rdotl);
        rvdot[k] = fma(wt1, fma(sa[k].x1mth2, cos2u, sa[k].rvK), rvdotl);
    }

    double sinsu[kN], cossu[kN], sini[kN], cosi[kN], si0[kN], ci0[kN];
    AZ_LANES {
        si0[k] = sa[k].sinio;
        ci0[k] = sa[k].cosio;
    }
    rotate_small_n<kN>(sinu, cosu, dsu, sinsu, cossu);
    rotate_small_n<kN>(si0, ci0, dinc, sini, cosi);
    AZ_LANES {
        double snod, cnod;
        sincos_full(xnode[k], snod, cnod);
        const double xmx = -snod * cosi[k];
        const double xmy = cnod * cosi[k];
        const double ux = fma(xmx, sinsu[k], cnod * cossu[k]);
        const double uy = fma(xmy, sinsu[k], snod * cossu[k]);
        const double uz = sini[k] * sinsu[k];
        const double vx = fma(xmx, cossu[k], -(cnod * sinsu[k]));
        const double vy = fma(xmy, cossu[k], -(snod * sinsu[k]));
        const double vz = sini[k] * cossu[k];
        const double rs = mrt[k] * g.radiusEarthKm;
        o[k].rx = rs * ux;
        o[k].ry = rs * uy;
        o[k].rz = rs * uz;
        o[k].vx = fma(mvt[k], ux, rvdot[k] * vx) * g.vkmpersec;
        o[k].vy = fma(mvt[k], uy, rvdot[k] * vy) * g.vkmpersec;
        o[k].vz = fma(mvt[k], uz, rvdot[k] * vz) * g.vkmpersec;
        o[k].mrt = mrt[k];
    }
}

// ---- near-earth secular + drag update, then the shared core (src/Sgp4Batch.zig:113-157) -----------
// `col(i)` returns column i of the satellite handled by this warp (shared-memory broadcast read);
// t[] are kN epochs (minutes since the element epoch) of that one satellite.
template <int kN, typename ColFn>
AZ_HD void sgp4_cell(ColFn col, const double (&t)[kN], const GravConsts &g, CellOut (&o)[kN]) {
    double t2[kN], xmdf[kN], argpm[kN], nodem[kN], tempa[kN], tempe[kN], templ[kN], mm[kN];
    {
        const double mdot = col(kMdot), mo = col(kMo), argpdot = col(kArgpdot), argpo = col(kArgpo);
        const double xnodcf = col(kXnodcf), nodedot = col(kNodedot), nodeo = col(kNodeo);
        const double cc1 = col(kCc1), bc4 = col(kBc4), t2cof = col(kT2cof);
        AZ_LANES {
            t2[k] = t[k] * t[k];
            xmdf[k] = fma(mdot, t[k], mo);
            argpm[k] = fma(argpdot, t[k], argpo);
            nodem[k] = fma(xnodcf, t2[k], fma(nodedot, t[k], nodeo));
            tempa[k] = fma(-cc1, t[k], 1.0);
            tempe[k] = bc4 * t[k];
            templ[k] = t2cof * t2[k];
            mm[k] = xmdf[k];
        }
    }
    if (col(kIsimp) == 0.0) {  // warp-uniform: a warp works on one satellite (src/Sgp4Batch.zig:133-145)
        const double eta = col(kEta), xmcof = col(kXmcof), delmo = col(kDelmo), omgcof = col(kOmgcof);
        const double d2 = col(kD2), d3 = col(kD3), d4 = col(kD4), bc5 = col(kBc5), sinmao = col(kSinmao);
        const double t3cof = col(kT3cof), t4cof = col(kT4cof), t5cof = col(kT5cof);
        double sm[kN], cm[kN], tho[kN];
        bool big = false, small = true, micro = true;
        AZ_LANES {
            sincos_full(xmdf[k], sm[k], cm[k]);
            const double dm = fma(eta, cm[k], 1.0);
            const double delm = xmcof * (dm * dm * dm - delmo);
            tho[k] = fma(omgcof, t[k], delm);
            mm[k] = xmdf[k] + tho[k];
            argpm[k] -= tho[k];
            big |= abs_gt(tho[k], kHiQuarter);
            small &= !abs_gt(tho[k], kHiTiny);
            micro &= !abs_gt(tho[k], kHiMicro);
        }
        // sin(mm) = sin(xmdf + tho): tho is a drag-sized angle (1e-6 .. 1e-3 rad over days for catalogued objects),
        // rotate instead of a second reduction, with the shortest series that covers it.  The choice is made once for
        // the thread's lanes, outside the lane loops.
        double sd[kN], cd[kN];
        AZ_LANES sincos_micro(tho[k], sd[k], cd[k]);  // the usual case, straight-line; larger angles redo it below
        if (!micro) {
            if (small) {
                AZ_LANES sincos_tiny(tho[k], sd[k], cd[k]);
            } else if (!big) {
                AZ_LANES sincos_quarter(tho[k], sd[k], cd[k]);
            } else {
                AZ_LANES sincos_full(tho[k], sd[k], cd[k]);
            }
        }
        AZ_LANES {
            const double sinmm = fma(sm[k], cd[k], cm[k] * sd[k]);
            const double t3 = t2[k] * t[k];
            const double t4 = t3 * t[k];
            tempa[k] = tempa[k] - d2 * t2[k] - d3 * t3 - d4 * t4;
            tempe[k] = fma(bc5, sinmm - sinmao, tempe[k]);
            templ[k] = templ[k] + t3cof * t3 + t4 * fma(t[k], t5cof, t4cof);
        }
    }
    double am[kN], em[kN];
    SatAngles sa[kN];
    {
        const double abase = col(kAbase), ecco = col(kEcco), no = col(kNo);
        SatAngles a0;
        a0.sinio = col(kSinio); a0.cosio = col(kCosio); a0.aycof = col(kAycof); a0.xlcof = col(kXlcof);
        a0.x1mth2 = col(kX1mth2);
        a0.mrtA = col(kMrtA); a0.mrtB = col(kMrtB); a0.dsuK = col(kDsuK); a0.nodeK = col(kNodeK);
        a0.dincK = col(kDincK); a0.rvK = col(kRvK);
        AZ_LANES {
            am[k] = abase * tempa[k] * tempa[k];
            em[k] = floor_at(ecco - tempe[k], kHiEmFloor, AZK(emFloor));
            mm[k] = fma(no, templ[k], mm[k]);
            sa[k] = a0;
        }
    }
    kepler_posvel<kN>(am, em, mm, argpm, nodem, sa, g, o);
}

// Angle of the unit vector (s, c) = (sin a, cos a), a in (-pi, pi].  An fp32 arctangent (idle FMA/XU pipes) is snapped
// to the lattice a0 = k / 128 rad, whose sines and cosines sit in a 13 KB table (L1-resident; az_angle_table.inc,
// tools/gen_angle_table.py); d = sin(a - a0) = s cos a0 - c sin a0 with |d| <= 2^-8 + 2e-5, and the three-term arcsine
// finishes it: the x^7 term is below 7e-19.  8 fp64 instructions, where libdevice's atan2 takes several times as many.
// A common scale error eps of (s, c) moves the result by eps d <
// 4e-3 eps.  The sign of a zero s survives the conversion, so the branch cut at +-pi falls where atan2 puts it.
struct AnglePair { double s, c; };
static __device__ const AnglePair __align__(16) kAngleTabDev[807] = {
#include "az_angle_table.inc"
};
static const AnglePair kAngleTabHost[807] = {  // the same entries for tests/host_emul
#include "az_angle_table.inc"
};
// fp32 arctangent of (s, c) within 2e-5 rad, branch-free: octant reduction by min / max, a five-term odd polynomial
// (1.2e-5 on [0, 1]), the octant undone with selects.  libdevice's atan2f is accurate to 2 ulp, which the lattice snap
// below throws away, and brings 6 branches and a division subroutine per call into an otherwise straight-line epilogue.
AZ_HD float atan2_seed(float s, float c) {
    const float ay = fabsf(s), ax = fabsf(c);
    const float mx = fmaxf(ax, ay), mn = fminf(ax, ay);
#ifdef __CUDA_ARCH__
    const float t = __fdividef(mn, mx);
#else
    const float t = mn / mx;
#endif
    const float t2 = t * t;
    float p = fmaf(t2, 0.020812865f, -0.085092984f);
    p = fmaf(p, t2, 0.18011868f);
    p = fmaf(p, t2, -0.33029541f);
    p = fmaf(p, t2, 0.99986577f);
    float r = p * t;
    r = (ay > ax) ? 1.57079637f - r : r;
    r = (c < 0.0f) ? 3.14159274f - r : r;
    return copysignf(r, s);
}

AZ_HD double angle_of_unit(double s, double c) {
    const float kf = rintf(atan2_seed((float)s, (float)c) * 128.0f);  // |k| <= 402
    const double a0 = (double)(kf * 0.0078125f);                      // exact
#ifdef __CUDA_ARCH__
    const AnglePair t = kAngleTabDev[(int)kf + 403];
#else
    const AnglePair t = kAngleTabHost[(int)kf + 403];
#endif
    const double d = fma(s, t.c, -(c * t.s));  // |d| <= 2^-8 + 2e-5
    const double x2 = d * d;
    const double u = x2 * fma(x2, 0.075, 1.0 / 6.0);  // asin(d) = d (1 + x2 (1/6 + 3/40 x2))
    return a0 + fma(d, u, d);
}

// ---- deep space (src/Sdp4Batch.zig:16-125,199-526; src/Sdp4.zig:681-866) --------------------------------
// One record per deep-space satellite, read with warp-uniform loads (a warp works on one satellite).
struct Sdp4Sat {
    double mo, mdot, argpo, argpdot, nodeo, nodedot, xnodcf, cc1, bc4, t2cof, ecco, no, inclo;
    double se2, se3, si2, si3, sl2, sl3, sl4, sgh2, sgh3, sgh4, sh2, sh3;  // solar periodics
    double ee2, e3, xi2, xi3, xl2, xl3, xl4, xgh2, xgh3, xgh4, xh2, xh3;  // lunar periodics
    double zmol, zmos, dedt, didt, dmdt, domdt, dnodt;
    // Resonance terms d_i sin(phi_b - g_i) folded on the basis angles phi_b (see resonance_accel): the acceleration is
    // sum_b rp[b] sin(phi_b) + rq[b] cos(phi_b).  Half-day (irez 2) basis: 2w+l, l, w+l, l-w, 2w+2l, 2l, w+2l, 2l-w;
    // synchronous (irez 1): l, 2l, 3l in the first three slots.
    double rp[8], rq[8];
    double xlamo, xfact, gsto;
    double abase, invNo;       // (xke / no)^(2/3) and 1 / no: the semi-major axis follows no by a short series
    double sinio, cosio;       // of inclo: the perturbed inclination is a small rotation away
    double epochJd;
    int irez, pad_;
};

constexpr double kStepp = 720.0;      // src/Sdp4.zig:51-52
constexpr double kStep2 = 259200.0;
constexpr double kRptim = 4.37526908801129966e-3;

// resonance accelerations at (xli, xni, atime)  (src/Sdp4.zig:824-866).
// The reference evaluates ten (half-day) or three (synchronous) sines and cosines of phase-shifted combinations of
// two angles, w = argpo + argpdot atime and l = xli.  Here sin/cos(w) and sin/cos(l) are the only range-reducing
// evaluations; the combinations come from angle addition and the constant phases g_i are folded into per-satellite
// coefficient pairs on the host (sdp4_record): d sin(phi - g) = (d cos g) sin(phi) - (d sin g) cos(phi).
AZ_HD void resonance_accel(const Sdp4Sat &e, double xli, double xni, double atime, double &xndt, double &xnddt,
                           double &xldot) {
    xldot = xni + e.xfact;
    double sl, cl;
    sincos_full(xli, sl, cl);
    const double s2l = 2.0 * sl * cl, c2l = fma(-2.0 * sl, sl, 1.0);
    if (e.irez == 2) {
        double so, co;
        sincos_full(fma(e.argpdot, atime, e.argpo), so, co);
        const double s2o = 2.0 * so * co, c2o = fma(-2.0 * so, so, 1.0);
        double sb[8], cb[8];
        rotate(s2o, c2o, sl, cl, sb[0], cb[0]);    // 2w + l
        sb[1] = sl; cb[1] = cl;                    // l
        rotate(so, co, sl, cl, sb[2], cb[2]);      // w + l
        rotate(sl, cl, -so, co, sb[3], cb[3]);     // l - w
        sb[4] = 2.0 * sb[2] * cb[2]; cb[4] = fma(-2.0 * sb[2], sb[2], 1.0);  // 2w + 2l
        sb[5] = s2l; cb[5] = c2l;                  // 2l
        rotate(so, co, s2l, c2l, sb[6], cb[6]);    // w + 2l
        rotate(s2l, c2l, -so, co, sb[7], cb[7]);   // 2l - w
        double acc = 0.0, d1 = 0.0, d2 = 0.0;
#pragma unroll
        for (int b = 0; b < 8; ++b) {
            acc = fma(e.rp[b], sb[b], fma(e.rq[b], cb[b], acc));
            const double dc = fma(e.rp[b], cb[b], -(e.rq[b] * sb[b]));  // d/dphi of the term
            if (b < 4) d1 += dc;
            else d2 += dc;
        }
        xndt = acc;
        xnddt = fma(2.0, d2, d1) * xldot;
    } else {
        const double s3l = fma(sl, c2l, cl * s2l), c3l = fma(cl, c2l, -(sl * s2l));
        xndt = fma(e.rp[0], sl, fma(e.rq[0], cl, fma(e.rp[1], s2l, fma(e.rq[1], c2l, fma(e.rp[2], s3l, e.rq[2] * c3l)))));
        const double dc1 = fma(e.rp[0], cl, -(e.rq[0] * sl));
        const double dc2 = fma(e.rp[1], c2l, -(e.rq[1] * s2l));
        const double dc3 = fma(e.rp[2], c3l, -(e.rq[2] * s3l));
        xnddt = fma(3.0, dc3, fma(2.0, dc2, dc1)) * xldot;
    }
}

// one 720-minute Euler-Maclaurin step of the resonance integrator (src/Sdp4.zig:796-801)
AZ_HD void resonance_step(const Sdp4Sat &e, double &xli, double &xni, double &atime, double delt) {
    double xndt, xnddt, xldot;
    resonance_accel(e, xli, xni, atime, xndt, xnddt, xldot);
    xli += xldot * delt + xndt * kStep2;
    xni += xndt * delt + xnddt * kStep2;
    atime += delt;
}

// number of whole 720-minute steps the reference's loop `while |t - atime| >= 720` takes from atime = 0
AZ_HD int resonance_node(double t) {
    const double a = fabs(t);
    int n = (int)(a * (1.0 / kStepp));  // a first guess (a division costs ~20 instructions); the two lines below settle it
    if ((double)n * kStepp > a) --n;
    if (a - (double)n * kStepp >= kStepp) ++n;  // a guard: 1.0 / kStepp rounds up, so the guess is never one short
    return n;
}

// kN deep-space cells of ONE satellite (kN epochs per thread, like sgp4_cell).  (xli, xni)[k] is the integrator state
// at the lattice node atime[k] = +-720*n nearest below |t[k]| (unused when irez == 0).  st[k] receives a kernel-level
// status (0 ok, 1 decayed, 2 invalid ecc) with the scalar path's checks (src/Sdp4.zig:913-967); a failing lane is
// carried through with harmless operands so the other lanes are unaffected.
// Every statement is a lane loop, so the two or three independent cells interleave on the fp64 pipe; the rare
// alternatives (Lyddane low-inclination form, a large inclination excursion, a large resonance libration) are chosen by
// flags folded over the lanes and fall back to per-lane code only when the lanes disagree.
template <int kN>
AZ_HD void sdp4_cell_n(const Sdp4Sat &e, const double (&t)[kN], const double (&xli)[kN], const double (&xni)[kN],
                       const double (&atime)[kN], const GravConsts &g, CellOut (&o)[kN], int (&st)[kN]) {
    double tempa[kN], tempe[kN], templ[kN], mm[kN], argpm[kN], nodem[kN], em[kN], inclm[kN], am[kN];
    AZ_LANES {
        st[k] = 0;
        const double t2 = t[k] * t[k];
        tempa[k] = fma(-e.cc1, t[k], 1.0);
        tempe[k] = e.bc4 * t[k];
        templ[k] = e.t2cof * t2;
        // secular gravity + drag, then luni-solar secular rates (src/Sdp4Batch.zig:212-236)
        mm[k] = fma(e.dmdt, t[k], fma(e.mdot, t[k], e.mo));
        argpm[k] = fma(e.domdt, t[k], fma(e.argpdot, t[k], e.argpo));
        nodem[k] = fma(e.dnodt, t[k], fma(e.xnodcf, t2, fma(e.nodedot, t[k], e.nodeo)));
        em[k] = fma(e.dedt, t[k], e.ecco);
        inclm[k] = fma(e.didt, t[k], e.inclo);
        am[k] = e.abase * tempa[k] * tempa[k];  // (xke / no)^(2/3) tempa^2 (src/Sdp4.zig:913-916 with nm = no)
    }

    if (e.irez != 0) {  // final partial step from the lattice node (src/Sdp4.zig:803-819); uniform: one satellite
        double xndt[kN], xnddt[kN], xldot[kN];
        AZ_LANES resonance_accel(e, xli[k], xni[k], atime[k], xndt[k], xnddt[k], xldot[k]);
        AZ_LANES {
            const double ft = t[k] - atime[k];
            const double hft2 = 0.5 * ft * ft;
            const double nmr = fma(xnddt[k], hft2, fma(xndt[k], ft, xni[k]));
            const double xl = fma(xndt[k], hft2, fma(xldot[k], ft, xli[k]));
            // theta = (gsto + t rptim) mod 2pi in the reference; the mean anomaly only ever enters a sine/cosine, whose
            // range reduction absorbs the multiple of 2pi
            const double theta = fma(t[k], AZK(rptim), e.gsto);
            mm[k] = (e.irez == 2) ? xl - 2.0 * nodem[k] + 2.0 * theta : xl - nodem[k] - argpm[k] + theta;
            const double nm = e.no + (nmr - e.no);
            if (nm <= 0.0) st[k] = 1;
            // (xke / nm)^(2/3) = abase (1 + x)^(-2/3), x = (nm - no) / no: the resonance libration of the mean motion is
            // a few 1e-4 of no, so a degree-6 binomial series replaces the reference's division + cube root
            const double x = (nmr - e.no) * e.invNo;
            if (abs_gt(x, 0x3f689374u)) {  // |x| > 3e-3 (never seen for catalogued objects): the general evaluation
                const double cr = cbrt(g.xke / (nm > 0.0 ? nm : e.no));
                am[k] = cr * cr * tempa[k] * tempa[k];
            } else {
                // binomial coefficients of (1 + x)^(-2/3); those of x^3 .. x^6 rounded to 21 significant bits (immediate
                // operands): on |x| <= 3e-3 that moves the factor by < 7e-15
                double p = fma(x, 0x1.9899ep-2 /* 2618/6561 */, -0x1.b0a2fp-2 /* -308/729 */);
                p = fma(p, x, 0x1.cf8ap-2 /* 110/243 */);
                p = fma(p, x, -0x1.f9addp-2 /* -40/81 */);
                p = fma(p, x, AZK(bin2));
                p = fma(p, x, AZK(bin1));
                am[k] *= fma(p, x, 1.0);
            }
        }
    }

    AZ_LANES {
        em[k] -= tempe[k];
        if (st[k] == 0 && (ge_one(em[k]) || em[k] < -0.001)) st[k] = 2;
        em[k] = floor_at(em[k], kHiEmFloor, AZK(emFloor));
        if (st[k] == 0 && am[k] < 0.95) st[k] = 1;
        mm[k] = fma(e.no, templ[k], mm[k]);
    }

    // luni-solar periodics, dpper (src/Sdp4.zig:681-759)
    double pe[kN], pinc[kN], pl[kN], pgh[kN], ph[kN];
    {
        double sz[kN], cz[kN];
        AZ_LANES sincos_full(fma(AZK(zns), t[k], e.zmos), sz[k], cz[k]);
        AZ_LANES {
            // zf = zm + 2 ze sin(zm): the second sine/cosine is a rotation of the first by an angle below 2 ze
            double sd, cd, sinzf, coszf;
            sincos_tiny(AZK(zes2) * sz[k], sd, cd);  // |.| <= 0.0335
            rotate(sz[k], cz[k], sd, cd, sinzf, coszf);
            const double f2 = fma(0.5 * sinzf, sinzf, -0.25);
            const double f3 = -0.5 * sinzf * coszf;
            pe[k] = fma(e.se2, f2, e.se3 * f3);
            pinc[k] = fma(e.si2, f2, e.si3 * f3);
            pl[k] = fma(e.sl2, f2, fma(e.sl3, f3, e.sl4 * sinzf));
            pgh[k] = fma(e.sgh2, f2, fma(e.sgh3, f3, e.sgh4 * sinzf));
            ph[k] = fma(e.sh2, f2, e.sh3 * f3);
        }
        AZ_LANES sincos_full(fma(AZK(znl), t[k], e.zmol), sz[k], cz[k]);
        AZ_LANES {
            double sd, cd, sinzf, coszf;
            sincos_quarter(AZK(zel2) * sz[k], sd, cd);  // |.| <= 0.1098
            rotate(sz[k], cz[k], sd, cd, sinzf, coszf);
            const double f2 = fma(0.5 * sinzf, sinzf, -0.25);
            const double f3 = -0.5 * sinzf * coszf;
            pe[k] += fma(e.ee2, f2, e.e3 * f3);
            pinc[k] += fma(e.xi2, f2, e.xi3 * f3);
            pl[k] += fma(e.xl2, f2, fma(e.xl3, f3, e.xl4 * sinzf));
            pgh[k] += fma(e.xgh2, f2, fma(e.xgh3, f3, e.xgh4 * sinzf));
            ph[k] += fma(e.xh2, f2, e.xh3 * f3);
        }
    }

    double sinip[kN], cosip[kN];
    bool smallInc = true, allNormal = true, allLyddane = true;
    AZ_LANES {
        const double dincl = fma(e.didt, t[k], pinc[k]);  // inclm - inclo: luni-solar secular + periodic, ~1e-3 rad over years
        inclm[k] += pinc[k];
        em[k] += pe[k];
        smallInc &= !abs_gt(dincl, kHiTiny);
        allNormal &= inclm[k] >= 0.2;
        allLyddane &= !(inclm[k] >= 0.2);
    }
    if (smallInc) {  // the perturbed inclination is a small rotation away from the element set's
        AZ_LANES {
            double sd, cd;
            sincos_tiny(fma(e.didt, t[k], pinc[k]), sd, cd);
            rotate(e.sinio, e.cosio, sd, cd, sinip[k], cosip[k]);
        }
    } else {
        AZ_LANES sincos_full(inclm[k], sinip[k], cosip[k]);
    }
    if (allNormal) {
        AZ_LANES {
            const double phs = ph[k] * rcp(sinip[k]);
            argpm[k] += fma(-cosip[k], phs, pgh[k]);
            nodem[k] += phs;
            mm[k] += pl[k];
        }
    } else {
        // Lyddane modification for near-equatorial orbits (src/Sdp4.zig:735-758): the usual case for a geostationary
        // belt object.  nodem <- atan2(alfdp, betdp): the vector is normalised and its angle taken with the fp32-seeded
        // extraction of the geodetic epilogue instead of libdevice's atan2.
        (void)allLyddane;
        AZ_LANES {
            if (inclm[k] >= 0.2) {
                const double phs = ph[k] * rcp(sinip[k]);
                argpm[k] += fma(-cosip[k], phs, pgh[k]);
                nodem[k] += phs;
                mm[k] += pl[k];
            } else {
                const double nod = mod_twopi(nodem[k]);
                double sinop, cosop;
                sincos_full(nod, sinop, cosop);
                const double alfdp = sinip[k] * sinop + (ph[k] * cosop + pinc[k] * cosip[k] * sinop);
                const double betdp = sinip[k] * cosop + (-ph[k] * sinop + pinc[k] * cosip[k] * cosop);
                const double xls = mm[k] + argpm[k] + cosip[k] * nod;
                const double dls = pl[k] + pgh[k] - pinc[k] * nod * sinip[k];
                const double r2 = fma(alfdp, alfdp, betdp * betdp);
                double nn;
                if (r2 > 1.0e-280) {
                    const double ir = rsqrt_nr(r2);
                    nn = angle_of_unit(alfdp * ir, betdp * ir);
                } else {
                    nn = 0.0;  // atan2(0, 0)
                }
                if (fabs(nod - nn) > kPi) nn += (nn < nod) ? kTwoPi : -kTwoPi;
                nodem[k] = nn;
                mm[k] += pl[k];
                argpm[k] = xls + dls - mm[k] - cosip[k] * nn;
            }
        }
    }
    SatAngles sa[kN];
    AZ_LANES {
        if (inclm[k] < 0.0) {  // src/Sdp4.zig:932-936 (sin flips sign with the inclination, cos does not)
            sinip[k] = -sinip[k];
            nodem[k] += kPi;
            argpm[k] -= kPi;
        }
        em[k] = floor_at(em[k], kHiEmFloor, AZK(emFloor));
        if (ge_one(em[k])) {  // failing lane: flag it, and keep the shared Kepler loop well conditioned
            if (st[k] == 0) st[k] = 2;
            em[k] = 0.5;
        }
        if (!(am[k] >= 0.95)) am[k] = 1.0;
        // inclination-dependent terms re-derived per cell (src/Sdp4Batch.zig:326-339)
        const double cosip2 = cosip[k] * cosip[k];
        // 1 + cos ip.  Near 180 degrees it cancels: cos ip is known to 1e-16 absolute, so 1 + cos ip ~ 1.5e-12 (the guard
        // below) would keep four digits, and xlcof ~ 1/(1 + cos ip) moves the argument of latitude by kilometres.  A
        // retrograde cell takes the identity 1 + cos = sin^2 / (1 - cos) instead, exact to the digits of sin ip (the
        // small rotation of the element set's sin/cos forms it to 1e-20 absolute); other cells keep 1 + cos ip.
        const double den = cosip[k] < 0.0 ? sinip[k] * sinip[k] * rcp(1.0 - cosip[k]) : 1.0 + cosip[k];
        sa[k].sinio = sinip[k];
        sa[k].cosio = cosip[k];
        sa[k].aycof = -0.5 * g.j3oj2 * sinip[k];
        sa[k].xlcof = -0.25 * g.j3oj2 * sinip[k] * fma(5.0, cosip[k], 3.0) * rcp(fabs(den) > 1.5e-12 ? den : 1.5e-12);
        sa[k].x1mth2 = 1.0 - cosip2;
        sa[k].fold(fma(3.0, cosip2, -1.0), fma(7.0, cosip2, -1.0));
    }
    kepler_posvel<kN>(am, em, mm, argpm, nodem, sa, g, o);
    AZ_LANES if (st[k] == 0 && o[k].mrt < 1.0) st[k] = 1;
}

// One deep-space cell (the single-epoch form of the above).
AZ_HD int sdp4_cell(const Sdp4Sat &e, double t, double xli, double xni, double atime, const GravConsts &g,
                    CellOut &o) {
    const double t1[1] = {t}, l1[1] = {xli}, n1[1] = {xni}, a1[1] = {atime};
    CellOut o1[1];
    int st[1];
    sdp4_cell_n<1>(e, t1, l1, n1, a1, g, o1, st);
    o = o1[0];
    return st[0];
}

// ---- output-mode epilogue (src/Constellation.zig:478-509, src/WorldCoordinateSystem.zig:98-121) ----
AZ_HD void eci_to_ecef(double &x, double &y, double sinG, double cosG) {
    const double ex = fma(x, cosG, y * sinG);
    const double ey = fma(y, cosG, -(x * sinG));
    x = ex;
    y = ey;
}

// ECEF -> (geodetic latitude rad, longitude rad, altitude km) on WGS84.  The reference iterates
// lat <- atan2(z + e2 N sin(lat), p) up to 10 times until the step is below 1e-12 rad
// (src/WorldCoordinateSystem.zig:98-121); its fixed point is the exact geodetic latitude.  Here the same latitude comes
// from Bowring's closed form on the parametric latitude u -- tan(lat) = (z + e'^2 b sin^3 u) / (p - e^2 a cos^3 u) --
// started from his height-corrected u (tan u = (b z / a p)(1 + e'^2 b / r)) and evaluated twice: 2e-13 rad after the
// first evaluation, rounding level after the second, for 100 km .. 70,000 km altitude at every latitude.  No
// trigonometry inside: three normalisations (rsqrt) and two angle extractions at the end.  The altitude uses
// p cos(lat) + z sin(lat) - a sqrt(1 - e2 sin^2(lat)), which equals the reference's p / cos(lat) - N without its
// cancellation near the poles.
AZ_HD void ecef_to_geodetic(double &x, double &y, double &z) {
    constexpr double a = 6378.137;
    constexpr double f = 1.0 / 298.257223563;
    constexpr double e2 = 2.0 * f - f * f;
    constexpr double b = a * (1.0 - f);
    constexpr double ep2b = e2 / (1.0 - e2) * b;  // e'^2 b
    constexpr double e2a = e2 * a;
    const double p2 = fma(x, x, y * y);
    if (!(p2 > 1.0e-280)) {  // on the polar axis: atan2(0, 0) = 0 for the longitude, like the reference
        const double az = fabs(z);
        x = (z < 0.0) ? -0.5 * kPi : 0.5 * kPi;
        y = 0.0;
        z = az - b;
        return;
    }
    // Reciprocal square roots carry one Newton step (1.5e-12) where that is provably enough: the Heron correction in
    // sqrt_from_rsqrt squares the error; angle_of_unit sees a common scale error of its arguments 4e-3 times smaller;
    // the height-corrected start needs its 0.7 % term to a few digits.
    const double ip = rsqrt_nr1(p2);
    const double p = sqrt_from_rsqrt(p2, ip);
    const double lon = angle_of_unit(y * ip, x * ip);
    // Bowring's step from the height-corrected parametric latitude, once: within 2.2e-13 rad (1.4 micrometres on the
    // ground) of the converged latitude for every height from 100 km to 50,000 km (a second step reaches 3e-16 for
    // 17 more instructions; the reference's own loop stops when a step moves the latitude by less than 1e-12,
    // src/WorldCoordinateSystem.zig:107-113)
    const double ir = rsqrt_seed(fma(z, z, p2));
    double su = b * z * fma(ep2b, ir, 1.0), cu = a * p;
    const double hq = rsqrt_nr1(fma(su, su, cu * cu));
    su *= hq;
    cu *= hq;
    const double num = fma(ep2b * su * su, su, z);
    const double den = fma(-e2a * cu * cu, cu, p);
    const double h = rsqrt_nr1(fma(num, num, den * den));
    const double sl = num * h, cl = den * h;
    const double w2 = fma(-e2 * sl, sl, 1.0);
    x = angle_of_unit(sl, cl);
    y = lon;
    z = fma(p, cl, z * sl) - a * sqrt_from_rsqrt(w2, rsqrt_nr1(w2));
}

}  // namespace az
