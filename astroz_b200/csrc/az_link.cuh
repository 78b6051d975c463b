// az_link.cuh -- K17: orbits from pairs of uncorrelated tracks.  __host__ __device__, so the kernels (az_link.cu) and
// the host emulation (tests/host_emul/emul_link.cu) run this source.
//
// Inputs: tracks in K12's observation layout (az_correlate.cuh), each in time order, and pairs (a, b) of track indices.
//
// Anchor: a track's middle observation, index floor(c / 2), among its c observations that give a line of sight from a
// known origin with every component of it used (sigma < inf): both angles of an optical observation (origin the
// station, range unknown); range, azimuth and elevation of a radar observation (origin the station, range known); the
// three position components of a TEME or ECEF state (origin the geocentre, range |r| known).  The geometry is K13's
// (iod_geom).  Each anchor gives a TEME origin R, a unit vector L and a range interval [lo, hi]: lo = hi = the range
// when it is known; otherwise the positive roots of |R + rho L| = r_min and = r_max.  A track with no anchor is TOO_FEW.
//
// Pair: the track whose anchor is earlier is track 1, so (a, b) and (b, a) are the same pair; anchors at the same time
// make the pair BAD_PAIR.  The link's epoch is track 2's anchor time, tof = t2 - t1 seconds.
//
// Hypotheses: a known range is one; an unknown one kLinkRanges points rho_k = lo (hi / lo)^(k / (N - 1)), with k = 0
// and k = N - 1 exactly lo and hi.  Every (rho1, rho2, direction) cell solves K9's lambert_solve(R1 + rho1 L1,
// R2 + rho2 L2, tof, mu, +z or -z, max_revs); each OK slot is the two-body state (r2, v2) at the epoch, kept when K13's
// admissibility holds (finite, e < 1, perigee >= the model's earth radius).
//
// Coarse score: each admissible state is propagated two-body (iod_kepler) to the probe observations -- the first,
// anchor and last observation of each track, each observation once -- and scored by K8's residual rules (iod_score);
// F_probe is the sum of squared weighted residuals.  The kLinkSeeds least (F_probe, key) are the seeds, key =
// revs << 18 | retrograde << 17 | right branch << 16 | i1 << 8 | i2; keys are unique, so the order in which the cells are
// reduced does not matter.
//
// Refinement: Levenberg-Marquardt on each seed's unknown ranges (0, 1 or 2 variables) with revs, direction and branch
// fixed (link_branch solves that one slot), scored over every observation of both tracks (F), the Jacobian by forward
// differences of kLinkStep of each range.  A step is clamped to the range intervals; a step whose state has no solution
// on the seed's branch, is not admissible or does not lower F is rejected and the damping multiplied by 10 (an accepted
// step divides it by 10).  The refinement stops when a proposed step moves every range by at most kLinkTol of itself,
// or after kLinkIter steps.  The winner is the least (F, key); wrms = sqrt(F / used residuals of both tracks).
//
// Conversion: K13's (iod_epoch_state, K8's fit to the one TEME state at the epoch, B* held, iod_final_status).
#pragma once

#include "az_iod.cuh"

namespace az {

// per-pair status bytes (ASTROZ_LINK_*): the first four are K13's
enum LinkStatus : uint8_t {
    kLinkOk = kIodOk, kLinkTooFew = kIodTooFew, kLinkNoCandidate = kIodNoCandidate,
    kLinkConversionFailed = kIodConversionFailed, kLinkBadTrack = kIodBadTrack, kLinkBadPair = 5
};
constexpr uint8_t kLinkRetrograde = 1, kLinkRightBranch = 2;   // flags
constexpr uint32_t kLinkRanges = 32;    // hypotheses of an unknown range
constexpr int kLinkSeeds = 4;           // seeds refined per pair
constexpr int kLinkIter = 30;           // Levenberg-Marquardt steps per seed
constexpr double kLinkTol = 1e-10;      // relative range step that ends a refinement
constexpr double kLinkStep = 1e-7;      // forward-difference step, relative to the range
constexpr int kLinkProbes = 6;

// Observation i gives an anchor: every component of its line of sight used
AZ_HD bool link_anchor_obs(const CorrObsArrays &a, uint32_t i) {
    const double *sg = a.sigma + (size_t)i * 6;
    const int need = a.kind[i] == kObsOptical ? 2 : 3;
    for (int c = 0; c < need; ++c)
        if (!(sg[c] < INFINITY)) return false;
    return true;
}

// The positive root of |R + rho L| = r for |R| < r, without cancellation
AZ_HD double link_range_root(const double *R, const double *L, double r) {
    const double b = iod_dot(R, L), c = iod_dot(R, R) - r * r;
    const double d = std::sqrt(b * b - c);
    return b > 0.0 ? -c / (b + d) : d - b;
}

struct LinkAnchor {
    uint32_t index;     // the observation
    double t;           // its jdFull
    double R[3], L[3];  // origin and unit line of sight, TEME
    double lo, hi;      // range interval, km; lo == hi when the range is known
    uint32_t n;         // hypotheses: 1 or kLinkRanges
};

// The index of track [begin, end)'s anchor observation, end when it has none
AZ_HD uint32_t link_anchor_index(const CorrObsArrays &a, uint32_t begin, uint32_t end) {
    uint32_t c = 0;
    for (uint32_t i = begin; i < end; ++i) c += link_anchor_obs(a, i);
    if (c == 0) return end;
    uint32_t k = c / 2, i = begin;
    for (;; ++i)
        if (link_anchor_obs(a, i) && k-- == 0) return i;
}

// Track [begin, end)'s anchor; false when it has none
AZ_HD bool link_anchor(const CorrObsArrays &a, uint32_t begin, uint32_t end, double rMin, double rMax, LinkAnchor &an) {
    const uint32_t i = link_anchor_index(a, begin, end);
    if (i == end) return false;
    IodGeom g;
    iod_geom(a, i, g);
    an.index = i;
    an.t = g.t;
    const int kind = a.kind[i];
    if (kind == kObsOptical) {
        for (int q = 0; q < 3; ++q) an.R[q] = g.R[q], an.L[q] = g.L[q];
        an.lo = link_range_root(an.R, an.L, rMin);
        an.hi = link_range_root(an.R, an.L, rMax);
        an.n = kLinkRanges;
        return true;
    }
    for (int q = 0; q < 3; ++q) an.R[q] = 0.0;
    if (kind == kObsRadar) {   // the station's TEME position, as iod_geom rotates it
        CorrObs o;
        corr_obs(a, i, o);
        for (int q = 0; q < 3; ++q) an.R[q] = o.st.r[q];
        iod_to_teme(an.R[0], an.R[1], o.sg, o.cg);
    }
    double d[3];
    for (int q = 0; q < 3; ++q) d[q] = g.s[q] - an.R[q];
    const double rho = iod_norm(d);
    for (int q = 0; q < 3; ++q) an.L[q] = d[q] / rho;
    an.lo = an.hi = rho;
    an.n = 1;
    return true;
}

// Hypothesis k of an anchor
AZ_HD double link_range(const LinkAnchor &an, uint32_t k) {
    if (an.n == 1 || k == 0) return an.lo;
    if (k == an.n - 1) return an.hi;
    return an.lo * std::pow(an.hi / an.lo, (double)k / (double)(an.n - 1));
}

struct LinkPair {
    IodTrack tr[2];          // track 1 (the earlier anchor), track 2
    LinkAnchor an[2];
    uint32_t probe[kLinkProbes];
    int nProbe;
    double tof;              // seconds from anchor 1 to anchor 2
    uint32_t used;           // used residuals of both tracks
    uint8_t status;          // kLinkOk, or the pair's status before any scoring
};

// Pair (ia, ib) of the t tracks of offsets.  ia or ib >= t, ia == ib, or an anchor range interval that is not
// 0 < lo <= hi < inf: BAD_PAIR (the host call refuses all of these); a track K13 would call BAD_TRACK: BAD_TRACK; no
// anchor: TOO_FEW; anchors at the same time: BAD_PAIR.
AZ_HD void link_pair(const CorrObsArrays &a, const uint32_t *offsets, uint32_t t, uint32_t ia, uint32_t ib,
                     double rMin, double rMax, LinkPair &p) {
    p.nProbe = 0;
    p.tof = 0.0;
    p.used = 0;
    p.status = kLinkBadPair;
    if (ia >= t || ib >= t || ia == ib) return;
    iod_track(a, offsets[ia], offsets[ia + 1], p.tr[0]);
    iod_track(a, offsets[ib], offsets[ib + 1], p.tr[1]);
    p.status = kLinkBadTrack;
    if (p.tr[0].status == kIodBadTrack || p.tr[1].status == kIodBadTrack) return;
    p.status = kLinkTooFew;
    for (int k = 0; k < 2; ++k)
        if (!link_anchor(a, p.tr[k].begin, p.tr[k].end, rMin, rMax, p.an[k])) return;
    p.status = kLinkBadPair;
    if (p.an[0].t == p.an[1].t) return;
    if (p.an[1].t < p.an[0].t) {
        const IodTrack tt = p.tr[0];
        p.tr[0] = p.tr[1];
        p.tr[1] = tt;
        const LinkAnchor aa = p.an[0];
        p.an[0] = p.an[1];
        p.an[1] = aa;
    }
    for (int k = 0; k < 2; ++k)
        if (!(p.an[k].lo > 0.0 && p.an[k].lo <= p.an[k].hi && p.an[k].hi < INFINITY)) return;
    p.tof = iod_seconds(p.an[1].t, p.an[0].t);
    p.used = p.tr[0].used + p.tr[1].used;
    for (int k = 0; k < 2; ++k) {
        const uint32_t ix[3] = {p.tr[k].begin, p.an[k].index, p.tr[k].end - 1};
        for (int q = 0; q < 3; ++q)
            if (q == 0 || (ix[q] != ix[q - 1] && ix[q] != ix[0])) p.probe[p.nProbe++] = ix[q];
    }
    p.status = kLinkOk;
}

// Cells of a pair: (i1, i2, direction), direction fastest
AZ_HD uint32_t link_cells(const LinkPair &p) { return p.an[0].n * p.an[1].n * 2; }

AZ_HD uint32_t link_key(uint32_t slot, uint32_t dir, uint32_t i1, uint32_t i2) {
    const uint32_t M = (slot + 1) / 2, right = M > 0 && (slot & 1) == 0;
    return M << 18 | dir << 17 | right << 16 | i1 << 8 | i2;
}
AZ_HD uint8_t link_flags(uint32_t key) {
    return (uint8_t)((key >> 17 & 1 ? kLinkRetrograde : 0) | (key >> 16 & 1 ? kLinkRightBranch : 0));
}
AZ_HD uint32_t link_key_slot(uint32_t key) {
    const uint32_t M = key >> 18;
    return M == 0 ? 0 : (key >> 16 & 1) ? 2 * M : 2 * M - 1;
}

// r1 = R1 + rho1 L1, r2 = R2 + rho2 L2
AZ_HD void link_positions(const LinkPair &p, const double (&x)[2], double (&r1)[3], double (&r2)[3]) {
    for (int q = 0; q < 3; ++q) {
        r1[q] = p.an[0].R[q] + x[0] * p.an[0].L[q];
        r2[q] = p.an[1].R[q] + x[1] * p.an[1].L[q];
    }
}

// The seeds of a lane: the kLinkSeeds least (F, key), ascending
struct LinkSeeds {
    double F[kLinkSeeds];
    uint32_t key[kLinkSeeds];
};

AZ_HD void link_seeds_init(LinkSeeds &s) {
    for (int q = 0; q < kLinkSeeds; ++q) s.F[q] = INFINITY, s.key[q] = 0xFFFFFFFFu;
}

AZ_HD void link_seed_insert(LinkSeeds &s, double F, uint32_t key) {
    if (!iod_better(F, key, s.F[kLinkSeeds - 1], s.key[kLinkSeeds - 1])) return;
    int q = kLinkSeeds - 1;
    for (; q > 0 && iod_better(F, key, s.F[q - 1], s.key[q - 1]); --q) s.F[q] = s.F[q - 1], s.key[q] = s.key[q - 1];
    s.F[q] = F;
    s.key[q] = key;
}

// F_probe of the state s at the epoch
AZ_HD double link_probe_score(const CorrObsArrays &a, const LinkPair &p, const double (&s)[6], double mu) {
    double F = 0.0;
    for (int q = 0; q < p.nProbe; ++q) {
        IodTrack one;
        one.begin = p.probe[q];
        one.end = p.probe[q] + 1;
        F += iod_score(a, one, s, p.an[1].t, mu);
    }
    return F;
}

// Cell c: every OK, admissible slot scored into seeds.  Returns the states scored.
AZ_HD uint32_t link_cell(const CorrObsArrays &a, const LinkPair &p, uint32_t c, uint32_t maxRevs, double mu, double rE,
                         LinkSeeds &seeds) {
    const uint32_t dir = c & 1, i2 = (c >> 1) % p.an[1].n, i1 = (c >> 1) / p.an[1].n;
    const double x[2] = {link_range(p.an[0], i1), link_range(p.an[1], i2)};
    double r1[3], r2[3];
    link_positions(p, x, r1, r2);
    const double n[3] = {0.0, 0.0, dir ? -1.0 : 1.0};
    uint32_t scored = 0;
    lambert_solve(r1, r2, p.tof, mu, n, maxRevs, [&](uint32_t slot, uint8_t st, int, const double *, const double *v2) {
        if (st != kLamOk) return;
        const double s[6] = {r2[0], r2[1], r2[2], v2[0], v2[1], v2[2]};
        if (!iod_admissible(s, mu, rE)) return;
        ++scored;
        const double F = link_probe_score(a, p, s, mu);
        if (F < INFINITY) link_seed_insert(seeds, F, link_key(slot, dir, i1, i2));
    });
    return scored;
}

// The state at the epoch of ranges x on slot `slot` and direction dir alone (lambert_solve's steps for that slot);
// false when the slot has no solution there or the state is not admissible.
AZ_HD bool link_branch(const LinkPair &p, const double (&x)[2], uint32_t dir, uint32_t slot, double mu, double rE,
                       double (&s)[6]) {
    double r1[3], r2[3];
    link_positions(p, x, r1, r2);
    const double n[3] = {0.0, 0.0, dir ? -1.0 : 1.0};
    LambertGeom g;
    if (lambert_geometry(r1, r2, p.tof, mu, n, g) != kLamOk) return false;
    const int M = (int)((slot + 1) / 2);
    if (lambert_mmax(g.T, g.lam, (uint32_t)M) < M) return false;
    double xx = lambert_guess(g.T, g.lam, slot);
    if (!lambert_householder(g.T, g.lam, M, xx)) return false;
    double v1[3], v2[3];
    lambert_velocities(g, mu, xx, v1, v2);
    for (int q = 0; q < 3; ++q) s[q] = r2[q], s[3 + q] = v2[q];
    return iod_admissible(s, mu, rE);
}

// F of state s[0] over every observation of both tracks and, for nvar > 0, the normal equations N (upper triangle
// N00, N01, N11) and b of the forward differences s[1 + j] at steps 1 / inv[1 + j].  +inf when a propagation fails or
// F is not finite.
AZ_HD double link_normal(const CorrObsArrays &a, const LinkPair &p, const double (*s)[6], int nvar, const double *inv,
                         double (&N)[3], double (&b)[2], double mu) {
    N[0] = N[1] = N[2] = b[0] = b[1] = 0.0;
    double F = 0.0;
    const double tRef = p.an[1].t;
    for (int k = 0; k < 2; ++k) {
        for (uint32_t i = p.tr[k].begin; i < p.tr[k].end; ++i) {
            CorrObs o;
            corr_obs(a, i, o);
            auto eval = [&](int q, double jdFull, const double (&)[1], double (&f)[6]) {
                return iod_kepler(s[q], s[q] + 3, iod_seconds(jdFull, tRef), mu, f, f + 3);
            };
            double obs[6], sc[6], r[6], J[12];
            if (!obs_residual_rows(eval, nvar, inv, o.jdFull, tRef, o.kind, o.value, o.w, o.sg, o.cg, o.st, obs, sc, r,
                                   J, 1))
                return INFINITY;
            for (int c = 0; c < 6; ++c) {
                F += r[c] * r[c];
                if (nvar > 0) {
                    N[0] += J[c] * J[c];
                    b[0] += J[c] * r[c];
                }
                if (nvar > 1) {
                    N[1] += J[c] * J[6 + c];
                    N[2] += J[6 + c] * J[6 + c];
                    b[1] += J[6 + c] * r[c];
                }
            }
        }
    }
    return F < INFINITY ? F : INFINITY;
}

// A refined seed
struct LinkBest {
    double F;
    uint32_t key;
    double s[6];
    double x[2];
    bool converged;   // the refinement ended on its step tolerance (or had no variable), not at kLinkIter
};

AZ_HD void link_best_init(LinkBest &w) {
    w.F = INFINITY;
    w.key = 0xFFFFFFFFu;
    for (int c = 0; c < 6; ++c) w.s[c] = 0.0;
    w.x[0] = w.x[1] = 0.0;
    w.converged = false;
}

// The Jacobian's states at x: s[1 + j] at x + h_j on variable j (h_j = kLinkStep x, negated when it would leave the
// interval); false when one has no solution on the branch.
AZ_HD bool link_jacobian_states(const LinkPair &p, const double (&x)[2], const int (&var)[2], int nvar, uint32_t dir,
                                uint32_t slot, double mu, double rE, double (*s)[6], double (&inv)[3]) {
    for (int j = 0; j < nvar; ++j) {
        const int v = var[j];
        double h = kLinkStep * x[v];
        if (x[v] + h > p.an[v].hi) h = -h;
        double xh[2] = {x[0], x[1]};
        xh[v] = x[v] + h;
        h = xh[v] - x[v];   // the step actually taken
        inv[1 + j] = 1.0 / h;
        if (!link_branch(p, xh, dir, slot, mu, rE, s[1 + j])) return false;
    }
    return true;
}

// Refine the seed `key` (Levenberg-Marquardt on its unknown ranges) into w
AZ_HD void link_refine(const CorrObsArrays &a, const LinkPair &p, uint32_t key, double mu, double rE, LinkBest &w) {
    link_best_init(w);
    const uint32_t slot = link_key_slot(key), dir = key >> 17 & 1;
    double x[2] = {link_range(p.an[0], key >> 8 & 0xFF), link_range(p.an[1], key & 0xFF)};
    int var[2] = {0, 0}, nvar = 0;
    for (int k = 0; k < 2; ++k)
        if (p.an[k].n > 1) var[nvar++] = k;
    double s[3][6], inv[3] = {1.0, 1.0, 1.0}, N[3], b[2];
    if (!link_branch(p, x, dir, slot, mu, rE, s[0])) return;
    bool jac = link_jacobian_states(p, x, var, nvar, dir, slot, mu, rE, s, inv);
    double F = link_normal(a, p, s, jac ? nvar : 0, inv, N, b, mu);
    double lambda = 1e-3;
    bool converged = nvar == 0;
#ifdef __CUDA_ARCH__
#pragma unroll 1
#endif
    for (int it = 0; jac && nvar > 0 && F < INFINITY && it < kLinkIter; ++it) {
        double d[2] = {0.0, 0.0};
        const double a00 = N[0] * (1.0 + lambda);
        if (nvar == 1) {
            d[0] = b[0] / a00;
        } else {
            const double a11 = N[2] * (1.0 + lambda), det = a00 * a11 - N[1] * N[1];
            d[0] = (b[0] * a11 - N[1] * b[1]) / det;
            d[1] = (a00 * b[1] - N[1] * b[0]) / det;
        }
        double xn[2] = {x[0], x[1]};
        bool small = true, finite = true;
        for (int j = 0; j < nvar; ++j) {
            const int v = var[j];
            finite = finite && std::fabs(d[j]) < INFINITY;
            xn[v] = fmin(fmax(x[v] + d[j], p.an[v].lo), p.an[v].hi);
            small = small && std::fabs(xn[v] - x[v]) <= kLinkTol * std::fabs(xn[v]);
        }
        double sn[6], Fn = INFINITY;
        if (finite && link_branch(p, xn, dir, slot, mu, rE, sn)) {
            double Nn[3], bn[2];
            const double (*sp)[6] = &sn;
            Fn = link_normal(a, p, sp, 0, inv, Nn, bn, mu);
        }
        if (Fn < F) {
            x[0] = xn[0], x[1] = xn[1];
            for (int c = 0; c < 6; ++c) s[0][c] = sn[c];
            F = Fn;
            lambda = fmax(lambda * 0.1, 1e-12);
            if ((converged = small)) break;
            jac = link_jacobian_states(p, x, var, nvar, dir, slot, mu, rE, s, inv);
            if (jac) {
                const double Fj = link_normal(a, p, s, nvar, inv, N, b, mu);
                jac = Fj < INFINITY;
            }
        } else {
            lambda *= 10.0;
            if ((converged = small && finite) || !finite) break;
        }
    }
    if (!(F < INFINITY)) return;
    w.F = F;
    w.key = key;
    for (int c = 0; c < 6; ++c) w.s[c] = s[0][c];
    w.x[0] = x[0];
    w.x[1] = x[1];
    w.converged = converged;
}

}  // namespace az
