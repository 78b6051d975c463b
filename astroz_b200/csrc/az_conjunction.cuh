// az_conjunction.cuh -- K11: assessment of candidate conjunctions: time of closest approach, miss, encounter-plane
// covariance and the short-encounter 2-D probability of collision.  __host__ __device__, so the kernels
// (az_conjunction.cu) and the host emulation (tests/host_emul/emul_conjunction.cu) run this source.
//
// Candidate i pairs catalogue rows p = primary[i] and s = secondary[i] (each with K10's element columns, covariance P
// and model byte) around the guess time jd + fr, with a half window w [min] and a combined hard-body radius R [km]:
//   nominal   each row's state at dt minutes from the guess: tsince = ts0 + dt, ts0 = ((jd + fr) - epoch) * 1440 formed
//             as K10 forms it, under the row's own model (sgp4_cell<1> on fit_columns, or the K2a-lattice SDP4 cell);
//             dr = r_s - r_p, dv = v_s - v_p;
//   TCA       a root of g = dr . dv where g goes from - to +, inside [-w, w] (conj_tca); several roots: the one with the
//             least |dr|; none: the window end with the smaller |dr|, status kConjWindowEdge;
//   Sigma     each row's 6 x 6 covariance at the TCA from K10's cov_query (same B*-held, zero-P and status rules), in
//             TEME or that row's own RTN frame;
//   plane     z = dv / |dv|, x = the part of dr perpendicular to z, normalised (exact hit: conj_geometry's fixed choice),
//             y = z x x; C2 = the (x, y) block of the position covariances Sigma_p + Sigma_s (uncorrelated objects);
//             |dv| = 0: kConjNoPlane, C2 and Pc zero;
//   Pc        the integral of N((u, v); (d, 0), C2) over the disk u^2 + v^2 <= R^2, d = |dr perpendicular to z|.
// A candidate's bytes depend on its own inputs and its two rows alone.
#pragma once

#include "az_covariance.cuh"

namespace az {

// per-candidate status bytes (ASTROZ_CONJ_*); 1 and 2 mean what K10's do; kConjNotPsd is K14's alone
enum ConjStatus : uint8_t {
    kConjOk = 0, kConjInitFailed = 1, kConjCellFailed = 2, kConjWindowEdge = 3, kConjNoPlane = 4, kConjBadPair = 5,
    kConjNotPsd = 6
};

// record words: dt_tca [min], miss [km], relative speed [km/s], (dr, dv) in the primary's RTN frame, C2 (xx, xy, yy)
// [km^2], Pc
constexpr int kConjRecordWords = 13;
constexpr int kConjRecRtn = 3, kConjRecC2 = 9, kConjRecPc = 12;

constexpr int kConjSamples = 32;       // samples of g per round: one per lane
constexpr double kConjTol = 1e-9;      // [min]: a bracket this narrow ends the search (then one secant step)
constexpr int kConjMaxRounds = 16;     // refinement rounds per bracket: width / 31^16 is below any tolerance
constexpr int kConjGauss = 16;         // Gauss-Legendre nodes per quadrature panel
constexpr int kConjBreaks = 64;        // candidate panel edges (conj_break)

// Sample l of the 32 spanning [a, b]: a, ..., b, both ends exact
AZ_HD double conj_node(double a, double b, int l) { return l == kConjSamples - 1 ? b : fma((double)l, (b - a) / 31.0, a); }

AZ_HD int conj_ctz(uint32_t v) {
#ifdef __CUDA_ARCH__
    return __ffs(v) - 1;
#else
    return __builtin_ctz(v);
#endif
}

// The TCA search.  S.round(a, b) evaluates the 32 samples conj_node(a, b, l) and returns the mask of g < 0; S.g(l) and
// S.d2(l) (= |dr|^2) read sample l of the last round.  Returns kConjOk or kConjWindowEdge with tca = dt [min].
// The first round brackets every - to + change of g over [-w, w]; each bracket is cut 31x per round until it is
// kConjTol wide, and the root is the secant of its ends.  With several brackets the root of least |dr| is kept (the
// first on a tie).
template <typename Sampler>
AZ_HD uint8_t conj_tca(Sampler &S, double w, double &tca) {
    const uint32_t neg = S.round(-w, w);
    uint32_t br = neg & ~(neg >> 1) & 0x7fffffffu;   // bit l: g(t_l) < 0 <= g(t_l+1)
    if (!br) {
        tca = S.d2(kConjSamples - 1) < S.d2(0) ? w : -w;
        return kConjWindowEdge;
    }
    const bool several = (br & (br - 1)) != 0;
    double best = 0.0;
    tca = 0.0;
    for (bool first = true; br; first = false) {
        const int l = conj_ctz(br);
        br &= br - 1;
        double a = conj_node(-w, w, l), b = conj_node(-w, w, l + 1), ga = 0.0, gb = 0.0;
        for (int it = 0; it < kConjMaxRounds; ++it) {
            const uint32_t nb = ~S.round(a, b);
            int k = nb ? conj_ctz(nb) : kConjSamples - 1;   // the first sample with g >= 0
            k = k < 1 ? 1 : k;
            const double a1 = conj_node(a, b, k - 1), b1 = conj_node(a, b, k);
            ga = S.g(k - 1);
            gb = S.g(k);
            a = a1;
            b = b1;
            if (b - a <= kConjTol) break;
        }
        const double den = ga - gb;
        const double t = den < 0.0 ? a + (b - a) * (ga / den) : a;
        if (several) {
            S.round(t, t);
            const double d2 = S.d2(0);
            if (first || d2 < best) {
                best = d2;
                tca = t;
            }
        } else {
            tca = t;
        }
    }
    return kConjOk;
}

// Word (a, b), a <= b, of a 21-word upper triangle
AZ_HD int conj_tri6(int a, int b) { return a * 6 - a * (a - 1) / 2 + (b - a); }

// The Pc integral's parameters in C2's principal axes: semi-axes s1 >= s2 [km] (sqrt of the eigenvalues), the disk
// centre's offset (m1, m2) from the mean along them, the radius R; kind 0 the quadrature, 1 s2 = 0 (a 1-D normal
// difference), 2 C2 = 0 (the indicator d < R), 3 no plane (Pc = 0).
struct ConjPc {
    double s1, s2, m1, m2, R, d;
    int kind;
};

// C2 = [[xx, xy], [xy, yy]] and the disk centre (d, 0), radius R -> principal-axis parameters
AZ_HD ConjPc conj_pc_params(double xx, double xy, double yy, double d, double R) {
    ConjPc p{0.0, 0.0, 0.0, 0.0, R, d, 0};
    const double half = 0.5 * (xx + yy), q = std::hypot(0.5 * (xx - yy), xy);
    const double l1 = half + q, det = xx * yy - xy * xy;
    const double l2 = (l1 > 0.0 && det > 0.0) ? det / l1 : 0.0;
    const double phi = 0.5 * std::atan2(2.0 * xy, xx - yy);
    p.s1 = l1 > 0.0 ? std::sqrt(l1) : 0.0;
    p.s2 = std::sqrt(l2);
    p.m1 = d * std::cos(phi);
    p.m2 = -d * std::sin(phi);
    p.kind = l1 > 0.0 ? (l2 > 0.0 ? 0 : 1) : 2;
    return p;
}

// The encounter geometry at the TCA: states fp, fs (TEME), their Sigma words sp, ss in `frame`, radius R -> record
// words 1 .. 11 and the Pc parameters; returns kConjOk or kConjNoPlane.
AZ_HD uint8_t conj_geometry(const double (&fp)[6], const double (&fs)[6], const double (&sp)[kCovWords],
                            const double (&ss)[kCovWords], int frame, double R, double *rec, ConjPc &pc) {
    double dr[3], dv[3], Rp[3][3];
    for (int c = 0; c < 3; ++c) {
        dr[c] = fs[c] - fp[c];
        dv[c] = fs[3 + c] - fp[3 + c];
    }
    const double miss = std::sqrt(dr[0] * dr[0] + dr[1] * dr[1] + dr[2] * dr[2]);
    const double speed = std::sqrt(dv[0] * dv[0] + dv[1] * dv[1] + dv[2] * dv[2]);
    rec[1] = miss;
    rec[2] = speed;
    cov_rtn(fp, Rp);
    for (int c = 0; c < 3; ++c) {
        rec[kConjRecRtn + c] = Rp[c][0] * dr[0] + Rp[c][1] * dr[1] + Rp[c][2] * dr[2];
        rec[kConjRecRtn + 3 + c] = Rp[c][0] * dv[0] + Rp[c][1] * dv[1] + Rp[c][2] * dv[2];
    }
    pc = ConjPc{0.0, 0.0, 0.0, 0.0, R, 0.0, 3};
    for (int q = 0; q < 3; ++q) rec[kConjRecC2 + q] = 0.0;
    if (!(speed > 0.0)) return kConjNoPlane;
    double z[3], x[3], y[3];
    for (int c = 0; c < 3; ++c) z[c] = dv[c] / speed;
    const double along = dr[0] * z[0] + dr[1] * z[1] + dr[2] * z[2];
    for (int c = 0; c < 3; ++c) x[c] = dr[c] - along * z[c];
    double d = std::sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
    if (d > 0.0) {
        for (int c = 0; c < 3; ++c) x[c] /= d;
    } else {   // exact hit: x from the TEME axis least aligned with z (the first on a tie)
        int k = 0;
        for (int c = 1; c < 3; ++c)
            if (std::fabs(z[c]) < std::fabs(z[k])) k = c;
        for (int c = 0; c < 3; ++c) x[c] = (c == k ? 1.0 : 0.0) - z[k] * z[c];
        const double xn = std::sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
        for (int c = 0; c < 3; ++c) x[c] /= xn;
    }
    y[0] = z[1] * x[2] - z[2] * x[1];
    y[1] = z[2] * x[0] - z[0] * x[2];
    y[2] = z[0] * x[1] - z[1] * x[0];
    // C2 = sum over both objects of E Sigma_pos E^T, E's rows x and y taken into the frame Sigma is stated in
    double c2[3] = {0.0, 0.0, 0.0};
    for (int o = 0; o < 2; ++o) {
        const double(&f)[6] = o ? fs : fp;
        const double(&sg)[kCovWords] = o ? ss : sp;
        double ex[3], ey[3];
        if (frame == kCovFrameRtn) {
            double Ro[3][3];
            cov_rtn(f, Ro);
            for (int c = 0; c < 3; ++c) {
                ex[c] = Ro[c][0] * x[0] + Ro[c][1] * x[1] + Ro[c][2] * x[2];
                ey[c] = Ro[c][0] * y[0] + Ro[c][1] * y[1] + Ro[c][2] * y[2];
            }
        } else {
            for (int c = 0; c < 3; ++c) {
                ex[c] = x[c];
                ey[c] = y[c];
            }
        }
        double cx[3], cy[3];   // Sigma_pos ex, Sigma_pos ey
        for (int a = 0; a < 3; ++a) {
            cx[a] = cy[a] = 0.0;
            for (int b = 0; b < 3; ++b) {
                const double s = sg[a <= b ? conj_tri6(a, b) : conj_tri6(b, a)];
                cx[a] += s * ex[b];
                cy[a] += s * ey[b];
            }
        }
        c2[0] += ex[0] * cx[0] + ex[1] * cx[1] + ex[2] * cx[2];
        c2[1] += ex[0] * cy[0] + ex[1] * cy[1] + ex[2] * cy[2];
        c2[2] += ey[0] * cy[0] + ey[1] * cy[1] + ey[2] * cy[2];
    }
    for (int q = 0; q < 3; ++q) rec[kConjRecC2 + q] = c2[q];
    pc = conj_pc_params(c2[0], c2[1], c2[2], d, R);
    return kConjOk;
}

// Phi(hi) - Phi(lo), lo <= hi, from erfc of same-sign arguments so far tails keep their digits
AZ_HD double conj_phi_diff(double lo, double hi) {
    constexpr double k = 0.70710678118654752440;
    if (lo >= 0.0) return 0.5 * (erfc(lo * k) - erfc(hi * k));
    if (hi <= 0.0) return 0.5 * (erfc(-hi * k) - erfc(-lo * k));
    return 1.0 - 0.5 * (erfc(hi * k) + erfc(-lo * k));
}

// The closed forms: kind 1 (one semi-axis 0), 2 (C2 = 0) and 3 (no plane); false for the quadrature
AZ_HD bool conj_pc_closed(const ConjPc &p, double &pc) {
    if (p.kind == 0) return false;
    if (p.kind == 3) pc = 0.0;
    else if (p.kind == 2) pc = p.d < p.R ? 1.0 : 0.0;
    else {
        const double m2 = std::fabs(p.m2);
        if (m2 < p.R) {
            const double h = std::sqrt((p.R - m2) * (p.R + m2));
            pc = conj_phi_diff((-h - p.m1) / p.s1, (h - p.m1) / p.s1);
        } else {
            pc = 0.0;
        }
    }
    return true;
}

// The quadrature runs over theta in [-pi/2, pi/2], u1 = R sin(theta) along the major axis and the chord half-length
// R cos(theta) along the minor one, integrand R cos(theta) phi(u1; m1, s1) P(|u2 - m2| <= R cos(theta); s2): smooth
// at the disk's edge.  Panel edges are where it turns sharp: the levels E = E_min + L of the major axis's exponent
// (E = (u1 - m1)^2 / 2 s1^2, E_min its least value on the disk) and the same levels of the minor axis's exponent in
// the chord half-length, L over kConjLevels.  Candidate idx -> theta, or kConjNoBreak when it falls outside the disk.
constexpr int kConjLevels = 10;
constexpr double kConjNoBreak = 1e300;
AZ_HD double conj_level(int c) {
    constexpr double L[kConjLevels] = {0.0, 0.5, 2.0, 4.5, 8.0, 12.5, 18.0, 24.5, 32.0, 50.0};
    return L[c];
}

AZ_HD double conj_break(const ConjPc &p, int idx) {
    constexpr double kHalfPi = 1.57079632679489661923;
    if (idx == 0) return -kHalfPi;
    if (idx == 1) return kHalfPi;
    if (idx == 2) return 0.0;
    if (idx < 3 + 2 * kConjLevels) {   // major axis: u1 = m1 -/+ s1 sqrt(delta^2 + 2 L)
        const int c = (idx - 3) >> 1;
        const double delta = fmax(std::fabs(p.m1) - p.R, 0.0) / p.s1;
        const double u = p.m1 + ((idx - 3) & 1 ? 1.0 : -1.0) * p.s1 * std::sqrt(delta * delta + 2.0 * conj_level(c));
        return std::fabs(u) < p.R ? std::asin(u / p.R) : kConjNoBreak;
    }
    const int j = idx - 3 - 2 * kConjLevels;
    if (j >= 4 * kConjLevels) return kConjNoBreak;
    // minor axis: chord half-length h = |m2| -/+ s2 sqrt(gamma^2 + 2 L), theta = -/+ acos(h / R)
    const int c = j >> 2;
    const double m2 = std::fabs(p.m2);
    const double gamma = fmax(m2 - p.R, 0.0) / p.s2;
    const double h = m2 + ((j >> 1) & 1 ? 1.0 : -1.0) * p.s2 * std::sqrt(gamma * gamma + 2.0 * conj_level(c));
    if (!(h > 0.0 && h < p.R)) return kConjNoBreak;
    const double t = std::acos(h / p.R);
    return j & 1 ? t : -t;
}

// Rank of candidate i among the valid ones of raw[kConjBreaks] (ties by index), -1 when invalid (invalid ones sort
// last, so the valid ranks are 0 .. K-1)
AZ_HD int conj_rank(const double *raw, int i) {
    const double v = raw[i];
    if (v == kConjNoBreak) return -1;
    int r = 0;
    for (int j = 0; j < kConjBreaks; ++j) {
        const double u = raw[j];
        r += (u < v || (u == v && j < i)) ? 1 : 0;
    }
    return r;
}

AZ_HD double conj_gl(int q, bool weight) {
    constexpr double x[kConjGauss / 2] = {0.09501250983763744, 0.2816035507792589, 0.45801677765722737,
                                          0.6178762444026438, 0.755404408355003, 0.8656312023878318,
                                          0.9445750230732326, 0.9894009349916499};
    constexpr double w[kConjGauss / 2] = {0.18945061045506864, 0.18260341504492364, 0.16915651939500265,
                                          0.1495959888165767, 0.12462897125553407, 0.0951585116824926,
                                          0.062253523938647456, 0.027152459411754176};
    const int h = q < kConjGauss / 2 ? kConjGauss / 2 - 1 - q : q - kConjGauss / 2;
    return weight ? w[h] : (q < kConjGauss / 2 ? -x[h] : x[h]);
}

// Lane `lane`'s share of the quadrature: nodes k = lane, lane + 32, ... of the (K - 1) panels between the sorted edges
// bp[0 .. K-1], each kConjGauss Gauss-Legendre nodes
AZ_HD double conj_partial(const ConjPc &p, const double *bp, int K, int lane) {
    constexpr double kInvSqrt2Pi = 0.39894228040143267794;
    const double m2 = std::fabs(p.m2);
    double acc = 0.0;
    for (int k = lane; k < (K - 1) * kConjGauss; k += kConjSamples) {
        const int pan = k / kConjGauss, q = k % kConjGauss;
        const double t0 = bp[pan], t1 = bp[pan + 1], hw = 0.5 * (t1 - t0);
        if (!(hw > 0.0)) continue;
        const double th = 0.5 * (t0 + t1) + hw * conj_gl(q, false);
        const double st = std::sin(th), ct = std::cos(th);
        const double u = p.R * st, h = p.R * ct;
        const double z = (u - p.m1) / p.s1;
        const double outer = std::exp(-0.5 * z * z) * kInvSqrt2Pi / p.s1;
        const double inner = conj_phi_diff((-h - m2) / p.s2, (h - m2) / p.s2);
        acc += hw * conj_gl(q, true) * h * outer * inner;
    }
    return acc;
}

// Set 0 .. 7 of a row at tsince ts [min]: near-earth columns col(c), or a deep-space record with its lattice
template <typename ColFn>
AZ_HD bool conj_eval_near(ColFn col, double ts, const GravConsts &g, double (&f)[6]) {
    const double t[1] = {ts};
    CellOut o[1];
    sgp4_cell<1>(col, t, g, o);
    f[0] = o[0].rx; f[1] = o[0].ry; f[2] = o[0].rz;
    f[3] = o[0].vx; f[4] = o[0].vy; f[5] = o[0].vz;
    return true;
}
AZ_HD bool conj_eval_deep(const Sdp4Sat &e, const double2 *lattice, double ts, const GravConsts &g, double (&f)[6]) {
    CellOut o;
    const int st = pairs_sdp4_at(e, lattice, kFitLatticeNodes, ts, g, o);
    f[0] = o.rx; f[1] = o.ry; f[2] = o.rz;
    f[3] = o.vx; f[4] = o.vy; f[5] = o.vz;
    return st == 0;
}

// The fixed reduction order of the 32 lane shares (the device's shuffle-down tree): v[0] receives the sum
AZ_HD void conj_tree(double *v) {
    for (int off = kConjSamples / 2; off > 0; off >>= 1)
        for (int l = 0; l < off; ++l) v[l] += v[l + off];
}

}  // namespace az
