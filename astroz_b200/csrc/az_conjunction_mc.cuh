// az_conjunction_mc.cuh -- K14: Monte Carlo collision probability of candidate conjunctions.  __host__ __device__, so
// the kernels (az_conjunction_mc.cu) and the host emulation (tests/host_emul/emul_conjunction_mc.cu) run this source.
//
// Candidate i is K11's (az_conjunction.cuh): rows p = primary[i] != s = secondary[i] with element columns, covariance
// P and a model byte, the guess time jd + fr, the half window w [min] and the hard-body radius R [km]; plus samples,
// first and seed.  For each row o:
//   nominal   x^ = Model::vars_of(el) over nvar = cov_nvar(P) variables (B* held when P's B* row is zero, as K10 and
//             K11 hold it); INIT_FAILED when the set of x^ cannot be built under the row's model or the byte is > 1;
//   factor    S = D^-1/2 P D^-1/2 over the nvar variables (D = diag P; a zero-variance variable has a zero row and
//             column), S = L L^T by a semidefinite Cholesky: a pivot in [-1e-12, 1e-12] zeroes its column, a pivot
//             below -1e-12 (or a negative variance) is kConjNotPsd;
//   sample k  x_k = x^ + D^1/2 L z, k in [first, first + samples), z the row's normals of sample k (mc_row_normals).
// Per sample: both rows' sets of x_k (fit_build_set_of<Model>(x_k, 0, ...); deep space with K11's lattices over
// [ts0 - w, ts0 + w]), conj_tca over [-w, w] on them -- K11's TCA applied to the drawn sets -- and the miss |dr| at
// that TCA.  A sample is failed when a set cannot be built, a deep-space cell fails or the miss is not finite (a
// near-earth set that decays inside the window propagates to NaN), and is then neither a hit nor a miss; it is an edge
// when conj_tca returns kConjWindowEdge (and still scored); a hit when miss < R.
// A sample's result depends on its candidate's inputs and its index k alone.
#pragma once

#include "az_conjunction.cuh"

namespace az {

// the counts words (hits, edge, failed) and the sample words (dt_tca [min], miss [km])
constexpr int kMcCountWords = 3;
constexpr int kMcSampleWords = 2;
constexpr int kMcBlocks = 7;                 // Philox blocks per sample: 14 normals, 7 per row
constexpr double kMcPivotZero = 1e-12;       // |pivot| at most this: a zero column of L

// ---- Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC 2011) --------------------------
struct McU4 {
    uint32_t x, y, z, w;
};

AZ_HD void mc_mulhilo(uint32_t a, uint32_t b, uint32_t &hi, uint32_t &lo) {
    const uint64_t p = (uint64_t)a * b;
    hi = (uint32_t)(p >> 32);
    lo = (uint32_t)p;
}

// Ten rounds on counter c under key (k0, k1)
AZ_HD McU4 mc_philox(McU4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        if (r) {
            k0 += 0x9E3779B9u;
            k1 += 0xBB67AE85u;
        }
        uint32_t hi0, lo0, hi1, lo1;
        mc_mulhilo(0xD2511F53u, c.x, hi0, lo0);
        mc_mulhilo(0xCD9E8D57u, c.z, hi1, lo1);
        c = McU4{hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0};
    }
    return c;
}

// A uniform in (0, 1] from two words: ((a 2^21 + (b >> 11)) + 0.5) 2^-53, the sum rounded in fp64
AZ_HD double mc_uniform(uint32_t a, uint32_t b) {
    const uint64_t u = ((uint64_t)a << 21) + (b >> 11);
    return ((double)u + 0.5) * 0x1p-53;
}

// Normals 2j and 2j + 1 of sample k under `seed`: block j = Philox of counter (j, k lo, k hi, 0) under key (seed lo,
// seed hi), Box-Muller on its uniforms (a, b) and (c, d)
AZ_HD void mc_normal_pair(uint64_t seed, uint64_t k, int j, double &n0, double &n1) {
    const McU4 o = mc_philox(McU4{(uint32_t)j, (uint32_t)k, (uint32_t)(k >> 32), 0u}, (uint32_t)seed,
                             (uint32_t)(seed >> 32));
    const double u1 = mc_uniform(o.x, o.y), u2 = mc_uniform(o.z, o.w);
    const double r = std::sqrt(-2.0 * std::log(u1)), t = detail::kHTwoPi * u2;
    n0 = r * std::cos(t);
    n1 = r * std::sin(t);
}

// Row o's seven normals of sample k: normals 7 o .. 7 o + 6 of the fourteen (the B* normal is drawn when B* is held)
AZ_HD void mc_row_normals(uint64_t seed, uint64_t k, int o, double (&z)[kFitVars]) {
    double all[2 * kMcBlocks];
    const int j0 = o ? 3 : 0, j1 = o ? kMcBlocks : 4;   // the blocks holding normals 7 o .. 7 o + 6
    for (int j = j0; j < j1; ++j) mc_normal_pair(seed, k, j, all[2 * j], all[2 * j + 1]);
    for (int v = 0; v < kFitVars; ++v) z[v] = all[kFitVars * o + v];
}

// ---- the factor ---------------------------------------------------------------------------------------------------
struct McFactor {
    double sd[kFitVars];     // sqrt(P_jj), 0 for a zero-variance or unused variable
    double L[kFitN];         // lower triangle of L by rows: entry (a, b), b <= a, at fit_tri(b, a)
};

// P's 28 words over nvar variables -> F; false when P is not positive semidefinite by the pivot rule
AZ_HD bool mc_factor(const double *P, int nvar, McFactor &F) {
    for (int q = 0; q < kFitN; ++q) F.L[q] = 0.0;
    for (int j = 0; j < kFitVars; ++j) {
        const double v = j < nvar ? P[fit_tri(j, j)] : 0.0;
        if (v < 0.0) return false;
        F.sd[j] = std::sqrt(v);
    }
    for (int j = 0; j < nvar; ++j) {
        if (F.sd[j] == 0.0) continue;   // a zero row and column of S
        double piv = 1.0;
        for (int c = 0; c < j; ++c) piv -= F.L[fit_tri(c, j)] * F.L[fit_tri(c, j)];
        if (piv < -kMcPivotZero) return false;
        if (piv <= kMcPivotZero) continue;
        const double d = std::sqrt(piv);
        F.L[fit_tri(j, j)] = d;
        for (int a = j + 1; a < nvar; ++a) {
            if (F.sd[a] == 0.0) continue;
            double s = P[fit_tri(j, a)] / (F.sd[j] * F.sd[a]);
            for (int c = 0; c < j; ++c) s -= F.L[fit_tri(c, a)] * F.L[fit_tri(c, j)];
            F.L[fit_tri(j, a)] = s / d;
        }
    }
    return true;
}

// x = xh + D^1/2 L z over the factor's variables; the others keep xh
AZ_HD void mc_draw(const McFactor &F, const double (&xh)[kFitVars], const double (&z)[kFitVars],
                   double (&x)[kFitVars]) {
    for (int a = 0; a < kFitVars; ++a) {
        double s = 0.0;
        for (int b = 0; b <= a; ++b) s += F.L[fit_tri(b, a)] * z[b];
        x[a] = xh[a] + F.sd[a] * s;
    }
}

// The row's nominal variables, factor and status: kConjOk, kConjInitFailed (the nominal set cannot be built, or
// model > 1) or kConjNotPsd
AZ_HD uint8_t mc_row(const double (&el)[8], const double *P, int model, const Gravity &grav, double (&xh)[kFitVars],
                     McFactor &F) {
    if (model > 1) return kConjInitFailed;
    double inv;
    bool built;
    if (model) {
        FitDeepSpace::vars_of(el, xh);
        Sdp4Sat set;
        built = fit_build_set_of<FitDeepSpace>(xh, 0, el[0], grav, set, inv);
    } else {
        FitNearEarth::vars_of(el, xh);
        double cols[kSgp4Cols];
        built = fit_build_set_of<FitNearEarth>(xh, 0, el[0], grav, cols, inv);
    }
    if (!built) return kConjInitFailed;
    return mc_factor(P, cov_nvar(P), F) ? kConjOk : kConjNotPsd;
}

// A candidate's status from its rows' (the primary's first)
AZ_HD uint8_t mc_status(uint8_t sp, uint8_t ss) {
    if (sp == kConjInitFailed || ss == kConjInitFailed) return kConjInitFailed;
    return sp != kConjOk ? sp : ss;
}

// The miss at the TCA from the two TEME states, as conj_geometry forms it
AZ_HD double mc_miss(const double (&fp)[6], const double (&fs)[6]) {
    double dr[3];
    for (int c = 0; c < 3; ++c) dr[c] = fs[c] - fp[c];
    return std::sqrt(dr[0] * dr[0] + dr[1] * dr[1] + dr[2] * dr[2]);
}

// Work items: candidate i's samples in blocks of B, ceil(samples / B) items
AZ_HD uint64_t mc_items(uint64_t samples, uint32_t B) { return samples / B + (samples % B ? 1 : 0); }

// The candidate of work item q: the least i < m with prefix[i] > q (prefix inclusive, non-decreasing, q < prefix[m-1])
AZ_HD uint32_t mc_candidate(const uint64_t *prefix, uint32_t m, uint64_t q) {
    uint32_t lo = 0, hi = m - 1;
    while (lo < hi) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (prefix[mid] > q) hi = mid;
        else lo = mid + 1;
    }
    return lo;
}

}  // namespace az
