// TEST INFRASTRUCTURE ONLY: runs K12 (az_correlate.cuh, __host__ __device__) on the CPU: every row's sets built once,
// every (track, row) pair scored by corr_pair_sums / corr_d2 and the lists kept by corr_insert, as correlate_kernel and
// correlate_deep_kernel do per thread.  emul_correlate is astroz_cuda_correlate_device's definition on host buffers
// (and can return the whole d2 matrix); emul_corr_pair the rows, sums and d2 of one pair; emul_fit_obs_sums the sums
// fit_accumulate_obs forms over the same observations; emul_chi2_quantile the gate.  Not part of the shipped library;
// nothing in astroz_b200/ references it.
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#include "az_correlate.cuh"

using namespace az;

namespace {

struct Row {
    int deep = 0, nvar = -1;   // -1: not built
    double el[8], P[kFitN], inv[kFitSets] = {};
    double cols[kFitSets][kSgp4Cols];
    Sdp4Sat sets[kFitSets];
    double2 lattice[kFitSets][2 * kFitLatticeNodes];
};

// row s's sets (the whole lattice: fit_deep_eval does not depend on its extent); false when they cannot be built
bool build_row(Row &r, const double *elements, uint32_t n, const double *covariance, const uint8_t *model,
               const Gravity &gr, uint32_t s) {
    const uint8_t md = model ? model[s] : 0;
    for (int c = 0; c < 8; ++c) r.el[c] = elements[(size_t)c * n + s];
    for (int q = 0; q < kFitN; ++q) r.P[q] = covariance ? covariance[(size_t)s * kFitN + q] : 0.0;
    r.deep = md == 1;
    r.nvar = -1;
    if (md > 1) return false;
    const int nvar = corr_nvar(r.P);
    double x[kFitVars];
    bool built = true;
    if (!r.deep) {
        FitNearEarth::vars_of(r.el, x);
        for (int k = 0; k <= nvar; ++k) built = fit_build_set(x, k, r.el[0], gr, r.cols[k], r.inv[k]) && built;
    } else {
        FitDeepSpace::vars_of(r.el, x);
        for (int k = 0; k <= nvar; ++k)
            built = fit_build_set_of<FitDeepSpace>(x, k, r.el[0], gr, r.sets[k], r.inv[k]) && built;
        if (built)
            for (int k = 0; k <= nvar; ++k)
                for (int dir = 0; dir < 2; ++dir) fit_deep_lattice(r.sets[k], dir, kFitLatticeNodes, r.lattice[k]);
    }
    if (built) r.nvar = nvar;
    return built;
}

template <typename Fn>
auto with_eval(const Row &r, const GravConsts &g, Fn fn) {
    if (!r.deep)
        return fn([&r, &g](int k, double, const double (&ts)[1], double (&f)[6]) {
            CellOut o[1];
            sgp4_cell<1>([&r, k](int c) { return r.cols[k][c]; }, ts, g, o);
            f[0] = o[0].rx; f[1] = o[0].ry; f[2] = o[0].rz;
            f[3] = o[0].vx; f[4] = o[0].vy; f[5] = o[0].vz;
            return true;
        });
    return fn([&r, &g](int k, double jdFull, const double (&)[1], double (&f)[6]) {
        return fit_deep_eval(r.sets[k], r.lattice[k], jdFull, g, f);
    });
}

}  // namespace

extern "C" double emul_chi2_quantile(uint32_t k, double p) { return corr_chi2_quantile(k, p); }

extern "C" size_t emul_corr_scratch_bytes(uint32_t n, uint32_t t, uint32_t best) {
    return corr_scratch_bytes(n, t, best);
}

// d2_all[t][n] (nullable): each pair's d2, NaN for a failed pair, a row that is not built or a bad track
extern "C" int emul_correlate(const double *elements, uint32_t n, int grav, const double *covariance,
                              const uint8_t *model, const uint32_t *offsets, uint32_t t, const double *jd,
                              const double *fr, const uint8_t *kind, const double *value, const double *sigma,
                              const uint32_t *station, const double *stations, double gateProbability, uint32_t best,
                              uint32_t *rows, double *d2, uint32_t *used, uint32_t *nGate, uint32_t *nFailed,
                              uint8_t *status, uint8_t *rowStatus, double *d2All) {
    const Gravity gr = gravity(grav);
    const GravConsts g = grav_consts(gr);
    const CorrObsArrays in{jd, fr, kind, value, sigma, station, stations};
    std::vector<Row> cat(n);
    for (uint32_t s = 0; s < n; ++s)
        rowStatus[s] = build_row(cat[s], elements, n, covariance, model, gr, s) ? kCovOk : kCovInitFailed;
    for (uint32_t j = 0; j < t; ++j) {
        const uint32_t b = offsets[j], e = offsets[j + 1];
        const bool sized = e > b && e - b <= kCorrMaxTrack;
        used[j] = sized ? corr_used(in, b, e) : 0;
        double bd[kCorrMaxBest];
        uint32_t br[kCorrMaxBest];
        corr_empty(bd, br);
        uint32_t ng = 0, nf = 0;
        const bool bad = corr_bad_track(b, e, used[j]);
        const double gate = bad ? NAN : corr_chi2_quantile(used[j], gateProbability);
        for (uint32_t s = 0; s < n; ++s) {
            double dd = NAN;
            const Row &r = cat[s];
            if (!bad && r.nvar >= 0) {
                double acc[kFitSumWords], J[kFitVars * 6];
                const bool ok = with_eval(r, g, [&](auto eval) {
                    return corr_pair_sums(eval, r.nvar, r.inv, r.el[0], in, b, e, J, acc);
                });
                dd = ok ? corr_d2(acc, r.P, r.nvar) : NAN;
                if (!(std::fabs(dd) < INFINITY)) {
                    ++nf;
                    dd = NAN;
                } else {
                    dd = dd > 0.0 ? dd : 0.0;
                    if (dd <= gate) ++ng;
                    corr_insert(bd, br, dd, s);
                }
            }
            if (d2All) d2All[(size_t)j * n + s] = dd;
        }
        for (uint32_t i = 0; i < best; ++i) {
            rows[(size_t)j * best + i] = br[i];
            d2[(size_t)j * best + i] = bd[i];
        }
        nGate[j] = ng;
        nFailed[j] = nf;
        status[j] = bad ? kCorrBadTrack : corr_status(ng, br[0]);
    }
    return 0;
}

// One pair, row s against the observations [b, e): z[L][6], G[L][7][6] (entry (j, c), zero past nvar), the sums
// (FitSums word layout), the nominal states f0[L][6]; returns d2 (unclamped), NaN when the pair fails or the row is not
// built.
extern "C" double emul_corr_pair(const double *elements, uint32_t n, int grav, const double *covariance,
                                 const uint8_t *model, uint32_t s, uint32_t b, uint32_t e, const double *jd,
                                 const double *fr, const uint8_t *kind, const double *value, const double *sigma,
                                 const uint32_t *station, const double *stations, double *z, double *G, double *sums,
                                 double *f0) {
    const Gravity gr = gravity(grav);
    const GravConsts g = grav_consts(gr);
    const CorrObsArrays in{jd, fr, kind, value, sigma, station, stations};
    static Row r;
    if (!build_row(r, elements, n, covariance, model, gr, s)) return NAN;
    return with_eval(r, g, [&](auto eval) {
        for (uint32_t i = b; i < e; ++i) {
            CorrObs o;
            corr_obs(in, i, o);
            double obs[6], sc[6], rr[6], J[kFitVars * 6] = {};
            obs_residual_rows(eval, r.nvar, r.inv, o.jdFull, r.el[0], o.kind, o.value, o.w, o.sg, o.cg, o.st, obs, sc,
                              rr, J, 1);
            std::memcpy(z + (size_t)(i - b) * 6, rr, sizeof rr);
            std::memcpy(G + (size_t)(i - b) * kFitVars * 6, J, sizeof J);
            const double ts[1] = {mul_rn(sub_rn(o.jdFull, r.el[0]), 1440.0)};
            double f[6];
            eval(0, o.jdFull, ts, f);
            std::memcpy(f0 + (size_t)(i - b) * 6, f, sizeof f);
        }
        double acc[kFitSumWords], J[kFitVars * 6];
        const bool ok = corr_pair_sums(eval, r.nvar, r.inv, r.el[0], in, b, e, J, acc);
        std::memcpy(sums, acc, sizeof acc);
        return ok ? corr_d2(acc, r.P, r.nvar) : NAN;
    });
}

// The element fit's sums over the same observations under row s's sets with nvar stepped sets (fit_accumulate_obs,
// stride 1, the sums zeroed first): FitSums words
extern "C" int emul_fit_obs_sums(const double *elements, uint32_t n, int grav, const double *covariance,
                                 const uint8_t *model, uint32_t s, uint32_t b, uint32_t e, const double *jd,
                                 const double *fr, const uint8_t *kind, const double *value, const double *sigma,
                                 const uint32_t *station, const double *stations, double *sums) {
    const Gravity gr = gravity(grav);
    const GravConsts g = grav_consts(gr);
    const CorrObsArrays in{jd, fr, kind, value, sigma, station, stations};
    static Row r;
    if (!build_row(r, elements, n, covariance, model, gr, s)) return -1;
    return with_eval(r, g, [&](auto eval) {
        double acc[kFitSumWords] = {}, J[kFitVars * 6];
        bool ok = true;
        for (uint32_t i = b; i < e; ++i) {
            CorrObs o;
            corr_obs(in, i, o);
            ok = fit_accumulate_obs(eval, r.nvar, r.inv, o.jdFull, r.el[0], o.kind, o.value, o.w, o.sg, o.cg, o.st, J,
                                    acc, 1) && ok;
        }
        std::memcpy(sums, acc, sizeof acc);
        return ok ? 0 : -1;
    });
}
