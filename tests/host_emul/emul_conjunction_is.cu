// TEST INFRASTRUCTURE ONLY: runs K15 (az_conjunction_is.cuh, __host__ __device__) on the CPU.  The sampling restates
// the warp of conjunction_is_kernel / conjunction_is_deep_kernel serially on K14's host restatement (Row, HostSampler
// of emul_conjunction_mc.cu); the proposal restates is_proposal_kernel, with K11's record, states and status passed in
// from K11's host build (emul_conjunction.cu), as the device call takes them from K11's launch.
// emul_conjunction_is is astroz_cuda_conjunction_is_device's definition on host buffers, with two extra outputs for
// the tests: G[m][2][14] of each linear proposal and v[m][record] = exp(-u . c) of each recorded sample.  Not part of
// the shipped library; nothing in astroz_b200/ references it.
#include "emul_conjunction_mc.cu"

#include "az_conjunction_is.cuh"

namespace {

struct PropRow {
    int deep = 0, nvar = 0;
    double el[8], P[kFitN], inv[kFitSets] = {}, ts0 = 0.0;
    double cols[kFitSets][kSgp4Cols];
    Sdp4Sat sets[kFitSets];
    double2 lattice[kFitSets][2 * kFitLatticeNodes];

    bool eval(int k, double ts, const GravConsts &g, double (&f)[6]) const {
        if (!deep) return conj_eval_near([this, k](int c) { return cols[k][c]; }, ts, g, f);
        return conj_eval_deep(sets[k], lattice[k], ts, g, f);
    }
};

// The linear shift of one candidate (rows idx, K11's TCA and TEME states st[12]) -> c, |c|^2 and G; false: PLAIN
bool linear_shift(const double *elements, uint32_t n, const Gravity &gr, const double *covariance,
                  const uint8_t *model, const uint32_t (&idx)[2], double jdFull, double w, double tca, const double *st,
                  double (&c)[kIsShift], double &cc, double (&G)[2][2][kFitVars]) {
    static PropRow rows[2];
    const GravConsts g = grav_consts(gr);
    double e[2][3], d[2], fp[6], fs[6];
    for (int q = 0; q < 6; ++q) {
        fp[q] = st[q];
        fs[q] = st[6 + q];
    }
    if (!is_plane(fp, fs, e, d)) return false;
    for (int o = 0; o < 2; ++o) {
        PropRow &r = rows[o];
        const uint32_t s = idx[o];
        r.deep = model ? model[s] : 0;
        for (int q = 0; q < 8; ++q) r.el[q] = elements[(size_t)q * n + s];
        std::memcpy(r.P, covariance + (size_t)s * kFitN, sizeof r.P);
        r.nvar = cov_nvar(r.P);
        r.ts0 = pairs_tsince_deep(jdFull, r.el[0]);
        double x[kFitVars];
        bool built = true;
        if (!r.deep) {
            FitNearEarth::vars_of(r.el, x);
            for (int k = 0; k <= r.nvar; ++k) built = fit_build_set(x, k, r.el[0], gr, r.cols[k], r.inv[k]) && built;
        } else {
            FitDeepSpace::vars_of(r.el, x);
            for (int k = 0; k <= r.nvar; ++k)
                built = fit_build_set_of<FitDeepSpace>(x, k, r.el[0], gr, r.sets[k], r.inv[k]) && built;
            if (built) {
                const double hi = r.ts0 + w, lo = r.ts0 - w;
                const int nodes[2] = {fit_lattice_nodes(hi > 0.0 ? hi : 0.0), fit_lattice_nodes(lo < 0.0 ? -lo : 0.0)};
                for (int k = 0; k <= r.nvar; ++k)
                    for (int dir = 0; dir < 2; ++dir) fit_deep_lattice(r.sets[k], dir, nodes[dir], r.lattice[k]);
            }
        }
        if (!built) return false;
        const double ts = r.ts0 + tca;
        auto eval = [&r, &g, ts](int k, double, const double (&)[1], double (&f)[6]) { return r.eval(k, ts, g, f); };
        double J[kCovJacWords], f0[6], sig[kCovWords];
        if (cov_query(eval, r.nvar, r.inv, r.P, 0.0, 0.0, kCovFrameTeme, J, 1, f0, sig) != kCovOk) return false;
        McFactor F;
        if (!mc_factor(r.P, r.nvar, F)) return false;
        is_row_map(J, F, e, o ? 1.0 : -1.0, G[o]);
    }
    return is_linear_shift(G[0], G[1], d, c, cc);
}

}  // namespace

extern "C" int emul_conjunction_is(const double *elements, uint32_t n, int grav, const double *covariance,
                                   const uint8_t *model, const uint32_t *primary, const uint32_t *secondary,
                                   const double *jd, const double *fr, const double *window, const double *hbr,
                                   const uint64_t *samples, const uint64_t *first, const uint64_t *seed,
                                   const double *shift, const double *k11Record, const double *k11States,
                                   const uint8_t *k11Status, uint32_t m, uint32_t record, uint64_t *counts,
                                   double *proposal, uint8_t *kind, double *sampleOut, uint8_t *status, double *gmap,
                                   double *vOut) {
    const Gravity gr = gravity(grav);
    const GravConsts g = grav_consts(gr);
    const double nan = std::numeric_limits<double>::quiet_NaN();
    static Row rows[2];
    for (uint32_t i = 0; i < m; ++i) {
        uint64_t *cnt = counts + (size_t)i * kIsCountWords;
        double *prop = proposal + (size_t)i * kIsProposalWords;
        for (int q = 0; q < kIsCountWords; ++q) cnt[q] = 0;
        for (int q = 0; q < kIsProposalWords; ++q) prop[q] = 0.0;
        for (int q = 0; q < 2 * kIsShift; ++q) gmap[(size_t)i * 2 * kIsShift + q] = 0.0;
        kind[i] = kIsPlain;
        for (size_t q = 0; q < (size_t)record * kIsSampleWords; ++q)
            sampleOut[(size_t)i * record * kIsSampleWords + q] = nan;
        for (size_t q = 0; q < record; ++q) vOut[(size_t)i * record + q] = nan;
        const uint32_t idx[2] = {primary[i], secondary[i]};
        if (idx[0] >= n || idx[1] >= n || idx[0] == idx[1]) {
            status[i] = kConjBadPair;
            continue;
        }
        const double jdFull = add_rn(jd[i], fr[i]), w = window[i];
        uint8_t so[2];
        for (int o = 0; o < 2; ++o) {
            Row &r = rows[o];
            const uint32_t s = idx[o];
            r.deep = model ? model[s] : 0;
            for (int c = 0; c < 8; ++c) r.el[c] = elements[(size_t)c * n + s];
            r.ts0 = pairs_tsince_deep(jdFull, r.el[0]);
            so[o] = mc_row(r.el, covariance + (size_t)s * kFitN, r.deep, gr, r.xh, r.F);
        }
        status[i] = mc_status(so[0], so[1]);
        if (status[i] != kConjOk) continue;
        // the proposal
        double c[kIsShift] = {}, cc = 0.0;
        if (shift) {
            for (int q = 0; q < kIsShift; ++q) c[q] = shift[(size_t)i * kIsShift + q];
            cc = is_norm2(c);
            kind[i] = kIsGiven;
        } else if (k11Status[i] == kConjOk || k11Status[i] == kConjWindowEdge) {
            double G[2][2][kFitVars];
            if (linear_shift(elements, n, gr, covariance, model, idx, jdFull, w, k11Record[(size_t)i * kConjRecordWords],
                             k11States + (size_t)i * 12, c, cc, G)) {
                kind[i] = kIsLinear;
                for (int o = 0; o < 2; ++o)
                    for (int r = 0; r < 2; ++r)
                        for (int b = 0; b < kFitVars; ++b)
                            gmap[(size_t)i * 2 * kIsShift + r * kIsShift + kFitVars * o + b] = G[o][r][b];
            } else {
                for (int q = 0; q < kIsShift; ++q) c[q] = 0.0;
                cc = 0.0;
            }
        }
        for (int q = 0; q < kIsShift; ++q) prop[q] = c[q];
        prop[kIsShift] = is_log_scale(cc);
        // the samples
        const uint64_t f0 = first ? first[i] : 0, sd = seed ? seed[i] : 0;
        uint64_t V[4] = {0, 0, 0, 0}, V2[4] = {0, 0, 0, 0}, overflow = 0;
        for (uint64_t j = 0; j < samples[i]; ++j) {
            bool built = true;
            double uc[2];
            for (int o = 0; o < 2; ++o) {
                double z[kFitVars], x[kFitVars];
                mc_row_normals(sd, f0 + j, o, z);
                uc[o] = is_shift_normals(c + kFitVars * o, z);
                mc_draw(rows[o].F, rows[o].xh, z, x);
                built = rows[o].build(x, gr, w) && built;
            }
            const double ucs = uc[0] + uc[1];
            double out0 = nan, out1 = nan, out2 = nan, v = nan;
            if (built) {
                HostSampler S{rows[0], rows[1], g};
                double tca = 0.0;
                const uint8_t st = conj_tca(S, w, tca);
                double fp[6], fs[6];
                bool good = rows[0].eval(rows[0].ts0 + tca, g, fp) && S.ok;
                good = rows[1].eval(rows[1].ts0 + tca, g, fs) && good;
                const double miss = mc_miss(fp, fs);
                if (good && std::isfinite(miss)) {
                    cnt[0] += miss < hbr[i] ? 1 : 0;
                    cnt[1] += st == kConjWindowEdge ? 1 : 0;
                    out0 = tca;
                    out1 = miss;
                    out2 = -ucs + prop[kIsShift];
                    v = exp(-ucs);
                    if (miss < hbr[i]) is_hit(v, V, V2, overflow);
                } else {
                    ++cnt[2];
                }
            } else {
                ++cnt[2];
            }
            if (j < record) {
                double *d = sampleOut + ((size_t)i * record + j) * kIsSampleWords;
                d[0] = out0;
                d[1] = out1;
                d[2] = out2;
                vOut[(size_t)i * record + j] = v;
            }
        }
        cnt[3] = overflow;
        for (int q = 0; q < 4; ++q) {
            cnt[kIsCountV + q] = V[q];
            cnt[kIsCountV2 + q] = V2[q];
        }
    }
    return 0;
}
