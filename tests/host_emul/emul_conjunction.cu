// TEST INFRASTRUCTURE ONLY: runs K11 (az_conjunction.cuh, __host__ __device__) on the CPU with the warp of
// conjunction_kernel / conjunction_deep_kernel (az_conjunction.cu) restated serially: the 32 samples of a search round
// in a loop, the two covariance queries one after the other, the 32 lane shares of the Pc quadrature and their fixed
// reduction tree.  emul_conjunction is astroz_cuda_conjunction_device's definition on host buffers; emul_conj_pc the
// Pc of one encounter plane.  Not part of the shipped library; nothing in astroz_b200/ references it.
#include <cmath>
#include <cstdint>
#include <cstring>

#include "az_conjunction.cuh"

using namespace az;

namespace {

struct Row {
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

struct HostSampler {
    const Row &p, &s;
    const GravConsts &gc;
    double gs[kConjSamples], d2s[kConjSamples];
    bool ok = true;
    uint32_t round(double a, double b) {
        uint32_t neg = 0;
        for (int l = 0; l < kConjSamples; ++l) {
            const double t = conj_node(a, b, l);
            double fp[6], fs[6];
            ok = p.eval(0, p.ts0 + t, gc, fp) && ok;
            ok = s.eval(0, s.ts0 + t, gc, fs) && ok;
            double gg = 0.0, dd = 0.0;
            for (int c = 0; c < 3; ++c) {
                const double dr = fs[c] - fp[c], dv = fs[3 + c] - fp[3 + c];
                gg += dr * dv;
                dd += dr * dr;
            }
            gs[l] = gg;
            d2s[l] = dd;
            if (gg < 0.0) neg |= 1u << l;
        }
        return neg;
    }
    double g(int l) const { return gs[l]; }
    double d2(int l) const { return d2s[l]; }
};

void zero(uint32_t i, uint8_t st, double *record, double *states, double *stateCov, uint8_t *status) {
    std::memset(record + (size_t)i * kConjRecordWords, 0, sizeof(double) * kConjRecordWords);
    if (states) std::memset(states + (size_t)i * 12, 0, sizeof(double) * 12);
    if (stateCov) std::memset(stateCov + (size_t)i * 2 * kCovWords, 0, sizeof(double) * 2 * kCovWords);
    status[i] = st;
}

}  // namespace

extern "C" double emul_conj_pc(double xx, double xy, double yy, double d, double R) {
    const ConjPc p = conj_pc_params(xx, xy, yy, d, R);
    double pc = 0.0;
    if (conj_pc_closed(p, pc)) return pc;
    double raw[kConjBreaks], bp[kConjBreaks], share[kConjSamples];
    for (int k = 0; k < kConjBreaks; ++k) raw[k] = conj_break(p, k);
    int K = 0;
    for (int k = 0; k < kConjBreaks; ++k) {
        const int r = conj_rank(raw, k);
        if (r >= 0) {
            bp[r] = raw[k];
            ++K;
        }
    }
    for (int l = 0; l < kConjSamples; ++l) share[l] = conj_partial(p, bp, K, l);
    conj_tree(share);
    return share[0];
}

extern "C" int emul_conjunction(const double *elements, uint32_t n, int grav, const double *covariance,
                                const uint8_t *model, const uint32_t *primary, const uint32_t *secondary,
                                const double *jd, const double *fr, const double *window, const double *hbr,
                                uint32_t m, int frame, double *record, double *states, double *stateCov,
                                uint8_t *status) {
    const Gravity gr = gravity(grav);
    const GravConsts g = grav_consts(gr);
    static Row rows[2];
    for (uint32_t i = 0; i < m; ++i) {
        const uint32_t idx[2] = {primary[i], secondary[i]};
        if (idx[0] >= n || idx[1] >= n || idx[0] == idx[1]) {
            zero(i, kConjBadPair, record, states, stateCov, status);
            continue;
        }
        const double jdFull = add_rn(jd[i], fr[i]), w = window[i];
        bool built = true, known = true;
        for (int o = 0; o < 2; ++o) {
            Row &r = rows[o];
            const uint32_t s = idx[o];
            r.deep = model ? model[s] : 0;
            known = known && r.deep <= 1;
            if (!known) break;
            for (int c = 0; c < 8; ++c) r.el[c] = elements[(size_t)c * n + s];
            std::memcpy(r.P, covariance + (size_t)s * kFitN, sizeof r.P);
            r.nvar = cov_nvar(r.P);
            r.ts0 = pairs_tsince_deep(jdFull, r.el[0]);
            double x[kFitVars];
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
        }
        if (!known || !built) {
            zero(i, kConjInitFailed, record, states, stateCov, status);
            continue;
        }
        HostSampler S{rows[0], rows[1], g};
        double tca = 0.0;
        uint8_t st = conj_tca(S, w, tca);
        double f[2][6], sig[2][kCovWords];
        bool ok = S.ok;
        for (int o = 0; o < 2 && ok; ++o) {
            const Row &r = rows[o];
            const double ts = r.ts0 + tca;
            auto eval = [&r, &g, ts](int k, double, const double (&)[1], double (&ff)[6]) { return r.eval(k, ts, g, ff); };
            double J[kCovJacWords];
            ok = cov_query(eval, r.nvar, r.inv, r.P, 0.0, 0.0, frame, J, 1, f[o], sig[o]) == kCovOk;
        }
        if (!ok) {
            zero(i, kConjCellFailed, record, states, stateCov, status);
            continue;
        }
        double *rec = record + (size_t)i * kConjRecordWords;
        ConjPc pc;
        if (conj_geometry(f[0], f[1], sig[0], sig[1], frame, hbr[i], rec, pc) == kConjNoPlane) st = kConjNoPlane;
        rec[0] = tca;
        rec[kConjRecPc] = emul_conj_pc(rec[kConjRecC2], rec[kConjRecC2 + 1], rec[kConjRecC2 + 2], pc.d, hbr[i]);
        if (st == kConjNoPlane) rec[kConjRecPc] = 0.0;
        if (states) std::memcpy(states + (size_t)i * 12, f, sizeof f);
        if (stateCov) std::memcpy(stateCov + (size_t)i * 2 * kCovWords, sig, sizeof sig);
        status[i] = st;
    }
    return 0;
}
