// TEST INFRASTRUCTURE ONLY: runs K14 (az_conjunction_mc.cuh, __host__ __device__) on the CPU with the warp of
// conjunction_mc_kernel / conjunction_mc_deep_kernel (az_conjunction_mc.cu) restated serially: each sample's two sets
// drawn and built one after the other, the 32 samples of a search round in a loop returning the same mask.
// emul_conjunction_mc is astroz_cuda_conjunction_mc_device's definition on host buffers; emul_philox, emul_normals,
// emul_factor and emul_draw expose the generator, the factor and the draws.  Not part of the shipped library; nothing
// in astroz_b200/ references it.
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>

#include "az_conjunction_mc.cuh"

using namespace az;

namespace {

struct Row {
    int deep = 0;
    double el[8], xh[kFitVars], ts0 = 0.0;
    McFactor F;
    double cols[kSgp4Cols];
    Sdp4Sat set;
    double2 lattice[2 * kFitLatticeNodes];

    bool eval(double ts, const GravConsts &g, double (&f)[6]) const {
        if (!deep) return conj_eval_near([this](int c) { return cols[c]; }, ts, g, f);
        return conj_eval_deep(set, lattice, ts, g, f);
    }
    // the set of x; false when it cannot be built
    bool build(const double (&x)[kFitVars], const Gravity &gr, double w) {
        double inv;
        if (!deep) return fit_build_set_of<FitNearEarth>(x, 0, el[0], gr, cols, inv);
        if (!fit_build_set_of<FitDeepSpace>(x, 0, el[0], gr, set, inv)) return false;
        const double hi = ts0 + w, lo = ts0 - w;
        const int nodes[2] = {fit_lattice_nodes(hi > 0.0 ? hi : 0.0), fit_lattice_nodes(lo < 0.0 ? -lo : 0.0)};
        for (int dir = 0; dir < 2; ++dir) fit_deep_lattice(set, dir, nodes[dir], lattice);
        return true;
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
            ok = p.eval(p.ts0 + t, gc, fp) && ok;
            ok = s.eval(s.ts0 + t, gc, fs) && ok;
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

}  // namespace

extern "C" void emul_philox(const uint32_t *ctr, const uint32_t *key, uint32_t n, uint32_t *out) {
    for (uint32_t i = 0; i < n; ++i) {
        const McU4 o = mc_philox(McU4{ctr[4 * i], ctr[4 * i + 1], ctr[4 * i + 2], ctr[4 * i + 3]}, key[2 * i],
                                 key[2 * i + 1]);
        out[4 * i] = o.x;
        out[4 * i + 1] = o.y;
        out[4 * i + 2] = o.z;
        out[4 * i + 3] = o.w;
    }
}

// the 14 normals of samples k[0 .. n) under seed: z[n][14]
extern "C" void emul_normals(uint64_t seed, const uint64_t *k, uint32_t n, double *z) {
    for (uint32_t i = 0; i < n; ++i)
        for (int o = 0; o < 2; ++o) {
            double r[kFitVars];
            mc_row_normals(seed, k[i], o, r);
            for (int v = 0; v < kFitVars; ++v) z[14 * i + kFitVars * o + v] = r[v];
        }
}

// the factor of P's words over cov_nvar(P) variables: sd[7], L[7][7] (dense, lower); 1 when positive semidefinite
extern "C" int emul_factor(const double *P, double *sd, double *L) {
    McFactor F;
    const int ok = mc_factor(P, cov_nvar(P), F) ? 1 : 0;
    for (int a = 0; a < kFitVars; ++a) {
        sd[a] = F.sd[a];
        for (int b = 0; b < kFitVars; ++b) L[a * kFitVars + b] = b <= a ? F.L[fit_tri(b, a)] : 0.0;
    }
    return ok;
}

// the drawn variables of row o (element columns el[8], model, P words) for samples k[0 .. n): x[n][7]; the status
extern "C" int emul_draw(const double *el, int model, const double *P, uint64_t seed, int o, const uint64_t *k,
                         uint32_t n, double *x, int grav) {
    double e[8], xh[kFitVars];
    std::memcpy(e, el, sizeof e);
    McFactor F;
    const uint8_t st = mc_row(e, P, model, gravity(grav), xh, F);
    if (st != kConjOk) return st;
    for (uint32_t i = 0; i < n; ++i) {
        double z[kFitVars], xs[kFitVars];
        mc_row_normals(seed, k[i], o, z);
        mc_draw(F, xh, z, xs);
        std::memcpy(x + (size_t)kFitVars * i, xs, sizeof xs);
    }
    return st;
}

extern "C" int emul_conjunction_mc(const double *elements, uint32_t n, int grav, const double *covariance,
                                   const uint8_t *model, const uint32_t *primary, const uint32_t *secondary,
                                   const double *jd, const double *fr, const double *window, const double *hbr,
                                   const uint64_t *samples, const uint64_t *first, const uint64_t *seed, uint32_t m,
                                   uint32_t record, uint64_t *counts, double *sampleOut, uint8_t *status) {
    const Gravity gr = gravity(grav);
    const GravConsts g = grav_consts(gr);
    const double nan = std::numeric_limits<double>::quiet_NaN();
    static Row rows[2];
    for (uint32_t i = 0; i < m; ++i) {
        uint64_t *cnt = counts + (size_t)i * kMcCountWords;
        cnt[0] = cnt[1] = cnt[2] = 0;
        for (size_t q = 0; q < (size_t)record * kMcSampleWords; ++q) sampleOut[(size_t)i * record * kMcSampleWords + q] = nan;
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
        const uint64_t f0 = first ? first[i] : 0, sd = seed ? seed[i] : 0;
        for (uint64_t j = 0; j < samples[i]; ++j) {
            bool built = true;
            for (int o = 0; o < 2; ++o) {
                double z[kFitVars], x[kFitVars];
                mc_row_normals(sd, f0 + j, o, z);
                mc_draw(rows[o].F, rows[o].xh, z, x);
                built = rows[o].build(x, gr, w) && built;
            }
            double out0 = nan, out1 = nan;
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
                } else {
                    ++cnt[2];
                }
            } else {
                ++cnt[2];
            }
            if (j < record) {
                sampleOut[((size_t)i * record + j) * kMcSampleWords] = out0;
                sampleOut[((size_t)i * record + j) * kMcSampleWords + 1] = out1;
            }
        }
    }
    return 0;
}
