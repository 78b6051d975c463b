// TEST INFRASTRUCTURE ONLY: runs the observation fits of K8 (az_fit.cuh + az_obs.cuh, __host__ __device__) and the
// measurement model on the CPU, with the evaluation passes of fit_obs_kernel and fit_obs_deep_kernel (az_fit_obs.cu)
// restated serially: 32 lane partials over observations l, l + 32, ..., then the xor-butterfly over masks 16, 8, 4, 2,
// 1.  emul_fit_obs is astroz_cuda_fit_observations, emul_fit_obs_mixed the _mixed call, emul_observe
// astroz_cuda_observe.  Not part of the shipped library; nothing in astroz_b200/ references it.
#include <cmath>
#include <cstdint>
#include <cstring>

#include "az_obs.cuh"

using namespace az;

namespace {

struct Obs {
    int kind;
    double jdFull, value[6], w[6], sg, cg;
    ObsStation st;
};

struct Batch {
    const double *jd, *fr, *value, *sigma, *stations;
    const uint32_t *station;
    const uint8_t *kind;
};

int load(const Batch &b, uint32_t i, Obs &o) {
    o.kind = b.kind[i];
    o.jdFull = add_rn(b.jd[i], b.fr[i]);
    for (int c = 0; c < 6; ++c) o.value[c] = b.value[(size_t)i * 6 + c];
    const int used = obs_weights(o.kind, o.value, b.sigma + (size_t)i * 6, o.w);
    double llh[3] = {0.0, 0.0, 0.0};
    if (obs_uses_station(o.kind))
        for (int c = 0; c < 3; ++c) llh[c] = b.stations[(size_t)b.station[i] * 3 + c];
    obs_frame(o.kind, o.jdFull, llh, o.sg, o.cg, o.st);
    return used;
}

uint32_t residuals(const Batch &b, uint32_t begin, uint32_t end) {
    uint32_t used = 0;
    for (uint32_t i = begin; i < end; ++i) {
        Obs o;
        used += (uint32_t)load(b, i, o);
    }
    return used;
}

template <typename ObsFn>
bool lane_sums(uint32_t begin, uint32_t end, ObsFn obs, FitSums &sum) {
    static thread_local double lanes[32][kFitSumWords];
    std::memset(lanes, 0, sizeof lanes);
    double J[kFitVars * 6];
    bool ok = true;
    for (uint32_t lane = 0; lane < 32; ++lane)
        for (uint32_t i = begin + lane; i < end; i += 32) ok = obs(i, J, lanes[lane]) && ok;
    if (!ok) return false;
    for (int m = 16; m > 0; m >>= 1) {
        double next[32][kFitSumWords];
        for (int l = 0; l < 32; ++l)
            for (int q = 0; q < kFitSumWords; ++q) next[l][q] = lanes[l][q] + lanes[l ^ m][q];
        std::memcpy(lanes, next, sizeof lanes);
    }
    std::memcpy(fit_words(sum), lanes[0], sizeof lanes[0]);
    return true;
}

TleRecord record(const double *el0) {
    TleRecord t;
    t.epochJd = el0[0]; t.revPerDay = el0[1]; t.ecc = el0[2]; t.inclDeg = el0[3];
    t.raanDeg = el0[4]; t.argpDeg = el0[5]; t.maDeg = el0[6]; t.bstar = el0[7];
    return t;
}

struct Out {
    double *fitted, *wrms, *cov;
    uint32_t *nRes, *iters;
    uint8_t *status;
};

template <typename Model, typename PassFn>
void run(const double *el0, const Gravity &gr, int fitBstar, uint32_t maxIter, uint32_t nRes, PassFn pass, uint32_t n,
         uint32_t s, const Out &o) {
    const int nvar = fitBstar ? kFitVars : kFitVars - 1;
    FitResult r;
    FitSums fin = {};
    bool fitted = false;
    auto final = [&](const FitSums &sums) {
        fin = sums;
        fitted = true;
    };
    fit_satellite_run(el0, gr, fitBstar != 0, maxIter, nRes, pass, final, r, Model{});
    double cov[kFitN] = {};
    if (fitted) fit_covariance(fin, nvar, cov);
    for (int c = 0; c < 8; ++c) o.fitted[(size_t)c * n + s] = r.el[c];
    std::memcpy(o.cov + (size_t)s * kFitN, cov, sizeof cov);
    o.wrms[s] = fitted && nRes ? std::sqrt(fin.F / nRes) : 0.0;
    o.nRes[s] = nRes;
    o.iters[s] = r.iters;
    o.status[s] = r.status;
}

}  // namespace

extern "C" int emul_fit_obs(const double *elements, uint32_t n, int grav, const uint32_t *offsets, const double *jd,
                            const double *fr, const double *value, const double *sigma, const uint32_t *station,
                            const uint8_t *kind, const double *stations, int fitBstar, uint32_t maxIter,
                            double *fitted, double *wrms, uint32_t *nResiduals, double *covariance,
                            uint32_t *iterations, uint8_t *status) {
    const Gravity gr = gravity(grav);
    const GravConsts g = grav_consts(gr);
    const int nvar = fitBstar ? kFitVars : kFitVars - 1;
    const Batch b{jd, fr, value, sigma, stations, station, kind};
    const Out out{fitted, wrms, covariance, nResiduals, iterations, status};
    for (uint32_t s = 0; s < n; ++s) {
        double el0[8];
        for (int c = 0; c < 8; ++c) el0[c] = elements[(size_t)c * n + s];
        const uint32_t begin = offsets[s], end = offsets[s + 1];
        auto pass = [&](const double (&x)[kFitVars], FitSums &sum) -> bool {
            double sets[kFitSets][kSgp4Cols], inv[kFitSets];
            for (int k = 0; k <= nvar; ++k)
                if (!fit_build_set(x, k, el0[0], gr, sets[k], inv[k])) return false;
            auto eval = [&](int k, double, const double (&ts)[1], double (&f)[6]) {
                CellOut o[1];
                sgp4_cell<1>([&sets, k](int c) { return sets[k][c]; }, ts, g, o);
                f[0] = o[0].rx; f[1] = o[0].ry; f[2] = o[0].rz;
                f[3] = o[0].vx; f[4] = o[0].vy; f[5] = o[0].vz;
                return true;
            };
            return lane_sums(begin, end, [&](uint32_t i, double *J, double *acc) {
                Obs o;
                load(b, i, o);
                fit_accumulate_obs(eval, nvar, inv, o.jdFull, el0[0], o.kind, o.value, o.w, o.sg, o.cg, o.st, J,
                                   acc, 1);
                return true;
            }, sum);
        };
        run<FitNearEarth>(el0, gr, fitBstar, maxIter, residuals(b, begin, end), pass, n, s, out);
    }
    return 0;
}

extern "C" int emul_fit_obs_mixed(const double *elements, uint32_t n, int grav, const uint32_t *offsets,
                                  const double *jd, const double *fr, const double *value, const double *sigma,
                                  const uint32_t *station, const uint8_t *kind, const double *stations, int fitBstar,
                                  uint32_t maxIter, double *fitted, double *wrms, uint32_t *nResiduals,
                                  double *covariance, uint32_t *iterations, uint8_t *status) {
    emul_fit_obs(elements, n, grav, offsets, jd, fr, value, sigma, station, kind, stations, fitBstar, maxIter, fitted,
                 wrms, nResiduals, covariance, iterations, status);
    const Gravity gr = gravity(grav);
    const GravConsts g = grav_consts(gr);
    const int nvar = fitBstar ? kFitVars : kFitVars - 1;
    const Batch b{jd, fr, value, sigma, stations, station, kind};
    const Out out{fitted, wrms, covariance, nResiduals, iterations, status};
    for (uint32_t s = 0; s < n; ++s) {
        double el0[8];
        for (int c = 0; c < 8; ++c) el0[c] = elements[(size_t)c * n + s];
        {
            NearEarth ne;
            if (build_near_earth(record(el0), gr, ne) != kDeepSpace) continue;
        }
        const uint32_t begin = offsets[s], end = offsets[s + 1];
        int nodes[2];
        {
            double fwd = 0.0, bwd = 0.0;
            for (uint32_t i = begin; i < end; ++i) {
                const double ts = pairs_tsince_deep(add_rn(jd[i], fr[i]), el0[0]);
                if (ts > 0.0) fwd = std::fmax(fwd, ts);
                else bwd = std::fmax(bwd, -ts);
            }
            nodes[0] = fit_lattice_nodes(fwd);
            nodes[1] = fit_lattice_nodes(bwd);
        }
        auto pass = [&](const double (&x)[kFitVars], FitSums &sum) -> bool {
            Sdp4Sat sets[kFitSets];
            double2 lattice[kFitSets][2 * kFitLatticeNodes];
            double inv[kFitSets];
            for (int k = 0; k <= nvar; ++k)
                if (!fit_build_set_of<FitDeepSpace>(x, k, el0[0], gr, sets[k], inv[k])) return false;
            for (int k = 0; k <= nvar; ++k)
                for (int dir = 0; dir < 2; ++dir) fit_deep_lattice(sets[k], dir, nodes[dir], lattice[k]);
            auto eval = [&](int k, double jdFull, const double (&)[1], double (&f)[6]) {
                return fit_deep_eval(sets[k], lattice[k], jdFull, g, f);
            };
            return lane_sums(begin, end, [&](uint32_t i, double *J, double *acc) {
                Obs o;
                load(b, i, o);
                return fit_accumulate_obs(eval, nvar, inv, o.jdFull, el0[0], o.kind, o.value, o.w, o.sg, o.cg, o.st,
                                          J, acc, 1);
            }, sum);
        };
        run<FitDeepSpace>(el0, gr, fitBstar, maxIter, residuals(b, begin, end), pass, n, s, out);
    }
    return 0;
}

extern "C" int emul_observe(const double *states, const double *jd, const double *fr, const uint8_t *kind,
                            const uint32_t *station, uint32_t m, const double *stations, double *values) {
    for (uint32_t i = 0; i < m; ++i) {
        double f[6], h[6], sc[6], llh[3] = {0.0, 0.0, 0.0};
        for (int c = 0; c < 6; ++c) f[c] = states[(size_t)i * 6 + c];
        if (obs_uses_station(kind[i]))
            for (int c = 0; c < 3; ++c) llh[c] = stations[(size_t)station[i] * 3 + c];
        double sg, cg;
        ObsStation st;
        obs_frame(kind[i], add_rn(jd[i], fr[i]), llh, sg, cg, st);
        obs_model(kind[i], f, sg, cg, st, h, sc);
        std::memcpy(values + (size_t)i * 6, h, sizeof h);
    }
    return 0;
}

// The cost, floor and sums one observation batch adds under the element set el (near-earth, fit_bstar): the words of
// FitSums after a pass (F, pos2, vel2, floor, N[28], g[7]) and the used residual count.  For the sigma = inf checks.
extern "C" int emul_obs_sums(const double *el, int grav, uint32_t m, const double *jd, const double *fr,
                             const double *value, const double *sigma, const uint32_t *station, const uint8_t *kind,
                             const double *stations, double *words, uint32_t *nResiduals) {
    const Gravity gr = gravity(grav);
    const GravConsts g = grav_consts(gr);
    const Batch b{jd, fr, value, sigma, stations, station, kind};
    double x[kFitVars];
    fit_vars_of(el, x);
    double sets[kFitSets][kSgp4Cols], inv[kFitSets];
    for (int k = 0; k < kFitSets; ++k)
        if (!fit_build_set(x, k, el[0], gr, sets[k], inv[k])) return -1;
    auto eval = [&](int k, double, const double (&ts)[1], double (&f)[6]) {
        CellOut o[1];
        sgp4_cell<1>([&sets, k](int c) { return sets[k][c]; }, ts, g, o);
        f[0] = o[0].rx; f[1] = o[0].ry; f[2] = o[0].rz;
        f[3] = o[0].vx; f[4] = o[0].vy; f[5] = o[0].vz;
        return true;
    };
    FitSums sum = {};
    lane_sums(0, m, [&](uint32_t i, double *J, double *acc) {
        Obs o;
        load(b, i, o);
        return fit_accumulate_obs(eval, kFitVars, inv, o.jdFull, el[0], o.kind, o.value, o.w, o.sg, o.cg, o.st, J,
                                  acc, 1);
    }, sum);
    std::memcpy(words, fit_words(sum), sizeof sum);
    *nResiduals = residuals(b, 0, m);
    return 0;
}

// station (lat deg, lon deg, h km) -> ECEF, and ecef_to_geodetic of it (lat, lon rad, h km): the round trip
extern "C" void emul_station(const double *llh, double *ecef, double *back) {
    ObsStation st;
    obs_station(llh, st);
    double x = st.r[0], y = st.r[1], z = st.r[2];
    std::memcpy(ecef, st.r, sizeof st.r);
    ecef_to_geodetic(x, y, z);
    back[0] = x;
    back[1] = y;
    back[2] = z;
}

// fit_accumulate_obs for one observation against given TEME states: f[k][6] is the state of set k (k = 0 nominal,
// 1 .. nvar the stepped sets), inv[1 + j] the inverse steps.  words receives the FitSums words.  For the wrap checks.
extern "C" void emul_obs_accumulate(int kind, const double *f, int nvar, const double *inv, double jdFull,
                                    const double *value, const double *sigma, const double *llh, double *words) {
    auto eval = [&](int k, double, const double (&)[1], double (&out)[6]) {
        for (int c = 0; c < 6; ++c) out[c] = f[6 * k + c];
        return true;
    };
    double w[6], sg, cg, J[kFitVars * 6];
    ObsStation st;
    obs_weights(kind, value, sigma, w);
    obs_frame(kind, jdFull, llh, sg, cg, st);
    FitSums sum = {};
    fit_accumulate_obs(eval, nvar, inv, jdFull, jdFull, kind, value, w, sg, cg, st, J, fit_words(sum), 1);
    std::memcpy(words, fit_words(sum), sizeof sum);
}
