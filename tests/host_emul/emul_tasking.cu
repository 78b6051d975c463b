// TEST INFRASTRUCTURE ONLY: runs K18 (az_tasking.cuh, __host__ __device__) on the CPU: every row's sets built once,
// every (row, slot) scored by task_score against every sensor, and the greedy picks and posteriors of the definition.
// emul_tasking is astroz_cuda_tasking_device's definition on host buffers; emul_task_slot scores one slot under given
// covariances (gains, cell words, nominal states, visibility masks) for the brute-force statement of the schedule;
// emul_task_update is the gain / spread / posterior of one cell.  Not part of the shipped library; nothing in
// astroz_b200/ references it.
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#include "az_tasking.cuh"

using namespace az;

namespace {

struct Row {
    int deep = 0, nvar = -1;   // -1: not built
    double el[8], inv[kFitSets] = {};
    double cols[kFitSets][kSgp4Cols];
    Sdp4Sat sets[kFitSets];
    double2 lattice[kFitSets][2 * kFitLatticeNodes];
};

bool build_row(Row &r, const double *elements, uint32_t n, const double *covariance, const uint8_t *model,
               const Gravity &gr, uint32_t s) {
    const uint8_t md = model ? model[s] : 0;
    double P[kFitN];
    for (int c = 0; c < 8; ++c) r.el[c] = elements[(size_t)c * n + s];
    for (int q = 0; q < kFitN; ++q) P[q] = covariance ? covariance[(size_t)s * kFitN + q] : 0.0;
    r.deep = md == 1;
    r.nvar = -1;
    if (md > 1) return false;
    const int nvar = corr_nvar(P);
    double x[kFitVars];
    bool built = true;
    if (!r.deep) {
        FitNearEarth::vars_of(r.el, x);
        for (int k = 0; k <= nvar && built; ++k) built = fit_build_set(x, k, r.el[0], gr, r.cols[k], r.inv[k]);
    } else {
        FitDeepSpace::vars_of(r.el, x);
        for (int k = 0; k <= nvar && built; ++k)
            built = fit_build_set_of<FitDeepSpace>(x, k, r.el[0], gr, r.sets[k], r.inv[k]);
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

struct Scene {
    Gravity gr;
    GravConsts g;
    std::vector<Row> rows;
    std::vector<TaskSensor> sensors;
};

void scene(Scene &sc, const double *elements, uint32_t n, int grav, const double *covariance, const uint8_t *model,
           const uint8_t *kind, const uint32_t *station, const double *sigma, const double *limits, uint32_t S,
           const double *stations, uint8_t *rowStatus) {
    sc.gr = gravity(grav);
    sc.g = grav_consts(sc.gr);
    sc.rows.resize(n);
    for (uint32_t s = 0; s < n; ++s) {
        const bool ok = build_row(sc.rows[s], elements, n, covariance, model, sc.gr, s);
        if (rowStatus) rowStatus[s] = ok ? kCovOk : kCovInitFailed;
    }
    sc.sensors.resize(S);
    for (uint32_t k = 0; k < S; ++k) task_sensor(kind, station, stations, sigma, limits, (int)k, sc.sensors[k]);
}

// Slot t under covariances P[n][28]: gain[S][n] (NaN: not visible), cell[S][n][kTaskCellWords], visible[n] masks,
// failed[n] cells, f0[n][6] nominal states (nullable)
void score_slot(const Scene &sc, uint32_t n, uint32_t S, double jdFull, const double *sun, const double *P,
                double *gain, double *cell, uint32_t *visible, uint32_t *failed, double *f0) {
    double u[3] = {0.0, 0.0, 0.0};
    if (sun) task_sun(sun, u);
    for (uint32_t s = 0; s < n; ++s) {
        for (uint32_t k = 0; k < S; ++k) gain[(size_t)k * n + s] = NAN;
        visible[s] = failed[s] = 0;
        const Row &r = sc.rows[s];
        if (r.nvar < 0) continue;
        with_eval(r, sc.g, [&](auto eval) {
            if (f0) {
                const double ts[1] = {mul_rn(sub_rn(jdFull, r.el[0]), 1440.0)};
                double f[6];
                for (int c = 0; c < 6; ++c) f[c] = NAN;
                eval(0, jdFull, ts, f);
                std::memcpy(f0 + (size_t)s * 6, f, sizeof f);
            }
            visible[s] = task_score(
                eval, r.nvar, r.inv, r.el[0], jdFull, sc.sensors.data(), (int)S, u, P + (size_t)s * kFitN,
                [&](int k, double g, const double (&h)[6], const double (&spread)[4],
                    const double (&G)[4][kFitVars]) {
                    double *c = cell + ((size_t)k * n + s) * kTaskCellWords;
                    for (int q = 0; q < 4; ++q) {
                        c[q] = h[q];
                        c[4 + q] = spread[q];
                    }
                    for (int q = 0; q < 4; ++q)
                        for (int j = 0; j < kFitVars; ++j) c[8 + q * kFitVars + j] = G[q][j];
                    gain[(size_t)k * n + s] = g;
                },
                failed[s]);
            return 0;
        });
    }
}

}  // namespace

extern "C" size_t emul_task_scratch_bytes(uint32_t n, uint32_t S) { return task_scratch_bytes(n, S); }

extern "C" int emul_tasking(const double *elements, uint32_t n, int grav, const double *covariance,
                            const uint8_t *model, const uint8_t *kind, const uint32_t *station, const double *sigma,
                            const double *limits, uint32_t S, const double *stations, const double *jd,
                            const double *fr, uint32_t T, const double *sun, double gainMin, uint32_t *taskRow,
                            double *taskGain, double *taskValue, double *taskSpread, uint32_t *nCandidates,
                            double *posterior, uint32_t *nTasks, uint32_t *nVisible, uint32_t *nFailed,
                            uint8_t *rowStatus) {
    Scene sc;
    scene(sc, elements, n, grav, covariance, model, kind, station, sigma, limits, S, stations, rowStatus);
    for (uint32_t s = 0; s < n; ++s) {
        for (int q = 0; q < kFitN; ++q)
            posterior[(size_t)s * kFitN + q] = covariance ? covariance[(size_t)s * kFitN + q] : 0.0;
        nTasks[s] = nVisible[s] = nFailed[s] = 0;
    }
    std::vector<double> gain((size_t)S * n), cell((size_t)S * n * kTaskCellWords);
    std::vector<uint32_t> vis(n), fail(n), taken(n, kTaskIdle);
    for (uint32_t t = 0; t < T; ++t) {
        score_slot(sc, n, S, add_rn(jd[t], fr[t]), sun ? sun + (size_t)t * 3 : nullptr, posterior, gain.data(),
                   cell.data(), vis.data(), fail.data(), nullptr);
        for (uint32_t s = 0; s < n; ++s) {
            for (uint32_t b = vis[s]; b; b &= b - 1) ++nVisible[s];
            nFailed[s] += fail[s];
        }
        std::vector<uint32_t> picks(S, kTaskIdle);
        for (uint32_t k = 0; k < S; ++k) {
            double bg = -INFINITY;
            uint32_t br = kTaskIdle, cnt = 0;
            for (uint32_t s = 0; s < n; ++s) {
                const double g = gain[(size_t)k * n + s];
                if (!(g > gainMin) || taken[s] == t) continue;
                ++cnt;
                if (g > bg || (g == bg && s < br)) {
                    bg = g;
                    br = s;
                }
            }
            const size_t o = (size_t)k * T + t;
            taskRow[o] = br;
            nCandidates[o] = cnt;
            taskGain[o] = br == kTaskIdle ? 0.0 : bg;
            for (int q = 0; q < 4; ++q) {
                taskValue[o * 4 + q] = br == kTaskIdle ? 0.0 : cell[((size_t)k * n + br) * kTaskCellWords + q];
                taskSpread[o * 4 + q] = br == kTaskIdle ? 0.0 : cell[((size_t)k * n + br) * kTaskCellWords + 4 + q];
            }
            if (br != kTaskIdle) taken[br] = t;
            picks[k] = br;
        }
        for (uint32_t k = 0; k < S; ++k) {
            const uint32_t s = picks[k];
            if (s == kTaskIdle) continue;
            const double *c = cell.data() + ((size_t)k * n + s) * kTaskCellWords;
            double G[4][kFitVars], L[kFitVars][kFitVars], g, spread[4];
            for (int q = 0; q < 4; ++q)
                for (int j = 0; j < kFitVars; ++j) G[q][j] = c[8 + q * kFitVars + j];
            task_cholesky(posterior + (size_t)s * kFitN, L);
            task_update(G, L, sc.sensors[k].sigma, g, spread, posterior + (size_t)s * kFitN);
            ++nTasks[s];
        }
    }
    return 0;
}

// One slot under covariances P[n][28] (the brute-force statement's per-cell function)
extern "C" int emul_task_slot(const double *elements, uint32_t n, int grav, const double *covariance,
                              const uint8_t *model, const uint8_t *kind, const uint32_t *station,
                              const double *sigma, const double *limits, uint32_t S, const double *stations,
                              double jd, double fr, const double *sun, const double *P, double *gain, double *cell,
                              uint32_t *visible, uint32_t *failed, double *f0, uint8_t *rowStatus) {
    Scene sc;
    scene(sc, elements, n, grav, covariance, model, kind, station, sigma, limits, S, stations, rowStatus);
    score_slot(sc, n, S, add_rn(jd, fr), sun, P, gain, cell, visible, failed, f0);
    return 0;
}

// The gain, spread and posterior of one cell: G[4][7] weighted rows, P[28], sigma[4]; returns 0, or -1 on failure
extern "C" int emul_task_update(const double *G, const double *P, const double *sigma, double *gain, double *spread,
                                double *Pplus) {
    double Gm[4][kFitVars], L[kFitVars][kFitVars], sp[4], sg[6];
    for (int q = 0; q < 4; ++q)
        for (int j = 0; j < kFitVars; ++j) Gm[q][j] = G[q * kFitVars + j];
    for (int c = 0; c < 6; ++c) sg[c] = c < 4 ? sigma[c] : INFINITY;
    task_cholesky(P, L);
    const bool ok = task_update(Gm, L, sg, *gain, sp, Pplus);
    std::memcpy(spread, sp, sizeof sp);
    return ok ? 0 : -1;
}
