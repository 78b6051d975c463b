// TEST INFRASTRUCTURE ONLY: runs K13 (az_iod.cuh, __host__ __device__) on the CPU.  emul_iod is
// astroz_cuda_initial_orbits_device's definition on host buffers: each track's summary, every generator slot built and
// scored by iod_slot (the winner is the least (F, key), so the order the lanes visit the slots in does not matter), the
// winner carried to the epoch, then the conversion by emul_fit_mixed (emul_fit.cu and emul_fit_deep.cu, linked into the
// same library) and iod_final_status.  The other entries expose the methods one at a time.  Not part of the shipped
// library; nothing in astroz_b200/ references it.
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#include "az_iod.cuh"

using namespace az;

extern "C" int emul_fit_mixed(const double *elements, uint32_t n, int grav, const uint32_t *offsets, const double *jd,
                              const double *fr, const double *pos, const double *vel, double posSigma, double velSigma,
                              int fitBstar, uint32_t maxIter, double *fitted, double *rms, uint32_t *iterations,
                              uint8_t *status);

// init[8][t] (nullable) receives the osculating initial sets, fitStatus[t] (nullable) the conversion fit's status
extern "C" int emul_iod(const uint32_t *offsets, uint32_t t, const double *jd, const double *fr, const uint8_t *kind,
                        const double *value, const double *sigma, const uint32_t *station, const double *stations,
                        const double *bstar, int grav, double *elements, double *state, double *wrms, uint8_t *method,
                        uint32_t *candidates, double *conv, uint8_t *deep, uint8_t *status, double *init,
                        uint8_t *fitStatusOut) {
    const Gravity gr = gravity(grav);
    const CorrObsArrays in{jd, fr, kind, value, sigma, station, stations};
    std::vector<double> el0((size_t)8 * t), fjd(t), ffr(t), pos((size_t)3 * t), vel((size_t)3 * t), rms((size_t)2 * t);
    std::vector<uint32_t> off(t + 1), iters(t);
    std::vector<uint8_t> iod(t), fit(t);
    for (uint32_t j = 0; j < t; ++j) {
        IodTrack tr;
        iod_track(in, offsets[j], offsets[j + 1], tr);
        IodBest best;
        iod_best_init(best);
        uint32_t scored = 0;
        if (tr.status == kIodOk)
            for (uint32_t g = 0, slots = iod_slots(tr); g < slots; ++g)
                scored += iod_slot(in, tr, g, gr.mu, gr.radiusEarthKm, best);
        uint8_t st = tr.status;
        double s[6] = {0, 0, 0, 0, 0, 0}, el[8] = {0, 0, -1.0, 0, 0, 0, 0, 0};
        uint8_t dp = 0;
        if (st == kIodOk) {
            if (!(best.F < INFINITY)) st = kIodNoCandidate;
            else if (!iod_epoch_state(best, tr.epoch, gr.mu, bstar ? bstar[j] : 0.0, gr, s, el, dp)) st = kIodNoCandidate;
        }
        if (st != kIodOk) {
            for (int c = 0; c < 6; ++c) s[c] = 0.0;
            for (int c = 0; c < 8; ++c) el[c] = c == 2 ? -1.0 : 0.0;
            dp = 0;
        }
        const bool ok = st == kIodOk;
        const uint32_t mid = tr.begin + (tr.end - tr.begin) / 2;
        for (int c = 0; c < 8; ++c) el0[(size_t)c * t + j] = el[c];
        fjd[j] = ok ? jd[mid] : 0.0;
        ffr[j] = ok ? fr[mid] : 0.0;
        for (int c = 0; c < 3; ++c) pos[3 * j + c] = s[c], vel[3 * j + c] = s[3 + c];
        off[j] = j;
        iod[j] = st;
        for (int c = 0; c < 6; ++c) state[(size_t)j * 6 + c] = s[c];
        wrms[j] = ok ? std::sqrt(best.F / tr.used) : 0.0;
        method[j] = ok ? (uint8_t)(best.key >> 16) : kIodNone;
        candidates[j] = scored;
        deep[j] = dp;
    }
    off[t] = t;
    if (init) std::memcpy(init, el0.data(), sizeof(double) * 8 * t);
    if (t)
        emul_fit_mixed(el0.data(), t, grav, off.data(), fjd.data(), ffr.data(), pos.data(), vel.data(), kIodFitPosSigma,
                       kIodFitVelSigma, 0, kIodFitIter, elements, rms.data(), iters.data(), fit.data());
    for (uint32_t j = 0; j < t; ++j) {
        status[j] = iod_final_status(iod[j], fit[j], rms[2 * j], rms[2 * j + 1]);
        conv[2 * j] = iod[j] == kIodOk ? rms[2 * j] : 0.0;
        conv[2 * j + 1] = iod[j] == kIodOk ? rms[2 * j + 1] : 0.0;
        if (iod[j] != kIodOk)
            for (int c = 0; c < 8; ++c) elements[(size_t)c * t + j] = 0.0;
        if (fitStatusOut) fitStatusOut[j] = fit[j];
    }
    return 0;
}

extern "C" int emul_iod_kepler(const double *s0, double dt, double mu, double *s) {
    return iod_kepler(s0, s0 + 3, dt, mu, s, s + 3) ? 0 : -1;
}
extern "C" void emul_iod_gibbs(const double *r1, const double *r2, const double *r3, double mu, double *v2) {
    iod_gibbs(r1, r2, r3, mu, v2);
}
extern "C" void emul_iod_herrick_gibbs(const double *r1, const double *r2, const double *r3, double t1, double t2,
                                       double t3, double mu, double *v2) {
    iod_herrick_gibbs(r1, r2, r3, t1, t2, t3, mu, v2);
}
extern "C" void emul_iod_coe(const double *s, double mu, double epochJd, double bstar, double *el) {
    double e[8];
    iod_coe(s, mu, epochJd, bstar, e);
    std::memcpy(el, e, sizeof e);
}
extern "C" int emul_iod_admissible(const double *s, double mu, double rE) { return iod_admissible(s, mu, rE); }
// Gauss on one triplet: L[3][3], R[3][3], t[3] seconds; states[3][6] and roots[3] of the refined candidates, in root
// order.  Returns the octic's root count above rE; *refined the candidates emitted.
extern "C" int emul_iod_gauss(const double *L, const double *R, const double *t, double mu, double rE, double *states,
                              int *roots, int *refined) {
    double Lm[3][3], Rm[3][3], tm[3];
    std::memcpy(Lm, L, sizeof Lm);
    std::memcpy(Rm, R, sizeof Rm);
    std::memcpy(tm, t, sizeof tm);
    int n = 0;
    const int nr = iod_gauss(Lm, Rm, tm, mu, rE, [&](const double (&s)[6], int root) {
        std::memcpy(states + 6 * n, s, sizeof s);
        roots[n++] = root;
    });
    *refined = n;
    return nr;
}
extern "C" int emul_iod_octic_roots(double a, double b, double c, double rE, double *roots) {
    double r[3];
    const int n = iod_octic_roots(a, b, c, rE, r);
    std::memcpy(roots, r, sizeof(double) * n);
    return n;
}
extern "C" int emul_iod_triplet(int q, uint32_t c, uint32_t *ix) {
    uint32_t x[3];
    if (!iod_triplet(q, c, x)) return 0;
    std::memcpy(ix, x, sizeof x);
    return 1;
}
