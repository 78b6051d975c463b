// TEST INFRASTRUCTURE ONLY: runs K17 (az_link.cuh, __host__ __device__) on the CPU.  emul_link is
// astroz_cuda_link_tracks_device's definition on host buffers: each pair's summary, every cell solved and scored into
// one seed list (the seeds are the least (F_probe, key), so the order the lanes visit the cells in does not matter),
// each seed refined, the least (F, key) converted by emul_fit_mixed (emul_fit.cu and emul_fit_deep.cu, linked into the
// same library) and iod_final_status.  The other entries expose the anchors, the probe scores and the seeds.  Not part of
// the shipped library; nothing in astroz_b200/ references it.
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#include "az_link.cuh"

using namespace az;

extern "C" int emul_fit_mixed(const double *elements, uint32_t n, int grav, const uint32_t *offsets, const double *jd,
                              const double *fr, const double *pos, const double *vel, double posSigma, double velSigma,
                              int fitBstar, uint32_t maxIter, double *fitted, double *rms, uint32_t *iterations,
                              uint8_t *status);

static CorrObsArrays arrays(const double *jd, const double *fr, const uint8_t *kind, const double *value,
                            const double *sigma, const uint32_t *station, const double *stations) {
    return CorrObsArrays{jd, fr, kind, value, sigma, station, stations};
}

// seedF / seedKey [p][kLinkSeeds] (nullable) receive each pair's seeds, converged[p] (nullable) whether the winner's
// refinement ended on its step tolerance
extern "C" int emul_link(const uint32_t *offsets, uint32_t t, const double *jd, const double *fr, const uint8_t *kind,
                         const double *value, const double *sigma, const uint32_t *station, const double *stations,
                         const uint32_t *pairs, uint32_t p, const double *bstar, double rMin, double rMax,
                         uint32_t maxRevs, int grav, double *elements, double *state, double *rho, uint8_t *revs,
                         uint8_t *flags, double *wrms, uint32_t *used, uint32_t *hypotheses, double *conv,
                         uint8_t *deep, uint8_t *status, double *seedF, uint32_t *seedKey, uint8_t *converged) {
    const Gravity gr = gravity(grav);
    const CorrObsArrays in = arrays(jd, fr, kind, value, sigma, station, stations);
    std::vector<double> el0((size_t)8 * p), fjd(p), ffr(p), pos((size_t)3 * p), vel((size_t)3 * p), rms((size_t)2 * p);
    std::vector<uint32_t> off(p + 1), iters(p);
    std::vector<uint8_t> st0(p), fit(p);
    for (uint32_t j = 0; j < p; ++j) {
        LinkPair pr;
        link_pair(in, offsets, t, pairs[2 * j], pairs[2 * j + 1], rMin, rMax, pr);
        LinkSeeds seeds;
        link_seeds_init(seeds);
        uint32_t scored = 0;
        if (pr.status == kLinkOk)
            for (uint32_t c = 0, cells = link_cells(pr); c < cells; ++c)
                scored += link_cell(in, pr, c, maxRevs, gr.mu, gr.radiusEarthKm, seeds);
        LinkBest best;
        link_best_init(best);
        for (int q = 0; q < kLinkSeeds; ++q) {
            if (seedF) seedF[(size_t)j * kLinkSeeds + q] = seeds.F[q];
            if (seedKey) seedKey[(size_t)j * kLinkSeeds + q] = seeds.key[q];
            if (!(seeds.F[q] < INFINITY)) continue;
            LinkBest w;
            link_refine(in, pr, seeds.key[q], gr.mu, gr.radiusEarthKm, w);
            if (iod_better(w.F, w.key, best.F, best.key)) best = w;
        }
        uint8_t st = pr.status;
        double s[6] = {0, 0, 0, 0, 0, 0}, el[8] = {0, 0, -1.0, 0, 0, 0, 0, 0};
        uint8_t dp = 0;
        if (st == kLinkOk) {
            IodBest w;
            w.F = best.F;
            w.key = best.key;
            w.tRef = pr.an[1].t;
            for (int c = 0; c < 6; ++c) w.s[c] = best.s[c];
            if (!(best.F < INFINITY)) st = kLinkNoCandidate;
            else if (!iod_epoch_state(w, pr.an[1].t, gr.mu, bstar ? bstar[j] : 0.0, gr, s, el, dp)) st = kLinkNoCandidate;
        }
        const bool ok = st == kLinkOk;
        if (!ok) {
            for (int c = 0; c < 6; ++c) s[c] = 0.0;
            for (int c = 0; c < 8; ++c) el[c] = c == 2 ? -1.0 : 0.0;
            dp = 0;
        }
        const uint32_t ep = pr.an[1].index;
        for (int c = 0; c < 8; ++c) el0[(size_t)c * p + j] = el[c];
        fjd[j] = ok ? jd[ep] : 0.0;
        ffr[j] = ok ? fr[ep] : 0.0;
        for (int c = 0; c < 3; ++c) pos[3 * j + c] = s[c], vel[3 * j + c] = s[3 + c];
        off[j] = j;
        st0[j] = st;
        for (int c = 0; c < 6; ++c) state[(size_t)j * 6 + c] = s[c];
        rho[2 * j] = ok ? best.x[0] : 0.0;
        rho[2 * j + 1] = ok ? best.x[1] : 0.0;
        revs[j] = ok ? (uint8_t)(best.key >> 18) : 0;
        flags[j] = ok ? link_flags(best.key) : 0;
        wrms[j] = ok ? std::sqrt(best.F / pr.used) : 0.0;
        used[j] = pr.status == kLinkOk ? pr.used : 0;
        hypotheses[j] = pr.status == kLinkOk ? scored : 0;
        deep[j] = dp;
        if (converged) converged[j] = ok && best.converged;
    }
    off[p] = p;
    if (p)
        emul_fit_mixed(el0.data(), p, grav, off.data(), fjd.data(), ffr.data(), pos.data(), vel.data(), kIodFitPosSigma,
                       kIodFitVelSigma, 0, kIodFitIter, elements, rms.data(), iters.data(), fit.data());
    for (uint32_t j = 0; j < p; ++j) {
        status[j] = iod_final_status(st0[j], fit[j], rms[2 * j], rms[2 * j + 1]);
        conv[2 * j] = st0[j] == kLinkOk ? rms[2 * j] : 0.0;
        conv[2 * j + 1] = st0[j] == kLinkOk ? rms[2 * j + 1] : 0.0;
        if (st0[j] != kLinkOk)
            for (int c = 0; c < 8; ++c) elements[(size_t)c * p + j] = 0.0;
    }
    return 0;
}

// Track [begin, end)'s anchor: out = {index, t, R[3], L[3], lo, hi, n}; 0 when it has none
extern "C" int emul_link_anchor(uint32_t begin, uint32_t end, const double *jd, const double *fr, const uint8_t *kind,
                                const double *value, const double *sigma, const uint32_t *station,
                                const double *stations, double rMin, double rMax, double *out) {
    LinkAnchor an;
    if (!link_anchor(arrays(jd, fr, kind, value, sigma, station, stations), begin, end, rMin, rMax, an)) return 0;
    out[0] = an.index;
    out[1] = an.t;
    for (int q = 0; q < 3; ++q) out[2 + q] = an.R[q], out[5 + q] = an.L[q];
    out[8] = an.lo;
    out[9] = an.hi;
    out[10] = an.n;
    return 1;
}

extern "C" double emul_link_range(double lo, double hi, uint32_t n, uint32_t k) {
    LinkAnchor an;
    an.lo = lo;
    an.hi = hi;
    an.n = n;
    return link_range(an, k);
}

// Every admissible state of pair (ia, ib): keys[cap], F[cap] (F_probe, +inf when a propagation failed) and the epoch
// states[cap][6], in cell and slot order; probes[6] the probe observations.  Returns the count, -1 - status when the
// pair is not OK.
extern "C" int emul_link_hypotheses(const uint32_t *offsets, uint32_t t, const double *jd, const double *fr,
                                    const uint8_t *kind, const double *value, const double *sigma,
                                    const uint32_t *station, const double *stations, uint32_t ia, uint32_t ib,
                                    double rMin, double rMax, uint32_t maxRevs, int grav, uint32_t cap, uint32_t *keys,
                                    double *F, double *states, uint32_t *probes, int *nProbe) {
    const Gravity gr = gravity(grav);
    const CorrObsArrays in = arrays(jd, fr, kind, value, sigma, station, stations);
    LinkPair pr;
    link_pair(in, offsets, t, ia, ib, rMin, rMax, pr);
    if (pr.status != kLinkOk) return -1 - pr.status;
    for (int q = 0; q < pr.nProbe; ++q) probes[q] = pr.probe[q];
    *nProbe = pr.nProbe;
    uint32_t n = 0;
    for (uint32_t c = 0, cells = link_cells(pr); c < cells; ++c) {
        const uint32_t dir = c & 1, i2 = (c >> 1) % pr.an[1].n, i1 = (c >> 1) / pr.an[1].n;
        const double x[2] = {link_range(pr.an[0], i1), link_range(pr.an[1], i2)};
        double r1[3], r2[3];
        link_positions(pr, x, r1, r2);
        const double nz[3] = {0.0, 0.0, dir ? -1.0 : 1.0};
        lambert_solve(r1, r2, pr.tof, gr.mu, nz, maxRevs,
                      [&](uint32_t slot, uint8_t st, int, const double *, const double *v2) {
                          if (st != kLamOk) return;
                          const double s[6] = {r2[0], r2[1], r2[2], v2[0], v2[1], v2[2]};
                          if (!iod_admissible(s, gr.mu, gr.radiusEarthKm) || n >= cap) return;
                          keys[n] = link_key(slot, dir, i1, i2);
                          F[n] = link_probe_score(in, pr, s, gr.mu);
                          std::memcpy(states + 6 * (size_t)n, s, sizeof s);
                          ++n;
                      });
    }
    return (int)n;
}
