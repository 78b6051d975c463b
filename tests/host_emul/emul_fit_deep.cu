// TEST INFRASTRUCTURE ONLY: runs the deep-space element fit (az_fit.cuh's FitDeepSpace, __host__ __device__) on the
// CPU, with the evaluation pass of fit_deep_kernel (az_fit.cu) restated serially: the sets and their resonance
// lattices, 32 lane partials over observations l, l + 32, ..., then the xor-butterfly over masks 16, 8, 4, 2, 1.
// Linked with emul_fit.cu, whose emul_fit fits the near-earth rows, into one library.  emul_fit_mixed is the _mixed
// calls (fit_kernel, then fit_deep_kernel on the deep-space rows); emul_deep_states evaluates the deep-space query
// through fit_deep_kernel's lattice or stepped fresh from atime = 0.  Not part of the shipped library; nothing in
// astroz_b200/ references it.
#include <cmath>
#include <cstdint>
#include <cstring>

#include "az_fit.cuh"

using namespace az;

extern "C" int emul_fit(const double *elements, uint32_t n, int grav, const uint32_t *offsets, const double *jd,
                        const double *fr, const double *pos, const double *vel, double posSigma, double velSigma,
                        int fitBstar, uint32_t maxIter, double *fitted, double *rms, uint32_t *iterations,
                        uint8_t *status);

// 32 lane partials, lane l over observations l, l + 32, ..., then the butterfly: fit_kernel / fit_deep_kernel's sums
template <typename ObsFn>
static bool emul_lane_sums(uint32_t begin, uint32_t end, ObsFn obs, FitSums &sum) {
    double lanes[32][kFitSumWords] = {};
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

// fit_deep_kernel's lattice extent: nodes per direction from the satellite's largest forward and backward |tsince|
static void emul_lattice_nodes(const double *jd, const double *fr, uint32_t begin, uint32_t end, double epochJd,
                               int (&nodes)[2]) {
    double fwd = 0.0, bwd = 0.0;
    for (uint32_t i = begin; i < end; ++i) {
        const double ts = pairs_tsince_deep(add_rn(jd[i], fr[i]), epochJd);
        if (ts > 0.0) fwd = std::fmax(fwd, ts);
        else bwd = std::fmax(bwd, -ts);
    }
    nodes[0] = fit_lattice_nodes(fwd);
    nodes[1] = fit_lattice_nodes(bwd);
}

static TleRecord emul_record(const double *el0) {
    TleRecord t;
    t.epochJd = el0[0]; t.revPerDay = el0[1]; t.ecc = el0[2]; t.inclDeg = el0[3];
    t.raanDeg = el0[4]; t.argpDeg = el0[5]; t.maDeg = el0[6]; t.bstar = el0[7];
    return t;
}

// astroz_cuda_fit_elements_mixed on the CPU: every row through emul_fit, then the deep-space rows again under
// FitDeepSpace with fit_deep_kernel's pass.
extern "C" int emul_fit_mixed(const double *elements, uint32_t n, int grav, const uint32_t *offsets, const double *jd,
                              const double *fr, const double *pos, const double *vel, double posSigma, double velSigma,
                              int fitBstar, uint32_t maxIter, double *fitted, double *rms, uint32_t *iterations,
                              uint8_t *status) {
    emul_fit(elements, n, grav, offsets, jd, fr, pos, vel, posSigma, velSigma, fitBstar, maxIter, fitted, rms,
             iterations, status);
    const Gravity gr = gravity(grav);
    const GravConsts g = grav_consts(gr);
    const int nvar = fitBstar ? kFitVars : kFitVars - 1;
    for (uint32_t s = 0; s < n; ++s) {
        double el0[8];
        for (int c = 0; c < 8; ++c) el0[c] = elements[(size_t)c * n + s];
        {
            NearEarth ne;
            if (build_near_earth(emul_record(el0), gr, ne) != kDeepSpace) continue;
        }
        const uint32_t begin = offsets[s], end = offsets[s + 1];
        const uint32_t nObs = end > begin ? end - begin : 0;
        int nodes[2];
        emul_lattice_nodes(jd, fr, begin, end, el0[0], nodes);
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
            return emul_lane_sums(begin, end, [&](uint32_t i, double *J, double *acc) {
                return fit_accumulate_model(eval, nvar, inv, add_rn(jd[i], fr[i]), el0[0], pos + (size_t)i * 3,
                                            vel ? vel + (size_t)i * 3 : nullptr, 1.0 / posSigma, 1.0 / velSigma, J,
                                            acc, 1);
            }, sum);
        };
        FitResult r;
        fit_satellite(el0, gr, fitBstar != 0, maxIter, nObs, vel != nullptr, pass, r, FitDeepSpace{});
        for (int c = 0; c < 8; ++c) fitted[(size_t)c * n + s] = r.el[c];
        rms[2 * s] = r.rmsPos;
        rms[2 * s + 1] = r.rmsVel;
        iterations[s] = r.iters;
        status[s] = r.status;
    }
    return 0;
}

// The deep-space model's TEME states of one element set el[8] at m epochs, as the fit evaluates them: the record the
// fit builds for these elements, queried through fit_deep_kernel's lattice (fresh = 0) or through a lattice of node 0
// alone, so that every query steps the resonance integrator from atime = 0 (fresh = 1).  out[m][6]; st[m] the cell
// statuses.  Returns 0, or -1 when the set is not a deep-space set.
extern "C" int emul_deep_states(const double *el, int grav, const double *jd, const double *fr, uint32_t m, int fresh,
                                double *out, uint8_t *st) {
    const Gravity gr = gravity(grav);
    const GravConsts g = grav_consts(gr);
    Sdp4Sat rec;
    if (!FitDeepSpace::build(emul_record(el), gr, rec)) return -1;
    double2 lattice[2 * kFitLatticeNodes];
    int nodes[2];
    emul_lattice_nodes(jd, fr, 0, m, el[0], nodes);
    for (int dir = 0; dir < 2; ++dir) fit_deep_lattice(rec, dir, nodes[dir], lattice);
    const double2 node0[2] = {make_double2(rec.xlamo, rec.no), make_double2(rec.xlamo, rec.no)};
    for (uint32_t i = 0; i < m; ++i) {
        const double jdFull = add_rn(jd[i], fr[i]);
        double f[6];
        if (fresh) {
            CellOut o;
            st[i] = pairs_sdp4_query<0, true>(rec, node0, 1, jdFull, g, o);
            f[0] = o.rx; f[1] = o.ry; f[2] = o.rz; f[3] = o.vx; f[4] = o.vy; f[5] = o.vz;
        } else {
            st[i] = fit_deep_eval(rec, lattice, jdFull, g, f) ? 0 : 1;
        }
        std::memcpy(out + 6 * (size_t)i, f, sizeof f);
    }
    return 0;
}
