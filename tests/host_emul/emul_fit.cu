// TEST INFRASTRUCTURE ONLY: runs the element fit of K8 (az_fit.cuh, __host__ __device__) on the CPU, with the
// evaluation pass of az_fit.cu restated serially: 32 lane partials over observations l, l + 32, ..., then the same
// xor-butterfly over masks 16, 8, 4, 2, 1.  Not part of the shipped library; nothing in astroz_b200/ references it.
#include <cstdint>
#include <cstring>

#include "az_fit.cuh"

using namespace az;

extern "C" int emul_fit(const double *elements, uint32_t n, int grav, const uint32_t *offsets, const double *jd,
                        const double *fr, const double *pos, const double *vel, double posSigma, double velSigma,
                        int fitBstar, uint32_t maxIter, double *fitted, double *rms, uint32_t *iterations,
                        uint8_t *status) {
    const Gravity gr = gravity(grav);
    const GravConsts g = grav_consts(gr);
    const int nvar = fitBstar ? kFitVars : kFitVars - 1;
    for (uint32_t s = 0; s < n; ++s) {
        double el0[8];
        for (int c = 0; c < 8; ++c) el0[c] = elements[(size_t)c * n + s];
        const uint32_t begin = offsets[s], end = offsets[s + 1];
        const uint32_t nObs = end > begin ? end - begin : 0;
        auto pass = [&](const double (&x)[kFitVars], FitSums &sum) -> bool {
            double sets[kFitSets][kSgp4Cols], inv[kFitSets];
            for (int k = 0; k <= nvar; ++k)
                if (!fit_build_set(x, k, el0[0], gr, sets[k], inv[k])) return false;
            auto set = [&sets](int k) { return [&sets, k](int c) { return sets[k][c]; }; };
            double lanes[32][kFitSumWords] = {};
            double J[kFitVars * 6];
            for (uint32_t lane = 0; lane < 32; ++lane)
                for (uint32_t i = begin + lane; i < end; i += 32)
                    fit_accumulate(set, nvar, inv, add_rn(jd[i], fr[i]), el0[0], pos + (size_t)i * 3,
                                   vel ? vel + (size_t)i * 3 : nullptr, 1.0 / posSigma, 1.0 / velSigma, g, J,
                                   lanes[lane], 1);
            for (int m = 16; m > 0; m >>= 1) {
                double next[32][kFitSumWords];
                for (int l = 0; l < 32; ++l)
                    for (int q = 0; q < kFitSumWords; ++q) next[l][q] = lanes[l][q] + lanes[l ^ m][q];
                std::memcpy(lanes, next, sizeof lanes);
            }
            std::memcpy(fit_words(sum), lanes[0], sizeof lanes[0]);
            return true;
        };
        FitResult r;
        fit_satellite(el0, gr, fitBstar != 0, maxIter, nObs, vel != nullptr, pass, r);
        for (int c = 0; c < 8; ++c) fitted[(size_t)c * n + s] = r.el[c];
        rms[2 * s] = r.rmsPos;
        rms[2 * s + 1] = r.rmsVel;
        iterations[s] = r.iters;
        status[s] = r.status;
    }
    return 0;
}
