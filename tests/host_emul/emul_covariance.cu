// TEST INFRASTRUCTURE ONLY: runs K10 (az_covariance.cuh, __host__ __device__) on the CPU with the work items of
// covariance_kernel and covariance_deep_kernel (az_covariance.cu) restated serially: chunks of `chunk` queries, each
// walking the satellite segments it overlaps, sets (and deep-space lattices up to the segment's largest |tsince|)
// built per segment.  emul_propagate_covariance is astroz_cuda_propagate_covariance with the chunk as a parameter
// (the library's is cov_chunk(m)).  Not part of the shipped library; nothing in astroz_b200/ references it.
#include <cmath>
#include <cstdint>
#include <cstring>

#include "az_covariance.cuh"

using namespace az;

extern "C" uint32_t emul_cov_chunk(uint32_t m) { return cov_chunk(m); }

extern "C" int emul_propagate_covariance(const double *elements, uint32_t n, int grav, const double *covariance,
                                         const uint8_t *model, const uint32_t *offsets, const double *jd,
                                         const double *fr, uint32_t m, int frame, uint32_t chunk, double *state,
                                         double *stateCov, double *jacobian, uint8_t *status) {
    const Gravity gr = gravity(grav);
    const GravConsts g = grav_consts(gr);
    for (uint64_t cb64 = 0; cb64 < m; cb64 += chunk) {
        const uint32_t cb = (uint32_t)cb64, ce = (uint32_t)(cb64 + chunk < m ? cb64 + chunk : m);
        for (uint32_t s = cov_first_sat(offsets, n, cb); s < n && offsets[s] < ce; ++s) {
            const uint32_t b = offsets[s] > cb ? offsets[s] : cb, e = offsets[s + 1] < ce ? offsets[s + 1] : ce;
            if (b >= e) continue;
            const int deep = model ? model[s] : 0;
            double el0[8], P[kFitN];
            for (int c = 0; c < 8; ++c) el0[c] = elements[(size_t)c * n + s];
            std::memcpy(P, covariance + (size_t)s * kFitN, sizeof P);
            const int nvar = cov_nvar(P);
            double x[kFitVars], inv[kFitSets] = {};
            double cols[kFitSets][kSgp4Cols];
            Sdp4Sat sets[kFitSets];
            double2 lattice[kFitSets][2 * kFitLatticeNodes];
            bool built = true;
            if (!deep) {
                FitNearEarth::vars_of(el0, x);
                for (int k = 0; k <= nvar; ++k) built = fit_build_set(x, k, el0[0], gr, cols[k], inv[k]) && built;
            } else {
                FitDeepSpace::vars_of(el0, x);
                for (int k = 0; k <= nvar; ++k)
                    built = fit_build_set_of<FitDeepSpace>(x, k, el0[0], gr, sets[k], inv[k]) && built;
                if (built) {
                    double fwd = 0.0, bwd = 0.0;
                    for (uint32_t i = b; i < e; ++i) {
                        const double ts = pairs_tsince_deep(add_rn(jd[i], fr[i]), el0[0]);
                        if (ts > 0.0) fwd = std::fmax(fwd, ts);
                        else bwd = std::fmax(bwd, -ts);
                    }
                    const int nodes[2] = {fit_lattice_nodes(fwd), fit_lattice_nodes(bwd)};
                    for (int k = 0; k <= nvar; ++k)
                        for (int dir = 0; dir < 2; ++dir) fit_deep_lattice(sets[k], dir, nodes[dir], lattice[k]);
                }
            }
            auto evalNear = [&](int k, double, const double (&ts)[1], double (&f)[6]) {
                CellOut o[1];
                sgp4_cell<1>([&cols, k](int c) { return cols[k][c]; }, ts, g, o);
                f[0] = o[0].rx; f[1] = o[0].ry; f[2] = o[0].rz;
                f[3] = o[0].vx; f[4] = o[0].vy; f[5] = o[0].vz;
                return true;
            };
            auto evalDeep = [&](int k, double jdFull, const double (&)[1], double (&f)[6]) {
                return fit_deep_eval(sets[k], lattice[k], jdFull, g, f);
            };
            for (uint32_t i = b; i < e; ++i) {
                double f0[6], sig[kCovWords], J[kCovJacWords];
                uint8_t st = kCovInitFailed;
                if (built) {
                    const double jdFull = add_rn(jd[i], fr[i]);
                    st = deep ? cov_query(evalDeep, nvar, inv, P, jdFull, el0[0], frame, J, 1, f0, sig)
                              : cov_query(evalNear, nvar, inv, P, jdFull, el0[0], frame, J, 1, f0, sig);
                } else {
                    cov_zero(J, 1, f0, sig);
                }
                if (state) std::memcpy(state + (size_t)i * 6, f0, sizeof f0);
                std::memcpy(stateCov + (size_t)i * kCovWords, sig, sizeof sig);
                if (jacobian) std::memcpy(jacobian + (size_t)i * kCovJacWords, J, sizeof J);
                status[i] = st;
            }
        }
    }
    return 0;
}
