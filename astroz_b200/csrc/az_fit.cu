// az_fit.cu -- K8: fit SGP4 mean elements to TEME ephemerides on the device, one warp per satellite.
//
// The fit itself (variables, steps, damping schedule, stopping rule) is az_fit.cuh's fit_satellite; this file gives it
// its evaluation pass.  Every lane of the warp runs the same Levenberg-Marquardt control flow on the same values:
//   1. lanes 0 .. nvar build one element set each (nominal, then one per stepped variable) with build_near_earth into
//      the warp's shared-memory slice of near-earth columns;
//   2. lane l evaluates sgp4_cell<1> under every set for observations l, l + 32, ... of the satellite, and accumulates
//      its partial cost, J^T J (28 entries) and J^T r; those partials and the observation's Jacobian columns sit in
//      the lane's column of shared memory, which keeps the registers for the propagation;
//   3. an xor-butterfly over masks 16, 8, 4, 2, 1 sums the partials: both partners of a pair add the same two values,
//      so every lane ends with the same bits, and the 7 x 7 solve and the accept / reject decision agree on all lanes.
// The order of every sum is fixed by the lane and observation indices alone, so a satellite's result does not depend
// on which other satellites share the launch or where it sits in the batch.
#include "az_fit.cuh"
#include "az_kernels.cuh"

namespace az {

constexpr int kFitWarps = 2;   // warps per CTA: 2 x 23 KB of shared memory
constexpr int kFitThreads = kFitWarps * 32;

struct FitWarpSmem {
    double sets[kFitSets][kSgp4Cols];
    double inv[kFitSets];
    double J[kFitVars * 6][32];   // this observation's Jacobian, entry (j, c) of lane l at J[j * 6 + c][l]
    double acc[kFitSumWords][32]; // lane l's partial FitSums, word q at acc[q][l]
};

__global__ void __launch_bounds__(kFitThreads) fit_kernel(const FitArgs a) {
    __shared__ FitWarpSmem smem[kFitWarps];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t s = blockIdx.x * kFitWarps + warp;
    if (s >= a.n) return;
    FitWarpSmem &w = smem[warp];
    const Gravity grav = gravity(a.grav);
    double el0[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) el0[c] = __ldg(a.elements + (size_t)c * a.n + s);
    const uint32_t begin = __ldg(a.offsets + s), end = __ldg(a.offsets + s + 1);
    const uint32_t nObs = end > begin ? end - begin : 0;
    const int nvar = a.fitBstar ? kFitVars : kFitVars - 1;

    auto pass = [&](const double (&x)[kFitVars], FitSums &sum) -> bool {
        bool ok = true;
        if ((int)lane <= nvar) ok = fit_build_set(x, (int)lane, el0[0], grav, w.sets[lane], w.inv[lane]);
        const bool allOk = __all_sync(0xffffffffu, ok);
        __syncwarp();
        if (!allOk) return false;
        auto set = [&w](int k) { return [&w, k](int c) { return w.sets[k][c]; }; };
#pragma unroll
        for (int q = 0; q < kFitSumWords; ++q) w.acc[q][lane] = 0.0;
        for (uint32_t i = begin + lane; i < end; i += 32) {
            const double jdFull = add_rn(__ldg(a.jd + i), __ldg(a.fr + i));
            fit_accumulate(set, nvar, w.inv, jdFull, el0[0], a.pos + (size_t)i * 3,
                           a.vel ? a.vel + (size_t)i * 3 : nullptr, a.wp, a.wv, a.g, &w.J[0][lane], &w.acc[0][lane],
                           32);
        }
        double *v = fit_words(sum);
#pragma unroll
        for (int q = 0; q < kFitSumWords; ++q) v[q] = w.acc[q][lane];
#pragma unroll
        for (int m = 16; m > 0; m >>= 1) {
#pragma unroll
            for (int q = 0; q < kFitSumWords; ++q) v[q] += __shfl_xor_sync(0xffffffffu, v[q], m);
        }
        __syncwarp();   // the sets are read by every lane before the next pass rebuilds them
        return true;
    };
    FitResult r;
    fit_satellite(el0, grav, a.fitBstar != 0, a.maxIter, nObs, a.vel != nullptr, pass, r);
    if (lane == 0) {
#pragma unroll
        for (int c = 0; c < 8; ++c) a.fitted[(size_t)c * a.n + s] = r.el[c];
        a.rms[2 * (size_t)s] = r.rmsPos;
        a.rms[2 * (size_t)s + 1] = r.rmsVel;
        a.iterations[s] = r.iters;
        a.status[s] = r.status;
    }
}

cudaError_t launch_fit(const FitArgs &a, cudaStream_t stream) {
    if (a.n == 0) return cudaSuccess;
    const uint32_t blocks = (a.n + kFitWarps - 1) / kFitWarps;
    fit_kernel<<<blocks, kFitThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

}  // namespace az
