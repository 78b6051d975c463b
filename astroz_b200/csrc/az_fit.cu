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
//
// fit_deep_kernel fits the deep-space sets the same way under az_fit.cuh's FitDeepSpace model: lanes 0 .. nvar build
// one Sdp4Sat record each, lanes 0 .. 2 nvar + 1 then build the resonance lattice of one (set, direction) each, and the
// observations go through pairs_sdp4_query against those records and lattices.
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

// One warp per CTA for the deep-space fit: its 29 KB of shared memory stays under the 48 KB static limit, and 7 such
// CTAs (7 warps) fit an SM's 228 KB, where 2-warp CTAs would need the opt-in to dynamic shared memory for 6.
struct FitDeepWarpSmem {
    Sdp4Sat sets[kFitSets];
    double2 lattice[kFitSets][2 * kFitLatticeNodes];   // set k: pairs_sdp4_query's [2][kFitLatticeNodes] layout
    double inv[kFitSets];
    double J[kFitVars * 6][32];
    double acc[kFitSumWords][32];
};

__global__ void __launch_bounds__(32) fit_deep_kernel(const FitArgs a) {
    __shared__ FitDeepWarpSmem smem;
    FitDeepWarpSmem &w = smem;
    const uint32_t lane = threadIdx.x;
    const uint32_t s = blockIdx.x;
    if (s >= a.n) return;
    const Gravity grav = gravity(a.grav);
    double el0[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) el0[c] = __ldg(a.elements + (size_t)c * a.n + s);
    {   // only the deep-space rows: the near-earth fit writes every other row
        TleRecord t;
        t.epochJd = el0[0]; t.revPerDay = el0[1]; t.ecc = el0[2]; t.inclDeg = el0[3];
        t.raanDeg = el0[4]; t.argpDeg = el0[5]; t.maDeg = el0[6]; t.bstar = el0[7];
        NearEarth ne;
        if (build_near_earth(t, grav, ne) != kDeepSpace) return;
    }
    const uint32_t begin = __ldg(a.offsets + s), end = __ldg(a.offsets + s + 1);
    const uint32_t nObs = end > begin ? end - begin : 0;
    const int nvar = a.fitBstar ? kFitVars : kFitVars - 1;
    // the lattice's extent in each direction, from the satellite's largest forward and backward |tsince|
    int nodes[2];
    {
        double fwd = 0.0, bwd = 0.0;
        for (uint32_t i = begin + lane; i < end; i += 32) {
            const double ts = pairs_tsince_deep(add_rn(__ldg(a.jd + i), __ldg(a.fr + i)), el0[0]);
            if (ts > 0.0) fwd = fmax(fwd, ts);
            else bwd = fmax(bwd, -ts);
        }
#pragma unroll
        for (int m = 16; m > 0; m >>= 1) {
            fwd = fmax(fwd, __shfl_xor_sync(0xffffffffu, fwd, m));
            bwd = fmax(bwd, __shfl_xor_sync(0xffffffffu, bwd, m));
        }
        nodes[0] = fit_lattice_nodes(fwd);
        nodes[1] = fit_lattice_nodes(bwd);
    }

    auto pass = [&](const double (&x)[kFitVars], FitSums &sum) -> bool {
        bool ok = true;
        if ((int)lane <= nvar)
            ok = fit_build_set_of<FitDeepSpace>(x, (int)lane, el0[0], grav, w.sets[lane], w.inv[lane]);
        if (!__all_sync(0xffffffffu, ok)) return false;
        __syncwarp();
        if ((int)lane < 2 * (nvar + 1)) {
            const int k = lane >> 1, dir = lane & 1;
            fit_deep_lattice(w.sets[k], dir, nodes[dir], w.lattice[k]);
        }
        __syncwarp();
        auto eval = [&w, &a](int k, double jdFull, const double (&)[1], double (&f)[6]) {
            return fit_deep_eval(w.sets[k], w.lattice[k], jdFull, a.g, f);
        };
#pragma unroll
        for (int q = 0; q < kFitSumWords; ++q) w.acc[q][lane] = 0.0;
        bool cellsOk = true;
        for (uint32_t i = begin + lane; i < end; i += 32) {
            const double jdFull = add_rn(__ldg(a.jd + i), __ldg(a.fr + i));
            cellsOk = fit_accumulate_model(eval, nvar, w.inv, jdFull, el0[0], a.pos + (size_t)i * 3,
                                           a.vel ? a.vel + (size_t)i * 3 : nullptr, a.wp, a.wv, &w.J[0][lane],
                                           &w.acc[0][lane], 32) && cellsOk;
        }
        const bool allOk = __all_sync(0xffffffffu, cellsOk);   // every lane has read the sets and lattices
        if (!allOk) return false;
        double *v = fit_words(sum);
#pragma unroll
        for (int q = 0; q < kFitSumWords; ++q) v[q] = w.acc[q][lane];
#pragma unroll
        for (int m = 16; m > 0; m >>= 1) {
#pragma unroll
            for (int q = 0; q < kFitSumWords; ++q) v[q] += __shfl_xor_sync(0xffffffffu, v[q], m);
        }
        __syncwarp();
        return true;
    };
    FitResult r;
    fit_satellite(el0, grav, a.fitBstar != 0, a.maxIter, nObs, a.vel != nullptr, pass, r, FitDeepSpace{});
    if (lane == 0) {
#pragma unroll
        for (int c = 0; c < 8; ++c) a.fitted[(size_t)c * a.n + s] = r.el[c];
        a.rms[2 * (size_t)s] = r.rmsPos;
        a.rms[2 * (size_t)s + 1] = r.rmsVel;
        a.iterations[s] = r.iters;
        a.status[s] = r.status;
    }
}

cudaError_t launch_fit_deep(const FitArgs &a, cudaStream_t stream) {
    if (a.n == 0) return cudaSuccess;
    fit_deep_kernel<<<a.n, 32, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_fit(const FitArgs &a, cudaStream_t stream) {
    if (a.n == 0) return cudaSuccess;
    const uint32_t blocks = (a.n + kFitWarps - 1) / kFitWarps;
    fit_kernel<<<blocks, kFitThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

}  // namespace az
