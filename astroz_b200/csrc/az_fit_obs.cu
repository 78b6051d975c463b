// az_fit_obs.cu -- K8 from sensor observations: the element fit of az_fit.cu with az_obs.cuh's measurement layer
// between the model's TEME state and the residual, and the formal covariance of the fitted variables at the end.
//
// fit_obs_kernel and fit_obs_deep_kernel are fit_kernel and fit_deep_kernel with one change each: an observation is
// (kind, value[6], sigma[6], station) instead of a TEME position and velocity, and goes through fit_accumulate_obs.
// The driver (fit_satellite_run: variables, steps, damping, stopping rule), the warp layout, the lane order of every
// sum and the xor-butterfly are theirs, so a satellite's result does not depend on the rest of the batch.  The
// satellite's used scalar residuals are counted once before the fit (an integer warp sum); at the final iterate lane 0
// inverts J^T W J (fit_covariance).  Stations are read through the read-only path: a station's geometry is formed
// per observation, a few dozen flops beside the ~8 propagations of each observation per pass.
//
// observe_kernel evaluates the measurement model alone, one thread per observation.
#include "az_kernels.cuh"
#include "az_obs.cuh"

namespace az {

constexpr int kFitObsWarps = 2;   // warps per CTA, as fit_kernel
constexpr int kFitObsThreads = kFitObsWarps * 32;

struct FitObsWarpSmem {
    double sets[kFitSets][kSgp4Cols];
    double inv[kFitSets];
    double J[kFitVars * 6][32];
    double acc[kFitSumWords][32];
};

struct FitObsDeepWarpSmem {
    Sdp4Sat sets[kFitSets];
    double2 lattice[kFitSets][2 * kFitLatticeNodes];
    double inv[kFitSets];
    double J[kFitVars * 6][32];
    double acc[kFitSumWords][32];
};

// Observation i: its kind, time, observed values, weights, GMST and station.
struct FitObsIn {
    int kind;
    double jdFull;
    double value[6], w[6];
    double sg, cg;
    ObsStation st;
};

__device__ __forceinline__ int fit_obs_load(const FitObsArgs &a, uint32_t i, FitObsIn &o) {
    o.kind = __ldg(a.kind + i);
    o.jdFull = add_rn(__ldg(a.jd + i), __ldg(a.fr + i));
    double sigma[6];
#pragma unroll
    for (int c = 0; c < 6; ++c) {
        o.value[c] = __ldg(a.value + (size_t)i * 6 + c);
        sigma[c] = __ldg(a.sigma + (size_t)i * 6 + c);
    }
    const int used = obs_weights(o.kind, o.value, sigma, o.w);
    double llh[3] = {0.0, 0.0, 0.0};
    if (obs_uses_station(o.kind)) {
        const uint32_t k = __ldg(a.station + i);
#pragma unroll
        for (int c = 0; c < 3; ++c) llh[c] = __ldg(a.stations + (size_t)k * 3 + c);
    }
    obs_frame(o.kind, o.jdFull, llh, o.sg, o.cg, o.st);
    return used;
}

// the satellite's used scalar residuals: lane partials, then an integer warp sum
__device__ __forceinline__ uint32_t fit_obs_residuals(const FitObsArgs &a, uint32_t begin, uint32_t end,
                                                      uint32_t lane) {
    uint32_t used = 0;
    for (uint32_t i = begin + lane; i < end; i += 32) {
        double value[6], sigma[6], w[6];
        const int kind = __ldg(a.kind + i);
        for (int c = 0; c < 6; ++c) {
            value[c] = __ldg(a.value + (size_t)i * 6 + c);
            sigma[c] = __ldg(a.sigma + (size_t)i * 6 + c);
        }
        used += (uint32_t)obs_weights(kind, value, sigma, w);
    }
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) used += __shfl_xor_sync(0xffffffffu, used, m);
    return used;
}

// lane 0's outputs of satellite s
__device__ __forceinline__ void fit_obs_store(const FitObsArgs &a, uint32_t s, const FitResult &r, bool fitted,
                                              const FitSums &fin, uint32_t nRes, int nvar, uint8_t model) {
    double cov[kFitN];
    for (int q = 0; q < kFitN; ++q) cov[q] = 0.0;
    if (fitted) fit_covariance(fin, nvar, cov);
#pragma unroll
    for (int c = 0; c < 8; ++c) a.fitted[(size_t)c * a.n + s] = r.el[c];
    for (int q = 0; q < kFitN; ++q) a.covariance[(size_t)s * kFitN + q] = cov[q];
    a.wrms[s] = fitted && nRes ? std::sqrt(fin.F / nRes) : 0.0;
    a.nResiduals[s] = nRes;
    a.iterations[s] = r.iters;
    a.status[s] = r.status;
    a.model[s] = model;
}

// the xor-butterfly of fit_kernel over the lanes' partial sums
__device__ __forceinline__ void fit_obs_reduce(const double (&acc)[kFitSumWords][32], uint32_t lane, FitSums &sum) {
    double *v = fit_words(sum);
#pragma unroll
    for (int q = 0; q < kFitSumWords; ++q) v[q] = acc[q][lane];
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) {
#pragma unroll
        for (int q = 0; q < kFitSumWords; ++q) v[q] += __shfl_xor_sync(0xffffffffu, v[q], m);
    }
}

__global__ void __launch_bounds__(kFitObsThreads) fit_obs_kernel(const FitObsArgs a) {
    __shared__ FitObsWarpSmem smem[kFitObsWarps];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t s = blockIdx.x * kFitObsWarps + warp;
    if (s >= a.n) return;
    FitObsWarpSmem &w = smem[warp];
    const Gravity grav = gravity(a.grav);
    double el0[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) el0[c] = __ldg(a.elements + (size_t)c * a.n + s);
    const uint32_t begin = __ldg(a.offsets + s), end = __ldg(a.offsets + s + 1);
    const int nvar = a.fitBstar ? kFitVars : kFitVars - 1;
    const uint32_t nRes = fit_obs_residuals(a, begin, end, lane);

    auto pass = [&](const double (&x)[kFitVars], FitSums &sum) -> bool {
        bool ok = true;
        if ((int)lane <= nvar) ok = fit_build_set(x, (int)lane, el0[0], grav, w.sets[lane], w.inv[lane]);
        const bool allOk = __all_sync(0xffffffffu, ok);
        __syncwarp();
        if (!allOk) return false;
        auto eval = [&w, &a](int k, double, const double (&ts)[1], double (&f)[6]) {
            CellOut o[1];
            sgp4_cell<1>([&w, k](int c) { return w.sets[k][c]; }, ts, a.g, o);
            f[0] = o[0].rx; f[1] = o[0].ry; f[2] = o[0].rz;
            f[3] = o[0].vx; f[4] = o[0].vy; f[5] = o[0].vz;
            return true;
        };
#pragma unroll
        for (int q = 0; q < kFitSumWords; ++q) w.acc[q][lane] = 0.0;
        for (uint32_t i = begin + lane; i < end; i += 32) {
            FitObsIn o;
            fit_obs_load(a, i, o);
            fit_accumulate_obs(eval, nvar, w.inv, o.jdFull, el0[0], o.kind, o.value, o.w, o.sg, o.cg, o.st,
                               &w.J[0][lane], &w.acc[0][lane], 32);
        }
        fit_obs_reduce(w.acc, lane, sum);
        __syncwarp();   // the sets are read by every lane before the next pass rebuilds them
        return true;
    };
    FitResult r;
    FitSums fin = {};
    bool fitted = false;
    auto final = [&](const FitSums &sums) {
        fin = sums;
        fitted = true;
    };
    fit_satellite_run(el0, grav, a.fitBstar != 0, a.maxIter, nRes, pass, final, r, FitNearEarth{});
    if (lane == 0) fit_obs_store(a, s, r, fitted, fin, nRes, nvar, 0);
}

// One warp per CTA, as fit_deep_kernel.
__global__ void __launch_bounds__(32) fit_obs_deep_kernel(const FitObsArgs a) {
    __shared__ FitObsDeepWarpSmem smem;
    FitObsDeepWarpSmem &w = smem;
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
    const int nvar = a.fitBstar ? kFitVars : kFitVars - 1;
    const uint32_t nRes = fit_obs_residuals(a, begin, end, lane);
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
            FitObsIn o;
            fit_obs_load(a, i, o);
            cellsOk = fit_accumulate_obs(eval, nvar, w.inv, o.jdFull, el0[0], o.kind, o.value, o.w, o.sg, o.cg,
                                         o.st, &w.J[0][lane], &w.acc[0][lane], 32) && cellsOk;
        }
        const bool allOk = __all_sync(0xffffffffu, cellsOk);   // every lane has read the sets and lattices
        if (!allOk) return false;
        fit_obs_reduce(w.acc, lane, sum);
        __syncwarp();
        return true;
    };
    FitResult r;
    FitSums fin = {};
    bool fitted = false;
    auto final = [&](const FitSums &sums) {
        fin = sums;
        fitted = true;
    };
    fit_satellite_run(el0, grav, a.fitBstar != 0, a.maxIter, nRes, pass, final, r, FitDeepSpace{});
    if (lane == 0) fit_obs_store(a, s, r, fitted, fin, nRes, nvar, 1);
}

__global__ void __launch_bounds__(256) observe_kernel(const double *states, const double *jd, const double *fr,
                                                      const uint8_t *kind, const uint32_t *station,
                                                      const double *stations, uint32_t m, double *values) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const int k = __ldg(kind + i);
    double f[6], h[6], sc[6], llh[3] = {0.0, 0.0, 0.0};
#pragma unroll
    for (int c = 0; c < 6; ++c) f[c] = __ldg(states + (size_t)i * 6 + c);
    if (obs_uses_station(k)) {
        const uint32_t row = __ldg(station + i);
#pragma unroll
        for (int c = 0; c < 3; ++c) llh[c] = __ldg(stations + (size_t)row * 3 + c);
    }
    double sg, cg;
    ObsStation st;
    obs_frame(k, add_rn(__ldg(jd + i), __ldg(fr + i)), llh, sg, cg, st);
    obs_model(k, f, sg, cg, st, h, sc);
#pragma unroll
    for (int c = 0; c < 6; ++c) values[(size_t)i * 6 + c] = h[c];
}

cudaError_t launch_fit_obs(const FitObsArgs &a, cudaStream_t stream) {
    if (a.n == 0) return cudaSuccess;
    fit_obs_kernel<<<(a.n + kFitObsWarps - 1) / kFitObsWarps, kFitObsThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_fit_obs_deep(const FitObsArgs &a, cudaStream_t stream) {
    if (a.n == 0) return cudaSuccess;
    fit_obs_deep_kernel<<<a.n, 32, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_observe(const double *states, const double *jd, const double *fr, const uint8_t *kind,
                           const uint32_t *station, const double *stations, uint32_t m, double *values,
                           cudaStream_t stream) {
    if (m == 0) return cudaSuccess;
    observe_kernel<<<(m + 255) / 256, 256, 0, stream>>>(states, jd, fr, kind, station, stations, m, values);
    return cudaGetLastError();
}

}  // namespace az
