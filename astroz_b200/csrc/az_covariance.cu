// az_covariance.cu -- K10: state covariance at query times from a fitted element set's covariance (az_covariance.cuh).
//
// Work is balanced over queries, not satellites: a work item is a chunk of cov_chunk(m) consecutive queries (queries
// are grouped by satellite through offsets), one warp per chunk, so one object with 10^6 times spreads over many warps
// and a batch of one query per object still fills the GPU.
// The warp binary-searches offsets for its chunk's first satellite and walks the satellite segments that overlap the
// chunk.  Per segment, lanes 0 .. nvar build the nominal and stepped sets into the warp's shared memory (deep space:
// Sdp4Sat records and each set's K2a lattice up to the segment's largest |tsince|); each lane then takes queries
// l, l + 32, ... of the segment, runs 1 + nvar propagations, builds J in its shared-memory column, forms J P J^T with P
// broadcast from shared memory and stores its outputs.  No sum runs across queries, so the bytes of a query do not
// depend on the chunking.  covariance_kernel (2 warps per CTA) handles the model-0 segments, covariance_deep_kernel (1
// warp per CTA, under 48 KB of static shared memory) the model-1 segments; each leaves the other's queries alone.
#include "az_covariance.cuh"
#include "az_kernels.cuh"

namespace az {

constexpr int kCovWarps = 2;   // warps per CTA of the near-earth kernel
constexpr int kCovThreads = kCovWarps * 32;

struct CovWarpSmem {
    double sets[kFitSets][kSgp4Cols];
    double inv[kFitSets];
    double P[kFitN];
    double J[kCovJacWords][32];
};

struct CovDeepWarpSmem {
    Sdp4Sat sets[kFitSets];
    double2 lattice[kFitSets][2 * kFitLatticeNodes];
    double inv[kFitSets];
    double P[kFitN];
    double J[kCovJacWords][32];
};

// query i's outputs from the lane's J column
__device__ __forceinline__ void cov_store(const CovArgs &a, uint32_t i, uint8_t st, const double (&f0)[6],
                                          const double (&sig)[kCovWords], const double (&J)[kCovJacWords][32],
                                          uint32_t lane) {
    if (a.state) {
#pragma unroll
        for (int c = 0; c < 6; ++c) a.state[(size_t)i * 6 + c] = f0[c];
    }
#pragma unroll
    for (int q = 0; q < kCovWords; ++q) a.sigma[(size_t)i * kCovWords + q] = sig[q];
    if (a.jacobian) {
#pragma unroll 6
        for (int q = 0; q < kCovJacWords; ++q) a.jacobian[(size_t)i * kCovJacWords + q] = J[q][lane];
    }
    a.status[i] = st;
}

// The queries of work item `item`: [cb, ce); false past the last query
__device__ __forceinline__ bool cov_item(const CovArgs &a, uint32_t item, uint32_t &cb, uint32_t &ce) {
    const uint64_t b = (uint64_t)item * a.chunk;
    if (b >= a.m) return false;
    cb = (uint32_t)b;
    ce = (uint32_t)(b + a.chunk < a.m ? b + a.chunk : a.m);
    return true;
}

// Segment s of the chunk: its element columns and P (into smem, lanes 0 .. 27); the caller syncs the warp after
__device__ __forceinline__ void cov_load_sat(const CovArgs &a, uint32_t s, uint32_t lane, double (&el0)[8],
                                             double (&P)[kFitN]) {
#pragma unroll
    for (int c = 0; c < 8; ++c) el0[c] = __ldg(a.elements + (size_t)c * a.n + s);
    if (lane < (uint32_t)kFitN) P[lane] = __ldg(a.covariance + (size_t)s * kFitN + lane);
}

__global__ void __launch_bounds__(kCovThreads) covariance_kernel(const CovArgs a) {
    __shared__ CovWarpSmem smem[kCovWarps];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint32_t cb, ce;
    if (!cov_item(a, blockIdx.x * kCovWarps + warp, cb, ce)) return;
    CovWarpSmem &w = smem[warp];
    const Gravity grav = gravity(a.grav);
    for (uint32_t s = cov_first_sat(a.offsets, a.n, cb); s < a.n; ++s) {
        const uint32_t sb = __ldg(a.offsets + s);
        if (sb >= ce) break;
        const uint32_t b = sb > cb ? sb : cb, e0 = __ldg(a.offsets + s + 1), e = e0 < ce ? e0 : ce;
        if (b >= e || (a.model && __ldg(a.model + s) != 0)) continue;
        double el0[8];
        __syncwarp();   // every lane is done with the previous segment's sets
        cov_load_sat(a, s, lane, el0, w.P);
        __syncwarp();
        const int nvar = cov_nvar(w.P);
        double x[kFitVars];
        FitNearEarth::vars_of(el0, x);
        bool ok = true;
        if ((int)lane <= nvar) ok = fit_build_set(x, (int)lane, el0[0], grav, w.sets[lane], w.inv[lane]);
        const bool built = __all_sync(0xffffffffu, ok);
        __syncwarp();
        auto eval = [&w, &a](int k, double, const double (&ts)[1], double (&f)[6]) {
            CellOut o[1];
            sgp4_cell<1>([&w, k](int c) { return w.sets[k][c]; }, ts, a.g, o);
            f[0] = o[0].rx; f[1] = o[0].ry; f[2] = o[0].rz;
            f[3] = o[0].vx; f[4] = o[0].vy; f[5] = o[0].vz;
            return true;
        };
        for (uint32_t i = b + lane; i < e; i += 32) {
            double f0[6], sig[kCovWords];
            uint8_t st = kCovInitFailed;
            if (built) {
                const double jdFull = add_rn(__ldg(a.jd + i), __ldg(a.fr + i));
                st = cov_query(eval, nvar, w.inv, w.P, jdFull, el0[0], a.frame, &w.J[0][lane], 32, f0, sig);
            } else {
                cov_zero(&w.J[0][lane], 32, f0, sig);
            }
            cov_store(a, i, st, f0, sig, w.J, lane);
        }
    }
}

__global__ void __launch_bounds__(32) covariance_deep_kernel(const CovArgs a) {
    __shared__ CovDeepWarpSmem smem;
    CovDeepWarpSmem &w = smem;
    const uint32_t lane = threadIdx.x;
    uint32_t cb, ce;
    if (!cov_item(a, blockIdx.x, cb, ce)) return;
    const Gravity grav = gravity(a.grav);
    for (uint32_t s = cov_first_sat(a.offsets, a.n, cb); s < a.n; ++s) {
        const uint32_t sb = __ldg(a.offsets + s);
        if (sb >= ce) break;
        const uint32_t b = sb > cb ? sb : cb, e0 = __ldg(a.offsets + s + 1), e = e0 < ce ? e0 : ce;
        if (b >= e || !a.model || __ldg(a.model + s) != 1) continue;
        double el0[8];
        __syncwarp();
        cov_load_sat(a, s, lane, el0, w.P);
        __syncwarp();
        const int nvar = cov_nvar(w.P);
        double x[kFitVars];
        FitDeepSpace::vars_of(el0, x);
        bool ok = true;
        if ((int)lane <= nvar) ok = fit_build_set_of<FitDeepSpace>(x, (int)lane, el0[0], grav, w.sets[lane], w.inv[lane]);
        const bool built = __all_sync(0xffffffffu, ok);
        __syncwarp();
        if (built) {   // the lattices up to the segment's largest |tsince| (fit_deep_eval does not depend on it)
            double fwd = 0.0, bwd = 0.0;
            for (uint32_t i = b + lane; i < e; i += 32) {
                const double ts = pairs_tsince_deep(add_rn(__ldg(a.jd + i), __ldg(a.fr + i)), el0[0]);
                if (ts > 0.0) fwd = fmax(fwd, ts);
                else bwd = fmax(bwd, -ts);
            }
#pragma unroll
            for (int m = 16; m > 0; m >>= 1) {
                fwd = fmax(fwd, __shfl_xor_sync(0xffffffffu, fwd, m));
                bwd = fmax(bwd, __shfl_xor_sync(0xffffffffu, bwd, m));
            }
            const int nodes[2] = {fit_lattice_nodes(fwd), fit_lattice_nodes(bwd)};
            if ((int)lane < 2 * (nvar + 1)) {
                const int k = lane >> 1, dir = lane & 1;
                fit_deep_lattice(w.sets[k], dir, nodes[dir], w.lattice[k]);
            }
            __syncwarp();
        }
        auto eval = [&w, &a](int k, double jdFull, const double (&)[1], double (&f)[6]) {
            return fit_deep_eval(w.sets[k], w.lattice[k], jdFull, a.g, f);
        };
        for (uint32_t i = b + lane; i < e; i += 32) {
            double f0[6], sig[kCovWords];
            uint8_t st = kCovInitFailed;
            if (built) {
                const double jdFull = add_rn(__ldg(a.jd + i), __ldg(a.fr + i));
                st = cov_query(eval, nvar, w.inv, w.P, jdFull, el0[0], a.frame, &w.J[0][lane], 32, f0, sig);
            } else {
                cov_zero(&w.J[0][lane], 32, f0, sig);
            }
            cov_store(a, i, st, f0, sig, w.J, lane);
        }
    }
}

cudaError_t launch_covariance(const CovArgs &args, cudaStream_t stream) {
    if (args.m == 0 || args.n == 0) return cudaSuccess;
    CovArgs a = args;
    a.chunk = cov_chunk(a.m);
    const uint32_t chunks = (uint32_t)(((uint64_t)a.m + a.chunk - 1) / a.chunk);
    covariance_kernel<<<(chunks + kCovWarps - 1) / kCovWarps, kCovThreads, 0, stream>>>(a);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess || !a.model) return e;
    covariance_deep_kernel<<<chunks, 32, 0, stream>>>(a);
    return cudaGetLastError();
}

}  // namespace az
