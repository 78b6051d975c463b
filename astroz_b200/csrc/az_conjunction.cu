// az_conjunction.cu -- K11: assessment of candidate conjunctions (az_conjunction.cuh), one warp per candidate.
//
// The warp loads both rows' element columns and covariance words, and lanes (row, set) build each row's nominal and
// stepped sets into the warp's shared-memory slots (deep space: Sdp4Sat records and, lanes (row, set, direction), each
// set's K2a lattice over the window).  In each search round the 32 lanes evaluate g at the 32 samples of the bracket
// and a ballot picks the sign change.  Lanes 0 and 1 then run K10's cov_query for the primary and the secondary at the
// TCA; every lane forms the plane from their shared-memory results, the lanes rank the 64 candidate panel edges, spread
// the Pc quadrature nodes over themselves and reduce in a fixed order, and lane 0 stores.  No sum crosses candidates.
// conjunction_kernel (4 warps per CTA) takes the pairs of two near-earth rows; conjunction_deep_kernel (2 warps per
// CTA, slots sized for deep-space sets and lattices) every other pair, bad pairs included; each leaves the other's
// candidates alone.
#include "az_conjunction.cuh"
#include "az_kernels.cuh"

namespace az {

constexpr int kConjNearWarps = 4;
constexpr int kConjDeepWarps = 2;

// Measurement builds only: AZ_CONJ_ONE_KERNEL=1 sends every candidate to conjunction_deep_kernel (deep-sized slots for
// every pair), the alternative to the class split that DESIGN.md section 3 (K11) times.
#ifndef AZ_CONJ_ONE_KERNEL
#define AZ_CONJ_ONE_KERNEL 0
#endif

struct ConjNearSlot {
    double cols[kFitSets][kSgp4Cols];
};
struct ConjDeepSlot {
    union {
        double cols[kFitSets][kSgp4Cols];
        struct {
            Sdp4Sat sets[kFitSets];
            double2 lattice[kFitSets][2 * kFitLatticeNodes];
        } ds;
    };
};

template <bool kDeep>
struct ConjWarpSmem {
    typename std::conditional<kDeep, ConjDeepSlot, ConjNearSlot>::type obj[2];
    double inv[2][kFitSets];
    double P[2][kFitN];
    double J[2][kCovJacWords];
    double f[2][6];
    double sig[2][kCovWords];
    double raw[kConjBreaks], bp[kConjBreaks];
    double rec[kConjRecordWords];
};

template <bool kDeep>
__device__ __forceinline__ bool conj_eval(const ConjWarpSmem<kDeep> &w, int o, int deep, int k, double ts,
                                          const GravConsts &g, double (&f)[6]) {
    if constexpr (kDeep) {
        if (deep) return conj_eval_deep(w.obj[o].ds.sets[k], w.obj[o].ds.lattice[k], ts, g, f);
    }
    return conj_eval_near([&w, o, k](int c) { return w.obj[o].cols[k][c]; }, ts, g, f);
}

template <bool kDeep>
struct ConjWarpSampler {
    const ConjWarpSmem<kDeep> &w;
    const GravConsts &gc;
    double ts0[2];
    int deep[2];
    uint32_t lane;
    double gv = 0.0, dv2 = 0.0;
    bool ok = true;
    __device__ uint32_t round(double a, double b) {
        const double t = conj_node(a, b, (int)lane);
        double fp[6], fs[6];
        ok = conj_eval(w, 0, deep[0], 0, ts0[0] + t, gc, fp) && ok;
        ok = conj_eval(w, 1, deep[1], 0, ts0[1] + t, gc, fs) && ok;
        double gg = 0.0, dd = 0.0;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const double dr = fs[c] - fp[c], dv = fs[3 + c] - fp[3 + c];
            gg += dr * dv;
            dd += dr * dr;
        }
        gv = gg;
        dv2 = dd;
        return __ballot_sync(0xffffffffu, gg < 0.0);
    }
    __device__ double g(int l) const { return __shfl_sync(0xffffffffu, gv, l); }
    __device__ double d2(int l) const { return __shfl_sync(0xffffffffu, dv2, l); }
};

__device__ __forceinline__ void conj_store_zero(const ConjArgs &a, uint32_t i, uint8_t st, uint32_t lane) {
    if (lane < (uint32_t)kConjRecordWords) a.record[(size_t)i * kConjRecordWords + lane] = 0.0;
    if (a.states && lane < 12) a.states[(size_t)i * 12 + lane] = 0.0;
    if (a.sigma)
        for (uint32_t q = lane; q < 2 * kCovWords; q += 32) a.sigma[(size_t)i * 2 * kCovWords + q] = 0.0;
    if (lane == 0) a.status[i] = st;
}

template <bool kDeep>
__device__ __forceinline__ void conj_candidate(const ConjArgs &a, uint32_t i, ConjWarpSmem<kDeep> &w, uint32_t lane) {
    const uint32_t idx[2] = {__ldg(a.primary + i), __ldg(a.secondary + i)};
    const bool bad = idx[0] >= a.n || idx[1] >= a.n || idx[0] == idx[1];
    const int mdl[2] = {bad || !a.model ? 0 : (int)__ldg(a.model + idx[0]),
                        bad || !a.model ? 0 : (int)__ldg(a.model + idx[1])};
    const bool near = !AZ_CONJ_ONE_KERNEL && !bad && mdl[0] == 0 && mdl[1] == 0;
    if (near == kDeep) return;   // the other kernel's candidate
    if (bad) return conj_store_zero(a, i, kConjBadPair, lane);
    if (mdl[0] > 1 || mdl[1] > 1) return conj_store_zero(a, i, kConjInitFailed, lane);
    const Gravity grav = gravity(a.grav);
    const double jdFull = add_rn(__ldg(a.jd + i), __ldg(a.fr + i)), win = __ldg(a.window + i);
    // lanes (o, k): row o = lane / 16 builds its set k
    const uint32_t o = lane >> 4, k = lane & 15;
    double el[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) el[c] = __ldg(a.elements + (size_t)c * a.n + idx[o]);
    const double ts0[2] = {pairs_tsince_deep(jdFull, __ldg(a.elements + idx[0])),
                           pairs_tsince_deep(jdFull, __ldg(a.elements + idx[1]))};
    __syncwarp();   // every lane is done with the previous candidate's slots
    for (uint32_t q = lane; q < 2 * kFitN; q += 32)
        w.P[q / kFitN][q % kFitN] = __ldg(a.covariance + (size_t)idx[q / kFitN] * kFitN + q % kFitN);
    __syncwarp();
    const int nvar[2] = {cov_nvar(w.P[0]), cov_nvar(w.P[1])};
    bool ok = true;
    if ((int)k <= nvar[o]) {
        double x[kFitVars];
        if (kDeep && mdl[o]) {
            FitDeepSpace::vars_of(el, x);
            if constexpr (kDeep) ok = fit_build_set_of<FitDeepSpace>(x, (int)k, el[0], grav, w.obj[o].ds.sets[k], w.inv[o][k]);
        } else {
            FitNearEarth::vars_of(el, x);
            ok = fit_build_set(x, (int)k, el[0], grav, w.obj[o].cols[k], w.inv[o][k]);
        }
    }
    if (!__all_sync(0xffffffffu, ok)) return conj_store_zero(a, i, kConjInitFailed, lane);
    __syncwarp();
    if constexpr (kDeep) {   // lanes (o, set, direction): the lattices over [ts0 - w, ts0 + w]
        const uint32_t set = (lane >> 1) & 7, dir = lane & 1;
        if (mdl[o] && (int)set <= nvar[o]) {
            const double hi = ts0[o] + win, lo = ts0[o] - win;
            const int nodes = fit_lattice_nodes(dir == 0 ? (hi > 0.0 ? hi : 0.0) : (lo < 0.0 ? -lo : 0.0));
            fit_deep_lattice(w.obj[o].ds.sets[set], (int)dir, nodes, w.obj[o].ds.lattice[set]);
        }
        __syncwarp();
    }
    ConjWarpSampler<kDeep> S{w, a.g, {ts0[0], ts0[1]}, {mdl[0], mdl[1]}, lane};
    double tca = 0.0;
    uint8_t st = conj_tca(S, win, tca);
    ok = __all_sync(0xffffffffu, S.ok);
    if (ok && lane < 2) {
        const int r = (int)lane, dp = mdl[r];
        const double ts = ts0[r] + tca;
        auto eval = [&w, &a, r, dp, ts](int kk, double, const double (&)[1], double (&f)[6]) {
            return conj_eval(w, r, dp, kk, ts, a.g, f);
        };
        ok = cov_query(eval, nvar[r], w.inv[r], w.P[r], 0.0, 0.0, a.frame, w.J[r], 1, w.f[r], w.sig[r]) == kCovOk;
    }
    if (!__all_sync(0xffffffffu, ok)) return conj_store_zero(a, i, kConjCellFailed, lane);
    __syncwarp();
    double rec[kConjRecordWords];
    ConjPc pc;
    if (conj_geometry(w.f[0], w.f[1], w.sig[0], w.sig[1], a.frame, __ldg(a.hbr + i), rec, pc) == kConjNoPlane)
        st = kConjNoPlane;
    rec[0] = tca;
    double p = 0.0;
    if (!conj_pc_closed(pc, p)) {
        w.raw[lane] = conj_break(pc, (int)lane);
        w.raw[lane + 32] = conj_break(pc, (int)lane + 32);
        __syncwarp();
        const int r0 = conj_rank(w.raw, (int)lane), r1 = conj_rank(w.raw, (int)lane + 32);
        const int K = __popc(__ballot_sync(0xffffffffu, r0 >= 0)) + __popc(__ballot_sync(0xffffffffu, r1 >= 0));
        const double v0 = w.raw[lane], v1 = w.raw[lane + 32];
        __syncwarp();
        if (r0 >= 0) w.bp[r0] = v0;
        if (r1 >= 0) w.bp[r1] = v1;
        __syncwarp();
        p = conj_partial(pc, w.bp, K, (int)lane);
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) p += __shfl_down_sync(0xffffffffu, p, off);
    }
    rec[kConjRecPc] = p;
    if (lane == 0) {
#pragma unroll
        for (int q = 0; q < kConjRecordWords; ++q) w.rec[q] = rec[q];
        a.status[i] = st;
    }
    __syncwarp();
    // one word per lane: the 13 record words, the 12 state words and the 42 Sigma words
    if (lane < (uint32_t)kConjRecordWords) a.record[(size_t)i * kConjRecordWords + lane] = w.rec[lane];
    if (a.states && lane < 12) a.states[(size_t)i * 12 + lane] = w.f[lane / 6][lane % 6];
    if (a.sigma)
        for (uint32_t q = lane; q < 2 * kCovWords; q += 32)
            a.sigma[(size_t)i * 2 * kCovWords + q] = w.sig[q / kCovWords][q % kCovWords];
}

__global__ void __launch_bounds__(kConjNearWarps * 32) conjunction_kernel(const ConjArgs a) {
    __shared__ ConjWarpSmem<false> smem[kConjNearWarps];
    const uint32_t warp = threadIdx.x >> 5, i = blockIdx.x * kConjNearWarps + warp;
    if (i < a.m) conj_candidate<false>(a, i, smem[warp], threadIdx.x & 31);
}

__global__ void __launch_bounds__(kConjDeepWarps * 32) conjunction_deep_kernel(const ConjArgs a) {
    __shared__ ConjWarpSmem<true> smem[kConjDeepWarps];
    const uint32_t warp = threadIdx.x >> 5, i = blockIdx.x * kConjDeepWarps + warp;
    if (i < a.m) conj_candidate<true>(a, i, smem[warp], threadIdx.x & 31);
}

cudaError_t launch_conjunction(const ConjArgs &a, cudaStream_t stream) {
    if (a.m == 0) return cudaSuccess;
    if (!AZ_CONJ_ONE_KERNEL) {
        conjunction_kernel<<<(a.m + kConjNearWarps - 1) / kConjNearWarps, kConjNearWarps * 32, 0, stream>>>(a);
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    conjunction_deep_kernel<<<(a.m + kConjDeepWarps - 1) / kConjDeepWarps, kConjDeepWarps * 32, 0, stream>>>(a);
    return cudaGetLastError();
}

}  // namespace az
