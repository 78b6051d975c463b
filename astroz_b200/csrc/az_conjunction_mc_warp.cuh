// az_conjunction_mc_warp.cuh -- the warp-level work of K14 (az_conjunction_mc.cu) and K15 (az_conjunction_is.cu):
// the persistent item loop, shared by a compile-time flag.  The Args type chooses it: ConjMcArgs
// is K14's plain sampling, ConjIsArgs K15's, which adds its candidate's shift to the normals, records log w and sums
// the hits' weights (az_conjunction_is.cuh).  Also the one launch sequence of both (mc_launch).
#pragma once

#include <cub/device/device_scan.cuh>
#include <limits>
#include <type_traits>

#include "az_conjunction_is.cuh"
#include "az_kernels.cuh"

namespace az {

constexpr uint32_t kMcNearB = 16, kMcDeepB = 8;   // samples per work item
constexpr int kMcNearWarps = 4;
constexpr int kMcDeepWarps = 2;
constexpr int kMcPrepThreads = 128;

template <class Args>
constexpr bool mc_is() { return std::is_same<Args, ConjIsArgs>::value; }

struct McNearSlot {
    double cols[kMcNearB][kSgp4Cols];
};
struct McDeepSlot {
    union {
        double cols[kMcDeepB][kSgp4Cols];
        struct {
            Sdp4Sat sets[kMcDeepB];
            double2 lattice[kMcDeepB][2 * kFitLatticeNodes];
        } ds;
    };
};

template <bool kDeep>
struct McWarpSmem {
    typename std::conditional<kDeep, McDeepSlot, McNearSlot>::type obj[2];
};

template <bool kDeep>
__device__ __forceinline__ bool mc_eval(const McWarpSmem<kDeep> &w, int o, int deep, int k, double ts,
                                        const GravConsts &g, double (&f)[6]) {
    if constexpr (kDeep) {
        if (deep) return conj_eval_deep(w.obj[o].ds.sets[k], w.obj[o].ds.lattice[k], ts, g, f);
    }
    return conj_eval_near([&w, o, k](int c) { return w.obj[o].cols[k][c]; }, ts, g, f);
}

// K11's warp sampler on the drawn sets of one sample: lane l evaluates sample l of the round for both rows
template <bool kDeep>
struct McWarpSampler {
    const McWarpSmem<kDeep> &w;
    const GravConsts &gc;
    double ts0[2];
    int deep[2];
    int set;
    uint32_t lane;
    double gv = 0.0, dv2 = 0.0;
    bool ok = true;
    __device__ uint32_t round(double a, double b) {
        const double t = conj_node(a, b, (int)lane);
        double fp[6], fs[6];
        ok = mc_eval(w, 0, deep[0], set, ts0[0] + t, gc, fp) && ok;
        ok = mc_eval(w, 1, deep[1], set, ts0[1] + t, gc, fs) && ok;
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

__device__ __forceinline__ bool mc_bad(const ConjMcArgs &a, uint32_t i, uint32_t (&idx)[2], int (&mdl)[2]) {
    idx[0] = __ldg(a.primary + i);
    idx[1] = __ldg(a.secondary + i);
    const bool bad = idx[0] >= a.n || idx[1] >= a.n || idx[0] == idx[1];
    mdl[0] = bad || !a.model ? 0 : (int)__ldg(a.model + idx[0]);
    mdl[1] = bad || !a.model ? 0 : (int)__ldg(a.model + idx[1]);
    return bad;
}

__device__ __forceinline__ void mc_load_el(const ConjMcArgs &a, uint32_t row, double (&el)[8]) {
#pragma unroll
    for (int c = 0; c < 8; ++c) el[c] = __ldg(a.elements + (size_t)c * a.n + row);
}

// A 256-bit sum S (four u64, least significant first) added to the words at g, the carries passed upward
__device__ __forceinline__ void is_atomic_add256(unsigned long long *g, const uint64_t (&S)[4]) {
    unsigned long long carry = 0;
    for (int k = 0; k < 4; ++k) {
        const unsigned long long add = S[k] + carry;
        unsigned long long next = add < carry ? 1 : 0;
        if (add) {
            const unsigned long long old = atomicAdd(g + k, add);
            next += old + add < old ? 1 : 0;
        }
        carry = next;
    }
}

// One work item: candidate i, samples blk B .. blk B + B - 1 counted from first
template <bool kDeep, class Args>
__device__ __forceinline__ void mc_item(const Args &a, uint32_t i, uint64_t blk, McWarpSmem<kDeep> &w,
                                        uint32_t lane) {
    constexpr bool kIs = mc_is<Args>();
    constexpr uint32_t B = kDeep ? kMcDeepB : kMcNearB;
    uint32_t idx[2];
    int mdl[2];
    mc_bad(a, i, idx, mdl);
    const Gravity grav = gravity(a.grav);
    const double jdFull = add_rn(__ldg(a.jd + i), __ldg(a.fr + i)), win = __ldg(a.window + i), R = __ldg(a.hbr + i);
    const uint64_t samples = __ldg(a.samples + i), first = a.first ? __ldg(a.first + i) : 0;
    const uint64_t seed = a.seed ? __ldg(a.seed + i) : 0;
    const uint64_t base = blk * B;                                   // sample offset of the item's first sample
    const uint32_t valid = samples - base < B ? (uint32_t)(samples - base) : B;
    const double ts0[2] = {pairs_tsince_deep(jdFull, __ldg(a.elements + idx[0])),
                           pairs_tsince_deep(jdFull, __ldg(a.elements + idx[1]))};
    // lanes (o, j): row o draws and builds its set of sample j
    const uint32_t o = kDeep ? (lane >> 3) & 1 : lane >> 4, j = lane & (B - 1);
    const bool mine = (!kDeep || lane < 2 * B) && j < valid;
    __syncwarp();   // every lane is done with the previous item's slots
    bool ok = false;
    double uc = 0.0;   // K15: u . c over row o's normals of sample j
    if (mine) {
        double el[8], xh[kFitVars], z[kFitVars], x[kFitVars], inv;
        McFactor F;
        mc_load_el(a, idx[o], el);
        const double *P = a.covariance + (size_t)idx[o] * kFitN;
        mc_factor(P, cov_nvar(P), F);   // positive semidefinite: the prepare step checked it
        mc_row_normals(seed, first + base + j, (int)o, z);
        if constexpr (kIs) uc = is_shift_normals(a.prop + (size_t)i * kIsProposalWords + kFitVars * o, z);
        if (kDeep && mdl[o]) {
            FitDeepSpace::vars_of(el, xh);
            mc_draw(F, xh, z, x);
            if constexpr (kDeep) ok = fit_build_set_of<FitDeepSpace>(x, 0, el[0], grav, w.obj[o].ds.sets[j], inv);
        } else {
            FitNearEarth::vars_of(el, xh);
            mc_draw(F, xh, z, x);
            ok = fit_build_set_of<FitNearEarth>(x, 0, el[0], grav, w.obj[o].cols[j], inv);
        }
    }
    const uint32_t built = __ballot_sync(0xffffffffu, ok);   // bit o B + j: row o's set of sample j
    __syncwarp();
    if constexpr (kDeep) {   // lanes (row, sample, direction): the lattices over [ts0 - w, ts0 + w]
        const uint32_t lo_ = lane >> 4, set = (lane >> 1) & 7, dir = lane & 1;
        if (mdl[lo_] && (built >> (lo_ * B + set) & 1u)) {
            const double hi = ts0[lo_] + win, lo = ts0[lo_] - win;
            const int nodes = fit_lattice_nodes(dir == 0 ? (hi > 0.0 ? hi : 0.0) : (lo < 0.0 ? -lo : 0.0));
            fit_deep_lattice(w.obj[lo_].ds.sets[set], (int)dir, nodes, w.obj[lo_].ds.lattice[set]);
        }
        __syncwarp();
    }
    uint64_t hits = 0, edge = 0, failed = 0;
    uint64_t overflow = 0, V[4] = {0, 0, 0, 0}, V2[4] = {0, 0, 0, 0};
    const bool rec = base < a.record;
    for (uint32_t s = 0; s < valid; ++s) {
        double out0 = std::numeric_limits<double>::quiet_NaN(), out1 = out0, out2 = out0;
        double ucs = 0.0;   // K15: u . c of sample s, the primary's part plus the secondary's
        if constexpr (kIs) ucs = __shfl_sync(0xffffffffu, uc, (int)s) + __shfl_sync(0xffffffffu, uc, (int)(B + s));
        if ((built >> s & 1u) && (built >> (B + s) & 1u)) {
            McWarpSampler<kDeep> S{w, a.g, {ts0[0], ts0[1]}, {mdl[0], mdl[1]}, (int)s, lane};
            double tca = 0.0;
            const uint8_t st = conj_tca(S, win, tca);
            double fp[6], fs[6];
            bool good = mc_eval(w, 0, mdl[0], (int)s, ts0[0] + tca, a.g, fp) && S.ok;
            good = mc_eval(w, 1, mdl[1], (int)s, ts0[1] + tca, a.g, fs) && good;
            const double miss = mc_miss(fp, fs);
            if (__all_sync(0xffffffffu, good && std::isfinite(miss))) {
                hits += miss < R ? 1 : 0;
                edge += st == kConjWindowEdge ? 1 : 0;
                out0 = tca;
                out1 = miss;
                if constexpr (kIs) {
                    out2 = -ucs + a.prop[(size_t)i * kIsProposalWords + kIsShift];
                    if (lane == 0 && miss < R) is_hit(exp(-ucs), V, V2, overflow);
                }
            } else {
                ++failed;
            }
        } else {
            ++failed;
        }
        if (lane == 0 && rec && base + s < a.record) {
            constexpr int kSample = kIs ? kIsSampleWords : kMcSampleWords;
            double *d = a.sampleOut + ((size_t)i * a.record + base + s) * kSample;
            d[0] = out0;
            d[1] = out1;
            if constexpr (kIs) d[2] = out2;
        }
    }
    if (lane == 0) {
        constexpr int kCount = kIs ? kIsCountWords : kMcCountWords;
        unsigned long long *c = reinterpret_cast<unsigned long long *>(a.counts + (size_t)i * kCount);
        if (hits) atomicAdd(c, (unsigned long long)hits);
        if (edge) atomicAdd(c + 1, (unsigned long long)edge);
        if (failed) atomicAdd(c + 2, (unsigned long long)failed);
        if constexpr (kIs) {
            if (overflow) atomicAdd(c + 3, (unsigned long long)overflow);
            is_atomic_add256(c + kIsCountV, V);
            is_atomic_add256(c + kIsCountV2, V2);
        }
    }
}

// Persistent warps over the work items of one half of the prefix: items [lo, prefix[m - 1]) of `prefix`
template <bool kDeep, class Args>
__device__ __forceinline__ void mc_run(const Args &a, const uint64_t *prefix, uint64_t lo, McWarpSmem<kDeep> &w,
                                       uint32_t warp, uint32_t warps) {
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t total = prefix[a.m - 1];
    for (uint64_t q = lo + blockIdx.x * (uint64_t)warps + warp; q < total; q += (uint64_t)gridDim.x * warps) {
        const uint32_t i = mc_candidate(prefix, a.m, q);
        const uint64_t start = i ? prefix[i - 1] : lo;
        mc_item<kDeep>(a, i, q - start, w, lane);
    }
}

// The scratch of the sampling steps: items[2m], prefix[2m] (u64), then the scan's temporary storage at a 256-byte
// offset
inline size_t mc_scan_offset(uint32_t m) { return ((size_t)32 * m + 255) & ~size_t(255); }

static cudaError_t mc_grid(const void *kernel, int threads, int *blocks) {
    int dev = 0, sms = 0, per = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, kernel, threads, 0);
    *blocks = sms * (per > 0 ? per : 1);
    return e;
}

// Candidate statuses and work items (prepare), their scan into the scratch at `scratch`, then the near-earth pairs'
// items (nearKernel) and every other pair's (deepKernel) on persistent grids
template <class Args>
cudaError_t mc_launch(const Args &a, void (*prepare)(const Args, uint64_t *),
                      void (*nearKernel)(const Args, const uint64_t *), void (*deepKernel)(const Args, const uint64_t *),
                      void *scratch, cudaStream_t stream) {
    uint64_t *items = static_cast<uint64_t *>(scratch), *prefix = items + (size_t)2 * a.m;
    prepare<<<(a.m + kMcPrepThreads - 1) / kMcPrepThreads, kMcPrepThreads, 0, stream>>>(a, items);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    size_t scan = 0;
    if ((e = conj_mc_scratch_bytes(a.m, &scan)) != cudaSuccess) return e;
    scan -= mc_scan_offset(a.m);
    e = cub::DeviceScan::InclusiveSum(static_cast<char *>(scratch) + mc_scan_offset(a.m), scan, items, prefix,
                                      (uint64_t)2 * a.m, stream);
    if (e != cudaSuccess) return e;
    int blocks = 0;
    if ((e = mc_grid(reinterpret_cast<const void *>(nearKernel), kMcNearWarps * 32, &blocks)) != cudaSuccess) return e;
    nearKernel<<<blocks, kMcNearWarps * 32, 0, stream>>>(a, prefix);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    if ((e = mc_grid(reinterpret_cast<const void *>(deepKernel), kMcDeepWarps * 32, &blocks)) != cudaSuccess) return e;
    deepKernel<<<blocks, kMcDeepWarps * 32, 0, stream>>>(a, prefix);
    return cudaGetLastError();
}

}  // namespace az
