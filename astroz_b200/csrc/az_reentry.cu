// az_reentry.cu -- K19: reentry prediction of catalogue rows and their covariance draws (az_reentry.cuh).
//
// Four steps on one stream:
//   1. reentry_build_kernel, one thread per request: the request's status, K14's nominal variables and factor, B_row,
//      epoch and model into the scratch; counts zeroed, the words no trajectory writes filled; and the request's work
//      items into four quarters of one array: near-earth sample items (ceil(samples / 32) blocks of 32 consecutive
//      samples), near-earth nominal flags, then the same two for deep-space rows;
//   2. a CUB inclusive scan of that array (K14's work-item scan over four quarters instead of two);
//   3. reentry_kernel (near-earth) and reentry_deep_kernel, persistent grids whose warps stride over their class's
//      items: first the sample items, each one row's 32 samples, then the nominal items, 32 consecutive nominals of the
//      class, each lane's request found by binary search in the prefix.  Each lane builds its set in the warp's shared
//      slot, takes its epoch state and integrates its own trajectory; lane 0 adds a sample item's counts with 64-bit
//      atomics.
// No floating-point sum crosses trajectories: the counts are integer sums, so no byte depends on the launch shape, the
// batch or the order of the work items.
#include "../../include/astroz_b200.h"
#include "az_conjunction_mc_warp.cuh"
#include "az_reentry.cuh"

namespace az {

static_assert(ASTROZ_REENTRY_RECORD_WORDS == kReRecordWords && ASTROZ_REENTRY_SAMPLE_WORDS == kReSampleWords &&
                  ASTROZ_REENTRY_COUNT_WORDS == kReCountWords && ASTROZ_REENTRY_STATE_WORDS == kReStateWords,
              "reentry layouts");
static_assert(ASTROZ_REENTRY_OK == kReOk && ASTROZ_REENTRY_INIT_FAILED == kReInitFailed &&
                  ASTROZ_REENTRY_NOT_PSD == kReNotPsd && ASTROZ_REENTRY_BAD_ROW == kReBadRow,
              "reentry request statuses");
static_assert(ASTROZ_REENTRY_TRAJ_REENTERED == kReReentered && ASTROZ_REENTRY_TRAJ_ABOVE == kReAbove &&
                  ASTROZ_REENTRY_TRAJ_INIT_FAILED == kReTrajInitFailed &&
                  ASTROZ_REENTRY_TRAJ_NONPHYSICAL == kReNonphysical && ASTROZ_REENTRY_TRAJ_STOPPED == kReStopped,
              "reentry trajectory statuses");

constexpr uint32_t kReLanes = 32;   // trajectories per work item
constexpr int kReWarps = 2;
constexpr int kReBuildThreads = 128;

template <bool kDeep>
struct ReWarpSmem;
template <>
struct ReWarpSmem<false> {
    union {
        double cols[kReLanes][kSgp4Cols];   // the sets, until each lane has its epoch state ...
        double y[kReLanes][6];              // ... then each lane's interval start state
    };
};
template <>
struct ReWarpSmem<true> {
    union {
        Sdp4Sat sets[kReLanes];
        double y[kReLanes][6];
    };
};

// The scratch: rows[m] (256-byte aligned), items[4m] and prefix[4m] (u64), then the scan's temporary storage
static size_t re_rows_bytes(uint32_t m) { return ((size_t)sizeof(ReentryRow) * m + 255) & ~size_t(255); }
static size_t re_items_bytes(uint32_t m) { return ((size_t)64 * m + 255) & ~size_t(255); }

__global__ void __launch_bounds__(kReBuildThreads) reentry_build_kernel(const ReentryArgs a, ReentryRow *rows,
                                                                         uint64_t *items) {
    const uint32_t i = blockIdx.x * kReBuildThreads + threadIdx.x;
    if (i >= a.m) return;
    const double nan = std::numeric_limits<double>::quiet_NaN();
    const uint32_t row = __ldg(a.rows + i);
    ReentryRow R;
    R.B = nan;
    R.model = 0;
    R.status = kReBadRow;
    if (row < a.n) {
        double el[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) el[c] = __ldg(a.elements + (size_t)c * a.n + row);
        const int model = a.model ? (int)__ldg(a.model + row) : 0;
        reentry_row(el, a.covariance + (size_t)row * kFitN, model, gravity(a.grav), a.ballistic != nullptr,
                    a.ballistic ? __ldg(a.ballistic + i) : 0.0, R);
    }
    rows[i] = R;
    a.status[i] = (uint8_t)R.status;
    for (int q = 0; q < kReCountWords; ++q) a.counts[(size_t)i * kReCountWords + q] = 0;
    const bool ok = R.status == kReOk, deep = R.model != 0;
    const uint64_t samples = __ldg(a.samples + i);
    const uint64_t n = ok ? mc_items(samples, kReLanes) : 0;
    items[i] = deep ? 0 : n;
    items[(size_t)a.m + i] = ok && !deep ? 1 : 0;
    items[(size_t)2 * a.m + i] = deep ? n : 0;
    items[(size_t)3 * a.m + i] = ok && deep ? 1 : 0;
    if (!ok) {   // the nominal is not run
        double *o = a.out + (size_t)i * kReRecordWords;
        for (int q = 0; q < 5; ++q) o[q] = nan;
        o[5] = R.B;
        o[6] = o[7] = 0.0;
        if (a.states)
            for (int q = 0; q < kReStateWords; ++q) a.states[(size_t)i * kReStateWords + q] = nan;
        a.nominalStatus[i] = kReTrajInitFailed;
    }
    // the rows no sample writes: past samples[i], or every row of a request that is not OK
    const uint64_t from = ok ? (samples < a.record ? samples : a.record) : 0;
    for (uint64_t r = from; r < a.record; ++r)
        for (int q = 0; q < kReSampleWords; ++q) a.sampleOut[((size_t)i * a.record + r) * kReSampleWords + q] = nan;
}

// Work item q of one class: sample items first, then nominal items
template <bool kDeep>
__device__ __forceinline__ void re_item(const ReentryArgs &a, const ReentryRow *rows, const uint64_t *prefix,
                                        uint64_t q, ReWarpSmem<kDeep> &w, uint32_t lane) {
    const ReentryCall &c = a.call;
    const uint64_t *sp = prefix + (kDeep ? (size_t)2 * a.m : 0), *np = sp + a.m;
    const uint64_t lo = kDeep ? prefix[(size_t)2 * a.m - 1] : 0, sEnd = sp[a.m - 1];
    const bool sample = q < sEnd - lo;
    uint32_t i = 0;
    uint64_t j = 0, k = 0, seed = 0;
    bool valid;
    if (sample) {   // one row's samples blk 32 .. blk 32 + 31
        const uint64_t qq = lo + q;
        i = mc_candidate(sp, a.m, qq);
        const uint64_t blk = qq - (i ? sp[i - 1] : lo);
        j = blk * kReLanes + lane;
        valid = j < __ldg(a.samples + i);
        k = (a.first ? __ldg(a.first + i) : 0) + j;
        seed = a.seed ? __ldg(a.seed + i) : 0;
    } else {        // 32 consecutive nominals of the class
        const uint64_t v = (q - (sEnd - lo)) * kReLanes + lane;
        valid = v < np[a.m - 1] - sEnd;
        if (valid) i = mc_candidate(np, a.m, sEnd + v);
    }
    const ReentryRow &R = rows[i];
    double x[kFitVars], B = 0.0, f = 1.0, y0[6];
    bool built = false;
    __syncwarp();   // every lane is done with the previous item's slot
    if (valid) {
        const Gravity grav = gravity(a.grav);   // formed here: it is dead once the set is built
        reentry_params(R, sample, seed, k, c.sigma, x, B, f);
        if constexpr (kDeep) built = reentry_epoch_deep(x, R.epoch, grav, a.g, w.sets[lane], y0);
        else built = reentry_epoch_near(x, R.epoch, grav, a.g, w.cols[lane], y0);
    }
    ReentryOut o;
    o.counts[0] = o.counts[1] = 0;
    __syncwarp();   // every lane has its epoch state: the slot now holds the start states
    if (valid) {
        if (built) reentry_integrate(y0, R.epoch, B, f, c, w.y[lane], o);
        else reentry_fail(o, kReTrajInitFailed);
        if (sample) {
            if (j < a.record) {
                double *d = a.sampleOut + ((size_t)i * a.record + j) * kReSampleWords;
                d[0] = o.dt;
                d[1] = o.lat;
                d[2] = o.lon;
                d[3] = (double)(o.counts[0] + o.counts[1]);
            }
        } else {
            double *d = a.out + (size_t)i * kReRecordWords;
            d[0] = o.dt;
            d[1] = o.lat;
            d[2] = o.lon;
            d[3] = o.speed;
            d[4] = o.fpa;
            d[5] = B;
            d[6] = (double)o.counts[0];
            d[7] = (double)o.counts[1];
            if (a.states)
                for (int q2 = 0; q2 < kReStateWords; ++q2) a.states[(size_t)i * kReStateWords + q2] = o.y[q2];
            a.nominalStatus[i] = o.status;
        }
    }
    if (sample) {   // warp-uniform: a sample item is one row's
        const uint32_t re = __popc(__ballot_sync(0xffffffffu, valid && o.status == kReReentered));
        const uint32_t ab = __popc(__ballot_sync(0xffffffffu, valid && o.status == kReAbove));
        const uint32_t fa = __popc(__ballot_sync(0xffffffffu, valid && reentry_failed(o.status)));
        if (lane == 0) {
            unsigned long long *cn = reinterpret_cast<unsigned long long *>(a.counts + (size_t)i * kReCountWords);
            if (re) atomicAdd(cn, (unsigned long long)re);
            if (ab) atomicAdd(cn + 1, (unsigned long long)ab);
            if (fa) atomicAdd(cn + 2, (unsigned long long)fa);
        }
    }
}

// Persistent warps over one class's items
template <bool kDeep>
__device__ __forceinline__ void re_run(const ReentryArgs &a, const ReentryRow *rows, const uint64_t *prefix,
                                       ReWarpSmem<kDeep> &w) {
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint64_t *sp = prefix + (kDeep ? (size_t)2 * a.m : 0), *np = sp + a.m;
    const uint64_t lo = kDeep ? prefix[(size_t)2 * a.m - 1] : 0, sEnd = sp[a.m - 1];
    const uint64_t total = (sEnd - lo) + mc_items(np[a.m - 1] - sEnd, kReLanes);
    for (uint64_t q = blockIdx.x * (uint64_t)kReWarps + warp; q < total; q += (uint64_t)gridDim.x * kReWarps)
        re_item<kDeep>(a, rows, prefix, q, w, lane);
}

__global__ void __launch_bounds__(kReWarps * 32) reentry_kernel(const ReentryArgs a, const ReentryRow *rows,
                                                                 const uint64_t *prefix) {
    __shared__ ReWarpSmem<false> smem[kReWarps];
    re_run<false>(a, rows, prefix, smem[threadIdx.x >> 5]);
}

__global__ void __launch_bounds__(kReWarps * 32) reentry_deep_kernel(const ReentryArgs a, const ReentryRow *rows,
                                                                      const uint64_t *prefix) {
    __shared__ ReWarpSmem<true> smem[kReWarps];
    re_run<true>(a, rows, prefix, smem[threadIdx.x >> 5]);
}

cudaError_t reentry_scratch_bytes(uint32_t m, size_t *bytes) {
    size_t scan = 0;
    const cudaError_t e = cub::DeviceScan::InclusiveSum(nullptr, scan, (const uint64_t *)nullptr, (uint64_t *)nullptr,
                                                        (uint64_t)4 * (m ? m : 1));
    *bytes = re_rows_bytes(m) + re_items_bytes(m) + scan;
    return e;
}

cudaError_t launch_reentry(const ReentryArgs &a, cudaStream_t stream) {
    if (a.m == 0) return cudaSuccess;
    char *base = static_cast<char *>(a.scratch);
    ReentryRow *rows = reinterpret_cast<ReentryRow *>(base);
    uint64_t *items = reinterpret_cast<uint64_t *>(base + re_rows_bytes(a.m)), *prefix = items + (size_t)4 * a.m;
    reentry_build_kernel<<<(a.m + kReBuildThreads - 1) / kReBuildThreads, kReBuildThreads, 0, stream>>>(a, rows, items);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    size_t scan = 0;
    if ((e = reentry_scratch_bytes(a.m, &scan)) != cudaSuccess) return e;
    scan -= re_rows_bytes(a.m) + re_items_bytes(a.m);
    e = cub::DeviceScan::InclusiveSum(base + re_rows_bytes(a.m) + re_items_bytes(a.m), scan, items, prefix,
                                      (uint64_t)4 * a.m, stream);
    if (e != cudaSuccess) return e;
    int blocks = 0;
    if ((e = mc_grid(reinterpret_cast<const void *>(reentry_kernel), kReWarps * 32, &blocks)) != cudaSuccess) return e;
    reentry_kernel<<<blocks, kReWarps * 32, 0, stream>>>(a, rows, prefix);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    if ((e = mc_grid(reinterpret_cast<const void *>(reentry_deep_kernel), kReWarps * 32, &blocks)) != cudaSuccess)
        return e;
    reentry_deep_kernel<<<blocks, kReWarps * 32, 0, stream>>>(a, rows, prefix);
    return cudaGetLastError();
}

}  // namespace az
