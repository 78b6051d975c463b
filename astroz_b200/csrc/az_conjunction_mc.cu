// az_conjunction_mc.cu -- K14: Monte Carlo collision probability of candidate conjunctions (az_conjunction_mc.cuh).
//
// Four steps on one stream:
//   1. mc_prepare_kernel, one thread per candidate: the status (bad pair, model byte, nominal sets, factors), counts
//      zeroed, the NaN rows of sample_out that no sample writes, and the candidate's work items -- ceil(samples / B)
//      blocks of B consecutive samples, B = 16 for a pair of near-earth rows and 8 otherwise -- into two halves of one
//      array (near-earth pairs, then every other pair);
//   2. a CUB inclusive scan of that array into the prefix of work items;
//   3. conjunction_mc_kernel and conjunction_mc_deep_kernel, persistent grids whose warps stride over their half's
//      work items, each item's candidate found by binary search in the prefix.  Lanes (row, sample) draw and build the
//      2B sets into the warp's shared-memory slots (deep space: then lanes (row, sample, direction) build the 32
//      lattices); the warp then runs conj_tca on each sample in turn, one evaluation per lane per row per round, and
//      lane 0 stores the samples' words and adds the block's (hits, edge, failed) with 64-bit atomics.
// No floating-point sum crosses samples or candidates: the counts are integer sums, so no result depends on the launch
// shape, the batch or the order of the work items.
#include "az_conjunction_mc_warp.cuh"

namespace az {

__global__ void __launch_bounds__(kMcPrepThreads) mc_prepare_kernel(const ConjMcArgs a, uint64_t *items) {
    const uint32_t i = blockIdx.x * kMcPrepThreads + threadIdx.x;
    if (i >= a.m) return;
    uint32_t idx[2];
    int mdl[2];
    uint8_t st = kConjBadPair;
    const bool bad = mc_bad(a, i, idx, mdl);
    if (!bad) {
        const Gravity grav = gravity(a.grav);
        uint8_t so[2];
        for (int o = 0; o < 2; ++o) {
            double el[8], xh[kFitVars];
            McFactor F;
            mc_load_el(a, idx[o], el);
            so[o] = mc_row(el, a.covariance + (size_t)idx[o] * kFitN, mdl[o], grav, xh, F);
        }
        st = mc_status(so[0], so[1]);
    }
    a.status[i] = st;
    for (int q = 0; q < kMcCountWords; ++q) a.counts[(size_t)i * kMcCountWords + q] = 0;
    const uint64_t samples = __ldg(a.samples + i);
    const bool near = !bad && mdl[0] == 0 && mdl[1] == 0;
    const uint64_t n = st == kConjOk ? mc_items(samples, near ? kMcNearB : kMcDeepB) : 0;
    items[i] = near ? n : 0;
    items[(size_t)a.m + i] = near ? 0 : n;
    // the rows no sample writes: past samples[i], or every row of a failed candidate
    const uint64_t from = st == kConjOk ? (samples < a.record ? samples : a.record) : 0;
    for (uint64_t r = from; r < a.record; ++r)
        for (int q = 0; q < kMcSampleWords; ++q)
            a.sampleOut[((size_t)i * a.record + r) * kMcSampleWords + q] = std::numeric_limits<double>::quiet_NaN();
}

__global__ void __launch_bounds__(kMcNearWarps * 32) conjunction_mc_kernel(const ConjMcArgs a, const uint64_t *prefix) {
    __shared__ McWarpSmem<false> smem[kMcNearWarps];
    const uint32_t warp = threadIdx.x >> 5;
    mc_run<false>(a, prefix, 0, smem[warp], warp, kMcNearWarps);
}

__global__ void __launch_bounds__(kMcDeepWarps * 32) conjunction_mc_deep_kernel(const ConjMcArgs a,
                                                                                const uint64_t *prefix) {
    __shared__ McWarpSmem<true> smem[kMcDeepWarps];
    const uint32_t warp = threadIdx.x >> 5;
    mc_run<true>(a, prefix + a.m, prefix[a.m - 1], smem[warp], warp, kMcDeepWarps);
}

cudaError_t conj_mc_scratch_bytes(uint32_t m, size_t *bytes) {
    size_t scan = 0;
    const cudaError_t e = cub::DeviceScan::InclusiveSum(nullptr, scan, (const uint64_t *)nullptr, (uint64_t *)nullptr,
                                                        (uint64_t)2 * (m ? m : 1));
    *bytes = mc_scan_offset(m) + scan;
    return e;
}

cudaError_t launch_conjunction_mc(const ConjMcArgs &a, cudaStream_t stream) {
    if (a.m == 0) return cudaSuccess;
    return mc_launch(a, mc_prepare_kernel, conjunction_mc_kernel, conjunction_mc_deep_kernel, a.scratch, stream);
}

}  // namespace az
