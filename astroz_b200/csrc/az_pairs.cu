// az_pairs.cu -- K6: propagate n arbitrary (satellite, time) queries in one device call.
//
// Replaces a loop of Satrec.sgp4(jd, fr) calls, one per observation (bindings/python/src/satrec.zig:169-201); the
// reference has no batched counterpart.  Pipeline on one stream:
//   1. key:   key[i] = the query's table position (near-earth table index, then nSgp4 + deep-space index; nRows for a
//             row outside the catalog), idx[i] = i;
//   2. sort:  cub::DeviceRadixSort::SortPairs on the bits the row count needs -- near-earth queries first, grouped by
//             satellite, then deep-space ones, then bad rows.  A warp then sees one or two satellites: its 39 column
//             loads are broadcasts of one 312-byte column set instead of 32 scattered gathers, and the isimp / irez
//             branches are warp-uniform except at group boundaries;
//   3. split: one thread finds the near / deep / bad boundaries in the sorted keys (nothing is read back);
//   4. sgp4_pairs_kernel over the near-earth segment, sdp4_pairs_kernel over the rest.  One query per thread; results
//             go to the query's original index.
#include "az_kernels.cuh"
#include "az_pairs.cuh"

#include <cub/device/device_radix_sort.cuh>

namespace az {

constexpr int kPairsThreads = 128;

__global__ void pairs_key_kernel(const uint32_t *__restrict__ sat, const uint32_t *__restrict__ rowKey, uint32_t nRows,
                                 uint32_t n, uint32_t *__restrict__ keys, uint32_t *__restrict__ idx) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t s = __ldg(sat + i);
    keys[i] = s < nRows ? __ldg(rowKey + s) : nRows;
    idx[i] = i;
}

// split[0] = first sorted position whose key is not near-earth, split[1] = first whose key is a bad row
__global__ void pairs_split_kernel(const uint32_t *__restrict__ keys, uint32_t n, uint32_t nSgp4, uint32_t nRows,
                                   uint32_t *__restrict__ split) {
    const uint32_t bound = threadIdx.x == 0 ? nSgp4 : nRows;
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (keys[mid] < bound) lo = mid + 1;
        else hi = mid;
    }
    split[threadIdx.x] = lo;
}

template <bool kVel>
__device__ __forceinline__ void pairs_store(const PairsArgs &a, uint32_t q, const CellOut &o, uint8_t st) {
    double *p = a.pos + (size_t)q * 3;
    __stcs(p, o.rx);
    __stcs(p + 1, o.ry);
    __stcs(p + 2, o.rz);
    if (kVel) {
        double *v = a.vel + (size_t)q * 3;
        __stcs(v, o.vx);
        __stcs(v + 1, o.vy);
        __stcs(v + 2, o.vz);
    }
    if (a.status) a.status[q] = st;
}

// Near-earth segment [0, split[0]) of the sorted queries, grid-stride.
template <int kMode, bool kVel>
__global__ void __launch_bounds__(kPairsThreads) sgp4_pairs_kernel(const PairsArgs a) {
    const uint32_t end = __ldg(a.split);
    for (uint32_t i = blockIdx.x * kPairsThreads + threadIdx.x; i < end; i += gridDim.x * kPairsThreads) {
        const uint32_t s = __ldg(a.keysSorted + i), q = __ldg(a.idxSorted + i);
        const double *base = a.sgp4Tiles + (size_t)(s / kTileSats) * kSgp4TileDoubles + (s % kTileSats);
        auto col = [base](int c) { return __ldg(base + c * kTileSats); };
        const double jdFull = add_rn(__ldg(a.jd + q), __ldg(a.fr + q));
        CellOut o;
        const uint8_t st = pairs_sgp4_query<kMode, kVel>(col, jdFull, a.refJd, __ldg(a.toff + s), a.g, o);
        pairs_store<kVel>(a, q, o, st);
    }
}

// Deep-space and bad-row segment [split[0], n), grid-stride.
template <int kMode, bool kVel>
__global__ void __launch_bounds__(kPairsThreads) sdp4_pairs_kernel(const PairsArgs a) {
    const uint32_t begin = __ldg(a.split), bad = __ldg(a.split + 1);
    for (uint32_t i = begin + blockIdx.x * kPairsThreads + threadIdx.x; i < a.n; i += gridDim.x * kPairsThreads) {
        const uint32_t q = __ldg(a.idxSorted + i);
        CellOut o;
        uint8_t st;
        if (i < bad) {
            const uint32_t d = __ldg(a.keysSorted + i) - a.nSgp4;
            const double jdFull = add_rn(__ldg(a.jd + q), __ldg(a.fr + q));
            st = pairs_sdp4_query<kMode, kVel>(a.sdp4[d], a.lattice + (size_t)d * 2 * a.latticeNodes, a.latticeNodes,
                                               jdFull, a.g, o);
        } else {  // not a catalog row: nothing is read for it
            o.rx = o.ry = o.rz = o.vx = o.vy = o.vz = 0.0;
            st = kCellBadSatellite;
        }
        pairs_store<kVel>(a, q, o, st);
    }
}

// Partial min / max of jd + fr: one pair per CTA, then one CTA folds the partials into range[0..1].
constexpr int kRangeThreads = 256;
constexpr int kRangeBlocks = 264;
__global__ void __launch_bounds__(kRangeThreads) pairs_range_kernel(const double *__restrict__ jd,
                                                                   const double *__restrict__ fr, uint32_t n,
                                                                   double *__restrict__ partial, double *range) {
    __shared__ double smin[kRangeThreads], smax[kRangeThreads];
    double lo = INFINITY, hi = -INFINITY;
    if (partial) {
        for (uint32_t i = blockIdx.x * kRangeThreads + threadIdx.x; i < n; i += gridDim.x * kRangeThreads) {
            const double j = add_rn(__ldg(jd + i), __ldg(fr + i));
            lo = fmin(lo, j);
            hi = fmax(hi, j);
        }
    } else {  // fold pass: jd = the partial minima, fr = the partial maxima
        for (uint32_t i = threadIdx.x; i < n; i += kRangeThreads) {
            lo = fmin(lo, jd[i]);
            hi = fmax(hi, fr[i]);
        }
    }
    smin[threadIdx.x] = lo;
    smax[threadIdx.x] = hi;
    __syncthreads();
    for (int w = kRangeThreads / 2; w > 0; w >>= 1) {
        if (threadIdx.x < w) {
            smin[threadIdx.x] = fmin(smin[threadIdx.x], smin[threadIdx.x + w]);
            smax[threadIdx.x] = fmax(smax[threadIdx.x], smax[threadIdx.x + w]);
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        if (partial) {
            partial[blockIdx.x] = smin[0];
            partial[kRangeBlocks + blockIdx.x] = smax[0];
        } else {
            range[0] = smin[0];
            range[1] = smax[0];
        }
    }
}

size_t pairs_range_scratch_doubles() { return 2 * kRangeBlocks + 2; }

cudaError_t launch_pairs_range(const double *jd, const double *fr, uint32_t n, double *scratch, cudaStream_t stream) {
    if (n == 0) return cudaErrorInvalidValue;
    const uint32_t blocks = std::min<uint32_t>(kRangeBlocks, (n + kRangeThreads - 1) / kRangeThreads);
    double *partial = scratch + 2;
    pairs_range_kernel<<<blocks, kRangeThreads, 0, stream>>>(jd, fr, n, partial, nullptr);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    pairs_range_kernel<<<1, kRangeThreads, 0, stream>>>(partial, partial + kRangeBlocks, blocks, nullptr, scratch);
    return cudaGetLastError();
}

static int sort_bits(uint32_t nRows) {
    int bits = 1;
    while (bits < 32 && (nRows >> bits) != 0) ++bits;  // keys run 0 .. nRows inclusive
    return bits;
}

cudaError_t pairs_sort_scratch_bytes(uint32_t n, uint32_t nRows, size_t *bytes) {
    *bytes = 0;
    return cub::DeviceRadixSort::SortPairs(nullptr, *bytes, (const uint32_t *)nullptr, (uint32_t *)nullptr,
                                           (const uint32_t *)nullptr, (uint32_t *)nullptr, (int)n, 0, sort_bits(nRows));
}

static int resident_ctas() {
    static int cached[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132 * 16;
    if (cached[dev] == 0) {
        int sms = 0;
        if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
        cached[dev] = sms * 16;
    }
    return cached[dev];
}

template <int kMode, bool kVel>
static cudaError_t launch_pairs_kernels(const PairsArgs &a, uint32_t ctas, cudaStream_t stream) {
    if (a.nSgp4) {
        sgp4_pairs_kernel<kMode, kVel><<<ctas, kPairsThreads, 0, stream>>>(a);
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    sdp4_pairs_kernel<kMode, kVel><<<ctas, kPairsThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_pairs(const PairsArgs &a, int mode, cudaStream_t stream) {
    if (a.n == 0) return cudaSuccess;
    if (mode < 0 || mode > 2) return cudaErrorInvalidValue;
    const uint32_t blocks = (a.n + kPairsThreads - 1) / kPairsThreads;
    pairs_key_kernel<<<blocks, kPairsThreads, 0, stream>>>(a.sat, a.rowKey, a.nRows, a.n, a.keys, a.idx);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    size_t bytes = a.sortScratchBytes;
    e = cub::DeviceRadixSort::SortPairs(a.sortScratch, bytes, a.keys, a.keysSorted, a.idx, a.idxSorted, (int)a.n, 0,
                                        sort_bits(a.nRows), stream);
    if (e != cudaSuccess) return e;
    pairs_split_kernel<<<1, 2, 0, stream>>>(a.keysSorted, a.n, a.nSgp4, a.nRows, a.split);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    const uint32_t ctas = std::min<uint32_t>(blocks, (uint32_t)resident_ctas());
    const bool vel = a.vel != nullptr;
    if (mode == 0) return vel ? launch_pairs_kernels<0, true>(a, ctas, stream) : launch_pairs_kernels<0, false>(a, ctas, stream);
    if (mode == 1) return vel ? launch_pairs_kernels<1, true>(a, ctas, stream) : launch_pairs_kernels<1, false>(a, ctas, stream);
    return vel ? launch_pairs_kernels<2, true>(a, ctas, stream) : launch_pairs_kernels<2, false>(a, ctas, stream);
}

}  // namespace az
