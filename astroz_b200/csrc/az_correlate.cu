// az_correlate.cu -- K12: sensor tracks correlated with catalogue rows (az_correlate.cuh).
//
// A dense sweep of (track, row) pairs.  correlate_gate_kernel counts each track's used residuals and forms its gate,
// one thread per track.  A scoring CTA takes one chunk of kCorrThreads tracks (one thread each) and one chunk of
// consecutive rows (corr_shape).  It streams the chunk's rows through shared memory kCorrWarps at a time, each warp
// building one row's nominal and stepped sets (lanes 0 .. nvar; deep space also the K2a lattices over the CTA's span of
// observation times, which fit_deep_eval does not depend on), so a row's sets are built once per CTA visit, never once
// per pair.  The stages are double-buffered: the warps build stage s + 1 and then score stage s, one barrier per stage.
// Every thread runs its whole track against each row of the stage (sums in track order, corr_pair_sums), keeps its
// ordered list in registers and counts the in-gate and failed pairs; at the end it stores the chunk's list and counts
// to scratch.  correlate_kernel scores the near-earth rows (model 0; a model byte > 1 fails init there) and
// correlate_deep_kernel the deep-space rows (model 1); each leaves the other's rows alone.  correlate_merge_kernel
// merges a track's row-chunk lists in (d^2, row) order and sums the integer counts, so no byte depends on the shape.
#include "az_correlate.cuh"
#include "az_kernels.cuh"

namespace az {

constexpr int kCorrStages = 2;   // the double buffer

struct CorrNearRow {
    double sets[kFitSets][kSgp4Cols];
};
struct CorrDeepRow {
    Sdp4Sat sets[kFitSets];
    double2 lattice[kFitSets][2 * kFitLatticeNodes];
};

template <typename Row>
struct CorrSmem {
    Row row[kCorrStages][kCorrWarps];
    double inv[kCorrStages][kCorrWarps][kFitSets];
    double P[kCorrStages][kCorrWarps][kFitN];
    double epoch[kCorrStages][kCorrWarps];
    uint32_t index[kCorrStages][kCorrWarps];
    int nvar[kCorrStages][kCorrWarps];   // -1: no row to score in this slot
    double span[kCorrWarps][2];          // the CTA's earliest and latest observation jdFull
};

// The row class each kernel scores
struct CorrNear {
    using Row = CorrNearRow;
    using Model = FitNearEarth;
    static constexpr int kClass = 0;
    __device__ static bool takes(uint8_t model) { return model != 1; }
    __device__ static void lattices(Row &, int, double, double, double, uint32_t) {}
    __device__ static auto evaluator(const Row &r, const GravConsts &g) {
        return [&r, &g](int k, double, const double (&ts)[1], double (&f)[6]) {
            CellOut o[1];
            sgp4_cell<1>([&r, k](int c) { return r.sets[k][c]; }, ts, g, o);
            f[0] = o[0].rx; f[1] = o[0].ry; f[2] = o[0].rz;
            f[3] = o[0].vx; f[4] = o[0].vy; f[5] = o[0].vz;
            return true;
        };
    }
};

struct CorrDeep {
    using Row = CorrDeepRow;
    using Model = FitDeepSpace;
    static constexpr int kClass = 1;
    __device__ static bool takes(uint8_t model) { return model == 1; }
    // lanes 2k + dir build direction dir of set k's lattice over [jdLo, jdHi]
    __device__ static void lattices(Row &r, int nvar, double epoch, double jdLo, double jdHi, uint32_t lane) {
        const double hi = pairs_tsince_deep(jdHi, epoch), lo = pairs_tsince_deep(jdLo, epoch);
        const int nodes[2] = {fit_lattice_nodes(hi > 0.0 ? hi : 0.0), fit_lattice_nodes(lo < 0.0 ? -lo : 0.0)};
        if ((int)lane < 2 * (nvar + 1)) {
            const int k = lane >> 1, dir = lane & 1;
            fit_deep_lattice(r.sets[k], dir, nodes[dir], r.lattice[k]);
        }
    }
    __device__ static auto evaluator(const Row &r, const GravConsts &g) {
        return [&r, &g](int k, double jdFull, const double (&)[1], double (&f)[6]) {
            return fit_deep_eval(r.sets[k], r.lattice[k], jdFull, g, f);
        };
    }
};

// The scratch of corr_scratch_bytes: gates, then the partial lists and counts of list l = class * rowChunks + chunk
struct CorrScratch {
    double *gate;
    double *d2;        // [lists][t][best]
    uint32_t *rows;    // [lists][t][best]
    uint32_t *counts;  // [lists][t][2]
};

static CorrScratch corr_scratch(void *p, uint32_t t, uint32_t best, const CorrShape &s) {
    const size_t lists = (size_t)2 * s.rowChunks * t;
    CorrScratch c;
    c.gate = static_cast<double *>(p);
    c.d2 = c.gate + t;
    c.rows = reinterpret_cast<uint32_t *>(c.d2 + lists * best);
    c.counts = c.rows + lists * best;
    return c;
}

__device__ __forceinline__ CorrObsArrays corr_arrays(const CorrArgs &a) {
    return CorrObsArrays{a.jd, a.fr, a.kind, a.value, a.sigma, a.station, a.stations};
}

__global__ void __launch_bounds__(128) correlate_gate_kernel(const CorrArgs a, double *gate) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= a.t) return;
    const uint32_t begin = __ldg(a.offsets + j), end = __ldg(a.offsets + j + 1);
    const bool sized = end > begin && end - begin <= kCorrMaxTrack;
    const uint32_t used = sized ? corr_used(corr_arrays(a), begin, end) : 0;
    a.used[j] = used;
    gate[j] = corr_bad_track(begin, end, used) ? NAN : corr_chi2_quantile(used, a.gateProbability);
}

// Warp `w` builds row s (when inChunk) into slot (buf, w); lane 0 of the first track chunk writes its row status.
template <typename K>
__device__ __forceinline__ void corr_build(const CorrArgs &a, CorrSmem<typename K::Row> &sm, int buf, int w,
                                           uint32_t s, bool inChunk, uint32_t lane, const Gravity &grav) {
    const uint8_t md = inChunk ? (a.model ? __ldg(a.model + s) : 0) : 0;
    if (!inChunk || !K::takes(md)) {
        if (lane == 0) sm.nvar[buf][w] = -1;
        return;
    }
    double el0[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) el0[c] = __ldg(a.elements + (size_t)c * a.n + s);
    double *P = sm.P[buf][w];
    if (lane < (uint32_t)kFitN) P[lane] = a.covariance ? __ldg(a.covariance + (size_t)s * kFitN + lane) : 0.0;
    __syncwarp();
    const int nvar = corr_nvar(P);
    double x[kFitVars];
    K::Model::vars_of(el0, x);
    bool ok = md <= 1;
    if (ok && (int)lane <= nvar)
        ok = fit_build_set_of<typename K::Model>(x, (int)lane, el0[0], grav, sm.row[buf][w].sets[lane],
                                                 sm.inv[buf][w][lane]);
    const bool built = __all_sync(0xffffffffu, ok);
    __syncwarp();
    if (built) {
        K::lattices(sm.row[buf][w], nvar, el0[0], sm.span[0][0], sm.span[0][1], lane);
        __syncwarp();
    }
    if (lane == 0) {
        sm.nvar[buf][w] = built ? nvar : -1;
        sm.epoch[buf][w] = el0[0];
        sm.index[buf][w] = s;
        if (blockIdx.x == 0) a.rowStatus[s] = built ? kCovOk : kCovInitFailed;
    }
}

template <typename K>
__device__ __forceinline__ void correlate_body(const CorrArgs &a, const CorrShape &shape, const CorrScratch &sc) {
    __shared__ CorrSmem<typename K::Row> sm;
    const uint32_t tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint32_t j = blockIdx.x * kCorrThreads + tid, q = blockIdx.y;
    const uint32_t r0 = q * shape.rows, r1 = r0 + shape.rows < a.n ? r0 + shape.rows : a.n;
    const double gate = j < a.t ? sc.gate[j] : NAN;
    const bool valid = gate == gate;
    const uint32_t begin = valid ? __ldg(a.offsets + j) : 0, end = valid ? __ldg(a.offsets + j + 1) : 0;
    const CorrObsArrays in = corr_arrays(a);
    if (K::kClass == 1) {   // the CTA's span of observation times, for the lattices
        double lo = INFINITY, hi = -INFINITY;
        for (uint32_t i = begin; i < end; ++i) {
            const double t = add_rn(__ldg(a.jd + i), __ldg(a.fr + i));
            lo = fmin(lo, t);
            hi = fmax(hi, t);
        }
#pragma unroll
        for (int m = 16; m > 0; m >>= 1) {
            lo = fmin(lo, __shfl_xor_sync(0xffffffffu, lo, m));
            hi = fmax(hi, __shfl_xor_sync(0xffffffffu, hi, m));
        }
        if (lane == 0) {
            sm.span[warp][0] = lo;
            sm.span[warp][1] = hi;
        }
        __syncthreads();
        if (tid == 0) {
#pragma unroll
            for (int w = 1; w < kCorrWarps; ++w) {
                sm.span[0][0] = fmin(sm.span[0][0], sm.span[w][0]);
                sm.span[0][1] = fmax(sm.span[0][1], sm.span[w][1]);
            }
            if (!(sm.span[0][0] <= sm.span[0][1])) sm.span[0][0] = sm.span[0][1] = 0.0;   // no valid track
        }
        __syncthreads();
    }
    const Gravity grav = gravity(a.grav);
    const uint32_t stages = (r1 - r0 + kCorrWarps - 1) / kCorrWarps;
    corr_build<K>(a, sm, 0, warp, r0 + warp, r0 + warp < r1, lane, grav);
    __syncthreads();
    double bd[kCorrMaxBest];
    uint32_t br[kCorrMaxBest];
    corr_empty(bd, br);
    uint32_t nGate = 0, nFailed = 0;
    double J[kFitVars * 6];
    for (uint32_t s = 0; s < stages; ++s) {
        const int buf = s & 1;
        if (s + 1 < stages) {
            const uint32_t row = r0 + (s + 1) * kCorrWarps + warp;
            corr_build<K>(a, sm, buf ^ 1, warp, row, row < r1, lane, grav);
        }
        if (valid) {
#pragma unroll 1
            for (int w = 0; w < kCorrWarps; ++w) {
                const int nvar = sm.nvar[buf][w];
                if (nvar < 0) continue;
                double acc[kFitSumWords];
                const bool ok = corr_pair_sums(K::evaluator(sm.row[buf][w], a.g), nvar, sm.inv[buf][w],
                                               sm.epoch[buf][w], in, begin, end, J, acc);
                double d2 = ok ? corr_d2(acc, sm.P[buf][w], nvar) : NAN;
                if (!(fabs(d2) < INFINITY)) {
                    ++nFailed;
                    continue;
                }
                d2 = d2 > 0.0 ? d2 : 0.0;
                if (d2 <= gate) ++nGate;
                corr_insert(bd, br, d2, sm.index[buf][w]);
            }
        }
        __syncthreads();
    }
    if (!valid) return;
    const size_t l = ((size_t)K::kClass * shape.rowChunks + q) * a.t + j;
#pragma unroll
    for (int i = 0; i < kCorrMaxBest; ++i) {
        if ((uint32_t)i < a.best) {
            sc.d2[l * a.best + i] = bd[i];
            sc.rows[l * a.best + i] = br[i];
        }
    }
    sc.counts[l * 2] = nGate;
    sc.counts[l * 2 + 1] = nFailed;
}

__global__ void __launch_bounds__(kCorrThreads) correlate_kernel(const CorrArgs a, const CorrShape shape,
                                                                 const CorrScratch sc) {
    correlate_body<CorrNear>(a, shape, sc);
}

__global__ void __launch_bounds__(kCorrThreads) correlate_deep_kernel(const CorrArgs a, const CorrShape shape,
                                                                      const CorrScratch sc) {
    correlate_body<CorrDeep>(a, shape, sc);
}

__global__ void __launch_bounds__(128) correlate_merge_kernel(const CorrArgs a, const CorrShape shape,
                                                              const CorrScratch sc, uint32_t lists) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= a.t) return;
    double bd[kCorrMaxBest];
    uint32_t br[kCorrMaxBest];
    corr_empty(bd, br);
    uint32_t nGate = 0, nFailed = 0;
    const double gate = sc.gate[j];
    const bool valid = gate == gate;
    if (valid) {
        for (uint32_t c = 0; c < lists; ++c) {
            const size_t l = (size_t)c * a.t + j;
            for (uint32_t i = 0; i < a.best; ++i) {
                const uint32_t r = sc.rows[l * a.best + i];
                if (r == kCorrEmptyRow) break;
                corr_insert(bd, br, sc.d2[l * a.best + i], r);
            }
            nGate += sc.counts[l * 2];
            nFailed += sc.counts[l * 2 + 1];
        }
    }
#pragma unroll
    for (int i = 0; i < kCorrMaxBest; ++i) {
        if ((uint32_t)i < a.best) {
            a.d2[(size_t)j * a.best + i] = bd[i];
            a.rows[(size_t)j * a.best + i] = br[i];
        }
    }
    a.nGate[j] = nGate;
    a.nFailed[j] = nFailed;
    a.status[j] = valid ? corr_status(nGate, br[0]) : kCorrBadTrack;
}

cudaError_t launch_correlate(const CorrArgs &a, cudaStream_t stream) {
    const CorrShape shape = corr_shape(a.n, a.t);
    const CorrScratch sc = corr_scratch(a.scratch, a.t, a.best, shape);
    if (a.t) correlate_gate_kernel<<<(a.t + 127) / 128, 128, 0, stream>>>(a, sc.gate);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    uint32_t lists = 0;
    if (a.n) {   // a catalogue with no tracks still gets its row status
        const dim3 grid(shape.trackChunks ? shape.trackChunks : 1, shape.rowChunks);
        correlate_kernel<<<grid, kCorrThreads, 0, stream>>>(a, shape, sc);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
        lists = shape.rowChunks;
        if (a.model) {
            correlate_deep_kernel<<<grid, kCorrThreads, 0, stream>>>(a, shape, sc);
            if ((e = cudaGetLastError()) != cudaSuccess) return e;
            lists = 2 * shape.rowChunks;
        }
    }
    if (a.t) correlate_merge_kernel<<<(a.t + 127) / 128, 128, 0, stream>>>(a, shape, sc, lists);
    return cudaGetLastError();
}

}  // namespace az
