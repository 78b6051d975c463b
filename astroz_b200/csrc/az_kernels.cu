// az_kernels.cu -- hand-written sm_90a kernels of the batch SGP4/SDP4 path.
//
//   K1  sgp4_grid_kernel    near-earth (n_sats x n_times) grid   -- replaces sgp4Batch8 + the
//                           Constellation hot loop (src/simdKernels.zig:9-13, src/Constellation.zig:405-434,478-509)
//   K2a sdp4_lattice_kernel resonance checkpoints on the 720-min lattice (src/Sdp4.zig:787-801)
//   K2  sdp4_grid_kernel    deep-space grid -- replaces sdp4Batch8 (src/simdKernels.zig:15-19,
//                           src/Constellation.zig:448-476)
//
// Mapping (K1): a CTA owns one 8-satellite tile of the element table and one stripe of epochs.  The
// tile (2,496 B, SoA) is staged into shared memory with a single TMA bulk copy (cp.async.bulk +
// mbarrier).  Each warp takes satellites of the tile in turn; its 32 lanes are 32 consecutive epochs of
// that satellite, so every per-satellite constant is a conflict-free shared-memory broadcast, the drag
// model branch (isimp) is warp-uniform, and the Kepler iteration count is near-uniform across the warp
// (same eccentricity).  All arithmetic is fp64 on the CUDA cores; there is no contraction to give the
// tensor cores.
#include "az_kernels.cuh"
#include "az_device_f32.cuh"
#include "az_screen.cuh"

#include <algorithm>

namespace az {

// ---------------------------------------------------------------------------------------------------
// TMA bulk copy + mbarrier helpers (PTX ISA: cp.async.bulk, mbarrier)
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_addr(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    uint32_t done;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(smem_addr(bar)), "r"(parity)
            : "memory");
    } while (!done);
}
// global -> shared bulk copy performed by the TMA unit; completion is signalled on `bar` in bytes
__device__ __forceinline__ void tma_bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_addr(dst)),
                 "l"(src), "r"(bytes), "r"(smem_addr(bar))
                 : "memory");
}

// ---------------------------------------------------------------------------------------------------
// output stage shared by K1 / K2: frame conversion, then either
//   * local block (either layout): each lane stores its 24-byte records directly (streaming stores; the
//     L2 merges the column stores of a warp-run into full lines before they reach HBM);
//   * fused all-gather (satellite-major): a warp's 32 consecutive epochs form one contiguous 768-byte
//     run; the 32 x (x,y,z) records are transposed through shared memory and leave as 128-bit stores to
//     each peer mapping over NVLink, or as one multimem.st to the NVLS multicast address.
// ---------------------------------------------------------------------------------------------------
template <int kMode, bool kVel>
__device__ __forceinline__ void to_output_frame(const GridArgs &a, uint32_t t, CellOut &o) {
    if (kMode != 0) {
        const double sg = __ldg(a.gsin + t), cg = __ldg(a.gcos + t);
        eci_to_ecef(o.rx, o.ry, sg, cg);
        if (kVel) eci_to_ecef(o.vx, o.vy, sg, cg);  // pure rotation, no omega x r (src/Constellation.zig:501-506)
        if (kMode == 2) ecef_to_geodetic(o.rx, o.ry, o.rz);
    }
}

// direct 24-byte record stores; idx in doubles.  For the local satellite-major block this needs no staging through
// shared memory (the L2 merges the three 8-byte column stores of a warp-run),
// so the staged 128-bit path is used only where every byte crosses NVLink (fused all-gather).
template <int kLayout, bool kVel>
__device__ __forceinline__ void store_direct(const GridArgs &a, uint32_t row, uint32_t t, const CellOut &o) {
    const size_t idx = (kLayout == 0) ? ((size_t)row * a.nTimes + t) * 3 : ((size_t)t * a.outNumSats + row) * 3;
    double *p = a.pos + idx;
    __stcs(p, o.rx);
    __stcs(p + 1, o.ry);
    __stcs(p + 2, o.rz);
    if (kVel) {
        double *v = a.vel + idx;
        __stcs(v, o.vx);
        __stcs(v + 1, o.vy);
        __stcs(v + 2, o.vz);
    }
}

__device__ __forceinline__ void st_multimem_16(double *mc, double2 v) {
    // 16 bytes to the multicast address: NVSwitch delivers the write to every GPU mapped by the object
    asm volatile("multimem.st.weak.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc), "r"(__double2loint(v.x)),
                 "r"(__double2hiint(v.x)), "r"(__double2loint(v.y)), "r"(__double2hiint(v.y))
                 : "memory");
}
__device__ __forceinline__ void st_multimem_8(double *mc, double v) {
    asm volatile("multimem.st.weak.global.f64 [%0], %1;" ::"l"(mc), "d"(v) : "memory");
}

constexpr int kStageDoubles = 32 * 3;  // one warp-run of positions (or velocities)

// Emit one warp-run: epochs [tw, tw+32) of output row `row`.  All 32 lanes must call this; `valid`
// masks lanes past the end of the time axis.  stage = this warp's 2 * kStageDoubles scratch.
template <bool kVel, int kGather>
__device__ __forceinline__ void emit_run_sat_major(const GridArgs &a, uint32_t row, uint32_t tw, uint32_t count,
                                                   int lane, bool valid, const CellOut &o, double *stage) {
    if (valid) {
        stage[lane * 3 + 0] = o.rx;
        stage[lane * 3 + 1] = o.ry;
        stage[lane * 3 + 2] = o.rz;
        if (kVel) {
            stage[kStageDoubles + lane * 3 + 0] = o.vx;
            stage[kStageDoubles + lane * 3 + 1] = o.vy;
            stage[kStageDoubles + lane * 3 + 2] = o.vz;
        }
    }
    __syncwarp();
    const size_t base = ((size_t)row * a.nTimes + tw) * 3;  // in doubles; src/Constellation.zig:46-51
    // 128-bit path only for a full run whose destination is 16-byte aligned in every target mapping (the
    // mappings share their alignment: symmetric allocations, and the caller's row/epoch shift is common)
    const double *probe = (kGather == 1) ? a.mcPos : (kGather == 2 ? a.peerPos[0] : a.pos);
    const bool vec = (count == 32) && ((reinterpret_cast<uintptr_t>(probe + base) & 15u) == 0) &&
                     (!kVel || ((reinterpret_cast<uintptr_t>((kGather == 1) ? a.mcVel : (kGather == 2 ? a.peerVel[0] : a.vel)) & 15u) ==
                                (reinterpret_cast<uintptr_t>(probe) & 15u)));
#pragma unroll
    for (int which = 0; which < (kVel ? 2 : 1); ++which) {
        const double *src = stage + which * kStageDoubles;
        if (vec) {
#pragma unroll
            for (int c = lane; c < kStageDoubles / 2; c += 32) {
                const double2 v = *reinterpret_cast<const double2 *>(src + 2 * c);
                if (kGather == 1) {
                    st_multimem_16((which ? a.mcVel : a.mcPos) + base + 2 * c, v);
                } else if (kGather == 2) {
                    for (int p = 0; p < a.nPeers; ++p)
                        __stcs(reinterpret_cast<double2 *>((which ? a.peerVel[p] : a.peerPos[p]) + base + 2 * c), v);
                } else {
                    __stcs(reinterpret_cast<double2 *>((which ? a.vel : a.pos) + base + 2 * c), v);
                }
            }
        } else {  // ragged tail or odd alignment: 8-byte stores
            for (uint32_t i = lane; i < count * 3; i += 32) {
                const double v = src[i];
                if (kGather == 0) {
                    __stcs((which ? a.vel : a.pos) + base + i, v);
                } else if (kGather == 1) {
                    st_multimem_8((which ? a.mcVel : a.mcPos) + base + i, v);
                } else {
                    for (int p = 0; p < a.nPeers; ++p) __stcs((which ? a.peerVel[p] : a.peerPos[p]) + base + i, v);
                }
            }
        }
    }
    __syncwarp();
}

// ---------------------------------------------------------------------------------------------------
// K1: near-earth grid
// ---------------------------------------------------------------------------------------------------
template <int kLayout, int kMode, bool kVel, int kWarps, int kStripe, int kMinBlocks, int kLanes, int kGather>
__global__ void __launch_bounds__(kWarps * 32, kMinBlocks) sgp4_grid_kernel(const GridArgs a) {
    __shared__ __align__(128) double tile[kSgp4TileDoubles];
    __shared__ __align__(16) double stageAll[kGather != 0 ? kWarps * 2 * kStageDoubles : 2];
    __shared__ __align__(8) uint64_t bar;

    const uint32_t tileIdx = blockIdx.x;
    if (threadIdx.x == 0) {
        mbar_init(&bar, 1);
    }
    __syncthreads();
    // Programmatic dependent launch (launch_k1 sets the attribute for back-to-back grids of a stream): this CTA may have
    // been scheduled while the previous kernel's last wave was still draining.  Nothing of global memory is touched
    // before the wait -- it returns once that kernel has completed and its writes are visible, i.e. ordinary stream
    // order -- and the next grid in the stream is then allowed to start filling the slots this grid's tail leaves free.
    // (Both are no-ops for a launch without the attribute.)
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;");
    if (threadIdx.x == 0) {
        mbar_expect_tx(&bar, kSgp4TileBytes);
        tma_bulk_g2s(tile, a.sgp4Tiles + (size_t)tileIdx * kSgp4TileDoubles, kSgp4TileBytes, &bar);
    }

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t t0 = blockIdx.y * a.stripe;
    const uint32_t t1 = min(t0 + a.stripe, a.nTimes);
    double *stage = stageAll + (kGather != 0 ? warp * 2 * kStageDoubles : 0);
    mbar_wait(&bar, 0);

    if constexpr (kLayout == 1 && kGather == 0) {
        // ---- time-major: for one epoch a tile's satellites are consecutive 24-byte records of the block (when
        // their output rows are consecutive, i.e. an all-near-earth catalog).  Each warp takes PAIRS of adjacent
        // satellites: a pair's two records are 48 contiguous, 16-byte aligned bytes per epoch, so the warp can
        // transpose its own 64 epochs x 2 satellites through a private shared-memory patch and emit 128-bit
        // stores without any CTA-wide barrier (per-lane 24-byte stores at a stride of n_sats*24 B touch a different row's
        // sector with every word; a CTA-wide 192-byte-row transpose costs two barriers per run).
        // The L2 merges the neighbouring pairs' halves of each 32-byte sector before it is written back.
        constexpr int kRun = 32 * kLanes;
        // The patch IS the pair's slice of the output: 48 contiguous bytes per epoch, epochs back to back.  Lanes write
        // their 24-byte records at a 48-byte pitch (two-way bank conflict on the stores); the read-back is then one
        // conflict-free LDS.128 per lane at 16 * lane, and lane = 3 e + ch addresses chunk ch of epoch e with no
        // division: 30 lanes move 10 epochs per pass.
        constexpr int kRow = 6;
        __shared__ __align__(16) double tposAll[kWarps * kRun * kRow];
        __shared__ __align__(16) double tvelAll[kVel ? kWarps * kRun * kRow : 2];
        double *tpos = tposAll + warp * kRun * kRow;
        double *tvel = tvelAll + (kVel ? warp * kRun * kRow : 0);
        const uint32_t sat0 = tileIdx * kTileSats;
        const uint32_t nReal = min((uint32_t)kTileSats, a.nSats - sat0);
        const bool evenStride = (((size_t)a.outNumSats * 3) & 1) == 0;
#pragma unroll 1
        for (int pr = warp; 2 * pr < (int)nReal; pr += kWarps) {
            const uint32_t satA = sat0 + 2 * pr;
            const int nPair = min(2, (int)nReal - 2 * pr);
            const uint32_t rowA = __ldg(a.orig + satA);
            const uint32_t rowB = nPair == 2 ? __ldg(a.orig + satA + 1) : rowA;
            const bool actA = !a.mask || a.mask[rowA] != 0;  // laneActive, src/Constellation.zig:530-533
            const bool actB = nPair == 2 && (!a.mask || a.mask[rowB] != 0);
            if (!actA && !actB) continue;
            // both records of an epoch leave as three 16-byte chunks when the pair's rows are adjacent in the block
            // (an all-near-earth catalog, or a mixed one where no deep-space row falls between them) and 16-byte aligned,
            // as six 8-byte words when adjacent but unaligned; a satellite without its partner (masked, or a deep-space
            // row in between) leaves as three 8-byte words per epoch -- always transposed through the patch, so a store
            // instruction covers whole contiguous records of 5-10 rows instead of 32 rows' single words
            const bool adjacent = actA && actB && rowB == rowA + 1;  // the pair's 48 bytes per epoch are contiguous
            const bool paired = adjacent && evenStride &&
                                ((reinterpret_cast<uintptr_t>(a.pos + (size_t)rowA * 3) & 15u) == 0) &&
                                (!kVel || (reinterpret_cast<uintptr_t>(a.vel + (size_t)rowA * 3) & 15u) == 0);
#pragma unroll 1
            for (uint32_t tw = t0; tw < t1; tw += kRun) {
#pragma unroll 1
                for (int m = 0; m < nPair; ++m) {
                    if (!(m == 0 ? actA : actB)) continue;
                    const uint32_t sat = satA + m;
                    const double *colBase = tile + 2 * pr + m;
                    auto col = [colBase](int i) { return colBase[i * kTileSats]; };
                    const double toff = __ldg(a.toff + sat);
                    const uint32_t row = m == 0 ? rowA : rowB;
                    double ts[kLanes];
#pragma unroll
                    for (int k = 0; k < kLanes; ++k) ts[k] = __ldg(a.tbase + min(tw + 32u * k + lane, t1 - 1)) + toff;
                    CellOut o[kLanes];
                    sgp4_cell<kLanes>(col, ts, a.g, o);
#pragma unroll
                    for (int k = 0; k < kLanes; ++k) {
                        const uint32_t tk = tw + 32u * k + lane;
                        if (tk >= t1) continue;
                        if (a.status) a.status[(size_t)row * a.nTimes + tk] = (o[k].mrt < 1.0) ? 1 : 0;
                        to_output_frame<kMode, kVel>(a, tk, o[k]);
                        double *p = tpos + (32 * k + lane) * kRow + m * 3;
                        p[0] = o[k].rx; p[1] = o[k].ry; p[2] = o[k].rz;
                        if (kVel) {
                            double *v = tvel + (32 * k + lane) * kRow + m * 3;
                            v[0] = o[k].vx; v[1] = o[k].vy; v[2] = o[k].vz;
                        }
                    }
                }
                __syncwarp();
                const uint32_t count = min((uint32_t)kRun, t1 - tw);  // epochs in this run
                const uint32_t e = (uint32_t)lane / 3u, ch = (uint32_t)lane - 3u * e;  // lane = 3 e + ch; lanes 30, 31 idle
                const size_t step = (size_t)a.outNumSats * 30;                       // ten epochs, in doubles
                if (paired) {  // warp-uniform
                    size_t dst = ((size_t)(tw + e) * a.outNumSats + rowA) * 3 + 2 * ch;
                    const double2 *sp = reinterpret_cast<const double2 *>(tpos) + lane;
                    const double2 *sv = reinterpret_cast<const double2 *>(tvel) + lane;
                    if (lane < 30) {
                        for (uint32_t j = e; j < count; j += 10, dst += step, sp += 30, sv += 30) {
                            __stcs(reinterpret_cast<double2 *>(a.pos + dst), *sp);
                            if (kVel) __stcs(reinterpret_cast<double2 *>(a.vel + dst), *sv);
                        }
                    }
                } else if (adjacent) {
                    // contiguous but not 16-byte aligned (odd first row, or an odd row count): the pair's six words per
                    // epoch as 8-byte stores, lane = 6 e + w -- a store instruction still fills whole 48-byte runs (five
                    // rows per pass), half the cache-line visits of storing the two satellites separately
                    const uint32_t e6 = (uint32_t)lane / 6u, w = (uint32_t)lane - 6u * e6;
                    if (lane < 30) {
                        size_t dst = ((size_t)(tw + e6) * a.outNumSats + rowA) * 3 + w;
                        const size_t step5 = (size_t)a.outNumSats * 15;
                        const double *sp = tpos + lane, *sv = tvel + lane;
                        for (uint32_t j = e6; j < count; j += 5, dst += step5, sp += 30, sv += 30) {
                            __stcs(a.pos + dst, *sp);
                            if (kVel) __stcs(a.vel + dst, *sv);
                        }
                    }
                } else if (lane < 30) {
#pragma unroll 1
                    for (int m = 0; m < nPair; ++m) {
                        if (!(m == 0 ? actA : actB)) continue;
                        size_t dst = ((size_t)(tw + e) * a.outNumSats + (m == 0 ? rowA : rowB)) * 3 + ch;
                        const double *sp = tpos + e * kRow + m * 3 + ch, *sv = tvel + e * kRow + m * 3 + ch;
                        for (uint32_t j = e; j < count; j += 10, dst += step, sp += 10 * kRow, sv += 10 * kRow) {
                            __stcs(a.pos + dst, *sp);
                            if (kVel) __stcs(a.vel + dst, *sv);
                        }
                    }
                }
                __syncwarp();
            }
        }
        return;
    }

#pragma unroll 1
    for (int sl = warp; sl < kTileSats; sl += kWarps) {
        const uint32_t sat = tileIdx * kTileSats + sl;
        if (sat >= a.nSats) break;  // padding lanes of the last tile (src/Constellation.zig:146,493)
        const double *colBase = tile + sl;
        auto col = [colBase](int i) { return colBase[i * kTileSats]; };
        const double toff = __ldg(a.toff + sat);
        const uint32_t row = __ldg(a.orig + sat);
        if (a.mask && a.mask[row] == 0) continue;  // laneActive, src/Constellation.zig:530-533
        // a thread owns kLanes epochs of this satellite, 32 apart, so each warp-run is 32 consecutive epochs
        // (one contiguous 768-byte run of the satellite-major block).  The loop is warp-uniform.
#pragma unroll 1
        for (uint32_t tw = t0; tw < t1; tw += 32 * kLanes) {
            double ts[kLanes];
#pragma unroll
            for (int k = 0; k < kLanes; ++k)
                ts[k] = __ldg(a.tbase + min(tw + 32u * k + lane, t1 - 1)) + toff;  // src/Constellation.zig:425
            CellOut o[kLanes];
            sgp4_cell<kLanes>(col, ts, a.g, o);
#pragma unroll
            for (int k = 0; k < kLanes; ++k) {
                const uint32_t twk = tw + 32u * k;
                if (twk >= t1) break;  // warp-uniform
                const uint32_t tk = twk + lane;
                const bool valid = tk < t1;
                if (valid) {
                    if (a.status) a.status[(size_t)row * a.nTimes + tk] = (o[k].mrt < 1.0) ? 1 : 0;
                    to_output_frame<kMode, kVel>(a, tk, o[k]);
                }
                if (kGather != 0) {
                    emit_run_sat_major<kVel, kGather>(a, row, twk, min(32u, t1 - twk), lane, valid, o[k], stage);
                } else if (valid) {
                    store_direct<kLayout, kVel>(a, row, tk, o[k]);
                }
            }
        }
    }
}

// K1t: one satellite x a long time axis (replaces sgp4Times8 / Sgp4.propagateN, src/simdKernels.zig:21-24,
// src/Sgp4.zig:753-785; the path behind Satrec.sgp4_array and sgp4_propagate_batch).  With a single
// satellite K1 would keep one warp per CTA busy; here every thread of every CTA takes epochs of that
// satellite (kLanes each), its 39 constants sitting in shared memory.
constexpr int kTimesThreads = 128;
constexpr int kTimesLanes = 2;
template <int kMode, bool kVel>
__global__ void __launch_bounds__(kTimesThreads, 4) sgp4_times_kernel(const GridArgs a) {
    __shared__ double cols[kSgp4Cols];
    if (threadIdx.x < kSgp4Cols) cols[threadIdx.x] = __ldg(a.sgp4Tiles + threadIdx.x * kTileSats);  // lane 0 of tile 0
    __syncthreads();
    auto col = [&](int i) { return cols[i]; };
    const double toff = __ldg(a.toff);
    const uint32_t row = __ldg(a.orig);
    const uint32_t base = blockIdx.x * (kTimesThreads * kTimesLanes) + threadIdx.x;
    if (base >= a.nTimes) return;
    double ts[kTimesLanes];
#pragma unroll
    for (int k = 0; k < kTimesLanes; ++k) {
        const uint32_t tc = min(base + k * kTimesThreads, a.nTimes - 1);
        ts[k] = a.jdArr ? ((__ldg(a.jdArr + tc) + __ldg(a.frArr + tc)) - a.epochJd) * 1440.0  // satrec.zig:263
                        : __ldg(a.tbase + tc) + toff;
    }
    CellOut o[kTimesLanes];
    sgp4_cell<kTimesLanes>(col, ts, a.g, o);
#pragma unroll
    for (int k = 0; k < kTimesLanes; ++k) {
        const uint32_t t = base + k * kTimesThreads;
        if (t < a.nTimes) {
            if (a.status) a.status[(size_t)row * a.nTimes + t] = (o[k].mrt < 1.0) ? 1 : 0;
            to_output_frame<kMode, kVel>(a, t, o[k]);
            const size_t idx = ((size_t)row * a.nTimes + t) * a.recStride;
            double *p = a.pos + idx;
            __stcs(p, o[k].rx);
            __stcs(p + 1, o[k].ry);
            __stcs(p + 2, o[k].rz);
            if (kVel) {
                double *v = a.vel + idx;
                __stcs(v, o[k].vx);
                __stcs(v + 1, o[k].vy);
                __stcs(v + 2, o[k].vz);
            }
        }
    }
}

template <int kMode, bool kVel>
static cudaError_t launch_k1t(const GridArgs &a, cudaStream_t stream) {
    const uint32_t per = kTimesThreads * kTimesLanes;
    sgp4_times_kernel<kMode, kVel><<<(a.nTimes + per - 1) / per, kTimesThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

// Launch-shape sweep scaffolding (tools/sweep_variants.py) is compiled only with -DAZ_TUNING; the shipped library
// carries the chosen shapes alone.
#ifdef AZ_TUNING
struct Sgp4Variant {
    const char *name;
    int warps, stripe, minBlocks, lanes;
};
static const Sgp4Variant kVariants[] = {
    {"w4_s256_b4_l1", 4, 256, 4, 1}, {"w4_s256_b3_l2", 4, 256, 3, 2}, {"w4_s512_b3_l2", 4, 512, 3, 2},
    {"w4_s256_b2_l2", 4, 256, 2, 2}, {"w8_s256_b1_l2", 8, 256, 1, 2}, {"w4_s512_b4_l1", 4, 512, 4, 1},
    {"w2_s256_b4_l2", 2, 256, 4, 2}, {"w4_s768_b3_l2", 4, 768, 3, 2}, {"w4_s768_b2_l3", 4, 768, 2, 3},
    {"w8_s512_b2_l2", 8, 512, 2, 2}, {"w4_s256_b6_l1", 4, 256, 6, 1}, {"w4_s256_b7_l1", 4, 256, 7, 1},
    {"w4_s256_b8_l1", 4, 256, 8, 1}, {"w8_s256_b4_l1", 8, 256, 4, 1}, {"w4_s256_b5_l2", 4, 256, 5, 2},
    {"w4_s384_b2_l3", 4, 384, 2, 3}, {"w4_s288_b2_l3", 4, 288, 2, 3}, {"w4_s768_b2_l4", 4, 768, 2, 4},
    {"w4_s512_b2_l4", 4, 512, 2, 4}, {"w8_s768_b1_l3", 8, 768, 1, 3}, {"w4_s384_b3_l3", 4, 384, 3, 3},
    {"w4_s768_b1_l4", 4, 768, 1, 4}, {"w8_s384_b1_l4", 8, 384, 1, 4},
};
int sgp4_variant_count() { return (int)(sizeof(kVariants) / sizeof(kVariants[0])); }
const char *sgp4_variant_name(int v) { return (v >= 0 && v < sgp4_variant_count()) ? kVariants[v].name : "?"; }
#else
int sgp4_variant_count() { return 0; }
const char *sgp4_variant_name(int) { return "?"; }
#endif

// resident CTA slots of the current device for the near-earth grid (3 CTAs of 128 threads per SM at 158 registers)
static int k1_resident_slots() {
    static int cached[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132 * 3;
    if (cached[dev] == 0) {
        int sms = 0;
        if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
        cached[dev] = sms * 3;
    }
    return cached[dev];
}
// ASTROZ_PDL=0 turns the programmatic dependent launch of back-to-back K1 grids off (measurement / bisecting)
static bool k1_pdl_enabled() {
    static const bool on = [] {
        const char *e = std::getenv("ASTROZ_PDL");
        return !(e && e[0] == '0');
    }();
    return on;
}
static uint32_t g_k1StripeOverride = 0;  // measurement only (ASTROZ_K1_STRIPE): epochs per CTA, 0 = automatic
void set_sgp4_stripe(uint32_t epochs) { g_k1StripeOverride = epochs; }

template <int kLayout, int kMode, bool kVel, int kWarps, int kStripe, int kMinBlocks, int kLanes, int kGather = 0>
static cudaError_t launch_k1(const GridArgs &a0, cudaStream_t stream) {
    const uint32_t tiles = (a0.nSats + kTileSats - 1) / kTileSats;
    if (tiles == 0 || a0.nTimes == 0) return cudaSuccess;
    // Epochs per CTA.  kStripe is the shape's stripe for a grid that fills the GPU many times over (fewest CTA
    // prologues: barrier, TMA tile copy).  A small grid -- a 1/8 satellite shard of the headline catalog is 211 tiles --
    // is cut finer, down to one pass of the CTA's warps (32 * kLanes epochs), until it gives every SM's resident CTA
    // slots about eight CTAs each, so that the last, partly filled wave is a small fraction of the launch.
    GridArgs a = a0;
    constexpr uint32_t kPass = 32 * kLanes;
    uint32_t stripe = kStripe;
    const uint32_t slots = (uint32_t)k1_resident_slots();
    while (stripe > kPass && (uint64_t)tiles * ((a.nTimes + stripe - 1) / stripe) < 8ull * slots) {
        const uint32_t half = ((stripe / 2 + kPass - 1) / kPass) * kPass;
        if (half >= stripe) break;
        stripe = half;
    }
    if (g_k1StripeOverride) stripe = std::max(kPass, g_k1StripeOverride / kPass * kPass);
    a.stripe = stripe;
    dim3 grid(tiles, (a.nTimes + stripe - 1) / stripe);
    if (kGather == 0 && k1_pdl_enabled()) {
        // back-to-back grids of one stream (a chunked host call, a caller's time loop): let the next grid's CTAs be
        // scheduled into the slots this grid's last wave leaves free; the kernel waits for its predecessor before it
        // touches global memory (griddepcontrol.wait at its top), so stream order is what the data sees
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = grid;
        cfg.blockDim = dim3(kWarps * 32);
        cfg.dynamicSmemBytes = 0;
        cfg.stream = stream;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        return cudaLaunchKernelEx(&cfg, sgp4_grid_kernel<kLayout, kMode, kVel, kWarps, kStripe, kMinBlocks, kLanes, kGather>, a);
    }
    sgp4_grid_kernel<kLayout, kMode, kVel, kWarps, kStripe, kMinBlocks, kLanes, kGather>
        <<<grid, kWarps * 32, 0, stream>>>(a);
    return cudaGetLastError();
}

// Shipped launch shapes (warps per CTA, epochs per stripe, resident CTAs per SM, epochs per thread).  The plain
// satellite-major TEME/ECEF grid: three epochs per thread (nine independent fp64 chains per scheduler), 3 resident CTAs / SM
// (164 registers).  On one H100 80GB HBM3 SXM (power limit 700 W, maximum SM clock 1980 MHz) the 23 shapes of the
// AZ_TUNING sweep (tools/sweep_variants.py: 20 steps per shape from a card not yet at its power cap) put this one first on
// the headline grid: 0.386 ms per step, against 0.392 ms for two epochs per thread (4, 256, 3, 2) and 0.441 ms for three
// epochs at 2 CTAs / SM; two passes agreed to 0.3 %.  The time-major grids take the same three epochs
// per thread; only the satellite-major geodetic grid, whose epilogue needs the registers itself, keeps two.
#ifndef AZ_K1_STRIPE
#define AZ_K1_STRIPE 384
#endif
#ifndef AZ_K1_BLOCKS
#define AZ_K1_BLOCKS 3
#endif
#ifndef AZ_K1_LANES
#define AZ_K1_LANES 3
#endif
#ifndef AZ_DEFAULT_K1
#define AZ_DEFAULT_K1 4, AZ_K1_STRIPE, AZ_K1_BLOCKS, AZ_K1_LANES
#endif
#define AZ_COMPACT_K1 4, 256, 3, 2
// epochs per thread of the time-major and geodetic specialisations (2: the compact shape, 3: stripe 384 x 3 CTAs / SM)
#ifndef AZ_TM_LANES
#define AZ_TM_LANES 3
#endif
#ifndef AZ_GEO_LANES
#define AZ_GEO_LANES 2
#endif
#if AZ_TM_LANES == 3
#define AZ_TIME_MAJOR_K1 4, 384, 3, 3   // three resident CTAs (168-register cap): the transposing patch costs registers
#else
#define AZ_TIME_MAJOR_K1 AZ_COMPACT_K1
#endif
#ifndef AZ_TM_ECEF_LANES
#define AZ_TM_ECEF_LANES 3   // with the table-reduced sincos the registers are there
#endif
#if AZ_TM_ECEF_LANES == 3
#define AZ_TM_ECEF_K1 4, 384, 3, 3
#else
#define AZ_TM_ECEF_K1 AZ_COMPACT_K1
#endif
#if AZ_GEO_LANES == 3
#define AZ_GEODETIC_K1 AZ_DEFAULT_K1
#else
#define AZ_GEODETIC_K1 AZ_COMPACT_K1
#endif

// The launch shape (epochs per thread) follows the time axis, identically for the local and the fused all-gather store
// stages, so a cell is computed by the same instruction stream -- and to the same bits -- whichever way it leaves the SM.
template <int kLayout, int kMode, bool kVel, int kGather>
static cudaError_t launch_k1_shaped(const GridArgs &a, cudaStream_t stream) {
    if constexpr (kMode == 2 && kLayout == 1) {  // geodetic: two epochs per thread satellite-major, three time-major
        return launch_k1<kLayout, kMode, kVel, AZ_TM_ECEF_K1, kGather>(a, stream);
    } else if constexpr (kMode == 2) {
        return launch_k1<kLayout, kMode, kVel, AZ_GEODETIC_K1, kGather>(a, stream);
    } else if constexpr (kLayout == 1 && kMode == 0) {
        return launch_k1<kLayout, kMode, kVel, AZ_TIME_MAJOR_K1, kGather>(a, stream);
    } else if constexpr (kLayout == 1) {
        return launch_k1<kLayout, kMode, kVel, AZ_TM_ECEF_K1, kGather>(a, stream);
    } else {
        // a thread's epochs are 32 apart: short or ragged time axes pad up to 32 * lanes, so take the widest shape
        // that does not add padded warp-runs (16 epochs x 10^6 Monte-Carlo draws: one lane, not three)
        const uint32_t runs1 = (a.nTimes + 31) / 32, runs2 = (a.nTimes + 63) / 64 * 2, runs3 = (a.nTimes + 95) / 96 * 3;
        if (runs3 <= runs2 && runs3 <= runs1) return launch_k1<kLayout, kMode, kVel, AZ_DEFAULT_K1, kGather>(a, stream);
        if (runs2 <= runs1) return launch_k1<kLayout, kMode, kVel, AZ_COMPACT_K1, kGather>(a, stream);
        return launch_k1<kLayout, kMode, kVel, 4, 256, 4, 1, kGather>(a, stream);
    }
}

template <int kLayout, int kMode, bool kVel>
static cudaError_t launch_k1_variant(const GridArgs &a, cudaStream_t stream, int variant) {
#ifdef AZ_TUNING
    if (kLayout == 0 && kMode == 0 && kVel) {  // tuning variants exist for the headline specialisation only
        switch (variant) {
            case 0: return launch_k1<0, 0, true, 4, 256, 4, 1>(a, stream);
            case 1: return launch_k1<0, 0, true, 4, 256, 3, 2>(a, stream);
            case 2: return launch_k1<0, 0, true, 4, 512, 3, 2>(a, stream);
            case 3: return launch_k1<0, 0, true, 4, 256, 2, 2>(a, stream);
            case 4: return launch_k1<0, 0, true, 8, 256, 1, 2>(a, stream);
            case 5: return launch_k1<0, 0, true, 4, 512, 4, 1>(a, stream);
            case 6: return launch_k1<0, 0, true, 2, 256, 4, 2>(a, stream);
            case 7: return launch_k1<0, 0, true, 4, 768, 3, 2>(a, stream);
            case 8: return launch_k1<0, 0, true, 4, 768, 2, 3>(a, stream);
            case 9: return launch_k1<0, 0, true, 8, 512, 2, 2>(a, stream);
            case 10: return launch_k1<0, 0, true, 4, 256, 6, 1>(a, stream);
            case 11: return launch_k1<0, 0, true, 4, 256, 7, 1>(a, stream);
            case 12: return launch_k1<0, 0, true, 4, 256, 8, 1>(a, stream);
            case 13: return launch_k1<0, 0, true, 8, 256, 4, 1>(a, stream);
            case 14: return launch_k1<0, 0, true, 4, 256, 5, 2>(a, stream);
            case 15: return launch_k1<0, 0, true, 4, 384, 2, 3>(a, stream);
            case 16: return launch_k1<0, 0, true, 4, 288, 2, 3>(a, stream);
            case 17: return launch_k1<0, 0, true, 4, 768, 2, 4>(a, stream);
            case 18: return launch_k1<0, 0, true, 4, 512, 2, 4>(a, stream);
            case 19: return launch_k1<0, 0, true, 8, 768, 1, 3>(a, stream);
            case 20: return launch_k1<0, 0, true, 4, 384, 3, 3>(a, stream);
            case 21: return launch_k1<0, 0, true, 4, 768, 1, 4>(a, stream);
            case 22: return launch_k1<0, 0, true, 8, 384, 1, 4>(a, stream);
            default: break;
        }
    }
#else
    (void)variant;
#endif
    return launch_k1_shaped<kLayout, kMode, kVel, 0>(a, stream);
}

cudaError_t launch_sgp4_grid(const GridArgs &a, int mode, int layout, cudaStream_t stream, int variant) {
    if (a.gather != 0) {  // fused all-gather: satellite-major TEME only
        if (layout != 0 || mode != 0) return cudaErrorInvalidValue;
        const bool gv = (a.gather == 1 ? a.mcVel : a.peerVel[0]) != nullptr;
        if (a.gather == 1) return gv ? launch_k1_shaped<0, 0, true, 1>(a, stream) : launch_k1_shaped<0, 0, false, 1>(a, stream);
        return gv ? launch_k1_shaped<0, 0, true, 2>(a, stream) : launch_k1_shaped<0, 0, false, 2>(a, stream);
    }
    const bool vel = a.vel != nullptr;
    if (a.nSats == 1 && a.nTimes >= 64 && a.mask == nullptr) {  // single satellite: spread the time axis over the whole GPU
        // one row: satellite-major and time-major coincide when the block has a single row
        if (layout == 0 || a.outNumSats == 1) {
            if (mode == 0) return vel ? launch_k1t<0, true>(a, stream) : launch_k1t<0, false>(a, stream);
            if (mode == 1) return vel ? launch_k1t<1, true>(a, stream) : launch_k1t<1, false>(a, stream);
            if (mode == 2) return vel ? launch_k1t<2, true>(a, stream) : launch_k1t<2, false>(a, stream);
        }
    }
#define AZ_K1(L, M)                                                               \
    if (layout == L && mode == M)                                                 \
        return vel ? launch_k1_variant<L, M, true>(a, stream, variant)            \
                   : launch_k1_variant<L, M, false>(a, stream, variant);
    AZ_K1(0, 0) AZ_K1(0, 1) AZ_K1(0, 2) AZ_K1(1, 0) AZ_K1(1, 1) AZ_K1(1, 2)
#undef AZ_K1
    return cudaErrorInvalidValue;
}

// ---------------------------------------------------------------------------------------------------
// K2a: resonance lattice.  thread = (deep-space satellite, direction); node k holds the integrator
// state after k steps of +-720 min from atime = 0 (src/Sdp4.zig:787-801, carry == fresh integration
// by src/Sdp4Batch.zig:603-629).
// ---------------------------------------------------------------------------------------------------
__global__ void sdp4_lattice_kernel(const Sdp4Sat *__restrict__ sats, uint32_t nSats, double2 *__restrict__ lattice,
                                    int nodes) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nSats * 2) return;
    const uint32_t sat = i >> 1;
    const Sdp4Sat e = sats[sat];
    const double delt = (i & 1) ? -kStepp : kStepp;
    double2 *out = lattice + (size_t)i * nodes;
    double xli = e.xlamo, xni = e.no, atime = 0.0;
    out[0] = make_double2(xli, xni);
    if (e.irez == 0) return;
#pragma unroll 1
    for (int k = 1; k < nodes; ++k) {
        resonance_step(e, xli, xni, atime, delt);
        out[k] = make_double2(xli, xni);
    }
}

cudaError_t launch_sdp4_lattice(const Sdp4Sat *sats, uint32_t nSats, double2 *lattice, int nodes, cudaStream_t stream) {
    if (nSats == 0) return cudaSuccess;
    const uint32_t threads = 64, total = nSats * 2;
    sdp4_lattice_kernel<<<(total + threads - 1) / threads, threads, 0, stream>>>(sats, nSats, lattice, nodes);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------
// K2: deep-space grid.  CTA = one satellite x one stripe of epochs; the satellite record sits in shared
// memory; a lane is one epoch, so the resonance class branch (irez) is uniform across the CTA.
// ---------------------------------------------------------------------------------------------------
constexpr int kSdp4Threads = 128;
constexpr int kSdp4Stripe = 512;

#ifndef AZ_K2_LANES
#define AZ_K2_LANES 1
#endif
constexpr int kSdp4Lanes = AZ_K2_LANES;  // epochs per thread, 32 apart (each warp-run is 32 consecutive epochs, like K1)

template <int kLayout, int kMode, bool kVel, int kGather, int kMinBlocks>
__global__ void __launch_bounds__(kSdp4Threads, kMinBlocks) sdp4_grid_kernel(const GridArgs a) {
    __shared__ Sdp4Sat e;
    __shared__ __align__(16) double stageAll[kGather != 0 ? (kSdp4Threads / 32) * 2 * kStageDoubles : 2];
    __shared__ __align__(16) double tmPatch[(kLayout == 1 && kGather == 0) ? (kSdp4Threads / 32) * (kVel ? 192 : 96) : 2];
    const uint32_t sat = blockIdx.x;
    {
        const double *src = reinterpret_cast<const double *>(a.sdp4 + sat);
        double *dst = reinterpret_cast<double *>(&e);
        for (int i = threadIdx.x; i < (int)(sizeof(Sdp4Sat) / 8); i += kSdp4Threads) dst[i] = __ldg(src + i);
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double *stage = stageAll + (kGather != 0 ? warp * 2 * kStageDoubles : 0);
    const uint32_t row = __ldg(a.orig + sat);
    const uint32_t t0 = blockIdx.y * kSdp4Stripe;
    const uint32_t t1 = min(t0 + (uint32_t)kSdp4Stripe, a.nTimes);
    constexpr uint32_t kRun = 32 * kSdp4Lanes;
#pragma unroll 1
    for (uint32_t tw = t0 + warp * kRun; tw < t1; tw += (kSdp4Threads / 32) * kRun) {  // warp-uniform
        double ts[kSdp4Lanes], xli[kSdp4Lanes], xni[kSdp4Lanes], atime[kSdp4Lanes];
#pragma unroll
        for (int k = 0; k < kSdp4Lanes; ++k) {
            const uint32_t tc = min(tw + 32u * k + lane, t1 - 1);
            ts[k] = a.tsince ? __ldg(a.tsince + tc)
                             : (__ldg(a.jdFull + tc) - e.epochJd) * 1440.0;  // src/Constellation.zig:465
            xli[k] = e.xlamo;
            xni[k] = e.no;
            atime[k] = 0.0;
            if (e.irez != 0) {
                const int node = resonance_node(ts[k]);
                const int have = min(node, a.latticeNodes - 1);
                const double2 st = __ldg(a.lattice + ((size_t)sat * 2 + (ts[k] > 0.0 ? 0 : 1)) * a.latticeNodes + have);
                const double delt = ts[k] > 0.0 ? kStepp : -kStepp;
                xli[k] = st.x;
                xni[k] = st.y;
                atime[k] = delt * (double)have;
                for (int j = have; j < node; ++j) resonance_step(e, xli[k], xni[k], atime[k], delt);  // beyond the lattice
            }
        }
        CellOut o[kSdp4Lanes];
        int st[kSdp4Lanes];
        sdp4_cell_n<kSdp4Lanes>(e, ts, xli, xni, atime, a.g, o, st);
#pragma unroll
        for (int k = 0; k < kSdp4Lanes; ++k) {
            const uint32_t twk = tw + 32u * k;
            if (twk >= t1) break;  // warp-uniform
            const uint32_t t = twk + lane;
            const bool valid = t < t1;
            if (valid && a.status) a.status[(size_t)row * a.nTimes + t] = (uint8_t)st[k];
            if (st[k] != 0) {  // zero fill, per satellite (src/Constellation.zig:468-471,511-528 does it per batch of 8)
                o[k].rx = o[k].ry = o[k].rz = o[k].vx = o[k].vy = o[k].vz = 0.0;
            } else if (valid) {
                to_output_frame<kMode, kVel>(a, t, o[k]);
            }
            if (kGather != 0) {
                emit_run_sat_major<kVel, kGather>(a, row, twk, min(32u, t1 - twk), lane, valid, o[k], stage);
            } else if (kLayout == 1) {
                // time-major: the warp's 32 records of this satellite sit n_sats * 24 bytes apart.  Transposed through
                // the warp's patch they leave as whole 24-byte records, lane = 3 e + w, ten rows per store instruction,
                // instead of one word of 32 different rows each
                double *tp = tmPatch + warp * (kVel ? 192 : 96);
                if (valid) {
                    tp[lane * 3 + 0] = o[k].rx; tp[lane * 3 + 1] = o[k].ry; tp[lane * 3 + 2] = o[k].rz;
                    if (kVel) { tp[96 + lane * 3 + 0] = o[k].vx; tp[96 + lane * 3 + 1] = o[k].vy; tp[96 + lane * 3 + 2] = o[k].vz; }
                }
                __syncwarp();
                const uint32_t count = min(32u, t1 - twk);
                const uint32_t e = (uint32_t)lane / 3u, w = (uint32_t)lane - 3u * e;
                if (lane < 30) {
                    size_t dst = ((size_t)(twk + e) * a.outNumSats + row) * 3 + w;
                    const size_t step = (size_t)a.outNumSats * 30;
                    const double *sp = tp + lane;
                    for (uint32_t j = e; j < count; j += 10, dst += step, sp += 30) {
                        __stcs(a.pos + dst, *sp);
                        if (kVel) __stcs(a.vel + dst, sp[96]);
                    }
                }
                __syncwarp();
            } else if (valid) {
                store_direct<kLayout, kVel>(a, row, t, o[k]);
            }
        }
    }
}

#ifndef AZ_DEFAULT_K2_BLOCKS
#define AZ_DEFAULT_K2_BLOCKS 6
#endif
static int g_k2Variant = -1;  // tuning only (ASTROZ_SDP4_VARIANT): 0 -> 3, 1 -> 4, 2 -> 5 resident CTAs per SM
void set_sdp4_variant(int v) { g_k2Variant = v; }

template <int kLayout, int kMode, bool kVel, int kGather = 0>
static cudaError_t launch_k2(const GridArgs &a, cudaStream_t stream) {
    const uint32_t stripes = (a.nTimes + kSdp4Stripe - 1) / kSdp4Stripe;
    if (a.nSats == 0 || stripes == 0) return cudaSuccess;
    dim3 grid(a.nSats, stripes);
#ifdef AZ_TUNING
    if (kLayout == 0 && kMode == 0 && kVel && kGather == 0 && g_k2Variant >= 0) {
        if (g_k2Variant == 1) { sdp4_grid_kernel<0, 0, true, 0, 4><<<grid, kSdp4Threads, 0, stream>>>(a); return cudaGetLastError(); }
        if (g_k2Variant == 2) { sdp4_grid_kernel<0, 0, true, 0, 5><<<grid, kSdp4Threads, 0, stream>>>(a); return cudaGetLastError(); }
        if (g_k2Variant == 0) { sdp4_grid_kernel<0, 0, true, 0, 3><<<grid, kSdp4Threads, 0, stream>>>(a); return cudaGetLastError(); }
    }
#endif
    sdp4_grid_kernel<kLayout, kMode, kVel, kGather, AZ_DEFAULT_K2_BLOCKS><<<grid, kSdp4Threads, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_sdp4_grid(const GridArgs &a, int mode, int layout, cudaStream_t stream) {
    if (a.gather != 0) {
        if (layout != 0 || mode != 0) return cudaErrorInvalidValue;
        const bool gv = (a.gather == 1 ? a.mcVel : a.peerVel[0]) != nullptr;
        if (a.gather == 1) return gv ? launch_k2<0, 0, true, 1>(a, stream) : launch_k2<0, 0, false, 1>(a, stream);
        return gv ? launch_k2<0, 0, true, 2>(a, stream) : launch_k2<0, 0, false, 2>(a, stream);
    }
    const bool vel = a.vel != nullptr;
#define AZ_K2(L, M) \
    if (layout == L && mode == M) return vel ? launch_k2<L, M, true>(a, stream) : launch_k2<L, M, false>(a, stream);
    AZ_K2(0, 0) AZ_K2(0, 1) AZ_K2(0, 2) AZ_K2(1, 0) AZ_K2(1, 1) AZ_K2(1, 2)
#undef AZ_K2
    return cudaErrorInvalidValue;
}

// ---------------------------------------------------------------------------------------------------
// K3: fused propagate + single-target screen (src/Constellation.zig:683-756).  Pass 1 propagates the
// target over the whole time axis (n_times cells).  Pass 2 is the K1 cell core with the store stage
// replaced by a running (min distance^2, first epoch index) per satellite: a warp owns one satellite
// over ALL epochs, reduces with shuffles and writes 12 bytes -- the 48 B/cell result block never exists.
// The reference rotates both vectors to ECEF with the same GMST first (:724,739); a common rotation
// leaves the distance unchanged, so it is skipped.  Both passes group epochs into lanes the same way
// (screen_lane_cells), so a satellite with the target's elements meets the track at distance 0.
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) sgp4_track_kernel(const ScreenArgs a) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t tw = (i >> 5) * (32u * kScreenLanes), lane = i & 31u;
    if (tw >= a.nTimes) return;
    const double *tile = a.sgp4Tiles + (size_t)(a.targetIdx / kTileSats) * kSgp4TileDoubles + (a.targetIdx % kTileSats);
    auto col = [tile](int c) { return __ldg(tile + c * kTileSats); };
    auto tbase = [&a](uint32_t t) { return __ldg(a.tbase + t); };
    uint32_t tk[kScreenLanes];
    CellOut o[kScreenLanes];
    screen_lane_cells(col, tbase, __ldg(a.toff + a.targetIdx), a.nTimes, tw, lane, a.g, tk, o);
#pragma unroll
    for (int k = 0; k < kScreenLanes; ++k) {
        if (tk[k] >= a.nTimes) continue;
        a.track[(size_t)tk[k] * 3 + 0] = o[k].rx;
        a.track[(size_t)tk[k] * 3 + 1] = o[k].ry;
        a.track[(size_t)tk[k] * 3 + 2] = o[k].rz;
    }
}

constexpr int kScreenWarps = 4;

__global__ void __launch_bounds__(kScreenWarps * 32, 3) sgp4_screen_kernel(const ScreenArgs a) {
    __shared__ __align__(128) double tile[kSgp4TileDoubles];
    __shared__ __align__(8) uint64_t bar;
    const uint32_t tileIdx = blockIdx.x;
    if (threadIdx.x == 0) mbar_init(&bar, 1);
    __syncthreads();
    if (threadIdx.x == 0) {
        mbar_expect_tx(&bar, kSgp4TileBytes);
        tma_bulk_g2s(tile, a.sgp4Tiles + (size_t)tileIdx * kSgp4TileDoubles, kSgp4TileBytes, &bar);
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    mbar_wait(&bar, 0);
#pragma unroll 1
    for (int sl = warp; sl < kTileSats; sl += kScreenWarps) {
        const uint32_t sat = tileIdx * kTileSats + sl;
        if (sat >= a.nSats) break;
        const double *colBase = tile + sl;
        auto col = [colBase](int i) { return colBase[i * kTileSats]; };
        const double toff = __ldg(a.toff + sat);
        auto tbase = [&a](uint32_t t) { return __ldg(a.tbase + t); };
        double best = a.thresholdSq;   // src/Constellation.zig:703-706: start at threshold^2, index 0
        uint32_t bestT = 0;
        if (sat != a.targetIdx) {
#pragma unroll 1
            for (uint32_t tw = 0; tw < a.nTimes; tw += 32 * kScreenLanes) {
                uint32_t tk[kScreenLanes];
                CellOut o[kScreenLanes];
                screen_lane_cells(col, tbase, toff, a.nTimes, tw, (uint32_t)lane, a.g, tk, o);
#pragma unroll
                for (int k = 0; k < kScreenLanes; ++k) {
                    if (tk[k] < a.nTimes) {
                        const double *tg = a.track + (size_t)tk[k] * 3;
                        const double dx = __ldg(tg) - o[k].rx, dy = __ldg(tg + 1) - o[k].ry, dz = __ldg(tg + 2) - o[k].rz;
                        const double d2 = screen_d2(dx, dy, dz);
                        if (d2 < best) {  // strict: the earliest epoch of the minimum wins (:745-748)
                            best = d2;
                            bestT = tk[k];
                        }
                    }
                }
            }
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) {
                const double ob = __shfl_xor_sync(0xffffffffu, best, off);
                const uint32_t ot = __shfl_xor_sync(0xffffffffu, bestT, off);
                if (ob < best || (ob == best && ot < bestT)) {
                    best = ob;
                    bestT = ot;
                }
            }
        }
        if (lane == 0) {
            a.minDist[sat] = sqrt(best);  // :753-755
            a.minT[sat] = (best < a.thresholdSq) ? bestT : 0u;
        }
    }
}

cudaError_t launch_sgp4_screen(const ScreenArgs &a, cudaStream_t stream) {
    if (a.nSats == 0 || a.nTimes == 0) return cudaSuccess;
    const uint32_t trackThreads = (a.nTimes + 32 * kScreenLanes - 1) / (32 * kScreenLanes) * 32;
    sgp4_track_kernel<<<(trackThreads + 127) / 128, 128, 0, stream>>>(a);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    const uint32_t tiles = (a.nSats + kTileSats - 1) / kTileSats;
    sgp4_screen_kernel<<<tiles, kScreenWarps * 32, 0, stream>>>(a);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------
// K4: coarse all-vs-all screen (bindings/python/src/conjunction.zig:11-149).  Same cell list and the same
// multiplicative hash as the reference; differences: the table is built with atomicExch (chain order is
// irrelevant to the result set), cell coordinates of a chain member are recomputed from its position
// instead of stored, and only the own cell + 13 lexicographically-forward neighbours are visited -- each
// cross-cell pair is met exactly once from the side whose offset is forward, same-cell pairs by other > s --
// instead of 27 cells with an other > s filter.  Output order is not the reference's (by epoch, then by
// satellite): callers get the same SET of (s, other, t) triples.  The per-(satellite, epoch) search is
// coarse_search (az_screen.cuh).
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ const double *coarse_pos(const CoarseArgs &a, uint32_t s, uint32_t t) {
    return a.pos + ((a.layout == 0) ? ((size_t)s * a.nTimes + t) * 3 : ((size_t)t * a.nSats + s) * 3);
}

__global__ void __launch_bounds__(256) coarse_build_kernel(const CoarseArgs a) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= a.nSats) return;
    const uint32_t tb = blockIdx.y, t = a.t0 + tb;
    const double *p = coarse_pos(a, s, t);
    if (!coarse_member(a.validMask, s, __ldg(p))) return;
    const uint32_t h = coarse_bucket(p, 1.0 / a.threshold, (1u << a.tableBits) - 1u);
    a.next[(size_t)tb * a.nSats + s] = atomicExch(a.head + ((size_t)tb << a.tableBits) + h, s);
}

__global__ void __launch_bounds__(256) coarse_pairs_kernel(const CoarseArgs a) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= a.nSats) return;
    const uint32_t tb = blockIdx.y, t = a.t0 + tb;
    const double *p = coarse_pos(a, s, t);
    if (!coarse_member(a.validMask, s, __ldg(p))) return;
    coarse_search(s, p, 1.0 / a.threshold, a.threshold * a.threshold, a.head + ((size_t)tb << a.tableBits),
                  a.next + (size_t)tb * a.nSats, (1u << a.tableBits) - 1u, a.validMask,
                  [&](uint32_t other) { return coarse_pos(a, other, t); },
                  [&](uint32_t other) {
                      const unsigned long long k = atomicAdd(a.count, 1ULL);
                      if (k < a.maxResults) {
                          a.pairs[2 * k] = min(s, other);
                          a.pairs[2 * k + 1] = max(s, other);
                          a.tIdx[k] = t;
                      }
                  });
}

cudaError_t launch_coarse_screen(const CoarseArgs &a, cudaStream_t stream) {
    if (a.nSats == 0 || a.tCount == 0) return cudaSuccess;
    cudaError_t e = cudaMemsetAsync(a.head, 0xff, ((size_t)a.tCount << a.tableBits) * 4, stream);
    if (e != cudaSuccess) return e;
    dim3 grid((a.nSats + 255) / 256, a.tCount);
    coarse_build_kernel<<<grid, 256, 0, stream>>>(a);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    coarse_pairs_kernel<<<grid, 256, 0, stream>>>(a);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------
// fp32 precision-study kernel (BASELINE config 5; no reference path).  Same mapping as K1.
// ---------------------------------------------------------------------------------------------------
template <bool kPhase64>
__global__ void __launch_bounds__(128, 4) sgp4_grid_f32_kernel(const GridArgs a) {
    __shared__ __align__(128) double tile[kSgp4TileDoubles];
    __shared__ __align__(8) uint64_t bar;
    const uint32_t tileIdx = blockIdx.x;
    if (threadIdx.x == 0) mbar_init(&bar, 1);
    __syncthreads();
    if (threadIdx.x == 0) {
        mbar_expect_tx(&bar, kSgp4TileBytes);
        tma_bulk_g2s(tile, a.sgp4Tiles + (size_t)tileIdx * kSgp4TileDoubles, kSgp4TileBytes, &bar);
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t t0 = blockIdx.y * 256, t1 = min(t0 + 256u, a.nTimes);
    mbar_wait(&bar, 0);
#pragma unroll 1
    for (int sl = warp; sl < kTileSats; sl += 4) {
        const uint32_t sat = tileIdx * kTileSats + sl;
        if (sat >= a.nSats) break;
        const double *colBase = tile + sl;
        auto col = [colBase](int i) { return colBase[i * kTileSats]; };
        const double toff = __ldg(a.toff + sat);
        const uint32_t row = __ldg(a.orig + sat);
#pragma unroll 1
        for (uint32_t t = t0 + lane; t < t1; t += 32) {
            CellOut o;
            sgp4_cell_f32<kPhase64>(col, __ldg(a.tbase + t) + toff, a.g, o);
            store_direct<0, true>(a, row, t, o);
        }
    }
}

cudaError_t launch_sgp4_grid_f32(const GridArgs &a, int phase64, cudaStream_t stream) {
    const uint32_t tiles = (a.nSats + kTileSats - 1) / kTileSats, stripes = (a.nTimes + 255) / 256;
    if (tiles == 0 || stripes == 0) return cudaSuccess;
    if (!a.vel) return cudaErrorInvalidValue;
    dim3 grid(tiles, stripes);
    if (phase64) sgp4_grid_f32_kernel<true><<<grid, 128, 0, stream>>>(a);
    else sgp4_grid_f32_kernel<false><<<grid, 128, 0, stream>>>(a);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------
// fp64 roofline denominator.  Two figures:
//   * the pipe's arithmetic peak: SMs x 64 DFMA lanes x 2 FLOP x the maximum SM clock;
//   * a live DFMA microbenchmark: 8 independent chains per thread, each x = fma(x, a, 0.5) -- the multiplier sits in one
//     register every instruction re-reads from the operand-reuse cache and the addend is an immediate, so the register
//     file serves one fresh 64-bit pair per DFMA (tools/fp64_probe.cu compares it with patterns that read more pairs),
//     run long enough for the clocks to settle
//     (~0.2 s of warm-up), best of 10.
// bench.py reports the roofline against the larger of the two.
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) dfma_peak_kernel(double *out, int iters, double a) {
    double x[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) x[k] = threadIdx.x * 1e-9 + k;
#pragma unroll 1
    for (int i = 0; i < iters; ++i) {
#pragma unroll
        for (int r = 0; r < 8; ++r) {
#pragma unroll
            for (int k = 0; k < 8; ++k) x[k] = fma(x[k], a, 0.5);  // SASS: DFMA R, R, Ra.reuse, 0.5 -- one live register read
        }
    }
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < 8; ++k) s += x[k];
    if (s == 1234.5678) out[0] = s;  // keep the chains alive without a real store
}

cudaError_t fp64_pipe_peak(double *flops) {
    int dev = 0, sms = 0, khz = 0;
    cudaError_t rc = cudaGetDevice(&dev);
    if (rc != cudaSuccess) return rc;
    rc = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (rc != cudaSuccess) return rc;
    rc = cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, dev);
    if (rc != cudaSuccess) return rc;
    *flops = (double)sms * 64.0 * 2.0 * (double)khz * 1e3;  // sm_90: 64 fp64 FMA lanes per SM
    return cudaSuccess;
}

cudaError_t measure_fp64_peak(double *flops) {
    int dev = 0, sms = 0;
    cudaError_t rc = cudaGetDevice(&dev);
    if (rc != cudaSuccess) return rc;
    rc = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (rc != cudaSuccess) return rc;
    double *d = nullptr;
    rc = cudaMalloc(&d, 8);
    if (rc != cudaSuccess) return rc;
    const int blocks = sms * 8, threads = 256, iters = 4096;  // 2^27 FLOP per block: ~4.2 ms per launch at an H100's peak
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    float best = 1e30f;
    for (int rep = 0; rep < 60; ++rep) {
        cudaEventRecord(e0);
        dfma_peak_kernel<<<blocks, threads>>>(d, iters, 0.999999);
        cudaEventRecord(e1);
        rc = cudaEventSynchronize(e1);
        if (rc != cudaSuccess) break;
        float ms = 0;
        cudaEventElapsedTime(&ms, e0, e1);
        if (rep >= 50) best = std::min(best, ms);
    }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    cudaFree(d);
    if (rc != cudaSuccess) return rc;
    *flops = 2.0 * 64.0 * (double)iters * (double)blocks * (double)threads / (best * 1e-3);
    return cudaSuccess;
}

}  // namespace az
