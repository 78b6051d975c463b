// az_screen.cuh -- per-thread logic of the two conjunction screens: K3's lane shape and K4's per-(satellite, epoch)
// cell-list search.  __host__ __device__, so tests/host_emul/emul_screen.cu runs the kernels' own code on the CPU.
#pragma once

#include <stdint.h>

#include "az_device.cuh"

namespace az {

template <typename T>
AZ_HD T ld_ro(const T *p) {  // read-only load: through the texture path on the device
#ifdef __CUDA_ARCH__
    return __ldg(p);
#else
    return *p;
#endif
}

// ---- K3: single-target screen ---------------------------------------------------------------------------------------
// Thread `lane` of a warp evaluates epochs tw + 32k + lane (k < kScreenLanes) of a run of 32 * kScreenLanes epochs in one
// sgp4_cell call; an epoch past the end of the axis evaluates the last epoch instead and is dropped by the caller.
// sgp4_cell chooses its series per thread over all of a thread's cells, so a cell's low bits depend on this grouping:
// the target track (pass 1) and the screen (pass 2) both use it, and a copy of the target reproduces the track exactly.
constexpr int kScreenLanes = 2;

template <typename ColFn, typename TimeFn>
AZ_HD void screen_lane_cells(ColFn col, TimeFn tbase, double toff, uint32_t nTimes, uint32_t tw, uint32_t lane,
                             const GravConsts &g, uint32_t (&tk)[kScreenLanes], CellOut (&o)[kScreenLanes]) {
    double ts[kScreenLanes];
#pragma unroll
    for (int k = 0; k < kScreenLanes; ++k) {
        tk[k] = tw + 32u * k + lane;
        ts[k] = tbase(tk[k] < nTimes ? tk[k] : nTimes - 1) + toff;
    }
    sgp4_cell<kScreenLanes>(col, ts, g, o);
}

// K3's own distance: contracted, unlike the reference's (src/Constellation.zig:743).  The reference also rotates
// both vectors to ECEF first, which K3 skips, so its d^2 differs from the reference's in the last bits either way.
AZ_HD double screen_d2(double dx, double dy, double dz) { return fma(dx, dx, fma(dy, dy, dz * dz)); }

// ---- K4: all-vs-all coarse screen (bindings/python/src/conjunction.zig:11-149) --------------------------------------
constexpr uint32_t kCoarseEmpty = 0xffffffffu;

AZ_HD uint32_t spatial_hash(uint32_t cx, uint32_t cy, uint32_t cz) {  // conjunction.zig:139-148
    uint32_t h = cx;
    h *= 2654435761u;
    h ^= cy;
    h *= 2654435761u;
    h ^= cz;
    h *= 2654435761u;
    return h;
}

// Cell coordinate floor(v) of v = position / threshold (formed as position * (1 / threshold), like the reference).
// Values beyond the int range saturate to INT32_MIN / INT32_MAX and NaN gives 0: the device conversion's behaviour,
// restated for the host, where the C cast is undefined.  Saturation is monotonic, so two positions closer than the
// threshold still land in the same or adjacent cells and no hit is lost; far positions that share a saturated cell
// are only extra candidates for the distance test.
AZ_HD int32_t coarse_cell(double v) {
#ifdef __CUDA_ARCH__
    return __double2int_rd(v);
#else
    if (v != v) return 0;
    const double f = floor(v);
    return f >= 2147483647.0 ? INT32_MAX : f <= -2147483648.0 ? INT32_MIN : (int32_t)f;
#endif
}

// A row takes part at an epoch when it is not masked out and its x is finite (conjunction.zig:60-63).  NaN or inf in y
// or z still enter the table; their distances compare false, so they never make a hit.
AZ_HD bool coarse_member(const uint8_t *validMask, uint32_t s, double x) {
    return !(validMask && validMask[s] == 0) && isfinite(x);
}

AZ_HD uint32_t coarse_bucket(const double *p, double inv, uint32_t mask) {
    return spatial_hash((uint32_t)coarse_cell(ld_ro(p) * inv), (uint32_t)coarse_cell(ld_ro(p + 1) * inv),
                        (uint32_t)coarse_cell(ld_ro(p + 2) * inv)) & mask;
}

// The reference's distance test (conjunction.zig:119-124): each product rounded, summed left to right, strict `<`.
// Written in rounded operations so nvcc cannot fuse it into FMAs, which decide differently within a few ulps of thr2.
AZ_HD bool coarse_hit(double dx, double dy, double dz, double thr2) {
    return add_rn(add_rn(mul_rn(dx, dx), mul_rn(dy, dy)), mul_rn(dz, dz)) < thr2;
}

// Every partner `other` of row s at one epoch: own cell + the 13 lexicographically forward neighbour cells, so a
// cross-cell pair is met exactly once (from the side whose offset is forward) and a same-cell pair by other > s.
// head / next: that epoch's bucket heads and chains; pos(i) the row's position; hit(other) is called once per pair.
// Neighbour coordinates are formed in uint32 (wrapping, like the hash's own arithmetic) so a saturated cell has no
// signed overflow.
template <typename PosFn, typename HitFn>
AZ_HD void coarse_search(uint32_t s, const double *p, double inv, double thr2, const uint32_t *head, const uint32_t *next,
                         uint32_t mask, const uint8_t *validMask, PosFn pos, HitFn hit) {
    const double sx = ld_ro(p), sy = ld_ro(p + 1), sz = ld_ro(p + 2);
    const uint32_t scx = (uint32_t)coarse_cell(sx * inv), scy = (uint32_t)coarse_cell(sy * inv),
                   scz = (uint32_t)coarse_cell(sz * inv);
#ifdef __CUDA_ARCH__
#pragma unroll 1
#endif
    for (int n = 13; n < 27; ++n) {  // offsets (dx,dy,dz) in lexicographic order: index 13 is (0,0,0), 14..26 are forward
        const uint32_t ncx = scx + (uint32_t)(n / 9 - 1), ncy = scy + (uint32_t)((n / 3) % 3 - 1),
                       ncz = scz + (uint32_t)(n % 3 - 1);
        uint32_t idx = ld_ro(head + (spatial_hash(ncx, ncy, ncz) & mask));
        while (idx != kCoarseEmpty) {
            const uint32_t other = idx;
            idx = ld_ro(next + other);
            if (other == s || (n == 13 && other < s)) continue;
            if (validMask && validMask[other] == 0) continue;
            const double *q = pos(other);
            const double ox = ld_ro(q), oy = ld_ro(q + 1), oz = ld_ro(q + 2);
            if ((uint32_t)coarse_cell(ox * inv) != ncx || (uint32_t)coarse_cell(oy * inv) != ncy ||
                (uint32_t)coarse_cell(oz * inv) != ncz)
                continue;  // hash collision: another cell in the same bucket (conjunction.zig:112-113)
            if (coarse_hit(sx - ox, sy - oy, sz - oz, thr2)) hit(other);
        }
    }
}

}  // namespace az
