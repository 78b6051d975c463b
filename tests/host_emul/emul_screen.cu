// TEST INFRASTRUCTURE ONLY: runs the per-thread code of the two conjunction screens (az_screen.cuh, __host__ __device__)
// on the CPU, so the hit sets of K4 and the lane shape of K3 can be checked without a GPU.  Not part of the shipped
// library; nothing in astroz_b200/ references it.
#include <cstdint>
#include <vector>

#include "az_screen.cuh"
#include "az_tables.hpp"

using namespace az;

// K4 over a whole block, epoch by epoch: the table build of coarse_build_kernel (chains in row order instead of atomic
// order, which does not change the set) and coarse_search per row.  Returns the number of hits; the first max_results
// go to pairs[k][2] (smaller row first) and t_idx[k].
extern "C" uint64_t emul_coarse_screen(const double *pos, uint32_t ns, uint32_t nt, int layout, double threshold,
                                       const uint8_t *valid_mask, uint32_t *pairs, uint32_t *t_idx,
                                       uint64_t max_results) {
    constexpr uint32_t kBits = 16, kMask = (1u << kBits) - 1u;
    std::vector<uint32_t> head(1u << kBits), next(ns);
    auto at = [&](uint32_t s, uint32_t t) {
        return pos + (layout == 0 ? ((size_t)s * nt + t) * 3 : ((size_t)t * ns + s) * 3);
    };
    const double inv = 1.0 / threshold, thr2 = threshold * threshold;
    uint64_t count = 0;
    for (uint32_t t = 0; t < nt; ++t) {
        std::fill(head.begin(), head.end(), kCoarseEmpty);
        for (uint32_t s = 0; s < ns; ++s) {
            if (!coarse_member(valid_mask, s, at(s, t)[0])) continue;
            const uint32_t h = coarse_bucket(at(s, t), inv, kMask);
            next[s] = head[h];
            head[h] = s;
        }
        for (uint32_t s = 0; s < ns; ++s) {
            if (!coarse_member(valid_mask, s, at(s, t)[0])) continue;
            coarse_search(s, at(s, t), inv, thr2, head.data(), next.data(), kMask, valid_mask,
                          [&](uint32_t other) { return at(other, t); },
                          [&](uint32_t other) {
                              if (count < max_results) {
                                  pairs[2 * count] = s < other ? s : other;
                                  pairs[2 * count + 1] = s < other ? other : s;
                                  t_idx[count] = t;
                              }
                              ++count;
                          });
        }
    }
    return count;
}

static void track_cells(const CatalogTables &cat, const double *times, uint32_t nt, const double *epoch_offsets,
                        uint32_t sat, int lanes, double *out) {
    const GravConsts g = grav_consts(cat.grav);
    const double *tile = cat.sgp4Tiles.data() + (size_t)(sat / kTileSats) * kSgp4TileDoubles + sat % kTileSats;
    auto col = [tile](int c) { return tile[c * kTileSats]; };
    auto tbase = [times](uint32_t t) { return times[t]; };
    for (uint32_t tw = 0; tw < nt; tw += 32 * kScreenLanes) {
        for (uint32_t lane = 0; lane < 32; ++lane) {
            uint32_t tk[kScreenLanes];
            CellOut o[kScreenLanes];
            screen_lane_cells(col, tbase, epoch_offsets[sat], nt, tw, lane, g, tk, o);
            for (int k = 0; k < kScreenLanes; ++k) {
                if (tk[k] >= nt) continue;
                if (lanes == 1) {
                    const double ts[1] = {times[tk[k]] + epoch_offsets[sat]};
                    CellOut o1[1];
                    sgp4_cell<1>(col, ts, g, o1);
                    o[k] = o1[0];
                }
                out[3 * tk[k]] = o[k].rx;
                out[3 * tk[k] + 1] = o[k].ry;
                out[3 * tk[k] + 2] = o[k].rz;
            }
        }
    }
}

// Positions of near-earth row `sat` at tsince = times[t] + epoch_offsets[sat], in K3's lane shape (lanes = 2:
// screen_lane_cells, what both passes of K3 evaluate) or one cell per call (lanes = 1: sgp4_cell<1>).  out[nt][3].
extern "C" int emul_screen_track(const char *const *l1, const char *const *l2, uint32_t n, int grav, const double *times,
                                 uint32_t nt, const double *epoch_offsets, uint32_t sat, int lanes, double *out) {
    CatalogTables cat;
    int rc = build_catalog(l1, l2, n, grav, cat);
    if (rc != kOk) return rc;
    if (sat >= cat.nSgp4 || nt == 0) return -20;
    track_cells(cat, times, nt, epoch_offsets, sat, lanes, out);
    return 0;
}

// K3 on the CPU: the target's track and every other near-earth row in the screen's lane shape, K3's distance, the
// running (min d^2, first epoch) with the threshold as the start value, and the final sqrt.
extern "C" int emul_screen_conjunction(const char *const *l1, const char *const *l2, uint32_t n, int grav,
                                       const double *times, uint32_t nt, const double *epoch_offsets, uint32_t target,
                                       double threshold, double *min_dist, uint32_t *min_t) {
    CatalogTables cat;
    int rc = build_catalog(l1, l2, n, grav, cat);
    if (rc != kOk) return rc;
    const uint32_t ns = cat.nSgp4;
    if (target >= ns || nt == 0) return -20;
    std::vector<double> track((size_t)nt * 3), cells((size_t)nt * 3);
    track_cells(cat, times, nt, epoch_offsets, target, 2, track.data());
    const double thr2 = threshold * threshold;
    for (uint32_t s = 0; s < ns; ++s) {
        double best = thr2;
        uint32_t bestT = 0;
        if (s != target) {
            track_cells(cat, times, nt, epoch_offsets, s, 2, cells.data());
            for (uint32_t t = 0; t < nt; ++t) {
                const double d2 = screen_d2(track[3 * t] - cells[3 * t], track[3 * t + 1] - cells[3 * t + 1],
                                            track[3 * t + 2] - cells[3 * t + 2]);
                if (d2 < best) {
                    best = d2;
                    bestT = t;
                }
            }
        }
        min_dist[s] = sqrt(best);
        min_t[s] = best < thr2 ? bestT : 0u;
    }
    return 0;
}
