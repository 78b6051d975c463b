// az_link.cu -- K17: orbits from pairs of tracks (az_link.cuh).
//
// link_kernel runs one warp per pair, kLinkWarps pairs per CTA.  Every lane forms the pair's summary (the loads are
// broadcasts), then lane l takes the cells l, l + 32, ... of the (rho1, rho2, direction) grid, solves each cell's
// Lambert problem and scores every admissible slot on the probe observations into its own kLinkSeeds least
// (F_probe, key).  A butterfly merges the lanes' seed lists (keys are unique, so the order of the merge does not
// matter) and every lane ends with the pair's seeds; lane q < kLinkSeeds refines seed q over every observation of both
// tracks.  A second butterfly over (F, key) picks the winner, a ballot names its lane, and lane 0 writes the outputs
// and the winner's state and osculating initial set into K13's conversion batch.  K13's conversion fits then run on
// the same stream (launch_iod_conversion), and link_finish_kernel writes the statuses and conversion residuals.  A
// pair's bytes depend on its two tracks alone.
#include "az_kernels.cuh"
#include "az_link.cuh"

namespace az {

constexpr int kLinkWarps = 4;

__global__ void __launch_bounds__(kLinkWarps * 32) link_kernel(const LinkArgs a, const IodScratch sc) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t j = blockIdx.x * kLinkWarps + (threadIdx.x >> 5);
    if (j >= a.p) return;
    const CorrObsArrays in{a.jd, a.fr, a.kind, a.value, a.sigma, a.station, a.stations};
    const Gravity grav = gravity(a.grav);
    const double mu = grav.mu, rE = grav.radiusEarthKm;
    LinkPair pr;
    link_pair(in, a.offsets, a.t, __ldg(a.pairs + 2 * (size_t)j), __ldg(a.pairs + 2 * (size_t)j + 1), a.rMin, a.rMax,
              pr);
    LinkSeeds seeds;
    link_seeds_init(seeds);
    uint32_t scored = 0;
    if (pr.status == kLinkOk) {
        const uint32_t cells = link_cells(pr);
#pragma unroll 1
        for (uint32_t c = lane; c < cells; c += 32) scored += link_cell(in, pr, c, a.maxRevs, mu, rE, seeds);
    }
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) {
        double oF[kLinkSeeds];
        uint32_t oKey[kLinkSeeds];
#pragma unroll
        for (int q = 0; q < kLinkSeeds; ++q) {
            oF[q] = __shfl_xor_sync(0xffffffffu, seeds.F[q], m);
            oKey[q] = __shfl_xor_sync(0xffffffffu, seeds.key[q], m);
        }
#pragma unroll
        for (int q = 0; q < kLinkSeeds; ++q) link_seed_insert(seeds, oF[q], oKey[q]);
        scored += __shfl_xor_sync(0xffffffffu, scored, m);
    }
    LinkBest best;
    link_best_init(best);
    if (lane < (uint32_t)kLinkSeeds && seeds.F[lane] < INFINITY) link_refine(in, pr, seeds.key[lane], mu, rE, best);
    double F = best.F;
    uint32_t key = best.key;
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) {
        const double oF = __shfl_xor_sync(0xffffffffu, F, m);
        const uint32_t oKey = __shfl_xor_sync(0xffffffffu, key, m);
        if (iod_better(oF, oKey, F, key)) F = oF, key = oKey;
    }
    const uint32_t won = __ballot_sync(0xffffffffu, best.key == key && best.F == F);
    const int src = won ? __ffs(won) - 1 : 0;
    double s[6], x[2];
#pragma unroll
    for (int c = 0; c < 6; ++c) s[c] = __shfl_sync(0xffffffffu, best.s[c], src);
    x[0] = __shfl_sync(0xffffffffu, best.x[0], src);
    x[1] = __shfl_sync(0xffffffffu, best.x[1], src);
    if (lane != 0) return;
    uint8_t status = pr.status;
    double state[6] = {0, 0, 0, 0, 0, 0}, el[8] = {0, 0, -1.0, 0, 0, 0, 0, 0};   // e = -1: the fit refuses the set
    uint8_t deep = 0;
    if (status == kLinkOk) {
        if (!(F < INFINITY)) status = kLinkNoCandidate;
        else {
            IodBest w;
            w.F = F;
            w.key = key;
            w.tRef = pr.an[1].t;
            for (int c = 0; c < 6; ++c) w.s[c] = s[c];
            const double bstar = a.bstar ? __ldg(a.bstar + j) : 0.0;
            if (!iod_epoch_state(w, pr.an[1].t, mu, bstar, grav, state, el, deep)) status = kLinkNoCandidate;
        }
    }
    const bool ok = status == kLinkOk;
    if (!ok) {
        for (int c = 0; c < 6; ++c) state[c] = 0.0;
        for (int c = 0; c < 8; ++c) el[c] = c == 2 ? -1.0 : 0.0;
        deep = 0;
    }
    const uint32_t ep = pr.an[1].index;
    for (int c = 0; c < 8; ++c) sc.init[(size_t)c * a.p + j] = el[c];
    sc.jd[j] = ok ? __ldg(a.jd + ep) : 0.0;
    sc.fr[j] = ok ? __ldg(a.fr + ep) : 0.0;
    for (int c = 0; c < 3; ++c) {
        sc.pos[(size_t)j * 3 + c] = state[c];
        sc.vel[(size_t)j * 3 + c] = state[3 + c];
    }
    sc.offsets[j] = j;
    if (j + 1 == a.p) sc.offsets[a.p] = a.p;
    sc.iodStatus[j] = status;
    for (int c = 0; c < 6; ++c) a.state[(size_t)j * 6 + c] = state[c];
    a.rho[2 * (size_t)j] = ok ? x[0] : 0.0;
    a.rho[2 * (size_t)j + 1] = ok ? x[1] : 0.0;
    a.revs[j] = ok ? (uint8_t)(key >> 18) : 0;
    a.flags[j] = ok ? link_flags(key) : 0;
    a.wrms[j] = ok ? std::sqrt(F / pr.used) : 0.0;
    const bool scoredPair = pr.status == kLinkOk;
    a.used[j] = scoredPair ? pr.used : 0;
    a.hypotheses[j] = scoredPair ? scored : 0;
    a.deepSpace[j] = deep;
}

__global__ void __launch_bounds__(128) link_finish_kernel(const LinkArgs a, const IodScratch sc) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= a.p) return;
    const uint8_t st = sc.iodStatus[j];
    const double dr = sc.rms[2 * (size_t)j], dv = sc.rms[2 * (size_t)j + 1];
    a.status[j] = iod_final_status(st, sc.fitStatus[j], dr, dv);
    a.conv[2 * (size_t)j] = st == kLinkOk ? dr : 0.0;
    a.conv[2 * (size_t)j + 1] = st == kLinkOk ? dv : 0.0;
    if (st != kLinkOk)
        for (int c = 0; c < 8; ++c) a.elements[(size_t)c * a.p + j] = 0.0;
}

cudaError_t launch_link(const LinkArgs &a, cudaStream_t stream) {
    if (a.p == 0) return cudaSuccess;
    const IodScratch sc = iod_scratch(a.scratch, a.p);
    link_kernel<<<(a.p + kLinkWarps - 1) / kLinkWarps, kLinkWarps * 32, 0, stream>>>(a, sc);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    if ((e = launch_iod_conversion(sc, a.p, a.grav, a.g, a.elements, stream)) != cudaSuccess) return e;
    link_finish_kernel<<<(a.p + 127) / 128, 128, 0, stream>>>(a, sc);
    return cudaGetLastError();
}

}  // namespace az
