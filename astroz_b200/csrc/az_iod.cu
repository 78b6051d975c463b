// az_iod.cu -- K13: initial orbits of tracks (az_iod.cuh).
//
// iod_kernel runs one warp per track, kIodWarps tracks per CTA.  Every lane reads the track's summary (the loads are
// broadcasts), then lane l takes the track's generator slots l, l + 32, ... (iod_slots: a state observation, a Gibbs or
// Herrick-Gibbs triplet, a Lambert direction or a Gauss triplet), builds their candidates and scores each over every
// observation of the track; the lanes walk the observations in the same order, so each observation load is a warp
// broadcast.  A butterfly over (F, key) picks the winner (keys are unique, so the order of the reduction does not
// matter), a ballot names its lane, and lane 0 propagates the winner to the epoch and writes the state, the
// osculating initial set and one TEME-state observation per track into the conversion batch.  K8's own fit kernels
// then run over that batch on the same stream (launch_fit, launch_fit_deep), B* held, and iod_finish_kernel writes the
// statuses and conversion residuals.  A track's bytes depend on that track alone.
#include "az_iod.cuh"
#include "az_kernels.cuh"

namespace az {

constexpr int kIodWarps = 4;

IodScratch iod_scratch(void *p, uint32_t t) {
    IodScratch s;
    s.init = static_cast<double *>(p);
    s.jd = s.init + (size_t)8 * t;
    s.fr = s.jd + t;
    s.pos = s.fr + t;
    s.vel = s.pos + (size_t)3 * t;
    s.rms = s.vel + (size_t)3 * t;
    s.offsets = reinterpret_cast<uint32_t *>(s.rms + (size_t)2 * t);
    s.iters = s.offsets + t + 1;
    s.fitStatus = reinterpret_cast<uint8_t *>(s.iters + t);
    s.iodStatus = s.fitStatus + t;
    return s;
}

size_t iod_scratch_bytes(uint32_t t) { return (size_t)t * (8 + 2 + 6 + 2) * 8 + ((size_t)2 * t + 1) * 4 + 2 * (size_t)t; }

__global__ void __launch_bounds__(kIodWarps * 32) iod_kernel(const IodArgs a, const IodScratch sc) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t j = blockIdx.x * kIodWarps + (threadIdx.x >> 5);
    if (j >= a.t) return;
    const CorrObsArrays in{a.jd, a.fr, a.kind, a.value, a.sigma, a.station, a.stations};
    const Gravity grav = gravity(a.grav);
    const double mu = grav.mu, rE = grav.radiusEarthKm;
    IodTrack tr;
    iod_track(in, __ldg(a.offsets + j), __ldg(a.offsets + j + 1), tr);
    IodBest best;
    iod_best_init(best);
    uint32_t scored = 0;
    if (tr.status == kIodOk) {
        const uint32_t slots = iod_slots(tr);
#pragma unroll 1
        for (uint32_t g = lane; g < slots; g += 32) scored += iod_slot(in, tr, g, mu, rE, best);
    }
    double F = best.F;
    uint32_t key = best.key;
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) {
        const double oF = __shfl_xor_sync(0xffffffffu, F, m);
        const uint32_t oKey = __shfl_xor_sync(0xffffffffu, key, m);
        if (iod_better(oF, oKey, F, key)) F = oF, key = oKey;
        scored += __shfl_xor_sync(0xffffffffu, scored, m);
    }
    const uint32_t won = __ballot_sync(0xffffffffu, best.key == key && best.F == F);
    const int src = won ? __ffs(won) - 1 : 0;
    double s[6];
#pragma unroll
    for (int c = 0; c < 6; ++c) s[c] = __shfl_sync(0xffffffffu, best.s[c], src);
    const double tRef = __shfl_sync(0xffffffffu, best.tRef, src);
    if (lane != 0) return;
    uint8_t status = tr.status;
    double state[6] = {0, 0, 0, 0, 0, 0}, el[8] = {0, 0, -1.0, 0, 0, 0, 0, 0};   // e = -1: the fit refuses the set
    uint8_t deep = 0;
    if (status == kIodOk) {
        if (!(F < INFINITY)) status = kIodNoCandidate;
        else {
            IodBest w;
            w.F = F;
            w.key = key;
            w.tRef = tRef;
            for (int c = 0; c < 6; ++c) w.s[c] = s[c];
            const double bstar = a.bstar ? __ldg(a.bstar + j) : 0.0;
            if (!iod_epoch_state(w, tr.epoch, mu, bstar, grav, state, el, deep)) status = kIodNoCandidate;
        }
    }
    if (status != kIodOk) {
        for (int c = 0; c < 6; ++c) state[c] = 0.0;
        for (int c = 0; c < 8; ++c) el[c] = c == 2 ? -1.0 : 0.0;
        deep = 0;
    }
    const uint32_t mid = tr.begin + (tr.end - tr.begin) / 2;
    const bool ok = status == kIodOk;
    for (int c = 0; c < 8; ++c) sc.init[(size_t)c * a.t + j] = el[c];
    sc.jd[j] = ok ? __ldg(a.jd + mid) : 0.0;
    sc.fr[j] = ok ? __ldg(a.fr + mid) : 0.0;
    for (int c = 0; c < 3; ++c) {
        sc.pos[(size_t)j * 3 + c] = state[c];
        sc.vel[(size_t)j * 3 + c] = state[3 + c];
    }
    sc.offsets[j] = j;
    if (j + 1 == a.t) sc.offsets[a.t] = a.t;
    sc.iodStatus[j] = status;
    for (int c = 0; c < 6; ++c) a.state[(size_t)j * 6 + c] = state[c];
    a.wrms[j] = ok ? std::sqrt(F / tr.used) : 0.0;
    a.method[j] = ok ? (uint8_t)(key >> 16) : kIodNone;
    a.candidates[j] = scored;
    a.deepSpace[j] = deep;
}

__global__ void __launch_bounds__(128) iod_finish_kernel(const IodArgs a, const IodScratch sc) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= a.t) return;
    const uint8_t iod = sc.iodStatus[j];
    const double dr = sc.rms[2 * (size_t)j], dv = sc.rms[2 * (size_t)j + 1];
    a.status[j] = iod_final_status(iod, sc.fitStatus[j], dr, dv);
    a.conv[2 * (size_t)j] = iod == kIodOk ? dr : 0.0;
    a.conv[2 * (size_t)j + 1] = iod == kIodOk ? dv : 0.0;
    if (iod != kIodOk)
        for (int c = 0; c < 8; ++c) a.elements[(size_t)c * a.t + j] = 0.0;
}

cudaError_t launch_iod_conversion(const IodScratch &sc, uint32_t t, int grav, const GravConsts &g, double *elements,
                                  cudaStream_t stream) {
    FitArgs f{};
    f.elements = sc.init;
    f.n = t;
    f.offsets = sc.offsets;
    f.jd = sc.jd;
    f.fr = sc.fr;
    f.pos = sc.pos;
    f.vel = sc.vel;
    f.wp = 1.0 / kIodFitPosSigma;
    f.wv = 1.0 / kIodFitVelSigma;
    f.fitBstar = 0;
    f.maxIter = kIodFitIter;
    f.grav = grav;
    f.g = g;
    f.fitted = elements;
    f.rms = sc.rms;
    f.iterations = sc.iters;
    f.status = sc.fitStatus;
    cudaError_t e = launch_fit(f, stream);
    if (e != cudaSuccess) return e;
    return launch_fit_deep(f, stream);
}

cudaError_t launch_iod(const IodArgs &a, cudaStream_t stream) {
    if (a.t == 0) return cudaSuccess;
    const IodScratch sc = iod_scratch(a.scratch, a.t);
    iod_kernel<<<(a.t + kIodWarps - 1) / kIodWarps, kIodWarps * 32, 0, stream>>>(a, sc);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    if ((e = launch_iod_conversion(sc, a.t, a.grav, a.g, a.elements, stream)) != cudaSuccess) return e;
    iod_finish_kernel<<<(a.t + 127) / 128, 128, 0, stream>>>(a, sc);
    return cudaGetLastError();
}

}  // namespace az
