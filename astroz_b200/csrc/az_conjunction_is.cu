// az_conjunction_is.cu -- K15: importance-sampled collision probability of candidate conjunctions
// (az_conjunction_is.cuh).
//
// One stream:
//   1. linear shifts only: K11's launch (launch_conjunction, TEME, states on) into the scratch;
//   2. is_proposal_kernel, one warp per candidate: a given shift is copied; otherwise, on a K11 status of OK or
//      WINDOW_EDGE, lanes (row, set) rebuild each row's nominal and stepped sets in K11's layout (deep space with their
//      lattices), lanes 0 and 1 run K10's cov_query at K11's TCA for J and form their row's block of G, and lane 0
//      forms c and l0.  Anything else, or a failed J or C = 0, is PLAIN (c = 0);
//   3. is_prepare_kernel (K14's prepare step on K15's layouts, which also delivers the proposal) and the CUB scan;
//   4. conjunction_is_kernel and conjunction_is_deep_kernel: K14's persistent item loop with the shift added to the
//      normals and the weighted sums accumulated (az_conjunction_mc_warp.cuh).
// The counts are integer sums and the proposal depends on its candidate alone, so no result depends on the launch
// shape, the batch or the order of the work items.
#include "az_conjunction_mc_warp.cuh"

namespace az {

constexpr int kIsPropWarps = 2;

struct IsPropSmem {
    union {
        double cols[kFitSets][kSgp4Cols];
        struct {
            Sdp4Sat sets[kFitSets];
            double2 lattice[kFitSets][2 * kFitLatticeNodes];
        } ds;
    } obj[2];
    double inv[2][kFitSets];
    double P[2][kFitN];
    double J[2][kCovJacWords];
    double f[2][6];
    double sig[2][kCovWords];
    double G[2][2][kFitVars];
    double c[kIsShift + 1];
};

__device__ __forceinline__ bool is_eval(const IsPropSmem &w, int o, int deep, int k, double ts, const GravConsts &g,
                                        double (&f)[6]) {
    if (deep) return conj_eval_deep(w.obj[o].ds.sets[k], w.obj[o].ds.lattice[k], ts, g, f);
    return conj_eval_near([&w, o, k](int c) { return w.obj[o].cols[k][c]; }, ts, g, f);
}

// The linear shift of candidate i from K11's TCA tca and TEME states st[12] into w.c (c, then |c|^2); false: PLAIN
__device__ __forceinline__ bool is_linear_warp(const ConjIsArgs &a, uint32_t i, double tca, const double *st,
                                               IsPropSmem &w, uint32_t lane) {
    const uint32_t idx[2] = {__ldg(a.primary + i), __ldg(a.secondary + i)};
    const int mdl[2] = {a.model ? (int)__ldg(a.model + idx[0]) : 0, a.model ? (int)__ldg(a.model + idx[1]) : 0};
    const Gravity grav = gravity(a.grav);
    const double jdFull = add_rn(__ldg(a.jd + i), __ldg(a.fr + i)), win = __ldg(a.window + i);
    // lanes (o, k): row o = lane / 16 builds its set k
    const uint32_t o = lane >> 4, k = lane & 15;
    double el[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) el[c] = __ldg(a.elements + (size_t)c * a.n + idx[o]);
    const double ts0[2] = {pairs_tsince_deep(jdFull, __ldg(a.elements + idx[0])),
                           pairs_tsince_deep(jdFull, __ldg(a.elements + idx[1]))};
    for (uint32_t q = lane; q < 2 * kFitN; q += 32)
        w.P[q / kFitN][q % kFitN] = __ldg(a.covariance + (size_t)idx[q / kFitN] * kFitN + q % kFitN);
    __syncwarp();
    const int nvar[2] = {cov_nvar(w.P[0]), cov_nvar(w.P[1])};
    bool ok = true;
    if ((int)k <= nvar[o]) {
        double x[kFitVars];
        if (mdl[o]) {
            FitDeepSpace::vars_of(el, x);
            ok = fit_build_set_of<FitDeepSpace>(x, (int)k, el[0], grav, w.obj[o].ds.sets[k], w.inv[o][k]);
        } else {
            FitNearEarth::vars_of(el, x);
            ok = fit_build_set(x, (int)k, el[0], grav, w.obj[o].cols[k], w.inv[o][k]);
        }
    }
    if (!__all_sync(0xffffffffu, ok)) return false;
    __syncwarp();
    {   // lanes (o, set, direction): the deep-space lattices over [ts0 - w, ts0 + w]
        const uint32_t set = (lane >> 1) & 7, dir = lane & 1;
        if (mdl[o] && (int)set <= nvar[o]) {
            const double hi = ts0[o] + win, lo = ts0[o] - win;
            const int nodes = fit_lattice_nodes(dir == 0 ? (hi > 0.0 ? hi : 0.0) : (lo < 0.0 ? -lo : 0.0));
            fit_deep_lattice(w.obj[o].ds.sets[set], (int)dir, nodes, w.obj[o].ds.lattice[set]);
        }
        __syncwarp();
    }
    double e[2][3], d[2];
    double fp[6], fs[6];
    for (int c = 0; c < 6; ++c) {
        fp[c] = st[c];
        fs[c] = st[6 + c];
    }
    ok = is_plane(fp, fs, e, d);
    if (ok && lane < 2) {   // lane r: row r's J at the TCA and its block of G
        const int r = (int)lane, dp = mdl[r];
        const double ts = ts0[r] + tca;
        auto eval = [&w, &a, r, dp, ts](int kk, double, const double (&)[1], double (&f)[6]) {
            return is_eval(w, r, dp, kk, ts, a.g, f);
        };
        ok = cov_query(eval, nvar[r], w.inv[r], w.P[r], 0.0, 0.0, kCovFrameTeme, w.J[r], 1, w.f[r], w.sig[r]) ==
             kCovOk;
        McFactor F;
        ok = mc_factor(w.P[r], nvar[r], F) && ok;
        if (ok) is_row_map(w.J[r], F, e, r ? 1.0 : -1.0, w.G[r]);
    }
    if (!__all_sync(0xffffffffu, ok)) return false;
    __syncwarp();
    if (lane == 0) {
        double c[kIsShift], cc;
        ok = is_linear_shift(w.G[0], w.G[1], d, c, cc);
        for (int q = 0; q < kIsShift; ++q) w.c[q] = c[q];
        w.c[kIsShift] = cc;
    }
    return __shfl_sync(0xffffffffu, ok, 0);
}

__global__ void __launch_bounds__(kIsPropWarps * 32) is_proposal_kernel(const ConjIsArgs a, const double *k11Record,
                                                                       const double *k11States,
                                                                       const uint8_t *k11Status, double *prop,
                                                                       uint8_t *propKind) {
    __shared__ IsPropSmem smem[kIsPropWarps];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31, i = blockIdx.x * kIsPropWarps + warp;
    if (i >= a.m) return;
    IsPropSmem &w = smem[warp];
    double *out = prop + (size_t)i * kIsProposalWords;
    if (a.shift) {
        if (lane == 0) {
            const double *c = a.shift + (size_t)i * kIsShift;
            for (int q = 0; q < kIsShift; ++q) out[q] = c[q];
            out[kIsShift] = is_log_scale(is_norm2(c));
            propKind[i] = kIsGiven;
        }
        return;
    }
    const uint8_t k11 = k11Status[i];
    const bool linear = (k11 == kConjOk || k11 == kConjWindowEdge) &&
                        is_linear_warp(a, i, k11Record[(size_t)i * kConjRecordWords], k11States + (size_t)i * 12, w,
                                       lane);
    __syncwarp();
    if (lane < (uint32_t)kIsProposalWords)
        out[lane] = !linear ? 0.0 : lane < (uint32_t)kIsShift ? w.c[lane] : is_log_scale(w.c[kIsShift]);
    if (lane == 0) propKind[i] = linear ? kIsLinear : kIsPlain;
}

// K14's prepare step (mc_prepare_kernel) on K15's layouts, one thread per candidate: the status, zeroed counts, the NaN
// rows of sample_out that no sample writes, the work items, and the proposal (zero and PLAIN when not OK)
__global__ void __launch_bounds__(kMcPrepThreads) is_prepare_kernel(const ConjIsArgs a, uint64_t *items) {
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
    for (int q = 0; q < kIsCountWords; ++q) a.counts[(size_t)i * kIsCountWords + q] = 0;
    if (a.proposal)
        for (int q = 0; q < kIsProposalWords; ++q)
            a.proposal[(size_t)i * kIsProposalWords + q] = st == kConjOk ? a.prop[(size_t)i * kIsProposalWords + q] : 0.0;
    if (a.kind) a.kind[i] = st == kConjOk ? a.propKind[i] : (uint8_t)kIsPlain;
    const uint64_t samples = __ldg(a.samples + i);
    const bool near = !bad && mdl[0] == 0 && mdl[1] == 0;
    const uint64_t n = st == kConjOk ? mc_items(samples, near ? kMcNearB : kMcDeepB) : 0;
    items[i] = near ? n : 0;
    items[(size_t)a.m + i] = near ? 0 : n;
    const uint64_t from = st == kConjOk ? (samples < a.record ? samples : a.record) : 0;
    for (uint64_t r = from; r < a.record; ++r)
        for (int q = 0; q < kIsSampleWords; ++q)
            a.sampleOut[((size_t)i * a.record + r) * kIsSampleWords + q] = std::numeric_limits<double>::quiet_NaN();
}

// K14's near-earth kernel fits 4 CTAs per SM at 128 registers; the weights would take this one to 162 and 3 CTAs
__global__ void __launch_bounds__(kMcNearWarps * 32, 4) conjunction_is_kernel(const ConjIsArgs a, const uint64_t *prefix) {
    __shared__ McWarpSmem<false> smem[kMcNearWarps];
    const uint32_t warp = threadIdx.x >> 5;
    mc_run<false>(a, prefix, 0, smem[warp], warp, kMcNearWarps);
}

__global__ void __launch_bounds__(kMcDeepWarps * 32) conjunction_is_deep_kernel(const ConjIsArgs a,
                                                                                const uint64_t *prefix) {
    __shared__ McWarpSmem<true> smem[kMcDeepWarps];
    const uint32_t warp = threadIdx.x >> 5;
    mc_run<true>(a, prefix + a.m, prefix[a.m - 1], smem[warp], warp, kMcDeepWarps);
}

// The scratch: K14's (work items, prefix, scan), then from a 256-byte offset K11's record[m][13] and states[m][12],
// the proposals[m][15], K11's status[m] and the kinds[m]
static size_t is_k11_offset(size_t mcBytes) { return (mcBytes + 255) & ~size_t(255); }

cudaError_t conj_is_scratch_bytes(uint32_t m, size_t *bytes) {
    size_t mc = 0;
    const cudaError_t e = conj_mc_scratch_bytes(m, &mc);
    *bytes = is_k11_offset(mc) + (size_t)8 * (kConjRecordWords + 12 + kIsProposalWords) * m + (size_t)2 * m;
    return e;
}

cudaError_t launch_conjunction_is(const ConjIsArgs &a, cudaStream_t stream) {
    if (a.m == 0) return cudaSuccess;
    size_t mc = 0;
    cudaError_t e = conj_mc_scratch_bytes(a.m, &mc);
    if (e != cudaSuccess) return e;
    double *rec = reinterpret_cast<double *>(static_cast<char *>(a.scratch) + is_k11_offset(mc));
    double *states = rec + (size_t)kConjRecordWords * a.m, *prop = states + (size_t)12 * a.m;
    uint8_t *k11Status = reinterpret_cast<uint8_t *>(prop + (size_t)kIsProposalWords * a.m), *kind = k11Status + a.m;
    if (!a.shift) {
        ConjArgs c{};
        c.elements = a.elements;
        c.covariance = a.covariance;
        c.model = a.model;
        c.n = a.n;
        c.primary = a.primary;
        c.secondary = a.secondary;
        c.jd = a.jd;
        c.fr = a.fr;
        c.window = a.window;
        c.hbr = a.hbr;
        c.m = a.m;
        c.frame = kCovFrameTeme;
        c.grav = a.grav;
        c.g = a.g;
        c.record = rec;
        c.states = states;
        c.status = k11Status;
        if ((e = launch_conjunction(c, stream)) != cudaSuccess) return e;
    }
    is_proposal_kernel<<<(a.m + kIsPropWarps - 1) / kIsPropWarps, kIsPropWarps * 32, 0, stream>>>(a, rec, states,
                                                                                                 k11Status, prop, kind);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    ConjIsArgs b = a;
    b.prop = prop;
    b.propKind = kind;
    return mc_launch(b, is_prepare_kernel, conjunction_is_kernel, conjunction_is_deep_kernel, a.scratch, stream);
}

}  // namespace az
