// az_tasking.cu -- K18: sensor tasking (az_tasking.cuh).
//
// One build launch, then two or three launches per slot on the caller's stream, with no host synchronisation:
//   task_build_kernel     one thread per row: the row's nominal and stepped sets (deep space: Sdp4Sat records and the
//                         whole K2a lattice of each set) into the row's scratch slot, its nvar and status; the counters
//                         zeroed, posterior = covariance (the working P); threads < S resolve the sensors' frames;
//   task_score_kernel     one thread per row of its class (near-earth, deep space), the row's sets read from scratch:
//                         task_score at the slot, each sensor's gain (NaN: not visible) and visible cell words into
//                         scratch, the row's visible and failed counters;
//   task_select_kernel    one CTA: for k = 0 .. S-1 a block-wide (gain desc, row asc) reduction over the rows not yet
//                         taken in the slot, the task outputs, and then one thread per taken row writes its P+.
// The reductions are exact (a max and an integer count), so no byte depends on the CTA shape.
#include "az_kernels.cuh"
#include "az_tasking.cuh"

namespace az {

constexpr int kTaskThreads = 128;
constexpr int kTaskSelectThreads = 256;

// The scratch of task_scratch_bytes
struct TaskScratch {
    TaskSensor *sensors;   // [S]
    char *rows;            // [n][task_row_bytes()]
    double *inv;           // [n][kFitSets]
    int *nvar;             // [n], -1: not built
    double *gain;          // [S][n]
    double *cell;          // [S][n][kTaskCellWords]
    uint32_t *taken;       // [n] the last slot that took the row
};

static TaskScratch task_scratch(void *p, uint32_t n, uint32_t S) {
    TaskScratch c;
    char *b = static_cast<char *>(p);
    c.sensors = reinterpret_cast<TaskSensor *>(b);
    b += ((sizeof(TaskSensor) * S) + 15) & ~size_t(15);
    c.rows = b;
    b += (size_t)n * task_row_bytes();
    c.inv = reinterpret_cast<double *>(b);
    c.gain = c.inv + (size_t)n * kFitSets;
    c.cell = c.gain + (size_t)S * n;
    c.nvar = reinterpret_cast<int *>(c.cell + (size_t)S * n * kTaskCellWords);
    c.taken = reinterpret_cast<uint32_t *>(c.nvar + n);
    return c;
}

struct TaskDeepRow {
    Sdp4Sat sets[kFitSets];
    double2 lattice[kFitSets][2 * kFitLatticeNodes];
};

__global__ void __launch_bounds__(kTaskThreads) task_build_kernel(const TaskArgs a, const TaskScratch sc) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < a.S) task_sensor(a.kind, a.station, a.stations, a.sigma, a.limits, (int)s, sc.sensors[s]);
    if (s >= a.n) return;
    const uint8_t md = a.model ? a.model[s] : 0;
    double el0[8], P[kFitN];
#pragma unroll
    for (int c = 0; c < 8; ++c) el0[c] = a.elements[(size_t)c * a.n + s];
#pragma unroll
    for (int q = 0; q < kFitN; ++q) {
        P[q] = a.covariance ? a.covariance[(size_t)s * kFitN + q] : 0.0;
        a.posterior[(size_t)s * kFitN + q] = P[q];
    }
    const int nvar = corr_nvar(P);
    const Gravity grav = gravity(a.grav);
    double *inv = sc.inv + (size_t)s * kFitSets;
    char *slot = sc.rows + (size_t)s * task_row_bytes();
    bool built = md <= 1;
    double x[kFitVars];
    if (built && md == 0) {
        FitNearEarth::vars_of(el0, x);
        double(*cols)[kSgp4Cols] = reinterpret_cast<double(*)[kSgp4Cols]>(slot);
#pragma unroll 1
        for (int k = 0; k <= nvar && built; ++k) built = fit_build_set(x, k, el0[0], grav, cols[k], inv[k]);
    } else if (built) {
        FitDeepSpace::vars_of(el0, x);
        TaskDeepRow &r = *reinterpret_cast<TaskDeepRow *>(slot);
#pragma unroll 1
        for (int k = 0; k <= nvar && built; ++k)
            built = fit_build_set_of<FitDeepSpace>(x, k, el0[0], grav, r.sets[k], inv[k]);
#pragma unroll 1
        for (int k = 0; k <= nvar && built; ++k)
            for (int dir = 0; dir < 2; ++dir) fit_deep_lattice(r.sets[k], dir, kFitLatticeNodes, r.lattice[k]);
    }
    sc.nvar[s] = built ? nvar : -1;
    sc.taken[s] = kTaskIdle;
    a.nTasks[s] = a.nVisible[s] = a.nFailed[s] = 0;
    a.rowStatus[s] = built ? kCovOk : kCovInitFailed;
}

struct TaskNear {
    __device__ static bool takes(uint8_t model) { return model != 1; }
    __device__ static auto evaluator(const char *slot, const GravConsts &g) {
        const double(*cols)[kSgp4Cols] = reinterpret_cast<const double(*)[kSgp4Cols]>(slot);
        return [cols, &g](int k, double, const double (&ts)[1], double (&f)[6]) {
            CellOut o[1];
            sgp4_cell<1>([cols, k](int c) { return cols[k][c]; }, ts, g, o);
            f[0] = o[0].rx; f[1] = o[0].ry; f[2] = o[0].rz;
            f[3] = o[0].vx; f[4] = o[0].vy; f[5] = o[0].vz;
            return true;
        };
    }
};

struct TaskDeep {
    __device__ static bool takes(uint8_t model) { return model == 1; }
    __device__ static auto evaluator(const char *slot, const GravConsts &g) {
        const TaskDeepRow *r = reinterpret_cast<const TaskDeepRow *>(slot);
        return [r, &g](int k, double jdFull, const double (&)[1], double (&f)[6]) {
            return fit_deep_eval(r->sets[k], r->lattice[k], jdFull, g, f);
        };
    }
};

template <typename K>
__device__ __forceinline__ void task_score_body(const TaskArgs &a, const TaskScratch &sc, uint32_t t) {
    __shared__ TaskSensor sensors[kTaskMaxSensors];
    for (uint32_t k = threadIdx.x; k < a.S; k += blockDim.x) sensors[k] = sc.sensors[k];
    __syncthreads();
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= a.n) return;
    const uint8_t md = a.model ? __ldg(a.model + s) : 0;
    if (!K::takes(md)) return;
    const int nvar = sc.nvar[s];
    if (nvar < 0) {
        for (uint32_t k = 0; k < a.S; ++k) sc.gain[(size_t)k * a.n + s] = NAN;
        return;
    }
    double u[3] = {0.0, 0.0, 0.0};
    if (a.sun) task_sun(a.sun + (size_t)t * 3, u);
    const double jdFull = add_rn(__ldg(a.jd + t), __ldg(a.fr + t));
    const double epoch = __ldg(a.elements + s);
    double P[kFitN];
#pragma unroll
    for (int q = 0; q < kFitN; ++q) P[q] = a.posterior[(size_t)s * kFitN + q];
    uint32_t failed = 0;
    const uint32_t visible = task_score(
        K::evaluator(sc.rows + (size_t)s * task_row_bytes(), a.g), nvar, sc.inv + (size_t)s * kFitSets, epoch, jdFull,
        sensors, (int)a.S, u, P,
        [&](int k, double g, const double (&h)[6], const double (&spread)[4], const double (&G)[4][kFitVars]) {
            double *c = sc.cell + ((size_t)k * a.n + s) * kTaskCellWords;
            for (int q = 0; q < 4; ++q) {
                c[q] = h[q];
                c[4 + q] = spread[q];
            }
            for (int q = 0; q < 4; ++q)
                for (int j = 0; j < kFitVars; ++j) c[8 + q * kFitVars + j] = G[q][j];
            sc.gain[(size_t)k * a.n + s] = g;
        },
        failed);
    uint32_t nv = 0;
    for (uint32_t k = 0; k < a.S; ++k) {
        if (visible >> k & 1u) ++nv;
        else sc.gain[(size_t)k * a.n + s] = NAN;
    }
    a.nVisible[s] += nv;
    a.nFailed[s] += failed;
}

__global__ void __launch_bounds__(kTaskThreads) task_score_kernel(const TaskArgs a, const TaskScratch sc, uint32_t t) {
    task_score_body<TaskNear>(a, sc, t);
}

__global__ void __launch_bounds__(kTaskThreads) task_score_deep_kernel(const TaskArgs a, const TaskScratch sc,
                                                                       uint32_t t) {
    task_score_body<TaskDeep>(a, sc, t);
}

// (g, r) ahead of (bg, br): larger gain, then lower row
__device__ __forceinline__ bool task_ahead(double g, uint32_t r, double bg, uint32_t br) {
    return g > bg || (g == bg && r < br);
}

__global__ void __launch_bounds__(kTaskSelectThreads) task_select_kernel(const TaskArgs a, const TaskScratch sc,
                                                                          uint32_t t) {
    constexpr int kWarps = kTaskSelectThreads / 32;
    __shared__ double wg[kWarps];
    __shared__ uint32_t wr[kWarps], wc[kWarps];
    __shared__ uint32_t picks[kTaskMaxSensors];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (uint32_t k = 0; k < a.S; ++k) {
        double bg = -INFINITY;
        uint32_t br = kTaskIdle, cnt = 0;
        for (uint32_t s = tid; s < a.n; s += kTaskSelectThreads) {
            const double g = sc.gain[(size_t)k * a.n + s];
            if (!(g > a.gainMin) || sc.taken[s] == t) continue;
            ++cnt;
            if (task_ahead(g, s, bg, br)) {
                bg = g;
                br = s;
            }
        }
#pragma unroll
        for (int m = 16; m > 0; m >>= 1) {
            const double og = __shfl_xor_sync(0xffffffffu, bg, m);
            const uint32_t orow = __shfl_xor_sync(0xffffffffu, br, m);
            cnt += __shfl_xor_sync(0xffffffffu, cnt, m);
            if (task_ahead(og, orow, bg, br)) {
                bg = og;
                br = orow;
            }
        }
        if (lane == 0) {
            wg[warp] = bg;
            wr[warp] = br;
            wc[warp] = cnt;
        }
        __syncthreads();
        if (tid == 0) {
            for (int w = 1; w < kWarps; ++w) {
                cnt += wc[w];
                if (task_ahead(wg[w], wr[w], bg, br)) {
                    bg = wg[w];
                    br = wr[w];
                }
            }
            const size_t o = (size_t)k * a.T + t;
            a.taskRow[o] = br;
            a.nCandidates[o] = cnt;
            a.taskGain[o] = br == kTaskIdle ? 0.0 : bg;
            const double *c = sc.cell + ((size_t)k * a.n + br) * kTaskCellWords;
            for (int q = 0; q < 4; ++q) {
                a.taskValue[o * 4 + q] = br == kTaskIdle ? 0.0 : c[q];
                a.taskSpread[o * 4 + q] = br == kTaskIdle ? 0.0 : c[4 + q];
            }
            if (br != kTaskIdle) sc.taken[br] = t;
            picks[k] = br;
        }
        __syncthreads();
    }
    // the taken rows' posteriors: distinct rows, one thread each
    if (tid < a.S && picks[tid] != kTaskIdle) {
        const uint32_t s = picks[tid];
        const double *c = sc.cell + ((size_t)tid * a.n + s) * kTaskCellWords;
        double G[4][kFitVars], L[kFitVars][kFitVars], P[kFitN], g, spread[4];
        for (int q = 0; q < 4; ++q)
            for (int j = 0; j < kFitVars; ++j) G[q][j] = c[8 + q * kFitVars + j];
        for (int q = 0; q < kFitN; ++q) P[q] = a.posterior[(size_t)s * kFitN + q];
        task_cholesky(P, L);
        task_update(G, L, sc.sensors[tid].sigma, g, spread, a.posterior + (size_t)s * kFitN);
        ++a.nTasks[s];
    }
}

cudaError_t launch_tasking(const TaskArgs &a, cudaStream_t stream) {
    const TaskScratch sc = task_scratch(a.scratch, a.n, a.S);
    const uint32_t threads = a.n > a.S ? a.n : a.S;
    task_build_kernel<<<(threads + kTaskThreads - 1) / kTaskThreads, kTaskThreads, 0, stream>>>(a, sc);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    const uint32_t blocks = (a.n + kTaskThreads - 1) / kTaskThreads;
    for (uint32_t t = 0; t < a.T; ++t) {
        if (a.n) {
            task_score_kernel<<<blocks, kTaskThreads, 0, stream>>>(a, sc, t);
            if (a.model) task_score_deep_kernel<<<blocks, kTaskThreads, 0, stream>>>(a, sc, t);
        }
        task_select_kernel<<<1, kTaskSelectThreads, 0, stream>>>(a, sc, t);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
    }
    return cudaSuccess;
}

}  // namespace az
