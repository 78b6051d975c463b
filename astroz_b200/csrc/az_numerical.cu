// az_numerical.cu -- K7: numerical propagation of a batch of initial states (RK4 / Dormand-Prince 8(7), two-body with
// optional J2 and drag), one state per thread.  The per-state cores are in az_numerical.cuh.
//
// A state's whole trajectory is one thread's sequential loop; its state, its DP87 step size and the stages of the
// current attempt live in registers (tools/numerical_timing.py and DESIGN.md section 3 "K7 numerical" give the register
// counts of the eight specialisations).  The states of a batch are independent, so the batch is the parallel axis, and
// a state's bits depend on its own inputs alone.
#include "az_numerical.cuh"

namespace az {
namespace {

constexpr int kNumThreads = 64;

template <int kInt, int kForces>
__global__ void __launch_bounds__(kNumThreads) numerical_kernel(NumArgs a) {
    const uint32_t i = blockIdx.x * kNumThreads + threadIdx.x;
    if (i >= a.n) return;
    double y0[6];
#pragma unroll
    for (int c = 0; c < 6; ++c) y0[c] = a.states[(size_t)i * 6 + c];
    DragBody d{0.0, 0.0, 0.0};
    if (kForces & kForceDrag) d = DragBody{a.cd[i], a.area[i], a.mass[i]};
    uint64_t counts[2];
    const size_t samples = (size_t)a.steps.nFull + a.steps.nTail + 1;
    const uint8_t st = propagate_state<kInt, kForces>(y0, d, a.p, a.steps, a.out + (size_t)i * samples * 6, counts);
    a.status[i] = st;
    if (a.counts) {
        a.counts[(size_t)i * 2] = counts[0];
        a.counts[(size_t)i * 2 + 1] = counts[1];
    }
}

template <int kInt>
cudaError_t launch_forces(const NumArgs &a, int forces, dim3 grid, cudaStream_t s) {
    switch (forces) {
        case 0: numerical_kernel<kInt, 0><<<grid, kNumThreads, 0, s>>>(a); break;
        case kForceJ2: numerical_kernel<kInt, kForceJ2><<<grid, kNumThreads, 0, s>>>(a); break;
        case kForceDrag: numerical_kernel<kInt, kForceDrag><<<grid, kNumThreads, 0, s>>>(a); break;
        case kForceJ2 | kForceDrag: numerical_kernel<kInt, kForceJ2 | kForceDrag><<<grid, kNumThreads, 0, s>>>(a); break;
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

// The model-list specialisations: the integrator is a template parameter, the list a __grid_constant__ launch parameter
// the same for every thread, so each branch on a model's kind is warp-uniform and the list is read in place.
template <int kInt>
__global__ void __launch_bounds__(kNumThreads) numerical_models_kernel(const __grid_constant__ ModelArgs m) {
    const NumArgs &a = m.a;
    const uint32_t i = blockIdx.x * kNumThreads + threadIdx.x;
    if (i >= a.n) return;
    double y0[6];
#pragma unroll
    for (int c = 0; c < 6; ++c) y0[c] = a.states[(size_t)i * 6 + c];
    uint64_t counts[2];
    const size_t samples = (size_t)a.steps.nFull + a.steps.nTail + 1;
    const uint8_t st = propagate_state_models<kInt>(y0, m.models, i, a.p, a.steps, a.out + (size_t)i * samples * 6,
                                                    counts);
    a.status[i] = st;
    if (a.counts) {
        a.counts[(size_t)i * 2] = counts[0];
        a.counts[(size_t)i * 2 + 1] = counts[1];
    }
}

// Maneuver schedules: one state per thread, the list a __grid_constant__ parameter as above; each thread walks its own
// impulses, so a warp's lanes diverge where their schedules differ.
template <int kInt>
__global__ void __launch_bounds__(kNumThreads) maneuvers_kernel(const __grid_constant__ ManeuverArgs a) {
    const uint32_t i = blockIdx.x * kNumThreads + threadIdx.x;
    if (i >= a.n) return;
    double y0[6];
#pragma unroll
    for (int c = 0; c < 6; ++c) y0[c] = a.states[(size_t)i * 6 + c];
    const uint32_t b = a.offsets[a.first + i], e = a.offsets[a.first + i + 1];
    ManeuverRow row{a.times + (size_t)i * a.maxSamples, a.out + (size_t)i * a.maxSamples * 6, a.maxSamples, 0};
    uint64_t counts[2];
    const uint8_t st = maneuver_state_models<kInt>(y0, a.models, i, a.p, a.t0, a.tf, a.h, a.impulses + b, e - b, row,
                                                   counts);
    a.status[i] = st;
    a.count[i] = row.count;
    if (a.counts) {
        a.counts[(size_t)i * 2] = counts[0];
        a.counts[(size_t)i * 2 + 1] = counts[1];
    }
}

}  // namespace

cudaError_t launch_maneuvers(const ManeuverArgs &a, int integrator, cudaStream_t s) {
    if (a.n == 0) return cudaSuccess;
    const dim3 grid((a.n + kNumThreads - 1) / kNumThreads);
    if (integrator == kIntRk4) {
        maneuvers_kernel<kIntRk4><<<grid, kNumThreads, 0, s>>>(a);
    } else if (integrator == kIntDp87) {
        maneuvers_kernel<kIntDp87><<<grid, kNumThreads, 0, s>>>(a);
    } else {
        return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

cudaError_t launch_numerical_models(const ModelArgs &m, int integrator, cudaStream_t s) {
    if (m.a.n == 0) return cudaSuccess;
    const dim3 grid((m.a.n + kNumThreads - 1) / kNumThreads);
    if (integrator == kIntRk4) {
        numerical_models_kernel<kIntRk4><<<grid, kNumThreads, 0, s>>>(m);
    } else if (integrator == kIntDp87) {
        numerical_models_kernel<kIntDp87><<<grid, kNumThreads, 0, s>>>(m);
    } else {
        return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

cudaError_t launch_numerical(const NumArgs &a, int integrator, int forces, cudaStream_t s) {
    if (a.n == 0) return cudaSuccess;
    const dim3 grid((a.n + kNumThreads - 1) / kNumThreads);
    if (integrator == kIntRk4) return launch_forces<kIntRk4>(a, forces, grid, s);
    if (integrator == kIntDp87) return launch_forces<kIntDp87>(a, forces, grid, s);
    return cudaErrorInvalidValue;
}

}  // namespace az
