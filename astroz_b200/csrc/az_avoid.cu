// az_avoid.cu -- K16: collision-avoidance manoeuvre trials (az_avoid.cuh).
//
// One stream, no synchronisation:
//   1. avoid_prepare_kernel (a thread per trial): the checks, K10's first catalogue (one primary copy per trial) and
//      its query offsets;
//   2. launch_covariance on it at the burn times: x(t_b) and J;
//   3. avoid_burn_kernel: the post-burn state and the conversion batch;
//   4. launch_fit + launch_fit_deep (K8, B* held, K13's weights): the new sets;
//   5. launch_covariance on the new sets at the burn times: J';
//   6. avoid_transport_kernel: the conversion status, P' and K11's catalogue of two rows per trial;
//   7. launch_conjunction (K11, TEME) into the caller's record and status;
//   8. avoid_finish_kernel: the status precedence, zeros, the optional outputs.
// Every step works on one trial per row or query, so a trial's bytes do not depend on the batch or its order.
#include "az_avoid.cuh"
#include "az_kernels.cuh"

namespace az {

constexpr int kAvoidThreads = 128;

__global__ void __launch_bounds__(kAvoidThreads) avoid_prepare_kernel(const AvoidArgs a, const AvoidScratch s) {
    const uint32_t k = blockIdx.x * kAvoidThreads + threadIdx.x;
    if (k < a.t) avoid_prepare(a, s, k);
}

__global__ void __launch_bounds__(kAvoidThreads) avoid_burn_kernel(const AvoidArgs a, const AvoidScratch s) {
    const uint32_t k = blockIdx.x * kAvoidThreads + threadIdx.x;
    if (k < a.t) avoid_burn(a, s, k);
}

__global__ void __launch_bounds__(kAvoidThreads) avoid_transport_kernel(const AvoidArgs a, const AvoidScratch s) {
    const uint32_t k = blockIdx.x * kAvoidThreads + threadIdx.x;
    if (k < a.t) avoid_transport(a, s, k);
}

__global__ void __launch_bounds__(kAvoidThreads) avoid_finish_kernel(const AvoidArgs a, const AvoidScratch s) {
    const uint32_t k = blockIdx.x * kAvoidThreads + threadIdx.x;
    if (k < a.t) avoid_finish(a, s, k);
}

// K10 over the t queries of a one-query-per-row catalogue at the burn times
static cudaError_t avoid_covariance_pass(const AvoidArgs &a, const AvoidScratch &s, const double *elements, double *J,
                                         double *state, uint8_t *status, cudaStream_t stream) {
    CovArgs c{};
    c.elements = elements;
    c.covariance = s.P1;
    c.model = s.model1;
    c.n = a.t;
    c.offsets = s.offsets;
    c.jd = a.burnJd;
    c.fr = a.burnFr;
    c.m = a.t;
    c.frame = kCovFrameTeme;
    c.grav = a.grav;
    c.g = a.g;
    c.state = state;
    c.sigma = s.sig;
    c.jacobian = J;
    c.status = status;
    return launch_covariance(c, stream);
}

cudaError_t launch_avoid(const AvoidArgs &a, cudaStream_t stream) {
    if (a.t == 0) return cudaSuccess;
    const AvoidScratch s = avoid_scratch(a.scratch, a.t);
    const uint32_t blocks = (a.t + kAvoidThreads - 1) / kAvoidThreads;
    avoid_prepare_kernel<<<blocks, kAvoidThreads, 0, stream>>>(a, s);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    if ((e = avoid_covariance_pass(a, s, s.el1, s.J, s.state, s.cov1St, stream)) != cudaSuccess) return e;
    avoid_burn_kernel<<<blocks, kAvoidThreads, 0, stream>>>(a, s);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    FitArgs f{};
    f.elements = s.init;
    f.n = a.t;
    f.offsets = s.offsets;
    f.jd = a.burnJd;
    f.fr = a.burnFr;
    f.pos = s.pos;
    f.vel = s.vel;
    f.wp = 1.0 / kIodFitPosSigma;
    f.wv = 1.0 / kIodFitVelSigma;
    f.fitBstar = 0;
    f.maxIter = kIodFitIter;
    f.grav = a.grav;
    f.g = a.g;
    f.fitted = s.fitted;
    f.rms = s.rms;
    f.iterations = s.iters;
    f.status = s.fitSt;
    if ((e = launch_fit(f, stream)) != cudaSuccess) return e;
    if ((e = launch_fit_deep(f, stream)) != cudaSuccess) return e;
    if ((e = avoid_covariance_pass(a, s, s.fitted, s.J2, nullptr, s.cov2St, stream)) != cudaSuccess) return e;
    avoid_transport_kernel<<<blocks, kAvoidThreads, 0, stream>>>(a, s);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    ConjArgs c{};
    c.elements = s.el2;
    c.covariance = s.P2;
    c.model = s.model2;
    c.n = 2 * a.t;
    c.primary = s.pri2;
    c.secondary = s.sec2;
    c.jd = s.jd2;
    c.fr = s.fr2;
    c.window = s.win2;
    c.hbr = s.hbr2;
    c.m = a.t;
    c.frame = kCovFrameTeme;
    c.grav = a.grav;
    c.g = a.g;
    c.record = a.record;
    c.status = a.status;
    if ((e = launch_conjunction(c, stream)) != cudaSuccess) return e;
    avoid_finish_kernel<<<blocks, kAvoidThreads, 0, stream>>>(a, s);
    return cudaGetLastError();
}

}  // namespace az
