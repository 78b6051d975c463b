// az_lambert.cu -- K9: batched Lambert solves and porkchop grids on the device, one problem (or cell) per thread.
//
// The per-problem arithmetic is az_lambert.cuh's lambert_solve; this file gives it its two shapes:
//   lambert_kernel:   problem i writes its S = 2 max_revs + 1 slots at [i][S];
//   porkchop_kernel:  cell (p, d, a) of P pairs x D departures x A arrivals, arrival index fastest, so a warp shares one
//                     chaser state and its neighbouring tofs have nearly the same revolution count.
// TEME is treated as inertial over a transfer: the frame's slow precession is far below the solver's closure.
// Compiled with -fmad=false, so the host build of the core equals a scalar C statement of it bit for bit wherever no
// libm / libdevice transcendental differs.
#include "az_lambert.cuh"

namespace az {

constexpr int kLamThreads = 128;

__global__ void __launch_bounds__(kLamThreads) lambert_kernel(const LambertArgs a) {
    const size_t i = (size_t)blockIdx.x * kLamThreads + threadIdx.x;
    if (i >= a.n) return;
    double r1[3], r2[3], n[3] = {0.0, 0.0, 1.0};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        r1[k] = __ldg(a.r1 + 3 * i + k);
        r2[k] = __ldg(a.r2 + 3 * i + k);
        if (a.normal) n[k] = __ldg(a.normal + 3 * i + k);
    }
    const size_t base = i * (2 * (size_t)a.maxRevs + 1);
    lambert_solve(r1, r2, __ldg(a.tof + i), a.mu, n, a.maxRevs,
                  [&](uint32_t s, uint8_t st, int it, const double v1[3], const double v2[3]) {
                      const size_t o = base + s;
#pragma unroll
                      for (int k = 0; k < 3; ++k) {
                          a.v1[3 * o + k] = v1[k];
                          a.v2[3 * o + k] = v2[k];
                      }
                      a.status[o] = st;
                      if (a.iterations) a.iterations[o] = (uint8_t)it;
                  });
}

__global__ void __launch_bounds__(kLamThreads) porkchop_kernel(const PorkchopArgs a) {
    const size_t cell = (size_t)blockIdx.x * kLamThreads + threadIdx.x;
    const size_t perPair = (size_t)a.D * a.A;
    if (cell >= (size_t)a.P * perPair) return;
    const size_t p = cell / perPair, rem = cell - p * perPair;
    const uint32_t d = (uint32_t)(rem / a.A), ar = (uint32_t)(rem - (size_t)d * a.A);
    const size_t di = p * a.D + d, ai = p * a.A + ar;
    double dv[2] = {0.0, 0.0};
    uint8_t slot = 0, status = kLamStateFailed;
    if ((!a.depStatus || __ldg(a.depStatus + di) == 0) && (!a.arrStatus || __ldg(a.arrStatus + ai) == 0)) {
        double rc[3], vc[3], rt[3], vt[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            rc[k] = __ldg(a.depPos + di * a.stride + k);
            vc[k] = __ldg(a.depVel + di * a.stride + k);
            rt[k] = __ldg(a.arrPos + ai * a.stride + k);
            vt[k] = __ldg(a.arrVel + ai * a.stride + k);
        }
        const double tof = ((__ldg(a.arrJd + ar) - __ldg(a.depJd + d)) + (__ldg(a.arrFr + ar) - __ldg(a.depFr + d))) *
                           86400.0;
        lambert_porkchop_cell(rc, vc, rt, vt, tof, a.mu, a.maxRevs, dv, slot, status);
    }
    a.dv[2 * cell] = dv[0];
    a.dv[2 * cell + 1] = dv[1];
    a.slot[cell] = slot;
    a.status[cell] = status;
}

cudaError_t launch_lambert(const LambertArgs &a, cudaStream_t stream) {
    if (a.n == 0) return cudaSuccess;
    lambert_kernel<<<(a.n + kLamThreads - 1) / kLamThreads, kLamThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_porkchop(const PorkchopArgs &a, cudaStream_t stream) {
    const size_t cells = (size_t)a.P * a.D * a.A;
    if (cells == 0) return cudaSuccess;
    porkchop_kernel<<<(unsigned)((cells + kLamThreads - 1) / kLamThreads), kLamThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

}  // namespace az
