// TEST INFRASTRUCTURE ONLY: runs the product's fp64 math primitives (az_math.cuh, az_device.cuh, both included
// unchanged) over host arrays, either in a plain host loop -- the host build tests/host_emul runs -- or in a small
// kernel on the device, where the MUFU seeds (rcp.approx / rsqrt.approx) and the __constant__ table are the ones the
// propagation kernels use.  Not part of the shipped library; nothing in astroz_b200/ references it.
#include <cstdint>

#include "az_device.cuh"

using namespace az;

// One primitive on one element: inputs (x, y, z), outputs (a, b).  Operands each primitive reads are listed beside it.
enum ProbeOp : int {
    kRcpSeed, kRcpFast, kRcp, kDivNr,                       // (x) / (x) / (x) / (x / y)
    kRsqrtSeed, kRsqrtNr, kRsqrtNr1, kSqrt, kSqrtNr1,        // (x); kSqrtNr1 = sqrt_from_rsqrt(x, rsqrt_nr1(x))
    kSinCosFull, kSinCosQuarter, kSinCosTiny, kSinCosMicro,  // (x) -> (sin, cos)
    kRotateSmall,                                            // rotate_small_n<1>((x, y) = (sin a, cos a), d = z)
    kAtan2Seed, kAngleOfUnit,                                // (x, y) = (s, c)
    kResonanceNode,                                          // (x)
    kAbsGt, kAbsLt, kGeOne, kHalfOf, kExpo,                  // (x, high-word limit y)
    kFloorAt, kClampAbs,                                     // (x, high word y, value z)
    kNumOps
};

AZ_HD void probe_one(int op, double x, double y, double z, double &a, double &b) {
    b = 0.0;
    switch (op) {
        case kRcpSeed: a = rcp_seed(x); break;
        case kRcpFast: a = rcp_fast(x); break;
        case kRcp: a = rcp(x); break;
        case kDivNr: a = div_nr(x, y); break;
        case kRsqrtSeed: a = rsqrt_seed(x); break;
        case kRsqrtNr: a = rsqrt_nr(x); break;
        case kRsqrtNr1: a = rsqrt_nr1(x); break;
        case kSqrt: a = sqrt_(x); break;
        case kSqrtNr1: a = sqrt_from_rsqrt(x, rsqrt_nr1(x)); break;
        case kSinCosFull: sincos_full(x, a, b); break;
        case kSinCosQuarter: sincos_quarter(x, a, b); break;
        case kSinCosTiny: sincos_tiny(x, a, b); break;
        case kSinCosMicro: sincos_micro(x, a, b); break;
        case kRotateSmall: {
            const double s0[1] = {x}, c0[1] = {y}, d[1] = {z};
            double s[1], c[1];
            rotate_small_n<1>(s0, c0, d, s, c);
            a = s[0];
            b = c[0];
            break;
        }
        case kAtan2Seed: a = (double)atan2_seed((float)x, (float)y); break;
        case kAngleOfUnit: a = angle_of_unit(x, y); break;
        case kResonanceNode: a = (double)resonance_node(x); break;
        case kAbsGt: a = abs_gt(x, (uint32_t)y) ? 1.0 : 0.0; break;
        case kAbsLt: a = abs_lt(x, (uint32_t)y) ? 1.0 : 0.0; break;
        case kGeOne: a = ge_one(x) ? 1.0 : 0.0; break;
        case kHalfOf: a = half_of(x); break;
        case kExpo: a = (double)expo(x); break;
        case kFloorAt: a = floor_at(x, (uint32_t)y, z); break;
        case kClampAbs: a = clamp_abs(x, (uint32_t)y, z); break;
        default: a = b = 0.0; break;
    }
}

__global__ void probe_kernel(int op, const double *x, const double *y, const double *z, int n, double *a, double *b) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) probe_one(op, x[i], y[i], z[i], a[i], b[i]);
}

// Runs `op` over n elements on the host (device == 0) or on the current CUDA device (device != 0).  Returns 0, -1 for
// an unknown op, or the cudaError_t of the first failing CUDA call.
extern "C" int probe_eval(int op, const double *x, const double *y, const double *z, int n, double *a, double *b,
                          int device) {
    if (op < 0 || op >= kNumOps || n < 0) return -1;
    if (!device) {
        for (int i = 0; i < n; ++i) probe_one(op, x[i], y[i], z[i], a[i], b[i]);
        return 0;
    }
    if (n == 0) return 0;
    const size_t bytes = (size_t)n * sizeof(double);
    double *d[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
    cudaError_t rc = cudaSuccess;
    for (int k = 0; k < 5 && rc == cudaSuccess; ++k) rc = cudaMalloc(&d[k], bytes);
    if (rc == cudaSuccess) rc = cudaMemcpy(d[0], x, bytes, cudaMemcpyHostToDevice);
    if (rc == cudaSuccess) rc = cudaMemcpy(d[1], y, bytes, cudaMemcpyHostToDevice);
    if (rc == cudaSuccess) rc = cudaMemcpy(d[2], z, bytes, cudaMemcpyHostToDevice);
    if (rc == cudaSuccess) {
        probe_kernel<<<(n + 127) / 128, 128>>>(op, d[0], d[1], d[2], n, d[3], d[4]);
        rc = cudaGetLastError();
    }
    if (rc == cudaSuccess) rc = cudaMemcpy(a, d[3], bytes, cudaMemcpyDeviceToHost);
    if (rc == cudaSuccess) rc = cudaMemcpy(b, d[4], bytes, cudaMemcpyDeviceToHost);
    for (int k = 0; k < 5; ++k)
        if (d[k]) cudaFree(d[k]);
    return (int)rc;
}

// The selector thresholds and table values the primitives are used with, so the tests read them from the product
// headers instead of restating them: high words kHiTiny, kHiQuarter, kHiClamp, kHiEmFloor, kHiMicro, kHiLinear, then
// the values tinyLimit, quarterLimit, clamp, emFloor, microLimit, linearLimit.
extern "C" int probe_constants(double *out, int n) {
    const double v[12] = {(double)kHiTiny, (double)kHiQuarter, (double)kHiClamp, (double)kHiEmFloor, (double)kHiMicro,
                          (double)kHiLinear, kMathHost.tinyLimit, kMathHost.quarterLimit, kMathHost.clamp,
                          kMathHost.emFloor, kMathHost.microLimit, kMathHost.linearLimit};
    for (int i = 0; i < n && i < 12; ++i) out[i] = v[i];
    return 12;
}
