// TEST INFRASTRUCTURE ONLY: K14's Philox4x32-10 (az_conjunction_mc.cuh, included unchanged) and curand's
// curand_Philox4x32_10 on the device over the same counters and keys, so the in-repo generator can be compared with
// the vendor's bit for bit.  Not part of the shipped library; nothing in astroz_b200/ references it.
#include <cuda_runtime.h>
#include <curand_kernel.h>

#include "az_conjunction_mc.cuh"

using namespace az;

__global__ void probe_philox_kernel(const uint4 *ctr, const uint2 *key, uint32_t n, uint4 *ours, uint4 *theirs) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint4 c = ctr[i];
    const uint2 k = key[i];
    const McU4 o = mc_philox(McU4{c.x, c.y, c.z, c.w}, k.x, k.y);
    ours[i] = make_uint4(o.x, o.y, o.z, o.w);
    theirs[i] = curand_Philox4x32_10(c, k);
}

// ctr[n][4], key[n][2] host arrays -> ours[n][4], theirs[n][4]; returns a cudaError_t
extern "C" int probe_philox(const uint32_t *ctr, const uint32_t *key, uint32_t n, uint32_t *ours, uint32_t *theirs) {
    uint4 *dc = nullptr, *d1 = nullptr, *d2 = nullptr;
    uint2 *dk = nullptr;
    cudaError_t e = cudaMalloc(&dc, sizeof(uint4) * n);
    if (e == cudaSuccess) e = cudaMalloc(&dk, sizeof(uint2) * n);
    if (e == cudaSuccess) e = cudaMalloc(&d1, sizeof(uint4) * n);
    if (e == cudaSuccess) e = cudaMalloc(&d2, sizeof(uint4) * n);
    if (e == cudaSuccess) e = cudaMemcpy(dc, ctr, sizeof(uint4) * n, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(dk, key, sizeof(uint2) * n, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        probe_philox_kernel<<<(n + 255) / 256, 256>>>(dc, dk, n, d1, d2);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpy(ours, d1, sizeof(uint4) * n, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(theirs, d2, sizeof(uint4) * n, cudaMemcpyDeviceToHost);
    cudaFree(dc);
    cudaFree(dk);
    cudaFree(d1);
    cudaFree(d2);
    return (int)e;
}
