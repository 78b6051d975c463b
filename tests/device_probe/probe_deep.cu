// TEST INFRASTRUCTURE ONLY: runs the product's deep-space cell (sdp4_cell, az_device.cuh, included unchanged) from
// a caller-supplied resonance state (xli, xni, atime), either in a plain host loop or in a small kernel on the device,
// where the MUFU seeds and the __constant__ tables are the ones the propagation kernels use.  This reaches branches of
// the cell that no element set does.  Not part of the shipped library; nothing in astroz_b200/ references it.
#include <cstdint>

#include "az_tables.hpp"

using namespace az;

__global__ void sdp4_cell_kernel(const Sdp4Sat e, const GravConsts g, const double *t, const double *xli,
                                 const double *xni, const double *atime, int n, double *out, int *st) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    CellOut c;
    st[i] = sdp4_cell(e, t[i], xli[i], xni[i], atime[i], g, c);
    const double r[6] = {c.rx, c.ry, c.rz, c.vx, c.vy, c.vz};
    for (int j = 0; j < 6; ++j) out[6 * i + j] = r[j];
}

// sdp4_cell of one deep-space element set at n cells (tsince, xli, xni, atime), on the host (device == 0) or the device.
// out [n][6] = (r, v) as the cell returns them, status [n].  Returns 0, -1 for an element set that is not a valid
// deep-space set, or the cudaError_t of the first failing CUDA call.
extern "C" int probe_sdp4_cell(const char *l1, const char *l2, int grav, const double *t, const double *xli,
                               const double *xni, const double *atime, int n, double *out, int *status, int device) {
    CatalogTables cat;
    const char *a1[1] = {l1}, *a2[1] = {l2};
    if (n < 0 || build_catalog(a1, a2, 1, grav, cat) != kOk || cat.nSdp4 != 1) return -1;
    const Sdp4Sat &e = cat.sdp4[0];
    const GravConsts g = grav_consts(cat.grav);
    if (!device) {
        for (int i = 0; i < n; ++i) {
            CellOut c;
            status[i] = sdp4_cell(e, t[i], xli[i], xni[i], atime[i], g, c);
            const double r[6] = {c.rx, c.ry, c.rz, c.vx, c.vy, c.vz};
            for (int j = 0; j < 6; ++j) out[6 * i + j] = r[j];
        }
        return 0;
    }
    if (n == 0) return 0;
    const size_t bytes = (size_t)n * sizeof(double);
    double *d[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
    int *dst = nullptr;
    const double *src[4] = {t, xli, xni, atime};
    cudaError_t rc = cudaSuccess;
    for (int k = 0; k < 4 && rc == cudaSuccess; ++k) rc = cudaMalloc(&d[k], bytes);
    if (rc == cudaSuccess) rc = cudaMalloc(&d[4], 6 * bytes);
    if (rc == cudaSuccess) rc = cudaMalloc(&dst, (size_t)n * sizeof(int));
    for (int k = 0; k < 4 && rc == cudaSuccess; ++k) rc = cudaMemcpy(d[k], src[k], bytes, cudaMemcpyHostToDevice);
    if (rc == cudaSuccess) {
        sdp4_cell_kernel<<<(n + 127) / 128, 128>>>(e, g, d[0], d[1], d[2], d[3], n, d[4], dst);
        rc = cudaGetLastError();
    }
    if (rc == cudaSuccess) rc = cudaMemcpy(out, d[4], 6 * bytes, cudaMemcpyDeviceToHost);
    if (rc == cudaSuccess) rc = cudaMemcpy(status, dst, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost);
    for (int k = 0; k < 5; ++k)
        if (d[k]) cudaFree(d[k]);
    if (dst) cudaFree(dst);
    return (int)rc;
}
