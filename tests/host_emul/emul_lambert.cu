// TEST INFRASTRUCTURE ONLY: runs the per-problem core of K9 (az_lambert.cuh, __host__ __device__) on the CPU, so the
// solver's arithmetic can be checked against the scalar C statement in a container without a GPU.  Not part of the
// shipped library; nothing in astroz_b200/ references it.
#include <cstdint>

#define AZ_LAMBERT_CORES_ONLY
#include "az_lambert.cuh"

using namespace az;

// n problems (normal nullable: +z): v1 / v2 [n][S][3], status / iters [n][S]
extern "C" void emul_lambert(const double *r1, const double *r2, const double *tof, const double *normal, uint32_t n,
                             double mu, uint32_t maxRevs, double *v1, double *v2, uint8_t *status, uint8_t *iters) {
    const size_t S = 2 * (size_t)maxRevs + 1;
    const double z[3] = {0.0, 0.0, 1.0};
    for (uint32_t i = 0; i < n; ++i)
        lambert_solve(r1 + 3 * i, r2 + 3 * i, tof[i], mu, normal ? normal + 3 * i : z, maxRevs,
                      [&](uint32_t s, uint8_t st, int it, const double a[3], const double b[3]) {
                          const size_t o = i * S + s;
                          for (int k = 0; k < 3; ++k) v1[3 * o + k] = a[k], v2[3 * o + k] = b[k];
                          status[o] = st;
                          iters[o] = (uint8_t)it;
                      });
}

// n porkchop cells: chaser (rc, vc), target (rt, vt) [n][3], tof [n]; dv [n][2], slot / status [n]
extern "C" void emul_porkchop(const double *rc, const double *vc, const double *rt, const double *vt, const double *tof,
                              uint32_t n, double mu, uint32_t maxRevs, double *dv, uint8_t *slot, uint8_t *status) {
    for (uint32_t i = 0; i < n; ++i)
        lambert_porkchop_cell(rc + 3 * i, vc + 3 * i, rt + 3 * i, vt + 3 * i, tof[i], mu, maxRevs, dv + 2 * i, slot[i],
                              status[i]);
}
