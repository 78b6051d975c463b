// TEST INFRASTRUCTURE ONLY: runs the per-state cores of K7 (az_numerical.cuh, __host__ __device__) on the CPU, so the
// arithmetic of the numerical propagation path can be checked against the scalar restatement in a container without a
// GPU.  Not part of the shipped library; nothing in astroz_b200/ references it.
#include <cstdint>

#define AZ_NUMERICAL_CORES_ONLY
#include "az_numerical.cuh"

using namespace az;

// The product's tableau as the host build holds it (the device copy is initialised from the same macro), and the
// compile-time zero pattern the unrolled stage loops rely on: nz[i][j] for a (j < 12), nz[i][12] for b8, nz[i][13] b7.
extern "C" void emul_numerical_tableau(double *c, double *a, double *b8, double *b7, uint8_t *nz) {
    for (int i = 0; i < 13; ++i) {
        c[i] = kDp87Host.c[i];
        b8[i] = kDp87Host.b8[i];
        b7[i] = kDp87Host.b7[i];
        for (int j = 0; j < 12; ++j) {
            a[i * 12 + j] = kDp87Host.a[i][j];
            nz[i * 14 + j] = dp87_a_nz(i, j);
        }
        nz[i * 14 + 12] = dp87_b8_nz(i);
        nz[i * 14 + 13] = dp87_b7_nz(i);
    }
}

template <int kInt>
static uint8_t one(int forces, const double *y0, const DragBody &d, const NumParams &p, const StepTable &steps,
                   double *out, uint64_t *counts) {
    switch (forces) {
        case 0: return propagate_state<kInt, 0>(y0, d, p, steps, out, counts);
        case 1: return propagate_state<kInt, 1>(y0, d, p, steps, out, counts);
        case 2: return propagate_state<kInt, 2>(y0, d, p, steps, out, counts);
        default: return propagate_state<kInt, 3>(y0, d, p, steps, out, counts);
    }
}

// n states over the K step sizes `steps` of a loop with step dt: par = {mu, j2, r_eq, rtol, atol}; cd / area / mass per
// state (drag); out[n][K + 1][6], status[n], counts[n][2].  Returns -1 when the steps do not fold into a StepTable.
extern "C" int emul_numerical(const double *states, uint32_t n, const double *steps, uint32_t K, double dt,
                              const double *par, int forces, const double *cd, const double *area, const double *mass,
                              int integrator, double *out, uint8_t *status, uint64_t *counts) {
    StepTable table{dt, 0, 0, {}};
    for (uint32_t k = 0; k < K; ++k)
        if (!step_table_push(table, steps[k])) return -1;
    const NumParams p{par[0], par[1], par[2], par[3], par[4]};
    for (uint32_t i = 0; i < n; ++i) {
        DragBody d{0.0, 0.0, 0.0};
        if (forces & kForceDrag) d = DragBody{cd[i], area[i], mass[i]};
        double *o = out + (size_t)i * (K + 1) * 6;
        status[i] = integrator == kIntRk4 ? one<kIntRk4>(forces, states + 6 * i, d, p, table, o, counts + 2 * i)
                                          : one<kIntDp87>(forces, states + 6 * i, d, p, table, o, counts + 2 * i);
    }
    return 0;
}
