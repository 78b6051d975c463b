// TEST INFRASTRUCTURE ONLY: runs the model-list cores of K7 (az_numerical.cuh, __host__ __device__) on the CPU, so the
// arithmetic of every force model, Composite, per-state coefficients and position tables can be checked against the
// scalar restatement without a GPU.  Not part of the shipped library; nothing in astroz_b200/ references it.
#include <cstdint>
#include <cstring>

#define AZ_NUMERICAL_CORES_ONLY
#include "az_numerical.cuh"

using namespace az;

// n states over the K step sizes `steps` of a loop with step dt, under the list models[count] (astroz_force_model_t
// layout, host pointers): out[n][K + 1][6], status[n], counts[n][2].  Returns -1 when the steps do not fold into a
// StepTable or the list is empty or too long.
extern "C" int emul_numerical_models(const double *states, uint32_t n, const double *steps, uint32_t K, double dt,
                                     const ForceModel *models, uint32_t count, double rtol, double atol, int integrator,
                                     double *out, uint8_t *status, uint64_t *counts) {
    StepTable table{dt, 0, 0, {}};
    for (uint32_t k = 0; k < K; ++k)
        if (!step_table_push(table, steps[k])) return -1;
    if (count == 0 || count > kMaxModels) return -1;
    ModelList L{};
    L.count = count;
    std::memcpy(L.m, models, count * sizeof(ForceModel));
    const NumParams p{0.0, 0.0, 0.0, rtol, atol};
    for (uint32_t i = 0; i < n; ++i) {
        double *o = out + (size_t)i * (K + 1) * 6;
        status[i] = integrator == kIntRk4 ? propagate_state_models<kIntRk4>(states + 6 * i, L, i, p, table, o, counts + 2 * i)
                                          : propagate_state_models<kIntDp87>(states + 6 * i, L, i, p, table, o, counts + 2 * i);
    }
    return 0;
}

// The list's acceleration at s[n][6] for batch items items[n] during interval k: out[n][3]
extern "C" void emul_models_accel(const ForceModel *models, uint32_t count, const double *s, const uint64_t *items,
                                  uint32_t k, uint32_t n, double *out) {
    ModelList L{};
    L.count = count;
    std::memcpy(L.m, models, count * sizeof(ForceModel));
    for (uint32_t j = 0; j < n; ++j) {
        ListForces f{L, (uint32_t)items[j]};
        f.interval(k);
        f(s + 6 * j, out + 3 * j);
    }
}
