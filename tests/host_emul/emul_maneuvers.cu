// TEST INFRASTRUCTURE ONLY: runs the K7 maneuver core (maneuver_with in az_numerical.cuh, __host__ __device__) on the
// CPU, so the loop, the four burns and the samples can be checked against the scalar restatement
// (tests/numerical_oracle/maneuvers.c) without a GPU.  Not part of the shipped library.
#include <cstdint>
#include <cstring>

#define AZ_NUMERICAL_CORES_ONLY
#include "az_numerical.cuh"

using namespace az;

// n states, state i with impulses imp[offsets[i] .. offsets[i + 1]), under models[count] (astroz_force_model_t layout,
// host pointers): times[n][cap], out[n][cap][6], nSamples[n], status[n], counts[n][2].  -1 for an empty or too long
// list.
extern "C" int emul_maneuvers(const double *states, uint32_t n, double t0, double duration, double h, double mu,
                              const uint32_t *offsets, const Impulse *imp, const ForceModel *models, uint32_t count,
                              double rtol, double atol, int integrator, uint32_t cap, double *times, double *out,
                              uint64_t *nSamples, uint8_t *status, uint64_t *counts) {
    if (count == 0 || count > kMaxModels) return -1;
    ModelList L{};
    L.count = count;
    std::memcpy(L.m, models, count * sizeof(ForceModel));
    const NumParams p{mu, 0.0, 0.0, rtol, atol};
    for (uint32_t i = 0; i < n; ++i) {
        ManeuverRow row{times + (size_t)i * cap, out + (size_t)i * cap * 6, cap, 0};
        const Impulse *b = imp + offsets[i];
        const uint32_t m = offsets[i + 1] - offsets[i];
        status[i] = integrator == kIntRk4
                        ? maneuver_state_models<kIntRk4>(states + 6 * i, L, i, p, t0, t0 + duration, h, b, m, row,
                                                         counts + 2 * i)
                        : maneuver_state_models<kIntDp87>(states + 6 * i, L, i, p, t0, t0 + duration, h, b, m, row,
                                                          counts + 2 * i);
        nSamples[i] = row.count;
    }
    return 0;
}
