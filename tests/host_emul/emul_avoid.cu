// TEST INFRASTRUCTURE ONLY: runs K16 (az_avoid.cuh, __host__ __device__) on the CPU.  emul_avoid is
// astroz_cuda_conjunction_maneuver_device's definition on host buffers: the four per-trial steps of az_avoid.cu in
// loops, composed with the host builds of K10 (emul_propagate_covariance, emul_covariance.cu, at the library's chunk),
// K8 (emul_fit_mixed, emul_fit.cu and emul_fit_deep.cu) and K11 (emul_conjunction, emul_conjunction.cu), all linked
// into the same library.  Not part of the shipped library; nothing in astroz_b200/ references it.
#include <cstdint>
#include <vector>

#include "az_avoid.cuh"

using namespace az;

extern "C" int emul_fit_mixed(const double *elements, uint32_t n, int grav, const uint32_t *offsets, const double *jd,
                              const double *fr, const double *pos, const double *vel, double posSigma, double velSigma,
                              int fitBstar, uint32_t maxIter, double *fitted, double *rms, uint32_t *iterations,
                              uint8_t *status);
extern "C" int emul_propagate_covariance(const double *elements, uint32_t n, int grav, const double *covariance,
                                         const uint8_t *model, const uint32_t *offsets, const double *jd,
                                         const double *fr, uint32_t m, int frame, uint32_t chunk, double *state,
                                         double *stateCov, double *jacobian, uint8_t *status);
extern "C" int emul_conjunction(const double *elements, uint32_t n, int grav, const double *covariance,
                                const uint8_t *model, const uint32_t *primary, const uint32_t *secondary,
                                const double *jd, const double *fr, const double *window, const double *hbr,
                                uint32_t m, int frame, double *record, double *states, double *stateCov,
                                uint8_t *status);

extern "C" uint64_t emul_avoid_scratch_bytes(uint32_t t) { return avoid_scratch_bytes(t); }

extern "C" int emul_avoid(const double *elements, uint32_t n, int grav, const double *covariance, const uint8_t *model,
                          const uint32_t *primary, const uint32_t *secondary, const double *jd, const double *fr,
                          const double *window, const double *hbr, uint32_t m, const uint32_t *candidate,
                          const double *burnJd, const double *burnFr, const double *dv, const double *dvSigma,
                          uint32_t t, double *record, double *newElements, double *newCovariance, double *residual,
                          uint8_t *status) {
    if (t == 0) return 0;
    std::vector<double> buf((avoid_scratch_bytes(t) + 7) / 8);
    AvoidArgs a;
    a.elements = elements;
    a.covariance = covariance;
    a.model = model;
    a.n = n;
    a.primary = primary;
    a.secondary = secondary;
    a.jd = jd;
    a.fr = fr;
    a.window = window;
    a.hbr = hbr;
    a.m = m;
    a.candidate = candidate;
    a.burnJd = burnJd;
    a.burnFr = burnFr;
    a.dv = dv;
    a.dvSigma = dvSigma;
    a.t = t;
    a.grav = grav;
    a.g = grav_consts(gravity(grav));
    a.scratch = buf.data();
    a.record = record;
    a.newElements = newElements;
    a.newCovariance = newCovariance;
    a.residual = residual;
    a.status = status;
    const AvoidScratch s = avoid_scratch(buf.data(), t);
    for (uint32_t k = 0; k < t; ++k) avoid_prepare(a, s, k);
    emul_propagate_covariance(s.el1, t, grav, s.P1, s.model1, s.offsets, burnJd, burnFr, t, kCovFrameTeme, cov_chunk(t),
                              s.state, s.sig, s.J, s.cov1St);
    for (uint32_t k = 0; k < t; ++k) avoid_burn(a, s, k);
    emul_fit_mixed(s.init, t, grav, s.offsets, burnJd, burnFr, s.pos, s.vel, kIodFitPosSigma, kIodFitVelSigma, 0,
                   kIodFitIter, s.fitted, s.rms, s.iters, s.fitSt);
    emul_propagate_covariance(s.fitted, t, grav, s.P1, s.model1, s.offsets, burnJd, burnFr, t, kCovFrameTeme,
                              cov_chunk(t), nullptr, s.sig, s.J2, s.cov2St);
    for (uint32_t k = 0; k < t; ++k) avoid_transport(a, s, k);
    emul_conjunction(s.el2, 2 * t, grav, s.P2, s.model2, s.pri2, s.sec2, s.jd2, s.fr2, s.win2, s.hbr2, t, kCovFrameTeme,
                     record, nullptr, nullptr, status);
    for (uint32_t k = 0; k < t; ++k) avoid_finish(a, s, k);
    return 0;
}

// The transport of one trial: J, J' (6 x 7 words), P (28), the pre-burn TEME state, sigma[3] (nullable), zero -> P'
extern "C" int emul_avoid_covariance(const double *J, const double *Jp, const double *P, const double *x,
                                     const double *sigma, int zero, double *Pn) {
    double xs[6];
    for (int c = 0; c < 6; ++c) xs[c] = x[c];
    return avoid_covariance(J, Jp, P, xs, sigma, zero != 0, Pn) ? 0 : -1;
}
