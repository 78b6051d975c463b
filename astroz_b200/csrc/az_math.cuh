// az_math.cuh -- fp64 device math for the SGP4/SDP4 grid kernels (sm_90a).
//
// Replaces src/simdMath.zig (sincosN :29-97, modTwoPiN :110-122, atan2N :124-177, pow15N :180-182,
// pow23N :201-212) of the reference.  Design differences, all deliberate:
//   * sincos: branch-free Cody-Waite (pi/2 = 21-bit head + 53-bit tail, FMA) + polynomial kernels fitted for this
//     pipe (immediate-encodable high-order coefficients, tools/fit_sincos_imm.py), < 2e-16 absolute;
//     no Payne-Hanek slow path (arguments here are bounded by |x| < ~1e5 rad: years of mean anomaly).
//   * atan2 is never needed on the SGP4 path: the true-longitude unit vector (sinu, cosu) is already
//     normalised, so the short-period rotation is applied with an angle-addition (see kernels).
//   * reciprocal / rsqrt: MUFU seed (rcp.approx.ftz.f64 / rsqrt.approx.ftz.f64) + Newton steps in
//     FMA form -- no special-case slow path, operands are O(1) by construction.
#pragma once

#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

// The per-cell cores are __host__ __device__ so tests/host_emul can run the *same arithmetic* on the
// CPU in unit tests when no GPU is present.  The shipped library exposes no host propagation path.
#define AZ_HD __host__ __device__ __forceinline__

namespace az {

AZ_HD int dbl_lo(double x) {
#ifdef __CUDA_ARCH__
    return __double2loint(x);
#else
    uint64_t b; memcpy(&b, &x, 8); return (int)(uint32_t)b;
#endif
}
AZ_HD double dbl_xor_hi(double x, unsigned mask) {  // flip bits of the high word (sign control)
#ifdef __CUDA_ARCH__
    return __hiloint2double(__double2hiint(x) ^ (int)mask, __double2loint(x));
#else
    uint64_t b; memcpy(&b, &x, 8); b ^= (uint64_t)mask << 32; memcpy(&x, &b, 8); return x;
#endif
}

AZ_HD uint32_t dbl_hi(double x) {
#ifdef __CUDA_ARCH__
    return (uint32_t)__double2hiint(x);
#else
    uint64_t b; memcpy(&b, &x, 8); return (uint32_t)(b >> 32);
#endif
}
AZ_HD double dbl_with_hi(double x, uint32_t hi) {
#ifdef __CUDA_ARCH__
    return __hiloint2double((int)hi, __double2loint(x));
#else
    uint64_t b; memcpy(&b, &x, 8); b = (b & 0xffffffffull) | ((uint64_t)hi << 32); memcpy(&x, &b, 8); return x;
#endif
}

// Rounded fp64 operations nvcc may not contract into an FMA, for expressions that must equal a host evaluation bit for
// bit (the host compiler does not contract).
AZ_HD double add_rn(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
AZ_HD double sub_rn(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dsub_rn(a, b);
#else
    return a - b;
#endif
}
AZ_HD double mul_rn(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}

// Magnitude tests that only steer control flow (which series to use, whether to iterate again) are done on the
// HIGH WORD of the double with integer instructions: a DSETP occupies the half-rate fp64 pipe like a DFMA does,
// the integer pipe has idle issue slots.  Ignoring
// the low word moves a threshold by at most 2^-20 relative, far inside the margin of every series it selects.
// NaN compares as larger than any limit, so a poisoned lane takes the general path.
constexpr uint32_t kHiTiny = 0x3fa99999u;     // 0.05
constexpr uint32_t kHiQuarter = 0x3fe8f5c2u;  // 0.78
constexpr uint32_t kHiClamp = 0x3fee6666u;    // 0.95
constexpr uint32_t kHiEmFloor = 0x3eb0c6f7u;  // 1e-6
constexpr uint32_t kHiMicro = 0x3f60624du;    // 2e-3
constexpr uint32_t kHiLinear = 0x3e45798eu;   // 1e-8
AZ_HD uint32_t abs_hi(double x) { return dbl_hi(x) & 0x7fffffffu; }
AZ_HD bool abs_gt(double x, uint32_t hiLimit) { return abs_hi(x) > hiLimit; }
AZ_HD bool abs_lt(double x, uint32_t hiLimit) { return abs_hi(x) < hiLimit; }
// max(x, floor) for a positive floor given by (hiFloor, value): negative x has the sign bit set and compares low
AZ_HD double floor_at(double x, uint32_t hiFloor, double floorValue) {
    return ((int)dbl_hi(x) < (int)hiFloor) ? floorValue : x;
}
// x >= 1.0, exactly (1.0 has a zero low word): any double >= 1 has a high word >= 0x3ff00000 as a signed integer,
// any smaller or negative one does not; a NaN with the sign bit clear (the device's canonical NaN) compares as >= 1
// and is flagged by the callers, one with the sign bit set compares as negative
AZ_HD bool ge_one(double x) { return (int)dbl_hi(x) >= 0x3ff00000; }
// clamp to +-limit (limit given by its high word and value), sign preserved
AZ_HD double clamp_abs(double x, uint32_t hiLimit, double limit) {
    const uint32_t h = dbl_hi(x);
    return ((h & 0x7fffffffu) > hiLimit) ? dbl_xor_hi(limit, h & 0x80000000u) : x;
}
// x / 2 for a normal x well away from underflow (here: reciprocal square roots of O(1) quantities): one integer
// subtract on the exponent field instead of a DMUL
AZ_HD double half_of(double x) { return dbl_with_hi(x, dbl_hi(x) - 0x00100000u); }
// biased exponent field; |x| < 2^(expo(x) - 1022)
AZ_HD int expo(double x) { return (int)((dbl_hi(x) >> 20) & 0x7ffu); }

constexpr double kPi = 3.14159265358979323846264338327950288;
constexpr double kTwoPi = 6.28318530717958647692528676655900577;

// Every fp64 literal whose low 32 bits are non-zero lives in __constant__ memory: fp64 instructions take
// constant-bank operands (c[bank][offset]) for free, whereas an immediate costs two UMOV / IMAD.MOV issue
// slots each time it is materialised -- in the first build that was about a third of the instructions per cell,
// making the kernel issue-bound instead of fp64-pipe-bound.
// sin / cos kernels on |r| <= pi/4 (tools/fit_sincos_imm.py): sin r = r + r^3 (s1 + s2 z + ... + s6 z^5),
// cos r = 1 - z/2 + z^2 (c1 + ... + c5 z^4), z = r^2.  s6, s4 and c5 are fp64 numbers whose low 32 bits are zero --
// the instruction encodes such an operand as an immediate, so the Horner step that multiplies by it reads two register
// pairs instead of three (a DFMA with three fresh register-pair sources can hold the fp64 pipe longer; tools/fp64_probe.cu
// measures it) -- and the other coefficients were re-solved with those fixed.  Max error in exact arithmetic
// 3.4e-17 (sin), 8.4e-17 (cos): on this interval a sixth cosine coefficient buys nothing, so the cosine kernel is one
// FMA shorter than fdlibm's, whose unconstrained minimax set reads 6e-18 / 5e-19 before the ~1e-16 of rounding all carry.
#define AZ_S4 0x1.71de3p-19
#define AZ_S6 0x1.5d61ep-33
#define AZ_C5 0x1.1bc3fp-29
// pi/2 = kPio2A (21 significant bits: k * kPio2A is exact for |k| < 2^32) + kPio2B (the next 53 bits); the third part,
// 1.06e-23, is below 1e-17 for every |x| < 1e6
#define AZ_PIO2A 0x1.921fbp+0
#define AZ_PIO2B 0x1.5110b4611a626p-22

struct MathTable {
    double s1, s2, s3, s4, s5, s6;          // sine kernel
    double c1, c2, c3, c4, c5, c6;          // cosine kernel (c6 unused: five coefficients)
    double twoOverPi, pio2Hi, pio2Mid, pio2Lo;
    double ts3, ts5, ts7, tc4, tc6, tc8;    // truncated Taylor series for |x| <= 0.05
    double quarterLimit, tinyLimit, clamp, emFloor, keplerTol, invTwoPi, twoPi, pi, microLimit, linearLimit;
    // deep-space constants (src/Sdp4.zig:15-52): solar / lunar mean motions, twice their eccentricities, the earth's
    // rotation rate per minute, and the two leading binomial coefficients of (1 + x)^(-2/3)
    double zns, znl, zes2, zel2, rptim, bin1, bin2;
    double stepInv, stepMid;                // 1024 / (2 pi) and the second word of 2 pi / 1024 (sincos_full)
};
#define AZ_MATH_TABLE_INIT                                                                                    \
    {                                                                                                         \
        -0x1.5555555555480p-3, 0x1.11111111053aep-7, -0x1.a01a019093f40p-13,                                  \
            AZ_S4, -0x1.ae5c4d5ed16f4p-26, AZ_S6,                                                             \
            0x1.5555555552f61p-5, -0x1.6c16c167479e5p-10, 0x1.a019fa88a4117p-16,                              \
            -0x1.27e01d2809545p-22, AZ_C5, 0.0,                                                               \
            6.36619772367581382433e-01, AZ_PIO2A, AZ_PIO2B,                                                  \
            -1.49738490485916983692e-33, -1.0 / 6.0, 1.0 / 120.0, -1.0 / 5040.0, 1.0 / 24.0, -1.0 / 720.0,    \
            1.0 / 40320.0, 0.78, 0.05, 0.95, 1.0e-6, 2.0e-15, 1.0 / 6.28318530717958647692528676655900577,    \
            6.28318530717958647692528676655900577, 3.14159265358979323846264338327950288, 2.0e-3, 1.0e-8,     \
            1.19459e-5, 1.5835218e-4, 2.0 * 0.01675, 2.0 * 0.05490, 4.37526908801129966e-3, -2.0 / 3.0, 5.0 / 9.0, \
            256.0 * 6.36619772367581382433e-01, AZ_PIO2B / 256.0                                            \
    }
static __constant__ MathTable kMathDev = AZ_MATH_TABLE_INIT;
static const MathTable kMathHost = AZ_MATH_TABLE_INIT;
#ifdef __CUDA_ARCH__
#define AZK(name) (::az::kMathDev.name)
#else
#define AZK(name) (::az::kMathHost.name)
#endif

// ---- reciprocal -------------------------------------------------------------------------------
AZ_HD double rcp_seed(double x) {
#ifdef __CUDA_ARCH__
    double y;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));  // 1e-6 relative (2^-20.0 measured on an H100)
    return y;
#else
    return (double)(1.0f / (float)x);  // ~2^-23
#endif
}
// the seed's error squared, from below: 1e-12 relative on the device, 2^-46 with the host's fp32 seed.  Enough for
// Newton correction steps (the fixed point does not depend on it) and for factors of J3- and e-sized terms
AZ_HD double rcp_fast(double x) {
    double y = rcp_seed(x);
    double e = fma(-x, y, 1.0);
    return fma(y, e, y);
}
// full precision (<= 1 ulp)
AZ_HD double rcp(double x) {
    double y = rcp_seed(x);
    double e = fma(-x, y, 1.0);
    y = fma(y, e, y);
    e = fma(-x, y, 1.0);
    return fma(y, e, y);
}
// a / b with one residual correction (<= 1 ulp for well-scaled operands)
AZ_HD double div_nr(double a, double b) {
    double y = rcp(b);
    double q = a * y;
    double r = fma(-b, q, a);
    return fma(r, y, q);
}

// ---- rsqrt / sqrt -----------------------------------------------------------------------------
AZ_HD double rsqrt_seed(double x) {
#ifdef __CUDA_ARCH__
    double y;
    asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));  // 1e-6 relative (2^-20.1 measured on an H100)
    return y;
#else
    return (double)(1.0f / sqrtf((float)x));
#endif
}
// 1/sqrt(x), <= 1 ulp
AZ_HD double rsqrt_nr(double x) {
    double y = rsqrt_seed(x);
    double r = fma(-x * y, y, 1.0);  // 1 - x y^2
    y = fma(half_of(y), r, y);
    r = fma(-x * y, y, 1.0);
    y = fma(half_of(y), r, y);
    return y;
}
// 1/sqrt(x) to 1.5e-12 on the device, 1.5 * 2^-46 on the host (one Newton step leaves 3/2 the square of the seed's
// error, from below): enough wherever a Heron correction (sqrt_from_rsqrt squares the error), a
// scale-invariant angle extraction, or a later iteration of the caller's own fixed point follows
AZ_HD double rsqrt_nr1(double x) {
    double y = rsqrt_seed(x);
    const double r = fma(-x * y, y, 1.0);
    return fma(half_of(y), r, y);
}
// sqrt(x) from y ~ 1/sqrt(x): one Heron correction
AZ_HD double sqrt_from_rsqrt(double x, double y) {
    double s = x * y;
    double r = fma(-s, s, x);
    return fma(half_of(y), r, s);
}
AZ_HD double sqrt_(double x) { return sqrt_from_rsqrt(x, rsqrt_nr(x)); }

// ---- sin / cos --------------------------------------------------------------------------------
// kernels on |r| <= pi/4 in fdlibm's form (sin r = r + r^3 P(z), cos r = 1 - z/2 + z^2 Q(z)); coefficients above
AZ_HD double ksin(double r, double r2) {
    double p = fma(r2, AZ_S6, AZK(s5));  // s6, s4 (c5 below) are immediates; s5 / c4 ride in a register as the addend
    p = fma(p, r2, AZ_S4);
    p = fma(p, r2, AZK(s3));
    p = fma(p, r2, AZK(s2));
    p = fma(p, r2, AZK(s1));
    return fma(p, r2 * r, r);
}
AZ_HD double kcos(double r2) {
    double p = fma(r2, AZ_C5, AZK(c4));
    p = fma(p, r2, AZK(c3));
    p = fma(p, r2, AZK(c2));
    p = fma(p, r2, AZK(c1));
    p = fma(p, r2, -0.5);
    return fma(p, r2, 1.0);
}

// sin and cos of x, |x| <~ 1e5.
#ifndef AZ_SINCOS_TABLE
#define AZ_SINCOS_TABLE 1
#endif
#if AZ_SINCOS_TABLE
// Reduction to the 1024-point lattice of the circle: x = k h + r, h = 2 pi / 1024, |r| <= h / 2 = 3.07e-3 (Cody-Waite
// with h = hi + mid, hi 21 bits so k hi is exact).  (sin, cos)(k h) come from a 16 KB table (az_sincos_table.inc,
// L1-resident, 40-digit values rounded once); on |r| <= 3.07e-3 sin r = r + r^3 (-1/6 + r^2 / 120) and
// cos r = 1 + r^2 (-1/2 + r^2 / 24) are exact to 5e-21 / 1.2e-18, and the angle addition finishes it: 14 fp64
// instructions and no quadrant logic, against 18 plus four selects for the pi/2 reduction with the |r| <= pi/4 kernels
// (which stay, for the arguments that need no reduction).  1/120 and 1/24 are 21-bit immediates: their rounding moves
// the result by 6e-22 and 9e-19.
struct SinCosPair { double s, c; };
static __device__ const SinCosPair __align__(16) kSinCosTabDev[1024] = {
#include "az_sincos_table.inc"
};
static const SinCosPair kSinCosTabHost[1024] = {  // the same entries for tests/host_emul
#include "az_sincos_table.inc"
};
#define AZ_STEP_A 0x1.921fbp-8  // AZ_PIO2A / 256
AZ_HD void sincos_full(double x, double &s, double &c) {
    constexpr double kMagic = 6755399441055744.0;  // 1.5 * 2^52: round-to-nearest-integer trick (imm32-encodable)
    double kf = fma(x, AZK(stepInv), kMagic);
    const unsigned q = (unsigned)dbl_lo(kf) & 1023u;
    kf -= kMagic;
    double r = fma(-kf, AZ_STEP_A, x);  // exact product (21-bit constant), one rounding
    r = fma(-kf, AZK(stepMid), r);
#ifdef __CUDA_ARCH__
    const SinCosPair t = kSinCosTabDev[q];
#else
    const SinCosPair t = kSinCosTabHost[q];
#endif
    const double r2 = r * r;
    const double sr = fma(r * r2, fma(r2, 0x1.11111p-7, AZK(ts3)), r);
    const double cr = fma(r2, fma(r2, 0x1.55555p-5, -0.5), 1.0);
    s = fma(t.s, cr, t.c * sr);
    c = fma(t.c, cr, -(t.s * sr));
}
#else
// Cody-Waite with pi/2 = hi + mid (FMA keeps k*hi exact enough).
AZ_HD void sincos_full(double x, double &s, double &c) {
    constexpr double kMagic = 6755399441055744.0;  // 1.5 * 2^52: round-to-nearest-integer trick (imm32-encodable)
    double kf = fma(x, AZK(twoOverPi), kMagic);
    const unsigned q = (unsigned)dbl_lo(kf);
    kf -= kMagic;
    double r = fma(-kf, AZ_PIO2A, x);  // exact product (21-bit constant), one rounding
    r = fma(-kf, AZK(pio2Mid), r);     // pio2Mid = AZ_PIO2B
    double r2 = r * r;
    double sr = ksin(r, r2);
    double cr = kcos(r2);
    double a = (q & 1) ? cr : sr;
    double b = (q & 1) ? sr : cr;
    // sign flips through the high word: sin negative in quadrants 2,3; cos negative in 1,2
    s = dbl_xor_hi(a, (q & 2u) << 30);
    c = dbl_xor_hi(b, ((q + 1u) & 2u) << 30);
}
#endif

// |x| <= pi/4: the kernels alone, no range reduction.  Used for the Kepler offset E-u (|.| <= e).
AZ_HD void sincos_quarter(double x, double &s, double &c) {
    double x2 = x * x;
    s = ksin(x, x2);
    c = kcos(x2);
}

// |x| <= 0.05: truncated Taylor series, abs error < 1e-17.  Used for the J2 short-period angles
// (|x| <= 1.5 * 0.5 * j2 / pl^2 ~ 8e-4 for any orbit above the surface).
AZ_HD void sincos_tiny(double x, double &s, double &c) {
    double x2 = x * x;
    double p = fma(x2, AZK(ts7), AZK(ts5));
    p = fma(x2, p, AZK(ts3));
    s = fma(x * x2, p, x);
    double q = fma(x2, AZK(tc8), AZK(tc6));
    q = fma(x2, q, AZK(tc4));
    q = fma(x2, q, -0.5);
    c = fma(x2, q, 1.0);
}

// |x| <= 2e-3 (the J2 short-period angles of any orbit above the surface are < 1e-3): abs error < 3e-16 (sin: 4e-8 |x|^3)
AZ_HD void sincos_micro(double x, double &s, double &c) {
    // -1/6 and 1/24 rounded to 21 significant bits (immediate operands): the rounding moves sin by |x|^3 * 4e-8 <= 3e-16
    // (the omitted x^5 / 120 has the other sign and cancels part of it) and cos by x^4 * 1e-8 <= 2e-19 on this range
    double x2 = x * x;
    s = fma(x * x2, -0x1.55555p-3, x);
    c = fma(x2, fma(x2, AZK(tc4), -0.5), 1.0);
}

// rotate the unit vector (s0, c0) = (sin a, cos a) by angle d given (sd, cd): returns sin/cos(a + d)
AZ_HD void rotate(double s0, double c0, double sd, double cd, double &s, double &c) {
    s = fma(s0, cd, c0 * sd);
    c = fma(c0, cd, -(s0 * sd));
}

// sin/cos(a + d) for an arbitrary d, picking the cheapest exact-enough evaluation of (sin d, cos d)
AZ_HD void rotate_small(double s0, double c0, double d, double &s, double &c) {
    double sd, cd;
    if (!abs_gt(d, kHiTiny)) sincos_tiny(d, sd, cd);
    else sincos_full(d, sd, cd);  // never taken for physical orbits; keeps the identity exact
    rotate(s0, c0, sd, cd, s, c);
}

// floored modulo 2*pi (Zig @mod semantics), result in [0, 2pi)
AZ_HD double mod_twopi(double x) {
    double n = floor(x * AZK(invTwoPi));
    double r = fma(-n, AZK(twoPi), x);
    r = (r < 0.0) ? r + AZK(twoPi) : r;
    return (r >= AZK(twoPi)) ? r - AZK(twoPi) : r;
}

// accurate atan2 for the SDP4 Lyddane branch only (rare): CUDA's own
AZ_HD double atan2_(double y, double x) { return atan2(y, x); }

}  // namespace az
