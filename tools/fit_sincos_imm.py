#!/usr/bin/env python
"""Design of the sin/cos kernels whose high-order coefficients are fp64 numbers with a zero low word (CPU tool).

A DFMA that reads three fresh 64-bit register pairs can occupy the fp64 pipe longer than one that reads two
(tools/fp64_probe.cu measures it), and ptxas keeps polynomial coefficients in registers, so a Horner step fma(p, z, c) with c in a
register is such an instruction.  An fp64 operand whose low 32 bits are zero is encoded in the instruction as an
immediate and costs no register read.  This script re-fits the |r| <= pi/4 kernels
    sin r = r + r^3 (s1 + s2 z + ... + s6 z^5),   cos r = 1 - z/2 + z^2 (c1 + c2 z + ... + c6 z^5),   z = r^2
with chosen coefficients constrained to 21 significant bits: they are rounded one at a time from the highest order
down, and after each rounding the remaining (full-precision) ones are re-solved by weighted least squares on Chebyshev
nodes, so they absorb most of the perturbation.  Prints the coefficient tables and the maximum error.
    python tools/fit_sincos_imm.py            (the shipped design)
    python tools/fit_sincos_imm.py 6 6        (other coefficient counts, immediates at the same Horner positions)
"""
import struct
import sys

import mpmath as mp

mp.mp.dps = 60
PIO4 = mp.pi / 4 * (1 + mp.mpf(2) ** -20)   # a little beyond pi/4: the Cody-Waite reduction lands within half a ulp of it


def imm(x):
    """nearest double whose low 32 bits are zero"""
    b = struct.unpack("<Q", struct.pack("<d", float(x)))[0]
    lo = b & 0xffffffff
    b -= lo
    if lo >= 0x80000000:
        b += 1 << 32
    return mp.mpf(struct.unpack("<d", struct.pack("<Q", b))[0])


def dbl(x):
    return mp.mpf(float(x))


def nodes(n):
    return [PIO4 * mp.cos(mp.pi * (2 * k + 1) / (2 * n)) for k in range(n)]


def fit(target, n_coef, imm_idx, weight):
    """coefficients c[0..n_coef) of sum c_k z^k ~ target(z); those whose index is in imm_idx are immediates.  They are
    rounded one at a time from the highest order down, the free ones re-solved after each rounding."""
    rs = [r for r in nodes(160) if r > 0]
    zs = [r * r for r in rs]
    fixed = {}
    order = sorted(imm_idx, reverse=True)
    for step in range(len(order) + 1):
        free = [k for k in range(n_coef) if k not in fixed]
        A = mp.matrix(len(zs), len(free))
        b = mp.matrix(len(zs), 1)
        for i, (r, z) in enumerate(zip(rs, zs)):
            w = weight(r)
            for j, k in enumerate(free):
                A[i, j] = w * z ** k
            b[i] = w * (target(r) - sum(fixed[k] * z ** k for k in fixed))
        sol = mp.lu_solve(A.T * A, A.T * b)
        coef = dict(fixed)
        for j, k in enumerate(free):
            coef[k] = sol[j]
        if step == len(order):
            break
        fixed[order[step]] = imm(coef[order[step]])
    out = [dbl(coef[k]) if k not in fixed else fixed[k] for k in range(n_coef)]
    return out, sorted(fixed)


def max_err(f, g, n=4001):
    worst = mp.mpf(0)
    for i in range(n):
        r = PIO4 * (mp.mpf(2 * i) / (n - 1) - 1)
        worst = max(worst, abs(f(r) - g(r)))
    return worst


def main():
    # shipped design: sin with six coefficients, s6 and s4 immediates (they are the multiplier-side constants of Horner
    # steps 1 and 2; s5 is the addend of step 1 and sits in a register anyway); cos with FIVE coefficients, c5 immediate
    # -- on |r| <= pi/4 the sixth cosine coefficient buys nothing at this accuracy, so the kernel is one FMA shorter
    n_s, imm_s = 6, [5, 3]
    n_c, imm_c = 5, [4]
    if len(sys.argv) > 2:
        n_s, n_c = int(sys.argv[1]), int(sys.argv[2])
        imm_s, imm_c = [n_s - 1, n_s - 3], [n_c - 1]
    s, s_imm = fit(lambda r: (mp.sin(r) - r) / r ** 3, n_s, imm_s, lambda r: r ** 3)
    c, c_imm = fit(lambda r: (mp.cos(r) - 1 + r * r / 2) / r ** 4, n_c, imm_c, lambda r: r ** 4)

    def psin(r):
        z = r * r
        p = s[-1]
        for k in range(n_s - 2, -1, -1):
            p = p * z + s[k]
        return r + r ** 3 * p

    def pcos(r):
        z = r * r
        p = c[-1]
        for k in range(n_c - 2, -1, -1):
            p = p * z + c[k]
        return 1 - z / 2 + z * z * p

    print("sin: immediates at orders", [k + 1 for k in s_imm], " max |err| (exact arithmetic) =", mp.nstr(max_err(mp.sin, psin), 4))
    for k, v in enumerate(s):
        print(f"  s{k + 1} = {float(v)!r}   {float(v).hex()}")
    print("cos: immediates at orders", [k + 1 for k in c_imm], " max |err| (exact arithmetic) =", mp.nstr(max_err(mp.cos, pcos), 4))
    for k, v in enumerate(c):
        print(f"  c{k + 1} = {float(v)!r}   {float(v).hex()}")


if __name__ == "__main__":
    main()
