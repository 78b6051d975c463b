// TEST INFRASTRUCTURE ONLY: the deep-space cell (sdp4_cell_n, az_device.cuh) on the CPU with the product's host tables.
// emul_deep_regimes restates the cell's arithmetic for one lane and reports, per (satellite, epoch), the quantities that
// choose each of its branches, so a fixture can prove which branch it reaches; emul_deep_cell runs the product's own
// sdp4_cell from a caller-supplied resonance state (xli, xni, atime), which reaches branches no element set does.
// Not part of the shipped library; nothing in astroz_b200/ references it.
#include <cmath>
#include <cstdint>
#include <limits>

#include "az_tables.hpp"

using namespace az;

// Columns of one emul_deep_regimes row.
enum DeepRegime : int {
    kRegX,        // resonance libration x = (nm - no) / no (0 when irez == 0): the binomial series holds |x| <= 3e-3
    kRegDincl,    // inclm - inclo after dpper: a small rotation of sin/cos(inclo) while |dincl| <= 0.05 (kHiTiny)
    kRegInclm,    // inclm after dpper (before the sign flip): Lyddane below 0.2, flipped below 0
    kRegOpc,      // 1 + cos(inclm) = 2 cos^2(inclm / 2), without cancellation: xlcof's guard is 1.5e-12
    kRegNodDiff,  // Lyddane: nod - atan2(alfdp, betdp), wrapped by 2 pi when above pi in magnitude (NaN otherwise)
    kRegR2,       // Lyddane: alfdp^2 + betdp^2, atan2(0, 0) at or below 1e-280 (NaN otherwise)
    kRegEmPre,    // em after drag, before the floor and dpper: status 2 at >= 1 or < -0.001
    kRegEmPost,   // em after dpper, before the floor: status 2 at >= 1
    kRegAm,       // am: status 1 below 0.95
    kRegNm,       // nm (no when irez == 0): status 1 at <= 0
    kRegKep1,     // the general Kepler loop's first step before the +-0.95 clamp
    kRegStatus,   // the status sdp4_cell sets (-1 for near-earth rows)
    kRegMrt,      // the radius sdp4_cell reaches, in earth radii: status 1 below 1
    kNumDeepRegimes
};

static bool load_deep(const char *l1, const char *l2, int grav, Sdp4Sat &e, GravConsts &g) {
    CatalogTables cat;
    const char *a1[1] = {l1}, *a2[1] = {l2};
    if (build_catalog(a1, a2, 1, grav, cat) != kOk || cat.nSdp4 != 1) return false;
    e = cat.sdp4[0];
    g = grav_consts(cat.grav);
    return true;
}

// the kernel's lattice walk from node 0 to the node below |t|
static void walk(const Sdp4Sat &e, double t, double &xli, double &xni, double &atime) {
    xli = e.xlamo;
    xni = e.no;
    atime = 0.0;
    if (e.irez == 0) return;
    const int node = resonance_node(t);
    const double delt = t > 0.0 ? kStepp : -kStepp;
    for (int j = 0; j < node; ++j) resonance_step(e, xli, xni, atime, delt);
}

static void regimes_of(const Sdp4Sat &e, const GravConsts &g, double t, double *o) {
    const double nan = std::numeric_limits<double>::quiet_NaN();
    for (int i = 0; i < kNumDeepRegimes; ++i) o[i] = nan;
    double xli, xni, atime;
    walk(e, t, xli, xni, atime);

    const double t2 = t * t;
    const double tempa = fma(-e.cc1, t, 1.0), tempe = e.bc4 * t, templ = e.t2cof * t2;
    double mm = fma(e.dmdt, t, fma(e.mdot, t, e.mo));
    double argpm = fma(e.domdt, t, fma(e.argpdot, t, e.argpo));
    double nodem = fma(e.dnodt, t, fma(e.xnodcf, t2, fma(e.nodedot, t, e.nodeo)));
    double em = fma(e.dedt, t, e.ecco);
    double inclm = fma(e.didt, t, e.inclo);
    double am = e.abase * tempa * tempa;
    o[kRegX] = 0.0;
    o[kRegNm] = e.no;
    if (e.irez != 0) {
        double xndt, xnddt, xldot;
        resonance_accel(e, xli, xni, atime, xndt, xnddt, xldot);
        const double ft = t - atime, hft2 = 0.5 * ft * ft;
        const double nmr = fma(xnddt, hft2, fma(xndt, ft, xni));
        const double xl = fma(xndt, hft2, fma(xldot, ft, xli));
        const double theta = fma(t, kMathHost.rptim, e.gsto);
        mm = (e.irez == 2) ? xl - 2.0 * nodem + 2.0 * theta : xl - nodem - argpm + theta;
        const double nm = e.no + (nmr - e.no);
        o[kRegNm] = nm;
        o[kRegX] = (nmr - e.no) * e.invNo;
        am = std::pow(g.xke / (nm > 0.0 ? nm : e.no), 2.0 / 3.0) * tempa * tempa;
    }
    em -= tempe;
    o[kRegEmPre] = em;
    o[kRegAm] = am;
    em = std::fmax(em, 1.0e-6);
    mm = fma(e.no, templ, mm);

    // dpper with libm sines (selection quantities only)
    double zm = e.zmos + kMathHost.zns * t, zf = zm + kMathHost.zes2 * std::sin(zm);
    double sz = std::sin(zf), f2 = 0.5 * sz * sz - 0.25, f3 = -0.5 * sz * std::cos(zf);
    double pe = e.se2 * f2 + e.se3 * f3, pinc = e.si2 * f2 + e.si3 * f3;
    double pl = e.sl2 * f2 + e.sl3 * f3 + e.sl4 * sz, pgh = e.sgh2 * f2 + e.sgh3 * f3 + e.sgh4 * sz;
    double ph = e.sh2 * f2 + e.sh3 * f3;
    zm = e.zmol + kMathHost.znl * t;
    zf = zm + kMathHost.zel2 * std::sin(zm);
    sz = std::sin(zf);
    f2 = 0.5 * sz * sz - 0.25;
    f3 = -0.5 * sz * std::cos(zf);
    pe += e.ee2 * f2 + e.e3 * f3;
    pinc += e.xi2 * f2 + e.xi3 * f3;
    pl += e.xl2 * f2 + e.xl3 * f3 + e.xl4 * sz;
    pgh += e.xgh2 * f2 + e.xgh3 * f3 + e.xgh4 * sz;
    ph += e.xh2 * f2 + e.xh3 * f3;

    o[kRegDincl] = fma(e.didt, t, pinc);
    inclm += pinc;
    em += pe;
    o[kRegInclm] = inclm;
    o[kRegEmPost] = em;
    const double ch = std::cos(0.5 * inclm);
    o[kRegOpc] = 2.0 * ch * ch;
    const double sinip = std::sin(inclm), cosip = std::cos(inclm);
    if (inclm >= 0.2) {
        const double phs = ph / sinip;
        argpm += pgh - cosip * phs;
        nodem += phs;
        mm += pl;
    } else {
        const double nod = std::fmod(std::fmod(nodem, 2.0 * M_PI) + 2.0 * M_PI, 2.0 * M_PI);
        const double alfdp = sinip * std::sin(nod) + (ph * std::cos(nod) + pinc * cosip * std::sin(nod));
        const double betdp = sinip * std::cos(nod) + (-ph * std::sin(nod) + pinc * cosip * std::cos(nod));
        const double r2 = alfdp * alfdp + betdp * betdp;
        const double nn = r2 > 1.0e-280 ? std::atan2(alfdp, betdp) : 0.0;
        o[kRegNodDiff] = nod - nn;
        o[kRegR2] = r2;
        const double xls = mm + argpm + cosip * nod, dls = pl + pgh - pinc * nod * sinip;
        double nnw = nn;
        if (std::fabs(nod - nn) > M_PI) nnw += (nn < nod) ? 2.0 * M_PI : -2.0 * M_PI;
        nodem = nnw;
        mm += pl;
        argpm = xls + dls - mm - cosip * nnw;
    }
    double sini = sinip;
    if (inclm < 0.0) {
        sini = -sini;
        argpm -= M_PI;
    }
    em = std::fmax(em, 1.0e-6);
    if (em >= 1.0) em = 0.5;
    if (!(am >= 0.95)) am = 1.0;
    // kepler_posvel's prologue and the general loop's first step
    const double den = std::fmax(o[kRegOpc], 1.5e-12);
    const double xlcof = -0.25 * g.j3oj2 * sini * (3.0 + 5.0 * cosip) / den, aycof = -0.5 * g.j3oj2 * sini;
    const double temp = 1.0 / (am * (1.0 - em * em));
    const double axnl = em * std::cos(argpm), aynl = em * std::sin(argpm) + temp * aycof;
    const double u = mm + argpm + temp * xlcof * axnl;
    const double esine = axnl * std::sin(u) - aynl * std::cos(u), ecose = axnl * std::cos(u) + aynl * std::sin(u);
    o[kRegKep1] = esine / (1.0 - ecose);

    CellOut c;
    o[kRegStatus] = (double)sdp4_cell(e, t, xli, xni, atime, g, c);
    o[kRegMrt] = c.mrt;
}

// Rows [n][nt][kNumDeepRegimes] for element sets (l1, l2) at epochs jd + fr; near-earth rows are NaN with status -1.
extern "C" int emul_deep_regimes(const char *const *l1, const char *const *l2, uint32_t n, int grav, const double *jd,
                                 const double *fr, uint32_t nt, double *out) {
    for (uint32_t s = 0; s < n; ++s) {
        Sdp4Sat e;
        GravConsts g;
        const bool deep = load_deep(l1[s], l2[s], grav, e, g);
        for (uint32_t k = 0; k < nt; ++k) {
            double *o = out + ((size_t)s * nt + k) * kNumDeepRegimes;
            if (!deep) {
                for (int i = 0; i < kNumDeepRegimes; ++i) o[i] = std::numeric_limits<double>::quiet_NaN();
                o[kRegStatus] = -1.0;
                continue;
            }
            regimes_of(e, g, ((jd[k] + fr[k]) - e.epochJd) * 1440.0, o);
        }
    }
    return 0;
}

// The product's sdp4_cell for one deep-space element set at n (tsince, xli, xni, atime) cells.  pos / vel [n][3] (zero
// where the status is not 0), status [n].  Returns 0, or -1 when the element set is not a valid deep-space set.
extern "C" int emul_deep_cell(const char *l1, const char *l2, int grav, const double *t, const double *xli,
                              const double *xni, const double *atime, uint32_t n, double *pos, double *vel,
                              int32_t *status) {
    Sdp4Sat e;
    GravConsts g;
    if (!load_deep(l1, l2, grav, e, g)) return -1;
    for (uint32_t i = 0; i < n; ++i) {
        CellOut c;
        const int st = sdp4_cell(e, t[i], xli[i], xni[i], atime[i], g, c);
        const double r[6] = {c.rx, c.ry, c.rz, c.vx, c.vy, c.vz};
        for (int j = 0; j < 3; ++j) {
            pos[3 * i + j] = st ? 0.0 : r[j];
            vel[3 * i + j] = st ? 0.0 : r[3 + j];
        }
        status[i] = st;
    }
    return 0;
}
