// TEST INFRASTRUCTURE ONLY: runs the per-query cores of the product's (satellite, time) pairs path (az_pairs.cuh,
// __host__ __device__) on the CPU with the product's own host tables, so the arithmetic of K6 can be checked against
// the oracle in a container without a GPU.  Not part of the shipped library; nothing in astroz_b200/ references it.
#include <cstdint>
#include <vector>

#include "az_pairs.cuh"
#include "az_tables.hpp"

using namespace az;

// The per-query device functions of the pairs path (az_pairs.cuh) for nq queries (sat[i], jd[i], fr[i]): gathered
// column access into the near-earth tiles, the tsince expression, GMST and the output epilogues.  The deep-space
// resonance state is read from a short lattice (`nodes` checkpoints per direction, built on the host the way K2a
// builds it), so queries beyond it exercise the step-on path.  tsince[i] receives the query's minutes since epoch,
// refJd[0] the catalog's reference epoch, epochOut[i] the satellite's epoch.
extern "C" int emul_pairs(const char *const *l1, const char *const *l2, uint32_t n, int grav, const uint32_t *sat,
                          const double *jd, const double *fr, uint32_t nq, int mode, int nodes, double *pos,
                          double *vel, uint8_t *status, double *tsince, double *refJd, double *epochOut) {
    CatalogTables cat;
    int rc = build_catalog(l1, l2, n, grav, cat);
    if (rc != kOk) return rc;
    const GravConsts g = grav_consts(cat.grav);
    std::vector<uint32_t> key(n);
    for (uint32_t i = 0; i < cat.nSgp4; ++i) key[cat.sgp4Orig[i]] = i;
    for (uint32_t d = 0; d < cat.nSdp4; ++d) key[cat.sdp4Orig[d]] = cat.nSgp4 + d;
    std::vector<double2> lattice((size_t)cat.nSdp4 * 2 * nodes);
    for (uint32_t i = 0; i < cat.nSdp4 * 2; ++i) {
        const Sdp4Sat &e = cat.sdp4[i >> 1];
        const double delt = (i & 1) ? -kStepp : kStepp;
        double2 *out = lattice.data() + (size_t)i * nodes;
        double xli = e.xlamo, xni = e.no, atime = 0.0;
        for (int k = 0; k < nodes; ++k) {
            if (k > 0 && e.irez != 0) resonance_step(e, xli, xni, atime, delt);
            out[k] = make_double2(xli, xni);
        }
    }
    refJd[0] = cat.referenceEpochJd;
    for (uint32_t q = 0; q < nq; ++q) {
        if (sat[q] >= n) return -20;
        const uint32_t k = key[sat[q]];
        const double jdFull = add_rn(jd[q], fr[q]);
        CellOut o{};
        uint8_t st;
        if (k < cat.nSgp4) {
            const double *base = cat.sgp4Tiles.data() + (size_t)(k / kTileSats) * kSgp4TileDoubles + (k % kTileSats);
            auto col = [base](int c) { return base[c * kTileSats]; };
            const double toff = (cat.referenceEpochJd - cat.sgp4Epoch[k]) * 1440.0;  // upload_toff
            tsince[q] = pairs_tsince_near(jdFull, cat.referenceEpochJd, toff);
            epochOut[q] = cat.sgp4Epoch[k];
            if (mode == 0) st = pairs_sgp4_query<0, true>(col, jdFull, cat.referenceEpochJd, toff, g, o);
            else if (mode == 1) st = pairs_sgp4_query<1, true>(col, jdFull, cat.referenceEpochJd, toff, g, o);
            else st = pairs_sgp4_query<2, true>(col, jdFull, cat.referenceEpochJd, toff, g, o);
        } else {
            const uint32_t d = k - cat.nSgp4;
            const Sdp4Sat &e = cat.sdp4[d];
            const double2 *lat = lattice.data() + (size_t)d * 2 * nodes;
            tsince[q] = pairs_tsince_deep(jdFull, e.epochJd);
            epochOut[q] = e.epochJd;
            if (mode == 0) st = pairs_sdp4_query<0, true>(e, lat, nodes, jdFull, g, o);
            else if (mode == 1) st = pairs_sdp4_query<1, true>(e, lat, nodes, jdFull, g, o);
            else st = pairs_sdp4_query<2, true>(e, lat, nodes, jdFull, g, o);
        }
        pos[3 * q] = o.rx; pos[3 * q + 1] = o.ry; pos[3 * q + 2] = o.rz;
        vel[3 * q] = o.vx; vel[3 * q + 1] = o.vy; vel[3 * q + 2] = o.vz;
        status[q] = st;
    }
    return 0;
}
