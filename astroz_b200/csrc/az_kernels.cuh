// az_kernels.cuh -- launch interface of the grid kernels (internal to the library).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "az_device.cuh"

namespace az {

// Arguments of one (n_sats x n_times) grid launch.  All pointers are device pointers.
struct GridArgs {
    // near-earth table (K1) or deep-space records (K2)
    const double *sgp4Tiles = nullptr;   // [tiles][kSgp4Cols][8]
    const Sdp4Sat *sdp4 = nullptr;       // [nSats]
    const double2 *lattice = nullptr;    // K2: [nSats][2][latticeNodes] (xli, xni) at atime = +-720*k
    int latticeNodes = 0;
    const uint32_t *orig = nullptr;      // output row of each table satellite (padded for K1)
    const uint8_t *mask = nullptr;       // nullable: per output row, 0 = leave that satellite's rows untouched
    uint32_t nSats = 0;                  // real satellites in the table
    // time axis
    const double *tbase = nullptr;       // K1: minutes of each epoch relative to the reference epoch
    const double *toff = nullptr;        // K1: per-satellite (reference - epoch) * 1440, padded
    const double *jdFull = nullptr;      // K2: jd + fr per epoch
    const double *tsince = nullptr;      // K2: if set, minutes since epoch are taken from here instead
    const double *jdArr = nullptr;       // K1t: if set, tsince = ((jd[t] + fr[t]) - epochJd) * 1440 on the device
    const double *frArr = nullptr;
    double epochJd = 0.0;
    const double *gsin = nullptr;        // sin/cos(GMST) per epoch when mode != TEME
    const double *gcos = nullptr;
    uint32_t nTimes = 0;
    uint32_t stripe = 0;                 // K1: epochs per CTA, chosen at launch from the CTA count (0 = the shape's default)
    // outputs
    double *pos = nullptr;
    double *vel = nullptr;               // nullable
    uint8_t *status = nullptr;           // nullable, [outRow][nTimes]
    uint32_t outNumSats = 0;             // row count of the output block (time-major stride)
    uint32_t recStride = 3;              // K1t only: doubles between consecutive epochs (6 = x y z vx vy vz records)
    // fused all-gather (satellite-major only): when gather != 0 the result block is written to every GPU
    // of the box from inside the kernel -- gather 1: one multimem.st per 16 bytes to the NVLS multicast
    // mapping of the symmetric buffer (mcPos/mcVel); gather 2: plain stores to each peer mapping.
    int gather = 0;
    int nPeers = 0;
    double *mcPos = nullptr;
    double *mcVel = nullptr;
    double *peerPos[8] = {};
    double *peerVel[8] = {};
    GravConsts g{};
};

constexpr int kMaxPeers = 8;

// K1: near-earth grid.  variant selects a tuning configuration (0 = default).
cudaError_t launch_sgp4_grid(const GridArgs &a, int mode, int layout, cudaStream_t stream, int variant);
// K2a: resonance lattice pre-pass (one thread per deep-space satellite, sequential 720-min steps).
cudaError_t launch_sdp4_lattice(const Sdp4Sat *sats, uint32_t nSats, double2 *lattice, int nodes, cudaStream_t stream);
// K2: deep-space grid.
cudaError_t launch_sdp4_grid(const GridArgs &a, int mode, int layout, cudaStream_t stream);
// K3: fused propagate + single-target conjunction screen (src/Constellation.zig:683-756).  No position block
// is written: per satellite the minimum distance to the target over all epochs (and its epoch index).
struct ScreenArgs {
    const double *sgp4Tiles = nullptr;
    const double *toff = nullptr;     // per-satellite epoch offsets (padded)
    const double *tbase = nullptr;    // times[n_times]
    uint32_t nSats = 0, nTimes = 0;
    uint32_t targetIdx = 0;
    double thresholdSq = 0.0;
    double *track = nullptr;          // scratch [n_times][3]: target positions
    double *minDist = nullptr;        // out [nSats]
    uint32_t *minT = nullptr;         // out [nSats]
    GravConsts g{};
};
cudaError_t launch_sgp4_screen(const ScreenArgs &a, cudaStream_t stream);

// K4: all-vs-all coarse conjunction screen over a device-resident position block
// (bindings/python/src/conjunction.zig:11-149): per epoch a cell list (cell edge = threshold) in a hash table,
// then each satellite checks its own and 13 forward neighbour cells.
struct CoarseArgs {
    const double *pos = nullptr;       // [nSats][nTimes][3] (layout 0) or [nTimes][nSats][3] (layout 1)
    const uint8_t *validMask = nullptr;  // nullable, per satellite
    uint32_t nSats = 0, nTimes = 0;
    int layout = 1;
    double threshold = 0.0;
    uint32_t t0 = 0, tCount = 0;       // epoch batch handled by this launch pair
    uint32_t tableBits = 16;
    uint32_t *head = nullptr;          // [tCount][1 << tableBits]
    uint32_t *next = nullptr;          // [tCount][nSats]
    uint32_t *pairs = nullptr;         // [maxResults][2]
    uint32_t *tIdx = nullptr;          // [maxResults]
    uint32_t maxResults = 0;
    unsigned long long *count = nullptr;  // device counter (total hits, may exceed maxResults)
};
cudaError_t launch_coarse_screen(const CoarseArgs &a, cudaStream_t stream);

// fp32 study kernel (BASELINE config 5): same grid / layout as K1 (satellite-major TEME, fp64 output words),
// arithmetic in fp32; phase64 != 0 forms the secular angles in fp64 first.
cudaError_t launch_sgp4_grid_f32(const GridArgs &a, int phase64, cudaStream_t stream);

// K6: n (satellite, time) queries in one call (az_pairs.cu).  All pointers are device pointers.
struct PairsArgs {
    // the handle's tables
    const double *sgp4Tiles = nullptr;   // [tiles][kSgp4Cols][8]
    const double *toff = nullptr;        // per near-earth table index: (referenceEpochJd - epoch) * 1440
    const Sdp4Sat *sdp4 = nullptr;
    const double2 *lattice = nullptr;    // [nSdp4][2][latticeNodes]
    int latticeNodes = 0;
    const uint32_t *rowKey = nullptr;    // per catalog row: near-earth table index, or nSgp4 + deep-space index
    uint32_t nRows = 0, nSgp4 = 0;
    double refJd = 0.0;
    // queries
    const uint32_t *sat = nullptr;
    const double *jd = nullptr, *fr = nullptr;
    uint32_t n = 0;
    // scratch: keys / indices before and after the sort, the segment bounds, the sort's temporary storage
    uint32_t *keys = nullptr, *idx = nullptr, *keysSorted = nullptr, *idxSorted = nullptr, *split = nullptr;
    void *sortScratch = nullptr;
    size_t sortScratchBytes = 0;
    // outputs, indexed by query
    double *pos = nullptr;
    double *vel = nullptr;               // nullable
    uint8_t *status = nullptr;           // nullable
    GravConsts g{};
};
cudaError_t launch_pairs(const PairsArgs &a, int mode, cudaStream_t stream);
// temporary storage the sort of n queries over nRows catalog rows needs
cudaError_t pairs_sort_scratch_bytes(uint32_t n, uint32_t nRows, size_t *bytes);
// min / max of jd + fr over n queries into scratch[0..1] (scratch: pairs_range_scratch_doubles() doubles)
cudaError_t launch_pairs_range(const double *jd, const double *fr, uint32_t n, double *scratch, cudaStream_t stream);
size_t pairs_range_scratch_doubles();

// K8: fit SGP4 mean elements to TEME ephemerides, one warp per satellite (az_fit.cu, az_fit.cuh).  All pointers are
// device pointers.
struct FitArgs {
    const double *elements = nullptr;    // [8][n] initial columns: epoch JD, n rev/day, e, i, node, w, M deg, B*
    uint32_t n = 0;
    const uint32_t *offsets = nullptr;   // [n + 1]: satellite s owns observations [offsets[s], offsets[s + 1])
    const double *jd = nullptr, *fr = nullptr;
    const double *pos = nullptr;         // [m][3] TEME km
    const double *vel = nullptr;         // [m][3] TEME km/s, nullable
    double wp = 1.0, wv = 1.0;           // 1 / pos_sigma, 1 / vel_sigma
    int fitBstar = 1;
    uint32_t maxIter = 25;
    int grav = 1;                        // ASTROZ_WGS72 / ASTROZ_WGS84
    GravConsts g{};
    double *fitted = nullptr;            // [8][n]
    double *rms = nullptr;               // [n][2]: position km, velocity km/s
    uint32_t *iterations = nullptr;      // [n]
    uint8_t *status = nullptr;           // [n] ASTROZ_FIT_*
};
cudaError_t launch_fit(const FitArgs &a, cudaStream_t stream);
// The deep-space sets of the batch only (initial period > 225 min), under the deep-space model: every other row is left
// as it is, so queued after launch_fit on the same arguments it completes a mixed batch.
cudaError_t launch_fit_deep(const FitArgs &a, cudaStream_t stream);

// K8 from sensor observations (az_fit_obs.cu, az_obs.cuh): TEME or ECEF states, radar, optical angles.  Device pointers.
struct FitObsArgs {
    const double *elements = nullptr;    // [8][n]
    uint32_t n = 0;
    const uint32_t *offsets = nullptr;   // [n + 1]
    const double *jd = nullptr, *fr = nullptr;
    const double *value = nullptr;       // [m][6]
    const double *sigma = nullptr;       // [m][6]: +inf = component not used
    const uint32_t *station = nullptr;   // [m]: row of stations (radar and optical kinds)
    const uint8_t *kind = nullptr;       // [m] ASTROZ_OBS_*
    const double *stations = nullptr;    // [k][3]: geodetic lat deg, lon deg, height km (WGS84)
    int fitBstar = 1;
    uint32_t maxIter = 25;
    int grav = 1;
    GravConsts g{};
    double *fitted = nullptr;            // [8][n]
    double *wrms = nullptr;              // [n]: sqrt(cost / used residuals)
    uint32_t *nResiduals = nullptr;      // [n]
    double *covariance = nullptr;        // [n][28]: upper triangle of the fitted variables' covariance
    uint32_t *iterations = nullptr;      // [n]
    uint8_t *status = nullptr;           // [n]
    uint8_t *model = nullptr;            // [n]: 0 near-earth variables, 1 deep-space (equinoctial) variables
};
cudaError_t launch_fit_obs(const FitObsArgs &a, cudaStream_t stream);
// the deep-space rows only, under the deep-space model (as launch_fit_deep)
cudaError_t launch_fit_obs_deep(const FitObsArgs &a, cudaStream_t stream);
// h(kind, state) of m observations, one thread each: states[m][6] TEME -> values[m][6] (zero past the kind's count)
cudaError_t launch_observe(const double *states, const double *jd, const double *fr, const uint8_t *kind,
                           const uint32_t *station, const double *stations, uint32_t m, double *values,
                           cudaStream_t stream);

// K10: fitted covariances carried to state covariances at query times (az_covariance.cu, az_covariance.cuh).  Device
// pointers.
struct CovArgs {
    const double *elements = nullptr;    // [8][n]
    const double *covariance = nullptr;  // [n][28]: upper triangle of P in the fit's variables
    const uint8_t *model = nullptr;      // [n], nullable (all 0): 0 near-earth variables, 1 deep-space variables
    uint32_t n = 0;
    const uint32_t *offsets = nullptr;   // [n + 1]: satellite s owns queries [offsets[s], offsets[s + 1])
    const double *jd = nullptr, *fr = nullptr;
    uint32_t m = 0;
    uint32_t chunk = 0;                  // queries per work item: launch_covariance sets cov_chunk(m)
    int frame = 0;                       // ASTROZ_COV_FRAME_*
    int grav = 1;
    GravConsts g{};
    double *state = nullptr;             // [m][6] TEME, nullable
    double *sigma = nullptr;             // [m][21]
    double *jacobian = nullptr;          // [m][6][7], nullable
    uint8_t *status = nullptr;           // [m] ASTROZ_COV_*
};
// the near-earth rows' queries (model 0), then on the same stream the deep-space rows' (model 1)
cudaError_t launch_covariance(const CovArgs &a, cudaStream_t stream);

// K11: candidate conjunctions assessed at their TCA (az_conjunction.cu, az_conjunction.cuh).  Device pointers.
struct ConjArgs {
    const double *elements = nullptr;    // [8][n]
    const double *covariance = nullptr;  // [n][28]: upper triangle of P in the fit's variables
    const uint8_t *model = nullptr;      // [n], nullable (all 0)
    uint32_t n = 0;
    const uint32_t *primary = nullptr, *secondary = nullptr;  // [m] rows
    const double *jd = nullptr, *fr = nullptr;                 // [m] guess times
    const double *window = nullptr;      // [m] half window [min]
    const double *hbr = nullptr;         // [m] combined hard-body radius [km]
    uint32_t m = 0;
    int frame = 0;                       // ASTROZ_COV_FRAME_* of the per-object Sigma
    int grav = 1;
    GravConsts g{};
    double *record = nullptr;            // [m][13]
    double *states = nullptr;            // [m][2][6] TEME at the TCA, nullable
    double *sigma = nullptr;             // [m][2][21], nullable
    uint8_t *status = nullptr;           // [m] ASTROZ_CONJ_*
};
// the pairs of two near-earth rows, then on the same stream every other pair
cudaError_t launch_conjunction(const ConjArgs &a, cudaStream_t stream);

// K14: Monte Carlo collision probability of candidate conjunctions (az_conjunction_mc.cu, az_conjunction_mc.cuh).
// Device pointers.
struct ConjMcArgs {
    const double *elements = nullptr;    // [8][n]
    const double *covariance = nullptr;  // [n][28]
    const uint8_t *model = nullptr;      // [n], nullable (all 0)
    uint32_t n = 0;
    const uint32_t *primary = nullptr, *secondary = nullptr;  // [m] rows
    const double *jd = nullptr, *fr = nullptr;                 // [m] guess times
    const double *window = nullptr;      // [m] half window [min]
    const double *hbr = nullptr;         // [m] combined hard-body radius [km]
    const uint64_t *samples = nullptr;   // [m]
    const uint64_t *first = nullptr;     // [m], nullable (all 0)
    const uint64_t *seed = nullptr;      // [m], nullable (all 0)
    uint32_t m = 0;
    uint32_t record = 0;                 // sample words kept per candidate
    int grav = 1;
    GravConsts g{};
    void *scratch = nullptr;             // conj_mc_scratch_bytes(m)
    uint64_t *counts = nullptr;          // [m][3] hits, edge, failed
    double *sampleOut = nullptr;         // [m][record][2] dt_tca, miss; nullable when record = 0
    uint8_t *status = nullptr;           // [m] ASTROZ_CONJ_*
};
cudaError_t conj_mc_scratch_bytes(uint32_t m, size_t *bytes);
// the candidates' statuses and work items, their scan, the near-earth pairs' items, then every other pair's
cudaError_t launch_conjunction_mc(const ConjMcArgs &a, cudaStream_t stream);

// K15: importance-sampled collision probability (az_conjunction_is.cu, az_conjunction_is.cuh).  Device pointers.  The
// inherited fields are K14's, except counts [m][12] (hits, edge, failed, overflow, V_hit[4], V2_hit[4]), sampleOut
// [m][record][3] (dt_tca, miss, log w) and scratch (conj_is_scratch_bytes(m)).
struct ConjIsArgs : ConjMcArgs {
    const double *shift = nullptr;       // [m][14] given shifts, nullable: the linear shift
    double *proposal = nullptr;          // [m][15] c, l0; nullable
    uint8_t *kind = nullptr;             // [m] ASTROZ_CONJ_IS_*, nullable
    const double *prop = nullptr;        // set by launch_conjunction_is: the proposals in the scratch ...
    const uint8_t *propKind = nullptr;   // ... and their kinds
};
cudaError_t conj_is_scratch_bytes(uint32_t m, size_t *bytes);
// for linear shifts K11's assessment into the scratch and the proposal kernel; then K14's steps with the shift
cudaError_t launch_conjunction_is(const ConjIsArgs &a, cudaStream_t stream);

// K12: sensor tracks correlated with catalogue rows (az_correlate.cu, az_correlate.cuh).  Device pointers.
struct CorrArgs {
    const double *elements = nullptr;    // [8][n]
    const double *covariance = nullptr;  // [n][28], nullable (every P zero)
    const uint8_t *model = nullptr;      // [n], nullable (all 0)
    uint32_t n = 0;
    const uint32_t *offsets = nullptr;   // [t + 1]: track j owns observations [offsets[j], offsets[j + 1])
    uint32_t t = 0;
    const double *jd = nullptr, *fr = nullptr;
    const uint8_t *kind = nullptr;
    const double *value = nullptr, *sigma = nullptr;   // [m][6]
    const uint32_t *station = nullptr;
    const double *stations = nullptr;
    double gateProbability = 0.999;
    uint32_t best = 4;
    int grav = 1;
    GravConsts g{};
    void *scratch = nullptr;             // corr_scratch_bytes(n, t, best)
    uint32_t *rows = nullptr;            // [t][best]
    double *d2 = nullptr;                // [t][best]
    uint32_t *used = nullptr, *nGate = nullptr, *nFailed = nullptr;   // [t]
    uint8_t *status = nullptr;           // [t] ASTROZ_CORR_*
    uint8_t *rowStatus = nullptr;        // [n] ASTROZ_COV_OK / ASTROZ_COV_INIT_FAILED
};
// the gates, the near-earth rows, the deep-space rows (when model is given) and the merge, on one stream
cudaError_t launch_correlate(const CorrArgs &a, cudaStream_t stream);

// K13: initial orbits of tracks (az_iod.cu, az_iod.cuh).  Device pointers.
struct IodArgs {
    const uint32_t *offsets = nullptr;   // [t + 1]: track j owns observations [offsets[j], offsets[j + 1]), time-ordered
    uint32_t t = 0;
    const double *jd = nullptr, *fr = nullptr;
    const uint8_t *kind = nullptr;
    const double *value = nullptr, *sigma = nullptr;   // [m][6]
    const uint32_t *station = nullptr;
    const double *stations = nullptr;
    const double *bstar = nullptr;       // [t], nullable (all 0)
    int grav = 1;
    GravConsts g{};
    void *scratch = nullptr;             // iod_scratch_bytes(t)
    double *elements = nullptr;          // [8][t] converted sets, epoch = the track's epoch
    double *state = nullptr;             // [t][6] TEME state at the epoch
    double *wrms = nullptr;              // [t]
    uint8_t *method = nullptr;           // [t] ASTROZ_IOD_METHOD_*
    uint32_t *candidates = nullptr;      // [t]
    double *conv = nullptr;              // [t][2] conversion |dr| km, |dv| km/s
    uint8_t *deepSpace = nullptr;        // [t]
    uint8_t *status = nullptr;           // [t] ASTROZ_IOD_*
};
size_t iod_scratch_bytes(uint32_t t);
// the IOD kernel, K8's near-earth and deep-space fits over one TEME state per track, and the finishing kernel
cudaError_t launch_iod(const IodArgs &a, cudaStream_t stream);
// The scratch of iod_scratch_bytes(t): the conversion batch and the fit's outputs (K13's, and K17's per pair)
struct IodScratch {
    double *init;       // [8][t] osculating initial sets
    double *jd, *fr;    // [t] the epoch observation's time
    double *pos, *vel;  // [t][3] TEME state at the epoch
    double *rms;        // [t][2]
    uint32_t *offsets;  // [t + 1] = 0, 1, ..., t
    uint32_t *iters;    // [t]
    uint8_t *fitStatus, *iodStatus;   // [t]
};
IodScratch iod_scratch(void *p, uint32_t t);
// K8's near-earth and deep-space fits of each initial set to its one TEME state, B* held, into elements[8][t]
cudaError_t launch_iod_conversion(const IodScratch &sc, uint32_t t, int grav, const GravConsts &g, double *elements,
                                  cudaStream_t stream);

// K17: orbits from pairs of tracks (az_link.cu, az_link.cuh)
struct LinkArgs {
    const uint32_t *offsets = nullptr;   // [t + 1]: track j owns observations [offsets[j], offsets[j + 1]), time-ordered
    uint32_t t = 0;
    const double *jd = nullptr, *fr = nullptr;
    const uint8_t *kind = nullptr;
    const double *value = nullptr, *sigma = nullptr;   // [m][6]
    const uint32_t *station = nullptr;
    const double *stations = nullptr;
    const uint32_t *pairs = nullptr;     // [p][2]
    uint32_t p = 0;
    const double *bstar = nullptr;       // [p], nullable (all 0)
    double rMin = 0.0, rMax = 0.0;       // km
    uint32_t maxRevs = 0;
    int grav = 1;
    GravConsts g{};
    void *scratch = nullptr;             // iod_scratch_bytes(p)
    double *elements = nullptr;          // [8][p] converted sets, epoch = the later anchor's time
    double *state = nullptr;             // [p][6] TEME state at the epoch
    double *rho = nullptr;               // [p][2] the winner's ranges, track 1 (earlier anchor) first
    uint8_t *revs = nullptr;             // [p]
    uint8_t *flags = nullptr;            // [p] ASTROZ_LINK_RETROGRADE | ASTROZ_LINK_RIGHT_BRANCH
    double *wrms = nullptr;              // [p]
    uint32_t *used = nullptr;            // [p] used residuals of both tracks
    uint32_t *hypotheses = nullptr;      // [p] admissible states scored
    double *conv = nullptr;              // [p][2] conversion |dr| km, |dv| km/s
    uint8_t *deepSpace = nullptr;        // [p]
    uint8_t *status = nullptr;           // [p] ASTROZ_LINK_*
};
// the link kernel, K13's conversion fits, and the finishing kernel
cudaError_t launch_link(const LinkArgs &a, cudaStream_t stream);

// K18: sensor tasking (az_tasking.cu, az_tasking.cuh).  Device pointers.
struct TaskArgs {
    const double *elements = nullptr;    // [8][n]
    const double *covariance = nullptr;  // [n][28], nullable (every P zero)
    const uint8_t *model = nullptr;      // [n], nullable (all 0)
    uint32_t n = 0;
    const uint8_t *kind = nullptr;       // [S] ASTROZ_OBS_RADAR / ASTROZ_OBS_OPTICAL
    const uint32_t *station = nullptr;   // [S] into stations
    const double *sigma = nullptr;       // [S][4]
    const double *limits = nullptr;      // [S][4] ASTROZ_TASK_LIMIT_*
    uint32_t S = 0;
    const double *stations = nullptr;    // [k][3]
    const double *jd = nullptr, *fr = nullptr;   // [T]
    uint32_t T = 0;
    const double *sun = nullptr;         // [T][3], nullable when no sensor is optical
    double gainMin = 0.0;
    int grav = 1;
    GravConsts g{};
    void *scratch = nullptr;             // task_scratch_bytes(n, S)
    uint32_t *taskRow = nullptr;         // [S][T]
    double *taskGain = nullptr;          // [S][T]
    double *taskValue = nullptr, *taskSpread = nullptr;   // [S][T][4]
    uint32_t *nCandidates = nullptr;     // [S][T]
    double *posterior = nullptr;         // [n][28]
    uint32_t *nTasks = nullptr, *nVisible = nullptr, *nFailed = nullptr;   // [n]
    uint8_t *rowStatus = nullptr;        // [n] ASTROZ_COV_OK / ASTROZ_COV_INIT_FAILED
};
// the build kernel, then per slot the near-earth and deep-space scoring kernels and the one-CTA select kernel
cudaError_t launch_tasking(const TaskArgs &a, cudaStream_t stream);

// K19: reentry prediction (az_reentry.cu, az_reentry.cuh).  The call's scalars as the trajectories read them (from the
// launch's parameters on the device) ...
struct ReentryCall {
    double hi;          // interface height [km]
    double horizon;     // [s] after epoch
    double step;        // output interval [s]
    double scale;       // density_scale
    double sigma;       // density_sigma
    double omega;       // the atmosphere's rotation rate [rad/s]
    double mu, rEq, j2; // the call's grav
};
// ... and the arrays, device pointers.
struct ReentryArgs {
    const double *elements = nullptr;    // [8][n]
    const double *covariance = nullptr;  // [n][28]
    const uint8_t *model = nullptr;      // [n], nullable (all 0)
    uint32_t n = 0;
    const uint32_t *rows = nullptr;      // [m] catalogue rows
    const double *ballistic = nullptr;   // [m] B [m^2/kg], nullable (12.741621 B*)
    const uint64_t *samples = nullptr;   // [m]
    const uint64_t *first = nullptr;     // [m], nullable (all 0)
    const uint64_t *seed = nullptr;      // [m], nullable (all 0)
    uint32_t m = 0;
    uint32_t record = 0;                 // sample words kept per request
    ReentryCall call{};
    int grav = 1;
    GravConsts g{};
    void *scratch = nullptr;             // reentry_scratch_bytes(m)
    double *out = nullptr;               // [m][8] nominal records
    double *states = nullptr;            // [m][6] TEME state at the nominal crossing, nullable
    uint8_t *nominalStatus = nullptr;    // [m] ASTROZ_REENTRY_TRAJ_*
    uint64_t *counts = nullptr;          // [m][3] reentered, above, failed
    double *sampleOut = nullptr;         // [m][record][4]; nullable when record = 0
    uint8_t *status = nullptr;           // [m] ASTROZ_REENTRY_*
};
cudaError_t reentry_scratch_bytes(uint32_t m, size_t *bytes);
// the build kernel, the work-item scan, the near-earth items, then the deep-space items
cudaError_t launch_reentry(const ReentryArgs &a, cudaStream_t stream);

// K16: collision-avoidance manoeuvre trials (az_avoid.cu, az_avoid.cuh; AvoidArgs and avoid_scratch_bytes are there).
// K10 at the burn, the burn, K8's conversion, K10 on the new sets, the covariance transport, K11, the finishing kernel
struct AvoidArgs;
cudaError_t launch_avoid(const AvoidArgs &a, cudaStream_t stream);

// DFMA throughput microbenchmark: returns achieved fp64 FLOP/s (FMA = 2).
cudaError_t measure_fp64_peak(double *flops);
// Arithmetic peak of the fp64 pipe: SMs x 64 lanes x 2 FLOP x the maximum SM clock.
cudaError_t fp64_pipe_peak(double *flops);

int sgp4_variant_count();
void set_sdp4_variant(int v);
void set_sgp4_stripe(uint32_t epochs);  // measurement only: fixed epochs per CTA for the near-earth grid, 0 = automatic
const char *sgp4_variant_name(int variant);

}  // namespace az
