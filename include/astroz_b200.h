/*
 * astroz_b200.h -- C ABI of the H100-native batch SGP4/SDP4 propagator.
 *
 * Drop-in boundary for the propagation path of ATTron/astroz (reference paths relative to the
 * reference repo root).  Every entry point names the reference interface it replaces.
 * Plain pointers and sizes only; no torch / C++ types.  All functions return an int32 from the
 * reference's own error-code space (src/c_api/error.zig:3-19) extended with CUDA codes.
 *
 * Threading / ownership (same contract as the reference, src/c_api/allocator.zig:9-18 and
 * src/Constellation.zig:88,294): handles are not thread-safe; caller owns every I/O buffer and the
 * library never retains it; device memory is owned by the handle and released by the matching *_free.
 * A handle keeps ONE copy of its per-call device scratch (time axis, epoch offsets, mask): calls on a handle
 * must be issued on one stream, or the caller synchronises between calls that use different streams.
 *
 * Failed cells.  Deep-space cells are checked like the reference's scalar path (src/Sdp4.zig:913-967: mean
 * motion <= 0, eccentricity >= 1 or < -0.001, semi-major axis < 0.95, radius < 1 earth radius) and a failing
 * cell is zero-filled, per satellite (the reference's batch path zero-fills the 8 satellites of the batch,
 * src/Constellation.zig:468-471,511-528, and applies only the first three checks, src/Sdp4Batch.zig:293-324).
 * Near-earth cells are never zero-filled -- the reference's near-earth batch path has no reachable failure
 * (src/Sgp4Batch.zig:147-150) -- the state is stored and the optional status byte reports radius < 1 earth
 * radius as ASTROZ_CELL_DECAYED (the scalar path's check, src/Sgp4.zig:588-590) as a diagnostic.
 */
#ifndef ASTROZ_B200_H
#define ASTROZ_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- error codes: src/c_api/error.zig:3-19 (+ CUDA extensions <= -200) ------------------------- */
#define ASTROZ_OK                    0
#define ASTROZ_BAD_TLE_LENGTH      (-1)
#define ASTROZ_BAD_CHECKSUM        (-2)
#define ASTROZ_DEEP_SPACE          (-10)   /* deepSpaceNotSupported */
#define ASTROZ_INVALID_ECC         (-11)
#define ASTROZ_DECAYED             (-12)
#define ASTROZ_VALUE_ERROR         (-20)
#define ASTROZ_ALLOC_FAILED        (-100)
#define ASTROZ_NULL_POINTER        (-101)
#define ASTROZ_NOT_INITIALIZED     (-102)
#define ASTROZ_UNKNOWN             (-999)
#define ASTROZ_CUDA_ERROR          (-200)  /* any CUDA runtime failure; see astroz_cuda_last_error() */
#define ASTROZ_NO_DEVICE           (-201)  /* no CUDA device: the library never falls back to a CPU path */

/* ---- per-cell status bytes (kernel-level codes, src/simdKernels.zig:30-37) --------------------- */
#define ASTROZ_CELL_OK           0
#define ASTROZ_CELL_DECAYED      1
#define ASTROZ_CELL_INVALID_ECC  2
#define ASTROZ_CELL_BAD_SATELLITE 3   /* pairs calls: the query's satellite row is not in the catalog */

/* gravity model selector: src/c_api/sgp4.zig:17-20 (0 = WGS84, 1 = WGS72) */
#define ASTROZ_WGS84 0
#define ASTROZ_WGS72 1

/* src/Constellation.zig:30-42 */
#define ASTROZ_MODE_TEME      0
#define ASTROZ_MODE_ECEF      1
#define ASTROZ_MODE_GEODETIC  2
#define ASTROZ_LAYOUT_SATELLITE_MAJOR 0   /* (n_sats, n_times, 3) */
#define ASTROZ_LAYOUT_TIME_MAJOR      1   /* (n_times, n_sats, 3) */

typedef void *astroz_constellation_t;
typedef void *astroz_sgp4_t;

/* replaces astroz_version (src/c_api/root.zig:13-15): (major<<16)|(minor<<8)|patch */
uint32_t astroz_cuda_version(void);
/* number of visible CUDA devices (0 when none) */
int32_t astroz_cuda_device_count(void);
/* text of the last CUDA failure seen on this thread ("" if none); pointer valid until the next call */
const char *astroz_cuda_last_error(void);

/* pinned host buffers for zero-staging device<->host copies of the output block */
void *astroz_cuda_host_alloc(size_t bytes);
void astroz_cuda_host_free(void *p);
/* Caller-owned buffers.  The host-buffer calls accept ANY host memory.  A buffer from astroz_cuda_host_alloc, or
 * one page-locked with astroz_cuda_host_register (cudaHostRegister: costs about as much as touching the pages once,
 * so it pays for blocks that are reused), receives the result by direct DMA.  Plain pageable memory (a numpy array, a
 * Zig slice from the page allocator) is served through a ring of pinned slots inside the handle: the result leaves the
 * GPU in 32 MB pieces at the full PCIe rate and a small pool of host threads (ASTROZ_COPY_THREADS, default 12, streaming stores) copies
 * each landed piece to its place while the next ones are in flight. */
int32_t astroz_cuda_host_register(void *p, size_t bytes);
int32_t astroz_cuda_host_unregister(void *p);

/* ------------------------------------------------------------------------------------------------
 * Constellation: replaces Constellation.init / propagate / resetCarry / deinit
 * (src/Constellation.zig:101-200, 245-308, 214-218, 202-210).
 * ---------------------------------------------------------------------------------------------- */

/* Parse n TLEs (NUL-terminated 69-column lines, src/Tle.zig:49-101), classify each as SGP4 or SDP4
 * exactly as src/Constellation.zig:115-126, build the device element tables on `device`.
 * device = -1: a MULTI-DEVICE handle -- the catalog is cut into contiguous, 8-row-aligned satellite ranges of
 * equal cost, one per visible GPU (the analogue of the reference's thread fan-out over one propagate call,
 * src/Constellation.zig:327-385).  The environment variable ASTROZ_DEVICES caps the number of GPUs used, the way
 * ASTROZ_THREADS caps the reference's threads (src/Constellation.zig:61-74); ASTROZ_DEVICE_LIST="0,2,3" names
 * ordinals explicitly.  The host-buffer calls (astroz_cuda_constellation_propagate, astroz_cuda_sgp4_propagate_into)
 * then run every GPU at once, each copying its rows over its own PCIe link into its slice of the caller's block;
 * results are bit-identical to a single-device handle.  Entry points that take DEVICE pointers need a
 * single-device handle and return ASTROZ_VALUE_ERROR otherwise.  (The three host constructors accept -1.)
 * Errors: BAD_TLE_LENGTH, INVALID_ECC, DECAYED (first offending TLE aborts, as the reference). */
int32_t astroz_cuda_constellation_create(const char *const *line1, const char *const *line2, uint32_t n,
                                         int32_t grav, int32_t device, astroz_constellation_t *out);

/* Same, from a text blob of 2- or 3-line element sets (src/Tle.zig:103-132 MultiIterator semantics). */
int32_t astroz_cuda_constellation_create_from_text(const char *text, size_t len, int32_t grav, int32_t device,
                                                   astroz_constellation_t *out);

/* Same, from numeric mean elements (the fields Tle.parseOmm fills from an OMM record, src/Tle.zig:134-215):
 * epoch_jd, mean motion [rev/day], eccentricity, inclination / RAAN / argument of perigee / mean anomaly [deg],
 * B* [1/earth radii].  No text round trip, so Monte-Carlo draws keep their full fp64 values. */
int32_t astroz_cuda_constellation_create_from_elements(const double *epoch_jd, const double *mean_motion_rev_day,
                                                       const double *ecc, const double *incl_deg, const double *raan_deg,
                                                       const double *argp_deg, const double *ma_deg, const double *bstar,
                                                       uint32_t n, int32_t grav, int32_t device,
                                                       astroz_constellation_t *out);

/* Same, with the eight element columns already resident in HBM on `device` (DEVICE pointers): classification,
 * Sgp4.initElements / Sdp4.initElements (src/Sgp4.zig:108-417, src/Sdp4.zig:174-657) and the table build of
 * src/Constellation.zig:101-200 run on the GPU, one element set per thread; nothing but counts, epochs and the row
 * maps (16 B per set) returns to the host.  For Monte-Carlo draws and OMM streams generated on the device. */
int32_t astroz_cuda_constellation_create_from_elements_device(
    const double *d_epoch_jd, const double *d_mean_motion_rev_day, const double *d_ecc, const double *d_incl_deg,
    const double *d_raan_deg, const double *d_argp_deg, const double *d_ma_deg, const double *d_bstar, uint32_t n,
    int32_t grav, int32_t device, astroz_constellation_t *out);

void astroz_cuda_constellation_free(astroz_constellation_t h);

/* numSatellites / numSgp4 / numSdp4 (src/Constellation.zig:82,89,95) */
int32_t astroz_cuda_constellation_counts(astroz_constellation_t h, uint32_t *n, uint32_t *n_sgp4, uint32_t *n_sdp4);
/* per-satellite epoch JD (n doubles) and class (n int32: 0 SGP4, 1 SDP4 irez0, 2 irez1, 3 irez2) */
int32_t astroz_cuda_constellation_epochs(astroz_constellation_t h, double *epochs);
int32_t astroz_cuda_constellation_classes(astroz_constellation_t h, int32_t *classes);
/* referenceEpochJd (src/Constellation.zig:92,139-140); settable so satellite shards of one catalog
 * share the whole catalog's reference epoch */
int32_t astroz_cuda_constellation_get_reference_epoch(astroz_constellation_t h, double *jd);
int32_t astroz_cuda_constellation_set_reference_epoch(astroz_constellation_t h, double jd);

/* Constellation.propagate (src/Constellation.zig:245-308) with HOST buffers.
 * pos / vel: n*n_times*3 doubles each (vel may be NULL), written per `layout`; `mode` selects TEME/ECEF/geodetic.
 * Cells whose propagation fails are zero-filled (src/Constellation.zig:511-528).  Includes the
 * host->device copy of jd/fr and the device->host copy of the result block. */
int32_t astroz_cuda_constellation_propagate(astroz_constellation_t h, const double *jd, const double *fr,
                                            uint32_t n_times, double *pos, double *vel, int32_t mode, int32_t layout);

/* Same computation, results left in HBM (d_pos / d_vel are DEVICE pointers on the handle's device).
 * out_num_sats / out_sat_offset place this handle's satellites inside a larger output block
 * (the reference's numSatellites-as-stride convention, src/Constellation.zig:46-51 and
 * bindings/python/src/sgp4.zig:216); pass n and 0 for a stand-alone constellation.
 * d_status (nullable): n*n_times bytes, satellite-major, per-cell ASTROZ_CELL_* code: this handle's satellite i at
 * i*n_times whatever out_num_sats / out_sat_offset are (the status block is not part of the larger block).
 * stream: a cudaStream_t (NULL = the handle's own stream); the call is asynchronous on it. */
int32_t astroz_cuda_constellation_propagate_device(astroz_constellation_t h, const double *jd, const double *fr,
                                                   uint32_t n_times, double *d_pos, double *d_vel, uint8_t *d_status,
                                                   int32_t mode, int32_t layout, uint32_t out_num_sats,
                                                   uint32_t out_sat_offset, void *stream);

/* Arbitrary (satellite, time) pairs: replaces a loop of Satrec.sgp4(jd, fr) calls, one per observation
 * (bindings/python/src/satrec.zig:169-201); the reference has no batched counterpart.  For catalogue workloads that are
 * not grids: correlating observations, orbit-determination residuals, sensor tasking, "where was object k at t_k".
 * Query i propagates catalog row sat[i] (the row numbering of propagate's output block) to jd[i] + fr[i]; pos[i] /
 * vel[i] / status[i] are what propagate would store in that row at that epoch, in the same frame and units:
 *   near earth: tsince = ((jd + fr) - referenceEpochJd) * 1440 + (referenceEpochJd - epoch) * 1440, the grid's
 *               expression to the bit (set_reference_epoch applies); deep space: ((jd + fr) - epoch) * 1440;
 *   ECEF / geodetic: the GMST of the query's own jd + fr, the grid's rotation and geodetic epilogue;
 *   failed cells: a deep-space cell failing the scalar checks is zero-filled with its ASTROZ_CELL_* code; a near-earth
 *   cell is always stored, its status byte flags ASTROZ_CELL_DECAYED only.
 * A query's result depends on (sat, jd, fr) alone: any permutation or duplication of the query list gives the same bits
 * per query.  (Propagation runs one query per thread, so results equal the grid's cells to 1e-10 km, not to the bit:
 * the grid picks some small-angle series per thread over 2-3 epochs.)
 * Host buffers: pos[n][3], vel[n][3] (nullable), status[n] (nullable).  sat[i] >= n_satellites: ASTROZ_VALUE_ERROR,
 * nothing written.  Device memory stays bounded: the queries are processed in chunks, upload / kernels / download
 * overlapped like astroz_cuda_sgp4_array; pageable buffers go through the handle's pinned ring and copy pool.
 * n = 0 is a no-op.  Multi-device handles (device = -1) return ASTROZ_VALUE_ERROR. */
int32_t astroz_cuda_constellation_propagate_pairs(astroz_constellation_t h, const uint32_t *sat, const double *jd,
                                                  const double *fr, uint32_t n, int32_t mode,
                                                  double *pos, double *vel, uint8_t *status);
/* Same with DEVICE pointers on the handle's device.  A query whose sat is out of range gets zeros and
 * ASTROZ_CELL_BAD_SATELLITE; nothing is read for it.  Asynchronous on `stream` (NULL = the handle's stream) except when
 * the catalog has deep-space members: the min / max of jd + fr is then reduced on the device and read back (16 bytes,
 * a synchronisation point) to grow the resonance lattice.  Multi-device handles return ASTROZ_VALUE_ERROR. */
int32_t astroz_cuda_constellation_propagate_pairs_device(astroz_constellation_t h, const uint32_t *d_sat,
                                                         const double *d_jd, const double *d_fr, uint32_t n,
                                                         int32_t mode, double *d_pos, double *d_vel,
                                                         uint8_t *d_status, void *stream);

/* Fused propagate + all-gather for satellite-sharded multi-GPU runs (SURVEY.md section 8e; no reference
 * counterpart -- the reference is single-process).  TEME, satellite-major.  This handle's rows
 * [out_sat_offset, out_sat_offset + n) of the (out_num_sats, n_times, 3) block are written, from inside the
 * propagation kernels, into EVERY GPU's copy of the block:
 *   mc_pos / mc_vel != NULL : NVLS multicast mappings of a symmetric allocation -- one multimem.st per
 *                             16 bytes, NVSwitch replicates it to all GPUs (this one included);
 *   otherwise               : peer_pos[0..n_peers) / peer_vel[...] are the per-GPU mappings of the block
 *                             (this GPU's own mapping included) and each run is stored to all of them.
 * peer_vel / mc_vel may be NULL (positions only).  Asynchronous on `stream`; the caller synchronises the
 * ranks (e.g. a symmetric-memory barrier) before reading other ranks' rows. */
int32_t astroz_cuda_constellation_propagate_gather(astroz_constellation_t h, const double *jd, const double *fr,
                                                   uint32_t n_times, void *const *peer_pos, void *const *peer_vel,
                                                   uint32_t n_peers, void *mc_pos, void *mc_vel,
                                                   uint32_t out_num_sats, uint32_t out_sat_offset, void *stream);

/* A page-locked result block of n * n_times * 3 doubles placed for the handle that will fill it: on a multi-device
 * handle each device's satellite range of a satellite-major block is bound to the NUMA node that device hangs off
 * (mbind), so every GPU writes node-local host memory over its own PCIe link -- a plain pinned allocation lives on one
 * node, and every GPU's writes then share that node's memory controllers.  Free with astroz_cuda_host_free. */
int32_t astroz_cuda_constellation_host_block(astroz_constellation_t h, uint32_t n_times, int32_t layout, double **out);

/* Devices behind a handle: *n_devices (1 for a single-device handle); device_ids[n_devices] (nullable) their CUDA
 * ordinals; first_rows[n_devices + 1] (nullable) the first catalog row of each device's satellite range, then n. */
int32_t astroz_cuda_constellation_devices(astroz_constellation_t h, int32_t *n_devices, int32_t *device_ids,
                                          uint32_t *first_rows);

/* The north star's all-gather behind one handle, without an external communicator: propagate (TEME,
 * satellite-major) and leave the WHOLE (n, n_times, 3) position block -- and velocity block when velocities != 0 --
 * in the HBM of EVERY device of a multi-device handle.  Each device's propagation kernels store their rows, run by
 * run, straight into all devices' copies over NVLink (peer mappings from cudaDeviceEnablePeerAccess), so the
 * transfer overlaps the fp64 work; the call returns when every copy is complete.  d_pos[k] / d_vel[k] receive the
 * block pointers on device k (owned by the handle, valid until the next call or free); arrays of n_devices entries.
 * On a single-device handle the block is simply left on that device. */
int32_t astroz_cuda_constellation_propagate_replicated(astroz_constellation_t h, const double *jd, const double *fr,
                                                       uint32_t n_times, int32_t velocities, double **d_pos,
                                                       double **d_vel);

/* Constellation.resetCarry (src/Constellation.zig:214-218).  The device path re-derives the SDP4
 * resonance state from a 720-minute lattice on every call, so this is a semantic no-op kept for drop-in use. */
int32_t astroz_cuda_constellation_reset_carry(astroz_constellation_t h);

/* stateless near-earth path: replaces Constellation.propagateConstellation (src/Constellation.zig:541-605)
 * as called by SatrecArray.propagate_into / Sgp4Constellation.propagate_into
 * (bindings/python/src/satrec.zig:896-988, bindings/python/src/sgp4.zig:171-268):
 *   tsince[sat][t] = times[t] + epoch_offsets[sat]   (minutes)
 * Only the SGP4 satellites of `h` take part, in catalog order: satellite i -> output row i.
 * epoch_offsets: n_sgp4 doubles.  reference_jd is used for GMST when mode != TEME.
 * satellite_mask (nullable, n_sgp4 bytes): rows whose byte is 0 are not computed and not written
 * (src/Constellation.zig:436-446,530-533).  out_num_sats (0 = n_sgp4): row count of the output block, the
 * reference's output_stride (bindings/python/src/sgp4.zig:215-216).  HOST buffers of out_num_sats*n_times*3. */
int32_t astroz_cuda_sgp4_propagate_into(astroz_constellation_t h, const double *times, uint32_t n_times,
                                        const double *epoch_offsets, double *pos, double *vel, int32_t mode,
                                        double reference_jd, int32_t layout, const uint8_t *satellite_mask,
                                        uint32_t out_num_sats);
/* device-resident variant of the above (d_pos/d_vel device pointers; the mask is still a HOST array) */
int32_t astroz_cuda_sgp4_propagate_into_device(astroz_constellation_t h, const double *times, uint32_t n_times,
                                               const double *epoch_offsets, double *d_pos, double *d_vel,
                                               int32_t mode, double reference_jd, int32_t layout,
                                               const uint8_t *satellite_mask, uint32_t out_num_sats, void *stream);

/* stateless deep-space path: replaces Constellation.propagateSdp4Constellation (src/Constellation.zig:611-674) as
 * called by sdp4_batch_propagate_into (bindings/python/src/satrec.zig:505-644).  Only the SDP4 satellites of `h` take
 * part, in catalog order: deep-space satellite i -> output row sat_offset + i of a block with out_num_sats rows
 * (0 = numSdp4), tsince = (jd[t] + fr[t] - epoch) * 1440 (src/Sdp4Batch.zig:199-215).  HOST buffers; rows of other
 * satellites are not touched. */
int32_t astroz_cuda_sdp4_propagate_into(astroz_constellation_t h, const double *jd, const double *fr, uint32_t n_times,
                                        double *pos, double *vel, int32_t mode, int32_t layout, uint32_t out_num_sats,
                                        uint32_t sat_offset);
/* device-resident variant (d_pos / d_vel DEVICE pointers to the whole out_num_sats-row block) */
int32_t astroz_cuda_sdp4_propagate_into_device(astroz_constellation_t h, const double *jd, const double *fr,
                                               uint32_t n_times, double *d_pos, double *d_vel, int32_t mode,
                                               int32_t layout, uint32_t out_num_sats, uint32_t sat_offset, void *stream);

/* Fused propagate + single-target conjunction screen: replaces Constellation.screenConstellation
 * (src/Constellation.zig:683-756) as called by Sgp4Constellation.screen_conjunction
 * (bindings/python/src/sgp4.zig).  Near-earth satellites only, tsince = times[t] + epoch_offsets[sat].
 * out_min_dists[n_sgp4]: minimum distance (km) to satellite `target_idx` over all times, or `threshold`
 * when never closer; out_min_t[n_sgp4]: index of the (first) time of that minimum, 0 when none.  The
 * target's own entry stays (threshold, 0).  No position block is produced or copied: 12 bytes per
 * satellite come back.  reference_jd is accepted for signature parity (a common GMST rotation does not
 * change distances).  HOST buffers. */
int32_t astroz_cuda_sgp4_screen(astroz_constellation_t h, const double *times, uint32_t n_times,
                                const double *epoch_offsets, uint32_t target_idx, double threshold,
                                double reference_jd, double *out_min_dists, uint32_t *out_min_t);

/* All-vs-all coarse conjunction screen: replaces coarse_screen / coarseScreen
 * (bindings/python/src/conjunction.zig:11-149).  d_positions: DEVICE block (num_sats, num_times, 3) for
 * layout 0 or (num_times, num_sats, 3) for layout 1 (e.g. left in HBM by *_propagate_device);
 * d_valid_mask: nullable per-satellite bytes.  Every (s, other, t) with s < other closer than `threshold`
 * at epoch t is appended to d_pairs[2k], d_pairs[2k+1], d_t_indices[k] (device buffers of max_results
 * entries; order unspecified -- the reference emits the same set ordered by epoch).  *count receives the
 * number of hits found, which may exceed max_results (then only max_results were stored).  Synchronous. */
int32_t astroz_cuda_constellation_coarse_screen_device(astroz_constellation_t h, const double *d_positions,
                                                       uint32_t num_sats, uint32_t num_times, int32_t layout,
                                                       double threshold, const uint8_t *d_valid_mask, uint32_t *d_pairs,
                                                       uint32_t *d_t_indices, uint32_t max_results, uint64_t *count);

/* The all-vs-all branch of astroz.screen(source, times, threshold) (bindings/python/astroz/__init__.py:535-650):
 * propagate the near-earth satellites (tsince = times[t] + epoch_offsets[sat], TEME, positions only), keep the
 * block in HBM, run the coarse screen on it, return only the hits.  pairs / t_indices: HOST buffers of
 * max_results entries. */
int32_t astroz_cuda_sgp4_screen_all(astroz_constellation_t h, const double *times, uint32_t n_times,
                                    const double *epoch_offsets, double threshold, uint32_t *pairs, uint32_t *t_indices,
                                    uint32_t max_results, uint64_t *count);

/* block until everything queued on the handle's stream has finished */
int32_t astroz_cuda_constellation_synchronize(astroz_constellation_t h);

/* Kernel timing is opt-in: enabled != 0 makes every later propagate call on the handle record CUDA events around its
 * kernels (about a dozen microseconds of stream time per call, which is why it is off by default; the environment
 * variable ASTROZ_TIMING=1 turns it on for new handles).  astroz_cuda_constellation_last_kernel_ms returns
 * ASTROZ_NOT_INITIALIZED for a call made with timing off. */
int32_t astroz_cuda_constellation_set_timing(astroz_constellation_t h, int32_t enabled);

/* device time (ms, CUDA events on the launching stream) of the propagation kernels of the last
 * propagate call on this handle: [0] SGP4 grid kernel, [1] span of all grid launches of the call (the two grids of a
 * mixed catalog run side by side on two streams, so [1] < [0] + [2] there), [2] SDP4 grid kernel.
 * After a HOST-buffer call (whose grid is launched in chunks so copies overlap compute) all three slots hold the span
 * from the first kernel of the first chunk to the last kernel of the last chunk; on a multi-device handle, the
 * maximum over its devices. */
int32_t astroz_cuda_constellation_last_kernel_ms(astroz_constellation_t h, float ms[3]);

/* ------------------------------------------------------------------------------------------------
 * Single satellite: replaces sgp4_init / sgp4_free / sgp4_propagate / sgp4_propagate_batch
 * (src/c_api/root.zig:48-59, src/c_api/sgp4.zig:16-100) -- extended to deep-space objects the way
 * Satrec.twoline2rv falls back to SDP4 (bindings/python/src/satrec.zig:135-160).
 * ---------------------------------------------------------------------------------------------- */
int32_t astroz_cuda_sgp4_init(const char *line1, const char *line2, int32_t grav, int32_t device, astroz_sgp4_t *out);
void astroz_cuda_sgp4_free(astroz_sgp4_t h);
/* 1 if the object is propagated with SDP4 (Satrec.is_deep_space) */
int32_t astroz_cuda_sgp4_is_deep_space(astroz_sgp4_t h);
int32_t astroz_cuda_sgp4_epoch(astroz_sgp4_t h, double *epoch_jd);
/* Mean elements behind the python-sgp4 attribute getters of Satrec (bindings/python/src/satrec.zig:395-470):
 * out[10] = ecco, inclo, nodeo, argpo, mo (rad), no_kozai (rad/min), bstar, a (un-Kozai'd semi-major axis, earth
 * radii: Sgp4.Elements.a, src/Sgp4.zig:206-228), no_unkozai (rad/min), epoch JD. */
int32_t astroz_cuda_sgp4_elements(astroz_sgp4_t h, double *out10);
/* one time: pos[3] km, vel[3] km/s (TEME) */
int32_t astroz_cuda_sgp4_propagate(astroz_sgp4_t h, double tsince, double pos[3], double vel[3]);
/* count times (minutes since epoch); results[count][6] = x y z vx vy vz (src/c_api/sgp4.zig:60-100) */
int32_t astroz_cuda_sgp4_propagate_batch(astroz_sgp4_t h, const double *times, double *results, uint32_t count);

/* Satrec.sgp4_array_into(jd, fr, positions, velocities) (bindings/python/src/satrec.zig:299-343): count absolute
 * epochs jd[i] + fr[i]; tsince = ((jd + fr) - epoch_jd) * 1440 is formed on the device in fp64 (the same
 * expression, :263).  results[count][6] = x y z vx vy vz.  Near-earth objects run on the time-parallel kernel. */
int32_t astroz_cuda_sgp4_array(astroz_sgp4_t h, const double *jd, const double *fr, double epoch_jd, double *results,
                               uint32_t count);

/* BASELINE config 5 (fp32 tolerance study; defined by this project, the reference has no such path): the
 * near-earth satellites of `h` propagated with the arithmetic in fp32 -- phase64 = 0: everything in fp32;
 * phase64 = 1: the three secular angles formed and reduced in fp64, the rest in fp32.  Satellite-major TEME,
 * results widened to fp64 words so they can be compared with astroz_cuda_constellation_propagate_device. */
int32_t astroz_cuda_constellation_propagate_device_f32(astroz_constellation_t h, const double *jd, const double *fr,
                                                       uint32_t n_times, double *d_pos, double *d_vel, int32_t phase64,
                                                       void *stream);

/* ------------------------------------------------------------------------------------------------
 * Numerical propagation of a batch of initial states: replaces propagate_numerical (bindings/python/src/propagator.zig:
 * 13-193), which integrates ONE state per call on one CPU thread, with n independent states in one device call.
 * State i's trajectory is what propagate_numerical(states[i], t0, duration, dt, mu, ...) returns for it:
 *   samples: Propagator.propagate (src/propagators/Propagator.zig:22-48) -- the state at t0, then after each step of
 *            while (t < t_end) { step = min(dt, t_end - t); ...; t += step; }, t_end = t0 + duration; every state shares
 *            this sequence, given by astroz_cuda_numerical_times;
 *   forces:  two-body, then J2 (forces & ASTROZ_FORCE_J2), then exponential-atmosphere drag (forces & ASTROZ_FORCE_DRAG:
 *            rho0 1.225 kg/m^3, H 7.249 km, none above 1500 km), ForceModel.zig:42-111 and :351-375; drag takes cd,
 *            area [m^2] and mass [kg] per state;
 *   integrator: ASTROZ_INTEGRATOR_RK4 (Integrator.zig:21-58) or ASTROZ_INTEGRATOR_DP87 (Dormand-Prince 8(7),
 *            Integrator.zig:60-269: hMin 0.001 s, hMax 3600 s, h starting at 60 s and carried from interval to interval,
 *            10,000 accepted substeps per interval at most) with tolerances rtol / atol.
 * Units: km, km/s, s, km^3/s^2.  Outputs: out[n][samples][6] (x y z vx vy vz), status[n] (ASTROZ_NUMERICAL_*),
 * steps[n][2] (nullable): accepted and rejected steps (RK4: one accepted step per interval).
 * Where the reference never returns -- a DP87 step rejected at hMin is retried with the same state and step forever
 * (e.g. a state whose error norm is not finite at any step size, such as one at the centre; a re-entry under drag does
 * not stop, its stiff drag term only shrinks the steps) -- the state stops: status ASTROZ_NUMERICAL_STOPPED and its
 * remaining samples zero-filled, like the library's failed cells.
 * ASTROZ_VALUE_ERROR, nothing written: dt <= 0; t0, duration, dt, mu, rtol, atol (or j2 / r_eq when used) not finite;
 * j2 missing with J2 on; r_eq missing with J2 or drag on; drag arrays missing with drag on; an unknown integrator or
 * force bit; a sampling loop that would not end or more than 2^32 - 2 steps; an output size that overflows;
 * device = -1 (these calls run on one device). */
#define ASTROZ_FORCE_J2        1
#define ASTROZ_FORCE_DRAG      2
#define ASTROZ_INTEGRATOR_RK4  0
#define ASTROZ_INTEGRATOR_DP87 1
#define ASTROZ_NUMERICAL_OK            0
#define ASTROZ_NUMERICAL_STOPPED       1   /* the reference would loop forever; remaining samples zero-filled */
#define ASTROZ_NUMERICAL_SUBSTEP_LIMIT 2   /* some DP87 interval hit 10,000 substeps: that sample is the reference's, not
                                              at its nominal time */
#define ASTROZ_NUMERICAL_NON_FINITE    3   /* an RK4 trajectory went to NaN or inf (the values are kept) */
/* per-satellite status bytes of the element fits (astroz_cuda_fit_elements below) */
#define ASTROZ_FIT_CONVERGED            0   /* the cost stopped changing, or reached the rounding floor */
#define ASTROZ_FIT_ITERATION_LIMIT      1   /* max_iter steps tried: the best accepted iterate is returned */
#define ASTROZ_FIT_INIT_FAILED          2   /* the initial set fails SGP4 init (e outside [0, 1), perigee below 1 ER) */
#define ASTROZ_FIT_DEEP_SPACE           3   /* period > 225 min: astroz_cuda_fit_elements[_device] do not fit deep-space
                                               sets (the _mixed calls do, and never return this) */
#define ASTROZ_FIT_TOO_FEW_OBSERVATIONS 4   /* fewer scalar residuals than fitted variables */

/* The sample times of the batch calls (Propagator.zig:32-45 evaluated on the host, the one home of the sampling rule):
 * *count = number of samples; times (nullable) receives them.  Same argument errors as the batch calls. */
int32_t astroz_cuda_numerical_times(double t0, double duration, double dt, double *times, uint64_t *count);

/* HOST buffers: states[n][6]; drag_cd / drag_area / drag_mass [n] each (NULL unless drag is on); out / status / steps as
 * above.  States are processed in chunks, upload / kernel / download overlapped; pageable buffers go through a pinned
 * ring and the host copy pool, pinned and registered ones receive their results by direct DMA.  The device slots are
 * returned before the call returns; per device, two streams and (after the first pageable transfer) the 96 MB pinned
 * ring stay for the life of the process.  n = 0 is a no-op. */
int32_t astroz_cuda_propagate_numerical(const double *states, uint32_t n, double t0, double duration, double dt,
                                        double mu, int32_t forces, const double *j2, const double *r_eq,
                                        const double *drag_cd, const double *drag_area, const double *drag_mass,
                                        int32_t integrator, double rtol, double atol, int32_t device, double *out,
                                        uint8_t *status, uint64_t *steps);
/* Same with DEVICE pointers on `device` (j2 / r_eq stay host scalars).  Asynchronous on `stream` (a cudaStream_t, NULL =
 * the legacy default stream): the step sizes travel in the launch's parameters, so the call queues one kernel and
 * returns. */
int32_t astroz_cuda_propagate_numerical_device(const double *d_states, uint32_t n, double t0, double duration,
                                               double dt, double mu, int32_t forces, const double *j2,
                                               const double *r_eq, const double *d_drag_cd,
                                               const double *d_drag_area, const double *d_drag_mass,
                                               int32_t integrator, double rtol, double atol, int32_t device,
                                               double *d_out, uint8_t *d_status, uint64_t *d_steps, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Numerical propagation under a caller's ordered list of force models: the force models of the reference's propagators
 * module (src/propagators/ForceModel.zig) for a batch of states.  State i's trajectory is what Propagator.propagate
 * (src/propagators/Propagator.zig:22-48) returns for states[i] with the chosen integrator and, as its force, the list:
 *   one model: that model's acceleration as it is (bindings/python/src/propagator.zig:138-146);
 *   several:   Composite (ForceModel.zig:365-374): a total starting at zero, the models added in list order, component by
 *              component (the order changes the low bits and is part of the result).  At most 16 models; kinds repeat.
 * Sampling, integrators, tolerances, status bytes, zero-filled stopped states and step counts are those of
 * astroz_cuda_propagate_numerical above.
 * Each model's fields, by kind (the reference's parameters, with its arithmetic line for line):
 *   ASTROZ_MODEL_TWO_BODY      mu                                               ForceModel.zig:42-56
 *   ASTROZ_MODEL_J2 / J3 / J4  mu, coef (j2 / j3 / j4), r_eq                    :58-80, :113-143, :145-176
 *   ASTROZ_MODEL_DRAG          r_eq, rho0, scale_height, c (cd), area, mass, max_altitude          :82-111
 *   ASTROZ_MODEL_IMPROVED_DRAG r_eq, c (cd), area, mass, max_altitude, f107     :268-349 (five layers, the atmosphere
 *                              rotating at 7.2921150e-5 rad/s, zero below 100 km and above max_altitude)
 *   ASTROZ_MODEL_SRP           c (cr), area, mass, r_eq, pos (sunPos)           :178-228 (P = 4.56e-6 N/m^2, AU =
 *                              1.495978707e8 km, src/constants.zig:27-28; cylindrical shadow of radius r_eq)
 *   ASTROZ_MODEL_THIRD_BODY    mu, pos                                          :230-266 (Battin's formula)
 * Fields a kind does not use are ignored.  Flags: ASTROZ_MODEL_PER_STATE_C / _AREA / _MASS take c / area / mass from
 * c_per_state / area_per_state / mass_per_state[n] instead (drag kinds and SRP); ASTROZ_MODEL_POS_TABLE takes pos from
 * pos_table[K][3] instead (SRP and third body), K = samples - 1: row k holds for every force evaluation of output interval
 * k, DP87 substeps and rejected attempts included -- the batch form of updateSunPos / updatePos between steps.
 * The reference's quirks are kept: J3's x / y terms carry an extra 1/r, J4 divides by r^9, ImprovedDrag is zero below
 * 100 km.
 * ASTROZ_VALUE_ERROR, nothing written or allocated: n_models 0 or > 16; an unknown kind or flag; a non-finite scalar field
 * the kind uses; a flag set and its pointer NULL; device = -1; and every error of astroz_cuda_propagate_numerical. */
#define ASTROZ_MODEL_TWO_BODY      0
#define ASTROZ_MODEL_J2            1
#define ASTROZ_MODEL_J3            2
#define ASTROZ_MODEL_J4            3
#define ASTROZ_MODEL_DRAG          4
#define ASTROZ_MODEL_IMPROVED_DRAG 5
#define ASTROZ_MODEL_SRP           6
#define ASTROZ_MODEL_THIRD_BODY    7
#define ASTROZ_MODEL_PER_STATE_C    1u
#define ASTROZ_MODEL_PER_STATE_AREA 2u
#define ASTROZ_MODEL_PER_STATE_MASS 4u
#define ASTROZ_MODEL_POS_TABLE      8u
#define ASTROZ_MAX_MODELS          16
typedef struct {
    int32_t kind;
    uint32_t flags;
    double mu;
    double coef;
    double r_eq;
    double rho0;
    double scale_height;
    double max_altitude;
    double f107;
    double c;
    double area;
    double mass;
    double pos[3];
    const double *c_per_state;
    const double *area_per_state;
    const double *mass_per_state;
    const double *pos_table;
} astroz_force_model_t;

/* HOST buffers: states[n][6], the per-state arrays [n] and position tables [K][3] the models name, out / status / steps
 * as astroz_cuda_propagate_numerical.  The same chunked pipeline; the position tables are uploaded once per call. */
int32_t astroz_cuda_propagate_numerical_models(const double *states, uint32_t n, double t0, double duration, double dt,
                                               const astroz_force_model_t *models, uint32_t n_models,
                                               int32_t integrator, double rtol, double atol, int32_t device,
                                               double *out, uint8_t *status, uint64_t *steps);
/* Same with DEVICE pointers on `device` for the states, outputs and every per-state array and position table the models
 * name (the descriptors themselves are host memory).  Asynchronous on `stream`: the model list travels in the launch's
 * parameters, so the call queues one kernel and returns. */
int32_t astroz_cuda_propagate_numerical_models_device(const double *d_states, uint32_t n, double t0, double duration,
                                                      double dt, const astroz_force_model_t *models, uint32_t n_models,
                                                      int32_t integrator, double rtol, double atol, int32_t device,
                                                      double *d_out, uint8_t *d_status, uint64_t *d_steps,
                                                      void *stream);

/* ------------------------------------------------------------------------------------------------
 * Impulsive maneuvers: the loop of Spacecraft.propagate (src/Spacecraft.zig:172-323) for a batch of states, each with
 * its own impulse schedule.  State i fires impulses[impulse_offsets[i] .. impulse_offsets[i + 1]) in list order (the
 * list is not sorted), under the model list `models` with RK4 or DP87:
 *   y = y0; t = t0; tf = t0 + duration; sample (t, y); idx = 0
 *   while t < tf:
 *       while idx < count and imp[idx].time <= t + h:     (an impulse before t0 fires at once)
 *           dt = imp[idx].time - t; if dt > 0: step dt, t += dt, sample
 *           burn imp[idx] (a phasing burn samples its coast and advances t); sample; idx += 1
 *       s = min(h, tf - t); step s; t += s; sample    (s <= 0 after a phasing coast that passes tf)
 *       stop when 0.5 v^2 - mu / r > 0, is NaN, or r > 100,000 km (status ASTROZ_MANEUVER_ABNORMAL)
 * Burns, operation for operation as the reference's:
 *   ASTROZ_IMPULSE_ABSOLUTE      velocity += p[0..2]                                   (calculations.zig:480-485)
 *   ASTROZ_IMPULSE_PROGRADE      velocity += v / |v| * p[0]                            (Spacecraft.zig:260-263)
 *   ASTROZ_IMPULSE_PHASE         the prograde dv of calculatePhaseChange(|r|, p[0], p[1]) (:310-323), a coast of
 *                                `while t < tEnd { step h; sample (t + h); t += h }`, tEnd = t + 2 pi sqrt(r^3 / mu)
 *                                * p[1], then the negated dv (:237-252)
 *   ASTROZ_IMPULSE_PLANE_CHANGE  applyPlaneChange (:272-307): nothing below 1e-10 rad; otherwise dv = (hx sin di,
 *                                hy sin di, hz cos di) * 2 |v| sin(angle / 2) / |h|, h = r x v -- the reference's
 *                                "simplified" direction, not the textbook plane change.
 * mu is the central body's parameter (the reference's orbitingObject.mu): the phasing burn and the abnormal-orbit test
 * use it.  A DP87 state carries its step size through every step: partial steps to a burn, coasts and regular steps (a
 * step of 1e-14 s or less makes no attempt and leaves the step size at min(step size, that step)).
 * Departures from the reference: the inputs are states, not TLEs, and tf = t0 + duration; where the reference never
 * returns, the state stops (ASTROZ_NUMERICAL_STOPPED: a DP87 rejection at hMin, or a sample count that would pass
 * 2^32 - 2); position tables are refused (their rows follow K7's shared output intervals, which do not exist here).
 * Outputs: rows of max_samples samples per state: times[n][max_samples], out[n][max_samples][6]; n_samples[n] = the
 * number of samples state i's trajectory has, also when that is more than max_samples (only the first max_samples are
 * written); samples past n_samples are zero.  Sample times repeat (the sample before and after a burn) and can decrease
 * (the negative last step).  status[n]: ASTROZ_MANEUVER_TRUNCATED first, then the ASTROZ_NUMERICAL_* codes, then
 * ASTROZ_MANEUVER_ABNORMAL; steps[n][2] (nullable) as for the batch calls.
 * ASTROZ_VALUE_ERROR, nothing read, written or allocated: h <= 0; t0, duration, h, mu, rtol or atol not finite; a
 * regular sampling loop that would not end; an unknown impulse kind; a non-finite impulse time or parameter; orbits <= 0;
 * offsets that decrease or offsets[n] != m (host call); max_samples = 0; every model-list error, and a position table;
 * an unknown integrator; device = -1. */
#define ASTROZ_IMPULSE_ABSOLUTE     0   /* p = dv[3] km/s */
#define ASTROZ_IMPULSE_PROGRADE     1   /* p[0] = dv km/s */
#define ASTROZ_IMPULSE_PHASE        2   /* p[0] = angle rad, p[1] = orbits (> 0) */
#define ASTROZ_IMPULSE_PLANE_CHANGE 3   /* p[0] = delta inclination rad, p[1] = delta RAAN rad */
typedef struct {
    double time;
    int32_t kind;
    uint32_t reserved;
    double p[3];
} astroz_impulse_t;
#define ASTROZ_MANEUVER_ABNORMAL  4     /* the reference's abnormal-orbit stop; the trajectory ends at that sample */
#define ASTROZ_MANEUVER_TRUNCATED 5     /* more than max_samples samples: the first max_samples are written */

/* HOST buffers: states[n][6], impulse_offsets[n + 1], impulses[m], the per-state arrays the models name, outputs as
 * above.  The chunked pipeline of astroz_cuda_propagate_numerical; the schedules are uploaded once per call. */
int32_t astroz_cuda_propagate_maneuvers(const double *states, uint32_t n, double t0, double duration, double h, double mu,
                                        const uint32_t *impulse_offsets, const astroz_impulse_t *impulses, uint32_t m,
                                        const astroz_force_model_t *models, uint32_t n_models, int32_t integrator,
                                        double rtol, double atol, uint32_t max_samples, int32_t device, double *times,
                                        double *out, uint64_t *n_samples, uint8_t *status, uint64_t *steps);
/* Same with DEVICE pointers on `device` for the states, offsets, impulses, per-state arrays and outputs (the descriptors
 * are host memory).  Asynchronous on `stream`: the call queues one kernel and returns, so it reads neither offsets nor
 * impulses -- they must pass the host call's checks (astroz_b200.numerical.propagate_maneuvers_batch_device checks
 * them before they go up). */
int32_t astroz_cuda_propagate_maneuvers_device(const double *d_states, uint32_t n, double t0, double duration, double h,
                                               double mu, const uint32_t *d_impulse_offsets,
                                               const astroz_impulse_t *d_impulses, uint32_t m,
                                               const astroz_force_model_t *models, uint32_t n_models, int32_t integrator,
                                               double rtol, double atol, uint32_t max_samples, int32_t device,
                                               double *d_times, double *d_out, uint64_t *d_n_samples, uint8_t *d_status,
                                               uint64_t *d_steps, void *stream);

/* ---- element fits (K8): SGP4 mean elements from TEME ephemerides ------------------------------------------------------
 * For each satellite s of a batch, Levenberg-Marquardt finds the near-earth mean elements whose SGP4 states best match
 * its observations in the weighted least-squares sense, residuals (pos - model) / pos_sigma and (vel - model) / vel_sigma.
 *   elements[8][n]: initial columns as astroz_cuda_constellation_create_from_elements takes them -- epoch JD, mean motion
 *            [rev/day], eccentricity, inclination, RAAN, argument of perigee, mean anomaly [deg], B*; grav ASTROZ_WGS72 or
 *            ASTROZ_WGS84.  The epoch is held: the fitted elements are mean elements at that epoch;
 *   observations: satellite s owns [offsets[s], offsets[s + 1]) of jd[m], fr[m], pos[m][3] (TEME km) and vel[m][3]
 *            (TEME km/s, nullable: positions only); tsince = ((jd + fr) - epoch) * 1440, as propagate_pairs forms it;
 *   variables: n, e cos w, e sin w, i, RAAN, M + w and B* (held at its initial value when fit_bstar = 0); forward-
 *            difference Jacobian, Marquardt damping x10 / /10, at most max_iter steps (25 is a good default);
 *   model:   every trial set goes through the library's near-earth init and propagation, so the fitted columns passed to
 *            create_from_elements and propagated with propagate_pairs at the observation times give back the RMS.
 * Outputs: fitted[8][n] (epoch unchanged; RAAN, w and M in [0, 360)), rms[n][2] (sqrt of the mean squared position
 * residual [km], and velocity residual [km/s] or 0 without velocities), iterations[n] (steps tried), status[n]
 * (ASTROZ_FIT_*).  A satellite that does not converge returns its best accepted iterate; one that is not fitted (init
 * failure, deep space, too few observations) returns its initial columns with zero RMS.  No output is NaN.  A
 * satellite's bytes depend on its own inputs alone, not on the rest of the batch.
 * ASTROZ_VALUE_ERROR, nothing written: device = -1 (a fit runs on one device); pos_sigma or vel_sigma not finite or
 * <= 0; max_iter = 0; an unknown grav; and for the host call offsets that decrease or offsets[n] != m, or a non-finite
 * element or observation value.  n = 0 is a no-op.  Without a device: ASTROZ_NO_DEVICE.
 * HOST buffers: the inputs go up once (pageable ones through a pinned ring, pinned ones by direct DMA), one launch fits
 * the batch, and the call returns with the results in place. */
int32_t astroz_cuda_fit_elements(const double *elements, uint32_t n, int32_t grav, const uint32_t *offsets,
                                 const double *jd, const double *fr, const double *pos, const double *vel, uint32_t m,
                                 double pos_sigma, double vel_sigma, int32_t fit_bstar, uint32_t max_iter,
                                 int32_t device, double *fitted, double *rms, uint32_t *iterations, uint8_t *status);
/* Same with DEVICE pointers on `device` (the observation count is d_offsets[n]).  One launch on `stream`: no allocation,
 * no synchronisation, and only the scalar arguments are checked -- the offsets and values must be valid. */
int32_t astroz_cuda_fit_elements_device(const double *d_elements, uint32_t n, int32_t grav, const uint32_t *d_offsets,
                                        const double *d_jd, const double *d_fr, const double *d_pos,
                                        const double *d_vel, double pos_sigma, double vel_sigma, int32_t fit_bstar,
                                        uint32_t max_iter, int32_t device, double *d_fitted, double *d_rms,
                                        uint32_t *d_iterations, uint8_t *d_status, void *stream);
/* Mixed batches: the calls above, plus the deep-space sets (initial period > 225 min) fitted under SDP4.  Same arguments,
 * checks and return codes.  Each call queues the near-earth fit and then the deep-space fit over the whole batch on one
 * stream; the second overwrites only the deep-space rows, so every near-earth row is the bytes astroz_cuda_fit_elements
 * gives it.  A deep-space set:
 *   variables: equinoctial -- n, e cos(w + RAAN), e sin(w + RAAN), tan(i/2) cos RAAN, tan(i/2) sin RAAN, M + w + RAAN and
 *            B* -- well conditioned at i = 0 and e = 0 (GEO).  They diverge as i -> 180 deg: retrograde deep-space sets
 *            near i = 180 deg are out of scope;
 *   class:   held: a trial set whose period falls to 225 min or below counts as a set that cannot be built (a rejected
 *            step, or the backward difference);
 *   model:   every trial set goes through the library's deep-space init and the propagate_pairs deep-space query (its
 *            resonance integrator included), so create_from_elements + propagate_pairs give back the RMS.  An observation
 *            the model cannot propagate (decayed, eccentricity out of range) fails the pass: ASTROZ_FIT_INIT_FAILED for
 *            the initial set, a rejected step for a trial set. */
int32_t astroz_cuda_fit_elements_mixed(const double *elements, uint32_t n, int32_t grav, const uint32_t *offsets,
                                       const double *jd, const double *fr, const double *pos, const double *vel,
                                       uint32_t m, double pos_sigma, double vel_sigma, int32_t fit_bstar,
                                       uint32_t max_iter, int32_t device, double *fitted, double *rms,
                                       uint32_t *iterations, uint8_t *status);
int32_t astroz_cuda_fit_elements_mixed_device(const double *d_elements, uint32_t n, int32_t grav,
                                              const uint32_t *d_offsets, const double *d_jd, const double *d_fr,
                                              const double *d_pos, const double *d_vel, double pos_sigma,
                                              double vel_sigma, int32_t fit_bstar, uint32_t max_iter, int32_t device,
                                              double *d_fitted, double *d_rms, uint32_t *d_iterations,
                                              uint8_t *d_status, void *stream);

/* ---- element fits (K8) from sensor observations: Earth-fixed states, radar and optical angles, with covariance ---------
 * astroz_cuda_fit_elements[_mixed] with a measurement layer between the model's TEME state and the residual.  The
 * variables, steps, damping, stopping rule, deep-space handling and the mixed calls' row rule are K8's.  Observation i
 * of satellite s ([offsets[s], offsets[s + 1]) as in K8) is jd[i] + fr[i], kind[i] (ASTROZ_OBS_*), value[i][6] and
 * sigma[i][6] (components past the kind's count are ignored), and station[i], a row of stations[k][3] = (geodetic
 * latitude deg, longitude deg, height km) on WGS84, read by the radar and optical kinds only (station may be NULL when
 * no observation uses one):
 *   TEME_STATE  x y z [km], vx vy vz [km/s]: K8's observation;
 *   ECEF_STATE  r_ecef = Rz(GMST) r, the rotation of propagate_pairs' ECEF output (GMST of the observation's jd + fr),
 *               and the Earth-fixed velocity v_ecef = Rz(GMST) v - omega x r_ecef (omega = 360.98564736629 deg/day).
 *               Unlike this kind, the library's ECEF output mode leaves omega x r out, as the reference does;
 *   RADAR       range [km], azimuth [rad, from north through east], elevation [rad], range-rate [km/s] in the station's
 *               geodetic horizon frame: rho = r_ecef - r_station, range-rate = rho . v_ecef / |rho|;
 *   OPTICAL     topocentric right ascension and declination [rad] in TEME: rho = r_teme - Rz(GMST)^T r_station.
 * Observations are geometric and instantaneous: no light time, aberration or refraction.  Polar motion and the TEME ->
 * GCRF rotation are the caller's: optical angles must be in TEME.
 *   residuals: (observed - model) / sigma.  Azimuth and right-ascension differences are wrapped to (-pi, pi] and
 *              multiplied by the cosine of the observed elevation / declination (sigma is an arc on the sky).  sigma =
 *              +inf: the component is not used (a radar without range-rate, a position-only fix);
 *   outputs:   fitted[8][n] and iterations[n], status[n] as K8; wrms[n] = sqrt(cost / used residuals), dimensionless,
 *              about 1 when the sigmas are right; n_residuals[n] the used scalar residuals (ASTROZ_FIT_TOO_FEW_
 *              OBSERVATIONS when fewer than the fitted variables); covariance[n][28] the upper triangle, row by row, of
 *              the 7 x 7 covariance (J^T W J)^-1 of the fitted variables at the final iterate, in the fit's own
 *              variables and order (near-earth: n, e cos w, e sin w, i, RAAN, M + w, B*; deep space: K8's equinoctial
 *              set), units rev/day, rad and 1/ER.  The B* row and column are zero when B* is held.  All 28 words zero:
 *              the normal matrix was not positive definite (or the satellite was not fitted); model[n] 0 when row s
 *              was fitted in the near-earth variables, 1 in the deep-space ones (the _mixed calls' deep-space rows):
 *              the variables its covariance is stated in.
 * ASTROZ_VALUE_ERROR, nothing written: device = -1, max_iter = 0, an unknown grav; and for the host calls offsets that
 * decrease or offsets[n] != m, a non-finite element or time, an unknown kind, a station index >= k (kinds that read
 * one), a sigma that is <= 0 or NaN, a non-finite value in a used component (or the elevation / declination of a used
 * azimuth / right ascension), a station that is not finite or whose latitude is outside [-90, 90]. */
#define ASTROZ_OBS_TEME_STATE 0
#define ASTROZ_OBS_ECEF_STATE 1
#define ASTROZ_OBS_RADAR      2
#define ASTROZ_OBS_OPTICAL    3
#define ASTROZ_OBS_VALUES     6    /* columns of value and sigma */
#define ASTROZ_FIT_COVARIANCE_WORDS 28
/* HOST buffers: one upload (pageable through a pinned ring, pinned by direct DMA), one launch, plain copies back. */
int32_t astroz_cuda_fit_observations(const double *elements, uint32_t n, int32_t grav, const uint32_t *offsets,
                                     const double *jd, const double *fr, const double *value, const double *sigma,
                                     const uint32_t *station, const uint8_t *kind, uint32_t m, const double *stations,
                                     uint32_t k, int32_t fit_bstar, uint32_t max_iter, int32_t device, double *fitted,
                                     double *wrms, uint32_t *n_residuals, double *covariance, uint32_t *iterations,
                                     uint8_t *status, uint8_t *model);
/* Mixed batches: deep-space rows fitted under SDP4 too, as astroz_cuda_fit_elements_mixed. */
int32_t astroz_cuda_fit_observations_mixed(const double *elements, uint32_t n, int32_t grav, const uint32_t *offsets,
                                           const double *jd, const double *fr, const double *value,
                                           const double *sigma, const uint32_t *station, const uint8_t *kind,
                                           uint32_t m, const double *stations, uint32_t k, int32_t fit_bstar,
                                           uint32_t max_iter, int32_t device, double *fitted, double *wrms,
                                           uint32_t *n_residuals, double *covariance, uint32_t *iterations,
                                           uint8_t *status, uint8_t *model);
/* DEVICE pointers on `device` (the observation count is d_offsets[n]): one launch (two for _mixed) on `stream`, no
 * allocation, no synchronisation; only the scalar arguments are checked -- kinds, stations and sigmas must be valid. */
int32_t astroz_cuda_fit_observations_device(const double *d_elements, uint32_t n, int32_t grav,
                                            const uint32_t *d_offsets, const double *d_jd, const double *d_fr,
                                            const double *d_value, const double *d_sigma, const uint32_t *d_station,
                                            const uint8_t *d_kind, const double *d_stations, int32_t fit_bstar,
                                            uint32_t max_iter, int32_t device, double *d_fitted, double *d_wrms,
                                            uint32_t *d_n_residuals, double *d_covariance, uint32_t *d_iterations,
                                            uint8_t *d_status, uint8_t *d_model, void *stream);
int32_t astroz_cuda_fit_observations_mixed_device(const double *d_elements, uint32_t n, int32_t grav,
                                                  const uint32_t *d_offsets, const double *d_jd, const double *d_fr,
                                                  const double *d_value, const double *d_sigma,
                                                  const uint32_t *d_station, const uint8_t *d_kind,
                                                  const double *d_stations, int32_t fit_bstar, uint32_t max_iter,
                                                  int32_t device, double *d_fitted, double *d_wrms,
                                                  uint32_t *d_n_residuals, double *d_covariance,
                                                  uint32_t *d_iterations, uint8_t *d_status, uint8_t *d_model,
                                                  void *stream);
/* The measurement model alone, one thread per observation: states[m][6] (TEME km, km/s) at jd[i] + fr[i] ->
 * values[m][6], the kind's values (azimuth and right ascension in [0, 2 pi)), zero past its count.  For per-observation
 * residuals and outlier editing; no visibility search: h is evaluated at the times given.  ASTROZ_VALUE_ERROR, nothing
 * written: device = -1; for the host call an unknown kind, a station index >= k, a bad station, a non-finite time.
 * The _device form checks only its scalars and runs on `stream`. */
int32_t astroz_cuda_observe(const double *states, const double *jd, const double *fr, const uint8_t *kind,
                            const uint32_t *station, uint32_t m, const double *stations, uint32_t k, int32_t device,
                            double *values);
int32_t astroz_cuda_observe_device(const double *d_states, const double *d_jd, const double *d_fr,
                                   const uint8_t *d_kind, const uint32_t *d_station, uint32_t m,
                                   const double *d_stations, int32_t device, double *d_values, void *stream);
/* ---- state covariance (K10): a fitted element set's covariance carried to any time, in TEME or RTN ----------------------
 * Satellite s has element columns elements[8][n], a covariance covariance[n][28] (the upper triangle, row by row, of a
 * 7 x 7 matrix P in the element fit's variables: the layout astroz_cuda_fit_observations returns; any positive
 * semi-definite P, not only a fit's) and model[s] (NULL: all 0), the variables P is stated in: 0 the near-earth set
 * (n, e cos w, e sin w, i, RAAN, M + w, B*), 1 the deep-space equinoctial set -- the fit's model output.  Query i of
 * satellite s ([offsets[s], offsets[s + 1]), offsets[0] = 0, offsets[n] = m) is at jd[i] + fr[i]:
 *   nominal:   the TEME state f(x) of the fit's model (SGP4 for model 0, SDP4 with the K2a lattice for model 1) at
 *              tsince = ((jd + fr) - epoch) * 1440, x the variables of the element columns;
 *   Jacobian:  J = df/dx (6 x 7) by the fit's forward differences: a step of 1e-8 in each variable (the backward step
 *              when the forward set cannot be built), divided by the step actually taken;
 *   B* held:   when P's B* row is all zero the B* set is not built or propagated and J's B* column is zero;
 *   frame:     ASTROZ_COV_FRAME_TEME, or ASTROZ_COV_FRAME_RTN of the nominal state: R = r / |r|, N = r x v / |r x v|,
 *              T = N x R.  The one rotation is applied to the position and the velocity blocks: there is no omega x r
 *              term, so the RTN velocity block is the TEME velocity covariance rotated, not that of a rotating frame;
 *   outputs:   state_covariance[m][21] the upper triangle, row by row, of Sigma = J P J^T [km^2, km^2/s, km^2/s^2];
 *              state[m][6] (nullable) the nominal TEME state [km, km/s]; jacobian[m][6][7] (nullable) J in the output
 *              frame; status[m] (ASTROZ_COV_*): INIT_FAILED when a set cannot be built under the row's model (model 0
 *              on a deep-space set, model 1 on a near-earth set, a stepped set that fails in both directions),
 *              CELL_FAILED when a deep-space cell of the nominal or a stepped set fails (decay, eccentricity).  A
 *              failed query is zero in every output; a zero P is not an error (zero Sigma, the state filled).
 *   deep space, B* free: SDP4's drag barely moves a deep-space orbit, so its B* column is rounding noise and a fit's
 *              B* variance is huge; Sigma is then dominated by their product.  Zero the B* row of P for such rows, or
 *              supply a B* variance of your own;
 * A query's bytes depend on its satellite's inputs and its own time alone: no sum runs across queries.
 * ASTROZ_VALUE_ERROR, nothing written: device = -1, an unknown grav or frame; and for the host call offsets that
 * decrease, offsets[0] != 0 or offsets[n] != m, a non-finite element, time or covariance word, a model byte > 1. */
#define ASTROZ_COV_OK          0
#define ASTROZ_COV_INIT_FAILED 1
#define ASTROZ_COV_CELL_FAILED 2
#define ASTROZ_COV_FRAME_TEME  0
#define ASTROZ_COV_FRAME_RTN   1
#define ASTROZ_STATE_COVARIANCE_WORDS 21
/* HOST buffers: one upload (pageable through a pinned ring, pinned by direct DMA), one launch per model, plain copies
 * back. */
int32_t astroz_cuda_propagate_covariance(const double *elements, uint32_t n, int32_t grav, const double *covariance,
                                         const uint8_t *model, const uint32_t *offsets, const double *jd,
                                         const double *fr, uint32_t m, int32_t frame, int32_t device, double *state,
                                         double *state_covariance, double *jacobian, uint8_t *status);
/* DEVICE pointers on `device`: two launches on `stream` (near-earth rows, then deep-space rows; one when d_model is
 * NULL), no allocation, no synchronisation; only the scalar arguments are checked. */
int32_t astroz_cuda_propagate_covariance_device(const double *d_elements, uint32_t n, int32_t grav,
                                                const double *d_covariance, const uint8_t *d_model,
                                                const uint32_t *d_offsets, const double *d_jd, const double *d_fr,
                                                uint32_t m, int32_t frame, int32_t device, double *d_state,
                                                double *d_state_covariance, double *d_jacobian, uint8_t *d_status,
                                                void *stream);
/* ---- conjunction assessment (K11): TCA, miss and 2-D Pc of candidate conjunctions from fitted covariances ------------
 * Candidates come from any screen, a conjunction message or the caller's own logic; nothing here finds them.  The
 * catalogue is K10's: elements[8][n], covariance[n][28] in the fit's variables and model[n] (NULL: all 0).  Candidate i
 * pairs rows primary[i] != secondary[i] around the guess time jd[i] + fr[i], with a half window window_min[i] > 0
 * [min] and a combined hard-body radius hbr_km[i] >= 0 [km]:
 *   states:    each row's nominal TEME state under its own model at dt minutes from the guess, tsince = ((jd + fr) -
 *              epoch) * 1440 + dt (K10's nominal at dt = 0); dr = r_s - r_p, dv = v_s - v_p;
 *   TCA:       a root of g = dr . dv where g goes from - to + in [-w, w], found by 32-point sampling rounds that cut the
 *              bracket 31x each until it is 1e-9 min wide, then one secant step.  Several roots in the first round's
 *              32 samples: the one of least |dr|.  No root: the window end with the smaller |dr|, status WINDOW_EDGE;
 *   Sigma:     each row's 6 x 6 state covariance at the TCA by K10's definition (forward-difference J, B* held when P's
 *              B* row is zero, a zero P gives a zero Sigma), in TEME or in that row's own RTN frame (frame);
 *   plane:     z = dv / |dv|, x = dr's part perpendicular to z, normalised (an exact hit takes x from the TEME axis
 *              least aligned with z), y = z x x.  C2 = the (x, y) block of Sigma_p + Sigma_s: the two objects'
 *              errors are assumed UNCORRELATED;
 *   Pc:        the short-encounter 2-D probability: the integral of N((u, v); (d, 0), C2) over the disk u^2 + v^2 <=
 *              R^2, d = |dr perpendicular to z|.  It assumes a straight-line relative motion over the encounter with
 *              constant covariance; for slow encounters (GEO pairs, co-orbiting objects) that assumption fails and
 *              Pc is not the collision probability.  Computed in C2's principal axes as a 1-D Gauss-Legendre
 *              integral of normal-CDF differences, with exact limits for a singular C2;
 *   outputs:   record[m][13]: dt_tca [min from jd + fr], miss [km], relative speed [km/s], dr and dv in the primary's
 *              RTN frame (6 words, no omega x r term), C2 (xx, xy, yy) [km^2], Pc; states[m][2][6] (nullable) the two
 *              TEME states at the TCA; state_covariance[m][2][21] (nullable) each row's Sigma words, as K10's;
 *              status[m] (ASTROZ_CONJ_*).  INIT_FAILED and CELL_FAILED mean what K10's do (and INIT_FAILED a model
 *              byte > 1 on the device call); every output is zero then and for BAD_PAIR (device call only: a row
 *              outside the catalogue, or primary == secondary).  WINDOW_EDGE and NO_PLANE (|dv| = 0: C2 and Pc zero)
 *              fill the other outputs.
 * A candidate's bytes depend on its own inputs and its two rows alone: no sum runs across candidates.
 * ASTROZ_VALUE_ERROR, nothing written: device = -1, an unknown grav or frame; and for the host call a row outside the
 * catalogue, primary == secondary, a half window <= 0, a radius < 0, a model byte > 1 or any non-finite input. */
#define ASTROZ_CONJ_OK           0
#define ASTROZ_CONJ_INIT_FAILED  1
#define ASTROZ_CONJ_CELL_FAILED  2
#define ASTROZ_CONJ_WINDOW_EDGE  3
#define ASTROZ_CONJ_NO_PLANE     4
#define ASTROZ_CONJ_BAD_PAIR     5
#define ASTROZ_CONJ_RECORD_WORDS 13
/* HOST buffers: one upload (pageable through a pinned ring, pinned by direct DMA), one launch per pair class, plain
 * copies back. */
int32_t astroz_cuda_conjunction(const double *elements, uint32_t n, int32_t grav, const double *covariance,
                                const uint8_t *model, const uint32_t *primary, const uint32_t *secondary,
                                const double *jd, const double *fr, const double *window_min, const double *hbr_km,
                                uint32_t m, int32_t frame, int32_t device, double *record, double *states,
                                double *state_covariance, uint8_t *status);
/* DEVICE pointers on `device`: two launches on `stream` (pairs of near-earth rows, then every other pair), no
 * allocation, no synchronisation; only the scalar arguments are checked. */
int32_t astroz_cuda_conjunction_device(const double *d_elements, uint32_t n, int32_t grav, const double *d_covariance,
                                       const uint8_t *d_model, const uint32_t *d_primary, const uint32_t *d_secondary,
                                       const double *d_jd, const double *d_fr, const double *d_window_min,
                                       const double *d_hbr_km, uint32_t m, int32_t frame, int32_t device,
                                       double *d_record, double *d_states, double *d_state_covariance,
                                       uint8_t *d_status, void *stream);
/* ---- Monte Carlo collision probability (K14): draws of both element sets from their covariances ---------------------
 * The catalogue and candidates are astroz_cuda_conjunction's; candidate i also has samples[i], first[i] (NULL: all 0)
 * and seed[i] (NULL: all 0).  For each row o:
 *   nominal:   x^ = the row's fit variables, over nvar = 7 or 6 (B* held when P's B* row is zero, as K10 and K11);
 *   factor:    S = D^-1/2 P D^-1/2 (D = diag P; a zero-variance variable has a zero row and column) factored S = L L^T
 *              by a semidefinite Cholesky: a pivot in [-1e-12, 1e-12] zeroes its column, one below -1e-12 or a
 *              negative variance is NOT_PSD;
 *   sample k:  x_k = x^ + D^1/2 L z, k in [first, first + samples), z from Philox4x32-10 under key (seed lo, seed hi):
 *              block j = 0 .. 6 of counter (j, k lo, k hi, 0) gives words (a, b, c, d), uniforms u1 = ((a 2^21 +
 *              (b >> 11)) + 0.5) 2^-53 and u2 likewise from (c, d), and Box-Muller normals 2j (r cos) and 2j + 1
 *              (r sin), r = sqrt(-2 ln u1), angle 2 pi u2.  Normals 0 .. 6 go to the primary's variables in order,
 *              7 .. 13 to the secondary's (the B* normal is drawn when B* is held).
 * Per sample: both drawn sets under their rows' models, astroz_cuda_conjunction's TCA search over [-w, w] on them and
 * the miss |dr| at that TCA.  A sample is FAILED when a drawn set cannot be built or a deep-space cell fails (it is
 * then neither a hit nor a miss), an EDGE when the search ends at a window end (still scored), a HIT when miss < R.
 * Pc = hits / (samples - failed).  The errors of the two objects are UNCORRELATED; no linear or short-encounter
 * assumption is made.
 * Outputs: counts[m][3] (hits, edge, failed); sample_out[m][record][2] (dt_tca [min from jd + fr], miss [km]) of
 * samples first .. first + record - 1, NaN for a failed sample, an index past samples[i] and every sample of a failed
 * candidate; status[m]: OK, INIT_FAILED (a nominal set cannot be built, or a model byte > 1 on the device call),
 * NOT_PSD, BAD_PAIR (device call only); counts of a candidate that is not OK are zero.
 * A sample's words depend on its candidate's inputs and its index k alone, and counts are integer sums: the bytes do
 * not depend on the batch, the order, the split of [first, first + samples) or the call form.  Counts over [0, 2N)
 * equal those over [0, N) plus those over [N, 2N): a run is extended by calling again with first = N.  Equal seeds
 * give equal draws; pass different seeds for independent estimates.
 * ASTROZ_VALUE_ERROR, nothing written: device = -1, an unknown grav; and for the host call every input check of
 * astroz_cuda_conjunction, first + samples above 2^64 - 1, record > 0 with a NULL sample_out. */
#define ASTROZ_CONJ_NOT_PSD              6
#define ASTROZ_CONJ_MC_COUNT_WORDS       3
#define ASTROZ_CONJ_MC_SAMPLE_WORDS      2
/* HOST buffers: one upload (pageable through a pinned ring, pinned by direct DMA), the launches, plain copies back. */
int32_t astroz_cuda_conjunction_mc(const double *elements, uint32_t n, int32_t grav, const double *covariance,
                                   const uint8_t *model, const uint32_t *primary, const uint32_t *secondary,
                                   const double *jd, const double *fr, const double *window_min, const double *hbr_km,
                                   const uint64_t *samples, const uint64_t *first, const uint64_t *seed, uint32_t m,
                                   uint32_t record, int32_t device, uint64_t *counts, double *sample_out,
                                   uint8_t *status);
/* DEVICE pointers on `device`: the launches on `stream`, no allocation, no synchronisation; only the scalar arguments
 * are checked (a bad pair gets BAD_PAIR).  d_scratch holds *bytes of astroz_cuda_conjunction_mc_scratch_bytes(m,
 * bytes), 16-byte aligned, for the work-item scan. */
int32_t astroz_cuda_conjunction_mc_device(const double *d_elements, uint32_t n, int32_t grav,
                                          const double *d_covariance, const uint8_t *d_model,
                                          const uint32_t *d_primary, const uint32_t *d_secondary, const double *d_jd,
                                          const double *d_fr, const double *d_window_min, const double *d_hbr_km,
                                          const uint64_t *d_samples, const uint64_t *d_first, const uint64_t *d_seed,
                                          uint32_t m, uint32_t record, int32_t device, uint64_t *d_counts,
                                          double *d_sample_out, uint8_t *d_status, void *d_scratch, void *stream);
/* The scratch of the device call for m candidates (the scan's size is the device's: ASTROZ_NO_DEVICE without one). */
int32_t astroz_cuda_conjunction_mc_scratch_bytes(uint32_t m, uint64_t *bytes);
/* ---- importance-sampled collision probability (K15): K14's draws shifted onto the collision point, weighted exactly --
 * The catalogue, candidates, samples, first, seed, factor, status rules and normals are astroz_cuda_conjunction_mc's.
 * u in R^14 are K14's normals of sample k (0 .. 6 the primary's, 7 .. 13 the secondary's) and c in R^14 the
 * candidate's shift:
 *   draw:      z = u + c, x_k = x^ + D^1/2 L z for each row; then K14's sets, TCA search, miss and FAILED / EDGE /
 *              HIT rules;
 *   weight:    log w_k = -u . c - |c|^2 / 2 = log phi(z) - log phi(z - c), exactly;
 *   estimate:  Pc = (1 / N) sum over hits of w_k, N = samples[i]: unbiased for P(hit) whatever the shift.  A FAILED
 *              draw counts as a non-hit, so where draws fail this estimates K14's hits / (N - failed) times
 *              (1 - P(failed));
 *   proposal:  shift NULL: LINEAR, from astroz_cuda_conjunction's assessment of the nominal pair (TEME): its TCA, plane
 *              (x, y) and in-plane miss d = (dr . x, dr . y).  J_o is row o's forward-difference Jacobian of its TEME
 *              position at the TCA (astroz_cuda_propagate_covariance's, B* held when P's B* row is zero), G = [-Pi J_p
 *              D_p^1/2 L_p | Pi J_s D_s^1/2 L_s] (2 x 14, Pi the projection on x, y) and c = -G^T C+ d, the least-norm
 *              shift with d + G c = 0 (C = G G^T, C+ by its 2 x 2 eigen-decomposition, an eigenvalue <= 1e-14 trace
 *              counting as zero); |c|^2 = d^T C+ d.  A nominal WINDOW_EDGE is still LINEAR.  PLAIN (c = 0, K14's
 *              draws): the nominal assessment is not OK or WINDOW_EDGE, a Jacobian cannot be formed, or C = 0.
 *              shift non-NULL: GIVEN, c = shift[i][14];
 *   sums:      each hit's v = exp(-u . c) and v^2 (v * v in fp64) rounded to multiples of 2^-128 and summed as unsigned
 *              256-bit integers (four u64 words, least significant first); a hit with v >= 2^31 enters neither sum
 *              and counts in overflow.  l0 = -|c|^2 / 2 is not accumulated: Pc = e^l0 V_hit 2^-128 / N.
 * Outputs: counts[m][12] (hits, edge, failed, overflow, V_hit[4], V2_hit[4]); proposal[m][15] (nullable: c, l0);
 * proposal_kind[m] (nullable: ASTROZ_CONJ_IS_*); sample_out[m][record][3] (dt_tca [min from jd + fr], miss [km], log
 * w) of samples first .. first + record - 1, NaN where K14's are; status[m] as K14's.  A candidate that is not OK has
 * zero counts and proposal words, PLAIN and NaN sample words.
 * The counts are integer sums: the bytes do not depend on the batch, the order, the split of [first, first + samples)
 * or the call form, and counts over [0, 2N) equal those over [0, N) plus those over [N, 2N).
 * ASTROZ_VALUE_ERROR, nothing written: every refusal of astroz_cuda_conjunction_mc, and a non-finite shift word. */
#define ASTROZ_CONJ_IS_COUNT_WORDS       12
#define ASTROZ_CONJ_IS_PROPOSAL_WORDS    15
#define ASTROZ_CONJ_IS_SAMPLE_WORDS      3
#define ASTROZ_CONJ_IS_LINEAR            0
#define ASTROZ_CONJ_IS_GIVEN             1
#define ASTROZ_CONJ_IS_PLAIN             2
/* HOST buffers: one upload (pageable through a pinned ring, pinned by direct DMA), the launches, plain copies back. */
int32_t astroz_cuda_conjunction_is(const double *elements, uint32_t n, int32_t grav, const double *covariance,
                                   const uint8_t *model, const uint32_t *primary, const uint32_t *secondary,
                                   const double *jd, const double *fr, const double *window_min, const double *hbr_km,
                                   const uint64_t *samples, const uint64_t *first, const uint64_t *seed,
                                   const double *shift, uint32_t m, uint32_t record, int32_t device, uint64_t *counts,
                                   double *proposal, uint8_t *proposal_kind, double *sample_out, uint8_t *status);
/* DEVICE pointers on `device`: the launches on `stream`, no allocation, no synchronisation; only the scalar arguments
 * are checked (a bad pair gets BAD_PAIR).  d_scratch holds *bytes of astroz_cuda_conjunction_is_scratch_bytes(m,
 * bytes), 16-byte aligned: the work-item scan and the nominal assessment of linear shifts. */
int32_t astroz_cuda_conjunction_is_device(const double *d_elements, uint32_t n, int32_t grav,
                                          const double *d_covariance, const uint8_t *d_model,
                                          const uint32_t *d_primary, const uint32_t *d_secondary, const double *d_jd,
                                          const double *d_fr, const double *d_window_min, const double *d_hbr_km,
                                          const uint64_t *d_samples, const uint64_t *d_first, const uint64_t *d_seed,
                                          const double *d_shift, uint32_t m, uint32_t record, int32_t device,
                                          uint64_t *d_counts, double *d_proposal, uint8_t *d_proposal_kind,
                                          double *d_sample_out, uint8_t *d_status, void *d_scratch, void *stream);
/* The scratch of the device call for m candidates (the scan's size is the device's: ASTROZ_NO_DEVICE without one). */
int32_t astroz_cuda_conjunction_is_scratch_bytes(uint32_t m, uint64_t *bytes);
/* ---- collision-avoidance manoeuvre trials (K16): burn the primary, refit it, carry its covariance, reassess -----------
 * The catalogue and candidates are astroz_cuda_conjunction's.  The PRIMARY of a candidate is the object that burns: to
 * plan a burn of the other object, swap the two.  Trial k takes candidate[k] < m, a burn time burn_jd[k] + burn_fr[k],
 * an impulsive dv_rtn[k][3] [km/s] in the primary's RTN frame at the burn (R = r / |r|, N = r x v / |r x v|, T = N x R)
 * and dv_sigma[k][3] (NULL: all 0), the 1-sigma execution error per RTN axis [km/s] (independent axes, uncorrelated with
 * the orbit error).  Per trial:
 *   burn:       ts_b = ((burn_jd + burn_fr) - epoch) * 1440, formed as astroz_cuda_propagate_covariance forms tsince,
 *               must come before the window: ts_b <= ts0 - w (ts0 the candidate's guess tsince, w its half window).
 *               x(t_b) and J (6 x 7, TEME) are astroz_cuda_propagate_covariance's nominal and Jacobian of the primary's
 *               row at t_b (B* held when P's B* row is zero); the post-burn state is x(t_b) + [0; R dv];
 *   conversion: the element fit (astroz_cuda_fit_elements_mixed's kernels, no other least squares) from the primary's
 *               own set to the one TEME state at t_b, B* held at the primary's B*, pos_sigma 1 km, vel_sigma 1e-3
 *               km/s, at most 50 iterations; the class follows the primary's set.  THE EPOCH STAYS THE PRIMARY'S
 *               EPOCH: the new set meets the post-burn state at t_b and shares the nominal's drag history, where a set
 *               re-epoched at the burn would restart SGP4's drag terms there and drift from the nominal even for a zero
 *               burn.  CONVERSION_FAILED: the fit does not converge, its residuals exceed 1e-6 km / 1e-9 km/s, or the
 *               new set cannot be built or propagated under the primary's model byte (a burn that moves the period
 *               across 225 min);
 *   zero burn:  dv = (0, 0, 0): the new row is the primary's set, copied (no fit), so with dv_sigma zero the trial's
 *               record is astroz_cuda_conjunction's record of the nominal pair bit for bit;
 *   covariance: J' = the Jacobian of the new set at t_b (same routine), J'6 its six orbital columns.  A (7 x 7): rows
 *               0-5 J'6^-1 (J - J'(:, B*) e_B*^T), row 6 e_B*^T (B* carried over, a held B* stays held).  P' = A P A^T
 *               + [J'6^-1 [0 0; 0 R diag(sigma^2) R^T] J'6^-T, 0; 0, 0].  J'6^-1 by LU with partial pivoting on J'6
 *               equilibrated by rows, then columns, to a largest |entry| of 1: a pivot |u| <= 1e-12 is singular
 *               (CONVERSION_FAILED);
 *   reassess:   astroz_cuda_conjunction (TEME) on the pair (new row with P' and the primary's model byte, the
 *               secondary's row) with the candidate's guess, window and radius.
 * THE RETURNED ROW IS AN ORDINARY CATALOGUE ROW: appended to the catalogue (elements, P', the primary's model byte) it
 * gives the trial's record bit for bit from astroz_cuda_conjunction, and it feeds the Monte Carlo, importance-sampling,
 * pairs and screening calls unchanged, which is how a chosen burn is verified with K15 or the post-burn orbit screened.
 * Outputs: record[T][13] astroz_cuda_conjunction's record (dt_tca from the candidate's guess); elements[T][8] (nullable)
 * the new set; covariance[T][28] (nullable) P'; residual[T][2] (nullable) the conversion residuals [km, km/s], 0 for a
 * zero burn; status[T], the first that applies: BAD_TRIAL / BAD_PAIR (device call only: candidate index >= m, burn not
 * before the window / a bad row pair); INIT_FAILED (a model byte > 1 on the device call, or the primary's set cannot be
 * built at t_b) / CELL_FAILED (its deep-space cell fails at t_b); CONVERSION_FAILED; then astroz_cuda_conjunction's
 * statuses of the post-burn pair.  A trial that is not assessed (stopped before the reassessment, or INIT_FAILED /
 * CELL_FAILED of the post-burn pair in it) has every output zero.
 * Precision of P': J and J' are forward differences, and their B* columns are quantised at about ulp(|r|) / 1e-8 (1e-4
 * km per unit B* in LEO).  A's B* column is the difference of two such columns mapped through J'6^-1, so on a row with
 * B* free whose B* variance dwarfs its orbital ones, P''s phase (lambda) entries carry that noise: measured up to 0.21
 * of sqrt(P'_jj P'_kk) on fitted LEO rows (an along-track error of a few cm at the burn), the same size in any build.
 * Rows with B* held do not carry it.  The reassessment's C2 agrees between builds within 5e-3 of its trace.
 * Limits: impulsive burns of one object, one burn per trial; the errors of the two objects are uncorrelated.
 * A trial's bytes depend on its own inputs, its candidate and its two rows alone: not on the batch, its order or the
 * call form.
 * ASTROZ_VALUE_ERROR, nothing written: device = -1, an unknown grav, T >= 2^31; and for the host call every refusal of
 * astroz_cuda_conjunction, a candidate index >= m, a burn not before its window, a non-finite burn time, dv or sigma
 * word, a negative sigma. */
#define ASTROZ_CONJ_CONVERSION_FAILED  7
#define ASTROZ_CONJ_BAD_TRIAL          8
/* HOST buffers: one upload (pageable through a pinned ring, pinned by direct DMA), the launches, plain copies back. */
int32_t astroz_cuda_conjunction_maneuver(const double *elements, uint32_t n, int32_t grav, const double *covariance,
                                         const uint8_t *model, const uint32_t *primary, const uint32_t *secondary,
                                         const double *jd, const double *fr, const double *window_min,
                                         const double *hbr_km, uint32_t m, const uint32_t *candidate,
                                         const double *burn_jd, const double *burn_fr, const double *dv_rtn,
                                         const double *dv_sigma, uint32_t t, int32_t device, double *record,
                                         double *new_elements, double *new_covariance, double *residual,
                                         uint8_t *status);
/* DEVICE pointers on `device`: the launches on `stream`, no allocation, no synchronisation; only the scalar arguments
 * are checked (a bad candidate index or burn time gets BAD_TRIAL, a bad pair BAD_PAIR).  d_scratch holds *bytes of
 * astroz_cuda_conjunction_maneuver_scratch_bytes(t, bytes), 16-byte aligned. */
int32_t astroz_cuda_conjunction_maneuver_device(const double *d_elements, uint32_t n, int32_t grav,
                                                const double *d_covariance, const uint8_t *d_model,
                                                const uint32_t *d_primary, const uint32_t *d_secondary,
                                                const double *d_jd, const double *d_fr, const double *d_window_min,
                                                const double *d_hbr_km, uint32_t m, const uint32_t *d_candidate,
                                                const double *d_burn_jd, const double *d_burn_fr,
                                                const double *d_dv_rtn, const double *d_dv_sigma, uint32_t t,
                                                int32_t device, double *d_record, double *d_new_elements,
                                                double *d_new_covariance, double *d_residual, uint8_t *d_status,
                                                void *d_scratch, void *stream);
/* The scratch of the device call for t trials. */
int32_t astroz_cuda_conjunction_maneuver_scratch_bytes(uint32_t t, uint64_t *bytes);
/* ---- track correlation (K12): which catalogue rows predict a sensor track within their uncertainty ----------------------
 * The catalogue is K10's: elements[8][n], covariance[n][28] in the fit's variables (NULL: every P zero, a plain TLE
 * catalogue) and model[n] (NULL: all 0).  Track j is the observations [offsets[j], offsets[j + 1]) (offsets[0] = 0,
 * offsets[t] = m) in the layout of astroz_cuda_fit_observations: jd[i] + fr[i], kind[i], value[i][6], sigma[i][6],
 * station[i] into stations[k][3].  For each (track, row) pair, x the row's variables:
 *   sets:      the row's nominal and stepped sets as K10 builds them (B* held when P's B* row is zero); when P is all zero
 *              no stepped set is built or propagated;
 *   rows:      per observation, the weighted residual z and weighted Jacobian rows G of the element fit (azimuth and
 *              right ascension wrapped, scaled by the cosine of the observed elevation / declination), at K10's time;
 *   distance:  d2 = z^T (I + G P G^T)^-1 z over the track's stacked residuals, evaluated as |z|^2 - b^T (I + P N)^-1 P b
 *              with b = G^T z and N = G^T G summed in track order (a 7 x 7 solve, exact for any positive semi-definite
 *              P), clamped at 0.  For one observation it is r^T (H Sigma H^T + R)^-1 r; for a track it accounts for the
 *              element error its residuals share;
 *   gate:      the chi-square quantile of k degrees of freedom at gate_probability, k = used[j] the track's used scalar
 *              residuals (astroz_cuda_chi2_quantile);
 *   failure:   a deep-space cell that fails, or sums that are not finite: the pair is skipped and counted.
 * Outputs per track: rows[t][best] and d2[t][best] the best smallest (d2, row) over the evaluated pairs, by d2 and then
 * row index, in or out of the gate (empty slots 0xFFFFFFFF / +inf); used[t] = k; n_gate[t] the rows with d2 <= gate;
 * n_failed[t] the skipped pairs; status[t] (ASTROZ_CORR_*): OK at least one row in the gate, UNCORRELATED none,
 * NO_ROW no pair evaluated, BAD_TRACK (device call only) an empty track, k = 0 or more than ASTROZ_CORR_MAX_TRACK
 * observations (every other output of the track empty or zero).  Per row: row_status[n] ASTROZ_COV_OK, or
 * ASTROZ_COV_INIT_FAILED when its sets cannot be built under its model (or, device call only, its model byte is > 1):
 * such a row takes part in no pair.
 * A track's bytes depend on its own observations and the catalogue alone: not on other tracks, their order, the batch
 * split or the call form.  Every pair is scored: there is no pre-screen.
 * ASTROZ_VALUE_ERROR, nothing written: device = -1, an unknown grav, best outside [1, ASTROZ_CORR_MAX_BEST],
 * gate_probability outside (0, 1); and for the host call offsets that decrease or do not run from 0 to m, an empty
 * track, a track of more than ASTROZ_CORR_MAX_TRACK observations or with no used residual, every observation check of
 * astroz_cuda_fit_observations, a non-finite element, covariance word or time, a model byte > 1. */
#define ASTROZ_CORR_OK           0
#define ASTROZ_CORR_UNCORRELATED 1
#define ASTROZ_CORR_NO_ROW       2
#define ASTROZ_CORR_BAD_TRACK    3
#define ASTROZ_CORR_MAX_TRACK    256
#define ASTROZ_CORR_MAX_BEST     8
/* HOST buffers: one upload (pageable through a pinned ring, pinned by direct DMA), the launches, plain copies back. */
int32_t astroz_cuda_correlate(const double *elements, uint32_t n, int32_t grav, const double *covariance,
                              const uint8_t *model, const uint32_t *offsets, uint32_t t, const double *jd,
                              const double *fr, const uint8_t *kind, const double *value, const double *sigma,
                              const uint32_t *station, uint32_t m, const double *stations, uint32_t k,
                              double gate_probability, uint32_t best, int32_t device, uint32_t *rows, double *d2,
                              uint32_t *used, uint32_t *n_gate, uint32_t *n_failed, uint8_t *status,
                              uint8_t *row_status);
/* DEVICE pointers on `device`: the launches on `stream`, no allocation, no synchronisation; only the scalar arguments
 * are checked (kinds, stations and sigmas must be valid; a bad track gets BAD_TRACK).  d_scratch holds
 * *bytes of astroz_cuda_correlate_scratch_bytes(n, t, best, bytes), 8-byte aligned, for the row chunks' partial lists. */
int32_t astroz_cuda_correlate_device(const double *d_elements, uint32_t n, int32_t grav, const double *d_covariance,
                                     const uint8_t *d_model, const uint32_t *d_offsets, uint32_t t, const double *d_jd,
                                     const double *d_fr, const uint8_t *d_kind, const double *d_value,
                                     const double *d_sigma, const uint32_t *d_station, const double *d_stations,
                                     double gate_probability, uint32_t best, int32_t device, void *d_scratch,
                                     uint32_t *d_rows, double *d_d2, uint32_t *d_used, uint32_t *d_n_gate,
                                     uint32_t *d_n_failed, uint8_t *d_status, uint8_t *d_row_status, void *stream);
int32_t astroz_cuda_correlate_scratch_bytes(uint32_t n, uint32_t t, uint32_t best, uint64_t *bytes);
/* The gate: the quantile x of the chi-square distribution of k >= 1 degrees of freedom at probability p in (0, 1), by
 * the function the kernels evaluate.  ASTROZ_VALUE_ERROR for k = 0 or p outside (0, 1). */
int32_t astroz_cuda_chi2_quantile(uint32_t k, double p, double *x);
/* ---- sensor tasking (K18): which catalogue row each sensor should observe at each slot --------------------------------
 * New capability: the reference has no tasking, so these calls replace nothing in it.
 * The catalogue is K10's: elements[8][n], covariance[n][28] in the fit's variables (NULL: every P zero) and model[n]
 * (NULL: all 0).  Sensor k of s (1 <= s <= ASTROZ_TASK_MAX_SENSORS) is kind[k] (ASTROZ_OBS_RADAR or ASTROZ_OBS_OPTICAL),
 * station[k] into stations[K][3] (lat deg, lon deg, h km on WGS84), sigma[k][4] (radar range km / azimuth rad /
 * elevation rad / range-rate km/s, optical RA / Dec rad; +inf: not measured) and limits[k][4], indexed by
 * ASTROZ_TASK_LIMIT_*: the minimum elevation (rad), the maximum range (km, +inf allowed), the maximum Sun elevation at
 * the station (rad) and the minimum solar exclusion angle (rad), the last two for optical sensors only.  Slots are
 * jd[t] + fr[t] (non-decreasing); sun[t][3] is the Sun's direction in TEME at each slot, of any length (required when a
 * sensor is optical).  For each cell (row, sensor, slot), at K10's time:
 *   visible:   the radar elevation of the nominal state above the station's geodetic horizon >= the minimum and the
 *              range <= the maximum (no refraction); optical sensors also need the object sunlit under a cylindrical
 *              shadow of radius 6378.137 km, the Sun's elevation at the station <= its limit and the angle between the
 *              line of sight and the Sun >= the exclusion angle;
 *   rows:      the predicted measurement h, and the weighted Jacobian rows G of the element fit with h as the
 *              observation (azimuth / RA scaled by the cosine of the predicted elevation / declination), from the
 *              row's nominal and stepped sets as K10 builds them (stepped sets propagated only where a sensor sees it);
 *   gain:      g = 1/2 log det(I + G P G^T) nats, the information of one observation about the row's variables, formed
 *              as 1/2 log det(I + L^T G^T G L) with P = L L^T (K12's semi-definite Cholesky): 0 exactly when P = 0;
 *   spread:    sqrt((G P G^T)_cc) sigma_c, the predicted 1-sigma of each measured component (azimuth / RA as an arc);
 *   failure:   a deep-space cell that fails (decay, eccentricity) is not visible and is counted.
 * Schedule: slot by slot, sensor k = 0 .. s-1 takes the row of largest g (then lowest row index) among the rows visible
 * to it with g > gain_min not taken by a lower sensor in the slot, or idles; each taken row's covariance becomes the
 * Kalman posterior of that one observation, P+ = L (I + L^T G^T G L)^-1 L^T (symmetric, 28 words), before the next
 * slot.  The elements are not changed; a held B* row stays zero.
 * Outputs per (sensor, slot): task_row[s][t] (0xFFFFFFFF idle), task_gain[s][t], task_value[s][t][4] the pointing (the
 * prediction h), task_spread[s][t][4], n_candidates[s][t] the rows that qualified when the sensor chose (idle: the
 * gain, value and spread are 0).  Per row: posterior[n][28], n_tasks[n], n_visible[n] the visible (sensor, slot)
 * cells, n_failed[n] the failed cells, row_status[n] ASTROZ_COV_OK or ASTROZ_COV_INIT_FAILED (such a row takes part in
 * nothing).  No byte depends on the launch shape or the call form.
 * ASTROZ_VALUE_ERROR, nothing written: device = -1, an unknown grav, s = 0 or s > ASTROZ_TASK_MAX_SENSORS, t = 0,
 * gain_min negative or not finite; and for the host call an unknown sensor kind, a station index >= K, a sigma that is
 * not positive or a sensor with no used component, a minimum elevation or maximum Sun elevation outside [-pi/2, pi/2],
 * a maximum range not > 0, an exclusion angle outside [0, pi], non-finite or decreasing slot times, sun NULL with an
 * optical sensor or a Sun row that is zero or not finite, a non-finite element or covariance word, a model byte > 1. */
#define ASTROZ_TASK_MAX_SENSORS       32
#define ASTROZ_TASK_LIMIT_EL_MIN      0
#define ASTROZ_TASK_LIMIT_RANGE_MAX   1
#define ASTROZ_TASK_LIMIT_SUN_EL_MAX  2
#define ASTROZ_TASK_LIMIT_EXCLUSION   3
/* HOST buffers: one upload (pageable through a pinned ring, pinned by direct DMA), the launches, plain copies back. */
int32_t astroz_cuda_tasking(const double *elements, uint32_t n, int32_t grav, const double *covariance,
                            const uint8_t *model, const uint8_t *kind, const uint32_t *station, const double *sigma,
                            const double *limits, uint32_t s, const double *stations, uint32_t k, const double *jd,
                            const double *fr, uint32_t t, const double *sun, double gain_min, int32_t device,
                            uint32_t *task_row, double *task_gain, double *task_value, double *task_spread,
                            uint32_t *n_candidates, double *posterior, uint32_t *n_tasks, uint32_t *n_visible,
                            uint32_t *n_failed, uint8_t *row_status);
/* DEVICE pointers on `device`: one build launch, then two launches per slot (three with model given) on `stream`, no
 * allocation, no synchronisation; only the scalar arguments are checked (sensors, slots and Sun rows must be valid).
 * d_scratch holds *bytes of astroz_cuda_tasking_scratch_bytes(n, s, bytes), 16-byte aligned. */
int32_t astroz_cuda_tasking_device(const double *d_elements, uint32_t n, int32_t grav, const double *d_covariance,
                                   const uint8_t *d_model, const uint8_t *d_kind, const uint32_t *d_station,
                                   const double *d_sigma, const double *d_limits, uint32_t s, const double *d_stations,
                                   const double *d_jd, const double *d_fr, uint32_t t, const double *d_sun,
                                   double gain_min, int32_t device, void *d_scratch, uint32_t *d_task_row,
                                   double *d_task_gain, double *d_task_value, double *d_task_spread,
                                   uint32_t *d_n_candidates, double *d_posterior, uint32_t *d_n_tasks,
                                   uint32_t *d_n_visible, uint32_t *d_n_failed, uint8_t *d_row_status, void *stream);
int32_t astroz_cuda_tasking_scratch_bytes(uint32_t n, uint32_t s, uint64_t *bytes);
/* ---- initial orbits (K13): an element set for a track no catalogue row predicts ---------------------------------------
 * New capability: the reference has no initial orbit determination, so these calls replace nothing in it.
 * Track j is the observations [offsets[j], offsets[j + 1]) in the layout of astroz_cuda_correlate, in time order (the
 * host call sorts each track stably by jd + fr; the device call reports a track out of order as BAD_TRACK).  Its epoch
 * is the time of its middle observation, index floor(m_j / 2).  mu is the gravity model's (grav).
 *   geometry:   the inverses of the measurement model: TEME and ECEF states give a TEME state, radar range / azimuth /
 *               elevation a TEME position (range-rate is scored only), optical angles a TEME line of sight from the
 *               station.  A method builds only from observations whose geometry components are all used: a TEME or
 *               ECEF state without its velocity, for one, builds nothing (it is scored only), so a track of such
 *               states alone is TOO_FEW;
 *   candidates: every state observation; with >= 3 radar positions a Gibbs and a Herrick-Gibbs velocity for the middle
 *               of every triplet of a fixed table of up to 30 (first, middle, last always among them); with exactly 2,
 *               the zero-revolution Lambert transfer for the normals +z and -z; with >= 3 optical observations Gauss'
 *               method on every triplet with |L1 . (L2 x L3)| >= 1e-12, every real root above 1 earth radius of its
 *               8th-degree polynomial refined by universal-variable f and g (Curtis, Algorithm 5.6).  A candidate that
 *               is not finite, has e >= 1 or a perigee radius below 1 earth radius is rejected;
 *   score:      each candidate propagated two-body to every observation of the track and scored by the element fit's
 *               residual rules: F = sum of squared weighted residuals.  The least (F, method, triplet, root) wins;
 *   conversion: the winner two-body at the epoch -> osculating elements (n in rev/day, B* = bstar[j], 0 when bstar is
 *               NULL) -> astroz_cuda_fit_elements_mixed's own fit to that one TEME state at the epoch with B* held.
 * Outputs per track: elements[8][t] the converted set (epoch = the track's epoch), state[t][6] the TEME state at the
 * epoch, wrms[t] = sqrt(F / used residuals), method[t] (ASTROZ_IOD_METHOD_*), candidates[t] the candidates scored,
 * conv[t][2] the converted set's |dr| [km] and |dv| [km/s] from the state at the epoch, deep_space[t] 1 when the set
 * is an SDP4 (period > 225 min) set, status[t] (ASTROZ_IOD_*): OK; TOO_FEW fewer usable observations than any method
 * needs (1 state, 2 radar, 3 optical); NO_CANDIDATE every candidate rejected; CONVERSION_FAILED the fit did not
 * converge or left |dr| > 1e-6 km or |dv| > 1e-9 km/s (the outputs are kept); BAD_TRACK (device call only) an empty
 * track, more than ASTROZ_IOD_MAX_TRACK observations, no used residual or out of time order.  Except for
 * CONVERSION_FAILED, a track that is not OK has zero elements, state, wrms and conv and method NONE.
 * A track's bytes depend on that track alone: not on other tracks, their order, the batch split or the call form.
 * ASTROZ_VALUE_ERROR, nothing written: device = -1, an unknown grav; and for the host call offsets that decrease or do
 * not run from 0 to m, an empty track, a track longer than ASTROZ_IOD_MAX_TRACK or with no used residual, every
 * observation check of astroz_cuda_fit_observations, a non-finite bstar. */
#define ASTROZ_IOD_OK                0
#define ASTROZ_IOD_TOO_FEW           1
#define ASTROZ_IOD_NO_CANDIDATE      2
#define ASTROZ_IOD_CONVERSION_FAILED 3
#define ASTROZ_IOD_BAD_TRACK         4
#define ASTROZ_IOD_MAX_TRACK         256
#define ASTROZ_IOD_METHOD_STATE         0
#define ASTROZ_IOD_METHOD_GIBBS         1
#define ASTROZ_IOD_METHOD_HERRICK_GIBBS 2
#define ASTROZ_IOD_METHOD_LAMBERT       3
#define ASTROZ_IOD_METHOD_GAUSS         4
#define ASTROZ_IOD_METHOD_NONE          255
/* HOST buffers: each track's observations are first sorted into host staging, which goes up through the pinned ring
 * whether the caller's arrays are pinned or not; then the launches and plain copies back. */
int32_t astroz_cuda_initial_orbits(const uint32_t *offsets, uint32_t t, const double *jd, const double *fr,
                                   const uint8_t *kind, const double *value, const double *sigma,
                                   const uint32_t *station, uint32_t m, const double *stations, uint32_t k,
                                   const double *bstar, int32_t grav, int32_t device, double *elements, double *state,
                                   double *wrms, uint8_t *method, uint32_t *candidates, double *conv,
                                   uint8_t *deep_space, uint8_t *status);
/* DEVICE pointers on `device`: four launches on `stream` (the IOD kernel, the near-earth and deep-space conversion fits,
 * the finishing kernel), no allocation, no synchronisation; only the scalar arguments are checked (kinds, stations and
 * sigmas must be valid; a bad track gets BAD_TRACK).  d_scratch holds *bytes of
 * astroz_cuda_initial_orbits_scratch_bytes(t, bytes), 8-byte aligned. */
int32_t astroz_cuda_initial_orbits_device(const uint32_t *d_offsets, uint32_t t, const double *d_jd,
                                          const double *d_fr, const uint8_t *d_kind, const double *d_value,
                                          const double *d_sigma, const uint32_t *d_station, const double *d_stations,
                                          const double *d_bstar, int32_t grav, int32_t device, void *d_scratch,
                                          double *d_elements, double *d_state, double *d_wrms, uint8_t *d_method,
                                          uint32_t *d_candidates, double *d_conv, uint8_t *d_deep_space,
                                          uint8_t *d_status, void *stream);
int32_t astroz_cuda_initial_orbits_scratch_bytes(uint32_t t, uint64_t *bytes);

/* ---- track linking (K17): an element set from two tracks of one unknown object ---------------------------------------
 * New capability: the reference has no track linking, so these calls replace nothing in it.
 * Tracks as in astroz_cuda_initial_orbits; pairs[p][2] the track pairs to test.
 *   anchor:     a track's middle observation among those that give a line of sight with every component used (both
 *               optical angles; radar range, azimuth and elevation; the position of a TEME or ECEF state, from the
 *               geocentre): a TEME origin R, unit vector L and range, known except for optical observations;
 *   pair:       the track with the earlier anchor is track 1, so (a, b) and (b, a) give the same bytes; the epoch is
 *               track 2's anchor time;
 *   hypotheses: a known range is one; an unknown one ASTROZ_LINK_RANGES geometric points from the root of
 *               |R + rho L| = r_min to the root of |R + rho L| = r_max (km; r_min above every station's radius);
 *   transfers:  every (rho1, rho2) and normal +z, -z: Lambert (astroz_cuda_lambert's solver, 0 .. max_revs
 *               revolutions, both branches) from R1 + rho1 L1 to R2 + rho2 L2, the state (r2, v2) at the epoch kept
 *               when finite with e < 1 and perigee >= 1 earth radius;
 *   score:      each state two-body against the first, anchor and last observation of each track (F_probe, the
 *               element fit's residual rules); the ASTROZ_LINK_SEEDS least are refined by Levenberg-Marquardt on their
 *               unknown ranges (revolutions, direction and branch fixed) over every observation of both tracks; the
 *               least F wins;
 *   conversion: astroz_cuda_initial_orbits' (the epoch state -> osculating elements, B* = bstar[p] or 0 -> the mixed
 *               element fit to that one state, B* held) and its thresholds.
 * Outputs per pair: elements[8][p], state[p][6] at the epoch, rho[p][2] the winner's ranges (track 1 first), revs[p],
 * flags[p] (ASTROZ_LINK_RETROGRADE: normal -z; ASTROZ_LINK_RIGHT_BRANCH), wrms[p] = sqrt(F / used), used[p] the used
 * residuals of both tracks, hypotheses[p] the admissible states scored, conv[p][2], deep_space[p], status[p]
 * (ASTROZ_LINK_*): OK; TOO_FEW a track without an anchor; NO_CANDIDATE no admissible state; CONVERSION_FAILED as for
 * initial orbits (outputs kept); BAD_TRACK (device call only) as for initial orbits; BAD_PAIR (device call only) a
 * pair index >= t, a == b, or equal anchor times.  Except for CONVERSION_FAILED a pair that is not OK has zero
 * elements, state, rho, revs, flags, wrms and conv; used and hypotheses are zero unless the pair was scored.
 * A pair's bytes depend on its two tracks alone: not on other pairs, their order, the batch split or the call form.
 * ASTROZ_VALUE_ERROR, nothing written: device = -1, an unknown grav, max_revs > ASTROZ_LAMBERT_MAX_REVS, r_min not
 * finite or <= 0, r_max not finite or <= r_min; and for the host call every refusal of astroz_cuda_initial_orbits
 * (bstar now per pair), a pair index >= t, a == b, equal anchor times and r_min <= the largest station radius. */
#define ASTROZ_LINK_OK                0
#define ASTROZ_LINK_TOO_FEW           1
#define ASTROZ_LINK_NO_CANDIDATE      2
#define ASTROZ_LINK_CONVERSION_FAILED 3
#define ASTROZ_LINK_BAD_TRACK         4
#define ASTROZ_LINK_BAD_PAIR          5
#define ASTROZ_LINK_RETROGRADE        1
#define ASTROZ_LINK_RIGHT_BRANCH      2
#define ASTROZ_LINK_RANGES            32
#define ASTROZ_LINK_SEEDS             4
/* HOST buffers: each track's observations are first sorted into host staging, as for astroz_cuda_initial_orbits. */
int32_t astroz_cuda_link_tracks(const uint32_t *offsets, uint32_t t, const double *jd, const double *fr,
                                const uint8_t *kind, const double *value, const double *sigma, const uint32_t *station,
                                uint32_t m, const double *stations, uint32_t k, const uint32_t *pairs, uint32_t p,
                                const double *bstar, double r_min, double r_max, uint32_t max_revs, int32_t grav,
                                int32_t device, double *elements, double *state, double *rho, uint8_t *revs,
                                uint8_t *flags, double *wrms, uint32_t *used, uint32_t *hypotheses, double *conv,
                                uint8_t *deep_space, uint8_t *status);
/* DEVICE pointers on `device`: four launches on `stream` (the link kernel, the two conversion fits, the finishing
 * kernel), no allocation, no synchronisation; only the scalar arguments are checked.  d_scratch holds *bytes of
 * astroz_cuda_link_tracks_scratch_bytes(p, bytes), 8-byte aligned. */
int32_t astroz_cuda_link_tracks_device(const uint32_t *d_offsets, uint32_t t, const double *d_jd, const double *d_fr,
                                       const uint8_t *d_kind, const double *d_value, const double *d_sigma,
                                       const uint32_t *d_station, const double *d_stations, const uint32_t *d_pairs,
                                       uint32_t p, const double *d_bstar, double r_min, double r_max,
                                       uint32_t max_revs, int32_t grav, int32_t device, void *d_scratch,
                                       double *d_elements, double *d_state, double *d_rho, uint8_t *d_revs,
                                       uint8_t *d_flags, double *d_wrms, uint32_t *d_used, uint32_t *d_hypotheses,
                                       double *d_conv, uint8_t *d_deep_space, uint8_t *d_status, void *stream);
int32_t astroz_cuda_link_tracks_scratch_bytes(uint32_t p, uint64_t *bytes);

/* One TLE line pair read by the library's own parser (src/Tle.zig:49-101) into the eight element columns above, the
 * numbers astroz_cuda_constellation_create would use.  ASTROZ_BAD_TLE_LENGTH when the pair cannot be read. */
int32_t astroz_cuda_parse_tle(const char *line1, const char *line2, double *elements);

/* ---- Lambert transfers (K9): replaces astroz.lambert(mu, r1, r2, tof) (bindings/python/src/orbital_mechanics.zig:37-97,
 * src/OrbitalMechanics.zig:122-183) with a batched multi-revolution solver.  The reference's lambertSolverSimple does not
 * solve Lambert's problem (its departure velocity, propagated for tof, misses r2: SURVEY.md appendix C); these calls
 * return the true solutions, by Izzo's algorithm (Celest. Mech. Dyn. Astron. 121, 2015).
 * Problem i: positions r1[i], r2[i] [km], time of flight tof[i] [s], gravitational parameter mu [km^3/s^2] and a unit
 * normal normal[i] (nullable: +z for every problem) that sets the sense of motion:
 *   direction: ih = r1 x r2 / |r1 x r2|; ih . n > 0 is the short way (transfer angle < pi), ih . n < 0 the long way.  A
 *              retrograde transfer is a negated normal;
 *   slots:     S = 2 max_revs + 1 per problem: slot 0 is the zero-revolution solution, slot 2M - 1 the left and slot 2M
 *              the right branch of M revolutions.  A slot of M revolutions exists when tof >= its minimum time of flight;
 *   numerics:  Householder iterations on Izzo's x until |dx| < 1e-13, at most 15; the minimum time of flight by Halley
 *              iterations, for the largest candidate M only;
 *   outputs:   v1[n][S][3], v2[n][S][3] [km/s], status[n][S] (ASTROZ_LAMBERT_*), iterations[n][S] (nullable: Householder
 *              steps taken, 15 for NOT_CONVERGED, 0 when no iteration ran).  A slot that is not OK is zero-filled.
 * A problem's bytes depend on its own inputs alone, never on its position in a batch.
 * ASTROZ_VALUE_ERROR, nothing written: mu not finite or <= 0; max_revs > 127 (slot indices stay inside a byte); device
 * = -1 or not a visible ordinal; an output size that overflows; and for the host call a non-finite r1, r2, tof or normal.
 * n = 0 is a no-op.  Without a device: ASTROZ_NO_DEVICE. */
#define ASTROZ_LAMBERT_OK            0
#define ASTROZ_LAMBERT_NO_SOLUTION   1   /* tof <= 0, or no M-revolution solution at this tof */
#define ASTROZ_LAMBERT_DEGENERATE    2   /* |r1| = 0, |r2| = 0, |r1 x r2| < 1e-12 |r1| |r2| (the reference's |sin dnu|
                                            < 1e-12 rule, OrbitalMechanics.zig:158) or ih . n = 0 */
#define ASTROZ_LAMBERT_NOT_CONVERGED 3   /* 15 Householder steps without |dx| < 1e-13 */
#define ASTROZ_LAMBERT_STATE_FAILED  4   /* porkchop only: an endpoint's propagation status was not 0 */
#define ASTROZ_LAMBERT_MAX_REVS      127

/* HOST buffers: r1[n][3], r2[n][3], tof[n], normal[n][3] (nullable), outputs as above.  Compute-bound: the inputs go up
 * at once (pageable ones through a pinned ring), one launch solves the batch, the results come back by plain copies. */
int32_t astroz_cuda_lambert(const double *r1, const double *r2, const double *tof, const double *normal, uint32_t n,
                            double mu, uint32_t max_revs, int32_t device, double *v1, double *v2, uint8_t *status,
                            uint8_t *iterations);
/* Same with DEVICE pointers on `device`.  One launch on `stream` (a cudaStream_t, NULL = the legacy default stream): no
 * allocation, no synchronisation, and only the scalar arguments are checked -- the values must be finite. */
int32_t astroz_cuda_lambert_device(const double *d_r1, const double *d_r2, const double *d_tof, const double *d_normal,
                                   uint32_t n, double mu, uint32_t max_revs, int32_t device, double *d_v1,
                                   double *d_v2, uint8_t *d_status, uint8_t *d_iterations, void *stream);

/* Porkchop grids: the cost of transfers between n_pairs (chaser, target) pairs over a grid of departure and arrival
 * epochs.  Cell (p, d, a), arrival index fastest:
 *   endpoints: the chaser's state at departure d, d_dep[p][d][6] (x y z vx vy vz, km and km/s), and the target's at
 *              arrival a, d_arr[p][a][6], each with a status byte (d_dep_status[p][d], d_arr_status[p][a], nullable: all
 *              valid).  States may come from anywhere: propagate_pairs_device, K7 trajectories, ephemerides.  TEME (or
 *              any frame) is treated as inertial over the transfer;
 *   time:      tof = ((arr_jd[a] - dep_jd[d]) + (arr_fr[a] - dep_fr[d])) * 86400, evaluated in that order;
 *   direction: prograde relative to the chaser: the normal is the chaser's r x v at departure;
 *   selection: every feasible slot of max_revs revolutions is solved and the one with the least
 *              |v1 - v_chaser| + |v_target - v2| kept, the lowest slot on a tie;
 *   outputs:   d_dv[p][d][a][2] (|dv1|, |dv2| km/s), d_slot[p][d][a] (the slot kept), d_status[p][d][a]: OK, or
 *              ASTROZ_LAMBERT_STATE_FAILED when an endpoint's status byte is not 0, or slot 0's status when no slot is
 *              OK (dv 0 and slot 0 then).
 * Asynchronous on `stream`; ASTROZ_VALUE_ERROR as for astroz_cuda_lambert_device, and when n_pairs * n_dep * n_arr
 * overflows. */
int32_t astroz_cuda_lambert_porkchop_device(const double *d_dep, const uint8_t *d_dep_status, const double *d_arr,
                                            const uint8_t *d_arr_status, uint32_t n_pairs, const double *d_dep_jd,
                                            const double *d_dep_fr, uint32_t n_dep, const double *d_arr_jd,
                                            const double *d_arr_fr, uint32_t n_arr, double mu, uint32_t max_revs,
                                            int32_t device, double *d_dv, uint8_t *d_slot, uint8_t *d_status,
                                            void *stream);
/* The whole porkchop from a handle's catalogue, HOST buffers: pair p departs from catalog row chaser[p] and arrives at
 * catalog row target[p].  The pairs are cut into chunks on the handle's two-slot pipeline; for each chunk the handle's
 * pairs path (astroz_cuda_constellation_propagate_pairs, TEME, its status bytes) gives the chaser rows x departures
 * and the target rows x arrivals, then the porkchop kernel above runs on them.  dv[n_pairs][n_dep][n_arr][2],
 * slot / status[n_pairs][n_dep][n_arr].
 * ASTROZ_VALUE_ERROR, nothing written: a row outside the catalog; a multi-device handle (device = -1); mu not finite or
 * <= 0; max_revs > 127; a non-finite epoch; an output size that overflows.  n_pairs, n_dep or n_arr = 0 is a no-op. */
int32_t astroz_cuda_constellation_porkchop(astroz_constellation_t h, const uint32_t *chaser, const uint32_t *target,
                                           uint32_t n_pairs, const double *dep_jd, const double *dep_fr, uint32_t n_dep,
                                           const double *arr_jd, const double *arr_fr, uint32_t n_arr, double mu,
                                           uint32_t max_revs, double *dv, uint8_t *slot, uint8_t *status);

/* ---- reentry prediction (K19): catalogue rows and their covariance draws carried down to the interface -------------
 * Request i names catalogue row rows[i] (element columns, covariance words, model byte, as astroz_cuda_conjunction_mc)
 * with samples[i], first[i] (NULL: all 0) and seed[i] (NULL: all 0).  A trajectory starts at the row's epoch from the
 * TEME state (tsince 0) of a set built under the row's model with grav: the row's own set for the NOMINAL, a drawn set
 * for SAMPLE k.  It is integrated by astroz_cuda_propagate_numerical's Dormand-Prince 8(7) (rtol 1e-9, atol 1e-12,
 * its step control and stop rules) over intervals of step_s seconds until the first crossing of the interface height
 * h_i [km] or horizon_days after epoch.
 *   force:     two-body + the textbook J2 acceleration (mu, equatorial radius and J2 of grav), and drag quadratic in the
 *              speed relative to a co-rotating atmosphere: a = -1/2 B f rho(h) |v_rel| v_rel 1e3 km/s^2, v_rel = v -
 *              w x r, w = 7.292115e-5 rad/s about TEME z.  h is the WGS-84 geodetic height of the TEME position (the
 *              height of the ECEF output mode's conversion; no GMST is needed for it).  rho(h) = density_scale x the
 *              piecewise-exponential atmosphere of Vallado, Fundamentals of Astrodynamics and Applications, Table 8-4:
 *              rho0 exp(-(h - h0) / H) in the band with the largest h0 <= h, the last band above 1000 km.  None of the
 *              numerical propagator's own force models is used or changed;
 *   B:         B_row = ballistic[i] [m^2/kg], or 12.741621 B* when ballistic is NULL (B* = B rho0 / 2, rho0 =
 *              0.15696615 kg m^-2 ER^-1).  A sample's B_k = B_row + 12.741621 (B*_k - B*_row) (B_row when B* is held).
 *              B <= 0 or non-finite: the trajectory is NONPHYSICAL;
 *   draws:     astroz_cuda_conjunction_mc's factor and draws of the PRIMARY under the request's seed: sample k's set is
 *              that call's primary set of sample k.  Normal 7 (block 3's second normal) gives the density factor
 *              f_k = exp(density_sigma z_7); the nominal has f = 1 (the median density);
 *   crossing:  after each interval, the cubic Hermite of position over it from its end states.  A crossing when the
 *              end height is <= h_i, or when the radial velocity goes from - to + inside the interval and the
 *              Hermite's minimum height (golden-section search to 1e-9 of the interval) is <= h_i (a perigee dip).  The crossing time is the root of the
 *              Hermite's height - h_i, by bisection to 2^-30 of the interval; the state there is the Hermite and its
 *              derivative.  A start at or below h_i crosses at dt = 0.
 * Outputs: record[m][8] of the nominal (dt [min from epoch, +inf when still above at the horizon], geodetic latitude
 * and east longitude [deg] by the ECEF mode's GMST, inertial speed [km/s], inertial flight-path angle [deg], B used,
 * accepted and rejected DP87 attempts; NaN where not defined); states[m][6] (nullable: TEME state at the nominal
 * crossing, NaN unless REENTERED); nominal_status[m] (ASTROZ_REENTRY_TRAJ_*); counts[m][3] (reentered, above, failed:
 * INIT_FAILED, NONPHYSICAL or STOPPED samples); sample_out[m][record][4] (dt, latitude, longitude, attempts) of samples
 * first .. first + record - 1, NaN past samples[i] and for every sample of a request that is not OK; status[m]: OK,
 * INIT_FAILED (the row's set cannot be built, or a model byte > 1 on the device call), NOT_PSD, BAD_ROW (device call
 * only).  A request that is not OK runs nothing: its counts are zero and its nominal is INIT_FAILED.
 * A sample's words depend on its row's inputs, the call's scalars, the seed and k alone, and counts are integer sums:
 * the bytes do not depend on the batch, the order, the split of [first, first + samples) or the call form.
 * Lunisolar and higher zonal terms are not modelled: transfer-orbit predictions are indicative only.
 * ASTROZ_VALUE_ERROR, nothing written: device = -1, an unknown grav, h_i outside [60, 200] km, horizon_days outside
 * (0, 3660], step_s outside [1, 3600], density_sigma outside [0, 2], density_scale <= 0 or non-finite; and for the host
 * call a row outside the catalogue, non-finite elements or covariance words, a model byte > 1, a non-finite ballistic,
 * first + samples above 2^64 - 1, record > 0 with a NULL sample_out. */
#define ASTROZ_REENTRY_RECORD_WORDS        8
#define ASTROZ_REENTRY_SAMPLE_WORDS        4
#define ASTROZ_REENTRY_COUNT_WORDS         3
#define ASTROZ_REENTRY_STATE_WORDS         6
#define ASTROZ_REENTRY_OK                  0
#define ASTROZ_REENTRY_INIT_FAILED         1
#define ASTROZ_REENTRY_NOT_PSD             2
#define ASTROZ_REENTRY_BAD_ROW             3
#define ASTROZ_REENTRY_TRAJ_REENTERED      0
#define ASTROZ_REENTRY_TRAJ_ABOVE          1
#define ASTROZ_REENTRY_TRAJ_INIT_FAILED    2   /* the set cannot be built, or its epoch state fails */
#define ASTROZ_REENTRY_TRAJ_NONPHYSICAL    3   /* B <= 0 or non-finite */
#define ASTROZ_REENTRY_TRAJ_STOPPED        4   /* the integrator's stop rule or substep limit, or a non-finite state */
/* HOST buffers: one upload (pageable through a pinned ring, pinned by direct DMA), the launches, plain copies back. */
int32_t astroz_cuda_reentry(const double *elements, uint32_t n, int32_t grav, const double *covariance,
                            const uint8_t *model, const uint32_t *rows, const double *ballistic, const uint64_t *samples,
                            const uint64_t *first, const uint64_t *seed, uint32_t m, double h_i, double horizon_days,
                            double step_s, double density_scale, double density_sigma, uint32_t record, int32_t device,
                            double *record_out, double *states, uint8_t *nominal_status, uint64_t *counts,
                            double *sample_out, uint8_t *status);
/* DEVICE pointers on `device`: the launches on `stream`, no allocation, no synchronisation; only the scalar arguments
 * are checked (a row outside the catalogue gets BAD_ROW).  d_scratch holds *bytes of
 * astroz_cuda_reentry_scratch_bytes(m, bytes), 256-byte aligned. */
int32_t astroz_cuda_reentry_device(const double *d_elements, uint32_t n, int32_t grav, const double *d_covariance,
                                   const uint8_t *d_model, const uint32_t *d_rows, const double *d_ballistic,
                                   const uint64_t *d_samples, const uint64_t *d_first, const uint64_t *d_seed,
                                   uint32_t m, double h_i, double horizon_days, double step_s, double density_scale,
                                   double density_sigma, uint32_t record, int32_t device, double *d_record_out,
                                   double *d_states, uint8_t *d_nominal_status, uint64_t *d_counts,
                                   double *d_sample_out, uint8_t *d_status, void *d_scratch, void *stream);
/* The scratch of the device call for m requests (the scan's size is the device's: ASTROZ_NO_DEVICE without one). */
int32_t astroz_cuda_reentry_scratch_bytes(uint32_t m, uint64_t *bytes);

/* ---- measurement helpers --------------------------------------------------------------------- */
/* DFMA microbenchmark on `device`: achieved fp64 TFLOP/s (FMA = 2) -- the measured roofline denominator */
int32_t astroz_cuda_fp64_peak(int32_t device, double *tflops);
/* Arithmetic peak of the fp64 pipe of `device`: SMs x 64 FMA lanes x 2 FLOP x the maximum SM clock, in TFLOP/s.
 * bench.py reports the roofline against the larger of this and the live microbenchmark. */
int32_t astroz_cuda_fp64_pipe_peak(int32_t device, double *tflops);

#ifdef __cplusplus
}
#endif
#endif /* ASTROZ_B200_H */
