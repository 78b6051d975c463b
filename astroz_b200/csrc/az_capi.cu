// az_capi.cu -- extern "C" boundary (include/astroz_b200.h).  Host orchestration: the device branch of
// src/Constellation.zig (init :101-200, propagate :245-308, propagateConstellation :541-605) and the
// single-satellite exports of src/c_api/sgp4.zig.  No CPU propagation path exists in this library:
// without a CUDA device every propagate call returns ASTROZ_NO_DEVICE / ASTROZ_CUDA_ERROR.
#include "../../include/astroz_b200.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <sys/mman.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <condition_variable>
#include <cstddef>
#include <initializer_list>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <thread>
#include <vector>

#include "az_avoid.cuh"
#include "az_covariance.cuh"
#include "az_conjunction.cuh"
#include "az_conjunction_is.cuh"
#include "az_correlate.cuh"
#include "az_tasking.cuh"
#include "az_fit.cuh"
#include "az_hostcopy.cuh"
#include "az_ingest.cuh"
#include "az_iod.cuh"
#include "az_link.cuh"
#include "az_kernels.cuh"
#include "az_lambert.cuh"
#include "az_numerical.cuh"
#include "az_obs.cuh"
#include "az_tables.hpp"

namespace {

thread_local std::string g_lastError;
std::mutex g_blockMutex;
std::map<void *, size_t> g_blocks;  // blocks made by astroz_cuda_constellation_host_block: host_free unregisters + unmaps

int32_t cuda_fail(cudaError_t e, const char *what) {
    g_lastError = std::string(what) + ": " + cudaGetErrorString(e);
    return (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver) ? ASTROZ_NO_DEVICE : ASTROZ_CUDA_ERROR;
}
#define AZ_CUDA(expr)                                        \
    do {                                                     \
        cudaError_t _e = (expr);                             \
        if (_e != cudaSuccess) return cuda_fail(_e, #expr);  \
    } while (0)

int32_t status_to_code(int st) {  // kernel-level code -> C API code (src/c_api/sgp4.zig:22-28)
    switch (st) {
        case az::kOk: return ASTROZ_OK;
        case az::kDecayed: return ASTROZ_DECAYED;
        case az::kInvalidEcc: return ASTROZ_INVALID_ECC;
        case az::kDeepSpace: return ASTROZ_DEEP_SPACE;
        case az::kOom: return ASTROZ_ALLOC_FAILED;
        case az::kBadTle: return ASTROZ_BAD_TLE_LENGTH;
        default: return ASTROZ_UNKNOWN;
    }
}

// ASTROZ_NO_DEVICE when no CUDA device is visible (`message` becomes the last error); *count = the device count
int32_t check_device_present(int *count, const char *message) {
    if (cudaGetDeviceCount(count) != cudaSuccess || *count == 0) {
        g_lastError = message;
        return ASTROZ_NO_DEVICE;
    }
    return ASTROZ_OK;
}

// check_device_present, then ASTROZ_VALUE_ERROR unless `device` is one of the visible ordinals
int32_t check_device_ordinal(int device) {
    int count = 0;
    const int32_t rc = check_device_present(&count, "no CUDA device available (this library has no CPU propagation path)");
    if (rc != ASTROZ_OK) return rc;
    if (device < 0 || device >= count) {
        g_lastError = "device index out of range";
        return ASTROZ_VALUE_ERROR;
    }
    return ASTROZ_OK;
}

using az::DevBuf;

// Worker threads of a multi-device handle: one per shard after the first (the caller's thread serves shard 0), parked on
// a condition variable between calls, so a call does not wait for thread creation before its last shard's first launch.
struct ShardWorkers {
    std::mutex m;
    std::condition_variable wake, done;
    std::vector<std::thread> threads;
    const std::function<int32_t(size_t)> *work = nullptr;
    std::vector<int32_t> rc;
    std::vector<std::string> err;
    uint64_t generation = 0;
    size_t pending = 0;
    bool stop = false;

    void start(size_t nShards);
    int32_t run(const std::function<int32_t(size_t)> &w);
    ~ShardWorkers() {
        {
            std::lock_guard<std::mutex> lk(m);
            stop = true;
        }
        wake.notify_all();
        for (auto &t : threads) t.join();
    }
};

struct Constellation {
    int device = 0;
    az::CatalogTables cat;
    az::GravConsts g{};
    double sdp4EpochMin = INFINITY, sdp4EpochMax = -INFINITY;  // epoch span of the deep-space records
    cudaStream_t stream = nullptr, copyStream = nullptr, auxStream = nullptr;  // aux: the deep-space grid of a mixed call
    cudaEvent_t forkEv = nullptr, joinEv = nullptr;
    // element tables (resident for the life of the handle)
    DevBuf<double> dTiles, dToff;
    DevBuf<uint32_t> dSgp4Orig, dSdp4Orig, dIdentity, dSdp4Identity;
    DevBuf<az::Sdp4Sat> dSdp4;
    // per-call time axis: tbase | jdFull | gsin | gcos
    // host staging rotates over kSlots pinned buffers so the host can queue several calls ahead of the GPU
    // without stalling on the previous call's asynchronous upload
    static constexpr int kSlots = 4;
    DevBuf<double> dTime;
    az::PinnedBuf<double> hTimeSlot[kSlots];
    cudaEvent_t slotCopied[kSlots] = {};
    bool slotPending[kSlots] = {};  // slotCopied[k] was recorded after an upload from slot k
    int slot = 0;                   // the slot of the current call
    // the time axis last uploaded by upload_time_axis: a repeated call with the same jd/fr (a propagation loop over a
    // fixed grid) reuses the device copy instead of re-uploading it
    std::vector<double> cachedJd, cachedFr;
    bool cachedGmst = false, cacheValid = false;
    double cachedRef = 0.0, cachedJdMin = 0.0, cachedJdMax = 0.0;
    cudaEvent_t axisReady = nullptr;   // recorded after the cached axis' upload
    cudaStream_t axisStream = nullptr;
    // stateless-path epoch offsets
    DevBuf<double> dToffCall;
    DevBuf<uint8_t> dMask;
    az::PinnedBuf<double> hToffCall;
    cudaEvent_t toffCopied = nullptr;
    bool toffPending = false;
    // resonance lattice (depends on the elements only; grown when a call reaches further in time)
    DevBuf<double2> dLattice;
    int latticeNodes = 0;
    // staging for the host-buffer API
    DevBuf<double> dPos, dVel;
    // (satellite, time) pairs (K6): catalog row -> table key (built on first use), sort keys / indices and segment
    // bounds, the sort's temporary storage, the jd-range reduction, and the host call's two slots of queries / results
    DevBuf<uint32_t> dRowKey, dPairsKeys;
    DevBuf<char> dPairsSort;
    DevBuf<double> dPairsRange, dPairsIn, dPairsOut;
    uint32_t pairsChunk = 1u << 21;  // queries per chunk of the host call (ASTROZ_PAIRS_CHUNK)
    // coarse-screen scratch: hash heads / chains for one batch of epochs, hit buffers, counter
    DevBuf<uint32_t> dHead, dNext, dPairs, dTIdx;
    DevBuf<unsigned long long> dCount;
    // kernel timing: start / end events of K1, K2 and the call's span (TimedSpan), and the set of them the last timed
    // call recorded (bit k = ev[k])
    cudaEvent_t ev[3][2] = {};
    unsigned timedSet = 0;
    bool timing = false;  // kernel-time events are recorded only on request (astroz_cuda_constellation_set_timing): the
                          // timed event records cost stream time, which is not work
    cudaEvent_t chunkDone[64] = {};  // grid chunk k of a host-buffer propagate has finished
    // the two-slot pipeline of the pairs call and sgp4_array, and the pinned ring every pageable transfer goes through
    az::ChunkPipeline pipe;
    int variant = -1;  // -1 = shipped default; >= 0 selects a tuning variant (ASTROZ_SGP4_VARIANT)
    int chunks = 8;
    // Multi-device handle (device = -1 at creation): the catalog is cut into contiguous satellite ranges, one
    // single-device shard each (the analogue of the reference's thread fan-out, src/Constellation.zig:327-385, with
    // ASTROZ_DEVICES in the role of ASTROZ_THREADS, :61-74).  The top-level object then holds only the catalog.
    std::vector<Constellation *> shards;
    std::vector<uint32_t> shardRow0;   // first catalog row of each shard, plus the end (size = shards + 1)
    std::vector<uint32_t> shardNear0;  // first near-earth index of each shard, plus the end
    std::vector<uint32_t> shardDeep0;  // first deep-space index of each shard, plus the end
    DevBuf<double> dFullPos, dFullVel; // per shard: the WHOLE block, for the replicated (all-gather) propagate
    ShardWorkers *workers = nullptr;   // multi-device handle: parked host threads, one per shard after the first
    bool multi() const { return !shards.empty(); }

    // The members are destroyed after this body, on the device it makes current.
    ~Constellation() {
        delete workers;  // joins them: no shard is in use after this line
        for (Constellation *sh : shards) delete sh;
        shards.clear();
        if (!stream) return;  // never opened on a device (a Satrec that was only inspected): nothing to release
        cudaSetDevice(device);
        for (auto &e : slotCopied) if (e) cudaEventDestroy(e);
        if (toffCopied) cudaEventDestroy(toffCopied);
        if (axisReady) cudaEventDestroy(axisReady);
        for (auto &pair : ev) for (auto &e : pair) if (e) cudaEventDestroy(e);
        for (auto &e : chunkDone) if (e) cudaEventDestroy(e);
        if (stream) cudaStreamDestroy(stream);
        if (copyStream) cudaStreamDestroy(copyStream);
        if (auxStream) cudaStreamDestroy(auxStream);
        if (forkEv) cudaEventDestroy(forkEv);
        if (joinEv) cudaEventDestroy(joinEv);
    }
};

int32_t upload_toff(Constellation *c) {  // src/Constellation.zig:153
    const size_t n = c->cat.sgp4Epoch.size();
    if (n == 0) return ASTROZ_OK;
    std::vector<double> off(n);
    for (size_t i = 0; i < n; ++i) off[i] = (c->cat.referenceEpochJd - c->cat.sgp4Epoch[i]) * 1440.0;
    AZ_CUDA(c->dToff.reserve(n));
    AZ_CUDA(cudaMemcpy(c->dToff.p, off.data(), n * 8, cudaMemcpyHostToDevice));
    return ASTROZ_OK;
}

int32_t open_device(Constellation *c, int device) {
    const int32_t rc = check_device_ordinal(device);
    if (rc != ASTROZ_OK) return rc;
    c->device = device;
    AZ_CUDA(cudaSetDevice(device));
    AZ_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    AZ_CUDA(cudaStreamCreateWithFlags(&c->copyStream, cudaStreamNonBlocking));
    AZ_CUDA(cudaStreamCreateWithFlags(&c->auxStream, cudaStreamNonBlocking));
    AZ_CUDA(cudaEventCreateWithFlags(&c->forkEv, cudaEventDisableTiming));
    AZ_CUDA(cudaEventCreateWithFlags(&c->joinEv, cudaEventDisableTiming));
    for (auto &e : c->slotCopied) AZ_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    AZ_CUDA(cudaEventCreateWithFlags(&c->toffCopied, cudaEventDisableTiming));
    AZ_CUDA(cudaEventCreateWithFlags(&c->axisReady, cudaEventDisableTiming));
    for (auto &pair : c->ev)
        for (auto &ev : pair) AZ_CUDA(cudaEventCreate(&ev));
    for (auto &ev : c->chunkDone) AZ_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    AZ_CUDA(c->pipe.create());
    if (const char *v = std::getenv("ASTROZ_SGP4_VARIANT")) c->variant = std::atoi(v);
    if (const char *v = std::getenv("ASTROZ_SDP4_VARIANT")) az::set_sdp4_variant(std::atoi(v));
    if (const char *v = std::getenv("ASTROZ_TIMING")) c->timing = std::atoi(v) != 0;
    if (const char *v = std::getenv("ASTROZ_K1_STRIPE")) az::set_sgp4_stripe((uint32_t)std::max(0, std::atoi(v)));
    if (const char *v = std::getenv("ASTROZ_D2H_CHUNKS")) c->chunks = std::max(1, std::min(64, std::atoi(v)));
    if (const char *v = std::getenv("ASTROZ_PAIRS_CHUNK")) c->pairsChunk = (uint32_t)std::max(1024, std::min(1 << 26, std::atoi(v)));
    return ASTROZ_OK;
}

int32_t finish_create(Constellation *c, int device) {
    int32_t rc0 = open_device(c, device);
    if (rc0 != ASTROZ_OK) return rc0;
    c->g = az::grav_consts(c->cat.grav);
    const az::CatalogTables &t = c->cat;
    if (t.nSgp4) {
        AZ_CUDA(c->dTiles.reserve(t.sgp4Tiles.size()));
        AZ_CUDA(cudaMemcpy(c->dTiles.p, t.sgp4Tiles.data(), t.sgp4Tiles.size() * 8, cudaMemcpyHostToDevice));
        AZ_CUDA(c->dSgp4Orig.reserve(t.sgp4Orig.size()));
        AZ_CUDA(cudaMemcpy(c->dSgp4Orig.p, t.sgp4Orig.data(), t.sgp4Orig.size() * 4, cudaMemcpyHostToDevice));
        std::vector<uint32_t> ident(t.sgp4Orig.size());
        for (size_t i = 0; i < ident.size(); ++i) ident[i] = (uint32_t)std::min<size_t>(i, t.nSgp4 - 1);
        AZ_CUDA(c->dIdentity.reserve(ident.size()));
        AZ_CUDA(cudaMemcpy(c->dIdentity.p, ident.data(), ident.size() * 4, cudaMemcpyHostToDevice));
        int32_t rc = upload_toff(c);
        if (rc != ASTROZ_OK) return rc;
    }
    if (t.nSdp4) {
        AZ_CUDA(c->dSdp4.reserve(t.nSdp4));
        AZ_CUDA(cudaMemcpy(c->dSdp4.p, t.sdp4.data(), t.nSdp4 * sizeof(az::Sdp4Sat), cudaMemcpyHostToDevice));
        AZ_CUDA(c->dSdp4Orig.reserve(t.nSdp4));
        AZ_CUDA(cudaMemcpy(c->dSdp4Orig.p, t.sdp4Orig.data(), t.nSdp4 * 4, cudaMemcpyHostToDevice));
        for (const az::Sdp4Sat &r : t.sdp4) {
            c->sdp4EpochMin = std::min(c->sdp4EpochMin, r.epochJd);
            c->sdp4EpochMax = std::max(c->sdp4EpochMax, r.epochJd);
        }
    }
    return ASTROZ_OK;
}

// Devices of a device = -1 handle: ASTROZ_DEVICE_LIST="0,2,3" names ordinals explicitly (an ordinal may repeat: several
// shards on one GPU, which is how the sharding is exercised on a one-GPU box); otherwise the first ASTROZ_DEVICES of the
// visible devices (all of them when unset) -- the device-count knob in the role of ASTROZ_THREADS
// (src/Constellation.zig:61-74).
std::vector<int> multi_device_list() {
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess) count = 0;
    std::vector<int> devs;
    if (const char *lst = std::getenv("ASTROZ_DEVICE_LIST")) {
        const char *p = lst;
        while (*p) {
            char *end = nullptr;
            const long v = std::strtol(p, &end, 10);
            if (end == p) break;
            if (v >= 0 && v < count) devs.push_back((int)v);
            p = (*end == ',') ? end + 1 : end;
        }
        if (!devs.empty()) return devs;
    }
    int want = count;
    if (const char *v = std::getenv("ASTROZ_DEVICES")) {
        const int k = std::atoi(v);
        if (k >= 1) want = std::min(count, k);
    }
    for (int d = 0; d < want; ++d) devs.push_back(d);
    return devs;
}

// Open the handle on `device` (>= 0), or cut the catalog into one shard per device (device = -1).
int32_t finish_create_any(Constellation *c, int device) {
    if (device >= 0) return finish_create(c, device);
    if (device != -1) {
        g_lastError = "device must be a CUDA ordinal, or -1 for every visible device (ASTROZ_DEVICES caps the count)";
        return ASTROZ_VALUE_ERROR;
    }
    const std::vector<int> devs = multi_device_list();
    const az::CatalogTables &t = c->cat;
    // satellite ranges of equal cost (a deep-space cell costs ~2.4 near-earth cells), cut on multiples of 8 rows so every
    // shard's rows start 64-byte aligned in either layout
    size_t want = std::min<size_t>(devs.size(), std::max<uint32_t>(1u, t.n / 64));
    if (want <= 1) return finish_create(c, devs.empty() ? 0 : devs[0]);
    std::vector<double> prefix(t.n + 1, 0.0);
    for (uint32_t i = 0; i < t.n; ++i) prefix[i + 1] = prefix[i] + (t.classes[i] == 0 ? 1.0 : 2.4);
    std::vector<uint32_t> cut(1, 0u);
    for (size_t k = 1; k < want; ++k) {
        const double target = prefix[t.n] * (double)k / (double)want;
        uint32_t r = (uint32_t)(std::lower_bound(prefix.begin(), prefix.end(), target) - prefix.begin());
        r = std::min(t.n, (r + 4) / 8 * 8);
        if (r > cut.back() && r < t.n) cut.push_back(r);
    }
    cut.push_back(t.n);
    c->g = az::grav_consts(t.grav);
    c->device = devs[0];
    c->shardRow0 = cut;
    c->shardNear0.assign(1, 0u);
    c->shardDeep0.assign(1, 0u);
    for (size_t k = 0; k + 1 < cut.size(); ++k) {
        Constellation *sh = new (std::nothrow) Constellation();
        if (!sh) return ASTROZ_ALLOC_FAILED;
        c->shards.push_back(sh);
        az::slice_catalog(t, cut[k], cut[k + 1], sh->cat);
        c->shardNear0.push_back(c->shardNear0.back() + sh->cat.nSgp4);
        c->shardDeep0.push_back(c->shardDeep0.back() + sh->cat.nSdp4);
        const int32_t rc = finish_create(sh, devs[k % devs.size()]);
        if (rc != ASTROZ_OK) return rc;
    }
    return ASTROZ_OK;
}

// Device-side ingest (K5, az_ingest.cu): the element columns are already in HBM; classification, initialisation and
// the table scatter run there.  The host keeps only what later calls need: counts, epochs, classes, row maps.
int32_t ingest_on_device(Constellation *c, az::IngestArgs a, int grav) {
    cudaStream_t s = c->stream;
    az::CatalogTables &t = c->cat;
    t = az::CatalogTables{};
    t.n = a.n;
    t.grav = az::gravity(grav);
    a.grav = t.grav;
    c->g = az::grav_consts(t.grav);
    if (a.n == 0) return ASTROZ_OK;
    const uint32_t blocks = az::ingest_block_count(a.n);
    DevBuf<uint8_t> flags;
    DevBuf<uint32_t> counts;   // blockNear | blockDeep | totals[2]
    DevBuf<unsigned long long> fail;
    DevBuf<int32_t> classes;
    AZ_CUDA(flags.reserve(a.n));
    AZ_CUDA(counts.reserve((size_t)blocks * 2 + 2));
    AZ_CUDA(fail.reserve(1));
    AZ_CUDA(classes.reserve(a.n));
    a.flags = flags.p;
    a.blockNear = counts.p;
    a.blockDeep = counts.p + blocks;
    a.totals = counts.p + 2 * (size_t)blocks;
    a.firstFail = fail.p;
    a.classes = classes.p;
    AZ_CUDA(cudaMemsetAsync(fail.p, 0xff, 8, s));
    AZ_CUDA(az::launch_ingest_classify(a, s));
    uint32_t totals[2] = {0, 0};
    unsigned long long firstFail = ~0ull;
    AZ_CUDA(cudaMemcpyAsync(totals, a.totals, 8, cudaMemcpyDeviceToHost, s));
    AZ_CUDA(cudaMemcpyAsync(&firstFail, fail.p, 8, cudaMemcpyDeviceToHost, s));
    AZ_CUDA(cudaStreamSynchronize(s));
    if (firstFail != ~0ull) {
        g_lastError = "element set " + std::to_string(firstFail >> 8) + " failed to initialise";
        return status_to_code((int)(firstFail & 0xff));
    }
    t.nSgp4 = totals[0];
    t.nSdp4 = totals[1];
    const uint32_t padded = t.sgp4Padded();
    if (t.nSgp4) {
        AZ_CUDA(c->dTiles.reserve((size_t)t.sgp4Tiles_count() * az::kSgp4TileDoubles));
        AZ_CUDA(c->dSgp4Orig.reserve(padded));
        AZ_CUDA(c->dIdentity.reserve(padded));
    }
    if (t.nSdp4) {
        AZ_CUDA(c->dSdp4.reserve(t.nSdp4));
        AZ_CUDA(c->dSdp4Orig.reserve(t.nSdp4));
    }
    a.tiles = c->dTiles.p;
    a.sgp4Orig = c->dSgp4Orig.p;
    a.identity = c->dIdentity.p;
    a.sdp4 = c->dSdp4.p;
    a.sdp4Orig = c->dSdp4Orig.p;
    AZ_CUDA(az::launch_ingest_build(a, s));
    t.epochs.resize(a.n);
    t.classes.resize(a.n);
    t.sgp4Orig.resize(padded);
    t.sdp4Orig.resize(t.nSdp4);
    AZ_CUDA(cudaMemcpyAsync(t.epochs.data(), a.epochJd, (size_t)a.n * 8, cudaMemcpyDeviceToHost, s));
    AZ_CUDA(cudaMemcpyAsync(t.classes.data(), classes.p, (size_t)a.n * 4, cudaMemcpyDeviceToHost, s));
    if (padded) AZ_CUDA(cudaMemcpyAsync(t.sgp4Orig.data(), c->dSgp4Orig.p, (size_t)padded * 4, cudaMemcpyDeviceToHost, s));
    if (t.nSdp4) AZ_CUDA(cudaMemcpyAsync(t.sdp4Orig.data(), c->dSdp4Orig.p, (size_t)t.nSdp4 * 4, cudaMemcpyDeviceToHost, s));
    AZ_CUDA(cudaMemcpyAsync(&firstFail, fail.p, 8, cudaMemcpyDeviceToHost, s));
    AZ_CUDA(cudaStreamSynchronize(s));
    if (firstFail != ~0ull) {
        g_lastError = "element set " + std::to_string(firstFail >> 8) + " failed to initialise";
        return status_to_code((int)(firstFail & 0xff));
    }
    t.sgp4Epoch.resize(padded);
    for (uint32_t i = 0; i < padded; ++i) t.sgp4Epoch[i] = t.epochs[t.sgp4Orig[i]];
    if (t.nSgp4) t.referenceEpochJd = t.sgp4Epoch[0];  // src/Constellation.zig:139-140
    for (uint32_t i = 0; i < t.nSdp4; ++i) {
        c->sdp4EpochMin = std::min(c->sdp4EpochMin, t.epochs[t.sdp4Orig[i]]);
        c->sdp4EpochMax = std::max(c->sdp4EpochMax, t.epochs[t.sdp4Orig[i]]);
    }
    return upload_toff(c);
}

cudaStream_t call_stream(const Constellation *c, void *stream) {
    return stream ? static_cast<cudaStream_t>(stream) : c->stream;
}

// ASTROZ_VALUE_ERROR for a multi-device handle at an entry point that works on one GPU
int32_t refuse_multi(const Constellation *c) {
    if (c && c->multi()) {
        g_lastError = "this entry point works on ONE GPU: create the handle with device >= 0 (a device = -1 handle "
                      "spans several GPUs)";
        return ASTROZ_VALUE_ERROR;
    }
    return ASTROZ_OK;
}

// Column k of the device time axis dTime: tbase | jdFull | gsin | gcos
double *time_col(Constellation *c, int k) { return c->dTime.p + (size_t)k * (c->dTime.cap / 4); }

// Host staging for an nt-epoch time axis: the next pinned slot of the rotation, column k at *h + k * nt, once the
// upload that last used it has finished.  Every writer of dTime comes through here (or says so itself).
int32_t time_slot(Constellation *c, size_t nt, double **h) {
    c->cacheValid = false;
    c->slot = (c->slot + 1) % Constellation::kSlots;
    const int k = c->slot;
    if (c->slotPending[k]) {  // kSlots calls ago: almost always long finished
        AZ_CUDA(cudaEventSynchronize(c->slotCopied[k]));
        c->slotPending[k] = false;
    }
    AZ_CUDA(c->hTimeSlot[k].reserve(nt * 4));
    AZ_CUDA(c->dTime.reserve(nt * 4));
    *h = c->hTimeSlot[k].p;
    return ASTROZ_OK;
}

// Queue the upload of the staged columns `cols` (bit k = column k) of the current slot and mark the slot in flight.
int32_t upload_time_slot(Constellation *c, size_t nt, unsigned cols, cudaStream_t s) {
    const double *h = c->hTimeSlot[c->slot].p;
    for (int k = 0; k < 4; ++k)
        if (cols & (1u << k))
            AZ_CUDA(cudaMemcpyAsync(time_col(c, k), h + k * nt, nt * 8, cudaMemcpyHostToDevice, s));
    AZ_CUDA(cudaEventRecord(c->slotCopied[c->slot], s));
    c->slotPending[c->slot] = true;
    return ASTROZ_OK;
}

// Time axis of the stateless near-earth path on s: `times` (minutes from the reference) into column 0, sin / cos of GMST
// into columns 2 and 3 when mode != TEME, and the per-call epoch offsets, padded to whole tiles, into dToffCall.
int32_t stage_stateless_axis(Constellation *c, const double *times, uint32_t nt, const double *offsets, int mode,
                             double reference_jd, cudaStream_t s) {
    double *tb;
    int32_t rc = time_slot(c, nt, &tb);
    if (rc != ASTROZ_OK) return rc;
    double *gs = tb + 2 * (size_t)nt, *gc = tb + 3 * (size_t)nt;
    for (uint32_t t = 0; t < nt; ++t) {
        tb[t] = times[t];
        if (mode != 0) {  // src/Constellation.zig:573-581
            const double gm = az::julian_to_gmst(reference_jd + times[t] / 1440.0);
            gs[t] = std::sin(gm);
            gc[t] = std::cos(gm);
        }
    }
    rc = upload_time_slot(c, nt, (mode != 0) ? 0xDu : 0x1u, s);
    if (rc != ASTROZ_OK) return rc;
    const uint32_t ns = c->cat.nSgp4, padded = c->cat.sgp4Padded();
    if (c->toffPending) {  // the previous call's upload of the offsets must have left the staging buffer
        AZ_CUDA(cudaEventSynchronize(c->toffCopied));
        c->toffPending = false;
    }
    AZ_CUDA(c->hToffCall.reserve(padded));
    for (uint32_t i = 0; i < padded; ++i) c->hToffCall.p[i] = offsets[std::min(i, ns - 1)];
    AZ_CUDA(c->dToffCall.reserve(padded));
    AZ_CUDA(cudaMemcpyAsync(c->dToffCall.p, c->hToffCall.p, (size_t)padded * 8, cudaMemcpyHostToDevice, s));
    AZ_CUDA(cudaEventRecord(c->toffCopied, s));
    c->toffPending = true;
    return ASTROZ_OK;
}

// Kernel timing (astroz_cuda_constellation_last_kernel_ms).  A timed call starts a new record with time_begin, then
// marks the start and end of each span it times; events are recorded only while timing is on.
enum TimedSpan { kTimeK1 = 0, kTimeK2 = 1, kTimeSpan = 2 };

void time_begin(Constellation *c) { c->timedSet = 0; }

cudaError_t time_mark(Constellation *c, TimedSpan k, bool end, cudaStream_t s) {
    if (!c->timing) return cudaSuccess;
    if (end) c->timedSet |= 1u << k;
    return cudaEventRecord(c->ev[k][end], s);
}

// Queue launch() on s between the start and end marks of span k (no marks when `timed` is false).
template <class F> cudaError_t in_span(Constellation *c, TimedSpan k, bool timed, cudaStream_t s, F &&launch) {
    cudaError_t e = timed ? time_mark(c, k, false, s) : cudaSuccess;
    if (e == cudaSuccess) e = launch();
    if (e == cudaSuccess && timed) e = time_mark(c, k, true, s);
    return e;
}

// A call of one grid pass: a new timing record holding span k around launch()
template <class F> int32_t timed_pass(Constellation *c, TimedSpan k, cudaStream_t s, F &&launch) {
    time_begin(c);
    AZ_CUDA(in_span(c, k, true, s, launch));
    return ASTROZ_OK;
}

int32_t ensure_lattice(Constellation *c, int nodes, cudaStream_t s) {
    nodes = std::min(std::max(nodes, 2), 16384);
    if (nodes <= c->latticeNodes) return ASTROZ_OK;
    nodes = std::max(nodes, 32);
    AZ_CUDA(cudaStreamSynchronize(s));  // a previous launch may still read the old lattice
    AZ_CUDA(c->dLattice.reserve((size_t)c->cat.nSdp4 * 2 * nodes));
    AZ_CUDA(az::launch_sdp4_lattice(c->dSdp4.p, c->cat.nSdp4, c->dLattice.p, nodes, s));
    c->latticeNodes = nodes;
    return ASTROZ_OK;
}

struct Launch {  // one grid pass over (satellite range) x (time range)
    uint32_t tile0 = 0, tileCount = 0;  // near-earth tiles
    bool deepSpace = true;              // include the deep-space satellites
    uint32_t t0 = 0, nt = 0;            // epoch range
};

// Queue the kernels for `L` on stream s.  Time arrays must already be on the device.
struct GatherTargets {  // fused all-gather destinations (see astroz_cuda_constellation_propagate_gather)
    int kind = 0;      // 0 none, 1 multicast, 2 peer stores
    int nPeers = 0;
    double *mcPos = nullptr, *mcVel = nullptr;
    double *peerPos[az::kMaxPeers] = {}, *peerVel[az::kMaxPeers] = {};
};

// The two builders of a grid pass's arguments: the handle's tables, its gravity constants, the satellite count and the
// time-axis columns from epoch t0 (dTime as last staged, so they are built after the staging).  The caller adds the
// outputs and whatever selects a kernel path of its own (tsince, jdArr, mask, gather), which the builders leave null.
// K1 (near-earth) over tiles [tile0, tile0 + tileCount) of the table, with epoch offsets `toff` and output rows `orig`
// indexed from the table's first satellite.
az::GridArgs near_pass(Constellation *c, const double *toff, const uint32_t *orig, uint32_t tile0 = 0,
                       uint32_t tileCount = UINT32_MAX, uint32_t t0 = 0) {
    const size_t first = (size_t)tile0 * az::kTileSats;
    az::GridArgs a;
    a.g = c->g;
    a.sgp4Tiles = c->dTiles.p + (size_t)tile0 * az::kSgp4TileDoubles;
    a.toff = toff + first;
    a.orig = orig + first;
    a.nSats = (uint32_t)std::min<uint64_t>(c->cat.nSgp4 - first, (uint64_t)tileCount * az::kTileSats);
    a.tbase = time_col(c, 0) + t0;
    a.gsin = time_col(c, 2) + t0;
    a.gcos = time_col(c, 3) + t0;
    return a;
}

// K2 (deep space) over every deep-space record, with output rows `orig`.  The lattice must already reach the call.
az::GridArgs deep_pass(Constellation *c, const uint32_t *orig, uint32_t t0 = 0) {
    az::GridArgs a;
    a.g = c->g;
    a.sdp4 = c->dSdp4.p;
    a.orig = orig;
    a.nSats = c->cat.nSdp4;
    a.lattice = c->dLattice.p;
    a.latticeNodes = c->latticeNodes;
    a.jdFull = time_col(c, 1) + t0;
    a.gsin = time_col(c, 2) + t0;
    a.gcos = time_col(c, 3) + t0;
    return a;
}

int32_t queue_grid(Constellation *c, const Launch &L, uint32_t ntTotal, double *dPos, double *dVel, uint8_t *dStatus,
                   int mode, int layout, uint32_t outNumSats, uint32_t outSatOffset, cudaStream_t s, bool timeIt,
                   const GatherTargets *gt = nullptr) {
    if (layout == 0 && L.nt != ntTotal) {
        g_lastError = "internal: satellite-major launches cover the whole time axis";
        return ASTROZ_UNKNOWN;
    }
    // The status block is the handle's own n x ntTotal bytes, satellite-major, whatever block the positions land in:
    // the kernels index it by output row and a.nTimes, which is the chunk length for a time-major chunk, so it only
    // comes with launches over the whole time axis.
    if (dStatus && (L.t0 != 0 || L.nt != ntTotal)) {
        g_lastError = "internal: a status block needs a launch over the whole time axis";
        return ASTROZ_UNKNOWN;
    }
    // outputs: rows are shifted by outSatOffset, epochs by t0
    const size_t shift = (layout == 0) ? ((size_t)outSatOffset * ntTotal + L.t0) * 3
                                       : ((size_t)L.t0 * outNumSats + outSatOffset) * 3;
    auto outputs = [&](az::GridArgs a) {
        a.nTimes = (layout == 0) ? ntTotal : L.nt;  // satellite-major rows are ntTotal long
        a.outNumSats = outNumSats;
        a.pos = dPos ? dPos + shift : nullptr;
        a.vel = dVel ? dVel + shift : nullptr;
        if (gt && gt->kind) {
            a.gather = gt->kind;
            a.nPeers = gt->nPeers;
            a.mcPos = gt->mcPos ? gt->mcPos + shift : nullptr;
            a.mcVel = gt->mcVel ? gt->mcVel + shift : nullptr;
            for (int p = 0; p < gt->nPeers; ++p) {
                a.peerPos[p] = gt->peerPos[p] ? gt->peerPos[p] + shift : nullptr;
                a.peerVel[p] = gt->peerVel[p] ? gt->peerVel[p] + shift : nullptr;
            }
        }
        a.status = dStatus;  // row i of the handle at i * ntTotal, not shifted by outSatOffset
        return a;
    };
    const bool doK1 = L.tileCount && c->cat.nSgp4, doK2 = L.deepSpace && c->cat.nSdp4;
    // A mixed call runs its two grids side by side: the deep-space grid is small (a few waves of CTAs at lower
    // fp64-pipe utilisation) and goes first, on the auxiliary stream, so the near-earth CTAs fill the SMs as it drains.
    const bool fork = doK1 && doK2;
    cudaStream_t s2 = fork ? c->auxStream : s;
    if (timeIt) {
        time_begin(c);
        AZ_CUDA(time_mark(c, kTimeSpan, false, s));
    }
    if (fork) {
        AZ_CUDA(cudaEventRecord(c->forkEv, s));
        AZ_CUDA(cudaStreamWaitEvent(s2, c->forkEv, 0));
    }
    if (doK2) {
        const az::GridArgs k2 = outputs(deep_pass(c, c->dSdp4Orig.p, L.t0));
        AZ_CUDA(in_span(c, kTimeK2, timeIt, s2, [&] { return az::launch_sdp4_grid(k2, mode, layout, s2); }));
    }
    if (doK1) {
        const az::GridArgs k1 = outputs(near_pass(c, c->dToff.p, c->dSgp4Orig.p, L.tile0, L.tileCount, L.t0));
        AZ_CUDA(in_span(c, kTimeK1, timeIt, s, [&] { return az::launch_sgp4_grid(k1, mode, layout, s, c->variant); }));
    }
    if (fork) {
        AZ_CUDA(cudaEventRecord(c->joinEv, s2));
        AZ_CUDA(cudaStreamWaitEvent(s, c->joinEv, 0));
    }
    if (timeIt) AZ_CUDA(time_mark(c, kTimeSpan, true, s));
    return ASTROZ_OK;
}

// Satellites [row0, row0 + n) x epochs [t0, t0 + m) of a block of totalRows satellites x nt epochs, 3 doubles per cell,
// in `layout`: `rows` runs of rowBytes, `pitch` bytes apart, from double `at` of the block.  A satellite-major range
// covers whole rows (t0 = 0, m = nt).  A dense device block of those cells holds the same runs back to back.
struct HostRows {
    size_t at, rows, rowBytes, pitch;
};

HostRows host_rows(int layout, uint32_t row0, uint32_t n, uint32_t totalRows, uint32_t t0, uint32_t m, uint32_t nt) {
    if (layout == 0) return {((size_t)row0 * nt + t0) * 3, n, (size_t)m * 24, (size_t)nt * 24};  // a run per satellite
    return {((size_t)t0 * totalRows + row0) * 3, m, (size_t)n * 24, (size_t)totalRows * 24};       // a run per epoch
}

// Place the dense device blocks dPos / dVel at `h` in the caller's host blocks pos / vel once the work queued so far on
// c->stream has finished (recorded in `ready`): pinned and registered memory gets a DMA on the copy stream, pageable
// memory gets ring-sized pieces through the pinned ring, delivered by propagate_host_wait.
int32_t place_rows(Constellation *c, cudaEvent_t ready, const double *dPos, const double *dVel, double *pos,
                   double *vel, const HostRows &h) {
    AZ_CUDA(cudaEventRecord(ready, c->stream));
    AZ_CUDA(cudaStreamWaitEvent(c->copyStream, ready, 0));
    for (int which = 0; which < (vel ? 2 : 1); ++which) {
        double *dst = which ? vel : pos;
        AZ_CUDA(c->pipe.ring.deliver(az::is_pageable(dst), ready, which ? dVel : dPos, dst + h.at, h.rows, h.rowBytes,
                                     h.pitch, c->copyStream));
    }
    return ASTROZ_OK;
}

int32_t propagate_host_wait(Constellation *c) {
    if (!c->stream) return ASTROZ_OK;
    AZ_CUDA(cudaSetDevice(c->device));
    AZ_CUDA(c->pipe.ring.drain(c->copyStream));
    AZ_CUDA(cudaStreamSynchronize(c->copyStream));
    AZ_CUDA(cudaStreamSynchronize(c->stream));
    return ASTROZ_OK;
}

// Build the time axis on the host exactly as the reference does (src/Constellation.zig:266-284) and
// queue its upload on s.
int32_t upload_time_axis(Constellation *c, const double *jd, const double *fr, uint32_t nt, int mode, cudaStream_t s,
                         double *jdMin, double *jdMax) {
    if (c->cacheValid && c->cachedJd.size() == nt && c->cachedRef == c->cat.referenceEpochJd &&
        (mode == 0 || c->cachedGmst) && std::memcmp(c->cachedJd.data(), jd, (size_t)nt * 8) == 0 &&
        std::memcmp(c->cachedFr.data(), fr, (size_t)nt * 8) == 0) {
        *jdMin = c->cachedJdMin;
        *jdMax = c->cachedJdMax;
        if (s != c->axisStream) AZ_CUDA(cudaStreamWaitEvent(s, c->axisReady, 0));
        return ASTROZ_OK;
    }
    double *tb;
    int32_t rc = time_slot(c, nt, &tb);
    if (rc != ASTROZ_OK) return rc;
    double *jf = tb + nt, *gs = tb + 2 * (size_t)nt, *gc = tb + 3 * (size_t)nt;
    double lo = INFINITY, hi = -INFINITY;
    for (uint32_t t = 0; t < nt; ++t) {
        const double j = jd[t] + fr[t];
        jf[t] = j;
        tb[t] = (j - c->cat.referenceEpochJd) * 1440.0;
        lo = std::min(lo, j);
        hi = std::max(hi, j);
        if (mode != 0) {
            const double gm = az::julian_to_gmst(j);
            gs[t] = std::sin(gm);
            gc[t] = std::cos(gm);
        }
    }
    *jdMin = lo;
    *jdMax = hi;
    rc = upload_time_slot(c, nt, (mode != 0) ? 0xFu : 0x3u, s);
    if (rc != ASTROZ_OK) return rc;
    AZ_CUDA(cudaEventRecord(c->axisReady, s));
    c->axisStream = s;
    c->cachedJd.assign(jd, jd + nt);
    c->cachedFr.assign(fr, fr + nt);
    c->cachedGmst = (mode != 0);
    c->cachedRef = c->cat.referenceEpochJd;
    c->cachedJdMin = lo;
    c->cachedJdMax = hi;
    c->cacheValid = true;
    return ASTROZ_OK;
}

int32_t prepare_deep_space(Constellation *c, double jdMin, double jdMax, cudaStream_t s) {
    if (c->cat.nSdp4 == 0) return ASTROZ_OK;
    const double eMin = c->sdp4EpochMin, eMax = c->sdp4EpochMax;
    const double reach = std::max(std::fabs((jdMax - eMin) * 1440.0), std::fabs((jdMin - eMax) * 1440.0));
    return ensure_lattice(c, (int)std::floor(reach / az::kStepp) + 2, s);
}

int32_t check_args(Constellation *c, const void *jd, const void *fr, const void *pos, int mode, int layout) {
    if (!c || !jd || !fr || !pos) return ASTROZ_NULL_POINTER;
    if (mode < 0 || mode > 2 || layout < 0 || layout > 1) {
        g_lastError = "invalid output mode / layout";
        return ASTROZ_VALUE_ERROR;
    }
    return ASTROZ_OK;
}

// Open a freshly built handle on `device` (finish_create_any) and hand it to the caller; freed on failure.
int32_t publish(std::unique_ptr<Constellation> c, int device, astroz_constellation_t *out) {
    const int32_t rc = finish_create_any(c.get(), device);
    if (rc != ASTROZ_OK) return rc;
    *out = c.release();
    return ASTROZ_OK;
}

struct Sgp4Single {
    std::unique_ptr<Constellation> c;
    int device = 0;
    bool opened = false;  // streams, events and the device tables are created by the first propagation call
    double epochJd = 0;
    bool deep = false;
    double elements[10] = {};  // ecco inclo nodeo argpo mo no_kozai bstar a no_unkozai epochJd
};

}  // namespace

// ================================================================================================
extern "C" {
#pragma GCC visibility push(default)

uint32_t astroz_cuda_version(void) { return (0u << 16) | (1u << 8) | 0u; }

int32_t astroz_cuda_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}

const char *astroz_cuda_last_error(void) { return g_lastError.c_str(); }

void *astroz_cuda_host_alloc(size_t bytes) {
    void *p = nullptr;
    if (cudaMallocHost(&p, bytes ? bytes : 8) != cudaSuccess) return nullptr;
    return p;
}
void astroz_cuda_host_free(void *p) {
    if (!p) return;
    size_t mapped = 0;
    {
        std::lock_guard<std::mutex> g(g_blockMutex);
        auto it = g_blocks.find(p);
        if (it != g_blocks.end()) {
            mapped = it->second;
            g_blocks.erase(it);
        }
    }
    if (mapped) {  // a block from astroz_cuda_constellation_host_block
        cudaHostUnregister(p);
        munmap(p, mapped);
        return;
    }
    cudaFreeHost(p);
}

int32_t astroz_cuda_constellation_create(const char *const *line1, const char *const *line2, uint32_t n, int32_t grav,
                                         int32_t device, astroz_constellation_t *out) {
    if (!out || (n && (!line1 || !line2))) return ASTROZ_NULL_POINTER;
    *out = nullptr;
    std::unique_ptr<Constellation> c(new (std::nothrow) Constellation());
    if (!c) return ASTROZ_ALLOC_FAILED;
    const int rc = az::build_catalog(line1, line2, n, grav, c->cat);
    if (rc != az::kOk) return status_to_code(rc);
    return publish(std::move(c), device, out);
}

int32_t astroz_cuda_constellation_create_from_text(const char *text, size_t len, int32_t grav, int32_t device,
                                                   astroz_constellation_t *out) {
    if (!text || !out) return ASTROZ_NULL_POINTER;
    std::vector<std::string> l1, l2;
    az::split_tle_text(text, len, l1, l2);
    std::vector<const char *> p1(l1.size()), p2(l2.size());
    for (size_t i = 0; i < l1.size(); ++i) {
        p1[i] = l1[i].c_str();
        p2[i] = l2[i].c_str();
    }
    return astroz_cuda_constellation_create(p1.data(), p2.data(), (uint32_t)l1.size(), grav, device, out);
}

int32_t astroz_cuda_constellation_create_from_elements(const double *epoch_jd, const double *mean_motion_rev_day,
                                                       const double *ecc, const double *incl_deg, const double *raan_deg,
                                                       const double *argp_deg, const double *ma_deg, const double *bstar,
                                                       uint32_t n, int32_t grav, int32_t device,
                                                       astroz_constellation_t *out) {
    if (!out || (n && (!epoch_jd || !mean_motion_rev_day || !ecc || !incl_deg || !raan_deg || !argp_deg || !ma_deg || !bstar)))
        return ASTROZ_NULL_POINTER;
    *out = nullptr;
    std::vector<az::TleRecord> recs(n);
    for (uint32_t i = 0; i < n; ++i) {
        az::TleRecord &t = recs[i];
        t.satnum = i;
        t.epochJd = epoch_jd[i];
        t.revPerDay = mean_motion_rev_day[i];
        t.ecc = ecc[i];
        t.inclDeg = incl_deg[i];
        t.raanDeg = raan_deg[i];
        t.argpDeg = argp_deg[i];
        t.maDeg = ma_deg[i];
        t.bstar = bstar[i];
    }
    std::unique_ptr<Constellation> c(new (std::nothrow) Constellation());
    if (!c) return ASTROZ_ALLOC_FAILED;
    const int rc = az::build_catalog_records(recs.data(), n, grav, c->cat);
    if (rc != az::kOk) return status_to_code(rc);
    return publish(std::move(c), device, out);
}

int32_t astroz_cuda_constellation_create_from_elements_device(
    const double *d_epoch_jd, const double *d_mean_motion_rev_day, const double *d_ecc, const double *d_incl_deg,
    const double *d_raan_deg, const double *d_argp_deg, const double *d_ma_deg, const double *d_bstar, uint32_t n,
    int32_t grav, int32_t device, astroz_constellation_t *out) {
    if (!out || (n && (!d_epoch_jd || !d_mean_motion_rev_day || !d_ecc || !d_incl_deg || !d_raan_deg || !d_argp_deg ||
                       !d_ma_deg || !d_bstar)))
        return ASTROZ_NULL_POINTER;
    *out = nullptr;
    std::unique_ptr<Constellation> c(new (std::nothrow) Constellation());
    if (!c) return ASTROZ_ALLOC_FAILED;
    int32_t e = open_device(c.get(), device);
    if (e != ASTROZ_OK) return e;
    az::IngestArgs a;
    a.epochJd = d_epoch_jd;
    a.revPerDay = d_mean_motion_rev_day;
    a.ecc = d_ecc;
    a.inclDeg = d_incl_deg;
    a.raanDeg = d_raan_deg;
    a.argpDeg = d_argp_deg;
    a.maDeg = d_ma_deg;
    a.bstar = d_bstar;
    a.n = n;
    e = ingest_on_device(c.get(), a, grav);
    if (e != ASTROZ_OK) return e;
    *out = c.release();
    return ASTROZ_OK;
}

void astroz_cuda_constellation_free(astroz_constellation_t h) { delete static_cast<Constellation *>(h); }

int32_t astroz_cuda_constellation_counts(astroz_constellation_t h, uint32_t *n, uint32_t *ns, uint32_t *nd) {
    if (!h) return ASTROZ_NULL_POINTER;
    Constellation *c = static_cast<Constellation *>(h);
    if (n) *n = c->cat.n;
    if (ns) *ns = c->cat.nSgp4;
    if (nd) *nd = c->cat.nSdp4;
    return ASTROZ_OK;
}

int32_t astroz_cuda_constellation_epochs(astroz_constellation_t h, double *epochs) {
    if (!h || !epochs) return ASTROZ_NULL_POINTER;
    Constellation *c = static_cast<Constellation *>(h);
    std::memcpy(epochs, c->cat.epochs.data(), c->cat.epochs.size() * 8);
    return ASTROZ_OK;
}

int32_t astroz_cuda_constellation_classes(astroz_constellation_t h, int32_t *classes) {
    if (!h || !classes) return ASTROZ_NULL_POINTER;
    Constellation *c = static_cast<Constellation *>(h);
    std::memcpy(classes, c->cat.classes.data(), c->cat.classes.size() * 4);
    return ASTROZ_OK;
}

int32_t astroz_cuda_constellation_get_reference_epoch(astroz_constellation_t h, double *jd) {
    if (!h || !jd) return ASTROZ_NULL_POINTER;
    *jd = static_cast<Constellation *>(h)->cat.referenceEpochJd;
    return ASTROZ_OK;
}

int32_t astroz_cuda_constellation_set_reference_epoch(astroz_constellation_t h, double jd) {
    if (!h) return ASTROZ_NULL_POINTER;
    Constellation *c = static_cast<Constellation *>(h);
    if (c->multi()) {
        c->cat.referenceEpochJd = jd;
        for (Constellation *sh : c->shards) {
            const int32_t rc = astroz_cuda_constellation_set_reference_epoch(sh, jd);
            if (rc != ASTROZ_OK) return rc;
        }
        return ASTROZ_OK;
    }
    AZ_CUDA(cudaSetDevice(c->device));
    // kernels still reading the old offsets may sit on the handle's stream or on a caller's stream that was given to a
    // _device call: the whole device is drained, this is a cold configuration call
    AZ_CUDA(cudaDeviceSynchronize());
    c->cat.referenceEpochJd = jd;
    c->cacheValid = false;
    return upload_toff(c);
}

int32_t astroz_cuda_constellation_propagate_device(astroz_constellation_t h, const double *jd, const double *fr,
                                                   uint32_t n_times, double *d_pos, double *d_vel, uint8_t *d_status,
                                                   int32_t mode, int32_t layout, uint32_t out_num_sats,
                                                   uint32_t out_sat_offset, void *stream) {
    Constellation *c = static_cast<Constellation *>(h);
    int32_t rc = refuse_multi(c);
    if (rc == ASTROZ_OK) rc = check_args(c, jd, fr, d_pos, mode, layout);
    if (rc != ASTROZ_OK) return rc;
    if (n_times == 0 || c->cat.n == 0) return ASTROZ_OK;
    if (out_num_sats < out_sat_offset + c->cat.n) {  // src/Constellation.zig:255-257 reports a short buffer this way
        g_lastError = "output block smaller than numSatellites rows";
        return ASTROZ_DECAYED;
    }
    AZ_CUDA(cudaSetDevice(c->device));
    cudaStream_t s = call_stream(c, stream);
    double jdMin, jdMax;
    rc = upload_time_axis(c, jd, fr, n_times, mode, s, &jdMin, &jdMax);
    if (rc != ASTROZ_OK) return rc;
    rc = prepare_deep_space(c, jdMin, jdMax, s);
    if (rc != ASTROZ_OK) return rc;
    Launch L;
    L.tileCount = c->cat.sgp4Tiles_count();
    L.nt = n_times;
    return queue_grid(c, L, n_times, d_pos, d_vel, d_status, mode, layout, out_num_sats, out_sat_offset, s, true);
}

// ---- deep-space members only (Constellation.propagateSdp4Constellation, src/Constellation.zig:611-674) --------
static int32_t sdp4_into_common(Constellation *c, const double *jd, const double *fr, uint32_t nt, double *dPos,
                                double *dVel, int mode, int layout, uint32_t outNumSats, uint32_t satOffset,
                                cudaStream_t s) {
    const uint32_t nd = c->cat.nSdp4;
    if (c->dSdp4Identity.cap < nd) {
        std::vector<uint32_t> ident(nd);
        for (uint32_t i = 0; i < nd; ++i) ident[i] = i;  // origIndices = sat_offset + i, satrec.zig:628-631
        AZ_CUDA(c->dSdp4Identity.reserve(nd));
        AZ_CUDA(cudaMemcpy(c->dSdp4Identity.p, ident.data(), (size_t)nd * 4, cudaMemcpyHostToDevice));
    }
    double jdMin, jdMax;
    int32_t rc = upload_time_axis(c, jd, fr, nt, mode, s, &jdMin, &jdMax);
    if (rc != ASTROZ_OK) return rc;
    rc = prepare_deep_space(c, jdMin, jdMax, s);
    if (rc != ASTROZ_OK) return rc;
    az::GridArgs a = deep_pass(c, c->dSdp4Identity.p);
    a.nTimes = nt;
    a.outNumSats = outNumSats;
    const size_t shift = (layout == 0) ? (size_t)satOffset * nt * 3 : (size_t)satOffset * 3;
    a.pos = dPos + shift;
    a.vel = dVel ? dVel + shift : nullptr;
    return timed_pass(c, kTimeK2, s, [&] { return az::launch_sdp4_grid(a, mode, layout, s); });
}

static int32_t sdp4_into_check(Constellation *c, uint32_t out_num_sats, uint32_t sat_offset, uint32_t *rows) {
    *rows = out_num_sats ? out_num_sats : c->cat.nSdp4;
    if (*rows < sat_offset + c->cat.nSdp4) {  // src/Constellation.zig:626-628 reports a short buffer this way
        g_lastError = "output block smaller than sat_offset + numSdp4 rows";
        return ASTROZ_DECAYED;
    }
    return ASTROZ_OK;
}

int32_t astroz_cuda_sdp4_propagate_into_device(astroz_constellation_t h, const double *jd, const double *fr,
                                               uint32_t n_times, double *d_pos, double *d_vel, int32_t mode,
                                               int32_t layout, uint32_t out_num_sats, uint32_t sat_offset, void *stream) {
    Constellation *c = static_cast<Constellation *>(h);
    int32_t rc = refuse_multi(c);
    if (rc == ASTROZ_OK) rc = check_args(c, jd, fr, d_pos, mode, layout);
    if (rc != ASTROZ_OK) return rc;
    if (n_times == 0 || c->cat.nSdp4 == 0) return ASTROZ_OK;
    uint32_t rows;
    rc = sdp4_into_check(c, out_num_sats, sat_offset, &rows);
    if (rc != ASTROZ_OK) return rc;
    AZ_CUDA(cudaSetDevice(c->device));
    cudaStream_t s = call_stream(c, stream);
    return sdp4_into_common(c, jd, fr, n_times, d_pos, d_vel, mode, layout, rows, sat_offset, s);
}

int32_t astroz_cuda_sdp4_propagate_into(astroz_constellation_t h, const double *jd, const double *fr, uint32_t n_times,
                                        double *pos, double *vel, int32_t mode, int32_t layout, uint32_t out_num_sats,
                                        uint32_t sat_offset) {
    Constellation *c = static_cast<Constellation *>(h);
    int32_t rc = refuse_multi(c);
    if (rc == ASTROZ_OK) rc = check_args(c, jd, fr, pos, mode, layout);
    if (rc != ASTROZ_OK) return rc;
    const uint32_t nd = c->cat.nSdp4;
    if (n_times == 0 || nd == 0) return ASTROZ_OK;
    uint32_t rows;
    rc = sdp4_into_check(c, out_num_sats, sat_offset, &rows);
    if (rc != ASTROZ_OK) return rc;
    AZ_CUDA(cudaSetDevice(c->device));
    // the deep-space rows are computed as a dense block on the device and placed in the caller's (possibly wider)
    // block; rows that belong to other satellites are never touched
    const size_t dense = (size_t)nd * n_times * 3;
    AZ_CUDA(c->dPos.reserve(dense));
    if (vel) AZ_CUDA(c->dVel.reserve(dense));
    double *dVel = vel ? c->dVel.p : nullptr;
    rc = sdp4_into_common(c, jd, fr, n_times, c->dPos.p, dVel, mode, layout, nd, 0, c->stream);
    if (rc != ASTROZ_OK) return rc;
    c->pipe.ring.discard();
    rc = place_rows(c, c->chunkDone[0], c->dPos.p, dVel, pos, vel, host_rows(layout, sat_offset, nd, rows, 0, n_times,
                                                                              n_times));
    if (rc != ASTROZ_OK) return rc;
    return propagate_host_wait(c);
}

int32_t astroz_cuda_constellation_propagate_device_f32(astroz_constellation_t h, const double *jd, const double *fr,
                                                       uint32_t n_times, double *d_pos, double *d_vel, int32_t phase64,
                                                       void *stream) {
    Constellation *c = static_cast<Constellation *>(h);
    if (const int32_t rc = refuse_multi(c); rc != ASTROZ_OK) return rc;
    if (!c || !jd || !fr || !d_pos || !d_vel) return ASTROZ_NULL_POINTER;
    if (n_times == 0 || c->cat.nSgp4 == 0) return ASTROZ_OK;
    AZ_CUDA(cudaSetDevice(c->device));
    cudaStream_t s = call_stream(c, stream);
    double jdMin, jdMax;
    int32_t rc = upload_time_axis(c, jd, fr, n_times, ASTROZ_MODE_TEME, s, &jdMin, &jdMax);
    if (rc != ASTROZ_OK) return rc;
    az::GridArgs a = near_pass(c, c->dToff.p, c->dSgp4Orig.p);
    a.nTimes = n_times;
    a.pos = d_pos;
    a.vel = d_vel;
    a.outNumSats = c->cat.n;
    return timed_pass(c, kTimeK1, s, [&] { return az::launch_sgp4_grid_f32(a, phase64, s); });
}

int32_t astroz_cuda_constellation_propagate_gather(astroz_constellation_t h, const double *jd, const double *fr,
                                                   uint32_t n_times, void *const *peer_pos, void *const *peer_vel,
                                                   uint32_t n_peers, void *mc_pos, void *mc_vel, uint32_t out_num_sats,
                                                   uint32_t out_sat_offset, void *stream) {
    Constellation *c = static_cast<Constellation *>(h);
    if (const int32_t rc = refuse_multi(c); rc != ASTROZ_OK) return rc;
    if (!c || !jd || !fr) return ASTROZ_NULL_POINTER;
    if (!mc_pos && (!peer_pos || n_peers == 0)) return ASTROZ_NULL_POINTER;
    if (n_peers > (uint32_t)az::kMaxPeers) {
        g_lastError = "at most 8 peers (one NVSwitch domain)";
        return ASTROZ_VALUE_ERROR;
    }
    if (n_times == 0 || c->cat.n == 0) return ASTROZ_OK;
    if (out_num_sats < out_sat_offset + c->cat.n) {
        g_lastError = "output block smaller than numSatellites rows";
        return ASTROZ_DECAYED;
    }
    GatherTargets gt;
    gt.kind = mc_pos ? 1 : 2;
    gt.nPeers = (int)n_peers;
    gt.mcPos = static_cast<double *>(mc_pos);
    gt.mcVel = static_cast<double *>(mc_vel);
    for (uint32_t p = 0; p < n_peers && peer_pos; ++p) {
        gt.peerPos[p] = static_cast<double *>(peer_pos[p]);
        gt.peerVel[p] = peer_vel ? static_cast<double *>(peer_vel[p]) : nullptr;
        if (!gt.peerPos[p]) return ASTROZ_NULL_POINTER;
    }
    AZ_CUDA(cudaSetDevice(c->device));
    cudaStream_t s = call_stream(c, stream);
    double jdMin, jdMax;
    int32_t rc = upload_time_axis(c, jd, fr, n_times, ASTROZ_MODE_TEME, s, &jdMin, &jdMax);
    if (rc != ASTROZ_OK) return rc;
    rc = prepare_deep_space(c, jdMin, jdMax, s);
    if (rc != ASTROZ_OK) return rc;
    Launch L;
    L.tileCount = c->cat.sgp4Tiles_count();
    L.nt = n_times;
    return queue_grid(c, L, n_times, nullptr, nullptr, nullptr, ASTROZ_MODE_TEME, ASTROZ_LAYOUT_SATELLITE_MAJOR,
                      out_num_sats, out_sat_offset, s, true, &gt);
}

// Host-buffer propagate, in a queue half and a wait half (deliveries to pageable memory are drained in the latter):
// queue = upload the time axis, launch the grid in chunks, start each chunk's device->host copy as soon as its kernels
// finish; wait = drain the streams.  This handle's rows land at rows [rowOffset, rowOffset + n) of a host block with
// totalRows rows (its own block when rowOffset = 0, totalRows = n).
static int32_t propagate_host_queue(Constellation *c, const double *jd, const double *fr, uint32_t n_times, double *pos,
                                    double *vel, int32_t mode, int32_t layout, uint32_t rowOffset, uint32_t totalRows) {
    const uint32_t n = c->cat.n;
    if (n_times == 0 || n == 0) return ASTROZ_OK;
    AZ_CUDA(cudaSetDevice(c->device));
    const size_t total = (size_t)n * n_times * 3;
    AZ_CUDA(c->dPos.reserve(total));
    if (vel) AZ_CUDA(c->dVel.reserve(total));
    double *dPos = c->dPos.p, *dVel = vel ? c->dVel.p : nullptr;
    cudaStream_t s = c->stream;
    double jdMin, jdMax;
    int32_t rc = upload_time_axis(c, jd, fr, n_times, mode, s, &jdMin, &jdMax);
    if (rc != ASTROZ_OK) return rc;
    rc = prepare_deep_space(c, jdMin, jdMax, s);
    if (rc != ASTROZ_OK) return rc;

    // Pipeline: the grid is cut into chunks whose output is one contiguous block of the result, so the
    // device->host copy of chunk i (copy stream) overlaps the kernels of chunk i+1 (compute stream).
    const uint32_t tiles = c->cat.sgp4Tiles_count();
    const bool bySat = (layout == 0) && c->cat.nSdp4 == 0;  // near-earth rows are the identity map
    const bool byTime = (layout == 1);
    uint32_t units = bySat ? tiles : (byTime ? n_times : 1);
    uint32_t nChunks = (bySat || byTime) ? std::min<uint32_t>((uint32_t)c->chunks, units) : 1;
    if (total * 8 < (8u << 20)) nChunks = 1;
    uint32_t per = (units + nChunks - 1) / nChunks;
    // a thread's epochs are 32 apart and the kernels start their runs at multiples of 64 / 96 epochs from the start of the
    // launch: time chunks that start on multiples of 192 keep every thread's set of epochs -- and with it the series each
    // cell takes, i.e. every result bit -- the same however the call is chunked (one device or many, any chunk count)
    if (byTime && nChunks > 1) per = (per + 191) / 192 * 192;
    c->pipe.ring.discard();
    // last_kernel_ms after a host-buffer call: the span from the first kernel of the first chunk to the last kernel of
    // the last chunk (copies overlapping) in all three slots
    time_begin(c);
    AZ_CUDA(time_mark(c, kTimeSpan, false, s));
    for (uint32_t k = 0; k < nChunks; ++k) {
        const uint32_t u0 = k * per, u1 = std::min(units, u0 + per);
        if (u0 >= u1) break;
        Launch L;
        uint32_t r0 = 0, r1 = n;  // the chunk's satellites
        if (bySat) {
            L.tile0 = u0; L.tileCount = u1 - u0; L.deepSpace = false; L.t0 = 0; L.nt = n_times;
            r0 = u0 * az::kTileSats;
            r1 = (uint32_t)std::min<size_t>(n, (size_t)u1 * az::kTileSats);
        } else if (byTime) {
            L.tile0 = 0; L.tileCount = tiles; L.deepSpace = true; L.t0 = u0; L.nt = u1 - u0;
        } else {
            L.tile0 = 0; L.tileCount = tiles; L.deepSpace = true; L.t0 = 0; L.nt = n_times;
        }
        rc = queue_grid(c, L, n_times, dPos, dVel, nullptr, mode, layout, n, 0, s, false);
        if (rc != ASTROZ_OK) return rc;
        // the device block is this handle's alone: the chunk's cells sit there as they would in a host block of n rows
        const size_t off = host_rows(layout, r0, r1 - r0, n, L.t0, L.nt, n_times).at;
        rc = place_rows(c, c->chunkDone[k], dPos + off, dVel ? dVel + off : nullptr, pos, vel,
                        host_rows(layout, rowOffset + r0, r1 - r0, totalRows, L.t0, L.nt, n_times));
        if (rc != ASTROZ_OK) return rc;
    }
    AZ_CUDA(time_mark(c, kTimeSpan, true, s));
    return ASTROZ_OK;
}

// Run `work(k)` (queue + wait of shard k) for every shard of a multi-device handle, one host thread per shard: the
// launches and copies of the devices are issued side by side instead of one device after the other.
void ShardWorkers::start(size_t nShards) {
    rc.assign(nShards, ASTROZ_OK);
    err.assign(nShards, std::string());
    for (size_t k = 1; k < nShards; ++k)
        threads.emplace_back([this, k] {
            uint64_t seen = 0;
            for (;;) {
                const std::function<int32_t(size_t)> *w;
                {
                    std::unique_lock<std::mutex> lk(m);
                    wake.wait(lk, [&] { return stop || generation != seen; });
                    if (stop) return;
                    seen = generation;
                    w = work;
                }
                const int32_t r = (*w)(k);
                std::lock_guard<std::mutex> lk(m);
                rc[k] = r;
                if (r != ASTROZ_OK) err[k] = g_lastError;  // thread-local in the worker: carry it back
                if (--pending == 0) done.notify_one();
            }
        });
}

int32_t ShardWorkers::run(const std::function<int32_t(size_t)> &w) {
    {
        std::lock_guard<std::mutex> lk(m);
        work = &w;
        pending = threads.size();
        ++generation;
    }
    wake.notify_all();
    const int32_t r0 = w(0);
    const std::string e0 = (r0 != ASTROZ_OK) ? g_lastError : std::string();
    std::unique_lock<std::mutex> lk(m);
    done.wait(lk, [&] { return pending == 0; });
    rc[0] = r0;
    err[0] = e0;
    for (size_t k = 0; k < rc.size(); ++k)
        if (rc[k] != ASTROZ_OK) {
            g_lastError = err[k];
            return rc[k];
        }
    return ASTROZ_OK;
}

static int32_t for_each_shard(Constellation *c, const std::function<int32_t(size_t)> &work) {
    if (!c->workers) {  // first call through this handle (calls on one handle are serial, include/astroz_b200.h)
        c->workers = new ShardWorkers();
        c->workers->start(c->shards.size());
    }
    return c->workers->run(work);
}

// A host-buffer call on every device of the handle: queue(target, row0, near0) then propagate_host_wait(target), on the
// handle itself (row0 = near0 = 0), or on each shard side by side with its first catalog row and first near-earth index.
// Each shard computes its own satellite range and copies it over its own PCIe link into its slice of the caller's
// block: no collective is needed for a host-resident result.
static int32_t queue_and_wait(Constellation *c,
                              const std::function<int32_t(Constellation *, uint32_t, uint32_t)> &queue) {
    if (!c->multi()) {
        const int32_t rc = queue(c, 0, 0);
        if (rc != ASTROZ_OK) return rc;
        return propagate_host_wait(c);
    }
    return for_each_shard(c, [&](size_t k) -> int32_t {
        Constellation *sh = c->shards[k];
        const int32_t q = queue(sh, c->shardRow0[k], c->shardNear0[k]);
        const int32_t w = propagate_host_wait(sh);   // also drains what was queued before a failure
        return q != ASTROZ_OK ? q : w;
    });
}

int32_t astroz_cuda_constellation_propagate(astroz_constellation_t h, const double *jd, const double *fr,
                                            uint32_t n_times, double *pos, double *vel, int32_t mode, int32_t layout) {
    Constellation *c = static_cast<Constellation *>(h);
    const int32_t rc = check_args(c, jd, fr, pos, mode, layout);
    if (rc != ASTROZ_OK) return rc;
    if (n_times == 0 || c->cat.n == 0) return ASTROZ_OK;
    return queue_and_wait(c, [&](Constellation *sh, uint32_t row0, uint32_t) {
        return propagate_host_queue(sh, jd, fr, n_times, pos, vel, mode, layout, row0, c->cat.n);
    });
}

// ---- (satellite, time) pairs (K6, az_pairs.cu) ----------------------------------------------------------------------
// Catalog row -> sort key: its near-earth table index, or nSgp4 + its deep-space index (the catalog's, built once).
static int32_t pairs_row_keys(Constellation *c, cudaStream_t s) {
    const az::CatalogTables &t = c->cat;
    if (c->dRowKey.cap >= t.n) return ASTROZ_OK;
    std::vector<uint32_t> key(t.n, 0);
    for (uint32_t i = 0; i < t.nSgp4; ++i) key[t.sgp4Orig[i]] = i;
    for (uint32_t d = 0; d < t.nSdp4; ++d) key[t.sdp4Orig[d]] = t.nSgp4 + d;
    AZ_CUDA(c->dRowKey.reserve(t.n));
    AZ_CUDA(cudaMemcpyAsync(c->dRowKey.p, key.data(), (size_t)t.n * 4, cudaMemcpyHostToDevice, s));  // staged: returns
    return ASTROZ_OK;                                                                                 // after the copy-out
}

// Queue key / sort / split / K6 for n device-resident queries on s.  The lattice must already reach every query.
static int32_t pairs_queue(Constellation *c, const uint32_t *dSat, const double *dJd, const double *dFr, uint32_t n,
                           int mode, double *dPos, double *dVel, uint8_t *dStatus, cudaStream_t s) {
    const az::CatalogTables &t = c->cat;
    int32_t rc = pairs_row_keys(c, s);
    if (rc != ASTROZ_OK) return rc;
    size_t sortBytes = 0;
    AZ_CUDA(az::pairs_sort_scratch_bytes(n, t.n, &sortBytes));
    AZ_CUDA(c->dPairsKeys.reserve((size_t)n * 4 + 2));
    AZ_CUDA(c->dPairsSort.reserve(std::max<size_t>(sortBytes, 16)));
    az::PairsArgs a;
    a.sgp4Tiles = c->dTiles.p;
    a.toff = c->dToff.p;
    a.sdp4 = c->dSdp4.p;
    a.lattice = c->dLattice.p;
    a.latticeNodes = c->latticeNodes;
    a.rowKey = c->dRowKey.p;
    a.nRows = t.n;
    a.nSgp4 = t.nSgp4;
    a.refJd = t.referenceEpochJd;
    a.sat = dSat;
    a.jd = dJd;
    a.fr = dFr;
    a.n = n;
    uint32_t *k = c->dPairsKeys.p;
    a.keys = k;
    a.idx = k + n;
    a.keysSorted = k + 2 * (size_t)n;
    a.idxSorted = k + 3 * (size_t)n;
    a.split = k + 4 * (size_t)n;
    a.sortScratch = c->dPairsSort.p;
    a.sortScratchBytes = c->dPairsSort.cap;
    a.pos = dPos;
    a.vel = dVel;
    a.status = dStatus;
    a.g = c->g;
    AZ_CUDA(az::launch_pairs(a, mode, s));
    time_begin(c);  // the pairs kernels are not timed
    return ASTROZ_OK;
}

static int32_t pairs_check(Constellation *c, int32_t mode) {
    if (!c) return ASTROZ_NULL_POINTER;
    if (const int32_t rc = refuse_multi(c); rc != ASTROZ_OK) return rc;
    if (mode < 0 || mode > 2) {
        g_lastError = "invalid output mode";
        return ASTROZ_VALUE_ERROR;
    }
    return ASTROZ_OK;
}

int32_t astroz_cuda_constellation_propagate_pairs_device(astroz_constellation_t h, const uint32_t *d_sat,
                                                         const double *d_jd, const double *d_fr, uint32_t n,
                                                         int32_t mode, double *d_pos, double *d_vel,
                                                         uint8_t *d_status, void *stream) {
    Constellation *c = static_cast<Constellation *>(h);
    int32_t rc = pairs_check(c, mode);
    if (rc != ASTROZ_OK) return rc;
    if (n == 0) return ASTROZ_OK;
    if (!d_sat || !d_jd || !d_fr || !d_pos) return ASTROZ_NULL_POINTER;
    AZ_CUDA(cudaSetDevice(c->device));
    cudaStream_t s = call_stream(c, stream);
    if (c->cat.nSdp4) {
        // the resonance lattice is grown to the furthest query: min / max of jd + fr on the device, 16 bytes back
        // (this call's one synchronisation point)
        AZ_CUDA(c->dPairsRange.reserve(az::pairs_range_scratch_doubles()));
        AZ_CUDA(az::launch_pairs_range(d_jd, d_fr, n, c->dPairsRange.p, s));
        double range[2];
        AZ_CUDA(cudaMemcpyAsync(range, c->dPairsRange.p, 16, cudaMemcpyDeviceToHost, s));
        AZ_CUDA(cudaStreamSynchronize(s));
        rc = prepare_deep_space(c, range[0], range[1], s);
        if (rc != ASTROZ_OK) return rc;
    }
    return pairs_queue(c, d_sat, d_jd, d_fr, n, mode, d_pos, d_vel, d_status, s);
}

// Host buffers: chunks of pairsChunk queries through the handle's two-slot pipeline (az::ChunkPipeline).
int32_t astroz_cuda_constellation_propagate_pairs(astroz_constellation_t h, const uint32_t *sat, const double *jd,
                                                  const double *fr, uint32_t n, int32_t mode, double *pos, double *vel,
                                                  uint8_t *status) {
    Constellation *c = static_cast<Constellation *>(h);
    int32_t rc = pairs_check(c, mode);
    if (rc != ASTROZ_OK) return rc;
    if (n == 0) return ASTROZ_OK;
    if (!sat || !jd || !fr || !pos) return ASTROZ_NULL_POINTER;
    const az::CatalogTables &t = c->cat;
    for (uint32_t i = 0; i < n; ++i)
        if (sat[i] >= t.n) {
            g_lastError = "query " + std::to_string(i) + ": satellite row " + std::to_string(sat[i]) + " is not in the " +
                          std::to_string(t.n) + "-row catalog";
            return ASTROZ_VALUE_ERROR;
        }
    AZ_CUDA(cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    if (t.nSdp4) {
        double lo = INFINITY, hi = -INFINITY;
        for (uint32_t i = 0; i < n; ++i) {
            const double j = jd[i] + fr[i];
            lo = std::min(lo, j);
            hi = std::max(hi, j);
        }
        rc = prepare_deep_space(c, lo, hi, st);
        if (rc != ASTROZ_OK) return rc;
    }
    const uint32_t chunk = std::min(n, c->pairsChunk);
    const az::HostIn in[3] = {{jd, 8}, {fr, 8}, {sat, 4}};
    const az::HostOut out[3] = {{pos, 24}, {vel, 24}, {status, 1}};
    AZ_CUDA(c->dPairsIn.reserve(az::chunk_slots_bytes(in, 3, n, chunk) / 8));
    AZ_CUDA(c->dPairsOut.reserve(az::chunk_slots_bytes(out, 3, n, chunk) / 8));
    int32_t queued = ASTROZ_OK;  // pairs_queue's own code; its message is the last error
    const cudaError_t e = c->pipe.run(
        st, c->copyStream, n, chunk, 3, in, 3, out, c->dPairsIn.p, c->dPairsOut.p,
        [&](uint32_t, uint32_t, uint32_t m, void *const *dIn, void *const *dOut, cudaStream_t s) {
            queued = pairs_queue(c, static_cast<const uint32_t *>(dIn[2]), static_cast<const double *>(dIn[0]),
                                 static_cast<const double *>(dIn[1]), m, mode, static_cast<double *>(dOut[0]),
                                 static_cast<double *>(dOut[1]), static_cast<uint8_t *>(dOut[2]), s);
            return queued == ASTROZ_OK ? cudaSuccess : cudaErrorUnknown;  // stops the run; `queued` is returned
        });
    if (queued != ASTROZ_OK) return queued;
    AZ_CUDA(e);
    return ASTROZ_OK;
}

int32_t astroz_cuda_constellation_reset_carry(astroz_constellation_t h) { return h ? ASTROZ_OK : ASTROZ_NULL_POINTER; }

int32_t astroz_cuda_constellation_synchronize(astroz_constellation_t h) {
    if (!h) return ASTROZ_NULL_POINTER;
    Constellation *c = static_cast<Constellation *>(h);
    if (c->multi()) {
        for (Constellation *sh : c->shards) {
            const int32_t rc = astroz_cuda_constellation_synchronize(sh);
            if (rc != ASTROZ_OK) return rc;
        }
        return ASTROZ_OK;
    }
    if (!c->stream) return ASTROZ_OK;
    AZ_CUDA(cudaSetDevice(c->device));
    AZ_CUDA(cudaStreamSynchronize(c->stream));
    AZ_CUDA(cudaStreamSynchronize(c->copyStream));
    return ASTROZ_OK;
}

int32_t astroz_cuda_constellation_set_timing(astroz_constellation_t h, int32_t enabled) {
    if (!h) return ASTROZ_NULL_POINTER;
    Constellation *c = static_cast<Constellation *>(h);
    c->timing = enabled != 0;
    time_begin(c);
    for (Constellation *sh : c->shards) {
        sh->timing = c->timing;
        time_begin(sh);
    }
    return ASTROZ_OK;
}

int32_t astroz_cuda_constellation_last_kernel_ms(astroz_constellation_t h, float ms[3]) {
    if (!h || !ms) return ASTROZ_NULL_POINTER;
    Constellation *c = static_cast<Constellation *>(h);
    ms[0] = ms[1] = ms[2] = 0.f;
    if (c->multi()) {  // the devices run side by side: the slowest one is the call's kernel time
        for (Constellation *sh : c->shards) {
            float one[3];
            const int32_t rc = astroz_cuda_constellation_last_kernel_ms(sh, one);
            if (rc != ASTROZ_OK) return rc;
            for (int k = 0; k < 3; ++k) ms[k] = std::max(ms[k], one[k]);
        }
        return ASTROZ_OK;
    }
    if (!c->timedSet) return ASTROZ_NOT_INITIALIZED;
    AZ_CUDA(cudaSetDevice(c->device));
    float t[3] = {0.f, 0.f, 0.f};  // by TimedSpan; 0 for a span the call did not time
    for (int k = 0; k < 3; ++k)
        if (c->timedSet & (1u << k)) {
            AZ_CUDA(cudaEventSynchronize(c->ev[k][1]));
            AZ_CUDA(cudaEventElapsedTime(&t[k], c->ev[k][0], c->ev[k][1]));
        }
    ms[0] = t[kTimeK1];
    ms[2] = t[kTimeK2];
    // the two grids of a mixed call overlap: ms[1] is the span of the whole call where one was timed
    ms[1] = (c->timedSet & (1u << kTimeSpan)) ? t[kTimeSpan] : ms[0] + ms[2];
    if (c->timedSet == (1u << kTimeSpan)) ms[0] = ms[2] = ms[1];  // a host-buffer call times its span only
    return ASTROZ_OK;
}

// ---- stateless near-earth path -----------------------------------------------------------------
static int32_t sgp4_into_common(Constellation *c, const double *times, uint32_t nt, const double *epoch_offsets,
                                double *dPos, double *dVel, int mode, double reference_jd, int layout, cudaStream_t s,
                                uint32_t recStride = 3, const uint8_t *mask = nullptr, uint32_t outNumSats = 0) {
    const uint32_t ns = c->cat.nSgp4;
    const int32_t rc = stage_stateless_axis(c, times, nt, epoch_offsets, mode, reference_jd, s);
    if (rc != ASTROZ_OK) return rc;
    az::GridArgs a = near_pass(c, c->dToffCall.p, c->dIdentity.p);  // satellite i -> row i, src/Constellation.zig:561-565
    a.nTimes = nt;
    a.pos = dPos;
    a.vel = dVel;
    a.outNumSats = outNumSats ? outNumSats : ns;
    a.recStride = recStride;
    if (mask) {  // pageable host bytes: the copy is staged by the driver before the call returns
        AZ_CUDA(c->dMask.reserve(ns));
        AZ_CUDA(cudaMemcpyAsync(c->dMask.p, mask, ns, cudaMemcpyHostToDevice, s));
        a.mask = c->dMask.p;
    }
    return timed_pass(c, kTimeK1, s, [&] { return az::launch_sgp4_grid(a, mode, layout, s, c->variant); });
}

int32_t astroz_cuda_sgp4_propagate_into_device(astroz_constellation_t h, const double *times, uint32_t n_times,
                                               const double *epoch_offsets, double *d_pos, double *d_vel, int32_t mode,
                                               double reference_jd, int32_t layout, const uint8_t *satellite_mask,
                                               uint32_t out_num_sats, void *stream) {
    Constellation *c = static_cast<Constellation *>(h);
    int32_t rc = refuse_multi(c);
    if (rc == ASTROZ_OK) rc = check_args(c, times, epoch_offsets, d_pos, mode, layout);
    if (rc != ASTROZ_OK) return rc;
    if (n_times == 0 || c->cat.nSgp4 == 0) return ASTROZ_OK;
    if (out_num_sats && out_num_sats < c->cat.nSgp4) {
        g_lastError = "out_num_sats smaller than the number of near-earth satellites";
        return ASTROZ_VALUE_ERROR;
    }
    AZ_CUDA(cudaSetDevice(c->device));
    cudaStream_t s = call_stream(c, stream);
    return sgp4_into_common(c, times, n_times, epoch_offsets, d_pos, d_vel, mode, reference_jd, layout, s, 3,
                            satellite_mask, out_num_sats);
}

// Host-buffer form of the stateless near-earth path, in queue / wait halves like propagate_host_queue.  Near-earth
// satellite i of this handle lands in row rowOffset + i of a host block with `rows` rows; epoch_offsets / mask are
// already offset to this handle's first satellite.
static int32_t sgp4_into_host_queue(Constellation *c, const double *times, uint32_t n_times, const double *epoch_offsets,
                                    double *pos, double *vel, int32_t mode, double reference_jd, int32_t layout,
                                    const uint8_t *mask, uint32_t rows, uint32_t rowOffset) {
    const uint32_t ns = c->cat.nSgp4;
    if (n_times == 0 || ns == 0) return ASTROZ_OK;
    AZ_CUDA(cudaSetDevice(c->device));
    cudaStream_t s = c->stream;
    // the near-earth rows are computed as a dense (ns, n_times) block on the device and placed in the caller's
    // (possibly wider) block; rows that belong to other satellites are never touched
    const size_t dense = (size_t)ns * n_times * 3;
    AZ_CUDA(c->dPos.reserve(dense));
    if (vel) AZ_CUDA(c->dVel.reserve(dense));
    double *dVel = vel ? c->dVel.p : nullptr;
    const HostRows at = host_rows(layout, rowOffset, ns, rows, 0, n_times, n_times);
    if (mask) {  // masked rows must keep the caller's contents: stage the caller's rows, overwrite the active ones
        for (int which = 0; which < (vel ? 2 : 1); ++which) {
            double *dst = which ? dVel : c->dPos.p;
            const double *src = (which ? vel : pos) + at.at;
            if (at.pitch == at.rowBytes) AZ_CUDA(cudaMemcpyAsync(dst, src, dense * 8, cudaMemcpyHostToDevice, s));
            else AZ_CUDA(cudaMemcpy2DAsync(dst, at.rowBytes, src, at.pitch, at.rowBytes, at.rows, cudaMemcpyHostToDevice,
                                           s));
        }
    }
    const int32_t rc = sgp4_into_common(c, times, n_times, epoch_offsets, c->dPos.p, dVel, mode, reference_jd, layout, s,
                                        3, mask, ns);
    if (rc != ASTROZ_OK) return rc;
    c->pipe.ring.discard();
    return place_rows(c, c->chunkDone[0], c->dPos.p, dVel, pos, vel, at);
}

int32_t astroz_cuda_sgp4_propagate_into(astroz_constellation_t h, const double *times, uint32_t n_times,
                                        const double *epoch_offsets, double *pos, double *vel, int32_t mode,
                                        double reference_jd, int32_t layout, const uint8_t *satellite_mask,
                                        uint32_t out_num_sats) {
    Constellation *c = static_cast<Constellation *>(h);
    int32_t rc = check_args(c, times, epoch_offsets, pos, mode, layout);
    if (rc != ASTROZ_OK) return rc;
    const uint32_t ns = c->cat.nSgp4;
    if (n_times == 0 || ns == 0) return ASTROZ_OK;
    const uint32_t rows = out_num_sats ? out_num_sats : ns;
    if (rows < ns) {
        g_lastError = "out_num_sats smaller than the number of near-earth satellites";
        return ASTROZ_VALUE_ERROR;
    }
    return queue_and_wait(c, [&](Constellation *sh, uint32_t, uint32_t near0) {
        return sgp4_into_host_queue(sh, times, n_times, epoch_offsets + near0, pos, vel, mode, reference_jd, layout,
                                    satellite_mask ? satellite_mask + near0 : nullptr, rows, near0);
    });
}

int32_t astroz_cuda_sgp4_screen(astroz_constellation_t h, const double *times, uint32_t n_times,
                                const double *epoch_offsets, uint32_t target_idx, double threshold,
                                double reference_jd, double *out_min_dists, uint32_t *out_min_t) {
    Constellation *c = static_cast<Constellation *>(h);
    if (const int32_t rc = refuse_multi(c); rc != ASTROZ_OK) return rc;
    if (!c || !times || !epoch_offsets || !out_min_dists || !out_min_t) return ASTROZ_NULL_POINTER;
    const uint32_t ns = c->cat.nSgp4;
    if (ns == 0 || n_times == 0) return ASTROZ_OK;
    if (target_idx >= ns) {
        g_lastError = "target index out of range";
        return ASTROZ_VALUE_ERROR;
    }
    AZ_CUDA(cudaSetDevice(c->device));
    cudaStream_t s = c->stream;
    int32_t rc = stage_stateless_axis(c, times, n_times, epoch_offsets, ASTROZ_MODE_TEME, reference_jd, s);
    if (rc != ASTROZ_OK) return rc;
    // scratch: target track [nt][3] | minDist [ns] | minT [ns] (as doubles' worth of space)
    AZ_CUDA(c->dPos.reserve((size_t)n_times * 3 + 2 * (size_t)ns + 2));
    az::ScreenArgs a;
    a.sgp4Tiles = c->dTiles.p;
    a.toff = c->dToffCall.p;
    a.tbase = time_col(c, 0);
    a.nSats = ns;
    a.nTimes = n_times;
    a.targetIdx = target_idx;
    a.thresholdSq = threshold * threshold;
    a.track = c->dPos.p;
    a.minDist = c->dPos.p + (size_t)n_times * 3;
    a.minT = reinterpret_cast<uint32_t *>(a.minDist + ns);
    a.g = c->g;
    rc = timed_pass(c, kTimeK1, s, [&] { return az::launch_sgp4_screen(a, s); });
    if (rc != ASTROZ_OK) return rc;
    AZ_CUDA(cudaMemcpyAsync(out_min_dists, a.minDist, (size_t)ns * 8, cudaMemcpyDeviceToHost, s));
    AZ_CUDA(cudaMemcpyAsync(out_min_t, a.minT, (size_t)ns * 4, cudaMemcpyDeviceToHost, s));
    AZ_CUDA(cudaStreamSynchronize(s));
    return ASTROZ_OK;
}

// ---- all-vs-all coarse screen ----------------------------------------------------------------------
static int32_t coarse_screen_run(Constellation *c, const double *dPositions, uint32_t ns, uint32_t nt, int layout,
                                 double threshold, const uint8_t *dMask, uint32_t *dPairs, uint32_t *dT,
                                 uint32_t maxResults, uint64_t *count, cudaStream_t s) {
    constexpr uint32_t kBits = 16, kBatch = 128;  // 128 epochs per pass: 32 MB of bucket heads
    const uint32_t batch = std::min(kBatch, nt);
    AZ_CUDA(c->dHead.reserve((size_t)batch << kBits));
    AZ_CUDA(c->dNext.reserve((size_t)batch * ns));
    AZ_CUDA(c->dCount.reserve(1));
    AZ_CUDA(cudaMemsetAsync(c->dCount.p, 0, 8, s));
    for (uint32_t t0 = 0; t0 < nt; t0 += batch) {
        az::CoarseArgs a;
        a.pos = dPositions;
        a.validMask = dMask;
        a.nSats = ns;
        a.nTimes = nt;
        a.layout = layout;
        a.threshold = threshold;
        a.t0 = t0;
        a.tCount = std::min(batch, nt - t0);
        a.tableBits = kBits;
        a.head = c->dHead.p;
        a.next = c->dNext.p;
        a.pairs = dPairs;
        a.tIdx = dT;
        a.maxResults = maxResults;
        a.count = c->dCount.p;
        AZ_CUDA(az::launch_coarse_screen(a, s));
    }
    unsigned long long found = 0;
    AZ_CUDA(cudaMemcpyAsync(&found, c->dCount.p, 8, cudaMemcpyDeviceToHost, s));
    AZ_CUDA(cudaStreamSynchronize(s));
    *count = found;
    return ASTROZ_OK;
}

int32_t astroz_cuda_constellation_coarse_screen_device(astroz_constellation_t h, const double *d_positions,
                                                       uint32_t num_sats, uint32_t num_times, int32_t layout,
                                                       double threshold, const uint8_t *d_valid_mask, uint32_t *d_pairs,
                                                       uint32_t *d_t_indices, uint32_t max_results, uint64_t *count) {
    Constellation *c = static_cast<Constellation *>(h);
    if (const int32_t rc = refuse_multi(c); rc != ASTROZ_OK) return rc;
    if (!c || !d_positions || !count || (max_results && (!d_pairs || !d_t_indices))) return ASTROZ_NULL_POINTER;
    if (layout < 0 || layout > 1 || !(threshold > 0.0)) {
        g_lastError = "coarse screen: layout must be 0/1 and threshold positive";
        return ASTROZ_VALUE_ERROR;
    }
    *count = 0;
    if (num_sats == 0 || num_times == 0) return ASTROZ_OK;
    AZ_CUDA(cudaSetDevice(c->device));
    return coarse_screen_run(c, d_positions, num_sats, num_times, layout, threshold, d_valid_mask, d_pairs, d_t_indices,
                             max_results, count, c->stream);
}

int32_t astroz_cuda_sgp4_screen_all(astroz_constellation_t h, const double *times, uint32_t n_times,
                                    const double *epoch_offsets, double threshold, uint32_t *pairs, uint32_t *t_indices,
                                    uint32_t max_results, uint64_t *count) {
    Constellation *c = static_cast<Constellation *>(h);
    if (const int32_t rc = refuse_multi(c); rc != ASTROZ_OK) return rc;
    if (!c || !times || !epoch_offsets || !count || (max_results && (!pairs || !t_indices))) return ASTROZ_NULL_POINTER;
    if (!(threshold > 0.0)) return ASTROZ_VALUE_ERROR;
    *count = 0;
    const uint32_t ns = c->cat.nSgp4;
    if (ns == 0 || n_times == 0) return ASTROZ_OK;
    AZ_CUDA(cudaSetDevice(c->device));
    cudaStream_t s = c->stream;
    AZ_CUDA(c->dPos.reserve((size_t)ns * n_times * 3));
    // positions only, time-major: a warp of the screen kernels then reads 32 neighbouring satellites of one epoch
    int32_t rc = sgp4_into_common(c, times, n_times, epoch_offsets, c->dPos.p, nullptr, ASTROZ_MODE_TEME, 0.0,
                                  ASTROZ_LAYOUT_TIME_MAJOR, s);
    if (rc != ASTROZ_OK) return rc;
    AZ_CUDA(c->dPairs.reserve((size_t)std::max<uint32_t>(max_results, 1) * 2));
    AZ_CUDA(c->dTIdx.reserve(std::max<uint32_t>(max_results, 1)));
    rc = coarse_screen_run(c, c->dPos.p, ns, n_times, ASTROZ_LAYOUT_TIME_MAJOR, threshold, nullptr, c->dPairs.p,
                           c->dTIdx.p, max_results, count, s);
    if (rc != ASTROZ_OK) return rc;
    const size_t stored = (size_t)std::min<uint64_t>(*count, max_results);
    if (stored) {
        AZ_CUDA(cudaMemcpyAsync(pairs, c->dPairs.p, stored * 8, cudaMemcpyDeviceToHost, s));
        AZ_CUDA(cudaMemcpyAsync(t_indices, c->dTIdx.p, stored * 4, cudaMemcpyDeviceToHost, s));
        AZ_CUDA(cudaStreamSynchronize(s));
    }
    return ASTROZ_OK;
}

// ---- single satellite ----------------------------------------------------------------------------
int32_t astroz_cuda_sgp4_init(const char *line1, const char *line2, int32_t grav, int32_t device, astroz_sgp4_t *out) {
    if (!line1 || !line2 || !out) return ASTROZ_NULL_POINTER;
    *out = nullptr;
    // python-sgp4 style code builds thousands of Satrec objects only to hand them to a SatrecArray: parsing and
    // classification happen here, on the host; device resources come with the first propagation of THIS satellite.
    const int32_t drc = check_device_ordinal(device);
    if (drc != ASTROZ_OK) return drc;
    std::unique_ptr<Sgp4Single> s(new (std::nothrow) Sgp4Single());
    if (!s) return ASTROZ_ALLOC_FAILED;
    s->c.reset(new (std::nothrow) Constellation());
    if (!s->c) return ASTROZ_ALLOC_FAILED;
    const char *l1[1] = {line1}, *l2[1] = {line2};
    const int brc = az::build_catalog(l1, l2, 1, grav, s->c->cat);
    if (brc != az::kOk) return status_to_code(brc);
    s->device = device;
    s->epochJd = s->c->cat.epochs[0];
    s->deep = s->c->cat.nSdp4 == 1;
    {  // mean elements for the python-sgp4 attribute getters (bindings/python/src/satrec.zig:395-470)
        az::TleRecord t;
        az::NearEarth ne;
        double period = 0.0, perigee = 0.0;
        if (az::parse_tle(line1, line2, t) == az::kOk &&
            az::build_common(t, az::gravity(grav), ne, period, perigee) == az::kOk) {
            const double e[10] = {ne.ecco, ne.inclo, ne.nodeo, ne.argpo, ne.mo, ne.no_kozai, ne.bstar, ne.a, ne.no, ne.epochJd};
            std::memcpy(s->elements, e, sizeof e);
        }
    }
    *out = s.release();
    return ASTROZ_OK;
}

static int32_t ensure_open(Sgp4Single *s) {
    if (s->opened) return ASTROZ_OK;
    const int32_t rc = finish_create(s->c.get(), s->device);
    if (rc == ASTROZ_OK) s->opened = true;
    return rc;
}

int32_t astroz_cuda_sgp4_elements(astroz_sgp4_t h, double *out10) {
    if (!h || !out10) return ASTROZ_NULL_POINTER;
    std::memcpy(out10, static_cast<Sgp4Single *>(h)->elements, sizeof(double) * 10);
    return ASTROZ_OK;
}

void astroz_cuda_sgp4_free(astroz_sgp4_t h) { delete static_cast<Sgp4Single *>(h); }

int32_t astroz_cuda_sgp4_is_deep_space(astroz_sgp4_t h) { return h && static_cast<Sgp4Single *>(h)->deep ? 1 : 0; }

int32_t astroz_cuda_sgp4_epoch(astroz_sgp4_t h, double *epoch_jd) {
    if (!h || !epoch_jd) return ASTROZ_NULL_POINTER;
    *epoch_jd = static_cast<Sgp4Single *>(h)->epochJd;
    return ASTROZ_OK;
}

int32_t astroz_cuda_sgp4_propagate_batch(astroz_sgp4_t h, const double *times, double *results, uint32_t count) {
    Sgp4Single *s = static_cast<Sgp4Single *>(h);
    if (!s || !times || !results) return ASTROZ_NULL_POINTER;
    if (count == 0) return ASTROZ_OK;
    {
        const int32_t orc = ensure_open(s);
        if (orc != ASTROZ_OK) return orc;
    }
    Constellation *c = s->c.get();
    AZ_CUDA(cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const size_t n3 = (size_t)count * 3;
    AZ_CUDA(c->dPos.reserve(2 * n3));
    double *dPos = c->dPos.p, *dVel = c->dPos.p + n3;
    const double zero = 0.0;
    if (!s->deep && count >= 64) {
        // the time-parallel kernel (K1t) writes x y z vx vy vz records straight into one block that is copied to
        // `results` in a single transfer (src/c_api/sgp4.zig:60-100 layout)
        const int32_t rc = sgp4_into_common(c, times, count, &zero, dPos, dPos + 3, ASTROZ_MODE_TEME, 0.0,
                                            ASTROZ_LAYOUT_SATELLITE_MAJOR, st, 6);
        if (rc != ASTROZ_OK) return rc;
        AZ_CUDA(cudaMemcpyAsync(results, dPos, n3 * 16, cudaMemcpyDeviceToHost, st));
        AZ_CUDA(cudaStreamSynchronize(st));
        return ASTROZ_OK;
    }
    // a position block and a velocity block, interleaved into records here: below 64 epochs K1 runs one epoch per
    // thread instead of K1t's two (the series a cell takes, and so its bits, may differ between the two)
    DevBuf<uint8_t> dSt;
    std::vector<uint8_t> cell;
    if (!s->deep) {
        const int32_t rc = sgp4_into_common(c, times, count, &zero, dPos, dVel, ASTROZ_MODE_TEME, 0.0,
                                            ASTROZ_LAYOUT_SATELLITE_MAJOR, st);
        if (rc != ASTROZ_OK) return rc;
    } else {
        // deep space: minutes since epoch go to the kernel directly (no Julian-date round trip)
        double *tb;
        int32_t rc = time_slot(c, count, &tb);
        if (rc != ASTROZ_OK) return rc;
        double reach = 0.0;
        for (uint32_t i = 0; i < count; ++i) {
            tb[i] = times[i];
            reach = std::max(reach, std::fabs(times[i]));
        }
        rc = upload_time_slot(c, count, 0x1u, st);
        if (rc != ASTROZ_OK) return rc;
        rc = ensure_lattice(c, (int)std::floor(reach / az::kStepp) + 2, st);
        if (rc != ASTROZ_OK) return rc;
        AZ_CUDA(dSt.reserve(count));
        az::GridArgs a = deep_pass(c, c->dSdp4Orig.p);
        a.tsince = time_col(c, 0);
        a.nTimes = count;
        a.pos = dPos;
        a.vel = dVel;
        a.status = dSt.p;
        a.outNumSats = 1;
        cell.resize(count);
        AZ_CUDA(az::launch_sdp4_grid(a, ASTROZ_MODE_TEME, ASTROZ_LAYOUT_SATELLITE_MAJOR, st));
        AZ_CUDA(cudaMemcpyAsync(cell.data(), dSt.p, count, cudaMemcpyDeviceToHost, st));
    }
    std::vector<double> pv(2 * n3);
    AZ_CUDA(cudaMemcpyAsync(pv.data(), dPos, 2 * n3 * 8, cudaMemcpyDeviceToHost, st));
    AZ_CUDA(cudaStreamSynchronize(st));
    int32_t rc = ASTROZ_OK;
    for (uint8_t code : cell)
        if (code != 0) rc = status_to_code(code);  // failing cells stay zero-filled; last failure reported
    for (uint32_t i = 0; i < count; ++i) {
        double *r = results + (size_t)i * 6;
        const double *p = pv.data() + (size_t)i * 3, *v = p + n3;
        r[0] = p[0]; r[1] = p[1]; r[2] = p[2];
        r[3] = v[0]; r[4] = v[1]; r[5] = v[2];
    }
    return rc;
}

int32_t astroz_cuda_sgp4_array(astroz_sgp4_t h, const double *jd, const double *fr, double epoch_jd, double *results,
                               uint32_t count) {
    Sgp4Single *s = static_cast<Sgp4Single *>(h);
    if (!s || !jd || !fr || !results) return ASTROZ_NULL_POINTER;
    if (count == 0) return ASTROZ_OK;
    {
        const int32_t orc = ensure_open(s);
        if (orc != ASTROZ_OK) return orc;
    }
    Constellation *c = s->c.get();
    if (s->deep || count < 64) {  // deep space / tiny: host-side tsince, then the batch entry point
        std::vector<double> ts(count);
        for (uint32_t i = 0; i < count; ++i) ts[i] = ((jd[i] + fr[i]) - epoch_jd) * 1440.0;
        return astroz_cuda_sgp4_propagate_batch(h, ts.data(), results, count);
    }
    AZ_CUDA(cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    c->cacheValid = false;  // dTime holds [jd | fr] slots here
    // A long axis ("1 year at one second" = 31.5 M epochs: 0.5 GB of jd/fr in, 1.5 GB of records out) is cut into
    // chunks on the handle's two-slot pipeline (az::ChunkPipeline): while chunk k is propagated, chunk k+1's epochs
    // are staged and uploaded and chunk k-1's records travel back, so the call runs at the PCIe rate of its 48 B/epoch
    // result instead of the sum of three serial phases.  jd / fr usually are pageable (numpy) and go up through the
    // pinned ring; pageable results come back through it too, in ring-sized pieces.
    constexpr uint32_t kChunk = 1u << 21;   // epochs per chunk: 32 MB of epochs, 96 MB of records
    const uint32_t nChunks = (count + kChunk - 1) / kChunk;
    const uint32_t chunk = ((count + nChunks - 1) / nChunks + 31) / 32 * 32;   // balanced: no short last chunk
    const az::HostIn in[2] = {{jd, 8}, {fr, 8}};
    const az::HostOut out[1] = {{results, 48}};
    AZ_CUDA(c->dTime.reserve(az::chunk_slots_bytes(in, 2, count, chunk) / 8));
    AZ_CUDA(c->dPos.reserve(az::chunk_slots_bytes(out, 1, count, chunk) / 8));
    auto launch = [&](uint32_t k, uint32_t t0, uint32_t n, void *const *dIn, void *const *dOut, cudaStream_t s) {
        double *dJd = static_cast<double *>(dIn[0]), *dRec = static_cast<double *>(dOut[0]);
        az::GridArgs a = near_pass(c, c->dToff.p, c->dIdentity.p);
        a.jdArr = dJd;
        a.frArr = static_cast<double *>(dIn[1]);
        a.epochJd = epoch_jd;
        a.nTimes = n;
        a.pos = dRec;
        a.vel = dRec + 3;
        a.outNumSats = 1;
        a.recStride = 6;
        // K1's span: from before the first chunk's kernel to after the last one's
        cudaError_t e = k == 0 ? time_mark(c, kTimeK1, false, s) : cudaSuccess;
        if (e == cudaSuccess)
            e = az::launch_sgp4_grid(a, ASTROZ_MODE_TEME, ASTROZ_LAYOUT_SATELLITE_MAJOR, s, c->variant);
        if (e == cudaSuccess && t0 + n == count) e = time_mark(c, kTimeK1, true, s);
        return e;
    };
    time_begin(c);
    AZ_CUDA(c->pipe.run(st, c->copyStream, count, chunk, 2, in, 1, out, c->dTime.p, c->dPos.p, launch));
    return ASTROZ_OK;
}

int32_t astroz_cuda_sgp4_propagate(astroz_sgp4_t h, double tsince, double pos[3], double vel[3]) {
    if (!h || !pos || !vel) return ASTROZ_NULL_POINTER;
    double r[6];
    int32_t rc = astroz_cuda_sgp4_propagate_batch(h, &tsince, r, 1);
    std::memcpy(pos, r, 24);
    std::memcpy(vel, r + 3, 24);
    return rc;
}

// ---- result blocks placed next to the GPUs that fill them ---------------------------------------------------------
// A multi-device handle writes one host block from several GPUs at once.  A plain pinned allocation sits on the NUMA
// node of the thread that made it, so half the GPUs of a two-socket box write across the socket interconnect and all of
// them into one node's memory controllers.  astroz_cuda_constellation_host_block maps the block anonymously, binds each device's slice of a
// satellite-major block to the NUMA node of that device (mbind), touches it, and page-locks the whole range.
static int device_numa_node(int device) {
    char bus[32] = {};
    if (cudaDeviceGetPCIBusId(bus, sizeof bus, device) != cudaSuccess) {
        (void)cudaGetLastError();
        return -1;
    }
    for (char *p = bus; *p; ++p) *p = (char)std::tolower(*p);
    const std::string path = std::string("/sys/bus/pci/devices/") + bus + "/numa_node";
    FILE *f = std::fopen(path.c_str(), "r");
    if (!f) return -1;
    int node = -1;
    if (std::fscanf(f, "%d", &node) != 1) node = -1;
    std::fclose(f);
    return node;
}

static void bind_to_node(char *begin, char *end, int node) {
#ifdef SYS_mbind
    if (node < 0 || node >= 64) return;
    const long page = sysconf(_SC_PAGESIZE);
    char *b = reinterpret_cast<char *>((reinterpret_cast<uintptr_t>(begin) + page - 1) / page * page);
    char *e = reinterpret_cast<char *>(reinterpret_cast<uintptr_t>(end) / page * page);
    if (e <= b) return;
    unsigned long mask = 1ul << node;
    (void)syscall(SYS_mbind, b, (unsigned long)(e - b), 2 /* MPOL_BIND */, &mask, 64ul, 0u);  // best effort
#else
    (void)begin; (void)end; (void)node;
#endif
}

int32_t astroz_cuda_constellation_host_block(astroz_constellation_t h, uint32_t n_times, int32_t layout, double **out) {
    if (!h || !out) return ASTROZ_NULL_POINTER;
    *out = nullptr;
    Constellation *c = static_cast<Constellation *>(h);
    const size_t bytes = std::max<size_t>((size_t)c->cat.n * n_times * 24, 4096);
    void *p = mmap(nullptr, bytes, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
    if (p == MAP_FAILED) return ASTROZ_ALLOC_FAILED;
    char *base = static_cast<char *>(p);
    if (c->multi() && layout == ASTROZ_LAYOUT_SATELLITE_MAJOR) {
        for (size_t k = 0; k < c->shards.size(); ++k)
            bind_to_node(base + (size_t)c->shardRow0[k] * n_times * 24, base + (size_t)c->shardRow0[k + 1] * n_times * 24,
                         device_numa_node(c->shards[k]->device));
    } else if (!c->multi()) {
        bind_to_node(base, base + bytes, device_numa_node(c->device));
    }   // time-major over several devices: rows interleave, the default (first-touch) placement stays
    {   // touch every page so the placement happens now, on the bound node, not at the first DMA
        const long page = sysconf(_SC_PAGESIZE);
        for (size_t o = 0; o < bytes; o += (size_t)page) base[o] = 0;
    }
    const cudaError_t e = cudaHostRegister(p, bytes, cudaHostRegisterPortable);
    if (e != cudaSuccess) {
        munmap(p, bytes);
        return cuda_fail(e, "cudaHostRegister");
    }
    {
        std::lock_guard<std::mutex> g(g_blockMutex);
        g_blocks[p] = bytes;
    }
    *out = static_cast<double *>(p);
    return ASTROZ_OK;
}

// ---- caller-owned buffers: explicit page-locking ------------------------------------------------------------
int32_t astroz_cuda_host_register(void *p, size_t bytes) {
    if (!p) return ASTROZ_NULL_POINTER;
    AZ_CUDA(cudaHostRegister(p, bytes, cudaHostRegisterPortable));
    return ASTROZ_OK;
}
int32_t astroz_cuda_host_unregister(void *p) {
    if (!p) return ASTROZ_NULL_POINTER;
    AZ_CUDA(cudaHostUnregister(p));
    return ASTROZ_OK;
}

// ---- multi-device handles --------------------------------------------------------------------------------
int32_t astroz_cuda_constellation_devices(astroz_constellation_t h, int32_t *n_devices, int32_t *device_ids,
                                          uint32_t *first_rows) {
    if (!h || !n_devices) return ASTROZ_NULL_POINTER;
    Constellation *c = static_cast<Constellation *>(h);
    if (!c->multi()) {
        *n_devices = 1;
        if (device_ids) device_ids[0] = c->device;
        if (first_rows) { first_rows[0] = 0; first_rows[1] = c->cat.n; }
        return ASTROZ_OK;
    }
    *n_devices = (int32_t)c->shards.size();
    for (size_t k = 0; k < c->shards.size(); ++k) {
        if (device_ids) device_ids[k] = c->shards[k]->device;
        if (first_rows) first_rows[k] = c->shardRow0[k];
    }
    if (first_rows) first_rows[c->shards.size()] = c->cat.n;
    return ASTROZ_OK;
}

// Peer mappings between every pair of distinct devices of the handle (cudaMalloc memory of one is then directly
// addressable from kernels on the other: NVLink loads/stores).  Idempotent.
static int32_t enable_peers(Constellation *c) {
    for (Constellation *a : c->shards)
        for (Constellation *b : c->shards) {
            if (a->device == b->device) continue;
            int can = 0;
            AZ_CUDA(cudaDeviceCanAccessPeer(&can, a->device, b->device));
            if (!can) {
                g_lastError = "devices " + std::to_string(a->device) + " and " + std::to_string(b->device) +
                              " have no peer access (no NVLink / P2P path)";
                return ASTROZ_CUDA_ERROR;
            }
            AZ_CUDA(cudaSetDevice(a->device));
            const cudaError_t e = cudaDeviceEnablePeerAccess(b->device, 0);
            if (e == cudaErrorPeerAccessAlreadyEnabled) (void)cudaGetLastError();
            else if (e != cudaSuccess) return cuda_fail(e, "cudaDeviceEnablePeerAccess");
        }
    return ASTROZ_OK;
}

int32_t astroz_cuda_constellation_propagate_replicated(astroz_constellation_t h, const double *jd, const double *fr,
                                                       uint32_t n_times, int32_t velocities, double **d_pos,
                                                       double **d_vel) {
    Constellation *c = static_cast<Constellation *>(h);
    if (!c || !jd || !fr || !d_pos || (velocities && !d_vel)) return ASTROZ_NULL_POINTER;
    const uint32_t n = c->cat.n;
    const size_t total = (size_t)n * n_times * 3;
    if (!c->multi()) {  // one device: the block is simply left in HBM
        if (n_times == 0 || n == 0) return ASTROZ_OK;
        AZ_CUDA(cudaSetDevice(c->device));
        AZ_CUDA(c->dFullPos.reserve(total));
        if (velocities) AZ_CUDA(c->dFullVel.reserve(total));
        int32_t rc = astroz_cuda_constellation_propagate_device(c, jd, fr, n_times, c->dFullPos.p,
                                                                velocities ? c->dFullVel.p : nullptr, nullptr,
                                                                ASTROZ_MODE_TEME, ASTROZ_LAYOUT_SATELLITE_MAJOR, n, 0, nullptr);
        if (rc != ASTROZ_OK) return rc;
        AZ_CUDA(cudaStreamSynchronize(c->stream));
        d_pos[0] = c->dFullPos.p;
        if (velocities) d_vel[0] = c->dFullVel.p;
        return ASTROZ_OK;
    }
    if (n_times == 0 || n == 0) return ASTROZ_OK;
    int32_t rc = enable_peers(c);
    if (rc != ASTROZ_OK) return rc;
    const size_t ns = c->shards.size();
    if (ns > (size_t)az::kMaxPeers) {
        g_lastError = "at most 8 devices (one NVSwitch domain)";
        return ASTROZ_VALUE_ERROR;
    }
    for (Constellation *sh : c->shards) {  // every device holds the whole block
        AZ_CUDA(cudaSetDevice(sh->device));
        AZ_CUDA(sh->dFullPos.reserve(total));
        if (velocities) AZ_CUDA(sh->dFullVel.reserve(total));
    }
    void *pp[az::kMaxPeers] = {}, *pv[az::kMaxPeers] = {};
    for (size_t k = 0; k < ns; ++k) {
        pp[k] = c->shards[k]->dFullPos.p;
        pv[k] = velocities ? c->shards[k]->dFullVel.p : nullptr;
    }
    // one fused launch per device: its rows are stored, run by run, into every device's copy of the block
    int32_t first = ASTROZ_OK;
    for (size_t k = 0; k < ns; ++k) {
        rc = astroz_cuda_constellation_propagate_gather(c->shards[k], jd, fr, n_times, pp, velocities ? pv : nullptr,
                                                        (uint32_t)ns, nullptr, nullptr, n, c->shardRow0[k], nullptr);
        if (rc != ASTROZ_OK && first == ASTROZ_OK) first = rc;
    }
    for (size_t k = 0; k < ns; ++k) {  // all stores have landed once every device's stream has drained
        rc = propagate_host_wait(c->shards[k]);
        if (rc != ASTROZ_OK && first == ASTROZ_OK) first = rc;
        d_pos[k] = c->shards[k]->dFullPos.p;
        if (velocities) d_vel[k] = c->shards[k]->dFullVel.p;
    }
    return first;
}

// ---- numerical propagation (K7, az_numerical.cu) -------------------------------------------------------------------
// ASTROZ_VALUE_ERROR with `why` as the last error: the argument checks' refusal
static int32_t value_error(const char *why) {
    g_lastError = why;
    return ASTROZ_VALUE_ERROR;
}
// The sampling rule of Propagator.propagate (src/propagators/Propagator.zig:32-45), stated here and nowhere else:
//   t = t0; t_end = t0 + duration; while (t < t_end) { step = min(dt, t_end - t); ...; t += step; }
// *count = samples (the initial state plus one per step); times (nullable) receives the sample times, table (nullable)
// the step sizes K7 integrates over.  Nothing is allocated.  A loop that would not end (t + step == t) or run more than
// kMaxNumSteps steps, and non-finite or non-positive inputs, are ASTROZ_VALUE_ERROR.
static constexpr uint64_t kMaxNumSteps = 0xfffffffeull;  // K7 counts intervals in 32 bits
static int32_t numerical_schedule(double t0, double duration, double dt, double *times, az::StepTable *table,
                                  uint64_t *count) {
    const double tEnd = t0 + duration;
    if (!std::isfinite(t0) || !std::isfinite(duration) || !std::isfinite(dt) || !std::isfinite(tEnd) || !(dt > 0.0))
        return value_error("t0, duration and dt must be finite and dt > 0");
    if (duration / dt > (double)kMaxNumSteps) return value_error("duration / dt exceeds the step limit");
    if (table) *table = az::StepTable{dt, 0, 0, {}};
    double t = t0;
    uint64_t k = 0;
    if (times) times[0] = t;
    while (t < tEnd) {
        const double step = std::min(dt, tEnd - t);
        if (t + step == t || ++k > kMaxNumSteps)
            return value_error("the sampling loop would not end: t0 + step rounds to t0");
        if (table && !az::step_table_push(*table, step))
            return value_error("the sampling loop's steps do not fit the step table");
        t += step;
        if (times) times[k] = t;
    }
    *count = k + 1;
    return ASTROZ_OK;
}

// Argument checks of every batch call, before anything is read, written or allocated.  On success a receives n, the
// steps and the tolerances.
static int32_t numerical_check(uint32_t n, double t0, double duration, double dt, int32_t integrator, double rtol,
                               double atol, int32_t device, az::NumArgs *a) {
    if (device < 0) return value_error("numerical propagation runs on one device: pass its ordinal");
    if (integrator != az::kIntRk4 && integrator != az::kIntDp87)
        return value_error("integrator must be RK4 (0) or DP87 (1)");
    if (!std::isfinite(rtol) || !std::isfinite(atol)) return value_error("rtol and atol must be finite");
    uint64_t samples = 0;
    const int32_t rc = numerical_schedule(t0, duration, dt, nullptr, &a->steps, &samples);
    if (rc != ASTROZ_OK) return rc;
    if ((uint64_t)n * samples > SIZE_MAX / 48) return value_error("the output size overflows");
    a->n = n;
    a->p.rtol = rtol;
    a->p.atol = atol;
    return ASTROZ_OK;
}

// Checks of the fixed force set (two-body, J2, exponential drag), before anything is read, written or allocated.  On
// success p receives mu, j2 and r_eq.
static int32_t forces_check(double mu, int32_t forces, const double *j2, const double *r_eq, const double *cd,
                            const double *area, const double *mass, az::NumParams *p) {
    if (forces & ~(az::kForceJ2 | az::kForceDrag)) return value_error("unknown force bit");
    if (!std::isfinite(mu)) return value_error("mu must be finite");
    if ((forces & az::kForceJ2) && (!j2 || !std::isfinite(*j2))) return value_error("J2 needs a finite j2");
    if (forces && (!r_eq || !std::isfinite(*r_eq))) return value_error("J2 and drag need a finite r_eq");
    if ((forces & az::kForceDrag) && (!cd || !area || !mass))
        return value_error("drag needs drag_cd, drag_area and drag_mass");
    p->mu = mu;
    p->j2 = (forces & az::kForceJ2) ? *j2 : 0.0;
    p->rEq = forces ? *r_eq : 0.0;
    return ASTROZ_OK;
}

// Per-device state of the host-buffer call: its two streams and its two-slot pipeline (whose pinned ring of three 32 MB
// pieces is allocated on the first pageable transfer).  Process-wide, created on first use and never destroyed, like
// the host copy pool; a mutex serialises the calls that share it.  The device slots are not kept: each call allocates
// them stream-ordered and returns them before it returns.
struct NumericalContext {
    std::mutex m;
    cudaStream_t stream = nullptr, copyStream = nullptr;
    az::ChunkPipeline pipe;
};

static int32_t numerical_context(int device, NumericalContext **out) {
    static std::mutex created;
    static std::map<int, NumericalContext *> contexts;
    std::lock_guard<std::mutex> lk(created);
    NumericalContext *&c = contexts[device];
    if (!c) {
        std::unique_ptr<NumericalContext> fresh(new (std::nothrow) NumericalContext());
        if (!fresh) return ASTROZ_ALLOC_FAILED;
        AZ_CUDA(cudaSetDevice(device));
        AZ_CUDA(cudaStreamCreateWithFlags(&fresh->stream, cudaStreamNonBlocking));
        AZ_CUDA(cudaStreamCreateWithFlags(&fresh->copyStream, cudaStreamNonBlocking));
        AZ_CUDA(fresh->pipe.create());
        c = fresh.release();
    }
    *out = c;
    return ASTROZ_OK;
}

// A stream-ordered device allocation returned to the pool on `s` when it goes out of scope (also on an error return).
struct StreamBuf {
    void *p = nullptr;
    cudaStream_t s = nullptr;
    explicit StreamBuf(cudaStream_t stream) : s(stream) {}
    StreamBuf(const StreamBuf &) = delete;
    StreamBuf &operator=(const StreamBuf &) = delete;
    ~StreamBuf() { release(); }
    cudaError_t alloc(size_t bytes) { return cudaMallocAsync(&p, bytes, s); }
    cudaError_t release() {
        void *q = p;
        p = nullptr;
        return q ? cudaFreeAsync(q, s) : cudaSuccess;
    }
};

int32_t astroz_cuda_numerical_times(double t0, double duration, double dt, double *times, uint64_t *count) {
    if (!count) return ASTROZ_NULL_POINTER;
    uint64_t k = 0;
    int32_t rc = numerical_schedule(t0, duration, dt, nullptr, nullptr, &k);  // validate before writing anything
    if (rc == ASTROZ_OK && times) rc = numerical_schedule(t0, duration, dt, times, nullptr, &k);
    if (rc != ASTROZ_OK) return rc;
    *count = k;
    return ASTROZ_OK;
}

int32_t astroz_cuda_propagate_numerical_device(const double *d_states, uint32_t n, double t0, double duration,
                                               double dt, double mu, int32_t forces, const double *j2,
                                               const double *r_eq, const double *d_drag_cd,
                                               const double *d_drag_area, const double *d_drag_mass,
                                               int32_t integrator, double rtol, double atol, int32_t device,
                                               double *d_out, uint8_t *d_status, uint64_t *d_steps, void *stream) {
    az::NumArgs a{};
    int32_t rc = forces_check(mu, forces, j2, r_eq, d_drag_cd, d_drag_area, d_drag_mass, &a.p);
    if (rc == ASTROZ_OK) rc = numerical_check(n, t0, duration, dt, integrator, rtol, atol, device, &a);
    if (rc != ASTROZ_OK) return rc;
    if (n == 0) return ASTROZ_OK;
    if (!d_states || !d_out || !d_status) return ASTROZ_NULL_POINTER;
    if ((rc = check_device_ordinal(device)) != ASTROZ_OK) return rc;
    AZ_CUDA(cudaSetDevice(device));
    a.states = d_states;
    a.cd = d_drag_cd;
    a.area = d_drag_area;
    a.mass = d_drag_mass;
    a.out = d_out;
    a.status = d_status;
    a.counts = d_steps;
    // the step table travels in the launch's parameters: nothing is uploaded, the call only queues the kernel
    AZ_CUDA(az::launch_numerical(a, integrator, forces, static_cast<cudaStream_t>(stream)));
    return ASTROZ_OK;
}

// Host buffers: chunks of states, each chunk's trajectory block at most kNumChunkBytes (eight ring pieces), through the
// device's two-slot pipeline (az::ChunkPipeline).  `cols` are the per-state input columns the kernel reads ([n] doubles
// each; the fixed drag set has three, a model list one per per-state array it names); `tabs` are whole arrays of
// tabBytes each, uploaded once per call before the first chunk (a model list's position tables, a maneuver call's
// schedules).  The per-state results are the columns res[nRes]; rowBytes, the bytes of one state's trajectory, sizes the
// chunks.  For each chunk, launch(first, m, dStates, dRes, dCols, dTabs, s) queues the kernel.
static constexpr size_t kNumChunkBytes = 256u << 20;
static constexpr int kNumMaxCols = 3 * (int)az::kMaxModels, kNumMaxTabs = (int)az::kMaxModels;
using NumLaunch = std::function<cudaError_t(const double *const *dCols, const double *const *dTabs, cudaStream_t s)>;
// one chunk: its first state, its state count, its device states and result columns, the per-state columns and tables
using NumRowsLaunch =
    std::function<cudaError_t(uint32_t first, uint32_t m, const double *dStates, void *const *dRes,
                              const double *const *dCols, const double *const *dTabs, cudaStream_t s)>;
static int32_t numerical_host_rows(uint32_t n, const double *states, int nCols, const double *const *cols, int nTabs,
                                   const double *const *tabs, size_t tabBytes, int32_t device, int nRes,
                                   const az::HostOut *res, size_t rowBytes, const NumRowsLaunch &launch) {
    NumericalContext *c = nullptr;
    int32_t rc = numerical_context(device, &c);
    if (rc != ASTROZ_OK) return rc;
    std::lock_guard<std::mutex> lk(c->m);
    AZ_CUDA(cudaSetDevice(device));
    cudaStream_t st = c->stream;
    const uint32_t chunk = (uint32_t)std::max<size_t>(1, std::min<size_t>(n, kNumChunkBytes / rowBytes));
    az::HostIn in[1 + kNumMaxCols] = {{states, 48}};
    for (int q = 0; q < nCols; ++q) in[1 + q] = {cols[q], 8};
    StreamBuf dIn(st), dOut(st), dTab(st);
    AZ_CUDA(dIn.alloc(az::chunk_slots_bytes(in, 1 + nCols, n, chunk)));
    AZ_CUDA(dOut.alloc(az::chunk_slots_bytes(res, nRes, n, chunk)));
    const double *dTabs[kNumMaxTabs] = {};
    if (nTabs) {
        AZ_CUDA(dTab.alloc(nTabs * tabBytes));
        for (int t = 0; t < nTabs; ++t) {
            double *at = static_cast<double *>(dTab.p) + t * (tabBytes / 8);
            AZ_CUDA(cudaMemcpyAsync(at, tabs[t], tabBytes, cudaMemcpyHostToDevice, st));
            dTabs[t] = at;
        }
    }
    AZ_CUDA(c->pipe.run(st, c->copyStream, n, chunk, 1 + nCols, in, nRes, res, dIn.p, dOut.p,
                        [&](uint32_t, uint32_t first, uint32_t m, void *const *dI, void *const *dO, cudaStream_t s) {
                            const double *dCols[kNumMaxCols] = {};
                            for (int q = 0; q < nCols; ++q) dCols[q] = static_cast<const double *>(dI[1 + q]);
                            return launch(first, m, static_cast<const double *>(dI[0]), dO, dCols, dTabs, s);
                        }));
    // give the slots back before returning (the default pool keeps nothing across a synchronisation)
    AZ_CUDA(dIn.release());
    AZ_CUDA(dOut.release());
    AZ_CUDA(dTab.release());
    AZ_CUDA(cudaStreamSynchronize(st));
    return ASTROZ_OK;
}

// K7's results: trajectory rows, status bytes and step counts.  a holds the checked arguments; for each chunk its n,
// states, out, status and counts are set to the chunk's and launch(dCols, dTabs, s) queues the kernel.
static int32_t numerical_host(az::NumArgs &a, const double *states, int nCols, const double *const *cols, int nTabs,
                              const double *const *tabs, size_t tabBytes, int32_t device, double *out, uint8_t *status,
                              uint64_t *steps, const NumLaunch &launch) {
    const size_t rowBytes = ((size_t)a.steps.nFull + a.steps.nTail + 1) * 48;  // one state's trajectory
    const az::HostOut res[3] = {{out, rowBytes}, {status, 1}, {steps, 16}};
    return numerical_host_rows(a.n, states, nCols, cols, nTabs, tabs, tabBytes, device, 3, res, rowBytes,
                               [&](uint32_t, uint32_t m, const double *dStates, void *const *dO,
                                   const double *const *dCols, const double *const *dTabs, cudaStream_t s) {
                                   a.n = m;
                                   a.states = dStates;
                                   a.out = static_cast<double *>(dO[0]);
                                   a.status = static_cast<uint8_t *>(dO[1]);
                                   a.counts = static_cast<uint64_t *>(dO[2]);
                                   return launch(dCols, dTabs, s);
                               });
}

int32_t astroz_cuda_propagate_numerical(const double *states, uint32_t n, double t0, double duration, double dt,
                                        double mu, int32_t forces, const double *j2, const double *r_eq,
                                        const double *drag_cd, const double *drag_area, const double *drag_mass,
                                        int32_t integrator, double rtol, double atol, int32_t device, double *out,
                                        uint8_t *status, uint64_t *steps) {
    az::NumArgs a{};
    int32_t rc = forces_check(mu, forces, j2, r_eq, drag_cd, drag_area, drag_mass, &a.p);
    if (rc == ASTROZ_OK) rc = numerical_check(n, t0, duration, dt, integrator, rtol, atol, device, &a);
    if (rc != ASTROZ_OK) return rc;
    if (n == 0) return ASTROZ_OK;
    if (!states || !out || !status) return ASTROZ_NULL_POINTER;
    if ((rc = check_device_ordinal(device)) != ASTROZ_OK) return rc;
    const bool drag = (forces & az::kForceDrag) != 0;
    const double *cols[3] = {drag_cd, drag_area, drag_mass};
    return numerical_host(a, states, drag ? 3 : 0, cols, 0, nullptr, 0, device, out, status, steps,
                          [&](const double *const *dCols, const double *const *, cudaStream_t s) {
                              a.cd = drag ? dCols[0] : nullptr;
                              a.area = drag ? dCols[1] : nullptr;
                              a.mass = drag ? dCols[2] : nullptr;
                              return az::launch_numerical(a, integrator, forces, s);
                          });
}

// ---- model lists (astroz_force_model_t) ----
static_assert(sizeof(astroz_force_model_t) == sizeof(az::ForceModel), "astroz_force_model_t is az::ForceModel");
static_assert(offsetof(astroz_force_model_t, pos) == offsetof(az::ForceModel, pos), "pos");
static_assert(offsetof(astroz_force_model_t, c_per_state) == offsetof(az::ForceModel, c_arr), "c_per_state");
static_assert(offsetof(astroz_force_model_t, pos_table) == offsetof(az::ForceModel, pos_table), "pos_table");
static_assert(ASTROZ_MAX_MODELS == az::kMaxModels && ASTROZ_MODEL_THIRD_BODY + 1 == az::kModelKinds, "model kinds");
static_assert(ASTROZ_MODEL_PER_STATE_C == az::kModelPerStateC && ASTROZ_MODEL_PER_STATE_AREA == az::kModelPerStateArea &&
                  ASTROZ_MODEL_PER_STATE_MASS == az::kModelPerStateMass && ASTROZ_MODEL_POS_TABLE == az::kModelPosTable,
              "model flags");

// Checks of a model list, before anything is read, written or allocated, and the list as the kernel reads it: each
// model's pointers kept only where its flags name them.
static int32_t models_check(const astroz_force_model_t *models, uint32_t nModels, az::ModelList *list) {
    if (nModels == 0 || nModels > az::kMaxModels) return value_error("a model list has 1 to 16 models");
    if (!models) return value_error("models is NULL");
    *list = az::ModelList{};
    list->count = nModels;
    constexpr uint32_t kPerState = az::kModelPerStateC | az::kModelPerStateArea | az::kModelPerStateMass;
    for (uint32_t j = 0; j < nModels; ++j) {
        const astroz_force_model_t &d = models[j];
        az::ForceModel &m = list->m[j];
        std::memcpy(&m, &d, sizeof m);
        m.c_arr = m.area_arr = m.mass_arr = m.pos_table = nullptr;
        // the scalar fields the kind reads, and the flags it accepts
        double used[10];
        int nUsed = 0;
        auto use = [&](std::initializer_list<double> v) {
            for (double x : v) used[nUsed++] = x;
        };
        uint32_t allowed = 0;
        switch (d.kind) {
            case az::kModelTwoBody: use({d.mu}); break;
            case az::kModelJ2:
            case az::kModelJ3:
            case az::kModelJ4: use({d.mu, d.coef, d.r_eq}); break;
            case az::kModelDrag: use({d.r_eq, d.rho0, d.scale_height, d.max_altitude}), allowed = kPerState; break;
            case az::kModelImprovedDrag: use({d.r_eq, d.max_altitude, d.f107}), allowed = kPerState; break;
            case az::kModelSrp: use({d.r_eq}), allowed = kPerState | az::kModelPosTable; break;
            case az::kModelThirdBody: use({d.mu}), allowed = az::kModelPosTable; break;
            default: return value_error("unknown model kind");
        }
        if (d.flags & ~allowed) return value_error("a model flag its kind does not take");
        if (allowed & kPerState) {
            const double *arr[3] = {d.c_per_state, d.area_per_state, d.mass_per_state};
            const double sc[3] = {d.c, d.area, d.mass};
            const double **dst[3] = {&m.c_arr, &m.area_arr, &m.mass_arr};
            for (int q = 0; q < 3; ++q) {
                if (d.flags & (az::kModelPerStateC << q)) {
                    if (!arr[q]) return value_error("a per-state flag is set and its array is NULL");
                    *dst[q] = arr[q];
                } else {
                    use({sc[q]});
                }
            }
        }
        if (allowed & az::kModelPosTable) {
            if (d.flags & az::kModelPosTable) {
                if (!d.pos_table) return value_error("ASTROZ_MODEL_POS_TABLE is set and pos_table is NULL");
                m.pos_table = d.pos_table;
            } else {
                use({d.pos[0], d.pos[1], d.pos[2]});
            }
        }
        for (int q = 0; q < nUsed; ++q)
            if (!std::isfinite(used[q])) return value_error("a model's scalar parameter is not finite");
    }
    return ASTROZ_OK;
}

int32_t astroz_cuda_propagate_numerical_models_device(const double *d_states, uint32_t n, double t0, double duration,
                                                      double dt, const astroz_force_model_t *models, uint32_t n_models,
                                                      int32_t integrator, double rtol, double atol, int32_t device,
                                                      double *d_out, uint8_t *d_status, uint64_t *d_steps,
                                                      void *stream) {
    az::ModelArgs ma{};
    int32_t rc = models_check(models, n_models, &ma.models);
    if (rc == ASTROZ_OK) rc = numerical_check(n, t0, duration, dt, integrator, rtol, atol, device, &ma.a);
    if (rc != ASTROZ_OK) return rc;
    if (n == 0) return ASTROZ_OK;
    if (!d_states || !d_out || !d_status) return ASTROZ_NULL_POINTER;
    if ((rc = check_device_ordinal(device)) != ASTROZ_OK) return rc;
    AZ_CUDA(cudaSetDevice(device));
    ma.a.states = d_states;
    ma.a.out = d_out;
    ma.a.status = d_status;
    ma.a.counts = d_steps;
    // the step table and the model list travel in the launch's parameters: the call only queues the kernel
    AZ_CUDA(az::launch_numerical_models(ma, integrator, static_cast<cudaStream_t>(stream)));
    return ASTROZ_OK;
}

int32_t astroz_cuda_propagate_numerical_models(const double *states, uint32_t n, double t0, double duration, double dt,
                                               const astroz_force_model_t *models, uint32_t n_models,
                                               int32_t integrator, double rtol, double atol, int32_t device,
                                               double *out, uint8_t *status, uint64_t *steps) {
    az::ModelArgs ma{};
    int32_t rc = models_check(models, n_models, &ma.models);
    if (rc == ASTROZ_OK) rc = numerical_check(n, t0, duration, dt, integrator, rtol, atol, device, &ma.a);
    if (rc != ASTROZ_OK) return rc;
    if (n == 0) return ASTROZ_OK;
    if (!states || !out || !status) return ASTROZ_NULL_POINTER;
    if ((rc = check_device_ordinal(device)) != ASTROZ_OK) return rc;
    // per-state columns in list order, and the position tables ([K][3] each)
    const double *cols[kNumMaxCols];
    const double **colOf[kNumMaxCols];
    const double *tabs[kNumMaxTabs];
    const double **tabOf[kNumMaxTabs];
    int nCols = 0, nTabs = 0;
    for (uint32_t j = 0; j < n_models; ++j) {
        az::ForceModel &m = ma.models.m[j];
        for (const double **p : {&m.c_arr, &m.area_arr, &m.mass_arr})
            if (*p) cols[nCols] = *p, colOf[nCols++] = p;
        if (m.pos_table) tabs[nTabs] = m.pos_table, tabOf[nTabs++] = &m.pos_table;
    }
    const size_t tabBytes = ((size_t)ma.a.steps.nFull + ma.a.steps.nTail) * 24;
    return numerical_host(ma.a, states, nCols, cols, nTabs, tabs, tabBytes, device, out, status, steps,
                          [&](const double *const *dCols, const double *const *dTabs, cudaStream_t s) {
                              for (int q = 0; q < nCols; ++q) *colOf[q] = dCols[q];
                              for (int t = 0; t < nTabs; ++t) *tabOf[t] = dTabs[t];
                              return az::launch_numerical_models(ma, integrator, s);
                          });
}

// ---- impulsive maneuvers (K7 maneuvers, az_numerical.cu) ----
static_assert(sizeof(astroz_impulse_t) == sizeof(az::Impulse) &&
                  offsetof(astroz_impulse_t, p) == offsetof(az::Impulse, p),
              "astroz_impulse_t is az::Impulse");
static_assert(ASTROZ_IMPULSE_ABSOLUTE == az::kImpAbsolute && ASTROZ_IMPULSE_PROGRADE == az::kImpPrograde &&
                  ASTROZ_IMPULSE_PHASE == az::kImpPhase && ASTROZ_IMPULSE_PLANE_CHANGE == az::kImpPlaneChange &&
                  ASTROZ_MANEUVER_ABNORMAL == az::kManAbnormal && ASTROZ_MANEUVER_TRUNCATED == az::kManTruncated,
              "impulse kinds and maneuver status bytes");

// Checks of every maneuver call, before anything is read, written or allocated (the impulses and offsets only where
// they are host memory).  On success a receives the scalars and the model list.
static int32_t maneuvers_check(uint32_t n, double t0, double duration, double h, double mu,
                               const uint32_t *offsets, const astroz_impulse_t *impulses, uint32_t m, bool host,
                               const astroz_force_model_t *models, uint32_t nModels, int32_t integrator, double rtol,
                               double atol, uint32_t maxSamples, int32_t device, az::ManeuverArgs *a) {
    int32_t rc = models_check(models, nModels, &a->models);
    if (rc != ASTROZ_OK) return rc;
    for (uint32_t j = 0; j < nModels; ++j)
        if (models[j].flags & ASTROZ_MODEL_POS_TABLE)
            return value_error("position tables follow K7's shared output intervals: a maneuver call refuses them");
    az::NumArgs na{};
    if ((rc = numerical_check(n, t0, duration, h, integrator, rtol, atol, device, &na)) != ASTROZ_OK) return rc;
    if (!std::isfinite(mu)) return value_error("mu must be finite");
    if (maxSamples == 0) return value_error("max_samples must be at least 1");
    if ((uint64_t)n * maxSamples > SIZE_MAX / 56) return value_error("the output size overflows");
    if (host) {
        if (!offsets || (m && !impulses)) return ASTROZ_NULL_POINTER;
        for (uint32_t i = 0; i < n; ++i)
            if (offsets[i + 1] < offsets[i]) return value_error("impulse_offsets decrease");
        if (offsets[n] != m) return value_error("impulse_offsets[n] must equal m");
        for (uint32_t k = 0; k < m; ++k) {
            const astroz_impulse_t &b = impulses[k];
            if (b.kind < ASTROZ_IMPULSE_ABSOLUTE || b.kind > ASTROZ_IMPULSE_PLANE_CHANGE)
                return value_error("unknown impulse kind");
            if (!std::isfinite(b.time) || !std::isfinite(b.p[0]) || !std::isfinite(b.p[1]) || !std::isfinite(b.p[2]))
                return value_error("an impulse's time or parameter is not finite");
            if (b.kind == ASTROZ_IMPULSE_PHASE && !(b.p[1] > 0.0)) return value_error("a phasing burn needs orbits > 0");
        }
    }
    a->n = n;
    a->t0 = t0;
    a->tf = t0 + duration;
    a->h = h;
    a->p = az::NumParams{mu, 0.0, 0.0, rtol, atol};
    a->maxSamples = maxSamples;
    return ASTROZ_OK;
}

int32_t astroz_cuda_propagate_maneuvers_device(const double *d_states, uint32_t n, double t0, double duration, double h,
                                               double mu, const uint32_t *d_impulse_offsets,
                                               const astroz_impulse_t *d_impulses, uint32_t m,
                                               const astroz_force_model_t *models, uint32_t n_models, int32_t integrator,
                                               double rtol, double atol, uint32_t max_samples, int32_t device,
                                               double *d_times, double *d_out, uint64_t *d_n_samples, uint8_t *d_status,
                                               uint64_t *d_steps, void *stream) {
    az::ManeuverArgs a{};
    int32_t rc = maneuvers_check(n, t0, duration, h, mu, nullptr, nullptr, m, false, models, n_models, integrator, rtol,
                                 atol, max_samples, device, &a);
    if (rc != ASTROZ_OK) return rc;
    if (n == 0) return ASTROZ_OK;
    if (!d_states || !d_impulse_offsets || (m && !d_impulses) || !d_times || !d_out || !d_n_samples || !d_status)
        return ASTROZ_NULL_POINTER;
    if ((rc = check_device_ordinal(device)) != ASTROZ_OK) return rc;
    AZ_CUDA(cudaSetDevice(device));
    a.states = d_states;
    a.offsets = d_impulse_offsets;
    a.impulses = reinterpret_cast<const az::Impulse *>(d_impulses);
    a.times = d_times;
    a.out = d_out;
    a.count = d_n_samples;
    a.status = d_status;
    a.counts = d_steps;
    // the scalars and the model list travel in the launch's parameters: the call only queues the kernel
    AZ_CUDA(az::launch_maneuvers(a, integrator, static_cast<cudaStream_t>(stream)));
    return ASTROZ_OK;
}

int32_t astroz_cuda_propagate_maneuvers(const double *states, uint32_t n, double t0, double duration, double h, double mu,
                                        const uint32_t *impulse_offsets, const astroz_impulse_t *impulses, uint32_t m,
                                        const astroz_force_model_t *models, uint32_t n_models, int32_t integrator,
                                        double rtol, double atol, uint32_t max_samples, int32_t device, double *times,
                                        double *out, uint64_t *n_samples, uint8_t *status, uint64_t *steps) {
    az::ManeuverArgs a{};
    int32_t rc = maneuvers_check(n, t0, duration, h, mu, impulse_offsets, impulses, m, true, models, n_models,
                                 integrator, rtol, atol, max_samples, device, &a);
    if (rc != ASTROZ_OK) return rc;
    if (n == 0) return ASTROZ_OK;
    if (!states || !times || !out || !n_samples || !status) return ASTROZ_NULL_POINTER;
    if ((rc = check_device_ordinal(device)) != ASTROZ_OK) return rc;
    // per-state columns in list order (as for model lists), and the schedules as one whole array: the impulses, then
    // the offsets, uploaded once per call
    const double *cols[kNumMaxCols];
    const double **colOf[kNumMaxCols];
    int nCols = 0;
    for (uint32_t j = 0; j < n_models; ++j) {
        az::ForceModel &fm = a.models.m[j];
        for (const double **p : {&fm.c_arr, &fm.area_arr, &fm.mass_arr})
            if (*p) cols[nCols] = *p, colOf[nCols++] = p;
    }
    const size_t impBytes = (size_t)m * sizeof(astroz_impulse_t), offBytes = ((size_t)n + 1) * 4;
    std::vector<double> sched((impBytes + offBytes + 7) / 8);
    if (m) std::memcpy(sched.data(), impulses, impBytes);
    std::memcpy(reinterpret_cast<char *>(sched.data()) + impBytes, impulse_offsets, offBytes);
    const double *tabs[1] = {sched.data()};
    const size_t rowSamples = max_samples;
    const az::HostOut res[5] = {
        {times, rowSamples * 8}, {out, rowSamples * 48}, {n_samples, 8}, {status, 1}, {steps, 16}};
    return numerical_host_rows(n, states, nCols, cols, 1, tabs, sched.size() * 8, device, 5, res, rowSamples * 56,
                               [&](uint32_t first, uint32_t cm, const double *dStates, void *const *dO,
                                   const double *const *dCols, const double *const *dTabs, cudaStream_t s) {
                                   for (int q = 0; q < nCols; ++q) *colOf[q] = dCols[q];
                                   a.n = cm;
                                   a.first = first;
                                   a.states = dStates;
                                   a.impulses = reinterpret_cast<const az::Impulse *>(dTabs[0]);
                                   a.offsets = reinterpret_cast<const uint32_t *>(
                                       reinterpret_cast<const char *>(dTabs[0]) + impBytes);
                                   a.times = static_cast<double *>(dO[0]);
                                   a.out = static_cast<double *>(dO[1]);
                                   a.count = static_cast<uint64_t *>(dO[2]);
                                   a.status = static_cast<uint8_t *>(dO[3]);
                                   a.counts = static_cast<uint64_t *>(dO[4]);
                                   return az::launch_maneuvers(a, integrator, s);
                               });
}

// ---- whole-batch host calls: element fits, observe, covariance, conjunctions, correlation, initial orbits, Lambert --
// Their input checks, each rule stated once, and their one staging path.  The checks run before anything is read on,
// written to or allocated on the device, in the order scalars, null pointers, values, device lookup.

static bool all_finite(const double *p, size_t count) {
    for (size_t i = 0; i < count; ++i)
        if (!std::isfinite(p[i])) return false;
    return true;
}

static int32_t grav_check(int32_t grav) {
    if (grav != ASTROZ_WGS72 && grav != ASTROZ_WGS84) return value_error("grav must be ASTROZ_WGS72 or ASTROZ_WGS84");
    return ASTROZ_OK;
}

// Group g of `groups` owns items [offsets[g], offsets[g + 1]) of m: the offsets are non-decreasing and end at m
// (`wrong_end` is the refusal when they do not).  As the call states, offsets[0] must also be 0 (zero_first), and with
// max_track > 0 the groups are tracks of 1 to max_track observations (`too_long` is the refusal of a longer one).
static int32_t offsets_check(const uint32_t *offsets, uint32_t groups, uint32_t m, const char *wrong_end,
                             bool zero_first = false, uint32_t max_track = 0, const char *too_long = nullptr) {
    if (zero_first && offsets[0] != 0) return value_error("offsets[0] must be 0");
    for (uint32_t g = 0; g < groups; ++g) {
        if (offsets[g + 1] < offsets[g]) return value_error("offsets must be non-decreasing");
        if (max_track == 0) continue;
        if (offsets[g + 1] == offsets[g]) return value_error("a track has no observation");
        if (offsets[g + 1] - offsets[g] > max_track) return value_error(too_long);
    }
    if (offsets[groups] != m) return value_error(wrong_end);
    return ASTROZ_OK;
}

// Catalogue rows: n element columns [8][n], and their covariance [n][28] when it is given.
static int32_t rows_check(const double *elements, const double *covariance, uint32_t n) {
    if (!all_finite(elements, (size_t)8 * n)) return value_error("elements must be finite");
    if (covariance && !all_finite(covariance, (size_t)az::kFitN * n)) return value_error("covariance words must be finite");
    return ASTROZ_OK;
}

// The rows' model bytes, when given.
static int32_t model_bytes_check(const uint8_t *model, uint32_t n) {
    if (model)
        for (uint32_t s = 0; s < n; ++s)
            if (model[s] > 1) return value_error("a model byte is not 0 (near-earth) or 1 (deep space)");
    return ASTROZ_OK;
}

// Every one of t tracks has a residual the scoring uses.
static int32_t used_residuals_check(const az::CorrObsArrays &in, const uint32_t *offsets, uint32_t t) {
    for (uint32_t j = 0; j < t; ++j)
        if (az::corr_used(in, offsets[j], offsets[j + 1]) == 0) return value_error("a track has no used residual");
    return ASTROZ_OK;
}

// One piece of a whole-batch call's device block: `bytes` long, uploaded from host `in` before the launch or copied to
// host `out` after it (neither: scratch, or an optional array the caller did not pass).
struct BatchPiece {
    size_t bytes;
    const void *in;
    void *out;
};
static BatchPiece upload(const void *src, size_t bytes) { return {bytes, src, nullptr}; }
static BatchPiece result(void *dst, size_t bytes) { return {bytes, nullptr, dst}; }
static BatchPiece scratch(size_t bytes) { return {bytes, nullptr, nullptr}; }

// A stream-ordered device block cut into the 16-byte aligned pieces of a list, at least 16 bytes in all: every piece
// has an address in the block, an empty one too.
struct DeviceBlock {
    StreamBuf buf;
    std::vector<size_t> at;
    explicit DeviceBlock(cudaStream_t s) : buf(s) {}
    cudaError_t alloc(std::initializer_list<BatchPiece> pieces) {
        size_t total = 0;
        for (const BatchPiece &p : pieces) at.push_back(total), total += (p.bytes + 15) & ~size_t(15);
        return buf.alloc(std::max<size_t>(total, 16));
    }
    char *piece(int k) const { return static_cast<char *>(buf.p) + at[k]; }
    double *f64(int k) const { return reinterpret_cast<double *>(piece(k)); }
    uint32_t *u32(int k) const { return reinterpret_cast<uint32_t *>(piece(k)); }
    uint8_t *u8(int k) const { return reinterpret_cast<uint8_t *>(piece(k)); }
};
using BatchLaunch = std::function<cudaError_t(const DeviceBlock &d, cudaStream_t s)>;

// The host form of every whole-batch call, after its checks.  These calls are compute-bound (a fit propagates each
// observation some 8 x iterations times for its ~56 bytes, a Lambert slot runs some 5 iterations of fp64
// transcendentals for 56 bytes in), so there is no chunk pipeline to overlap transfers with: the whole batch goes up at
// once into one device block -- pageable sources through the device's pinned ring, pinned ones by direct DMA, decided
// per array -- launch(d, stream) queues the kernels on the device's stream with d.piece(k) the device copy of
// pieces[k], each result comes back by a plain copy, and the block is returned before the call returns.
static int32_t whole_batch(int32_t device, std::initializer_list<BatchPiece> pieces, const BatchLaunch &launch) {
    int32_t rc = check_device_ordinal(device);
    if (rc != ASTROZ_OK) return rc;
    NumericalContext *c = nullptr;
    if ((rc = numerical_context(device, &c)) != ASTROZ_OK) return rc;
    std::lock_guard<std::mutex> lk(c->m);
    AZ_CUDA(cudaSetDevice(device));
    cudaStream_t st = c->stream;
    DeviceBlock d(st);
    AZ_CUDA(d.alloc(pieces));
    const size_t byteSize = 1;
    int k = 0;
    for (const BatchPiece &p : pieces) {
        void *const dst[1] = {d.piece(k++)};
        if (p.in && p.bytes) AZ_CUDA(c->pipe.ring.upload(az::is_pageable(p.in), 1, &p.in, dst, &byteSize, p.bytes, st));
    }
    AZ_CUDA(launch(d, st));
    k = 0;
    for (const BatchPiece &p : pieces) {
        char *const src = d.piece(k++);
        if (p.out && p.bytes) AZ_CUDA(cudaMemcpyAsync(p.out, src, p.bytes, cudaMemcpyDeviceToHost, st));
    }
    AZ_CUDA(d.buf.release());
    AZ_CUDA(cudaStreamSynchronize(st));
    return ASTROZ_OK;
}

// ---- element fits (K8, az_fit.cu) ------------------------------------------------------------------------------------
static_assert(ASTROZ_FIT_CONVERGED == az::kFitConverged && ASTROZ_FIT_ITERATION_LIMIT == az::kFitIterLimit &&
                  ASTROZ_FIT_INIT_FAILED == az::kFitInitFailed && ASTROZ_FIT_DEEP_SPACE == az::kFitDeepSpace &&
                  ASTROZ_FIT_TOO_FEW_OBSERVATIONS == az::kFitTooFew,
              "fit status bytes");

// Scalar checks of both fit calls, before anything is read, written or allocated; a receives the scalars.
static int32_t fit_check(uint32_t n, int32_t grav, double pos_sigma, double vel_sigma, int32_t fit_bstar,
                         uint32_t max_iter, int32_t device, az::FitArgs *a) {
    if (device < 0) return value_error("an element fit runs on one device: pass its ordinal");
    const int32_t rc = grav_check(grav);
    if (rc != ASTROZ_OK) return rc;
    if (!std::isfinite(pos_sigma) || !(pos_sigma > 0.0) || !std::isfinite(vel_sigma) || !(vel_sigma > 0.0))
        return value_error("pos_sigma and vel_sigma must be finite and > 0");
    if (max_iter == 0) return value_error("max_iter must be at least 1");
    a->n = n;
    a->grav = grav;
    a->g = az::grav_consts(az::gravity(grav));
    a->wp = 1.0 / pos_sigma;
    a->wv = 1.0 / vel_sigma;
    a->fitBstar = fit_bstar != 0;
    a->maxIter = max_iter;
    return ASTROZ_OK;
}

// The kernels one fit call queues on its stream: launch_fit, or launch_fit_mixed below.
using FitLaunch = cudaError_t (*)(const az::FitArgs &a, cudaStream_t stream);

// Both call forms: a holds fit_check's scalars, the arrays are on the device, launch(a, st) queues the kernels.
static cudaError_t fit_run(az::FitArgs a, const double *elements, const uint32_t *offsets, const double *jd,
                           const double *fr, const double *pos, const double *vel, double *fitted, double *rms,
                           uint32_t *iterations, uint8_t *status, cudaStream_t st, FitLaunch launch) {
    a.elements = elements;
    a.offsets = offsets;
    a.jd = jd;
    a.fr = fr;
    a.pos = pos;
    a.vel = vel;
    a.fitted = fitted;
    a.rms = rms;
    a.iterations = iterations;
    a.status = status;
    return launch(a, st);
}

// The device-pointer calls.
static int32_t fit_device(const double *d_elements, uint32_t n, int32_t grav, const uint32_t *d_offsets,
                          const double *d_jd, const double *d_fr, const double *d_pos, const double *d_vel,
                          double pos_sigma, double vel_sigma, int32_t fit_bstar, uint32_t max_iter, int32_t device,
                          double *d_fitted, double *d_rms, uint32_t *d_iterations, uint8_t *d_status, void *stream,
                          FitLaunch launch) {
    az::FitArgs a{};
    int32_t rc = fit_check(n, grav, pos_sigma, vel_sigma, fit_bstar, max_iter, device, &a);
    if (rc != ASTROZ_OK) return rc;
    if (n == 0) return ASTROZ_OK;
    if (!d_elements || !d_offsets || !d_jd || !d_fr || !d_pos || !d_fitted || !d_rms || !d_iterations || !d_status)
        return ASTROZ_NULL_POINTER;
    if ((rc = check_device_ordinal(device)) != ASTROZ_OK) return rc;
    AZ_CUDA(cudaSetDevice(device));
    AZ_CUDA(fit_run(a, d_elements, d_offsets, d_jd, d_fr, d_pos, d_vel, d_fitted, d_rms, d_iterations, d_status,
                    static_cast<cudaStream_t>(stream), launch));
    return ASTROZ_OK;
}

// A mixed batch: the near-earth fit writes every row (DEEP_SPACE on the deep-space ones), then the deep-space fit
// overwrites the deep-space rows on the same stream.  The near-earth rows are therefore the near-earth call's bytes.
static cudaError_t launch_fit_mixed(const az::FitArgs &a, cudaStream_t st) {
    const cudaError_t e = az::launch_fit(a, st);
    return e != cudaSuccess ? e : az::launch_fit_deep(a, st);
}

int32_t astroz_cuda_fit_elements_device(const double *d_elements, uint32_t n, int32_t grav, const uint32_t *d_offsets,
                                        const double *d_jd, const double *d_fr, const double *d_pos,
                                        const double *d_vel, double pos_sigma, double vel_sigma, int32_t fit_bstar,
                                        uint32_t max_iter, int32_t device, double *d_fitted, double *d_rms,
                                        uint32_t *d_iterations, uint8_t *d_status, void *stream) {
    return fit_device(d_elements, n, grav, d_offsets, d_jd, d_fr, d_pos, d_vel, pos_sigma, vel_sigma, fit_bstar,
                      max_iter, device, d_fitted, d_rms, d_iterations, d_status, stream, az::launch_fit);
}

int32_t astroz_cuda_fit_elements_mixed_device(const double *d_elements, uint32_t n, int32_t grav,
                                              const uint32_t *d_offsets, const double *d_jd, const double *d_fr,
                                              const double *d_pos, const double *d_vel, double pos_sigma,
                                              double vel_sigma, int32_t fit_bstar, uint32_t max_iter, int32_t device,
                                              double *d_fitted, double *d_rms, uint32_t *d_iterations,
                                              uint8_t *d_status, void *stream) {
    return fit_device(d_elements, n, grav, d_offsets, d_jd, d_fr, d_pos, d_vel, pos_sigma, vel_sigma, fit_bstar,
                      max_iter, device, d_fitted, d_rms, d_iterations, d_status, stream, launch_fit_mixed);
}

static int32_t fit_host(const double *elements, uint32_t n, int32_t grav, const uint32_t *offsets, const double *jd,
                        const double *fr, const double *pos, const double *vel, uint32_t m, double pos_sigma,
                        double vel_sigma, int32_t fit_bstar, uint32_t max_iter, int32_t device, double *fitted,
                        double *rms, uint32_t *iterations, uint8_t *status, FitLaunch launch) {
    az::FitArgs a{};
    int32_t rc = fit_check(n, grav, pos_sigma, vel_sigma, fit_bstar, max_iter, device, &a);
    if (rc != ASTROZ_OK) return rc;
    if (n == 0) return ASTROZ_OK;
    if (!elements || !offsets || !fitted || !rms || !iterations || !status) return ASTROZ_NULL_POINTER;
    if (m && (!jd || !fr || !pos)) return ASTROZ_NULL_POINTER;
    if ((rc = offsets_check(offsets, n, m, "offsets[n] must equal the observation count m")) != ASTROZ_OK) return rc;
    if (!all_finite(elements, (size_t)8 * n) || !all_finite(jd, m) || !all_finite(fr, m) ||
        !all_finite(pos, (size_t)3 * m) || (vel && !all_finite(vel, (size_t)3 * m)))
        return value_error("elements and observations must be finite");
    return whole_batch(device,
                       {upload(elements, (size_t)64 * n), upload(offsets, (size_t)4 * (n + 1)), upload(jd, (size_t)8 * m),
                        upload(fr, (size_t)8 * m), upload(pos, (size_t)24 * m), upload(vel, vel ? (size_t)24 * m : 0),
                        result(fitted, (size_t)64 * n), result(rms, (size_t)16 * n), result(iterations, (size_t)4 * n),
                        result(status, n)},
                       [&](const DeviceBlock &d, cudaStream_t st) {
                           return fit_run(a, d.f64(0), d.u32(1), d.f64(2), d.f64(3), d.f64(4),
                                          vel ? d.f64(5) : nullptr, d.f64(6), d.f64(7), d.u32(8), d.u8(9), st, launch);
                       });
}

int32_t astroz_cuda_fit_elements(const double *elements, uint32_t n, int32_t grav, const uint32_t *offsets,
                                 const double *jd, const double *fr, const double *pos, const double *vel, uint32_t m,
                                 double pos_sigma, double vel_sigma, int32_t fit_bstar, uint32_t max_iter,
                                 int32_t device, double *fitted, double *rms, uint32_t *iterations, uint8_t *status) {
    return fit_host(elements, n, grav, offsets, jd, fr, pos, vel, m, pos_sigma, vel_sigma, fit_bstar, max_iter, device,
                    fitted, rms, iterations, status, az::launch_fit);
}

int32_t astroz_cuda_fit_elements_mixed(const double *elements, uint32_t n, int32_t grav, const uint32_t *offsets,
                                       const double *jd, const double *fr, const double *pos, const double *vel,
                                       uint32_t m, double pos_sigma, double vel_sigma, int32_t fit_bstar,
                                       uint32_t max_iter, int32_t device, double *fitted, double *rms,
                                       uint32_t *iterations, uint8_t *status) {
    return fit_host(elements, n, grav, offsets, jd, fr, pos, vel, m, pos_sigma, vel_sigma, fit_bstar, max_iter, device,
                    fitted, rms, iterations, status, launch_fit_mixed);
}

// ---- element fits from sensor observations (K8, az_fit_obs.cu, az_obs.cuh) ----------------------------------------
static_assert(ASTROZ_OBS_TEME_STATE == az::kObsTemeState && ASTROZ_OBS_ECEF_STATE == az::kObsEcefState &&
                  ASTROZ_OBS_RADAR == az::kObsRadar && ASTROZ_OBS_OPTICAL == az::kObsOptical &&
                  ASTROZ_OBS_VALUES == az::kObsValues && ASTROZ_FIT_COVARIANCE_WORDS == az::kFitN,
              "observation kinds and layouts");

// Scalar checks of the observation fits, before anything is read, written or allocated; a receives the scalars.
static int32_t fit_obs_check(uint32_t n, int32_t grav, int32_t fit_bstar, uint32_t max_iter, int32_t device,
                             az::FitObsArgs *a) {
    if (device < 0) return value_error("an element fit runs on one device: pass its ordinal");
    const int32_t rc = grav_check(grav);
    if (rc != ASTROZ_OK) return rc;
    if (max_iter == 0) return value_error("max_iter must be at least 1");
    a->n = n;
    a->grav = grav;
    a->g = az::grav_consts(az::gravity(grav));
    a->fitBstar = fit_bstar != 0;
    a->maxIter = max_iter;
    return ASTROZ_OK;
}

// Host-side value checks of m observations and k stations.  sigma = nullptr: astroz_cuda_observe, which has no sigmas
// and reads no values.
static int32_t obs_values_check(const double *jd, const double *fr, const double *value, const double *sigma,
                                const uint32_t *station, const uint8_t *kind, uint32_t m, const double *stations,
                                uint32_t k) {
    if (k && !stations) return ASTROZ_NULL_POINTER;
    for (uint32_t s = 0; s < k; ++s) {
        const double *st = stations + (size_t)s * 3;
        if (!std::isfinite(st[0]) || !std::isfinite(st[1]) || !std::isfinite(st[2]))
            return value_error("stations must be finite");
        if (!(std::fabs(st[0]) <= 90.0)) return value_error("a station latitude is outside [-90, 90] deg");
    }
    if (!all_finite(jd, m) || !all_finite(fr, m)) return value_error("observation times must be finite");
    for (uint32_t i = 0; i < m; ++i) {
        if (kind[i] >= az::kObsKinds) return value_error("unknown observation kind");
        if (az::obs_uses_station(kind[i])) {
            if (!station) return ASTROZ_NULL_POINTER;
            if (station[i] >= k) return value_error("a station index is not below the station count k");
        }
        if (!sigma) continue;
        const double *v = value + (size_t)i * 6, *sg = sigma + (size_t)i * 6;
        const int count = az::obs_count(kind[i]), wr = az::obs_wrapped(kind[i]);
        for (int c = 0; c < count; ++c) {
            if (!(sg[c] > 0.0)) return value_error("sigma must be > 0 (+inf: component not used)");
            if (sg[c] < INFINITY && !std::isfinite(v[c])) return value_error("a used observation value is not finite");
        }
        if (wr >= 0 && sg[wr] < INFINITY && !std::isfinite(v[az::obs_partner(kind[i])]))
            return value_error("a used azimuth or right ascension needs a finite elevation or declination");
    }
    return ASTROZ_OK;
}

static cudaError_t launch_fit_obs_mixed(const az::FitObsArgs &a, cudaStream_t st) {
    const cudaError_t e = az::launch_fit_obs(a, st);
    return e != cudaSuccess ? e : az::launch_fit_obs_deep(a, st);
}
using FitObsLaunch = cudaError_t (*)(const az::FitObsArgs &a, cudaStream_t stream);

// Both call forms: a holds fit_obs_check's scalars, the arrays are on the device, launch(a, st) queues the kernels.
static cudaError_t fit_obs_run(az::FitObsArgs a, const double *elements, const uint32_t *offsets, const double *jd,
                               const double *fr, const double *value, const double *sigma, const uint32_t *station,
                               const uint8_t *kind, const double *stations, double *fitted, double *wrms,
                               uint32_t *n_residuals, double *covariance, uint32_t *iterations, uint8_t *status,
                               uint8_t *model, cudaStream_t st, FitObsLaunch launch) {
    a.elements = elements;
    a.offsets = offsets;
    a.jd = jd;
    a.fr = fr;
    a.value = value;
    a.sigma = sigma;
    a.station = station;
    a.kind = kind;
    a.stations = stations;
    a.fitted = fitted;
    a.wrms = wrms;
    a.nResiduals = n_residuals;
    a.covariance = covariance;
    a.iterations = iterations;
    a.status = status;
    a.model = model;
    return launch(a, st);
}

static int32_t fit_obs_device(const double *d_elements, uint32_t n, int32_t grav, const uint32_t *d_offsets,
                              const double *d_jd, const double *d_fr, const double *d_value, const double *d_sigma,
                              const uint32_t *d_station, const uint8_t *d_kind, const double *d_stations,
                              int32_t fit_bstar, uint32_t max_iter, int32_t device, double *d_fitted, double *d_wrms,
                              uint32_t *d_n_residuals, double *d_covariance, uint32_t *d_iterations,
                              uint8_t *d_status, uint8_t *d_model, void *stream, FitObsLaunch launch) {
    az::FitObsArgs a{};
    int32_t rc = fit_obs_check(n, grav, fit_bstar, max_iter, device, &a);
    if (rc != ASTROZ_OK) return rc;
    if (n == 0) return ASTROZ_OK;
    if (!d_elements || !d_offsets || !d_jd || !d_fr || !d_value || !d_sigma || !d_kind || !d_fitted || !d_wrms ||
        !d_n_residuals || !d_covariance || !d_iterations || !d_status || !d_model)
        return ASTROZ_NULL_POINTER;
    if ((rc = check_device_ordinal(device)) != ASTROZ_OK) return rc;
    AZ_CUDA(cudaSetDevice(device));
    AZ_CUDA(fit_obs_run(a, d_elements, d_offsets, d_jd, d_fr, d_value, d_sigma, d_station, d_kind, d_stations,
                        d_fitted, d_wrms, d_n_residuals, d_covariance, d_iterations, d_status, d_model,
                        static_cast<cudaStream_t>(stream), launch));
    return ASTROZ_OK;
}

static int32_t fit_obs_host(const double *elements, uint32_t n, int32_t grav, const uint32_t *offsets,
                            const double *jd, const double *fr, const double *value, const double *sigma,
                            const uint32_t *station, const uint8_t *kind, uint32_t m, const double *stations,
                            uint32_t k, int32_t fit_bstar, uint32_t max_iter, int32_t device, double *fitted,
                            double *wrms, uint32_t *n_residuals, double *covariance, uint32_t *iterations,
                            uint8_t *status, uint8_t *model, FitObsLaunch launch) {
    az::FitObsArgs a{};
    int32_t rc = fit_obs_check(n, grav, fit_bstar, max_iter, device, &a);
    if (rc != ASTROZ_OK) return rc;
    if (n == 0) return ASTROZ_OK;
    if (!elements || !offsets || !fitted || !wrms || !n_residuals || !covariance || !iterations || !status || !model)
        return ASTROZ_NULL_POINTER;
    if (m && (!jd || !fr || !value || !sigma || !kind)) return ASTROZ_NULL_POINTER;
    if ((rc = offsets_check(offsets, n, m, "offsets[n] must equal the observation count m")) != ASTROZ_OK) return rc;
    if ((rc = rows_check(elements, nullptr, n)) != ASTROZ_OK) return rc;
    if ((rc = obs_values_check(jd, fr, value, sigma, station, kind, m, stations, k)) != ASTROZ_OK) return rc;
    return whole_batch(device,
                       {upload(elements, (size_t)64 * n), upload(offsets, (size_t)4 * (n + 1)), upload(jd, (size_t)8 * m),
                        upload(fr, (size_t)8 * m), upload(value, (size_t)48 * m), upload(sigma, (size_t)48 * m),
                        upload(station, station ? (size_t)4 * m : 0), upload(kind, m), upload(stations, (size_t)24 * k),
                        result(fitted, (size_t)64 * n), result(wrms, (size_t)8 * n), result(n_residuals, (size_t)4 * n),
                        result(covariance, (size_t)8 * az::kFitN * n), result(iterations, (size_t)4 * n),
                        result(status, n), result(model, n)},
                       [&](const DeviceBlock &d, cudaStream_t st) {
                           return fit_obs_run(a, d.f64(0), d.u32(1), d.f64(2), d.f64(3), d.f64(4), d.f64(5),
                                              station ? d.u32(6) : nullptr, d.u8(7), k ? d.f64(8) : nullptr, d.f64(9),
                                              d.f64(10), d.u32(11), d.f64(12), d.u32(13), d.u8(14), d.u8(15), st,
                                              launch);
                       });
}

int32_t astroz_cuda_fit_observations(const double *elements, uint32_t n, int32_t grav, const uint32_t *offsets,
                                     const double *jd, const double *fr, const double *value, const double *sigma,
                                     const uint32_t *station, const uint8_t *kind, uint32_t m, const double *stations,
                                     uint32_t k, int32_t fit_bstar, uint32_t max_iter, int32_t device, double *fitted,
                                     double *wrms, uint32_t *n_residuals, double *covariance, uint32_t *iterations,
                                     uint8_t *status, uint8_t *model) {
    return fit_obs_host(elements, n, grav, offsets, jd, fr, value, sigma, station, kind, m, stations, k, fit_bstar,
                        max_iter, device, fitted, wrms, n_residuals, covariance, iterations, status, model,
                        az::launch_fit_obs);
}

int32_t astroz_cuda_fit_observations_mixed(const double *elements, uint32_t n, int32_t grav, const uint32_t *offsets,
                                           const double *jd, const double *fr, const double *value,
                                           const double *sigma, const uint32_t *station, const uint8_t *kind,
                                           uint32_t m, const double *stations, uint32_t k, int32_t fit_bstar,
                                           uint32_t max_iter, int32_t device, double *fitted, double *wrms,
                                           uint32_t *n_residuals, double *covariance, uint32_t *iterations,
                                           uint8_t *status, uint8_t *model) {
    return fit_obs_host(elements, n, grav, offsets, jd, fr, value, sigma, station, kind, m, stations, k, fit_bstar,
                        max_iter, device, fitted, wrms, n_residuals, covariance, iterations, status, model,
                        launch_fit_obs_mixed);
}

int32_t astroz_cuda_fit_observations_device(const double *d_elements, uint32_t n, int32_t grav,
                                            const uint32_t *d_offsets, const double *d_jd, const double *d_fr,
                                            const double *d_value, const double *d_sigma, const uint32_t *d_station,
                                            const uint8_t *d_kind, const double *d_stations, int32_t fit_bstar,
                                            uint32_t max_iter, int32_t device, double *d_fitted, double *d_wrms,
                                            uint32_t *d_n_residuals, double *d_covariance, uint32_t *d_iterations,
                                            uint8_t *d_status, uint8_t *d_model, void *stream) {
    return fit_obs_device(d_elements, n, grav, d_offsets, d_jd, d_fr, d_value, d_sigma, d_station, d_kind, d_stations,
                          fit_bstar, max_iter, device, d_fitted, d_wrms, d_n_residuals, d_covariance, d_iterations,
                          d_status, d_model, stream, az::launch_fit_obs);
}

int32_t astroz_cuda_fit_observations_mixed_device(const double *d_elements, uint32_t n, int32_t grav,
                                                  const uint32_t *d_offsets, const double *d_jd, const double *d_fr,
                                                  const double *d_value, const double *d_sigma,
                                                  const uint32_t *d_station, const uint8_t *d_kind,
                                                  const double *d_stations, int32_t fit_bstar, uint32_t max_iter,
                                                  int32_t device, double *d_fitted, double *d_wrms,
                                                  uint32_t *d_n_residuals, double *d_covariance,
                                                  uint32_t *d_iterations, uint8_t *d_status, uint8_t *d_model,
                                                  void *stream) {
    return fit_obs_device(d_elements, n, grav, d_offsets, d_jd, d_fr, d_value, d_sigma, d_station, d_kind, d_stations,
                          fit_bstar, max_iter, device, d_fitted, d_wrms, d_n_residuals, d_covariance, d_iterations,
                          d_status, d_model, stream, launch_fit_obs_mixed);
}

int32_t astroz_cuda_observe(const double *states, const double *jd, const double *fr, const uint8_t *kind,
                            const uint32_t *station, uint32_t m, const double *stations, uint32_t k, int32_t device,
                            double *values) {
    if (device < 0) return value_error("observe runs on one device: pass its ordinal");
    if (m == 0) return ASTROZ_OK;
    if (!states || !jd || !fr || !kind || !values) return ASTROZ_NULL_POINTER;
    const int32_t rc = obs_values_check(jd, fr, nullptr, nullptr, station, kind, m, stations, k);
    if (rc != ASTROZ_OK) return rc;
    return whole_batch(device,
                       {upload(states, (size_t)48 * m), upload(jd, (size_t)8 * m), upload(fr, (size_t)8 * m),
                        upload(kind, m), upload(station, station ? (size_t)4 * m : 0), upload(stations, (size_t)24 * k),
                        result(values, (size_t)48 * m)},
                       [&](const DeviceBlock &d, cudaStream_t st) {
                           return az::launch_observe(d.f64(0), d.f64(1), d.f64(2), d.u8(3),
                                                     station ? d.u32(4) : nullptr, k ? d.f64(5) : nullptr, m,
                                                     d.f64(6), st);
                       });
}

int32_t astroz_cuda_observe_device(const double *d_states, const double *d_jd, const double *d_fr,
                                   const uint8_t *d_kind, const uint32_t *d_station, uint32_t m,
                                   const double *d_stations, int32_t device, double *d_values, void *stream) {
    if (device < 0) return value_error("observe runs on one device: pass its ordinal");
    if (m == 0) return ASTROZ_OK;
    if (!d_states || !d_jd || !d_fr || !d_kind || !d_values) return ASTROZ_NULL_POINTER;
    int32_t rc = check_device_ordinal(device);
    if (rc != ASTROZ_OK) return rc;
    AZ_CUDA(cudaSetDevice(device));
    AZ_CUDA(az::launch_observe(d_states, d_jd, d_fr, d_kind, d_station, d_stations, m, d_values,
                               static_cast<cudaStream_t>(stream)));
    return ASTROZ_OK;
}

// ---- state covariance (K10, az_covariance.cu, az_covariance.cuh) ----------------------------------------------------
static_assert(ASTROZ_COV_OK == az::kCovOk && ASTROZ_COV_INIT_FAILED == az::kCovInitFailed &&
                  ASTROZ_COV_CELL_FAILED == az::kCovCellFailed && ASTROZ_COV_FRAME_TEME == az::kCovFrameTeme &&
                  ASTROZ_COV_FRAME_RTN == az::kCovFrameRtn && ASTROZ_STATE_COVARIANCE_WORDS == az::kCovWords,
              "covariance status bytes, frames and layout");

// Scalar checks of the covariance calls, before anything is read, written or allocated; a receives the scalars.
static int32_t cov_check(uint32_t n, int32_t grav, uint32_t m, int32_t frame, int32_t device, az::CovArgs *a) {
    if (device < 0) return value_error("covariance propagation runs on one device: pass its ordinal");
    const int32_t rc = grav_check(grav);
    if (rc != ASTROZ_OK) return rc;
    if (frame != ASTROZ_COV_FRAME_TEME && frame != ASTROZ_COV_FRAME_RTN)
        return value_error("frame must be ASTROZ_COV_FRAME_TEME or ASTROZ_COV_FRAME_RTN");
    a->n = n;
    a->m = m;
    a->grav = grav;
    a->g = az::grav_consts(az::gravity(grav));
    a->frame = frame;
    return ASTROZ_OK;
}

// Both call forms: a holds cov_check's scalars, the arrays are on the device.
static cudaError_t cov_run(az::CovArgs a, const double *elements, const double *covariance, const uint8_t *model,
                           const uint32_t *offsets, const double *jd, const double *fr, double *state,
                           double *state_covariance, double *jacobian, uint8_t *status, cudaStream_t st) {
    a.elements = elements;
    a.covariance = covariance;
    a.model = model;
    a.offsets = offsets;
    a.jd = jd;
    a.fr = fr;
    a.state = state;
    a.sigma = state_covariance;
    a.jacobian = jacobian;
    a.status = status;
    return az::launch_covariance(a, st);
}

int32_t astroz_cuda_propagate_covariance_device(const double *d_elements, uint32_t n, int32_t grav,
                                                const double *d_covariance, const uint8_t *d_model,
                                                const uint32_t *d_offsets, const double *d_jd, const double *d_fr,
                                                uint32_t m, int32_t frame, int32_t device, double *d_state,
                                                double *d_state_covariance, double *d_jacobian, uint8_t *d_status,
                                                void *stream) {
    az::CovArgs a{};
    int32_t rc = cov_check(n, grav, m, frame, device, &a);
    if (rc != ASTROZ_OK) return rc;
    if (n == 0 || m == 0) return ASTROZ_OK;
    if (!d_elements || !d_covariance || !d_offsets || !d_jd || !d_fr || !d_state_covariance || !d_status)
        return ASTROZ_NULL_POINTER;
    if ((rc = check_device_ordinal(device)) != ASTROZ_OK) return rc;
    AZ_CUDA(cudaSetDevice(device));
    AZ_CUDA(cov_run(a, d_elements, d_covariance, d_model, d_offsets, d_jd, d_fr, d_state, d_state_covariance,
                    d_jacobian, d_status, static_cast<cudaStream_t>(stream)));
    return ASTROZ_OK;
}

int32_t astroz_cuda_propagate_covariance(const double *elements, uint32_t n, int32_t grav, const double *covariance,
                                         const uint8_t *model, const uint32_t *offsets, const double *jd,
                                         const double *fr, uint32_t m, int32_t frame, int32_t device, double *state,
                                         double *state_covariance, double *jacobian, uint8_t *status) {
    az::CovArgs a{};
    int32_t rc = cov_check(n, grav, m, frame, device, &a);
    if (rc != ASTROZ_OK) return rc;
    if (!offsets) return ASTROZ_NULL_POINTER;
    if (n && (!elements || !covariance)) return ASTROZ_NULL_POINTER;
    if (m && (!jd || !fr || !state_covariance || !status)) return ASTROZ_NULL_POINTER;
    if ((rc = offsets_check(offsets, n, m, "offsets[n] must equal the query count m", true)) != ASTROZ_OK) return rc;
    if ((rc = rows_check(elements, covariance, n)) != ASTROZ_OK) return rc;
    if (!all_finite(jd, m) || !all_finite(fr, m)) return value_error("query times must be finite");
    if ((rc = model_bytes_check(model, n)) != ASTROZ_OK) return rc;
    if (n == 0 || m == 0) return ASTROZ_OK;
    return whole_batch(device,
                       {upload(elements, (size_t)64 * n), upload(covariance, (size_t)8 * az::kFitN * n),
                        upload(model, model ? (size_t)n : 0), upload(offsets, (size_t)4 * (n + 1)),
                        upload(jd, (size_t)8 * m), upload(fr, (size_t)8 * m), result(state, state ? (size_t)48 * m : 0),
                        result(state_covariance, (size_t)8 * az::kCovWords * m),
                        result(jacobian, jacobian ? (size_t)8 * az::kCovJacWords * m : 0), result(status, m)},
                       [&](const DeviceBlock &d, cudaStream_t st) {
                           return cov_run(a, d.f64(0), d.f64(1), model ? d.u8(2) : nullptr, d.u32(3), d.f64(4),
                                          d.f64(5), state ? d.f64(6) : nullptr, d.f64(7),
                                          jacobian ? d.f64(8) : nullptr, d.u8(9), st);
                       });
}

// ---- conjunction assessment (K11, az_conjunction.cu, az_conjunction.cuh) -------------------------------------------
static_assert(ASTROZ_CONJ_OK == az::kConjOk && ASTROZ_CONJ_INIT_FAILED == az::kConjInitFailed &&
                  ASTROZ_CONJ_CELL_FAILED == az::kConjCellFailed && ASTROZ_CONJ_WINDOW_EDGE == az::kConjWindowEdge &&
                  ASTROZ_CONJ_NO_PLANE == az::kConjNoPlane && ASTROZ_CONJ_BAD_PAIR == az::kConjBadPair &&
                  ASTROZ_CONJ_RECORD_WORDS == az::kConjRecordWords,
              "conjunction status bytes and record layout");

// Scalar checks of the conjunction calls, before anything is read, written or allocated; a receives the scalars.
static int32_t conj_check(uint32_t n, int32_t grav, uint32_t m, int32_t frame, int32_t device, az::ConjArgs *a) {
    if (device < 0) return value_error("conjunction assessment runs on one device: pass its ordinal");
    const int32_t rc = grav_check(grav);
    if (rc != ASTROZ_OK) return rc;
    if (frame != ASTROZ_COV_FRAME_TEME && frame != ASTROZ_COV_FRAME_RTN)
        return value_error("frame must be ASTROZ_COV_FRAME_TEME or ASTROZ_COV_FRAME_RTN");
    a->n = n;
    a->m = m;
    a->grav = grav;
    a->g = az::grav_consts(az::gravity(grav));
    a->frame = frame;
    return ASTROZ_OK;
}

// Both call forms: a holds conj_check's scalars, the arrays are on the device.
static cudaError_t conj_run(az::ConjArgs a, const double *elements, const double *covariance, const uint8_t *model,
                            const uint32_t *primary, const uint32_t *secondary, const double *jd, const double *fr,
                            const double *window_min, const double *hbr_km, double *record, double *states,
                            double *state_covariance, uint8_t *status, cudaStream_t st) {
    a.elements = elements;
    a.covariance = covariance;
    a.model = model;
    a.primary = primary;
    a.secondary = secondary;
    a.jd = jd;
    a.fr = fr;
    a.window = window_min;
    a.hbr = hbr_km;
    a.record = record;
    a.states = states;
    a.sigma = state_covariance;
    a.status = status;
    return az::launch_conjunction(a, st);
}

// The value checks of astroz_cuda_conjunction's host call on its catalogue and candidates (pointers already checked).
static int32_t conj_inputs_check(const double *elements, uint32_t n, const double *covariance, const uint8_t *model,
                                 const uint32_t *primary, const uint32_t *secondary, const double *jd, const double *fr,
                                 const double *window_min, const double *hbr_km, uint32_t m) {
    for (uint32_t i = 0; i < m; ++i) {
        if (primary[i] >= n || secondary[i] >= n) return value_error("a candidate's row is outside the catalogue");
        if (primary[i] == secondary[i]) return value_error("a candidate pairs a row with itself");
        if (!(window_min[i] > 0.0) || !std::isfinite(window_min[i]))
            return value_error("half windows must be finite and > 0 minutes");
        if (!(hbr_km[i] >= 0.0) || !std::isfinite(hbr_km[i]))
            return value_error("hard-body radii must be finite and >= 0 km");
    }
    int32_t rc = rows_check(elements, covariance, n);
    if (rc != ASTROZ_OK) return rc;
    if (!all_finite(jd, m) || !all_finite(fr, m)) return value_error("guess times must be finite");
    return model_bytes_check(model, n);
}

int32_t astroz_cuda_conjunction_device(const double *d_elements, uint32_t n, int32_t grav, const double *d_covariance,
                                       const uint8_t *d_model, const uint32_t *d_primary, const uint32_t *d_secondary,
                                       const double *d_jd, const double *d_fr, const double *d_window_min,
                                       const double *d_hbr_km, uint32_t m, int32_t frame, int32_t device,
                                       double *d_record, double *d_states, double *d_state_covariance,
                                       uint8_t *d_status, void *stream) {
    az::ConjArgs a{};
    int32_t rc = conj_check(n, grav, m, frame, device, &a);
    if (rc != ASTROZ_OK) return rc;
    if (m == 0) return ASTROZ_OK;
    if ((n && (!d_elements || !d_covariance)) || !d_primary || !d_secondary || !d_jd || !d_fr || !d_window_min ||
        !d_hbr_km || !d_record || !d_status)
        return ASTROZ_NULL_POINTER;
    if ((rc = check_device_ordinal(device)) != ASTROZ_OK) return rc;
    AZ_CUDA(cudaSetDevice(device));
    AZ_CUDA(conj_run(a, d_elements, d_covariance, d_model, d_primary, d_secondary, d_jd, d_fr, d_window_min, d_hbr_km,
                     d_record, d_states, d_state_covariance, d_status, static_cast<cudaStream_t>(stream)));
    return ASTROZ_OK;
}

int32_t astroz_cuda_conjunction(const double *elements, uint32_t n, int32_t grav, const double *covariance,
                                const uint8_t *model, const uint32_t *primary, const uint32_t *secondary,
                                const double *jd, const double *fr, const double *window_min, const double *hbr_km,
                                uint32_t m, int32_t frame, int32_t device, double *record, double *states,
                                double *state_covariance, uint8_t *status) {
    az::ConjArgs a{};
    int32_t rc = conj_check(n, grav, m, frame, device, &a);
    if (rc != ASTROZ_OK) return rc;
    if (n && (!elements || !covariance)) return ASTROZ_NULL_POINTER;
    if (m && (!primary || !secondary || !jd || !fr || !window_min || !hbr_km || !record || !status))
        return ASTROZ_NULL_POINTER;
    if ((rc = conj_inputs_check(elements, n, covariance, model, primary, secondary, jd, fr, window_min, hbr_km, m)) !=
        ASTROZ_OK)
        return rc;
    if (m == 0) return ASTROZ_OK;
    return whole_batch(device,
                       {upload(elements, (size_t)64 * n), upload(covariance, (size_t)8 * az::kFitN * n),
                        upload(model, model ? (size_t)n : 0), upload(primary, (size_t)4 * m),
                        upload(secondary, (size_t)4 * m), upload(jd, (size_t)8 * m), upload(fr, (size_t)8 * m),
                        upload(window_min, (size_t)8 * m), upload(hbr_km, (size_t)8 * m),
                        result(record, (size_t)8 * az::kConjRecordWords * m),
                        result(states, states ? (size_t)96 * m : 0),
                        result(state_covariance, state_covariance ? (size_t)16 * az::kCovWords * m : 0),
                        result(status, m)},
                       [&](const DeviceBlock &d, cudaStream_t st) {
                           return conj_run(a, d.f64(0), d.f64(1), model ? d.u8(2) : nullptr, d.u32(3), d.u32(4),
                                           d.f64(5), d.f64(6), d.f64(7), d.f64(8), d.f64(9),
                                           states ? d.f64(10) : nullptr, state_covariance ? d.f64(11) : nullptr,
                                           d.u8(12), st);
                       });
}

// ---- Monte Carlo collision probability (K14, az_conjunction_mc.cu, az_conjunction_mc.cuh) ----------------------------
static_assert(ASTROZ_CONJ_NOT_PSD == az::kConjNotPsd && ASTROZ_CONJ_MC_COUNT_WORDS == az::kMcCountWords &&
                  ASTROZ_CONJ_MC_SAMPLE_WORDS == az::kMcSampleWords,
              "Monte Carlo status byte and layouts");

// Scalar checks of the Monte Carlo calls: conj_check's, the frame unused
static int32_t conj_mc_check(uint32_t n, int32_t grav, uint32_t m, uint32_t record, int32_t device,
                             az::ConjMcArgs *a) {
    az::ConjArgs c{};
    const int32_t rc = conj_check(n, grav, m, ASTROZ_COV_FRAME_TEME, device, &c);
    if (rc != ASTROZ_OK) return rc;
    a->n = n;
    a->m = m;
    a->record = record;
    a->grav = grav;
    a->g = c.g;
    return ASTROZ_OK;
}

// Both call forms: a holds conj_mc_check's scalars, the arrays are on the device.
static cudaError_t conj_mc_run(az::ConjMcArgs a, const double *elements, const double *covariance,
                               const uint8_t *model, const uint32_t *primary, const uint32_t *secondary,
                               const double *jd, const double *fr, const double *window_min, const double *hbr_km,
                               const uint64_t *samples, const uint64_t *first, const uint64_t *seed, void *scratch,
                               uint64_t *counts, double *sample_out, uint8_t *status, cudaStream_t st) {
    a.elements = elements;
    a.covariance = covariance;
    a.model = model;
    a.primary = primary;
    a.secondary = secondary;
    a.jd = jd;
    a.fr = fr;
    a.window = window_min;
    a.hbr = hbr_km;
    a.samples = samples;
    a.first = first;
    a.seed = seed;
    a.scratch = scratch;
    a.counts = counts;
    a.sampleOut = sample_out;
    a.status = status;
    return az::launch_conjunction_mc(a, st);
}

int32_t astroz_cuda_conjunction_mc_scratch_bytes(uint32_t m, uint64_t *bytes) {
    if (!bytes) return ASTROZ_NULL_POINTER;
    int count = 0;
    const int32_t rc = check_device_present(&count, "no CUDA device available (the scan's scratch is the device's)");
    if (rc != ASTROZ_OK) return rc;
    size_t b = 0;
    AZ_CUDA(az::conj_mc_scratch_bytes(m, &b));
    *bytes = b;
    return ASTROZ_OK;
}

int32_t astroz_cuda_conjunction_mc_device(const double *d_elements, uint32_t n, int32_t grav,
                                          const double *d_covariance, const uint8_t *d_model,
                                          const uint32_t *d_primary, const uint32_t *d_secondary, const double *d_jd,
                                          const double *d_fr, const double *d_window_min, const double *d_hbr_km,
                                          const uint64_t *d_samples, const uint64_t *d_first, const uint64_t *d_seed,
                                          uint32_t m, uint32_t record, int32_t device, uint64_t *d_counts,
                                          double *d_sample_out, uint8_t *d_status, void *d_scratch, void *stream) {
    az::ConjMcArgs a{};
    int32_t rc = conj_mc_check(n, grav, m, record, device, &a);
    if (rc != ASTROZ_OK) return rc;
    if (m == 0) return ASTROZ_OK;
    if ((n && (!d_elements || !d_covariance)) || !d_primary || !d_secondary || !d_jd || !d_fr || !d_window_min ||
        !d_hbr_km || !d_samples || !d_counts || !d_status || !d_scratch || (record && !d_sample_out))
        return ASTROZ_NULL_POINTER;
    if ((rc = check_device_ordinal(device)) != ASTROZ_OK) return rc;
    AZ_CUDA(cudaSetDevice(device));
    AZ_CUDA(conj_mc_run(a, d_elements, d_covariance, d_model, d_primary, d_secondary, d_jd, d_fr, d_window_min,
                        d_hbr_km, d_samples, d_first, d_seed, d_scratch, d_counts, d_sample_out, d_status,
                        static_cast<cudaStream_t>(stream)));
    return ASTROZ_OK;
}

int32_t astroz_cuda_conjunction_mc(const double *elements, uint32_t n, int32_t grav, const double *covariance,
                                   const uint8_t *model, const uint32_t *primary, const uint32_t *secondary,
                                   const double *jd, const double *fr, const double *window_min, const double *hbr_km,
                                   const uint64_t *samples, const uint64_t *first, const uint64_t *seed, uint32_t m,
                                   uint32_t record, int32_t device, uint64_t *counts, double *sample_out,
                                   uint8_t *status) {
    az::ConjMcArgs a{};
    int32_t rc = conj_mc_check(n, grav, m, record, device, &a);
    if (rc != ASTROZ_OK) return rc;
    if (n && (!elements || !covariance)) return ASTROZ_NULL_POINTER;
    if (m && (!primary || !secondary || !jd || !fr || !window_min || !hbr_km || !samples || !counts || !status))
        return ASTROZ_NULL_POINTER;
    if (m && record && !sample_out) return value_error("record > 0 needs sample_out");
    for (uint32_t i = 0; i < m; ++i) {
        if (primary[i] >= n || secondary[i] >= n) return value_error("a candidate's row is outside the catalogue");
        if (primary[i] == secondary[i]) return value_error("a candidate pairs a row with itself");
        if (!(window_min[i] > 0.0) || !std::isfinite(window_min[i]))
            return value_error("half windows must be finite and > 0 minutes");
        if (!(hbr_km[i] >= 0.0) || !std::isfinite(hbr_km[i]))
            return value_error("hard-body radii must be finite and >= 0 km");
        if (first && samples[i] > UINT64_MAX - first[i])
            return value_error("first + samples must not exceed 2^64 - 1");
    }
    if ((rc = rows_check(elements, covariance, n)) != ASTROZ_OK) return rc;
    if (!all_finite(jd, m) || !all_finite(fr, m)) return value_error("guess times must be finite");
    if ((rc = model_bytes_check(model, n)) != ASTROZ_OK) return rc;
    if (m == 0) return ASTROZ_OK;
    if ((rc = check_device_ordinal(device)) != ASTROZ_OK) return rc;
    size_t scratchBytes = 0;
    AZ_CUDA(cudaSetDevice(device));
    AZ_CUDA(az::conj_mc_scratch_bytes(m, &scratchBytes));
    return whole_batch(device,
                       {upload(elements, (size_t)64 * n), upload(covariance, (size_t)8 * az::kFitN * n),
                        upload(model, model ? (size_t)n : 0), upload(primary, (size_t)4 * m),
                        upload(secondary, (size_t)4 * m), upload(jd, (size_t)8 * m), upload(fr, (size_t)8 * m),
                        upload(window_min, (size_t)8 * m), upload(hbr_km, (size_t)8 * m),
                        upload(samples, (size_t)8 * m), upload(first, first ? (size_t)8 * m : 0),
                        upload(seed, seed ? (size_t)8 * m : 0), scratch(scratchBytes),
                        result(counts, (size_t)8 * az::kMcCountWords * m),
                        result(sample_out, (size_t)8 * az::kMcSampleWords * record * m), result(status, m)},
                       [&](const DeviceBlock &d, cudaStream_t st) {
                           return conj_mc_run(a, d.f64(0), d.f64(1), model ? d.u8(2) : nullptr, d.u32(3), d.u32(4),
                                              d.f64(5), d.f64(6), d.f64(7), d.f64(8),
                                              reinterpret_cast<const uint64_t *>(d.piece(9)),
                                              first ? reinterpret_cast<const uint64_t *>(d.piece(10)) : nullptr,
                                              seed ? reinterpret_cast<const uint64_t *>(d.piece(11)) : nullptr,
                                              d.piece(12), reinterpret_cast<uint64_t *>(d.piece(13)),
                                              record ? d.f64(14) : nullptr, d.u8(15), st);
                       });
}

// ---- reentry prediction (K19, az_reentry.cu, az_reentry.cuh) ---------------------------------------------------------
// Scalar checks of the reentry calls, before anything is read, written or allocated; a receives the scalars.
static int32_t reentry_check(uint32_t n, int32_t grav, uint32_t m, double h_i, double horizon_days, double step_s,
                             double density_scale, double density_sigma, uint32_t record, int32_t device,
                             az::ReentryArgs *a) {
    if (device < 0) return value_error("reentry prediction runs on one device: pass its ordinal");
    const int32_t rc = grav_check(grav);
    if (rc != ASTROZ_OK) return rc;
    if (!(h_i >= 60.0 && h_i <= 200.0)) return value_error("h_i must be in [60, 200] km");
    if (!(horizon_days > 0.0 && horizon_days <= 3660.0)) return value_error("horizon_days must be in (0, 3660]");
    if (!(step_s >= 1.0 && step_s <= 3600.0)) return value_error("step_s must be in [1, 3600] s");
    if (!(density_sigma >= 0.0 && density_sigma <= 2.0)) return value_error("density_sigma must be in [0, 2]");
    if (!(density_scale > 0.0) || !std::isfinite(density_scale))
        return value_error("density_scale must be finite and > 0");
    a->n = n;
    a->m = m;
    a->record = record;
    const az::Gravity gr = az::gravity(grav);
    a->call = {h_i, horizon_days * 86400.0, step_s, density_scale, density_sigma, 7.292115e-5, gr.mu, gr.radiusEarthKm,
               gr.j2};
    a->grav = grav;
    a->g = az::grav_consts(gr);
    return ASTROZ_OK;
}

// Both call forms: a holds reentry_check's scalars, the arrays are on the device.
static cudaError_t reentry_run(az::ReentryArgs a, const double *elements, const double *covariance,
                               const uint8_t *model, const uint32_t *rows, const double *ballistic,
                               const uint64_t *samples, const uint64_t *first, const uint64_t *seed, void *scratch,
                               double *record_out, double *states, uint8_t *nominal_status, uint64_t *counts,
                               double *sample_out, uint8_t *status, cudaStream_t st) {
    a.elements = elements;
    a.covariance = covariance;
    a.model = model;
    a.rows = rows;
    a.ballistic = ballistic;
    a.samples = samples;
    a.first = first;
    a.seed = seed;
    a.scratch = scratch;
    a.out = record_out;
    a.states = states;
    a.nominalStatus = nominal_status;
    a.counts = counts;
    a.sampleOut = sample_out;
    a.status = status;
    return az::launch_reentry(a, st);
}

int32_t astroz_cuda_reentry_scratch_bytes(uint32_t m, uint64_t *bytes) {
    if (!bytes) return ASTROZ_NULL_POINTER;
    int count = 0;
    const int32_t rc = check_device_present(&count, "no CUDA device available (the scan's scratch is the device's)");
    if (rc != ASTROZ_OK) return rc;
    size_t b = 0;
    AZ_CUDA(az::reentry_scratch_bytes(m, &b));
    *bytes = b;
    return ASTROZ_OK;
}

int32_t astroz_cuda_reentry_device(const double *d_elements, uint32_t n, int32_t grav, const double *d_covariance,
                                   const uint8_t *d_model, const uint32_t *d_rows, const double *d_ballistic,
                                   const uint64_t *d_samples, const uint64_t *d_first, const uint64_t *d_seed,
                                   uint32_t m, double h_i, double horizon_days, double step_s, double density_scale,
                                   double density_sigma, uint32_t record, int32_t device, double *d_record_out,
                                   double *d_states, uint8_t *d_nominal_status, uint64_t *d_counts,
                                   double *d_sample_out, uint8_t *d_status, void *d_scratch, void *stream) {
    az::ReentryArgs a{};
    int32_t rc = reentry_check(n, grav, m, h_i, horizon_days, step_s, density_scale, density_sigma, record, device, &a);
    if (rc != ASTROZ_OK) return rc;
    if (m == 0) return ASTROZ_OK;
    if ((n && (!d_elements || !d_covariance)) || !d_rows || !d_samples || !d_record_out || !d_nominal_status ||
        !d_counts || !d_status || !d_scratch || (record && !d_sample_out))
        return ASTROZ_NULL_POINTER;
    if ((rc = check_device_ordinal(device)) != ASTROZ_OK) return rc;
    AZ_CUDA(cudaSetDevice(device));
    AZ_CUDA(reentry_run(a, d_elements, d_covariance, d_model, d_rows, d_ballistic, d_samples, d_first, d_seed,
                        d_scratch, d_record_out, d_states, d_nominal_status, d_counts, d_sample_out, d_status,
                        static_cast<cudaStream_t>(stream)));
    return ASTROZ_OK;
}

int32_t astroz_cuda_reentry(const double *elements, uint32_t n, int32_t grav, const double *covariance,
                            const uint8_t *model, const uint32_t *rows, const double *ballistic, const uint64_t *samples,
                            const uint64_t *first, const uint64_t *seed, uint32_t m, double h_i, double horizon_days,
                            double step_s, double density_scale, double density_sigma, uint32_t record, int32_t device,
                            double *record_out, double *states, uint8_t *nominal_status, uint64_t *counts,
                            double *sample_out, uint8_t *status) {
    az::ReentryArgs a{};
    int32_t rc = reentry_check(n, grav, m, h_i, horizon_days, step_s, density_scale, density_sigma, record, device, &a);
    if (rc != ASTROZ_OK) return rc;
    if (n && (!elements || !covariance)) return ASTROZ_NULL_POINTER;
    if (m && (!rows || !samples || !record_out || !nominal_status || !counts || !status)) return ASTROZ_NULL_POINTER;
    if (m && record && !sample_out) return value_error("record > 0 needs sample_out");
    for (uint32_t i = 0; i < m; ++i) {
        if (rows[i] >= n) return value_error("a request's row is outside the catalogue");
        if (first && samples[i] > UINT64_MAX - first[i])
            return value_error("first + samples must not exceed 2^64 - 1");
    }
    if (ballistic && !all_finite(ballistic, m)) return value_error("ballistic coefficients must be finite");
    if ((rc = rows_check(elements, covariance, n)) != ASTROZ_OK) return rc;
    if ((rc = model_bytes_check(model, n)) != ASTROZ_OK) return rc;
    if (m == 0) return ASTROZ_OK;
    if ((rc = check_device_ordinal(device)) != ASTROZ_OK) return rc;
    size_t scratchBytes = 0;
    AZ_CUDA(cudaSetDevice(device));
    AZ_CUDA(az::reentry_scratch_bytes(m, &scratchBytes));
    return whole_batch(device,
                       {upload(elements, (size_t)64 * n), upload(covariance, (size_t)8 * az::kFitN * n),
                        upload(model, model ? (size_t)n : 0), upload(rows, (size_t)4 * m),
                        upload(ballistic, ballistic ? (size_t)8 * m : 0), upload(samples, (size_t)8 * m),
                        upload(first, first ? (size_t)8 * m : 0), upload(seed, seed ? (size_t)8 * m : 0),
                        scratch(scratchBytes), result(record_out, (size_t)8 * ASTROZ_REENTRY_RECORD_WORDS * m),
                        result(states, states ? (size_t)8 * ASTROZ_REENTRY_STATE_WORDS * m : 0),
                        result(nominal_status, m), result(counts, (size_t)8 * ASTROZ_REENTRY_COUNT_WORDS * m),
                        result(sample_out, (size_t)8 * ASTROZ_REENTRY_SAMPLE_WORDS * record * m), result(status, m)},
                       [&](const DeviceBlock &d, cudaStream_t st) {
                           return reentry_run(a, d.f64(0), d.f64(1), model ? d.u8(2) : nullptr, d.u32(3),
                                              ballistic ? d.f64(4) : nullptr,
                                              reinterpret_cast<const uint64_t *>(d.piece(5)),
                                              first ? reinterpret_cast<const uint64_t *>(d.piece(6)) : nullptr,
                                              seed ? reinterpret_cast<const uint64_t *>(d.piece(7)) : nullptr,
                                              d.piece(8), d.f64(9), states ? d.f64(10) : nullptr, d.u8(11),
                                              reinterpret_cast<uint64_t *>(d.piece(12)), record ? d.f64(13) : nullptr,
                                              d.u8(14), st);
                       });
}

// ---- importance-sampled collision probability (K15, az_conjunction_is.cu, az_conjunction_is.cuh) ---------------------
static_assert(ASTROZ_CONJ_IS_COUNT_WORDS == az::kIsCountWords && ASTROZ_CONJ_IS_PROPOSAL_WORDS == az::kIsProposalWords &&
                  ASTROZ_CONJ_IS_SAMPLE_WORDS == az::kIsSampleWords && ASTROZ_CONJ_IS_LINEAR == az::kIsLinear &&
                  ASTROZ_CONJ_IS_GIVEN == az::kIsGiven && ASTROZ_CONJ_IS_PLAIN == az::kIsPlain,
              "importance-sampling layouts and proposal kinds");

// Both call forms: a holds conj_mc_check's scalars, the arrays are on the device.
static cudaError_t conj_is_run(az::ConjIsArgs a, const double *elements, const double *covariance,
                               const uint8_t *model, const uint32_t *primary, const uint32_t *secondary,
                               const double *jd, const double *fr, const double *window_min, const double *hbr_km,
                               const uint64_t *samples, const uint64_t *first, const uint64_t *seed,
                               const double *shift, void *scratch, uint64_t *counts, double *proposal,
                               uint8_t *proposal_kind, double *sample_out, uint8_t *status, cudaStream_t st) {
    a.elements = elements;
    a.covariance = covariance;
    a.model = model;
    a.primary = primary;
    a.secondary = secondary;
    a.jd = jd;
    a.fr = fr;
    a.window = window_min;
    a.hbr = hbr_km;
    a.samples = samples;
    a.first = first;
    a.seed = seed;
    a.shift = shift;
    a.scratch = scratch;
    a.counts = counts;
    a.proposal = proposal;
    a.kind = proposal_kind;
    a.sampleOut = sample_out;
    a.status = status;
    return az::launch_conjunction_is(a, st);
}

int32_t astroz_cuda_conjunction_is_scratch_bytes(uint32_t m, uint64_t *bytes) {
    if (!bytes) return ASTROZ_NULL_POINTER;
    int count = 0;
    const int32_t rc = check_device_present(&count, "no CUDA device available (the scan's scratch is the device's)");
    if (rc != ASTROZ_OK) return rc;
    size_t b = 0;
    AZ_CUDA(az::conj_is_scratch_bytes(m, &b));
    *bytes = b;
    return ASTROZ_OK;
}

int32_t astroz_cuda_conjunction_is_device(const double *d_elements, uint32_t n, int32_t grav,
                                          const double *d_covariance, const uint8_t *d_model,
                                          const uint32_t *d_primary, const uint32_t *d_secondary, const double *d_jd,
                                          const double *d_fr, const double *d_window_min, const double *d_hbr_km,
                                          const uint64_t *d_samples, const uint64_t *d_first, const uint64_t *d_seed,
                                          const double *d_shift, uint32_t m, uint32_t record, int32_t device,
                                          uint64_t *d_counts, double *d_proposal, uint8_t *d_proposal_kind,
                                          double *d_sample_out, uint8_t *d_status, void *d_scratch, void *stream) {
    az::ConjIsArgs a{};
    int32_t rc = conj_mc_check(n, grav, m, record, device, &a);
    if (rc != ASTROZ_OK) return rc;
    if (m == 0) return ASTROZ_OK;
    if ((n && (!d_elements || !d_covariance)) || !d_primary || !d_secondary || !d_jd || !d_fr || !d_window_min ||
        !d_hbr_km || !d_samples || !d_counts || !d_status || !d_scratch || (record && !d_sample_out))
        return ASTROZ_NULL_POINTER;
    if ((rc = check_device_ordinal(device)) != ASTROZ_OK) return rc;
    AZ_CUDA(cudaSetDevice(device));
    AZ_CUDA(conj_is_run(a, d_elements, d_covariance, d_model, d_primary, d_secondary, d_jd, d_fr, d_window_min,
                        d_hbr_km, d_samples, d_first, d_seed, d_shift, d_scratch, d_counts, d_proposal,
                        d_proposal_kind, d_sample_out, d_status, static_cast<cudaStream_t>(stream)));
    return ASTROZ_OK;
}

int32_t astroz_cuda_conjunction_is(const double *elements, uint32_t n, int32_t grav, const double *covariance,
                                   const uint8_t *model, const uint32_t *primary, const uint32_t *secondary,
                                   const double *jd, const double *fr, const double *window_min, const double *hbr_km,
                                   const uint64_t *samples, const uint64_t *first, const uint64_t *seed,
                                   const double *shift, uint32_t m, uint32_t record, int32_t device, uint64_t *counts,
                                   double *proposal, uint8_t *proposal_kind, double *sample_out, uint8_t *status) {
    az::ConjIsArgs a{};
    int32_t rc = conj_mc_check(n, grav, m, record, device, &a);
    if (rc != ASTROZ_OK) return rc;
    if (n && (!elements || !covariance)) return ASTROZ_NULL_POINTER;
    if (m && (!primary || !secondary || !jd || !fr || !window_min || !hbr_km || !samples || !counts || !status))
        return ASTROZ_NULL_POINTER;
    if (m && record && !sample_out) return value_error("record > 0 needs sample_out");
    for (uint32_t i = 0; i < m; ++i) {
        if (primary[i] >= n || secondary[i] >= n) return value_error("a candidate's row is outside the catalogue");
        if (primary[i] == secondary[i]) return value_error("a candidate pairs a row with itself");
        if (!(window_min[i] > 0.0) || !std::isfinite(window_min[i]))
            return value_error("half windows must be finite and > 0 minutes");
        if (!(hbr_km[i] >= 0.0) || !std::isfinite(hbr_km[i]))
            return value_error("hard-body radii must be finite and >= 0 km");
        if (first && samples[i] > UINT64_MAX - first[i])
            return value_error("first + samples must not exceed 2^64 - 1");
    }
    if ((rc = rows_check(elements, covariance, n)) != ASTROZ_OK) return rc;
    if (!all_finite(jd, m) || !all_finite(fr, m)) return value_error("guess times must be finite");
    if ((rc = model_bytes_check(model, n)) != ASTROZ_OK) return rc;
    if (shift && !all_finite(shift, (size_t)az::kIsShift * m)) return value_error("shift words must be finite");
    if (m == 0) return ASTROZ_OK;
    if ((rc = check_device_ordinal(device)) != ASTROZ_OK) return rc;
    size_t scratchBytes = 0;
    AZ_CUDA(cudaSetDevice(device));
    AZ_CUDA(az::conj_is_scratch_bytes(m, &scratchBytes));
    return whole_batch(device,
                       {upload(elements, (size_t)64 * n), upload(covariance, (size_t)8 * az::kFitN * n),
                        upload(model, model ? (size_t)n : 0), upload(primary, (size_t)4 * m),
                        upload(secondary, (size_t)4 * m), upload(jd, (size_t)8 * m), upload(fr, (size_t)8 * m),
                        upload(window_min, (size_t)8 * m), upload(hbr_km, (size_t)8 * m),
                        upload(samples, (size_t)8 * m), upload(first, first ? (size_t)8 * m : 0),
                        upload(seed, seed ? (size_t)8 * m : 0), upload(shift, shift ? (size_t)8 * az::kIsShift * m : 0),
                        scratch(scratchBytes), result(counts, (size_t)8 * az::kIsCountWords * m),
                        result(proposal, proposal ? (size_t)8 * az::kIsProposalWords * m : 0),
                        result(proposal_kind, proposal_kind ? (size_t)m : 0),
                        result(sample_out, (size_t)8 * az::kIsSampleWords * record * m), result(status, m)},
                       [&](const DeviceBlock &d, cudaStream_t st) {
                           return conj_is_run(a, d.f64(0), d.f64(1), model ? d.u8(2) : nullptr, d.u32(3), d.u32(4),
                                              d.f64(5), d.f64(6), d.f64(7), d.f64(8),
                                              reinterpret_cast<const uint64_t *>(d.piece(9)),
                                              first ? reinterpret_cast<const uint64_t *>(d.piece(10)) : nullptr,
                                              seed ? reinterpret_cast<const uint64_t *>(d.piece(11)) : nullptr,
                                              shift ? d.f64(12) : nullptr, d.piece(13),
                                              reinterpret_cast<uint64_t *>(d.piece(14)),
                                              proposal ? d.f64(15) : nullptr, proposal_kind ? d.u8(16) : nullptr,
                                              record ? d.f64(17) : nullptr, d.u8(18), st);
                       });
}

// ---- collision-avoidance manoeuvre trials (K16, az_avoid.cu, az_avoid.cuh) -------------------------------------------
static_assert(ASTROZ_CONJ_CONVERSION_FAILED == az::kConjConversionFailed && ASTROZ_CONJ_BAD_TRIAL == az::kConjBadTrial,
              "manoeuvre status bytes");

// Scalar checks of the manoeuvre calls, before anything is read, written or allocated; a receives the scalars.
static int32_t avoid_check(uint32_t n, int32_t grav, uint32_t m, uint32_t t, int32_t device, az::AvoidArgs *a) {
    if (device < 0) return value_error("manoeuvre trials run on one device: pass its ordinal");
    const int32_t rc = grav_check(grav);
    if (rc != ASTROZ_OK) return rc;
    if (t >= 0x80000000u) return value_error("t must be below 2^31 (the reassessment's catalogue has 2t rows)");
    a->n = n;
    a->m = m;
    a->t = t;
    a->grav = grav;
    a->g = az::grav_consts(az::gravity(grav));
    return ASTROZ_OK;
}

// Both call forms: a holds avoid_check's scalars, the arrays are on the device.
static cudaError_t avoid_run(az::AvoidArgs a, const double *elements, const double *covariance, const uint8_t *model,
                             const uint32_t *primary, const uint32_t *secondary, const double *jd, const double *fr,
                             const double *window_min, const double *hbr_km, const uint32_t *candidate,
                             const double *burn_jd, const double *burn_fr, const double *dv_rtn,
                             const double *dv_sigma, void *scratch, double *record, double *new_elements,
                             double *new_covariance, double *residual, uint8_t *status, cudaStream_t st) {
    a.elements = elements;
    a.covariance = covariance;
    a.model = model;
    a.primary = primary;
    a.secondary = secondary;
    a.jd = jd;
    a.fr = fr;
    a.window = window_min;
    a.hbr = hbr_km;
    a.candidate = candidate;
    a.burnJd = burn_jd;
    a.burnFr = burn_fr;
    a.dv = dv_rtn;
    a.dvSigma = dv_sigma;
    a.scratch = scratch;
    a.record = record;
    a.newElements = new_elements;
    a.newCovariance = new_covariance;
    a.residual = residual;
    a.status = status;
    return az::launch_avoid(a, st);
}

int32_t astroz_cuda_conjunction_maneuver_scratch_bytes(uint32_t t, uint64_t *bytes) {
    if (!bytes) return ASTROZ_NULL_POINTER;
    *bytes = az::avoid_scratch_bytes(t);
    return ASTROZ_OK;
}

int32_t astroz_cuda_conjunction_maneuver_device(const double *d_elements, uint32_t n, int32_t grav,
                                                const double *d_covariance, const uint8_t *d_model,
                                                const uint32_t *d_primary, const uint32_t *d_secondary,
                                                const double *d_jd, const double *d_fr, const double *d_window_min,
                                                const double *d_hbr_km, uint32_t m, const uint32_t *d_candidate,
                                                const double *d_burn_jd, const double *d_burn_fr,
                                                const double *d_dv_rtn, const double *d_dv_sigma, uint32_t t,
                                                int32_t device, double *d_record, double *d_new_elements,
                                                double *d_new_covariance, double *d_residual, uint8_t *d_status,
                                                void *d_scratch, void *stream) {
    az::AvoidArgs a{};
    int32_t rc = avoid_check(n, grav, m, t, device, &a);
    if (rc != ASTROZ_OK) return rc;
    if (t == 0) return ASTROZ_OK;
    if ((n && (!d_elements || !d_covariance)) || (m && (!d_primary || !d_secondary || !d_jd || !d_fr ||
                                                        !d_window_min || !d_hbr_km)) ||
        !d_candidate || !d_burn_jd || !d_burn_fr || !d_dv_rtn || !d_record || !d_status || !d_scratch)
        return ASTROZ_NULL_POINTER;
    if ((rc = check_device_ordinal(device)) != ASTROZ_OK) return rc;
    AZ_CUDA(cudaSetDevice(device));
    AZ_CUDA(avoid_run(a, d_elements, d_covariance, d_model, d_primary, d_secondary, d_jd, d_fr, d_window_min, d_hbr_km,
                      d_candidate, d_burn_jd, d_burn_fr, d_dv_rtn, d_dv_sigma, d_scratch, d_record, d_new_elements,
                      d_new_covariance, d_residual, d_status, static_cast<cudaStream_t>(stream)));
    return ASTROZ_OK;
}

int32_t astroz_cuda_conjunction_maneuver(const double *elements, uint32_t n, int32_t grav, const double *covariance,
                                         const uint8_t *model, const uint32_t *primary, const uint32_t *secondary,
                                         const double *jd, const double *fr, const double *window_min,
                                         const double *hbr_km, uint32_t m, const uint32_t *candidate,
                                         const double *burn_jd, const double *burn_fr, const double *dv_rtn,
                                         const double *dv_sigma, uint32_t t, int32_t device, double *record,
                                         double *new_elements, double *new_covariance, double *residual,
                                         uint8_t *status) {
    az::AvoidArgs a{};
    int32_t rc = avoid_check(n, grav, m, t, device, &a);
    if (rc != ASTROZ_OK) return rc;
    if (n && (!elements || !covariance)) return ASTROZ_NULL_POINTER;
    if (m && (!primary || !secondary || !jd || !fr || !window_min || !hbr_km)) return ASTROZ_NULL_POINTER;
    if (t && (!candidate || !burn_jd || !burn_fr || !dv_rtn || !record || !status)) return ASTROZ_NULL_POINTER;
    if ((rc = conj_inputs_check(elements, n, covariance, model, primary, secondary, jd, fr, window_min, hbr_km, m)) !=
        ASTROZ_OK)
        return rc;
    if (!all_finite(burn_jd, t) || !all_finite(burn_fr, t)) return value_error("burn times must be finite");
    if (!all_finite(dv_rtn, (size_t)3 * t)) return value_error("dv words must be finite");
    if (dv_sigma)
        for (size_t q = 0; q < (size_t)3 * t; ++q)
            if (!(dv_sigma[q] >= 0.0) || !std::isfinite(dv_sigma[q]))
                return value_error("execution sigmas must be finite and >= 0 km/s");
    for (uint32_t k = 0; k < t; ++k) {
        const uint32_t c = candidate[k];
        if (c >= m) return value_error("a trial's candidate index is not below m");
        const double epoch = elements[primary[c]];
        const double tsb = az::pairs_tsince_deep(az::add_rn(burn_jd[k], burn_fr[k]), epoch);
        const double ts0 = az::pairs_tsince_deep(az::add_rn(jd[c], fr[c]), epoch);
        if (!(tsb <= ts0 - window_min[c])) return value_error("a burn does not come before its candidate's window");
    }
    if (t == 0) return ASTROZ_OK;
    return whole_batch(device,
                       {upload(elements, (size_t)64 * n), upload(covariance, (size_t)8 * az::kFitN * n),
                        upload(model, model ? (size_t)n : 0), upload(primary, (size_t)4 * m),
                        upload(secondary, (size_t)4 * m), upload(jd, (size_t)8 * m), upload(fr, (size_t)8 * m),
                        upload(window_min, (size_t)8 * m), upload(hbr_km, (size_t)8 * m),
                        upload(candidate, (size_t)4 * t), upload(burn_jd, (size_t)8 * t),
                        upload(burn_fr, (size_t)8 * t), upload(dv_rtn, (size_t)24 * t),
                        upload(dv_sigma, dv_sigma ? (size_t)24 * t : 0), scratch(az::avoid_scratch_bytes(t)),
                        result(record, (size_t)8 * az::kConjRecordWords * t),
                        result(new_elements, new_elements ? (size_t)64 * t : 0),
                        result(new_covariance, new_covariance ? (size_t)8 * az::kFitN * t : 0),
                        result(residual, residual ? (size_t)16 * t : 0), result(status, t)},
                       [&](const DeviceBlock &d, cudaStream_t st) {
                           return avoid_run(a, d.f64(0), d.f64(1), model ? d.u8(2) : nullptr, d.u32(3), d.u32(4),
                                            d.f64(5), d.f64(6), d.f64(7), d.f64(8), d.u32(9), d.f64(10), d.f64(11),
                                            d.f64(12), dv_sigma ? d.f64(13) : nullptr, d.piece(14), d.f64(15),
                                            new_elements ? d.f64(16) : nullptr, new_covariance ? d.f64(17) : nullptr,
                                            residual ? d.f64(18) : nullptr, d.u8(19), st);
                       });
}

// ---- track correlation (K12, az_correlate.cu, az_correlate.cuh) -------------------------------------------------------
static_assert(ASTROZ_CORR_OK == az::kCorrOk && ASTROZ_CORR_UNCORRELATED == az::kCorrUncorrelated &&
                  ASTROZ_CORR_NO_ROW == az::kCorrNoRow && ASTROZ_CORR_BAD_TRACK == az::kCorrBadTrack &&
                  ASTROZ_CORR_MAX_TRACK == az::kCorrMaxTrack && ASTROZ_CORR_MAX_BEST == az::kCorrMaxBest,
              "correlation status bytes and limits");

// Scalar checks of the correlation calls, before anything is read, written or allocated; a receives the scalars.
static int32_t corr_check(uint32_t n, int32_t grav, uint32_t t, double gate_probability, uint32_t best,
                          int32_t device, az::CorrArgs *a) {
    if (device < 0) return value_error("track correlation runs on one device: pass its ordinal");
    const int32_t rc = grav_check(grav);
    if (rc != ASTROZ_OK) return rc;
    if (best < 1 || best > (uint32_t)az::kCorrMaxBest) return value_error("best must be in [1, ASTROZ_CORR_MAX_BEST]");
    if (!(gate_probability > 0.0 && gate_probability < 1.0)) return value_error("gate_probability must be in (0, 1)");
    a->n = n;
    a->t = t;
    a->grav = grav;
    a->g = az::grav_consts(az::gravity(grav));
    a->gateProbability = gate_probability;
    a->best = best;
    return ASTROZ_OK;
}

int32_t astroz_cuda_correlate_scratch_bytes(uint32_t n, uint32_t t, uint32_t best, uint64_t *bytes) {
    if (!bytes) return ASTROZ_NULL_POINTER;
    if (best < 1 || best > (uint32_t)az::kCorrMaxBest) return value_error("best must be in [1, ASTROZ_CORR_MAX_BEST]");
    *bytes = az::corr_scratch_bytes(n, t, best);
    return ASTROZ_OK;
}

int32_t astroz_cuda_chi2_quantile(uint32_t k, double p, double *x) {
    if (!x) return ASTROZ_NULL_POINTER;
    if (k == 0 || !(p > 0.0 && p < 1.0)) return value_error("the chi-square quantile needs k >= 1 and p in (0, 1)");
    *x = az::corr_chi2_quantile(k, p);
    return ASTROZ_OK;
}

// Both call forms: a holds corr_check's scalars, the arrays and the scratch are on the device.
static cudaError_t corr_run(az::CorrArgs a, const double *elements, const double *covariance, const uint8_t *model,
                            const uint32_t *offsets, const double *jd, const double *fr, const uint8_t *kind,
                            const double *value, const double *sigma, const uint32_t *station,
                            const double *stations, void *scratch, uint32_t *rows, double *d2, uint32_t *used,
                            uint32_t *n_gate, uint32_t *n_failed, uint8_t *status, uint8_t *row_status,
                            cudaStream_t st) {
    a.elements = elements;
    a.covariance = covariance;
    a.model = model;
    a.offsets = offsets;
    a.jd = jd;
    a.fr = fr;
    a.kind = kind;
    a.value = value;
    a.sigma = sigma;
    a.station = station;
    a.stations = stations;
    a.scratch = scratch;
    a.rows = rows;
    a.d2 = d2;
    a.used = used;
    a.nGate = n_gate;
    a.nFailed = n_failed;
    a.status = status;
    a.rowStatus = row_status;
    return az::launch_correlate(a, st);
}

int32_t astroz_cuda_correlate_device(const double *d_elements, uint32_t n, int32_t grav, const double *d_covariance,
                                     const uint8_t *d_model, const uint32_t *d_offsets, uint32_t t, const double *d_jd,
                                     const double *d_fr, const uint8_t *d_kind, const double *d_value,
                                     const double *d_sigma, const uint32_t *d_station, const double *d_stations,
                                     double gate_probability, uint32_t best, int32_t device, void *d_scratch,
                                     uint32_t *d_rows, double *d_d2, uint32_t *d_used, uint32_t *d_n_gate,
                                     uint32_t *d_n_failed, uint8_t *d_status, uint8_t *d_row_status, void *stream) {
    az::CorrArgs a{};
    int32_t rc = corr_check(n, grav, t, gate_probability, best, device, &a);
    if (rc != ASTROZ_OK) return rc;
    if (n == 0 && t == 0) return ASTROZ_OK;
    if ((n && (!d_elements || !d_row_status)) || !d_offsets || !d_scratch)
        return ASTROZ_NULL_POINTER;
    if (t && (!d_jd || !d_fr || !d_kind || !d_value || !d_sigma || !d_rows || !d_d2 || !d_used || !d_n_gate ||
              !d_n_failed || !d_status))
        return ASTROZ_NULL_POINTER;
    if ((rc = check_device_ordinal(device)) != ASTROZ_OK) return rc;
    AZ_CUDA(cudaSetDevice(device));
    AZ_CUDA(corr_run(a, d_elements, d_covariance, d_model, d_offsets, d_jd, d_fr, d_kind, d_value, d_sigma, d_station,
                     d_stations, d_scratch, d_rows, d_d2, d_used, d_n_gate, d_n_failed, d_status, d_row_status,
                     static_cast<cudaStream_t>(stream)));
    return ASTROZ_OK;
}

int32_t astroz_cuda_correlate(const double *elements, uint32_t n, int32_t grav, const double *covariance,
                              const uint8_t *model, const uint32_t *offsets, uint32_t t, const double *jd,
                              const double *fr, const uint8_t *kind, const double *value, const double *sigma,
                              const uint32_t *station, uint32_t m, const double *stations, uint32_t k,
                              double gate_probability, uint32_t best, int32_t device, uint32_t *rows, double *d2,
                              uint32_t *used, uint32_t *n_gate, uint32_t *n_failed, uint8_t *status,
                              uint8_t *row_status) {
    az::CorrArgs a{};
    int32_t rc = corr_check(n, grav, t, gate_probability, best, device, &a);
    if (rc != ASTROZ_OK) return rc;
    if (!offsets) return ASTROZ_NULL_POINTER;
    if (n && (!elements || !row_status)) return ASTROZ_NULL_POINTER;
    if (t && (!rows || !d2 || !used || !n_gate || !n_failed || !status)) return ASTROZ_NULL_POINTER;
    if (m && (!jd || !fr || !kind || !value || !sigma)) return ASTROZ_NULL_POINTER;
    if ((rc = offsets_check(offsets, t, m, "offsets[t] must equal the observation count m", true, az::kCorrMaxTrack,
                            "a track is longer than ASTROZ_CORR_MAX_TRACK observations")) != ASTROZ_OK)
        return rc;
    if ((rc = obs_values_check(jd, fr, value, sigma, station, kind, m, stations, k)) != ASTROZ_OK) return rc;
    if ((rc = used_residuals_check({jd, fr, kind, value, sigma, station, stations}, offsets, t)) != ASTROZ_OK)
        return rc;
    if ((rc = rows_check(elements, covariance, n)) != ASTROZ_OK) return rc;
    if ((rc = model_bytes_check(model, n)) != ASTROZ_OK) return rc;
    if (n == 0 && t == 0) return ASTROZ_OK;
    return whole_batch(device,
                       {upload(elements, (size_t)64 * n),
                        upload(covariance, covariance ? (size_t)8 * az::kFitN * n : 0),
                        upload(model, model ? (size_t)n : 0), upload(offsets, (size_t)4 * (t + 1)),
                        upload(jd, (size_t)8 * m), upload(fr, (size_t)8 * m), upload(kind, m),
                        upload(value, (size_t)48 * m), upload(sigma, (size_t)48 * m),
                        upload(station, station ? (size_t)4 * m : 0), upload(stations, (size_t)24 * k),
                        scratch(az::corr_scratch_bytes(n, t, best)), result(rows, (size_t)4 * best * t),
                        result(d2, (size_t)8 * best * t), result(used, (size_t)4 * t), result(n_gate, (size_t)4 * t),
                        result(n_failed, (size_t)4 * t), result(status, t), result(row_status, n)},
                       [&](const DeviceBlock &d, cudaStream_t st) {
                           return corr_run(a, d.f64(0), covariance ? d.f64(1) : nullptr, model ? d.u8(2) : nullptr,
                                           d.u32(3), d.f64(4), d.f64(5), d.u8(6), d.f64(7), d.f64(8),
                                           station ? d.u32(9) : nullptr, k ? d.f64(10) : nullptr, d.piece(11),
                                           d.u32(12), d.f64(13), d.u32(14), d.u32(15), d.u32(16), d.u8(17), d.u8(18),
                                           st);
                       });
}

// ---- sensor tasking (K18, az_tasking.cu, az_tasking.cuh) --------------------------------------------------------------
static_assert(ASTROZ_TASK_MAX_SENSORS == az::kTaskMaxSensors && ASTROZ_TASK_LIMIT_EL_MIN == az::kTaskElMin &&
                  ASTROZ_TASK_LIMIT_RANGE_MAX == az::kTaskRangeMax &&
                  ASTROZ_TASK_LIMIT_SUN_EL_MAX == az::kTaskSunElMax &&
                  ASTROZ_TASK_LIMIT_EXCLUSION == az::kTaskExclusion,
              "tasking limits");

// Scalar checks of the tasking calls, before anything is read, written or allocated; a receives the scalars.
static int32_t task_check(uint32_t n, int32_t grav, uint32_t s, uint32_t t, double gain_min, int32_t device,
                          az::TaskArgs *a) {
    if (device < 0) return value_error("sensor tasking runs on one device: pass its ordinal");
    const int32_t rc = grav_check(grav);
    if (rc != ASTROZ_OK) return rc;
    if (s == 0 || s > (uint32_t)az::kTaskMaxSensors) return value_error("s must be in [1, ASTROZ_TASK_MAX_SENSORS]");
    if (t == 0) return value_error("t must be at least 1");
    if (!(gain_min >= 0.0 && gain_min < INFINITY)) return value_error("gain_min must be finite and >= 0");
    a->n = n;
    a->S = s;
    a->T = t;
    a->grav = grav;
    a->g = az::grav_consts(az::gravity(grav));
    a->gainMin = gain_min;
    return ASTROZ_OK;
}

// The sensors, slots and Sun rows of the host call.
static int32_t task_values_check(const uint8_t *kind, const uint32_t *station, const double *sigma,
                                 const double *limits, uint32_t s, uint32_t k, const double *jd, const double *fr,
                                 uint32_t t, const double *sun) {
    bool optical = false;
    for (uint32_t q = 0; q < s; ++q) {
        if (kind[q] != az::kObsRadar && kind[q] != az::kObsOptical)
            return value_error("a sensor kind is not ASTROZ_OBS_RADAR or ASTROZ_OBS_OPTICAL");
        optical = optical || kind[q] == az::kObsOptical;
        if (station[q] >= k) return value_error("a sensor's station index is not below the station count k");
        int used = 0;
        for (int c = 0; c < az::obs_count(kind[q]); ++c) {
            const double sg = sigma[(size_t)q * 4 + c];
            if (!(sg > 0.0)) return value_error("sensor sigma must be > 0 (+inf: component not measured)");
            used += sg < INFINITY;
        }
        if (used == 0) return value_error("a sensor measures no component");
        const double *lim = limits + (size_t)q * 4;
        const double halfPi = 0.5 * az::kPi;
        if (!(std::fabs(lim[az::kTaskElMin]) <= halfPi) || !(std::fabs(lim[az::kTaskSunElMax]) <= halfPi))
            return value_error("an elevation limit is outside [-pi/2, pi/2]");
        if (!(lim[az::kTaskRangeMax] > 0.0)) return value_error("range_max must be > 0 (+inf allowed)");
        if (!(lim[az::kTaskExclusion] >= 0.0 && lim[az::kTaskExclusion] <= az::kPi))
            return value_error("an exclusion angle is outside [0, pi]");
    }
    if (!all_finite(jd, t) || !all_finite(fr, t)) return value_error("slot times must be finite");
    for (uint32_t i = 1; i < t; ++i)
        if ((jd[i] - jd[i - 1]) + (fr[i] - fr[i - 1]) < 0.0) return value_error("slot times must be non-decreasing");
    if (optical && !sun) return value_error("an optical sensor needs the Sun's direction at every slot");
    if (sun)
        for (uint32_t i = 0; i < t; ++i) {
            const double *u = sun + (size_t)i * 3;
            if (!all_finite(u, 3) || (u[0] == 0.0 && u[1] == 0.0 && u[2] == 0.0))
                return value_error("a Sun direction is zero or not finite");
        }
    return ASTROZ_OK;
}

int32_t astroz_cuda_tasking_scratch_bytes(uint32_t n, uint32_t s, uint64_t *bytes) {
    if (!bytes) return ASTROZ_NULL_POINTER;
    if (s == 0 || s > (uint32_t)az::kTaskMaxSensors) return value_error("s must be in [1, ASTROZ_TASK_MAX_SENSORS]");
    *bytes = az::task_scratch_bytes(n, s);
    return ASTROZ_OK;
}

// Both call forms: a holds task_check's scalars, the arrays and the scratch are on the device.
static cudaError_t tasking_run(az::TaskArgs a, const double *elements, const double *covariance, const uint8_t *model,
                               const uint8_t *kind, const uint32_t *station, const double *sigma,
                               const double *limits, const double *stations, const double *jd, const double *fr,
                               const double *sun, void *scratch, uint32_t *task_row, double *task_gain,
                               double *task_value, double *task_spread, uint32_t *n_candidates, double *posterior,
                               uint32_t *n_tasks, uint32_t *n_visible, uint32_t *n_failed, uint8_t *row_status,
                               cudaStream_t st) {
    a.elements = elements;
    a.covariance = covariance;
    a.model = model;
    a.kind = kind;
    a.station = station;
    a.sigma = sigma;
    a.limits = limits;
    a.stations = stations;
    a.jd = jd;
    a.fr = fr;
    a.sun = sun;
    a.scratch = scratch;
    a.taskRow = task_row;
    a.taskGain = task_gain;
    a.taskValue = task_value;
    a.taskSpread = task_spread;
    a.nCandidates = n_candidates;
    a.posterior = posterior;
    a.nTasks = n_tasks;
    a.nVisible = n_visible;
    a.nFailed = n_failed;
    a.rowStatus = row_status;
    return az::launch_tasking(a, st);
}

int32_t astroz_cuda_tasking_device(const double *d_elements, uint32_t n, int32_t grav, const double *d_covariance,
                                   const uint8_t *d_model, const uint8_t *d_kind, const uint32_t *d_station,
                                   const double *d_sigma, const double *d_limits, uint32_t s, const double *d_stations,
                                   const double *d_jd, const double *d_fr, uint32_t t, const double *d_sun,
                                   double gain_min, int32_t device, void *d_scratch, uint32_t *d_task_row,
                                   double *d_task_gain, double *d_task_value, double *d_task_spread,
                                   uint32_t *d_n_candidates, double *d_posterior, uint32_t *d_n_tasks,
                                   uint32_t *d_n_visible, uint32_t *d_n_failed, uint8_t *d_row_status, void *stream) {
    az::TaskArgs a{};
    int32_t rc = task_check(n, grav, s, t, gain_min, device, &a);
    if (rc != ASTROZ_OK) return rc;
    if (!d_kind || !d_station || !d_sigma || !d_limits || !d_stations || !d_jd || !d_fr || !d_scratch ||
        !d_task_row || !d_task_gain || !d_task_value || !d_task_spread || !d_n_candidates)
        return ASTROZ_NULL_POINTER;
    if (n && (!d_elements || !d_posterior || !d_n_tasks || !d_n_visible || !d_n_failed || !d_row_status))
        return ASTROZ_NULL_POINTER;
    if ((rc = check_device_ordinal(device)) != ASTROZ_OK) return rc;
    AZ_CUDA(cudaSetDevice(device));
    AZ_CUDA(tasking_run(a, d_elements, d_covariance, d_model, d_kind, d_station, d_sigma, d_limits, d_stations, d_jd,
                        d_fr, d_sun, d_scratch, d_task_row, d_task_gain, d_task_value, d_task_spread, d_n_candidates,
                        d_posterior, d_n_tasks, d_n_visible, d_n_failed, d_row_status,
                        static_cast<cudaStream_t>(stream)));
    return ASTROZ_OK;
}

int32_t astroz_cuda_tasking(const double *elements, uint32_t n, int32_t grav, const double *covariance,
                            const uint8_t *model, const uint8_t *kind, const uint32_t *station, const double *sigma,
                            const double *limits, uint32_t s, const double *stations, uint32_t k, const double *jd,
                            const double *fr, uint32_t t, const double *sun, double gain_min, int32_t device,
                            uint32_t *task_row, double *task_gain, double *task_value, double *task_spread,
                            uint32_t *n_candidates, double *posterior, uint32_t *n_tasks, uint32_t *n_visible,
                            uint32_t *n_failed, uint8_t *row_status) {
    az::TaskArgs a{};
    int32_t rc = task_check(n, grav, s, t, gain_min, device, &a);
    if (rc != ASTROZ_OK) return rc;
    if (!kind || !station || !sigma || !limits || !stations || !jd || !fr || !task_row || !task_gain ||
        !task_value || !task_spread || !n_candidates)
        return ASTROZ_NULL_POINTER;
    if (n && (!elements || !posterior || !n_tasks || !n_visible || !n_failed || !row_status))
        return ASTROZ_NULL_POINTER;
    if ((rc = obs_values_check(nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 0, stations, k)) != ASTROZ_OK)
        return rc;
    if ((rc = task_values_check(kind, station, sigma, limits, s, k, jd, fr, t, sun)) != ASTROZ_OK) return rc;
    if ((rc = rows_check(elements, covariance, n)) != ASTROZ_OK) return rc;
    if ((rc = model_bytes_check(model, n)) != ASTROZ_OK) return rc;
    return whole_batch(device,
                       {upload(elements, (size_t)64 * n),
                        upload(covariance, covariance ? (size_t)8 * az::kFitN * n : 0),
                        upload(model, model ? (size_t)n : 0), upload(kind, s), upload(station, (size_t)4 * s),
                        upload(sigma, (size_t)32 * s), upload(limits, (size_t)32 * s),
                        upload(stations, (size_t)24 * k), upload(jd, (size_t)8 * t), upload(fr, (size_t)8 * t),
                        upload(sun, sun ? (size_t)24 * t : 0), scratch(az::task_scratch_bytes(n, s)),
                        result(task_row, (size_t)4 * s * t), result(task_gain, (size_t)8 * s * t),
                        result(task_value, (size_t)32 * s * t), result(task_spread, (size_t)32 * s * t),
                        result(n_candidates, (size_t)4 * s * t), result(posterior, (size_t)8 * az::kFitN * n),
                        result(n_tasks, (size_t)4 * n), result(n_visible, (size_t)4 * n),
                        result(n_failed, (size_t)4 * n), result(row_status, n)},
                       [&](const DeviceBlock &d, cudaStream_t st) {
                           return tasking_run(a, d.f64(0), covariance ? d.f64(1) : nullptr,
                                              model ? d.u8(2) : nullptr, d.u8(3), d.u32(4), d.f64(5), d.f64(6),
                                              d.f64(7), d.f64(8), d.f64(9), sun ? d.f64(10) : nullptr, d.piece(11),
                                              d.u32(12), d.f64(13), d.f64(14), d.f64(15), d.u32(16), d.f64(17),
                                              d.u32(18), d.u32(19), d.u32(20), d.u8(21), st);
                       });
}

// ---- initial orbits (K13, az_iod.cu, az_iod.cuh) ----------------------------------------------------------------------
static_assert(ASTROZ_IOD_OK == az::kIodOk && ASTROZ_IOD_TOO_FEW == az::kIodTooFew &&
                  ASTROZ_IOD_NO_CANDIDATE == az::kIodNoCandidate &&
                  ASTROZ_IOD_CONVERSION_FAILED == az::kIodConversionFailed &&
                  ASTROZ_IOD_BAD_TRACK == az::kIodBadTrack && ASTROZ_IOD_MAX_TRACK == az::kIodMaxTrack &&
                  ASTROZ_IOD_METHOD_STATE == az::kIodState && ASTROZ_IOD_METHOD_GIBBS == az::kIodGibbs &&
                  ASTROZ_IOD_METHOD_HERRICK_GIBBS == az::kIodHerrickGibbs &&
                  ASTROZ_IOD_METHOD_LAMBERT == az::kIodLambert && ASTROZ_IOD_METHOD_GAUSS == az::kIodGauss &&
                  ASTROZ_IOD_METHOD_NONE == az::kIodNone,
              "initial-orbit status and method bytes");

// Scalar checks of the initial-orbit calls, before anything is read, written or allocated; a receives the scalars.
static int32_t iod_check(uint32_t t, int32_t grav, int32_t device, az::IodArgs *a) {
    if (device < 0) return value_error("initial orbit determination runs on one device: pass its ordinal");
    const int32_t rc = grav_check(grav);
    if (rc != ASTROZ_OK) return rc;
    a->t = t;
    a->grav = grav;
    a->g = az::grav_consts(az::gravity(grav));
    return ASTROZ_OK;
}

int32_t astroz_cuda_initial_orbits_scratch_bytes(uint32_t t, uint64_t *bytes) {
    if (!bytes) return ASTROZ_NULL_POINTER;
    *bytes = az::iod_scratch_bytes(t);
    return ASTROZ_OK;
}

// Both call forms: a holds iod_check's scalars, the arrays and the scratch are on the device.
static cudaError_t iod_run(az::IodArgs a, const uint32_t *offsets, const double *jd, const double *fr,
                           const uint8_t *kind, const double *value, const double *sigma, const uint32_t *station,
                           const double *stations, const double *bstar, void *scratch, double *elements,
                           double *state, double *wrms, uint8_t *method, uint32_t *candidates, double *conv,
                           uint8_t *deep_space, uint8_t *status, cudaStream_t st) {
    a.offsets = offsets;
    a.jd = jd;
    a.fr = fr;
    a.kind = kind;
    a.value = value;
    a.sigma = sigma;
    a.station = station;
    a.stations = stations;
    a.bstar = bstar;
    a.scratch = scratch;
    a.elements = elements;
    a.state = state;
    a.wrms = wrms;
    a.method = method;
    a.candidates = candidates;
    a.conv = conv;
    a.deepSpace = deep_space;
    a.status = status;
    return az::launch_iod(a, st);
}

int32_t astroz_cuda_initial_orbits_device(const uint32_t *d_offsets, uint32_t t, const double *d_jd,
                                          const double *d_fr, const uint8_t *d_kind, const double *d_value,
                                          const double *d_sigma, const uint32_t *d_station, const double *d_stations,
                                          const double *d_bstar, int32_t grav, int32_t device, void *d_scratch,
                                          double *d_elements, double *d_state, double *d_wrms, uint8_t *d_method,
                                          uint32_t *d_candidates, double *d_conv, uint8_t *d_deep_space,
                                          uint8_t *d_status, void *stream) {
    az::IodArgs a{};
    int32_t rc = iod_check(t, grav, device, &a);
    if (rc != ASTROZ_OK) return rc;
    if (t == 0) return ASTROZ_OK;
    if (!d_offsets || !d_jd || !d_fr || !d_kind || !d_value || !d_sigma || !d_scratch || !d_elements || !d_state ||
        !d_wrms || !d_method || !d_candidates || !d_conv || !d_deep_space || !d_status)
        return ASTROZ_NULL_POINTER;
    if ((rc = check_device_ordinal(device)) != ASTROZ_OK) return rc;
    AZ_CUDA(cudaSetDevice(device));
    AZ_CUDA(iod_run(a, d_offsets, d_jd, d_fr, d_kind, d_value, d_sigma, d_station, d_stations, d_bstar, d_scratch,
                    d_elements, d_state, d_wrms, d_method, d_candidates, d_conv, d_deep_space, d_status,
                    static_cast<cudaStream_t>(stream)));
    return ASTROZ_OK;
}

// The observations of each track sorted stably by jd + fr, into host staging: what the track calls upload.
struct SortedTracks {
    std::vector<double> jd, fr, value, sigma;
    std::vector<uint8_t> kind;
    std::vector<uint32_t> station;
};

static SortedTracks sorted_tracks(const uint32_t *offsets, uint32_t t, const double *jd, const double *fr,
                                  const uint8_t *kind, const double *value, const double *sigma,
                                  const uint32_t *station, uint32_t m) {
    std::vector<uint32_t> order(m);
    for (uint32_t i = 0; i < m; ++i) order[i] = i;
    for (uint32_t j = 0; j < t; ++j)
        std::stable_sort(order.begin() + offsets[j], order.begin() + offsets[j + 1], [&](uint32_t p, uint32_t q) {
            return az::add_rn(jd[p], fr[p]) < az::add_rn(jd[q], fr[q]);
        });
    SortedTracks s;
    s.jd.resize(m);
    s.fr.resize(m);
    s.value.resize((size_t)6 * m);
    s.sigma.resize((size_t)6 * m);
    s.kind.resize(m);
    s.station.resize(station ? m : 0);
    for (uint32_t i = 0; i < m; ++i) {
        const uint32_t p = order[i];
        s.jd[i] = jd[p];
        s.fr[i] = fr[p];
        s.kind[i] = kind[p];
        std::memcpy(&s.value[(size_t)6 * i], value + (size_t)6 * p, 48);
        std::memcpy(&s.sigma[(size_t)6 * i], sigma + (size_t)6 * p, 48);
        if (station) s.station[i] = station[p];
    }
    return s;
}

// Every check, then each track's observations sorted stably by jd + fr into host staging, which is what goes up (the
// caller's pinned arrays are not read by DMA: the staging copy is pageable).
int32_t astroz_cuda_initial_orbits(const uint32_t *offsets, uint32_t t, const double *jd, const double *fr,
                                   const uint8_t *kind, const double *value, const double *sigma,
                                   const uint32_t *station, uint32_t m, const double *stations, uint32_t k,
                                   const double *bstar, int32_t grav, int32_t device, double *elements, double *state,
                                   double *wrms, uint8_t *method, uint32_t *candidates, double *conv,
                                   uint8_t *deep_space, uint8_t *status) {
    az::IodArgs a{};
    int32_t rc = iod_check(t, grav, device, &a);
    if (rc != ASTROZ_OK) return rc;
    if (!offsets) return ASTROZ_NULL_POINTER;
    if (t && (!elements || !state || !wrms || !method || !candidates || !conv || !deep_space || !status))
        return ASTROZ_NULL_POINTER;
    if (m && (!jd || !fr || !kind || !value || !sigma)) return ASTROZ_NULL_POINTER;
    if ((rc = offsets_check(offsets, t, m, "offsets[t] must equal the observation count m", true, az::kIodMaxTrack,
                            "a track is longer than ASTROZ_IOD_MAX_TRACK observations")) != ASTROZ_OK)
        return rc;
    if ((rc = obs_values_check(jd, fr, value, sigma, station, kind, m, stations, k)) != ASTROZ_OK) return rc;
    if ((rc = used_residuals_check({jd, fr, kind, value, sigma, station, stations}, offsets, t)) != ASTROZ_OK)
        return rc;
    if (bstar && !all_finite(bstar, t)) return value_error("bstar must be finite");
    if (t == 0) return ASTROZ_OK;
    const SortedTracks so = sorted_tracks(offsets, t, jd, fr, kind, value, sigma, station, m);
    return whole_batch(device,
                       {upload(offsets, (size_t)4 * (t + 1)), upload(so.jd.data(), (size_t)8 * m),
                        upload(so.fr.data(), (size_t)8 * m), upload(so.kind.data(), m),
                        upload(so.value.data(), (size_t)48 * m), upload(so.sigma.data(), (size_t)48 * m),
                        upload(so.station.data(), station ? (size_t)4 * m : 0), upload(stations, (size_t)24 * k),
                        upload(bstar, bstar ? (size_t)8 * t : 0), scratch(az::iod_scratch_bytes(t)),
                        result(elements, (size_t)64 * t), result(state, (size_t)48 * t), result(wrms, (size_t)8 * t),
                        result(method, t), result(candidates, (size_t)4 * t), result(conv, (size_t)16 * t),
                        result(deep_space, t), result(status, t)},
                       [&](const DeviceBlock &d, cudaStream_t st) {
                           return iod_run(a, d.u32(0), d.f64(1), d.f64(2), d.u8(3), d.f64(4), d.f64(5),
                                          station ? d.u32(6) : nullptr, k ? d.f64(7) : nullptr,
                                          bstar ? d.f64(8) : nullptr, d.piece(9), d.f64(10), d.f64(11), d.f64(12),
                                          d.u8(13), d.u32(14), d.f64(15), d.u8(16), d.u8(17), st);
                       });
}

// ---- track linking (K17, az_link.cu, az_link.cuh) ----------------------------------------------------------------------
static_assert(ASTROZ_LINK_OK == az::kLinkOk && ASTROZ_LINK_TOO_FEW == az::kLinkTooFew &&
                  ASTROZ_LINK_NO_CANDIDATE == az::kLinkNoCandidate &&
                  ASTROZ_LINK_CONVERSION_FAILED == az::kLinkConversionFailed &&
                  ASTROZ_LINK_BAD_TRACK == az::kLinkBadTrack && ASTROZ_LINK_BAD_PAIR == az::kLinkBadPair &&
                  ASTROZ_LINK_RETROGRADE == az::kLinkRetrograde && ASTROZ_LINK_RIGHT_BRANCH == az::kLinkRightBranch &&
                  ASTROZ_LINK_RANGES == az::kLinkRanges && ASTROZ_LINK_SEEDS == az::kLinkSeeds,
              "track-link status, flag and size constants");

// Scalar checks of the link calls, before anything is read, written or allocated; a receives the scalars.
static int32_t link_check(uint32_t t, uint32_t p, double r_min, double r_max, uint32_t max_revs, int32_t grav,
                          int32_t device, az::LinkArgs *a) {
    if (device < 0) return value_error("track linking runs on one device: pass its ordinal");
    const int32_t rc = grav_check(grav);
    if (rc != ASTROZ_OK) return rc;
    if (max_revs > az::kLamMaxRevs) return value_error("max_revs must be at most ASTROZ_LAMBERT_MAX_REVS");
    if (!(r_min > 0.0) || !std::isfinite(r_min)) return value_error("r_min must be finite and positive");
    if (!(r_max > r_min) || !std::isfinite(r_max)) return value_error("r_max must be finite and above r_min");
    a->t = t;
    a->p = p;
    a->rMin = r_min;
    a->rMax = r_max;
    a->maxRevs = max_revs;
    a->grav = grav;
    a->g = az::grav_consts(az::gravity(grav));
    return ASTROZ_OK;
}

int32_t astroz_cuda_link_tracks_scratch_bytes(uint32_t p, uint64_t *bytes) {
    if (!bytes) return ASTROZ_NULL_POINTER;
    *bytes = az::iod_scratch_bytes(p);
    return ASTROZ_OK;
}

// Both call forms: a holds link_check's scalars, the arrays and the scratch are on the device.
static cudaError_t link_run(az::LinkArgs a, const uint32_t *offsets, const double *jd, const double *fr,
                            const uint8_t *kind, const double *value, const double *sigma, const uint32_t *station,
                            const double *stations, const uint32_t *pairs, const double *bstar, void *scratch,
                            double *elements, double *state, double *rho, uint8_t *revs, uint8_t *flags, double *wrms,
                            uint32_t *used, uint32_t *hypotheses, double *conv, uint8_t *deep_space, uint8_t *status,
                            cudaStream_t st) {
    a.offsets = offsets;
    a.jd = jd;
    a.fr = fr;
    a.kind = kind;
    a.value = value;
    a.sigma = sigma;
    a.station = station;
    a.stations = stations;
    a.pairs = pairs;
    a.bstar = bstar;
    a.scratch = scratch;
    a.elements = elements;
    a.state = state;
    a.rho = rho;
    a.revs = revs;
    a.flags = flags;
    a.wrms = wrms;
    a.used = used;
    a.hypotheses = hypotheses;
    a.conv = conv;
    a.deepSpace = deep_space;
    a.status = status;
    return az::launch_link(a, st);
}

int32_t astroz_cuda_link_tracks_device(const uint32_t *d_offsets, uint32_t t, const double *d_jd, const double *d_fr,
                                       const uint8_t *d_kind, const double *d_value, const double *d_sigma,
                                       const uint32_t *d_station, const double *d_stations, const uint32_t *d_pairs,
                                       uint32_t p, const double *d_bstar, double r_min, double r_max,
                                       uint32_t max_revs, int32_t grav, int32_t device, void *d_scratch,
                                       double *d_elements, double *d_state, double *d_rho, uint8_t *d_revs,
                                       uint8_t *d_flags, double *d_wrms, uint32_t *d_used, uint32_t *d_hypotheses,
                                       double *d_conv, uint8_t *d_deep_space, uint8_t *d_status, void *stream) {
    az::LinkArgs a{};
    int32_t rc = link_check(t, p, r_min, r_max, max_revs, grav, device, &a);
    if (rc != ASTROZ_OK) return rc;
    if (p == 0) return ASTROZ_OK;
    if (!d_offsets || !d_jd || !d_fr || !d_kind || !d_value || !d_sigma || !d_pairs || !d_scratch || !d_elements ||
        !d_state || !d_rho || !d_revs || !d_flags || !d_wrms || !d_used || !d_hypotheses || !d_conv ||
        !d_deep_space || !d_status)
        return ASTROZ_NULL_POINTER;
    if ((rc = check_device_ordinal(device)) != ASTROZ_OK) return rc;
    AZ_CUDA(cudaSetDevice(device));
    AZ_CUDA(link_run(a, d_offsets, d_jd, d_fr, d_kind, d_value, d_sigma, d_station, d_stations, d_pairs, d_bstar,
                     d_scratch, d_elements, d_state, d_rho, d_revs, d_flags, d_wrms, d_used, d_hypotheses, d_conv,
                     d_deep_space, d_status, static_cast<cudaStream_t>(stream)));
    return ASTROZ_OK;
}

// Every check of astroz_cuda_initial_orbits, then the pairs' and the range bounds'; the tracks go up sorted, as there.
int32_t astroz_cuda_link_tracks(const uint32_t *offsets, uint32_t t, const double *jd, const double *fr,
                                const uint8_t *kind, const double *value, const double *sigma, const uint32_t *station,
                                uint32_t m, const double *stations, uint32_t k, const uint32_t *pairs, uint32_t p,
                                const double *bstar, double r_min, double r_max, uint32_t max_revs, int32_t grav,
                                int32_t device, double *elements, double *state, double *rho, uint8_t *revs,
                                uint8_t *flags, double *wrms, uint32_t *used, uint32_t *hypotheses, double *conv,
                                uint8_t *deep_space, uint8_t *status) {
    az::LinkArgs a{};
    int32_t rc = link_check(t, p, r_min, r_max, max_revs, grav, device, &a);
    if (rc != ASTROZ_OK) return rc;
    if (!offsets) return ASTROZ_NULL_POINTER;
    if (p && (!pairs || !elements || !state || !rho || !revs || !flags || !wrms || !used || !hypotheses || !conv ||
              !deep_space || !status))
        return ASTROZ_NULL_POINTER;
    if (m && (!jd || !fr || !kind || !value || !sigma)) return ASTROZ_NULL_POINTER;
    if ((rc = offsets_check(offsets, t, m, "offsets[t] must equal the observation count m", true, az::kIodMaxTrack,
                            "a track is longer than ASTROZ_IOD_MAX_TRACK observations")) != ASTROZ_OK)
        return rc;
    if ((rc = obs_values_check(jd, fr, value, sigma, station, kind, m, stations, k)) != ASTROZ_OK) return rc;
    if ((rc = used_residuals_check({jd, fr, kind, value, sigma, station, stations}, offsets, t)) != ASTROZ_OK)
        return rc;
    if (bstar && !all_finite(bstar, p)) return value_error("bstar must be finite");
    for (uint32_t q = 0; q < k; ++q) {
        az::ObsStation st;
        az::obs_station(stations + (size_t)3 * q, st);
        if (!(r_min > std::sqrt(st.r[0] * st.r[0] + st.r[1] * st.r[1] + st.r[2] * st.r[2])))
            return value_error("r_min must exceed every station's radius");
    }
    for (uint64_t q = 0; q < 2 * (uint64_t)p; ++q)
        if (pairs[q] >= t) return value_error("a pair names a track index >= t");
    if (p == 0) return ASTROZ_OK;
    const SortedTracks so = sorted_tracks(offsets, t, jd, fr, kind, value, sigma, station, m);
    const az::CorrObsArrays in{so.jd.data(), so.fr.data(), so.kind.data(), so.value.data(), so.sigma.data(),
                               station ? so.station.data() : nullptr, stations};
    std::vector<double> anchorT(t, NAN);
    for (uint32_t j = 0; j < t; ++j) {
        const uint32_t i = az::link_anchor_index(in, offsets[j], offsets[j + 1]);
        if (i != offsets[j + 1]) anchorT[j] = az::add_rn(so.jd[i], so.fr[i]);
    }
    for (uint32_t q = 0; q < p; ++q) {
        if (pairs[2 * q] == pairs[2 * q + 1]) return value_error("a pair names one track twice");
        if (anchorT[pairs[2 * q]] == anchorT[pairs[2 * q + 1]])
            return value_error("the two tracks of a pair have their anchors at the same time");
    }
    return whole_batch(device,
                       {upload(offsets, (size_t)4 * (t + 1)), upload(so.jd.data(), (size_t)8 * m),
                        upload(so.fr.data(), (size_t)8 * m), upload(so.kind.data(), m),
                        upload(so.value.data(), (size_t)48 * m), upload(so.sigma.data(), (size_t)48 * m),
                        upload(so.station.data(), station ? (size_t)4 * m : 0), upload(stations, (size_t)24 * k),
                        upload(pairs, (size_t)8 * p), upload(bstar, bstar ? (size_t)8 * p : 0),
                        scratch(az::iod_scratch_bytes(p)), result(elements, (size_t)64 * p),
                        result(state, (size_t)48 * p), result(rho, (size_t)16 * p), result(revs, p), result(flags, p),
                        result(wrms, (size_t)8 * p), result(used, (size_t)4 * p), result(hypotheses, (size_t)4 * p),
                        result(conv, (size_t)16 * p), result(deep_space, p), result(status, p)},
                       [&](const DeviceBlock &d, cudaStream_t st) {
                           return link_run(a, d.u32(0), d.f64(1), d.f64(2), d.u8(3), d.f64(4), d.f64(5),
                                           station ? d.u32(6) : nullptr, k ? d.f64(7) : nullptr, d.u32(8),
                                           bstar ? d.f64(9) : nullptr, d.piece(10), d.f64(11), d.f64(12), d.f64(13),
                                           d.u8(14), d.u8(15), d.f64(16), d.u32(17), d.u32(18), d.f64(19), d.u8(20),
                                           d.u8(21), st);
                       });
}

int32_t astroz_cuda_parse_tle(const char *line1, const char *line2, double *elements) {
    if (!line1 || !line2 || !elements) return ASTROZ_NULL_POINTER;
    az::TleRecord t;
    if (az::parse_tle(line1, line2, t) != az::kOk) return ASTROZ_BAD_TLE_LENGTH;
    const double cols[8] = {t.epochJd, t.revPerDay, t.ecc, t.inclDeg, t.raanDeg, t.argpDeg, t.maDeg, t.bstar};
    std::memcpy(elements, cols, sizeof cols);
    return ASTROZ_OK;
}

// ---- Lambert transfers (K9, az_lambert.cu) ---------------------------------------------------------------------------
static_assert(ASTROZ_LAMBERT_OK == az::kLamOk && ASTROZ_LAMBERT_NO_SOLUTION == az::kLamNoSolution &&
                  ASTROZ_LAMBERT_DEGENERATE == az::kLamDegenerate &&
                  ASTROZ_LAMBERT_NOT_CONVERGED == az::kLamNotConverged &&
                  ASTROZ_LAMBERT_STATE_FAILED == az::kLamStateFailed && ASTROZ_LAMBERT_MAX_REVS == az::kLamMaxRevs,
              "lambert status bytes");

// Scalar checks of every Lambert call, before anything is read, written or allocated.
static int32_t lambert_check(double mu, uint32_t max_revs, int32_t device) {
    if (device < 0) return value_error("a Lambert call runs on one device: pass its ordinal");
    if (!std::isfinite(mu) || !(mu > 0.0)) return value_error("mu must be finite and > 0");
    if (max_revs > az::kLamMaxRevs) return value_error("max_revs must be at most 127");
    return ASTROZ_OK;
}

// lambert_check, and the grid's size: its byte count and its CTA count (one cell per thread) must be representable.
static int32_t porkchop_check(uint32_t n_pairs, uint32_t n_dep, uint32_t n_arr, double mu, uint32_t max_revs,
                              int32_t device) {
    const int32_t rc = lambert_check(mu, max_revs, device);
    if (rc != ASTROZ_OK) return rc;
    const uint64_t perPair = (uint64_t)n_dep * n_arr;
    if (n_pairs && perPair > (uint64_t)0x7fffffff * 128 / n_pairs) return value_error("the porkchop grid is too large");
    return ASTROZ_OK;
}

// Both call forms, on device arrays.
static cudaError_t lambert_run(const double *r1, const double *r2, const double *tof, const double *normal,
                               uint32_t n, double mu, uint32_t max_revs, double *v1, double *v2, uint8_t *status,
                               uint8_t *iterations, cudaStream_t st) {
    return az::launch_lambert(az::LambertArgs{r1, r2, tof, normal, n, max_revs, mu, v1, v2, status, iterations}, st);
}

int32_t astroz_cuda_lambert_device(const double *d_r1, const double *d_r2, const double *d_tof, const double *d_normal,
                                   uint32_t n, double mu, uint32_t max_revs, int32_t device, double *d_v1,
                                   double *d_v2, uint8_t *d_status, uint8_t *d_iterations, void *stream) {
    int32_t rc = lambert_check(mu, max_revs, device);
    if (rc != ASTROZ_OK) return rc;
    if (n == 0) return ASTROZ_OK;
    if (!d_r1 || !d_r2 || !d_tof || !d_v1 || !d_v2 || !d_status) return ASTROZ_NULL_POINTER;
    if ((rc = check_device_ordinal(device)) != ASTROZ_OK) return rc;
    AZ_CUDA(cudaSetDevice(device));
    AZ_CUDA(lambert_run(d_r1, d_r2, d_tof, d_normal, n, mu, max_revs, d_v1, d_v2, d_status, d_iterations,
                        static_cast<cudaStream_t>(stream)));
    return ASTROZ_OK;
}

int32_t astroz_cuda_lambert(const double *r1, const double *r2, const double *tof, const double *normal, uint32_t n,
                            double mu, uint32_t max_revs, int32_t device, double *v1, double *v2, uint8_t *status,
                            uint8_t *iterations) {
    const int32_t rc = lambert_check(mu, max_revs, device);
    if (rc != ASTROZ_OK) return rc;
    if (n == 0) return ASTROZ_OK;
    if (!r1 || !r2 || !tof || !v1 || !v2 || !status) return ASTROZ_NULL_POINTER;
    if (!all_finite(r1, (size_t)3 * n) || !all_finite(r2, (size_t)3 * n) || !all_finite(tof, n) ||
        (normal && !all_finite(normal, (size_t)3 * n)))
        return value_error("r1, r2, tof and normal must be finite");
    const size_t slots = (size_t)n * (2 * (size_t)max_revs + 1);
    return whole_batch(device,
                       {upload(r1, (size_t)24 * n), upload(r2, (size_t)24 * n),
                        upload(normal, normal ? (size_t)24 * n : 0), upload(tof, (size_t)8 * n),
                        result(v1, 24 * slots), result(v2, 24 * slots), result(status, slots),
                        result(iterations, iterations ? slots : 0)},
                       [&](const DeviceBlock &d, cudaStream_t st) {
                           return lambert_run(d.f64(0), d.f64(1), d.f64(3), normal ? d.f64(2) : nullptr, n, mu,
                                              max_revs, d.f64(4), d.f64(5), d.u8(6), iterations ? d.u8(7) : nullptr,
                                              st);
                       });
}

int32_t astroz_cuda_lambert_porkchop_device(const double *d_dep, const uint8_t *d_dep_status, const double *d_arr,
                                            const uint8_t *d_arr_status, uint32_t n_pairs, const double *d_dep_jd,
                                            const double *d_dep_fr, uint32_t n_dep, const double *d_arr_jd,
                                            const double *d_arr_fr, uint32_t n_arr, double mu, uint32_t max_revs,
                                            int32_t device, double *d_dv, uint8_t *d_slot, uint8_t *d_status,
                                            void *stream) {
    int32_t rc = porkchop_check(n_pairs, n_dep, n_arr, mu, max_revs, device);
    if (rc != ASTROZ_OK) return rc;
    if (!n_pairs || !n_dep || !n_arr) return ASTROZ_OK;
    if (!d_dep || !d_arr || !d_dep_jd || !d_dep_fr || !d_arr_jd || !d_arr_fr || !d_dv || !d_slot || !d_status)
        return ASTROZ_NULL_POINTER;
    if ((rc = check_device_ordinal(device)) != ASTROZ_OK) return rc;
    AZ_CUDA(cudaSetDevice(device));
    const az::PorkchopArgs a{d_dep,    d_dep + 3, d_arr,    d_arr + 3, 6,     d_dep_status, d_arr_status,
                             d_dep_jd, d_dep_fr,  d_arr_jd, d_arr_fr,  n_pairs, n_dep,      n_arr,
                             max_revs, mu,        d_dv,     d_slot,    d_status};
    AZ_CUDA(az::launch_porkchop(a, static_cast<cudaStream_t>(stream)));
    return ASTROZ_OK;
}

// Host buffers: chunks of pairs through the handle's two-slot pipeline (az::ChunkPipeline), each chunk's grid block at
// most kPorkchopChunkBytes with its endpoint states.  A chunk's queries are its pairs' catalog rows (the pipeline's input
// columns, one row per departure or arrival) against the time axes tiled over the chunk's pairs (uploaded once); the
// handle's pairs path fills the endpoint states, then the porkchop kernel runs on them, all on the handle's stream.
static constexpr size_t kPorkchopChunkBytes = 32u << 20;
int32_t astroz_cuda_constellation_porkchop(astroz_constellation_t h, const uint32_t *chaser, const uint32_t *target,
                                           uint32_t n_pairs, const double *dep_jd, const double *dep_fr, uint32_t n_dep,
                                           const double *arr_jd, const double *arr_fr, uint32_t n_arr, double mu,
                                           uint32_t max_revs, double *dv, uint8_t *slot, uint8_t *status) {
    Constellation *c = static_cast<Constellation *>(h);
    if (!c) return ASTROZ_NULL_POINTER;
    int32_t rc = refuse_multi(c);
    if (rc == ASTROZ_OK) rc = porkchop_check(n_pairs, n_dep, n_arr, mu, max_revs, c->device);
    if (rc != ASTROZ_OK) return rc;
    if (!n_pairs || !n_dep || !n_arr) return ASTROZ_OK;
    if (!chaser || !target || !dep_jd || !dep_fr || !arr_jd || !arr_fr || !dv || !slot || !status)
        return ASTROZ_NULL_POINTER;
    const az::CatalogTables &t = c->cat;
    for (uint32_t p = 0; p < n_pairs; ++p)
        if (chaser[p] >= t.n || target[p] >= t.n) {
            g_lastError = "pair " + std::to_string(p) + ": a catalog row is not in the " + std::to_string(t.n) +
                          "-row catalog";
            return ASTROZ_VALUE_ERROR;
        }
    if (!all_finite(dep_jd, n_dep) || !all_finite(dep_fr, n_dep) || !all_finite(arr_jd, n_arr) ||
        !all_finite(arr_fr, n_arr))
        return value_error("the departure and arrival epochs must be finite");
    const size_t D = n_dep, A = n_arr;
    AZ_CUDA(cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    if (t.nSdp4) {
        double lo = INFINITY, hi = -INFINITY;
        for (size_t i = 0; i < D; ++i) lo = std::min(lo, dep_jd[i] + dep_fr[i]), hi = std::max(hi, dep_jd[i] + dep_fr[i]);
        for (size_t i = 0; i < A; ++i) lo = std::min(lo, arr_jd[i] + arr_fr[i]), hi = std::max(hi, arr_jd[i] + arr_fr[i]);
        if ((rc = prepare_deep_space(c, lo, hi, st)) != ASTROZ_OK) return rc;
    }
    const size_t pairBytes = D * A * 18 + (D + A) * 49;   // grid block, and endpoint states and status bytes
    const uint32_t chunk = (uint32_t)std::max<size_t>(1, std::min<size_t>(n_pairs, kPorkchopChunkBytes / pairBytes));
    std::vector<uint32_t> satC((size_t)n_pairs * D), satT((size_t)n_pairs * A);
    for (size_t p = 0; p < n_pairs; ++p) {
        std::fill_n(satC.begin() + p * D, D, chaser[p]);
        std::fill_n(satT.begin() + p * A, A, target[p]);
    }
    // device scratch: tiled dep jd | dep fr | arr jd | arr fr, then dep pos | dep vel | arr pos | arr vel, status bytes
    const size_t qd = (size_t)chunk * D, qa = (size_t)chunk * A;
    std::vector<double> tiles(2 * qd + 2 * qa);
    for (size_t q = 0; q < qd; ++q) tiles[q] = dep_jd[q % D], tiles[qd + q] = dep_fr[q % D];
    for (size_t q = 0; q < qa; ++q) tiles[2 * qd + q] = arr_jd[q % A], tiles[2 * qd + qa + q] = arr_fr[q % A];
    StreamBuf dScratch(st), dIn(st), dOut(st);
    AZ_CUDA(dScratch.alloc((tiles.size() + 6 * qd + 6 * qa) * 8 + qd + qa));
    double *dTiles = static_cast<double *>(dScratch.p);
    AZ_CUDA(cudaMemcpyAsync(dTiles, tiles.data(), tiles.size() * 8, cudaMemcpyHostToDevice, st));
    const double *depJd = dTiles, *depFr = dTiles + qd, *arrJd = dTiles + 2 * qd, *arrFr = dTiles + 2 * qd + qa;
    double *depPos = dTiles + tiles.size(), *depVel = depPos + 3 * qd, *arrPos = depVel + 3 * qd,
           *arrVel = arrPos + 3 * qa;
    uint8_t *depSt = reinterpret_cast<uint8_t *>(arrVel + 3 * qa), *arrSt = depSt + qd;
    const az::HostIn in[2] = {{satC.data(), 4 * D}, {satT.data(), 4 * A}};
    const az::HostOut out[3] = {{dv, 16 * D * A}, {slot, D * A}, {status, D * A}};
    AZ_CUDA(dIn.alloc(az::chunk_slots_bytes(in, 2, n_pairs, chunk)));
    AZ_CUDA(dOut.alloc(az::chunk_slots_bytes(out, 3, n_pairs, chunk)));
    int32_t queued = ASTROZ_OK;  // pairs_queue's own code; its message is the last error
    const cudaError_t e = c->pipe.run(
        st, c->copyStream, n_pairs, chunk, 2, in, 3, out, dIn.p, dOut.p,
        [&](uint32_t, uint32_t, uint32_t m, void *const *dI, void *const *dO, cudaStream_t s) {
            queued = pairs_queue(c, static_cast<const uint32_t *>(dI[0]), depJd, depFr, (uint32_t)(m * D),
                                 ASTROZ_MODE_TEME, depPos, depVel, depSt, s);
            if (queued == ASTROZ_OK)
                queued = pairs_queue(c, static_cast<const uint32_t *>(dI[1]), arrJd, arrFr, (uint32_t)(m * A),
                                     ASTROZ_MODE_TEME, arrPos, arrVel, arrSt, s);
            if (queued != ASTROZ_OK) return cudaErrorUnknown;  // stops the run; `queued` is returned
            const az::PorkchopArgs a{depPos, depVel, arrPos, arrVel, 3, depSt, arrSt, depJd, depFr, arrJd, arrFr,
                                     m, n_dep, n_arr, max_revs, mu, static_cast<double *>(dO[0]),
                                     static_cast<uint8_t *>(dO[1]), static_cast<uint8_t *>(dO[2])};
            return az::launch_porkchop(a, s);
        });
    if (queued != ASTROZ_OK) return queued;
    AZ_CUDA(e);
    AZ_CUDA(dIn.release());
    AZ_CUDA(dOut.release());
    AZ_CUDA(dScratch.release());
    AZ_CUDA(cudaStreamSynchronize(st));
    return ASTROZ_OK;
}

int32_t astroz_cuda_fp64_peak(int32_t device, double *tflops) {
    if (!tflops) return ASTROZ_NULL_POINTER;
    int n = 0;
    const int32_t rc = check_device_present(&n, "no CUDA device available");
    if (rc != ASTROZ_OK) return rc;
    AZ_CUDA(cudaSetDevice(device));
    double flops = 0;
    AZ_CUDA(az::measure_fp64_peak(&flops));
    *tflops = flops * 1e-12;
    return ASTROZ_OK;
}

int32_t astroz_cuda_fp64_pipe_peak(int32_t device, double *tflops) {
    if (!tflops) return ASTROZ_NULL_POINTER;
    int n = 0;
    const int32_t rc = check_device_present(&n, "no CUDA device available");
    if (rc != ASTROZ_OK) return rc;
    AZ_CUDA(cudaSetDevice(device));
    double flops = 0;
    AZ_CUDA(az::fp64_pipe_peak(&flops));
    *tflops = flops * 1e-12;
    return ASTROZ_OK;
}

#pragma GCC visibility pop
}  // extern "C"
