// az_hostcopy.cu -- the pinned ring, the host copy pool and the two-slot chunk pipeline behind az_hostcopy.cuh.
#include "az_hostcopy.cuh"

#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <functional>
#include <initializer_list>
#include <mutex>
#include <thread>

namespace az {
namespace {

// Piece size: large enough that (a) the wake-up of the copy threads is amortised and (b) each thread's share (a few MB)
// is above libc's non-temporal threshold, so the destination lines are streamed instead of read for ownership first.
constexpr size_t kPieceBytes = 32u << 20;

// Streaming copy for the landed pieces: the destination is written once and not read again by this library, so the
// stores bypass the cache (no read-for-ownership of the destination lines, no eviction of the caller's working set):
// a third less memory traffic per byte than a cached copy.  AVX2 hosts; anything else uses memcpy.
#if defined(__x86_64__) && defined(__GNUC__)
#include <immintrin.h>
__attribute__((target("avx2"))) void stream_copy_avx2(char *dst, const char *src, size_t n) {
    const size_t head = (32 - (reinterpret_cast<uintptr_t>(dst) & 31)) & 31;
    if (head) {
        const size_t h = std::min(head, n);
        std::memcpy(dst, src, h);
        dst += h; src += h; n -= h;
    }
    size_t i = 0;
    for (; i + 128 <= n; i += 128) {
        const __m256i a = _mm256_loadu_si256(reinterpret_cast<const __m256i *>(src + i));
        const __m256i b = _mm256_loadu_si256(reinterpret_cast<const __m256i *>(src + i + 32));
        const __m256i c = _mm256_loadu_si256(reinterpret_cast<const __m256i *>(src + i + 64));
        const __m256i d = _mm256_loadu_si256(reinterpret_cast<const __m256i *>(src + i + 96));
        _mm256_stream_si256(reinterpret_cast<__m256i *>(dst + i), a);
        _mm256_stream_si256(reinterpret_cast<__m256i *>(dst + i + 32), b);
        _mm256_stream_si256(reinterpret_cast<__m256i *>(dst + i + 64), c);
        _mm256_stream_si256(reinterpret_cast<__m256i *>(dst + i + 96), d);
    }
    _mm_sfence();
    if (i < n) std::memcpy(dst + i, src + i, n - i);
}
void stream_copy(char *dst, const char *src, size_t n) {
    static const bool avx2 = __builtin_cpu_supports("avx2");
    if (avx2 && n >= (64u << 10)) stream_copy_avx2(dst, src, n);
    else std::memcpy(dst, src, n);
}
#else
void stream_copy(char *dst, const char *src, size_t n) { std::memcpy(dst, src, n); }
#endif

class CopyPool {  // process-wide, created on first use, never destroyed (workers sleep on the condition variable)
public:
    static CopyPool &get() {
        static CopyPool *p = new CopyPool();
        return *p;
    }
    // copy `rows` rows of rowBytes from a contiguous source to a destination with pitch hpitch, split over the pool
    void copy(char *dst, const char *src, size_t rows, size_t rowBytes, size_t hpitch) {
        const size_t total = rows * rowBytes;
        const int parts = (int)std::max<size_t>(1, std::min<size_t>(workers_.size(), total / (1u << 20)));
        if (parts <= 1 || workers_.empty()) {
            run(dst, src, rowBytes, hpitch, 0, total);
            return;
        }
        std::atomic<int> left(parts);
        std::mutex dm;
        std::condition_variable dcv;
        for (int k = 0; k < parts; ++k) {
            const size_t b0 = total * k / parts, b1 = total * (k + 1) / parts;
            push([=, &left, &dm, &dcv] {
                run(dst, src, rowBytes, hpitch, b0, b1);
                if (left.fetch_sub(1) == 1) {
                    std::lock_guard<std::mutex> g(dm);
                    dcv.notify_one();
                }
            });
        }
        std::unique_lock<std::mutex> g(dm);
        dcv.wait(g, [&] { return left.load() == 0; });
    }

private:
    CopyPool() {
        int n = 12;
        if (const char *v = std::getenv("ASTROZ_COPY_THREADS")) n = std::max(0, std::min(64, std::atoi(v)));
        const unsigned hw = std::thread::hardware_concurrency();
        if (hw && (unsigned)n > hw) n = (int)hw;
        for (int i = 0; i < n; ++i) workers_.emplace_back([this] { loop(); });
        for (auto &t : workers_) t.detach();
    }
    // bytes [b0, b1) of the logical contiguous source, scattered to rows of the destination
    static void run(char *dst, const char *src, size_t rowBytes, size_t hpitch, size_t b0, size_t b1) {
        if (hpitch == rowBytes) {
            stream_copy(dst + b0, src + b0, b1 - b0);
            return;
        }
        size_t b = b0;
        while (b < b1) {
            const size_t r = b / rowBytes, o = b % rowBytes;
            const size_t len = std::min(rowBytes - o, b1 - b);
            stream_copy(dst + r * hpitch + o, src + b, len);
            b += len;
        }
    }
    void push(std::function<void()> f) {
        {
            std::lock_guard<std::mutex> g(m_);
            q_.push_back(std::move(f));
        }
        cv_.notify_one();
    }
    void loop() {
        for (;;) {
            std::function<void()> f;
            {
                std::unique_lock<std::mutex> g(m_);
                cv_.wait(g, [&] { return !q_.empty(); });
                f = std::move(q_.front());
                q_.pop_front();
            }
            f();
        }
    }
    std::vector<std::thread> workers_;
    std::mutex m_;
    std::condition_variable cv_;
    std::deque<std::function<void()>> q_;
};

}  // namespace

bool is_pageable(const void *p) {
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        (void)cudaGetLastError();
        return true;
    }
    return a.type == cudaMemoryTypeUnregistered;
}

HostRing::~HostRing() {
    for (cudaEvent_t e : ev_)
        if (e) cudaEventDestroy(e);
}

cudaError_t HostRing::ensure_ring() {
    if (ring_.p) return cudaSuccess;
    for (cudaEvent_t &e : ev_)
        if (!e) {
            const cudaError_t r = cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
            if (r != cudaSuccess) return r;
        }
    return ring_.reserve(kPieceBytes * kSlots);
}

char *HostRing::slot(size_t i) const { return ring_.p + (i % kSlots) * kPieceBytes; }

cudaError_t HostRing::deliver(bool pageable, cudaEvent_t ready, const void *dsrc, void *hdst, size_t rows,
                              size_t rowBytes, size_t hpitch, cudaStream_t copy) {
    if (!pageable) {
        if (rows == 1 || hpitch == rowBytes)
            return cudaMemcpyAsync(hdst, dsrc, rows * rowBytes, cudaMemcpyDeviceToHost, copy);
        return cudaMemcpy2DAsync(hdst, hpitch, dsrc, rowBytes, rowBytes, rows, cudaMemcpyDeviceToHost, copy);
    }
    const char *src = static_cast<const char *>(dsrc);
    char *dst = static_cast<char *>(hdst);
    if (rows == 1 || hpitch == rowBytes) {  // one contiguous run: cut by bytes
        const size_t total = rows * rowBytes;
        for (size_t b = 0; b < total; b += kPieceBytes) {
            const size_t len = std::min(kPieceBytes, total - b);
            plan_.push_back(Piece{src + b, dst + b, 1, len, len, ready});
        }
    } else if (rowBytes > kPieceBytes) {     // very wide rows: each row cut by bytes
        for (size_t r = 0; r < rows; ++r)
            for (size_t b = 0; b < rowBytes; b += kPieceBytes) {
                const size_t len = std::min(kPieceBytes, rowBytes - b);
                plan_.push_back(Piece{src + r * rowBytes + b, dst + r * hpitch + b, 1, len, len, ready});
            }
    } else {                                // whole rows per piece
        const size_t per = std::max<size_t>(1, kPieceBytes / rowBytes);
        for (size_t r = 0; r < rows; r += per)
            plan_.push_back(Piece{src + r * rowBytes, dst + r * hpitch, std::min(per, rows - r), rowBytes, hpitch, ready});
    }
    return cudaSuccess;
}

cudaError_t HostRing::drain(cudaStream_t copy) {
    if (plan_.empty()) return cudaSuccess;
    cudaError_t e = ensure_ring();
    CopyPool &pool = CopyPool::get();
    const size_t n = plan_.size();
    auto issue = [&](size_t i) -> cudaError_t {
        const Piece &p = plan_[i];
        cudaError_t r = cudaStreamWaitEvent(copy, p.ready, 0);
        if (r == cudaSuccess) r = cudaMemcpyAsync(slot(i), p.dsrc, p.rows * p.rowBytes, cudaMemcpyDeviceToHost, copy);
        if (r == cudaSuccess) r = cudaEventRecord(ev_[i % kSlots], copy);
        return r;
    };
    for (size_t i = 0; i < std::min<size_t>(kSlots, n) && e == cudaSuccess; ++i) e = issue(i);
    for (size_t i = 0; i < n && e == cudaSuccess; ++i) {
        e = cudaEventSynchronize(ev_[i % kSlots]);
        if (e != cudaSuccess) break;
        const Piece &p = plan_[i];
        pool.copy(p.hdst, slot(i), p.rows, p.rowBytes, p.hpitch);
        if (i + kSlots < n) e = issue(i + kSlots);
    }
    plan_.clear();
    return e;
}

cudaError_t HostRing::upload(bool pageable, int nArrays, const void *const *src, void *const *dst,
                             const size_t *elemBytes, size_t count, cudaStream_t s) {
    if (!pageable) {
        for (int a = 0; a < nArrays; ++a) {
            const cudaError_t e = cudaMemcpyAsync(dst[a], src[a], count * elemBytes[a], cudaMemcpyHostToDevice, s);
            if (e != cudaSuccess) return e;
        }
        return cudaSuccess;
    }
    cudaError_t e = ensure_ring();
    if (e != cudaSuccess) return e;
    size_t perElem = 0;
    for (int a = 0; a < nArrays; ++a) perElem += elemBytes[a];
    const size_t granule = kPieceBytes / perElem;  // elements per ring slot
    CopyPool &pool = CopyPool::get();
    for (size_t g0 = 0; g0 < count; g0 += granule, ++uploads_) {
        const size_t gn = std::min(granule, count - g0);
        const cudaEvent_t done = ev_[uploads_ % kSlots];
        char *stage = slot(uploads_);
        e = cudaEventSynchronize(done);  // the slot's last transfer is done (returns at once if none was recorded)
        size_t at = 0;
        for (int a = 0; a < nArrays && e == cudaSuccess; ++a) {
            const size_t b = gn * elemBytes[a];
            pool.copy(stage + at, static_cast<const char *>(src[a]) + g0 * elemBytes[a], 1, b, b);
            e = cudaMemcpyAsync(static_cast<char *>(dst[a]) + g0 * elemBytes[a], stage + at, b, cudaMemcpyHostToDevice, s);
            at += b;
        }
        if (e == cudaSuccess) e = cudaEventRecord(done, s);
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

#define AZ_TRY(expr) do { const cudaError_t e_ = (expr); if (e_ != cudaSuccess) return e_; } while (0)

ChunkPipeline::~ChunkPipeline() {
    for (cudaEvent_t e : {kernelDone[0], kernelDone[1], copyDone[0], copyDone[1], inputsDone})
        if (e) cudaEventDestroy(e);
}

cudaError_t ChunkPipeline::create() {
    for (cudaEvent_t *e : {&kernelDone[0], &kernelDone[1], &copyDone[0], &copyDone[1], &inputsDone})
        if (!*e) AZ_TRY(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
    return cudaSuccess;
}

// Slot reuse.  Chunk k takes slot k % 2, which chunk k-2 used, so before chunk k's inputs go up the pipeline waits on
// copyDone[slot], recorded on `copy` after chunk k-2's deliveries were queued.  For a pinned / registered destination
// that event completes once the D2H copy has read the slot.  For a pageable one it does not cover the data: the
// deliveries were only planned when it was recorded.  They were drained during chunk k-1, though (each chunk drains the
// previous chunk's plan before queueing its own deliveries), and drain returns only when every planned piece is in its
// final place, so chunk k-2's data has left the slot by then.  Uploads and deliveries share the ring's slots, and drain
// fills them without waiting for an upload: before each drain the pipeline waits on inputsDone, this chunk's inputs
// having left the ring.
cudaError_t ChunkPipeline::run(cudaStream_t stream, cudaStream_t copy, uint32_t n, uint32_t chunk, int nIn,
                               const HostIn *in, int nOut, const HostOut *out, void *dIn, void *dOut,
                               const ChunkLaunch &launch) {
    const uint32_t nChunks = (uint32_t)(((uint64_t)n + chunk - 1) / chunk), slots = nChunks > 1 ? 2 : 1;
    // the bytes of one slot: what a single chunk needs
    const size_t inSlot = chunk_slots_bytes(in, nIn, 1, chunk), outSlot = chunk_slots_bytes(out, nOut, 1, chunk);
    std::vector<const void *> src(nIn);
    std::vector<void *> dI(nIn), dO(nOut);
    std::vector<size_t> inBytes(nIn);
    std::vector<char> outPg(nOut);
    bool inPageable = false, outPageable = false;
    for (int a = 0; a < nIn; ++a) {
        inPageable = inPageable || is_pageable(in[a].p);
        inBytes[a] = in[a].bytes;
    }
    for (int j = 0; j < nOut; ++j) {
        outPg[j] = out[j].p && is_pageable(out[j].p);
        outPageable = outPageable || outPg[j];
    }
    auto chunks = [&]() -> cudaError_t {
        for (uint32_t k = 0; k < nChunks; ++k) {
            const uint32_t slot = k % slots, first = k * chunk, m = std::min(chunk, n - first);
            char *at = static_cast<char *>(dIn) + slot * inSlot;
            for (int a = 0; a < nIn; ++a) {
                src[a] = static_cast<const char *>(in[a].p) + (size_t)first * in[a].bytes;
                dI[a] = at;
                at += chunk_col_bytes(chunk, in[a].bytes);
            }
            at = static_cast<char *>(dOut) + slot * outSlot;
            for (int j = 0; j < nOut; ++j) {
                dO[j] = out[j].p ? at : nullptr;
                if (out[j].p) at += chunk_col_bytes(chunk, out[j].bytes);
            }
            if (k >= slots) AZ_TRY(cudaEventSynchronize(copyDone[slot]));  // chunk k-2's results have left this slot
            AZ_TRY(ring.upload(inPageable, nIn, src.data(), dI.data(), inBytes.data(), m, stream));
            AZ_TRY(cudaEventRecord(inputsDone, stream));
            AZ_TRY(launch(k, first, m, dI.data(), dO.data(), stream));
            const cudaEvent_t ready = kernelDone[slot];
            AZ_TRY(cudaEventRecord(ready, stream));
            if (outPageable) {  // chunk k-1's pageable results go through the ring while chunk k computes
                AZ_TRY(cudaEventSynchronize(inputsDone));
                AZ_TRY(ring.drain(copy));
            }
            AZ_TRY(cudaStreamWaitEvent(copy, ready, 0));
            for (int j = 0; j < nOut; ++j) {
                if (!out[j].p) continue;
                char *dst = static_cast<char *>(out[j].p) + (size_t)first * out[j].bytes;
                const size_t b = (size_t)m * out[j].bytes;
                AZ_TRY(ring.deliver(outPg[j], ready, dO[j], dst, 1, b, b, copy));
            }
            AZ_TRY(cudaEventRecord(copyDone[slot], copy));
        }
        AZ_TRY(ring.drain(copy));
        AZ_TRY(cudaStreamSynchronize(copy));
        return cudaStreamSynchronize(stream);
    };
    ring.discard();
    const cudaError_t e = chunks();
    if (e != cudaSuccess) {  // nothing may write to the caller's memory, or read the slots, after the return
        ring.discard();
        cudaStreamSynchronize(copy);
        cudaStreamSynchronize(stream);
    }
    return e;
}

}  // namespace az
