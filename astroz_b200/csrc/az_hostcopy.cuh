// az_hostcopy.cuh -- the handle's grow-only buffers, and the pinned transfers of the host-buffer entry points of
// az_capi.cu.  A DMA to or from PAGEABLE memory is staged by the driver through a small internal buffer, synchronously,
// at a fraction of the PCIe rate.  Instead such transfers go through a ring of pinned slots owned by the handle
// (full-rate DMA), and a small pool of host threads copies each piece between its slot and the caller's memory while
// the next pieces are in flight.  ChunkPipeline runs the host-buffer calls that cut their items into chunks over two
// device slots.
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <functional>
#include <vector>

namespace az {

// Grow-only buffer from Alloc / Free: device memory (DevBuf) or page-locked host memory (PinnedBuf).  A DevBuf is freed
// on the device that is current when it is destroyed.
template <typename T, cudaError_t (*Alloc)(void **, size_t), cudaError_t (*Free)(void *)>
struct GrowBuf {
    T *p = nullptr;
    size_t cap = 0;
    GrowBuf() = default;
    GrowBuf(const GrowBuf &) = delete;
    GrowBuf &operator=(const GrowBuf &) = delete;
    ~GrowBuf() {
        if (p) Free(p);
    }
    cudaError_t reserve(size_t n) {
        if (n <= cap) return cudaSuccess;
        if (p) Free(p);
        p = nullptr;
        cap = 0;
        cudaError_t e = Alloc(reinterpret_cast<void **>(&p), n * sizeof(T));
        if (e == cudaSuccess) cap = n;
        return e;
    }
};
template <typename T>
using DevBuf = GrowBuf<T, cudaMalloc, cudaFree>;
template <typename T>
using PinnedBuf = GrowBuf<T, cudaMallocHost, cudaFreeHost>;

// true unless p is device, managed, pinned or registered memory
bool is_pageable(const void *p);

class HostRing {
public:
    HostRing() = default;
    HostRing(const HostRing &) = delete;
    HostRing &operator=(const HostRing &) = delete;
    ~HostRing();

    // Send `rows` rows of rowBytes (contiguous on the device at dsrc) to the host at hdst with pitch hpitch, once
    // `ready` has completed.  A pinned / registered destination gets the copy queued on `copy` right away (the caller
    // has made `copy` wait for `ready`); a pageable one is planned as ring-sized pieces that drain() delivers.
    cudaError_t deliver(bool pageable, cudaEvent_t ready, const void *dsrc, void *hdst, size_t rows, size_t rowBytes,
                        size_t hpitch, cudaStream_t copy);
    // Deliver the planned pieces: up to kSlots of them in flight on `copy` while the pool copies the landed one to its
    // final place.  Returns when every planned piece is in place; the plan is empty afterwards, also on failure.
    cudaError_t drain(cudaStream_t copy);
    // Forget pieces a failed call planned and never drained.
    void discard() { plan_.clear(); }

    // Copy `count` elements of each of the nArrays host arrays src[a] (elemBytes[a] bytes per element) to the device
    // arrays dst[a] on stream s.  Pageable sources are staged through the ring slots, all arrays' elements of one
    // granule in one slot; a slot is refilled only after its previous upload has completed.
    cudaError_t upload(bool pageable, int nArrays, const void *const *src, void *const *dst, const size_t *elemBytes,
                       size_t count, cudaStream_t s);

private:
    static constexpr int kSlots = 3;
    struct Piece {  // one ring-sized piece of a planned delivery: rows x rowBytes, contiguous on the device
        const char *dsrc;
        char *hdst;
        size_t rows, rowBytes, hpitch;
        cudaEvent_t ready;
    };
    cudaError_t ensure_ring();
    char *slot(size_t i) const;

    PinnedBuf<char> ring_;
    cudaEvent_t ev_[kSlots] = {};  // recorded after each slot's last transfer
    std::vector<Piece> plan_;
    size_t uploads_ = 0;  // granules staged so far: the next upload takes slot uploads_ % kSlots
};

// A host column of a chunked call: item i at p + i * bytes.  An output column with p = nullptr is not wanted: it takes
// no device memory and its launch pointer is nullptr.
struct HostIn { const void *p; size_t bytes; };
struct HostOut { void *p; size_t bytes; };

// Device bytes of one column of a chunk within its slot: the next column starts 16-byte aligned.
inline size_t chunk_col_bytes(uint32_t chunk, size_t bytes) { return ((size_t)chunk * bytes + 15) & ~size_t(15); }
// Device bytes ChunkPipeline::run needs for the columns of one side (HostIn or HostOut) over n items in chunks of
// `chunk`: one slot, or two when n spans several chunks.
template <class Col>
size_t chunk_slots_bytes(const Col *cols, int nCols, uint32_t n, uint32_t chunk) {
    size_t b = 0;
    for (int k = 0; k < nCols; ++k)
        if (cols[k].p) b += chunk_col_bytes(chunk, cols[k].bytes);
    return (n > chunk ? 2 : 1) * b;
}

// launch(k, first, count, dIn, dOut, s) queues chunk k's work on s: items [first, first + count), with the device copy
// of input column a at dIn[a] and output column j to be written at dOut[j].
using ChunkLaunch = std::function<cudaError_t(uint32_t k, uint32_t first, uint32_t count, void *const *dIn,
                                              void *const *dOut, cudaStream_t s)>;

// The two-slot chunk pipeline of the host-buffer calls: n items are cut into chunks of `chunk` on two device slots.
// Chunk k's inputs go up and its work runs on `stream` while chunk k-1's results leave on `copy` (pinned / registered
// destinations) or through the ring and the copy pool (pageable ones); pageable inputs are staged through the ring too.
// Not copyable (the ring is not).
class ChunkPipeline {
public:
    ~ChunkPipeline();
    cudaError_t create();  // the events, on the current device

    // Run the chunks.  dIn / dOut are device memory of chunk_slots_bytes() for `in` / `out`.  Returns once every
    // result is in place and both streams are idle -- also on failure, when the ring's plan is forgotten first, so no
    // copy into the caller's memory is still queued after the call returns.
    cudaError_t run(cudaStream_t stream, cudaStream_t copy, uint32_t n, uint32_t chunk, int nIn, const HostIn *in,
                    int nOut, const HostOut *out, void *dIn, void *dOut, const ChunkLaunch &launch);

    HostRing ring;  // pinned transfers from / to pageable caller memory (also used outside run)

private:
    // slot k's work / result copy has finished; the current chunk's inputs are on the device
    cudaEvent_t kernelDone[2] = {}, copyDone[2] = {}, inputsDone = nullptr;
};

}  // namespace az
