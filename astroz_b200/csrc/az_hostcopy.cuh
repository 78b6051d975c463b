// az_hostcopy.cuh -- the handle's grow-only buffers, and the pinned transfers of the host-buffer entry points of
// az_capi.cu.  A DMA to or from PAGEABLE memory is staged by the driver through a small internal buffer, synchronously,
// at a fraction of the PCIe rate.  Instead such transfers go through a ring of pinned slots owned by the handle
// (full-rate DMA), and a small pool of host threads copies each piece between its slot and the caller's memory while
// the next pieces are in flight.
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>

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

}  // namespace az
