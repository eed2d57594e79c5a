// cuda_owned.h — single owners of the CUDA resources a context holds: device arrays, pinned host blocks, events and
// streams. Each owner is move-only and releases what it holds when it is reset, assigned over or destroyed, so a call that
// throws half-way (CUDA_CHECK in context.cpp) leaks nothing and leaves no freed pointer behind.
//
// Destructors ignore release errors, as teardown always has. Calls that allocate return the cudaError_t and leave the
// throwing to the caller. Only the CUDA runtime API header is included: the CPU tests compile this header with g++
// against a fake runtime that fails chosen calls (tests/test_cuda_owned_cpu.py).
#pragma once

#include <cuda_runtime_api.h>

#include <stddef.h>

#include <utility>

namespace hnb_rt {

// `size()` elements of T from `Alloc`, given back with `Free`.
template <typename T, cudaError_t (*Alloc)(void**, size_t), cudaError_t (*Free)(void*)> class Block {
  public:
    Block() = default;
    Block(Block&& o) noexcept { swap(o); }
    Block& operator=(Block&& o) noexcept {
        Block(std::move(o)).swap(*this);
        return *this;
    }
    ~Block() {
        if (p_) (void)Free(p_);
    }
    void swap(Block& o) noexcept {
        std::swap(p_, o.p_);
        std::swap(n_, o.n_);
    }
    // Releases the block held, then allocates `n` elements, not initialised. The owner is empty if this fails.
    cudaError_t alloc(size_t n) {
        reset();
        void* p = nullptr;
        const cudaError_t e = Alloc(&p, n * sizeof(T));
        if (e == cudaSuccess) {
            p_ = static_cast<T*>(p);
            n_ = n;
        }
        return e;
    }
    void reset() { Block().swap(*this); }
    T* get() const { return p_; }
    size_t size() const { return n_; }
    explicit operator bool() const { return p_ != nullptr; }

  private:
    T* p_ = nullptr;
    size_t n_ = 0;
};

template <typename T> using DeviceArray = Block<T, cudaMalloc, cudaFree>;
using PinnedBlock = Block<char, cudaMallocHost, cudaFreeHost>;

// Replaces the array with `n` zero-filled elements whose first `keep` (0: none) are copied from the old array, in order on
// `st`. Kernels queued earlier may still read the old array, so the stream is synchronised before it is released (an
// empty owner has nothing to wait for: this is then a zero-filled allocation). Only when every step succeeded does the
// new array replace the old one; on failure the owner keeps its old array and size, and the new array is released.
template <typename T> cudaError_t grow(DeviceArray<T>& a, size_t n, size_t keep, cudaStream_t st) {
    DeviceArray<T> next;
    cudaError_t e = next.alloc(n);
    if (e == cudaSuccess) e = cudaMemsetAsync(next.get(), 0, n * sizeof(T), st);
    if (e == cudaSuccess && keep) e = cudaMemcpyAsync(next.get(), a.get(), keep * sizeof(T), cudaMemcpyDeviceToDevice, st);
    if (e == cudaSuccess && a) e = cudaStreamSynchronize(st);
    if (e == cudaSuccess) a.swap(next);
    return e;
}

// A CUDA handle, either created here and destroyed with the owner, or borrowed from the caller and never destroyed.
// Converts to the handle it holds.
template <typename H, cudaError_t (*Create)(H*, unsigned), cudaError_t (*Destroy)(H)> class Handle {
  public:
    Handle() = default;
    Handle(Handle&& o) noexcept { swap(o); }
    Handle& operator=(Handle&& o) noexcept {
        Handle(std::move(o)).swap(*this);
        return *this;
    }
    ~Handle() {
        if (h_ && owned_) (void)Destroy(h_);
    }
    void swap(Handle& o) noexcept {
        std::swap(h_, o.h_);
        std::swap(owned_, o.owned_);
    }
    // Releases the handle held, then creates one that this owner destroys. The owner is empty if this fails.
    cudaError_t create(unsigned flags) {
        Handle().swap(*this);
        H h = nullptr;
        const cudaError_t e = Create(&h, flags);
        if (e == cudaSuccess) {
            h_ = h;
            owned_ = true;
        }
        return e;
    }
    void borrow(H h) {
        Handle().swap(*this);
        h_ = h;
    }
    H get() const { return h_; }
    operator H() const { return h_; }

  private:
    H h_ = nullptr;
    bool owned_ = false;
};

using Event = Handle<cudaEvent_t, cudaEventCreateWithFlags, cudaEventDestroy>;
using Stream = Handle<cudaStream_t, cudaStreamCreateWithFlags, cudaStreamDestroy>;

}  // namespace hnb_rt
