// buffers.h -- the host-side plumbing every native handle shares: owned device / pinned host allocations and the CUDA error check.
// Host code only.  A handle holds its buffers as members, so destroying the handle frees them: there is no list of buffers to keep.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>
#include <string>

#include "../../include/erasor_b200.h"

namespace erasor {

// One cudaMalloc (kPinned: cudaMallocHost) allocation, owned: move-only, freed by the destructor.  Nothing throws; the
// allocating calls return the CUDA error.
template <bool kPinned>
class CudaBuffer {
public:
    CudaBuffer() = default;
    // epoch: bumped by every allocation and every move into this buffer (a captured CUDA graph holds the old pointer)
    explicit CudaBuffer(uint64_t* epoch) : epoch_(epoch) {}
    CudaBuffer(const CudaBuffer&) = delete;
    CudaBuffer& operator=(const CudaBuffer&) = delete;
    CudaBuffer(CudaBuffer&& o) noexcept : p_(o.p_), cap_(o.cap_), epoch_(o.epoch_) { o.p_ = nullptr; o.cap_ = 0; }
    // the epoch stays with the buffer moved into, so std::swap keeps each buffer's own
    CudaBuffer& operator=(CudaBuffer&& o) noexcept {
        if (this != &o) {
            free();
            p_ = o.p_; cap_ = o.cap_;
            o.p_ = nullptr; o.cap_ = 0;
            if (epoch_) ++*epoch_;
        }
        return *this;
    }
    ~CudaBuffer() { free(); }

    void*  p() const { return p_; }
    size_t cap() const { return cap_; }
    template <class T> T* as() const { return static_cast<T*>(p_); }

    // exactly `bytes`; the old allocation is freed first and its contents are not kept
    cudaError_t allocate(size_t bytes) {
        free();
        if (epoch_) ++*epoch_;
        void* q = nullptr;
        const cudaError_t e = kPinned ? cudaMallocHost(&q, bytes) : cudaMalloc(&q, bytes);
        if (e != cudaSuccess) return e;
        p_ = q; cap_ = bytes;
        return cudaSuccess;
    }
    // at least `bytes`: a larger request reallocates with a quarter + 4 KiB of headroom, so that sizes creeping up from call to
    // call do not pay a cudaFree (a device-wide synchronisation) each time
    cudaError_t ensure(size_t bytes) { return bytes <= cap_ ? cudaSuccess : allocate(bytes + bytes / 4 + 4096); }

private:
    void free() {
        if (p_) {
            if (kPinned) cudaFreeHost(p_);
            else         cudaFree(p_);
        }
        p_ = nullptr; cap_ = 0;
    }
    void*     p_ = nullptr;
    size_t    cap_ = 0;
    uint64_t* epoch_ = nullptr;
};

using DeviceBuffer = CudaBuffer<false>;
using PinnedBuffer = CudaBuffer<true>;

}  // namespace erasor

// When `call` (a cudaError_t expression) fails: err = text + ": " + CUDA's message, and the enclosing function returns
// ERASOR_E_CUDA.  Each file wraps it in a one-line alias that passes #call itself, e.g.
//     #define CK(call) ERASOR_CUDA_TRY(h->err, call, #call)
// so that the message shows the call as written: an argument handed on to a second macro is macro-expanded before that macro
// could stringify it, and some CUDA entry points are macros.
#define ERASOR_CUDA_TRY(err, call, text)                                                           \
    do {                                                                                           \
        const cudaError_t e__ = (call);                                                            \
        if (e__ != cudaSuccess) {                                                                  \
            (err) = std::string(text) + ": " + cudaGetErrorString(e__);                            \
            return ERASOR_E_CUDA;                                                                  \
        }                                                                                          \
    } while (0)
