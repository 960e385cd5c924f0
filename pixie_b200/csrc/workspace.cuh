// Error reporting of the library, and the scratch memory of the stateless device operations behind the C ABI (those that
// take no handle): each of those returns the first failing cudaError_t and leaves the thread's last error clear.
#pragma once
#include <cuda_runtime.h>
#include <cstddef>
#include <string>

// Returns the status of `expr` from the enclosing operation when it is an error. The thread's last error is cleared first:
// the operations check it for launch errors, so a stale one would make the next, valid call fail.
#define PIXIE_TRY(expr) \
    do { const cudaError_t pixie_e_ = (expr); if (pixie_e_ != cudaSuccess) { cudaGetLastError(); return pixie_e_; } } while (0)

namespace pixie {

// The message pixie_last_error() returns, one per host thread, is the library's only error state (capi.cu). Both setters
// return 1, the C ABI's failure code.
// Refused input or state, e.g. "forward before finalize".
int fail(const std::string& message);
// A failed CUDA call: "<what>: <CUDA's description of e>". Also clears the thread's last error, so that the failure is not
// blamed on the next, valid call.
int fail(const std::string& what, cudaError_t e);

// One cudaMallocAsync on the operation's stream, handed out as 256-byte aligned typed arrays and freed on that stream
// when the workspace goes out of scope, so every return frees it.
class Workspace {
public:
    explicit Workspace(cudaStream_t st) : st_(st) {}
    ~Workspace() { if (base_ && cudaFreeAsync(base_, st_) != cudaSuccess) cudaGetLastError(); }
    Workspace(const Workspace&) = delete;
    Workspace& operator=(const Workspace&) = delete;

    // take_all() takes every array with take(). It runs once to size the scratch (take() returns null), then, after the
    // allocation, once more to hand out the arrays.
    template <class F> cudaError_t carve(F&& take_all) {
        take_all();
        void* p = nullptr;
        const cudaError_t e = cudaMallocAsync(&p, off_, st_);
        if (e != cudaSuccess) return e;
        base_ = static_cast<char*>(p);
        off_ = 0;
        take_all();
        return cudaSuccess;
    }
    template <class T> T* take(size_t count) {
        T* p = base_ ? reinterpret_cast<T*>(base_ + off_) : nullptr;
        off_ += (count * sizeof(T) + 255) & ~size_t(255);
        return p;
    }

private:
    cudaStream_t st_;
    char* base_ = nullptr;
    size_t off_ = 0;
};

}  // namespace pixie
