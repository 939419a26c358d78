// cuda_owner.h -- how the library holds CUDA resources: PG_CUDA (a failed call throws), owners of device memory, streams, events, pinned
// host blocks and IPC mappings, the functions that create them, and DeviceScope.  Host-only and header-only: any build can include it.
#pragma once
#include <cuda_runtime_api.h>
#include <cstdio>
#include <stdexcept>
#include <utility>

namespace pgb {

#define PG_CUDA(call)                                                                                         \
    do {                                                                                                      \
        cudaError_t e__ = (call);                                                                             \
        if (e__ != cudaSuccess) {                                                                             \
            char b__[512];                                                                                    \
            snprintf(b__, sizeof b__, "CUDA error %s at %s:%d: %s", cudaGetErrorName(e__), __FILE__, __LINE__, \
                     cudaGetErrorString(e__));                                                                \
            throw std::runtime_error(b__);                                                                    \
        }                                                                                                     \
    } while (0)

struct DevBuf {
    void* p = nullptr;
    size_t bytes = 0;
    DevBuf() {}
    DevBuf(DevBuf&& o) noexcept : p(o.p), bytes(o.bytes) { o.p = nullptr; o.bytes = 0; }
    DevBuf& operator=(DevBuf&& o) noexcept { std::swap(p, o.p); std::swap(bytes, o.bytes); return *this; }
    ~DevBuf() { release(); }
    void alloc(size_t n) {
        release();
        if (n == 0) n = 16;
        PG_CUDA(cudaMalloc(&p, n));
        bytes = n;
    }
    void ensure(size_t n) { if (n > bytes) alloc(n + n / 4); }
    void release() { if (p) cudaFree(p); p = nullptr; bytes = 0; }
    template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

// Owner of a stream, an event, a pinned host block or an IPC mapping, in the style of DevBuf.  Made by the make_* functions below;
// an IPC mapping owns the pointer cudaIpcOpenMemHandle returned.
template <class T, cudaError_t (*Release)(T)>
struct CudaOwned {
    T h = nullptr;
    CudaOwned() {}
    explicit CudaOwned(T x) : h(x) {}
    CudaOwned(CudaOwned&& o) noexcept : h(o.h) { o.h = nullptr; }
    CudaOwned& operator=(CudaOwned&& o) noexcept { std::swap(h, o.h); return *this; }
    ~CudaOwned() { if (h) Release(h); }
    operator T() const { return h; }
};
template <class T> cudaError_t free_pinned(T* p) { return cudaFreeHost(p); }
using Stream = CudaOwned<cudaStream_t, cudaStreamDestroy>;
using Event = CudaOwned<cudaEvent_t, cudaEventDestroy>;
template <class T> using Pinned = CudaOwned<T*, free_pinned<T>>;
using IpcMapping = CudaOwned<void*, cudaIpcCloseMemHandle>;

inline Stream make_stream() { cudaStream_t s; PG_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking)); return Stream(s); }
inline Event make_event(unsigned flags = cudaEventDefault) { cudaEvent_t e; PG_CUDA(cudaEventCreateWithFlags(&e, flags)); return Event(e); }
template <class T> Pinned<T> make_pinned(size_t n) { void* p; PG_CUDA(cudaHostAlloc(&p, n * sizeof(T), cudaHostAllocDefault)); return Pinned<T>((T*)p); }

// Binds device d to the calling thread for the scope's duration, then restores the device that was current.  Unchecked.
struct DeviceScope {
    int old = 0;
    explicit DeviceScope(int d) { cudaGetDevice(&old); cudaSetDevice(d); }
    ~DeviceScope() { cudaSetDevice(old); }
    DeviceScope(const DeviceScope&) = delete;
};

}   // namespace pgb
