// launch_util.cuh -- host-side launch helpers shared by the kernel launchers.
//
// Everything a launcher caches (SM count, opt-in shared-memory attribute of a kernel) is PER DEVICE: a C caller
// may drive several GPUs from one process (tier 1 takes device pointers and a stream), and
// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) only applies to the device that is current when it is called.
#pragma once
#include <cuda_runtime.h>
#include <mutex>
#include <vector>

namespace fseb {

constexpr int MAX_DEVICES = 64;

inline int current_device()
{
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= MAX_DEVICES) dev = 0;
    return dev;
}

inline int device_sm_count(int dev)
{
    static int sms[MAX_DEVICES];
    static std::once_flag once[MAX_DEVICES];
    std::call_once(once[dev], [dev] {
        int n = 132;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
        sms[dev] = n;
    });
    return sms[dev];
}

// Largest dynamic shared memory one block may opt in to (0 if the device cannot say).
inline int device_smem_optin(int dev)
{
    static int bytes[MAX_DEVICES];
    static std::once_flag once[MAX_DEVICES];
    std::call_once(once[dev], [dev] {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess || n < 0) n = 0;
        bytes[dev] = n;
    });
    return bytes[dev];
}

// One instance per kernel (function-local static in its launcher): remembers on which devices the kernel's
// dynamic shared-memory limit was already raised.
struct SmemOptIn {
    std::mutex mu;
    int granted[MAX_DEVICES] = {};       // bytes already requested on that device
    template <typename K>
    cudaError_t ensure(K kernel, int dev, int bytes)
    {
        std::lock_guard<std::mutex> lock(mu);
        if (granted[dev] >= bytes) return cudaSuccess;
        cudaError_t const e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
        if (e == cudaSuccess) granted[dev] = bytes;
        return e;
    }
};

// Grow-only device scratch, one buffer per (purpose, device, stream): successive calls on a stream reuse it (stream order makes
// that safe), a different stream gets its own.  Returns nullptr and sets *err on failure.
inline void* stream_scratch(int purpose, cudaStream_t stream, size_t bytes, cudaError_t* err)
{
    struct Slot { int purpose, dev; cudaStream_t s; void* p; size_t cap; };
    static std::mutex mu;
    static std::vector<Slot> slots;
    std::lock_guard<std::mutex> lock(mu);
    int const dev = current_device();
    Slot* hit = nullptr;
    for (auto& sl : slots) if (sl.purpose == purpose && sl.s == stream && sl.dev == dev) { hit = &sl; break; }
    if (!hit) { slots.push_back(Slot{ purpose, dev, stream, nullptr, 0 }); hit = &slots.back(); }
    *err = cudaSuccess;
    if (hit->cap < bytes) {
        if (hit->p) { cudaStreamSynchronize(stream); cudaFree(hit->p); hit->p = nullptr; hit->cap = 0; }
        *err = cudaMalloc(&hit->p, bytes);
        if (*err != cudaSuccess) return nullptr;
        hit->cap = bytes;
    }
    return hit->p;
}

}  // namespace fseb
