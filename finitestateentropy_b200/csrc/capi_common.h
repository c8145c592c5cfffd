// capi_common.h -- what the two C-ABI files share: capi.cu (device-pointer tier, the reference's one-block drop-ins, tables,
// generators) and host_pipeline.cu (whole batches on host buffers).
#pragma once
#include "common.cuh"
#include "launchers.h"
#include <cstdio>
#include <cstdlib>

#define FSEB_API extern "C" __attribute__((visibility("default")))

namespace fseb {

// There is no CPU fallback: a CUDA failure in a call that has no error value to return aborts with its name.
[[noreturn]] inline void die(const char* what, cudaError_t e)
{
    std::fprintf(stderr, "libfse_b200: %s failed: %s -- this library has no CPU fallback\n", what, cudaGetErrorString(e));
    std::abort();
}
#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) fseb::die(#call, e_); } while (0)

inline BatchGeom geom(size_t total, size_t blockSize, size_t slot)
{
    BatchGeom g;
    g.total = total; g.blockSize = (u32)blockSize; g.slot = (u32)slot;
    g.nBlocks = blockSize ? (u32)((total + blockSize - 1) / blockSize) : 0;
    return g;
}
inline size_t ok_or_generic(cudaError_t e) { return e == cudaSuccess ? 0 : (size_t)err(E_GENERIC); }

constexpr size_t FSE_ONE_BLOCK_MAX = (size_t)1 << 30;                   // same limit as the batch tier (FSEB_DECL_*)

typedef cudaError_t (*enc_fn)(const BatchGeom&, void*, u64*, const void*, unsigned, unsigned, cudaStream_t);
typedef cudaError_t (*dec_fn)(const BatchGeom&, void*, const void*, const u64*, u64*, const void*, cudaStream_t);

inline cudaError_t huf_dec_std(const BatchGeom& g, void* d, const void* c, const u64* cs, u64* r, const void* o, cudaStream_t s) { return launch_huf_decode(g, d, c, cs, r, o, s, 0); }

}  // namespace fseb
