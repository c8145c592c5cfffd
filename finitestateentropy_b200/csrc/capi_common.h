// capi_common.h -- what the two C-ABI files share: capi.cu (device-pointer tier, the reference's one-block drop-ins, tables,
// generators) and host_pipeline.cu (whole batches on host buffers, which runs capi.cu's chain helpers on each chunk).
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

// Huff0 forms: nStreams 4 or 1, every block in that form; 0, each block's form in dSingleStream, which must then be given
inline bool forms_given(int nStreams, const void* dSingleStream) { return nStreams || dSingleStream; }
// The form of a packed chain compress: every block in nStreams streams (4 or 1), or (0) each block's form in dSingleStream --
// read, or under zstd's literal policy (`literals`, with minLiterals and minGainLog) chosen by the device and written there.
struct ChainForm {
    int nStreams;
    unsigned char* dSingleStream;
    bool literals;
    unsigned minLiterals, minGainLog;
};
// The packed chain compress and decompress on device arrays (FSEB200_HUF_*_chains_packed, FSEB200_HUF_*_repeat_packed), argument
// checks included: what those entry points return.  Decompress: nStreams as ChainForm's, the forms in dSingleStream.
size_t huf_repeat_chains_packed(size_t nChains, const size_t* dChainStarts, size_t nBlocks, void* dOut, size_t outCapacity,
                                size_t* dOffsets, size_t* dCSizes, unsigned char* dKinds, const void* const* dSrcs,
                                const size_t* dSrcSizes, const int* dPreferRepeat, unsigned* const* dCTables, int* dRepeats,
                                const void** dChainHeaders, size_t* dChainHeaderSizes, const ChainForm& f, unsigned msv, unsigned tlog,
                                void* stream);
size_t huf_repeat_unpack(size_t nChains, const size_t* dChainStarts, size_t nBlocks, void* const* dDsts, const size_t* dDstSizes,
                         size_t* dResults, const void* dIn, const size_t* dOffsets, const unsigned char* dKinds,
                         const void* const* dChainHeaders, const size_t* dChainHeaderSizes, int nStreams, void* stream,
                         const unsigned char* dSingleStream = nullptr);

}  // namespace fseb
