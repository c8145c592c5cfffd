// huf_packed.cu -- the packed Huff0 decompress (include/fse_b200.h FSEB200_HUF_decompress{,1X}_packed): every block of a buffer
// FSEB200_HUF_compress{,1X}_packed wrote, located by its offsets, through the unchanged descriptor decoder of huf_decode.cu.
//
// Huff0's decoders already read a stored length equal to the block size as a raw copy and a length of 1 as RLE, so unlike FSE
// (fse_packed.cu) no block needs a path of its own.  Three steps, all on the stream:
//   1. a classify kernel derives the descriptors (source dIn + offset, size L) into stream scratch;
//   2. the descriptor decoder (pass A, pass B, the X2 verdict pass) on them;
//   3. a kernel gives an empty block (n == 0 and L == 0, what the packed compress stores for it) the result 0 -- the decoder
//      answers dstSize 0 with dstSize_tooSmall.
#include "common.cuh"
#include "launchers.h"
#include "launch_util.cuh"

namespace fseb {

namespace hufp {

struct HufUnpack {
    const u8* in; const u64* offset;
    const u64* dstSize; u64* result;
    const u8** decSrc; u64* decSize;                                // the derived descriptors, in stream scratch
    u32 nBlocks;
};

constexpr int THREADS = 256;

__global__ void __launch_bounds__(THREADS) huf_unpack_classify_kernel(HufUnpack g)
{
    u64 const b = (u64)blockIdx.x * THREADS + threadIdx.x;
    if (b >= g.nBlocks) return;
    u64 const off = g.offset[b];
    g.decSrc[b] = g.in + off;
    g.decSize[b] = g.offset[b + 1] - off;
}

__global__ void __launch_bounds__(THREADS) huf_unpack_empty_kernel(HufUnpack g)
{
    u64 const b = (u64)blockIdx.x * THREADS + threadIdx.x;
    if (b >= g.nBlocks) return;
    if (g.dstSize[b] == 0 && g.decSize[b] == 0) g.result[b] = 0;
}

}  // namespace hufp

cudaError_t launch_huf_decompress_packed(u8* const* dst, const u64* dstSize, u64* result, const u8* in, const u64* offset,
                                         u32 nBlocks, int nStreams, cudaStream_t stream)
{
    if (nBlocks == 0) return cudaSuccess;
    size_t const n = nBlocks;
    cudaError_t e;
    u8* const s = (u8*)stream_scratch(7, stream, 2 * sizeof(u64) * n, &e);
    if (e != cudaSuccess) return e;
    hufp::HufUnpack g;
    g.in = in; g.offset = offset; g.dstSize = dstSize; g.result = result;
    g.decSrc = (const u8**)s; g.decSize = (u64*)(s + 8 * n); g.nBlocks = nBlocks;
    unsigned const grid = (unsigned)((n + hufp::THREADS - 1) / hufp::THREADS);
    hufp::huf_unpack_classify_kernel<<<grid, hufp::THREADS, 0, stream>>>(g);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    BlockDescs d;
    d.dst = dst; d.dstCap = dstSize; d.result = result; d.src = g.decSrc; d.srcSize = g.decSize; d.nBlocks = nBlocks;
    if ((e = launch_huf_decode_blocks(d, nStreams, stream)) != cudaSuccess) return e;
    hufp::huf_unpack_empty_kernel<<<grid, hufp::THREADS, 0, stream>>>(g);
    return cudaGetLastError();
}

}  // namespace fseb
