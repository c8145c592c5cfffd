// frame.cu -- the device side of the .fse frame calls (include/fse_b200.h FSEB200_frame_{compress,decompress}_host).
//
// Frame layout (the reference's programs/fileio.c:266-285): block b is a 1-byte header { type:2 (0 compressed, 1 raw, 2 RLE),
// full:1, 0:5 }, then its regenerated size as 2 big-endian bytes unless it is full (n == blockSize), then its compressed size
// as 2 big-endian bytes if it is compressed, then its payload: the compressed bytes, the n source bytes of a raw block, or the
// one byte of an RLE block.
//
// Compress, per chunk, after the device packed compress of its blocks (fse_packed.cu / huf_encode.cu): the payloads are already
// the packed stream's stored blocks, in order, so the frame body is that stream with a header in front of each block.  A scan of
// header + stored length (pack_dev.cuh) gives each block's frame offset and writes its header; one CTA per block then moves its
// payload from the packed buffer behind it.  The chunk's frame body is one contiguous range.
// Decompress, per chunk: the compressed blocks go to the descriptor decoders with pointers into the chunk's frame bytes (the host
// builds the descriptors); raw and RLE blocks come from frame_stored_kernel, one CTA per block of a compact index.
#include "common.cuh"
#include "launchers.h"
#include "launch_util.cuh"
#include "pack_dev.cuh"

namespace fseb {
namespace frame {

// the packed compress's outputs for a chunk (offset: nBlocks + 1 entries) and the frame body they become
struct Body {
    const u8* packed; const u64* offset; const u64* value; const u64* srcSize;
    u8* out; u64* bodyOff;                                          // bodyOff[b]: where block b's header starts; stream scratch
    u64 blockSize; u32 nBlocks;
};

// header bytes of a block with compress value v and n source bytes; an error value stores nothing (the host reports it)
__device__ __forceinline__ u32 header_len(u64 v, u64 n, u64 blockSize)
{
    if (is_err(v)) return 0;
    return 1 + (n == blockSize ? 0 : 2) + (v >= 2 ? 2 : 0);
}

struct Headers {
    typedef Body Geo;
    typedef u64* Aux;
    static __device__ __forceinline__ u64 value(const Body& g, u64 b) { return g.value[b]; }
    static __device__ __forceinline__ u64 len(const Body& g, u64 b, u64 v)
    {
        return header_len(v, g.srcSize[b], g.blockSize) + (g.offset[b + 1] - g.offset[b]);
    }
    static __device__ __forceinline__ void place(const Body& g, u64*, u64 b, u64 v, u64 off, u64)
    {
        g.bodyOff[b] = off;
        if (is_err(v)) return;
        u64 const n = g.srcSize[b];
        bool const full = n == g.blockSize;
        u8* h = g.out + off;
        *h++ = (u8)(((v == 0 ? 1u : v == 1 ? 2u : 0u) << 6) | (full ? 0x20u : 0u));
        if (!full) { *h++ = (u8)(n >> 8); *h++ = (u8)n; }
        if (v >= 2) { *h++ = (u8)(v >> 8); *h++ = (u8)v; }
    }
};

// one CTA per block (blocks b0 + blockIdx.x): the stored payload behind its header
__global__ void __launch_bounds__(pack::COPY_THREADS) frame_payload_kernel(Body g, u64 b0)
{
    u64 const b = b0 + blockIdx.x;
    u64 const v = g.value[b];
    u32 const L = (u32)(g.offset[b + 1] - g.offset[b]);             // at most a block, 64 KB
    if (is_err(v) || L == 0) return;
    pack::cta_copy<pack::COPY_THREADS, pack::COPY_UNROLL>(g.out + g.bodyOff[b] + header_len(v, g.srcSize[b], g.blockSize),
                                                         g.packed + g.offset[b], L);
}

// raw and RLE blocks of a chunk: index[3 j .. 3 j + 2] = output offset, payload offset in the chunk's frame bytes, and
// n | kind << 32 (kind 1 raw, 2 RLE)
__global__ void __launch_bounds__(pack::COPY_THREADS) frame_stored_kernel(u8* out, const u8* in, const u64* index, u64 j0)
{
    const u64* const e = index + 3 * (j0 + blockIdx.x);
    u64 const w = e[2];
    u32 const n = (u32)w;
    if ((w >> 32) == 1) pack::cta_copy<pack::COPY_THREADS, pack::COPY_UNROLL>(out + e[0], in + e[1], n);
    else pack::cta_fill<false>(out + e[0], in + e[1], n);
}

constexpr u64 GRID_MAX = 1ull << 30;                                // CTAs per launch of the one-CTA-per-block kernels

}  // namespace frame

cudaError_t launch_frame_body(u8* out, const u8* packed, const u64* offset, const u64* value, const u64* srcSize, u32 nBlocks,
                              u64 blockSize, cudaStream_t stream)
{
    if (nBlocks == 0) return cudaSuccess;
    size_t const n = nBlocks;
    unsigned const tiles = (unsigned)((n + pack::PACK_TILE - 1) / pack::PACK_TILE);
    cudaError_t e;
    u64* const s = (u64*)stream_scratch(8, stream, sizeof(u64) * (n + tiles + 1), &e);
    if (e != cudaSuccess) return e;
    frame::Body g;
    g.packed = packed; g.offset = offset; g.value = value; g.srcSize = srcSize;
    g.out = out; g.bodyOff = s; g.blockSize = blockSize; g.nBlocks = nBlocks;
    u64* const tileSum = s + n;                                     // tiles + 1 words: the body's length goes to the last
    pack::pack_sums_kernel<frame::Headers><<<tiles, pack::PACK_THREADS, 0, stream>>>(g, tileSum);
    pack::pack_scan_tiles_kernel<<<1, pack::PACK_SCAN_THREADS, 0, stream>>>(tileSum, tiles, nullptr, tileSum + tiles);
    pack::pack_place_kernel<frame::Headers><<<tiles, pack::PACK_THREADS, 0, stream>>>(g, tileSum, nullptr);
    for (u64 b0 = 0; b0 < n; b0 += frame::GRID_MAX)
        frame::frame_payload_kernel<<<(unsigned)(n - b0 < frame::GRID_MAX ? n - b0 : frame::GRID_MAX), pack::COPY_THREADS, 0, stream>>>(g, b0);
    return cudaGetLastError();
}

cudaError_t launch_frame_stored(u8* out, const u8* in, const u64* index, u64 nStored, cudaStream_t stream)
{
    for (u64 j0 = 0; j0 < nStored; j0 += frame::GRID_MAX)
        frame::frame_stored_kernel<<<(unsigned)(nStored - j0 < frame::GRID_MAX ? nStored - j0 : frame::GRID_MAX), pack::COPY_THREADS, 0, stream>>>(out, in, index, j0);
    return cudaGetLastError();
}

}  // namespace fseb
