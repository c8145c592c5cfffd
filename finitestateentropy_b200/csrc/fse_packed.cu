// fse_packed.cu -- FSE and FSE-U16 blocks back to back in one device buffer: the packed compress and decompress calls
// (include/fse_b200.h FSEB200_FSE{,U16}_{compress,decompress}_packed) around the unchanged descriptor encoders and decoders of
// fse_codec.cu.
//
// Compress.  Unlike Huff0's, an FSE block's size is known only when its chain closes the stream (enc_stream_close), so its
// bytes are staged before their offset exists: block b is coded into a staging slot of FSE_compressBound(u * n) bytes in the
// caller's workspace, which makes its value exactly the reference's at that capacity.  Four steps, all on the stream:
//   1. the slots: a scan of the bounds in block order (pack_dev.cuh) writes the staging descriptors to stream scratch.  A block
//      the batch tier's limits settle takes no slot; a block whose slot ends past workSize gets a size the route kernel answers
//      without coding it, and workSpace_tooSmall in step 3;
//   2. the descriptor encode (route kernel, CTA and warp encoders) on the staging descriptors;
//   3. a scan of the stored lengths: the offsets, the capacity rule, the RLE unit written in place;
//   4. one copy kernel: the staged bytes of a compressed block, the source of a raw one (pack::cta_copy).
// Decompress.  A classify kernel derives descriptors (source dIn + offset, size L; size 0 for a raw or RLE block, which the
// decoder settles at once without writing), the descriptor decoder runs on them, then a raw / RLE kernel writes those blocks and
// their results.
#include "common.cuh"
#include "launchers.h"
#include "launch_util.cuh"
#include "pack_dev.cuh"

namespace fseb {

namespace fsep {

// The packed compress's arguments, and its staging descriptors in stream scratch (nBlocks entries each).
struct FsePack {
    u8* out; u64 outCap; u64* offset; u64* result;
    const u8* const* src; const u64* srcSize;
    u8* work; u64 workSize;
    u8** stageDst; u64* stageCap; u64* stageSize;
    u32 nBlocks;
};
// stageSize of a block whose slot does not fit: above the batch tier's limit, so the route kernel settles it uncoded
constexpr u64 NO_ROOM = ~0ull;

// FSE_compressBound (lib/fse.h:290-292) of block b in bytes; 0 for a block the limits settle (it takes no slot)
template <bool WIDE>
__device__ __forceinline__ u64 slot_bound(const FsePack& g, u64 b)
{
    u64 const n = fse_bytes(g.srcSize[b], WIDE);
    if ((WIDE && (reinterpret_cast<u64>(g.src[b]) & 1)) || n > FSE_BLOCK_MAX) return 0;
    return 512 + n + (n >> 7) + 4 + 8;
}

// step 1: staging slots, laid out in block order
template <bool WIDE> struct StageSlots {
    typedef FsePack Geo;
    typedef u64* Aux;
    static __device__ __forceinline__ u64 value(const FsePack& g, u64 b) { return slot_bound<WIDE>(g, b); }
    static __device__ __forceinline__ u64 len(const FsePack&, u64, u64 v) { return v; }
    static __device__ __forceinline__ void place(const FsePack& g, u64*, u64 b, u64 v, u64 off, u64)
    {
        bool const fits = v && off + v <= g.workSize;
        g.stageDst[b] = fits ? g.work + off : nullptr;
        g.stageCap[b] = fits ? v : 0;
        g.stageSize[b] = (v && !fits) ? NO_ROOM : g.srcSize[b];
    }
};

// bytes a block takes in the packed output, from its compress value (u = 2 for U16): the compressed size, the unit of an RLE
// block, a raw copy of the source for 0, nothing for an error
template <bool WIDE>
__device__ __forceinline__ u64 fse_packed_len(u64 v, u64 n)
{
    if (is_err(v)) return 0;
    if (v == 0) return WIDE ? 2 * n : n;                            // a value of 0 means n is within the limits
    if (v == 1) return WIDE ? 2 : 1;
    return v;
}

// step 3: offsets, the workspace and capacity verdicts, the RLE unit
template <bool WIDE> struct PackedBlocks {
    typedef FsePack Geo;
    typedef u64* Aux;
    static __device__ __forceinline__ u64 value(const FsePack& g, u64 b) { return g.result[b]; }
    static __device__ __forceinline__ u64 len(const FsePack& g, u64 b, u64 v) { return fse_packed_len<WIDE>(v, g.srcSize[b]); }
    static __device__ __forceinline__ void place(const FsePack& g, u64*, u64 b, u64 v, u64 off, u64 len)
    {
        g.offset[b] = off;
        if (g.stageSize[b] != g.srcSize[b]) g.result[b] = err(E_WKSP_TOO_SMALL);      // its slot did not fit: not coded, len 0
        else if (!is_err(v) && off + len > g.outCap) g.result[b] = err(E_DST_TOO_SMALL);
        else if (v == 1) {
            const u8* const s = g.src[b];
            g.out[off] = s[0];
            if (WIDE) g.out[off + 1] = s[1];
        }
    }
};

// step 4, one CTA per block (blocks b0 + blockIdx.x): the staged bytes of a compressed block, the source of a raw one
template <bool WIDE>
__global__ void __launch_bounds__(pack::COPY_THREADS)
fse_pack_copy_kernel(FsePack g, u64 b0)
{
    u64 const b = b0 + blockIdx.x;
    u64 const v = g.result[b];
    if (is_err(v) || v == 1) return;                                // errors store nothing; RLE units are placed already
    u32 const n = v ? (u32)v : (u32)(WIDE ? 2 * g.srcSize[b] : g.srcSize[b]);   // both at most FSE_compressBound(2^30)
    if (n == 0) return;
    pack::cta_copy<pack::COPY_THREADS, pack::COPY_UNROLL>(g.out + g.offset[b], v ? g.stageDst[b] : g.src[b], n);
}

// ---- decompress ----
struct FseUnpack {
    const u8* in; const u64* offset;
    u8* const* dst; const u64* dstSize; u64* result;
    const u8** decSrc; u64* decSize;                                // the derived descriptors, in stream scratch
    u32 nBlocks;
};
enum { DECODE = 0, RAW = 1, RLE = 2 };

// how block b is regenerated: the decoder's limit and alignment verdicts first (dec_desc_verdict: it gets L and answers them),
// then L == u * n is a raw copy, L == u an RLE block, anything else is decoded
template <bool WIDE>
__device__ __forceinline__ int stored_kind(const FseUnpack& g, u64 b, u64 L)
{
    if (WIDE && (reinterpret_cast<u64>(g.dst[b]) & 1)) return DECODE;
    u64 const nb = fse_bytes(g.dstSize[b], WIDE);
    if (L > FSE_BLOCK_MAX || nb > FSE_BLOCK_MAX) return DECODE;
    if (L == nb) return RAW;
    return L == (WIDE ? 2u : 1u) ? RLE : DECODE;
}

constexpr int CLASSIFY_THREADS = 256;
template <bool WIDE>
__global__ void __launch_bounds__(CLASSIFY_THREADS) fse_unpack_classify_kernel(FseUnpack g)
{
    u64 const b = (u64)blockIdx.x * CLASSIFY_THREADS + threadIdx.x;
    if (b >= g.nBlocks) return;
    u64 const off = g.offset[b], L = g.offset[b + 1] - off;
    g.decSrc[b] = g.in + off;
    g.decSize[b] = stored_kind<WIDE>(g, b, L) == DECODE ? L : 0;
}

// after the decoder, one CTA per block (blocks b0 + blockIdx.x): raw and RLE blocks and their results
template <bool WIDE>
__global__ void __launch_bounds__(pack::COPY_THREADS)
fse_unpack_stored_kernel(FseUnpack g, u64 b0)
{
    u64 const b = b0 + blockIdx.x;
    u64 const off = g.offset[b];
    int const kind = stored_kind<WIDE>(g, b, g.offset[b + 1] - off);
    if (kind == DECODE) return;
    u64 const n = g.dstSize[b];
    u32 const nb = (u32)(WIDE ? 2 * n : n);                         // at most 2^30
    if (kind == RAW) pack::cta_copy<pack::COPY_THREADS, pack::COPY_UNROLL>(g.dst[b], g.in + off, nb);
    else pack::cta_fill<WIDE>(g.dst[b], g.in + off, nb);
    if (threadIdx.x == 0) g.result[b] = n;
}

template <bool WIDE>
cudaError_t compress_packed(FsePack g, unsigned msv, unsigned tlog, cudaStream_t stream)
{
    size_t const n = g.nBlocks;
    unsigned const tiles = pack::tiles_of(n);
    cudaError_t e;
    u8* const s = (u8*)stream_scratch(5, stream, 3 * sizeof(u64) * n + sizeof(u64) * (tiles + 1), &e);
    if (e != cudaSuccess) return e;
    g.stageDst = (u8**)s; g.stageCap = (u64*)(s + 8 * n); g.stageSize = (u64*)(s + 16 * n);
    u64* const tileSum = (u64*)(s + 24 * n);                        // tiles + 1 words: the slots' total goes to the last
    // 1. staging slots
    pack::launch_pack<StageSlots<WIDE>>(g, tileSum, tileSum + tiles, nullptr, stream);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    // 2. the descriptor encode into the slots
    BlockDescs st;
    st.dst = g.stageDst; st.dstCap = g.stageCap; st.result = g.result; st.src = g.src; st.srcSize = g.stageSize; st.nBlocks = g.nBlocks;
    if ((e = launch_fse_encode_blocks(st, WIDE, msv, tlog, stream)) != cudaSuccess) return e;
    // 3. offsets and verdicts
    pack::launch_pack<PackedBlocks<WIDE>>(g, tileSum, g.offset + n, nullptr, stream);
    // 4. the bytes
    pack::launch_per_block(fse_pack_copy_kernel<WIDE>, n, stream, g);
    return cudaGetLastError();
}

template <bool WIDE>
cudaError_t decompress_packed(FseUnpack g, cudaStream_t stream)
{
    size_t const n = g.nBlocks;
    cudaError_t e;
    u8* const s = (u8*)stream_scratch(6, stream, 2 * sizeof(u64) * n, &e);
    if (e != cudaSuccess) return e;
    g.decSrc = (const u8**)s; g.decSize = (u64*)(s + 8 * n);
    fse_unpack_classify_kernel<WIDE><<<(unsigned)((n + CLASSIFY_THREADS - 1) / CLASSIFY_THREADS), CLASSIFY_THREADS, 0, stream>>>(g);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    BlockDescs d;
    d.dst = g.dst; d.dstCap = g.dstSize; d.result = g.result; d.src = g.decSrc; d.srcSize = g.decSize; d.nBlocks = g.nBlocks;
    if ((e = launch_fse_decode_blocks(d, WIDE, stream)) != cudaSuccess) return e;
    pack::launch_per_block(fse_unpack_stored_kernel<WIDE>, n, stream, g);
    return cudaGetLastError();
}

}  // namespace fsep

cudaError_t launch_fse_compress_packed(u8* out, u64 outCap, u64* offset, u64* result, const u8* const* src, const u64* srcSize,
                                       u32 nBlocks, u8* work, u64 workSize, bool wide, unsigned msv, unsigned tlog, cudaStream_t stream)
{
    if (nBlocks == 0) return cudaSuccess;
    fsep::FsePack g;
    g.out = out; g.outCap = outCap; g.offset = offset; g.result = result; g.src = src; g.srcSize = srcSize;
    g.work = work; g.workSize = workSize; g.stageDst = nullptr; g.stageCap = nullptr; g.stageSize = nullptr; g.nBlocks = nBlocks;
    return wide ? fsep::compress_packed<true>(g, msv, tlog, stream) : fsep::compress_packed<false>(g, msv, tlog, stream);
}

cudaError_t launch_fse_decompress_packed(u8* const* dst, const u64* dstSize, u64* result, const u8* in, const u64* offset,
                                         u32 nBlocks, bool wide, cudaStream_t stream)
{
    if (nBlocks == 0) return cudaSuccess;
    fsep::FseUnpack g;
    g.in = in; g.offset = offset; g.dst = dst; g.dstSize = dstSize; g.result = result;
    g.decSrc = nullptr; g.decSize = nullptr; g.nBlocks = nBlocks;
    return wide ? fsep::decompress_packed<true>(g, stream) : fsep::decompress_packed<false>(g, stream);
}

}  // namespace fseb
