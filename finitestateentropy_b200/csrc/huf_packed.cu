// huf_packed.cu -- the packed Huff0 decompress (include/fse_b200.h FSEB200_HUF_decompress{,1X}_packed): every block of a buffer
// FSEB200_HUF_compress{,1X}_packed wrote, located by its offsets, through the unchanged descriptor decoder of huf_decode.cu.
//
// Huff0's decoders already read a stored length equal to the block size as a raw copy and a length of 1 as RLE, so unlike FSE
// (fse_packed.cu) no block needs a path of its own.  Three steps, all on the stream:
//   1. a classify kernel derives the descriptors (source dIn + offset, size L) into stream scratch;
//   2. the descriptor decoder (pass A, pass B, the X2 verdict pass) on them;
//   3. a kernel gives an empty block (n == 0 and L == 0, what the packed compress stores for it) the result 0 -- the decoder
//      answers dstSize 0 with dstSize_tooSmall.
// It also holds the decompress of packed chains of table reuse (FSEB200_HUF_decompress{4X,1X,_mixed}_repeat_packed), below.
#include "common.cuh"
#include "launchers.h"
#include "launch_util.cuh"
#include "pack_dev.cuh"

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

// ---- packed chains of table reuse: every block of a buffer FSEB200_HUF_compress{4X,1X}_repeat_chains_packed wrote, from its
// offsets and kinds (0 raw, 1 RLE, 2 own tree header, 3 the previous table's header, anything else corrupt).  Five steps:
//   1. the chain geometry's verdict (huf_encode.cu's check kernel);
//   2. a scan over the blocks in order (pack_dev.cuh) counts the kind-2 blocks before each block and lists their positions:
//      the last kind-2 block before b is the newest one on that list whose count is not below the count at b's chain start,
//      so this plain scan stands in for a scan segmented by chain;
//   3. a resolve kernel, one thread per block, finds b's chain by binary search over the chain starts and derives the
//      header-descriptor batch: source (dIn + offset, L) and header for the Huffman kinds, and an action for the others --
//      every block the decoder must not touch gets a size above HUF_BLOCK_MAX, which it settles without reading or writing;
//   4. the header decoder of huf_decode.cu on that batch;
//   5. one CTA per block writes the raw and RLE blocks and the verdicts of the others, over what step 4 settled.
enum : u8 { ACT_DECODE = 0, ACT_RAW = 1, ACT_RLE = 2, ACT_SRC_WRONG = 3, ACT_CORRUPT = 4 };

struct HufChainUnpack {
    const u64* start; u32 nChains;
    u8* const* dst; const u64* dstSize; u64* result;
    const u8* in; const u64* offset; const u8* kind;
    const u8* const* chainHdr; const u64* chainHdrSize;
    const u32* malformed;
    u32* count;                                                     // scratch: kind-2 blocks before block b
    u32* newPos;                                                    // scratch: the positions of the kind-2 blocks, in order
    const u8** decSrc; u64* decSize; u64* decCap; const u8** hdr; u64* hdrSize; u8* act;   // scratch: the derived batch
    u32 nBlocks;
};

struct CountNew {
    typedef HufChainUnpack Geo;
    typedef u32* Aux;
    static __device__ __forceinline__ u64 value(const HufChainUnpack& g, u64 b) { return g.kind[b] == 2; }
    static __device__ __forceinline__ u64 len(const HufChainUnpack&, u64, u64 v) { return v; }
    static __device__ __forceinline__ void place(const HufChainUnpack& g, u32*, u64 b, u64 v, u64 off, u64)
    {
        g.count[b] = (u32)off;
        if (v) g.newPos[off] = (u32)b;
    }
};

__global__ void __launch_bounds__(THREADS) huf_chain_resolve_kernel(HufChainUnpack g)
{
    u64 const b = (u64)blockIdx.x * THREADS + threadIdx.x;
    if (b >= g.nBlocks) return;
    u64 const off = g.offset[b], L = g.offset[b + 1] - off, n = g.dstSize[b];
    const u8* hp = nullptr;
    u64 hs = 0;
    u8 act = ACT_CORRUPT;
    if (*g.malformed || n > HUF_BLOCK_MAX) act = ACT_SRC_WRONG;
    else switch (g.kind[b]) {
        case 0: act = L == n ? ACT_RAW : ACT_CORRUPT; break;
        case 1: act = L == 1 ? ACT_RLE : ACT_CORRUPT; break;
        case 2: act = ACT_DECODE; break;
        case 3: {
            u32 lo = 0, hi = g.nChains;                             // the chain: the last c with start[c] <= b (start[0] = 0 <= b < start[nChains])
            while (hi - lo > 1) { u32 const mid = lo + (hi - lo) / 2; if (g.start[mid] <= b) lo = mid; else hi = mid; }
            u32 const k = g.count[b];
            if (k > g.count[g.start[lo]]) {                         // a kind-2 block of this chain precedes b: the newest one
                u32 const j = g.newPos[k - 1];
                hp = g.in + g.offset[j]; hs = g.offset[j + 1] - g.offset[j];
            } else { hp = g.chainHdr[lo]; hs = g.chainHdrSize[lo]; }
            act = hs ? ACT_DECODE : ACT_CORRUPT;
            break;
        }
        default: break;
    }
    g.decSrc[b] = g.in + off; g.decSize[b] = L;
    g.decCap[b] = act == ACT_DECODE ? n : (u64)HUF_BLOCK_MAX + 1;   // the others: srcSize_wrong at once, replaced in step 5
    g.hdr[b] = hp; g.hdrSize[b] = act == ACT_DECODE ? hs : 0;
    g.act[b] = act;
}

__global__ void __launch_bounds__(pack::COPY_THREADS) huf_chain_stored_kernel(HufChainUnpack g, u64 b0)
{
    u64 const b = b0 + blockIdx.x;
    u8 const act = g.act[b];
    if (act == ACT_DECODE) return;
    u64 const n = g.dstSize[b];
    if (act == ACT_RAW) pack::cta_copy<pack::COPY_THREADS, pack::COPY_UNROLL>(g.dst[b], g.in + g.offset[b], (u32)n);
    else if (act == ACT_RLE) pack::cta_fill<false>(g.dst[b], g.in + g.offset[b], (u32)n);
    if (threadIdx.x == 0) g.result[b] = act == ACT_SRC_WRONG ? err(E_SRC_WRONG) : act == ACT_CORRUPT ? err(E_CORRUPT) : n;
}

}  // namespace hufp

cudaError_t launch_huf_decompress_repeat_packed(const u64* start, u32 nChains, u8* const* dst, const u64* dstSize, u64* result,
                                                const u8* in, const u64* offset, const u8* kind, const u8* const* chainHdr,
                                                const u64* chainHdrSize, u32 nBlocks, int nStreams, cudaStream_t stream,
                                                const u8* single)
{
    if (nBlocks == 0) return cudaSuccess;
    size_t const n = nBlocks;
    unsigned const tiles = pack::tiles_of(n);
    cudaError_t e;
    // 5 words, 2 counters and 1 action per block; tiles + 1 scan words; the geometry verdict
    size_t const words = 5 * n + (tiles + 1) + (2 * n * sizeof(u32) + n + 2 * sizeof(u32) + 7) / 8;
    u64* const s = (u64*)stream_scratch(12, stream, sizeof(u64) * words, &e);
    if (e != cudaSuccess) return e;
    hufp::HufChainUnpack g;
    g.start = start; g.nChains = nChains; g.dst = dst; g.dstSize = dstSize; g.result = result;
    g.in = in; g.offset = offset; g.kind = kind; g.chainHdr = chainHdr; g.chainHdrSize = chainHdrSize; g.nBlocks = nBlocks;
    g.decSrc = (const u8**)s; g.decSize = s + n; g.decCap = s + 2 * n; g.hdr = (const u8**)(s + 3 * n); g.hdrSize = s + 4 * n;
    u64* const tileSum = s + 5 * n;
    u32* const w = (u32*)(tileSum + tiles + 1);
    u32* const malformed = w;
    g.malformed = malformed; g.count = w + 2; g.newPos = w + 2 + n; g.act = (u8*)(w + 2 + 2 * n);
    if ((e = launch_huf_chain_check(start, nChains, nBlocks, malformed, stream)) != cudaSuccess) return e;
    pack::launch_pack<hufp::CountNew>(g, tileSum, tileSum + tiles, nullptr, stream);
    hufp::huf_chain_resolve_kernel<<<(unsigned)((n + hufp::THREADS - 1) / hufp::THREADS), hufp::THREADS, 0, stream>>>(g);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    HeaderDescs d;
    d.dst = dst; d.dstCap = g.decCap; d.result = result; d.src = g.decSrc; d.srcSize = g.decSize; d.nBlocks = nBlocks;
    d.hdr = g.hdr; d.hdrSize = g.hdrSize;
    if ((e = launch_huf_decode_headers(d, nStreams, stream, single)) != cudaSuccess) return e;
    pack::launch_per_block(hufp::huf_chain_stored_kernel, n, stream, g);
    return cudaGetLastError();
}

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
