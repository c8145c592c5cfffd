// frame.cu -- the device side of the .fse frame calls (include/fse_b200.h FSEB200_frame_{compress,decompress}_host{,_batch}).
//
// Frame layout (the reference's programs/fileio.c:266-285): a 5-byte frame header (LE32 magic, block-size id), then per block a
// 1-byte header { type:2 (0 compressed, 1 raw, 2 RLE), full:1, 0:5 }, then its regenerated size as 2 big-endian bytes unless it
// is full (n == blockSize), then its compressed size as 2 big-endian bytes if it is compressed, then its payload: the compressed
// bytes, the n source bytes of a raw block, or the one byte of an RLE block; then a 3-byte trailer holding 22 bits of the XXH32
// of the frame's data.
//
// Compress, per chunk of whole frames or pieces of one frame, after the device packed compress of its blocks (fse_packed.cu /
// huf_encode.cu): the payloads are already the packed stream's stored blocks, in order, so the chunk's frame bodies are that
// stream with a block header in front of each block, a frame header in front of each frame's first block and a trailer behind
// its last.  A scan of those lengths (pack_dev.cuh) gives each block's offset; one CTA per block then writes its headers, moves
// its payload from the packed buffer behind them and, for a frame whose hash xxh32_kernel computed, writes the trailer.  The
// device-memory call (frame_device.cu) lays out whole batches at once and decides per frame, between the scan and the writes,
// whether the frame is stored: a frame of an error block takes no bytes, and a frame that ends past the capacity is not written.
// Decompress, per chunk: the compressed blocks go to the descriptor decoders with pointers into the chunk's frame bytes (the host
// builds the descriptors); raw and RLE blocks come from frame_stored_kernel, one CTA per block of a compact index.
//
// xxh32_kernel hashes many byte ranges of one device buffer in one launch: the frames' data, before the compress writes the frame
// bodies over it, or the decoded output.  It is the public xxHash specification's XXH32 at seed 0, bit for bit.
#include "common.cuh"
#include "frame_walk.h"
#include "launchers.h"
#include "launch_util.cuh"
#include "pack_dev.cuh"

namespace fseb {
namespace frame {

// the packed compress's outputs for a chunk (offset: nBlocks + 1 entries) and the frame bodies they become.  role[b]: ROLE_FIRST
// if block b starts a frame, ROLE_LAST if it ends one, and ROLE_HASHED with the frame's index into hash[] in the upper 32 bits if the trailer
// is written here (otherwise the host writes it).  A block of 0 source bytes is the placeholder of an empty frame: no block
// header, no payload.
struct Body {
    const u8* packed; const u64* offset; const u64* value; const u64* srcSize; const u64* role; const u64* hash;
    u8* out; u64* bodyOff;                                          // bodyOff[b]: where block b's bytes start; scratch
    u64 blockSize; u32 nBlocks; u32 magic; u32 blockSizeId;
    // FrameStore only (else nullptr: every frame is written, and the host settles error frames): role[b] >> 32 is block b's
    // frame for every block; errBlock[f], the first block of frame f with an error value (~0: none); stored[f], frame f is written
    const u64* errBlock; const u8* stored;
};

using namespace fmt;

// frame header and trailer bytes around block b
__device__ __forceinline__ u32 frame_len(u64 role)
{
    return (u32)((role & ROLE_FIRST ? FRAME_HEADER : 0) + (role & ROLE_LAST ? FRAME_TRAILER : 0));
}

// header bytes of a block with compress value v and n source bytes; an error value stores nothing (the host reports it), and
// neither does an empty frame's placeholder
__device__ __forceinline__ u32 header_len(u64 v, u64 n, u64 blockSize)
{
    if (is_err(v) || n == 0) return 0;
    return 1 + (n == blockSize ? 0 : 2) + (v >= 2 ? 2 : 0);
}

struct Headers {
    typedef Body Geo;
    typedef u64* Aux;
    static __device__ __forceinline__ u64 value(const Body& g, u64 b) { return g.value[b]; }
    static __device__ __forceinline__ u64 len(const Body& g, u64 b, u64 v)
    {
        if (g.errBlock && g.errBlock[g.role[b] >> 32] != ~0ull) return 0;
        return frame_len(g.role[b]) + header_len(v, g.srcSize[b], g.blockSize) + (g.offset[b + 1] - g.offset[b]);
    }
    static __device__ __forceinline__ void place(const Body& g, u64*, u64 b, u64, u64 off, u64) { g.bodyOff[b] = off; }
};

// one CTA per block (blocks b0 + blockIdx.x) of a stored frame: its headers, the stored payload behind them, and the trailer of
// a frame it ends
__global__ void __launch_bounds__(pack::COPY_THREADS) frame_payload_kernel(Body g, u64 b0)
{
    u64 const b = b0 + blockIdx.x;
    u64 const v = g.value[b], role = g.role[b];
    if (g.stored && !g.stored[role >> 32]) return;
    u64 const n = g.srcSize[b];
    u32 const L = (u32)(g.offset[b + 1] - g.offset[b]);             // at most a block, 64 KB
    u32 const hl = header_len(v, n, g.blockSize);
    u8* h = g.out + g.bodyOff[b];
    u8* const at = h + (role & ROLE_FIRST ? FRAME_HEADER : 0) + hl;
    if (threadIdx.x == 0) {
        if (role & ROLE_FIRST) {
            for (int i = 0; i < 4; i++) *h++ = (u8)(g.magic >> (8 * i));
            *h++ = (u8)g.blockSizeId;
        }
        if (hl) {
            bool const full = n == g.blockSize;
            *h++ = (u8)(((v == 0 ? 1u : v == 1 ? 2u : 0u) << 6) | (full ? 0x20u : 0u));
            if (!full) { *h++ = (u8)(n >> 8); *h++ = (u8)n; }
            if (v >= 2) { *h++ = (u8)(v >> 8); *h++ = (u8)v; }
        }
    }
    if ((role & (ROLE_LAST | ROLE_HASHED)) == (ROLE_LAST | ROLE_HASHED) && threadIdx.x == 0) {
        u32 const c = ((u32)g.hash[role >> 32] >> 5) & ((1u << 22) - 1);
        at[L] = (u8)((c >> 16) | 0xC0u); at[L + 1] = (u8)(c >> 8); at[L + 2] = (u8)c;
    }
    if (is_err(v) || L == 0) return;
    pack::cta_copy<pack::COPY_THREADS, pack::COPY_UNROLL>(at, g.packed + g.offset[b], L);
}

// FrameStore: errBlock[f] = the first block of frame f whose value is an error (errBlock starts at ~0)
__global__ void frame_errors_kernel(Body g)
{
    u64 const b = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (b < g.nBlocks && is_err(g.value[b])) atomicMin(const_cast<u64*>(g.errBlock) + (g.role[b] >> 32), b);
}

// FrameStore, one thread per frame once the scan has placed every block: the frame's offset (its first block's), its length
// (up to the next frame's offset, or the total), its result and whether it is written
__global__ void frame_settle_kernel(Body g, FrameStore o, const u64* total, u8* stored)
{
    u32 const f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= o.nFrames) return;
    u64 const off = g.bodyOff[o.first[f]], end = f + 1 < o.nFrames ? g.bodyOff[o.first[f + 1]] : *total;
    u64 const e = g.errBlock[f];
    bool const fits = e == ~0ull && end <= o.capacity;
    o.offsets[f] = off;
    if (f + 1 == o.nFrames) o.offsets[o.nFrames] = end;
    o.results[f] = e != ~0ull ? g.value[e] : fits ? end - off : err(E_DST_TOO_SMALL);
    stored[f] = fits;
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

// XXH32 (seed 0) of ranges [desc[2 f], desc[2 f] + desc[2 f + 1]) of `base`, f < n, into hash[f].  Four lanes of a warp take one
// range, one lane per accumulator; a warp takes GROUPS ranges and a CTA WARPS warps.  Each round the warp stages TILE bytes of
// each of its ranges in shared memory with 16-byte cp.async copies, double-buffered so the next round's copies overlap this
// round's stripes; a round consumes STEP = TILE - 32 bytes, so the range's misalignment within its first 16 bytes, the round's
// stripes and a 15-byte tail all lie inside the tile.  The stripes are a chain of three dependent integer ops per 16 bytes per
// lane (IMAD, SHF, IMAD); the tail and the avalanche run on the range's first lane in its last round.
namespace xxh {
constexpr u32 P1 = 2654435761u, P2 = 2246822519u, P3 = 3266489917u, P4 = 668265263u, P5 = 374761393u;
constexpr int GROUPS = 8, WARPS = 2, THREADS = 32 * WARPS;
constexpr u32 TILE = 1024, STEP = TILE - 32, ROUND_STRIPES = STEP / 16, UNITS = TILE / 16;
// a group's tile sits PITCH bytes after the previous one: the 16 extra bytes put the 8 groups of a warp 4 banks apart, so the
// warp's 32 stripe words of one step fall on 32 distinct banks whenever the groups' ranges share their misalignment
constexpr u32 PITCH = TILE + 16;

__device__ __forceinline__ u32 rotl(u32 x, int r) { return __funnelshift_l(x, x, r); }
// the little-endian word at byte offset o of a staged tile: one aligned load, or the two aligned words around it
__device__ __forceinline__ u32 word_at(const u8* t, u32 o)
{
    const u32* const w = reinterpret_cast<const u32*>(t + (o & ~3u));
    return (o & 3) ? __funnelshift_r(w[0], w[1], 8 * (o & 3)) : w[0];
}
__device__ __forceinline__ void cp16(void* smem, const void* gmem)
{
    unsigned const s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
}  // namespace xxh

__global__ void __launch_bounds__(xxh::THREADS) xxh32_kernel(const u8* __restrict__ base, const u64* __restrict__ desc, u32 n,
                                                             u64* __restrict__ hash)
{
    using namespace xxh;
    __shared__ __align__(16) u8 sm[WARPS][2][GROUPS][PITCH];
    u32 const warp = threadIdx.x >> 5, lane = threadIdx.x & 31u, grp = lane >> 2, li = lane & 3u;
    u32 const f0 = (blockIdx.x * WARPS + warp) * GROUPS;
    // lane j < GROUPS holds range f0 + j; every lane gets its group's by a shuffle, and each range's bounds in the copy loop
    u64 myStart = 0, myLen = 0;
    if (lane < GROUPS && f0 + lane < n) { myStart = desc[2 * (f0 + lane)]; myLen = desc[2 * (f0 + lane) + 1]; }
    u64 const start = __shfl_sync(pack::FULL, myStart, grp), len = __shfl_sync(pack::FULL, myLen, grp);
    bool const live = f0 + grp < n;
    u64 const nS = len / 16;
    u32 const rounds = live ? (u32)(nS / ROUND_STRIPES) + 1 : 0;   // the last round also takes the tail
    u32 R = rounds;
    #pragma unroll
    for (int d = 16; d >= 1; d >>= 1) R = max(R, __shfl_xor_sync(pack::FULL, R, d));
    u32 const mis = (u32)(start & 15);

    auto stage = [&](u32 r) {
        #pragma unroll 1
        for (u32 j = 0; j < GROUPS; j++) {
            u64 const s = __shfl_sync(pack::FULL, myStart, j), e = s + __shfl_sync(pack::FULL, myLen, j);
            u64 const a = (s & ~(u64)15) + (u64)r * STEP;
            #pragma unroll
            for (u32 u = lane; u < UNITS; u += 32)
                if (f0 + j < n && a + 16 * u < e) cp16(&sm[warp][r & 1][j][16 * u], base + a + 16 * u);
        }
        asm volatile("cp.async.commit_group;\n" ::);
    };

    u32 v = li == 0 ? P1 + P2 : li == 1 ? P2 : li == 2 ? 0u : 0u - P1;
    if (R) stage(0);
    for (u32 r = 0; r < R; r++) {
        if (r + 1 < R) stage(r + 1);
        else asm volatile("cp.async.commit_group;\n" ::);
        asm volatile("cp.async.wait_group 1;\n" ::);
        __syncwarp();
        const u8* const t = sm[warp][r & 1][grp];
        u64 const s0 = (u64)r * ROUND_STRIPES;
        if (r < rounds) {
            u32 const k = (u32)min(nS - s0, (u64)ROUND_STRIPES);
            #pragma unroll 4
            for (u32 i = 0; i < k; i++) v = rotl(v + word_at(t, mis + 16 * i + 4 * li) * P2, 13) * P1;
        }
        u32 const base4 = lane & ~3u;                                 // the group's accumulators, for its merge
        u32 const a0 = __shfl_sync(pack::FULL, v, base4), a1 = __shfl_sync(pack::FULL, v, base4 + 1);
        u32 const a2 = __shfl_sync(pack::FULL, v, base4 + 2), a3 = __shfl_sync(pack::FULL, v, base4 + 3);
        if (r + 1 == rounds && li == 0) {
            u32 h = len >= 16 ? rotl(a0, 1) + rotl(a1, 7) + rotl(a2, 12) + rotl(a3, 18) : P5;
            h += (u32)len;
            u32 o = mis + 16 * (u32)(nS - s0), rem = (u32)(len & 15);
            for (; rem >= 4; rem -= 4, o += 4) h = rotl(h + word_at(t, o) * P3, 17) * P4;
            for (; rem; rem--, o++) h = rotl(h + t[o] * P5, 11) * P1;
            h ^= h >> 15; h *= P2; h ^= h >> 13; h *= P3; h ^= h >> 16;
            hash[f0 + grp] = h;
        }
        __syncwarp();
    }
    asm volatile("cp.async.wait_all;\n" ::);
}

}  // namespace frame

size_t frame_body_work(u32 nBlocks, u32 nFrames)
{
    return sizeof(u64) * ((size_t)nBlocks + pack::tiles_of(nBlocks) + 1 + nFrames) + nFrames;
}

cudaError_t launch_frame_body(u8* out, const u8* packed, const u64* offset, const u64* value, const u64* srcSize, const u64* role,
                              const u64* hash, u32 nBlocks, u64 blockSize, u32 magic, u32 blockSizeId, cudaStream_t stream,
                              const FrameStore* store)
{
    if (nBlocks == 0) return cudaSuccess;
    size_t const n = nBlocks;
    unsigned const tiles = pack::tiles_of(n);
    cudaError_t e = cudaSuccess;
    u64* const s = store ? (u64*)store->work : (u64*)stream_scratch(8, stream, frame_body_work(nBlocks, 0), &e);
    if (e != cudaSuccess) return e;
    frame::Body g;
    g.packed = packed; g.offset = offset; g.value = value; g.srcSize = srcSize;
    g.role = role; g.hash = hash; g.magic = magic; g.blockSizeId = blockSizeId;
    g.out = out; g.bodyOff = s; g.blockSize = blockSize; g.nBlocks = nBlocks;
    g.errBlock = nullptr; g.stored = nullptr;
    u64* const tileSum = s + n;                                     // tiles + 1 words: the body's length goes to the last
    if (store) {
        u64* const errBlock = tileSum + tiles + 1;
        u8* const stored = (u8*)(errBlock + store->nFrames);
        g.errBlock = errBlock; g.stored = stored;
        if ((e = cudaMemsetAsync(errBlock, 0xFF, sizeof(u64) * store->nFrames, stream)) != cudaSuccess) return e;
        frame::frame_errors_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(g);
        pack::launch_pack<frame::Headers>(g, tileSum, tileSum + tiles, nullptr, stream);
        frame::frame_settle_kernel<<<(store->nFrames + 255) / 256, 256, 0, stream>>>(g, *store, tileSum + tiles, stored);
    } else pack::launch_pack<frame::Headers>(g, tileSum, tileSum + tiles, nullptr, stream);
    pack::launch_per_block(frame::frame_payload_kernel, n, stream, g);
    return cudaGetLastError();
}

cudaError_t launch_frame_stored(u8* out, const u8* in, const u64* index, u64 nStored, cudaStream_t stream)
{
    pack::launch_per_block(frame::frame_stored_kernel, nStored, stream, out, in, index);
    return cudaGetLastError();
}

cudaError_t launch_xxh32_ranges(const u8* base, const u64* desc, u32 n, u64* hash, cudaStream_t stream)
{
    if (n == 0) return cudaSuccess;
    u32 const per = frame::xxh::GROUPS * frame::xxh::WARPS;
    frame::xxh32_kernel<<<(n + per - 1) / per, frame::xxh::THREADS, 0, stream>>>(base, desc, n, hash);
    return cudaGetLastError();
}

}  // namespace fseb
