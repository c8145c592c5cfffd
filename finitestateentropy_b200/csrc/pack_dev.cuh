// pack_dev.cuh -- placing variable-length blocks back to back in one device buffer, shared by the packed calls of both codecs
// (huf_encode.cu: Huff0 compress; fse_packed.cu: FSE / FSE-U16 compress and decompress) and the .fse frame calls (frame.cu).
//
// Offsets: a device-wide exclusive scan of per-block lengths, reduce-then-scan over tiles of PACK_TILE blocks -- the tiles'
// sums (pack_sums_kernel), their exclusive scan from 0 in one CTA (pack_scan_tiles_kernel), then the scan inside each tile,
// handing every block its offset (pack_place_kernel) -- in u64, so totals above 2^32 and batches of up to 2^32 - 1 blocks are
// exact.  What is scanned and what happens at the offsets is the caller's, through a placement P:
//   P::Geo                                 the kernels' argument (it has nBlocks); P::Aux a pointer the place step may use
//   P::value(g, b)                         the per-block word the length derives from (read once per block by the place step)
//   P::len(g, b, v)                        the bytes block b takes
//   P::place(g, aux, b, v, off, len)       what the place step does for block b at offset off
// Copies: cta_copy, one CTA moving one block with 16-byte aligned destination stores; cta_fill, one CTA writing a run of one unit.
#pragma once
#include "common.cuh"

namespace fseb {
namespace pack {

constexpr unsigned FULL = 0xFFFFFFFFu;
constexpr int PACK_THREADS = 256, PACK_ITEMS = 8, PACK_SCAN_THREADS = 1024, COPY_THREADS = 256, COPY_UNROLL = 4;
constexpr u32 PACK_TILE = PACK_THREADS * PACK_ITEMS;

// exclusive prefix of v over the CTA's NT threads in `excl`; returns the CTA's total.  sm: NT / 32 + 1 words.
template <int NT>
__device__ __forceinline__ u64 cta_exclusive_scan(u64 v, u64& excl, u64* sm)
{
    static_assert(NT % 32 == 0 && NT <= 1024, "one warp scans the warp totals");
    unsigned const lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    u64 incl = v;
    #pragma unroll
    for (int d = 1; d < 32; d <<= 1) { u64 const t = __shfl_up_sync(FULL, incl, d); if (lane >= (unsigned)d) incl += t; }
    if (lane == 31) sm[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        u64 const w = lane < NT / 32 ? sm[lane] : 0;
        u64 wi = w;
        #pragma unroll
        for (int d = 1; d < 32; d <<= 1) { u64 const t = __shfl_up_sync(FULL, wi, d); if (lane >= (unsigned)d) wi += t; }
        if (lane < NT / 32) sm[lane] = wi - w;
        if (lane == NT / 32 - 1) sm[NT / 32] = wi;
    }
    __syncthreads();
    excl = sm[warp] + incl - v;
    u64 const total = sm[NT / 32];
    __syncthreads();                                                // sm is free for the next call
    return total;
}

// step 1: the length of each tile of blocks
template <class P>
__global__ void __launch_bounds__(PACK_THREADS)
pack_sums_kernel(typename P::Geo g, u64* __restrict__ tileSum)
{
    __shared__ u64 sm[PACK_THREADS / 32 + 1];
    u64 const first = (u64)blockIdx.x * PACK_TILE + threadIdx.x * PACK_ITEMS;
    u64 s = 0;
    #pragma unroll
    for (int i = 0; i < PACK_ITEMS; i++) { u64 const b = first + i; if (b < g.nBlocks) s += P::len(g, b, P::value(g, b)); }
    u64 excl;
    u64 const t = cta_exclusive_scan<PACK_THREADS>(s, excl, sm);
    if (threadIdx.x == 0) tileSum[blockIdx.x] = t;
}

// step 2, one CTA: tile sums -> tile offsets (in place), from 0; the grand total goes to *totalOut
static __global__ void __launch_bounds__(PACK_SCAN_THREADS)
pack_scan_tiles_kernel(u64* __restrict__ tileSum, u32 nTiles, u64* __restrict__ totalOut)
{
    __shared__ u64 sm[PACK_SCAN_THREADS / 32 + 1];
    u64 run = 0;
    for (u32 t0 = 0; t0 < nTiles; t0 += PACK_SCAN_THREADS) {
        u32 const t = t0 + threadIdx.x;
        u64 const v = t < nTiles ? tileSum[t] : 0;
        u64 excl;
        u64 const tot = cta_exclusive_scan<PACK_SCAN_THREADS>(v, excl, sm);
        if (t < nTiles) tileSum[t] = run + excl;
        run += tot;
    }
    if (threadIdx.x == 0) *totalOut = run;
}

// step 3: offsets inside each tile, and P::place at each
template <class P>
__global__ void __launch_bounds__(PACK_THREADS)
pack_place_kernel(typename P::Geo g, const u64* __restrict__ tileOff, typename P::Aux __restrict__ aux)
{
    __shared__ u64 sm[PACK_THREADS / 32 + 1];
    u64 const first = (u64)blockIdx.x * PACK_TILE + threadIdx.x * PACK_ITEMS;
    u64 v[PACK_ITEMS], len[PACK_ITEMS], s = 0;
    #pragma unroll
    for (int i = 0; i < PACK_ITEMS; i++) {
        u64 const b = first + i;
        bool const in = b < g.nBlocks;
        v[i] = in ? P::value(g, b) : 0;
        len[i] = in ? P::len(g, b, v[i]) : 0;
        s += len[i];
    }
    u64 excl;
    cta_exclusive_scan<PACK_THREADS>(s, excl, sm);
    u64 off = tileOff[blockIdx.x] + excl;
    #pragma unroll
    for (int i = 0; i < PACK_ITEMS; i++) {
        u64 const b = first + i;
        if (b >= g.nBlocks) break;
        P::place(g, aux, b, v[i], off, len[i]);
        off += len[i];
    }
}

inline unsigned tiles_of(u64 n) { return (unsigned)((n + PACK_TILE - 1) / PACK_TILE); }
// the three steps for P; tileSum: tiles_of(g.nBlocks) words; the total goes to *totalOut
template <class P>
void launch_pack(const typename P::Geo& g, u64* tileSum, u64* totalOut, typename P::Aux aux, cudaStream_t stream)
{
    unsigned const tiles = tiles_of(g.nBlocks);
    pack_sums_kernel<P><<<tiles, PACK_THREADS, 0, stream>>>(g, tileSum);
    pack_scan_tiles_kernel<<<1, PACK_SCAN_THREADS, 0, stream>>>(tileSum, tiles, totalOut);
    pack_place_kernel<P><<<tiles, PACK_THREADS, 0, stream>>>(g, tileSum, aux);
}

// kernel(args..., b0), one CTA of COPY_THREADS per block b0 + blockIdx.x of [0, n), in launches of at most GRID_MAX CTAs
constexpr u64 GRID_MAX = 1ull << 30;
template <class... K, class... A>
void launch_per_block(void (*kernel)(K...), u64 n, cudaStream_t stream, A... args)
{
    for (u64 b0 = 0; b0 < n; b0 += GRID_MAX)
        kernel<<<(unsigned)(n - b0 < GRID_MAX ? n - b0 : GRID_MAX), COPY_THREADS, 0, stream>>>(args..., b0);
}

// n bytes from s to d by the NT threads of one CTA (n < 2^32; any alignment of either).  The destination's 16-byte aligned
// interior is written in whole 16-byte stores, the bytes before and after it one by one.  Every interior chunk's source bytes
// sit at the same misalignment sh in the source, so they are the bytes [sh, sh + 16) of two consecutive aligned 16-byte source
// pieces: a lane loads one piece, takes the next from its neighbour lane, and funnel-shifts the pair.  A piece is loaded only if
// it holds a byte of the source.  Every thread of the CTA must call it (the loop is CTA-uniform).
template <int NT, int UNROLL>
__device__ __forceinline__ void cta_copy(u8* const d, const u8* const s, u32 const n)
{
    u32 const tid = threadIdx.x, lane = tid & 31u;
    u32 const head = min((u32)(-reinterpret_cast<u64>(d) & 15), n);
    u32 const nChunks = (n - head) / 16, tailBeg = head + 16 * nChunks;
    if (tid < head) d[tid] = s[tid];
    if (tid < n - tailBeg) d[tailBeg + tid] = s[tailBeg + tid];
    u64 const sa = reinterpret_cast<u64>(s) + head;                 // source of chunk 0
    u32 const sh = (u32)(sa & 15), q = sh >> 2, r = 8 * (sh & 3);
    const uint4* const sp = reinterpret_cast<const uint4*>(sa - sh);    // chunk k: pieces k and k + 1 (k alone when sh == 0)
    uint4* const dp = reinterpret_cast<uint4*>(d + head);
    u32 const lastPiece = nChunks - (sh == 0);                      // pieces [0, lastPiece] hold source bytes (none if nChunks == 0)
    auto ld = [&](u32 k) { return (nChunks && k <= lastPiece) ? __ldg(sp + k) : make_uint4(0, 0, 0, 0); };
    #pragma unroll 1
    for (u32 k0 = 0; k0 < nChunks; k0 += NT * UNROLL) {             // CTA-uniform: every lane takes part in the shuffles
        uint4 a[UNROLL], c[UNROLL];
        #pragma unroll
        for (int j = 0; j < UNROLL; j++) {
            u32 const k = k0 + j * NT + tid;
            a[j] = ld(k);
            c[j] = (lane == 31 && sh) ? ld(k + 1) : make_uint4(0, 0, 0, 0);
        }
        #pragma unroll
        for (int j = 0; j < UNROLL; j++) {
            u32 const k = k0 + j * NT + tid;
            uint4 nx;
            nx.x = __shfl_down_sync(FULL, a[j].x, 1); nx.y = __shfl_down_sync(FULL, a[j].y, 1);
            nx.z = __shfl_down_sync(FULL, a[j].z, 1); nx.w = __shfl_down_sync(FULL, a[j].w, 1);
            if (lane == 31) nx = c[j];
            if (k >= nChunks) continue;
            u32 const x[8] = { a[j].x, a[j].y, a[j].z, a[j].w, nx.x, nx.y, nx.z, nx.w };
            u32 y[5];
            #pragma unroll
            for (int i = 0; i < 5; i++) y[i] = q == 0 ? x[i] : q == 1 ? x[i + 1] : q == 2 ? x[i + 2] : x[i + 3];
            dp[k] = make_uint4(__funnelshift_r(y[0], y[1], r), __funnelshift_r(y[1], y[2], r),
                               __funnelshift_r(y[2], y[3], r), __funnelshift_r(y[3], y[4], r));
        }
    }
}

// nb bytes of copies of the unit at s (1 byte; WIDE: 2 bytes, d even) to d by the CTA: 16-byte stores in the aligned interior
template <bool WIDE>
__device__ __forceinline__ void cta_fill(u8* const d, const u8* const s, u32 const nb)
{
    u32 const w = WIDE ? ((u32)s[0] | (u32)s[1] << 8) * 0x10001u : (u32)s[0] * 0x01010101u;
    u32 const head = min((u32)(-reinterpret_cast<u64>(d) & 15), nb);   // even for U16: the pattern stays in phase
    u32 const nChunks = (nb - head) / 16, tailBeg = head + 16 * nChunks;
    for (u32 i = threadIdx.x; i < head; i += blockDim.x) d[i] = (u8)(w >> (8 * (i & 3)));
    for (u32 i = tailBeg + threadIdx.x; i < nb; i += blockDim.x) d[i] = (u8)(w >> (8 * (i & 3)));
    uint4* const dp = reinterpret_cast<uint4*>(d + head);
    for (u32 k = threadIdx.x; k < nChunks; k += blockDim.x) dp[k] = make_uint4(w, w, w, w);
}

}  // namespace pack
}  // namespace fseb
