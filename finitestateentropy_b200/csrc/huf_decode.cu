// huf_decode.cu -- batched Huff0 4-stream decode for sm_90a (HBM-bound integer path, no tensor cores).
//
// Replaces, for a whole batch of independent blocks, the CPU chain
//   HUF_decompress            lib/huf_decompress.c:1056-1081  (raw / RLE / decoder choice)
//   HUF_readStats             lib/entropy_common.c:154-215
//   HUF_readDTableX1          lib/huf_decompress.c:118-185
//   HUF_decompress4X1_usingDTable_internal_body  lib/huf_decompress.c:262-354
// Decoded bytes are those of both CPU decoders (they agree on every valid stream); the error verdict produced here is
// the single-symbol (X1) decoder's.  Where the reference would have run its double-symbol decoder
// (HUF_selectDecoder, lib/huf_decompress.c:1029-1051) and this kernel rejects a stream, huf_x2_fixup.cu re-runs the
// block under the exact X2 end-of-stream rules (a stream accepted here is accepted by X2 with the same bytes).
//
// H100 mapping ("lane per stream, table column per bank"):
//   * one CTA = 64 consecutive blocks = 256 streams = 256 threads; a warp holds the SAME stream index of 32
//     DIFFERENT blocks (the even or the odd columns), so the 32 look-ups of a warp instruction hit 32 tables;
//   * ONE unified u16 table per block, column-interleaved tbl[row][64]: rows [0, CUT) hold full-resolution cells
//     (indexed by the top tableLog bits of the window) for the few windows that start a code longer than M bits
//     (Huff0 numbers the longest codes from 0, so these are exactly the windows below a per-block threshold),
//     rows >= CUT hold the M-bit first-level table minus its never-used head.  The row of window value x is
//         min(x, D + (x >> (tableLog - M))),   D = CUT - (CUT >> (tableLog - M))
//     -- one IMNMX instead of a compare/select, and the split M is chosen PER BLOCK to minimise the rows
//     (P14: M = 7, 283 rows; the round-1 layout needed 704).  306 rows of 128 B + an 8 KB stream ring + 1.25 KB of
//     per-block facts + 8 KB of output staging = 55.5 KB per CTA: FOUR CTAs (1024 lanes = 256 blocks) in the 228 KB of an SM, so the 248
//     blocks per SM of a 1 GiB batch on 132 SMs decode in one round;
//   * bit window: the lane keeps three raw 32-bit stream words w0..w2 and a bit offset r < 32; the 64-bit window is
//     recomputed from (w0,w1,w2) by two funnel shifts after every PAIR of symbols, and when r crosses 32 the words
//     rotate (predicated moves) and the next word is fetched from the lane's private shared-memory ring.  No
//     running 64-bit shift, no merge, 2 funnel shifts + 1 test per pair instead of round 1's 14-instruction refill;
//   * stream ring: 8 words per lane, word-interleaved ring[slot][tid] (bank = lane: conflict-free for any 32
//     cursors).  The lane tops it up itself with one 16-byte global load per 4 words, issued one top-up ahead into
//     registers (the load is in flight across ~16 symbols of work, nothing waits on it);
//   * output: 32 symbols are packed into one whole 32-byte sector per lane; the warp stages its 32 sectors in shared memory and
//     writes them transposed, 16 whole sectors per store instruction;
//   * blocks whose best table exceeds the row budget ("hard", e.g. near-flat 256-symbol alphabets), unaligned
//     segments and ragged tails take a per-symbol loop (canonical-code search for hard blocks).
// Single-stream blocks (HUF_decompress1X_DCtx, huf_decompress.c:1141-1176; descriptor batches only) run the same kernel with
// NS = 1: one lane per block column, 64 lanes = 2 warps per CTA (still the even or the odd columns per warp), no jump table;
// the table, ring, fast loop, head, tail, passes and the X2 verdict pass are those of the 4X form (DESIGN.md 4.1).
#include "common.cuh"
#include "launchers.h"
#include "huf_dev.cuh"
#include "launch_util.cuh"
#include <cstdlib>
#include <type_traits>

namespace fseb {
namespace hufd {

#ifndef FSEB200_HUFD_HEAD
#define FSEB200_HUFD_HEAD 1       // 0: descriptor batches decode misaligned segments per symbol (a build for measuring the head decode)
#endif

constexpr int G = 64;             // block columns per CTA
constexpr int THREADS = 4 * G;    // one lane per stream (4X)
constexpr int NWARPS = THREADS / 32;
constexpr int RW = 8;             // ring words per lane
constexpr u32 RING_BYTES = RW * THREADS * 4;
// The kernel's shape for NS streams per block: 4X = G columns x 4 lanes (8 warps), 1X = G columns x 1 lane (2 warps).
__host__ __device__ constexpr int threads_for(int ns) { return ns * G; }
__host__ __device__ constexpr u32 ring_bytes(int ns) { return RW * threads_for(ns) * 4; }
constexpr u32 NOERR = 0xFFFFFFFFu;
constexpr unsigned FULL = 0xFFFFFFFFu;
constexpr u32 MIN_ROWS = 160;     // a hard block parks its canonical-code arrays in 156 rows of its own column
constexpr u32 PARK_RANKEND = 128, PARK_LISTSTART = 142;
// HeaderDescs: a block's compressed size is not bounded by its dstSize there.  A stream longer than HDR_STREAM_MAX bytes can never
// be consumed exactly (at most 12 bits for each of <= 128 K symbols), so after its BIT_initDStream checks it gets the reference's
// end-of-stream verdict, corruption_detected, without being decoded; every other stream's bit count then fits 32 bits.
constexpr u64 HDR_STREAM_MAX = 1ull << 20;

struct __align__(16) Facts {      // per-CTA facts about its 64 block columns (1.25 KB)
    u32 bid[G];                   // batch index of the block in this column (NOBLOCK = empty column)
    u32 status[G];                // NOERR or (stage<<8 | error code), smallest wins
    u32 hsize[G];                 // tree-header bytes
    u16 dOff[G];                  // D of the row formula
    u16 cut[G];
    u8  tlog[G];
    u8  mbits[G];                 // M; == tlog for a main-only table
    u8  kind[G];                  // 0 = Huffman, 1 = raw copy, 2 = RLE, 3 = done/skip
    u8  hard[G];
};
template <int NW>
struct BuildScratchT {            // lives in the (not yet used) stream ring while tables are built, one set per warp
    u8  weights[NW][256];
    u8  sorted[NW][256];          // symbols in code order: weight ascending, symbol ascending
    u32 rankStats[NW][HUF_MAX_TLOG + 1];
    u16 rankRun[NW][HUF_MAX_TLOG + 2];
    u16 rankEnd[NW][HUF_MAX_TLOG + 2];         // end (exclusive) of weight w's range in tableLog-bit index space
    u16 listStart[NW][HUF_MAX_TLOG + 2];       // first position of weight w in the sorted symbol list
};
typedef BuildScratchT<NWARPS> BuildScratch;
static_assert(sizeof(BuildScratch) <= RING_BYTES, "build scratch must fit in the ring");
static_assert(sizeof(BuildScratchT<threads_for(1) / 32>) <= ring_bytes(1), "build scratch must fit in the 1X ring");
static_assert(sizeof(Facts) == 1280, "Facts layout");
constexpr u32 NOBLOCK = 0xFFFFFFFFu;

constexpr u32 STAGE_WARP_BYTES = 32 * 32;    // one 32-byte output sector per lane, staged for the warp's transposed store
__host__ __device__ constexpr u32 smem_bytes(u32 rows, bool staged, int ns = 4)
{
    return rows * (G * 2) + ring_bytes(ns) + (u32)sizeof(Facts) + (staged ? (u32)(threads_for(ns) / 32) * STAGE_WARP_BYTES : 0u);
}

__device__ __forceinline__ u32 lds_u16(u32 addr) { u16 v; asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(addr)); return v; }
__device__ __forceinline__ u32 lds_u32(u32 addr) { u32 v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr)); return v; }
__device__ __forceinline__ void sts_u32(u32 addr, u32 v) { asm volatile("st.shared.u32 [%0], %1;" :: "r"(addr), "r"(v) : "memory"); }

// symbols a stream decodes one at a time before its output position reaches a 32-byte boundary (descriptor batches)
__device__ __forceinline__ u32 head_symbols(const u8* outp) { return (u32)(0ull - reinterpret_cast<u64>(outp)) & 31u; }

// canonical-code look-up in tableLog-bit index space -> (nbBits | symbol << 8)
__device__ __forceinline__ u32 canon_cell(const u16* rankEnd, const u16* listStart, const u8* sorted, u32 idx, u32 tl)
{
    u32 w = 1;
    while (idx >= rankEnd[w]) w++;
    u32 const first = (w == 1) ? 0u : rankEnd[w - 1];
    u32 const k = listStart[w] + ((idx - first) >> (w - 1));
    return (tl + 1 - w) | ((u32)sorted[k] << 8);
}

// HUF_readStats (lib/entropy_common.c:158-215) with the whole warp: same verdicts as d_huf_read_stats.  The raw 4-bit form and
// the per-weight statistics are spread over the lanes (they were 7 % of this kernel's instructions on one lane); the
// FSE-compressed form (a serial 2-state decode of <= 255 weights) stays on lane 0.  All lanes return the same value.
__device__ u64 warp_huf_read_stats(u8* weights, u32* rankStats, u32* nbSymPtr, u32* tlPtr, const u8* in, u64 srcSize, unsigned lane)
{
    if (!srcSize) return err(E_SRC_WRONG);
    u64 iSize = in[0], oSize;
    if (iSize >= 128) {                                   // raw 4-bit weights (:167-177)
        oSize = iSize - 127;
        iSize = (oSize + 1) / 2;
        if (iSize + 1 > srcSize) return err(E_SRC_WRONG);
        if (oSize >= 256) return err(E_CORRUPT);
        for (u32 k = lane; k < (u32)iSize; k += 32) { u8 const v = in[1 + k]; weights[2 * k] = v >> 4; weights[2 * k + 1] = v & 15; }
    } else {                                              // FSE-compressed weights (:178-183)
        if (iSize + 1 > srcSize) return err(E_SRC_WRONG);
        oSize = 0;
        if (lane == 0) oSize = d_huf_read_weights_fse(weights, 256, in, iSize);
        oSize = __shfl_sync(FULL, oSize, 0);
        if (is_err(oSize)) return oSize;
    }
    if (lane <= HUF_MAX_TLOG) rankStats[lane] = 0;
    __syncwarp();
    u32 total = 0; bool bad = false;
    for (u32 n = lane; n < (u32)oSize; n += 32) {
        u32 const w = weights[n];
        if (w >= HUF_MAX_TLOG) bad = true;
        else { atomicAdd(&rankStats[w], 1u); total += (1u << w) >> 1; }
    }
    if (__any_sync(FULL, bad)) return err(E_CORRUPT);
    #pragma unroll
    for (int d = 16; d; d >>= 1) total += __shfl_xor_sync(FULL, total, d);
    if (total == 0) return err(E_CORRUPT);
    u32 const tl = hibit(total) + 1;
    if (tl > HUF_MAX_TLOG) return err(E_CORRUPT);
    u32 const rest = (1u << tl) - total;
    u32 const lastW = hibit(rest) + 1;
    if ((1u << hibit(rest)) != rest) return err(E_CORRUPT);
    __syncwarp();
    if (lane == 0) { weights[oSize] = (u8)lastW; rankStats[lastW]++; }
    __syncwarp();
    if ((rankStats[1] < 2) || (rankStats[1] & 1)) return err(E_CORRUPT);
    *tlPtr = tl;
    *nbSymPtr = (u32)(oSize + 1);
    return iSize + 1;
}

// Builds the unified table of block column `blk` with one warp.  EXT: the header is not the start of the block (HUF_readDTableX1
// on a caller's header, `csize` its bound): no hSize < cSize test, and the payload starts at the block's first byte.
template <bool EXT = false, class BS>
__device__ void setup_block(u16* tbl, Facts& fx, BS& bs, u32 rows, int blk, const u8* csrc, u64 csize, int warp)
{
    unsigned const lane = lane_id();
    u8* const weights = bs.weights[warp];
    u8* const sorted = bs.sorted[warp];
    u16* const rankEnd = bs.rankEnd[warp];
    u16* const listStart = bs.listStart[warp];
    u32 nbSym = 0, tl = 0, M = 0, cut = 0, nRows = 0;
    u64 h = warp_huf_read_stats(weights, bs.rankStats[warp], &nbSym, &tl, csrc, csize, lane);
    if (lane == 0) {
        if (!is_err(h) && tl > HUF_MAX_TLOG) h = err(E_TLOG_TOO_LARGE);      // huf_decompress.c:143
        if (!EXT && !is_err(h) && h >= csize) h = err(E_SRC_WRONG);           // huf_decompress.c:426
        if (!is_err(h)) {
            // rank ranges (huf_decompress.c:151-156): weight w covers 2^(w-1) cells per symbol, longest codes first
            u32 acc = 0, pos = 0;
            rankEnd[0] = 0; listStart[0] = 0;
            for (u32 w = 1; w <= tl; w++) {
                listStart[w] = (u16)pos; bs.rankRun[warp][w] = (u16)pos;
                pos += bs.rankStats[warp][w];
                acc += bs.rankStats[warp][w] << (w - 1);
                rankEnd[w] = (u16)(acc > 0xFFFF ? 0xFFFF : acc);
            }
            rankEnd[tl] = (u16)(1u << tl);
            rankEnd[tl + 1] = 0xFFFF;
            // split choice: first level of m bits + full resolution below CUT; rows = CUT + 2^m - CUT / 2^(tl-m)
            M = tl; cut = 0; nRows = 1u << tl;                                 // main-only
            for (u32 m = (tl > 10 ? 10 : tl - 1); m >= 4 && m < tl; m--) {
                u32 const g = 1u << (tl - m);
                u32 const T = rankEnd[tl - m];                                 // windows that start a code longer than m bits
                u32 const c = (T + g - 1) & ~(g - 1);
                u32 const r = c + (1u << m) - (c >> (tl - m));
                if (r < nRows) { nRows = r; M = m; cut = c; }
            }
            fx.hard[blk] = (u8)(nRows > rows);
            fx.tlog[blk] = (u8)tl;
            fx.mbits[blk] = (u8)M;
            fx.cut[blk] = (u16)cut;
            fx.dOff[blk] = (u16)(M < tl ? cut - (cut >> (tl - M)) : 0);
            fx.hsize[blk] = EXT ? 0u : (u32)h;
        } else {
            atomicMin(&fx.status[blk], (u32)(0u << 8 | (u32)(0 - h)));
        }
    }
    h = __shfl_sync(FULL, h, 0);
    if (is_err(h)) return;
    M = __shfl_sync(FULL, M, 0); cut = __shfl_sync(FULL, cut, 0); nRows = __shfl_sync(FULL, nRows, 0);
    __syncwarp();
    // sorted symbol list: stable by weight, then symbol order (huf_decompress.c:158-183 fills cells in that order)
    for (u32 base = 0; base < nbSym; base += 32) {
        u32 const s = base + lane;
        u32 const w = (s < nbSym) ? weights[s] : 0u;
        u32 const peers = __match_any_sync(FULL, w);
        if (w) sorted[bs.rankRun[warp][w] + __popc(peers & ((1u << lane) - 1))] = (u8)s;
        __syncwarp();
        if (w && (peers >> lane) == 1u) bs.rankRun[warp][w] = (u16)(bs.rankRun[warp][w] + __popc(peers));   // highest lane of the group
        __syncwarp();
    }
    u16* const col = tbl + blk;
    if (nRows <= rows) {
        u32 const D = (M < tl) ? cut - (cut >> (tl - M)) : 0u;
        for (u32 row = lane; row < nRows; row += 32) {
            u32 const x = (row < cut || M == tl) ? row : ((row - D) << (tl - M));
            col[row * G] = (u16)canon_cell(rankEnd, listStart, sorted, x, tl);
        }
    } else {   // hard block: park the code-ordered symbol list (2 per cell) and the rank arrays in the column
        for (u32 r = lane; r < 128; r += 32) col[r * G] = (u16)(sorted[2 * r] | (sorted[2 * r + 1] << 8));
        if (lane < HUF_MAX_TLOG + 2) { col[(PARK_RANKEND + lane) * G] = rankEnd[lane]; col[(PARK_LISTSTART + lane) * G] = listStart[lane]; }
    }
    __syncwarp();
}

// NS = streams per block: 4 (HUF_decompress, 4X) or 1 (HUF_decompress1X_DCtx, descriptor batches only).  4X: a lane per
// (column, stream), 8 warps.  1X: a lane per column, i.e. per block, 2 warps; five CTAs per SM at the pass-A budget.
template <bool PASS_A, class Geo, int NS>
__global__ void __launch_bounds__(NS * G, NS == 4 ? 4 : 5)
huf_decode_kernel(Geo g, u8* __restrict__ dst, const u8* __restrict__ cbuf, const u64* __restrict__ csizes,
                  u64* __restrict__ results, const u8* __restrict__ orig, u32 flags, u32 gEff, u32 rows,
                  const u32* __restrict__ list, const u32* __restrict__ listCount, u32* __restrict__ deferList, u32* __restrict__ deferCount)
{
    static_assert(NS == 4 || NS == 1, "4X or 1X");
    constexpr int NT = threads_for(NS);              // threads per CTA (THREADS for 4X)
    constexpr int NW = NT / 32;
    constexpr u32 RB = ring_bytes(NS);
    // Two passes share this kernel (PASS_A is true exactly when list == nullptr).
    // Pass A walks the batch in order with the four-CTAs-per-SM table budget; a
    // block whose smallest table does not fit that budget is not decoded but appended to deferList.  Pass B (deferList == nullptr)
    // walks that list with a larger budget (fewer CTAs per SM); what does not fit even there takes the per-symbol path.
    extern __shared__ __align__(16) unsigned char smem_raw[];
    // The ring comes first: its address is then (compile-time base) + an offset the hot loop builds with one OR.
    unsigned char* const ringRaw = smem_raw;
    BuildScratchT<NW>& bs = *reinterpret_cast<BuildScratchT<NW>*>(ringRaw);
    Facts& fx = *reinterpret_cast<Facts*>(ringRaw + RB);
    u16* const tbl = reinterpret_cast<u16*>(smem_raw + RB + sizeof(Facts));            // [rows][G]
    int const tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    u32 const blk0 = blockIdx.x * gEff;
    u32 const nWork = list ? *listCount : g.nBlocks;
    if (blk0 >= nWork) return;                                              // pass B is launched for the worst case: most CTAs find nothing
    u32 const blkEnd = min(blk0 + gEff, nWork);                             // this CTA owns work items [blk0, blkEnd)

    if (tid < G) { fx.bid[tid] = (blk0 + tid < blkEnd) ? (list ? list[blk0 + tid] : blk0 + tid) : NOBLOCK; fx.status[tid] = NOERR; fx.kind[tid] = 3; fx.hsize[tid] = 0; fx.tlog[tid] = 0; fx.mbits[tid] = 0; fx.cut[tid] = 0; fx.dOff[tid] = 0; fx.hard[tid] = 0; }
    __syncthreads();

    // ---- classify blocks and build tables: warp w handles columns w, w+NW, ... ----
    for (int j = warp; j < G; j += NW) {
        u32 const b = fx.bid[j];
        if (b == NOBLOCK) continue;                                     // warp-uniform
        u64 const n = dec_len(g, b);
        u64 const cs = dec_csize(g, csizes, b);
        int kind;
        if constexpr (std::is_same_v<Geo, HeaderDescs>) {              // HUF_decompress{4X,1X}1_DCtx or readDTableX1 + usingDTable: always Huffman
            if (n > HUF_BLOCK_MAX) { kind = 3; if (lane == 0) dec_out(g, results, b) = err(E_SRC_WRONG); }
            else kind = 0;
        } else if constexpr (!Geo::DESCS) {
            if (flags & 1u) kind = 0;                                  // HUF_decompress4X1 / 4X2 semantics: always a Huffman block
            else if (is_err(cs)) { kind = 3; if (lane == 0) results[b] = cs; }   // propagated compressor error
            else if (cs == 0) { kind = orig ? 1 : 3; if (lane == 0) results[b] = orig ? n : 0; }   // stored raw by the harness (bench.c:393-397)
            else if (n == 0) { kind = 3; if (lane == 0) results[b] = err(E_DST_TOO_SMALL); }        // huf_decompress.c:1063
            else if (cs > n) { kind = 3; if (lane == 0) results[b] = err(E_CORRUPT); }              // :1064
            else if (cs == n) kind = 1;                                                                // :1065
            else if (cs == 1) kind = 2;                                                                // :1066
            else kind = 0;
        } else {                                                        // HUF_decompress on the literal sizes, the library's limit first
            if (n == 0) { kind = 3; if (lane == 0) dec_out(g, results, b) = err(E_DST_TOO_SMALL); }             // huf_decompress.c:1063
            else if (n > HUF_BLOCK_MAX) { kind = 3; if (lane == 0) dec_out(g, results, b) = err(E_SRC_WRONG); } // capi.cu HUF_decompress
            else if (cs > n) { kind = 3; if (lane == 0) dec_out(g, results, b) = err(E_CORRUPT); }              // :1064
            else if (cs == n) kind = 1;                                                                            // :1065
            else if (cs == 1) kind = 2;                                                                            // :1066
            else kind = 0;
        }
        if (lane == 0) fx.kind[j] = (u8)kind;
        if (kind == 0) {
            if constexpr (std::is_same_v<Geo, HeaderDescs>) {
                u64 const hb = g.hdrSize[b];
                if (hb) setup_block<true>(tbl, fx, bs, rows, j, g.hdr[b], hb, warp);
                else setup_block(tbl, fx, bs, rows, j, dec_src(g, cbuf, b), cs, warp);
            } else setup_block(tbl, fx, bs, rows, j, dec_src(g, cbuf, b), cs, warp);
            if (deferList && fx.hard[j] && fx.status[j] == NOERR) {     // pass A: hand the block to the pass with the larger table budget
                if (lane == 0) { deferList[atomicAdd(deferCount, 1u)] = b; fx.kind[j] = 3; }
            }
        }
    }
    __syncthreads();                                  // tables and facts complete; the build scratch (ring) is free now

    // ---- per-lane stream set-up: thread -> (block column, stream); 1X: thread -> block column ----
    int const col = 2 * lane + (NS == 4 ? warp >> 2 : warp);   // a warp sees the 32 even (or odd) columns = 32 distinct banks
    int const strm = (NS == 4) ? warp & 3 : 0;
    u32 const b = fx.bid[col];
    bool const live = (b != NOBLOCK) && fx.kind[col] == 0 && fx.status[col] == NOERR;
    u32 const n = live ? dec_len(g, b) : 0;
    u32 const seg = (NS == 4) ? (n + 3) / 4 : n;
    u32 segLen = 0;                                  // symbols this lane must produce
    u8* outp = (Geo::DESCS && !live) ? nullptr : dec_dst(g, dst, b) + (u64)strm * seg;   // an empty column has no descriptor to read
    const u8* blockStart = nullptr;                  // the block's compressed bytes (the feeder's lower limit, dec_floor)
    u64 chunkTop = 0;                                // address just above chunk 0
    u32 expectBits = 0;                              // stream bits between chunkTop and the first byte of the stream
    u32 c0 = 0;                                      // bits to skip at the top of chunk 0: garbage above the stream + zero padding + end mark
    u32 const tl = fx.tlog[col];

    if (live) {
        const u8* const cs0 = dec_src(g, cbuf, b);
        u64 const cs = dec_csize(g, csizes, b);
        blockStart = cs0;
        const u8* const pay = cs0 + fx.hsize[col];
        u64 const psize = cs - fx.hsize[col];
        u32 code = 0;
        constexpr bool HDR = std::is_same_v<Geo, HeaderDescs>;
        bool tooLong = false;                        // HDR: a stream no decode can consume exactly (stage 5 verdict)
        if constexpr (NS == 4) {
            if (psize < 10) code = E_CORRUPT;                                            // huf_decompress.c:268
            else if (3 * seg > n) code = E_CORRUPT;                                      // dst too small for 4 segments (documented deviation, see DESIGN.md)
            else {
                u32 const l1 = rd16(pay), l2 = rd16(pay + 2), l3 = rd16(pay + 4);
                if ((u64)l1 + l2 + l3 + 6 > psize) code = E_CORRUPT;                     // :302 length4 overflow
                else {
                    u32 const l4 = (u32)(psize - 6 - l1 - l2 - l3);
                    u32 const off = 6 + (strm > 0 ? l1 : 0) + (strm > 1 ? l2 : 0) + (strm > 2 ? l3 : 0);
                    u32 const len = strm == 0 ? l1 : strm == 1 ? l2 : strm == 2 ? l3 : l4;
                    u64 const len64 = (HDR && strm == 3) ? psize - 6 - l1 - l2 - l3 : len;   // HDR: stream 4 may pass 2^32
                    if (HDR ? len64 < 1 : len < 1) code = E_SRC_WRONG;                   // BIT_initDStream, bitstream.h:274
                    else {
                        u8 const last = HDR ? pay[off + len64 - 1] : pay[off + len - 1];
                        if (last == 0) code = (HDR ? len64 >= 8 : len >= 8) ? E_GENERIC : E_CORRUPT;   // :282-284 / :303-306
                        else if (HDR && len64 > HDR_STREAM_MAX) tooLong = true;
                        else {
                            u64 const sBegin = (u64)(pay + off);
                            u64 const e = sBegin + len;                                  // one past the last byte
                            chunkTop = ((e - 1) & ~31ull) + 32;
                            c0 = (u32)(8 * (chunkTop - e)) + (8 - hibit(last));
                            expectBits = (u32)(8 * (chunkTop - sBegin));
                            segLen = (strm < 3) ? seg : n - 3 * seg;
                        }
                    }
                }
            }
        } else if (HDR && (psize < 1 || psize > HDR_STREAM_MAX)) {   // 1X, HDR: an external header leaves any payload size
            if (psize < 1) code = E_SRC_WRONG;                                           // BIT_initDStream, bitstream.h:274
            else if (pay[psize - 1] == 0) code = E_GENERIC;                              // bitstream.h:282-284 (psize >= 8)
            else tooLong = true;
        } else {                                     // 1X: one stream, the whole payload (huf_decompress.c:240-260, :722-747)
            u32 const len = (u32)psize;              // >= 1: setup_block rejected hSize >= cSize; < 128 KB: cSize < dstSize
            u8 const last = pay[len - 1];
            if (last == 0) code = (len >= 8) ? E_GENERIC : E_CORRUPT;                // bitstream.h:282-284 / :303-306
            else {
                u64 const sBegin = (u64)pay;
                u64 const e = sBegin + len;
                chunkTop = ((e - 1) & ~31ull) + 32;
                c0 = (u32)(8 * (chunkTop - e)) + (8 - hibit(last));
                expectBits = (u32)(8 * (chunkTop - sBegin));                        // < 8 * (128 KB + 32) bits
                segLen = n;
            }
        }
        if (code) atomicMin(&fx.status[col], (u32)((1u + strm) << 8 | code));
        if (tooLong) atomicMin(&fx.status[col], (u32)(5u << 8 | E_CORRUPT));     // behind every stream's init verdict, as :348-349
    }
    __syncthreads();                                  // init verdicts of all four streams are in
    bool const go = live && fx.status[col] == NOERR;
    if (!go) segLen = 0;

    // ---- stream feeder ----
    // Stream word j (j = 0 is the word just below chunkTop) is the little-endian u32 at chunkTop - 4(j+1); chunk q = words
    // 4q..4q+3 = one aligned 16 bytes.  Below the first byte of the stream the feeder delivers whatever lies there (the
    // previous stream, the jump table, the header): the reference pads with zeros instead, but those bits can only be
    // CONSUMED by a stream that is already over-read -- a code that straddles the stream start decodes, under any padding,
    // to a length beyond the bits that are left (prefix property) -- so the verdict "consumed == stream bits" is the same,
    // and a rejected block's bytes are not part of the contract.  That keeps the hot loop to ONE unconditional 16-byte load:
    // with a second, conditional load path inlined next to it, ptxas shared a scoreboard slot between the two and every
    // 16 symbols the window shift waited a DRAM round trip for a load it does not depend on.
    // Chunks that would lie below the compressed buffer itself (for descriptors: below the block's own first 32-byte sector)
    // re-read its first sector (address clamp, never dereferenced out of bounds).
    u32 const ringLane = (u32)__cvta_generic_to_shared(ringRaw) + tid * 4;      // + slot * (NT*4)
    // Chunks are fetched a PAIR at a time: one whole 32-byte sector, as two back-to-back 16-byte loads (sm_90 has no
    // 32-byte LDG).  The pair waits in eight registers; its two chunks enter the ring one after the other.
    u32 pLimit;                                      // last pair at or above the buffer start (descriptors: the block's first sector)
    if constexpr (Geo::DESCS) pLimit = go ? (u32)((chunkTop - dec_floor(g, cbuf, blockStart)) >> 5) - 1u : 0u;
    else pLimit = go ? (u32)((chunkTop - (reinterpret_cast<u64>(cbuf) & ~31ull)) >> 5) - 1u : 0u;
    u32 m0 = 0, m1 = 0, m2 = 0, m3 = 0, m4 = 0, m5 = 0, m6 = 0, m7 = 0;        // pending pair, memory order (m7 = highest address = first consumed)
    // L2 residency (pass A): all 131,072 streams of a 1 GiB batch are in flight at once and a lane takes ~50 us to use up a
    // 128-byte input line, so the live lines of the batch (one input + one partial output line per lane, 32 MiB) come close to
    // the 50 MB L2.  The accesses therefore say which lines are dead: the pair that finishes an input line (its lowest address:
    // the lane reads downward) is read evict_first.  The cache policy of an LDG is a UNIFORM operand on sm_90 (ptxas reads one
    // lane's register, it does not loop), so a per-lane choice of policy register would give the whole warp one arbitrary lane's
    // choice.  Instead both forms are issued under complementary per-lane predicates, each with a constant policy.
    // Pass B (two CTAs per SM, the live set is half as large) is a separate instantiation that keeps plain loads and the
    // one-sector prefetch.
    constexpr bool staged = PASS_A;
    auto load_pair = [&](u32 pr) {
        u64 const a = chunkTop - 32ull * (min(pr, pLimit) + 1);
        if (!staged) {
            asm volatile("ld.global.nc.v4.b32 {%0, %1, %2, %3}, [%8];\n\t"
                         "ld.global.nc.v4.b32 {%4, %5, %6, %7}, [%8+16];"
                         : "=r"(m0), "=r"(m1), "=r"(m2), "=r"(m3), "=r"(m4), "=r"(m5), "=r"(m6), "=r"(m7) : "l"(a));
            // ... and the L2 is asked for the sector two pairs further down the stream: the demand load above was itself
            // announced that way, so it is an L2 hit by now.
            asm volatile("prefetch.global.L2 [%0];" :: "l"(chunkTop - 32ull * (min(pr + 2, pLimit) + 1)));
            return;
        }
        u32 const dead = (a & 127) == 0;
        asm volatile("{\n\t.reg .pred p;\n\t.reg .b64 pol;\n\tsetp.ne.u32 p, %9, 0;\n\t"
                     "createpolicy.fractional.L2::evict_first.b64 pol, 1.0;\n\t"
                     "@p ld.global.nc.L2::cache_hint.v4.b32 {%0, %1, %2, %3}, [%8], pol;\n\t"
                     "@p ld.global.nc.L2::cache_hint.v4.b32 {%4, %5, %6, %7}, [%8+16], pol;\n\t"
                     "@!p ld.global.nc.v4.b32 {%0, %1, %2, %3}, [%8];\n\t"
                     "@!p ld.global.nc.v4.b32 {%4, %5, %6, %7}, [%8+16];\n\t}"
                     : "=r"(m0), "=r"(m1), "=r"(m2), "=r"(m3), "=r"(m4), "=r"(m5), "=r"(m6), "=r"(m7) : "l"(a), "r"(dead));
        {
            // ... and when this pair is the first one of its line (highest address), the whole line two lines further down the
            // stream is brought into the L2 by one bulk prefetch, ahead of the demand loads that use it.  Its address is a uniform
            // operand too, and here ptxas does loop over the issuing lanes (R2UR + UBLKPF + a BRA.U.ANY back edge).  Only lines
            // that lie wholly at or above the buffer's first pair are prefetched (pair pr + 11 is the lowest pair of that line).
            if ((a & 127) == 96 && pr + 11 <= pLimit) asm volatile("cp.async.bulk.prefetch.L2.global [%0], 128;" :: "l"(a - 352));
        }
    };

    u32 w0 = 0, w1 = 0, w2 = 0, r = 0;               // raw stream words: the window starts at bit r of w0 and spans w0..w2
    u32 kBase = 0;                                    // absolute index of the next stream word to fetch = kBase + (r >> 5): `r` is never reduced
    u32 q = 0;                                        // next chunk to enter the ring (chunks 0..q-1 are consumed or in it); chunk q -> slots (4q..4q+3) mod 8
    auto store_next = [&]() {                         // chunk q out of the pending pair; an odd q uses the pair up: fetch the next one
        u32 const a = ringLane + (q & 1) * (4 * NT * 4);
        bool const lowHalf = (q & 1) != 0;
        sts_u32(a, lowHalf ? m3 : m7); sts_u32(a + NT * 4, lowHalf ? m2 : m6);
        sts_u32(a + 2 * NT * 4, lowHalf ? m1 : m5); sts_u32(a + 3 * NT * 4, lowHalf ? m0 : m4);
        q++;
        if (!(q & 1)) load_pair(q >> 1);
    };
    // Words written but not yet fetched: U = 4q - (absolute index of the next word to fetch).  The ring is topped up at two
    // kinds of check, 8 symbols (at most 3 fetched words) apart: the group-start check stores the next chunk when U <= 4, the
    // mid-group check only when U <= 3.  Induction: U >= 5 after a group-start check, hence >= 2 at the mid-group one and
    // >= 4 after it, hence >= 1 at the next group start -- U stays in [1, 8] at every check, so it is recoverable from the
    // slot numbers alone, and the ring never runs dry whatever the code lengths.  On typical data only the group-start
    // check stores, so a load has 16 symbols of work to land before the next store of this WARP touches its registers (the
    // scoreboard is per warp, not per lane: a store every 8 symbols exposed the latency).
    auto unread = [&]() -> u32 { return 4 * q - kBase - (r >> 5); };
    auto top_up = [&](u32 threshold) { if (unread() <= threshold) store_next(); };

    if (go) {                                         // the first pair fills the ring, the window words come out of it
        u32 const k0 = c0 >> 5;                       // first word of the window: 0..8
        r = c0 & 31;
        q = 2 * (k0 >> 3);
        load_pair(q >> 1);
        store_next(); store_next();                   // ring full: words 4q-8 .. 4q-1; the next pair is on its way
        kBase = k0;
        auto fetch_word = [&]() -> u32 {              // word kBase lives in slot kBase & 7
            u32 const v = lds_u32(ringLane + (kBase & 7) * (NT * 4));
            kBase++;
            if (!(kBase & 7)) store_next();           // wrapped to slot 0 = everything fetched: the next chunk goes there
            return v;
        };
        w0 = fetch_word(); w1 = fetch_word(); w2 = fetch_word();
        top_up(4);                                    // bring the ring to >= 5 unread words
    }

    // ---- decode ----
    u32 const tblCol = (u32)__cvta_generic_to_shared(tbl) + col * 2;       // + row * 128
    u32 const M = fx.mbits[col];
    u32 const shX = 32 - (tl ? tl : 1);                // window >> shX = index at full resolution
    u32 const shY = 32 - (M ? M : 1);                // umulhi(window, mulY) = window >> (32 - M) = first-level index
    int const dOff = (int)fx.dOff[col];
    u32 const tblColD = tblCol + (u32)dOff * (G * 2);  // row = min(x - D, y) + D: the "+ D" lives in the base address
    bool const hardBlk = fx.hard[col] != 0;

    // slot stride S = NT * 4 (4X: 1024, 1X: 256): (r >> 5) * S = (r * (S / 32)) minus (r & 31) * (S / 32) < S, which the slot mask drops
    static_assert(NT * 4 % 32 == 0 && (NT * 4 & (NT * 4 - 1)) == 0, "slot stride: a power of two, a multiple of 32");
    u32 const tid4 = tid * 4;
    u32 const ringBase = (u32)__cvta_generic_to_shared(ringRaw);
    u32 const slotBias = kBase * (NT * 4);             // (kBase + (r >> 5)) * S, masked to the 8 slots: the low bits of r * (S / 32) fall to the mask
    u32 hi = __funnelshift_l(w1, w0, r), lo = __funnelshift_l(w2, w1, r);
    // Row of the window: min(x, D + y) = min(x - D, y) + D, as a signed minimum.  Plain shifts: a high multiply for one of them
    // (to move work from the busy ALU pipe to the FMA pipe) was slower: IMAD.HI throttled
    // that pipe outright (measured before the H100 port, not re-measured).
#define HUFD_LOOKUP(E, H) do { \
        int const a_ = (int)((H) >> shX) - dOff; \
        int const y_ = (int)((H) >> shY); \
        E = lds_u16((u32)min(a_, y_) * (G * 2) + tblColD); \
    } while (0)
    // After a pair of symbols: `r` has grown by their bits (it is never reduced: the funnel shifts take it modulo 32 and
    // bit 5 FLIPS exactly when a 32-bit word has been used up -- a pair is at most 24 bits).  Then the words rotate and the
    // next one comes out of the ring, all predicated; the window is recomputed from the raw words either way.  The slot of that
    // next word follows from `r` itself -- word kBase + (r >> 5), slot = index mod 8 -- as one multiply-add (FMA pipe) and one
    // AND-OR with the lane's column offset; the ring sits at the start of shared memory, so its base is an immediate of the load.
    // `r` must stay a clean bit count for that: the pair's two lengths are added by one byte-wise dot product of the packed
    // cells (len0 | sym0 << 8 | len1 << 16 | sym1 << 24) with 0x00010001 -- also on the FMA pipe.
#define HUFD_ADVANCE(PACKED) do { \
        u32 const rOld_ = r; \
        r = __dp4a((u32)(PACKED), 0x00010001u, r); \
        u32 const ra_ = ((rOld_ * (NT * 4 / 32u) + slotBias) & ((RW - 1) * NT * 4)) | tid4; \
        asm volatile("{\n\t.reg .pred p;\n\t.reg .b32 t;\n\t" \
                     "xor.b32 t, %4, %5;\n\tand.b32 t, t, 32;\n\tsetp.ne.u32 p, t, 0;\n\t" \
                     "@p mov.b32 %0, %1;\n\t@p mov.b32 %1, %2;\n\t@p ld.shared.u32 %2, [%3];\n\t}" \
                     : "+r"(w0), "+r"(w1), "+r"(w2) : "r"(ringBase + ra_), "r"(r), "r"(rOld_) : "memory"); \
        hi = __funnelshift_l(w1, w0, r); lo = __funnelshift_l(w2, w1, r); \
    } while (0)

    u32 pos = 0;
    // 32 symbols -> one whole 32-byte sector per lane.  Every lane writes its own stream, so a lane's own stores cannot coalesce
    // with its neighbours'; on sm_90 (no 32-byte STG) a lane writing its sector as two 16-byte stores costs 2.63 ms per GiB on
    // this access pattern alone (scripts/ubench/scatter.cu, H100).  So the warp stages its 32 sectors in shared memory and writes
    // them transposed: each 16-byte store of a lane is half of some lane's sector, and one warp instruction writes 16 whole
    // sectors (0.45 ms per GiB in the same benchmark).  Lanes leave the fast path at different trip counts: the loop runs the
    // warp's longest count and a finished lane only takes part in the transposed stores.  Pass B has no room for the staging
    // (its larger table budget keeps the near-flat alphabets off the per-symbol path): its lanes write their sectors directly.
    // Descriptor batches: a segment of seg = ceil(n / 4) bytes starts on a 32-byte boundary for about one stream in four, so a
    // lane whose segment start is misaligned first decodes the (-outp) & 31 symbols up to the next boundary one at a time
    // ("head", topped up like the tail loop) and then enters the fast loop there.  Hard blocks and segments with less than one
    // sector after the head stay on the per-symbol path.  The uniform geometry keeps its aligned-segments-only rule.
    constexpr bool withHead = Geo::DESCS && FSEB200_HUFD_HEAD;
    bool const fastOk = withHead ? go && !hardBlk && segLen >= head_symbols(outp) + 32u
                                 : go && !hardBlk && ((reinterpret_cast<u64>(outp) & 31) == 0);
    u32 const headN = (withHead && fastOk) ? head_symbols(outp) : 0u;
    if constexpr (withHead) {
        for (u32 i = 0; i < headN; i++) {            // <= 8 symbols (<= 3 words) between checks, as in the tail loop: the fast
            if ((i & 7) == 0) top_up(4);             // loop's first group-start check still finds 1 <= unread <= 8
            u32 e;
            HUFD_LOOKUP(e, hi);
            HUFD_ADVANCE(e);
            outp[pos++] = (u8)(e >> 8);
        }
    }
    u32 const nIter = fastOk ? (segLen - headN) >> 5 : 0u;
    u32 const nIterW = __reduce_max_sync(FULL, nIter);
    u32 const stageW = (u32)__cvta_generic_to_shared(tbl) + rows * (G * 2) + (u32)warp * STAGE_WARP_BYTES;
    for (u32 it = 0; it < nIterW; it++) {
        bool const act = it < nIter;
        u32 o[8];
        if (act) {
            #pragma unroll
            for (int h = 0; h < 8; h++) {
                if ((h & 3) == 0) top_up(4);                                     // group start: the common store
                else if ((h & 3) == 2 && __builtin_expect(__any_sync(__activemask(), unread() <= 3), 0)) top_up(3);   // mid-group: only when a lane ran low (vote among the lanes still decoding)
                u32 e0, e1, e2, e3, hi1;
                HUFD_LOOKUP(e0, hi); hi1 = __funnelshift_l(lo, hi, e0); HUFD_LOOKUP(e1, hi1);
                u32 const p01 = e0 | (e1 << 16);
                HUFD_ADVANCE(p01);
                HUFD_LOOKUP(e2, hi); hi1 = __funnelshift_l(lo, hi, e2); HUFD_LOOKUP(e3, hi1);
                u32 const p23 = e2 | (e3 << 16);
                HUFD_ADVANCE(p23);
                o[h] = __byte_perm(p01, p23, 0x7531);
            }
        }
        if (!staged) {
            if (act)
                asm volatile("st.global.v4.b32 [%0], {%1, %2, %3, %4};\n\tst.global.v4.b32 [%0+16], {%5, %6, %7, %8};"
                             :: "l"(outp + pos), "r"(o[0]), "r"(o[1]), "r"(o[2]), "r"(o[3]), "r"(o[4]), "r"(o[5]), "r"(o[6]), "r"(o[7]) : "memory");
            if (act) pos += 32;
            continue;
        }
        if (act)
            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};\n\tst.shared.v4.b32 [%0+16], {%5, %6, %7, %8};"
                         :: "r"(stageW + (u32)lane * 32), "r"(o[0]), "r"(o[1]), "r"(o[2]), "r"(o[3]), "r"(o[4]), "r"(o[5]), "r"(o[6]), "r"(o[7]) : "memory");
        __syncwarp();
        u64 const dstHere = reinterpret_cast<u64>(outp + pos);
        // Output line hints: the store that completes a 128-byte line (the lane writes upward: the sector at offset 96) is
        // evict_first; the stores before it are evict_last, so the L2 prefers to keep a partly written line until it is whole
        // rather than write it to DRAM in pieces (DESIGN 4.1 has the measurements; DRAM traffic itself was not measured).  A line
        // this loop will not finish (ragged tails, unaligned segments) is written evict_first throughout, so no line is left
        // evict_last.  As for the loads, the policy is chosen by per-lane predicates over two stores with constant policies.
        // Pass B (direct stores) runs at half the occupancy and keeps the default policy.
        u32 const o32 = (u32)dstHere - pos;                                      // low bits of outp
        bool const lineDone = ((((o32 + pos) | 127u) + 1u) - o32) <= headN + nIter * 32u;   // the fast path finishes this sector's line
        u32 const flags = (act ? 1u : 0u) | (lineDone ? 2u : 0u);
        #pragma unroll
        for (int k = 0; k < 2; k++) {                                            // lanes 2j, 2j+1 write the two halves of lane 16k + j's sector
            int const src = k * 16 + (lane >> 1);
            u32 const half = (u32)(lane & 1) * 16;
            u64 const q = __shfl_sync(FULL, dstHere, src);
            u32 const srcFlags = __shfl_sync(FULL, flags, src);
            u32 x0, x1, x2, x3;
            asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(x0), "=r"(x1), "=r"(x2), "=r"(x3) : "r"(stageW + (u32)src * 32 + half));
            u32 const keep = (srcFlags & 2u) && ((q + half) & 127) < 96;
            if (srcFlags & 1u)
                asm volatile("{\n\t.reg .pred p;\n\t.reg .b64 pl, pf;\n\tsetp.ne.u32 p, %5, 0;\n\t"
                             "createpolicy.fractional.L2::evict_last.b64 pl, 1.0;\n\t"
                             "createpolicy.fractional.L2::evict_first.b64 pf, 1.0;\n\t"
                             "@p st.global.L2::cache_hint.v4.b32 [%0], {%1, %2, %3, %4}, pl;\n\t"
                             "@!p st.global.L2::cache_hint.v4.b32 [%0], {%1, %2, %3, %4}, pf;\n\t}"
                             :: "l"(q + half), "r"(x0), "r"(x1), "r"(x2), "r"(x3), "r"(keep) : "memory");
        }
        __syncwarp();
        if (act) pos += 32;
    }
    // ragged tails, unaligned segments and hard blocks: one symbol at a time
    if (pos < segLen) {
        const u16* const colp = tbl + col;
        auto parked_cell = [&](u32 idx) -> u32 {
            u32 w = 1;
            while (idx >= colp[(PARK_RANKEND + w) * G]) w++;
            u32 const first = (w == 1) ? 0u : colp[(PARK_RANKEND + w - 1) * G];
            u32 const k = colp[(PARK_LISTSTART + w) * G] + ((idx - first) >> (w - 1));
            return (tl + 1 - w) | (((colp[(k >> 1) * G] >> (8 * (k & 1))) & 0xFFu) << 8);
        };
        u32 cnt = 0;
        while (pos < segLen) {
            if ((cnt++ & 7) == 0) top_up(4);
            u32 e;
            if (hardBlk) e = parked_cell(hi >> (32 - tl));
            else HUFD_LOOKUP(e, hi);
            HUFD_ADVANCE(e);
            outp[pos++] = (u8)(e >> 8);
        }
    }
#undef HUFD_LOOKUP
#undef HUFD_ADVANCE

    // ---- verdict: every stream must be consumed exactly (huf_decompress.c:348-349) ----
    if (go) {
        u64 const fetched = 4ull * q - unread();                        // absolute index of the next word to fetch; w0 is word fetched-3
        u64 const consumed = 32ull * (fetched - 3) + (r & 31);
        if (consumed != (u64)expectBits) atomicMin(&fx.status[col], (u32)(5u << 8 | E_CORRUPT));
    }
    __syncthreads();
    if (tid < G) {
        u32 const bb = fx.bid[tid];
        if (bb != NOBLOCK && fx.kind[tid] == 0) {
            u32 const st = fx.status[tid];
            u64 rv = (st == NOERR) ? (u64)dec_len(g, bb) : err(st & 0xFF);
            // Rejected only by the exact-consumption rule of the single-symbol decoder: where the reference would have run
            // its double-symbol decoder (always for HUF_decompress4X2, by HUF_selectDecoder for HUF_decompress) the verdict
            // is the second pass's (huf_x2_fixup.cu).
            if ((st >> 8) == 5u && ((flags & 2u) || (!(flags & 1u) && d_huf_select_decoder(dec_len(g, bb), dec_csize(g, csizes, bb))))) rv = HUF_X2_PENDING;
            dec_out(g, results, bb) = rv;
        }
    }
    // ---- raw / RLE blocks (huf_decompress.c:1065-1066; the harness' own 0-size convention, bench.c:393-402) ----
    for (int j = 0; j < G; j++) {
        int const kd = fx.kind[j];
        if (kd != 1 && kd != 2) continue;
        u32 const bb = fx.bid[j];
        u32 const nn = dec_len(g, bb);
        u64 const cs = dec_csize(g, csizes, bb);
        u8* const o = dec_dst(g, dst, bb);
        if (kd == 2) { u8 const v = dec_src(g, cbuf, bb)[0]; for (u32 i = tid; i < nn; i += NT) o[i] = v; }
        else {
            const u8* const s = (cs == 0) ? dec_orig(g, orig, bb) : dec_src(g, cbuf, bb);    // cs == 0 is never raw for descriptors
            for (u32 i = tid; i < nn; i += NT) o[i] = s[i];
        }
        if (tid == 0) dec_out(g, results, bb) = nn;
    }
}

// ---- mixed forms (single[b]: 0 4X, else 1X): the header decoder runs once per form over the same batch.  Each launch sees the other
// form's blocks with a size above HUF_BLOCK_MAX, which it settles as srcSize_wrong without reading or writing a byte; the 1X launch
// writes its verdicts to scratch, and the merge takes them for the 1X blocks.
constexpr int FORM_THREADS = 256;
struct HufMixedSplit {
    const u64* dstCap; const u8* single; u64* cap4; u64* cap1; const u64* res1; u64* result;
    u32 nBlocks;
};

__global__ void __launch_bounds__(FORM_THREADS) huf_mixed_split_kernel(HufMixedSplit g)
{
    u64 const b = (u64)blockIdx.x * FORM_THREADS + threadIdx.x;
    if (b >= g.nBlocks) return;
    u64 const n = g.dstCap[b], none = (u64)HUF_BLOCK_MAX + 1;
    bool const one = g.single[b] != 0;
    g.cap4[b] = one ? none : n;
    g.cap1[b] = one ? n : none;
}

__global__ void __launch_bounds__(FORM_THREADS) huf_mixed_merge_kernel(HufMixedSplit g)
{
    u64 const b = (u64)blockIdx.x * FORM_THREADS + threadIdx.x;
    if (b >= g.nBlocks) return;
    if (g.single[b]) g.result[b] = g.res1[b];
}

}  // namespace hufd

namespace {

// flags: bit 0 = every block is a Huffman block (HUF_decompress4X1 / 4X2 semantics: no raw / RLE forms);
//        bit 1 = verdicts of the double-symbol decoder for every block (HUF_decompress4X2);
//        0     = HUF_decompress: raw / RLE forms, decoder (and hence verdict on malformed input) by HUF_selectDecoder.
// NS = streams per block (1: HUF_decompress1X_DCtx, descriptors only: BlockDescs with flags 0, HeaderDescs with flags 1).
template <class Geo, int NS>
cudaError_t huf_decode(const Geo& g, void* dst, const void* cbuf, const u64* csizes, u64* results,
                       const void* orig, cudaStream_t stream, u32 flags)
{
    static SmemOptIn optinA, optinB;
    // Table rows per CTA.  Pass A: 306 rows + the 8 KB output staging -> 55.5 KB -> FOUR CTAs (256 blocks) per SM; pass B, for the
    // blocks whose tables need more (wide, flat alphabets): 808 rows, no staging -> two CTAs per SM.  FSEB200_HUFD_ROWS / _ROWS_B override;
    // each is clamped to what the device's per-block shared-memory opt-in limit holds for its pass (pass A with the staging).
    static u32 const reqA = [] { const char* e = std::getenv("FSEB200_HUFD_ROWS"); return e ? (u32)std::atoi(e) : 306u; }();
    static u32 const reqB = [] { const char* e = std::getenv("FSEB200_HUFD_ROWS_B"); return e ? (u32)std::atoi(e) : 808u; }();   // 0 = single pass
    if (g.nBlocks == 0) return cudaSuccess;
    int const dev = current_device();
    u32 const optin = (u32)device_smem_optin(dev);
    auto fit = [optin](bool staged) { u32 const fixed = hufd::smem_bytes(0, staged, NS); return optin > fixed ? (optin - fixed) / (hufd::G * 2) : 0u; };
    u32 const rowsA = max(hufd::MIN_ROWS, min(reqA, fit(true)));     // below MIN_ROWS the opt-in below fails and the call reports it
    u32 const rowsB = min(reqB, fit(false));
    size_t const smemA = hufd::smem_bytes(rowsA, true, NS);
    bool const twoPass = rowsB > rowsA;
    cudaError_t e = optinA.ensure(hufd::huf_decode_kernel<true, Geo, NS>, dev, (int)smemA);
    if (e == cudaSuccess && twoPass) e = optinB.ensure(hufd::huf_decode_kernel<false, Geo, NS>, dev, (int)hufd::smem_bytes(rowsB, false, NS));
    if (e != cudaSuccess) return e;
    u32* scratch = nullptr;
    if (twoPass) {
        scratch = (u32*)stream_scratch(1, stream, ((size_t)g.nBlocks + 1) * sizeof(u32), &e);
        if (e != cudaSuccess) return e;
        e = cudaMemsetAsync(scratch, 0, sizeof(u32), stream);              // [0] = number of deferred blocks, [1..] = their indices
        if (e != cudaSuccess) return e;
    }
    // Pass A grid shape.  Every lane decodes a whole stream, so a launch lasts one "round" however few blocks a CTA holds, and a
    // round is the faster the fewer warps share an SM .  A batch that fills most of
    // the machine is spread evenly -- every SM the same number of blocks per round, CTAs only partly full; a small batch (a pipeline
    // chunk, a scatter/gather piece, one block) packs its CTAs full instead, so that each SM hosts as few warps as possible.
    int perSm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, hufd::huf_decode_kernel<true, Geo, NS>, hufd::threads_for(NS), smemA) != cudaSuccess || perSm < 1) perSm = 1;
    u32 const slots = (u32)perSm * (u32)device_sm_count(dev);
    u32 gEff = (u32)hufd::G;
    if ((u64)g.nBlocks * 5 > (u64)slots * hufd::G * 4) {                 // more than 80 % of what the machine holds at once (threshold chosen before the H100 port, not re-tuned)
        u32 const rounds = (g.nBlocks + slots * hufd::G - 1) / (slots * hufd::G);
        gEff = (g.nBlocks + slots * rounds - 1) / (slots * rounds);
        if (gEff > (u32)hufd::G) gEff = hufd::G;
        if (gEff < 1) gEff = 1;
    }
    unsigned const grid = (g.nBlocks + gEff - 1) / gEff;
    hufd::huf_decode_kernel<true, Geo, NS><<<grid, hufd::threads_for(NS), smemA, stream>>>(g, (u8*)dst, (const u8*)cbuf, csizes, results, (const u8*)orig, flags, gEff, rowsA,
                                                                    nullptr, nullptr, twoPass ? scratch + 1 : nullptr, scratch);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    if (twoPass) {   // pass B over the deferred list; its length lives on the device, so the grid covers the worst case and idle CTAs leave at once
        unsigned const gridB = (g.nBlocks + hufd::G - 1) / hufd::G;
        hufd::huf_decode_kernel<false, Geo, NS><<<gridB, hufd::threads_for(NS), hufd::smem_bytes(rowsB, false, NS), stream>>>(g, (u8*)dst, (const u8*)cbuf, csizes, results, (const u8*)orig, flags,
                                                                                            (u32)hufd::G, rowsB, scratch + 1, scratch, nullptr, nullptr);
        e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    if (flags == 1u) return cudaSuccess;                                // X1-only semantics (HeaderDescs included): no verdict pass
    if constexpr (Geo::DESCS) return launch_huf_x2_fixup_blocks(g, NS, stream);
    else return launch_huf_x2_fixup(g, dst, cbuf, csizes, results, stream);
}
}  // namespace

cudaError_t launch_huf_decode(const BatchGeom& g, void* dst, const void* cbuf, const u64* csizes, u64* results,
                              const void* orig, cudaStream_t stream, u32 flags)
{
    return huf_decode<BatchGeom, 4>(g, dst, cbuf, csizes, results, orig, stream, flags);
}

// per-block descriptors (BlockDescs): the same passes, budgets and grid shape.  nStreams 4: HUF_decompress semantics on every
// block; 1: HUF_decompress1X_DCtx semantics (one lane per block).
cudaError_t launch_huf_decode_blocks(const BlockDescs& g, int nStreams, cudaStream_t stream)
{
    return nStreams == 1 ? huf_decode<BlockDescs, 1>(g, nullptr, nullptr, nullptr, nullptr, nullptr, stream, 0u)
                         : huf_decode<BlockDescs, 4>(g, nullptr, nullptr, nullptr, nullptr, nullptr, stream, 0u);
}

// header-less blocks (HeaderDescs): X1 verdicts only -- HUF_decompress{4X,1X}1_DCtx for a block with its own header, HUF_readDTableX1
// on the caller's header + HUF_decompress{4X,1X}1_usingDTable otherwise.  The same passes, budgets and grid shape.  nStreams 0: each
// block in the form single[b] names, one decode per form (hufd::HufMixedSplit).
cudaError_t launch_huf_decode_headers(const HeaderDescs& g, int nStreams, cudaStream_t stream, const u8* single)
{
    if (nStreams == 1) return huf_decode<HeaderDescs, 1>(g, nullptr, nullptr, nullptr, nullptr, nullptr, stream, 1u);
    if (nStreams) return huf_decode<HeaderDescs, 4>(g, nullptr, nullptr, nullptr, nullptr, nullptr, stream, 1u);
    if (g.nBlocks == 0) return cudaSuccess;
    size_t const n = g.nBlocks;
    cudaError_t e;
    u64* const s = (u64*)stream_scratch(13, stream, 3 * sizeof(u64) * n, &e);       // cap4, cap1, the 1X launch's verdicts
    if (e != cudaSuccess) return e;
    hufd::HufMixedSplit m;
    m.dstCap = g.dstCap; m.single = single; m.cap4 = s; m.cap1 = s + n; m.res1 = s + 2 * n; m.result = g.result; m.nBlocks = g.nBlocks;
    unsigned const grid = (unsigned)((n + hufd::FORM_THREADS - 1) / hufd::FORM_THREADS);
    hufd::huf_mixed_split_kernel<<<grid, hufd::FORM_THREADS, 0, stream>>>(m);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    HeaderDescs d = g;
    d.dstCap = m.cap4;
    if ((e = huf_decode<HeaderDescs, 4>(d, nullptr, nullptr, nullptr, nullptr, nullptr, stream, 1u)) != cudaSuccess) return e;
    d.dstCap = m.cap1; d.result = s + 2 * n;
    if ((e = huf_decode<HeaderDescs, 1>(d, nullptr, nullptr, nullptr, nullptr, nullptr, stream, 1u)) != cudaSuccess) return e;
    hufd::huf_mixed_merge_kernel<<<grid, hufd::FORM_THREADS, 0, stream>>>(m);
    return cudaGetLastError();
}

}  // namespace fseb
