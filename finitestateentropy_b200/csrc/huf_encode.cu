// huf_encode.cu -- batched Huff0 4-stream encode for sm_90a.
//
// Replaces, per block, the CPU chain
//   HUF_compress2 / HUF_compress_internal  lib/huf_compress.c:637-724,787-793 (table reuse: RepeatDescs, huf_plan_kernel)
//   HIST_count_wksp                        lib/hist.c:163-173
//   HUF_optimalTableLog                    lib/huf_compress.c:48-51
//   HUF_buildCTable_wksp (+HUF_sort, HUF_setMaxHeight)  lib/huf_compress.c:215-410
//   HUF_writeCTable (+HUF_compressWeights) lib/huf_compress.c:63-147
//   HUF_compress4X_usingCTable_internal / HUF_compress1X_usingCTable_internal_body  :457-502,552-603
// and returns the same value per block: 0 (not compressible / does not fit), 1 (RLE, byte in dst[0]),
// the compressed size, or an error code.  Compressed bytes are identical to the reference's.
// Both kernels take the stream count as a template parameter: 4 (above), or 1 for descriptor batches in the single-stream
// format -- HUF_compress1X per block (huf_compress.c:457-502,750-758): the same histograms, table and header, one stream.
// Packed output (PackedDescs, either format): the blocks back to back in one buffer, placed by a scan of their stored lengths
// that runs between the two kernels below (huf_pack_*_kernel).
//
// H100 mapping -- two kernels, because the work has two very different shapes:
//   1. huf_plan_kernel, ONE CTA PER 32 BLOCKS: histograms and sort warp per block, then the O(alphabet)
//      serial pieces with exact CPU tie-breaks (Huffman merge, depth limiter, canonical values, weight
//      header incl. its tiny FSE coder) LANE PER BLOCK in one warp, then stream sizes and verdict warp
//      per block again.  The serial chains are latency-bound: run on lane 0 of a warp per block they
//      left 31 lanes idle; side by side in one warp they cost about what one chain costs, and three
//      CTAs per SM keep the other CTAs' histograms running meanwhile.
//      Output: a 3.2 KB "plan" per block in a stream-ordered scratch buffer (code table, header,
//      verdict, the per-segment counts passed from the first phase to the last).
//   2. huf_emit_kernel, ONE CTA (4 warps) PER BLOCK, one warp per stream, no serial section and no
//      second look at the data: stream sizes and offsets are already known from the per-segment
//      histograms of the plan kernel.  (An earlier version gave each thread a contiguous run of
//      symbols staged in shared memory: runs are 128 bytes apart, i.e. all 32 lanes of a warp in the
//      same bank -- 525M bank conflicts per 256 MiB, short-scoreboard 38 stalls per issue.)
#include <mutex>
#include <type_traits>
#include <vector>
#include "common.cuh"
#include "launchers.h"
#include "launch_util.cuh"
#include "fse_dev.cuh"
#include "sink_dev.cuh"
#include "huf_build_dev.cuh"
#include "pack_dev.cuh"

namespace fseb {
namespace hufe {

constexpr unsigned FULL = 0xFFFFFFFFu;

struct __align__(16) Plan {        // per block, in global scratch
    u32 ctable[256];               // val | nbBits << 16
    u8  header[136];
    u32 hSize;
    u32 state;                     // PLAN_EMIT, PLAN_FINAL (the verdict is final: nothing to emit) or PLAN_EMIT_1X
    u32 total;                     // compressed size when state == 0
    u32 streamOff[4];              // byte offset of each stream from the start of the block
    u32 streamBytes[4];
    u16 segCount[4][256];          // plan kernel only: per-segment histograms (a segment count is <= HUF_BLOCK_MAX / 4 = 32768)
};
// Plan::state.  A mixed chain call runs two emit launches, 4X and 1X; a 1X block of such a call is PLAN_EMIT_1X, so the 4X launch
// passes it by as it passes a final verdict, and the 1X launch (the Emit1X view) passes by everything else.
enum : u32 { PLAN_EMIT = 0, PLAN_FINAL = 1, PLAN_EMIT_1X = 2 };

// ---------------------------------------------------------------------------------------------
// kernel 1: statistics, code table, tree header, stream sizes, verdict -- one CTA per group of 32 blocks
//   phase 1, warp per block: histograms, early verdicts, HUF_optimalTableLog, HUF_sort -> the group's node rows
//   phase 2, lane per block: warp 0, lane l builds block l's table (merge, lengths, HUF_setMaxHeight, canonical
//            values, weight header) -- the order-sensitive chains, 32 of them side by side instead of one per warp
//   phase 3, warp per block: stream bit totals, the writer's capacity rule, the final verdict, the plan
// ---------------------------------------------------------------------------------------------
constexpr int PLAN_WARPS = 8;
constexpr u32 GROUP = 32;                          // blocks per CTA, one per lane of the builder warp
constexpr u32 HDR_STRIDE = 34 + 224 + 1;           // words per lane in phase 2's header area: header (136 B) + d_huf_write_ctable's
                                                   // workspace (224 words), + 1 so that the lanes' areas start in different banks
constexpr u32 CT_ROW = HDR_STRIDE;                 // rows CT_ROW + s: code table cell of symbol s (phase 2 -> phase 3)
constexpr u32 ROWS = CT_ROW + 256;
constexpr u32 NODE_END = 0x7FFFFFFFu, LEAF_END = 0xFFFFFFFFu;   // empty queues in the merge (the reference's 1<<30 / 1<<31 barriers)
// Interleaved rows: word [r][c] belongs to block c of the group, so the 32 lanes of the builder warp always hit 32 different
// banks whatever their indices.  Row use by phase:
//   phase 1: rows 1 .. 256 node i = leaf of rank i (count); rows 257 .. 512 reused as the eight warps' segment histograms
//   phase 2: node i at row 1 + i (leaves 0 .. 255, internal nodes 256 .. 510), count | parent - 256 << 24, then count | length << 24;
//            row 0 = node -1 (length 0, read by HUF_setMaxHeight); then rows CT_ROW + s = code table cells and, once the tree is
//            dead, rows 0 .. CT_ROW - 1 as 32 contiguous per-lane areas of HDR_STRIDE words for the header writer
struct PlanCta {                   // 72.8 KB: three CTAs per SM
    u32 nd[ROWS][GROUP];
    u8  sym[256][GROUP];           // symbol of the leaf of rank i
    u64 res[GROUP];                // phase 2 result: header size or error code
    u16 msv[GROUP];
    u8  last[GROUP];               // rank of the last non-zero count
    u8  tlog[GROUP];               // HUF_optimalTableLog in phase 1, the maximum code length after phase 2
    u8  live[GROUP];               // 0: the verdict is already final
};
static_assert(ROWS >= 1 + 256 + PLAN_WARPS * 4 * 256 / GROUP, "segment histograms must fit in the rows above the leaves");
static_assert(ROWS >= 1 + 511 && CT_ROW >= 1 + 256, "node rows");
static_assert(HUF_BLOCK_MAX < (1u << 24), "node counts share a word with an 8-bit parent / length");
static_assert(sizeof(PlanCta) <= 76 * 1024, "three CTAs per SM");

// Stream bits of a block coded with the table whose cells (val | nbBits << 16) the lane holds for symbols i * 32 + lane, from
// count(k, i) = that symbol's count in segment k (4X) or in the whole block (1X).  One warp.
template <int NS, class Count>
__device__ __forceinline__ void stream_bits(const u32 (&cell)[8], Count count, u32 (&bits)[NS])
{
    #pragma unroll
    for (int k = 0; k < NS; k++) {
        u32 acc = 0;
        #pragma unroll
        for (u32 i = 0; i < 8; i++) acc += count(k, i) * (cell[i] >> 16);
        #pragma unroll
        for (int dlt = 16; dlt; dlt >>= 1) acc += __shfl_xor_sync(FULL, acc, dlt);
        bits[k] = acc;
    }
}

// The streams' places after a header of hs bytes with capLeft bytes after it, under the writer's capacity rule stream after stream
// (huf_compress.c:566-600, bitstream.h:190,246,258): offsets, lengths and the block's total; false if a stream does not fit.
template <int NS>
__device__ __forceinline__ bool place_streams(const u32 (&bits)[NS], u64 hs, u64 capLeft, u32 (&offs)[NS], u32 (&lens)[NS], u64& total)
{
    u64 op = (NS == 4) ? 6 : 0; bool fits = true;
    #pragma unroll
    for (int t = 0; t < NS; t++) {
        u64 const capk = capLeft - op;
        u64 const tot = (u64)bits[t] + 1;                                    // + end mark
        if (fits && (capk <= 8 || (tot >> 3) >= capk - 8)) fits = false;
        offs[t] = (u32)(hs + op); lens[t] = (u32)((tot + 7) >> 3);
        op += lens[t];
    }
    total = hs + op;
    return fits;
}

// HUF_compressCTable_internal with that table after a header of hs bytes, at capacity cap: the 4X size tests (huf_compress.c:564-565),
// the stream sizes, the capacity rule and the final compressibility test (:625).  1X: one stream, no jump table and no srcSize < 12
// test (:457-475).  A block that passes gets its plan: the cells, the header (hs bytes at hdr), the streams' offsets and lengths,
// hSize and total.
template <int NS, class Count>
__device__ __forceinline__ bool plan_streams(Plan& P, const u32 (&cell)[8], Count count, const u8* hdr, u64 hs, u64 cap, u32 n,
                                             unsigned lane, u64& total)
{
    u32 bits[NS], offs[NS], lens[NS];
    stream_bits<NS>(cell, count, bits);
    bool const fits = place_streams<NS>(bits, hs, cap - hs, offs, lens, total);
    if ((NS == 4 && (cap - hs < 6 + 1 + 1 + 1 + 8 || n < 12)) || !fits || total >= (u64)n - 1) return false;
    #pragma unroll
    for (u32 i = 0; i < 8; i++) P.ctable[i * 32 + lane] = cell[i];
    for (u32 i = lane; i < (u32)hs; i += 32) P.header[i] = hdr[i];
    #pragma unroll
    for (int k = 0; k < NS; k++) if (lane == (unsigned)k) { P.streamOff[k] = offs[k]; P.streamBytes[k] = lens[k]; }
    if (lane == 0) { P.hSize = (u32)hs; P.total = (u32)total; }
    return true;
}

// Stream mode NS: 4 or 1 streams per block, or 0 (mixed chains): per block, the form enc_single names.  by_form calls f with the
// block's stream count as a Form; under mode 0 that is a warp-uniform branch, since one warp owns one block at a time in both
// kernels that call it.
template <int S> using Form = std::integral_constant<int, S>;
template <int NS, class F>
__device__ __forceinline__ auto by_form(bool single, F f)
{
    if constexpr (NS == 0) return single ? f(Form<1>{}) : f(Form<4>{});
    else return f(Form<NS>{});
}

// HUF_estimateCompressedSize (huf_compress.c:422-430) of the table whose cells the lane holds as above, in bits before its >> 3,
// from the block's counts cnt[i] of symbols i * 32 + lane
__device__ __forceinline__ u32 estimate_bits(const u32 (&cell)[8], const u32 (&cnt)[8])
{
    u32 acc = 0;
    #pragma unroll
    for (u32 i = 0; i < 8; i++) acc += cnt[i] * (cell[i] >> 16);
    return __reduce_add_sync(FULL, acc);
}

// histogram of src[begin, end) into cnt[256] (shared memory), one warp
__device__ __forceinline__ void warp_hist_range(u32* cnt, const u8* s, u32 begin, u32 end, unsigned lane)
{
    u32 i = begin;
    u32 const head = min(end, (u32)((begin + 15) & ~15u));         // bytes up to 16-byte alignment of the OFFSET ...
    bool const vec = ((reinterpret_cast<u64>(s) & 15) == 0);       // ... which is alignment of the address when the block is aligned
    if (vec) {
        for (u32 k = i + lane; k < head; k += 32) atomicAdd(&cnt[s[k]], 1u);
        i = head;
        u32 const nvec = (end - i) / 16;
        const uint4* const gv = reinterpret_cast<const uint4*>(s + i);
        for (u32 v0 = 0; v0 < nvec; v0 += 128) {                   // four 16-byte loads in flight per lane before the first use
            uint4 x[4];
            #pragma unroll
            for (int h = 0; h < 4; h++) { u32 const vi = v0 + 32 * h + lane; x[h] = (vi < nvec) ? __ldg(gv + vi) : make_uint4(0, 0, 0, 0); }
            #pragma unroll
            for (int h = 0; h < 4; h++) {
                if (v0 + 32 * h + lane >= nvec) continue;
                u32 const wd[4] = { x[h].x, x[h].y, x[h].z, x[h].w };
                #pragma unroll
                for (int k = 0; k < 4; k++) {
                    u32 const y = wd[k];                             // one extract + one address + one shared atomic per byte
                    atomicAdd(&cnt[y & 0xFF], 1u); atomicAdd(&cnt[__byte_perm(y, 0, 0x4441)], 1u);
                    atomicAdd(&cnt[__byte_perm(y, 0, 0x4442)], 1u); atomicAdd(&cnt[y >> 24], 1u);
                }
            }
        }
        i += nvec * 16;
    }
    for (u32 k = i + lane; k < end; k += 32) atomicAdd(&cnt[s[k]], 1u);
}

// All four per-segment histograms of an aligned block whose segments are whole 2 KB batches (the 32 KB case): one
// software pipeline over the block, the next batch's four 16-byte loads are in flight while the current one is counted,
// on two alternating register sets (nothing touches a register with a load in flight).
__device__ __forceinline__ void warp_hist4_pipelined(u32 (*count4)[256], const u8* s, u32 n, u32 seg, unsigned lane)
{
    const uint4* const gv = reinterpret_cast<const uint4*>(s) + lane;
    u32 const B = n / 2048, perSeg = seg / 2048;
    auto load = [&](uint4 (&x)[4], u32 b) {
        #pragma unroll
        for (int h = 0; h < 4; h++) x[h] = __ldg(gv + b * 128 + 32 * h);
    };
    auto count = [&](const uint4 (&x)[4], u32 b) {
        u32* const cnt = count4[b / perSeg];
        #pragma unroll
        for (int h = 0; h < 4; h++) {
            u32 const wd[4] = { x[h].x, x[h].y, x[h].z, x[h].w };
            #pragma unroll
            for (int k = 0; k < 4; k++) {
                u32 const y = wd[k];                                 // one extract + one address + one shared atomic per byte
                atomicAdd(&cnt[y & 0xFF], 1u); atomicAdd(&cnt[__byte_perm(y, 0, 0x4441)], 1u);
                atomicAdd(&cnt[__byte_perm(y, 0, 0x4442)], 1u); atomicAdd(&cnt[y >> 24], 1u);
            }
        }
    };
    uint4 xa[4], xb[4];
    load(xa, 0);
    #pragma unroll 1
    for (u32 b = 0; b < B; b += 2) {
        if (b + 1 < B) load(xb, b + 1);
        count(xa, b);
        if (b + 2 < B) load(xa, b + 2);
        if (b + 1 < B) count(xb, b + 1);
    }
}

// NS = streams per block: 4 (HUF_compress2, the 4X format) or 1 (HUF_compress1X, descriptor batches only).  Phases 1 and 2 are
// the same for both; phase 3 sizes NS streams and applies that format's capacity rule.
// Geo = RepeatDescs: HUF_compress{4X,1X}_repeat per block (huf_compress.c:653-724), with the block's (table, flag) pair.  Phase 1
// takes the old-table exits that need no tree (prefer + valid before the histogram exits, validation under check, prefer + any
// flag after them) and marks the block; phase 2 builds trees only for the other blocks; phase 3 compares the estimates, saves a
// new table, and sizes the streams with the chosen table (hSize 0 for the old one).  S.live then also tells the three apart:
// 1 = new table, 2 = new table unless the estimates prefer the old one, 3 = old table.
// Geo = ChainDescs: the same phases with no flag, for every block of every chain; they write nothing but scratch.  Phase 1 records
// the argument verdict or the histogram exit that would apply (and keeps the counts either way: prefer + valid skips the exits),
// phase 2 builds every tree the exits leave, phase 3 plans the block with its new table.  huf_chain_kernel then decides.
// Geo = ChainPackedDescs: the same, at capacities HUF_compressBound(srcSize).
// Mixed chains (common.cuh Mixed): NS = 0, and phase 3 plans each block in the form its flag names.
template <class Geo, int NS>
__global__ void __launch_bounds__(32 * PLAN_WARPS, 3)
huf_plan_kernel(Geo g, u8* __restrict__ cbuf, u64* __restrict__ csizes, const u8* __restrict__ src,
                unsigned msvReq, unsigned tlogReq, Plan* __restrict__ plans)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    PlanCta& S = *reinterpret_cast<PlanCta*>(smem_raw);
    unsigned const lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    u32 const b0 = blockIdx.x * GROUP;
    constexpr bool REP = std::is_same_v<Geo, RepeatDescs>;
    constexpr bool CHAIN = std::is_base_of_v<ChainDescs, Geo>;                              // ChainDescs or ChainPackedDescs, or mixed
    static_assert(NS == 4 || NS == 1 || (NS == 0 && CHAIN), "4X, 1X, or mixed chains");
#define FSEB_FINAL(v) { if (lane == 0) {                                                                            \
        if constexpr (CHAIN) { g.fact[b].kind = CF_ARGS; g.fact[b].exitValue = (v); }                                  \
        else { P.state = 1; enc_out(g, csizes, b) = (v); }                                                             \
        S.live[c] = 0; } continue; }                                                    // next block of the loop

    // ---- phase 1: one warp per block ----
    u32 (*const count4)[256] = reinterpret_cast<u32 (*)[256]>(&S.nd[257][0] + warp * 4 * 256);
    #pragma unroll 1
    for (u32 c = warp; c < GROUP; c += PLAN_WARPS) {
        __syncwarp();                                                   // the previous block is done with count4
        u32 const b = b0 + c;
        if (b >= g.nBlocks) { if (lane == 0) S.live[c] = 0; continue; }
        u32 const n = enc_len(g, b);
        u64 const cap = enc_cap(g, b);
        const u8* const s = enc_src(g, src, b);
        Plan& P = plans[b];
        // argument checks of HUF_compress_internal (huf_compress.c:656-664), in its order
        if (!n) FSEB_FINAL(0);
        if (!cap) FSEB_FINAL(0);
        if (n > HUF_BLOCK_MAX) FSEB_FINAL(err(E_SRC_WRONG));
        if (tlogReq > HUF_MAX_TLOG) FSEB_FINAL(err(E_TLOG_TOO_LARGE));
        if (msvReq > HUF_MAX_SV) FSEB_FINAL(err(E_MSV_TOO_LARGE));
        unsigned const msvDecl = msvReq ? msvReq : HUF_MAX_SV;
        int flag = 0; bool prefer = false;
        if constexpr (REP) { flag = g.repeat[b]; prefer = g.prefer[b] != 0; }
        bool const oldNow = REP && prefer && flag == 2;                                           // :665-669: no histogram exit

        // histograms, one per 4X segment (HIST_count_wksp semantics for their sum, hist.c:163-173,128)
        u32 const seg = (n + 3) / 4;
        for (u32 i = lane; i < 4 * 256; i += 32) (&count4[0][0])[i] = 0;
        __syncwarp();
        if ((reinterpret_cast<u64>(s) & 15) == 0 && seg % 2048 == 0 && n == 4 * seg) warp_hist4_pipelined(count4, s, n, seg, lane);
        else {
            #pragma unroll 1
            for (u32 k = 0; k < 4; k++) {
                u32 const beg = min(k * seg, n), end = (k < 3) ? min((k + 1) * seg, n) : n;
                warp_hist_range(count4[k], s, beg, end, lane);
            }
        }
        __syncwarp();
        u32 cnt[8], top = 0, best = 0;
        #pragma unroll
        for (u32 i = 0; i < 8; i++) {
            u32 const sy = i * 32 + lane;
            cnt[i] = count4[0][sy] + count4[1][sy] + count4[2][sy] + count4[3][sy];
            if (cnt[i]) top = sy;
            best = max(best, cnt[i]);
        }
        #pragma unroll
        for (int dlt = 16; dlt; dlt >>= 1) { top = max(top, __shfl_xor_sync(FULL, top, dlt)); best = max(best, __shfl_xor_sync(FULL, best, dlt)); }
        if (!CHAIN && !oldNow) {
            if (msvDecl < 255 && top > msvDecl) FSEB_FINAL(err(E_MSV_TOO_SMALL));                 // hist.c:128
            if (best == n) {                                                                      // huf_compress.c:673
                if constexpr (!std::is_same_v<Geo, PackedDescs>) { if (lane == 0) enc_dst(g, cbuf, b)[0] = s[0]; }   // packed: placement writes it
                FSEB_FINAL(1);
            }
            if (best <= (n >> 7) + 4) FSEB_FINAL(0);                                              // :674
        }
        bool histExit = false;
        if constexpr (CHAIN) {                                                                    // the exit that applies unless prefer + valid
            bool const mst = msvReq != 0 && msvReq < 255 && top > msvReq;                        // msvDecl < 255 && top > msvDecl
            histExit = mst || best == n || best <= (n >> 7) + 4;
            if (lane == 0) {
                ChainFact& F = g.fact[b];
                F.kind = histExit ? CF_HIST : CF_TREE; F.msv = (u16)top;
                F.exitValue = mst ? err(E_MSV_TOO_SMALL) : best == n ? 1 : 0;
            }
        }
        u32 const msv = top;
        // segment counts for phase 3, compacted to u16
        #pragma unroll
        for (u32 k = 0; k < 4; k++)
            #pragma unroll
            for (u32 i = 0; i < 8; i++) P.segCount[k][i * 32 + lane] = (u16)count4[k][i * 32 + lane];
        if (CHAIN && histExit) { if (lane == 0) S.live[c] = 0; continue; }                     // its counts kept: prefer + valid skips the exit
        if constexpr (REP) {
            if (!oldNow && flag == 1) {                                                           // :679-683 HUF_validateCTable
                const u32* const old = g.ctable[b];
                bool bad = false;
                #pragma unroll
                for (u32 i = 0; i < 8; i++) { u32 const sy = i * 32 + lane; bad |= sy <= msv && cnt[i] && ((old[sy] >> 16) & 0xFFu) == 0; }
                if (__any_sync(FULL, bad)) { flag = 0; if (lane == 0) g.repeat[b] = 0; }
            }
            if (oldNow || (prefer && flag != 0)) {                                                // :685-689
                if (lane == 0) { S.msv[c] = (u16)msv; S.live[c] = 3; }
                continue;
            }
        }
        // HUF_sort (huf_compress.c:307-329): decreasing count, ties by increasing symbol == decreasing (count << 8 | 255 - symbol)
        u32 key[8], nnz = 0;
        #pragma unroll
        for (u32 i = 0; i < 8; i++) { u32 const sy = i * 32 + lane; key[i] = ((sy <= msv ? cnt[i] : 0u) << 8) | (255u - sy); nnz += __popc(__ballot_sync(FULL, cnt[i] != 0)); }
        warp_sort256_desc(key, lane);
        #pragma unroll
        for (u32 i = 0; i < 8; i++) {
            u32 const r = i * 32 + lane;
            if (r <= msv) { S.nd[1 + r][c] = key[i] >> 8; S.sym[r][c] = (u8)(255u - (key[i] & 0xFFu)); }
        }
        if (lane == 0) {
            S.nd[0][c] = 0;
            S.msv[c] = (u16)msv; S.last[c] = (u8)(nnz - 1); S.live[c] = (REP && flag != 0) ? 2 : 1;
            S.tlog[c] = (u8)d_optimal_tablelog(tlogReq ? tlogReq : HUF_DEF_TLOG, n, msv, 1);     // huf_compress.c:691
        }
    }
    __syncthreads();

    // ---- phase 2: warp 0, lane c builds block c's table (huf_compress.c:338-410, then :703-716) ----
    if (warp == 0) {
        u32 const c = lane;
        bool const live = REP ? (S.live[c] == 1 || S.live[c] == 2) : S.live[c];     // REP: no tree for an old-table block
        u32 const msv = S.msv[c];
        u32* const col = &S.nd[1][c];                                   // node i at col[i * GROUP]
        auto at = [&](int i) -> u32& { return col[i * (int)GROUP]; };
        u32* const ct = &S.nd[CT_ROW][c];                               // cell of symbol s at ct[s * GROUP]
        u64 res = 0;
        if (live) {
            int const last = S.last[c];
            int fresh = 256, leaf = last, inner = fresh;
            int const root = fresh + leaf - 1;
            {   u32 const x = at(leaf), y = at(leaf - 1);
                at(fresh) = x + y;                                      // parents 256 - 256 = 0 in the tag byte
                fresh++; leaf -= 2;
            }
            u32 cl = leaf >= 0 ? at(leaf) : LEAF_END, ci = at(inner);   // heads of the two queues, in registers
            while (fresh <= root) {                                     // on equal counts the internal node goes first
                int a, bb; u32 ca, cb;
                if (cl < ci) { a = leaf--; ca = cl; cl = leaf >= 0 ? at(leaf) : LEAF_END; } else { a = inner++; ca = ci; ci = inner < fresh ? at(inner) : NODE_END; }
                if (cl < ci) { bb = leaf--; cb = cl; cl = leaf >= 0 ? at(leaf) : LEAF_END; } else { bb = inner++; cb = ci; ci = inner < fresh ? at(inner) : NODE_END; }
                u32 const sum = ca + cb;
                at(fresh) = sum;
                if (inner == fresh) ci = sum;                           // the new node is the head of the inner queue
                u32 const tag = (u32)(fresh - 256) << 24;
                at(a) = ca | tag; at(bb) = cb | tag;
                fresh++;
            }
            // code lengths: parent -> length in the tag byte, root first (a parent's index is above its children's)
            at(root) &= 0xFFFFFFu;
            for (int m = root - 1; m >= 256; m--) { u32 const v = at(m); at(m) = (v & 0xFFFFFFu) | (((at(256 + (int)(v >> 24)) >> 24) + 1) << 24); }
            for (int m = 0; m <= last; m++) { u32 const v = at(m); at(m) = (v & 0xFFFFFFu) | (((at(256 + (int)(v >> 24)) >> 24) + 1) << 24); }
            u32 const mb = d_huf_limit_depth(PackedNodeView{ col, (int)GROUP }, (u32)last, S.tlog[c]);
            if (mb > HUF_MAX_TLOG) res = err(E_GENERIC);
            else {
                // canonical values (huf_compress.c:394-407): the longest lengths numbered from 0, symbol order inside a length
                u32 perLen[HUF_MAX_TLOG + 1], nextVal[HUF_MAX_TLOG + 1];
                for (u32 i = 0; i <= HUF_MAX_TLOG; i++) { perLen[i] = 0; nextVal[i] = 0; }
                for (int m = 0; m <= last; m++) perLen[at(m) >> 24]++;
                u32 v = 0;
                for (int m = (int)mb; m > 0; m--) { nextVal[m] = v; v = (v + perLen[m]) >> 1; }
                for (u32 r = 0; r <= msv; r++) ct[S.sym[r][c] * GROUP] = (int)r <= last ? at((int)r) >> 24 : 0u;
                for (u32 sy = 0; sy <= msv; sy++) { u32 const len = ct[sy * GROUP]; ct[sy * GROUP] = (nextVal[len]++ & 0xFFFF) | (len << 16); }
                S.tlog[c] = (u8)mb;
            }
        }
        __syncwarp();                                                   // every lane is done with the tree rows: header areas next
        if (live && !is_err(res)) {
            u64 const cap = enc_cap(g, b0 + c);
            u32* const area = &S.nd[0][0] + c * HDR_STRIDE;
            struct Col { const u32* p; __device__ u32 operator[](u32 i) const { return p[i * GROUP]; } };
            res = d_huf_write_ctable(reinterpret_cast<u8*>(area), cap < 136 ? cap : 136, Col{ ct }, msv, S.tlog[c], area + 34);
        }
        S.res[c] = res;
    }
    __syncthreads();

    // ---- phase 3: one warp per block -- RepeatDescs: the table-reuse choice; then plan_streams with the chosen table, the stream
    //      sizes from the per-segment histograms ----
    #pragma unroll 1
    for (u32 c = warp; c < GROUP; c += PLAN_WARPS) {
        if (!S.live[c]) continue;
        u32 const b = b0 + c;
        u32 const n = enc_len(g, b);
        u64 const cap = enc_cap(g, b);
        Plan& P = plans[b];
        u64 hs = S.res[c];
        auto const count = [&](auto form, int k, u32 i) {
            u32 const sy = i * 32 + lane;                                    // 1X: the four segment counts of a symbol add up to its block count
            return (decltype(form)::value == 4) ? (u32)P.segCount[k][sy] : (u32)P.segCount[0][sy] + P.segCount[1][sy] + P.segCount[2][sy] + P.segCount[3][sy];
        };
        auto const new_cells = [&](u32 (&cell)[8]) {
            u32 const msv = S.msv[c];
            #pragma unroll
            for (u32 i = 0; i < 8; i++) cell[i] = (i * 32 + lane <= msv) ? S.nd[CT_ROW + i * 32 + lane][c] : 0u;
        };
        auto const block_counts = [&](u32 (&sum)[8]) {
            #pragma unroll
            for (u32 i = 0; i < 8; i++) { u32 const sy = i * 32 + lane; sum[i] = (u32)P.segCount[0][sy] + P.segCount[1][sy] + P.segCount[2][sy] + P.segCount[3][sy]; }
        };
        const u8* const hdr = reinterpret_cast<const u8*>(&S.nd[0][0] + c * HDR_STRIDE);
        u32 cell[8];
        u64 total;
        auto const plan = [&](auto form) {                                   // plan_streams in the block's form
            return plan_streams<decltype(form)::value>(P, cell, [&](int k, u32 i) { return count(form, k, i); }, hdr, hs, cap, n, lane, total);
        };
        if constexpr (CHAIN) {                   // the plan with the new table (its cells also for saving it), its verdict and estimate
            ChainFact& F = g.fact[b];
            if (lane == 0) F.hSize = hs;
            if (is_err(hs) || hs + 12 >= n) continue;                                             // :714, or the old table
            u32 sum[8];
            new_cells(cell);
            block_counts(sum);
            bool const ok = by_form<NS>(enc_single(g, b), plan);
            if (!ok) {
                #pragma unroll
                for (u32 i = 0; i < 8; i++) P.ctable[i * 32 + lane] = cell[i];
                if constexpr (std::is_same_v<Geo, ChainPackedLiteralsDescs>)                    // for a 1X re-plan in the chain kernel
                    for (u32 i = lane; i < (u32)hs; i += 32) P.header[i] = hdr[i];
            }
            u32 const newBits = estimate_bits(cell, sum);
            if (lane == 0) { F.newBits = newBits; F.newValue = ok ? total : 0; }
            continue;
        }
        bool useOld = false;
        if constexpr (REP) useOld = S.live[c] == 3;
        if (!useOld) {
            if (is_err(hs)) FSEB_FINAL(hs);
            if constexpr (REP) {
                new_cells(cell);
                if (S.live[c] == 2) {                                                             // :703-713 the estimates, old and new
                    u32 old[8], sum[8];
                    #pragma unroll
                    for (u32 i = 0; i < 8; i++) old[i] = g.ctable[b][i * 32 + lane] & 0xFFFFFFu;  // byte 3 is padding
                    block_counts(sum);
                    useOld = (estimate_bits(old, sum) >> 3) <= hs + (estimate_bits(cell, sum) >> 3) || hs + 12 >= n;
                }
                if (!useOld && hs + 12 < n) {                                                     // :716-719 the new table is saved, the flag set to none
                    #pragma unroll
                    for (u32 i = 0; i < 8; i++) g.ctable[b][i * 32 + lane] = cell[i];
                    if (lane == 0) g.repeat[b] = 0;
                }
            }
            if (!useOld && hs + 12 >= n) FSEB_FINAL(0);                                           // :714
        }
        if constexpr (REP) {                                                                      // every cell: prefer + valid codes symbols above msv
            if (useOld) {                                                                         // HUF_compressCTable_internal at ostart
                hs = 0;
                #pragma unroll
                for (u32 i = 0; i < 8; i++) cell[i] = g.ctable[b][i * 32 + lane] & 0xFFFFFFu;      // byte 3 is padding
            }
        } else new_cells(cell);
        if (!by_form<NS>(enc_single(g, b), plan)) FSEB_FINAL(0);
        if (lane == 0) { P.state = 0; enc_out(g, csizes, b) = total; }
    }
#undef FSEB_FINAL
}

// ---------------------------------------------------------------------------------------------
// Chains (ChainDescs): the decisions HUF_compress_internal takes with a stream's (table, flag) state (huf_compress.c:653-724), one
// warp per chain walking its blocks in order, from the facts the plan kernel recorded.  The state lives in registers: lane l holds
// the table's cells for symbols i * 32 + l, as the plan kernel's phase 3 does.  Nothing a decision reads from memory depends on
// the state, so the next block's facts, counts and new cells are loaded while the current block is decided.
// ---------------------------------------------------------------------------------------------
constexpr int CHAIN_WARPS = 4;

// Chain geometry: start[0] == 0, start[nChains] == nBlocks, never decreasing.  One CTA; *malformed gets the verdict.
__global__ void __launch_bounds__(1024)
huf_chain_check_kernel(const u64* __restrict__ start, u32 nChains, u32 nBlocks, u32* __restrict__ malformed)
{
    bool bad = threadIdx.x == 0 && (start[0] != 0 || start[nChains] != nBlocks);
    for (u64 c = threadIdx.x; c < nChains; c += blockDim.x) bad |= start[c + 1] < start[c];
    bad = __syncthreads_or(bad);
    if (threadIdx.x == 0) *malformed = bad;
}

struct ChainBlock {                // what the decision for one block reads
    ChainFact f;
    u32 cnt[4][8];                 // segment counts of symbols i * 32 + lane
    u32 cell[8];                   // the new table's cells (CF_TREE with hSize + 12 < srcSize)
    u8* dst;
    u64 cap;
    u32 n;
    int prefer;
};
struct ChainBlockMixed : ChainBlock {
    bool single;                   // the block's form (mixed chains)
};
template <class Geo, class Blk>
__device__ __forceinline__ void chain_load(const Geo& g, const Plan* plans, u32 b, Blk& x, unsigned lane)
{
    x.f = g.fact[b];
    const Plan& P = plans[b];      // read whatever the kind: a plan the block did not fill is never used
    #pragma unroll
    for (int k = 0; k < 4; k++)
        #pragma unroll
        for (u32 i = 0; i < 8; i++) x.cnt[k][i] = P.segCount[k][i * 32 + lane];
    #pragma unroll
    for (u32 i = 0; i < 8; i++) x.cell[i] = P.ctable[i * 32 + lane];
    if constexpr (std::is_same_v<Geo, ChainDescs> || std::is_same_v<Geo, ChainMixedDescs>) x.dst = enc_dst(g, nullptr, b);
    else x.dst = nullptr;                                                                   // packed: no place yet, and none needed
    x.cap = enc_cap(g, b); x.n = enc_len(g, b); x.prefer = g.prefer[b];
    if constexpr (std::is_same_v<Blk, ChainBlockMixed>) x.single = enc_single(g, b);
}

// HUF_compressCTable_internal with the table T (cells, byte 3 cleared) after a header of hs bytes in the S-stream form: the 4X
// size tests (huf_compress.c:564-565), the capacity rule and the final test (:625).  The block's value, 0 or the size, goes to r;
// a size comes with its plan (the cells, hSize, the streams' places; the header bytes must be in the plan already), and then the
// block is emitted (returns true).  The chain's table has hs 0; the literal policy also re-plans a new table as 1X with its header.
// Mixed and literal chains only: the 4X and 1X kernels keep this step inline; a build that ran it through this helper for them too
// changed their SASS, and one chain of 32,768 blocks took 35 instead of 28 ms per GiB on an H100.
template <int S>
__device__ __forceinline__ bool chain_plan(Plan& P, const u32 (&T)[8], u64 hs, const ChainBlock& x, const u32 (&sum)[8], unsigned lane,
                                           u64& r)
{
    u32 const n = x.n;
    auto const count = [&](int k, u32 i) { return S == 4 ? x.cnt[k][i] : sum[i]; };
    u32 bits[S], offs[S], lens[S];
    u64 total;
    stream_bits<S>(T, count, bits);
    bool const fits = place_streams<S>(bits, hs, x.cap - hs, offs, lens, total);
    bool const ok = !(S == 4 && (x.cap - hs < 6 + 1 + 1 + 1 + 8 || n < 12)) && fits && total < (u64)n - 1;
    if (ok) {
        #pragma unroll
        for (u32 i = 0; i < 8; i++) P.ctable[i * 32 + lane] = T[i];
        #pragma unroll
        for (int k = 0; k < S; k++) if (lane == (unsigned)k) { P.streamOff[k] = offs[k]; P.streamBytes[k] = lens[k]; }
        if (lane == 0) { P.hSize = (u32)hs; P.total = (u32)total; }
    }
    r = ok ? total : 0;
    return ok;
}

// One step of zstd's literal coder (ZSTD_compressLiterals; the rule is stated once, in include/fse_b200.h) on block b of a chain
// whose state is (T, F): the form from F, the size threshold, HUF_compress{1X,4X}_repeat on the step's flag Fs (its candidate
// table is the block's new cells x.cell), then the block's kind.  The plan kernel planned the form n decides; a block F makes 1X
// (F == 2, 256 <= n < 1024) is re-planned here, from its new cells and header or from T.  Writes the block's value, kind, form and
// plan state; commits the candidate (T := x.cell, F := 1) and returns true only for kind 2.
__device__ __forceinline__ bool literals_step(const ChainPackedLiteralsDescs& g, Plan& P, u32 b, const ChainBlockMixed& x,
                                              const u32 (&sum)[8], u32 (&T)[8], int& F, unsigned lane)
{
    ChainFact const& f = x.f;
    u32 const n = x.n;
    bool const single = n < 256 || (F == 2 && n < 1024);
    u64 r = 0;
    u8 kind = 0;
    if (n > HUF_BLOCK_MAX) { r = err(E_SRC_WRONG); kind = 4; }
    else if (n >= (F == 2 ? 6u : g.minLiterals)) {
        int Fs = F;
        bool useOld = false, fresh = false;
        if (f.kind == CF_ARGS) r = f.exitValue;                                                   // huf_compress.c:656-664
        else if (x.prefer && Fs == 2) useOld = true;                                              // :665-669
        else if (f.kind == CF_HIST) r = f.exitValue;                                              // hist.c:128, :673-674
        else {
            if (Fs == 1) {                                                                        // :679-683 HUF_validateCTable
                bool bad = false;
                #pragma unroll
                for (u32 i = 0; i < 8; i++) bad |= sum[i] && (T[i] >> 16) == 0;
                if (__any_sync(FULL, bad)) Fs = 0;
            }
            if (x.prefer && Fs != 0) useOld = true;                                               // :685-689
            else if (is_err(f.hSize)) r = f.hSize;
            else {
                if (Fs != 0) {                                                                    // :703-713 the estimates, old and new
                    u32 oldBits = 0;
                    #pragma unroll
                    for (u32 i = 0; i < 8; i++) oldBits += sum[i] * (T[i] >> 16);
                    oldBits = __reduce_add_sync(FULL, oldBits);
                    useOld = (oldBits >> 3) <= f.hSize + (f.newBits >> 3) || f.hSize + 12 >= n;
                }
                if (!useOld && f.hSize + 12 < n) { fresh = true; Fs = 0; r = f.newValue; }        // :716-719 the candidate table
            }
        }
        if (useOld) single ? chain_plan<1>(P, T, 0, x, sum, lane, r) : chain_plan<4>(P, T, 0, x, sum, lane, r);
        else if (fresh && single && !x.single) chain_plan<1>(P, x.cell, f.hSize, x, sum, lane, r);   // planned 4X, coded 1X
        if (is_err(r) || r == 0 || r >= (u64)n - ((n >> g.minGainLog) + 2)) kind = 0;             // size_t: n < minGain rejects nothing
        else if (r == 1) {                                      // RLE, unless a 1X stream of < 8 symbols fit in one byte
            const u8* const s = g.src[b];
            kind = (n >= 8 || __all_sync(FULL, lane >= n || s[lane] == s[0])) ? 1 : 0;
        } else kind = Fs != 0 ? 3 : 2;
    }
    bool const commit = kind == 2;
    if (commit) {
        #pragma unroll
        for (u32 i = 0; i < 8; i++) T[i] = x.cell[i];
        F = 1;                                                                                    // the block carries the new table
    }
    if (lane == 0) {
        P.state = kind == 2 || kind == 3 ? (single ? PLAN_EMIT_1X : PLAN_EMIT) : PLAN_FINAL;
        g.result[b] = r; g.kind[b] = kind; g.single[b] = single;
    }
    return commit;
}

// The decisions restate the repeat plan's rules and plan_streams inline: this loop is serial and latency-bound, and built on shared
// helpers ptxas scheduled the next block's loads later (1 chain of 32,768 blocks: 5 % slower on an H100).
// Geo = ChainDescs: the state goes back to the chain's entries, the RLE byte to the block, its header to blkHdr / blkHdrSize.
// Geo = ChainPackedDescs: none of these (the placement writes the RLE byte and the kinds); end[c] records what chainState needs.
// NS = 0 (mixed chains): the old-table sizing in each block's form, and the 1X blocks to the 1X emit launch.
// Geo = ChainPackedLiteralsDescs (NS = 0): zstd's literal policy, each step on copies of the state; see literals_step.
template <int NS, class Geo>
__global__ void __launch_bounds__(32 * CHAIN_WARPS)
huf_chain_kernel(Geo g, Plan* __restrict__ plans, const u32* __restrict__ malformed)
{
    constexpr bool PACKED = std::is_base_of_v<ChainPackedDescs, Geo>;
    unsigned const lane = threadIdx.x & 31u;
    if (*malformed) {              // every verdict srcSize_wrong, nothing else written and nothing emitted
        for (u64 b = blockIdx.x * (u64)blockDim.x + threadIdx.x; b < g.nBlocks; b += (u64)gridDim.x * blockDim.x) {
            g.result[b] = err(E_SRC_WRONG);
            plans[b].state = 1;
        }
        return;
    }
    u64 const c = blockIdx.x * (u64)CHAIN_WARPS + (threadIdx.x >> 5);
    if (c >= g.nChains) return;
    u32 const b0 = (u32)g.start[c], b1 = (u32)g.start[c + 1];
    if (b0 == b1) return;
    u32 T[8];                      // the chain's table (byte 3, padding, cleared), flag and header
    const u32* const t0 = g.ctable[c];
    #pragma unroll
    for (u32 i = 0; i < 8; i++) T[i] = t0[i * 32 + lane] & 0xFFFFFFu;
    int F = g.repeat[c];
    const u8* H = g.hdr[c];
    u64 HS = g.hdrSize[c];
    bool saved = false;
    u32 lastNew = CHAIN_NONE, lastSaved = CHAIN_NONE;                                             // packed only
    using Blk = std::conditional_t<NS == 0, ChainBlockMixed, ChainBlock>;
    Blk nx;
    chain_load(g, plans, b0, nx, lane);
    #pragma unroll 1
    for (u32 b = b0; b < b1; b++) {
        Blk const x = nx;
        if (b + 1 < b1) chain_load(g, plans, b + 1, nx, lane);
        ChainFact const& f = x.f;
        u32 const n = x.n;
        u32 sum[8];                                                                               // block counts
        #pragma unroll
        for (u32 i = 0; i < 8; i++) sum[i] = x.cnt[0][i] + x.cnt[1][i] + x.cnt[2][i] + x.cnt[3][i];
        if constexpr (std::is_same_v<Geo, ChainPackedLiteralsDescs>) {
            if (literals_step(g, plans[b], b, x, sum, T, F, lane)) lastNew = lastSaved = b;
            continue;
        }
        u64 r = 0;
        bool useOld = false, emit = false;
        if (f.kind == CF_ARGS) r = f.exitValue;                                                   // huf_compress.c:656-664
        else if (x.prefer && F == 2) useOld = true;                                               // :665-669
        else if (f.kind == CF_HIST) {                                                             // hist.c:128, :673-674
            r = f.exitValue;
            if constexpr (!PACKED) { if (r == 1 && lane == 0) x.dst[0] = g.src[b][0]; }       // the RLE byte (packed: the placement's)
        } else {
            if (F == 1) {                                                                         // :679-683 HUF_validateCTable
                bool bad = false;
                #pragma unroll
                for (u32 i = 0; i < 8; i++) bad |= sum[i] && (T[i] >> 16) == 0;
                if (__any_sync(FULL, bad)) F = 0;
            }
            if (x.prefer && F != 0) useOld = true;                                                // :685-689
            else if (is_err(f.hSize)) r = f.hSize;
            else {
                if (F != 0) {                                                                     // :703-713 HUF_estimateCompressedSize, old and new
                    u32 oldBits = 0;
                    #pragma unroll
                    for (u32 i = 0; i < 8; i++) oldBits += sum[i] * (T[i] >> 16);
                    oldBits = __reduce_add_sync(FULL, oldBits);
                    useOld = (oldBits >> 3) <= f.hSize + (f.newBits >> 3) || f.hSize + 12 >= n;
                }
                if (!useOld && f.hSize + 12 < n) {                                                // :716-719 the new table is saved, the flag set to none
                    #pragma unroll
                    for (u32 i = 0; i < 8; i++) T[i] = x.cell[i];
                    saved = true; F = 0; r = f.newValue; emit = r != 0;
                    if constexpr (PACKED) lastSaved = b;
                }
            }
        }
        Plan& P = plans[b];
        if (useOld) {                                                                             // HUF_compressCTable_internal with the old table
            if constexpr (NS == 0) emit = x.single ? chain_plan<1>(P, T, 0, x, sum, lane, r) : chain_plan<4>(P, T, 0, x, sum, lane, r);
            else {                                                                                // chain_plan<NS> with hs 0, inline
                auto const count = [&](int k, u32 i) { return NS == 4 ? x.cnt[k][i] : sum[i]; };
                u32 bits[NS], offs[NS], lens[NS];
                u64 total;
                stream_bits<NS>(T, count, bits);
                bool const fits = place_streams<NS>(bits, 0, x.cap, offs, lens, total);
                bool const ok = !(NS == 4 && (x.cap < 6 + 1 + 1 + 1 + 8 || n < 12)) && fits && total < (u64)n - 1;   // :564-565, :625
                r = ok ? total : 0; emit = ok;
                if (ok) {
                    #pragma unroll
                    for (u32 i = 0; i < 8; i++) P.ctable[i * 32 + lane] = T[i];
                    #pragma unroll
                    for (int k = 0; k < NS; k++) if (lane == (unsigned)k) { P.streamOff[k] = offs[k]; P.streamBytes[k] = lens[k]; }
                    if (lane == 0) { P.hSize = 0; P.total = (u32)total; }
                }
            }
        }
        bool const coded = !is_err(r) && r >= 2;                                                  // 1X: a 1-byte stream is emitted, not coded
        if (lane == 0) {
            if constexpr (NS == 0) P.state = emit ? (x.single ? PLAN_EMIT_1X : PLAN_EMIT) : PLAN_FINAL;
            else P.state = emit ? PLAN_EMIT : PLAN_FINAL;
            g.result[b] = r;
            if constexpr (!PACKED) {
                g.blkHdr[b] = coded && F != 0 ? H : nullptr;
                g.blkHdrSize[b] = coded && F != 0 ? HS : 0;
            }
        }
        if constexpr (PACKED) { if (coded && F == 0) lastNew = b; }
        if (coded && F == 0) { F = 1; H = x.dst; HS = r; }                                        // the block carries the new table: check it next
    }
    if constexpr (PACKED) {
        if (lane == 0) g.end[c] = ChainEnd{ lastNew, lastSaved, F };
        return;
    }
    if (saved) {
        #pragma unroll
        for (u32 i = 0; i < 8; i++) g.ctable[c][i * 32 + lane] = T[i];
    }
    if (lane == 0) { g.repeat[c] = F; g.hdr[c] = H; g.hdrSize[c] = HS; }
}

// ---------------------------------------------------------------------------------------------
// kernel 2: emit -- one CTA (4 warps) per block, one warp per stream, no serial section.
// A stream is the concatenation, last symbol first, of the codes.  The warp walks its segment from the
// end, 512 symbols at a time on aligned data: lane l takes the 8 symbols of one 64-bit piece of each of two
// 256-symbol groups (coalesced global reads, nothing staged), concatenates their codes (<= 88 bits per group),
// ONE warp scan of the two bit counts (packed in one register) gives both bit offsets, and the lane ORs its bits
// into a circular shared-memory window of the stream (aligned 32-bit words of the destination, whose position is
// known from the plan) with four reds at consecutive words; completed words leave 128 at a time, 16 bytes per lane.
// What bounds it was measured, not assumed: shared-memory wavefronts first (8-byte code cells), the ALU pipe now.
// ---------------------------------------------------------------------------------------------
constexpr int THREADS = 128;

// A 16-byte piece of a stream window that touches the stream's first or last bytes: only local bytes [a0, endByte) belong to
// this stream (the neighbours are another warp's), so it goes out byte by byte.  Out of line: once or twice per stream.  One copy
// per geometry: shared, the uniform batch's copy would lose the global stores the compiler proves for its kernel parameters.
template <class Geo>
static __device__ __noinline__ void store_piece_exact(u32* gw, u32 j, uint4 v, u32 a0, u32 endByte)
{
    u32 const wd[4] = { v.x, v.y, v.z, v.w };
    u8* const pb = reinterpret_cast<u8*>(gw + j);
    for (u32 t = 0; t < 16; t++) { u32 const at = 4 * j + t; if (at >= a0 && at < endByte) pb[t] = (u8)(wd[t >> 2] >> (8 * (t & 3))); }
}

// The 1X emit launch of a mixed chain call: the blocks of geometry G whose plan is PLAN_EMIT_1X
template <class G> struct Emit1X : G {};
template <class G> struct EmitState { static constexpr u32 value = PLAN_EMIT; };
template <class G> struct EmitState<Emit1X<G>> { static constexpr u32 value = PLAN_EMIT_1X; };

// NS = streams per block.  4X: a CTA of 4 warps, one per stream.  1X (descriptor batches only): a CTA of ONE warp whose
// segment is the whole block, and no jump table -- the same warp loop, 3 KB of shared memory per CTA (DESIGN.md 4.2).
template <class Geo, int NS>
__global__ void __launch_bounds__(32 * NS)
huf_emit_kernel(Geo g, u8* __restrict__ cbuf, const u8* __restrict__ src, const Plan* __restrict__ plans, const u32* __restrict__ sharedCT)
{
    static_assert(NS == 4 || NS == 1, "4X or 1X");
    constexpr int NT = 32 * NS;                                     // threads per CTA (THREADS for 4X)
    constexpr u32 W = 512;                                          // words of stream window per warp (a double group adds <= 176, < 128 wait for the next flush)
    __shared__ u32 ctab[256];                                       // cells nbBits | code << 8.  4-byte cells: the kernel is bound by shared-memory
                                                                    // wavefronts, and an 8-byte cell per lane costs two
    constexpr u32 WP = W + 4;                                       // + 3 spill words (a put writes up to 4 consecutive words, never wrapping) + 1 unused
    __shared__ __align__(16) u32 winAll[NS * WP];
    int const tid = threadIdx.x;
    unsigned const lane = tid & 31u; int const k = tid >> 5;
    u32 const b = blockIdx.x;
    const Plan& P = plans[b];
    if (P.state != EmitState<Geo>::value) return;                          // verdict already delivered by the plan kernel (or the other launch's block)
    u32 const n = enc_len(g, b);
    const u8* const s = enc_src(g, src, b);
    u8* const d = enc_dst(g, cbuf, b);
    u32 const hSize = P.hSize, total = P.total;

    {   const u32* const ct = sharedCT ? sharedCT : P.ctable;       // one caller-supplied table for the whole batch, or the block's own
        if constexpr (NS == 4) {
            u32 const c0 = ct[tid], c1 = ct[tid + 128];
            ctab[tid] = (c0 >> 16) | (c0 << 8 & 0xFFFF00u); ctab[tid + 128] = (c1 >> 16) | (c1 << 8 & 0xFFFF00u);
        } else {
            #pragma unroll
            for (int i = tid; i < 256; i += NT) { u32 const c0 = ct[i]; ctab[i] = (c0 >> 16) | (c0 << 8 & 0xFFFF00u); }
        }
    }
    for (u32 i = tid; i < NS * WP; i += NT) winAll[i] = 0;
    // tree header and (4X) jump table straight to the block (byte stores: the word they end in is shared with stream 1)
    for (u32 i = tid; i < hSize; i += NT) d[i] = P.header[i];
    if (NS == 4 && tid < 3) { u32 const v = P.streamBytes[tid]; d[hSize + 2 * tid] = (u8)v; d[hSize + 2 * tid + 1] = (u8)(v >> 8); }
    __syncthreads();
    {
        u32 const seg = (NS == 4) ? (n + 3) / 4 : n;
        int const segBeg = (int)(k * seg);
        int const segEnd = (k < NS - 1) ? (int)((k + 1) * seg) : (int)n;
        u32 sTab = (u32)__cvta_generic_to_shared(ctab);
        asm volatile("mov.u32 %0, %0;" : "+r"(sTab));               // keep it in a register (otherwise re-derived from the CTA id before every look-up)
        // The stream is built in a circular window of aligned 32-bit words of the destination and flushed as it grows, so a
        // CTA needs 6 KB of shared memory instead of an image of the whole block (occupancy: 10+ CTAs per SM instead of 6).
        u32* const win = winAll + k * WP;
        u32 sWin = (u32)__cvta_generic_to_shared(win);
        asm volatile("mov.u32 %0, %0;" : "+r"(sWin));
        u8* const gstart = d + P.streamOff[k];
        u32 const a0 = (u32)(reinterpret_cast<u64>(gstart) & 15);   // the window is 16-byte aligned in the destination: it is flushed in 16-byte pieces
        u32* const gw = reinterpret_cast<u32*>(gstart - a0);        // word j of the window <-> gw[j]
        u32 const sBytes = (k < NS - 1) ? P.streamBytes[k] : total - P.streamOff[NS - 1];
        u32 const endByte = a0 + sBytes;                            // stream occupies local bytes [a0, endByte)
        u32 bitpos = 8u * a0;
        u32 flushed = 0;                                            // words already written out
        auto lds32 = [&](u32 a) -> u32 { u32 v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a)); return v; };
        auto lds64 = [&](u32 o) -> uint2 { u32 const e = lds32(sTab + (o >> 1)); return make_uint2(e >> 8, e & 0xFFu); };   // {code, nbBits} of the cell at 8 * symbol
        auto red_or = [&](u32 a, u32 v) { asm volatile("red.shared.or.b32 [%0], %1;" :: "r"(a), "r"(v) : "memory"); };
        // three consecutive words, unconditionally: a predicated red compiles to a branch around it (4 more instructions each,
        // 162 instructions per 8 symbols in all), and a zero operand costs the shared-memory pipe no more than a one-lane red
        auto red_or3 = [&](u32 a, u32 v0, u32 v1, u32 v2) {
            asm volatile("red.shared.or.b32 [%0], %1; red.shared.or.b32 [%0+4], %2; red.shared.or.b32 [%0+8], %3;" :: "r"(a), "r"(v0), "r"(v1), "r"(v2) : "memory");
        };
        // warp scan of the lanes' bit counts: exclusive prefix in `excl`, returns the warp total
        auto scan = [&](u32 held, u32& excl) -> u32 {
            u32 incl = held;
            #pragma unroll
            for (int dd = 1; dd < 32; dd <<= 1)                     // shfl.up's own predicate says whether a source lane exists
                asm volatile("{ .reg .pred p; .reg .u32 t; shfl.sync.up.b32 t|p, %0, %1, 0, 0xffffffff; @p add.u32 %0, %0, t; }" : "+r"(incl) : "r"(dd));
            excl = incl - held;
            return __shfl_sync(FULL, incl, 31);
        };
        // ORs up to 64 bits (a0 | a1 << 32) into the window at bit offset `at`.  Only the first word's position wraps: words
        // W .. W+2 of the window are spill cells for words 0 .. 2 of the next lap, folded in when those are flushed.
        auto put = [&](u32 at, u32 x0, u32 x1) {
            u32 const sh = at & 31;
            red_or3(sWin + ((at >> 3) & (4 * (W - 1))), x0 << sh, __funnelshift_l(x0, x1, sh), __funnelshift_l(x1, 0, sh));
        };
        // the same for up to 88 bits (z0 | z1 << 32 | z2 << 64): four words
        auto put96 = [&](u32 at, u32 z0, u32 z1, u32 z2) {
            u32 const sh = at & 31;
            asm volatile("red.shared.or.b32 [%0], %1; red.shared.or.b32 [%0+4], %2; red.shared.or.b32 [%0+8], %3; red.shared.or.b32 [%0+12], %4;"
                         :: "r"(sWin + ((at >> 3) & (4 * (W - 1)))), "r"(z0 << sh), "r"(__funnelshift_l(z0, z1, sh)), "r"(__funnelshift_l(z1, z2, sh)),
                            "r"(__funnelshift_l(z2, 0, sh)) : "memory");
        };
        // Final words leave 128 at a time, one 16-byte piece per lane (the 32-words-per-flush version spent 50 of 135
        // instructions per 8 symbols here).  Between flushes < 128 final words wait, a double group adds <= 176 (+ 3 spill): < W.
        auto flush = [&](bool all) {
            u32 const upTo = all ? (endByte + 3) / 4 : (bitpos >> 5);
            if (!all && flushed + 128 > upTo) return;               // warp-uniform
            __syncwarp();
            while (all ? flushed < upTo : flushed + 128 <= upTo) {
                u32 const j = flushed + 4 * lane;
                if (j < upTo) {
                    u32 const i = j & (W - 1);
                    uint4 v = *reinterpret_cast<uint4*>(win + i);
                    *reinterpret_cast<uint4*>(win + i) = make_uint4(0, 0, 0, 0);
                    if (i == 0) { v.x |= win[W]; v.y |= win[W + 1]; v.z |= win[W + 2]; win[W] = 0; win[W + 1] = 0; win[W + 2] = 0; }
                    if (!all && (j != 0 || a0 == 0)) *reinterpret_cast<uint4*>(gw + j) = v;   // interior piece: below bitpos, inside the stream
                    else store_piece_exact<Geo>(gw, j, v, a0, endByte);  // first / last pieces
                }
                flushed += 128;
            }
        };
        auto place = [&](u32 x0, u32 x1, u32 held) -> u32 {         // lane's `held` bits go to bitpos + exclusive prefix
            u32 excl; u32 const sum = scan(held, excl);
            put(bitpos + excl, x0, x1);
            return sum;
        };
        constexpr int PF = 4;
        int hiCur = segEnd;                                         // symbols [segBeg, hiCur) are still to be coded
        // ---- groups of 256 symbols on 8-byte-aligned data: lane l codes the 8 symbols of one 64-bit piece, highest byte first.
        //      One scan serves 8 symbols; the two 4-symbol halves (<= 44 bits each) are placed separately. ----
        {
            bool const al8 = ((reinterpret_cast<u64>(s) + (u64)segEnd) & 7) == 0;
            int const nBig = al8 ? (segEnd - segBeg) / 256 : 0;
            const uint2* gq = reinterpret_cast<const uint2*>(s + segEnd) - 1 - lane;         // group j: piece gq[-32 j]
            auto half = [&](u32 w, u32& a0, u32& a1) -> u32 {        // 4 symbols of one word -> up to 44 bits
                // a cell is used as a shift amount as it is: the funnel shift takes the low 5 bits (lengths <= 11, pairs <= 22)
                u32 const e0 = lds32(sTab + 4 * __byte_perm(w, 0, 0x4443)), e1 = lds32(sTab + 4 * __byte_perm(w, 0, 0x4442));
                u32 const e2 = lds32(sTab + 4 * __byte_perm(w, 0, 0x4441)), e3 = lds32(sTab + 4 * __byte_perm(w, 0, 0x4440));
                u32 const p01 = (e0 >> 8) | __funnelshift_l(0, e1 >> 8, e0), l01 = e0 + e1;
                u32 const p23 = (e2 >> 8) | __funnelshift_l(0, e3 >> 8, e2), l23 = e2 + e3;
                a0 = p01 | __funnelshift_l(0, p23, l01); a1 = __funnelshift_l(p23, 0, l01);
                return (l01 + l23) & 0xFFu;
            };
            // Z = X | Y << lx for two halves (X < 2^lx, lx <= 44, Y < 2^44): the lane's 8 symbols as one string of <= 88 bits, so
            // that they cost 4 window ORs instead of 6 -- the kernel is bound by shared-memory wavefronts, not by instructions
            auto merge = [&](u32 x0, u32 x1, u32 lx, u32 y0, u32 y1, u32& z0, u32& z1, u32& z2) {
                u32 const t0 = __funnelshift_l(0, y0, lx), t1 = __funnelshift_l(y0, y1, lx), t2 = __funnelshift_l(y1, 0, lx);   // Y << (lx & 31)
                bool const far = (lx & 32u) != 0;
                z0 = x0 | (far ? 0u : t0); z1 = x1 | (far ? t0 : t1); z2 = far ? t1 : t2;
            };
            // Two groups of 256 symbols per scan: the two bit counts ride in the halves of one register (each total < 2^16).
            auto big2 = [&](uint2 curA, uint2 curB) {
                u32 x0, x1, y0, y1, za0, za1, za2, zb0, zb1, zb2;
                u32 lx = half(curA.y, x0, x1), ly = half(curA.x, y0, y1);           // .y holds the higher addresses: emitted first
                merge(x0, x1, lx, y0, y1, za0, za1, za2);
                u32 const la = lx + ly;
                lx = half(curB.y, x0, x1); ly = half(curB.x, y0, y1);
                merge(x0, x1, lx, y0, y1, zb0, zb1, zb2);
                u32 const lb = lx + ly;
                u32 excl; u32 const sum = scan(la | (lb << 16), excl);
                u32 const sumA = sum & 0xFFFFu;
                put96(bitpos + (excl & 0xFFFFu), za0, za1, za2);
                put96(bitpos + sumA + (excl >> 16), zb0, zb1, zb2);
                bitpos += sumA + (sum >> 16);
                flush(false);
            };
            constexpr int PB = 2;                                   // pieces in flight per register set (2 x 256 B per warp)
            int const rounds = nBig / PB;
            uint2 bufA[PB], bufB[PB];
            #pragma unroll
            for (int i = 0; i < PB; i++) { bufA[i] = rounds > 0 ? __ldg(gq - 32 * i) : make_uint2(0, 0); bufB[i] = make_uint2(0, 0); }
            auto round = [&](uint2 (&X)[PB], uint2 (&Y)[PB], int r) {
                gq -= 32 * PB;
                uint2 const c0 = X[0], c1 = X[1];
                if (r + 1 < rounds) { Y[0] = __ldg(gq); Y[1] = __ldg(gq - 32); }
                big2(c0, c1);
            };
            int r = 0;
            #pragma unroll 1
            for (; r + 1 < rounds; r += 2) { round(bufA, bufB, r); round(bufB, bufA, r + 1); }
            if (r < rounds) round(bufA, bufB, r);
            hiCur -= 256 * rounds * PB;
        }
        // ---- full groups of 128 symbols on word-aligned data: lane l codes the 4 symbols of one 32-bit word, highest byte first ----
        bool const wordAligned = ((reinterpret_cast<u64>(s) + (u64)hiCur) & 3) == 0;
        int const nFull = wordAligned ? (hiCur - segBeg) / 128 : 0;
        {
            const u32* gp = reinterpret_cast<const u32*>(s + hiCur) - 1 - lane;             // group j: word gp[-32 j]
            auto group = [&](u32 o0, u32 o1, u32 o2, u32 o3) {      // table offsets of the 4 symbols, emission order
                uint2 const e0 = lds64(o0), e1 = lds64(o1), e2 = lds64(o2), e3 = lds64(o3);
                u32 const p01 = e0.x | (e1.x << e0.y), l01 = e0.y + e1.y;           // <= 22 bits
                u32 const p23 = e2.x | (e3.x << e2.y), l23 = e2.y + e3.y;
                u32 const a0 = p01 | (p23 << l01), a1 = __funnelshift_l(p23, 0, l01);
                bitpos += place(a0, a1, l01 + l23);
                flush(false);
            };
            // rounds of PF groups: a raw word is unpacked one round after its load was issued, and it is dead (unpacked into
            // table offsets) before the next load is issued into its register -- warps issue in order, so no instruction
            // may touch a register with a load in flight
            int const rounds = nFull / PF;
            u32 bufA[PF], bufB[PF];                                 // two register sets, used alternately: nothing is ever rotated
            #pragma unroll
            for (int i = 0; i < PF; i++) { bufA[i] = rounds > 0 ? __ldg(gp - 32 * i) : 0u; bufB[i] = 0u; }
            auto round = [&](u32 (&X)[PF], u32 (&Y)[PF], int r) {   // code the groups held in X, request the next round into Y
                gp -= 32 * PF;
                bool const more = r + 1 < rounds;
                #pragma unroll
                for (int i = 0; i < PF; i++) {
                    u32 const cur = X[i];
                    if (more) Y[i] = __ldg(gp - 32 * i);
                    group(8 * (cur >> 24), 8 * __byte_perm(cur, 0, 0x4442), 8 * __byte_perm(cur, 0, 0x4441), 8 * (cur & 0xFFu));
                }
            };
            int r = 0;
            #pragma unroll 1
            for (; r + 1 < rounds; r += 2) { round(bufA, bufB, r); round(bufB, bufA, r + 1); }
            if (r < rounds) round(bufA, bufB, r);
            for (int j = rounds * PF; j < nFull; j++) {             // < PF groups left
                u32 const cur = __ldg(reinterpret_cast<const u32*>(s + hiCur) - 1 - lane - 32 * j);
                group(8 * (cur >> 24), 8 * __byte_perm(cur, 0, 0x4442), 8 * __byte_perm(cur, 0, 0x4441), 8 * (cur & 0xFFu));
            }
        }
        // ---- what is left (a partial group, or everything when the segment end is not word aligned) ----
        {
            int const rest = hiCur - 128 * nFull;
            auto fetch = [&](int hi) -> u32 {                       // the 4 symbols below hi-4*lane as one little-endian word
                int const top = hi - 4 * (int)lane;                 // exclusive
                u32 v = 0;
                if (top - 4 >= segBeg && ((reinterpret_cast<u64>(s + top) & 3) == 0)) v = __ldg(reinterpret_cast<const u32*>(s + top - 4));
                else if (top > segBeg) {
                    #pragma unroll
                    for (int j = 0; j < 4; j++) { int const i = top - 1 - j; if (i >= segBeg) v |= (u32)s[i] << (8 * (3 - j)); }
                }
                return v;
            };
            #pragma unroll 1
            for (int hi = rest; hi > segBeg; hi -= 128) {
                u32 const cur = fetch(hi);
                int const nValid = hi - 4 * (int)lane - segBeg;     // symbols available to this lane
                u64 acc = 0; u32 held = 0;                          // up to 48 bits
                #pragma unroll
                for (int j = 0; j < 4; j++) {
                    uint2 const e = lds64(8 * ((cur >> (8 * (3 - j))) & 0xFF));
                    if (j < nValid) { acc |= (u64)e.x << held; held += e.y; }
                }
                bitpos += place((u32)acc, (u32)(acc >> 32), held);
                flush(false);
            }
        }
        if (lane == 0) red_or(sWin + 4 * ((bitpos >> 5) & (W - 1)), 1u << (bitpos & 31));    // end mark (bitstream.h:256)
        bitpos += 1;
        flush(true);                                                // the rest, byte-exact at both ends
    }
}

// ---------------------------------------------------------------------------------------------
// Packed output (PackedDescs): the plan kernel has settled every block's verdict, so every block's stored length is known
// before anything is written.  Between plan and emit, a device-wide exclusive scan of the stored lengths (pack_dev.cuh) gives
// each block its offset, and placement settles what the plan kernel left open: the capacity verdict (the plan is made final,
// emit skips the block), the RLE byte and the raw copy of a block whose verdict is 0.
// ---------------------------------------------------------------------------------------------
struct HufPlace {
    typedef PackedDescs Geo;
    typedef Plan* Aux;
    static __device__ __forceinline__ u64 value(const PackedDescs& g, u64 b) { return g.result[b]; }
    static __device__ __forceinline__ u64 len(const PackedDescs& g, u64 b, u64 v) { return packed_len(v, g.srcSize[b]); }
    // the capacity verdict (nothing is written for a block that does not fit), the RLE byte; returns the block's final value
    static __device__ __forceinline__ u64 place(const PackedDescs& g, Plan* plans, u64 b, u64 v, u64 off, u64 len)
    {
        g.offset[b] = off;
        if (!is_err(v) && off + len > g.outCap) { v = err(E_DST_TOO_SMALL); g.result[b] = v; plans[b].state = 1; }
        else if (v == 1) g.out[off] = g.src[b][0];                     // a 1X block coded into one byte: emit overwrites it
        return v;
    }
};

// raw copy of every block whose verdict is 0, one CTA per block
__global__ void __launch_bounds__(pack::COPY_THREADS)
huf_pack_raw_kernel(PackedDescs g)
{
    u32 const b = blockIdx.x;
    if (g.result[b] != 0) return;                                   // a verdict of 0 that fits; everything else is placed already
    u32 const n = (u32)g.srcSize[b];                                // a verdict of 0 means srcSize <= HUF_BLOCK_MAX
    if (n == 0) return;
    const u8* const s = g.src[b];
    u8* const d = g.out + g.offset[b];
    pack::cta_copy<pack::COPY_THREADS, pack::COPY_UNROLL>(d, s, n);
}

// ---------------------------------------------------------------------------------------------
// Packed chains (ChainPackedDescs): the placement runs after huf_chain_kernel, whose decisions fix every value.  It is HufPlace's
// on the pk view (offsets, capacity verdict, RLE byte), then the kind of the final value: 0 raw, 1 RLE, 2 coded with its own tree
// header, 3 coded with the stream's previous table (the chain kernel left hSize 0 in its plan), 4 nothing stored.  Malformed
// geometry writes only the kinds (4, as every value is srcSize_wrong).  The raw copies and the emit then run as for PackedDescs, and chainState writes the streams' state.
// ---------------------------------------------------------------------------------------------
struct HufChainPlace {
    typedef ChainPackedDescs Geo;
    typedef Plan* Aux;
    static __device__ __forceinline__ u64 value(const ChainPackedDescs& g, u64 b) { return g.result[b]; }
    static __device__ __forceinline__ u64 len(const ChainPackedDescs& g, u64 b, u64 v) { return packed_len(v, g.srcSize[b]); }
    static __device__ __forceinline__ void place(const ChainPackedDescs& g, Plan* plans, u64 b, u64 v, u64 off, u64 len)
    {
        if (!*g.malformed) v = HufPlace::place(g.pk, plans, b, v, off, len);
        g.kind[b] = is_err(v) ? 4 : v == 0 ? 0 : v == 1 ? 1 : plans[b].hSize ? 2 : 3;
    }
};

// Packed chains under the literal policy: the chain kernel has written every kind, and a raw block's value may be anything (an
// error, a size the minimum gain rejected), so the stored length follows the kind: n raw, 1 RLE, the value for kinds 2 and 3.
// The capacity verdict makes a block kind 4; the RLE byte is the source's first.  Malformed geometry (the chain kernel wrote only
// the values): kinds 4, nothing placed.
struct HufLiteralsPlace {
    typedef ChainPackedLiteralsDescs Geo;
    typedef Plan* Aux;
    static __device__ __forceinline__ u64 value(const Geo& g, u64 b) { return g.result[b]; }
    static __device__ __forceinline__ u64 len(const Geo& g, u64 b, u64 v)
    {
        if (*g.malformed) return 0;
        u8 const k = g.kind[b];
        return k == 0 ? g.srcSize[b] : k == 1 ? 1 : k == 4 ? 0 : v;
    }
    static __device__ __forceinline__ void place(const Geo& g, Plan* plans, u64 b, u64, u64 off, u64 len)
    {
        if (*g.malformed) { g.kind[b] = 4; return; }
        g.pk.offset[b] = off;
        u8 const k = g.kind[b];
        if (k != 4 && off + len > g.pk.outCap) { g.result[b] = err(E_DST_TOO_SMALL); plans[b].state = PLAN_FINAL; g.kind[b] = 4; }
        else if (k == 1) g.pk.out[off] = g.src[b][0];
    }
};

// raw copy of every block of kind 0 (the literal policy's placement), one CTA per block
__global__ void __launch_bounds__(pack::COPY_THREADS)
huf_pack_raw_kinds_kernel(PackedDescs g, const u8* __restrict__ kind)
{
    u32 const b = blockIdx.x;
    if (kind[b] != 0) return;
    u32 const n = (u32)g.srcSize[b];                                // kind 0 means srcSize <= HUF_BLOCK_MAX
    if (n == 0) return;
    pack::cta_copy<pack::COPY_THREADS, pack::COPY_UNROLL>(g.out + g.offset[b], g.src[b], n);
}

// The streams' state, one warp per chain, once every block's place is known: nothing unless the geometry is sound and the total
// (*total, which also becomes offset[nBlocks]) fits.  Then the chain's flag, the table of its last block that saved one (that
// block's plan holds it, whatever its value), and the header of its last kind-2 block, at its place in out.
__global__ void __launch_bounds__(32 * CHAIN_WARPS)
huf_chain_state_kernel(ChainPackedDescs g, const Plan* __restrict__ plans, const u64* __restrict__ total)
{
    if (*g.malformed) return;
    u64 const tot = *total;
    if (blockIdx.x == 0 && threadIdx.x == 0) g.pk.offset[g.nBlocks] = tot;
    if (tot > g.pk.outCap) return;
    unsigned const lane = threadIdx.x & 31u;
    u64 const c = blockIdx.x * (u64)CHAIN_WARPS + (threadIdx.x >> 5);
    if (c >= g.nChains || g.start[c] == g.start[c + 1]) return;
    ChainEnd const e = g.end[c];
    if (e.lastSaved != CHAIN_NONE) {
        const u32* const t = plans[e.lastSaved].ctable;
        #pragma unroll
        for (u32 i = 0; i < 8; i++) g.ctable[c][i * 32 + lane] = t[i * 32 + lane];
    }
    if (lane == 0) {
        g.repeat[c] = e.flag;
        if (e.lastNew != CHAIN_NONE) { g.hdr[c] = g.pk.out + g.pk.offset[e.lastNew]; g.hdrSize[c] = g.result[e.lastNew]; }
    }
}

// ---------------------------------------------------------------------------------------------
// Table reuse (SURVEY.md 8f-3): every block of the batch coded with ONE caller-supplied HUF_CElt table, i.e. per block
// HUF_compress4X_usingCTable (lib/huf_compress.c:552-610).  No histogram, no tree, no header: the plan kernel disappears and
// this warp-per-block pass only sums the code lengths of each 4X segment (stream sizes, the writer's capacity rule).
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32 * PLAN_WARPS)
huf_sizes_kernel(BatchGeom g, u64* __restrict__ csizes, const u8* __restrict__ src, const u32* __restrict__ ct, Plan* __restrict__ plans)
{
    __shared__ u8 nbOf[256];
    unsigned const lane = threadIdx.x & 31u;
    for (u32 i = threadIdx.x; i < 256; i += blockDim.x) nbOf[i] = (u8)(ct[i] >> 16);
    __syncthreads();
    u32 const b = blockIdx.x * PLAN_WARPS + (threadIdx.x >> 5);
    if (b >= g.nBlocks) return;
    u32 const n = block_len(g, b);
    const u8* const s = src + (u64)b * g.blockSize;
    u64 const cap = g.slot;
    Plan& P = plans[b];
    if (cap < 6 + 1 + 1 + 1 + 8 || n < 12) { if (lane == 0) { P.state = 1; csizes[b] = 0; } return; }   // huf_compress.c:564-565
    u32 const seg = (n + 3) / 4;
    u32 bits[4];
    #pragma unroll 1
    for (u32 k = 0; k < 4; k++) {
        u32 const beg = k * seg, end = (k < 3) ? (k + 1) * seg : n;
        u32 acc = 0;
        u32 i = beg + lane * 4;
        if ((reinterpret_cast<u64>(s + beg) & 3) == 0) {
            for (; i + 4 <= end; i += 128) {
                u32 const w = __ldg(reinterpret_cast<const u32*>(s + i));
                acc += nbOf[w & 0xFF] + nbOf[(w >> 8) & 0xFF] + nbOf[(w >> 16) & 0xFF] + nbOf[w >> 24];
            }
            for (u32 t = i; t < end && t < i + 4; t++) acc += nbOf[s[t]];      // the lane whose word straddles the end
        } else for (u32 t = beg + lane; t < end; t += 32) acc += nbOf[s[t]];
        #pragma unroll
        for (int dlt = 16; dlt; dlt >>= 1) acc += __shfl_xor_sync(FULL, acc, dlt);
        bits[k] = acc;
    }
    u32 offs[4], lens[4];
    u64 total;
    if (!place_streams<4>(bits, 0, cap, offs, lens, total)) { if (lane == 0) { P.state = 1; csizes[b] = 0; } return; }
    if (lane < 4) { P.streamOff[lane] = offs[lane]; P.streamBytes[lane] = lens[lane]; }
    if (lane == 0) { P.hSize = 0; P.state = 0; P.total = (u32)total; csizes[b] = total; }
}

}  // namespace hufe

cudaError_t launch_huf_encode_using_ctable(const BatchGeom& g, void* cbuf, u64* csizes, const void* src, const u32* dCTable, cudaStream_t stream)
{
    if (g.nBlocks == 0) return cudaSuccess;
    cudaError_t e;
    hufe::Plan* const plans = (hufe::Plan*)stream_scratch(2, stream, sizeof(hufe::Plan) * (size_t)g.nBlocks, &e);
    if (e != cudaSuccess) return e;
    unsigned const grid = (g.nBlocks + hufe::PLAN_WARPS - 1) / hufe::PLAN_WARPS;
    hufe::huf_sizes_kernel<<<grid, 32 * hufe::PLAN_WARPS, 0, stream>>>(g, csizes, (const u8*)src, dCTable, plans);
    hufe::huf_emit_kernel<BatchGeom, 4><<<g.nBlocks, hufe::THREADS, 0, stream>>>(g, (u8*)cbuf, (const u8*)src, plans, dCTable);
    return cudaGetLastError();
}

namespace {
// the emit kernel's geometry argument: packed chains are emitted as the packed blocks they are, everything else as itself
template <class Geo> const Geo& emit_view(const Geo& g) { return g; }
const PackedDescs& emit_view(const ChainPackedDescs& g) { return g.pk; }

template <class Geo, int NS>
cudaError_t huf_encode(const Geo& g, void* cbuf, u64* csizes, const void* src, unsigned msv, unsigned tlog, cudaStream_t stream)
{
    if (g.nBlocks == 0) return cudaSuccess;
    cudaError_t e;
    // Plan scratch (3.2 KB per block): the per-stream grow-only buffer launch_huf_encode_using_ctable also takes its plans from.
    hufe::Plan* const plans = (hufe::Plan*)stream_scratch(2, stream, sizeof(hufe::Plan) * (size_t)g.nBlocks, &e);
    if (e != cudaSuccess) return e;
    size_t const smem = sizeof(hufe::PlanCta);
    static SmemOptIn optin;
    e = optin.ensure(hufe::huf_plan_kernel<Geo, NS>, current_device(), (int)smem);
    if (e != cudaSuccess) return e;
    constexpr bool chain = std::is_base_of_v<ChainDescs, Geo>;
    constexpr bool chainPacked = std::is_base_of_v<ChainPackedDescs, Geo>;
    constexpr bool packed = std::is_same_v<Geo, PackedDescs>;
    using EmitGeo = std::conditional_t<chainPacked, PackedDescs,    // the plan holds the chosen table
                                       std::conditional_t<std::is_same_v<Geo, RepeatDescs> || chain, BlockDescs, Geo>>;
    u64* tileSum = nullptr;                                         // packed: one word per scan tile (packed chains: + the total)
    if constexpr (packed || chainPacked) {
        tileSum = (u64*)stream_scratch(4, stream, sizeof(u64) * (pack::tiles_of(g.nBlocks) + chainPacked), &e);
        if (e != cudaSuccess) return e;
    }
    Geo gx = g;
    u32* malformed = nullptr;                                       // chains: the geometry verdict, then one fact per block
    if constexpr (chain) {
        malformed = (u32*)stream_scratch(9, stream, sizeof(u32), &e);
        if (e == cudaSuccess) gx.fact = (ChainFact*)stream_scratch(10, stream, sizeof(ChainFact) * (size_t)g.nBlocks, &e);
        if constexpr (chainPacked) {                                // and one end record per chain
            gx.malformed = malformed;
            if (e == cudaSuccess) gx.end = (ChainEnd*)stream_scratch(11, stream, sizeof(ChainEnd) * ((size_t)g.nChains + 1), &e);
        }
        if (e != cudaSuccess) return e;
    }
    unsigned const grid = (g.nBlocks + hufe::GROUP - 1) / hufe::GROUP;
    hufe::huf_plan_kernel<Geo, NS><<<grid, 32 * hufe::PLAN_WARPS, smem, stream>>>(gx, (u8*)cbuf, csizes, (const u8*)src, msv, tlog, plans);
    if constexpr (packed) {                                         // offsets, capacity verdicts, RLE bytes, raw copies; then emit
        pack::launch_pack<hufe::HufPlace>(gx, tileSum, gx.offset + gx.nBlocks, plans, stream);
        hufe::huf_pack_raw_kernel<<<gx.nBlocks, pack::COPY_THREADS, 0, stream>>>(gx);
    }
    if constexpr (chain) {
        hufe::huf_chain_check_kernel<<<1, 1024, 0, stream>>>(gx.start, gx.nChains, gx.nBlocks, malformed);
        u64 const cgrid = ((u64)gx.nChains + hufe::CHAIN_WARPS - 1) / hufe::CHAIN_WARPS;
        hufe::huf_chain_kernel<NS, Geo><<<(unsigned)(cgrid ? cgrid : 1), 32 * hufe::CHAIN_WARPS, 0, stream>>>(gx, plans, malformed);
    }
    if constexpr (std::is_same_v<Geo, ChainPackedLiteralsDescs>) {  // offsets by the decided kinds, capacity verdicts, RLE bytes, raw copies
        pack::launch_pack<hufe::HufLiteralsPlace>(gx, tileSum, tileSum + pack::tiles_of(gx.nBlocks), plans, stream);
        hufe::huf_pack_raw_kinds_kernel<<<gx.nBlocks, pack::COPY_THREADS, 0, stream>>>(gx.pk, gx.kind);
    } else if constexpr (chainPacked) {                             // offsets, kinds, capacity verdicts, RLE bytes, raw copies; then emit
        pack::launch_pack<hufe::HufChainPlace>(gx, tileSum, tileSum + pack::tiles_of(gx.nBlocks), plans, stream);
        hufe::huf_pack_raw_kernel<<<gx.nBlocks, pack::COPY_THREADS, 0, stream>>>(gx.pk);
    }
    if constexpr (NS == 0) {                                        // mixed: a 4X launch and a 1X launch, each passing the other's blocks by
        hufe::Emit1X<EmitGeo> v1;
        if constexpr (chainPacked) static_cast<PackedDescs&>(v1) = gx.pk;
        else static_cast<BlockDescs&>(v1) = gx;
        EmitGeo const& v4 = v1;
        hufe::huf_emit_kernel<EmitGeo, 4><<<gx.nBlocks, 32 * 4, 0, stream>>>(v4, (u8*)cbuf, (const u8*)src, plans, nullptr);
        hufe::huf_emit_kernel<hufe::Emit1X<EmitGeo>, 1><<<gx.nBlocks, 32, 0, stream>>>(v1, (u8*)cbuf, (const u8*)src, plans, nullptr);
    } else hufe::huf_emit_kernel<EmitGeo, NS><<<gx.nBlocks, 32 * NS, 0, stream>>>(emit_view(gx), (u8*)cbuf, (const u8*)src, plans, nullptr);
    if constexpr (chainPacked) {                                    // the streams' state, if the total fits
        u64 const cgrid = ((u64)gx.nChains + hufe::CHAIN_WARPS - 1) / hufe::CHAIN_WARPS;
        hufe::huf_chain_state_kernel<<<(unsigned)(cgrid ? cgrid : 1), 32 * hufe::CHAIN_WARPS, 0, stream>>>(
            gx, plans, tileSum + pack::tiles_of(gx.nBlocks));
    }
    return cudaGetLastError();
}
}  // namespace

cudaError_t launch_huf_encode(const BatchGeom& g, void* cbuf, u64* csizes, const void* src,
                              unsigned msv, unsigned tlog, cudaStream_t stream)
{
    return huf_encode<BatchGeom, 4>(g, cbuf, csizes, src, msv, tlog, stream);
}

// The descriptor geometries (launchers.h launch_huf_encode_descs); the host never reads their arrays:
//   BlockDescs        HUF_compress2 / HUF_compress1X per block
//   PackedDescs       the same, with the scan and placement between plan and emit
//   RepeatDescs       HUF_compress4X_repeat / HUF_compress1X_repeat per block (table reuse)
//   ChainDescs        chains of table reuse: plan, the chains' decisions, emit -- the repeat call block after block per chain
//   ChainPackedDescs  packed chains: plan, the chains' decisions, the placement scan and raw copies, emit, the streams' state
//   Mixed<...>        either chain geometry with a form per block (stream mode 0): the same steps, and two emit launches (4X, 1X)
//   ChainPackedLiteralsDescs  packed chains under zstd's literal policy, stream mode 0 only: as Mixed<ChainPackedDescs>, the forms
//                     and kinds decided by the chain kernel, the placement and raw copies by kind
namespace {
// the geometry a call runs as when every block takes the form nStreams names: a Mixed<Base> runs as its Base
template <class Geo> struct OneForm { using type = Geo; };
template <class Base> struct OneForm<Mixed<Base>> { using type = Base; };
}  // namespace
template <class Geo>
cudaError_t launch_huf_encode_descs(const Geo& g, int nStreams, unsigned msv, unsigned tlog, cudaStream_t stream)
{
    using One = typename OneForm<Geo>::type;
    if constexpr (std::is_same_v<Geo, ChainPackedLiteralsDescs>) {
        return nStreams ? cudaErrorInvalidValue : huf_encode<Geo, 0>(g, nullptr, nullptr, nullptr, msv, tlog, stream);
    } else {
        if constexpr (!std::is_same_v<One, Geo>)
            if (nStreams == 0) return huf_encode<Geo, 0>(g, nullptr, nullptr, nullptr, msv, tlog, stream);
        return nStreams == 1 ? huf_encode<One, 1>(g, nullptr, nullptr, nullptr, msv, tlog, stream)
                             : huf_encode<One, 4>(g, nullptr, nullptr, nullptr, msv, tlog, stream);
    }
}
// defined for these geometries only: a call on any other fails to link
template cudaError_t launch_huf_encode_descs(const BlockDescs&, int, unsigned, unsigned, cudaStream_t);
template cudaError_t launch_huf_encode_descs(const PackedDescs&, int, unsigned, unsigned, cudaStream_t);
template cudaError_t launch_huf_encode_descs(const RepeatDescs&, int, unsigned, unsigned, cudaStream_t);
template cudaError_t launch_huf_encode_descs(const ChainDescs&, int, unsigned, unsigned, cudaStream_t);
template cudaError_t launch_huf_encode_descs(const ChainPackedDescs&, int, unsigned, unsigned, cudaStream_t);
template cudaError_t launch_huf_encode_descs(const ChainMixedDescs&, int, unsigned, unsigned, cudaStream_t);
template cudaError_t launch_huf_encode_descs(const ChainPackedMixedDescs&, int, unsigned, unsigned, cudaStream_t);
template cudaError_t launch_huf_encode_descs(const ChainPackedLiteralsDescs&, int, unsigned, unsigned, cudaStream_t);

// the chain geometry's verdict (start[0] == 0, start[nChains] == nBlocks, never decreasing) to *malformed, for the decoders
cudaError_t launch_huf_chain_check(const u64* start, u32 nChains, u32 nBlocks, u32* malformed, cudaStream_t stream)
{
    hufe::huf_chain_check_kernel<<<1, 1024, 0, stream>>>(start, nChains, nBlocks, malformed);
    return cudaGetLastError();
}

}  // namespace fseb
