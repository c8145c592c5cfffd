// fse_codec.cu -- batched FSE (tANS) block encode / decode for sm_90a, byte and 16-bit alphabets.
//
// Replaces, per block, the CPU chains
//   FSE_compress2 -> FSE_compress_wksp          lib/fse_compress.c:632-693
//       HIST_count_wksp, FSE_optimalTableLog, FSE_normalizeCount, FSE_writeNCount,
//       FSE_buildCTable_wksp, FSE_compress_usingCTable (2 interleaved states)
//   FSE_decompress -> FSE_decompress_wksp       lib/fse_decompress.c:255-283
//       FSE_readNCount, FSE_buildDTable, FSE_decompress_usingDTable (fast / safe variants)
//   FSE_compressU16 / FSE_decompressU16         lib/fseU16.c:203-251,306-329 (single state)
//
// What the format allows on a GPU (DESIGN.md section 4.3): a block is ONE dependent chain on decode
// (both states share one bitstream) and TWO on encode; each step is a table look-up whose index is
// the previous step's result, and the tables (CTable 10 KB, DTable 12-16 KB at tableLog 12) bound how
// many chains an SM keeps resident.  The batch kernels are cut around the chains:
//   fse_encode_cta_kernel  a CTA owns 16 blocks; all warps run the front half (histogram .. CTable), then one
//                          CHAIN warp walks the tables (lane pair = the two states of a block) and seven EMITTER
//                          warps turn its (state, nbBits) records into stream words (named-barrier ring)
//   fse_decode_cta_kernel  a CTA owns 8 blocks; its warps build the tables, then one lane per block decodes through
//                          a register bit window, check-free in the middle of the stream and on the exact
//                          byte-granular model (bitsrc_dev.cuh) near its ends
//   fse_encode_kernel      warp per block; takes the ragged last block and unaligned geometries
#include <cstdlib>
#include "common.cuh"
#include "launch_util.cuh"
#include "fse_dev.cuh"
#include "bitsrc_dev.cuh"

namespace fseb {
namespace fsek {

constexpr int WARPS = 4;
constexpr int THREADS = 32 * WARPS;
constexpr unsigned FULL = 0xFFFFFFFFu;

// ---- warp-cooperative symbol spreading ------------------------------------------------------
// Visit v (0..size-1) of the reference walk lands on cell (v*stride) & mask; cells above `high`
// (parked low-probability symbols) are skipped; the r-th accepted visit receives the symbol whose
// cumulative normalized count covers r.  put(cell, symbol) is called exactly once per cell.
// cum: u16[msv+2] exclusive cumulative counts of the positive norms (shared memory).
template <typename Put>
__device__ inline bool warp_spread(const short* norm, const u16* cum, unsigned msv, unsigned tl, Put put)
{
    unsigned const lane = lane_id();
    u32 const size = 1u << tl, mask = size - 1, stride = (size >> 1) + (size >> 3) + 3;
    // parked symbols, in symbol order, from the top cell downwards (tiny: one lane)
    u32 high = size - 1;
    if (lane == 0) for (u32 s = 0; s <= msv; s++) if (norm[s] == -1) put(high--, s);
    high = __shfl_sync(FULL, high, 0);
    u32 const nAccept = cum[msv + 1];
    u32 accepted = 0;
    for (u32 v0 = 0; v0 < size; v0 += 32) {
        u32 const v = v0 + lane;
        u32 const pos = (v * stride) & mask;
        bool const ok = pos <= high;
        u32 const votes = __ballot_sync(FULL, ok);
        u32 const r = accepted + __popc(votes & ((1u << lane) - 1));
        if (ok && r < nAccept) {
            u32 lo = 0, hi = msv + 1;                    // largest s with cum[s] <= r  (skips empty symbols)
            while (hi - lo > 1) { u32 const mid = (lo + hi) >> 1; if (cum[mid] <= r) lo = mid; else hi = mid; }
            put(pos, lo);
        }
        accepted += __popc(votes);
    }
    // the reference requires the walk to close on cell 0 after the last placement
    // (fse_decompress.c:113); with sum(|norm|) == size that is equivalent to accepting exactly nAccept visits.
    return accepted == nAccept;
}

// =================================================================================================
// decode
// =================================================================================================
template <bool WIDE> struct DecCfg;
template <> struct DecCfg<false> { static constexpr unsigned MSV = FSE_MAX_SV, TL = FSE_MAX_TLOG, CELLS = 1u << FSE_MAX_TLOG; };
template <> struct DecCfg<true>  { static constexpr unsigned MSV = U16_MAX_SV, TL = U16_MAX_TLOG, CELLS = 1u << U16_MAX_TLOG; };

// =================================================================================================
// decode, batch kernel.  A tANS decode is one serial chain per block (state -> cell -> bits -> state) that the
// format does not let us split, and its table is what limits how many chains an SM keeps resident.  So: a CTA
// owns DK blocks, its four warps parse the headers and build the tables (bytes: 12-bit next-state base + 4-bit
// nbBits in a u16 cell plus a separate symbol byte -- 12 KB instead of 16 KB per block), then warp 0 runs ONE LANE
// PER BLOCK.  A lane reads its stream straight from global memory through a 96-bit register window (aligned
// 32-bit words, next word prefetched) with a bit cursor, so a symbol costs two table loads and ~8 ALU ops.
// The reference's reader is byte-granular (BIT_reloadDStream); its bookkeeping only matters near the two ends
// of the stream, so the lane runs check-free chunks whose length is bounded so that every reload the reference
// would do in between returns "unfinished" (ptr stays >= start + 8) and the output bound holds, then hands the
// last few bytes to the exact byte-granular model (bitsrc_dev.cuh) which also produces the verdicts.
// =================================================================================================
constexpr int DTHREADS = 128;
template <bool WIDE> struct DecCta {
    static constexpr unsigned DK = WIDE ? 3 : 8;                    // blocks per CTA; two CTAs per SM
    static constexpr unsigned MSV = DecCfg<WIDE>::MSV, CELLS = DecCfg<WIDE>::CELLS;
    static constexpr unsigned TAB_BYTES = WIDE ? CELLS * 4 : CELLS * 3;
    static constexpr unsigned WB = WIDE ? 7 : 6;                    // most stream bytes one 4-symbol iteration can retire ((7 + 4 * tableLog) >> 3)
    struct alignas(16) Scratch { short norm[MSV + 1]; u16 cum[MSV + 3]; u16 nextOf[MSV + 1]; };
    struct alignas(16) Smem {
        u8 tab[DK][TAB_BYTES];
        Scratch scratch[DTHREADS / 32];
        u32 go[DK], tl[DK], fast[DK], hdr[DK];
    };
};
__device__ __forceinline__ u32 lds_u16(u32 addr) { u32 v; asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(addr)); return v; }
__device__ __forceinline__ u32 lds_u8(u32 addr)  { u32 v; asm volatile("ld.shared.u8 %0, [%1];"  : "=r"(v) : "r"(addr)); return v; }
__device__ __forceinline__ u32 lds_u32(u32 addr) { u32 v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr)); return v; }

// Table of one block, one warp.  bytes: tab = u16 cell[size] (nextState base | nbBits << 12) then u8 symbol[size];
// U16: u32 cell[size] (base | nbBits << 16 | symbol << 20).  Same construction as warp_build_dtable.
template <bool WIDE>
__device__ inline u64 warp_build_dtable_split(typename DecCta<WIDE>::Scratch& w, u8* tab, unsigned msv, unsigned tl, unsigned& fastOut)
{
    unsigned const lane = lane_id();
    u32 const size = 1u << tl;
    if (msv > DecCfg<WIDE>::MSV) return err(E_MSV_TOO_LARGE);
    if (tl > DecCfg<WIDE>::TL) return err(E_TLOG_TOO_LARGE);
    unsigned fast = 1;
    if (lane == 0) {
        u32 acc = 0;
        for (u32 s = 0; s <= msv; s++) {
            w.cum[s] = (u16)acc;
            int const n = w.norm[s];
            if (n == -1) w.nextOf[s] = 1;
            else { if (n >= (int)(1u << (tl - 1))) fast = 0; w.nextOf[s] = (u16)n; if (n > 0) acc += (u32)n; }
        }
        w.cum[msv + 1] = (u16)acc;
    }
    fastOut = __shfl_sync(FULL, fast, 0);
    __syncwarp();
    u16* const t16 = reinterpret_cast<u16*>(tab);
    u8*  const s8  = tab + 2 * DecCfg<false>::CELLS;
    u32* const c32 = reinterpret_cast<u32*>(tab);
    bool const closed = warp_spread(w.norm, w.cum, msv, tl, [&](u32 cell, u32 sym) { if (WIDE) c32[cell] = sym; else s8[cell] = (u8)sym; });
    __syncwarp();
    if (!closed) return err(E_GENERIC);
    for (u32 u0 = 0; u0 < size; u0 += 32) {                       // the k-th cell (ascending) of symbol s gets x = norm[s] + k  (fse_decompress.c:117-124)
        u32 const u = u0 + lane;
        u32 const sym = WIDE ? c32[u] : (u32)s8[u];
        u32 const peers = __match_any_sync(FULL, sym);
        u32 const x = w.nextOf[sym] + __popc(peers & ((1u << lane) - 1));
        __syncwarp();
        if ((peers >> lane) == 1u) w.nextOf[sym] = (u16)(w.nextOf[sym] + __popc(peers));
        u32 const nb = tl - hibit(x);
        u32 const ns = ((x << nb) - size) & 0xFFFF;
        if (WIDE) c32[u] = ns | (nb << 16) | (sym << 20); else t16[u] = (u16)(ns | (nb << 12));
        __syncwarp();
    }
    return 0;
}

// exact-model steps on the split table (tail of a stream)
template <bool WIDE>
__device__ __forceinline__ u32 tab_step(u32& state, BitSrc& b, u32 tabAddr, bool fast)
{
    if (WIDE) {
        u32 const cell = lds_u32(tabAddr + 4 * state);
        state = (cell & 0xFFFF) + (u32)bs_read(b, (cell >> 16) & 0xF);
        return cell >> 20;
    }
    u32 const cell = lds_u16(tabAddr + 2 * state);
    u32 const sym = lds_u8(tabAddr + 2 * DecCfg<false>::CELLS + state);
    u32 const nb = cell >> 12;
    state = (cell & 0xFFF) + (u32)(fast ? bs_read_fast(b, nb) : bs_read(b, nb));
    return sym;
}

// Descriptor blocks only: the verdict a block gets before its header is read (0: decode it).  The batch tier's limits on the
// literal sizes; a U16 destination must hold whole 16-bit symbols.
template <bool WIDE>
__device__ __forceinline__ u64 dec_desc_verdict(const BlockDescs& g, u32 b)
{
    if (WIDE && (reinterpret_cast<u64>(g.dst[b]) & 1)) return err(E_GENERIC);
    if (g.srcSize[b] > FSE_BLOCK_MAX || fse_dec_len(g, b, WIDE) > FSE_BLOCK_MAX) return err(E_SRC_WRONG);
    return 0;
}

// Geo: BatchGeom (uniform batch; csizes / orig carry the harness' stored-block conventions) or BlockDescs (sizes taken
// literally; a U16 block's capacity and result count symbols).
template <bool WIDE, class Geo>
__global__ void __launch_bounds__(DTHREADS, 2)
fse_decode_cta_kernel(Geo g, u8* __restrict__ dst, const u8* __restrict__ cbuf, const u64* __restrict__ csizes,
                      u64* __restrict__ results, const u8* __restrict__ orig)
{
    typedef DecCta<WIDE> C;
    constexpr unsigned DK = C::DK;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    typename C::Smem& sm = *reinterpret_cast<typename C::Smem*>(smem_raw);
    unsigned const lane = lane_id(), warp = threadIdx.x >> 5;
    u32 const b0 = blockIdx.x * DK;
    u32 const nHere = g.nBlocks - b0 < DK ? g.nBlocks - b0 : DK;
    if constexpr (Geo::DESCS) { csizes = g.srcSize; results = g.result; }    // indexed by block, as the uniform batch's

    // ---- phase 1: stored-block conventions, header, table: one warp per block ----
    if (threadIdx.x < DK) sm.go[threadIdx.x] = 0;
    __syncthreads();
    for (u32 blk = warp; blk < nHere; blk += DTHREADS / 32) {
        u32 const b = b0 + blk;
        u64 const cs = csizes[b];
        const u8* c;
        if constexpr (Geo::DESCS) {
            c = dec_src(g, cbuf, b);
            u64 const v = dec_desc_verdict<WIDE>(g, b);
            if (v) { if (lane == 0) results[b] = v; continue; }
        } else {
            u32 const n = block_len(g, b);
            u8* const out = dst + (u64)b * g.blockSize;
            c = cbuf + (u64)b * g.slot;
            if (is_err(cs)) { if (lane == 0) results[b] = cs; continue; }
            if (cs == 0 || (cs == 1 && !WIDE)) {                    // the harness' conventions for stored blocks (bench.c:393-402)
                if (orig) {
                    const u8* const o = orig + (u64)b * g.blockSize;
                    if (cs == 0) for (u32 i = lane; i < n; i += 32) out[i] = o[i];
                    else { u8 const v = o[0]; for (u32 i = lane; i < n; i += 32) out[i] = v; }
                }
                if (lane == 0) results[b] = orig ? n : 0;
                continue;
            }
        }
        typename C::Scratch& w = sm.scratch[warp];
        u64 h = 0; unsigned tl = 0, msv = C::MSV;
        if (lane == 0) {
            if (WIDE && cs < 2) h = err(E_SRC_WRONG);                                   // fseU16.c:317
            else h = d_read_ncount(w.norm, &msv, &tl, c, cs);
            if (!WIDE && !is_err(h) && tl > FSE_MAX_TLOG) h = err(E_TLOG_TOO_LARGE);    // fse_decompress.c:266
        }
        h = __shfl_sync(FULL, h, 0); tl = __shfl_sync(FULL, tl, 0); msv = __shfl_sync(FULL, msv, 0);
        if (is_err(h)) { if (lane == 0) results[b] = h; continue; }
        __syncwarp();
        unsigned fast = 0;
        u64 const e = warp_build_dtable_split<WIDE>(w, sm.tab[blk], msv, tl, fast);
        if (is_err(e)) { if (lane == 0) results[b] = e; continue; }
        if (lane == 0) { sm.go[blk] = 1; sm.tl[blk] = tl; sm.fast[blk] = fast; sm.hdr[blk] = (u32)h; }
        __syncwarp();
    }
    __syncthreads();
    if (warp != 0) return;

    // ---- phase 2: one lane per block ----
    bool const mine = lane < DK && sm.go[lane < DK ? lane : 0];
    u32 const blk = mine ? lane : 0;
    u32 const b = b0 + blk;
    u32 const tl = sm.tl[blk];
    bool const fastMode = sm.fast[blk] != 0;
    u32 const tabAddr = (u32)__cvta_generic_to_shared(sm.tab[blk]);
    u32 const symAddr = tabAddr + 2 * DecCfg<false>::CELLS;
    u32 nBytes; u8* out; const u8* cs0;
    if constexpr (Geo::DESCS) { nBytes = mine ? (u32)fse_dec_len(g, b, WIDE) : 0; out = dec_dst(g, dst, b); cs0 = dec_src(g, cbuf, b); }
    else { nBytes = mine ? block_len(g, b) : 0; out = dst + (u64)b * g.blockSize; cs0 = cbuf + (u64)b * g.slot; }
    long long const omax = WIDE ? nBytes / 2 : nBytes;              // symbols
    u64 const lowest = reinterpret_cast<u64>(cs0) & ~15ull;          // nothing below the block's own slot is ever read
    BitSrc bs; bs.s = cs0; bs.len = 0; bs.at = 0; bs.w = 0; bs.used = 0;
    u32 s1 = 0, s2 = 0;
    long long op = 0;
    u64 ret = 0;
    int mode = mine ? 0 : 2;                                        // 0 = chunked fast region, 1 = exact tail, 2 = finished
    bool openErr = false;
    if (mine) {
        u64 const cs = csizes[b]; u32 const h = sm.hdr[blk];
        u64 const e = bs_open(bs, cs0 + h, cs - h);
        if (!WIDE) {
            if (is_err(e)) { ret = e; mode = 2; }
            else { s1 = (u32)bs_read(bs, tl); bs_refill(bs); s2 = (u32)bs_read(bs, tl); bs_refill(bs); }
        } else {
            if (cs - h < 1) { ret = err(E_CORRUPT); mode = 2; }      // the reference dereferences a NULL stream here (documented deviation)
            else { openErr = is_err(e); s1 = (u32)bs_read(bs, tl); bs_refill(bs); }    // fseU16.c:286 ignores the verdict
        }
    }
    (void)openErr;

    // Bit window of the check-free region: a 64-bit shift register hi:lo with `avail` valid bits at the top (the stream is read
    // downwards: the next bit is bit 31 of hi), q = the next 32-bit word, already loaded, p = the address below q.  A symbol
    // costs: two table loads, split the cell, take the top nbBits of hi, add, shift the register (2), count -- 11 instructions;
    // every two symbols a predicated refill (8) appends q when avail <= 32 and requests the next word, whose only reader is the
    // next refill (this warp issues in order and has nobody to hide behind: the kernel's time is its instruction count times
    // ~3.3 cycles -- the 96-bit register window with a bit cursor that this replaces took 21 instructions per symbol, a third of
    // them in its four-register rotation with a 64-bit bounds check).
    // Addresses: the stream pointer and the output pointer are kept as (low, high) register halves and only the low half moves
    // -- a predicated 64-bit decrement costs four instructions (add, add-with-carry, two selects), the 32-bit one a single
    // add.  A block whose compressed slot or output straddles a 4 GiB address boundary takes the exact path instead (sameHi).
    u32 hi = 0, lo = 0, avail = 0, q = 0, pLo = 0, pHi = 0;        // (pHi:pLo) = address of the next word to request
    u32 oLo = 0, oHi = 0;
    bool windowed = false;
    auto ldw = [&](u64 a) -> u32 { return a >= lowest ? __ldg(reinterpret_cast<const u32*>(a)) : 0u; };
    bool const al4 = ((reinterpret_cast<u64>(out) & (WIDE ? 7 : 3)) == 0);   // the check-free loop stores 4 symbols at once
    // The window reads aligned words in [lowest, round_up_4(end of the compressed block)): for descriptors, that extent is the
    // block's own; the uniform batch bounds it by the slot.
    bool sameHi;
    if constexpr (Geo::DESCS)
        sameHi = ((reinterpret_cast<u64>(out) + nBytes) >> 32) == (reinterpret_cast<u64>(out) >> 32)
              && ((reinterpret_cast<u64>(cs0) + (mine ? csizes[b] : 0) + 3) >> 32) == (lowest >> 32);
    else
        sameHi = ((reinterpret_cast<u64>(out) + nBytes) >> 32) == (reinterpret_cast<u64>(out) >> 32)
              && ((reinterpret_cast<u64>(cs0) + g.slot + 16) >> 32) == (lowest >> 32);
    constexpr u32 MARGIN = 24;                                      // container bytes that stay unread below a chunk: the window (8) + q (4)
                                                                    // + the word in flight (4) + alignment (3) never reach below the stream start
    for (;;) {
        // chunk length: every reload in between must see ptr >= start + 8, every iteration needs 4 output slots
        u32 m = 0;
        if (mode == 0) {
            if (al4 && sameHi && bs.len >= 8 && bs.at >= MARGIN && bs.used <= 7) {
                u64 const ms = (bs.at - MARGIN) / C::WB, mo = (u64)((omax - op) / 4);
                m = (u32)(ms < mo ? ms : mo);
            }
            if (m == 0) mode = 1;
        }
        u32 mm = mode == 0 ? m : 0xFFFFFFFFu;
        #pragma unroll
        for (int d = 16; d; d >>= 1) mm = min(mm, __shfl_xor_sync(FULL, mm, d));
        if (mm == 0xFFFFFFFFu) break;
        if (mode == 0) {
            if (!windowed) {                                        // stand the window on (at, used)
                u64 const A = reinterpret_cast<u64>(bs.s) + bs.at + 8;
                u64 const top4 = (A + 3) & ~3ull;
                u32 const k = (u32)(8 * (top4 - A)) + bs.used;     // <= 31
                u32 const w0 = ldw(top4 - 4), w1 = ldw(top4 - 8);
                hi = __funnelshift_l(w1, w0, k); lo = w1 << k; avail = 64 - k;
                q = ldw(top4 - 12); pLo = (u32)(top4 - 16); pHi = (u32)((top4 - 16) >> 32);
                windowed = true;
            }
            u32 const pLo0 = pLo, avail0 = avail;
            {   u64 const oa = reinterpret_cast<u64>(out) + (u64)op * (WIDE ? 2 : 1); oLo = (u32)oa; oHi = (u32)(oa >> 32); }
            u32 const oLo0 = oLo;
#define FSEB_REFILL() asm volatile("{\n\t.reg .pred a;\n\t.reg .b32 t;\n\t.reg .b64 pa;\n\t" \
                "setp.le.u32 a, %3, 32;\n\t" \
                "shf.r.clamp.b32 t, %2, 0, %3;\n\t"          /* q >> avail (0 when avail == 32) */ \
                "@a or.b32 %0, %0, t;\n\t" \
                "@a shf.r.clamp.b32 %1, 0, %2, %3;\n\t"      /* q << (32 - avail) */ \
                "@a add.u32 %3, %3, 32;\n\t" \
                "mov.b64 pa, {%4, %5};\n\t" \
                "@a ld.global.nc.u32 %2, [pa];\n\t" \
                "@a add.u32 %4, %4, -4;\n\t}" \
                : "+r"(hi), "+r"(lo), "+r"(q), "+r"(avail), "+r"(pLo) : "r"(pHi) : "memory")
#define FSEB_STORE(V0, V1) do { \
                if (WIDE) asm volatile("{\n\t.reg .b64 oa;\n\tmov.b64 oa, {%0, %1};\n\tst.global.v2.u32 [oa], {%2, %3};\n\t}" :: "r"(oLo), "r"(oHi), "r"(V0), "r"(V1) : "memory"); \
                else      asm volatile("{\n\t.reg .b64 oa;\n\tmov.b64 oa, {%0, %1};\n\tst.global.u32 [oa], %2;\n\t}" :: "r"(oLo), "r"(oHi), "r"(V0) : "memory"); \
                oLo += WIDE ? 8 : 4; } while (0)
#define FSEB_PSTEP(ST, SYM) do { \
                u32 cell_, nb_, base_; \
                if (WIDE) { cell_ = lds_u32(tabAddr + 4 * ST); SYM = cell_ >> 20; nb_ = (cell_ >> 16) & 0xF; base_ = cell_ & 0xFFFF; } \
                else { cell_ = lds_u16(tabAddr + 2 * ST); SYM = lds_u8(symAddr + ST); nb_ = cell_ >> 12; base_ = cell_ & 0xFFF; } \
                ST = base_ + __funnelshift_l(hi, 0, nb_); \
                hi = __funnelshift_l(lo, hi, nb_); lo <<= nb_; avail -= nb_; } while (0)
            #pragma unroll 1
            for (u32 it = 0; it < mm; it++) {
                u32 a0, a1, a2, a3;
                if (!WIDE) {
                    FSEB_PSTEP(s1, a0); FSEB_PSTEP(s2, a1); FSEB_REFILL();
                    FSEB_PSTEP(s1, a2); FSEB_PSTEP(s2, a3); FSEB_REFILL();
                    FSEB_STORE(a0 | (a1 << 8) | (a2 << 16) | (a3 << 24), 0u);
                } else {
                    FSEB_PSTEP(s1, a0); FSEB_PSTEP(s1, a1); FSEB_REFILL();
                    FSEB_PSTEP(s1, a2); FSEB_PSTEP(s1, a3); FSEB_REFILL();
                    FSEB_STORE(a0 | (a1 << 16), a2 | (a3 << 16));
                }
            }
            op += (long long)((oLo - oLo0) / (WIDE ? 2 : 1));
#undef FSEB_PSTEP
#undef FSEB_REFILL
#undef FSEB_STORE
            u64 const tot = (u64)bs.used + 8ull * (pLo0 - pLo) + avail0 - avail;   // (64-bit left to right: avail may exceed avail0)   // bits retired in this chunk, carried into the byte-granular counters
            bs.at -= tot >> 3; bs.used = (unsigned)(tot & 7);
        }
    }
    // ---- exact tail on the byte-granular model ----
    if (mode == 1) {
        if (windowed) bs.w = ld64u(bs.s + bs.at);
        if (!WIDE) {
            ret = d_fse_decode_2state(out, op, omax, s1, s2, bs, [&](u32& s) { return tab_step<false>(s, bs, tabAddr, fastMode); });
        } else {
            u16* const o16 = reinterpret_cast<u16*>(out);
            while (bs_refill(bs) < SRC_DONE && op < omax) o16[op++] = (u16)tab_step<WIDE>(s1, bs, tabAddr, false);    // fseU16.c:289-293
            if (!bs_exhausted(bs)) ret = err(E_CORRUPT);                                                            // :295
            else {
                while (s1 && op < omax) o16[op++] = (u16)tab_step<WIDE>(s1, bs, tabAddr, false);                     // :297-298
                ret = s1 ? err(E_CORRUPT) : (u64)op * 2;
            }
        }
    }
    if constexpr (Geo::DESCS) { if (WIDE && !is_err(ret)) ret /= 2; }    // U16 descriptor results count symbols
    if (mine) results[b] = ret;
}

// =================================================================================================
// encode
// =================================================================================================
template <bool WIDE> struct EncCfg;
template <> struct EncCfg<false> { static constexpr unsigned MSV = FSE_MAX_SV, CELLS = 1u << FSE_MAX_TLOG; typedef u8 sym_t; };
template <> struct EncCfg<true>  { static constexpr unsigned MSV = U16_MAX_SV, CELLS = 1u << FSE_MAX_TLOG; typedef u16 sym_t; };   // tableLog <= 12 as linked (SURVEY a22)

template <bool WIDE>
struct EncWarp {
    u32   ct[1 + EncCfg<WIDE>::CELLS / 2 + 2 * (EncCfg<WIDE>::MSV + 1)];
    u32   count[EncCfg<WIDE>::MSV + 1];
    u32   start[EncCfg<WIDE>::MSV + 3];
    short norm[EncCfg<WIDE>::MSV + 1];
    u16   cum[EncCfg<WIDE>::MSV + 3];
    typename EncCfg<WIDE>::sym_t cellSym[EncCfg<WIDE>::CELLS];
    u32   cdfs[64], cdnb[64];     // deltaFindState / deltaNbBits of the 64 symbols of the current group (filled by the whole warp)
    u32   slot[64];               // (value | nbBits << 16) of up to 64 consecutive symbols, emission order
    u32   words[32];              // emit_group's staging area
};

// One block's stream as both encode kernels write it: a word-aligned image of 32-bit words from base32 (global), whose
// word 0 also covers `mis` header bytes that are never rewritten.  carry holds the carryBits (< 32) pending bits behind
// word wpos - 1.  Words from capWords on are dropped; overflow is judged from the bit total at the close (bitstream.h:246,258).
// The bit total is 32 * wpos + carryBits - 8 * mis, formed in 64 bits: a block of up to 2^30 bytes can pass 2^32 bits.
struct EncStream { u32* base32; u32 mis, capWords, carry, carryBits, wpos; };

// sbase: first stream byte (right behind the header); scap: the capacity the stream writer sees (slot - header).
__device__ __forceinline__ EncStream enc_stream_open(u8* sbase, u64 scap)
{
    EncStream st;
    st.mis = (u32)(reinterpret_cast<u64>(sbase) & 3);
    st.base32 = reinterpret_cast<u32*>(sbase - st.mis);
    st.capWords = (u32)((st.mis + (scap > 8 ? scap : 0)) / 4);
    st.carry = 0; st.carryBits = 8 * st.mis; st.wpos = 0;
    return st;
}

// Appends PER_LANE (1 or 2) records per lane to the stream, in lane order, r0 before r1.  A record is (value | nbBits << 16);
// value bits at and above nbBits are ignored.  words: the warp's staging area, 28 words (64 records of up to 12 bits + the carry).
template <int PER_LANE>
__device__ __forceinline__ void emit_group(u32 r0, u32 r1, u32* words, EncStream& st)
{
    unsigned const lane = lane_id();
    u32 const nb0 = r0 >> 16, v0 = r0 & ((1u << nb0) - 1);
    u32 nb = nb0, val = v0;
    if (PER_LANE == 2) { u32 const nb1 = r1 >> 16; val |= (r1 & ((1u << nb1) - 1)) << nb0; nb += nb1; }
    u32 incl = nb;                                                 // inclusive scan of bit lengths
    #pragma unroll
    for (int d = 1; d < 32; d <<= 1) { u32 const t = __shfl_up_sync(FULL, incl, d); if (lane >= (unsigned)d) incl += t; }
    u32 const sum = __shfl_sync(FULL, incl, 31);
    u32 const off = st.carryBits + incl - nb;
    if (lane < 28) words[lane] = (lane == 0) ? st.carry : 0u;
    __syncwarp();
    if (nb) {
        u64 const v = (u64)val << (off & 31);
        atomicOr(&words[off >> 5], (u32)v);
        if ((u32)(v >> 32)) atomicOr(&words[(off >> 5) + 1], (u32)(v >> 32));
    }
    __syncwarp();
    u32 const tot = st.carryBits + sum;
    u32 const full = tot >> 5;
    if (lane < full && st.wpos + lane < st.capWords) {
        if (st.wpos + lane == 0 && st.mis) {                       // word 0 also covers `mis` header bytes: leave them alone
            u8* const p8 = reinterpret_cast<u8*>(st.base32);
            for (u32 i = st.mis; i < 4; i++) p8[i] = (u8)(words[0] >> (8 * i));
        } else st.base32[st.wpos + lane] = words[lane];
    }
    st.carry = words[full]; st.carryBits = tot & 31; st.wpos += full;
    __syncwarp();
}

// Closes the stream (bitstream.h:190,254-260) and returns the block's result: the capacity rule on the 64-bit bit total, the
// partial last word flushed byte by byte, then the verdicts of fse_compress.c:669,674 (bytes) or fseU16.c:248 (U16).
template <bool WIDE>
__device__ inline u64 enc_stream_close(const EncStream& st, u32 hSize, u64 scap, u32 n)
{
    u64 const totalBits = 32ull * st.wpos + st.carryBits - 8 * st.mis;
    u64 streamBytes = 0;
    if (scap > 8 && (totalBits >> 3) < scap - 8) {
        streamBytes = (totalBits + 7) >> 3;
        if (lane_id() == 0 && st.carryBits > 8 * st.mis * (st.wpos == 0)) {
            u32 const nby = (st.carryBits + 7) / 8;
            u8* const p = reinterpret_cast<u8*>(st.base32 + st.wpos);
            for (u32 i = (st.wpos == 0 ? st.mis : 0); i < nby; i++) p[i] = (u8)(st.carry >> (8 * i));
        }
    }
    u64 const totalOut = hSize + streamBytes;
    if (!WIDE) return (streamBytes == 0 || totalOut >= (u64)n - 1) ? 0 : totalOut;
    return totalOut >= (u64)(n - 1) * 2 ? 0 : totalOut;
}

// Scratch of the front half of one block's compression.  `count` and `start` may alias the symbol-transform area
// of `ct` (they are dead before it is written); everything is shared memory.
template <bool WIDE>
struct EncFront {
    u32* ct; u32* count; u32* start; short* norm; u16* cum; typename EncCfg<WIDE>::sym_t* cellSym;
};

// Everything FSE_compress_wksp / FSE_compressU16 do before the first FSE_encodeSymbol: argument checks, histogram,
// rle / not-compressible verdicts, normalisation, the NCount header (written to d) and the CTable.  One warp.
// Returns true when the payload must be coded (hSize, tl set); false when `verdict` is already the block's result.
template <bool WIDE>
__device__ inline bool warp_encode_front(const EncFront<WIDE>& w, const typename EncCfg<WIDE>::sym_t* s, u32 n, u8* d, u64 cap,
                                         unsigned msvReq, unsigned tlogReq, u64& verdict, u32& hSizeOut, u32& tlOut, u32 chainBase = 0)
{
    typedef typename EncCfg<WIDE>::sym_t sym_t;
    unsigned const lane = lane_id();
    unsigned const MSVMAX = EncCfg<WIDE>::MSV;
#define FRONT_DONE(v) do { verdict = (v); return false; } while (0)
    // ---- argument checks (fse_compress.c:645-649,691 ; fseU16.c:216-220) ----
    unsigned msv = msvReq, tl = tlogReq;
    if (!WIDE) {
        if (tl > FSE_MAX_TLOG) FRONT_DONE(err(E_TLOG_TOO_LARGE));
        if (tl == 0) FRONT_DONE(err(E_TLOG_TOO_LARGE));               // FSE_WKSP_SIZE_U32(0,..) shifts by -1: the reference (gcc/x86-64) reports tableLog_tooLarge
        // :645 vs the stack workspace of :679-685.  FSE_WKSP_SIZE_U32 is unsigned 32-bit arithmetic: (msv + 1) * 2 wraps, so
        // maxSymbolValue 2^32-1 (and 2^31-1) passes the test and compresses as 255
        u32 const ctWords = 1u + (1u << (tl - 1)) + (msv + 1u) * 2u;  // FSE_CTABLE_SIZE_U32 of the request (:641)
        if (14340u < ctWords + 1024u) FRONT_DONE(err(E_TLOG_TOO_LARGE));
        if (n <= 1) FRONT_DONE(0);
        // the scratch after that CTable (:642-643) is 14340 - 4 * ctWords bytes; HIST_count_wksp refuses less than 4096 of it
        // (hist.c:168).  When the CTable alone exceeds the workspace the size wraps and the reference runs past its stack:
        // those requests are answered as at maxSymbolValue 255.
        if (4ull * ctWords <= 14340u && 14340u - 4ull * ctWords < 4096u) FRONT_DONE(err(E_WKSP_TOO_SMALL));
        if (!msv) msv = FSE_MAX_SV;
        if (msv > FSE_MAX_SV) msv = FSE_MAX_SV;                      // HIST_count_wksp clamps (hist.c:171)
    } else {
        if (n <= 1) FRONT_DONE(n);
        if (!msv) msv = U16_MAX_SV;
        if (!tl) tl = U16_DEF_TLOG;
        if (msv > U16_MAX_SV) FRONT_DONE(err(E_MSV_TOO_LARGE));
        if (tl > U16_MAX_TLOG) FRONT_DONE(err(E_TLOG_TOO_LARGE));
    }
    // ---- histogram: four interleaved copies (lane & 3) in the not-yet-built table area, 16-byte loads, 4 in flight ----
    u32 over = 0;
    {
        u32* const sub = w.ct;
        for (u32 i = lane; i < 4 * (MSVMAX + 1); i += 32) sub[i] = 0;
        __syncwarp();
        u32* const mine = sub + (lane & 3) * (MSVMAX + 1);
        u32 const lim = WIDE ? msv : 255u;
        auto add1 = [&](u32 v, u32 k) { if (WIDE && v > lim) over = 1; else atomicAdd(&mine[v], k); };
        const u8* const sb = reinterpret_cast<const u8*>(s);
        u32 const nB = WIDE ? 2 * n : n;
        u32 const head = min(nB, (u32)((16 - (reinterpret_cast<u64>(sb) & 15)) & 15));
        for (u32 k = lane; k < head / sizeof(sym_t); k += 32) add1(s[k], 1);
        u32 const nvec = (nB - head) / 16;
        const uint4* const gv = reinterpret_cast<const uint4*>(sb + head);
        for (u32 v0 = 0; v0 < nvec; v0 += 128) {
            uint4 x[4];
            #pragma unroll
            for (int h = 0; h < 4; h++) { u32 const vi = v0 + 32 * h + lane; x[h] = (vi < nvec) ? __ldg(gv + vi) : make_uint4(0, 0, 0, 0); }
            #pragma unroll
            for (int h = 0; h < 4; h++) {
                if (v0 + 32 * h + lane >= nvec) continue;
                u32 const wd[4] = { x[h].x, x[h].y, x[h].z, x[h].w };
                #pragma unroll
                for (int k = 0; k < 4; k++) {
                    u32 const y = wd[k];
                    if (WIDE) {
                        u32 const a0 = y & 0xFFFFu, a1 = y >> 16;
                        if (a0 == a1) add1(a0, 2); else { add1(a0, 1); add1(a1, 1); }
                    } else {
                        u32 const b0 = y & 0xFF, b1 = (y >> 8) & 0xFF, b2 = (y >> 16) & 0xFF, b3 = y >> 24;
                        if ((b0 == b1) & (b1 == b2) & (b2 == b3)) add1(b0, 4);
                        else { add1(b0, 1); add1(b1, 1); add1(b2, 1); add1(b3, 1); }
                    }
                }
            }
        }
        for (u32 k = (head + nvec * 16) / sizeof(sym_t) + lane; k < n; k += 32) add1(s[k], 1);
        __syncwarp();
        for (u32 i = lane; i <= MSVMAX; i += 32)
            w.count[i] = sub[i] + sub[(MSVMAX + 1) + i] + sub[2 * (MSVMAX + 1) + i] + sub[3 * (MSVMAX + 1) + i];
    }
    __syncwarp();
    over = __any_sync(FULL, over);
    if (WIDE && over) FRONT_DONE(err(E_MSV_TOO_SMALL));               // fseU16.c:131
    u32 top = 0, best = 0;
    for (u32 i = lane; i <= (WIDE ? msv : 255u); i += 32) { u32 const c = w.count[i]; if (c) top = i; best = c > best ? c : best; }
    #pragma unroll
    for (int dlt = 16; dlt; dlt >>= 1) { top = max(top, __shfl_xor_sync(FULL, top, dlt)); best = max(best, __shfl_xor_sync(FULL, best, dlt)); }
    if (!WIDE && msv < 255 && top > msv) FRONT_DONE(err(E_MSV_TOO_SMALL));            // hist.c:128
    msv = top;
    if (best == n) FRONT_DONE(1);                                      // rle
    if (!WIDE) {
        if (best == 1) FRONT_DONE(0);
        if (best < (n >> 7)) FRONT_DONE(0);
    }
    // ---- normalise + header (one lane) ----
    tl = d_optimal_tablelog(tl, n, msv, 2);
    u64 hdr = 0;
    if (lane == 0) {
        hdr = d_normalize(w.norm, tl, w.count, n, msv);
        if (!is_err(hdr)) hdr = d_write_ncount(d, cap, w.norm, msv, tl);
    }
    hdr = __shfl_sync(FULL, hdr, 0);
    if (is_err(hdr)) FRONT_DONE(hdr);
    u32 const hSize = (u32)hdr;
    // ---- CTable (fse_compress.c:66-169) ----
    u32 const size = 1u << tl;
    if (lane == 0) {
        u32 acc = 0, st = 0;
        for (u32 q = 0; q <= msv; q++) {
            w.cum[q] = (u16)acc; w.start[q] = st;
            int const nn = w.norm[q];
            if (nn > 0) acc += (u32)nn;
            st += (u32)(nn == -1 ? 1 : nn);
        }
        w.cum[msv + 1] = (u16)acc;
        ((u16*)w.ct)[0] = (u16)tl; ((u16*)w.ct)[1] = (u16)msv;
    }
    __syncwarp();
    warp_spread(w.norm, w.cum, msv, tl, [&](u32 cell, u32 sym) { w.cellSym[cell] = (typename EncCfg<WIDE>::sym_t)sym; });
    __syncwarp();
    {   u16* const next = ((u16*)w.ct) + 2;
        for (u32 u0 = 0; u0 < size; u0 += 32) {                       // next[start[s] + k] = size + u for the k-th cell u of s (:125-128)
            u32 const u = u0 + lane;
            u32 const sym = w.cellSym[u];
            u32 const peers = __match_any_sync(FULL, sym);
            u32 const at = w.start[sym] + __popc(peers & ((1u << lane) - 1));
            next[at] = (u16)(size + u);
            __syncwarp();
            if ((peers >> lane) == 1u) w.start[sym] += __popc(peers);
            __syncwarp();
        }
        u32* const tt = w.ct + 1 + (size >> 1);
        if (lane == 0) {
            u32 total = 0;
            for (u32 q = 0; q <= msv; q++) {
                int const nn = w.norm[q];
                if (chainBase) {                                    // chain form: { byte address of next[deltaFindState], (maxBitsOut - 1) << 16 | minStatePlus }
                    if (nn == 0) { tt[2 * q] = chainBase; tt[2 * q + 1] = ((tl - 1) << 16) | size; continue; }
                    if (nn == -1 || nn == 1) { tt[2 * q] = chainBase + 2 * (total - 1); tt[2 * q + 1] = ((tl - 1) << 16) | size; total++; }
                    else {
                        u32 const maxOut = tl - hibit((u32)nn - 1);
                        tt[2 * q] = chainBase + 2 * (total - (u32)nn); tt[2 * q + 1] = ((maxOut - 1) << 16) | ((u32)nn << maxOut);
                        total += (u32)nn;
                    }
                    continue;
                }
                if (nn == 0) { tt[2 * q + 1] = ((tl + 1) << 16) - size; tt[2 * q] = 0; continue; }
                if (nn == -1 || nn == 1) { tt[2 * q + 1] = (tl << 16) - size; tt[2 * q] = total - 1; total++; }
                else {
                    u32 const maxOut = tl - hibit((u32)nn - 1);
                    tt[2 * q + 1] = (maxOut << 16) - ((u32)nn << maxOut);
                    tt[2 * q] = total - (u32)nn; total += (u32)nn;
                }
            }
        }
    }
    __syncwarp();
    hSizeOut = hSize; tlOut = tl;
    return true;
#undef FRONT_DONE
}

// Descriptor batches reach the two encode kernels through block lists: fse_route_kernel settles the blocks the tier's limits
// decide and files every other block's index under the kernel that codes it.  list[i] is the i-th block of a kernel's list
// and *count the list's length; the kernels launch with grids for the whole batch and exit past the count.
struct ListedDescs : BlockDescs { const u32* list; const u32* count; };

// Geo: BatchGeom (blocks firstBlock + i) or ListedDescs (blocks list[i])
template <bool WIDE, class Geo>
__global__ void __launch_bounds__(THREADS)
fse_encode_kernel(Geo g, u32 firstBlock, u8* __restrict__ cbuf, u64* __restrict__ csizes, const u8* __restrict__ src,
                  unsigned msvReq, unsigned tlogReq)
{
    typedef typename EncCfg<WIDE>::sym_t sym_t;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    EncWarp<WIDE>& w = reinterpret_cast<EncWarp<WIDE>*>(smem_raw)[threadIdx.x >> 5];
    unsigned const lane = lane_id();
    u32 b;
    if constexpr (Geo::DESCS) {
        u32 const i = blockIdx.x * WARPS + (threadIdx.x >> 5);
        if (i >= *g.count) return;
        b = g.list[i];
    } else {
        b = firstBlock + blockIdx.x * WARPS + (threadIdx.x >> 5);
        if (b >= g.nBlocks) return;
    }
    u32 const nBytes = (u32)fse_enc_len(g, b, WIDE);
    u32 const n = WIDE ? nBytes / 2 : nBytes;                        // symbols
    const sym_t* const s = reinterpret_cast<const sym_t*>(enc_src(g, src, b));
    u8* const d = enc_dst(g, cbuf, b);
    u64 const cap = enc_cap(g, b);
#define FSEB_DONE(v) do { if (lane == 0) enc_out(g, csizes, b) = (v); return; } while (0)

    EncFront<WIDE> f; f.ct = w.ct; f.count = w.count; f.start = w.start; f.norm = w.norm; f.cum = w.cum; f.cellSym = w.cellSym;
    u64 verdict = 0; u32 hSize = 0, tl = 0;
    if (!warp_encode_front<WIDE>(f, s, n, d, cap, msvReq, tlogReq, verdict, hSize, tl)) FSEB_DONE(verdict);
    u32 const size = 1u << tl;
    // ---- encode (fse_compress.c:554-611 ; U16: fseU16.c:150-200) ----
    u64 const scap = cap - hSize;                                    // capacity seen by the stream writer
    if (!WIDE && (n <= 2 || scap <= 8)) FSEB_DONE(0);
    EncStream st = enc_stream_open(d + hSize, scap);
    const u16* const next = ((const u16*)w.ct) + 2;
    const u32* const tt = w.ct + 1 + (size >> 1);
    u32 state = 0; bool seeded = false;
    if (WIDE) { state = size; seeded = true; }
    // symbols are consumed from the end; index parity picks the chain (lane 0: even / the only chain, lane 1: odd)
    for (u32 hi = n; hi > 0;) {
        u32 const cnt = hi >= 64 ? 64 : hi;
        u32 const lo = hi - cnt;
        // slot j <-> symbol index hi-1-j.  The whole warp first fetches the group's symbols (coalesced) and their
        // transforms, so that the chain lanes only touch shared memory and their loads do not depend on the state.
        for (u32 j = lane; j < cnt; j += 32) {
            u32 const sym = (u32)s[hi - 1 - j];
            w.cdfs[j] = tt[2 * sym]; w.cdnb[j] = tt[2 * sym + 1];
        }
        __syncwarp();
        {
            unsigned const chains = WIDE ? 1u : 2u;
            if (lane < chains) {
                u32 const j0 = WIDE ? 0u : ((((hi - 1) & 1u) == lane) ? 0u : 1u);      // first slot of this chain in the group
                for (u32 j = j0; j < cnt; j += chains) {
                    u32 const dfs = w.cdfs[j], dnb = w.cdnb[j];
                    if (!seeded) {                                   // FSE_initCState2 (fse.h:503-512): no output
                        u32 const nb0 = (dnb + (1u << 15)) >> 16;
                        u32 const v0 = (nb0 << 16) - dnb;
                        state = next[(v0 >> nb0) + dfs];
                        seeded = true;
                        w.slot[j] = 0;
                    } else {                                         // FSE_encodeSymbol (fse.h:514-521)
                        u32 const nb = (state + dnb) >> 16;
                        w.slot[j] = (state & ((1u << nb) - 1)) | (nb << 16);
                        state = next[(state >> nb) + dfs];
                    }
                }
            }
        }
        __syncwarp();
        for (u32 j = 0; j < cnt; j += 32) emit_group<1>(j + lane < cnt ? w.slot[j + lane] : 0u, 0u, w.words, st);
        hi = lo;
    }
    // final states (fse_compress.c:608-609), end mark
    {   u32 const s0 = __shfl_sync(FULL, state, 0), s1 = __shfl_sync(FULL, state, 1);
        u32 k = 0;
        if (lane == 0) {
            if (!WIDE) w.slot[k++] = (s1 & (size - 1)) | (tl << 16);
            w.slot[k++] = (s0 & (size - 1)) | (tl << 16);
            w.slot[k++] = 1u | (1u << 16);
        }
        k = WIDE ? 2 : 3;
        __syncwarp();
        emit_group<1>(lane < k ? w.slot[lane] : 0u, 0u, w.words, st);
    }
    FSEB_DONE(enc_stream_close<WIDE>(st, hSize, scap, n));
#undef FSEB_DONE
}


// =================================================================================================
// encode, batch kernel.  The tANS chain is a serial dependency (state -> table -> state, ~50 cycles per symbol) and its
// tables (10 KB per block) are what limits how many chains an SM can keep resident, so the work is arranged
// around the chains: one CTA owns EK blocks; all warps run the front half (histogram .. CTable) of the blocks,
// then warp 0 becomes the CHAIN warp -- lane pair (2k, 2k+1) carries the two interleaved states of block k
// (U16: lane k carries the single state) and does nothing but table walks, dropping one (state, nbBits) record per
// symbol into a shared-memory ring -- while warps 1..7 are EMITTERS that turn ring groups into stream words
// (prefix scan of bit counts, OR into a staging word array, coalesced word stores).  Ring groups are handed
// over with named barriers (two buffers).  Only full blocks whose size is a multiple of 64 bytes and that
// start 16-byte aligned come here; everything else takes the warp-per-block kernel above.
// =================================================================================================
constexpr int ETHREADS = 256;
constexpr int GSTEPS = 32;             // chain steps per ring group
template <bool WIDE, int EK> struct EncCta {         // EK = blocks per CTA (16: one CTA per SM; 8: two)
    typedef typename EncCfg<WIDE>::sym_t sym_t;
    static constexpr unsigned CH = WIDE ? 1 : 2;
    static constexpr unsigned MSV = EncCfg<WIDE>::MSV, CELLS = EncCfg<WIDE>::CELLS;
    static constexpr unsigned CT_WORDS = ((2 + CELLS / 2 + 2 * (MSV + 1) + 8) + 3) & ~3u;    // u32 per block, 16-byte multiple
    static constexpr unsigned BUILDERS = WIDE ? EK / 4 : EK / 2;
    static constexpr unsigned RING_STRIDE = GSTEPS * CH + 2;                                 // u32 per block per buffer (+2 skews the banks)
    struct alignas(16) Scratch { short norm[MSV + 1]; u16 cum[MSV + 3]; sym_t cellSym[CELLS]; };
    struct alignas(16) Smem {
        u32 ct[EK * CT_WORDS];
        u32 ring[2 * EK * RING_STRIDE];
        u32 words[8 * 32];
        u32 active[EK], hSize[EK], tl[EK];
        Scratch scratch[BUILDERS];
    };
    struct alignas(16) DescSmem { u32 b[EK], len[EK]; };            // descriptor batches, behind Smem: block index, bytes
};
// named barriers 1,2 = ring buffer 0,1 full ; 3,4 = ring buffer 0,1 drained (immediate ids: the CTA then owns 5 barriers, not 16)
__device__ __forceinline__ void bar_sync(int id)
{
    switch (id) {
    case 1: asm volatile("bar.sync 1, 256;" ::: "memory"); break;
    case 2: asm volatile("bar.sync 2, 256;" ::: "memory"); break;
    case 3: asm volatile("bar.sync 3, 256;" ::: "memory"); break;
    default: asm volatile("bar.sync 4, 256;" ::: "memory"); break;
    }
}
__device__ __forceinline__ void bar_arrive(int id)
{
    switch (id) {
    case 1: asm volatile("bar.arrive 1, 256;" ::: "memory"); break;
    case 2: asm volatile("bar.arrive 2, 256;" ::: "memory"); break;
    case 3: asm volatile("bar.arrive 3, 256;" ::: "memory"); break;
    default: asm volatile("bar.arrive 4, 256;" ::: "memory"); break;
    }
}
static_assert(ETHREADS == 256, "barrier counts are spelled out");
__device__ __forceinline__ uint2 lds_v2(u32 addr) { uint2 v; asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(addr)); return v; }

template <class Geo> __device__ __forceinline__ u32 listed(const Geo& g, u32 i) { if constexpr (Geo::DESCS) return g.list[i]; else return i; }

// Geo: BatchGeom (blocks b0 .. nFast - 1, all of g.blockSize bytes) or ListedDescs (blocks list[0 .. *count), each its own
// size).  Blocks of different sizes share a CTA: each chain lane and emitter runs its own block's group count, the ring
// hand-over runs to the CTA's largest, and each block closes at its own count.
template <bool WIDE, int EK, class Geo>
__global__ void __launch_bounds__(ETHREADS, 16 / EK)
fse_encode_cta_kernel(Geo g, u32 nFast, u8* __restrict__ cbuf, u64* __restrict__ csizes, const u8* __restrict__ src,
                      unsigned msvReq, unsigned tlogReq)
{
    typedef EncCta<WIDE, EK> C;
    typedef typename C::sym_t sym_t;
    constexpr unsigned CH = C::CH;
    constexpr bool DESCS = Geo::DESCS;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    typename C::Smem& sm = *reinterpret_cast<typename C::Smem*>(smem_raw);
    typename C::DescSmem& sx = *reinterpret_cast<typename C::DescSmem*>(smem_raw + sizeof(typename C::Smem));   // DESCS only
    unsigned const lane = lane_id(), warp = threadIdx.x >> 5;
    u32 const b0 = blockIdx.x * EK;
    if constexpr (DESCS) { nFast = *g.count; if (b0 >= nFast) return; }
    u32 const nHere = nFast - b0 < (u32)EK ? nFast - b0 : (u32)EK;
    u32 nBytes = 0; u64 cap = 0;                                    // the uniform batch's, for every block
    if constexpr (!DESCS) { nBytes = (u32)g.blockSize; cap = g.slot; }
    u32 const n = WIDE ? nBytes / 2 : nBytes;

    // ---- phase 1: front half of every block, one warp per block ----
    if (threadIdx.x < EK) sm.active[threadIdx.x] = 0;
    __syncthreads();
    if (warp < C::BUILDERS) {
        for (u32 blk = warp; blk < nHere; blk += C::BUILDERS) {
            u32 const b = listed(g, b0 + blk);
            u32 const bBytes = DESCS ? (u32)fse_enc_len(g, b, WIDE) : nBytes;
            u32 const bn = WIDE ? bBytes / 2 : bBytes;
            u64 const bcap = DESCS ? enc_cap(g, b) : cap;
            EncFront<WIDE> f;
            f.ct = sm.ct + blk * C::CT_WORDS + 1;                  // +1: the symbol transforms (8-byte pairs) land 8-byte aligned
            f.count = f.ct + 1 + C::CELLS / 2; f.start = f.count + C::MSV + 1;      // dead before the transforms are written
            f.norm = sm.scratch[warp].norm; f.cum = sm.scratch[warp].cum; f.cellSym = sm.scratch[warp].cellSym;
            u8* const d = enc_dst(g, cbuf, b);
            u64 verdict = 0; u32 hSize = 0, tl = 0;
            u32 const nextAddr = (u32)__cvta_generic_to_shared(reinterpret_cast<u16*>(f.ct) + 2);
            bool go = warp_encode_front<WIDE>(f, reinterpret_cast<const sym_t*>(enc_src(g, src, b)), bn, d, bcap, msvReq, tlogReq, verdict, hSize, tl, nextAddr);
            if (go) {
                bool const usable = bcap - hSize > 8;
                if (!WIDE && (bn <= 2 || !usable)) { go = false; verdict = 0; }
                if (WIDE && !usable) { go = false; verdict = (u64)hSize >= (u64)(bn - 1) * 2 ? 0 : hSize; }
            }
            if (lane == 0) {
                sm.active[blk] = go; sm.hSize[blk] = hSize; sm.tl[blk] = tl;
                if constexpr (DESCS) { sx.b[blk] = b; sx.len[blk] = bBytes; }
                if (!go) enc_out(g, csizes, b) = verdict;
            }
            __syncwarp();
        }
    }
    __syncthreads();

    u32 const iters = nBytes / 16;                                 // 16 source bytes = 8 chain steps
    u32 nGroups = iters / 4;                                       // GSTEPS = 32 steps; descriptors: the CTA's largest block's
    if constexpr (DESCS) for (u32 k = 0; k < nHere; k++) if (sm.active[k]) nGroups = max(nGroups, sx.len[k] / 64);
    if (warp == 0) {
        // ---- chain warp ----
        u32 const blk = lane / CH, c = lane % CH;
        bool const act = blk < (u32)EK && sm.active[blk < (u32)EK ? blk : 0];
        u32 const bsafe = act ? blk : 0;
        u32 const tl = act ? sm.tl[bsafe] : 5u;
        u32 const size = 1u << tl;
        const u32* const ct = sm.ct + bsafe * C::CT_WORDS + 1;
        u32 const ttAddr = (u32)__cvta_generic_to_shared(ct + 1 + (size >> 1));
        u32 const myIters = DESCS ? (act ? sx.len[bsafe] / 16 : 0u) : iters;   // this lane's block
        u32 const myGroups = myIters / 4;
        const uint4* sp;
        if constexpr (DESCS) sp = reinterpret_cast<const uint4*>(act ? enc_src(g, src, sx.b[bsafe]) + sx.len[bsafe] : nullptr) - 1;
        else sp = reinterpret_cast<const uint4*>(src + (u64)(b0 + bsafe) * g.blockSize + g.blockSize) - 1;
        u32* const ringLane = sm.ring + bsafe * C::RING_STRIDE + c;
        u32 const selA = 0x4440u | (3 - c), selB = 0x4440u | (1 - c);  // byte pickers for even / odd steps of a register (bytes only)
        u32 state = WIDE ? size : 0u;
        // transforms of the 8 symbols this lane codes out of one 16-byte piece (descending addresses)
        auto fetch = [&](const uint4& v, uint2 (&t)[8]) {
            u32 const regs[4] = { v.w, v.z, v.y, v.x };
            #pragma unroll
            for (int q = 0; q < 8; q++) {
                u32 const r = regs[q >> 1];
                u32 const sym = WIDE ? ((q & 1) ? (r & 0xFFFFu) : (r >> 16)) : __byte_perm(r, 0, (q & 1) ? selB : selA);
                t[q] = lds_v2(ttAddr + sym * 8);
            }
        };
        uint4 q1 = make_uint4(0, 0, 0, 0), q2 = q1;              // pieces it+1, it+2 (in flight)
        uint2 t[8], tn[8];
        #pragma unroll
        for (int q = 0; q < 8; q++) { t[q] = make_uint2(0, 0); tn[q] = t[q]; }
        // closing group: final states (fse_compress.c:608-609), end mark (bitstream.h:254-260)
        auto close = [&](u32* rp) {
            rp[0] = (state & (size - 1)) | (tl << 16);
            rp[CH] = c == 0 ? (1u | (1u << 16)) : 0u;
            for (u32 q = 2; q < (u32)GSTEPS; q++) rp[q * CH] = 0;
        };
        if (act) {
            uint4 const q0 = __ldg(sp);
            if (myIters > 1) q1 = __ldg(sp - 1);
            if (myIters > 2) q2 = __ldg(sp - 2);
            fetch(q0, tn);
        }
        for (u32 grp = 0; grp < nGroups; grp++) {
            u32 const buf = grp & 1;
            if (grp >= 2) bar_sync(3 + buf);
            u32* rp = ringLane + buf * (EK * C::RING_STRIDE);
            bool const live = DESCS ? act && grp < myGroups : act;
            if constexpr (DESCS) { if (act && grp == myGroups) close(rp); }   // a block shorter than the CTA's longest closes early
            #pragma unroll
            for (u32 i4 = 0; i4 < 4; i4++, rp += 8 * CH) {          // fully unrolled: the two-deep queues rotate by renaming
                u32 const it = grp * 4 + i4;
                if (live) {
                    uint2 (&tc)[8] = (i4 & 1) ? t : tn;             // transforms of this piece (fetched one piece ago)
                    uint2 (&tf)[8] = (i4 & 1) ? tn : t;             // ... and where the next piece's go
                    uint4 const nx = (i4 & 1) ? q2 : q1;            // piece it+1
                    if (it + 3 < myIters) { if (i4 & 1) q2 = __ldg(sp - (it + 3)); else q1 = __ldg(sp - (it + 3)); }
                    if (it + 1 < myIters) fetch(nx, tf);            // off the chain's critical path
                    #pragma unroll
                    for (int q = 0; q < 8; q++) {
                        u32 const x = tc[q].x, y = tc[q].y;         // { byte address of next[deltaFindState], (maxBitsOut - 1) << 16 | minStatePlus }
                        u32 const yhi = y & 0xFFFF0000u;
                        u32 rec;
                        if (!WIDE && q == 0 && i4 == 0 && grp == 0) {   // FSE_initCState2 (fse.h:503-512): no output
                            u32 const dnb = (yhi + 0x10000u) - (y & 0xFFFFu);
                            u32 const nb0 = (dnb + (1u << 15)) >> 16;
                            u32 const v0 = (nb0 << 16) - dnb;
                            state = lds_u16(x + 2 * (v0 >> nb0));
                            rec = 0;
                        } else {                                    // FSE_encodeSymbol (fse.h:514-521): nbBitsOut = maxBitsOut - (state < minStatePlus)
                            u32 const r0 = state + yhi;             // state < 2^16: also state | (maxBitsOut-1) << 16
                            bool const p = r0 >= y;                 // state >= minStatePlus
                            u32 idx;
                            asm("shr.u32 %0, %1, %2;" : "=r"(idx) : "r"(state), "r"(y >> 16));
                            if (p) idx >>= 1;
                            rec = p ? r0 + 0x10000u : r0;           // (state, nbBits): the emitter masks the value
                            state = lds_u16(x + 2 * idx);
                        }
                        rp[q * CH] = rec;
                    }
                }
            }
            __syncwarp();
            bar_arrive(1 + buf);
        }
        {
            u32 const buf = nGroups & 1;
            if (nGroups >= 2) bar_sync(3 + buf);
            u32* const rp = ringLane + buf * (EK * C::RING_STRIDE);
            if (DESCS ? act && myGroups == nGroups : act) close(rp);
            __syncwarp();
            bar_arrive(1 + buf);
        }
    } else {
        // ---- emitter warps: blocks e, e+7, e+14 ----
        u32 const e = warp - 1;
        u32* const words = sm.words + warp * 32;
        EncStream st[3]; bool on[3]; u32 myGroups[3];
        #pragma unroll
        for (int k = 0; k < 3; k++) {
            u32 const blk = e + 7 * k;
            on[k] = blk < (u32)EK && sm.active[blk < (u32)EK ? blk : 0];
            u32 const hs = on[k] ? sm.hSize[blk] : 0;
            if constexpr (DESCS) {
                u32 const b = sx.b[on[k] ? blk : 0];
                myGroups[k] = on[k] ? sx.len[blk] / 64 : 0u;
                st[k] = enc_stream_open(on[k] ? enc_dst(g, cbuf, b) + hs : nullptr, on[k] ? enc_cap(g, b) - hs : 0);
            } else st[k] = enc_stream_open(cbuf + (u64)(b0 + (on[k] ? blk : 0)) * g.slot + hs, cap - hs);
        }
        for (u32 grp = 0; grp <= nGroups; grp++) {
            u32 const buf = grp & 1;
            bar_sync(1 + buf);
            #pragma unroll
            for (int k = 0; k < 3; k++) {
                if (!on[k] || (DESCS && grp > myGroups[k])) continue;
                const u32* const row = sm.ring + buf * (EK * C::RING_STRIDE) + (e + 7 * k) * C::RING_STRIDE;
                u32 r0, r1 = 0;
                if (WIDE) r0 = row[lane];
                else { uint2 const rr = reinterpret_cast<const uint2*>(row)[lane]; r0 = rr.x; r1 = rr.y; }
                emit_group<CH>(r0, r1, words, st[k]);
            }
            __syncwarp();
            if (grp + 2 <= nGroups) bar_arrive(3 + buf);
        }
        #pragma unroll
        for (int k = 0; k < 3; k++) {
            if (!on[k]) continue;
            u32 const blk = e + 7 * k;
            u32 const hSize = sm.hSize[blk];
            if constexpr (DESCS) {
                u32 const b = sx.b[blk];
                u64 const verdict = enc_stream_close<WIDE>(st[k], hSize, enc_cap(g, b) - hSize, WIDE ? sx.len[blk] / 2 : sx.len[blk]);
                if (lane == 0) enc_out(g, csizes, b) = verdict;
            } else {
                u64 const verdict = enc_stream_close<WIDE>(st[k], hSize, cap - hSize, n);
                if (lane == 0) csizes[b0 + blk] = verdict;
            }
        }
    }
}

// Descriptor batches: settles the blocks the batch tier's limits decide -- U16: a source at an odd address (GENERIC), one symbol
// or none (the count itself, as FSE_compressU16), more than 2^29 symbols; bytes: more than 2^30 (srcSize_wrong) -- and files
// every other block under the kernel that codes it, by the rule launch_enc applies to the uniform batch: a whole number of
// 64-byte groups (at least one) at a 16-byte aligned source goes to the CTA kernel, anything else to the warp-per-block kernel.
// lists: u32 count[2] (zeroed by the launcher), then the CTA kernel's list and the warp kernel's, nBlocks entries each.
constexpr int RTHREADS = 256;
template <bool WIDE>
__global__ void __launch_bounds__(RTHREADS) fse_route_kernel(BlockDescs g, u32* __restrict__ lists)
{
    u32 const b = blockIdx.x * RTHREADS + threadIdx.x;
    unsigned const lane = lane_id();
    int route = -1;
    if (b < g.nBlocks) {
        u64 const n = g.srcSize[b];
        u64 const a = reinterpret_cast<u64>(g.src[b]);
        u64 const bytes = fse_bytes(n, WIDE);
        if (WIDE && (a & 1)) g.result[b] = err(E_GENERIC);
        else if (WIDE && n <= 1) g.result[b] = n;
        else if (bytes > FSE_BLOCK_MAX) g.result[b] = err(E_SRC_WRONG);
        else route = (bytes >= 64 && bytes % 64 == 0 && (a & 15) == 0) ? 0 : 1;
    }
    #pragma unroll
    for (int r = 0; r < 2; r++) {                                   // one atomic per warp and list
        u32 const m = __ballot_sync(FULL, route == r);
        if (!m) continue;
        int const leader = __ffs(m) - 1;
        u32 base = 0;
        if ((int)lane == leader) base = atomicAdd(&lists[r], (u32)__popc(m));
        base = __shfl_sync(FULL, base, leader);
        if (route == r) lists[2 + (u64)r * g.nBlocks + base + __popc(m & ((1u << lane) - 1))] = b;
    }
}

}  // namespace fsek

template <bool WIDE, class Geo>
static cudaError_t launch_dec(const Geo& g, void* dst, const void* cbuf, const u64* csizes, u64* results, const void* orig, cudaStream_t stream)
{
    if (g.nBlocks == 0) return cudaSuccess;
    size_t const smemCta = sizeof(typename fsek::DecCta<WIDE>::Smem);
    static SmemOptIn optin;                                          // per device: the attribute belongs to the current device
    {   cudaError_t const e = optin.ensure(fsek::fse_decode_cta_kernel<WIDE, Geo>, current_device(), (int)smemCta);
        if (e != cudaSuccess) return e; }
    unsigned const DK = fsek::DecCta<WIDE>::DK;
    unsigned const grid = (g.nBlocks + DK - 1) / DK;
    fsek::fse_decode_cta_kernel<WIDE, Geo><<<grid, fsek::DTHREADS, smemCta, stream>>>(g, (u8*)dst, (const u8*)cbuf, csizes, results, (const u8*)orig);
    return cudaGetLastError();
}
template <bool WIDE, int EK, class Geo>
static cudaError_t launch_enc_cta(const Geo& g, u32 nFast, void* cbuf, u64* csizes, const void* src, unsigned msv, unsigned tlog, cudaStream_t stream)
{
    typedef fsek::EncCta<WIDE, EK> C;
    size_t const smemCta = sizeof(typename C::Smem) + (Geo::DESCS ? sizeof(typename C::DescSmem) : 0);
    static SmemOptIn optin;
    {   cudaError_t const e = optin.ensure(fsek::fse_encode_cta_kernel<WIDE, EK, Geo>, current_device(), (int)smemCta);
        if (e != cudaSuccess) return e; }
    unsigned const grid = (nFast + EK - 1) / EK;
    fsek::fse_encode_cta_kernel<WIDE, EK, Geo><<<grid, fsek::ETHREADS, smemCta, stream>>>(g, nFast, (u8*)cbuf, csizes, (const u8*)src, msv, tlog);
    return cudaGetLastError();
}
template <bool WIDE, class Geo>
static cudaError_t launch_enc_warp(const Geo& g, u32 firstBlock, u32 nWarpBlocks, void* cbuf, u64* csizes, const void* src, unsigned msv, unsigned tlog, cudaStream_t stream)
{
    size_t const smem = sizeof(fsek::EncWarp<WIDE>) * fsek::WARPS;
    static SmemOptIn optin;
    {   cudaError_t const e = optin.ensure(fsek::fse_encode_kernel<WIDE, Geo>, current_device(), (int)smem);
        if (e != cudaSuccess) return e; }
    unsigned const grid = (nWarpBlocks + fsek::WARPS - 1) / fsek::WARPS;
    fsek::fse_encode_kernel<WIDE, Geo><<<grid, fsek::THREADS, smem, stream>>>(g, firstBlock, (u8*)cbuf, csizes, (const u8*)src, msv, tlog);
    return cudaGetLastError();
}
static int enc_ek()                                                  // tuning knob: blocks per CTA of the chain-warp kernel
{
    static int const ek = [] { const char* const v = getenv("FSEB200_ENC_EK"); return (v && atoi(v) == 8) ? 8 : 16; }();
    return ek;
}
template <bool WIDE>
static cudaError_t launch_enc(const BatchGeom& g, void* cbuf, u64* csizes, const void* src, unsigned msv, unsigned tlog, cudaStream_t stream)
{
    if (g.nBlocks == 0) return cudaSuccess;
    // full, aligned blocks go to the chain-warp kernel; a ragged last block or an odd geometry to the warp-per-block kernel
    u64 const nFull = g.total / g.blockSize;
    bool const fast = g.blockSize >= 64 && g.blockSize % 64 == 0 && (reinterpret_cast<u64>(src) & 15) == 0;
    u32 const nFast = fast ? (u32)nFull : 0u;
    if (nFast) {
        cudaError_t const e = enc_ek() == 8 ? launch_enc_cta<WIDE, 8>(g, nFast, cbuf, csizes, src, msv, tlog, stream)
                                            : launch_enc_cta<WIDE, 16>(g, nFast, cbuf, csizes, src, msv, tlog, stream);
        if (e != cudaSuccess) return e;
    }
    if (nFast < g.nBlocks) return launch_enc_warp<WIDE>(g, nFast, g.nBlocks - nFast, cbuf, csizes, src, msv, tlog, stream);
    return cudaGetLastError();
}
// Descriptor batches: the route kernel writes the two block lists to stream scratch, then both encode kernels launch with grids
// for the whole batch (the host never sees the sizes) and exit past their list's count.
template <bool WIDE>
static cudaError_t launch_enc_blocks(const BlockDescs& g, unsigned msv, unsigned tlog, cudaStream_t stream)
{
    if (g.nBlocks == 0) return cudaSuccess;
    cudaError_t e;
    u32* const lists = (u32*)stream_scratch(3, stream, (2 + 2 * (size_t)g.nBlocks) * sizeof(u32), &e);
    if (e != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(lists, 0, 2 * sizeof(u32), stream)) != cudaSuccess) return e;
    fsek::fse_route_kernel<WIDE><<<(g.nBlocks + fsek::RTHREADS - 1) / fsek::RTHREADS, fsek::RTHREADS, 0, stream>>>(g, lists);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    fsek::ListedDescs cta, warp;
    static_cast<BlockDescs&>(cta) = g; cta.count = lists; cta.list = lists + 2;
    static_cast<BlockDescs&>(warp) = g; warp.count = lists + 1; warp.list = lists + 2 + g.nBlocks;
    e = enc_ek() == 8 ? launch_enc_cta<WIDE, 8>(cta, g.nBlocks, nullptr, nullptr, nullptr, msv, tlog, stream)
                      : launch_enc_cta<WIDE, 16>(cta, g.nBlocks, nullptr, nullptr, nullptr, msv, tlog, stream);
    if (e != cudaSuccess) return e;
    return launch_enc_warp<WIDE>(warp, 0, g.nBlocks, nullptr, nullptr, nullptr, msv, tlog, stream);
}

cudaError_t launch_fse_decode(const BatchGeom& g, void* dst, const void* cbuf, const u64* csizes, u64* results, const void* orig, cudaStream_t s)
{ return launch_dec<false>(g, dst, cbuf, csizes, results, orig, s); }
cudaError_t launch_fseu16_decode(const BatchGeom& g, void* dst, const void* cbuf, const u64* csizes, u64* results, const void* orig, cudaStream_t s)
{ return launch_dec<true>(g, dst, cbuf, csizes, results, orig, s); }
cudaError_t launch_fse_encode(const BatchGeom& g, void* cbuf, u64* csizes, const void* src, unsigned msv, unsigned tlog, cudaStream_t s)
{ return launch_enc<false>(g, cbuf, csizes, src, msv, tlog, s); }
cudaError_t launch_fseu16_encode(const BatchGeom& g, void* cbuf, u64* csizes, const void* src, unsigned msv, unsigned tlog, cudaStream_t s)
{ return launch_enc<true>(g, cbuf, csizes, src, msv, tlog, s); }
cudaError_t launch_fse_encode_blocks(const BlockDescs& g, bool wide, unsigned msv, unsigned tlog, cudaStream_t s)
{ return wide ? launch_enc_blocks<true>(g, msv, tlog, s) : launch_enc_blocks<false>(g, msv, tlog, s); }
cudaError_t launch_fse_decode_blocks(const BlockDescs& g, bool wide, cudaStream_t s)
{ return wide ? launch_dec<true>(g, nullptr, nullptr, nullptr, nullptr, nullptr, s) : launch_dec<false>(g, nullptr, nullptr, nullptr, nullptr, nullptr, s); }

}  // namespace fseb
