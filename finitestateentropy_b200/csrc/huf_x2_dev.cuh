// huf_x2_dev.cuh -- device restatement of the reference's DOUBLE-symbol Huff0 decoder, exact to the bit on any input:
//   HUF_readDTableX2 / HUF_fillDTableX2[Level2]        lib/huf_decompress.c:460-649
//   HUF_decodeSymbolX2 / HUF_decodeLastSymbolX2        lib/huf_decompress.c:659-683
//   HUF_decodeStreamX2                                 lib/huf_decompress.c:693-720
//   HUF_decompress{1,4}X2_usingDTable_internal_body    lib/huf_decompress.c:722-862
// and the payload decode both Huff0 decoders share (stream split, rejections, verdict), with the single-symbol stream loop
// HUF_decodeStreamX1 (:214-237) beside the double-symbol one.
// Used by the table-level entry points (micro.cu) and by the verdict fix-up pass of the batch decoder
// (huf_x2_fixup.cu).  One lane per stream on the byte-granular reader model (bitsrc_dev.cuh): these serve single calls and
// rejected blocks, not throughput.
#pragma once
#include "common.cuh"
#include "bitsrc_dev.cuh"
#include "huf_dev.cuh"

namespace fseb {

// dt = { header word, 2^L cells }; cell = { U16 sequence; BYTE nbBits; BYTE length } (huf_decompress.c:460).
// In an index space of width L (= the descriptor's maxTableLog) a symbol of code length n owns 2^(L-n) cells, weights
// ascending; where the shortest code still fits behind it, those cells are a scaled copy of the same layout for the second
// symbol (second symbols too long to fit leave single-symbol cells).  One lane.  Scratch: weights[256], listSym[256], listW[256].
__device__ inline u64 d_huf_build_dtable_x2(u32* dt, u32 hdr, u8* weights, u8* listSym, u8* listW, const u8* src, u64 srcSize)
{
    u32 rank[17]; u32 nb = 0, tl = 0;
    u32* const cells = dt + 1;
    u32 const L = hdr & 0xFF;
    dt[0] = hdr;
    if (L > HUF_MAX_TLOG) return err(E_TLOG_TOO_LARGE);
    u64 const h = d_huf_read_stats(weights, 256, rank, &nb, &tl, src, srcSize);
    if (is_err(h)) return h;
    if (tl > L) return err(E_TLOG_TOO_LARGE);                                        // :571
    u32 maxW = tl; while (rank[maxW] == 0) maxW--;
    u32 listStart[HUF_MAX_TLOG + 2], fill[HUF_MAX_TLOG + 2], first[HUF_MAX_TLOG + 2], next1[HUF_MAX_TLOG + 2], next2[HUF_MAX_TLOG + 2];
    u32 listSize = 0;
    for (u32 w = 1; w <= maxW; w++) { listStart[w] = listSize; fill[w] = listSize; listSize += rank[w]; }
    for (u32 s = 0; s < nb; s++) { u32 const ws = weights[s]; if (ws) { listSym[fill[ws]] = (u8)s; listW[fill[ws]] = (u8)ws; fill[ws]++; } }
    {   u32 acc = 0;
        for (u32 w = 1; w <= maxW; w++) { first[w] = acc; next1[w] = acc; acc += rank[w] << (w + (L - tl) - 1); }
    }
    u32 const minBits = tl + 1 - maxW;
    for (u32 i = 0; i < listSize; i++) {
        u32 const sym = listSym[i], w1 = listW[i], n = tl + 1 - w1;
        u32 const span = 1u << (L - n);
        u32* const sub = cells + next1[w1];
        next1[w1] += span;
        if (L - n >= minBits) {
            int minWeight = (int)n + ((int)tl + 1 - (int)L);
            if (minWeight < 1) minWeight = 1;
            for (u32 w = 1; w <= maxW; w++) next2[w] = first[w] >> n;
            if (minWeight > 1) { u32 const skip = next2[minWeight]; for (u32 u = 0; u < skip; u++) sub[u] = sym | (n << 16) | (1u << 24); }
            for (u32 j = listStart[minWeight]; j < listSize; j++) {
                u32 const s2 = listSym[j], w2 = listW[j], n2 = tl + 1 - w2;
                u32 const len2 = 1u << (L - n - n2);
                u32 const cell = ((sym + (s2 << 8)) & 0xFFFF) | ((n + n2) << 16) | (2u << 24);
                u32 const at = next2[w2];
                for (u32 u = 0; u < len2; u++) sub[at + u] = cell;
                next2[w2] += len2;
            }
        } else for (u32 u = 0; u < span; u++) sub[u] = sym | (n << 16) | (1u << 24);
    }
    dt[0] = (hdr & 0xFF0000FFu) | (1u << 8) | (L << 16);
    return h;
}

// One stream with the single-symbol table into out[p .. pe) (HUF_decodeStreamX1, huf_decompress.c:214-237): returns the
// BIT_initDStream verdict; *done = stream consumed exactly (:348-349).  dtab = { header word, HUF_DEltX1 { byte, nbBits } cells }.
__device__ inline u64 d_huf_decode_stream_x1(u8* out, long long p, long long const pe, const u8* s, u64 len, const u32* dtab, u32* done)
{
    const u16* const cells = reinterpret_cast<const u16*>(dtab + 1);
    u32 const dtLog = (dtab[0] >> 16) & 0xFF;
    BitSrc b;
    *done = 0;
    u64 const ie = bs_open(b, s, len);
    if (is_err(ie)) return ie;
    auto sym = [&]() { u32 const cell = cells[bs_peek_fast(b, dtLog)]; b.used += cell >> 8; out[p++] = (u8)cell; };
    while ((bs_refill(b) == SRC_MORE) & (p < pe - 3)) { sym(); sym(); sym(); sym(); }
    while (p < pe) sym();
    *done = bs_exhausted(b) ? 1u : 0u;
    return 0;
}

// One stream with the double-symbol table into out[p .. pe): returns the BIT_initDStream verdict; *done = stream consumed exactly.
__device__ inline u64 d_huf_decode_stream_x2(u8* out, long long p, long long const pe, const u8* s, u64 len, const u32* dtab, u32* done)
{
    const u32* const cells = dtab + 1;
    u32 const dtLog = (dtab[0] >> 16) & 0xFF;
    BitSrc b;
    *done = 0;
    u64 const ie = bs_open(b, s, len);
    if (is_err(ie)) return ie;
    auto sym2 = [&]() {                                              // HUF_decodeSymbolX2 :659-666
        u32 const cell = cells[bs_peek_fast(b, dtLog)];
        out[p] = (u8)cell; out[p + 1] = (u8)(cell >> 8);
        b.used += (cell >> 16) & 0xFF; p += cell >> 24;
    };
    while ((bs_refill(b) == SRC_MORE) & (p < pe - 7)) { sym2(); sym2(); sym2(); sym2(); }   // HUF_decodeStreamX2 :693-720
    while ((bs_refill(b) == SRC_MORE) & (p <= pe - 2)) sym2();
    while (p <= pe - 2) sym2();
    if (p < pe) {                                                    // HUF_decodeLastSymbolX2 :668-683
        u32 const cell = cells[bs_peek_fast(b, dtLog)];
        u32 const nbb = (cell >> 16) & 0xFF;
        out[p++] = (u8)cell;
        if ((cell >> 24) == 1) b.used += nbb;
        else if (b.used < 64) { b.used += nbb; if (b.used > 64) b.used = 64; }
    }
    *done = bs_exhausted(b) ? 1u : 0u;
    return 0;
}

typedef u64 (*HufStreamDecoder)(u8* out, long long p, long long pe, const u8* s, u64 len, const u32* dtab, u32* done);

// CTA-cooperative payload decode with a table image: four streams (HUF_decompress4X{1,2}_usingDTable, huf_decompress.c:262-354,
// 749-862) or one (HUF_decompress1X{1,2}_usingDTable, :240-260,722-747), thread k decoding stream k with DEC
// (d_huf_decode_stream_x1 or _x2).  Every thread of the CTA must call it (barriers inside).  s_init / s_done: 4-entry shared
// scratch.  Returns the reference's value (all threads).
template <HufStreamDecoder DEC>
__device__ inline u64 cta_huf_decode(bool four, const u32* dtab, const u8* c, u64 cs, u8* out, u64 n, u64* s_init, u32* s_done)
{
    int const tid = threadIdx.x;
    bool bad = four && cs < 10;                                                      // :268,751
    u64 l1 = 0, l2 = 0, l3 = 0, l4 = 0;
    if (four && !bad) {
        l1 = c[0] | ((u64)c[1] << 8); l2 = c[2] | ((u64)c[3] << 8); l3 = c[4] | ((u64)c[5] << 8);
        if (l1 + l2 + l3 + 6 > cs) bad = true; else l4 = cs - (l1 + l2 + l3 + 6);   // :787 (the reference would read out of bounds)
    }
    u64 const seg = four ? (n + 3) / 4 : n;
    if (four && !bad && 3 * seg > n) bad = true;                                     // dstSize < 6: the reference writes out of bounds (documented deviation)
    int const nStreams = four ? 4 : 1;
    if (tid < nStreams) {
        u64 ie = 0; u32 done = 0;
        if (!bad) {
            u64 const lens[4] = { four ? l1 : cs, l2, l3, l4 };
            u64 off = four ? 6 : 0; for (int k = 0; k < tid; k++) off += lens[k];
            long long const p = (long long)(seg * tid); long long const pe = (four && tid < 3) ? (long long)(seg * (tid + 1)) : (long long)n;
            ie = DEC(out, p, pe, c + off, lens[tid], dtab, &done);
        }
        s_init[tid] = ie; s_done[tid] = done;
    }
    __syncthreads();
    u64 r = n;
    if (bad) r = err(E_CORRUPT);
    else {
        bool initFailed = false; u32 all = 1;
        for (int k = 0; k < nStreams; k++) { if (!initFailed && is_err(s_init[k])) { r = s_init[k]; initFailed = true; } all &= s_done[k]; }   // CHECK_F in stream order (:788-791)
        if (!initFailed && !all) r = err(E_CORRUPT);                                 // :855-856
    }
    __syncthreads();
    return r;
}

}  // namespace fseb
