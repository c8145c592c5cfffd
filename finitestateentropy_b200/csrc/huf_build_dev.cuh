// huf_build_dev.cuh -- device-side Huffman code construction and tree-header writer.
//
//   HUF_buildCTable_wksp  lib/huf_compress.c:338-410  (HUF_sort :307-329, HUF_setMaxHeight :215-291)
//   HUF_writeCTable       lib/huf_compress.c:114-147  (HUF_compressWeights :63-103)
// Tie-breaks that decide the compressed bytes are kept: sort = decreasing count, ties by increasing
// symbol; the merge takes the internal node on equal counts; the depth limiter's repayment order;
// codes are canonical with the longest lengths numbered from 0, symbol order inside a length.
// CTable cell = val | nbBits << 16 (the {U16 val; BYTE nbBits} layout of huf_compress.c:106-109).
#pragma once
#include "common.cuh"
#include "fse_dev.cuh"
#include "sink_dev.cuh"

namespace fseb {

struct HNode { u32 count; u16 parent; u8 sym; u8 len; };

// Node views for d_huf_limit_depth: count(i), len(i), set_len(i, v) of the leaves in rank order.
struct HNodeView {                 // HNode array
    HNode* p;
    __device__ u32 count(int i) const { return p[i].count; }
    __device__ u32 len(int i) const { return p[i].len; }
    __device__ void set_len(int i, u32 v) const { p[i].len = (u8)v; }
};
struct PackedNodeView {            // one u32 per node, count in the low 24 bits and length above; node i at p[i * stride]
    u32* p; int stride;
    __device__ u32 count(int i) const { return p[i * stride] & 0xFFFFFFu; }
    __device__ u32 len(int i) const { return p[i * stride] >> 24; }
    __device__ void set_len(int i, u32 v) const { u32& x = p[i * stride]; x = (x & 0xFFFFFFu) | (v << 24); }
};

// HUF_setMaxHeight, one lane; node -1 must be addressable with length 0
template <class Nodes>
__device__ inline u32 d_huf_limit_depth(Nodes nd, u32 last, u32 maxBits)
{
    u32 const deepest = nd.len(last);
    if (deepest <= maxBits) return deepest;
    int debt = 0;
    u32 const unit = 1u << (deepest - maxBits);
    int n = (int)last;
    u32 const NONE = 0xF0F0F0F0u;
    u32 lastOfRank[HUF_MAX_TLOG + 2];
    while (nd.len(n) > maxBits) {
        debt += (int)(unit - (1u << (deepest - nd.len(n))));
        nd.set_len(n, maxBits); n--;
    }
    while (nd.len(n) == maxBits) n--;
    debt >>= (deepest - maxBits);
    for (u32 i = 0; i < HUF_MAX_TLOG + 2; i++) lastOfRank[i] = NONE;
    {   u32 cur = maxBits;
        for (int pos = n; pos >= 0; pos--) {
            if (nd.len(pos) >= cur) continue;
            cur = nd.len(pos);
            lastOfRank[maxBits - cur] = (u32)pos;
        }
    }
    while (debt > 0) {
        u32 dec = hibit((u32)debt) + 1;
        for (; dec > 1; dec--) {
            u32 const hi = lastOfRank[dec], lo = lastOfRank[dec - 1];
            if (hi == NONE) continue;
            if (lo == NONE) break;
            if (nd.count(hi) <= 2 * nd.count(lo)) break;
        }
        while (dec <= HUF_MAX_TLOG && lastOfRank[dec] == NONE) dec++;
        debt -= 1 << (dec - 1);
        if (lastOfRank[dec - 1] == NONE) lastOfRank[dec - 1] = lastOfRank[dec];
        nd.set_len(lastOfRank[dec], nd.len(lastOfRank[dec]) + 1);
        if (lastOfRank[dec] == 0) lastOfRank[dec] = NONE;
        else {
            lastOfRank[dec]--;
            if (nd.len(lastOfRank[dec]) != maxBits - dec) lastOfRank[dec] = NONE;
        }
    }
    while (debt < 0) {
        if (lastOfRank[1] == NONE) {
            while (nd.len(n) == maxBits) n--;
            nd.set_len(n + 1, nd.len(n + 1) - 1);
            lastOfRank[1] = (u32)(n + 1);
            debt++;
            continue;
        }
        nd.set_len(lastOfRank[1] + 1, nd.len(lastOfRank[1] + 1) - 1);
        lastOfRank[1]++;
        debt++;
    }
    return maxBits;
}

// CTA-cooperative (blockDim.x == 256).  count/ctable/lenOf/firstVal live in shared memory.
// store: HNode[2*256+2].  Returns the maximum code length, or an error code; contains barriers.
__device__ inline u64 cta_huf_build_ctable(u32* ctable, const u32* count, u32 msv, u32 maxBits,
                                           HNode* store, u32* lenOf, u32* firstVal)
{
    int const tid = threadIdx.x;
    HNode* const nd = store + 1;
    __shared__ u32 s_ret;
    if (!maxBits) maxBits = HUF_DEF_TLOG;
    if (msv > HUF_MAX_SV) return err(E_MSV_TOO_LARGE);
    for (int i = tid; i < 2 * 256 + 2; i += blockDim.x) { HNode z; z.count = 0; z.parent = 0; z.sym = 0; z.len = 0; store[i] = z; }
    __syncthreads();
    if ((u32)tid <= msv) {                                   // rank by counting == stable sort by decreasing count
        u32 const c = count[tid];
        u32 rank = 0;
        for (u32 jj = 0; jj <= msv; jj++) { u32 const cj = count[jj]; rank += (cj > c) | ((cj == c) & (jj < (u32)tid)); }
        nd[rank].count = c; nd[rank].sym = (u8)tid;
    }
    __syncthreads();
    if (tid == 0) {
        int last = (int)msv; while (nd[last].count == 0) last--;
        int fresh = 256, leaf = last, root = fresh + leaf - 1, inner = fresh;
        nd[fresh].count = nd[leaf].count + nd[leaf - 1].count;
        nd[leaf].parent = nd[leaf - 1].parent = (u16)fresh;
        fresh++; leaf -= 2;
        for (int n = fresh; n <= root; n++) nd[n].count = 1u << 30;
        nd[-1].count = 1u << 31;
        while (fresh <= root) {
            int const a = (nd[leaf].count < nd[inner].count) ? leaf-- : inner++;
            int const b = (nd[leaf].count < nd[inner].count) ? leaf-- : inner++;
            nd[fresh].count = nd[a].count + nd[b].count;
            nd[a].parent = nd[b].parent = (u16)fresh;
            fresh++;
        }
        nd[root].len = 0;
        for (int n = root - 1; n >= 256; n--) nd[n].len = (u8)(nd[nd[n].parent].len + 1);
        for (int n = 0; n <= last; n++) nd[n].len = (u8)(nd[nd[n].parent].len + 1);
        u32 const mb = d_huf_limit_depth(HNodeView{ nd }, (u32)last, maxBits);
        s_ret = mb;
        if (mb <= HUF_MAX_TLOG) {
            u32 perLen[HUF_MAX_TLOG + 1];
            for (u32 i = 0; i <= HUF_MAX_TLOG; i++) perLen[i] = 0;
            for (int n = 0; n <= last; n++) perLen[nd[n].len]++;
            u32 v = 0;
            for (u32 i = 0; i <= HUF_MAX_TLOG; i++) firstVal[i] = 0;
            for (int n = (int)mb; n > 0; n--) { firstVal[n] = v; v = (v + perLen[n]) >> 1; }
        }
    }
    __syncthreads();
    u32 const mb = s_ret;
    if (mb > HUF_MAX_TLOG) return err(E_GENERIC);
    if ((u32)tid <= msv) lenOf[nd[tid].sym] = nd[tid].len;
    __syncthreads();
    if ((u32)tid <= msv) {                                   // value = first value of the length + number of earlier symbols of that length
        u32 const len = lenOf[tid];
        u32 before = 0;
        for (u32 jj = 0; jj < (u32)tid; jj++) before += (lenOf[jj] == len);
        ctable[tid] = ((firstVal[len] + before) & 0xFFFF) | (len << 16);
    } else ctable[tid & 255] = 0;
    __syncthreads();
    return mb;
}

// 256 keys, element e = i * 32 + lane, sorted into DEcreasing order (bitonic network: shuffles for partners in other
// lanes, plain compare-exchange for partners in the same lane).  Keys must be distinct.
__device__ __forceinline__ void warp_sort256_desc(u32 (&key)[8], unsigned lane)
{
    #pragma unroll
    for (u32 k = 2; k <= 256; k <<= 1) {
        #pragma unroll
        for (u32 j = k >> 1; j > 0; j >>= 1) {
            if (j >= 32) {
                u32 const dj = j >> 5;
                #pragma unroll
                for (u32 i = 0; i < 8; i++) {
                    if (i & dj) continue;
                    u32 const e = i * 32;                          // lane bits do not matter for k >= 64
                    bool const desc = (k == 256) || ((e & k) != 0) ;
                    u32 const lo = min(key[i], key[i | dj]), hi = max(key[i], key[i | dj]);
                    key[i] = desc ? hi : lo; key[i | dj] = desc ? lo : hi;
                }
            } else {
                #pragma unroll
                for (u32 i = 0; i < 8; i++) {
                    u32 const e = i * 32 + lane;
                    u32 const other = __shfl_xor_sync(0xFFFFFFFFu, key[i], j);
                    bool const asc = (k == 256) ? false : ((e & k) == 0);
                    bool const takeMin = ((e & j) == 0) == asc;
                    key[i] = takeMin ? min(key[i], other) : max(key[i], other);
                }
            }
        }
    }
}

// HUF_compressWeights, one lane.  wksp: >= 160 u32 of scratch.
__device__ inline u64 d_huf_compress_weights(u8* out, u64 cap, const u8* w, u64 n, u32* wksp)
{
    unsigned* const count = wksp;                     // 13
    short* const norm = (short*)(wksp + 16);          // 13 shorts
    u32* const ct = wksp + 24;                        // 1 + 32 + 2*13 = 59
    u16* const cellSym = (u16*)(wksp + 84);           // 64 u16
    u32* const start = wksp + 116;                    // 15
    unsigned msv = HUF_MAX_TLOG, tl = 6, best = 0;
    if (n <= 1) return 0;
    for (unsigned i = 0; i <= HUF_MAX_TLOG; i++) count[i] = 0;
    for (u64 i = 0; i < n; i++) count[w[i]]++;
    while (!count[msv]) msv--;
    for (unsigned s = 0; s <= msv; s++) best = count[s] > best ? count[s] : best;
    if (best == n) return 1;
    if (best == 1) return 0;
    tl = d_optimal_tablelog(tl, n, msv, 2);
    u64 r = d_normalize(norm, tl, count, n, msv); if (is_err(r)) return r;
    r = d_write_ncount(out, cap, norm, msv, tl); if (is_err(r)) return r;
    u64 const o = r;
    d_build_ctable_serial(ct, norm, msv, tl, cellSym, start);
    r = d_fse_encode_serial(out + o, cap - o, w, n, ct);
    if (r == 0) return 0;
    return o + r;
}

// HUF_writeCTable, one lane.  `out` has room for min(cap,136) bytes where cap is the caller's capacity.
// ctable: anything indexable by symbol (a plain array, or a column of an interleaved one).
template <class CTable>
__device__ inline u64 d_huf_write_ctable(u8* out, u64 cap, CTable ctable, unsigned msv, unsigned huffLog, u32* wksp)
{
    u8* const weight = (u8*)(wksp + 160);             // 256 bytes
    if (msv > HUF_MAX_SV) return err(E_MSV_TOO_LARGE);
    for (unsigned n = 0; n < msv; n++) {
        unsigned const len = (ctable[n] >> 16) & 0xFF;
        weight[n] = (u8)(len ? huffLog + 1 - len : 0);
    }
    {   u64 const h = d_huf_compress_weights(out + 1, cap - 1, weight, msv, wksp);
        if (is_err(h)) return h;
        if ((h > 1) & (h < msv / 2)) { out[0] = (u8)h; return h + 1; }
    }
    if (msv > 128) return err(E_GENERIC);
    if (((msv + 1) / 2) + 1 > cap) return err(E_DST_TOO_SMALL);
    out[0] = (u8)(128 + (msv - 1));
    weight[msv] = 0;
    for (unsigned n = 0; n < msv; n += 2) out[(n / 2) + 1] = (u8)((weight[n] << 4) + weight[n + 1]);
    return ((msv + 1) / 2) + 1;
}

}  // namespace fseb
