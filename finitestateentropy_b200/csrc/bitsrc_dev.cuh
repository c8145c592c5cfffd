// bitsrc_dev.cuh -- exact device model of the reference's backward bit reader (BIT_DStream_t,
// lib/bitstream.h:91-102,272-448) and the 2-state tANS decoder on top of it
// (FSE_decompress_usingDTable_generic, lib/fse_decompress.c:178-238).  One lane per stream.
//
// This byte-granular form is used where error verdicts on malformed input must match the CPU
// library exactly and the stream is short (Huffman weight headers, single-lane fallbacks).
#pragma once
#include "common.cuh"

namespace fseb {

struct BitSrc {
    const u8* s; u64 len; u64 at; u64 w; unsigned used;
};
enum { SRC_MORE = 0, SRC_ENDBUF = 1, SRC_DONE = 2, SRC_OVER = 3 };

__device__ __forceinline__ u64 ld64u(const u8* p)
{
    return (u64)rd32(p) | ((u64)rd32(p + 4) << 32);
}

__device__ inline u64 bs_open(BitSrc& b, const u8* p, u64 len)
{
    b.s = p; b.len = len; b.at = 0; b.w = 0; b.used = 0;
    if (len < 1) return err(E_SRC_WRONG);
    if (len >= 8) {
        b.at = len - 8; b.w = ld64u(p + b.at);
        if (p[len - 1] == 0) return err(E_GENERIC);
        b.used = 8 - hibit(p[len - 1]);
    } else {
        b.w = p[0];
        for (u64 i = 1; i < len; i++) b.w += (u64)p[i] << (8 * i);
        if (p[len - 1] == 0) return err(E_CORRUPT);
        b.used = 8 - hibit(p[len - 1]);
        b.used += (unsigned)(8 - len) * 8;
    }
    return len;
}
__device__ __forceinline__ u64 bs_peek(const BitSrc& b, unsigned nb)
{
    u64 const mask = nb ? ((1ULL << nb) - 1) : 0;
    return (b.w >> ((64u - b.used - nb) & 63u)) & mask;
}
__device__ __forceinline__ u64 bs_peek_fast(const BitSrc& b, unsigned nb)
{
    return (b.w << (b.used & 63u)) >> ((64u - nb) & 63u);
}
__device__ __forceinline__ u64 bs_read(BitSrc& b, unsigned nb) { u64 v = bs_peek(b, nb); b.used += nb; return v; }
__device__ __forceinline__ u64 bs_read_fast(BitSrc& b, unsigned nb) { u64 v = bs_peek_fast(b, nb); b.used += nb; return v; }
__device__ inline int bs_refill_fast(BitSrc& b)
{
    if (b.at < 8) return SRC_OVER;
    b.at -= b.used >> 3; b.used &= 7; b.w = ld64u(b.s + b.at);
    return SRC_MORE;
}
__device__ inline int bs_refill(BitSrc& b)
{
    if (b.used > 64) return SRC_OVER;
    if (b.at >= 8) return bs_refill_fast(b);
    if (b.at == 0) return b.used < 64 ? SRC_ENDBUF : SRC_DONE;
    u64 nb = b.used >> 3; int st = SRC_MORE;
    if (b.at < nb) { nb = b.at; st = SRC_ENDBUF; }
    b.at -= nb; b.used -= (unsigned)nb * 8; b.w = ld64u(b.s + b.at);
    return st;
}
__device__ __forceinline__ bool bs_exhausted(const BitSrc& b) { return b.at == 0 && b.used == 64; }

__device__ __forceinline__ u8 fse_dec_step(u32& state, BitSrc& b, const u32* cells, bool fast)
{
    u32 const cell = cells[state];
    u32 const nb = cell >> 24;
    u64 const low = fast ? bs_read_fast(b, nb) : bs_read(b, nb);
    state = (cell & 0xFFFF) + (u32)low;
    return (u8)(cell >> 16);
}

// The 2-state loops of FSE_decompress_usingDTable_generic (fse_decompress.c:206-235), from output position op with states
// s1, s2 onwards: returns the decoded size or the reference's verdict.  step(state) decodes one symbol through the caller's
// table layout and advances that state and b.
template <typename Step>
__device__ __forceinline__ u64 d_fse_decode_2state(u8* out, long long op, long long omax, u32 s1, u32 s2, BitSrc& b, Step step)
{
    for (; (bs_refill(b) == SRC_MORE) & (op < omax - 3); op += 4) {
        out[op] = (u8)step(s1);
        out[op + 1] = (u8)step(s2);
        out[op + 2] = (u8)step(s1);
        out[op + 3] = (u8)step(s2);
    }
    for (;;) {
        if (op > omax - 2) return err(E_DST_TOO_SMALL);
        out[op++] = (u8)step(s1);
        if (bs_refill(b) == SRC_OVER) { out[op++] = (u8)step(s2); return (u64)op; }
        if (op > omax - 2) return err(E_DST_TOO_SMALL);
        out[op++] = (u8)step(s2);
        if (bs_refill(b) == SRC_OVER) { out[op++] = (u8)step(s1); return (u64)op; }
    }
}

// Exact single-lane 2-state decoder (byte symbols).  dt = {tableLog | fastMode<<16, cells...}.
__device__ inline u64 d_fse_decode_serial(u8* out, u64 cap, const u8* cSrc, u64 cSize, const u32* dt)
{
    unsigned const tl = dt[0] & 0xFFFF;
    bool const fast = (dt[0] >> 16) != 0;
    const u32* const cells = dt + 1;
    BitSrc b;
    {   u64 const e = bs_open(b, cSrc, cSize); if (is_err(e)) return e; }
    u32 const s1 = (u32)bs_read(b, tl); bs_refill(b);
    u32 const s2 = (u32)bs_read(b, tl); bs_refill(b);
    return d_fse_decode_2state(out, 0, (long long)cap, s1, s2, b, [&](u32& s) { return fse_dec_step(s, b, cells, fast); });
}

}  // namespace fseb
