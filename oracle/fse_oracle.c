/*
 * fse_oracle.c -- plain-C CPU restatement of the reference's block entropy-coding hot path.
 *
 * TEST INFRASTRUCTURE ONLY (see fse_oracle.h).  Written from the reference's behaviour, not
 * copied from its sources: one translation unit, byte-array/bit-position formulation, explicit
 * little-endian packing of the table layouts.  Parity is PINNED against the compiled reference
 * (oracle/_ref), tests/golden/ and SURVEY.md section 6.3 by tests/test_oracle_vs_ref.py.
 *
 * Known, documented deviations (all on inputs the reference itself treats as unsupported):
 *   - orc_huf_decode4x1 refuses dstSize < 6 (the reference would write 1 byte out of bounds,
 *     lib/huf_decompress.c:291-296,344-347); HUF_compress never emits such blocks (:565).
 *   - orc_fse_compress2 builds its CTable in private storage.  FSE_compress_wksp lays CTable+scratch
 *     out for the *requested* tableLog and maxSymbolValue (lib/fse_compress.c:641-643) but builds with
 *     the tableLog FSE_optimalTableLog returns (:658,667); the reference's call can fault on raised
 *     requests and where the requested CTable alone exceeds its workspace.  Those are answered as the
 *     same steps done one reference function at a time answer them (tests/table_logs.py:fse_steps).
 *   - orc_fse_decompress_u16 returns `corruption` for an empty payload where the reference
 *     dereferences a NULL stream pointer (lib/fseU16.c:286-287 with lib/bitstream.h:274).
 *
 * All `file:line` citations are relative to /root/reference/.
 */
#include "fse_oracle.h"
#include <string.h>

typedef uint8_t u8;
typedef uint16_t u16;
typedef uint32_t u32;
typedef uint64_t u64;

#define FSE_MIN_TLOG 5          /* lib/fse.h:675 */
#define FSE_MAX_TLOG 12         /* lib/fse.h:641,672 (memory usage 14) */
#define FSE_DEF_TLOG 11         /* lib/fse.h:644,674 */
#define FSE_ABS_TLOG 15         /* lib/fse.h:676 */
#define FSE_MAX_SV 255          /* lib/fse.h:653 */
#define U16_MAX_SV 286          /* lib/fseU16.h:49-51 */
#define U16_MAX_TLOG 13         /* lib/fseU16.c:43-45,97 */
#define U16_DEF_TLOG 12         /* lib/fseU16.c:46-48 */
#define HUF_MAX_TLOG 12         /* lib/huf.h:117 */
#define HUF_DEF_TLOG 11         /* lib/huf.h:118 */
#define HUF_MAX_SV 255          /* lib/huf.h:119 */
#define HUF_BLOCK_MAX (128 * 1024)  /* lib/huf.h:72 */

unsigned orc_is_error(size_t code) { return code > ORC_ERROR(ORC_MAXCODE); }   /* lib/error_private.h:79 */

static unsigned hibit(u32 v) { unsigned r = 0; while (v >>= 1) r++; return r; } /* lib/bitstream.h:139 (0 -> 0 here) */
static u32 rd16(const u8* p) { return (u32)p[0] | ((u32)p[1] << 8); }
static u32 rd32(const u8* p) { return rd16(p) | (rd16(p + 2) << 16); }
static u64 rd64(const u8* p) { return (u64)rd32(p) | ((u64)rd32(p + 4) << 32); }
static void wr16(u8* p, u32 v) { p[0] = (u8)v; p[1] = (u8)(v >> 8); }

/* ------------------------------------------------------------------------------------------
 * forward bit sink (wire format of lib/bitstream.h:57-63,183-260): bits are appended LSB-first;
 * closing adds a single 1 ("end mark").  Capacity rule (:190-191,246,258): the stream is refused
 * (size 0) when cap <= 8 or when floor(totalBits/8) >= cap-8, whatever the flush schedule was.
 * ------------------------------------------------------------------------------------------ */
typedef struct { u8* out; size_t cap; u64 acc; unsigned held; size_t nbytes; u64 nbits; int usable; } bsink;

static void sink_open(bsink* s, void* dst, size_t cap)
{
    s->out = (u8*)dst; s->cap = cap; s->acc = 0; s->held = 0; s->nbytes = 0; s->nbits = 0;
    s->usable = cap > 8;
}
static void sink_put(bsink* s, u32 value, unsigned nb)
{
    if (nb == 0) return;
    s->acc |= ((u64)value & (((u64)1 << nb) - 1)) << s->held;
    s->held += nb; s->nbits += nb;
    while (s->held >= 8) {
        if (s->nbytes < s->cap) s->out[s->nbytes] = (u8)s->acc;
        s->nbytes++; s->acc >>= 8; s->held -= 8;
    }
}
static size_t sink_close(bsink* s)
{
    if (!s->usable) return 0;
    sink_put(s, 1, 1);
    if ((s->nbits >> 3) >= (u64)(s->cap - 8)) return 0;
    if (s->held) { s->out[s->nbytes] = (u8)s->acc; s->nbytes++; }
    return s->nbytes;
}

/* ------------------------------------------------------------------------------------------
 * backward bit source: exact model of BIT_DStream_t (lib/bitstream.h:91-102,272-448).
 * `at` is the byte offset of the 64-bit window, `used` the bits already consumed from its top.
 * ------------------------------------------------------------------------------------------ */
typedef struct { const u8* s; size_t len; size_t at; u64 w; unsigned used; } bsrc;
enum { SRC_MORE = 0, SRC_ENDBUF = 1, SRC_DONE = 2, SRC_OVER = 3 };   /* lib/bitstream.h:99-102 */

static size_t src_open(bsrc* b, const void* data, size_t len)          /* lib/bitstream.h:272-318 */
{
    const u8* p = (const u8*)data;
    memset(b, 0, sizeof(*b));
    if (len < 1) return ORC_ERROR(ORC_SRC_WRONG);
    b->s = p; b->len = len;
    if (len >= 8) {
        b->at = len - 8; b->w = rd64(p + b->at);
        if (p[len - 1] == 0) return ORC_ERROR(ORC_GENERIC);
        b->used = 8 - hibit(p[len - 1]);
    } else {
        size_t i;
        b->at = 0; b->w = p[0];
        for (i = 1; i < len; i++) {              /* bytes 1..3 at their natural place, 4..6 at 32,40,48 */
            unsigned const sh = (unsigned)(8 * i);
            b->w += (u64)p[i] << sh;
        }
        if (p[len - 1] == 0) return ORC_ERROR(ORC_CORRUPT);
        b->used = 8 - hibit(p[len - 1]);
        b->used += (unsigned)(8 - len) * 8;
    }
    return len;
}
static u64 src_peek(const bsrc* b, unsigned nb)                         /* lib/bitstream.h:331-353 */
{
    u64 const mask = nb ? (((u64)1 << nb) - 1) : 0;
    return (b->w >> ((64u - b->used - nb) & 63u)) & mask;
}
static u64 src_peek_fast(const bsrc* b, unsigned nb)                    /* lib/bitstream.h:361-366, nb >= 1 */
{
    return (b->w << (b->used & 63u)) >> ((64u - nb) & 63u);
}
static u64 src_read(bsrc* b, unsigned nb) { u64 v = src_peek(b, nb); b->used += nb; return v; }
static u64 src_read_fast(bsrc* b, unsigned nb) { u64 v = src_peek_fast(b, nb); b->used += nb; return v; }
static int src_refill_fast(bsrc* b)                                     /* lib/bitstream.h:400-410 */
{
    if (b->at < 8) return SRC_OVER;
    b->at -= b->used >> 3; b->used &= 7; b->w = rd64(b->s + b->at);
    return SRC_MORE;
}
static int src_refill(bsrc* b)                                          /* lib/bitstream.h:416-440 */
{
    if (b->used > 64) return SRC_OVER;
    if (b->at >= 8) return src_refill_fast(b);
    if (b->at == 0) return b->used < 64 ? SRC_ENDBUF : SRC_DONE;
    {   size_t nb = b->used >> 3; int st = SRC_MORE;
        if (b->at < nb) { nb = b->at; st = SRC_ENDBUF; }
        b->at -= nb; b->used -= (unsigned)nb * 8; b->w = rd64(b->s + b->at);
        return st;
    }
}
static int src_exhausted(const bsrc* b) { return b->at == 0 && b->used == 64; }   /* lib/bitstream.h:445-448 */

/* ==========================================================================================
 * a1  histogram -- HIST_count / HIST_count_wksp (lib/hist.c:163-180; kernels :29-54,:66-133).
 * The result does not depend on which internal kernel runs.
 * ========================================================================================== */
size_t orc_hist_count(unsigned* count, unsigned* msvPtr, const void* src, size_t n)
{
    unsigned full[256];
    unsigned const declared = *msvPtr > 255 ? 255 : *msvPtr;
    const u8* p = (const u8*)src;
    unsigned top = 255, best = 0, s;
    size_t i;
    if (n == 0) { memset(count, 0, (declared + 1) * sizeof(*count)); *msvPtr = 0; return 0; }
    memset(full, 0, sizeof(full));
    for (i = 0; i < n; i++) full[p[i]]++;
    while (!full[top]) top--;
    if (declared < 255 && top > declared) return ORC_ERROR(ORC_MSV_TOO_SMALL);   /* hist.c:128 */
    for (s = 0; s < 256; s++) if (full[s] > best) best = full[s];
    memcpy(count, full, (declared + 1) * sizeof(*count));
    *msvPtr = top;
    return best;
}

/* a2  FSE_optimalTableLog_internal / FSE_minTableLog (lib/fse_compress.c:316-342) */
static unsigned min_tablelog(size_t srcSize, unsigned msv)
{
    unsigned const bySrc = hibit((u32)srcSize) + 1, bySym = hibit(msv) + 2;
    return bySrc < bySym ? bySrc : bySym;
}
unsigned orc_optimal_tablelog(unsigned maxTableLog, size_t srcSize, unsigned msv, unsigned minus)
{
    unsigned const bySrc = hibit((u32)(srcSize - 1)) - minus;
    unsigned const floorBits = min_tablelog(srcSize, msv);
    unsigned tl = maxTableLog ? maxTableLog : FSE_DEF_TLOG;
    if (bySrc < tl) tl = bySrc;
    if (floorBits > tl) tl = floorBits;
    if (tl < FSE_MIN_TLOG) tl = FSE_MIN_TLOG;
    if (tl > FSE_MAX_TLOG) tl = FSE_MAX_TLOG;
    return tl;
}

/* a3  FSE_normalizeCount + FSE_normalizeM2 (lib/fse_compress.c:348-494) */
static size_t normalize_fallback(short* norm, unsigned tl, const unsigned* count, size_t total, unsigned msv)
{
    enum { PENDING = -2 };
    u32 const lowThr = (u32)(total >> tl);
    u32 lowOne = (u32)((total * 3) >> (tl + 1));
    u32 given = 0, left, s;
    for (s = 0; s <= msv; s++) {
        if (count[s] == 0) { norm[s] = 0; continue; }
        if (count[s] <= lowThr) { norm[s] = -1; given++; total -= count[s]; continue; }
        if (count[s] <= lowOne) { norm[s] = 1; given++; total -= count[s]; continue; }
        norm[s] = PENDING;
    }
    left = ((u32)1 << tl) - given;
    if (left == 0) return 0;
    if ((total / left) > lowOne) {                      /* fse_compress.c:380-391 */
        lowOne = (u32)((total * 3) / (left * 2));
        for (s = 0; s <= msv; s++)
            if (norm[s] == PENDING && count[s] <= lowOne) { norm[s] = 1; given++; total -= count[s]; }
        left = ((u32)1 << tl) - given;
    }
    if (given == msv + 1) {                             /* :393-402 everything was tiny: top-up the first maximum */
        u32 argmax = 0, vmax = 0;
        for (s = 0; s <= msv; s++) if (count[s] > vmax) { vmax = count[s]; argmax = s; }
        norm[argmax] = (short)(norm[argmax] + (short)left);
        return 0;
    }
    if (total == 0) {                                   /* :404-409 round-robin over positive cells */
        for (s = 0; left > 0; s = (s + 1) % (msv + 1))
            if (norm[s] > 0) { left--; norm[s]++; }
        return 0;
    }
    {   u64 const vlog = 62 - tl;
        u64 const mid = ((u64)1 << (vlog - 1)) - 1;
        u64 const rstep = ((((u64)1 << vlog) * left) + mid) / total;
        u64 run = mid;
        for (s = 0; s <= msv; s++) {
            if (norm[s] != PENDING) continue;
            {   u64 const end = run + (u64)count[s] * rstep;
                u32 const w = (u32)(end >> vlog) - (u32)(run >> vlog);
                if (w < 1) return ORC_ERROR(ORC_GENERIC);
                norm[s] = (short)w; run = end;
            }
        }
    }
    return 0;
}

size_t orc_fse_normalize(short* norm, unsigned tl, const unsigned* count, size_t total, unsigned msv)
{
    static const u32 roundUp[8] = { 0, 473195, 504333, 520860, 550000, 700000, 750000, 830000 };  /* :445 */
    if (tl == 0) tl = FSE_DEF_TLOG;
    if (tl < FSE_MIN_TLOG) return ORC_ERROR(ORC_GENERIC);
    if (tl > FSE_MAX_TLOG) return ORC_ERROR(ORC_TLOG_TOO_LARGE);
    if (tl < min_tablelog(total, msv)) return ORC_ERROR(ORC_GENERIC);
    {   u64 const scale = 62 - tl;
        u64 const step = ((u64)1 << 62) / total;
        u64 const vstep = (u64)1 << (scale - 20);
        u32 const lowThr = (u32)(total >> tl);
        int toGive = 1 << tl;
        unsigned s, argmax = 0;
        short pmax = 0;
        for (s = 0; s <= msv; s++) {
            if (count[s] == total) return 0;            /* single symbol: caller should use RLE (:456) */
            if (count[s] == 0) { norm[s] = 0; continue; }
            if (count[s] <= lowThr) { norm[s] = -1; toGive--; continue; }
            {   u64 const scaled = (u64)count[s] * step;
                short p = (short)(scaled >> scale);
                if (p < 8) p = (short)(p + ((scaled - ((u64)p << scale)) > vstep * roundUp[p]));
                if (p > pmax) { pmax = p; argmax = s; }
                norm[s] = p; toGive -= p;
            }
        }
        if (-toGive >= (norm[argmax] >> 1)) {
            size_t const e = normalize_fallback(norm, tl, count, total, msv);
            if (orc_is_error(e)) return e;
        } else norm[argmax] = (short)(norm[argmax] + (short)toGive);
    }
    return tl;
}

/* a4  FSE_NCountWriteBound / FSE_writeNCount (lib/fse_compress.c:186-298) */
size_t orc_fse_ncount_bound(unsigned msv, unsigned tl)
{
    return msv ? (((size_t)(msv + 1) * tl) >> 3) + 3 : 512;
}

size_t orc_fse_write_ncount(void* dst, size_t cap, const short* norm, unsigned msv, unsigned tl)
{
    u8* const out = (u8*)dst;
    size_t o = 0;                                  /* bytes emitted so far */
    int const guarded = cap < orc_fse_ncount_bound(msv, tl);
    unsigned const alphabet = msv + 1;
    u32 acc; int held;
    int remaining, threshold, width;
    unsigned sym = 0; int afterZero = 0;
    if (tl > FSE_MAX_TLOG) return ORC_ERROR(ORC_TLOG_TOO_LARGE);
    if (tl < FSE_MIN_TLOG) return ORC_ERROR(ORC_GENERIC);
#define SPILL16() do { if (guarded && o + 2 > cap) return ORC_ERROR(ORC_DST_TOO_SMALL); \
                       out[o] = (u8)acc; out[o + 1] = (u8)(acc >> 8); o += 2; acc >>= 16; } while (0)
    acc = tl - FSE_MIN_TLOG; held = 4;
    remaining = (1 << tl) + 1; threshold = 1 << tl; width = (int)tl + 1;
    while (sym < alphabet && remaining > 1) {
        if (afterZero) {                           /* zero-run escape (:219-248) */
            unsigned from = sym;
            while (sym < alphabet && !norm[sym]) sym++;
            if (sym == alphabet) break;
            while (sym >= from + 24) { from += 24; acc += 0xFFFFu << held; SPILL16(); }
            while (sym >= from + 3) { from += 3; acc += 3u << held; held += 2; }
            acc += (sym - from) << held; held += 2;
            if (held > 16) { SPILL16(); held -= 16; }
        }
        {   int v = norm[sym++];
            int const cut = (2 * threshold - 1) - remaining;
            remaining -= v < 0 ? -v : v;
            v++;
            if (v >= threshold) v += cut;
            acc += (u32)v << held;
            held += width; held -= (v < cut);
            afterZero = (v == 1);
            if (remaining < 1) return ORC_ERROR(ORC_GENERIC);
            while (remaining < threshold) { width--; threshold >>= 1; }
        }
        if (held > 16) { SPILL16(); held -= 16; }
    }
    if (remaining != 1) return ORC_ERROR(ORC_GENERIC);
    if (guarded && o + 2 > cap) return ORC_ERROR(ORC_DST_TOO_SMALL);
    out[o] = (u8)acc; out[o + 1] = (u8)(acc >> 8);
    o += (size_t)((held + 7) / 8);
#undef SPILL16
    return o;
}

/* a8  FSE_readNCount (lib/entropy_common.c:41-144) */
size_t orc_fse_read_ncount(short* norm, unsigned* msvPtr, unsigned* tlPtr, const void* src, size_t hbSize)
{
    const u8* const in = (const u8*)src;
    ptrdiff_t const end = (ptrdiff_t)hbSize;
    ptrdiff_t ip = 0;
    int width, remaining, threshold, held;
    u32 bits; unsigned sym = 0; int afterZero = 0;
    if (hbSize < 4) {                              /* :55-64 pad to 4 bytes and retry */
        u8 pad[4] = { 0, 0, 0, 0 };
        size_t r;
        memcpy(pad, src, hbSize);
        r = orc_fse_read_ncount(norm, msvPtr, tlPtr, pad, sizeof(pad));
        if (orc_is_error(r)) return r;
        if (r > hbSize) return ORC_ERROR(ORC_CORRUPT);
        return r;
    }
    memset(norm, 0, (*msvPtr + 1) * sizeof(norm[0]));
    bits = rd32(in);
    width = (int)(bits & 0xF) + FSE_MIN_TLOG;
    if (width > FSE_ABS_TLOG) return ORC_ERROR(ORC_TLOG_TOO_LARGE);
    bits >>= 4; held = 4;
    *tlPtr = (unsigned)width;
    remaining = (1 << width) + 1; threshold = 1 << width; width++;
    while ((remaining > 1) & (sym <= *msvPtr)) {
        if (afterZero) {
            unsigned upto = sym;
            while ((bits & 0xFFFF) == 0xFFFF) {
                upto += 24;
                if (ip < end - 5) { ip += 2; bits = rd32(in + ip) >> held; }
                else { bits >>= 16; held += 16; }
            }
            while ((bits & 3) == 3) { upto += 3; bits >>= 2; held += 2; }
            upto += bits & 3; held += 2;
            if (upto > *msvPtr) return ORC_ERROR(ORC_MSV_TOO_SMALL);
            while (sym < upto) norm[sym++] = 0;
            if ((ip <= end - 7) || (ip + (held >> 3) <= end - 4)) {
                ip += held >> 3; held &= 7; bits = rd32(in + ip) >> held;
            } else bits >>= 2;
        }
        {   int const cut = (2 * threshold - 1) - remaining;
            int v;
            if ((bits & (u32)(threshold - 1)) < (u32)cut) { v = (int)(bits & (u32)(threshold - 1)); held += width - 1; }
            else { v = (int)(bits & (u32)(2 * threshold - 1)); if (v >= threshold) v -= cut; held += width; }
            v--;
            remaining -= v < 0 ? -v : v;
            norm[sym++] = (short)v;
            afterZero = !v;
            while (remaining < threshold) { width--; threshold >>= 1; }
            if ((ip <= end - 7) || (ip + (held >> 3) <= end - 4)) { ip += held >> 3; held &= 7; }
            else { held -= (int)(8 * (end - 4 - ip)); ip = end - 4; }
            bits = rd32(in + ip) >> (held & 31);
        }
    }
    if (remaining != 1) return ORC_ERROR(ORC_CORRUPT);
    if (held > 32) return ORC_ERROR(ORC_CORRUPT);
    *msvPtr = sym - 1;
    ip += (held + 7) >> 3;
    return (size_t)ip;
}

/* ------------------------------------------------------------------------------------------
 * symbol spreading shared by a5 and a9 (lib/fse_compress.c:96-122, lib/fse_decompress.c:91-114):
 * "-1" symbols are parked from the top cell downwards, the others walk the table with stride
 * (size/2 + size/8 + 3) (lib/fse.h:683) skipping the parked zone.  Returns 0 if the walk does
 * not close on cell 0.
 * ------------------------------------------------------------------------------------------ */
static int spread_symbols(u16* cellSym, const short* norm, unsigned msv, unsigned tl)
{
    u32 const size = (u32)1 << tl, mask = size - 1;
    u32 const stride = (size >> 1) + (size >> 3) + 3;
    u32 high = size - 1, pos = 0, s;
    for (s = 0; s <= msv; s++) if (norm[s] == -1) cellSym[high--] = (u16)s;
    for (s = 0; s <= msv; s++) {
        int k;
        for (k = 0; k < norm[s]; k++) {
            cellSym[pos] = (u16)s;
            do pos = (pos + stride) & mask; while (pos > high);
        }
    }
    return pos == 0;
}

/* a5  FSE_buildCTable_wksp (lib/fse_compress.c:66-169); image = {u16 tableLog,u16 maxSV} +
 * u16 nextState[size] + {i32 deltaFindState,u32 deltaNbBits}[maxSV+1] (lib/fse.h:295,483-486) */
size_t orc_fse_build_ctable(u32* ct, const short* norm, unsigned msv, unsigned tl)
{
    u32 const size = (u32)1 << tl;
    u16* const hdr = (u16*)(void*)ct;
    u16* const next = hdr + 2;
    u32* const tt = ct + 1 + (tl ? (size >> 1) : 1);
    u16 cellSym[1 << 13];
    u32 start[4096 + 2];
    u32 s, u;
    if (tl > 13 || msv > 4095) return ORC_ERROR(ORC_TLOG_TOO_LARGE);
    hdr[0] = (u16)tl; hdr[1] = (u16)msv;
    start[0] = 0;
    for (s = 1; s <= msv + 1; s++) start[s] = start[s - 1] + (u32)(norm[s - 1] == -1 ? 1 : norm[s - 1]);
    start[msv + 1] = size + 1;
    spread_symbols(cellSym, norm, msv, tl);
    for (u = 0; u < size; u++) next[start[cellSym[u]]++] = (u16)(size + u);   /* :125-128 */
    {   u32 total = 0;
        for (s = 0; s <= msv; s++) {
            int const n = norm[s];
            if (n == 0) { tt[2 * s + 1] = ((tl + 1) << 16) - size; continue; }     /* deltaFindState left untouched */
            if (n == -1 || n == 1) {
                tt[2 * s + 1] = (tl << 16) - size; tt[2 * s] = total - 1; total++;
            } else {
                u32 const maxOut = tl - hibit((u32)n - 1);
                tt[2 * s + 1] = (maxOut << 16) - ((u32)n << maxOut);
                tt[2 * s] = total - (u32)n; total += (u32)n;
            }
        }
    }
    return 0;
}

/* a9  FSE_buildDTable (lib/fse_decompress.c:71-126): {u16 tableLog,u16 fastMode} + cells.
 * wide==0: cell = {u16 newState,u8 symbol,u8 nbBits}; wide==1 (lib/fseU16.c:78-82):
 * {u16 newState, nbBits:4, symbol:12} */
static size_t build_dtable(u32* dt, const short* norm, unsigned msv, unsigned tl, int wide, unsigned msvLimit, unsigned tlLimit)
{
    u32 const size = (u32)1 << tl;
    u16 cellSym[1 << 13];
    u16 nextOf[4096 + 1];
    u32 s, u; unsigned fast = 1;
    if (msv > msvLimit) return ORC_ERROR(ORC_MSV_TOO_LARGE);
    if (tl > tlLimit) return ORC_ERROR(ORC_TLOG_TOO_LARGE);
    for (s = 0; s <= msv; s++) {
        if (norm[s] == -1) nextOf[s] = 1;
        else { if (norm[s] >= (short)(1 << (tl - 1))) fast = 0; nextOf[s] = (u16)norm[s]; }
    }
    dt[0] = tl | (fast << 16);
    if (!spread_symbols(cellSym, norm, msv, tl)) {
        /* the reference has already written header + symbols; it reports GENERIC (:113) */
        return ORC_ERROR(ORC_GENERIC);
    }
    for (u = 0; u < size; u++) {
        u32 const sym = cellSym[u];
        u32 const x = nextOf[sym]++;
        u32 const nb = tl - hibit(x);
        u32 const ns = ((x << nb) - size) & 0xFFFF;
        dt[1 + u] = wide ? (ns | (nb << 16) | (sym << 20)) : (ns | (sym << 16) | (nb << 24));
    }
    return 0;
}
size_t orc_fse_build_dtable(u32* dt, const short* norm, unsigned msv, unsigned tl)
{ return build_dtable(dt, norm, msv, tl, 0, FSE_MAX_SV, FSE_MAX_TLOG); }
size_t orc_fse_build_dtable_u16(u32* dt, const short* norm, unsigned msv, unsigned tl)
{ return build_dtable(dt, norm, msv, tl, 1, U16_MAX_SV, U16_MAX_TLOG); }

/* ==========================================================================================
 * a6  tANS encoder -- FSE_compress_usingCTable (lib/fse_compress.c:554-623, lib/fse.h:488-527).
 * Symbols are visited last to first; index parity selects the chain (even -> state 1,
 * odd -> state 2); a chain's first visit only seeds its state.  `chains`==1 is the U16
 * single-state variant (lib/fseU16.c:150-200) whose state starts at 2^tableLog.
 * ========================================================================================== */
typedef struct { const u16* next; const u32* tt; unsigned tl; } ctview;
static ctview ct_view(const u32* ct)
{
    ctview v;
    v.tl = ((const u16*)(const void*)ct)[0];
    v.next = ((const u16*)(const void*)ct) + 2;
    v.tt = ct + 1 + (v.tl ? ((u32)1 << (v.tl - 1)) : 1);
    return v;
}
static u32 enc_seed(const ctview* c, u32 sym)                              /* lib/fse.h:503-512 */
{
    u32 const dnb = c->tt[2 * sym + 1];
    u32 const nb = (dnb + (1u << 15)) >> 16;
    u32 const v = (nb << 16) - dnb;
    return c->next[(v >> nb) + (u32)(int32_t)c->tt[2 * sym]];
}
static u32 enc_step(bsink* s, const ctview* c, u32 state, u32 sym)       /* lib/fse.h:514-521 */
{
    u32 const nb = (state + c->tt[2 * sym + 1]) >> 16;
    sink_put(s, state, nb);
    return c->next[(state >> nb) + (u32)(int32_t)c->tt[2 * sym]];
}

size_t orc_fse_encode(void* dst, size_t cap, const void* src, size_t n, const u32* ct)
{
    ctview const c = ct_view(ct);
    const u8* const in = (const u8*)src;
    bsink s;
    u32 st[2] = { 0, 0 }; int seeded[2] = { 0, 0 };
    size_t i;
    if (n <= 2) return 0;
    sink_open(&s, dst, cap);
    if (!s.usable) return 0;
    for (i = n; i-- > 0;) {
        unsigned const k = (unsigned)(i & 1);
        if (!seeded[k]) { st[k] = enc_seed(&c, in[i]); seeded[k] = 1; }
        else st[k] = enc_step(&s, &c, st[k], in[i]);
    }
    sink_put(&s, st[1], c.tl);                                           /* fse_compress.c:608-609 */
    sink_put(&s, st[0], c.tl);
    return sink_close(&s);
}

static size_t fse_encode_u16(void* dst, size_t cap, const u16* in, size_t n, const u32* ct)
{
    ctview const c = ct_view(ct);
    bsink s; u32 st = (u32)1 << c.tl;
    size_t i;
    sink_open(&s, dst, cap);
    for (i = n; i-- > 0;) st = enc_step(&s, &c, st, in[i]);
    sink_put(&s, st, c.tl);
    return sink_close(&s);
}

/* a10  tANS decoder -- FSE_decompress_usingDTable (lib/fse_decompress.c:178-252) */
static u8 dec_step(u32* state, bsrc* b, const u32* cells, int fast)     /* lib/fse.h:600-622 */
{
    u32 const cell = cells[*state];
    u32 const nb = cell >> 24;
    u64 const low = fast ? src_read_fast(b, nb) : src_read(b, nb);
    *state = (cell & 0xFFFF) + (u32)low;
    return (u8)(cell >> 16);
}

size_t orc_fse_decode(void* dst, size_t cap, const void* cSrc, size_t cSize, const u32* dt)
{
    u8* const out = (u8*)dst;
    unsigned const tl = dt[0] & 0xFFFF;
    int const fast = (dt[0] >> 16) != 0;
    const u32* const cells = dt + 1;
    ptrdiff_t const omax = (ptrdiff_t)cap;
    ptrdiff_t op = 0;
    bsrc b; u32 s1, s2;
    {   size_t const e = src_open(&b, cSrc, cSize); if (orc_is_error(e)) return e; }
    s1 = (u32)src_read(&b, tl); src_refill(&b);
    s2 = (u32)src_read(&b, tl); src_refill(&b);
    for (; (src_refill(&b) == SRC_MORE) & (op < omax - 3); op += 4) {    /* :201-218 */
        out[op] = dec_step(&s1, &b, cells, fast);
        out[op + 1] = dec_step(&s2, &b, cells, fast);
        out[op + 2] = dec_step(&s1, &b, cells, fast);
        out[op + 3] = dec_step(&s2, &b, cells, fast);
    }
    for (;;) {                                                          /* :222-235 */
        if (op > omax - 2) return ORC_ERROR(ORC_DST_TOO_SMALL);
        out[op++] = dec_step(&s1, &b, cells, fast);
        if (src_refill(&b) == SRC_OVER) { out[op++] = dec_step(&s2, &b, cells, fast); break; }
        if (op > omax - 2) return ORC_ERROR(ORC_DST_TOO_SMALL);
        out[op++] = dec_step(&s2, &b, cells, fast);
        if (src_refill(&b) == SRC_OVER) { out[op++] = dec_step(&s1, &b, cells, fast); break; }
    }
    return (size_t)op;
}

static size_t fse_decode_u16(u16* out, size_t cap, const void* cSrc, size_t cSize, const u32* dt)  /* lib/fseU16.c:261-301 */
{
    unsigned const tl = dt[0] & 0xFFFF;
    const u32* const cells = dt + 1;
    size_t op = 0; bsrc b; u32 st;
    if (orc_is_error(src_open(&b, cSrc, cSize)) && cSize < 1) return ORC_ERROR(ORC_CORRUPT);
    st = (u32)src_read(&b, tl); src_refill(&b);
#define U16_STEP() do { u32 const cell = cells[st]; out[op++] = (u16)(cell >> 20); \
                        st = (cell & 0xFFFF) + (u32)src_read(&b, (cell >> 16) & 0xF); } while (0)
    while (src_refill(&b) < SRC_DONE && op < cap) U16_STEP();
    if (!src_exhausted(&b)) return ORC_ERROR(ORC_CORRUPT);
    while (st && op < cap) U16_STEP();
#undef U16_STEP
    if (st) return ORC_ERROR(ORC_CORRUPT);
    return op;
}

/* a7  FSE_compress_wksp / FSE_compress2 (lib/fse_compress.c:632-693) */
size_t orc_fse_compress2(void* dst, size_t cap, const void* src, size_t n, unsigned msv, unsigned tl)
{
    u8* const out = (u8*)dst;
    unsigned count[FSE_MAX_SV + 1]; short norm[FSE_MAX_SV + 1];
    u32 ct[1 + 2048 + 2 * (FSE_MAX_SV + 1)];
    size_t o = 0, r;
    if (tl > FSE_MAX_TLOG) return ORC_ERROR(ORC_TLOG_TOO_LARGE);
    /* :645 -- FSE_WKSP_SIZE_U32(tl,msv) (lib/fse.h:314) against the 14,340-byte stack workspace of :679-685 */
    if (tl == 0) return ORC_ERROR(ORC_TLOG_TOO_LARGE);   /* the same macro shifts by (0-1): as built (gcc, x86-64) the reference reports tableLog_tooLarge */
    /* the macro is unsigned 32-bit arithmetic: (msv + 1) * 2 wraps, so msv 2^32-1 (and 2^31-1) passes and compresses as 255 */
    {   u32 const ctWords = 1u + (1u << (tl - 1)) + (msv + 1u) * 2u;   /* FSE_CTABLE_SIZE_U32 of the request (:641) */
        if (14340u < ctWords + 1024u) return ORC_ERROR(ORC_TLOG_TOO_LARGE);
        if (n <= 1) return 0;
        /* :642-643 -- the scratch after that CTable is 14340 - 4*ctWords bytes; HIST_count_wksp refuses less than 4096
         * (hist.c:168).  Where the CTable alone exceeds the workspace the size wraps and the reference runs past its
         * stack; those requests are answered as at msv 255. */
        if (4ull * ctWords <= 14340u && 14340u - 4ull * ctWords < 4096u) return ORC_ERROR(ORC_WKSP_TOO_SMALL);
    }
    if (!msv) msv = FSE_MAX_SV;
    if (!tl) tl = FSE_DEF_TLOG;
    r = orc_hist_count(count, &msv, src, n);
    if (orc_is_error(r)) return r;
    if (r == n) return 1;
    if (r == 1) return 0;
    if (r < (n >> 7)) return 0;
    tl = orc_optimal_tablelog(tl, n, msv, 2);
    r = orc_fse_normalize(norm, tl, count, n, msv); if (orc_is_error(r)) return r;
    r = orc_fse_write_ncount(out, cap, norm, msv, tl); if (orc_is_error(r)) return r;
    o = r;
    r = orc_fse_build_ctable(ct, norm, msv, tl); if (orc_is_error(r)) return r;
    r = orc_fse_encode(out + o, cap - o, src, n, ct);
    if (r == 0) return 0;
    o += r;
    if (o >= n - 1) return 0;
    return o;
}

/* a11  FSE_decompress_wksp / FSE_decompress (lib/fse_decompress.c:255-283) */
static size_t fse_decompress_limited(void* dst, size_t cap, const void* cSrc, size_t cSize, u32* dt, unsigned maxLog)
{
    short norm[FSE_MAX_SV + 1];
    unsigned tl, msv = FSE_MAX_SV;
    size_t const h = orc_fse_read_ncount(norm, &msv, &tl, cSrc, cSize);
    size_t r;
    if (orc_is_error(h)) return h;
    if (tl > maxLog) return ORC_ERROR(ORC_TLOG_TOO_LARGE);
    r = orc_fse_build_dtable(dt, norm, msv, tl); if (orc_is_error(r)) return r;
    return orc_fse_decode(dst, cap, (const u8*)cSrc + h, cSize - h, dt);
}
size_t orc_fse_decompress(void* dst, size_t cap, const void* cSrc, size_t cSize)
{
    u32 dt[1 + 4096];
    return fse_decompress_limited(dst, cap, cSrc, cSize, dt, FSE_MAX_TLOG);
}

/* a22  FSE_countU16 / FSE_compressU16 / FSE_decompressU16 (lib/fseU16.c:121-145,203-251,306-329).
 * tableLog selection, normalisation and header use the *byte* build's limits (12). */
size_t orc_fse_compress_u16(void* dst, size_t cap, const u16* src, size_t n, unsigned msv, unsigned tl)
{
    u8* const out = (u8*)dst;
    unsigned count[U16_MAX_SV + 1]; short norm[U16_MAX_SV + 1];
    u32 ct[1 + 4096 + 2 * (U16_MAX_SV + 1)];
    size_t i, o, r; unsigned top, best = 0, s;
    if (n <= 1) return n;
    if (!msv) msv = U16_MAX_SV;
    if (!tl) tl = U16_DEF_TLOG;
    if (msv > U16_MAX_SV) return ORC_ERROR(ORC_MSV_TOO_LARGE);
    if (tl > U16_MAX_TLOG) return ORC_ERROR(ORC_TLOG_TOO_LARGE);
    memset(count, 0, sizeof(count));
    for (i = 0; i < n; i++) { if (src[i] > msv) return ORC_ERROR(ORC_MSV_TOO_SMALL); count[src[i]]++; }
    top = msv; while (!count[top]) top--;
    msv = top;
    for (s = 0; s <= msv; s++) if (count[s] > best) best = count[s];
    if (best == n) return 1;
    tl = orc_optimal_tablelog(tl, n, msv, 2);
    r = orc_fse_normalize(norm, tl, count, n, msv); if (orc_is_error(r)) return r;
    r = orc_fse_write_ncount(out, cap, norm, msv, tl); if (orc_is_error(r)) return r;
    o = r;
    r = orc_fse_build_ctable(ct, norm, msv, tl); if (orc_is_error(r)) return r;
    o += fse_encode_u16(out + o, cap - o, src, n, ct);
    if (o >= (n - 1) * 2) return 0;
    return o;
}

size_t orc_fse_decompress_u16(u16* dst, size_t cap, const void* cSrc, size_t cSize)
{
    short norm[U16_MAX_SV + 1];
    u32 dt[1 + 8192];
    unsigned tl, msv = U16_MAX_SV;
    size_t h, r;
    if (cSize < 2) return ORC_ERROR(ORC_SRC_WRONG);
    h = orc_fse_read_ncount(norm, &msv, &tl, cSrc, cSize); if (orc_is_error(h)) return h;
    r = orc_fse_build_dtable_u16(dt, norm, msv, tl); if (orc_is_error(r)) return r;
    return fse_decode_u16(dst, cap, (const u8*)cSrc + h, cSize - h, dt);
}

/* ==========================================================================================
 * a12  HUF_buildCTable_wksp (lib/huf_compress.c:338-410), HUF_sort (:307-329),
 *      HUF_setMaxHeight (:215-291).  cell image = val | nbBits<<16 (pad byte zeroed here).
 * ========================================================================================== */
typedef struct { u32 count; u16 parent; u8 sym; u8 len; } hnode;

static u32 limit_depth(hnode* nd, u32 last, u32 maxBits)               /* huf_compress.c:215-291 */
{
    u32 const deepest = nd[last].len;
    if (deepest <= maxBits) return deepest;
    {   int debt = 0;
        u32 const unit = 1u << (deepest - maxBits);
        int n = (int)last;
        u32 const NONE = 0xF0F0F0F0u;
        u32 lastOfRank[HUF_MAX_TLOG + 2];
        u32 i;
        while (nd[n].len > maxBits) {
            debt += (int)(unit - (1u << (deepest - nd[n].len)));
            nd[n].len = (u8)maxBits; n--;
        }
        while (nd[n].len == maxBits) n--;
        debt >>= (deepest - maxBits);
        for (i = 0; i < HUF_MAX_TLOG + 2; i++) lastOfRank[i] = NONE;
        {   u32 cur = maxBits; int pos;
            for (pos = n; pos >= 0; pos--) {
                if (nd[pos].len >= cur) continue;
                cur = nd[pos].len;
                lastOfRank[maxBits - cur] = (u32)pos;
            }
        }
        while (debt > 0) {
            u32 dec = hibit((u32)debt) + 1;
            for (; dec > 1; dec--) {
                u32 const hi = lastOfRank[dec], lo = lastOfRank[dec - 1];
                if (hi == NONE) continue;
                if (lo == NONE) break;
                if (nd[hi].count <= 2 * nd[lo].count) break;
            }
            while (dec <= HUF_MAX_TLOG && lastOfRank[dec] == NONE) dec++;
            debt -= 1 << (dec - 1);
            if (lastOfRank[dec - 1] == NONE) lastOfRank[dec - 1] = lastOfRank[dec];
            nd[lastOfRank[dec]].len++;
            if (lastOfRank[dec] == 0) lastOfRank[dec] = NONE;
            else {
                lastOfRank[dec]--;
                if (nd[lastOfRank[dec]].len != maxBits - dec) lastOfRank[dec] = NONE;
            }
        }
        while (debt < 0) {
            if (lastOfRank[1] == NONE) {
                while (nd[n].len == maxBits) n--;
                nd[n + 1].len--;
                lastOfRank[1] = (u32)(n + 1);
                debt++;
                continue;
            }
            nd[lastOfRank[1] + 1].len--;
            lastOfRank[1]++;
            debt++;
        }
    }
    return maxBits;
}

size_t orc_huf_build_ctable(u32* ctable, const unsigned* count, unsigned msv, unsigned maxBits)
{
    hnode store[2 * 256 + 2];
    hnode* const nd = store + 1;                   /* nd[-1] is the sentinel of :368 */
    int last, leaf, inner, fresh, root, n;
    if (!maxBits) maxBits = HUF_DEF_TLOG;
    if (msv > HUF_MAX_SV) return ORC_ERROR(ORC_MSV_TOO_LARGE);
    memset(store, 0, sizeof(store));
    /* stable sort by decreasing count == bucket+insertion sort of :307-329 */
    for (n = 0; n <= (int)msv; n++) {
        int pos = n;
        while (pos > 0 && count[n] > nd[pos - 1].count) { nd[pos] = nd[pos - 1]; pos--; }
        nd[pos].count = count[n]; nd[pos].sym = (u8)n;
    }
    last = (int)msv; while (nd[last].count == 0) last--;
    fresh = 256; leaf = last; root = fresh + leaf - 1; inner = fresh;
    nd[fresh].count = nd[leaf].count + nd[leaf - 1].count;
    nd[leaf].parent = nd[leaf - 1].parent = (u16)fresh;
    fresh++; leaf -= 2;
    for (n = fresh; n <= root; n++) nd[n].count = 1u << 30;
    nd[-1].count = 1u << 31;
    while (fresh <= root) {                        /* two-queue merge; ties prefer the internal node (:372-373) */
        int const a = (nd[leaf].count < nd[inner].count) ? leaf-- : inner++;
        int const b = (nd[leaf].count < nd[inner].count) ? leaf-- : inner++;
        nd[fresh].count = nd[a].count + nd[b].count;
        nd[a].parent = nd[b].parent = (u16)fresh;
        fresh++;
    }
    nd[root].len = 0;
    for (n = root - 1; n >= 256; n--) nd[n].len = (u8)(nd[nd[n].parent].len + 1);
    for (n = 0; n <= last; n++) nd[n].len = (u8)(nd[nd[n].parent].len + 1);
    maxBits = limit_depth(nd, (u32)last, maxBits);
    {   u16 perLen[HUF_MAX_TLOG + 1], firstVal[HUF_MAX_TLOG + 1];
        u8 lenOf[256];
        u16 v = 0;
        memset(perLen, 0, sizeof(perLen)); memset(firstVal, 0, sizeof(firstVal));
        if (maxBits > HUF_MAX_TLOG) return ORC_ERROR(ORC_GENERIC);
        for (n = 0; n <= last; n++) perLen[nd[n].len]++;
        for (n = (int)maxBits; n > 0; n--) { firstVal[n] = v; v = (u16)((v + perLen[n]) >> 1); }   /* :396-401 */
        for (n = 0; n <= (int)msv; n++) lenOf[nd[n].sym] = nd[n].len;
        for (n = 0; n <= (int)msv; n++) ctable[n] = (u32)firstVal[lenOf[n]]++ | ((u32)lenOf[n] << 16);
    }
    return maxBits;
}

/* a13  HUF_compressWeights + HUF_writeCTable (lib/huf_compress.c:63-147) */
static size_t compress_weights(void* dst, size_t cap, const u8* w, size_t n)
{
    u8* const out = (u8*)dst;
    unsigned count[HUF_MAX_TLOG + 1]; short norm[HUF_MAX_TLOG + 1];
    u32 ct[1 + 32 + 2 * (HUF_MAX_TLOG + 1)];
    unsigned msv = HUF_MAX_TLOG, tl = 6, best = 0, s;
    size_t i, o, r;
    if (n <= 1) return 0;
    memset(count, 0, sizeof(count));               /* HIST_count_simple, hist.c:29-54 */
    for (i = 0; i < n; i++) count[w[i]]++;
    while (!count[msv]) msv--;
    for (s = 0; s <= msv; s++) if (count[s] > best) best = count[s];
    if (best == n) return 1;
    if (best == 1) return 0;
    tl = orc_optimal_tablelog(tl, n, msv, 2);
    r = orc_fse_normalize(norm, tl, count, n, msv); if (orc_is_error(r)) return r;
    r = orc_fse_write_ncount(out, cap, norm, msv, tl); if (orc_is_error(r)) return r;
    o = r;
    r = orc_fse_build_ctable(ct, norm, msv, tl); if (orc_is_error(r)) return r;
    r = orc_fse_encode(out + o, cap - o, w, n, ct);
    if (r == 0) return 0;
    return o + r;
}

size_t orc_huf_write_ctable(void* dst, size_t cap, const u32* ctable, unsigned msv, unsigned huffLog)
{
    u8* const out = (u8*)dst;
    u8 weight[HUF_MAX_SV + 1];
    unsigned n;
    if (msv > HUF_MAX_SV) return ORC_ERROR(ORC_MSV_TOO_LARGE);
    for (n = 0; n < msv; n++) {
        unsigned const len = (ctable[n] >> 16) & 0xFF;
        weight[n] = (u8)(len ? huffLog + 1 - len : 0);
    }
    {   size_t const h = compress_weights(out + 1, cap - 1, weight, msv);
        if (orc_is_error(h)) return h;
        if ((h > 1) & (h < msv / 2)) { out[0] = (u8)h; return h + 1; }
    }
    if (msv > 128) return ORC_ERROR(ORC_GENERIC);
    if (((msv + 1) / 2) + 1 > cap) return ORC_ERROR(ORC_DST_TOO_SMALL);
    out[0] = (u8)(128 + (msv - 1));
    weight[msv] = 0;
    for (n = 0; n < msv; n += 2) out[(n / 2) + 1] = (u8)((weight[n] << 4) + weight[n + 1]);
    return ((msv + 1) / 2) + 1;
}

/* a14  HUF_compress1X/4X_usingCTable (lib/huf_compress.c:457-502,552-603) */
size_t orc_huf_encode1x(void* dst, size_t cap, const void* src, size_t n, const u32* ctable)
{
    const u8* const in = (const u8*)src;
    bsink s; size_t i;
    if (cap < 8) return 0;
    sink_open(&s, dst, cap);
    if (!s.usable) return 0;
    for (i = n; i-- > 0;) sink_put(&s, ctable[in[i]] & 0xFFFF, (ctable[in[i]] >> 16) & 0xFF);
    return sink_close(&s);
}

size_t orc_huf_encode4x(void* dst, size_t cap, const void* src, size_t n, const u32* ctable)
{
    const u8* in = (const u8*)src;
    u8* const out = (u8*)dst;
    size_t const seg = (n + 3) / 4;
    size_t o = 6; int k;
    if (cap < 6 + 1 + 1 + 1 + 8) return 0;
    if (n < 12) return 0;
    for (k = 0; k < 4; k++) {
        size_t const len = (k < 3) ? seg : n - 3 * seg;
        size_t const c = orc_huf_encode1x(out + o, cap - o, in + (size_t)k * seg, len, ctable);
        if (c == 0) return 0;
        if (k < 3) wr16(out + 2 * k, (u32)c);
        o += c;
    }
    return o;
}

/* a15  HUF_compress_internal / HUF_compress2 (lib/huf_compress.c:637-724,787-793), no table reuse */
size_t orc_huf_compress2(void* dst, size_t cap, const void* src, size_t n, unsigned msv, unsigned huffLog)
{
    u8* const out = (u8*)dst;
    unsigned count[HUF_MAX_SV + 1];
    u32 ctable[HUF_MAX_SV + 1];
    size_t r, o;
    if (!n) return 0;
    if (!cap) return 0;
    if (n > HUF_BLOCK_MAX) return ORC_ERROR(ORC_SRC_WRONG);
    if (huffLog > HUF_MAX_TLOG) return ORC_ERROR(ORC_TLOG_TOO_LARGE);
    if (msv > HUF_MAX_SV) return ORC_ERROR(ORC_MSV_TOO_LARGE);
    if (!msv) msv = HUF_MAX_SV;
    if (!huffLog) huffLog = HUF_DEF_TLOG;
    r = orc_hist_count(count, &msv, src, n); if (orc_is_error(r)) return r;
    if (r == n) { out[0] = ((const u8*)src)[0]; return 1; }
    if (r <= (n >> 7) + 4) return 0;
    huffLog = orc_optimal_tablelog(huffLog, n, msv, 1);
    r = orc_huf_build_ctable(ctable, count, msv, huffLog); if (orc_is_error(r)) return r;
    huffLog = (unsigned)r;
    r = orc_huf_write_ctable(out, cap, ctable, msv, huffLog); if (orc_is_error(r)) return r;
    if (r + 12 >= n) return 0;
    o = r;
    r = orc_huf_encode4x(out + o, cap - o, src, n, ctable);
    if (r == 0) return 0;
    o += r;
    if (o >= n - 1) return 0;
    return o;
}

/* a16  HUF_readStats (lib/entropy_common.c:154-215) */
size_t orc_huf_read_stats(u8* weights, size_t hwSize, u32* rankStats, u32* nbSymbolsPtr, u32* tlPtr,
                          const void* src, size_t srcSize)
{
    const u8* const in = (const u8*)src;
    size_t iSize, oSize, n;
    u32 total = 0;
    if (!srcSize) return ORC_ERROR(ORC_SRC_WRONG);
    iSize = in[0];
    if (iSize >= 128) {                            /* raw nibbles */
        oSize = iSize - 127;
        iSize = (oSize + 1) / 2;
        if (iSize + 1 > srcSize) return ORC_ERROR(ORC_SRC_WRONG);
        if (oSize >= hwSize) return ORC_ERROR(ORC_CORRUPT);
        for (n = 0; n < oSize; n += 2) {
            weights[n] = in[1 + n / 2] >> 4;
            weights[n + 1] = in[1 + n / 2] & 15;
        }
    } else {                                       /* FSE-compressed weights, tableLog <= 6 */
        u32 dt[1 + 64];
        if (iSize + 1 > srcSize) return ORC_ERROR(ORC_SRC_WRONG);
        oSize = fse_decompress_limited(weights, hwSize - 1, in + 1, iSize, dt, 6);
        if (orc_is_error(oSize)) return oSize;
    }
    memset(rankStats, 0, (HUF_MAX_TLOG + 1) * sizeof(u32));
    for (n = 0; n < oSize; n++) {
        if (weights[n] >= HUF_MAX_TLOG) return ORC_ERROR(ORC_CORRUPT);
        rankStats[weights[n]]++;
        total += (1u << weights[n]) >> 1;
    }
    if (total == 0) return ORC_ERROR(ORC_CORRUPT);
    {   u32 const tl = hibit(total) + 1;
        u32 const rest = (1u << tl) - total;
        u32 const lastW = hibit(rest) + 1;
        if (tl > HUF_MAX_TLOG) return ORC_ERROR(ORC_CORRUPT);
        *tlPtr = tl;
        if ((1u << hibit(rest)) != rest) return ORC_ERROR(ORC_CORRUPT);
        weights[oSize] = (u8)lastW;
        rankStats[lastW]++;
    }
    if ((rankStats[1] < 2) || (rankStats[1] & 1)) return ORC_ERROR(ORC_CORRUPT);
    *nbSymbolsPtr = (u32)(oSize + 1);
    return iSize + 1;
}

/* a17  HUF_readDTableX1_wksp (lib/huf_decompress.c:118-185).  dtable[0] must carry maxTableLog
 * in its low byte on entry (HUF_CREATE_STATIC_DTABLEX1, lib/huf.h:146-147). */
size_t orc_huf_read_dtable_x1(u32* dtable, const void* src, size_t srcSize)
{
    u8 weights[HUF_MAX_SV + 1];
    u32 rank[16 + 1];
    u32 tl = 0, nbSym = 0, n, next = 0;
    u16* const cells = (u16*)(void*)(dtable + 1);
    size_t const h = orc_huf_read_stats(weights, HUF_MAX_SV + 1, rank, &nbSym, &tl, src, srcSize);
    if (orc_is_error(h)) return h;
    if (tl > (dtable[0] & 0xFF) + 1) return ORC_ERROR(ORC_TLOG_TOO_LARGE);
    dtable[0] = (dtable[0] & 0xFF0000FFu) | (tl << 16);               /* tableType 0, tableLog */
    for (n = 1; n < tl + 1; n++) { u32 const cur = next; next += rank[n] << (n - 1); rank[n] = cur; }
    for (n = 0; n < nbSym; n++) {
        u32 const w = weights[n];
        u32 const span = (1u << w) >> 1;
        u32 const cell = n | ((tl + 1 - w) << 8);                      /* {byte, nbBits} */
        u32 u;
        for (u = 0; u < span; u++) cells[rank[w] + u] = (u16)cell;
        rank[w] += span;
    }
    return h;
}

/* a18  HUF_readDTableX2 (lib/huf_decompress.c:551-649 ; fill :468-549): the double-symbol table, always built at the
 * descriptor's maxTableLog L.  Cell = { U16 sequence; BYTE nbBits; BYTE length } (:460).
 * Formulation: symbols of weight >= 1 are listed by (weight, symbol).  In an index space of width L a symbol of code
 * length n owns 2^(L-n) consecutive cells, weights ascending, so weight w starts at first[w] = sum_{v<w} count[v] << (v+L-tl-1).
 * If the cells of a first symbol (L-n index bits left) can hold the shortest code, they are a scaled copy of the same
 * layout for the second symbol: weight w starts at first[w] >> n; second symbols too long to fit (weight < n + tl+1-L, at
 * least 1) leave the leading cells as single-symbol entries.  */
size_t orc_huf_read_dtable_x2(u32* dtable, const void* src, size_t srcSize)
{
    u8 weights[HUF_MAX_SV + 1];
    u32 rank[16 + 1];
    u8 listSym[HUF_MAX_SV + 1], listW[HUF_MAX_SV + 1];
    u32 listStart[HUF_MAX_TLOG + 2], fill[HUF_MAX_TLOG + 2], first[HUF_MAX_TLOG + 2];
    u32 tl = 0, nbSym = 0, maxW, w, s, listSize = 0;
    u32 const L = dtable[0] & 0xFF;
    u32* const cells = dtable + 1;
    size_t h;
    if (L > HUF_MAX_TLOG) return ORC_ERROR(ORC_TLOG_TOO_LARGE);          /* :586 */
    h = orc_huf_read_stats(weights, HUF_MAX_SV + 1, rank, &nbSym, &tl, src, srcSize);
    if (orc_is_error(h)) return h;
    if (tl > L) return ORC_ERROR(ORC_TLOG_TOO_LARGE);                     /* :593 */
    for (maxW = tl; rank[maxW] == 0; maxW--) {}
    /* symbols of weight >= 1 ordered by (weight, symbol) */
    for (w = 1; w <= maxW; w++) { listStart[w] = listSize; listSize += rank[w]; }
    listStart[maxW + 1] = listSize;
    for (w = 1; w <= maxW; w++) fill[w] = listStart[w];
    for (s = 0; s < nbSym; s++) { u32 const ws = weights[s]; if (ws) { listSym[fill[ws]] = (u8)s; listW[fill[ws]] = (u8)ws; fill[ws]++; } }
    {   u32 acc = 0;
        for (w = 1; w <= maxW; w++) { first[w] = acc; acc += rank[w] << (w + (L - tl) - 1); }
    }
    {   u32 const minBits = tl + 1 - maxW;                                /* shortest code */
        u32 next1[HUF_MAX_TLOG + 2];
        u32 i;
        for (w = 1; w <= maxW; w++) next1[w] = first[w];
        for (i = 0; i < listSize; i++) {
            u32 const sym = listSym[i], w1 = listW[i], n = tl + 1 - w1;
            u32 const start = next1[w1], span = 1u << (L - n);
            u32* const sub = cells + start;
            next1[w1] += span;
            if (L - n >= minBits) {                                       /* room for a second symbol */
                int minWeight = (int)n + ((int)tl + 1 - (int)L);
                u32 next2[HUF_MAX_TLOG + 2];
                u32 j, u;
                if (minWeight < 1) minWeight = 1;
                for (w = 1; w <= maxW; w++) next2[w] = first[w] >> n;
                if (minWeight > 1) {                                      /* too-long second symbols: single-symbol cells */
                    u32 const skip = next2[minWeight];
                    for (u = 0; u < skip; u++) sub[u] = sym | (n << 16) | (1u << 24);
                }
                for (j = listStart[minWeight]; j < listSize; j++) {
                    u32 const s2 = listSym[j], w2 = listW[j], n2 = tl + 1 - w2;
                    u32 const len2 = 1u << (L - n - n2);
                    u32 const at = next2[w2];
                    for (u = 0; u < len2; u++) sub[at + u] = ((sym + (s2 << 8)) & 0xFFFF) | ((n + n2) << 16) | (2u << 24);
                    next2[w2] += len2;
                }
            } else {
                u32 u;
                for (u = 0; u < span; u++) sub[u] = sym | (n << 16) | (1u << 24);
            }
        }
    }
    dtable[0] = (dtable[0] & 0xFF0000FFu) | (1u << 8) | (L << 16);         /* tableType 1, tableLog = maxTableLog (:645-647) */
    return h;
}

/* a19  HUF_decompress1X1/4X1_usingDTable_internal_body (lib/huf_decompress.c:194-354) */
static u8 huf_step(bsrc* b, const u16* cells, unsigned dtLog)          /* :194-201 */
{
    u32 const cell = cells[src_peek_fast(b, dtLog)];
    b->used += cell >> 8;
    return (u8)cell;
}
static void huf_finish_stream(u8* out, ptrdiff_t p, ptrdiff_t pEnd, bsrc* b, const u16* cells, unsigned dtLog)  /* :214-237 */
{
    while ((src_refill(b) == SRC_MORE) & (p < pEnd - 3)) {
        out[p++] = huf_step(b, cells, dtLog); out[p++] = huf_step(b, cells, dtLog);
        out[p++] = huf_step(b, cells, dtLog); out[p++] = huf_step(b, cells, dtLog);
    }
    while (p < pEnd) out[p++] = huf_step(b, cells, dtLog);
}

size_t orc_huf_decode1x1(void* dst, size_t dstSize, const void* cSrc, size_t cSize, const u32* dtable)
{
    bsrc b;
    size_t const e = src_open(&b, cSrc, cSize);
    if (orc_is_error(e)) return e;
    huf_finish_stream((u8*)dst, 0, (ptrdiff_t)dstSize, &b, (const u16*)(const void*)(dtable + 1), (dtable[0] >> 16) & 0xFF);
    if (!src_exhausted(&b)) return ORC_ERROR(ORC_CORRUPT);
    return dstSize;
}

size_t orc_huf_decode4x1(void* dst, size_t dstSize, const void* cSrc, size_t cSize, const u32* dtable)
{
    const u8* const in = (const u8*)cSrc;
    u8* const out = (u8*)dst;
    const u16* const cells = (const u16*)(const void*)(dtable + 1);
    unsigned const dtLog = (dtable[0] >> 16) & 0xFF;
    if (cSize < 10) return ORC_ERROR(ORC_CORRUPT);
    {   size_t const l1 = rd16(in), l2 = rd16(in + 2), l3 = rd16(in + 4);
        size_t const l4 = cSize - (l1 + l2 + l3 + 6);
        ptrdiff_t const seg = (ptrdiff_t)((dstSize + 3) / 4);
        ptrdiff_t const end = (ptrdiff_t)dstSize;
        ptrdiff_t p[4]; ptrdiff_t stop[4];
        bsrc b[4]; int k; int alive = 1;
        size_t e;
        if (l4 > cSize) return ORC_ERROR(ORC_CORRUPT);
        if (3 * seg > end) return ORC_ERROR(ORC_CORRUPT);             /* documented deviation: see file header */
        e = src_open(&b[0], in + 6, l1); if (orc_is_error(e)) return e;
        e = src_open(&b[1], in + 6 + l1, l2); if (orc_is_error(e)) return e;
        e = src_open(&b[2], in + 6 + l1 + l2, l3); if (orc_is_error(e)) return e;
        e = src_open(&b[3], in + 6 + l1 + l2 + l3, l4); if (orc_is_error(e)) return e;
        for (k = 0; k < 4; k++) { p[k] = k * seg; stop[k] = (k < 3) ? (k + 1) * seg : end; }
        while (alive & (p[3] < end - 3)) {                            /* :310-331 */
            int r;
            for (r = 0; r < 4; r++) for (k = 0; k < 4; k++) out[p[k]++] = huf_step(&b[k], cells, dtLog);
            for (k = 0; k < 4; k++) alive &= (src_refill_fast(&b[k]) == SRC_MORE);
        }
        if (p[0] > stop[0] || p[1] > stop[1] || p[2] > stop[2]) return ORC_ERROR(ORC_CORRUPT);
        for (k = 0; k < 4; k++) huf_finish_stream(out, p[k], stop[k], &b[k], cells, dtLog);
        for (k = 0; k < 4; k++) if (!src_exhausted(&b[k])) return ORC_ERROR(ORC_CORRUPT);
    }
    return dstSize;
}

/* a19 (double-symbol)  HUF_decompress1X2/4X2_usingDTable_internal_body (lib/huf_decompress.c:659-862).  A cell yields one
 * or two symbols per look-up; the last symbol of a stream is taken alone (:668-683). */
static void huf_finish_stream_x2(u8* out, ptrdiff_t p, ptrdiff_t pEnd, bsrc* b, const u32* cells, unsigned dtLog)   /* :693-720 */
{
#define ORC_X2() do { u32 const c_ = cells[src_peek_fast(b, dtLog)]; out[p] = (u8)c_; out[p + 1] = (u8)(c_ >> 8); \
                      b->used += (c_ >> 16) & 0xFF; p += c_ >> 24; } while (0)
    while ((src_refill(b) == SRC_MORE) & (p < pEnd - 7)) { ORC_X2(); ORC_X2(); ORC_X2(); ORC_X2(); }
    while ((src_refill(b) == SRC_MORE) & (p <= pEnd - 2)) ORC_X2();
    while (p <= pEnd - 2) ORC_X2();
#undef ORC_X2
    if (p < pEnd) {
        u32 const c = cells[src_peek_fast(b, dtLog)];
        unsigned const nb = (c >> 16) & 0xFF;
        out[p] = (u8)c;
        if ((c >> 24) == 1) b->used += nb;
        else if (b->used < 64) { b->used += nb; if (b->used > 64) b->used = 64; }
    }
}
size_t orc_huf_decode1x2(void* dst, size_t dstSize, const void* cSrc, size_t cSize, const u32* dtable)
{
    bsrc b;
    size_t const e = src_open(&b, cSrc, cSize);
    if (orc_is_error(e)) return e;
    huf_finish_stream_x2((u8*)dst, 0, (ptrdiff_t)dstSize, &b, dtable + 1, (dtable[0] >> 16) & 0xFF);
    if (!src_exhausted(&b)) return ORC_ERROR(ORC_CORRUPT);
    return dstSize;
}
/* Streams are independent: decoding them one after the other yields what the reference's interleaved loop (:797-845) yields
 * whenever it returns success, and a stream that is not consumed exactly is reported either way (:853-855). */
size_t orc_huf_decode4x2(void* dst, size_t dstSize, const void* cSrc, size_t cSize, const u32* dtable)
{
    const u8* const in = (const u8*)cSrc;
    u8* const out = (u8*)dst;
    unsigned const dtLog = (dtable[0] >> 16) & 0xFF;
    if (cSize < 10) return ORC_ERROR(ORC_CORRUPT);
    {   size_t const l1 = rd16(in), l2 = rd16(in + 2), l3 = rd16(in + 4);
        size_t const l4 = cSize - (l1 + l2 + l3 + 6);
        ptrdiff_t const seg = (ptrdiff_t)((dstSize + 3) / 4), end = (ptrdiff_t)dstSize;
        size_t const off[4] = { 6, 6 + l1, 6 + l1 + l2, 6 + l1 + l2 + l3 };
        size_t const len[4] = { l1, l2, l3, l4 };
        bsrc b[4]; int k;
        if (l4 > cSize) return ORC_ERROR(ORC_CORRUPT);
        if (3 * seg > end) return ORC_ERROR(ORC_CORRUPT);             /* same guard as the single-symbol restatement */
        for (k = 0; k < 4; k++) { size_t const e = src_open(&b[k], in + off[k], len[k]); if (orc_is_error(e)) return e; }
        for (k = 0; k < 4; k++) huf_finish_stream_x2(out, k * seg, (k < 3) ? (k + 1) * seg : end, &b[k], dtable + 1, dtLog);
        for (k = 0; k < 4; k++) if (!src_exhausted(&b[k])) return ORC_ERROR(ORC_CORRUPT);
    }
    return dstSize;
}

/* a20  HUF_selectDecoder / HUF_decompress (lib/huf_decompress.c:1001-1081) */
unsigned orc_huf_select_decoder(size_t dstSize, size_t cSize)
{
    static const u16 cost[16][4] = {               /* {X1 table, X1 per-256, X2 table, X2 per-256} */
        {0, 0, 1, 1}, {0, 0, 1, 1}, {38, 130, 1313, 74}, {448, 128, 1353, 74}, {556, 128, 1353, 74},
        {714, 128, 1418, 74}, {883, 128, 1437, 74}, {897, 128, 1515, 75}, {926, 128, 1613, 75},
        {947, 128, 1729, 77}, {1107, 128, 2083, 81}, {1177, 128, 2379, 87}, {1242, 128, 2415, 93},
        {1349, 128, 2644, 106}, {1455, 128, 2422, 124}, {722, 128, 1891, 145} };
    u32 const q = (cSize >= dstSize) ? 15 : (u32)(cSize * 16 / dstSize);
    u32 const d256 = (u32)(dstSize >> 8);
    u32 const t0 = cost[q][0] + cost[q][1] * d256;
    u32 t1 = cost[q][2] + cost[q][3] * d256;
    t1 += t1 >> 3;
    return t1 < t0;
}

/* HUF_decompress4X1 / HUF_decompress4X2 (lib/huf_decompress.c:416-449,917-952): header + payload with a fixed decoder */
size_t orc_huf_decompress4x1(void* dst, size_t dstSize, const void* cSrc, size_t cSize)
{
    u32 dtable[1 + 4096];
    size_t h;
    dtable[0] = (HUF_MAX_TLOG - 1) * 0x01000001u;
    h = orc_huf_read_dtable_x1(dtable, cSrc, cSize);
    if (orc_is_error(h)) return h;
    if (h >= cSize) return ORC_ERROR(ORC_SRC_WRONG);
    return orc_huf_decode4x1(dst, dstSize, (const u8*)cSrc + h, cSize - h, dtable);
}

size_t orc_huf_decompress4x2(void* dst, size_t dstSize, const void* cSrc, size_t cSize)
{
    u32 dtable[1 + 4096];
    size_t h;
    dtable[0] = HUF_MAX_TLOG * 0x01000001u;
    h = orc_huf_read_dtable_x2(dtable, cSrc, cSize);
    if (orc_is_error(h)) return h;
    if (h >= cSize) return ORC_ERROR(ORC_SRC_WRONG);
    return orc_huf_decode4x2(dst, dstSize, (const u8*)cSrc + h, cSize - h, dtable);
}

/* HUF_decompress (lib/huf_decompress.c:1056-1081): raw / RLE, then the decoder HUF_selectDecoder picks.  Both decoders
 * regenerate the same bytes for a valid stream; on malformed streams the double-symbol decoder accepts some the
 * single-symbol one rejects (HUF_decodeLastSymbolX2 clamps the bit count), so the choice is part of the verdict. */
size_t orc_huf_decompress(void* dst, size_t dstSize, const void* cSrc, size_t cSize)
{
    if (dstSize == 0) return ORC_ERROR(ORC_DST_TOO_SMALL);
    if (cSize > dstSize) return ORC_ERROR(ORC_CORRUPT);
    if (cSize == dstSize) { memcpy(dst, cSrc, dstSize); return dstSize; }
    if (cSize == 1) { memset(dst, *(const u8*)cSrc, dstSize); return dstSize; }
    return orc_huf_select_decoder(dstSize, cSize) ? orc_huf_decompress4x2(dst, dstSize, cSrc, cSize)
                                                  : orc_huf_decompress4x1(dst, dstSize, cSrc, cSize);
}

/* ==========================================================================================
 * measurement inputs: size-parametric restatements of the reference generators
 * ========================================================================================== */
static u32 lcg_next(u32* seed) { *seed = (*seed * 2654435761u) + 2246822519u; return *seed >> 11; }

void orc_probagen(void* buf, size_t size, double p)                   /* programs/probaGenerator.c:95-126 */
{
    u8 table[4096];
    int remaining = 4096; unsigned pos = 0, sym = 0;
    u8* out = (u8*)buf; size_t i; u32 seed = 1;
    if (p == 0.0) p = 0.005;
    while (remaining) {
        unsigned n = (unsigned)(remaining * p);
        unsigned end;
        if (!n) n = 1;
        end = pos + n;
        while (pos < end) table[pos++] = (u8)sym;
        sym++; remaining -= (int)n;
    }
    for (i = 0; i < size; i++) out[i] = table[lcg_next(&seed) & 4095];
}

void orc_gen_u16(u16* buf, size_t nb, unsigned start, double p, u32 seed)   /* programs/fuzzerU16.c:107-134 */
{
    u16 table[4096];
    u32 remaining = 4096, pos = 0; u16 v = (u16)start; size_t i;
    while (remaining) {
        u32 const n = (u32)(remaining * p) + 1;
        u32 const end = pos + n;
        while (pos < end) table[pos++] = v;
        v++; if (v >= U16_MAX_SV) v = 1;
        remaining -= n;
    }
    for (i = 0; i < nb; i++) buf[i] = table[lcg_next(&seed) & 4095];
}

/* XXH32 / XXH64 (public xxHash specification; the reference harness uses them for its self-checks,
 * programs/bench.c:311,444 and SURVEY.md section 6.3) */
static u32 rol32(u32 x, int r) { return (x << r) | (x >> (32 - r)); }
static u64 rol64(u64 x, int r) { return (x << r) | (x >> (64 - r)); }
#define P32_1 2654435761u
#define P32_2 2246822519u
#define P32_3 3266489917u
#define P32_4 668265263u
#define P32_5 374761393u
uint32_t orc_xxh32(const void* data, size_t len, uint32_t seed)
{
    const u8* p = (const u8*)data; const u8* const end = p + len; u32 h;
    if (len >= 16) {
        u32 v1 = seed + P32_1 + P32_2, v2 = seed + P32_2, v3 = seed, v4 = seed - P32_1;
        do {
            v1 = rol32(v1 + rd32(p) * P32_2, 13) * P32_1; p += 4;
            v2 = rol32(v2 + rd32(p) * P32_2, 13) * P32_1; p += 4;
            v3 = rol32(v3 + rd32(p) * P32_2, 13) * P32_1; p += 4;
            v4 = rol32(v4 + rd32(p) * P32_2, 13) * P32_1; p += 4;
        } while (p + 16 <= end);
        h = rol32(v1, 1) + rol32(v2, 7) + rol32(v3, 12) + rol32(v4, 18);
    } else h = seed + P32_5;
    h += (u32)len;
    while (p + 4 <= end) { h = rol32(h + rd32(p) * P32_3, 17) * P32_4; p += 4; }
    while (p < end) { h = rol32(h + (*p) * P32_5, 11) * P32_1; p++; }
    h ^= h >> 15; h *= P32_2; h ^= h >> 13; h *= P32_3; h ^= h >> 16;
    return h;
}
#define P64_1 11400714785074694791ULL
#define P64_2 14029467366897019727ULL
#define P64_3 1609587929392839161ULL
#define P64_4 9650029242287828579ULL
#define P64_5 2870177450012600261ULL
static u64 x64_round(u64 acc, u64 in) { return rol64(acc + in * P64_2, 31) * P64_1; }
static u64 x64_merge(u64 h, u64 v) { return (h ^ x64_round(0, v)) * P64_1 + P64_4; }
uint64_t orc_xxh64(const void* data, size_t len, uint64_t seed)
{
    const u8* p = (const u8*)data; const u8* const end = p + len; u64 h;
    if (len >= 32) {
        u64 v1 = seed + P64_1 + P64_2, v2 = seed + P64_2, v3 = seed, v4 = seed - P64_1;
        do {
            v1 = x64_round(v1, rd64(p)); p += 8; v2 = x64_round(v2, rd64(p)); p += 8;
            v3 = x64_round(v3, rd64(p)); p += 8; v4 = x64_round(v4, rd64(p)); p += 8;
        } while (p + 32 <= end);
        h = rol64(v1, 1) + rol64(v2, 7) + rol64(v3, 12) + rol64(v4, 18);
        h = x64_merge(h, v1); h = x64_merge(h, v2); h = x64_merge(h, v3); h = x64_merge(h, v4);
    } else h = seed + P64_5;
    h += (u64)len;
    while (p + 8 <= end) { h = rol64(h ^ x64_round(0, rd64(p)), 27) * P64_1 + P64_4; p += 8; }
    if (p + 4 <= end) { h = rol64(h ^ ((u64)rd32(p) * P64_1), 23) * P64_2 + P64_3; p += 4; }
    while (p < end) { h = rol64(h ^ ((*p) * P64_5), 11) * P64_1; p++; }
    h ^= h >> 33; h *= P64_2; h ^= h >> 29; h *= P64_3; h ^= h >> 32;
    return h;
}

/* ==========================================================================================
 * block loops of the reference harness (programs/bench.c:353-364 and :389-424)
 * ========================================================================================== */
size_t orc_compress_blocks(int codec, const void* src, size_t total, size_t blockSize, void* cbuf, size_t slot,
                           size_t* csizes, unsigned msv, unsigned tl)
{
    size_t const nb = (total + blockSize - 1) / blockSize;
    size_t b;
    for (b = 0; b < nb; b++) {
        size_t const off = b * blockSize;
        size_t const n = off + blockSize <= total ? blockSize : total - off;
        u8* const c = (u8*)cbuf + b * slot;
        const u8* const s = (const u8*)src + off;
        csizes[b] = codec == 0 ? orc_fse_compress2(c, slot, s, n, msv, tl)
                  : codec == 1 ? orc_huf_compress2(c, slot, s, n, msv, tl)
                  : orc_fse_compress_u16(c, slot, (const u16*)(const void*)s, n / 2, msv, tl);
    }
    return nb;
}

size_t orc_decompress_blocks(int codec, void* out, const void* orig, size_t total, size_t blockSize,
                             const void* cbuf, size_t slot, const size_t* csizes, size_t* results)
{
    size_t const nb = (total + blockSize - 1) / blockSize;
    size_t b;
    for (b = 0; b < nb; b++) {
        size_t const off = b * blockSize;
        size_t const n = off + blockSize <= total ? blockSize : total - off;
        const u8* const c = (const u8*)cbuf + b * slot;
        u8* const o = (u8*)out + off;
        size_t r;
        if (csizes[b] == 0) { memcpy(o, (const u8*)orig + off, n); r = n; }
        else if (csizes[b] == 1 && codec != 2) { memset(o, ((const u8*)orig)[off], n); r = n; }
        else if (codec == 0) r = orc_fse_decompress(o, n, c, csizes[b]);
        else if (codec == 1) r = orc_huf_decompress(o, n, c, csizes[b]);
        else { r = orc_fse_decompress_u16((u16*)(void*)o, n / 2, c, csizes[b]); if (!orc_is_error(r)) r *= 2; }
        if (results) results[b] = r;
    }
    return nb;
}
