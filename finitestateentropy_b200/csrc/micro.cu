// micro.cu -- single-CTA kernels behind the reference's table-level entry points (lib/fse.h:135-247,
// lib/hist.h:30-75, lib/huf.h:188-272 static section).  They run the very same device routines the
// batched kernels use, on one table, so that HIST_count / FSE_normalizeCount / FSE_buildCTable /
// FSE_buildDTable / HUF_buildCTable / HUF_readDTableX1 ... are honest drop-ins executing on the GPU.
#include "common.cuh"
#include "launchers.h"
#include "fse_dev.cuh"
#include "bitsrc_dev.cuh"
#include "sink_dev.cuh"
#include "huf_dev.cuh"
#include "huf_build_dev.cuh"
#include "huf_x2_dev.cuh"
#include "micro.h"

namespace fseb {

// ---- HIST_count (lib/hist.c:163-180): any size, one CTA ----
__global__ void __launch_bounds__(256) hist_kernel(const u8* src, u64 n, u32 declared, u32* out /*256 counts, then msv, then pad*/, u64* ret)
{
    __shared__ u32 h[8][256];
    __shared__ u32 tot[256];
    int const tid = threadIdx.x;
    for (int i = tid; i < 8 * 256; i += 256) (&h[0][0])[i] = 0;
    __syncthreads();
    u32* const mine = h[tid >> 5];
    for (u64 i = tid; i < n; i += 256) atomicAdd(&mine[src[i]], 1u);
    __syncthreads();
    {   u32 c = 0; for (int w = 0; w < 8; w++) c += h[w][tid]; tot[tid] = c; }
    __syncthreads();
    if (tid == 0) {
        if (declared > 255) declared = 255;
        if (n == 0) { for (u32 i = 0; i <= declared; i++) out[i] = 0; out[256] = 0; *ret = 0; return; }
        u32 top = 255; while (!tot[top]) top--;
        if (declared < 255 && top > declared) { *ret = err(E_MSV_TOO_SMALL); return; }
        u32 best = 0;
        for (u32 i = 0; i < 256; i++) best = tot[i] > best ? tot[i] : best;
        for (u32 i = 0; i <= declared; i++) out[i] = tot[i];
        out[256] = top; *ret = best;
    }
}

// ---- FSE_countU16 (lib/fseU16.c:121-145): histogram of 16-bit symbols, one CTA, counters in global scratch ----
// out: count u32[declared+1], then out[declared+1] = largest present symbol.  ret: largest count, 0 for an empty input, or
// maxSymbolValue_tooSmall if a symbol exceeds `declared` (the reference stops at the first such symbol; the counts it leaves
// behind are unspecified, ours are zeros).
__global__ void __launch_bounds__(256) hist16_kernel(const u16* src, u64 n, u32 declared, u32* out, u64* ret)
{
    __shared__ u32 s_bad, s_top, s_best;
    int const tid = threadIdx.x;
    for (u32 i = tid; i <= declared + 1; i += 256) out[i] = 0;
    if (tid == 0) { s_bad = 0; s_top = 0; s_best = 0; }
    __syncthreads();
    u32 bad = 0;
    for (u64 i = tid; i < n; i += 256) { u32 const v = src[i]; if (v > declared) bad = 1; else atomicAdd(&out[v], 1u); }
    if (bad) s_bad = 1;
    __syncthreads();
    if (s_bad) { for (u32 i = tid; i <= declared; i += 256) out[i] = 0; if (tid == 0) *ret = err(E_MSV_TOO_SMALL); return; }
    u32 top = 0, best = 0;
    for (u32 i = tid; i <= declared; i += 256) { u32 const c = out[i]; if (c) { top = i; best = c > best ? c : best; } }
    atomicMax(&s_top, top); atomicMax(&s_best, best);
    __syncthreads();
    if (tid == 0) { out[declared + 1] = n ? s_top : 0; *ret = n ? s_best : 0; }
}

// ---- everything O(alphabet)/O(table): one kernel, op-code dispatched ----
// buf layout: the offsets in micro.h, per op below; a[] carries scalars.
__global__ void __launch_bounds__(256) micro_kernel(int op, MicroArgs A, u8* buf, u64* ret)
{
    __shared__ u32 s_count[256];
    __shared__ u32 s_ct[256];
    __shared__ HNode s_nodes[2 * 256 + 2];
    __shared__ u32 s_a[256], s_b[256];
    __shared__ u32 s_w[384];
    int const tid = threadIdx.x;
    switch (op) {
    case MOP_NORMALIZE: {          // in: count u32[msv+1] @0 ; out: norm i16[msv+1] @MICRO_OUT
        if (tid == 0) *ret = d_normalize((short*)(buf + MICRO_OUT), (unsigned)A.a[0], (const unsigned*)buf, A.a[1], (unsigned)A.a[2]);
        break; }
    case MOP_WRITE_NCOUNT: {       // in: norm @0 ; out: bytes @MICRO_OUT
        if (tid == 0) *ret = d_write_ncount(buf + MICRO_OUT, A.a[0], (const short*)buf, (unsigned)A.a[1], (unsigned)A.a[2]);
        break; }
    case MOP_READ_NCOUNT: {        // in: header bytes @0 (size a0), msv in a1 ; out: norm @MICRO_OUT, msv/tl as u32 @MICRO_META
        if (tid == 0) {
            unsigned msv = (unsigned)A.a[1], tl = 0;
            *ret = d_read_ncount((short*)(buf + MICRO_OUT), &msv, &tl, buf, A.a[0]);
            ((u32*)(buf + MICRO_META))[0] = msv; ((u32*)(buf + MICRO_META))[1] = tl;
        }
        break; }
    case MOP_BUILD_CTABLE: {       // in: norm @0 ; out: ct @MICRO_OUT ; scratch @MICRO_WORK
        if (tid == 0) {
            unsigned const msv = (unsigned)A.a[0], tl = (unsigned)A.a[1];
            if (tl > 13 || msv > 4095) { *ret = err(E_TLOG_TOO_LARGE); break; }
            d_build_ctable_serial((u32*)(buf + MICRO_OUT), (const short*)buf, msv, tl, (u16*)(buf + MICRO_WORK), (u32*)(buf + MICRO_WORK + 32768));
            *ret = 0;
        }
        break; }
    case MOP_BUILD_DTABLE: {       // in: norm @0 ; out: dt @MICRO_OUT ; a2 = wide
        if (tid == 0) {
            unsigned const msv = (unsigned)A.a[0], tl = (unsigned)A.a[1];
            if (A.a[2]) *ret = d_build_dtable_serial<true>((u32*)(buf + MICRO_OUT), (const short*)buf, msv, tl, U16_MAX_SV, U16_MAX_TLOG, (u16*)(buf + MICRO_WORK), (u16*)(buf + MICRO_WORK + 32768));
            else *ret = d_build_dtable_serial<false>((u32*)(buf + MICRO_OUT), (const short*)buf, msv, tl, FSE_MAX_SV, FSE_MAX_TLOG, (u16*)(buf + MICRO_WORK), (u16*)(buf + MICRO_WORK + 32768));
        }
        break; }
    case MOP_HUF_BUILD_CTABLE: {   // in: count u32[256] @0 ; out: ctable u32[256] @MICRO_OUT
        s_count[tid] = ((u32)tid <= A.a[0]) ? ((const u32*)buf)[tid] : 0;
        __syncthreads();
        u64 const r = cta_huf_build_ctable(s_ct, s_count, (u32)A.a[0], (u32)A.a[1], s_nodes, s_a, s_b);
        if (!is_err(r)) ((u32*)(buf + MICRO_OUT))[tid] = s_ct[tid];
        if (tid == 0) *ret = r;
        break; }
    case MOP_HUF_WRITE_CTABLE: {   // in: ctable u32[256] @0 ; out: bytes @MICRO_OUT ; a0 = cap, a1 = msv, a2 = huffLog
        if (tid == 0) *ret = d_huf_write_ctable(buf + MICRO_OUT, A.a[0] < 136 ? A.a[0] : 136, (const u32*)buf, (unsigned)A.a[1], (unsigned)A.a[2], s_w);
        break; }
    case MOP_HUF_READ_STATS: {     // in: bytes @0 (a0) ; out: weights @MICRO_OUT (hwSize a1), rankStats u32[13] @MICRO_META, nbSym,tl @MICRO_META_HUF
        if (tid == 0) {
            u32 nb = 0, tl = 0;
            *ret = d_huf_read_stats(buf + MICRO_OUT, A.a[1], (u32*)(buf + MICRO_META), &nb, &tl, buf, A.a[0]);
            ((u32*)(buf + MICRO_META_HUF))[0] = nb; ((u32*)(buf + MICRO_META_HUF))[1] = tl;
        }
        break; }
    case MOP_HUF_READ_DTABLE_X1: { // in: bytes @0 (a0), a1 = DTable header word ; out: dtable u32[1+2048] @MICRO_DTABLE_X1
        if (tid == 0) {
            u8* const weights = buf + MICRO_OUT;
            u32 rank[17]; u32 nb = 0, tl = 0;
            u32* const dt = (u32*)(buf + MICRO_DTABLE_X1);
            u16* const cells = (u16*)(dt + 1);
            u64 const h = d_huf_read_stats(weights, 256, rank, &nb, &tl, buf, A.a[0]);
            u32 const hdr = (u32)A.a[1];
            dt[0] = hdr;
            if (is_err(h)) { *ret = h; break; }
            if (tl > (hdr & 0xFF) + 1) { *ret = err(E_TLOG_TOO_LARGE); break; }      // huf_decompress.c:143
            dt[0] = (hdr & 0xFF0000FFu) | (tl << 16);
            u32 next = 0;
            for (u32 n = 1; n < tl + 1; n++) { u32 const cur = next; next += rank[n] << (n - 1); rank[n] = cur; }
            for (u32 n = 0; n < nb; n++) {
                u32 const w = weights[n], span = (1u << w) >> 1, cell = n | ((tl + 1 - w) << 8);
                for (u32 u = 0; u < span; u++) cells[rank[w] + u] = (u16)cell;
                rank[w] += span;
            }
            *ret = h;
        }
        break; }
    // ---- payload coding with a caller-supplied table image (the *_usingCTable / *_usingDTable entry points): table @0,
    //      input @a2 = MICRO_PAYLOAD (a0 bytes), output @a3 (capacity a1).  One lane per stream; these serve single calls, not throughput.
    case MOP_FSE_ENCODE_CT: {      // FSE_compress_usingCTable (fse_compress.c:554-623)
        if (tid == 0) *ret = d_fse_encode_serial(buf + A.a[3], A.a[1], buf + A.a[2], A.a[0], (const u32*)buf);
        break; }
    case MOP_FSE_DECODE_DT: {      // FSE_decompress_usingDTable (fse_decompress.c:178-252)
        if (tid == 0) *ret = d_fse_decode_serial(buf + A.a[3], A.a[1], buf + A.a[2], A.a[0], (const u32*)buf);
        break; }
    case MOP_HUF_ENCODE4X_CT: {    // HUF_compress4X_usingCTable (huf_compress.c:552-603): lane k codes segment k, lane 0 assembles
        __shared__ u64 s_len[4];
        const u32* const ct = (const u32*)buf;
        const u8* const in = buf + A.a[2]; u8* const out = buf + A.a[3];
        u64 const n = A.a[0], cap = A.a[1];
        u64 const seg = (n + 3) / 4;
        bool const refuse = cap < 6 + 1 + 1 + 1 + 8 || n < 12;                       // :564-565
        u8* const stage = buf + A.a[3] + ((cap + 15) & ~15ull);                     // 4 private areas of `cap` bytes behind the output
        if (tid < 4 && !refuse) {
            u64 const beg = seg * tid, end = tid < 3 ? seg * (tid + 1) : n;
            BitSink sk; sink_open(sk, stage + tid * ((cap + 15) & ~15ull), cap);     // capacity is judged by lane 0 with the real remaining room
            for (u64 i = end; i-- > beg;) { u32 const e = ct[in[i]]; sink_put(sk, e & 0xFFFF, e >> 16); }
            sink_put(sk, 1, 1);                                                      // end mark
            s_len[tid] = sk.nbits;
            if (sk.held) { if (sk.nbytes < cap) sk.out[sk.nbytes] = (u8)sk.acc; }
        }
        __syncthreads();
        if (tid == 0) {
            if (refuse) { *ret = 0; break; }
            u64 op = 6; u64 r = 0; bool ok = true;
            for (int k = 0; k < 4 && ok; k++) {
                u64 const room = cap - op;                                           // BIT_initCStream / closeCStream rules (bitstream.h:183-260)
                u64 const bits = s_len[k], bytes = (bits + 7) >> 3;
                if (room <= 8 || (bits >> 3) >= room - 8) { ok = false; break; }
                const u8* const sp = stage + k * ((cap + 15) & ~15ull);
                for (u64 i = 0; i < bytes; i++) out[op + i] = sp[i];
                if (k < 3) { out[2 * k] = (u8)bytes; out[2 * k + 1] = (u8)(bytes >> 8); }
                op += bytes;
            }
            r = ok ? op : 0;
            *ret = r;
        }
        break; }
    case MOP_HUF_ENCODE1X_CT: {    // HUF_compress1X_usingCTable (huf_compress.c:457-502): one stream, last symbol first
        if (tid == 0) {
            const u32* const ct = (const u32*)buf; const u8* const in = buf + A.a[2];
            u64 const n = A.a[0], cap = A.a[1];
            if (cap < 8) { *ret = 0; break; }                                        // :470
            BitSink sk; sink_open(sk, buf + A.a[3], cap);
            if (!sk.usable) { *ret = 0; break; }
            for (u64 i = n; i-- > 0;) { u32 const e = ct[in[i]]; sink_put(sk, e & 0xFFFF, e >> 16); }
            *ret = sink_close(sk);
        }
        break; }
    case MOP_HUF_READ_DTABLE_X2: { // HUF_readDTableX2 (huf_decompress.c:551-649): in: bytes @0 (a0), a1 = DTable header word ; out: dtable u32[1+4096] @MICRO_DTABLE_X2
        if (tid == 0) *ret = d_huf_build_dtable_x2((u32*)(buf + MICRO_DTABLE_X2), (u32)A.a[1], buf + MICRO_OUT, buf + MICRO_META, buf + MICRO_META + 256, buf, A.a[0]);
        break; }
    case MOP_HUF_DECODE4X1_DT:     // HUF_decompress4X1_usingDTable (huf_decompress.c:262-354)
    case MOP_HUF_DECODE1X1_DT:     // HUF_decompress1X1_usingDTable (:240-260)
    case MOP_HUF_DECODE4X2_DT:     // HUF_decompress4X2_usingDTable (:749-862)
    case MOP_HUF_DECODE1X2_DT: {   // HUF_decompress1X2_usingDTable (:722-747)
        __shared__ u64 s_init[4]; __shared__ u32 s_done[4];
        bool const four = op == MOP_HUF_DECODE4X1_DT || op == MOP_HUF_DECODE4X2_DT;
        const u32* const dtab = (const u32*)buf; const u8* const c = buf + A.a[2]; u8* const out = buf + A.a[3];
        u64 const r = (op == MOP_HUF_DECODE4X1_DT || op == MOP_HUF_DECODE1X1_DT)
                    ? cta_huf_decode<d_huf_decode_stream_x1>(four, dtab, c, A.a[0], out, A.a[1], s_init, s_done)
                    : cta_huf_decode<d_huf_decode_stream_x2>(four, dtab, c, A.a[0], out, A.a[1], s_init, s_done);
        if (tid == 0) *ret = r;
        break; }
    default: if (tid == 0) *ret = err(E_GENERIC);
    }
}

cudaError_t launch_hist(const void* src, u64 n, u32 declared, u32* out, u64* ret, cudaStream_t s)
{ hist_kernel<<<1, 256, 0, s>>>((const u8*)src, n, declared, out, ret); return cudaGetLastError(); }
cudaError_t launch_hist16(const void* src, u64 n, u32 declared, u32* out, u64* ret, cudaStream_t s)
{ hist16_kernel<<<1, 256, 0, s>>>((const u16*)src, n, declared, out, ret); return cudaGetLastError(); }
cudaError_t launch_micro(int op, const MicroArgs& A, void* buf, u64* ret, cudaStream_t s)
{ micro_kernel<<<1, 256, 0, s>>>(op, A, (u8*)buf, ret); return cudaGetLastError(); }

}  // namespace fseb
