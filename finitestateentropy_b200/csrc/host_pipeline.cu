// host_pipeline.cu -- whole-batch calls on HOST buffers (what an unmodified host program would hand over; declarations:
// include/fse_b200.h): the slot pair FSEB200_{compress,decompress}_host, the packed pair FSEB200_{compress,decompress}_host_packed
// and the .fse frame calls.  Each cuts its batch into chunks that are copied in, processed and copied out on a ring of streams,
// so that PCIe transfers overlap the kernels; one driver, run_chunks, runs the chunks of every call.
#include "capi_common.h"
#include "fse_b200.h"
#include "launch_util.cuh"
#include "xxh32.h"
#include <algorithm>
#include <cstring>
#include <mutex>
#include <thread>
#include <vector>

using namespace fseb;

namespace {

// NS non-blocking streams and, per stream, grow-only device buffers by role and a pinned host image.  One ring per device and
// call family; its mutex serialises the calls of that family.
template <int NS_>
struct Ring {
    enum { NS = NS_ };
    cudaStream_t st[NS] = {};
    u8* dA[NS] = {};              // uncompressed side
    u8* dB[NS] = {};              // compressed slots / packed side
    u8* dW[NS] = {};              // FSE staging slots
    u64* dD[NS] = {};             // per-block words: sizes and results, or descriptors
    u64* hD[NS] = {};             // pinned host image of the per-block words
    size_t capA = 0, capB = 0, capW = 0, capD = 0, capH = 0;
    std::mutex mu;
    template <typename T> static cudaError_t grow(T* (&p)[NS], size_t& cap, size_t need, bool host)
    {
        if (need <= cap) return cudaSuccess;
        for (int i = 0; i < NS; i++) {
            if (p[i]) { cudaError_t const e = host ? cudaFreeHost(p[i]) : cudaFree(p[i]); p[i] = nullptr; if (e != cudaSuccess) return e; }
        }
        cap = 0;
        for (int i = 0; i < NS; i++) {
            cudaError_t const e = host ? cudaMallocHost((void**)&p[i], need) : cudaMalloc((void**)&p[i], need);
            if (e != cudaSuccess) return e;
        }
        cap = need;
        return cudaSuccess;
    }
    // `a`, `b`, `w` bytes, `d` device words and `h` pinned words per stream; the A and B sides get the decoders' slack
    cudaError_t ensure(size_t a, size_t b, size_t w, size_t d, size_t h)
    {
        cudaError_t e = cudaSuccess;
        for (int i = 0; i < NS && e == cudaSuccess; i++) if (!st[i]) e = cudaStreamCreateWithFlags(&st[i], cudaStreamNonBlocking);
        if (e == cudaSuccess) e = grow(dA, capA, a + 256, false);
        if (e == cudaSuccess) e = grow(dB, capB, b + 256, false);
        if (e == cudaSuccess) e = grow(dW, capW, w, false);
        if (e == cudaSuccess) e = grow(dD, capD, d * sizeof(u64), false);
        if (e == cudaSuccess) e = grow(hD, capH, h * sizeof(u64), true);
        return e;
    }
};
// the slot pair's ring and the packed pair's, which the frame calls share
Ring<4>& slot_ring() { static Ring<4> r[MAX_DEVICES]; return r[current_device()]; }
Ring<3>& packed_ring() { static Ring<3> r[MAX_DEVICES]; return r[current_device()]; }

// Runs the chunks [0, nChunks) of one call on ring R:
// - queue(ci, k) enqueues chunk ci on stream k = ci % NS;
// - finish(ci, k) runs on the host, in chunk order, `lag` chunks later: before chunk ci + lag is queued.  With lag <= NS the chunk
//   that last used a stream's buffers and pinned image has been finished before the stream takes its next chunk.  At lag 0
//   finish(ci) runs just before queue(ci); a call without a finish step passes a no-op there, and its stream reuse is ordered
//   by each stream alone;
// - the loop stops at the first CUDA error, or once a finish step sets *verdict;
// - every stream is drained, also after a failure, and the first error is returned.
template <int NS, class Queue, class Finish>
cudaError_t run_chunks(Ring<NS>& R, size_t nChunks, size_t lag, Queue queue, Finish finish, const size_t* verdict = nullptr)
{
    cudaError_t e = cudaSuccess;
    auto go = [&] { return e == cudaSuccess && !(verdict && *verdict); };
    for (size_t ci = 0; ci < nChunks + lag && go(); ci++) {
        if (ci >= lag) e = finish(ci - lag, (int)((ci - lag) % NS));
        if (go() && ci < nChunks) e = queue(ci, (int)(ci % NS));
    }
    for (int i = 0; i < NS; i++) {
        if (!R.st[i]) continue;
        cudaError_t const d = cudaStreamSynchronize(R.st[i]);
        if (e == cudaSuccess) e = d;
    }
    return e;
}

// Blocks per slot-pair chunk (FSEB200_HOST_CHUNK_BLOCKS, default 2048 = 64 MiB of 32 KB blocks): smaller chunks shorten the
// pipeline's fill and drain but leave the decode kernel a fraction of a wave per launch.
size_t chunk_blocks()
{
    static size_t const v = [] { const char* e = std::getenv("FSEB200_HOST_CHUNK_BLOCKS"); long n = e ? std::atol(e) : 2048; return (size_t)(n < 64 ? 64 : n > 65536 ? 65536 : n); }();
    return v;
}
}

// ================================================================================================
// the slot pair: one block size, chunks of chunk_blocks() blocks.  codec: 0 = FSE, 1 = HUF, 2 = FSE-U16.
// ================================================================================================
FSEB_API size_t FSEB200_compress_host(int codec, void* hCBuf, size_t slot, size_t* hCSizes, const void* hSrc, size_t srcTotal,
                                      size_t blockSize, unsigned maxSymbolValue, unsigned tableLog)
{
    if (blockSize == 0 || slot > 0xFFFFFFFFull || codec < 0 || codec > 2) return (size_t)err(E_SRC_WRONG);
    if (blockSize > (codec == 1 ? (size_t)HUF_BLOCK_MAX : FSE_ONE_BLOCK_MAX)) return (size_t)err(E_SRC_WRONG);
    enc_fn const fn = codec == 0 ? launch_fse_encode : codec == 1 ? launch_huf_encode : launch_fseu16_encode;
    auto& P = slot_ring();
    std::lock_guard<std::mutex> lock(P.mu);
    size_t const CB = chunk_blocks(), nb = (srcTotal + blockSize - 1) / blockSize;
    CK(P.ensure(CB * blockSize, CB * slot, 0, 2 * CB, 0));
    // queue: the chunk up, coded, its sizes down.  finish: wait for its sizes, then copy back only the used width of its slots
    // (strided 2-D copy): the compressed side of the PCIe traffic shrinks from `slot` to max(cSize) bytes per block.
    auto queue = [&](size_t ci, int k) -> cudaError_t {
        size_t const b0 = ci * CB, cb = nb - b0 < CB ? nb - b0 : CB;
        size_t const off = b0 * blockSize;
        size_t const bytes = (off + cb * blockSize <= srcTotal) ? cb * blockSize : srcTotal - off;
        cudaStream_t s = P.st[k];
        cudaError_t r;
        if ((r = cudaMemcpyAsync(P.dA[k], (const unsigned char*)hSrc + off, bytes, cudaMemcpyHostToDevice, s)) != cudaSuccess) return r;
        if ((r = fn(geom(bytes, blockSize, slot), P.dB[k], P.dD[k], P.dA[k], maxSymbolValue, tableLog, s)) != cudaSuccess) return r;
        return cudaMemcpyAsync(hCSizes + b0, P.dD[k], cb * sizeof(u64), cudaMemcpyDeviceToHost, s);
    };
    auto finish = [&](size_t ci, int k) -> cudaError_t {
        size_t const b0 = ci * CB, cb = nb - b0 < CB ? nb - b0 : CB;
        cudaStream_t s = P.st[k];
        cudaError_t const r = cudaStreamSynchronize(s);
        if (r != cudaSuccess) return r;
        size_t width = 0;
        for (size_t b = 0; b < cb; b++) { size_t const c = hCSizes[b0 + b]; if (!is_err(c) && c > width) width = c; }
        width = (width + 63) & ~(size_t)63; if (width > slot) width = slot;
        return width ? cudaMemcpy2DAsync((unsigned char*)hCBuf + b0 * slot, slot, P.dB[k], slot, width, cb, cudaMemcpyDeviceToHost, s) : cudaSuccess;
    };
    CK(run_chunks(P, (nb + CB - 1) / CB, P.NS - 1, queue, finish));
    return 0;
}

FSEB_API size_t FSEB200_decompress_host(int codec, void* hDst, size_t dstTotal, size_t blockSize, const void* hCBuf, size_t slot,
                                        const size_t* hCSizes, size_t* hResults, const void* hOrig)
{
    if (blockSize == 0 || slot > 0xFFFFFFFFull || codec < 0 || codec > 2) return (size_t)err(E_SRC_WRONG);
    if (blockSize > (codec == 1 ? (size_t)HUF_BLOCK_MAX : FSE_ONE_BLOCK_MAX)) return (size_t)err(E_SRC_WRONG);
    dec_fn const fn = codec == 0 ? launch_fse_decode : codec == 1 ? huf_dec_std : launch_fseu16_decode;
    auto& P = slot_ring();
    std::lock_guard<std::mutex> lock(P.mu);
    size_t const CB = chunk_blocks(), nb = (dstTotal + blockSize - 1) / blockSize;
    CK(P.ensure(CB * blockSize, CB * slot, 0, 2 * CB, 0));
    // queue: the used width of the chunk's slots and its sizes up, decoded, the blocks and results down.  No finish step: a
    // stream's buffers are reused in its own order.
    auto queue = [&](size_t ci, int k) -> cudaError_t {
        size_t const b0 = ci * CB, cb = nb - b0 < CB ? nb - b0 : CB;
        size_t const off = b0 * blockSize;
        size_t const bytes = (off + cb * blockSize <= dstTotal) ? cb * blockSize : dstTotal - off;
        cudaStream_t s = P.st[k];
        size_t width = 0;
        for (size_t bb = 0; bb < cb; bb++) { size_t const c = hCSizes[b0 + bb]; if (!is_err(c) && c > width) width = c; }
        width = (width + 16 + 63) & ~(size_t)63; if (width > slot) width = slot;     // +16: kernels read whole aligned 16-byte chunks
        cudaError_t r;
        if (width && (r = cudaMemcpy2DAsync(P.dB[k], slot, (const unsigned char*)hCBuf + b0 * slot, slot, width, cb, cudaMemcpyHostToDevice, s)) != cudaSuccess) return r;
        if ((r = cudaMemcpyAsync(P.dD[k], hCSizes + b0, cb * sizeof(u64), cudaMemcpyHostToDevice, s)) != cudaSuccess) return r;
        if ((r = fn(geom(bytes, blockSize, slot), P.dA[k], P.dB[k], P.dD[k], P.dD[k] + CB, nullptr, s)) != cudaSuccess) return r;
        if ((r = cudaMemcpyAsync((unsigned char*)hDst + off, P.dA[k], bytes, cudaMemcpyDeviceToHost, s)) != cudaSuccess) return r;
        return cudaMemcpyAsync(hResults + b0, P.dD[k] + CB, cb * sizeof(u64), cudaMemcpyDeviceToHost, s);
    };
    CK(run_chunks(P, (nb + CB - 1) / CB, 0, queue, [](size_t, int) { return cudaSuccess; }));
    if (hOrig) {   // raw / RLE blocks: regenerated on the host, exactly as bench.c:393-402 does
        for (size_t b = 0; b < nb; b++) {
            size_t const cs = hCSizes[b];
            if (cs > 1 || (cs == 1 && codec == 2)) continue;
            size_t const off = b * blockSize;
            size_t const n = off + blockSize <= dstTotal ? blockSize : dstTotal - off;
            if (cs == 0) std::memcpy((unsigned char*)hDst + off, (const unsigned char*)hOrig + off, n);
            else if (codec != 1) std::memset((unsigned char*)hDst + off, ((const unsigned char*)hOrig)[off], n);
            else continue;                                                  // HUF regenerates RLE blocks itself (lib/huf.h:62)
            hResults[b] = n;
        }
    }
    return 0;
}

// ================================================================================================
// the packed pair: blocks of any size on HOST buffers through the packed device calls, so the stream a host program keeps is
// the one the device packed calls produce -- one buffer and its offsets, raw and RLE blocks stored in place -- and decodes
// without the original.  Chunks of blocks, cut by a byte budget, run on the packed ring; inside a chunk the device packed calls
// run unchanged on chunk-local offsets with room for every block, and the host turns the results into the whole batch's:
// global offsets, the capacity rule, only the stored bytes copied down.
// codec: 0 = FSE, 1 = Huff0 4X, 2 = FSE-U16, 3 = Huff0 1X.
// ================================================================================================
namespace {
// Bytes per pipeline chunk (FSEB200_HOST_PACKED_CHUNK_BYTES, default 64 MiB).  A block counts its bytes plus 512 for its
// descriptors and staging overhead, so a chunk of tiny blocks stays bounded too; a block above the budget is a chunk of its own.
size_t chunk_budget()
{
    static size_t const v = [] { const char* e = std::getenv("FSEB200_HOST_PACKED_CHUNK_BYTES"); long long n = e ? std::atoll(e) : 64ll << 20; return (size_t)(n < 1 ? 1 : n); }();
    return v;
}
constexpr u64 BLOCK_OVERHEAD = 512;

struct HostChunk { size_t b0, b1; u64 a0, a1; };   // blocks [b0, b1); uncompressed bytes [a0, a1) of the batch
struct ChunkMax { size_t blocks = 0; u64 bytes = 0, packed = 0; };   // each the largest over the chunks

// chunks of blocks whose weight (uncompressed bytes + the packed bytes `packed(b)` + BLOCK_OVERHEAD) stays within the budget;
// `most` gets the largest block count, uncompressed bytes and packed bytes of a chunk
template <typename F>
std::vector<HostChunk> cut_chunks(const size_t* sizes, size_t nBlocks, u64 unit, F packed, ChunkMax& most)
{
    std::vector<HostChunk> out;
    size_t const budget = chunk_budget();
    HostChunk c = { 0, 0, 0, 0 };
    u64 w = 0, p = 0;
    auto close = [&] {
        out.push_back(c);
        most.blocks = std::max(most.blocks, c.b1 - c.b0); most.bytes = std::max(most.bytes, c.a1 - c.a0); most.packed = std::max(most.packed, p);
    };
    for (size_t b = 0; b < nBlocks; b++) {
        u64 const bytes = unit * sizes[b], pb = packed(b), wb = bytes + pb + BLOCK_OVERHEAD;
        if (c.b1 > c.b0 && w + wb > budget) { close(); c = { b, b, c.a1, c.a1 }; w = 0; p = 0; }
        c.b1 = b + 1; c.a1 += bytes; w += wb; p += pb;
    }
    close();
    return out;
}

// Queues chunk c of a host batch through the device packed compress in slot k: the source and the descriptors up, the packed
// call with room for every block.  On the device the slot's descriptor words are then: source pointers (cb), sizes (cb), offsets
// (cb + 1), values (cb).  codec as the host packed calls.
cudaError_t queue_packed_compress(Ring<3>& P, int k, const HostChunk& c, int codec, const void* hSrc, const size_t* hSrcSizes,
                                  unsigned maxSymbolValue, unsigned tableLog)
{
    bool const fse = codec == 0 || codec == 2, wide = codec == 2;
    u64 const unit = wide ? 2 : 1;
    size_t const cb = c.b1 - c.b0;
    u64 const bytes = c.a1 - c.a0;
    cudaStream_t const s = P.st[k];
    u64* const h = P.hD[k];
    u64* const d = P.dD[k];
    for (size_t b = 0, a = 0; b < cb; b++) { h[b] = reinterpret_cast<u64>(P.dA[k] + a); h[cb + b] = hSrcSizes[c.b0 + b]; a += unit * hSrcSizes[c.b0 + b]; }
    cudaError_t r;
    if (bytes && (r = cudaMemcpyAsync(P.dA[k], (const u8*)hSrc + c.a0, bytes, cudaMemcpyHostToDevice, s)) != cudaSuccess) return r;
    if ((r = cudaMemcpyAsync(d, h, 2 * cb * sizeof(u64), cudaMemcpyHostToDevice, s)) != cudaSuccess) return r;
    u64* const offs = d + 2 * cb;
    u64* const vals = d + 3 * cb + 1;
    if (fse) return launch_fse_compress_packed(P.dB[k], bytes, offs, vals, (const u8* const*)d, d + cb, (u32)cb, P.dW[k], P.capW, wide,
                                               maxSymbolValue, tableLog, s);
    PackedDescs g;
    g.out = P.dB[k]; g.outCap = bytes; g.offset = offs; g.result = vals;
    g.src = (const u8* const*)d; g.srcSize = d + cb; g.nBlocks = (u32)cb;
    return launch_huf_encode_packed(g, codec == 1 ? 4 : 1, maxSymbolValue, tableLog, s);
}
}

FSEB_API size_t FSEB200_compress_host_packed(int codec, void* hOut, size_t outCapacity, size_t* hOffsets, size_t* hCSizes,
                                             const void* hSrc, const size_t* hSrcSizes, size_t nBlocks,
                                             unsigned maxSymbolValue, unsigned tableLog)
{
    if (codec < 0 || codec > 3 || nBlocks > 0xFFFFFFFFull) return (size_t)err(E_SRC_WRONG);
    if (nBlocks == 0) return 0;
    if (!hOut || !hOffsets || !hCSizes || !hSrc || !hSrcSizes) return (size_t)err(E_SRC_WRONG);
    bool const fse = codec == 0 || codec == 2, wide = codec == 2;
    ChunkMax most;
    std::vector<HostChunk> const chunks = cut_chunks(hSrcSizes, nBlocks, wide ? 2 : 1, [](size_t) { return (u64)0; }, most);
    size_t maxW = 0;
    if (fse) for (const HostChunk& c : chunks) maxW = std::max(maxW, FSEB200_FSE_packed_workspace(c.b1 - c.b0, c.a1 - c.a0));
    auto& P = packed_ring();
    std::lock_guard<std::mutex> lock(P.mu);
    // a block stores at most its own bytes
    cudaError_t e = P.ensure(most.bytes, most.bytes, maxW, 4 * most.blocks + 1, 4 * most.blocks + 1);
    u64 total = 0;                                                  // global offset of the next chunk's first block
    // queue: the source and the descriptors up, the packed call with room for every block, offsets and values down
    auto queue = [&](size_t ci, int k) -> cudaError_t {
        size_t const cb = chunks[ci].b1 - chunks[ci].b0;
        cudaError_t const r = queue_packed_compress(P, k, chunks[ci], codec, hSrc, hSrcSizes, maxSymbolValue, tableLog);
        if (r != cudaSuccess) return r;
        return cudaMemcpyAsync(P.hD[k] + 2 * cb, P.dD[k] + 2 * cb, (2 * cb + 1) * sizeof(u64), cudaMemcpyDeviceToHost, P.st[k]);
    };
    // finish: global offsets, the capacity rule of one call over the whole batch, and the stored bytes -- a prefix of the chunk's
    // packed bytes, since the blocks that fit come first -- copied down
    auto finish = [&](size_t ci, int k) -> cudaError_t {
        const HostChunk& c = chunks[ci];
        size_t const cb = c.b1 - c.b0;
        cudaError_t r = cudaStreamSynchronize(P.st[k]);
        if (r != cudaSuccess) return r;
        const u64* const lo = P.hD[k] + 2 * cb;
        const u64* const vals = lo + cb + 1;
        u64 end = 0;
        for (size_t b = 0; b < cb; b++) {
            u64 const off = total + lo[b], len = lo[b + 1] - lo[b];
            u64 v = vals[b];
            if (!is_err(v) && off + len > outCapacity) v = err(E_DST_TOO_SMALL);
            else if (!is_err(v) && len) end = lo[b + 1];
            hOffsets[c.b0 + b] = (size_t)off; hCSizes[c.b0 + b] = (size_t)v;
        }
        if (end && (r = cudaMemcpyAsync((u8*)hOut + total, P.dB[k], end, cudaMemcpyDeviceToHost, P.st[k])) != cudaSuccess) return r;
        total += lo[cb];
        return cudaSuccess;
    };
    if (e == cudaSuccess) e = run_chunks(P, chunks.size(), P.NS - 1, queue, finish);
    if (e != cudaSuccess) return (size_t)err(E_GENERIC);
    hOffsets[nBlocks] = (size_t)total;
    return 0;
}

FSEB_API size_t FSEB200_decompress_host_packed(int codec, void* hDst, const size_t* hDstSizes, size_t* hResults,
                                               const void* hIn, const size_t* hOffsets, size_t nBlocks)
{
    if (codec < 0 || codec > 3 || nBlocks > 0xFFFFFFFFull) return (size_t)err(E_SRC_WRONG);
    if (nBlocks == 0) return 0;
    if (!hDst || !hDstSizes || !hResults || !hIn || !hOffsets) return (size_t)err(E_SRC_WRONG);
    for (size_t b = 0; b < nBlocks; b++) if (hOffsets[b + 1] < hOffsets[b]) return (size_t)err(E_SRC_WRONG);
    bool const fse = codec == 0 || codec == 2, wide = codec == 2;
    u64 const unit = wide ? 2 : 1;
    ChunkMax most;
    std::vector<HostChunk> const chunks = cut_chunks(hDstSizes, nBlocks, unit, [&](size_t b) { return (u64)(hOffsets[b + 1] - hOffsets[b]); }, most);
    auto& P = packed_ring();
    std::lock_guard<std::mutex> lock(P.mu);
    cudaError_t e = P.ensure(most.bytes, most.packed, 0, 4 * most.blocks + 1, 4 * most.blocks + 1);
    // queue: the chunk's packed bytes and descriptors up (offsets rebased to the chunk), the packed decompress, the blocks and
    // their results down
    auto queue = [&](size_t ci, int k) -> cudaError_t {
        const HostChunk& c = chunks[ci];
        size_t const cb = c.b1 - c.b0;
        u64 const in0 = hOffsets[c.b0], in = hOffsets[c.b1] - in0, bytes = c.a1 - c.a0;
        cudaStream_t const s = P.st[k];
        u64* const h = P.hD[k];
        u64* const d = P.dD[k];
        for (size_t b = 0, a = 0; b < cb; b++) { h[b] = reinterpret_cast<u64>(P.dA[k] + a); h[cb + b] = hDstSizes[c.b0 + b]; a += unit * hDstSizes[c.b0 + b]; }
        for (size_t b = 0; b <= cb; b++) h[2 * cb + b] = hOffsets[c.b0 + b] - in0;
        cudaError_t r;
        if (in && (r = cudaMemcpyAsync(P.dB[k], (const u8*)hIn + in0, in, cudaMemcpyHostToDevice, s)) != cudaSuccess) return r;
        if ((r = cudaMemcpyAsync(d, h, (3 * cb + 1) * sizeof(u64), cudaMemcpyHostToDevice, s)) != cudaSuccess) return r;
        u8* const* const dsts = (u8* const*)d;
        u64* const vals = d + 3 * cb + 1;
        r = fse ? launch_fse_decompress_packed(dsts, d + cb, vals, P.dB[k], d + 2 * cb, (u32)cb, wide, s)
                : launch_huf_decompress_packed(dsts, d + cb, vals, P.dB[k], d + 2 * cb, (u32)cb, codec == 1 ? 4 : 1, s);
        if (r != cudaSuccess) return r;
        if (bytes && (r = cudaMemcpyAsync((u8*)hDst + c.a0, P.dA[k], bytes, cudaMemcpyDeviceToHost, s)) != cudaSuccess) return r;
        return cudaMemcpyAsync(h + 3 * cb + 1, vals, cb * sizeof(u64), cudaMemcpyDeviceToHost, s);
    };
    // finish: the results of the chunk, once its stream is done; it runs before the chunk's stream and pinned image take the
    // next chunk
    auto finish = [&](size_t ci, int k) -> cudaError_t {
        size_t const cb = chunks[ci].b1 - chunks[ci].b0;
        cudaError_t const r = cudaStreamSynchronize(P.st[k]);
        if (r == cudaSuccess) std::memcpy(hResults + chunks[ci].b0, P.hD[k] + 3 * cb + 1, cb * sizeof(u64));
        return r;
    };
    if (e == cudaSuccess) e = run_chunks(P, chunks.size(), P.NS, queue, finish);
    return e == cudaSuccess ? 0 : (size_t)err(E_GENERIC);
}

// ================================================================================================
// frames: the .fse format of the reference's file tool (programs/fileio.c:266-626) on host buffers, through the packed
// pair's ring and chunk budget.  Compress: each chunk runs the device packed compress, then frame.cu lays its frame body out on the device --
// headers in front of the stored blocks -- so the body comes down in one copy to its place in the frame; a worker thread hashes
// the whole input meanwhile.  Decompress: the host walks the block headers first (the frame is in host memory), each chunk copies
// up exactly its own frame bytes, the compressed blocks go to the descriptor decoders and the raw and RLE blocks to frame.cu's
// stored-block kernel.  An FSE block may decode short, so a chunk's output offset is known only once every earlier chunk's
// results are in: a chunk is copied down, and hashed in frame order, in the lagged finish step.
// ================================================================================================
namespace {
constexpr u32 MAGIC_FSE = 0x183E2309u, MAGIC_HUF = 0x183E3309u;
constexpr u64 FRAME_HEADER = 5, FRAME_TRAILER = 3;
enum { BT_COMPRESSED = 0, BT_RAW = 1, BT_RLE = 2, BT_END = 3 };

u32 trailer_checksum(u32 h) { return (h >> 5) & ((1u << 22) - 1); }
u64 be16(const u8* p) { return (u64)p[0] << 8 | p[1]; }

struct FrameBlock { u64 head, payload, rSize, cSize; int type; };   // header and payload offsets in the frame

struct FrameWalk {
    size_t verdict = 0;             // 0, or the verdict where the walk stopped (the point FIO_decompressFilename stops at)
    int codec = 0;                  // 0 FSE, 1 Huff0
    std::vector<FrameBlock> blocks; // every block before that point
    u32 checksum = 0;               // the trailer's 22 bits (verdict 0)
};

// the reference's header walk, with its exit codes as verdicts; blocks that would overrun its buffers are corruption_detected
FrameWalk walk_frame(const u8* f, u64 size)
{
    FrameWalk w;
    auto stop = [&w](unsigned code) { w.verdict = (size_t)err(code); };
    if (size < FRAME_HEADER) { stop(E_SRC_WRONG); return w; }                                  // exit 30
    u32 const magic = (u32)f[0] | (u32)f[1] << 8 | (u32)f[2] << 16 | (u32)f[3] << 24;
    if (magic != MAGIC_FSE && magic != MAGIC_HUF) { stop(E_GENERIC); return w; }             // 31 (zlibh too)
    if (f[4] > 6) { stop(E_GENERIC); return w; }                                              // 32
    w.codec = magic == MAGIC_HUF;
    u64 const bs = (u64)1024 << f[4];
    u64 pos = FRAME_HEADER;
    if (pos >= size) { stop(E_SRC_WRONG); return w; }                                         // 34
    for (;;) {
        FrameBlock k;
        k.head = pos;
        k.type = f[pos] >> 6;
        if (k.type == BT_END) break;
        bool const full = f[pos] & 0x20;
        pos++;
        k.rSize = bs;
        if (!full) {
            if (pos + 2 > size) { stop(E_SRC_WRONG); return w; }                              // 35
            k.rSize = be16(f + pos); pos += 2;
        }
        if (k.type == BT_COMPRESSED) {
            if (pos + 2 > size) { stop(E_SRC_WRONG); return w; }                              // 36
            k.cSize = be16(f + pos); pos += 2;
        } else k.cSize = k.type == BT_RAW ? k.rSize : 1;
        if (k.cSize > bs + 4) { stop(E_CORRUPT); return w; }                                  // past its input buffer
        if (pos + k.cSize + 1 > size) { stop(E_SRC_WRONG); return w; }                        // 38: payload + next header byte
        if (k.type != BT_RAW && k.rSize > bs) { stop(E_CORRUPT); return w; }                  // past its output buffer
        k.payload = pos; pos += k.cSize;
        w.blocks.push_back(k);
    }
    if (pos + FRAME_TRAILER > size) { stop(E_SRC_WRONG); return w; }                          // 43
    w.checksum = (u32)be16(f + pos + 1) | (u32)(f[pos] & 0x3F) << 16;
    return w;
}
}

FSEB_API unsigned FSEB200_XXH32(const void* src, size_t srcSize, unsigned seed)
{
    Xxh32 x(seed);
    if (srcSize) x.update(src, srcSize);
    return x.digest();
}

FSEB_API size_t FSEB200_frame_compressBound(size_t srcSize, unsigned blockSizeId)
{
    if (blockSizeId > 6) return (size_t)err(E_SRC_WRONG);
    size_t const bs = (size_t)1024 << blockSizeId;
    // the all-raw frame: a full block takes 1 + bs bytes, a partial one 3 + n; a compressed block is shorter than n - 1 bytes
    // (lib/fse_compress.c, lib/huf_compress.c) behind at most 2 more header bytes, an RLE block 1 byte
    return FRAME_HEADER + srcSize + srcSize / bs + (srcSize % bs ? 3 : 0) + FRAME_TRAILER;
}


FSEB_API size_t FSEB200_frame_compress_host(int codec, unsigned blockSizeId, void* hFrame, size_t frameCapacity,
                                            const void* hSrc, size_t srcSize)
{
    if (codec < 0 || codec > 1 || blockSizeId > 6 || (!hSrc && srcSize) || (!hFrame && frameCapacity)) return (size_t)err(E_SRC_WRONG);
    if (frameCapacity < FRAME_HEADER + FRAME_TRAILER) return (size_t)err(E_DST_TOO_SMALL);
    u8* const out = (u8*)hFrame;
    u32 const magic = codec ? MAGIC_HUF : MAGIC_FSE;
    for (int i = 0; i < 4; i++) out[i] = (u8)(magic >> (8 * i));
    out[4] = (u8)blockSizeId;
    u32 hash = 0;
    std::thread hasher([&hash, hSrc, srcSize] { hash = FSEB200_XXH32(hSrc, srcSize, 0); });
    size_t const bs = (size_t)1024 << blockSizeId, nb = (srcSize + bs - 1) / bs;
    size_t verdict = 0;
    u64 body = 0;                                                   // frame body bytes written so far
    if (nb) {
        std::vector<size_t> sizes(nb, bs);
        sizes[nb - 1] = srcSize - (nb - 1) * bs;
        ChunkMax most;
        std::vector<HostChunk> const chunks = cut_chunks(sizes.data(), nb, 1, [](size_t) { return (u64)0; }, most);
        auto& P = packed_ring();
        std::lock_guard<std::mutex> lock(P.mu);
        // The body goes to the source's buffer once it is coded: the stored blocks plus at most 5 header bytes each.  Every block
        // but the last is full, so the chunk with the most blocks also has the most bytes.
        cudaError_t e = P.ensure(most.bytes + 5 * most.blocks, most.bytes, codec == 0 ? FSEB200_FSE_packed_workspace(most.blocks, most.bytes) : 0,
                                 4 * most.blocks + 1, 4 * most.blocks + 1);
        // queue: the packed compress, the frame body, the offsets and values down
        auto queue = [&](size_t ci, int k) -> cudaError_t {
            size_t const cb = chunks[ci].b1 - chunks[ci].b0;
            u64* const d = P.dD[k];
            cudaError_t r = queue_packed_compress(P, k, chunks[ci], codec, hSrc, sizes.data(), 255, 11);
            if (r == cudaSuccess) r = launch_frame_body(P.dA[k], P.dB[k], d + 2 * cb, d + 3 * cb + 1, d + cb, (u32)cb, bs, P.st[k]);
            if (r != cudaSuccess) return r;
            return cudaMemcpyAsync(P.hD[k] + 2 * cb, d + 2 * cb, (2 * cb + 1) * sizeof(u64), cudaMemcpyDeviceToHost, P.st[k]);
        };
        // finish: the first error value in block order stops the call (fileio.c:329); otherwise the body comes down if it fits
        auto finish = [&](size_t ci, int k) -> cudaError_t {
            const HostChunk& c = chunks[ci];
            size_t const cb = c.b1 - c.b0;
            cudaError_t const r = cudaStreamSynchronize(P.st[k]);
            if (r != cudaSuccess) return r;
            const u64* const lo = P.hD[k] + 2 * cb;
            const u64* const vals = lo + cb + 1;
            u64 len = lo[cb];
            for (size_t b = 0; b < cb && !verdict; b++) {
                u64 const v = vals[b];
                if (is_err(v)) verdict = (size_t)v;
                len += 1 + (sizes[c.b0 + b] == bs ? 0 : 2) + (v >= 2 ? 2 : 0);
            }
            if (!verdict && FRAME_HEADER + body + len + FRAME_TRAILER > frameCapacity) verdict = (size_t)err(E_DST_TOO_SMALL);
            if (verdict) return cudaSuccess;
            u64 const at = body;
            body += len;
            return cudaMemcpyAsync(out + FRAME_HEADER + at, P.dA[k], len, cudaMemcpyDeviceToHost, P.st[k]);
        };
        if (e == cudaSuccess) e = run_chunks(P, chunks.size(), P.NS - 1, queue, finish, &verdict);
        if (!verdict && e != cudaSuccess) verdict = (size_t)err(E_GENERIC);
    }
    hasher.join();
    if (verdict) return verdict;
    u8* const t = out + FRAME_HEADER + body;
    u32 const crc = trailer_checksum(hash);
    t[0] = (u8)((crc >> 16) | (BT_END << 6)); t[1] = (u8)(crc >> 8); t[2] = (u8)crc;
    return (size_t)(FRAME_HEADER + body + FRAME_TRAILER);
}

FSEB_API size_t FSEB200_frame_decompress_bound(const void* hFrame, size_t frameSize)
{
    if (!hFrame && frameSize) return (size_t)err(E_SRC_WRONG);
    FrameWalk const w = walk_frame((const u8*)hFrame, frameSize);
    if (w.verdict) return w.verdict;
    u64 total = 0;
    for (const FrameBlock& k : w.blocks) total += k.rSize;
    return (size_t)total;
}

FSEB_API size_t FSEB200_frame_decompress_host(void* hDst, size_t dstCapacity, const void* hFrame, size_t frameSize)
{
    if ((!hFrame && frameSize) || (!hDst && dstCapacity)) return (size_t)err(E_SRC_WRONG);
    const u8* const f = (const u8*)hFrame;
    u8* const dst = (u8*)hDst;
    FrameWalk const w = walk_frame(f, frameSize);
    const std::vector<FrameBlock>& blk = w.blocks;
    size_t const nb = blk.size();
    u64 nominal = 0;
    bool coded = false;
    for (const FrameBlock& k : blk) { nominal += k.rSize; coded |= k.type == BT_COMPRESSED; }
    if (!coded) {                                                   // every block's output size is known: settled here first
        if (nominal > dstCapacity) return (size_t)err(E_DST_TOO_SMALL);
        if (w.verdict) return w.verdict;
    }
    Xxh32 hash(0);
    size_t verdict = 0;
    u64 out = 0;                                                    // bytes regenerated so far
    if (nb) {
        std::vector<size_t> rs(nb);
        for (size_t b = 0; b < nb; b++) rs[b] = (size_t)blk[b].rSize;
        // a chunk's packed bytes are its frame bytes, headers included
        ChunkMax most;
        std::vector<HostChunk> const chunks = cut_chunks(rs.data(), nb, 1, [&](size_t b) { return blk[b].payload + blk[b].cSize - blk[b].head; }, most);
        std::vector<size_t> nCoded(chunks.size(), 0);
        for (size_t ci = 0; ci < chunks.size(); ci++)
            for (size_t b = chunks[ci].b0; b < chunks[ci].b1; b++) nCoded[ci] += blk[b].type == BT_COMPRESSED;
        auto& P = packed_ring();
        std::lock_guard<std::mutex> lock(P.mu);
        cudaError_t e = P.ensure(most.bytes, most.packed, 0, 5 * most.blocks, 5 * most.blocks);
        // Descriptor words of a chunk with nc compressed and ns stored blocks: destinations, capacities, sources and sizes of
        // the compressed ones (nc each), the stored-block index (3 ns), then the decoders' results (nc).
        auto queue = [&](size_t ci, int k) -> cudaError_t {
            const HostChunk& c = chunks[ci];
            size_t const cb = c.b1 - c.b0, nc = nCoded[ci], ns = cb - nc;
            u64 const f0 = blk[c.b0].head, in = blk[c.b1 - 1].payload + blk[c.b1 - 1].cSize - f0;
            cudaStream_t const s = P.st[k];
            u64* const h = P.hD[k];
            u64* const d = P.dD[k];
            u64* const index = h + 4 * nc;
            for (size_t b = c.b0, a = 0, j = 0, t = 0; b < c.b1; a += blk[b].rSize, b++) {
                const FrameBlock& x = blk[b];
                if (x.type == BT_COMPRESSED) {
                    h[j] = reinterpret_cast<u64>(P.dA[k] + a); h[nc + j] = x.rSize;
                    h[2 * nc + j] = reinterpret_cast<u64>(P.dB[k] + (x.payload - f0)); h[3 * nc + j] = x.cSize;
                    j++;
                } else {
                    index[3 * t] = a; index[3 * t + 1] = x.payload - f0; index[3 * t + 2] = x.rSize | (u64)x.type << 32;
                    t++;
                }
            }
            cudaError_t r;
            if ((r = cudaMemcpyAsync(P.dB[k], f + f0, in, cudaMemcpyHostToDevice, s)) != cudaSuccess) return r;
            if ((r = cudaMemcpyAsync(d, h, (4 * nc + 3 * ns) * sizeof(u64), cudaMemcpyHostToDevice, s)) != cudaSuccess) return r;
            u64* const res = d + 4 * nc + 3 * ns;
            if (nc) {
                BlockDescs g;
                g.dst = (u8* const*)d; g.dstCap = d + nc; g.result = res;
                g.src = (const u8* const*)(d + 2 * nc); g.srcSize = d + 3 * nc; g.nBlocks = (u32)nc;
                r = w.codec ? launch_huf_decode_blocks(g, 4, s) : launch_fse_decode_blocks(g, false, s);
                if (r != cudaSuccess) return r;
                if ((r = cudaMemcpyAsync(h + 4 * nc + 3 * ns, res, nc * sizeof(u64), cudaMemcpyDeviceToHost, s)) != cudaSuccess) return r;
            }
            return ns ? launch_frame_stored(P.dA[k], P.dB[k], d + 4 * nc, ns, s) : cudaSuccess;
        };
        // the chunk whose output has been copied down but not hashed yet
        struct { int k = 0; u64 a = 0, n = 0; } pend;
        auto hash_pending = [&]() -> cudaError_t {
            if (!pend.n) return cudaSuccess;
            cudaError_t const r = cudaStreamSynchronize(P.st[pend.k]);
            if (r == cudaSuccess) hash.update(dst + pend.a, pend.n);
            pend.n = 0;
            return r;
        };
        // finish: the first decoder error or overflow of dstCapacity in block order stops the call; otherwise the chunk's output
        // comes down to its true offset -- in one copy, or block by block when an FSE block decoded short -- and the previous
        // chunk's output, landed meanwhile, is hashed
        auto finish = [&](size_t ci, int k) -> cudaError_t {
            const HostChunk& c = chunks[ci];
            size_t const nc = nCoded[ci], ns = (c.b1 - c.b0) - nc;
            cudaError_t r = cudaStreamSynchronize(P.st[k]);
            if (r != cudaSuccess) return r;
            const u64* const res = P.hD[k] + 4 * nc + 3 * ns;
            u64 o = out;
            bool shortBlock = false;
            for (size_t b = c.b0, j = 0; b < c.b1 && !verdict; b++) {
                u64 n = blk[b].rSize;
                if (blk[b].type == BT_COMPRESSED) {
                    u64 const v = res[j++];
                    if (is_err(v)) { verdict = (size_t)v; break; }
                    shortBlock |= v != n;
                    n = v;
                }
                if (o + n > dstCapacity) verdict = (size_t)err(E_DST_TOO_SMALL);
                o += n;
            }
            if (verdict) return cudaSuccess;
            if (!shortBlock) {
                if (o > out && (r = cudaMemcpyAsync(dst + out, P.dA[k], o - out, cudaMemcpyDeviceToHost, P.st[k])) != cudaSuccess) return r;
            } else {
                u64 at = out;
                for (size_t b = c.b0, a = 0, j = 0; b < c.b1; a += blk[b].rSize, b++) {
                    u64 const n = blk[b].type == BT_COMPRESSED ? res[j++] : blk[b].rSize;
                    if (n && (r = cudaMemcpyAsync(dst + at, P.dA[k] + a, n, cudaMemcpyDeviceToHost, P.st[k])) != cudaSuccess) return r;
                    at += n;
                }
            }
            if ((r = hash_pending()) != cudaSuccess) return r;
            pend.k = k; pend.a = out; pend.n = o - out;
            out = o;
            return cudaSuccess;
        };
        if (e == cudaSuccess) e = run_chunks(P, chunks.size(), P.NS - 1, queue, finish, &verdict);
        if (e == cudaSuccess && !verdict) e = hash_pending();      // the last chunk's output, landed by the drain
        if (!verdict && e != cudaSuccess) verdict = (size_t)err(E_GENERIC);
    }
    if (verdict) return verdict;
    if (w.verdict) return w.verdict;
    if (trailer_checksum(hash.digest()) != w.checksum) return (size_t)err(E_CORRUPT);   // exit 44
    return (size_t)out;
}
