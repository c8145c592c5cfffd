// host_pipeline.cu -- whole-batch calls on HOST buffers (what an unmodified host program would hand over; declarations:
// include/fse_b200.h): the slot pair FSEB200_{compress,decompress}_host, the packed pair FSEB200_{compress,decompress}_host_packed,
// the packed Huff0 chain pair FSEB200_compress_host_repeat_chains_packed / FSEB200_decompress_host_repeat_packed and the .fse
// frame calls.  Each cuts its batch into chunks that are copied in, processed and copied out on a ring of streams,
// so that PCIe transfers overlap the kernels; one driver, run_chunks, runs the chunks of every call.
#include "capi_common.h"
#include "fse_b200.h"
#include "frame_walk.h"
#include "launch_util.cuh"
#include "xxh32.h"
#include <algorithm>
#include <cassert>
#include <atomic>
#include <cstring>
#include <condition_variable>
#include <memory>
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

// A chunk's per-block words, one layout per pipelined call: the same segment offsets in the pinned image and the device words,
// and `end`, which sizes Ring::ensure.  The packed pair, for cb blocks: block pointers, sizes, offsets (cb + 1), values.
struct PackedWords {
    size_t ptr = 0, size, offset, value, end;
    explicit PackedWords(size_t cb) : size(cb), offset(2 * cb), value(3 * cb + 1), end(4 * cb + 1) {}
};
// The frame compress, for cb blocks and nh device-hashed frames: queue_packed_compress's words, roles, hash ranges, hashes.
struct FrameCompressWords {
    PackedWords packed; size_t role, range, hash, end;
    FrameCompressWords(size_t cb, size_t nh) : packed(cb), role(packed.end), range(role + cb), hash(range + 2 * nh), end(hash + nh) {}
};
// The frame decompress, for nc compressed and ns stored blocks and nh device-hashed frames: the compressed blocks' destinations,
// capacities, sources and sizes (the FSE frames' first), the stored-block index, hash ranges, then the results and hashes.
struct FrameDecompressWords {
    size_t dst = 0, cap, src, srcSize, index, range, result, hash, end;
    FrameDecompressWords(size_t nc, size_t ns, size_t nh) : cap(nc), src(2 * nc), srcSize(3 * nc), index(4 * nc), range(index + 3 * ns),
        result(range + 2 * nh), hash(result + nc), end(hash + nh) {}
};

// chunks of blocks whose weight (uncompressed bytes + the packed bytes `packed(b)` + BLOCK_OVERHEAD) stays within the budget;
// `most` gets the largest block count, uncompressed bytes and packed bytes of a chunk.  With `whole` (the frame calls),
// whole[b] is the weight of the frame that starts at block b (0 inside a frame): a chunk also closes in front of a frame that
// fits the budget whole but not the rest of the chunk, so only frames above the budget span chunks.
template <typename F>
std::vector<HostChunk> cut_chunks(const size_t* sizes, size_t nBlocks, u64 unit, F packed, ChunkMax& most, const u64* whole = nullptr)
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
        bool const frameBreak = whole && whole[b] && whole[b] <= budget && w + whole[b] > budget;
        if (c.b1 > c.b0 && (w + wb > budget || frameBreak)) { close(); c = { b, b, c.a1, c.a1 }; w = 0; p = 0; }
        c.b1 = b + 1; c.a1 += bytes; w += wb; p += pb;
    }
    close();
    return out;
}

// Queues chunk c of a host batch through the device packed compress in slot k: the source and the descriptors up, the packed
// call with room for every block, its device words laid out as PackedWords.  codec as the host packed calls.
cudaError_t queue_packed_compress(Ring<3>& P, int k, const HostChunk& c, int codec, const void* hSrc, const size_t* hSrcSizes,
                                  unsigned maxSymbolValue, unsigned tableLog)
{
    bool const fse = codec == 0 || codec == 2, wide = codec == 2;
    u64 const unit = wide ? 2 : 1;
    size_t const cb = c.b1 - c.b0;
    PackedWords const L(cb);
    u64 const bytes = c.a1 - c.a0;
    cudaStream_t const s = P.st[k];
    u64* const h = P.hD[k];
    u64* const d = P.dD[k];
    for (size_t b = 0, a = 0; b < cb; b++) { h[L.ptr + b] = reinterpret_cast<u64>(P.dA[k] + a); h[L.size + b] = hSrcSizes[c.b0 + b]; a += unit * hSrcSizes[c.b0 + b]; }
    cudaError_t r;
    if (bytes && (r = cudaMemcpyAsync(P.dA[k], (const u8*)hSrc + c.a0, bytes, cudaMemcpyHostToDevice, s)) != cudaSuccess) return r;
    if ((r = cudaMemcpyAsync(d, h, L.offset * sizeof(u64), cudaMemcpyHostToDevice, s)) != cudaSuccess) return r;
    const u8* const* const src = (const u8* const*)(d + L.ptr);
    if (fse) return launch_fse_compress_packed(P.dB[k], bytes, d + L.offset, d + L.value, src, d + L.size, (u32)cb, P.dW[k], P.capW, wide,
                                               maxSymbolValue, tableLog, s);
    PackedDescs g;
    g.out = P.dB[k]; g.outCap = bytes; g.offset = d + L.offset; g.result = d + L.value;
    g.src = src; g.srcSize = d + L.size; g.nBlocks = (u32)cb;
    return launch_huf_encode_descs(g, codec == 1 ? 4 : 1, maxSymbolValue, tableLog, s);
}

// The finish of a packed compress chunk c whose offsets `lo` (chunk-local, cb + 1) and values have landed in the pinned image:
// global offsets, the capacity rule of one call over the whole batch (a block that does not fit gets dstSize_tooSmall and, where
// there are kinds, kind 4), and the stored bytes -- a prefix of the chunk's packed bytes at dOut, since the blocks that fit come
// first -- copied down on s.  `total` is the global offset of the chunk's first block and moves past the chunk.  Where there are
// kinds, a block stores bytes unless its kind is 4 (under the literal policy a raw block's value may be an error).
cudaError_t finish_packed(const HostChunk& c, const u64* lo, const u64* vals, const u8* kinds, const u8* dOut, cudaStream_t s,
                          u8* hOut, size_t outCapacity, size_t* hOffsets, size_t* hCSizes, unsigned char* hKinds, u64& total)
{
    size_t const cb = c.b1 - c.b0;
    u64 end = 0;
    for (size_t b = 0; b < cb; b++) {
        u64 const off = total + lo[b], len = lo[b + 1] - lo[b];
        u64 v = vals[b];
        bool const stores = kinds ? kinds[b] != 4 : !is_err(v);
        bool const over = stores && off + len > outCapacity;
        if (over) v = err(E_DST_TOO_SMALL);
        else if (stores && len) end = lo[b + 1];
        hOffsets[c.b0 + b] = (size_t)off; hCSizes[c.b0 + b] = (size_t)v;
        if (hKinds) hKinds[c.b0 + b] = over ? 4 : kinds[b];
    }
    u8* const at = hOut + total;
    total += lo[cb];
    return end ? cudaMemcpyAsync(at, dOut, end, cudaMemcpyDeviceToHost, s) : cudaSuccess;
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
    size_t const words = PackedWords(most.blocks).end;
    cudaError_t e = P.ensure(most.bytes, most.bytes, maxW, words, words);
    u64 total = 0;                                                  // global offset of the next chunk's first block
    // queue: the source and the descriptors up, the packed call with room for every block, offsets and values down
    auto queue = [&](size_t ci, int k) -> cudaError_t {
        PackedWords const L(chunks[ci].b1 - chunks[ci].b0);
        cudaError_t const r = queue_packed_compress(P, k, chunks[ci], codec, hSrc, hSrcSizes, maxSymbolValue, tableLog);
        if (r != cudaSuccess) return r;
        return cudaMemcpyAsync(P.hD[k] + L.offset, P.dD[k] + L.offset, (L.end - L.offset) * sizeof(u64), cudaMemcpyDeviceToHost, P.st[k]);
    };
    // finish: global offsets, the capacity rule of one call over the whole batch, and the stored bytes -- a prefix of the chunk's
    // packed bytes, since the blocks that fit come first -- copied down
    auto finish = [&](size_t ci, int k) -> cudaError_t {
        PackedWords const L(chunks[ci].b1 - chunks[ci].b0);
        cudaError_t const r = cudaStreamSynchronize(P.st[k]);
        if (r != cudaSuccess) return r;
        return finish_packed(chunks[ci], P.hD[k] + L.offset, P.hD[k] + L.value, nullptr, P.dB[k], P.st[k], (u8*)hOut, outCapacity,
                             hOffsets, hCSizes, nullptr, total);
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
    size_t const words = PackedWords(most.blocks).end;
    cudaError_t e = P.ensure(most.bytes, most.packed, 0, words, words);
    // queue: the chunk's packed bytes and descriptors up (offsets rebased to the chunk), the packed decompress, the blocks and
    // their results down
    auto queue = [&](size_t ci, int k) -> cudaError_t {
        const HostChunk& c = chunks[ci];
        size_t const cb = c.b1 - c.b0;
        PackedWords const L(cb);
        u64 const in0 = hOffsets[c.b0], in = hOffsets[c.b1] - in0, bytes = c.a1 - c.a0;
        cudaStream_t const s = P.st[k];
        u64* const h = P.hD[k];
        u64* const d = P.dD[k];
        for (size_t b = 0, a = 0; b < cb; b++) { h[L.ptr + b] = reinterpret_cast<u64>(P.dA[k] + a); h[L.size + b] = hDstSizes[c.b0 + b]; a += unit * hDstSizes[c.b0 + b]; }
        for (size_t b = 0; b <= cb; b++) h[L.offset + b] = hOffsets[c.b0 + b] - in0;
        cudaError_t r;
        if (in && (r = cudaMemcpyAsync(P.dB[k], (const u8*)hIn + in0, in, cudaMemcpyHostToDevice, s)) != cudaSuccess) return r;
        if ((r = cudaMemcpyAsync(d, h, L.value * sizeof(u64), cudaMemcpyHostToDevice, s)) != cudaSuccess) return r;
        u8* const* const dsts = (u8* const*)(d + L.ptr);
        u64* const vals = d + L.value;
        r = fse ? launch_fse_decompress_packed(dsts, d + L.size, vals, P.dB[k], d + L.offset, (u32)cb, wide, s)
                : launch_huf_decompress_packed(dsts, d + L.size, vals, P.dB[k], d + L.offset, (u32)cb, codec == 1 ? 4 : 1, s);
        if (r != cudaSuccess) return r;
        if (bytes && (r = cudaMemcpyAsync((u8*)hDst + c.a0, P.dA[k], bytes, cudaMemcpyDeviceToHost, s)) != cudaSuccess) return r;
        return cudaMemcpyAsync(h + L.value, vals, (L.end - L.value) * sizeof(u64), cudaMemcpyDeviceToHost, s);
    };
    // finish: the results of the chunk, once its stream is done; it runs before the chunk's stream and pinned image take the
    // next chunk
    auto finish = [&](size_t ci, int k) -> cudaError_t {
        PackedWords const L(chunks[ci].b1 - chunks[ci].b0);
        cudaError_t const r = cudaStreamSynchronize(P.st[k]);
        if (r == cudaSuccess) std::memcpy(hResults + chunks[ci].b0, P.hD[k] + L.value, (L.end - L.value) * sizeof(u64));
        return r;
    };
    if (e == cudaSuccess) e = run_chunks(P, chunks.size(), P.NS, queue, finish);
    return e == cudaSuccess ? 0 : (size_t)err(E_GENERIC);
}

// ================================================================================================
// packed chains of table reuse on HOST buffers: FSEB200_HUF_compress{4X,1X}_repeat_chains_packed and
// FSEB200_HUF_decompress{4X,1X}_repeat_packed through the packed pair's ring and chunk budget, chain boundaries ignored; each
// chunk runs the device call's helper (capi_common.h huf_repeat_chains_packed, huf_repeat_unpack) unchanged on chunk-local
// geometry.  Chains are contiguous ranges of blocks, so the chains that meet a chunk are a contiguous range of which only the
// first can have started in an earlier chunk: at most one chain crosses each chunk boundary, and its state (compress) or its last
// tree header (decompress) is all that passes from chunk to chunk.  codec: 1 = Huff0 4X, 3 = Huff0 1X; the mixed pair (a form
// per block, hSingleStream) and the literal-policy compress (the forms an output) run the same code with their own ChainForm.
// ================================================================================================
namespace {
// The most of a tree header a Huff0 decoder reads (HUF_readStats: 1 + 127 bytes in the FSE form, 1 + 64 raw); a header's size
// enters its verdict only through iSize + 1 > size, so a longer one is passed as its first HDR_MAX bytes with the same verdicts.
constexpr u64 HDR_MAX = 128;
constexpr size_t NONE = SIZE_MAX;

// start[0] == 0, start[nChains] == nBlocks, never decreasing: the device calls' geometry check
bool chains_sound(const size_t* start, size_t nChains, size_t nBlocks)
{
    if (start[0] != 0 || start[nChains] != nBlocks) return false;
    for (size_t c = 0; c < nChains; c++) if (start[c + 1] < start[c]) return false;
    return true;
}

// The chains [c0, c0 + n) that chunk c meets (sound geometry): c0 holds block b0, i.e. it is the last chain whose start is <= b0,
// as the decoder assigns blocks, and the last holds b1 - 1.  Their chunk-local starts are start - b0 clamped at 0, then cb.
struct ChunkChains {
    size_t c0, n;
    ChunkChains(const size_t* start, size_t nChains, const HostChunk& c)
    {
        auto holder = [&](size_t b) { return (size_t)(std::upper_bound(start, start + nChains + 1, b) - start) - 1; };
        c0 = holder(c.b0); n = holder(c.b1 - 1) - c0 + 1;
    }
    void local_starts(const size_t* start, const HostChunk& c, u64* out) const
    {
        for (size_t i = 0; i < n; i++) out[i] = std::max(start[c0 + i], c.b0) - c.b0;
        out[n] = c.b1 - c.b0;
    }
};

// The chain compress, for cb blocks and nc chunk-local chains: source pointers, sizes, prefer flags (two per word), chain starts
// (nc + 1) and, for the mixed call, the blocks' forms (eight per word) go up; offsets (cb + 1), values, kinds (eight per word) and,
// for the literal-policy call, the forms it chose come down.  The per-chain state views are ChainPool's at the chunk's first chain.
struct ChainCompressWords {
    size_t ptr = 0, size, prefer, start, single, offset, value, kind, singleOut, end;
    ChainCompressWords(size_t cb, size_t nc, bool mixed, bool lit) : size(cb), prefer(2 * cb), start(prefer + (cb + 1) / 2),
        single(start + nc + 1), offset(single + (mixed ? (cb + 7) / 8 : 0)), value(offset + cb + 1), kind(value + cb),
        singleOut(kind + (cb + 7) / 8), end(singleOut + (lit ? (cb + 7) / 8 : 0)) {}
};
// The chain decompress, for cb blocks, nc chunk-local chains and ne entry headers: destination pointers, sizes, offsets (cb + 1),
// kinds, chain starts, the chains' entry header pointers and sizes, ne header images of HDR_MAX bytes with a 32-byte sector of
// slack behind them (the decoder reads whole sectors) and, for the mixed call, the blocks' forms go up; values come down.
struct ChainDecompressWords {
    size_t ptr = 0, size, offset, kind, start, hdr, hdrSize, hdrBytes, single, value, end;
    ChainDecompressWords(size_t cb, size_t nc, size_t ne, bool mixed) : size(cb), offset(2 * cb), kind(3 * cb + 1), start(kind + (cb + 7) / 8),
        hdr(start + nc + 1), hdrSize(hdr + nc), hdrBytes(hdrSize + nc), single(hdrBytes + ne * (HDR_MAX / 8) + 4),
        value(single + (mixed ? (cb + 7) / 8 : 0)), end(value + cb) {}
};

// A compress call's per-chain state on the device, in u64 words for nChains chains: the tables (256 cells, 1 KiB each), pointers
// to them, the flags (two per word), the header pointers and the header sizes.  The device calls only carry a header pointer,
// so those go up as 0, and the host derives the exit headers from the kinds.  `h` is its pinned host image: 32,768 chains take
// 32 MiB each way, which pageable memory would copy at a fraction of the PCIe rate.  Grow-only, per device, used under the packed
// ring's mutex.
struct ChainPool {
    struct Layout {
        size_t table = 0, tptr, flag, hdr, hdrSize, end;
        explicit Layout(size_t n) : tptr(128 * n), flag(129 * n), hdr(flag + (n + 1) / 2), hdrSize(hdr + n), end(hdrSize + n) {}
    };
    u64* d = nullptr;
    u64* h = nullptr;
    size_t cap = 0;
    cudaError_t ensure(size_t words)
    {
        if (words <= cap) return cudaSuccess;
        cudaError_t e = cudaSuccess;
        if (d) e = cudaFree(d);
        if (h && e == cudaSuccess) e = cudaFreeHost(h);
        d = nullptr; h = nullptr; cap = 0;
        if (e == cudaSuccess) e = cudaMalloc((void**)&d, words * sizeof(u64));
        if (e == cudaSuccess) e = cudaMallocHost((void**)&h, words * sizeof(u64));
        if (e == cudaSuccess) cap = words;
        return e;
    }
};
ChainPool& chain_pool() { static ChainPool p[MAX_DEVICES]; return p[current_device()]; }

// one event per ring stream: chunk ci's chain call waits for chunk ci - 1's
template <int NS>
struct ChunkEvents {
    cudaEvent_t ev[NS] = {};
    cudaError_t create()
    {
        cudaError_t e = cudaSuccess;
        for (int i = 0; i < NS && e == cudaSuccess; i++) e = cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming);
        return e;
    }
    ~ChunkEvents() { for (cudaEvent_t x : ev) if (x) cudaEventDestroy(x); }
};

// the header a chunk-local chain enters a decompress chunk with: `n` bytes at `p`
struct EntryHeader { size_t chain; const u8* p; u64 n; };
}

namespace {
// `form` is the device call's; its dSingleStream is set per chunk to the device copy of hSingle, the blocks' forms -- read
// (nStreams 0) or, under the literal policy, written
size_t host_chains_compress(const ChainForm& form, size_t nChains, const size_t* hChainStarts, size_t nBlocks, void* hOut,
                            size_t outCapacity, size_t* hOffsets, size_t* hCSizes, unsigned char* hKinds, const void* hSrc,
                            const size_t* hSrcSizes, const int* hPreferRepeat, unsigned char* hSingle, unsigned* const* hCTables,
                            int* hRepeats, const void** hChainHeaders, size_t* hChainHeaderSizes, unsigned maxSymbolValue,
                            unsigned tableLog)
{
    bool const lit = form.literals, mixed = !form.nStreams && !lit;
    if (nBlocks > 0xFFFFFFFFull || nChains > 0xFFFFFFFFull) return (size_t)err(E_SRC_WRONG);
    if (nBlocks == 0) return 0;
    if (!hChainStarts || !hOut || !hOffsets || !hCSizes || !hKinds || !hSrc || !hSrcSizes || !hPreferRepeat || !hCTables ||
        !hRepeats || !hChainHeaders || !hChainHeaderSizes || !forms_given(form.nStreams, hSingle) ||
        (lit && (form.minGainLog < 1 || form.minGainLog > 31))) return (size_t)err(E_SRC_WRONG);
    if (!chains_sound(hChainStarts, nChains, nBlocks)) {            // the device call's verdicts, and nothing else written
        for (size_t b = 0; b < nBlocks; b++) { hCSizes[b] = (size_t)err(E_SRC_WRONG); hKinds[b] = 4; }
        return 0;
    }
    ChunkMax most;
    std::vector<HostChunk> const chunks = cut_chunks(hSrcSizes, nBlocks, 1, [](size_t) { return (u64)0; }, most);
    std::vector<ChunkChains> cc;
    size_t words = 0;
    for (const HostChunk& c : chunks) {
        cc.emplace_back(hChainStarts, nChains, c);
        words = std::max(words, ChainCompressWords(c.b1 - c.b0, cc.back().n, mixed, lit).end);
    }
    auto& P = packed_ring();
    std::lock_guard<std::mutex> lock(P.mu);
    ChainPool& S = chain_pool();
    ChainPool::Layout const SL(nChains);
    ChunkEvents<Ring<3>::NS> ev;
    cudaError_t e = P.ensure(most.bytes, most.bytes, 0, words, words);
    if (e == cudaSuccess) e = S.ensure(SL.end);
    if (e == cudaSuccess) e = ev.create();
    // the caller's state up once, on the first chunk's stream, through the pool's pinned image, which also takes it back down
    u64* const img = S.h;
    int* const flags = reinterpret_cast<int*>(img + SL.flag);
    if (e == cudaSuccess) {
        std::fill(img + SL.flag, img + SL.end, (u64)0);
        for (size_t c = 0; c < nChains; c++) {
            std::memcpy(img + SL.table + 128 * c, hCTables[c], 1024);
            img[SL.tptr + c] = reinterpret_cast<u64>(S.d + SL.table + 128 * c);
            flags[c] = hRepeats[c];
            img[SL.hdrSize + c] = hChainHeaderSizes[c];
        }
        e = cudaMemcpyAsync(S.d, img, SL.end * sizeof(u64), cudaMemcpyHostToDevice, P.st[0]);
    }
    // queue: the source and the descriptors up, then -- once chunk ci - 1's call has left the crossing chain's state -- the
    // device call with room for every block on views of the state at the chunk's first chain, then offsets, values, kinds down
    auto queue = [&](size_t ci, int k) -> cudaError_t {
        const HostChunk& c = chunks[ci];
        size_t const cb = c.b1 - c.b0, c0 = cc[ci].c0;
        ChainCompressWords const L(cb, cc[ci].n, mixed, lit);
        u64 const bytes = c.a1 - c.a0;
        cudaStream_t const s = P.st[k];
        u64* const h = P.hD[k], * const d = P.dD[k];
        for (size_t b = 0, a = 0; b < cb; b++) { h[L.ptr + b] = reinterpret_cast<u64>(P.dA[k] + a); h[L.size + b] = hSrcSizes[c.b0 + b]; a += hSrcSizes[c.b0 + b]; }
        std::memcpy(h + L.prefer, hPreferRepeat + c.b0, cb * sizeof(int));
        cc[ci].local_starts(hChainStarts, c, h + L.start);
        if (mixed) std::memcpy(h + L.single, hSingle + c.b0, cb);
        cudaError_t r;
        if (bytes && (r = cudaMemcpyAsync(P.dA[k], (const u8*)hSrc + c.a0, bytes, cudaMemcpyHostToDevice, s)) != cudaSuccess) return r;
        if ((r = cudaMemcpyAsync(d, h, L.offset * sizeof(u64), cudaMemcpyHostToDevice, s)) != cudaSuccess) return r;
        if (ci && (r = cudaStreamWaitEvent(s, ev.ev[(ci - 1) % P.NS], 0)) != cudaSuccess) return r;
        ChainForm f = form;
        if (!f.nStreams) f.dSingleStream = (unsigned char*)(d + (lit ? L.singleOut : L.single));
        size_t const v = huf_repeat_chains_packed(
            cc[ci].n, (const size_t*)(d + L.start), cb, P.dB[k], bytes, (size_t*)(d + L.offset), (size_t*)(d + L.value),
            (unsigned char*)(d + L.kind), (const void* const*)(d + L.ptr), (const size_t*)(d + L.size), (const int*)(d + L.prefer),
            (unsigned* const*)(S.d + SL.tptr) + c0, (int*)(S.d + SL.flag) + c0, (const void**)(S.d + SL.hdr) + c0,
            (size_t*)(S.d + SL.hdrSize) + c0, f, maxSymbolValue, tableLog, s);
        if (v) return cudaErrorLaunchFailure;
        if ((r = cudaEventRecord(ev.ev[k], s)) != cudaSuccess) return r;
        return cudaMemcpyAsync(h + L.offset, d + L.offset, (L.end - L.offset) * sizeof(u64), cudaMemcpyDeviceToHost, s);
    };
    u64 total = 0;
    auto finish = [&](size_t ci, int k) -> cudaError_t {
        ChainCompressWords const L(chunks[ci].b1 - chunks[ci].b0, cc[ci].n, mixed, lit);
        cudaError_t const r = cudaStreamSynchronize(P.st[k]);
        if (r != cudaSuccess) return r;
        if (lit) std::memcpy(hSingle + chunks[ci].b0, P.hD[k] + L.singleOut, chunks[ci].b1 - chunks[ci].b0);
        return finish_packed(chunks[ci], P.hD[k] + L.offset, P.hD[k] + L.value, (const u8*)(P.hD[k] + L.kind), P.dB[k], P.st[k],
                             (u8*)hOut, outCapacity, hOffsets, hCSizes, hKinds, total);
    };
    if (e == cudaSuccess) e = run_chunks(P, chunks.size(), P.NS - 1, queue, finish);
    bool const fits = total <= outCapacity;
    if (e == cudaSuccess && fits) e = cudaMemcpy(img, S.d, SL.hdr * sizeof(u64), cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) return (size_t)err(E_GENERIC);
    hOffsets[nBlocks] = (size_t)total;
    // the state goes back only if the whole stream fits: the tables and flags the calls left, and the header of each chain's
    // last kind-2 block, at its place in hOut, or the one it came in with
    if (fits)
        for (size_t c = 0; c < nChains; c++) {
            std::memcpy(hCTables[c], img + SL.table + 128 * c, 1024);
            hRepeats[c] = flags[c];
            for (size_t j = hChainStarts[c + 1]; j-- > hChainStarts[c];)
                if (hKinds[j] == 2) { hChainHeaders[c] = (const u8*)hOut + hOffsets[j]; hChainHeaderSizes[c] = hCSizes[j]; break; }
        }
    return 0;
}

// nStreams 4 (4X), 1 (1X) or 0 (mixed: the form of block b from hSingle[b])
size_t host_chains_decompress(int nStreams, size_t nChains, const size_t* hChainStarts, size_t nBlocks, void* hDst, const size_t* hDstSizes,
                              size_t* hResults, const void* hIn, const size_t* hOffsets, const unsigned char* hKinds,
                              const unsigned char* hSingle, const void* const* hChainHeaders, const size_t* hChainHeaderSizes)
{
    bool const mixed = nStreams == 0;
    if (nBlocks > 0xFFFFFFFFull || nChains > 0xFFFFFFFFull) return (size_t)err(E_SRC_WRONG);
    if (nBlocks == 0) return 0;
    if (!hChainStarts || !hDst || !hDstSizes || !hResults || !hIn || !hOffsets || !hKinds || !hChainHeaders || !hChainHeaderSizes ||
        !forms_given(nStreams, hSingle)) return (size_t)err(E_SRC_WRONG);
    for (size_t b = 0; b < nBlocks; b++) if (hOffsets[b + 1] < hOffsets[b]) return (size_t)err(E_SRC_WRONG);
    if (!chains_sound(hChainStarts, nChains, nBlocks)) {            // the device call's verdicts, and nothing else written
        for (size_t b = 0; b < nBlocks; b++) hResults[b] = (size_t)err(E_SRC_WRONG);
        return 0;
    }
    ChunkMax most;
    std::vector<HostChunk> const chunks = cut_chunks(hDstSizes, nBlocks, 1, [&](size_t b) { return (u64)(hOffsets[b + 1] - hOffsets[b]); }, most);
    // The device decoder finds a kind-3 block's header in its chunk when a kind-2 block of its chain precedes it there.  Otherwise
    // the chain's entry header is supplied: the chain's last kind-2 block before the chunk, or the caller's.  One walk over the
    // blocks, with the chain that holds each block and that chain's last kind-2 block so far.
    std::vector<ChunkChains> cc;
    std::vector<std::vector<EntryHeader>> entries(chunks.size());
    size_t words = 0;
    for (size_t ci = 0, ch = 0, last2 = NONE; ci < chunks.size(); ci++) {
        const HostChunk& c = chunks[ci];
        cc.emplace_back(hChainStarts, nChains, c);
        bool seen = false;                                          // chain ch has a kind-2 or kind-3 block in this chunk before b
        for (size_t b = c.b0; b < c.b1; b++) {
            while (hChainStarts[ch + 1] <= b) { ch++; last2 = NONE; seen = false; }
            unsigned char const k = hKinds[b];
            if (k == 3 && !seen)
                entries[ci].push_back(last2 != NONE ? EntryHeader{ ch - cc[ci].c0, (const u8*)hIn + hOffsets[last2], hOffsets[last2 + 1] - hOffsets[last2] }
                                                    : EntryHeader{ ch - cc[ci].c0, (const u8*)hChainHeaders[ch], hChainHeaderSizes[ch] });
            seen |= k == 2 || k == 3;
            if (k == 2) last2 = b;
        }
        words = std::max(words, ChainDecompressWords(c.b1 - c.b0, cc[ci].n, entries[ci].size(), mixed).end);
    }
    auto& P = packed_ring();
    std::lock_guard<std::mutex> lock(P.mu);
    cudaError_t e = P.ensure(most.bytes, most.packed, 0, words, words);
    // queue: the chunk's packed bytes and descriptors up (offsets rebased to the chunk, entry headers as images of at most HDR_MAX
    // bytes), the device decompress, the blocks and their values down
    auto queue = [&](size_t ci, int k) -> cudaError_t {
        const HostChunk& c = chunks[ci];
        size_t const cb = c.b1 - c.b0;
        ChainDecompressWords const L(cb, cc[ci].n, entries[ci].size(), mixed);
        u64 const in0 = hOffsets[c.b0], in = hOffsets[c.b1] - in0, bytes = c.a1 - c.a0;
        cudaStream_t const s = P.st[k];
        u64* const h = P.hD[k], * const d = P.dD[k];
        for (size_t b = 0, a = 0; b < cb; b++) { h[L.ptr + b] = reinterpret_cast<u64>(P.dA[k] + a); h[L.size + b] = hDstSizes[c.b0 + b]; a += hDstSizes[c.b0 + b]; }
        for (size_t b = 0; b <= cb; b++) h[L.offset + b] = hOffsets[c.b0 + b] - in0;
        std::memcpy(h + L.kind, hKinds + c.b0, cb);
        cc[ci].local_starts(hChainStarts, c, h + L.start);
        std::fill(h + L.hdr, h + L.hdrBytes, (u64)0);
        for (size_t j = 0; j < entries[ci].size(); j++) {
            const EntryHeader& x = entries[ci][j];
            u64 const n = std::min(x.n, HDR_MAX);
            if (n) std::memcpy((u8*)(h + L.hdrBytes) + j * HDR_MAX, x.p, n);
            h[L.hdr + x.chain] = reinterpret_cast<u64>((u8*)(d + L.hdrBytes) + j * HDR_MAX); h[L.hdrSize + x.chain] = n;
        }
        if (mixed) std::memcpy(h + L.single, hSingle + c.b0, cb);
        cudaError_t r;
        if (in && (r = cudaMemcpyAsync(P.dB[k], (const u8*)hIn + in0, in, cudaMemcpyHostToDevice, s)) != cudaSuccess) return r;
        if ((r = cudaMemcpyAsync(d, h, L.value * sizeof(u64), cudaMemcpyHostToDevice, s)) != cudaSuccess) return r;
        size_t const v = huf_repeat_unpack(
            cc[ci].n, (const size_t*)(d + L.start), cb, (void* const*)(d + L.ptr), (const size_t*)(d + L.size), (size_t*)(d + L.value),
            P.dB[k], (const size_t*)(d + L.offset), (const unsigned char*)(d + L.kind), (const void* const*)(d + L.hdr),
            (const size_t*)(d + L.hdrSize), nStreams, s, mixed ? (const unsigned char*)(d + L.single) : nullptr);
        if (v) return cudaErrorLaunchFailure;
        if (bytes && (r = cudaMemcpyAsync((u8*)hDst + c.a0, P.dA[k], bytes, cudaMemcpyDeviceToHost, s)) != cudaSuccess) return r;
        return cudaMemcpyAsync(h + L.value, d + L.value, cb * sizeof(u64), cudaMemcpyDeviceToHost, s);
    };
    auto finish = [&](size_t ci, int k) -> cudaError_t {
        const HostChunk& c = chunks[ci];
        ChainDecompressWords const L(c.b1 - c.b0, cc[ci].n, entries[ci].size(), mixed);
        cudaError_t const r = cudaStreamSynchronize(P.st[k]);
        if (r == cudaSuccess) std::memcpy(hResults + c.b0, P.hD[k] + L.value, (c.b1 - c.b0) * sizeof(u64));
        return r;
    };
    if (e == cudaSuccess) e = run_chunks(P, chunks.size(), P.NS, queue, finish);
    return e == cudaSuccess ? 0 : (size_t)err(E_GENERIC);
}
}  // namespace

FSEB_API size_t FSEB200_compress_host_repeat_chains_packed(int codec, size_t nChains, const size_t* hChainStarts, size_t nBlocks,
                                                           void* hOut, size_t outCapacity, size_t* hOffsets, size_t* hCSizes,
                                                           unsigned char* hKinds, const void* hSrc, const size_t* hSrcSizes,
                                                           const int* hPreferRepeat, unsigned* const* hCTables, int* hRepeats,
                                                           const void** hChainHeaders, size_t* hChainHeaderSizes,
                                                           unsigned maxSymbolValue, unsigned tableLog)
{
    if (codec != 1 && codec != 3) return (size_t)err(E_SRC_WRONG);
    return host_chains_compress(ChainForm{codec == 1 ? 4 : 1}, nChains, hChainStarts, nBlocks, hOut, outCapacity, hOffsets, hCSizes,
                                hKinds, hSrc, hSrcSizes, hPreferRepeat, nullptr, hCTables, hRepeats, hChainHeaders, hChainHeaderSizes,
                                maxSymbolValue, tableLog);
}
FSEB_API size_t FSEB200_decompress_host_repeat_packed(int codec, size_t nChains, const size_t* hChainStarts, size_t nBlocks,
                                                      void* hDst, const size_t* hDstSizes, size_t* hResults,
                                                      const void* hIn, const size_t* hOffsets, const unsigned char* hKinds,
                                                      const void* const* hChainHeaders, const size_t* hChainHeaderSizes)
{
    if (codec != 1 && codec != 3) return (size_t)err(E_SRC_WRONG);
    return host_chains_decompress(codec == 1 ? 4 : 1, nChains, hChainStarts, nBlocks, hDst, hDstSizes, hResults, hIn, hOffsets, hKinds,
                                  nullptr, hChainHeaders, hChainHeaderSizes);
}
FSEB_API size_t FSEB200_compress_host_mixed_repeat_chains_packed(size_t nChains, const size_t* hChainStarts, size_t nBlocks,
                                                                 void* hOut, size_t outCapacity, size_t* hOffsets, size_t* hCSizes,
                                                                 unsigned char* hKinds, const void* hSrc, const size_t* hSrcSizes,
                                                                 const int* hPreferRepeat, const unsigned char* hSingleStream,
                                                                 unsigned* const* hCTables, int* hRepeats, const void** hChainHeaders,
                                                                 size_t* hChainHeaderSizes, unsigned maxSymbolValue, unsigned tableLog)
{
    return host_chains_compress(ChainForm{0}, nChains, hChainStarts, nBlocks, hOut, outCapacity, hOffsets, hCSizes, hKinds, hSrc,
                                hSrcSizes, hPreferRepeat, const_cast<unsigned char*>(hSingleStream), hCTables, hRepeats, hChainHeaders,
                                hChainHeaderSizes, maxSymbolValue, tableLog);
}
FSEB_API size_t FSEB200_compress_host_literals_chains_packed(size_t nChains, const size_t* hChainStarts, size_t nBlocks,
                                                             void* hOut, size_t outCapacity, size_t* hOffsets, size_t* hCSizes,
                                                             unsigned char* hKinds, const void* hSrc, const size_t* hSrcSizes,
                                                             const int* hPreferRepeat, unsigned char* hSingleStream,
                                                             unsigned* const* hCTables, int* hRepeats, const void** hChainHeaders,
                                                             size_t* hChainHeaderSizes, unsigned maxSymbolValue, unsigned tableLog,
                                                             unsigned minLiterals, unsigned minGainLog)
{
    return host_chains_compress(ChainForm{0, nullptr, true, minLiterals, minGainLog}, nChains, hChainStarts, nBlocks, hOut, outCapacity,
                                hOffsets, hCSizes, hKinds, hSrc, hSrcSizes, hPreferRepeat, hSingleStream, hCTables, hRepeats,
                                hChainHeaders, hChainHeaderSizes, maxSymbolValue, tableLog);
}
FSEB_API size_t FSEB200_decompress_host_mixed_repeat_packed(size_t nChains, const size_t* hChainStarts, size_t nBlocks, void* hDst,
                                                            const size_t* hDstSizes, size_t* hResults, const void* hIn,
                                                            const size_t* hOffsets, const unsigned char* hKinds,
                                                            const unsigned char* hSingleStream, const void* const* hChainHeaders,
                                                            const size_t* hChainHeaderSizes)
{
    return host_chains_decompress(0, nChains, hChainStarts, nBlocks, hDst, hDstSizes, hResults, hIn, hOffsets, hKinds, hSingleStream,
                                  hChainHeaders, hChainHeaderSizes);
}

// ================================================================================================
// frames: the .fse format of the reference's file tool (programs/fileio.c:266-626) on host buffers, many frames per call (the
// one-frame calls are batches of one), through the packed pair's ring and chunk budget; DESIGN 5b describes the pipeline.
// ================================================================================================
namespace {
using namespace fmt;

// Frames of at most this many bytes that lie in one chunk are hashed on the device, the rest on host threads.  One frame is a
// serial chain on either side, slower on the device than on a host core, so the device wins while a chunk holds many frames to
// hash side by side.  Set at the measured crossover (DESIGN 5b: batches of 64 KiB to 16 MiB frames, each placement alone):
// the device is faster up to 1 MiB, the host from 4 MiB, and at 2 MiB each wins one direction.
constexpr u64 DEVICE_HASH_MAX = 1ull << 20;

void put_trailer(u8* t, u32 hash)
{
    u32 const crc = trailer_checksum(hash);
    t[0] = (u8)((crc >> 16) | (BT_END << 6)); t[1] = (u8)(crc >> 8); t[2] = (u8)crc;
}
u64 block_header_len(u64 v, u64 n, u64 bs) { return 1 + (n == bs ? 0 : 2) + (v >= 2 ? 2 : 0); }

struct FrameWalk {
    size_t verdict = 0;             // 0, or the verdict where the walk stopped (the point FIO_decompressFilename stops at)
    int codec = 0;                  // 0 FSE, 1 Huff0
    std::vector<FrameBlock> blocks; // every block before that point
    u32 checksum = 0;               // the trailer's 22 bits (verdict 0)
};

// the reference's header walk, with its exit codes as verdicts (frame_walk.h)
FrameWalk walk_frame(const u8* f, u64 size)
{
    FrameWalk w;
    WalkState s;
    FrameBlock k;
    u64 r;
    while ((r = walk_step(f, size, s, k)) == WALK_BLOCK) w.blocks.push_back(k);
    if (r != WALK_END) w.verdict = (size_t)r;
    w.codec = s.codec; w.checksum = s.checksum;
    return w;
}

// Device-to-host copies of one chunk, merged while both sides stay contiguous
struct CopyRun {
    cudaStream_t s; const u8* dev = nullptr; u8* host = nullptr; u64 n = 0;
    cudaError_t add(const u8* d, u8* h, u64 len)
    {
        if (!len || (n && dev + n == d && host + n == h)) { n += len; return cudaSuccess; }
        cudaError_t const r = flush();
        dev = d; host = h; n = len;
        return r;
    }
    cudaError_t flush() { cudaError_t const r = n ? cudaMemcpyAsync(host, dev, n, cudaMemcpyDeviceToHost, s) : cudaSuccess; n = 0; return r; }
};

// A batch of frames as a batch of blocks, as both frame directions run it: frame f's blocks are [fb[f], fb[f + 1]), block b has
// bytes[b] uncompressed bytes, and onDevice[f] says frame f's checksum comes from xxh32_kernel, nHashed[ci] of them in chunk ci.
struct FramePlan {
    std::vector<size_t> fb, bytes, hostFrames;                      // hostFrames: those hashed on host threads, in frame order
    std::vector<u32> frameOf, nHashed;
    std::vector<char> onDevice;
    std::vector<HostChunk> chunks; ChunkMax most;
};
struct FrameShape { size_t nBlocks; u64 hashLen; bool hashable; }; struct BlockShape { u64 bytes, stored; };

// frame(f): frame f's block count, the bytes its checksum covers, whether it has one; block(f, i): bytes and stored bytes.  A frame
// weighs its blocks' weights; it is hashed on the device if it covers at most DEVICE_HASH_MAX bytes and lies in one chunk.
template <class Frame, class Block>
FramePlan plan_frames(size_t nFrames, Frame frame, Block block)
{
    FramePlan p; p.fb.assign(nFrames + 1, 0);
    std::vector<FrameShape> shape(nFrames);
    for (size_t f = 0; f < nFrames; f++) { shape[f] = frame(f); p.fb[f + 1] = p.fb[f] + shape[f].nBlocks; }
    size_t const nb = p.fb[nFrames];
    p.frameOf.resize(nb); p.bytes.resize(nb);
    std::vector<u64> stored(nb), whole(nb, 0);                      // whole[b]: the weight of the frame that starts at block b
    for (size_t f = 0; f < nFrames; f++)
        for (size_t b = p.fb[f]; b < p.fb[f + 1]; b++) {
            BlockShape const k = block(f, b - p.fb[f]);
            p.frameOf[b] = (u32)f; p.bytes[b] = (size_t)k.bytes; stored[b] = k.stored;
            whole[p.fb[f]] += k.bytes + k.stored + BLOCK_OVERHEAD;
        }
    p.chunks = cut_chunks(p.bytes.data(), nb, 1, [&](size_t b) { return stored[b]; }, p.most, whole.data());
    p.onDevice.assign(nFrames, 0); p.nHashed.assign(p.chunks.size(), 0);
    for (size_t ci = 0; ci < p.chunks.size(); ci++)
        for (size_t b = p.chunks[ci].b0; b < p.chunks[ci].b1; b++) {
            size_t const f = p.frameOf[b];
            if (b != p.fb[f] || !shape[f].hashable) continue;
            p.onDevice[f] = shape[f].hashLen <= DEVICE_HASH_MAX && p.fb[f + 1] <= p.chunks[ci].b1;
            if (p.onDevice[f]) p.nHashed[ci]++;
            else p.hostFrames.push_back(f);
        }
    return p;
}

// XXH32 of `frames` on min(frames, cores) host threads, each taking frames in frame order and hashing a frame's pieces as fed,
// up to the one marked last.  join(), also the destructor's after a failure or an early stop, closes every frame and waits for
// the threads; digest(f) is read after it (a frame not among `frames`: the empty input's).
class HostHasher {
    struct Queue { std::vector<std::pair<const u8*, u64>> pieces; bool closed = false; std::condition_variable cv; };
    static constexpr size_t NONE = SIZE_MAX;
    std::vector<size_t> frames_, slot_;                             // slot_[f]: frame f's index in frames_, or NONE
    std::vector<Xxh32> state_;                                      // by slot
    std::vector<Queue> q_;
    std::mutex mu_;
    std::atomic<size_t> next_{0};
    std::vector<std::thread> threads_;
public:
    struct Piece { size_t f; const u8* p; u64 n; bool last; };
    HostHasher(size_t nFrames, const std::vector<size_t>& frames) : frames_(frames), slot_(nFrames, NONE), state_(frames.size()), q_(frames.size())
    {
        for (size_t j = 0; j < frames.size(); j++) slot_[frames[j]] = j;
        for (size_t i = 0; i < std::min(frames.size(), (size_t)std::max(1u, std::thread::hardware_concurrency())); i++)
            threads_.emplace_back([this] {
                for (size_t j; (j = next_++) < q_.size();)
                    for (std::vector<std::pair<const u8*, u64>> got;; got.clear()) {
                        {
                            std::unique_lock<std::mutex> lk(mu_);
                            q_[j].cv.wait(lk, [&] { return !q_[j].pieces.empty() || q_[j].closed; });
                            if (q_[j].pieces.empty()) break;
                            got.swap(q_[j].pieces);
                        }
                        for (const auto& x : got) state_[j].update(x.first, x.second);
                    }
            });
    }
    ~HostHasher() { join(); }
    void feed(const Piece& x)
    {
        assert(slot_[x.f] != NONE);                                 // only `frames` are fed
        Queue& q = q_[slot_[x.f]];
        { std::lock_guard<std::mutex> lk(mu_); if (x.n) q.pieces.push_back({ x.p, x.n }); q.closed |= x.last; }
        q.cv.notify_one();
    }
    void join() { for (size_t f : frames_) feed({ f, nullptr, 0, true }); for (std::thread& t : threads_) t.join(); threads_.clear(); }
    u32 digest(size_t f) const { return slot_[f] == NONE ? Xxh32().digest() : state_[slot_[f]].digest(); }
};

// A compress call's frames as they close in frame order: offsets, results under the capacity rule, empty-source frames written
struct FrameOutput {
    u8* out; size_t capacity; size_t* results;
    u8 empty[FRAME_HEADER + FRAME_TRAILER];                         // the frame of an empty source
    u64 total = 0;                                                  // offset of the next frame
    size_t closed = 0;                                              // frames [0, closed) have their offsets and results
    std::vector<char> stored;
    std::vector<u64> at;                                            // frame f's offset; at[nFrames]: the total
    FrameOutput(u8* o, size_t cap, size_t* res, size_t nFrames, u32 magic, unsigned blockSizeId)
        : out(o), capacity(cap), results(res), empty{ (u8)magic, (u8)(magic >> 8), (u8)(magic >> 16), (u8)(magic >> 24), (u8)blockSizeId },
          stored(nFrames, 0), at(nFrames + 1, 0) { put_trailer(empty + FRAME_HEADER, FSEB200_XXH32(nullptr, 0, 0)); }
    // frame f at `total` with `len` bytes or a verdict
    void close(size_t f, u64 len, size_t verdict)
    {
        at[f] = total; closed = f + 1;
        if (verdict) { results[f] = verdict; return; }
        stored[f] = total + len <= capacity;
        results[f] = stored[f] ? (size_t)len : (size_t)err(E_DST_TOO_SMALL);
        total += len;
    }
    void close_empty_until(size_t f)                                // the frames without blocks in front of frame f
    {
        for (size_t g = closed; g < f; g++) {
            u64 const pos = total;
            close(g, FRAME_HEADER + FRAME_TRAILER, 0);
            if (stored[g]) std::memcpy(out + pos, empty, sizeof(empty));
        }
    }
};

// How a frame that spans chunks is written.  ONE_FRAME (the one-frame call, which promises only that nothing past the capacity
// is written): straight to its place while it fits, and the call stops once the frame fails.  BATCH: to its place if its
// compressBound fits from its offset, else to a host stage copied in once it closes and fits; the other frames go on.
enum class Spanning { ONE_FRAME, BATCH };

// Arguments checked by the callers.  Returns 0 or generic; hResults, hOffsets (NULL for ONE_FRAME) as the batch call's.
size_t frame_compress_batch(Spanning spanning, int codec, unsigned blockSizeId, size_t nFrames, u8* out, size_t outCapacity,
                            size_t* hOffsets, size_t* hResults, const u8* src, const size_t* hSrcSizes)
{
    u64 const bs = (u64)1024 << blockSizeId;
    FramePlan const p = plan_frames(nFrames, [&](size_t f) { return FrameShape{ (size_t)((hSrcSizes[f] + bs - 1) / bs), hSrcSizes[f], true }; },
                                    [&](size_t f, size_t i) { return BlockShape{ std::min(bs, hSrcSizes[f] - i * bs), 0 }; });
    std::vector<u64> fsrc(nFrames + 1, 0);                          // frame f's source offset
    for (size_t f = 0; f < nFrames; f++) fsrc[f + 1] = fsrc[f] + hSrcSizes[f];
    HostHasher hasher(nFrames, p.hostFrames);
    for (size_t f : p.hostFrames) hasher.feed({ f, src + fsrc[f], hSrcSizes[f], true });
    u32 const magic = codec ? MAGIC_HUF : MAGIC_FSE;
    FrameOutput o(out, outCapacity, hResults, nFrames, magic, blockSizeId);
    // The frame being built across chunks (one at a time spans chunks): bytes so far, verdict, and where its pieces go -- its
    // place, or a host stage (Spanning)
    struct { u64 len = 0; size_t verdict = 0; u8* to = nullptr; std::unique_ptr<u8[]> stage; } cur;
    size_t const nb = p.bytes.size(), lastFrame = nb ? p.frameOf[nb - 1] : 0;     // the last frame with blocks
    size_t stop = 0;                                                // the last frame has failed: nothing left to decide
    cudaError_t e = cudaSuccess;
    if (nb) {
        auto& P = packed_ring();
        std::lock_guard<std::mutex> lock(P.mu);
        // The bodies go to the source's buffer once it is coded and hashed: the stored blocks plus at most 5 block-header bytes
        // and 8 frame-header and trailer bytes per block.
        size_t maxW = 0, words = 0;
        for (size_t ci = 0; ci < p.chunks.size(); ci++) {
            const HostChunk& c = p.chunks[ci];
            if (codec == 0) maxW = std::max(maxW, FSEB200_FSE_packed_workspace(c.b1 - c.b0, c.a1 - c.a0));
            words = std::max(words, FrameCompressWords(c.b1 - c.b0, p.nHashed[ci]).end);
        }
        e = P.ensure(p.most.bytes + 13 * p.most.blocks, p.most.bytes, maxW, words, words);
        // queue: the packed compress, the hashes, the frame bodies, the offsets and values down
        auto queue = [&](size_t ci, int k) -> cudaError_t {
            const HostChunk& c = p.chunks[ci];
            size_t const cb = c.b1 - c.b0;
            FrameCompressWords const L(cb, p.nHashed[ci]);
            u64* const h = P.hD[k], * const d = P.dD[k];
            cudaError_t r = queue_packed_compress(P, k, c, codec, src, p.bytes.data(), 255, 11);
            if (r != cudaSuccess) return r;
            for (size_t b = c.b0, j = 0; b < c.b1; b++) {
                size_t const f = p.frameOf[b];
                bool const last = b + 1 == p.fb[f + 1], hashed = last && p.onDevice[f];
                h[L.role + b - c.b0] = (b == p.fb[f] ? ROLE_FIRST : 0) | (last ? ROLE_LAST : 0) | (hashed ? ROLE_HASHED | (u64)j << 32 : 0);
                if (hashed) { h[L.range + 2 * j] = fsrc[f] - c.a0; h[L.range + 2 * j + 1] = hSrcSizes[f]; j++; }
            }
            cudaStream_t const s = P.st[k];
            if ((r = cudaMemcpyAsync(d + L.role, h + L.role, (L.hash - L.role) * sizeof(u64), cudaMemcpyHostToDevice, s)) != cudaSuccess) return r;
            if ((r = launch_xxh32_ranges(P.dA[k], d + L.range, p.nHashed[ci], d + L.hash, s)) != cudaSuccess) return r;
            r = launch_frame_body(P.dA[k], P.dB[k], d + L.packed.offset, d + L.packed.value, d + L.packed.size, d + L.role, d + L.hash,
                                  (u32)cb, bs, magic, blockSizeId, s);
            if (r != cudaSuccess) return r;
            return cudaMemcpyAsync(h + L.packed.offset, d + L.packed.offset, (L.packed.end - L.packed.offset) * sizeof(u64), cudaMemcpyDeviceToHost, s);
        };
        // finish: each frame's length and verdict from its blocks' values (an error value makes it an error frame of length 0),
        // the capacity rule, and the stored frames' bytes down from the chunk's body -- a run of whole frames in one copy, the
        // piece of a spanning frame to where `cur` says
        auto finish = [&](size_t ci, int k) -> cudaError_t {
            const HostChunk& c = p.chunks[ci];
            FrameCompressWords const L(c.b1 - c.b0, p.nHashed[ci]);
            cudaError_t r = cudaStreamSynchronize(P.st[k]); if (r != cudaSuccess) return r;
            const u64* const lo = P.hD[k] + L.packed.offset, * const vals = P.hD[k] + L.packed.value;
            CopyRun run; run.s = P.st[k];
            u64 dpos = 0;                                           // the body offset of the next block
            for (size_t b = c.b0; b < c.b1 && r == cudaSuccess;) {
                size_t const f = p.frameOf[b], e1 = std::min(c.b1, p.fb[f + 1]);
                bool const first = b == p.fb[f], last = e1 == p.fb[f + 1], spans = !(first && last);
                if (first) {
                    o.close_empty_until(f);
                    cur.len = 0; cur.verdict = 0; cur.to = nullptr; cur.stage.reset();
                    size_t const bound = FSEB200_frame_compressBound(hSrcSizes[f], blockSizeId);
                    if (spans && (spanning == Spanning::ONE_FRAME || o.total + bound <= outCapacity)) cur.to = out + o.total;
                    else if (spans) { cur.stage.reset(new u8[bound]); cur.to = cur.stage.get(); }
                }
                u64 const d0 = dpos, pieceAt = cur.len;
                for (; b < e1; b++) {
                    u64 const v = vals[b - c.b0], len = lo[b - c.b0 + 1] - lo[b - c.b0];
                    u64 const n = (b == p.fb[f] ? FRAME_HEADER : 0) + (b + 1 == p.fb[f + 1] ? FRAME_TRAILER : 0) +
                                  (is_err(v) ? 0 : block_header_len(v, p.bytes[b], bs) + len);
                    dpos += n;
                    if (cur.verdict) continue;
                    if (is_err(v)) cur.verdict = (size_t)v;
                    else cur.len += n;
                }
                bool const over = spanning == Spanning::ONE_FRAME && o.total + cur.len > outCapacity;
                if (f == lastFrame && (cur.verdict || over)) { stop = 1; break; }
                if (spans && !cur.verdict) r = run.add(P.dA[k] + d0, cur.to + pieceAt, dpos - d0);
                if (!last) continue;
                u64 const frameAt = o.total;
                o.close(f, cur.len, cur.verdict);
                if (o.stored[f] && !spans) r = run.add(P.dA[k] + d0, out + frameAt, cur.len);
                if (cur.stage) {                                    // its pieces land before the stage is copied or freed
                    if (r == cudaSuccess) r = run.flush();
                    if (r == cudaSuccess) r = cudaStreamSynchronize(P.st[k]);
                    if (r != cudaSuccess) return r;
                    if (o.stored[f]) std::memcpy(out + frameAt, cur.stage.get(), cur.len);
                    cur.stage.reset();
                }
            }
            if (r == cudaSuccess) r = run.flush();
            return r;
        };
        if (e == cudaSuccess) e = run_chunks(P, p.chunks.size(), P.NS - 1, queue, finish, &stop);
    }
    hasher.join();
    if (e != cudaSuccess) return (size_t)err(E_GENERIC);
    if (stop) o.close(lastFrame, cur.len, cur.verdict ? cur.verdict : (size_t)err(E_DST_TOO_SMALL));
    o.close_empty_until(nFrames);
    o.at[nFrames] = o.total;
    if (hOffsets) std::copy(o.at.begin(), o.at.end(), hOffsets);
    for (size_t f : p.hostFrames) if (o.stored[f]) put_trailer(out + o.at[f] + hResults[f] - FRAME_TRAILER, hasher.digest(f));
    return 0;
}

// What each decompress chunk copies up: runs of its frames' bytes, unless 4 KiB or more of other bytes lie between (frames that do
// not run, long tails); srcOff[b], block b's header there; the largest chunk's bytes; its compressed blocks, nFse of FSE frames.
struct ChunkInputs {
    struct Run { u64 from, n, to; };
    std::vector<std::vector<Run>> runs; std::vector<u64> srcOff; u64 most = 0; std::vector<size_t> nCoded, nFse;
};
ChunkInputs chunk_inputs(const FramePlan& p, const std::vector<FrameWalk>& walks, const size_t* hOffsets)
{
    ChunkInputs c;
    c.runs.resize(p.chunks.size()); c.srcOff.resize(p.bytes.size()); c.nCoded.assign(p.chunks.size(), 0); c.nFse.assign(p.chunks.size(), 0);
    for (size_t ci = 0; ci < p.chunks.size(); ci++) {
        std::vector<ChunkInputs::Run>& R = c.runs[ci];
        for (size_t b = p.chunks[ci].b0; b < p.chunks[ci].b1; b++) {
            size_t const f = p.frameOf[b];
            const FrameBlock& k = walks[f].blocks[b - p.fb[f]];
            u64 const a = hOffsets[f] + k.head, z = hOffsets[f] + k.payload + k.cSize;
            if (R.empty() || a >= R.back().from + R.back().n + 4096) R.push_back({ a, 0, R.empty() ? 0 : R.back().to + R.back().n });
            R.back().n = z - R.back().from;
            c.srcOff[b] = R.back().to + (a - R.back().from);
            c.nCoded[ci] += k.type == BT_COMPRESSED;
            c.nFse[ci] += k.type == BT_COMPRESSED && walks[f].codec == 0;
        }
        if (!R.empty()) c.most = std::max(c.most, R.back().to + R.back().n);
    }
    return c;
}

// Arguments checked by the callers; offsets non-decreasing.  Returns 0 or generic; hResults as FSEB200_frame_decompress_host_batch.
size_t frame_decompress_batch(size_t nFrames, u8* dst, const size_t* caps, size_t* hResults, const u8* in, const size_t* hOffsets)
{
    std::vector<FrameWalk> walks(nFrames);
    std::vector<u64> region(nFrames + 1, 0);                        // frame f's output region starts at dst + region[f]
    std::vector<u64> nominal(nFrames, 0);
    std::vector<size_t> verdict(nFrames, 0);                        // a decoder error or overflow, in block order
    for (size_t f = 0; f < nFrames; f++) {
        FrameWalk& w = walks[f] = walk_frame(in + hOffsets[f], hOffsets[f + 1] - hOffsets[f]);
        region[f + 1] = region[f] + caps[f];
        bool coded = false;
        for (const FrameBlock& k : w.blocks) { nominal[f] += k.rSize; coded |= k.type == BT_COMPRESSED; }
        // every block's output size is known: settled here first, as the single call does, and none of its blocks runs
        if (!coded && nominal[f] > caps[f]) verdict[f] = (size_t)err(E_DST_TOO_SMALL);
        if (!coded && (nominal[f] > caps[f] || w.verdict)) w.blocks.clear();
    }
    FramePlan const p = plan_frames(nFrames, [&](size_t f) { return FrameShape{ walks[f].blocks.size(), nominal[f], !walks[f].verdict }; },
                                    [&](size_t f, size_t i) { const FrameBlock& k = walks[f].blocks[i]; return BlockShape{ k.rSize, k.payload + k.cSize - k.head }; });
    size_t const nb = p.bytes.size();
    auto blk = [&](size_t b) -> const FrameBlock& { return walks[p.frameOf[b]].blocks[b - p.fb[p.frameOf[b]]]; };
    ChunkInputs const up = chunk_inputs(p, walks, hOffsets);
    auto layout = [&](size_t ci) { return FrameDecompressWords(up.nCoded[ci], p.chunks[ci].b1 - p.chunks[ci].b0 - up.nCoded[ci], p.nHashed[ci]); };
    std::vector<u64> done(nFrames, 0);                              // bytes regenerated so far
    std::vector<u32> devHash(nFrames, 0);
    HostHasher hasher(nFrames, p.hostFrames);
    std::vector<std::vector<HostHasher::Piece>> landed(p.chunks.size());    // each chunk's pieces of the host-hashed frames
    size_t fed = 0;                                                 // chunks [0, fed) went to the hasher
    cudaError_t e = cudaSuccess;
    if (nb) {
        auto& P = packed_ring();
        std::lock_guard<std::mutex> lock(P.mu);
        size_t words = 0;
        for (size_t ci = 0; ci < p.chunks.size(); ci++) words = std::max(words, layout(ci).end);
        e = P.ensure(p.most.bytes, up.most, 0, words, words);
        // queue: the frames' bytes and the descriptors up, the decoders, the stored blocks and the hashes, the results down
        auto queue = [&](size_t ci, int k) -> cudaError_t {
            const HostChunk& c = p.chunks[ci];
            FrameDecompressWords const L = layout(ci);
            size_t const nc = up.nCoded[ci];
            cudaStream_t const s = P.st[k];
            u64* const h = P.hD[k], * const d = P.dD[k];
            for (size_t b = c.b0, a = 0, jf = 0, jh = up.nFse[ci], t = 0, j = 0; b < c.b1; a += p.bytes[b], b++) {
                const FrameBlock& x = blk(b);
                size_t const f = p.frameOf[b];
                u64 const pay = up.srcOff[b] + (x.payload - x.head);
                if (b == p.fb[f] && p.onDevice[f]) { h[L.range + 2 * j] = a; h[L.range + 2 * j + 1] = nominal[f]; j++; }
                if (x.type == BT_COMPRESSED) {
                    size_t const i = walks[f].codec ? jh++ : jf++;
                    h[L.dst + i] = reinterpret_cast<u64>(P.dA[k] + a); h[L.cap + i] = x.rSize;
                    h[L.src + i] = reinterpret_cast<u64>(P.dB[k] + pay); h[L.srcSize + i] = x.cSize;
                } else {
                    u64* const index = h + L.index + 3 * t++;
                    index[0] = a; index[1] = pay; index[2] = x.rSize | (u64)x.type << 32;
                }
            }
            cudaError_t r;
            for (const ChunkInputs::Run& x : up.runs[ci])
                if ((r = cudaMemcpyAsync(P.dB[k] + x.to, in + x.from, x.n, cudaMemcpyHostToDevice, s)) != cudaSuccess) return r;
            if ((r = cudaMemcpyAsync(d, h, L.result * sizeof(u64), cudaMemcpyHostToDevice, s)) != cudaSuccess) return r;
            for (int huf = 0; huf < 2; huf++) {
                size_t const j0 = huf ? up.nFse[ci] : 0, n = huf ? nc - up.nFse[ci] : up.nFse[ci];
                if (!n) continue;
                BlockDescs g;
                g.dst = (u8* const*)(d + L.dst) + j0; g.dstCap = d + L.cap + j0; g.result = d + L.result + j0;
                g.src = (const u8* const*)(d + L.src) + j0; g.srcSize = d + L.srcSize + j0; g.nBlocks = (u32)n;
                if ((r = huf ? launch_huf_decode_blocks(g, 4, s) : launch_fse_decode_blocks(g, false, s)) != cudaSuccess) return r;
            }
            size_t const ns = c.b1 - c.b0 - nc;
            if (ns && (r = launch_frame_stored(P.dA[k], P.dB[k], d + L.index, ns, s)) != cudaSuccess) return r;
            if ((r = launch_xxh32_ranges(P.dA[k], d + L.range, p.nHashed[ci], d + L.hash, s)) != cudaSuccess) return r;
            return L.end > L.result ? cudaMemcpyAsync(h + L.result, d + L.result, (L.end - L.result) * sizeof(u64), cudaMemcpyDeviceToHost, s) : cudaSuccess;
        };
        auto feed_until = [&](size_t end) -> cudaError_t {          // in chunk order, once each chunk's copies have landed
            for (cudaError_t r; fed < end; fed++) {
                if (!landed[fed].empty() && (r = cudaStreamSynchronize(P.st[fed % P.NS])) != cudaSuccess) return r;
                for (const HostHasher::Piece& x : landed[fed]) hasher.feed(x);
            }
            return cudaSuccess;
        };
        size_t const lastFrame = p.frameOf[nb - 1];
        size_t stop = 0;                                            // the last frame has failed: nothing left to decide
        // finish: per frame, the first decoder error or overflow of its capacity in block order ends it; its output comes down
        // to its place -- runs of blocks and frames contiguous on both sides in one copy -- and then goes to the hasher
        auto finish = [&](size_t ci, int k) -> cudaError_t {
            const HostChunk& c = p.chunks[ci];
            FrameDecompressWords const L = layout(ci);
            cudaError_t r = cudaStreamSynchronize(P.st[k]); if (r != cudaSuccess) return r;
            const u64* const res = P.hD[k] + L.result, * const hashes = P.hD[k] + L.hash;
            CopyRun run; run.s = P.st[k];
            for (size_t b = c.b0, a = 0, jf = 0, jh = up.nFse[ci], t = 0; b < c.b1 && r == cudaSuccess; a += p.bytes[b], b++) {
                size_t const f = p.frameOf[b];
                const FrameBlock& x = blk(b);
                bool const last = b + 1 == p.fb[f + 1], onHost = !walks[f].verdict && !p.onDevice[f];
                if (b == p.fb[f] && p.onDevice[f]) devHash[f] = (u32)hashes[t++];
                u64 const n = x.type == BT_COMPRESSED ? res[walks[f].codec ? jh++ : jf++] : x.rSize;   // the block's result
                if (!verdict[f] && is_err(n)) verdict[f] = (size_t)n;
                if (!verdict[f] && done[f] + n > caps[f]) verdict[f] = (size_t)err(E_DST_TOO_SMALL);
                u8* const to = dst + region[f] + done[f];
                if (!verdict[f]) { r = run.add(P.dA[k] + a, to, n); done[f] += n; }
                if (onHost && (last || !verdict[f])) landed[ci].push_back({ f, to, verdict[f] ? 0 : n, last });
            }
            if (r == cudaSuccess) r = run.flush();
            if (r == cudaSuccess) r = feed_until(ci);               // the earlier chunks', landed meanwhile
            stop = verdict[lastFrame] != 0;
            return r;
        };
        if (e == cudaSuccess) e = run_chunks(P, p.chunks.size(), P.NS - 1, queue, finish, &stop);
        if (e == cudaSuccess) e = feed_until(p.chunks.size());     // the rest, landed by the drain
    }
    hasher.join();
    if (e != cudaSuccess) return (size_t)err(E_GENERIC);
    for (size_t f = 0; f < nFrames; f++) {
        if (verdict[f] || walks[f].verdict) { hResults[f] = verdict[f] ? verdict[f] : walks[f].verdict; continue; }
        // a device-hashed frame that decoded short is hashed here: its device hash covered the nominal layout, gaps included
        u32 const hash = !p.onDevice[f] ? hasher.digest(f) : done[f] != nominal[f] ? FSEB200_XXH32(dst + region[f], done[f], 0) : devHash[f];
        hResults[f] = trailer_checksum(hash) != walks[f].checksum ? (size_t)err(E_CORRUPT) : (size_t)done[f];   // exit 44
    }
    return 0;
}
}  // namespace

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

FSEB_API size_t FSEB200_frame_compress_host_batch(int codec, unsigned blockSizeId, size_t nFrames, void* hOut, size_t outCapacity,
                                                  size_t* hOffsets, size_t* hResults, const void* hSrc, const size_t* hSrcSizes)
{
    if (codec < 0 || codec > 1 || blockSizeId > 6 || nFrames > 0xFFFFFFFFull) return (size_t)err(E_SRC_WRONG);
    if (nFrames == 0) return 0;
    if (!hOut || !hOffsets || !hResults || !hSrcSizes) return (size_t)err(E_SRC_WRONG);
    if (!hSrc) for (size_t f = 0; f < nFrames; f++) if (hSrcSizes[f]) return (size_t)err(E_SRC_WRONG);
    return frame_compress_batch(Spanning::BATCH, codec, blockSizeId, nFrames, (u8*)hOut, outCapacity, hOffsets, hResults, (const u8*)hSrc,
                                hSrcSizes);
}

FSEB_API size_t FSEB200_frame_compress_host(int codec, unsigned blockSizeId, void* hFrame, size_t frameCapacity,
                                            const void* hSrc, size_t srcSize)
{
    if (codec < 0 || codec > 1 || blockSizeId > 6 || (!hSrc && srcSize) || (!hFrame && frameCapacity)) return (size_t)err(E_SRC_WRONG);
    if (frameCapacity < FRAME_HEADER + FRAME_TRAILER) return (size_t)err(E_DST_TOO_SMALL);
    size_t result = 0;
    size_t const r = frame_compress_batch(Spanning::ONE_FRAME, codec, blockSizeId, 1, (u8*)hFrame, frameCapacity, nullptr, &result,
                                          (const u8*)hSrc, &srcSize);
    return r ? r : result;
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

FSEB_API size_t FSEB200_frame_decompress_host_batch(size_t nFrames, void* hDst, const size_t* hDstCapacities, size_t* hResults,
                                                    const void* hIn, const size_t* hOffsets)
{
    if (nFrames > 0xFFFFFFFFull) return (size_t)err(E_SRC_WRONG);
    if (nFrames == 0) return 0;
    if (!hDst || !hDstCapacities || !hResults || !hIn || !hOffsets) return (size_t)err(E_SRC_WRONG);
    for (size_t f = 0; f < nFrames; f++) if (hOffsets[f + 1] < hOffsets[f]) return (size_t)err(E_SRC_WRONG);
    return frame_decompress_batch(nFrames, (u8*)hDst, hDstCapacities, hResults, (const u8*)hIn, hOffsets);
}

FSEB_API size_t FSEB200_frame_decompress_host(void* hDst, size_t dstCapacity, const void* hFrame, size_t frameSize)
{
    if ((!hFrame && frameSize) || (!hDst && dstCapacity)) return (size_t)err(E_SRC_WRONG);
    size_t const offsets[2] = { 0, frameSize };
    size_t result = 0;
    size_t const r = frame_decompress_batch(1, (u8*)hDst, &dstCapacity, &result, (const u8*)hFrame, offsets);
    return r ? r : result;
}
