// capi.cu -- the C-ABI boundary of libfse_b200.so (declarations: include/fse_b200.h).
//
// Tiers:
//   1. FSEB200_*_batch : device-pointer, stream-ordered, whole-batch entry points -- what the
//      per-chunk loops of the reference harness (programs/bench.c:353-364 and :389-424) collapse into.
//      FSEB200_{HUF,FSE,FSEU16}_*_blocks: the same for blocks given by per-block device descriptors (common.cuh BlockDescs),
//      and the *_packed calls for blocks stored back to back in one device buffer.
//      The same batches on HOST buffers (FSEB200_*_host, .fse frames) are host_pipeline.cu's.
//   2. the reference's own one-block-per-call symbols (lib/fse.h, lib/huf.h, lib/hist.h,
//      lib/fseU16.h) with HOST pointers: they stage the block through a private device workspace and
//      run the same kernels with a batch of one.  Correct drop-ins for unmodified callers; not the
//      fast path (one launch + two PCIe copies per call).  Beside them: the scalar helpers, the table
//      helpers and the measurement-input generators.
// There is no CPU implementation behind any data-path entry point: without a CUDA device every call
// aborts loudly.  Only scalar helpers (bounds, error names, table-log arithmetic) run on the host.
#include "capi_common.h"
#include "fse_b200.h"
#include "launch_util.cuh"
#include <cstring>
#include <mutex>

using namespace fseb;

static cudaError_t huf_dec_4x1(const BatchGeom& g, void* d, const void* c, const u64* cs, u64* r, const void* o, cudaStream_t s) { return launch_huf_decode(g, d, c, cs, r, o, s, 1); }
static cudaError_t huf_dec_4x2(const BatchGeom& g, void* d, const void* c, const u64* cs, u64* r, const void* o, cudaStream_t s) { return launch_huf_decode(g, d, c, cs, r, o, s, 3); }

namespace {

// Private device workspace of the host-pointer tier.
struct Workspace {
    std::mutex mu;
    cudaStream_t stream = nullptr;
    unsigned char* d[4] = { nullptr, nullptr, nullptr, nullptr };
    size_t cap[4] = { 0, 0, 0, 0 };
    void* get(int i, size_t bytes)
    {
        if (!stream) CK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
        bytes = (bytes + 64 + 255) & ~(size_t)255;          // slack: kernels read whole aligned 16-byte chunks
        if (cap[i] < bytes) {
            if (d[i]) CK(cudaFree(d[i]));
            CK(cudaMalloc(&d[i], bytes));
            CK(cudaMemset(d[i], 0, bytes));
            cap[i] = bytes;
        }
        return d[i];
    }
};
// one workspace per device: streams and buffers belong to the device that was current when they were created
Workspace& ws() { static Workspace w[MAX_DEVICES]; return w[current_device()]; }

// one block through the batched encoder; `zeroIsEmpty`: what to answer for srcSize == 0
size_t one_block_compress(enc_fn fn, void* dst, size_t dstCapacity, const void* src, size_t srcBytes,
                          unsigned msv, unsigned tlog, bool copyRleByte)
{
    Workspace& w = ws();
    std::lock_guard<std::mutex> lock(w.mu);
    size_t const cap = dstCapacity > 0xFFFFFF00ull ? 0xFFFFFF00ull : dstCapacity;
    unsigned char* dS = (unsigned char*)w.get(0, srcBytes);
    unsigned char* dC = (unsigned char*)w.get(1, cap);
    u64* dR = (u64*)w.get(2, 2 * sizeof(u64));
    u64 r = 0;
    if (srcBytes) CK(cudaMemcpyAsync(dS, src, srcBytes, cudaMemcpyHostToDevice, w.stream));
    BatchGeom g = geom(srcBytes ? srcBytes : 1, srcBytes ? srcBytes : 1, cap);
    if (!srcBytes) { g.total = 0; g.nBlocks = 1; }           // a single empty block (bench.c:513,538-544 produces those)
    CK(fn(g, dC, dR, dS, msv, tlog, w.stream));
    CK(cudaMemcpyAsync(&r, dR, sizeof(r), cudaMemcpyDeviceToHost, w.stream));
    CK(cudaStreamSynchronize(w.stream));
    if (!is_err(r)) {
        size_t const nOut = (r > 1) ? (size_t)r : ((r == 1 && copyRleByte) ? 1 : 0);
        if (nOut) { CK(cudaMemcpyAsync(dst, dC, nOut, cudaMemcpyDeviceToHost, w.stream)); CK(cudaStreamSynchronize(w.stream)); }
    }
    return (size_t)r;
}

size_t one_block_decompress(dec_fn fn, void* dst, size_t dstBytes, const void* cSrc, size_t cSrcSize)
{
    Workspace& w = ws();
    std::lock_guard<std::mutex> lock(w.mu);
    unsigned char* dC = (unsigned char*)w.get(0, cSrcSize);
    unsigned char* dO = (unsigned char*)w.get(1, dstBytes);
    u64* dS = (u64*)w.get(2, 2 * sizeof(u64));
    u64 hs[2] = { (u64)cSrcSize, 0 };
    if (cSrcSize) CK(cudaMemcpyAsync(dC, cSrc, cSrcSize, cudaMemcpyHostToDevice, w.stream));
    CK(cudaMemcpyAsync(dS, hs, sizeof(hs), cudaMemcpyHostToDevice, w.stream));
    BatchGeom g = geom(dstBytes ? dstBytes : 1, dstBytes ? dstBytes : 1, cSrcSize + 16);
    if (!dstBytes) { g.total = 0; g.nBlocks = 1; }
    CK(fn(g, dO, dC, dS, dS + 1, nullptr, w.stream));
    CK(cudaMemcpyAsync(hs, dS, sizeof(hs), cudaMemcpyDeviceToHost, w.stream));
    CK(cudaStreamSynchronize(w.stream));
    if (!is_err(hs[1]) && hs[1]) {
        size_t const nOut = hs[1] < dstBytes ? (size_t)hs[1] : dstBytes;
        CK(cudaMemcpyAsync(dst, dO, nOut, cudaMemcpyDeviceToHost, w.stream));
        CK(cudaStreamSynchronize(w.stream));
    }
    return (size_t)hs[1];
}

// runs one table-level op: uploads `in` at offset 0 of the scratch, returns the kernel's value; the
// caller then downloads what it needs from the scratch.
struct Micro {
    Workspace& w; unsigned char* buf; u64* ret; std::unique_lock<std::mutex> lock;
    explicit Micro(size_t bytes = 256 * 1024) : w(ws()), lock(w.mu) { buf = (unsigned char*)w.get(3, bytes < 256 * 1024 ? 256 * 1024 : bytes); ret = (u64*)w.get(2, 2 * sizeof(u64)); }
    void up(size_t off, const void* p, size_t n) { if (n) CK(cudaMemcpyAsync(buf + off, p, n, cudaMemcpyHostToDevice, w.stream)); }
    void down(void* p, size_t off, size_t n) { if (n) { CK(cudaMemcpyAsync(p, buf + off, n, cudaMemcpyDeviceToHost, w.stream)); CK(cudaStreamSynchronize(w.stream)); } }
    u64 run(int op, u64 a0 = 0, u64 a1 = 0, u64 a2 = 0, u64 a3 = 0)
    {
        MicroArgs A; A.a[0] = a0; A.a[1] = a1; A.a[2] = a2; A.a[3] = a3; A.a[4] = A.a[5] = 0;
        u64 r = 0;
        CK(launch_micro(op, A, buf, ret, w.stream));
        CK(cudaMemcpyAsync(&r, ret, sizeof(r), cudaMemcpyDeviceToHost, w.stream));
        CK(cudaStreamSynchronize(w.stream));
        return r;
    }
};

unsigned hibit_h(unsigned v) { unsigned r = 0; while (v >>= 1) r++; return r; }

}  // namespace

// ================================================================================================
// tier 1: batched, device-resident.  Geometry: programs/bench.c:530-548 (see common.cuh BatchGeom).
// ================================================================================================
#define FSEB_DECL_DEC(NAME, FN, MAXBLOCK) \
FSEB_API size_t NAME(void* dDst, size_t dstTotal, size_t blockSize, const void* dCBuf, size_t slot, \
                     const size_t* dCSizes, size_t* dResults, const void* dOrig, void* stream) \
{ \
    if (blockSize == 0 || blockSize > (MAXBLOCK) || slot > 0xFFFFFFFFull) return (size_t)err(E_SRC_WRONG); \
    return ok_or_generic(FN(geom(dstTotal, blockSize, slot), dDst, dCBuf, (const u64*)dCSizes, (u64*)dResults, dOrig, (cudaStream_t)stream)); \
}
#define FSEB_DECL_ENC(NAME, FN, MAXBLOCK) \
FSEB_API size_t NAME(void* dCBuf, size_t slot, size_t* dCSizes, const void* dSrc, size_t srcTotal, size_t blockSize, \
                     unsigned maxSymbolValue, unsigned tableLog, void* stream) \
{ \
    if (blockSize == 0 || blockSize > (MAXBLOCK) || slot > 0xFFFFFFFFull) return (size_t)err(E_SRC_WRONG); \
    return ok_or_generic(FN(geom(srcTotal, blockSize, slot), dCBuf, (u64*)dCSizes, dSrc, maxSymbolValue, tableLog, (cudaStream_t)stream)); \
}
FSEB_DECL_DEC(FSEB200_HUF_decompress_batch, huf_dec_std, HUF_BLOCK_MAX)
FSEB_DECL_ENC(FSEB200_HUF_compress_batch, launch_huf_encode, HUF_BLOCK_MAX)
FSEB_DECL_DEC(FSEB200_FSE_decompress_batch, launch_fse_decode, (1u << 30))
FSEB_DECL_ENC(FSEB200_FSE_compress_batch, launch_fse_encode, (1u << 30))
FSEB_DECL_DEC(FSEB200_FSEU16_decompress_batch, launch_fseu16_decode, (1u << 30))
FSEB_DECL_ENC(FSEB200_FSEU16_compress_batch, launch_fseu16_encode, (1u << 30))

// Table reuse across blocks (SURVEY.md 8f-3): the whole batch coded with ONE caller-supplied HUF_CElt table (256 cells on the device,
// the layout HUF_buildCTable produces: val | nbBits << 16).  dCSizes[b] is what HUF_compress4X_usingCTable (lib/huf.h:191,
// huf_compress.c:552-610) returns for block b with that table: 6 + the four stream sizes, or 0 (block shorter than 12 bytes, or a
// stream does not fit its slot).  No histogram, no tree, no header: the shape programs/bench.c:610-633 times for FSE and
// HUF_compress4X_repeat (huf_compress.c:664-712) reduces to when the previous table is kept.
FSEB_API size_t FSEB200_HUF_compress4X_usingCTable_batch(void* dCBuf, size_t slot, size_t* dCSizes, const void* dSrc, size_t srcTotal, size_t blockSize,
                                                         const unsigned* dCTable, void* stream)
{
    if (blockSize == 0 || blockSize > HUF_BLOCK_MAX || slot > 0xFFFFFFFFull || !dCTable) return (size_t)err(E_SRC_WRONG);
    return ok_or_generic(launch_huf_encode_using_ctable(geom(srcTotal, blockSize, slot), dCBuf, (u64*)dCSizes, dSrc, dCTable, (cudaStream_t)stream));
}

// Per-block descriptors (see common.cuh BlockDescs): every array and every buffer it points to is device memory, and the host never
// reads them -- the per-block verdicts (sizes above a block, capacities, parameters) all come from the kernels.
// nStreams: 4 for the 4X format (HUF_compress2 / HUF_decompress), 1 for the single-stream one (HUF_compress1X / HUF_decompress1X_DCtx).
namespace {
// the descriptor calls' argument checks, then `launch(descs)`
template <class Launch>
size_t blocks_call(size_t nBlocks, void* const* dDsts, const size_t* dDstSizes, size_t* dOut, const void* const* dSrcs, const size_t* dSrcSizes,
                   Launch launch)
{
    if (nBlocks == 0) return 0;
    if (nBlocks > 0xFFFFFFFFull || !dDsts || !dDstSizes || !dOut || !dSrcs || !dSrcSizes) return (size_t)err(E_SRC_WRONG);
    BlockDescs g;
    g.dst = (u8* const*)dDsts; g.dstCap = (const u64*)dDstSizes; g.result = (u64*)dOut;
    g.src = (const u8* const*)dSrcs; g.srcSize = (const u64*)dSrcSizes; g.nBlocks = (u32)nBlocks;
    return ok_or_generic(launch(g));
}
}
FSEB_API size_t FSEB200_HUF_compress_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstCapacities, size_t* dCSizes,
                                            const void* const* dSrcs, const size_t* dSrcSizes, unsigned maxSymbolValue, unsigned tableLog, void* stream)
{
    return blocks_call(nBlocks, dDsts, dDstCapacities, dCSizes, dSrcs, dSrcSizes,
                       [&](const BlockDescs& g) { return launch_huf_encode_descs(g, 4, maxSymbolValue, tableLog, (cudaStream_t)stream); });
}
FSEB_API size_t FSEB200_HUF_decompress_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstSizes, size_t* dResults,
                                              const void* const* dCSrcs, const size_t* dCSrcSizes, void* stream)
{
    return blocks_call(nBlocks, dDsts, dDstSizes, dResults, dCSrcs, dCSrcSizes,
                       [&](const BlockDescs& g) { return launch_huf_decode_blocks(g, 4, (cudaStream_t)stream); });
}
FSEB_API size_t FSEB200_HUF_compress1X_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstCapacities, size_t* dCSizes,
                                              const void* const* dSrcs, const size_t* dSrcSizes, unsigned maxSymbolValue, unsigned tableLog, void* stream)
{
    return blocks_call(nBlocks, dDsts, dDstCapacities, dCSizes, dSrcs, dSrcSizes,
                       [&](const BlockDescs& g) { return launch_huf_encode_descs(g, 1, maxSymbolValue, tableLog, (cudaStream_t)stream); });
}
FSEB_API size_t FSEB200_HUF_decompress1X_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstSizes, size_t* dResults,
                                                const void* const* dCSrcs, const size_t* dCSrcSizes, void* stream)
{
    return blocks_call(nBlocks, dDsts, dDstSizes, dResults, dCSrcs, dCSrcSizes,
                       [&](const BlockDescs& g) { return launch_huf_decode_blocks(g, 1, (cudaStream_t)stream); });
}
// Table reuse: the descriptor calls with each block's (table, repeat flag) pair (common.cuh RepeatDescs), and the decoders of what
// they produce, which take a block's tree header from wherever the caller says (common.cuh HeaderDescs).
namespace {
size_t huf_repeat_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstCapacities, size_t* dCSizes, const void* const* dSrcs,
                         const size_t* dSrcSizes, unsigned* const* dCTables, int* dRepeats, const int* dPreferRepeat, int nStreams,
                         unsigned msv, unsigned tlog, void* stream)
{
    if (nBlocks && (!dCTables || !dRepeats || !dPreferRepeat)) return (size_t)err(E_SRC_WRONG);
    return blocks_call(nBlocks, dDsts, dDstCapacities, dCSizes, dSrcs, dSrcSizes, [&](const BlockDescs& d) {
        RepeatDescs g;
        static_cast<BlockDescs&>(g) = d;
        g.ctable = (u32* const*)dCTables; g.repeat = dRepeats; g.prefer = dPreferRepeat;
        return launch_huf_encode_descs(g, nStreams, msv, tlog, (cudaStream_t)stream);
    });
}
// nStreams as forms_given's
size_t huf_header_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstSizes, size_t* dResults, const void* const* dCSrcs,
                         const size_t* dCSrcSizes, const void* const* dHeaders, const size_t* dHeaderSizes, int nStreams, void* stream,
                         const unsigned char* dSingleStream = nullptr)
{
    if (nBlocks && (!dHeaders || !dHeaderSizes || !forms_given(nStreams, dSingleStream))) return (size_t)err(E_SRC_WRONG);
    return blocks_call(nBlocks, dDsts, dDstSizes, dResults, dCSrcs, dCSrcSizes, [&](const BlockDescs& d) {
        HeaderDescs g;
        static_cast<BlockDescs&>(g) = d;
        g.hdr = (const u8* const*)dHeaders; g.hdrSize = (const u64*)dHeaderSizes;
        return launch_huf_decode_headers(g, nStreams, (cudaStream_t)stream, dSingleStream);
    });
}
}
// Mixed forms: per block, the 4X or the 1X header decoder, as dSingleStream[b] names (0: 4X).
FSEB_API size_t FSEB200_HUF_decompress_mixed_repeat_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstSizes, size_t* dResults,
                                                          const void* const* dCSrcs, const size_t* dCSrcSizes, const void* const* dHeaders,
                                                          const size_t* dHeaderSizes, const unsigned char* dSingleStream, void* stream)
{
    return huf_header_blocks(nBlocks, dDsts, dDstSizes, dResults, dCSrcs, dCSrcSizes, dHeaders, dHeaderSizes, 0, stream, dSingleStream);
}
FSEB_API size_t FSEB200_HUF_compress4X_repeat_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstCapacities, size_t* dCSizes,
                                                     const void* const* dSrcs, const size_t* dSrcSizes, unsigned* const* dCTables, int* dRepeats,
                                                     const int* dPreferRepeat, unsigned maxSymbolValue, unsigned tableLog, void* stream)
{
    return huf_repeat_blocks(nBlocks, dDsts, dDstCapacities, dCSizes, dSrcs, dSrcSizes, dCTables, dRepeats, dPreferRepeat, 4,
                             maxSymbolValue, tableLog, stream);
}
FSEB_API size_t FSEB200_HUF_compress1X_repeat_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstCapacities, size_t* dCSizes,
                                                     const void* const* dSrcs, const size_t* dSrcSizes, unsigned* const* dCTables, int* dRepeats,
                                                     const int* dPreferRepeat, unsigned maxSymbolValue, unsigned tableLog, void* stream)
{
    return huf_repeat_blocks(nBlocks, dDsts, dDstCapacities, dCSizes, dSrcs, dSrcSizes, dCTables, dRepeats, dPreferRepeat, 1,
                             maxSymbolValue, tableLog, stream);
}
// Chains: blocks of one stream in one call, the stream's state carried from block to block on the device (common.cuh ChainDescs).
namespace {
// nStreams as forms_given's
size_t huf_repeat_chains(size_t nChains, const size_t* dChainStarts, size_t nBlocks, void* const* dDsts, const size_t* dDstCapacities,
                         size_t* dCSizes, const void* const* dSrcs, const size_t* dSrcSizes, const int* dPreferRepeat,
                         unsigned* const* dCTables, int* dRepeats, const void** dChainHeaders, size_t* dChainHeaderSizes,
                         const void** dHeaders, size_t* dHeaderSizes, int nStreams, unsigned msv, unsigned tlog, void* stream,
                         const unsigned char* dSingleStream = nullptr)
{
    if (nBlocks && (nChains > 0xFFFFFFFFull || !dChainStarts || !dPreferRepeat || !dCTables || !dRepeats || !dChainHeaders ||
                    !dChainHeaderSizes || !dHeaders || !dHeaderSizes || !forms_given(nStreams, dSingleStream))) return (size_t)err(E_SRC_WRONG);
    return blocks_call(nBlocks, dDsts, dDstCapacities, dCSizes, dSrcs, dSrcSizes, [&](const BlockDescs& d) {
        ChainMixedDescs g;
        static_cast<BlockDescs&>(g) = d;
        g.start = (const u64*)dChainStarts; g.nChains = (u32)nChains; g.prefer = dPreferRepeat;
        g.ctable = (u32* const*)dCTables; g.repeat = dRepeats; g.hdr = (const u8**)dChainHeaders; g.hdrSize = (u64*)dChainHeaderSizes;
        g.blkHdr = (const u8**)dHeaders; g.blkHdrSize = (u64*)dHeaderSizes; g.fact = nullptr; g.single = dSingleStream;
        return launch_huf_encode_descs(g, nStreams, msv, tlog, (cudaStream_t)stream);
    });
}
}
FSEB_API size_t FSEB200_HUF_compress4X_repeat_chains(size_t nChains, const size_t* dChainStarts, size_t nBlocks, void* const* dDsts,
                                                     const size_t* dDstCapacities, size_t* dCSizes, const void* const* dSrcs,
                                                     const size_t* dSrcSizes, const int* dPreferRepeat, unsigned* const* dCTables,
                                                     int* dRepeats, const void** dChainHeaders, size_t* dChainHeaderSizes,
                                                     const void** dHeaders, size_t* dHeaderSizes, unsigned maxSymbolValue,
                                                     unsigned tableLog, void* stream)
{
    return huf_repeat_chains(nChains, dChainStarts, nBlocks, dDsts, dDstCapacities, dCSizes, dSrcs, dSrcSizes, dPreferRepeat, dCTables,
                             dRepeats, dChainHeaders, dChainHeaderSizes, dHeaders, dHeaderSizes, 4, maxSymbolValue, tableLog, stream);
}
FSEB_API size_t FSEB200_HUF_compress1X_repeat_chains(size_t nChains, const size_t* dChainStarts, size_t nBlocks, void* const* dDsts,
                                                     const size_t* dDstCapacities, size_t* dCSizes, const void* const* dSrcs,
                                                     const size_t* dSrcSizes, const int* dPreferRepeat, unsigned* const* dCTables,
                                                     int* dRepeats, const void** dChainHeaders, size_t* dChainHeaderSizes,
                                                     const void** dHeaders, size_t* dHeaderSizes, unsigned maxSymbolValue,
                                                     unsigned tableLog, void* stream)
{
    return huf_repeat_chains(nChains, dChainStarts, nBlocks, dDsts, dDstCapacities, dCSizes, dSrcs, dSrcSizes, dPreferRepeat, dCTables,
                             dRepeats, dChainHeaders, dChainHeaderSizes, dHeaders, dHeaderSizes, 1, maxSymbolValue, tableLog, stream);
}
FSEB_API size_t FSEB200_HUF_compress_mixed_repeat_chains(size_t nChains, const size_t* dChainStarts, size_t nBlocks, void* const* dDsts,
                                                         const size_t* dDstCapacities, size_t* dCSizes, const void* const* dSrcs,
                                                         const size_t* dSrcSizes, const int* dPreferRepeat,
                                                         const unsigned char* dSingleStream, unsigned* const* dCTables,
                                                         int* dRepeats, const void** dChainHeaders, size_t* dChainHeaderSizes,
                                                         const void** dHeaders, size_t* dHeaderSizes, unsigned maxSymbolValue,
                                                         unsigned tableLog, void* stream)
{
    return huf_repeat_chains(nChains, dChainStarts, nBlocks, dDsts, dDstCapacities, dCSizes, dSrcs, dSrcSizes, dPreferRepeat, dCTables,
                             dRepeats, dChainHeaders, dChainHeaderSizes, dHeaders, dHeaderSizes, 0, maxSymbolValue, tableLog, stream,
                             dSingleStream);
}
// Packed chains: the chain calls with every block stored back to back in one buffer and a kind byte per block
// (common.cuh ChainPackedDescs), and the decoders of that buffer.
namespace {
// the packed-chain geometry of a call's arguments, checked by the caller
void chain_packed_descs(ChainPackedDescs& g, size_t nChains, const size_t* dChainStarts, size_t nBlocks, void* dOut, size_t outCapacity,
                        size_t* dOffsets, size_t* dCSizes, unsigned char* dKinds, const void* const* dSrcs, const size_t* dSrcSizes,
                        const int* dPreferRepeat, unsigned* const* dCTables, int* dRepeats, const void** dChainHeaders,
                        size_t* dChainHeaderSizes)
{
    g.dst = nullptr; g.dstCap = nullptr; g.result = (u64*)dCSizes; g.src = (const u8* const*)dSrcs; g.srcSize = (const u64*)dSrcSizes;
    g.nBlocks = (u32)nBlocks;
    g.start = (const u64*)dChainStarts; g.nChains = (u32)nChains; g.prefer = dPreferRepeat;
    g.ctable = (u32* const*)dCTables; g.repeat = dRepeats; g.hdr = (const u8**)dChainHeaders; g.hdrSize = (u64*)dChainHeaderSizes;
    g.blkHdr = nullptr; g.blkHdrSize = nullptr; g.fact = nullptr;
    g.pk.out = (u8*)dOut; g.pk.outCap = outCapacity; g.pk.offset = (u64*)dOffsets; g.pk.result = g.result;
    g.pk.src = g.src; g.pk.srcSize = g.srcSize; g.pk.nBlocks = g.nBlocks;
    g.kind = dKinds; g.end = nullptr; g.malformed = nullptr;
}
}
size_t fseb::huf_repeat_chains_packed(size_t nChains, const size_t* dChainStarts, size_t nBlocks, void* dOut, size_t outCapacity,
                                      size_t* dOffsets, size_t* dCSizes, unsigned char* dKinds, const void* const* dSrcs,
                                      const size_t* dSrcSizes, const int* dPreferRepeat, unsigned* const* dCTables, int* dRepeats,
                                      const void** dChainHeaders, size_t* dChainHeaderSizes, const ChainForm& f, unsigned msv,
                                      unsigned tlog, void* stream)
{
    if (nBlocks == 0) return 0;
    if (nBlocks > 0xFFFFFFFFull || nChains > 0xFFFFFFFFull || !dChainStarts || !dOut || !dOffsets || !dCSizes || !dKinds || !dSrcs ||
        !dSrcSizes || !dPreferRepeat || !dCTables || !dRepeats || !dChainHeaders || !dChainHeaderSizes ||
        !forms_given(f.nStreams, f.dSingleStream) || (f.literals && (f.minGainLog < 1 || f.minGainLog > 31)))
        return (size_t)err(E_SRC_WRONG);
    ChainPackedDescs d;
    chain_packed_descs(d, nChains, dChainStarts, nBlocks, dOut, outCapacity, dOffsets, dCSizes, dKinds, dSrcs, dSrcSizes, dPreferRepeat,
                       dCTables, dRepeats, dChainHeaders, dChainHeaderSizes);
    if (f.literals) {
        ChainPackedLiteralsDescs g;
        static_cast<ChainPackedDescs&>(g) = d;
        g.single = f.dSingleStream; g.minLiterals = f.minLiterals; g.minGainLog = f.minGainLog;
        return ok_or_generic(launch_huf_encode_descs(g, 0, msv, tlog, (cudaStream_t)stream));
    }
    ChainPackedMixedDescs g;
    static_cast<ChainPackedDescs&>(g) = d;
    g.single = f.dSingleStream;
    return ok_or_generic(launch_huf_encode_descs(g, f.nStreams, msv, tlog, (cudaStream_t)stream));
}
size_t fseb::huf_repeat_unpack(size_t nChains, const size_t* dChainStarts, size_t nBlocks, void* const* dDsts, const size_t* dDstSizes,
                               size_t* dResults, const void* dIn, const size_t* dOffsets, const unsigned char* dKinds,
                               const void* const* dChainHeaders, const size_t* dChainHeaderSizes, int nStreams, void* stream,
                               const unsigned char* dSingleStream)
{
    if (nBlocks == 0) return 0;
    if (nBlocks > 0xFFFFFFFFull || nChains > 0xFFFFFFFFull || !dChainStarts || !dDsts || !dDstSizes || !dResults || !dIn ||
        !dOffsets || !dKinds || !dChainHeaders || !dChainHeaderSizes || !forms_given(nStreams, dSingleStream))
        return (size_t)err(E_SRC_WRONG);
    return ok_or_generic(launch_huf_decompress_repeat_packed((const u64*)dChainStarts, (u32)nChains, (u8* const*)dDsts,
                                                             (const u64*)dDstSizes, (u64*)dResults, (const u8*)dIn,
                                                             (const u64*)dOffsets, dKinds, (const u8* const*)dChainHeaders,
                                                             (const u64*)dChainHeaderSizes, (u32)nBlocks, nStreams, (cudaStream_t)stream,
                                                             dSingleStream));
}
FSEB_API size_t FSEB200_HUF_compress4X_repeat_chains_packed(size_t nChains, const size_t* dChainStarts, size_t nBlocks, void* dOut,
                                                            size_t outCapacity, size_t* dOffsets, size_t* dCSizes, unsigned char* dKinds,
                                                            const void* const* dSrcs, const size_t* dSrcSizes, const int* dPreferRepeat,
                                                            unsigned* const* dCTables, int* dRepeats, const void** dChainHeaders,
                                                            size_t* dChainHeaderSizes, unsigned maxSymbolValue, unsigned tableLog, void* stream)
{
    return huf_repeat_chains_packed(nChains, dChainStarts, nBlocks, dOut, outCapacity, dOffsets, dCSizes, dKinds, dSrcs, dSrcSizes,
                                    dPreferRepeat, dCTables, dRepeats, dChainHeaders, dChainHeaderSizes, ChainForm{4}, maxSymbolValue,
                                    tableLog, stream);
}
FSEB_API size_t FSEB200_HUF_compress1X_repeat_chains_packed(size_t nChains, const size_t* dChainStarts, size_t nBlocks, void* dOut,
                                                            size_t outCapacity, size_t* dOffsets, size_t* dCSizes, unsigned char* dKinds,
                                                            const void* const* dSrcs, const size_t* dSrcSizes, const int* dPreferRepeat,
                                                            unsigned* const* dCTables, int* dRepeats, const void** dChainHeaders,
                                                            size_t* dChainHeaderSizes, unsigned maxSymbolValue, unsigned tableLog, void* stream)
{
    return huf_repeat_chains_packed(nChains, dChainStarts, nBlocks, dOut, outCapacity, dOffsets, dCSizes, dKinds, dSrcs, dSrcSizes,
                                    dPreferRepeat, dCTables, dRepeats, dChainHeaders, dChainHeaderSizes, ChainForm{1}, maxSymbolValue,
                                    tableLog, stream);
}
FSEB_API size_t FSEB200_HUF_decompress4X_repeat_packed(size_t nChains, const size_t* dChainStarts, size_t nBlocks, void* const* dDsts,
                                                       const size_t* dDstSizes, size_t* dResults, const void* dIn, const size_t* dOffsets,
                                                       const unsigned char* dKinds, const void* const* dChainHeaders,
                                                       const size_t* dChainHeaderSizes, void* stream)
{
    return huf_repeat_unpack(nChains, dChainStarts, nBlocks, dDsts, dDstSizes, dResults, dIn, dOffsets, dKinds, dChainHeaders,
                             dChainHeaderSizes, 4, stream);
}
FSEB_API size_t FSEB200_HUF_decompress1X_repeat_packed(size_t nChains, const size_t* dChainStarts, size_t nBlocks, void* const* dDsts,
                                                       const size_t* dDstSizes, size_t* dResults, const void* dIn, const size_t* dOffsets,
                                                       const unsigned char* dKinds, const void* const* dChainHeaders,
                                                       const size_t* dChainHeaderSizes, void* stream)
{
    return huf_repeat_unpack(nChains, dChainStarts, nBlocks, dDsts, dDstSizes, dResults, dIn, dOffsets, dKinds, dChainHeaders,
                             dChainHeaderSizes, 1, stream);
}
FSEB_API size_t FSEB200_HUF_compress_mixed_repeat_chains_packed(size_t nChains, const size_t* dChainStarts, size_t nBlocks, void* dOut,
                                                                size_t outCapacity, size_t* dOffsets, size_t* dCSizes, unsigned char* dKinds,
                                                                const void* const* dSrcs, const size_t* dSrcSizes, const int* dPreferRepeat,
                                                                const unsigned char* dSingleStream, unsigned* const* dCTables, int* dRepeats,
                                                                const void** dChainHeaders, size_t* dChainHeaderSizes,
                                                                unsigned maxSymbolValue, unsigned tableLog, void* stream)
{
    return huf_repeat_chains_packed(nChains, dChainStarts, nBlocks, dOut, outCapacity, dOffsets, dCSizes, dKinds, dSrcs, dSrcSizes,
                                    dPreferRepeat, dCTables, dRepeats, dChainHeaders, dChainHeaderSizes,
                                    ChainForm{0, const_cast<unsigned char*>(dSingleStream)}, maxSymbolValue, tableLog, stream);
}
FSEB_API size_t FSEB200_HUF_compress_literals_chains_packed(size_t nChains, const size_t* dChainStarts, size_t nBlocks, void* dOut,
                                                            size_t outCapacity, size_t* dOffsets, size_t* dCSizes, unsigned char* dKinds,
                                                            const void* const* dSrcs, const size_t* dSrcSizes, const int* dPreferRepeat,
                                                            unsigned char* dSingleStream, unsigned* const* dCTables, int* dRepeats,
                                                            const void** dChainHeaders, size_t* dChainHeaderSizes, unsigned maxSymbolValue,
                                                            unsigned tableLog, unsigned minLiterals, unsigned minGainLog, void* stream)
{
    return huf_repeat_chains_packed(nChains, dChainStarts, nBlocks, dOut, outCapacity, dOffsets, dCSizes, dKinds, dSrcs, dSrcSizes,
                                    dPreferRepeat, dCTables, dRepeats, dChainHeaders, dChainHeaderSizes,
                                    ChainForm{0, dSingleStream, true, minLiterals, minGainLog}, maxSymbolValue, tableLog, stream);
}
FSEB_API size_t FSEB200_HUF_decompress_mixed_repeat_packed(size_t nChains, const size_t* dChainStarts, size_t nBlocks, void* const* dDsts,
                                                           const size_t* dDstSizes, size_t* dResults, const void* dIn, const size_t* dOffsets,
                                                           const unsigned char* dKinds, const unsigned char* dSingleStream,
                                                           const void* const* dChainHeaders, const size_t* dChainHeaderSizes, void* stream)
{
    return huf_repeat_unpack(nChains, dChainStarts, nBlocks, dDsts, dDstSizes, dResults, dIn, dOffsets, dKinds, dChainHeaders,
                             dChainHeaderSizes, 0, stream, dSingleStream);
}
FSEB_API size_t FSEB200_HUF_decompress4X_repeat_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstSizes, size_t* dResults,
                                                       const void* const* dCSrcs, const size_t* dCSrcSizes, const void* const* dHeaders,
                                                       const size_t* dHeaderSizes, void* stream)
{
    return huf_header_blocks(nBlocks, dDsts, dDstSizes, dResults, dCSrcs, dCSrcSizes, dHeaders, dHeaderSizes, 4, stream);
}
FSEB_API size_t FSEB200_HUF_decompress1X_repeat_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstSizes, size_t* dResults,
                                                       const void* const* dCSrcs, const size_t* dCSrcSizes, const void* const* dHeaders,
                                                       const size_t* dHeaderSizes, void* stream)
{
    return huf_header_blocks(nBlocks, dDsts, dDstSizes, dResults, dCSrcs, dCSrcSizes, dHeaders, dHeaderSizes, 1, stream);
}
// Packed output: the descriptor compress with every block stored back to back in one buffer (common.cuh PackedDescs).
namespace {
size_t huf_packed(size_t nBlocks, void* dOut, size_t outCapacity, size_t* dOffsets, size_t* dCSizes, const void* const* dSrcs,
                  const size_t* dSrcSizes, int nStreams, unsigned msv, unsigned tlog, void* stream)
{
    if (nBlocks == 0) return 0;
    if (nBlocks > 0xFFFFFFFFull || !dOut || !dOffsets || !dCSizes || !dSrcs || !dSrcSizes) return (size_t)err(E_SRC_WRONG);
    PackedDescs g;
    g.out = (u8*)dOut; g.outCap = outCapacity; g.offset = (u64*)dOffsets; g.result = (u64*)dCSizes;
    g.src = (const u8* const*)dSrcs; g.srcSize = (const u64*)dSrcSizes; g.nBlocks = (u32)nBlocks;
    return ok_or_generic(launch_huf_encode_descs(g, nStreams, msv, tlog, (cudaStream_t)stream));
}
}
FSEB_API size_t FSEB200_HUF_compress_packed(size_t nBlocks, void* dOut, size_t outCapacity, size_t* dOffsets, size_t* dCSizes,
                                            const void* const* dSrcs, const size_t* dSrcSizes, unsigned maxSymbolValue, unsigned tableLog, void* stream)
{
    return huf_packed(nBlocks, dOut, outCapacity, dOffsets, dCSizes, dSrcs, dSrcSizes, 4, maxSymbolValue, tableLog, stream);
}
FSEB_API size_t FSEB200_HUF_compress1X_packed(size_t nBlocks, void* dOut, size_t outCapacity, size_t* dOffsets, size_t* dCSizes,
                                              const void* const* dSrcs, const size_t* dSrcSizes, unsigned maxSymbolValue, unsigned tableLog, void* stream)
{
    return huf_packed(nBlocks, dOut, outCapacity, dOffsets, dCSizes, dSrcs, dSrcSizes, 1, maxSymbolValue, tableLog, stream);
}
// Packed decompress: the descriptor decoder on dIn + dOffsets[b] / dOffsets[b+1] - dOffsets[b], an empty block answered with 0.
namespace {
// the packed decompress calls' argument checks, then `launch(dsts, dstSizes, results, in, offsets, nBlocks)`
template <class Launch>
size_t unpacked_call(size_t nBlocks, void* const* dDsts, const size_t* dDstSizes, size_t* dResults, const void* dIn,
                     const size_t* dOffsets, Launch launch)
{
    if (nBlocks == 0) return 0;
    if (nBlocks > 0xFFFFFFFFull || !dDsts || !dDstSizes || !dResults || !dIn || !dOffsets) return (size_t)err(E_SRC_WRONG);
    return ok_or_generic(launch((u8* const*)dDsts, (const u64*)dDstSizes, (u64*)dResults, (const u8*)dIn, (const u64*)dOffsets, (u32)nBlocks));
}
}
FSEB_API size_t FSEB200_HUF_decompress_packed(size_t nBlocks, void* const* dDsts, const size_t* dDstSizes, size_t* dResults,
                                              const void* dIn, const size_t* dOffsets, void* stream)
{
    return unpacked_call(nBlocks, dDsts, dDstSizes, dResults, dIn, dOffsets,
                         [&](auto... a) { return launch_huf_decompress_packed(a..., 4, (cudaStream_t)stream); });
}
FSEB_API size_t FSEB200_HUF_decompress1X_packed(size_t nBlocks, void* const* dDsts, const size_t* dDstSizes, size_t* dResults,
                                                const void* dIn, const size_t* dOffsets, void* stream)
{
    return unpacked_call(nBlocks, dDsts, dDstSizes, dResults, dIn, dOffsets,
                         [&](auto... a) { return launch_huf_decompress_packed(a..., 1, (cudaStream_t)stream); });
}
FSEB_API size_t FSEB200_FSE_compress_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstCapacities, size_t* dCSizes,
                                            const void* const* dSrcs, const size_t* dSrcSizes, unsigned maxSymbolValue, unsigned tableLog, void* stream)
{
    return blocks_call(nBlocks, dDsts, dDstCapacities, dCSizes, dSrcs, dSrcSizes,
                       [&](const BlockDescs& g) { return launch_fse_encode_blocks(g, false, maxSymbolValue, tableLog, (cudaStream_t)stream); });
}
FSEB_API size_t FSEB200_FSE_decompress_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstCapacities, size_t* dResults,
                                              const void* const* dCSrcs, const size_t* dCSrcSizes, void* stream)
{
    return blocks_call(nBlocks, dDsts, dDstCapacities, dResults, dCSrcs, dCSrcSizes,
                       [&](const BlockDescs& g) { return launch_fse_decode_blocks(g, false, (cudaStream_t)stream); });
}
FSEB_API size_t FSEB200_FSEU16_compress_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstCapacities, size_t* dCSizes,
                                               const void* const* dSrcs, const size_t* dSrcSizes, unsigned maxSymbolValue, unsigned tableLog, void* stream)
{
    return blocks_call(nBlocks, dDsts, dDstCapacities, dCSizes, dSrcs, dSrcSizes,
                       [&](const BlockDescs& g) { return launch_fse_encode_blocks(g, true, maxSymbolValue, tableLog, (cudaStream_t)stream); });
}
FSEB_API size_t FSEB200_FSEU16_decompress_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstCapacities, size_t* dResults,
                                                 const void* const* dCSrcs, const size_t* dCSrcSizes, void* stream)
{
    return blocks_call(nBlocks, dDsts, dDstCapacities, dResults, dCSrcs, dCSrcSizes,
                       [&](const BlockDescs& g) { return launch_fse_decode_blocks(g, true, (cudaStream_t)stream); });
}

// Packed FSE / FSE-U16 blocks (include/fse_b200.h): the descriptor codecs with every block stored back to back in one buffer.
namespace {
size_t fse_packed(size_t nBlocks, void* dOut, size_t outCapacity, size_t* dOffsets, size_t* dCSizes, const void* const* dSrcs,
                  const size_t* dSrcSizes, unsigned msv, unsigned tlog, void* dWork, size_t workSize, bool wide, void* stream)
{
    if (nBlocks == 0) return 0;
    if (nBlocks > 0xFFFFFFFFull || !dOut || !dOffsets || !dCSizes || !dSrcs || !dSrcSizes || !dWork) return (size_t)err(E_SRC_WRONG);
    return ok_or_generic(launch_fse_compress_packed((u8*)dOut, outCapacity, (u64*)dOffsets, (u64*)dCSizes, (const u8* const*)dSrcs,
                                                    (const u64*)dSrcSizes, (u32)nBlocks, (u8*)dWork, workSize, wide, msv, tlog,
                                                    (cudaStream_t)stream));
}
}
FSEB_API size_t FSEB200_FSE_compress_packed(size_t nBlocks, void* dOut, size_t outCapacity, size_t* dOffsets, size_t* dCSizes,
                                            const void* const* dSrcs, const size_t* dSrcSizes, unsigned maxSymbolValue, unsigned tableLog,
                                            void* dWork, size_t workSize, void* stream)
{
    return fse_packed(nBlocks, dOut, outCapacity, dOffsets, dCSizes, dSrcs, dSrcSizes, maxSymbolValue, tableLog, dWork, workSize, false, stream);
}
FSEB_API size_t FSEB200_FSEU16_compress_packed(size_t nBlocks, void* dOut, size_t outCapacity, size_t* dOffsets, size_t* dCSizes,
                                               const void* const* dSrcs, const size_t* dSrcSizes, unsigned maxSymbolValue, unsigned tableLog,
                                               void* dWork, size_t workSize, void* stream)
{
    return fse_packed(nBlocks, dOut, outCapacity, dOffsets, dCSizes, dSrcs, dSrcSizes, maxSymbolValue, tableLog, dWork, workSize, true, stream);
}
FSEB_API size_t FSEB200_FSE_packed_workspace(size_t nBlocks, size_t srcBytes) { return srcBytes + (srcBytes >> 7) + 524 * nBlocks; }
FSEB_API size_t FSEB200_FSE_decompress_packed(size_t nBlocks, void* const* dDsts, const size_t* dDstSizes, size_t* dResults,
                                              const void* dIn, const size_t* dOffsets, void* stream)
{
    return unpacked_call(nBlocks, dDsts, dDstSizes, dResults, dIn, dOffsets,
                         [&](auto... a) { return launch_fse_decompress_packed(a..., false, (cudaStream_t)stream); });
}
FSEB_API size_t FSEB200_FSEU16_decompress_packed(size_t nBlocks, void* const* dDsts, const size_t* dDstSizes, size_t* dResults,
                                                 const void* dIn, const size_t* dOffsets, void* stream)
{
    return unpacked_call(nBlocks, dDsts, dDstSizes, dResults, dIn, dOffsets,
                         [&](auto... a) { return launch_fse_decompress_packed(a..., true, (cudaStream_t)stream); });
}

FSEB_API size_t FSEB200_batch_blocks(size_t total, size_t blockSize) { return blockSize ? (total + blockSize - 1) / blockSize : 0; }
FSEB_API int FSEB200_device_count(void) { int n = 0; return cudaGetDeviceCount(&n) == cudaSuccess ? n : 0; }

// ================================================================================================
// tier 2a: scalar helpers (host arithmetic only)
// ================================================================================================
FSEB_API unsigned FSE_versionNumber(void) { return 0 * 10000 + 9 * 100 + 0; }                 // lib/fse.h:43-47
FSEB_API size_t FSE_compressBound(size_t size) { return 512 + size + (size >> 7) + 4 + sizeof(size_t); }   // lib/fse.h:290-292
FSEB_API size_t HUF_compressBound(size_t size) { return huf_bound(size); }
FSEB_API unsigned FSE_isError(size_t code) { return code > (size_t)err(E_MAXCODE); }          // lib/error_private.h:79
FSEB_API unsigned HUF_isError(size_t code) { return FSE_isError(code); }
FSEB_API unsigned HIST_isError(size_t code) { return FSE_isError(code); }
FSEB_API const char* FSE_getErrorName(size_t code)                                             // lib/error_private.h:92-117
{
    if (!FSE_isError(code)) return "No error detected";
    switch ((unsigned)(0 - code)) {
    case E_GENERIC: return "Error (generic)";
    case E_DST_TOO_SMALL: return "Destination buffer is too small";
    case E_SRC_WRONG: return "Src size is incorrect";
    case E_CORRUPT: return "Corrupted block detected";
    case E_TLOG_TOO_LARGE: return "tableLog requires too much memory : unsupported";
    case E_MSV_TOO_LARGE: return "Unsupported max Symbol Value : too large";
    case E_MSV_TOO_SMALL: return "Specified maxSymbolValue is too small";
    case E_WKSP_TOO_SMALL: return "workspace buffer is too small";
    default: return "Unspecified error code";
    }
}
FSEB_API const char* HUF_getErrorName(size_t code) { return FSE_getErrorName(code); }

static unsigned optimal_tablelog_h(unsigned maxTableLog, size_t srcSize, unsigned msv, unsigned minus)   // lib/fse_compress.c:316-342
{
    unsigned const bySrc = hibit_h((unsigned)(srcSize - 1)) - minus;
    unsigned const a = hibit_h((unsigned)srcSize) + 1, b = hibit_h(msv) + 2;
    unsigned const floorBits = a < b ? a : b;
    unsigned tl = maxTableLog ? maxTableLog : FSE_DEF_TLOG;
    if (bySrc < tl) tl = bySrc;
    if (floorBits > tl) tl = floorBits;
    if (tl < FSE_MIN_TLOG) tl = FSE_MIN_TLOG;
    if (tl > FSE_MAX_TLOG) tl = FSE_MAX_TLOG;
    return tl;
}
FSEB_API unsigned FSE_optimalTableLog(unsigned maxTableLog, size_t srcSize, unsigned msv) { return optimal_tablelog_h(maxTableLog, srcSize, msv, 2); }
FSEB_API unsigned FSE_optimalTableLog_internal(unsigned maxTableLog, size_t srcSize, unsigned msv, unsigned minus) { return optimal_tablelog_h(maxTableLog, srcSize, msv, minus); }
FSEB_API unsigned HUF_optimalTableLog(unsigned maxTableLog, size_t srcSize, unsigned msv) { return optimal_tablelog_h(maxTableLog, srcSize, msv, 1); }
FSEB_API size_t FSE_NCountWriteBound(unsigned msv, unsigned tl) { return msv ? (((size_t)(msv + 1) * tl) >> 3) + 3 : 512; }   // lib/fse_compress.c:186-190

FSEB_API unsigned HUF_selectDecoder(size_t dstSize, size_t cSrcSize)                            // lib/huf_decompress.c:1001-1051
{
    static const unsigned short cost[16][4] = {
        {0, 0, 1, 1}, {0, 0, 1, 1}, {38, 130, 1313, 74}, {448, 128, 1353, 74}, {556, 128, 1353, 74},
        {714, 128, 1418, 74}, {883, 128, 1437, 74}, {897, 128, 1515, 75}, {926, 128, 1613, 75},
        {947, 128, 1729, 77}, {1107, 128, 2083, 81}, {1177, 128, 2379, 87}, {1242, 128, 2415, 93},
        {1349, 128, 2644, 106}, {1455, 128, 2422, 124}, {722, 128, 1891, 145} };
    unsigned const q = (cSrcSize >= dstSize) ? 15 : (unsigned)(cSrcSize * 16 / dstSize);
    unsigned const d256 = (unsigned)(dstSize >> 8);
    unsigned const t0 = cost[q][0] + cost[q][1] * d256;
    unsigned t1 = cost[q][2] + cost[q][3] * d256;
    t1 += t1 >> 3;
    return t1 < t0;
}

FSEB_API unsigned* FSE_createCTable(unsigned msv, unsigned tl)                                  // lib/fse_compress.c:305-312
{ if (tl > FSE_ABS_TLOG) tl = FSE_ABS_TLOG; return (unsigned*)std::malloc((1 + ((size_t)1 << (tl - 1)) + ((size_t)msv + 1) * 2) * sizeof(unsigned)); }
FSEB_API void FSE_freeCTable(unsigned* ct) { std::free(ct); }
FSEB_API unsigned* FSE_createDTable(unsigned tl)                                                // lib/fse_decompress.c:57-66
{ if (tl > FSE_ABS_TLOG) tl = FSE_ABS_TLOG; return (unsigned*)std::malloc((1 + ((size_t)1 << tl)) * sizeof(unsigned)); }
FSEB_API void FSE_freeDTable(unsigned* dt) { std::free(dt); }

// ================================================================================================
// tier 2b: one block per call, host pointers
// ================================================================================================
FSEB_API size_t FSE_compress2(void* dst, size_t cap, const void* src, size_t n, unsigned msv, unsigned tl)     // lib/fse.h:105
{
    if (n > FSE_ONE_BLOCK_MAX) return (size_t)err(E_SRC_WRONG);         // the kernels index a block with 32 bits
    return one_block_compress(launch_fse_encode, dst, cap, src, n, msv, tl, false);
}
FSEB_API size_t FSE_compress(void* dst, size_t cap, const void* src, size_t n)                                    // lib/fse.h:67 -> (255, 11)
{ return FSE_compress2(dst, cap, src, n, FSE_MAX_SV, FSE_DEF_TLOG); }
FSEB_API size_t FSE_decompress(void* dst, size_t cap, const void* cSrc, size_t cSize)                             // lib/fse.h:80
{
    if (cap > FSE_ONE_BLOCK_MAX || cSize > FSE_ONE_BLOCK_MAX) return (size_t)err(E_SRC_WRONG);
    return one_block_decompress(launch_fse_decode, dst, cap, cSrc, cSize);
}

FSEB_API size_t HUF_compress2(void* dst, size_t cap, const void* src, size_t n, unsigned msv, unsigned tl)      // lib/huf.h:86
{
    if (!n) return 0;                                                   // huf_compress.c:656
    if (!cap) return 0;
    if (n > HUF_BLOCK_MAX) return (size_t)err(E_SRC_WRONG);
    return one_block_compress(launch_huf_encode, dst, cap, src, n, msv, tl, true);
}
FSEB_API size_t HUF_compress(void* dst, size_t cap, const void* src, size_t n) { return HUF_compress2(dst, cap, src, n, 255, HUF_DEF_TLOG); }   // lib/huf.h:54
FSEB_API size_t HUF_compress4X_wksp(void* dst, size_t cap, const void* src, size_t n, unsigned msv, unsigned tl, void* wksp, size_t wkspSize)
{
    if (((size_t)wksp & 3) != 0) return (size_t)err(E_GENERIC);        // huf_compress.c:652-653
    if (wkspSize < (6 << 10)) return (size_t)err(E_WKSP_TOO_SMALL);
    return HUF_compress2(dst, cap, src, n, msv, tl);
}
FSEB_API size_t HUF_decompress(void* dst, size_t dstSize, const void* cSrc, size_t cSrcSize)                     // lib/huf.h:67
{
    if (dstSize == 0) return (size_t)err(E_DST_TOO_SMALL);
    if (dstSize > HUF_BLOCK_MAX) return (size_t)err(E_SRC_WRONG);      // kernels are sized for HUF_BLOCKSIZE_MAX (lib/huf.h:72)
    return one_block_decompress(huf_dec_std, dst, dstSize, cSrc, cSrcSize);
}
// Both regenerate identical bytes for valid input; on malformed input each returns its CPU namesake's verdict (the batch
// decoder runs the single-symbol rules, huf_x2_fixup.cu re-examines what those reject under the double-symbol rules).
FSEB_API size_t HUF_decompress4X1(void* dst, size_t dstSize, const void* cSrc, size_t cSrcSize)                  // lib/huf.h:155
{
    if (dstSize > HUF_BLOCK_MAX) return (size_t)err(E_SRC_WRONG);
    return one_block_decompress(huf_dec_4x1, dst, dstSize, cSrc, cSrcSize);   // never treats the input as raw / RLE (huf_decompress.c:416-449)
}
FSEB_API size_t HUF_decompress4X2(void* dst, size_t dstSize, const void* cSrc, size_t cSrcSize)                  // lib/huf.h:160
{
    if (dstSize > HUF_BLOCK_MAX) return (size_t)err(E_SRC_WRONG);
    return one_block_decompress(huf_dec_4x2, dst, dstSize, cSrc, cSrcSize);
}

FSEB_API size_t FSE_compressU16(void* dst, size_t cap, const unsigned short* src, size_t n, unsigned msv, unsigned tl)   // lib/fseU16.h:75
{
    if (n <= 1) return n;
    if (n > FSE_ONE_BLOCK_MAX / 2) return (size_t)err(E_SRC_WRONG);
    return one_block_compress(launch_fseu16_encode, dst, cap, src, n * 2, msv, tl, false);
}
FSEB_API size_t FSE_decompressU16(unsigned short* dst, size_t cap, const void* cSrc, size_t cSize)                 // lib/fseU16.h:79
{
    if (cSize < 2) return (size_t)err(E_SRC_WRONG);
    if (cap > FSE_ONE_BLOCK_MAX / 2 || cSize > FSE_ONE_BLOCK_MAX) return (size_t)err(E_SRC_WRONG);
    size_t const r = one_block_decompress(launch_fseu16_decode, dst, cap * 2, cSrc, cSize);
    return FSE_isError(r) ? r : r / 2;
}

// ================================================================================================
// tier 2c: statistics and tables, host pointers (single-CTA kernels, micro.cu)
// ================================================================================================
FSEB_API size_t HIST_count(unsigned* count, unsigned* msvPtr, const void* src, size_t n)                          // lib/hist.h:30
{
    Workspace& w = ws();
    std::lock_guard<std::mutex> lock(w.mu);
    unsigned char* dS = (unsigned char*)w.get(0, n);
    u32* dOut = (u32*)w.get(1, 260 * sizeof(u32));
    u64* dR = (u64*)w.get(2, 2 * sizeof(u64));
    unsigned const declared = *msvPtr > 255 ? 255 : *msvPtr;
    u32 out[257]; u64 r = 0;
    if (n) CK(cudaMemcpyAsync(dS, src, n, cudaMemcpyHostToDevice, w.stream));
    CK(launch_hist(dS, n, declared, dOut, dR, w.stream));
    CK(cudaMemcpyAsync(&r, dR, sizeof(r), cudaMemcpyDeviceToHost, w.stream));
    CK(cudaMemcpyAsync(out, dOut, sizeof(out), cudaMemcpyDeviceToHost, w.stream));
    CK(cudaStreamSynchronize(w.stream));
    if (is_err(r)) return (size_t)r;
    std::memcpy(count, out, (declared + 1) * sizeof(unsigned));
    *msvPtr = out[256];
    return (size_t)r;
}
FSEB_API size_t HIST_countFast(unsigned* count, unsigned* msvPtr, const void* src, size_t n) { return HIST_count(count, msvPtr, src, n); }
FSEB_API unsigned HIST_count_simple(unsigned* count, unsigned* msvPtr, const void* src, size_t n) { return (unsigned)HIST_count(count, msvPtr, src, n); }
FSEB_API size_t HIST_count_wksp(unsigned* count, unsigned* msvPtr, const void* src, size_t n, void* wksp, size_t wkspSize)
{
    if ((size_t)wksp & 3) return (size_t)err(E_GENERIC);                // hist.c:167-168
    if (wkspSize < 1024 * sizeof(unsigned)) return (size_t)err(E_WKSP_TOO_SMALL);
    return HIST_count(count, msvPtr, src, n);
}
FSEB_API size_t HIST_countFast_wksp(unsigned* count, unsigned* msvPtr, const void* src, size_t n, void* wksp, size_t wkspSize)
{ return HIST_count_wksp(count, msvPtr, src, n, wksp, wkspSize); }

FSEB_API size_t FSE_countU16(unsigned* count, unsigned* msvPtr, const unsigned short* src, size_t n)                   // lib/fseU16.c:121-145
{
    unsigned const declared = *msvPtr > 65535u ? 65535u : *msvPtr;       // a 16-bit symbol cannot exceed it
    if (n > FSE_ONE_BLOCK_MAX / 2) return (size_t)err(E_SRC_WRONG);
    Workspace& w = ws();
    std::lock_guard<std::mutex> lock(w.mu);
    unsigned char* dS = (unsigned char*)w.get(0, n * 2);
    u32* dOut = (u32*)w.get(1, ((size_t)declared + 2) * sizeof(u32));
    u64* dR = (u64*)w.get(2, 2 * sizeof(u64));
    u64 r = 0; u32 top = 0;
    if (n) CK(cudaMemcpyAsync(dS, src, n * 2, cudaMemcpyHostToDevice, w.stream));
    CK(launch_hist16(dS, n, declared, dOut, dR, w.stream));
    CK(cudaMemcpyAsync(&r, dR, sizeof(r), cudaMemcpyDeviceToHost, w.stream));
    CK(cudaMemcpyAsync(count, dOut, ((size_t)declared + 1) * sizeof(u32), cudaMemcpyDeviceToHost, w.stream));
    CK(cudaMemcpyAsync(&top, dOut + declared + 1, sizeof(top), cudaMemcpyDeviceToHost, w.stream));
    CK(cudaStreamSynchronize(w.stream));
    if (*msvPtr > declared) std::memset(count + declared + 1, 0, ((size_t)*msvPtr - declared) * sizeof(unsigned));
    if (is_err(r)) return (size_t)r;
    *msvPtr = top;
    return (size_t)r;
}

FSEB_API size_t FSE_normalizeCount(short* norm, unsigned tl, const unsigned* count, size_t total, unsigned msv)   // lib/fse.h:147
{
    if (msv > 4095) return (size_t)err(E_MSV_TOO_LARGE);
    Micro m; m.up(0, count, (msv + 1) * sizeof(unsigned));
    u64 const r = m.run(MOP_NORMALIZE, tl, total, msv);
    if (!is_err(r)) m.down(norm, MICRO_OUT, (msv + 1) * sizeof(short));
    return (size_t)r;
}
FSEB_API size_t FSE_writeNCount(void* buffer, size_t bufferSize, const short* norm, unsigned msv, unsigned tl)     // lib/fse.h:157
{
    if (msv > 1023) return (size_t)err(E_MSV_TOO_LARGE);
    Micro m; m.up(0, norm, (msv + 1) * sizeof(short));
    size_t const cap = bufferSize > 60000 ? 60000 : bufferSize;
    u64 const r = m.run(MOP_WRITE_NCOUNT, cap, msv, tl);
    if (!is_err(r)) m.down(buffer, MICRO_OUT, (size_t)r);
    return (size_t)r;
}
FSEB_API size_t FSE_readNCount(short* norm, unsigned* msvPtr, unsigned* tlPtr, const void* hdr, size_t hbSize)     // lib/fse.h:227
{
    if (*msvPtr > 1023) return (size_t)err(E_MSV_TOO_LARGE);
    Micro m;
    size_t const take = hbSize > 4000 ? 4000 : hbSize;                  // a header never exceeds FSE_NCOUNTBOUND (512)
    m.up(0, hdr, take);
    u64 const r = m.run(MOP_READ_NCOUNT, take, *msvPtr);
    unsigned const declared = *msvPtr;
    unsigned meta[2] = { 0, 0 };
    m.down(meta, MICRO_META, sizeof(meta));
    *tlPtr = meta[1];
    if (is_err(r)) { m.down(norm, MICRO_OUT, (declared + 1) * sizeof(short)); return (size_t)r; }
    m.down(norm, MICRO_OUT, (declared + 1) * sizeof(short));
    *msvPtr = meta[0];
    return (size_t)r;
}
FSEB_API size_t FSE_buildCTable(unsigned* ct, const short* norm, unsigned msv, unsigned tl)                          // lib/fse.h:163
{
    if (msv > FSE_MAX_SV) return (size_t)err(E_MSV_TOO_LARGE);
    Micro m; m.up(0, norm, (msv + 1) * sizeof(short));
    u64 const r = m.run(MOP_BUILD_CTABLE, msv, tl);
    if (!is_err(r)) m.down(ct, MICRO_OUT, (1 + (tl ? ((size_t)1 << (tl - 1)) : 1) + ((size_t)msv + 1) * 2) * sizeof(unsigned));
    return (size_t)r;
}
FSEB_API size_t FSE_buildDTable(unsigned* dt, const short* norm, unsigned msv, unsigned tl)                          // lib/fse.h:240
{
    if (msv > FSE_MAX_SV) return (size_t)err(E_MSV_TOO_LARGE);
    if (tl > FSE_MAX_TLOG) return (size_t)err(E_TLOG_TOO_LARGE);
    Micro m; m.up(0, norm, (msv + 1) * sizeof(short));
    u64 const r = m.run(MOP_BUILD_DTABLE, msv, tl, 0);
    if (!is_err(r)) m.down(dt, MICRO_OUT, (1 + ((size_t)1 << tl)) * sizeof(unsigned));
    return (size_t)r;
}
FSEB_API size_t HUF_buildCTable(unsigned* ctable, const unsigned* count, unsigned msv, unsigned maxNbBits)            // lib/huf.h:188
{
    if (msv > HUF_MAX_SV) return (size_t)err(E_MSV_TOO_LARGE);
    unsigned cnt[256];
    std::memcpy(cnt, count, (msv + 1) * sizeof(unsigned));             // CTable and count may overlap (huf.h:188 note)
    Micro m; m.up(0, cnt, (msv + 1) * sizeof(unsigned));
    u64 const r = m.run(MOP_HUF_BUILD_CTABLE, msv, maxNbBits);
    if (!is_err(r)) m.down(ctable, MICRO_OUT, (msv + 1) * sizeof(unsigned));
    return (size_t)r;
}
FSEB_API size_t HUF_writeCTable(void* dst, size_t maxDstSize, const unsigned* ctable, unsigned msv, unsigned huffLog)  // lib/huf.h:189
{
    if (msv > HUF_MAX_SV) return (size_t)err(E_MSV_TOO_LARGE);
    Micro m; m.up(0, ctable, (msv + 1) * sizeof(unsigned));
    u64 const r = m.run(MOP_HUF_WRITE_CTABLE, maxDstSize, msv, huffLog);
    if (!is_err(r)) m.down(dst, MICRO_OUT, (size_t)r);
    return (size_t)r;
}
FSEB_API size_t HUF_readStats(unsigned char* huffWeight, size_t hwSize, unsigned* rankStats, unsigned* nbSymbolsPtr,
                              unsigned* tableLogPtr, const void* src, size_t srcSize)                                   // lib/huf.h:225
{
    if (hwSize > 4000) hwSize = 4000;
    Micro m;
    size_t const take = srcSize > 256 ? 256 : srcSize;                  // a tree header never exceeds HUF_CTABLEBOUND (129)
    m.up(0, src, take);
    u64 const r = m.run(MOP_HUF_READ_STATS, take, hwSize);
    if (is_err(r)) return (size_t)r;
    unsigned meta[2];
    m.down(meta, MICRO_META_HUF, sizeof(meta));
    m.down(rankStats, MICRO_META, 13 * sizeof(unsigned));
    m.down(huffWeight, MICRO_OUT, meta[0]);
    *nbSymbolsPtr = meta[0]; *tableLogPtr = meta[1];
    return (size_t)r;
}
FSEB_API size_t HUF_readDTableX1(unsigned* DTable, const void* src, size_t srcSize)                                    // lib/huf.h:267
{
    Micro m;
    size_t const take = srcSize > 256 ? 256 : srcSize;
    m.up(0, src, take);
    u64 const r = m.run(MOP_HUF_READ_DTABLE_X1, take, DTable[0]);
    if (is_err(r)) return (size_t)r;
    unsigned hdr = 0;
    m.down(&hdr, MICRO_DTABLE_X1, sizeof(hdr));
    unsigned const tl = (hdr >> 16) & 0xFF;
    m.down(DTable, MICRO_DTABLE_X1, sizeof(unsigned) + ((size_t)1 << tl) * 2);
    return (size_t)r;
}

// ---- CTable inspection helpers (lib/huf.h:196-199,221): arithmetic on the 4-byte cells {U16 val; BYTE nbBits} ----
FSEB_API unsigned HUF_getNbBits(const void* symbolTable, unsigned symbolValue)                                      // huf_compress.c:200-205
{ return (((const unsigned*)symbolTable)[symbolValue] >> 16) & 0xFF; }
FSEB_API size_t HUF_estimateCompressedSize(const unsigned* CTable, const unsigned* count, unsigned maxSymbolValue)  // huf_compress.c:422-430
{
    size_t nbBits = 0;
    for (unsigned s = 0; s <= maxSymbolValue; s++) nbBits += (size_t)((CTable[s] >> 16) & 0xFF) * count[s];
    return nbBits >> 3;
}
FSEB_API int HUF_validateCTable(const unsigned* CTable, const unsigned* count, unsigned maxSymbolValue)             // huf_compress.c:432-439
{
    int bad = 0;
    for (unsigned s = 0; s <= maxSymbolValue; s++) bad |= (count[s] != 0) & (((CTable[s] >> 16) & 0xFF) == 0);
    return !bad;
}

// ---- constant-pattern tables for stored / single-symbol blocks (lib/fse.h:330-345 ; fse_compress.c:498-551, fse_decompress.c:134-176).
//      Pure fills of the ABI table layouts: host arithmetic like the other scalar helpers, no data path involved. ----
FSEB_API size_t FSE_buildCTable_raw(unsigned* ct, unsigned nbBits)
{
    if (nbBits < 1) return (size_t)err(E_GENERIC);
    if (nbBits > 15) return (size_t)err(E_TLOG_TOO_LARGE);               // the reference would overflow its U16 cells
    unsigned const tableSize = 1u << nbBits;
    unsigned short* const t16 = reinterpret_cast<unsigned short*>(ct) + 2;
    unsigned* const tt = ct + 1 + (tableSize >> 1);
    t16[-2] = (unsigned short)nbBits; t16[-1] = (unsigned short)(tableSize - 1);
    for (unsigned s = 0; s < tableSize; s++) t16[s] = (unsigned short)(tableSize + s);
    for (unsigned s = 0; s < tableSize; s++) { tt[2 * s] = s - 1; tt[2 * s + 1] = (nbBits << 16) - tableSize; }
    return 0;
}
FSEB_API size_t FSE_buildCTable_rle(unsigned* ct, unsigned char symbolValue)
{
    unsigned short* const t16 = reinterpret_cast<unsigned short*>(ct) + 2;
    unsigned* const tt = ct + 2;
    t16[-2] = 0; t16[-1] = symbolValue; t16[0] = 0; t16[1] = 0;
    tt[2 * symbolValue] = 0; tt[2 * symbolValue + 1] = 0;
    return 0;
}
FSEB_API size_t FSE_buildDTable_rle(unsigned* dt, unsigned char symbolValue)
{
    dt[0] = 0;                                                            // tableLog 0, fastMode 0
    dt[1] = (unsigned)symbolValue << 16;                                  // { newState 0, symbol, nbBits 0 }
    return 0;
}
FSEB_API size_t FSE_buildDTable_raw(unsigned* dt, unsigned nbBits)
{
    if (nbBits < 1) return (size_t)err(E_GENERIC);
    if (nbBits > 15) return (size_t)err(E_TLOG_TOO_LARGE);
    dt[0] = nbBits | (1u << 16);                                          // fastMode 1
    for (unsigned s = 0; s < (1u << nbBits); s++) dt[1 + s] = ((s & 0xFF) << 16) | (nbBits << 24);
    return 0;
}

// ---- payload coding with a caller-supplied table (the tables are ABI: fse.h:295-296,483-486,565-575 ; huf.h:136-149) ----
namespace {
constexpr size_t MICRO_MAX = (size_t)1 << 24;                           // single-call payloads above 16 MiB are refused (use the batch tier)
size_t al16(size_t v) { return (v + 15) & ~(size_t)15; }
// A caller's HUF_CElt table has HUF_CTABLE_SIZE_U32(maxSymbolValue) = maxSymbolValue+1 cells (lib/huf.h:136-139) and nothing tells
// us maxSymbolValue: read only the cells the payload can index (up to its largest byte) and hand the device a zero-padded 256-cell image.
void ctable_image(unsigned (&full)[256], const unsigned* CTable, const void* src, size_t srcSize)
{
    unsigned top = 0;
    const unsigned char* const p = (const unsigned char*)src;
    for (size_t i = 0; i < srcSize; i++) top = p[i] > top ? p[i] : top;
    std::memset(full, 0, sizeof(full));
    std::memcpy(full, CTable, ((size_t)top + 1) * sizeof(unsigned));
}
// HUF_compress{4,1}X_usingCTable: the output area, then `stages` private areas of the same size behind it (4X: one per stream).
size_t huf_encode_using_ctable(int opcode, size_t stages, void* dst, size_t dstSize, const void* src, size_t srcSize, const unsigned* CTable)
{
    if (srcSize > MICRO_MAX) return (size_t)err(E_SRC_WRONG);
    size_t const cap = dstSize < 2 * srcSize + 64 ? dstSize : 2 * srcSize + 64;
    size_t const outOff = MICRO_PAYLOAD + al16(srcSize + 16);
    Micro m(outOff + (1 + stages) * al16(cap) + 64);
    unsigned full[256]; ctable_image(full, CTable, src, srcSize);
    m.up(0, full, sizeof(full)); m.up(MICRO_PAYLOAD, src, srcSize);
    u64 const r = m.run(opcode, srcSize, cap, MICRO_PAYLOAD, outOff);
    if (!is_err(r) && r) m.down(dst, outOff, (size_t)r);
    return (size_t)r;
}
// HUF_decompress{4,1}X{1,2}_usingDTable: the DTable must be of `type` (0: X1, huf_decompress.c:367,434 ; 1: X2, :866,910); its
// image is the header word and 2^tableLog cells of cellBytes each.  On success the whole output capacity is copied back.
size_t huf_decode_using_dtable(int opcode, unsigned type, size_t cellBytes, void* dst, size_t maxDstSize, const void* cSrc, size_t cSrcSize,
                               const unsigned* DTable)
{
    unsigned const t = (DTable[0] >> 8) & 0xFF, tl = (DTable[0] >> 16) & 0xFF;
    if (t != type) return (size_t)err(E_GENERIC);
    if (tl > HUF_MAX_TLOG) return (size_t)err(E_TLOG_TOO_LARGE);
    if (cSrcSize > MICRO_MAX || maxDstSize > MICRO_MAX) return (size_t)err(E_SRC_WRONG);
    size_t const outOff = MICRO_PAYLOAD + al16(cSrcSize + 16);
    Micro m(outOff + maxDstSize + 64);
    m.up(0, DTable, sizeof(unsigned) + (cellBytes << tl)); m.up(MICRO_PAYLOAD, cSrc, cSrcSize);
    u64 const r = m.run(opcode, cSrcSize, maxDstSize, MICRO_PAYLOAD, outOff);
    if (!is_err(r)) m.down(dst, outOff, maxDstSize);
    return (size_t)r;
}
}
FSEB_API size_t FSE_compress_usingCTable(void* dst, size_t dstSize, const void* src, size_t srcSize, const unsigned* ct)   // lib/fse.h:222
{
    unsigned const tl = ct[0] & 0xFFFF, msv = ct[0] >> 16;
    if (tl > FSE_MAX_TLOG) return (size_t)err(E_TLOG_TOO_LARGE);
    if (msv > FSE_MAX_SV) return (size_t)err(E_MSV_TOO_LARGE);
    if (srcSize > MICRO_MAX) return (size_t)err(E_SRC_WRONG);
    size_t const cap = dstSize < 2 * srcSize + 64 ? dstSize : 2 * srcSize + 64;     // <= 12 bits per symbol: more room can never be used
    size_t const ctBytes = (1 + (tl ? ((size_t)1 << (tl - 1)) : 1) + 2 * ((size_t)msv + 1)) * sizeof(unsigned);   // FSE_CTABLE_SIZE_U32 ; rle tables: fse_compress.c:532
    size_t const outOff = MICRO_PAYLOAD + al16(srcSize + 16);
    Micro m(outOff + cap + 64);
    m.up(0, ct, ctBytes); m.up(MICRO_PAYLOAD, src, srcSize);
    u64 const r = m.run(MOP_FSE_ENCODE_CT, srcSize, cap, MICRO_PAYLOAD, outOff);
    if (!is_err(r) && r) m.down(dst, outOff, (size_t)r);
    return (size_t)r;
}
FSEB_API size_t FSE_decompress_usingDTable(void* dst, size_t maxDstSize, const void* cSrc, size_t cSrcSize, const unsigned* dt)   // lib/fse.h:247
{
    unsigned const tl = dt[0] & 0xFFFF;
    if (tl > FSE_MAX_TLOG) return (size_t)err(E_TLOG_TOO_LARGE);
    if (cSrcSize > MICRO_MAX || maxDstSize > MICRO_MAX) return (size_t)err(E_SRC_WRONG);
    size_t const outOff = MICRO_PAYLOAD + al16(cSrcSize + 16);
    Micro m(outOff + maxDstSize + 64);
    m.up(0, dt, (1 + ((size_t)1 << tl)) * sizeof(unsigned)); m.up(MICRO_PAYLOAD, cSrc, cSrcSize);
    u64 const r = m.run(MOP_FSE_DECODE_DT, cSrcSize, maxDstSize, MICRO_PAYLOAD, outOff);
    if (!is_err(r) && r) m.down(dst, outOff, (size_t)r);
    return (size_t)r;
}
FSEB_API size_t HUF_compress4X_usingCTable(void* dst, size_t dstSize, const void* src, size_t srcSize, const unsigned* CTable)   // lib/huf.h:191
{ return huf_encode_using_ctable(MOP_HUF_ENCODE4X_CT, 4, dst, dstSize, src, srcSize, CTable); }
FSEB_API size_t HUF_decompress4X1_usingDTable(void* dst, size_t maxDstSize, const void* cSrc, size_t cSrcSize, const unsigned* DTable)   // lib/huf.h:277
{ return huf_decode_using_dtable(MOP_HUF_DECODE4X1_DT, 0, 2, dst, maxDstSize, cSrc, cSrcSize, DTable); }
FSEB_API size_t HUF_decompress4X2_usingDTable(void* dst, size_t maxDstSize, const void* cSrc, size_t cSrcSize, const unsigned* DTable)   // lib/huf.h:280
{ return huf_decode_using_dtable(MOP_HUF_DECODE4X2_DT, 1, 4, dst, maxDstSize, cSrc, cSrcSize, DTable); }
FSEB_API size_t HUF_decompress1X2_usingDTable(void* dst, size_t maxDstSize, const void* cSrc, size_t cSrcSize, const unsigned* DTable)   // lib/huf.h:323
{ return huf_decode_using_dtable(MOP_HUF_DECODE1X2_DT, 1, 4, dst, maxDstSize, cSrc, cSrcSize, DTable); }
FSEB_API size_t HUF_decompress4X_usingDTable(void* dst, size_t maxDstSize, const void* cSrc, size_t cSrcSize, const unsigned* DTable)    // lib/huf.h:203
{
    // huf_decompress.c:980-997: dispatch on DTableDesc.tableType
    return ((DTable[0] >> 8) & 0xFF) ? HUF_decompress4X2_usingDTable(dst, maxDstSize, cSrc, cSrcSize, DTable)
                                     : HUF_decompress4X1_usingDTable(dst, maxDstSize, cSrc, cSrcSize, DTable);
}

// ---- single-stream Huff0 (lib/huf.h:288-320): the same device routines with one stream; HUF_compress1X is the reference's
//      driver (huf_compress.c:637-724 with HUF_singleStream) composed from the table-level calls above ----
FSEB_API size_t HUF_compress1X_usingCTable(void* dst, size_t dstSize, const void* src, size_t srcSize, const unsigned* CTable)      // lib/huf.h:290
{ return huf_encode_using_ctable(MOP_HUF_ENCODE1X_CT, 0, dst, dstSize, src, srcSize, CTable); }
FSEB_API size_t HUF_compress1X(void* dst, size_t dstSize, const void* src, size_t srcSize, unsigned maxSymbolValue, unsigned huffLog)   // lib/huf.h:288
{
    unsigned char* const ostart = (unsigned char*)dst;
    if (!srcSize || !dstSize) return 0;                                              // huf_compress.c:656-657
    if (srcSize > HUF_BLOCK_MAX) return (size_t)err(E_SRC_WRONG);
    if (huffLog > HUF_MAX_TLOG) return (size_t)err(E_TLOG_TOO_LARGE);
    if (maxSymbolValue > HUF_MAX_SV) return (size_t)err(E_MSV_TOO_LARGE);
    if (!maxSymbolValue) maxSymbolValue = HUF_MAX_SV;
    if (!huffLog) huffLog = HUF_DEF_TLOG;
    unsigned count[256]; unsigned ctable[256];
    size_t const largest = HIST_count(count, &maxSymbolValue, src, srcSize);
    if (is_err(largest)) return largest;
    if (largest == srcSize) { ostart[0] = ((const unsigned char*)src)[0]; return 1; }   // :673
    if (largest <= (srcSize >> 7) + 4) return 0;                                     // :674
    huffLog = HUF_optimalTableLog(huffLog, srcSize, maxSymbolValue);
    size_t const maxBits = HUF_buildCTable(ctable, count, maxSymbolValue, huffLog);
    if (is_err(maxBits)) return maxBits;
    huffLog = (unsigned)maxBits;
    for (unsigned s = maxSymbolValue + 1; s < 256; s++) ctable[s] = 0;
    size_t const hSize = HUF_writeCTable(ostart, dstSize, ctable, maxSymbolValue, huffLog);
    if (is_err(hSize)) return hSize;
    if (hSize + 12ul >= srcSize) return 0;                                           // :715
    size_t const cSize = HUF_compress1X_usingCTable(ostart + hSize, dstSize - hSize, src, srcSize, ctable);
    if (is_err(cSize)) return cSize;
    if (cSize == 0) return 0;
    if (hSize + cSize >= srcSize - 1) return 0;                                      // :625
    return hSize + cSize;
}
// ---- table reuse, one block per call (lib/huf.h:194-208,291-300): a batch of one through FSEB200_HUF_compress{4X,1X}_repeat_blocks,
//      the caller's table (256 cells) and flag copied in and out.  `repeat` is HUF_repeat {none 0, check 1, valid 2}; a NULL flag
//      acts as none and a NULL table as a zeroed one that is not returned. ----
namespace {
size_t huf_compress_repeat(int nStreams, void* dst, size_t dstSize, const void* src, size_t srcSize, unsigned maxSymbolValue, unsigned huffLog,
                           void* workSpace, size_t wkspSize, unsigned* hufTable, int* repeat, int preferRepeat)
{
    if (((size_t)workSpace & 3) != 0) return (size_t)err(E_GENERIC);                 // huf_compress.c:652-653
    if (wkspSize < (6 << 10)) return (size_t)err(E_WKSP_TOO_SMALL);
    if (!srcSize || !dstSize) return 0;                                              // :656-657, before anything is staged
    if (srcSize > HUF_BLOCK_MAX) return (size_t)err(E_SRC_WRONG);
    Workspace& w = ws();
    std::lock_guard<std::mutex> lock(w.mu);
    size_t const cap = dstSize > 0xFFFFFF00ull ? 0xFFFFFF00ull : dstSize;
    unsigned char* dS = (unsigned char*)w.get(0, srcSize);
    unsigned char* dC = (unsigned char*)w.get(1, cap);
    // descriptor words: dst, capacity, cSize, src, srcSize, table, flag | prefer << 32, then the table's 256 cells
    u64* dA = (u64*)w.get(2, 8 * sizeof(u64) + 256 * sizeof(unsigned));
    u32* const dT = (u32*)(dA + 8);
    struct { u64 a[8]; unsigned t[256]; } h;
    h.a[0] = (u64)dC; h.a[1] = cap; h.a[2] = 0; h.a[3] = (u64)dS; h.a[4] = srcSize; h.a[5] = (u64)dT;
    h.a[6] = (u64)(u32)(repeat ? *repeat : 0) | (u64)(u32)preferRepeat << 32;
    if (hufTable) std::memcpy(h.t, hufTable, sizeof(h.t)); else std::memset(h.t, 0, sizeof(h.t));
    CK(cudaMemcpyAsync(dS, src, srcSize, cudaMemcpyHostToDevice, w.stream));
    CK(cudaMemcpyAsync(dA, &h, sizeof(h), cudaMemcpyHostToDevice, w.stream));
    int* const dFlag = (int*)(dA + 6);
    size_t const r0 = (nStreams == 4 ? FSEB200_HUF_compress4X_repeat_blocks : FSEB200_HUF_compress1X_repeat_blocks)(
        1, (void* const*)dA, (const size_t*)(dA + 1), (size_t*)(dA + 2), (const void* const*)(dA + 3), (const size_t*)(dA + 4),
        (unsigned* const*)(dA + 5), dFlag, dFlag + 1, maxSymbolValue, huffLog, w.stream);
    if (is_err(r0)) return r0;
    CK(cudaMemcpyAsync(&h, dA, sizeof(h), cudaMemcpyDeviceToHost, w.stream));
    CK(cudaStreamSynchronize(w.stream));
    u64 const r = h.a[2];
    if (!is_err(r) && r) CK(cudaMemcpy(dst, dC, (size_t)r, cudaMemcpyDeviceToHost));   // 1: the RLE byte
    if (repeat) *repeat = (int)(u32)h.a[6];
    if (hufTable) std::memcpy(hufTable, h.t, sizeof(h.t));
    return (size_t)r;
}
}
FSEB_API size_t HUF_compress4X_repeat(void* dst, size_t dstSize, const void* src, size_t srcSize, unsigned maxSymbolValue, unsigned tableLog,
                                      void* workSpace, size_t wkspSize, unsigned* hufTable, int* repeat, int preferRepeat, int bmi2)   // lib/huf.h:204
{ (void)bmi2; return huf_compress_repeat(4, dst, dstSize, src, srcSize, maxSymbolValue, tableLog, workSpace, wkspSize, hufTable, repeat, preferRepeat); }
FSEB_API size_t HUF_compress1X_repeat(void* dst, size_t dstSize, const void* src, size_t srcSize, unsigned maxSymbolValue, unsigned tableLog,
                                      void* workSpace, size_t wkspSize, unsigned* hufTable, int* repeat, int preferRepeat, int bmi2)   // lib/huf.h:296
{ (void)bmi2; return huf_compress_repeat(1, dst, dstSize, src, srcSize, maxSymbolValue, tableLog, workSpace, wkspSize, hufTable, repeat, preferRepeat); }

// HUF_readCTable (lib/huf.h:231, huf_compress.c:149-198): the header is parsed on the GPU (HUF_readStats); what remains is the
// O(alphabet) canonical numbering of the codes, host arithmetic like the other table helpers.
FSEB_API size_t HUF_readCTable(unsigned* CTable, unsigned* maxSymbolValuePtr, const void* src, size_t srcSize, unsigned* hasZeroWeights)
{
    unsigned char w[256]; unsigned rank[17]; unsigned nbSym = 0, tl = 0;
    size_t const readSize = HUF_readStats(w, 256, rank, &nbSym, &tl, src, srcSize);
    if (is_err(readSize)) return readSize;
    if (tl > HUF_MAX_TLOG) return (size_t)err(E_TLOG_TOO_LARGE);
    if (nbSym > *maxSymbolValuePtr + 1) return (size_t)err(E_MSV_TOO_SMALL);
    unsigned nbBits[256]; unsigned short perRank[HUF_MAX_TLOG + 2] = { 0 }, valPerRank[HUF_MAX_TLOG + 2] = { 0 };
    *hasZeroWeights = 0;
    for (unsigned n = 0; n < nbSym; n++) { *hasZeroWeights |= (w[n] == 0); nbBits[n] = w[n] ? (tl + 1 - w[n]) & 0xFF : 0; perRank[nbBits[n]]++; }
    {   unsigned short mn = 0;
        for (unsigned n = tl; n > 0; n--) { valPerRank[n] = mn; mn = (unsigned short)(mn + perRank[n]); mn >>= 1; }
    }
    for (unsigned n = 0; n < nbSym; n++) CTable[n] = (unsigned)(valPerRank[nbBits[n]]++) | (nbBits[n] << 16);
    *maxSymbolValuePtr = nbSym - 1;
    return readSize;
}

FSEB_API size_t HUF_decompress1X2(void* dst, size_t dstSize, const void* cSrc, size_t cSrcSize)                                          // lib/huf.h:304
{
    static thread_local unsigned DTable[1 + 4096];
    DTable[0] = 12u * 0x01000001u;                                                  // HUF_CREATE_STATIC_DTABLEX2(DTable, HUF_TABLELOG_MAX)
    size_t const hSize = HUF_readDTableX2(DTable, cSrc, cSrcSize);
    if (is_err(hSize)) return hSize;
    if (hSize >= cSrcSize) return (size_t)err(E_SRC_WRONG);                         // huf_decompress.c:882
    return HUF_decompress1X2_usingDTable(dst, dstSize, (const unsigned char*)cSrc + hSize, cSrcSize - hSize, DTable);
}
FSEB_API size_t HUF_decompress1X_usingDTable_bmi2(void* dst, size_t maxDstSize, const void* cSrc, size_t cSrcSize, const unsigned* DTable, int bmi2)   // lib/huf.h:329
{ (void)bmi2; return HUF_decompress1X_usingDTable(dst, maxDstSize, cSrc, cSrcSize, DTable); }
FSEB_API size_t HUF_decompress4X_usingDTable_bmi2(void* dst, size_t maxDstSize, const void* cSrc, size_t cSrcSize, const unsigned* DTable, int bmi2)   // lib/huf.h:333
{ (void)bmi2; return HUF_decompress4X_usingDTable(dst, maxDstSize, cSrc, cSrcSize, DTable); }

FSEB_API size_t HUF_decompress1X1_usingDTable(void* dst, size_t maxDstSize, const void* cSrc, size_t cSrcSize, const unsigned* DTable)  // lib/huf.h:320
{ return huf_decode_using_dtable(MOP_HUF_DECODE1X1_DT, 0, 2, dst, maxDstSize, cSrc, cSrcSize, DTable); }
FSEB_API size_t HUF_decompress1X_usingDTable(void* dst, size_t maxDstSize, const void* cSrc, size_t cSrcSize, const unsigned* DTable)   // lib/huf.h:318
{
    return ((DTable[0] >> 8) & 0xFF) ? HUF_decompress1X2_usingDTable(dst, maxDstSize, cSrc, cSrcSize, DTable)      // huf_decompress.c:962-977
                                     : HUF_decompress1X1_usingDTable(dst, maxDstSize, cSrc, cSrcSize, DTable);
}
FSEB_API size_t HUF_decompress1X1(void* dst, size_t dstSize, const void* cSrc, size_t cSrcSize)                                          // lib/huf.h:302
{
    unsigned DTable[1 + 2048]; DTable[0] = 11u * 0x01000001u;                       // HUF_CREATE_STATIC_DTABLEX1(DTable, HUF_TABLELOG_MAX)
    size_t const hSize = HUF_readDTableX1(DTable, cSrc, cSrcSize);
    if (is_err(hSize)) return hSize;
    if (hSize >= cSrcSize) return (size_t)err(E_SRC_WRONG);                         // huf_decompress.c:380
    return HUF_decompress1X1_usingDTable(dst, dstSize, (const unsigned char*)cSrc + hSize, cSrcSize - hSize, DTable);
}

FSEB_API size_t HUF_readDTableX2(unsigned* DTable, const void* src, size_t srcSize)                                    // lib/huf.h:268
{
    Micro m;
    size_t const take = srcSize > 256 ? 256 : srcSize;
    m.up(0, src, take);
    u64 const r = m.run(MOP_HUF_READ_DTABLE_X2, take, DTable[0]);
    if (is_err(r)) return (size_t)r;
    unsigned const L = DTable[0] & 0xFF;
    m.down(DTable, MICRO_DTABLE_X2, sizeof(unsigned) * (1 + ((size_t)1 << L)));
    return (size_t)r;
}

// ================================================================================================
// measurement inputs (programs/probaGenerator.c:95-126, programs/fuzzerU16.c:107-134) generated in HBM
// ================================================================================================
FSEB_API size_t FSEB200_probagen(void* dDst, size_t nBytes, size_t streamOffset, double p, void* stream)
{
    unsigned char table[4096];
    int remaining = 4096; unsigned pos = 0, sym = 0;
    if (p == 0.0) p = 0.005;
    if (!(p > 0.0 && p <= 1.0)) return err(E_GENERIC);                  // a probability, not a percentage (the reference's CLI divides by 100)
    while (remaining) {
        unsigned n = (unsigned)(remaining * p);
        if (!n) n = 1;
        unsigned const end = pos + n;
        while (pos < end) table[pos++] = (unsigned char)sym;
        sym++; remaining -= (int)n;
    }
    void* dT = nullptr;
    cudaStream_t st = (cudaStream_t)stream;
    CK(cudaMallocAsync(&dT, sizeof(table), st));
    CK(cudaMemcpyAsync(dT, table, sizeof(table), cudaMemcpyHostToDevice, st));
    cudaError_t const e = launch_gen8(dDst, nBytes, streamOffset, dT, 1u, st);
    CK(cudaStreamSynchronize(st));                                     // `table` lives on this stack frame
    CK(cudaFreeAsync(dT, st));
    return ok_or_generic(e);
}
FSEB_API size_t FSEB200_genU16(void* dDst, size_t nSymbols, size_t streamOffset, unsigned start, double p, unsigned seed, void* stream)
{
    unsigned short table[4096];
    unsigned remaining = 4096, pos = 0; unsigned short v = (unsigned short)start;
    if (!(p >= 0.0 && p <= 1.0)) return err(E_GENERIC);
    while (remaining) {
        unsigned n = (unsigned)(remaining * p) + 1;
        if (n > remaining) n = remaining;
        unsigned const end = pos + n;
        while (pos < end) table[pos++] = v;
        v++; if (v >= U16_MAX_SV) v = 1;
        remaining -= n;
    }
    void* dT = nullptr;
    cudaStream_t st = (cudaStream_t)stream;
    CK(cudaMallocAsync(&dT, sizeof(table), st));
    CK(cudaMemcpyAsync(dT, table, sizeof(table), cudaMemcpyHostToDevice, st));
    cudaError_t const e = launch_gen16(dDst, nSymbols, streamOffset, dT, seed, st);
    CK(cudaStreamSynchronize(st));
    CK(cudaFreeAsync(dT, st));
    return ok_or_generic(e);
}
