// capi.cu -- the C-ABI boundary of libfse_b200.so (declarations: include/fse_b200.h).
//
// Two tiers:
//   1. FSEB200_*_batch : device-pointer, stream-ordered, whole-batch entry points -- what the
//      per-chunk loops of the reference harness (programs/bench.c:353-364 and :389-424) collapse into.
//      FSEB200_{HUF,FSE,FSEU16}_*_blocks: the same for blocks given by per-block device descriptors (common.cuh BlockDescs).
//   2. the reference's own one-block-per-call symbols (lib/fse.h, lib/huf.h, lib/hist.h,
//      lib/fseU16.h) with HOST pointers: they stage the block through a private device workspace and
//      run the same kernels with a batch of one.  Correct drop-ins for unmodified callers; not the
//      fast path (one launch + two PCIe copies per call).
// There is no CPU implementation behind any data-path entry point: without a CUDA device every call
// aborts loudly.  Only scalar helpers (bounds, error names, table-log arithmetic) run on the host.
#include "common.cuh"
#include "micro.h"
#include "fse_b200.h"
#include "launch_util.cuh"
#include "xxh32.h"
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <thread>
#include <vector>

namespace fseb {
cudaError_t launch_huf_decode(const BatchGeom&, void*, const void*, const u64*, u64*, const void*, cudaStream_t, u32 flags);
cudaError_t launch_huf_encode(const BatchGeom&, void*, u64*, const void*, unsigned, unsigned, cudaStream_t);
cudaError_t launch_huf_encode_using_ctable(const BatchGeom&, void*, u64*, const void*, const u32*, cudaStream_t);
cudaError_t launch_huf_encode_blocks(const BlockDescs&, int, unsigned, unsigned, cudaStream_t);
cudaError_t launch_huf_encode_packed(const PackedDescs&, int, unsigned, unsigned, cudaStream_t);
cudaError_t launch_huf_decode_blocks(const BlockDescs&, int, cudaStream_t);
cudaError_t launch_fse_decode(const BatchGeom&, void*, const void*, const u64*, u64*, const void*, cudaStream_t);
cudaError_t launch_fse_encode(const BatchGeom&, void*, u64*, const void*, unsigned, unsigned, cudaStream_t);
cudaError_t launch_fseu16_decode(const BatchGeom&, void*, const void*, const u64*, u64*, const void*, cudaStream_t);
cudaError_t launch_fseu16_encode(const BatchGeom&, void*, u64*, const void*, unsigned, unsigned, cudaStream_t);
cudaError_t launch_fse_encode_blocks(const BlockDescs&, bool, unsigned, unsigned, cudaStream_t);
cudaError_t launch_fse_decode_blocks(const BlockDescs&, bool, cudaStream_t);
cudaError_t launch_fse_compress_packed(u8*, u64, u64*, u64*, const u8* const*, const u64*, u32, u8*, u64, bool, unsigned, unsigned, cudaStream_t);
cudaError_t launch_fse_decompress_packed(u8* const*, const u64*, u64*, const u8*, const u64*, u32, bool, cudaStream_t);
cudaError_t launch_huf_decompress_packed(u8* const*, const u64*, u64*, const u8*, const u64*, u32, int, cudaStream_t);
cudaError_t launch_frame_body(u8*, const u8*, const u64*, const u64*, const u64*, u32, u64, cudaStream_t);
cudaError_t launch_frame_stored(u8*, const u8*, const u64*, u64, cudaStream_t);
cudaError_t launch_hist(const void*, u64, u32, u32*, u64*, cudaStream_t);
cudaError_t launch_hist16(const void*, u64, u32, u32*, u64*, cudaStream_t);
cudaError_t launch_micro(int, const MicroArgs&, void*, u64*, cudaStream_t);
cudaError_t launch_gen8(void*, u64, u64, const void*, u32, cudaStream_t);
cudaError_t launch_gen16(void*, u64, u64, const void*, u32, cudaStream_t);
}

using namespace fseb;

static cudaError_t huf_dec_std(const BatchGeom& g, void* d, const void* c, const u64* cs, u64* r, const void* o, cudaStream_t s) { return launch_huf_decode(g, d, c, cs, r, o, s, 0); }
static cudaError_t huf_dec_4x1(const BatchGeom& g, void* d, const void* c, const u64* cs, u64* r, const void* o, cudaStream_t s) { return launch_huf_decode(g, d, c, cs, r, o, s, 1); }
static cudaError_t huf_dec_4x2(const BatchGeom& g, void* d, const void* c, const u64* cs, u64* r, const void* o, cudaStream_t s) { return launch_huf_decode(g, d, c, cs, r, o, s, 3); }

#define FSEB_API extern "C" __attribute__((visibility("default")))

namespace {

[[noreturn]] void die(const char* what, cudaError_t e)
{
    std::fprintf(stderr, "libfse_b200: %s failed: %s -- this library has no CPU fallback\n", what, cudaGetErrorString(e));
    std::abort();
}
#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) die(#call, e_); } while (0)

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

BatchGeom geom(size_t total, size_t blockSize, size_t slot)
{
    BatchGeom g;
    g.total = total; g.blockSize = (u32)blockSize; g.slot = (u32)slot;
    g.nBlocks = blockSize ? (u32)((total + blockSize - 1) / blockSize) : 0;
    return g;
}
size_t ok_or_generic(cudaError_t e) { return e == cudaSuccess ? 0 : (size_t)err(E_GENERIC); }

typedef cudaError_t (*enc_fn)(const BatchGeom&, void*, u64*, const void*, unsigned, unsigned, cudaStream_t);
typedef cudaError_t (*dec_fn)(const BatchGeom&, void*, const void*, const u64*, u64*, const void*, cudaStream_t);

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
constexpr size_t FSE_ONE_BLOCK_MAX = (size_t)1 << 30;                   // same limit as the batch tier (FSEB_DECL_*)

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
size_t huf_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstSizes, size_t* dOut, const void* const* dSrcs, const size_t* dSrcSizes,
                  int nStreams, bool compress, unsigned msv, unsigned tlog, void* stream)
{
    if (nBlocks == 0) return 0;
    if (nBlocks > 0xFFFFFFFFull || !dDsts || !dDstSizes || !dOut || !dSrcs || !dSrcSizes) return (size_t)err(E_SRC_WRONG);
    BlockDescs g;
    g.dst = (u8* const*)dDsts; g.dstCap = (const u64*)dDstSizes; g.result = (u64*)dOut;
    g.src = (const u8* const*)dSrcs; g.srcSize = (const u64*)dSrcSizes; g.nBlocks = (u32)nBlocks;
    return ok_or_generic(compress ? launch_huf_encode_blocks(g, nStreams, msv, tlog, (cudaStream_t)stream)
                                  : launch_huf_decode_blocks(g, nStreams, (cudaStream_t)stream));
}
}
FSEB_API size_t FSEB200_HUF_compress_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstCapacities, size_t* dCSizes,
                                            const void* const* dSrcs, const size_t* dSrcSizes, unsigned maxSymbolValue, unsigned tableLog, void* stream)
{
    return huf_blocks(nBlocks, dDsts, dDstCapacities, dCSizes, dSrcs, dSrcSizes, 4, true, maxSymbolValue, tableLog, stream);
}
FSEB_API size_t FSEB200_HUF_decompress_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstSizes, size_t* dResults,
                                              const void* const* dCSrcs, const size_t* dCSrcSizes, void* stream)
{
    return huf_blocks(nBlocks, dDsts, dDstSizes, dResults, dCSrcs, dCSrcSizes, 4, false, 0, 0, stream);
}
FSEB_API size_t FSEB200_HUF_compress1X_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstCapacities, size_t* dCSizes,
                                              const void* const* dSrcs, const size_t* dSrcSizes, unsigned maxSymbolValue, unsigned tableLog, void* stream)
{
    return huf_blocks(nBlocks, dDsts, dDstCapacities, dCSizes, dSrcs, dSrcSizes, 1, true, maxSymbolValue, tableLog, stream);
}
FSEB_API size_t FSEB200_HUF_decompress1X_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstSizes, size_t* dResults,
                                                const void* const* dCSrcs, const size_t* dCSrcSizes, void* stream)
{
    return huf_blocks(nBlocks, dDsts, dDstSizes, dResults, dCSrcs, dCSrcSizes, 1, false, 0, 0, stream);
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
    return ok_or_generic(launch_huf_encode_packed(g, nStreams, msv, tlog, (cudaStream_t)stream));
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
size_t huf_unpacked(size_t nBlocks, void* const* dDsts, const size_t* dDstSizes, size_t* dResults, const void* dIn,
                    const size_t* dOffsets, int nStreams, void* stream)
{
    if (nBlocks == 0) return 0;
    if (nBlocks > 0xFFFFFFFFull || !dDsts || !dDstSizes || !dResults || !dIn || !dOffsets) return (size_t)err(E_SRC_WRONG);
    return ok_or_generic(launch_huf_decompress_packed((u8* const*)dDsts, (const u64*)dDstSizes, (u64*)dResults, (const u8*)dIn,
                                                      (const u64*)dOffsets, (u32)nBlocks, nStreams, (cudaStream_t)stream));
}
}
FSEB_API size_t FSEB200_HUF_decompress_packed(size_t nBlocks, void* const* dDsts, const size_t* dDstSizes, size_t* dResults,
                                              const void* dIn, const size_t* dOffsets, void* stream)
{
    return huf_unpacked(nBlocks, dDsts, dDstSizes, dResults, dIn, dOffsets, 4, stream);
}
FSEB_API size_t FSEB200_HUF_decompress1X_packed(size_t nBlocks, void* const* dDsts, const size_t* dDstSizes, size_t* dResults,
                                                const void* dIn, const size_t* dOffsets, void* stream)
{
    return huf_unpacked(nBlocks, dDsts, dDstSizes, dResults, dIn, dOffsets, 1, stream);
}
namespace {
size_t fse_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstCaps, size_t* dOut, const void* const* dSrcs, const size_t* dSrcSizes,
                  bool wide, bool compress, unsigned msv, unsigned tlog, void* stream)
{
    if (nBlocks == 0) return 0;
    if (nBlocks > 0xFFFFFFFFull || !dDsts || !dDstCaps || !dOut || !dSrcs || !dSrcSizes) return (size_t)err(E_SRC_WRONG);
    BlockDescs g;
    g.dst = (u8* const*)dDsts; g.dstCap = (const u64*)dDstCaps; g.result = (u64*)dOut;
    g.src = (const u8* const*)dSrcs; g.srcSize = (const u64*)dSrcSizes; g.nBlocks = (u32)nBlocks;
    return ok_or_generic(compress ? launch_fse_encode_blocks(g, wide, msv, tlog, (cudaStream_t)stream) : launch_fse_decode_blocks(g, wide, (cudaStream_t)stream));
}
}
FSEB_API size_t FSEB200_FSE_compress_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstCapacities, size_t* dCSizes,
                                            const void* const* dSrcs, const size_t* dSrcSizes, unsigned maxSymbolValue, unsigned tableLog, void* stream)
{
    return fse_blocks(nBlocks, dDsts, dDstCapacities, dCSizes, dSrcs, dSrcSizes, false, true, maxSymbolValue, tableLog, stream);
}
FSEB_API size_t FSEB200_FSE_decompress_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstCapacities, size_t* dResults,
                                              const void* const* dCSrcs, const size_t* dCSrcSizes, void* stream)
{
    return fse_blocks(nBlocks, dDsts, dDstCapacities, dResults, dCSrcs, dCSrcSizes, false, false, 0, 0, stream);
}
FSEB_API size_t FSEB200_FSEU16_compress_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstCapacities, size_t* dCSizes,
                                               const void* const* dSrcs, const size_t* dSrcSizes, unsigned maxSymbolValue, unsigned tableLog, void* stream)
{
    return fse_blocks(nBlocks, dDsts, dDstCapacities, dCSizes, dSrcs, dSrcSizes, true, true, maxSymbolValue, tableLog, stream);
}
FSEB_API size_t FSEB200_FSEU16_decompress_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstCapacities, size_t* dResults,
                                                 const void* const* dCSrcs, const size_t* dCSrcSizes, void* stream)
{
    return fse_blocks(nBlocks, dDsts, dDstCapacities, dResults, dCSrcs, dCSrcSizes, true, false, 0, 0, stream);
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
size_t fse_unpacked(size_t nBlocks, void* const* dDsts, const size_t* dDstSizes, size_t* dResults, const void* dIn,
                    const size_t* dOffsets, bool wide, void* stream)
{
    if (nBlocks == 0) return 0;
    if (nBlocks > 0xFFFFFFFFull || !dDsts || !dDstSizes || !dResults || !dIn || !dOffsets) return (size_t)err(E_SRC_WRONG);
    return ok_or_generic(launch_fse_decompress_packed((u8* const*)dDsts, (const u64*)dDstSizes, (u64*)dResults, (const u8*)dIn,
                                                      (const u64*)dOffsets, (u32)nBlocks, wide, (cudaStream_t)stream));
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
    return fse_unpacked(nBlocks, dDsts, dDstSizes, dResults, dIn, dOffsets, false, stream);
}
FSEB_API size_t FSEB200_FSEU16_decompress_packed(size_t nBlocks, void* const* dDsts, const size_t* dDstSizes, size_t* dResults,
                                                 const void* dIn, const size_t* dOffsets, void* stream)
{
    return fse_unpacked(nBlocks, dDsts, dDstSizes, dResults, dIn, dOffsets, true, stream);
}

FSEB_API size_t FSEB200_batch_blocks(size_t total, size_t blockSize) { return blockSize ? (total + blockSize - 1) / blockSize : 0; }
FSEB_API int FSEB200_device_count(void) { int n = 0; return cudaGetDeviceCount(&n) == cudaSuccess ? n : 0; }

// ================================================================================================
// tier 2a: scalar helpers (host arithmetic only)
// ================================================================================================
FSEB_API unsigned FSE_versionNumber(void) { return 0 * 10000 + 9 * 100 + 0; }                 // lib/fse.h:43-47
FSEB_API size_t FSE_compressBound(size_t size) { return 512 + size + (size >> 7) + 4 + sizeof(size_t); }   // lib/fse.h:290-292
FSEB_API size_t HUF_compressBound(size_t size) { return 129 + size + (size >> 8) + 8; }       // lib/huf.h:131-133
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
// ---- table reuse, one block per call (lib/huf.h:194-208,291-300): HUF_compress_internal's repeat logic (huf_compress.c:637-724) composed
//      from the table-level calls, every data step on the GPU.  `repeat` is HUF_repeat {none 0, check 1, valid 2}. ----
namespace {
size_t huf_compress_ctable_internal(bool four, unsigned char* ostart, unsigned char* op, unsigned char* oend, const void* src, size_t srcSize, const unsigned* CTable)
{
    size_t const cSize = four ? HUF_compress4X_usingCTable(op, (size_t)(oend - op), src, srcSize, CTable)      // huf_compress.c:612-627
                              : HUF_compress1X_usingCTable(op, (size_t)(oend - op), src, srcSize, CTable);
    if (is_err(cSize)) return cSize;
    if (cSize == 0) return 0;
    op += cSize;
    if ((size_t)(op - ostart) >= srcSize - 1) return 0;
    return (size_t)(op - ostart);
}
size_t huf_compress_repeat(bool four, void* dst, size_t dstSize, const void* src, size_t srcSize, unsigned maxSymbolValue, unsigned huffLog,
                           void* workSpace, size_t wkspSize, unsigned* oldHufTable, int* repeat, int preferRepeat)
{
    unsigned char* const ostart = (unsigned char*)dst; unsigned char* const oend = ostart + dstSize; unsigned char* op = ostart;
    if (((size_t)workSpace & 3) != 0) return (size_t)err(E_GENERIC);                 // :652-653
    if (wkspSize < (6 << 10)) return (size_t)err(E_WKSP_TOO_SMALL);
    if (!srcSize || !dstSize) return 0;
    if (srcSize > HUF_BLOCK_MAX) return (size_t)err(E_SRC_WRONG);
    if (huffLog > HUF_MAX_TLOG) return (size_t)err(E_TLOG_TOO_LARGE);
    if (maxSymbolValue > HUF_MAX_SV) return (size_t)err(E_MSV_TOO_LARGE);
    if (!maxSymbolValue) maxSymbolValue = HUF_MAX_SV;
    if (!huffLog) huffLog = HUF_DEF_TLOG;
    if (preferRepeat && repeat && *repeat == 2) return huf_compress_ctable_internal(four, ostart, op, oend, src, srcSize, oldHufTable);   // :665-669
    unsigned count[256]; unsigned ctable[256];
    size_t const largest = HIST_count(count, &maxSymbolValue, src, srcSize);
    if (is_err(largest)) return largest;
    if (largest == srcSize) { ostart[0] = ((const unsigned char*)src)[0]; return 1; }
    if (largest <= (srcSize >> 7) + 4) return 0;
    for (unsigned s2 = maxSymbolValue + 1; s2 < 256; s2++) count[s2] = 0;
    if (repeat && *repeat == 1 && !HUF_validateCTable(oldHufTable, count, maxSymbolValue)) *repeat = 0;                              // :679-683
    if (preferRepeat && repeat && *repeat != 0) return huf_compress_ctable_internal(four, ostart, op, oend, src, srcSize, oldHufTable);
    huffLog = HUF_optimalTableLog(huffLog, srcSize, maxSymbolValue);
    size_t const maxBits = HUF_buildCTable(ctable, count, maxSymbolValue, huffLog);
    if (is_err(maxBits)) return maxBits;
    huffLog = (unsigned)maxBits;
    for (unsigned s2 = maxSymbolValue + 1; s2 < 256; s2++) ctable[s2] = 0;                                                          // :699-701
    size_t const hSize = HUF_writeCTable(op, dstSize, ctable, maxSymbolValue, huffLog);
    if (is_err(hSize)) return hSize;
    if (repeat && *repeat != 0) {                                                                                                   // :706-713
        size_t const oldSize = HUF_estimateCompressedSize(oldHufTable, count, maxSymbolValue);
        size_t const newSize = HUF_estimateCompressedSize(ctable, count, maxSymbolValue);
        if (oldSize <= hSize + newSize || hSize + 12 >= srcSize) return huf_compress_ctable_internal(four, ostart, op, oend, src, srcSize, oldHufTable);
    }
    if (hSize + 12ul >= srcSize) return 0;
    op += hSize;
    if (repeat) *repeat = 0;
    if (oldHufTable) std::memcpy(oldHufTable, ctable, sizeof(ctable));
    return huf_compress_ctable_internal(four, ostart, op, oend, src, srcSize, ctable);
}
}
FSEB_API size_t HUF_compress4X_repeat(void* dst, size_t dstSize, const void* src, size_t srcSize, unsigned maxSymbolValue, unsigned tableLog,
                                      void* workSpace, size_t wkspSize, unsigned* hufTable, int* repeat, int preferRepeat, int bmi2)   // lib/huf.h:204
{ (void)bmi2; return huf_compress_repeat(true, dst, dstSize, src, srcSize, maxSymbolValue, tableLog, workSpace, wkspSize, hufTable, repeat, preferRepeat); }
FSEB_API size_t HUF_compress1X_repeat(void* dst, size_t dstSize, const void* src, size_t srcSize, unsigned maxSymbolValue, unsigned tableLog,
                                      void* workSpace, size_t wkspSize, unsigned* hufTable, int* repeat, int preferRepeat, int bmi2)   // lib/huf.h:296
{ (void)bmi2; return huf_compress_repeat(false, dst, dstSize, src, srcSize, maxSymbolValue, tableLog, workSpace, wkspSize, hufTable, repeat, preferRepeat); }

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

// ================================================================================================
// tier 1b: whole-batch calls on HOST buffers (what an unmodified host program would hand over):
// the batch is cut into chunks that are copied in, processed and copied out on alternating streams so
// that PCIe transfers overlap the kernels.  codec: 0 = FSE, 1 = HUF, 2 = FSE-U16.
// ================================================================================================
namespace {
struct HostPipe {
    enum { NS = 4 };
    cudaStream_t st[NS] = {};
    unsigned char* dA[NS] = {};   // uncompressed side
    unsigned char* dB[NS] = {};   // compressed slots
    u64* dS[NS] = {};             // sizes + results
    size_t capA = 0, capB = 0, capS = 0;
    std::mutex mu;
    void ensure(size_t a, size_t b, size_t s)
    {
        for (int i = 0; i < NS; i++) if (!st[i]) CK(cudaStreamCreateWithFlags(&st[i], cudaStreamNonBlocking));
        if (a > capA) { for (int i = 0; i < NS; i++) { if (dA[i]) CK(cudaFree(dA[i])); CK(cudaMalloc(&dA[i], a + 256)); } capA = a; }
        if (b > capB) { for (int i = 0; i < NS; i++) { if (dB[i]) CK(cudaFree(dB[i])); CK(cudaMalloc(&dB[i], b + 256)); } capB = b; }
        if (s > capS) { for (int i = 0; i < NS; i++) { if (dS[i]) CK(cudaFree(dS[i])); CK(cudaMalloc(&dS[i], 2 * s * sizeof(u64))); } capS = s; }
    }
};
HostPipe& pipe() { static HostPipe p[MAX_DEVICES]; return p[current_device()]; }
// Blocks per pipeline chunk (FSEB200_HOST_CHUNK_BLOCKS, default 2048 = 64 MiB of 32 KB blocks): smaller chunks shorten the
// pipeline's fill and drain but leave the decode kernel a fraction of a wave per launch.
size_t chunk_blocks()
{
    static size_t const v = [] { const char* e = std::getenv("FSEB200_HOST_CHUNK_BLOCKS"); long n = e ? std::atol(e) : 2048; return (size_t)(n < 64 ? 64 : n > 65536 ? 65536 : n); }();
    return v;
}
#define CHUNK_BLOCKS chunk_blocks()
}

FSEB_API size_t FSEB200_compress_host(int codec, void* hCBuf, size_t slot, size_t* hCSizes, const void* hSrc, size_t srcTotal,
                                      size_t blockSize, unsigned maxSymbolValue, unsigned tableLog)
{
    if (blockSize == 0 || slot > 0xFFFFFFFFull || codec < 0 || codec > 2) return (size_t)err(E_SRC_WRONG);
    if (blockSize > (codec == 1 ? (size_t)HUF_BLOCK_MAX : FSE_ONE_BLOCK_MAX)) return (size_t)err(E_SRC_WRONG);
    enc_fn const fn = codec == 0 ? launch_fse_encode : codec == 1 ? launch_huf_encode : launch_fseu16_encode;
    HostPipe& P = pipe();
    std::lock_guard<std::mutex> lock(P.mu);
    size_t const nb = (srcTotal + blockSize - 1) / blockSize;
    P.ensure(CHUNK_BLOCKS * blockSize, CHUNK_BLOCKS * slot, CHUNK_BLOCKS);
    size_t const nChunks = (nb + CHUNK_BLOCKS - 1) / CHUNK_BLOCKS;
    // Software pipeline over chunks: chunk i+1 is queued (H2D + kernels + sizes D2H) before chunk i is finished.
    // Finishing = wait for its sizes, then copy back only the used width of its slots (strided 2-D copy): the
    // compressed side of the PCIe traffic shrinks from `slot` to max(cSize) bytes per block.
    auto queue = [&](size_t ci) {
        int const k = (int)(ci % HostPipe::NS);
        size_t const b0 = ci * CHUNK_BLOCKS, cb = nb - b0 < CHUNK_BLOCKS ? nb - b0 : CHUNK_BLOCKS;
        size_t const off = b0 * blockSize;
        size_t const bytes = (off + cb * blockSize <= srcTotal) ? cb * blockSize : srcTotal - off;
        cudaStream_t s = P.st[k];
        CK(cudaMemcpyAsync(P.dA[k], (const unsigned char*)hSrc + off, bytes, cudaMemcpyHostToDevice, s));
        CK(fn(geom(bytes, blockSize, slot), P.dB[k], P.dS[k], P.dA[k], maxSymbolValue, tableLog, s));
        CK(cudaMemcpyAsync(hCSizes + b0, P.dS[k], cb * sizeof(u64), cudaMemcpyDeviceToHost, s));
    };
    auto finish = [&](size_t ci) {
        int const k = (int)(ci % HostPipe::NS);
        size_t const b0 = ci * CHUNK_BLOCKS, cb = nb - b0 < CHUNK_BLOCKS ? nb - b0 : CHUNK_BLOCKS;
        cudaStream_t s = P.st[k];
        CK(cudaStreamSynchronize(s));
        size_t width = 0;
        for (size_t b = 0; b < cb; b++) { size_t const c = hCSizes[b0 + b]; if (!is_err(c) && c > width) width = c; }
        width = (width + 63) & ~(size_t)63; if (width > slot) width = slot;
        if (width) CK(cudaMemcpy2DAsync((unsigned char*)hCBuf + b0 * slot, slot, P.dB[k], slot, width, cb, cudaMemcpyDeviceToHost, s));
    };
    for (size_t ci = 0; ci < nChunks; ci++) {
        if (ci >= (size_t)HostPipe::NS - 1) finish(ci - (HostPipe::NS - 1));     // frees the buffers chunk ci+... will reuse next
        queue(ci);
    }
    for (size_t ci = (nChunks >= (size_t)HostPipe::NS - 1 ? nChunks - (HostPipe::NS - 1) : 0); ci < nChunks; ci++) finish(ci);
    for (int i = 0; i < HostPipe::NS; i++) CK(cudaStreamSynchronize(P.st[i]));
    return 0;
}

FSEB_API size_t FSEB200_decompress_host(int codec, void* hDst, size_t dstTotal, size_t blockSize, const void* hCBuf, size_t slot,
                                        const size_t* hCSizes, size_t* hResults, const void* hOrig)
{
    if (blockSize == 0 || slot > 0xFFFFFFFFull || codec < 0 || codec > 2) return (size_t)err(E_SRC_WRONG);
    if (blockSize > (codec == 1 ? (size_t)HUF_BLOCK_MAX : FSE_ONE_BLOCK_MAX)) return (size_t)err(E_SRC_WRONG);
    dec_fn const fn = codec == 0 ? launch_fse_decode : codec == 1 ? huf_dec_std : launch_fseu16_decode;
    HostPipe& P = pipe();
    std::lock_guard<std::mutex> lock(P.mu);
    size_t const nb = (dstTotal + blockSize - 1) / blockSize;
    P.ensure(CHUNK_BLOCKS * blockSize, CHUNK_BLOCKS * slot, CHUNK_BLOCKS);
    int k = 0;
    (void)hOrig;   // raw / RLE blocks: regenerated on the host below, exactly as bench.c:393-402 does
    for (size_t b0 = 0; b0 < nb; b0 += CHUNK_BLOCKS, k = (k + 1) % HostPipe::NS) {
        size_t const cb = nb - b0 < CHUNK_BLOCKS ? nb - b0 : CHUNK_BLOCKS;
        size_t const off = b0 * blockSize;
        size_t const bytes = (off + cb * blockSize <= dstTotal) ? cb * blockSize : dstTotal - off;
        cudaStream_t s = P.st[k];
        size_t width = 0;
        for (size_t bb = 0; bb < cb; bb++) { size_t const c = hCSizes[b0 + bb]; if (!is_err(c) && c > width) width = c; }
        width = (width + 16 + 63) & ~(size_t)63; if (width > slot) width = slot;     // +16: kernels read whole aligned 16-byte chunks
        if (width) CK(cudaMemcpy2DAsync(P.dB[k], slot, (const unsigned char*)hCBuf + b0 * slot, slot, width, cb, cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(P.dS[k], hCSizes + b0, cb * sizeof(u64), cudaMemcpyHostToDevice, s));
        CK(fn(geom(bytes, blockSize, slot), P.dA[k], P.dB[k], P.dS[k], P.dS[k] + CHUNK_BLOCKS, nullptr, s));
        CK(cudaMemcpyAsync((unsigned char*)hDst + off, P.dA[k], bytes, cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(hResults + b0, P.dS[k] + CHUNK_BLOCKS, cb * sizeof(u64), cudaMemcpyDeviceToHost, s));
    }
    for (int i = 0; i < HostPipe::NS; i++) CK(cudaStreamSynchronize(P.st[i]));
    if (hOrig) {
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
// tier 1b, packed: blocks of any size on HOST buffers through the packed device calls, so the stream a host program keeps is
// the one the device packed calls produce -- one buffer and its offsets, raw and RLE blocks stored in place -- and decodes
// without the original.  Chunks of blocks, cut by a byte budget, run on alternating streams as in the slot form above; inside a
// chunk the device packed calls run unchanged on chunk-local offsets with room for every block, and the host turns the results
// into the whole batch's: global offsets, the capacity rule, only the stored bytes copied down.
// codec: 0 = FSE, 1 = Huff0 4X, 2 = FSE-U16, 3 = Huff0 1X.
// ================================================================================================
namespace {
struct PackedPipe {
    enum { NS = 3 };
    cudaStream_t st[NS] = {};
    u8* dA[NS] = {};              // uncompressed side
    u8* dB[NS] = {};              // packed side
    u8* dW[NS] = {};              // FSE staging slots
    u64* dD[NS] = {};             // per-block arrays: pointers, sizes, offsets (n + 1), values
    u64* hD[NS] = {};             // their pinned host images
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
    // `a`, `b`, `w` bytes, `d` words per slot; the packed side gets the decoders' slack
    cudaError_t ensure(size_t a, size_t b, size_t w, size_t d)
    {
        cudaError_t e = cudaSuccess;
        for (int i = 0; i < NS && e == cudaSuccess; i++) if (!st[i]) e = cudaStreamCreateWithFlags(&st[i], cudaStreamNonBlocking);
        if (e == cudaSuccess) e = grow(dA, capA, a + 256, false);
        if (e == cudaSuccess) e = grow(dB, capB, b + 256, false);
        if (e == cudaSuccess && w) e = grow(dW, capW, w, false);
        if (e == cudaSuccess) e = grow(dD, capD, d * sizeof(u64), false);
        if (e == cudaSuccess) e = grow(hD, capH, d * sizeof(u64), true);
        return e;
    }
    // waits for every stream, also after a failure; the first error
    cudaError_t drain()
    {
        cudaError_t first = cudaSuccess;
        for (int i = 0; i < NS; i++) if (st[i]) { cudaError_t const e = cudaStreamSynchronize(st[i]); if (first == cudaSuccess) first = e; }
        return first;
    }
};
PackedPipe& ppipe() { static PackedPipe p[MAX_DEVICES]; return p[current_device()]; }

// Bytes per pipeline chunk (FSEB200_HOST_PACKED_CHUNK_BYTES, default 64 MiB).  A block counts its bytes plus 512 for its
// descriptors and staging overhead, so a chunk of tiny blocks stays bounded too; a block above the budget is a chunk of its own.
size_t chunk_budget()
{
    static size_t const v = [] { const char* e = std::getenv("FSEB200_HOST_PACKED_CHUNK_BYTES"); long long n = e ? std::atoll(e) : 64ll << 20; return (size_t)(n < 1 ? 1 : n); }();
    return v;
}
constexpr u64 BLOCK_OVERHEAD = 512;

struct HostChunk { size_t b0, b1; u64 a0, a1; };   // blocks [b0, b1); uncompressed bytes [a0, a1) of the batch

// chunks of blocks whose weight (uncompressed bytes + the packed bytes `packed(b)` + BLOCK_OVERHEAD) stays within the budget
template <typename F>
std::vector<HostChunk> cut_chunks(const size_t* sizes, size_t nBlocks, u64 unit, F packed)
{
    std::vector<HostChunk> out;
    size_t const budget = chunk_budget();
    HostChunk c = { 0, 0, 0, 0 };
    u64 w = 0;
    for (size_t b = 0; b < nBlocks; b++) {
        u64 const bytes = unit * sizes[b], wb = bytes + packed(b) + BLOCK_OVERHEAD;
        if (c.b1 > c.b0 && w + wb > budget) { out.push_back(c); c = { b, b, c.a1, c.a1 }; w = 0; }
        c.b1 = b + 1; c.a1 += bytes; w += wb;
    }
    out.push_back(c);
    return out;
}

// Queues chunk c of a host batch through the device packed compress in slot k: the source and the descriptors up, the packed
// call with room for every block.  On the device the slot's descriptor words are then: source pointers (cb), sizes (cb), offsets
// (cb + 1), values (cb).  codec as the host packed calls.
cudaError_t queue_packed_compress(PackedPipe& P, int k, const HostChunk& c, int codec, const void* hSrc, const size_t* hSrcSizes,
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
    u64 const unit = wide ? 2 : 1;
    std::vector<HostChunk> const chunks = cut_chunks(hSrcSizes, nBlocks, unit, [](size_t) { return (u64)0; });
    size_t maxA = 0, maxW = 0, maxD = 0;
    for (const HostChunk& c : chunks) {
        size_t const cb = c.b1 - c.b0, a = (size_t)(c.a1 - c.a0);
        maxA = a > maxA ? a : maxA;
        maxD = 4 * cb + 1 > maxD ? 4 * cb + 1 : maxD;
        if (fse) { size_t const w = FSEB200_FSE_packed_workspace(cb, a); maxW = w > maxW ? w : maxW; }
    }
    PackedPipe& P = ppipe();
    std::lock_guard<std::mutex> lock(P.mu);
    cudaError_t e = P.ensure(maxA, maxA, maxW, maxD);             // a block stores at most its own bytes
    u64 total = 0;                                                  // global offset of the next chunk's first block
    // queue: the source and the descriptors up, the packed call with room for every block, offsets and values down
    auto queue = [&](size_t ci) -> cudaError_t {
        int const k = (int)(ci % PackedPipe::NS);
        size_t const cb = chunks[ci].b1 - chunks[ci].b0;
        cudaError_t const r = queue_packed_compress(P, k, chunks[ci], codec, hSrc, hSrcSizes, maxSymbolValue, tableLog);
        if (r != cudaSuccess) return r;
        return cudaMemcpyAsync(P.hD[k] + 2 * cb, P.dD[k] + 2 * cb, (2 * cb + 1) * sizeof(u64), cudaMemcpyDeviceToHost, P.st[k]);
    };
    // finish: global offsets, the capacity rule of one call over the whole batch, and the stored bytes -- a prefix of the chunk's
    // packed bytes, since the blocks that fit come first -- copied down
    auto finish = [&](size_t ci) -> cudaError_t {
        int const k = (int)(ci % PackedPipe::NS);
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
    size_t const nc = chunks.size(), lag = PackedPipe::NS - 1;
    for (size_t ci = 0; ci < nc + lag && e == cudaSuccess; ci++) {
        if (ci >= lag) e = finish(ci - lag);
        if (e == cudaSuccess && ci < nc) e = queue(ci);
    }
    cudaError_t const d = P.drain();
    if (e != cudaSuccess || d != cudaSuccess) return (size_t)err(E_GENERIC);
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
    std::vector<HostChunk> const chunks = cut_chunks(hDstSizes, nBlocks, unit, [&](size_t b) { return (u64)(hOffsets[b + 1] - hOffsets[b]); });
    size_t maxA = 0, maxB = 0, maxD = 0;
    for (const HostChunk& c : chunks) {
        size_t const cb = c.b1 - c.b0, a = (size_t)(c.a1 - c.a0), in = hOffsets[c.b1] - hOffsets[c.b0];
        maxA = a > maxA ? a : maxA;
        maxB = in > maxB ? in : maxB;
        maxD = 4 * cb + 1 > maxD ? 4 * cb + 1 : maxD;
    }
    PackedPipe& P = ppipe();
    std::lock_guard<std::mutex> lock(P.mu);
    cudaError_t e = P.ensure(maxA, maxB, 0, maxD);
    // collect: the results of the chunk that last used slot k, once its stream is done
    auto collect = [&](size_t ci) -> cudaError_t {
        int const k = (int)(ci % PackedPipe::NS);
        size_t const cb = chunks[ci].b1 - chunks[ci].b0;
        cudaError_t const r = cudaStreamSynchronize(P.st[k]);
        if (r == cudaSuccess) std::memcpy(hResults + chunks[ci].b0, P.hD[k] + 3 * cb + 1, cb * sizeof(u64));
        return r;
    };
    // queue: the chunk's packed bytes and descriptors up (offsets rebased to the chunk), the packed decompress, the blocks and
    // their results down
    auto queue = [&](size_t ci) -> cudaError_t {
        int const k = (int)(ci % PackedPipe::NS);
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
    size_t const nc = chunks.size();
    for (size_t ci = 0; ci < nc + PackedPipe::NS && e == cudaSuccess; ci++) {
        if (ci >= (size_t)PackedPipe::NS) e = collect(ci - PackedPipe::NS);
        if (e == cudaSuccess && ci < nc) e = queue(ci);
    }
    cudaError_t const d = P.drain();
    return e == cudaSuccess && d == cudaSuccess ? 0 : (size_t)err(E_GENERIC);
}

// ================================================================================================
// tier 1b, frames: the .fse format of the reference's file tool (programs/fileio.c:266-626) on host buffers, through the packed
// pipeline above.  Compress: each chunk runs the device packed compress, then frame.cu lays its frame body out on the device --
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
        std::vector<HostChunk> const chunks = cut_chunks(sizes.data(), nb, 1, [](size_t) { return (u64)0; });
        size_t maxA = 0, maxF = 0, maxW = 0, maxD = 0;
        for (const HostChunk& c : chunks) {
            size_t const cb = c.b1 - c.b0, a = (size_t)(c.a1 - c.a0);
            maxA = a > maxA ? a : maxA;
            maxF = a + 5 * cb > maxF ? a + 5 * cb : maxF;           // a body: the stored blocks plus at most 5 header bytes each
            maxD = 4 * cb + 1 > maxD ? 4 * cb + 1 : maxD;
            if (codec == 0) { size_t const w = FSEB200_FSE_packed_workspace(cb, a); maxW = w > maxW ? w : maxW; }
        }
        PackedPipe& P = ppipe();
        std::lock_guard<std::mutex> lock(P.mu);
        cudaError_t e = P.ensure(maxF, maxA, maxW, maxD);          // the body goes to the source's buffer once it is coded
        // queue: the packed compress, the frame body, the offsets and values down
        auto queue = [&](size_t ci) -> cudaError_t {
            int const k = (int)(ci % PackedPipe::NS);
            size_t const cb = chunks[ci].b1 - chunks[ci].b0;
            u64* const d = P.dD[k];
            cudaError_t r = queue_packed_compress(P, k, chunks[ci], codec, hSrc, sizes.data(), 255, 11);
            if (r == cudaSuccess) r = launch_frame_body(P.dA[k], P.dB[k], d + 2 * cb, d + 3 * cb + 1, d + cb, (u32)cb, bs, P.st[k]);
            if (r != cudaSuccess) return r;
            return cudaMemcpyAsync(P.hD[k] + 2 * cb, d + 2 * cb, (2 * cb + 1) * sizeof(u64), cudaMemcpyDeviceToHost, P.st[k]);
        };
        // finish: the first error value in block order stops the call (fileio.c:329); otherwise the body comes down if it fits
        auto finish = [&](size_t ci) -> cudaError_t {
            int const k = (int)(ci % PackedPipe::NS);
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
        size_t const nc = chunks.size(), lag = PackedPipe::NS - 1;
        for (size_t ci = 0; ci < nc + lag && e == cudaSuccess && !verdict; ci++) {
            if (ci >= lag) e = finish(ci - lag);
            if (e == cudaSuccess && !verdict && ci < nc) e = queue(ci);
        }
        cudaError_t const d = P.drain();
        if (!verdict && (e != cudaSuccess || d != cudaSuccess)) verdict = (size_t)err(E_GENERIC);
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
        auto span = [&](size_t b) { return blk[b].payload + blk[b].cSize - blk[b].head; };
        std::vector<HostChunk> const chunks = cut_chunks(rs.data(), nb, 1, [&](size_t b) { return span(b); });
        std::vector<size_t> nCoded(chunks.size(), 0);
        size_t maxA = 0, maxB = 0, maxD = 0;
        for (size_t ci = 0; ci < chunks.size(); ci++) {
            const HostChunk& c = chunks[ci];
            size_t const cb = c.b1 - c.b0, a = (size_t)(c.a1 - c.a0);
            size_t const in = (size_t)(blk[c.b1 - 1].payload + blk[c.b1 - 1].cSize - blk[c.b0].head);
            for (size_t b = c.b0; b < c.b1; b++) nCoded[ci] += blk[b].type == BT_COMPRESSED;
            maxA = a > maxA ? a : maxA;
            maxB = in > maxB ? in : maxB;
            maxD = 5 * cb > maxD ? 5 * cb : maxD;
        }
        PackedPipe& P = ppipe();
        std::lock_guard<std::mutex> lock(P.mu);
        cudaError_t e = P.ensure(maxA, maxB, 0, maxD);
        // Descriptor words of a chunk with nc compressed and ns stored blocks: destinations, capacities, sources and sizes of
        // the compressed ones (nc each), the stored-block index (3 ns), then the decoders' results (nc).
        auto queue = [&](size_t ci) -> cudaError_t {
            int const k = (int)(ci % PackedPipe::NS);
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
        auto finish = [&](size_t ci) -> cudaError_t {
            int const k = (int)(ci % PackedPipe::NS);
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
        size_t const nChunks = chunks.size(), lag = PackedPipe::NS - 1;
        for (size_t ci = 0; ci < nChunks + lag && e == cudaSuccess && !verdict; ci++) {
            if (ci >= lag) e = finish(ci - lag);
            if (e == cudaSuccess && !verdict && ci < nChunks) e = queue(ci);
        }
        if (e == cudaSuccess && !verdict) e = hash_pending();
        cudaError_t const d = P.drain();
        if (!verdict && (e != cudaSuccess || d != cudaSuccess)) verdict = (size_t)err(E_GENERIC);
    }
    if (verdict) return verdict;
    if (w.verdict) return w.verdict;
    if (trailer_checksum(hash.digest()) != w.checksum) return (size_t)err(E_CORRUPT);   // exit 44
    return (size_t)out;
}
