// launchers.h -- the host launchers that one source file defines and another calls, declared once.  Every file that defines or
// calls one includes this header, so a definition that drifts from its declaration fails to compile or to link (-z defs).
#pragma once
#include "common.cuh"
#include "micro.h"

namespace fseb {
// batch tier (common.cuh BatchGeom); huf_decode flags: see huf_decode.cu
cudaError_t launch_huf_decode(const BatchGeom& g, void* dst, const void* cbuf, const u64* csizes, u64* results, const void* orig,
                              cudaStream_t stream, u32 flags);
cudaError_t launch_huf_encode(const BatchGeom& g, void* cbuf, u64* csizes, const void* src, unsigned msv, unsigned tlog, cudaStream_t stream);
cudaError_t launch_huf_encode_using_ctable(const BatchGeom& g, void* cbuf, u64* csizes, const void* src, const u32* dCTable, cudaStream_t stream);
cudaError_t launch_huf_x2_fixup(const BatchGeom& g, void* dst, const void* cbuf, const u64* csizes, u64* results, cudaStream_t stream);
cudaError_t launch_fse_decode(const BatchGeom& g, void* dst, const void* cbuf, const u64* csizes, u64* results, const void* orig, cudaStream_t s);
cudaError_t launch_fse_encode(const BatchGeom& g, void* cbuf, u64* csizes, const void* src, unsigned msv, unsigned tlog, cudaStream_t s);
cudaError_t launch_fseu16_decode(const BatchGeom& g, void* dst, const void* cbuf, const u64* csizes, u64* results, const void* orig, cudaStream_t s);
cudaError_t launch_fseu16_encode(const BatchGeom& g, void* cbuf, u64* csizes, const void* src, unsigned msv, unsigned tlog, cudaStream_t s);

// per-block descriptors (common.cuh BlockDescs, PackedDescs, ...).  The Huff0 encoder of every descriptor geometry, instantiated
// for each in huf_encode.cu: nStreams 4 (the 4X format) or 1 (1X) for every block, or 0 for the per-block forms of Mixed<...> and
// ChainPackedLiteralsDescs (which takes 0 only).  A Mixed<Base> with nStreams 4 or 1 runs as its Base.
template <class Geo>
cudaError_t launch_huf_encode_descs(const Geo& g, int nStreams, unsigned msv, unsigned tlog, cudaStream_t stream);
cudaError_t launch_huf_decode_blocks(const BlockDescs& g, int nStreams, cudaStream_t stream);
cudaError_t launch_huf_chain_check(const u64* start, u32 nChains, u32 nBlocks, u32* malformed, cudaStream_t stream);
// nStreams 4 or 1 for every block, or 0: per block, the form single[b] names (0: 4X, else 1X)
cudaError_t launch_huf_decode_headers(const HeaderDescs& g, int nStreams, cudaStream_t stream, const u8* single = nullptr);
cudaError_t launch_huf_x2_fixup_blocks(const BlockDescs& g, int nStreams, cudaStream_t stream);
cudaError_t launch_fse_encode_blocks(const BlockDescs& g, bool wide, unsigned msv, unsigned tlog, cudaStream_t s);
cudaError_t launch_fse_decode_blocks(const BlockDescs& g, bool wide, cudaStream_t s);

// packed buffers (fse_packed.cu, huf_packed.cu) and .fse frame bodies (frame.cu)
cudaError_t launch_fse_compress_packed(u8* out, u64 outCap, u64* offset, u64* result, const u8* const* src, const u64* srcSize,
                                       u32 nBlocks, u8* work, u64 workSize, bool wide, unsigned msv, unsigned tlog, cudaStream_t stream);
cudaError_t launch_fse_decompress_packed(u8* const* dst, const u64* dstSize, u64* result, const u8* in, const u64* offset,
                                         u32 nBlocks, bool wide, cudaStream_t stream);
cudaError_t launch_huf_decompress_packed(u8* const* dst, const u64* dstSize, u64* result, const u8* in, const u64* offset,
                                         u32 nBlocks, int nStreams, cudaStream_t stream);
cudaError_t launch_huf_decompress_repeat_packed(const u64* start, u32 nChains, u8* const* dst, const u64* dstSize, u64* result,
                                                const u8* in, const u64* offset, const u8* kind, const u8* const* chainHdr,
                                                const u64* chainHdrSize, u32 nBlocks, int nStreams, cudaStream_t stream,
                                                const u8* single = nullptr);   // as launch_huf_decode_headers
// A whole batch of frames laid out at once (the device-memory call): frame f is blocks [first[f], first[f + 1]), role[b] >> 32
// is block b's frame, and every frame has a block (an empty frame a placeholder of 0 source bytes).  offsets (nFrames + 1) and
// results get the batch call's values, and only frames that end at or before `capacity` are written; work: frame_body_work bytes.
struct FrameStore { u32 nFrames; const u64* first; u64 capacity; u64* offsets; u64* results; void* work; };
size_t frame_body_work(u32 nBlocks, u32 nFrames);
cudaError_t launch_frame_body(u8* out, const u8* packed, const u64* offset, const u64* value, const u64* srcSize, const u64* role,
                              const u64* hash, u32 nBlocks, u64 blockSize, u32 magic, u32 blockSizeId, cudaStream_t stream,
                              const FrameStore* store = nullptr);
cudaError_t launch_frame_stored(u8* out, const u8* in, const u64* index, u64 nStored, cudaStream_t stream);
cudaError_t launch_xxh32_ranges(const u8* base, const u64* desc, u32 n, u64* hash, cudaStream_t stream);

// single-CTA table kernels (micro.cu) and generators (gen.cu)
cudaError_t launch_hist(const void* src, u64 n, u32 declared, u32* out, u64* ret, cudaStream_t s);
cudaError_t launch_hist16(const void* src, u64 n, u32 declared, u32* out, u64* ret, cudaStream_t s);
cudaError_t launch_micro(int op, const MicroArgs& A, void* buf, u64* ret, cudaStream_t s);
cudaError_t launch_gen8(void* out, u64 n, u64 offset, const void* dTable, u32 seed0, cudaStream_t st);
cudaError_t launch_gen16(void* out, u64 n, u64 offset, const void* dTable, u32 seed0, cudaStream_t st);
}  // namespace fseb
