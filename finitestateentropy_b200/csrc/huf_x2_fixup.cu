// huf_x2_fixup.cu -- second pass of the batch Huff0 decoder: the reference's verdict on malformed streams.
//
// HUF_decompress (lib/huf_decompress.c:1056-1081) decodes a block with the single- or the double-symbol decoder as
// HUF_selectDecoder says (:1029-1051).  On valid streams both regenerate the same bytes.  On malformed ones they differ at
// the very end of a stream: HUF_decodeLastSymbolX2 (:668-683) takes the first byte of a two-symbol cell, skips the bits of
// BOTH symbols and clamps the bit count, so the X2 decoder ACCEPTS some streams whose last code does not end exactly where
// the stream does -- which the X1 rule (every stream consumed exactly, :348-349) rejects.  A stream accepted by X1 is
// accepted by X2 with the same bytes, never the other way round.
//
// huf_decode_kernel is an X1 decoder.  Blocks it rejects at the end-of-stream check, and which the reference would have
// decoded with X2, are marked HUF_X2_PENDING; this kernel re-decodes exactly those blocks with the bit-exact model of
// the X2 decoder (huf_x2_dev.cuh), writing the bytes and the verdict the reference produces.  On well-formed batches it
// finds nothing to do: one coalesced sweep over the results.
#include "common.cuh"
#include "launchers.h"
#include "huf_x2_dev.cuh"
#include "launch_util.cuh"

namespace fseb {
namespace hufx {

constexpr int THREADS = 128;

// NS = streams per block of the batch: 4 (HUF_decompress) or 1 (HUF_decompress1X_DCtx)
template <class Geo, int NS>
__global__ void __launch_bounds__(THREADS)
huf_x2_fixup_kernel(Geo g, u8* __restrict__ dst, const u8* __restrict__ cbuf, const u64* __restrict__ csizes, u64* __restrict__ results)
{
    __shared__ u32 s_dt[1 + 4096];
    __shared__ u8 s_scratch[768];
    __shared__ u64 s_init[4];
    __shared__ u32 s_done[4];
    __shared__ u64 s_h;
    __shared__ u32 s_hits[THREADS];
    __shared__ u32 s_nhits;
    int const tid = threadIdx.x;
    u32 const per = (g.nBlocks + gridDim.x - 1) / gridDim.x;
    u32 const c0 = blockIdx.x * per;
    u32 const c1 = min(c0 + per, g.nBlocks);
    for (u32 base = c0; base < c1; base += THREADS) {
        if (tid == 0) s_nhits = 0;
        __syncthreads();
        u32 const b = base + tid;
        if (b < c1 && dec_out(g, results, b) == HUF_X2_PENDING) s_hits[atomicAdd(&s_nhits, 1u)] = b;
        __syncthreads();
        u32 const nh = s_nhits;
        for (u32 i = 0; i < nh; i++) {
            u32 const bb = s_hits[i];
            const u8* const c = dec_src(g, cbuf, bb);
            u64 const cs = dec_csize(g, csizes, bb);
            u64 const n = dec_len(g, bb);
            if (tid == 0) s_h = d_huf_build_dtable_x2(s_dt, HUF_MAX_TLOG * 0x01000001u, s_scratch, s_scratch + 256, s_scratch + 512, c, cs);   // HUF_CREATE_STATIC_DTABLEX2(.., HUF_TABLELOG_MAX), :944
            __syncthreads();
            u64 const h = s_h;
            u64 r;
            if (is_err(h)) r = h;                                                   // :934
            else if (h >= cs) r = err(E_SRC_WRONG);                                 // :935
            else r = cta_huf_decode<d_huf_decode_stream_x2>(NS == 4, s_dt, c + h, cs - h, dec_dst(g, dst, bb), n, s_init, s_done);
            if (tid == 0) dec_out(g, results, bb) = r;
            __syncthreads();
        }
    }
}

}  // namespace hufx

namespace {
template <class Geo, int NS>
cudaError_t huf_x2_fixup(const Geo& g, void* dst, const void* cbuf, const u64* csizes, u64* results, cudaStream_t stream)
{
    if (g.nBlocks == 0) return cudaSuccess;
    unsigned grid = 2u * (unsigned)device_sm_count(current_device());
    unsigned const need = (g.nBlocks + hufx::THREADS - 1) / hufx::THREADS;
    if (grid > need) grid = need;
    hufx::huf_x2_fixup_kernel<Geo, NS><<<grid, hufx::THREADS, 0, stream>>>(g, (u8*)dst, (const u8*)cbuf, csizes, results);
    return cudaGetLastError();
}
}  // namespace

cudaError_t launch_huf_x2_fixup(const BatchGeom& g, void* dst, const void* cbuf, const u64* csizes, u64* results, cudaStream_t stream)
{
    return huf_x2_fixup<BatchGeom, 4>(g, dst, cbuf, csizes, results, stream);
}

cudaError_t launch_huf_x2_fixup_blocks(const BlockDescs& g, int nStreams, cudaStream_t stream)
{
    return nStreams == 1 ? huf_x2_fixup<BlockDescs, 1>(g, nullptr, nullptr, nullptr, nullptr, stream)
                         : huf_x2_fixup<BlockDescs, 4>(g, nullptr, nullptr, nullptr, nullptr, stream);
}

}  // namespace fseb
