// frame_device.cu -- the .fse frame calls on DEVICE memory (include/fse_b200.h FSEB200_frame_{compress,decompress}_device,
// FSEB200_frame_decompress_bound_device): per frame exactly what the host batch calls give, with the geometry on the host and
// the bytes on the device.  DESIGN 5b describes both directions.
//
// Compress, all enqueued on the caller's stream: the host lays out the blocks (the words below) and uploads them from a pinned
// image; the device packed compress codes every block into scratch; the frame body (frame.cu) is scanned, each frame's offset,
// result and stored decision settled, and the stored frames written straight into dOut.  The checksums run meanwhile on a
// second stream that reads only the source, and the caller's stream waits for them on the device before the bodies are written.
//
// Decompress: a walk kernel (one frame per thread, frame_walk.h) counts each frame's blocks and reserves their places in the
// descriptor lists; the stream is synchronised once to learn the totals; a second walk fills the lists; the descriptor decoders
// and frame_stored_kernel regenerate the blocks; a settle kernel (one CTA per frame) walks each frame's results in block order;
// xxh32_kernel hashes the true outputs and a last kernel compares the trailers and writes the results.
#include "capi_common.h"
#include "fse_b200.h"
#include "frame_walk.h"
#include "launch_util.cuh"
#include "pack_dev.cuh"
#include <algorithm>
#include <cstring>
#include <mutex>
#include <vector>

using namespace fseb;
using namespace fseb::fmt;

namespace {

// Pinned host images of the words a call uploads.  An image is reused once the copy out of it has run (its event), so a call
// never waits for the device to upload its words.  Images come in powers of two from 64 KiB, so the pool holds a few images per
// call in flight at once: at most about twice the largest upload each, however the uploads grow.  Nothing is freed (freeing
// pinned memory would synchronise the device).
struct Pinned { u8* p = nullptr; size_t cap = 0; cudaEvent_t done = nullptr; int dev = 0; bool busy = false; };
std::mutex g_pinnedMu;
std::vector<Pinned*> g_pinned;

cudaError_t upload(void* dDst, const void* src, size_t bytes, cudaStream_t s)
{
    if (!bytes) return cudaSuccess;
    int const dev = current_device();
    Pinned* b = nullptr;
    {
        std::lock_guard<std::mutex> lk(g_pinnedMu);
        for (Pinned* x : g_pinned)
            if (!x->busy && x->dev == dev && x->cap >= bytes && cudaEventQuery(x->done) == cudaSuccess) { b = x; break; }
        if (b) b->busy = true;
    }
    cudaError_t e = cudaSuccess;
    if (!b) {
        b = new Pinned;
        b->dev = dev; b->busy = true;
        if ((e = cudaEventCreateWithFlags(&b->done, cudaEventDisableTiming)) == cudaSuccess) {
            size_t cap = (size_t)64 << 10;
            while (cap < bytes) cap <<= 1;
            if ((e = cudaMallocHost((void**)&b->p, cap)) == cudaSuccess) b->cap = cap;
        }
        std::lock_guard<std::mutex> lk(g_pinnedMu);
        g_pinned.push_back(b);                                      // kept even if it failed: cap 0 is never taken
    }
    if (e == cudaSuccess) {
        std::memcpy(b->p, src, bytes);
        e = cudaMemcpyAsync(dDst, b->p, bytes, cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess) e = cudaEventRecord(b->done, s);
    }
    std::lock_guard<std::mutex> lk(g_pinnedMu);
    b->busy = false;
    return e;
}

// The stream a compress call's checksums run on, forked from and joined back into the caller's stream by events: one per
// (device, caller's stream), so calls on different streams never queue behind each other's hashes
cudaError_t hash_stream(cudaStream_t caller, cudaStream_t* out)
{
    struct Slot { int dev; cudaStream_t caller, hash; };
    static std::mutex mu;
    static std::vector<Slot> slots;
    std::lock_guard<std::mutex> lk(mu);
    int const dev = current_device();
    for (const Slot& x : slots) if (x.dev == dev && x.caller == caller) { *out = x.hash; return cudaSuccess; }
    cudaError_t const e = cudaStreamCreateWithFlags(out, cudaStreamNonBlocking);
    if (e == cudaSuccess) slots.push_back({ dev, caller, *out });
    return e;
}

size_t up16(size_t n) { return (n + 15) & ~(size_t)15; }

// Scratch laid out in one stream-ordered allocation: take(bytes) hands out 16-byte aligned pieces in order
struct Carve {
    u8* base = nullptr; size_t at = 0;
    template <typename T> T* take(size_t bytes) { T* const p = (T*)(base + at); at += up16(bytes); return p; }
};

// Owns a stream-ordered allocation: freed on the stream when the call is done with it, also on an early return
struct StreamMem {
    void* p = nullptr; cudaStream_t s;
    explicit StreamMem(cudaStream_t st) : s(st) {}
    cudaError_t alloc(size_t bytes) { return cudaMallocAsync(&p, bytes ? bytes : 16, s); }
    ~StreamMem() { if (p) cudaFreeAsync(p, s); }
};

}  // namespace

// ================================================================================================
// decompress kernels
// ================================================================================================
namespace fseb {
namespace framedev {

// What the walk learns of frame f, and what the later passes settle
struct DecFrame {
    u64 nominal;            // the walked blocks' rSize sum
    u64 walkVerdict;        // where the header walk stopped, or 0
    u64 verdict;            // a stored frame's overflow up front, then the first decoder error or overflow in block order
    u64 nRun, nCoded;       // blocks that run, compressed ones among them
    u64 rec0, coded0, stored0, scratch0;   // their places: settle records, the codec's descriptor list, the stored index, scratch
    u64 done;               // bytes regenerated
    u32 checksum, codec, crossing, pad;    // crossing: the nominal output passes the capacity, so the blocks decode into scratch
};
struct Totals { u64 blocks, fse, huf, stored, scratch; };

struct Dec {
    const u8* in; const u64* off; const u64* region;                // frame f: in[off[f], off[f + 1]); output region[f] ..
    u8* dst; DecFrame* fr; Totals* tot; u64* bound; u32 nFrames;
    // after the sync
    u8** cdst; u64* ccap; const u8** csrc; u64* csize; u64* cres; u64* index; u64* rec; u8* scratch; u64 nFse;
    u64* hashDesc; u64* hash; u64 mis;                              // mis: dst's misalignment, the hash kernel's base being aligned
};

constexpr u64 REC_STORED = 1ull << 63;                              // rec[2 i + 1]: a stored block's rSize, or a coded block's result slot

// count pass, one frame per thread: the walk, the up-front verdicts of frames without compressed blocks, the bound, and the
// reservations of the frame's places in every list
__global__ void walk_count_kernel(Dec d)
{
    u64 const f = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= d.nFrames) return;
    const u8* const p = d.in + d.off[f];
    u64 const size = d.off[f + 1] - d.off[f];
    WalkState s;
    FrameBlock k;
    u64 r, nb = 0, nc = 0, nominal = 0;
    while ((r = walk_step(p, size, s, k)) == WALK_BLOCK) { nb++; nc += k.type == BT_COMPRESSED; nominal += k.rSize; }
    u64 const walkVerdict = r == WALK_END ? 0 : r;
    d.bound[f] = walkVerdict ? walkVerdict : nominal;
    if (!d.region) return;                                          // the bound call
    DecFrame x = {};
    u64 const cap = d.region[f + 1] - d.region[f];
    x.nominal = nominal; x.walkVerdict = walkVerdict; x.checksum = s.checksum; x.codec = (u32)s.codec;
    // every block's output size is known: settled here, as the host call does, and none of its blocks runs
    if (!nc && nominal > cap) x.verdict = err(E_DST_TOO_SMALL);
    if (nc || (nominal <= cap && !walkVerdict)) { x.nRun = nb; x.nCoded = nc; }
    x.crossing = x.nRun && nominal > cap;
    if (x.nRun) {
        x.rec0 = atomicAdd(&d.tot->blocks, x.nRun);
        x.coded0 = nc ? atomicAdd(x.codec ? &d.tot->huf : &d.tot->fse, nc) : 0;
        x.stored0 = nb > nc ? atomicAdd(&d.tot->stored, nb - nc) : 0;
        x.scratch0 = x.crossing ? atomicAdd(&d.tot->scratch, nominal) : 0;
    }
    d.fr[f] = x;
}

// fill pass, one frame per thread: the same walk again, each running block's descriptor (compressed), index entry (raw, RLE)
// and settle record.  Blocks decode at their nominal place: in the region, or in scratch for a crossing frame.
__global__ void walk_fill_kernel(Dec d)
{
    u64 const f = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= d.nFrames) return;
    DecFrame const x = d.fr[f];
    if (!x.nRun) return;
    const u8* const p = d.in + d.off[f];
    u64 const size = d.off[f + 1] - d.off[f];
    u8* const out = x.crossing ? d.scratch + x.scratch0 : d.dst + d.region[f];
    u64 const c0 = x.coded0 + (x.codec ? d.nFse : 0);
    WalkState s;
    FrameBlock k;
    u64 pos = 0, ci = 0, si = 0;
    for (u64 i = 0; i < x.nRun && walk_step(p, size, s, k) == WALK_BLOCK; i++) {
        u64* const rec = d.rec + 2 * (x.rec0 + i);
        rec[0] = pos;
        if (k.type == BT_COMPRESSED) {
            u64 const j = c0 + ci++;
            d.cdst[j] = out + pos; d.ccap[j] = k.rSize; d.csrc[j] = p + k.payload; d.csize[j] = k.cSize;
            rec[1] = j;
        } else {
            // absolute addresses: frame_stored_kernel runs with null bases
            u64* const e = d.index + 3 * (x.stored0 + si++);
            e[0] = reinterpret_cast<u64>(out + pos); e[1] = reinterpret_cast<u64>(p + k.payload); e[2] = k.rSize | (u64)k.type << 32;
            rec[1] = REC_STORED | k.rSize;
        }
        pos += k.rSize;
    }
}

// n bytes from s down to d <= s, the ranges possibly overlapping, by the CTA: each round every thread reads its 16 bytes of
// the round's 16 * blockDim.x, the CTA meets, then every thread writes them.  A round writes below what later rounds read.
__device__ void cta_move_down(u8* d, const u8* s, u64 n)
{
    for (u64 o = 0; o < n; o += 16ull * blockDim.x) {
        u64 const at = o + 16ull * threadIdx.x;
        u8 t[16];
        #pragma unroll
        for (int i = 0; i < 16; i++) if (at + i < n) t[i] = s[at + i];
        __syncthreads();
        #pragma unroll
        for (int i = 0; i < 16; i++) if (at + i < n) d[at + i] = t[i];
    }
    __syncthreads();
}

// settle, one CTA of pack::COPY_THREADS per frame (frames f0 + blockIdx.x): its blocks' results in block order, a tile of
// blocks at a time -- the first decoder error or the first block past the capacity ends the frame with its verdict; otherwise
// every block that does not sit where the true sizes put it (after a short FSE block, or every block of a crossing frame)
// moves there, one block after another; then the frame's hash range
__global__ void __launch_bounds__(pack::COPY_THREADS) settle_kernel(Dec d, u64 f0)
{
    constexpr int NT = pack::COPY_THREADS;
    __shared__ u64 sm[NT / 32 + 1];
    __shared__ u64 sNom[NT], sPos[NT], sLen[NT];
    __shared__ u64 sFail, sVerdict;
    u64 const f = f0 + blockIdx.x;
    DecFrame const x = d.fr[f];
    u8* const region = d.dst + d.region[f];
    u64 const cap = d.region[f + 1] - d.region[f];
    const u8* const from = x.crossing ? d.scratch + x.scratch0 : region;
    u64 done = 0, verdict = x.verdict;
    for (u64 i0 = 0; i0 < x.nRun && !verdict; i0 += NT) {
        u64 const i = i0 + threadIdx.x;
        bool const in = i < x.nRun;
        u64 nom = 0, n = 0;
        if (in) {
            const u64* const rec = d.rec + 2 * (x.rec0 + i);
            nom = rec[0];
            n = rec[1] & REC_STORED ? rec[1] & ~REC_STORED : d.cres[rec[1]];
        }
        bool const bad = in && is_err(n);
        u64 excl;
        u64 const tileLen = pack::cta_exclusive_scan<NT>(bad ? 0 : n, excl, sm);
        u64 const pos = done + excl;
        if (threadIdx.x == 0) sFail = ~0ull;
        __syncthreads();
        if (in && (bad || pos + n > cap)) atomicMin((unsigned long long*)&sFail, (unsigned long long)i);
        sNom[threadIdx.x] = nom; sPos[threadIdx.x] = pos; sLen[threadIdx.x] = n;
        __syncthreads();
        if (sFail == i) sVerdict = bad ? n : err(E_DST_TOO_SMALL);
        __syncthreads();
        if (sFail != ~0ull) { verdict = sVerdict; break; }
        u64 const m = x.nRun - i0 < NT ? x.nRun - i0 : NT;
        for (u64 j = 0; j < m; j++) {                                // CTA-uniform: shared values only
            if (!x.crossing && sNom[j] == sPos[j]) continue;
            if (x.crossing) pack::cta_copy<NT, pack::COPY_UNROLL>(region + sPos[j], from + sNom[j], (u32)sLen[j]);
            else cta_move_down(region + sPos[j], from + sNom[j], sLen[j]);
        }
        done += tileLen;
        __syncthreads();                                            // sNom, sPos, sLen are rewritten by the next tile
    }
    if (threadIdx.x == 0) {
        d.fr[f].verdict = verdict; d.fr[f].done = done;
        bool const hashed = !verdict && !x.walkVerdict;
        d.hashDesc[2 * f] = d.mis + d.region[f]; d.hashDesc[2 * f + 1] = hashed ? done : 0;
    }
}

// the results: a verdict, or the checksum's
__global__ void finish_kernel(Dec d, u64* results)
{
    u64 const f = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= d.nFrames) return;
    DecFrame const x = d.fr[f];
    u64 r = x.verdict ? x.verdict : x.walkVerdict;
    if (!r) r = trailer_checksum((u32)d.hash[f]) != x.checksum ? err(E_CORRUPT) : x.done;   // exit 44
    results[f] = r;
}

}  // namespace framedev
}  // namespace fseb

namespace {
using namespace fseb::framedev;

unsigned grid_of(u64 n, unsigned t) { return (unsigned)((n + t - 1) / t); }

// The walk of every frame on the device: Dec's first half, with the frames' offsets (and regions, unless the bound call) uploaded.
// Per-frame scratch: DecFrame, the totals, the bound, the hash ranges and hashes, the offsets and regions.
struct Walked { StreamMem mem; Dec d = {}; Totals tot = {}; explicit Walked(cudaStream_t s) : mem(s) {} };

cudaError_t walk_frames(Walked& w, size_t nFrames, const void* dIn, const size_t* hOffsets, const size_t* hCaps, void* dDst, cudaStream_t s)
{
    size_t const F = nFrames;
    std::vector<u64> words(2 * (F + 1));
    for (size_t f = 0; f <= F; f++) words[f] = hOffsets[f];
    if (hCaps) for (size_t f = 0; f < F; f++) words[F + 1 + f + 1] = words[F + 1 + f] + hCaps[f];
    size_t const bytes = up16(sizeof(DecFrame) * F) + up16(sizeof(Totals)) + up16(8 * F) * 4 + up16(8 * words.size());
    cudaError_t e;
    if ((e = w.mem.alloc(bytes)) != cudaSuccess) return e;
    Carve c; c.base = (u8*)w.mem.p;
    Dec& d = w.d;
    d.fr = c.take<DecFrame>(sizeof(DecFrame) * F); d.tot = c.take<Totals>(sizeof(Totals)); d.bound = c.take<u64>(8 * F);
    d.hashDesc = c.take<u64>(16 * F); d.hash = c.take<u64>(8 * F);
    u64* const up = c.take<u64>(8 * words.size());
    d.in = (const u8*)dIn; d.off = up; d.region = hCaps ? up + F + 1 : nullptr; d.nFrames = (u32)F;
    d.mis = reinterpret_cast<u64>(dDst) & 15; d.dst = (u8*)dDst;
    if ((e = cudaMemsetAsync(d.tot, 0, sizeof(Totals), s)) != cudaSuccess) return e;
    if ((e = upload(up, words.data(), 8 * words.size(), s)) != cudaSuccess) return e;
    walk_count_kernel<<<grid_of(F, 128), 128, 0, s>>>(d);
    return cudaGetLastError();
}

size_t frame_args_ok(size_t nFrames, const size_t* hOffsets)
{
    for (size_t f = 0; f < nFrames; f++) if (hOffsets[f + 1] < hOffsets[f]) return (size_t)err(E_SRC_WRONG);
    return 0;
}
}  // namespace

FSEB_API size_t FSEB200_frame_decompress_bound_device(size_t nFrames, size_t* hBounds, const void* dIn, const size_t* hOffsets, void* stream)
{
    if (nFrames > 0xFFFFFFFFull) return (size_t)err(E_SRC_WRONG);
    if (nFrames == 0) return 0;
    if (!hBounds || !dIn || !hOffsets) return (size_t)err(E_SRC_WRONG);
    if (size_t const r = frame_args_ok(nFrames, hOffsets)) return r;
    cudaStream_t const s = (cudaStream_t)stream;
    cudaError_t e;
    {
        Walked w(s);
        e = walk_frames(w, nFrames, dIn, hOffsets, nullptr, nullptr, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(hBounds, w.d.bound, 8 * nFrames, cudaMemcpyDeviceToHost, s);
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    return ok_or_generic(e);
}

FSEB_API size_t FSEB200_frame_decompress_device(size_t nFrames, void* dDst, const size_t* hDstCapacities, size_t* dResults,
                                                const void* dIn, const size_t* hOffsets, void* stream)
{
    if (nFrames > 0xFFFFFFFFull) return (size_t)err(E_SRC_WRONG);
    if (nFrames == 0) return 0;
    if (!dDst || !hDstCapacities || !dResults || !dIn || !hOffsets) return (size_t)err(E_SRC_WRONG);
    if (size_t const r = frame_args_ok(nFrames, hOffsets)) return r;
    cudaStream_t const s = (cudaStream_t)stream;
    Walked w(s);
    cudaError_t e = walk_frames(w, nFrames, dIn, hOffsets, hDstCapacities, dDst, s);
    // the one synchronisation: the totals size the lists and the launches
    if (e == cudaSuccess) e = cudaMemcpyAsync(&w.tot, w.d.tot, sizeof(Totals), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) return (size_t)err(E_GENERIC);
    Totals const t = w.tot;
    u64 const nc = t.fse + t.huf;
    if (t.fse > 0xFFFFFFFFull || t.huf > 0xFFFFFFFFull) return (size_t)err(E_SRC_WRONG);
    Dec d = w.d;
    StreamMem lists(s);
    size_t const bytes = up16(8 * nc) * 5 + up16(24 * t.stored) + up16(16 * t.blocks) + up16(t.scratch);
    if ((e = lists.alloc(bytes)) != cudaSuccess) return (size_t)err(E_GENERIC);
    Carve c; c.base = (u8*)lists.p;
    d.cdst = c.take<u8*>(8 * nc); d.ccap = c.take<u64>(8 * nc); d.csrc = c.take<const u8*>(8 * nc); d.csize = c.take<u64>(8 * nc);
    d.cres = c.take<u64>(8 * nc); d.index = c.take<u64>(24 * t.stored); d.rec = c.take<u64>(16 * t.blocks); d.scratch = c.take<u8>(t.scratch);
    d.nFse = t.fse;
    walk_fill_kernel<<<grid_of(nFrames, 128), 128, 0, s>>>(d);
    for (int huf = 0; huf < 2 && e == cudaSuccess; huf++) {
        u64 const j0 = huf ? t.fse : 0, n = huf ? t.huf : t.fse;
        if (!n) continue;
        BlockDescs g;
        g.dst = d.cdst + j0; g.dstCap = d.ccap + j0; g.result = d.cres + j0; g.src = d.csrc + j0; g.srcSize = d.csize + j0; g.nBlocks = (u32)n;
        e = huf ? launch_huf_decode_blocks(g, 4, s) : launch_fse_decode_blocks(g, false, s);
    }
    if (e == cudaSuccess && t.stored) e = launch_frame_stored(nullptr, nullptr, d.index, t.stored, s);
    if (e == cudaSuccess) {
        pack::launch_per_block(settle_kernel, nFrames, s, d);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = launch_xxh32_ranges(d.dst - d.mis, d.hashDesc, (u32)nFrames, d.hash, s);
    if (e == cudaSuccess) {
        finish_kernel<<<grid_of(nFrames, 128), 128, 0, s>>>(d, (u64*)dResults);
        e = cudaGetLastError();
    }
    return ok_or_generic(e);
}

// ================================================================================================
// compress
// ================================================================================================
FSEB_API size_t FSEB200_frame_compress_device(int codec, unsigned blockSizeId, size_t nFrames, void* dOut, size_t outCapacity,
                                              size_t* dOffsets, size_t* dResults, const void* dSrc, const size_t* hSrcSizes, void* stream)
{
    if (codec < 0 || codec > 1 || blockSizeId > 6 || nFrames > 0xFFFFFFFFull) return (size_t)err(E_SRC_WRONG);
    if (nFrames == 0) return 0;
    if (!dOut || !dOffsets || !dResults || !hSrcSizes) return (size_t)err(E_SRC_WRONG);
    if (!dSrc) for (size_t f = 0; f < nFrames; f++) if (hSrcSizes[f]) return (size_t)err(E_SRC_WRONG);
    cudaStream_t const s = (cudaStream_t)stream;
    size_t const F = nFrames;
    u64 const bs = (u64)1024 << blockSizeId;
    // the blocks: ceil(n / bs) per frame, and an empty frame's placeholder of 0 bytes
    u64 nb = 0, total = 0;
    for (size_t f = 0; f < F; f++) { nb += hSrcSizes[f] ? (hSrcSizes[f] + bs - 1) / bs : 1; total += hSrcSizes[f]; }
    if (nb > 0xFFFFFFFFull) return (size_t)err(E_SRC_WRONG);
    // uploaded words: block pointers, sizes and roles, the frames' hash ranges and first blocks; then the device's: the packed
    // offsets and values, the hashes, the body's work; then the packed bytes and the FSE workspace
    size_t const nUp = 3 * nb + 2 * F + F + 1;
    size_t const work = codec == 0 ? FSEB200_FSE_packed_workspace(nb, total) : 0;
    size_t const bytes = up16(8 * nUp) + up16(8 * (2 * nb + 1)) + up16(8 * F) + up16(frame_body_work((u32)nb, (u32)F)) + up16(total + 32) + up16(work);
    StreamMem mem(s);
    cudaError_t e = mem.alloc(bytes);
    if (e != cudaSuccess) return (size_t)err(E_GENERIC);
    Carve c; c.base = (u8*)mem.p;
    u64* const up = c.take<u64>(8 * nUp);
    u64* const offset = c.take<u64>(8 * (2 * nb + 1)); u64* const value = offset + nb + 1;
    u64* const hash = c.take<u64>(8 * F);
    void* const bodyWork = c.take<u8>(frame_body_work((u32)nb, (u32)F));
    u8* const packed = c.take<u8>(total + 32);
    u8* const fseWork = c.take<u8>(work);
    u64* const hPtr = up, * const hSize = up + nb, * const hRole = up + 2 * nb, * const hRange = up + 3 * nb, * const hFirst = hRange + 2 * F;
    // the source's 16-byte aligned base for xxh32_kernel's copies; the ranges are offsets from it
    const u8* const src = dSrc ? (const u8*)dSrc : packed;
    u64 const mis = reinterpret_cast<u64>(src) & 15;
    std::vector<u64> w(nUp);
    u64* const ptr = w.data(), * const size = ptr + nb, * const role = size + nb, * const range = role + nb, * const first = range + 2 * F;
    for (size_t f = 0, b = 0, at = 0; f < F; f++) {
        u64 const n = hSrcSizes[f], k = n ? (n + bs - 1) / bs : 1;
        first[f] = b;
        range[2 * f] = mis + at; range[2 * f + 1] = n;
        for (u64 i = 0; i < k; i++, b++) {
            size[b] = n ? std::min(bs, n - i * bs) : 0;
            ptr[b] = reinterpret_cast<u64>(n ? src + at + i * bs : packed);
            role[b] = (i == 0 ? ROLE_FIRST : 0) | (i + 1 == k ? ROLE_LAST | ROLE_HASHED : 0) | (u64)f << 32;
        }
        at += n;
    }
    first[F] = nb;
    if ((e = upload(up, w.data(), 8 * nUp, s)) != cudaSuccess) return (size_t)err(E_GENERIC);
    // the checksums, on the hash stream while the blocks are coded; they read only the source
    cudaStream_t hs;
    cudaEvent_t fork = nullptr, joined = nullptr;
    bool forked = false;                                            // the hash stream reads scratch: `s` must wait for it
    if ((e = hash_stream(s, &hs)) != cudaSuccess) return (size_t)err(E_GENERIC);
    if ((e = cudaEventCreateWithFlags(&fork, cudaEventDisableTiming)) == cudaSuccess &&
        (e = cudaEventCreateWithFlags(&joined, cudaEventDisableTiming)) == cudaSuccess &&
        (e = cudaEventRecord(fork, s)) == cudaSuccess && (e = cudaStreamWaitEvent(hs, fork, 0)) == cudaSuccess) {
        forked = true;
        e = launch_xxh32_ranges(src - mis, hRange, (u32)F, hash, hs);
        cudaError_t const r = cudaEventRecord(joined, hs);
        if (e == cudaSuccess) e = r;
    }
    // the device packed compress at the writer's (255, 11), with room for every block
    const u8* const* const srcs = (const u8* const*)hPtr;
    if (e == cudaSuccess) {
        if (codec == 0) e = launch_fse_compress_packed(packed, total, offset, value, srcs, hSize, (u32)nb, fseWork, work, false, 255, 11, s);
        else {
            PackedDescs g;
            g.out = packed; g.outCap = total; g.offset = offset; g.result = value; g.src = srcs; g.srcSize = hSize; g.nBlocks = (u32)nb;
            e = launch_huf_encode_descs(g, 4, 255, 11, s);
        }
    }
    // the stream waits on the device for the checksums (also after a failure, before the scratch is freed on it); then the
    // frame bodies, offsets and results
    if (forked) { cudaError_t const r = cudaStreamWaitEvent(s, joined, 0); if (e == cudaSuccess) e = r; }
    if (e == cudaSuccess) {
        FrameStore const st = { (u32)F, hFirst, outCapacity, (u64*)dOffsets, (u64*)dResults, bodyWork };
        e = launch_frame_body((u8*)dOut, packed, offset, value, hSize, hRole, hash, (u32)nb, bs, codec ? MAGIC_HUF : MAGIC_FSE,
                              blockSizeId, s, &st);
    }
    if (fork) cudaEventDestroy(fork);
    if (joined) cudaEventDestroy(joined);
    return ok_or_generic(e);
}
