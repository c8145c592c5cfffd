// common.cuh -- shared device/host helpers for the H100 (sm_90a) entropy-coding kernels.
//
// Error convention: identical to the reference's (lib/error_private.h:77-79,
// lib/error_public.h:45-56): every entry point returns size_t, errors are (size_t)-code.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>

namespace fseb {

enum : unsigned {
    E_OK = 0, E_GENERIC = 1, E_DST_TOO_SMALL = 2, E_SRC_WRONG = 3, E_CORRUPT = 4,
    E_TLOG_TOO_LARGE = 5, E_MSV_TOO_LARGE = 6, E_MSV_TOO_SMALL = 7, E_WKSP_TOO_SMALL = 8, E_MAXCODE = 9
};

typedef unsigned long long u64;
typedef uint32_t u32;
typedef uint16_t u16;
typedef uint8_t u8;

__host__ __device__ __forceinline__ u64 err(unsigned code) { return (u64)0 - (u64)code; }
__host__ __device__ __forceinline__ bool is_err(u64 r) { return r > err(E_MAXCODE); }

// constants fixed by the wire format (lib/fse.h:641-676, lib/huf.h:117-119,72)
constexpr unsigned FSE_MIN_TLOG = 5, FSE_MAX_TLOG = 12, FSE_DEF_TLOG = 11, FSE_ABS_TLOG = 15, FSE_MAX_SV = 255;
constexpr unsigned HUF_MAX_TLOG = 12, HUF_DEF_TLOG = 11, HUF_MAX_SV = 255, HUF_BLOCK_MAX = 128 * 1024;
constexpr unsigned U16_MAX_SV = 286, U16_MAX_TLOG = 13, U16_DEF_TLOG = 12;

// Transient per-block result of the batch Huff0 decoder: "rejected by the single-symbol end-of-stream rule, to be re-examined
// under the double-symbol decoder's rules" (huf_x2_fixup.cu replaces it before the call returns).  Neither a size nor an error code.
constexpr u64 HUF_X2_PENDING = 0x8000000000000004ull;

__device__ __forceinline__ unsigned hibit(unsigned v) { return 31u - (unsigned)__clz((int)v); }   // v != 0
__device__ __forceinline__ unsigned lane_id() { return threadIdx.x & 31u; }

// unaligned little-endian reads through a byte pointer (generic address space)
__device__ __forceinline__ u32 rd16(const u8* p) { return (u32)p[0] | ((u32)p[1] << 8); }
__device__ __forceinline__ u32 rd32(const u8* p) { return rd16(p) | (rd16(p + 2) << 16); }

// -------------------------------------------------------------------------------------------
// Uniform batch geometry: the split programs/bench.c:530-548 performs on a flat buffer.
//   block b covers [b*blockSize, min(total,(b+1)*blockSize)); compressed block b lives in the
//   fixed slot cbuf + b*slot (slot = FSE_compressBound(blockSize) in the reference harness).
// -------------------------------------------------------------------------------------------
struct BatchGeom {
    static constexpr bool DESCS = false;
    u64 total;       // uncompressed bytes in the whole batch
    u32 blockSize;   // uncompressed bytes per block (last block may be shorter)
    u32 slot;        // byte stride between compressed blocks == per-block dst capacity
    u32 nBlocks;
};
__host__ __device__ __forceinline__ u32 block_len(const BatchGeom& g, u32 b)
{
    u64 const off = (u64)b * g.blockSize;
    u64 const left = g.total - off;
    return left < g.blockSize ? (u32)left : g.blockSize;
}

// -------------------------------------------------------------------------------------------
// Descriptor geometry: block b is wherever the caller's device arrays say, every block with its own sizes.
//   compress:   src[b] / srcSize[b] = uncompressed input, dst[b] / dstCap[b] = output capacity, result[b] = cSize
//   decompress: src[b] / srcSize[b] = compressed input,   dst[b] / dstCap[b] = dstSize,         result[b] = regenerated size
// Contract (include/fse_b200.h): no destination overlaps another destination, a source or the arrays; `result` overlaps no
// other array (the emit kernel, the decoder's verdicts and the X2 pass read the sizes after earlier kernels wrote results);
// sources may overlap each other; a compressed input is readable up to the end of the 32-byte sector that holds its last byte.
// -------------------------------------------------------------------------------------------
struct BlockDescs {
    static constexpr bool DESCS = true;
    u8* const* dst;
    const u64* dstCap;
    u64* result;
    const u8* const* src;
    const u64* srcSize;
    u32 nBlocks;
};

// Table reuse (Huff0 compress only): a descriptor batch whose block b also carries its stream's (table, repeat flag) pair --
// ctable[b] = 256 HUF_CElt cells (val | nbBits << 16), repeat[b] = HUF_repeat as an int, prefer[b] = preferRepeat.  The plan
// kernel reads and writes the pair; the emit kernel sees the batch as the BlockDescs it derives from.
struct RepeatDescs : BlockDescs {
    u32* const* ctable;
    int* repeat;
    const int* prefer;
};
// Chains of table reuse (Huff0 compress only): chain c is blocks [start[c], start[c + 1]) of one stream, in order; the stream's
// (table, flag, header) state comes in through ctable[c] / repeat[c] / hdr[c] / hdrSize[c] and goes back out there, and block b
// gets the header it was coded with in blkHdr[b] / blkHdrSize[b].  The plan kernel sees only the blocks and writes nothing but
// scratch: the state-independent facts of block b go to fact[b], and huf_chain_kernel walks each chain's decisions from them.
struct __align__(16) ChainFact {
    u64 exitValue;                 // kind CF_ARGS / CF_HIST: the verdict of that exit
    u64 hSize;                     // kind CF_TREE: the new table's header size, or an error
    u64 newValue;                  // kind CF_TREE with hSize + 12 < srcSize: the verdict with the new table (its plan is complete)
    u32 newBits;                   // ... and its HUF_estimateCompressedSize in bits
    u16 msv;                       // largest symbol present (kinds CF_HIST and CF_TREE)
    u8 kind;
};
enum : u8 { CF_ARGS = 0, CF_HIST = 1, CF_TREE = 2 };   // an argument verdict, a histogram exit, a tree was built
struct ChainDescs : BlockDescs {
    const u64* start;              // nChains + 1 entries
    u32 nChains;
    const int* prefer;             // per block
    u32* const* ctable;            // per chain, in-out
    int* repeat;
    const u8** hdr;
    u64* hdrSize;
    const u8** blkHdr;             // per block, out
    u64* blkHdrSize;
    ChainFact* fact;               // per block, scratch
};
// Header-less decode (Huff0 only): block b's tree header is read from hdr[b] (hdrSize[b] bytes, the table's bound) and its
// payload starts at src[b][0]; hdrSize[b] == 0 means the block carries its own header.
struct HeaderDescs : BlockDescs {
    const u8* const* hdr;
    const u64* hdrSize;
};

// -------------------------------------------------------------------------------------------
// Packed geometry (Huff0 compress only): sources by descriptor, outputs back to back in one buffer.  Block b is stored at
// out + offset[b], offset[] being the exclusive prefix sum of the stored lengths (include/fse_b200.h); its capacity is
// HUF_compressBound(srcSize), so its verdict is that of the reference at that capacity.  `offset` has nBlocks + 1 entries.
// -------------------------------------------------------------------------------------------
struct PackedDescs {
    static constexpr bool DESCS = true;
    u8* out;
    u64 outCap;
    u64* offset;
    u64* result;
    const u8* const* src;
    const u64* srcSize;
    u32 nBlocks;
};
// HUF_compressBound (lib/huf.h:131-133): the capacity of a packed block of n source bytes
__host__ __device__ __forceinline__ u64 huf_bound(u64 n) { return 129 + n + (n >> 8) + 8; }
// bytes a block takes in the packed output, from its compress verdict: the compressed size, the RLE byte, a raw copy of the
// source when the verdict is 0 (0 bytes for an empty block), nothing for an error
__host__ __device__ __forceinline__ u64 packed_len(u64 v, u64 n) { return is_err(v) ? 0 : (v ? v : n); }

// The Huff0 kernels locate a block only through these accessors, one set per geometry.  The uniform geometry's pointer
// arguments are the batch's buffers; the descriptor geometry ignores them (its launchers pass nullptr).
// A size above what any Huff0 block can have is reported as HUF_BLOCK_MAX + 1: every verdict the kernels derive from it
// ("larger than a block", "larger than the compressed size") is the same as for the literal value.
__device__ __forceinline__ u32 clamp_len(u64 n) { return n > HUF_BLOCK_MAX ? HUF_BLOCK_MAX + 1 : (u32)n; }

// encoder: uncompressed source, its length, the output, its capacity, the compressed size
__device__ __forceinline__ const u8* enc_src(const BatchGeom& g, const u8* src, u32 b) { return src + (u64)b * g.blockSize; }
__device__ __forceinline__ u32 enc_len(const BatchGeom& g, u32 b) { return block_len(g, b); }
__device__ __forceinline__ u8* enc_dst(BatchGeom g, u8* cbuf, u32 b) { return cbuf + (u64)b * g.slot; }   // by value: the emit kernel then compiles as it did before the accessors
__device__ __forceinline__ u64 enc_cap(const BatchGeom& g, u32) { return g.slot; }
__device__ __forceinline__ u64& enc_out(const BatchGeom&, u64* csizes, u32 b) { return csizes[b]; }
__device__ __forceinline__ const u8* enc_src(const BlockDescs& g, const u8*, u32 b) { return g.src[b]; }
__device__ __forceinline__ u32 enc_len(const BlockDescs& g, u32 b) { return clamp_len(g.srcSize[b]); }
__device__ __forceinline__ u8* enc_dst(const BlockDescs& g, u8*, u32 b) { return g.dst[b]; }
__device__ __forceinline__ u64 enc_cap(const BlockDescs& g, u32 b) { u64 const c = g.dstCap[b]; return c > 0xFFFFFF00ull ? 0xFFFFFF00ull : c; }   // as one_block_compress
__device__ __forceinline__ u64& enc_out(const BlockDescs& g, u64*, u32 b) { return g.result[b]; }
// packed: enc_dst is valid only once the placement kernel has written offset[b] (the emit kernel's use)
__device__ __forceinline__ const u8* enc_src(const PackedDescs& g, const u8*, u32 b) { return g.src[b]; }
__device__ __forceinline__ u32 enc_len(const PackedDescs& g, u32 b) { return clamp_len(g.srcSize[b]); }
__device__ __forceinline__ u8* enc_dst(const PackedDescs& g, u8*, u32 b) { return g.out + g.offset[b]; }
__device__ __forceinline__ u64 enc_cap(const PackedDescs& g, u32 b) { return huf_bound(enc_len(g, b)); }
__device__ __forceinline__ u64& enc_out(const PackedDescs& g, u64*, u32 b) { return g.result[b]; }

// -------------------------------------------------------------------------------------------
// Packed chains of table reuse (Huff0 compress only): the chains of ChainDescs with every block's capacity HUF_compressBound(srcSize)
// and its bytes stored as PackedDescs stores them (`pk` is that view of the same call: out, outCap, offset, result, src, srcSize),
// plus one kind byte per block (include/fse_b200.h).  dst, dstCap, blkHdr and blkHdrSize are unused: a block's place is fixed
// only by the scan after the decisions, so huf_chain_kernel records per chain what the state write-back needs in end[c] instead
// of writing the state, and chainState writes it once the total is known to fit.
// -------------------------------------------------------------------------------------------
constexpr u32 CHAIN_NONE = 0xFFFFFFFFu;
struct ChainEnd {
    u32 lastNew;                   // the chain's last block coded with a new table (kind 2), or CHAIN_NONE
    u32 lastSaved;                 // the chain's last block that saved a table, or CHAIN_NONE
    int flag;                      // the flag after the chain's last block
};
struct ChainPackedDescs : ChainDescs {
    PackedDescs pk;
    u8* kind;                      // per block, out
    ChainEnd* end;                 // per chain, scratch
    const u32* malformed;          // scratch: the chain geometry's verdict
};
__device__ __forceinline__ u64 enc_cap(const ChainPackedDescs& g, u32 b) { return huf_bound(enc_len(g, b)); }
__device__ __forceinline__ u8* enc_dst(const ChainPackedDescs& g, u8*, u32 b) { return g.pk.out + g.pk.offset[b]; }   // after placement

// Mixed chains: ChainDescs or ChainPackedDescs whose blocks each choose their form -- single[b] == 0: HUF_compress4X_repeat,
// anything else: HUF_compress1X_repeat.  The kernels run them as stream mode 0 (huf_encode.cu); every other rule is the base's.
template <class Base>
struct Mixed : Base {
    const u8* single;              // per block
};
using ChainMixedDescs = Mixed<ChainDescs>;
using ChainPackedMixedDescs = Mixed<ChainPackedDescs>;
// Packed chains under zstd's literal-coding policy (include/fse_b200.h, FSEB200_HUF_compress_literals_chains_packed): the chain
// kernel chooses each block's form from the stream's flag and writes it to single[b], applies the size threshold minLiterals and
// the minimum gain (n >> minGainLog) + 2, and keeps a step's (table, flag) only when the block is stored with its own header.  The
// plan kernel plans the form n alone decides (1X below 256 bytes, else 4X); the chain kernel re-plans 256 <= n < 1024 as 1X when
// the flag is 2.  The chain kernel also writes each block's kind, which the placement (HufLiteralsPlace) stores by.
struct ChainPackedLiteralsDescs : ChainPackedDescs {
    u8* single;                    // per block, out
    u32 minLiterals;
    u32 minGainLog;                // 1 .. 31
};
// block b's form: true for one stream.  Only mixed geometry has a choice; the literal policy's plan takes the form n decides.
template <class Geo> __device__ __forceinline__ bool enc_single(const Geo&, u32) { return false; }
template <class Base> __device__ __forceinline__ bool enc_single(const Mixed<Base>& g, u32 b) { return g.single[b] != 0; }
__device__ __forceinline__ bool enc_single(const ChainPackedLiteralsDescs& g, u32 b) { return enc_len(g, b) < 256; }

// decoder: compressed source, its size, the output, the regenerated size, the result; `orig` (stored blocks) is uniform-only
__device__ __forceinline__ const u8* dec_src(const BatchGeom& g, const u8* cbuf, u32 b) { return cbuf + (u64)b * g.slot; }
__device__ __forceinline__ u64 dec_csize(const BatchGeom&, const u64* csizes, u32 b) { return csizes[b]; }
__device__ __forceinline__ u8* dec_dst(const BatchGeom& g, u8* dst, u32 b) { return dst + (u64)b * g.blockSize; }
__device__ __forceinline__ u32 dec_len(const BatchGeom& g, u32 b) { return block_len(g, b); }
__device__ __forceinline__ u64& dec_out(const BatchGeom&, u64* results, u32 b) { return results[b]; }
__device__ __forceinline__ const u8* dec_orig(const BatchGeom& g, const u8* orig, u32 b) { return orig + (u64)b * g.blockSize; }
__device__ __forceinline__ const u8* dec_src(const BlockDescs& g, const u8*, u32 b) { return g.src[b]; }
__device__ __forceinline__ u64 dec_csize(const BlockDescs& g, const u64*, u32 b) { return g.srcSize[b]; }
__device__ __forceinline__ u8* dec_dst(const BlockDescs& g, u8*, u32 b) { return g.dst[b]; }
__device__ __forceinline__ u32 dec_len(const BlockDescs& g, u32 b) { return clamp_len(g.dstCap[b]); }
__device__ __forceinline__ u64& dec_out(const BlockDescs& g, u64*, u32 b) { return g.result[b]; }
__device__ __forceinline__ const u8* dec_orig(const BlockDescs&, const u8*, u32) { return nullptr; }
// The lowest address the decoder's stream feeder may read for block b: the batch buffer's first 32-byte sector, or, for
// descriptors, the block's own first sector (a block may be the first bytes of an allocation).
__device__ __forceinline__ u64 dec_floor(const BatchGeom&, const u8* cbuf, const u8*) { return reinterpret_cast<u64>(cbuf) & ~31ull; }
__device__ __forceinline__ u64 dec_floor(const BlockDescs&, const u8*, const u8* block) { return reinterpret_cast<u64>(block) & ~31ull; }

// FSE and FSE-U16 blocks: the batch tier's limit is 2^30 bytes per source, capacity and compressed size (U16: 2^29 symbols).
// The U16 descriptor calls count uncompressed sizes in 16-bit symbols, as FSE_compressU16 / FSE_decompressU16 do; fse_bytes
// turns such a size into bytes and reports anything above the limit as FSE_BLOCK_MAX + 1, which the kernels answer with
// srcSize_wrong.  The uncompressed length of a block, in bytes, through either geometry:
constexpr u64 FSE_BLOCK_MAX = 1ull << 30;
__device__ __forceinline__ u64 fse_bytes(u64 v, bool wide)
{
    if (wide) return v > FSE_BLOCK_MAX / 2 ? FSE_BLOCK_MAX + 1 : 2 * v;
    return v > FSE_BLOCK_MAX ? FSE_BLOCK_MAX + 1 : v;
}
__device__ __forceinline__ u64 fse_enc_len(const BatchGeom& g, u32 b, bool) { return block_len(g, b); }
__device__ __forceinline__ u64 fse_enc_len(const BlockDescs& g, u32 b, bool wide) { return fse_bytes(g.srcSize[b], wide); }
__device__ __forceinline__ u64 fse_dec_len(const BatchGeom& g, u32 b, bool) { return block_len(g, b); }
__device__ __forceinline__ u64 fse_dec_len(const BlockDescs& g, u32 b, bool wide) { return fse_bytes(g.dstCap[b], wide); }

}  // namespace fseb
