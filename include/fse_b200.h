/*
 * fse_b200.h -- C-ABI of libfse_b200.so: the H100 (sm_90a) implementation of the FSE / Huff0 block
 * entropy-coding hot path of Cyan4973/FiniteStateEntropy.
 *
 * Plain C: pointers and sizes only.  Link with -lfse_b200 (the library carries its own CUDA runtime).
 * All `file:line` citations are relative to the reference tree (/root/reference).
 *
 * Conventions kept from the reference (lib/error_private.h:77-79, lib/error_public.h:45-56):
 *   - every function returns size_t; errors are (size_t)-code, test with FSE_isError()/HUF_isError();
 *   - compressors return 0 = "not compressible / does not fit, nothing stored" and 1 = "single symbol,
 *     use RLE" in-band (lib/fse.h:63-65, lib/huf.h:51-52; HUF also stores the byte in dst[0]);
 *   - tables are caller-owned `unsigned[]` with the reference's documented layouts and sizes
 *     (lib/fse.h:295-300, lib/huf.h:136-149).
 *
 * Tier 1 (FSEB200_*_batch) works on DEVICE memory and a CUDA stream, a whole batch per call; FSEB200_{HUF,FSE,FSEU16}_*_blocks
 * does the same for blocks of any size at any address, given by per-block device descriptors.
 * Tier 2 (the reference's own names) works on HOST memory, one block per synchronous call, and is
 * implemented by running the same kernels with a batch of one -- a correct drop-in for unmodified
 * callers (programs/bench.c, the fuzzers), not the fast path.
 * There is no CPU fallback: with no usable CUDA device a data-path call aborts with a message.
 */
#ifndef FSE_B200_H
#define FSE_B200_H
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------------
 * Tier 1 -- batched entry points (extension).  They replace the per-chunk loops of the reference
 * harness, programs/bench.c:353-364 (compress) and :389-424 (decompress), by one launch.
 *
 * Geometry (programs/bench.c:530-548): a flat buffer of `total` uncompressed bytes is cut into
 * ceil(total/blockSize) blocks of `blockSize` bytes (the last one shorter); compressed block b lives in
 * the fixed slot dCBuf + b*slot and may use `slot` bytes (bench.c uses FSE_compressBound(blockSize));
 * dCSizes[b] is exactly what the reference's FSE_compress2 / HUF_compress2 / FSE_compressU16 returns
 * for that block (0, 1, size, or an error code).  Bytes of a slot beyond the returned size are scratch.
 * Decompression writes block b at dDst + b*blockSize and dResults[b] = regenerated size or error code;
 * blocks with dCSizes[b]==0 (stored raw) or ==1 (RLE) are regenerated from dOrig as bench.c:393-402
 * does when dOrig != NULL (HUF additionally handles cSize==origSize / cSize==1 itself, lib/huf.h:60-63).
 * For the U16 codec sizes are in BYTES (a block holds blockSize/2 symbols, bench.c:221).
 * All pointers are device pointers; `stream` is a cudaStream_t (NULL = default stream).
 * The compressed buffer must be readable for 32 bytes past the last block's compressed bytes (the decoders load aligned 16- / 32-byte
 * pieces; what lies beyond a block's own bytes is never interpreted) -- bench.c's own buffer of nbChunks * FSE_compressBound() has it.
 * Alignment and stride: for the byte codecs (HUF, FSE) dSrc, dCBuf and dDst may have any byte alignment and `slot` any value,
 * odd or below FSE_compressBound(blockSize) (a block that does not fit its slot gets the reference's verdict for that
 * dstCapacity); buffers may straddle a 4 GiB address boundary.  FSE-U16 holds unsigned shorts: dSrc and dDst must be 2-byte
 * aligned and blockSize even; its dCBuf and `slot` are tested at even values.  The test-suite checks offsets 0, 1 (U16: 2),
 * 4, 8, 16, 32, 64 and 96 from a 512-byte aligned start, odd, 128-multiple and below-bound strides, and views across 2^32.
 * Return value: 0, or an error code if the launch itself could not be made.
 * ------------------------------------------------------------------------------------------------ */
size_t FSEB200_HUF_compress_batch(void* dCBuf, size_t slot, size_t* dCSizes, const void* dSrc, size_t srcTotal,
                                  size_t blockSize, unsigned maxSymbolValue, unsigned tableLog, void* stream);
size_t FSEB200_HUF_decompress_batch(void* dDst, size_t dstTotal, size_t blockSize, const void* dCBuf, size_t slot,
                                    const size_t* dCSizes, size_t* dResults, const void* dOrig, void* stream);
size_t FSEB200_FSE_compress_batch(void* dCBuf, size_t slot, size_t* dCSizes, const void* dSrc, size_t srcTotal,
                                  size_t blockSize, unsigned maxSymbolValue, unsigned tableLog, void* stream);
size_t FSEB200_FSE_decompress_batch(void* dDst, size_t dstTotal, size_t blockSize, const void* dCBuf, size_t slot,
                                    const size_t* dCSizes, size_t* dResults, const void* dOrig, void* stream);
size_t FSEB200_FSEU16_compress_batch(void* dCBuf, size_t slot, size_t* dCSizes, const void* dSrc, size_t srcTotal,
                                     size_t blockSize, unsigned maxSymbolValue, unsigned tableLog, void* stream);
size_t FSEB200_FSEU16_decompress_batch(void* dDst, size_t dstTotal, size_t blockSize, const void* dCBuf, size_t slot,
                                       const size_t* dCSizes, size_t* dResults, const void* dOrig, void* stream);
size_t FSEB200_batch_blocks(size_t total, size_t blockSize);

/* Tier 1, per-block descriptors (Huff0): block b has its own addresses and sizes, given by device arrays -- e.g. the
 * variable-size literal sections of a zstd-style caller, packed back to back.  All six arrays and every buffer they point to
 * are in DEVICE memory; the call is asynchronous on `stream` and the host never reads the arrays (no copy, no synchronize).
 *   compress:   dCSizes[b] = exactly what HUF_compress2(dDsts[b], dDstCapacities[b], dSrcs[b], dSrcSizes[b], maxSymbolValue,
 *               tableLog) returns: 0, 1 (the byte in dDsts[b][0]), a size or an error code; bytes [0, dCSizes[b]) are the
 *               reference's.  Per-block verdicts come from the kernels: srcSize > 128 KB gives srcSize_wrong, a bad
 *               maxSymbolValue / tableLog the reference's error, and a capacity above 2^32 acts as 0xFFFFFF00.
 *   decompress: dResults[b] = exactly what this library's HUF_decompress(dDsts[b], dDstSizes[b], dCSrcs[b], dCSrcSizes[b])
 *               returns, sizes taken literally: dstSize 0 gives dstSize_tooSmall, dstSize > 128 KB srcSize_wrong, cSize >
 *               dstSize corruption_detected, cSize == dstSize is a raw copy, cSize == 1 RLE, anything else is Huffman-decoded
 *               with the decoder (and verdict on malformed input) HUF_selectDecoder picks.  Unlike the uniform call, cSize 0
 *               does not mean "stored" and an error code in dCSrcSizes is not passed through.
 * Contract: no destination may overlap another destination, any source or the arrays (sources may overlap each other), and
 * the output array (dCSizes / dResults) may not overlap the other arrays: the kernels read the sizes again after writing it.  Each
 * compressed input must be readable up to the end of the 32-byte-aligned sector that holds its last byte (blocks packed back
 * to back meet this when the buffer has 32 bytes of slack).  Bytes of [dst, dst + capacity) beyond the returned size are
 * unspecified; nothing outside the destinations is written.
 * Return value: 0 (also for nBlocks == 0, which launches nothing); srcSize_wrong if nBlocks > 0xFFFFFFFF or an array is NULL
 * while nBlocks > 0; generic if a launch fails. */
size_t FSEB200_HUF_compress_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstCapacities, size_t* dCSizes,
                                   const void* const* dSrcs, const size_t* dSrcSizes,
                                   unsigned maxSymbolValue, unsigned tableLog, void* stream);
size_t FSEB200_HUF_decompress_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstSizes, size_t* dResults,
                                     const void* const* dCSrcs, const size_t* dCSrcSizes, void* stream);

/* Tier 1, per-block descriptors (single-stream Huff0, the "1X" format of lib/huf.h:288-335: tree header + one bitstream, no
 * jump table) -- e.g. the small literal sections a zstd-style caller codes as one stream.  Argument shape, asynchrony,
 * contract and return value are those of FSEB200_HUF_{compress,decompress}_blocks above; every block builds and carries its
 * own table.
 *   compress:   dCSizes[b] = exactly what HUF_compress1X(dDsts[b], dDstCapacities[b], dSrcs[b], dSrcSizes[b], maxSymbolValue,
 *               tableLog) returns: 0, 1 (the byte in dDsts[b][0]), a size or an error code; bytes [0, dCSizes[b]) are the
 *               reference's.  srcSize > 128 KB gives srcSize_wrong, a bad maxSymbolValue / tableLog the reference's error, and
 *               a capacity above 2^32 acts as 0xFFFFFF00.
 *   decompress: dResults[b] = exactly what HUF_decompress1X_DCtx(dctx, dDsts[b], dDstSizes[b], dCSrcs[b], dCSrcSizes[b])
 *               returns for a fresh HUF_CREATE_STATIC_DTABLEX2(dctx, HUF_TABLELOG_MAX), sizes taken literally: dstSize 0
 *               gives dstSize_tooSmall, cSize > dstSize corruption_detected, cSize == dstSize is a raw copy, cSize == 1 RLE,
 *               anything else is decoded with the decoder (and verdict on malformed input) HUF_selectDecoder picks.
 *               Deviation: the reference's 1X decoder has no block-size limit; here dstSize > 128 KB gives srcSize_wrong,
 *               as in FSEB200_HUF_decompress_blocks. */
size_t FSEB200_HUF_compress1X_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstCapacities, size_t* dCSizes,
                                     const void* const* dSrcs, const size_t* dSrcSizes,
                                     unsigned maxSymbolValue, unsigned tableLog, void* stream);
size_t FSEB200_HUF_decompress1X_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstSizes, size_t* dResults,
                                       const void* const* dCSrcs, const size_t* dCSrcSizes, void* stream);

/* Tier 1, per-block descriptors with table reuse (Huff0, 4X and 1X): the zstd-style literal coder's pattern, where each stream keeps
 * a (table, repeat flag) pair and every block decides whether to reuse the previous table, check it first, or build a new one.
 * Block b carries its stream's pair: dCTables[b] (device array of device pointers) = 256 HUF_CElt cells in this library's layout
 * (val | nbBits << 16, as HUF_buildCTable and HUF_readCTable give them), dRepeats[b] = a HUF_repeat (none 0, check 1, valid 2),
 * dPreferRepeat[b] = preferRepeat.  Blocks of one stream go to successive calls, so a batch with one block from each of many
 * streams is fully parallel.  Argument shape, asynchrony, limits, contract and return value are those of
 * FSEB200_HUF_{compress,decompress}{,1X}_blocks; all arrays and buffers are in device memory and the host never reads them.
 *   compress:   per block, exactly what HUF_compress4X_repeat(dDsts[b], dDstCapacities[b], dSrcs[b], dSrcSizes[b], maxSymbolValue,
 *               tableLog, wksp, sizeof wksp, dCTables[b], &dRepeats[b], dPreferRepeat[b], 0) does with a zeroed, aligned, large
 *               enough workspace (1X: HUF_compress1X_repeat): dCSizes[b] is its return value (0, 1 with the byte in dDsts[b][0],
 *               a size or an error code), bytes [0, dCSizes[b]) are its bytes, and dRepeats[b] and all 256 words of dCTables[b]
 *               hold what it leaves there.  A table is written only where the reference saves a new one (cells above the
 *               block's largest symbol zeroed), a flag only where the reference sets it to none.  Byte 3 of every cell the call
 *               stores is 0.  Flag values are taken literally, as the reference's comparisons with 0, 1 and 2 take them.
 *               The workspace checks have no counterpart here, and a capacity above 2^32 acts as 0xFFFFFF00.
 *               Telling the two kinds of block apart: for a block whose dCSizes[b] is 2 or more, dRepeats[b] != 0 after the call
 *               exactly when the block was coded with the old table and carries no tree header.
 *               No table may overlap another block's table, a source, a destination or an array.
 *   decompress: per block, with DT a fresh HUF_CREATE_STATIC_DTABLEX1(DT, HUF_TABLELOG_MAX):
 *               dHeaderSizes[b] == 0: the block carries its own tree header, and dResults[b] is exactly
 *                 HUF_decompress4X1_DCtx(DT, dDsts[b], dDstSizes[b], dCSrcs[b], dCSrcSizes[b]) (1X: HUF_decompress1X1_DCtx) --
 *                 no raw or RLE forms, and the single-symbol decoder's verdicts;
 *               otherwise h = HUF_readDTableX1(DT, dHeaders[b], dHeaderSizes[b]); dResults[b] is h if that is an error, else
 *                 HUF_decompress4X1_usingDTable(dDsts[b], dDstSizes[b], dCSrcs[b], dCSrcSizes[b], DT) (1X:
 *                 HUF_decompress1X1_usingDTable): the payload starts at dCSrcs[b][0].
 *               A header may lie anywhere, inside another block's compressed bytes included: typically the start of the block of
 *               the same stream that last carried a table, with dHeaderSizes[b] = that block's compressed size.  Headers may
 *               overlap each other and the sources, and must be readable to the end of their 32-byte sector, like compressed
 *               inputs.  Deviations, where the reference's call has no such limit: dstSize > 128 KB gives srcSize_wrong, and a 4X
 *               dstSize below 6 gives corruption_detected (the reference writes out of bounds there).  Any cSize is taken
 *               literally: a stream longer than any decode can consume gets the reference's corruption_detected. */
size_t FSEB200_HUF_compress4X_repeat_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstCapacities, size_t* dCSizes,
                                            const void* const* dSrcs, const size_t* dSrcSizes,
                                            unsigned* const* dCTables, int* dRepeats, const int* dPreferRepeat,
                                            unsigned maxSymbolValue, unsigned tableLog, void* stream);
size_t FSEB200_HUF_compress1X_repeat_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstCapacities, size_t* dCSizes,
                                            const void* const* dSrcs, const size_t* dSrcSizes,
                                            unsigned* const* dCTables, int* dRepeats, const int* dPreferRepeat,
                                            unsigned maxSymbolValue, unsigned tableLog, void* stream);
/* Tier 1, chains of table reuse (Huff0, 4X and 1X): whole runs of one stream's blocks in one call, the stream's state carried
 * from block to block on the device -- one long stream of literal blocks, as a zstd-style compressor makes from one file, needs
 * no call per block.  All arrays and buffers are in device memory, the call is asynchronous on `stream`, and the host never reads
 * the arrays.  Chain c is blocks [dChainStarts[c], dChainStarts[c+1]) in order (dChainStarts has nChains + 1 entries); block
 * descriptors (dDsts .. dSrcSizes), dPreferRepeat, dHeaders and dHeaderSizes are per block; dCTables[c], dRepeats[c],
 * dChainHeaders[c] and dChainHeaderSizes[c] are per chain, in-out: the stream's state when the chain starts, and when it ends.
 * Each chain gives exactly what this loop gives, from T = dCTables[c], F = dRepeats[c], H = (dChainHeaders[c], dChainHeaderSizes[c]):
 *     for (b = dChainStarts[c]; b < dChainStarts[c+1]; b++) {
 *         r = HUF_compress4X_repeat(dDsts[b], dDstCapacities[b], dSrcs[b], dSrcSizes[b], maxSymbolValue, tableLog,
 *                                   wksp, sizeof wksp, T, &F, dPreferRepeat[b], 0);          (1X: HUF_compress1X_repeat)
 *         dCSizes[b] = r;
 *         if (!isError(r) && r >= 2 && F != 0) { dHeaders[b] = H.ptr; dHeaderSizes[b] = H.size; }    coded with the old table
 *         else                                  { dHeaders[b] = NULL;  dHeaderSizes[b] = 0; }
 *         if (!isError(r) && r >= 2 && F == 0) { F = 1; H = (dDsts[b], r); }                        carries a new table: check it next
 *     }
 * and then writes T (only if a block saved a table), F and H back to the chain's entries; an empty chain writes nothing.  Each step
 * has the single-block semantics of FSEB200_HUF_compress{4X,1X}_repeat_blocks (a zeroed workspace, a table written only where the
 * reference saves one, byte 3 of stored cells 0, flag values taken literally, a capacity above 2^32 acting as 0xFFFFFF00).
 * dHeaders / dHeaderSizes are exactly the header arrays FSEB200_HUF_decompress{4X,1X}_repeat_blocks take: the blocks with
 * dCSizes[b] >= 2 decode in one such call; the caller handles those stored raw (0) or as RLE (1) itself.  A chain that enters with
 * F != 0 needs dChainHeaderSizes[c] = the size of that table's header source; its old-table blocks inherit it as given.
 * Returns 0 for nBlocks == 0 (nothing launched); srcSize_wrong, the device untouched, for nBlocks or nChains above 0xFFFFFFFF or a
 * NULL array while nBlocks > 0; generic if a launch fails.  Malformed chain geometry (dChainStarts[0] != 0,
 * dChainStarts[nChains] != nBlocks, or a decrease) is found on the device: then every dCSizes[b] is srcSize_wrong and nothing
 * else is written -- no destination, table, flag or header.
 * Contract: that of FSEB200_HUF_compress{4X,1X}_repeat_blocks, and no per-chain state array overlaps another array, and no table
 * belongs to two chains.  The decisions of a chain run one block after another on one warp: a single chain of many blocks takes
 * time in proportion to its length (DESIGN.md 4.2). */
size_t FSEB200_HUF_compress4X_repeat_chains(size_t nChains, const size_t* dChainStarts, size_t nBlocks,
                                            void* const* dDsts, const size_t* dDstCapacities, size_t* dCSizes,
                                            const void* const* dSrcs, const size_t* dSrcSizes, const int* dPreferRepeat,
                                            unsigned* const* dCTables, int* dRepeats, const void** dChainHeaders, size_t* dChainHeaderSizes,
                                            const void** dHeaders, size_t* dHeaderSizes,
                                            unsigned maxSymbolValue, unsigned tableLog, void* stream);
size_t FSEB200_HUF_compress1X_repeat_chains(size_t nChains, const size_t* dChainStarts, size_t nBlocks,
                                            void* const* dDsts, const size_t* dDstCapacities, size_t* dCSizes,
                                            const void* const* dSrcs, const size_t* dSrcSizes, const int* dPreferRepeat,
                                            unsigned* const* dCTables, int* dRepeats, const void** dChainHeaders, size_t* dChainHeaderSizes,
                                            const void** dHeaders, size_t* dHeaderSizes,
                                            unsigned maxSymbolValue, unsigned tableLog, void* stream);
size_t FSEB200_HUF_decompress4X_repeat_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstSizes, size_t* dResults,
                                              const void* const* dCSrcs, const size_t* dCSrcSizes,
                                              const void* const* dHeaders, const size_t* dHeaderSizes, void* stream);
size_t FSEB200_HUF_decompress1X_repeat_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstSizes, size_t* dResults,
                                              const void* const* dCSrcs, const size_t* dCSrcSizes,
                                              const void* const* dHeaders, const size_t* dHeaderSizes, void* stream);

/* Tier 1, per-block descriptors with packed output (Huff0, 4X and 1X): the blocks given by dSrcs / dSrcSizes are compressed and
 * stored back to back in one buffer, each at an offset the call computes on the device -- no per-block reservation, no
 * compaction pass, and the stream decodes with the descriptor decoders above.  Per block b, with n = dSrcSizes[b]:
 *   dCSizes[b]  = exactly what HUF_compress2(dst, HUF_compressBound(n), src, n, maxSymbolValue, tableLog) returns (the 1X call:
 *                 HUF_compress1X): 0, 1, a size or an error code -- except for a block that does not fit (below).
 *   stored length L[b]: dCSizes[b] >= 2: dCSizes[b], the reference's compressed bytes; 1: 1, the byte src[0] (RLE); 0: n, a raw
 *                 copy of the source (0 bytes for an empty block); an error code: 0, nothing stored.
 *                 L[b] <= n always (a compressed block is shorter than n - 1 bytes, lib/huf_compress.c:625), so an outCapacity
 *                 of sum(n) always holds every block; add 32 bytes of slack for the decoders' sector reads.
 *   dOffsets    has nBlocks + 1 entries: dOffsets[b] = L[0] + ... + L[b-1], dOffsets[nBlocks] = the total.  It is written in
 *                 full even when blocks do not fit, so a too-small call still tells the size it needs.
 *   capacity    block b is stored at dOut + dOffsets[b] only if dOffsets[b] + L[b] <= outCapacity; otherwise dCSizes[b] =
 *                 dstSize_tooSmall and nothing is written for it (a block whose value is an error code keeps it).  Nothing
 *                 outside [dOut, dOut + min(total, outCapacity)) is ever written.
 * Decoding: FSEB200_HUF_decompress_blocks (1X: FSEB200_HUF_decompress1X_blocks) with dCSrcs[b] = dOut + dOffsets[b],
 * dCSrcSizes[b] = L[b] = dOffsets[b+1] - dOffsets[b] and dDstSizes[b] = n regenerates every non-empty block whose dCSizes[b]
 * is not an error code (HUF_decompress reads cSize == dstSize as a raw copy and cSize == 1 as RLE, lib/huf.h:60-63) -- with the
 * reference's own exception: it cannot decode a few of its compressed blocks (a code of length 1 at tableLog 12 is written as
 * weight 12, which HUF_readStats rejects, entropy_common.c:191), and the decoders return its verdict for them.
 * All arrays and buffers are in DEVICE memory; the call is asynchronous on `stream` and the host never reads the arrays.
 * Contract: dOut, dOffsets and dCSizes overlap no source and no other array; sources may overlap each other.
 * Return value: 0 (also for nBlocks == 0, which launches nothing and writes nothing, not even dOffsets[0]); srcSize_wrong if
 * nBlocks > 0xFFFFFFFF or a pointer is NULL while nBlocks > 0; generic if a launch fails. */
size_t FSEB200_HUF_compress_packed(size_t nBlocks, void* dOut, size_t outCapacity, size_t* dOffsets, size_t* dCSizes,
                                   const void* const* dSrcs, const size_t* dSrcSizes,
                                   unsigned maxSymbolValue, unsigned tableLog, void* stream);
size_t FSEB200_HUF_compress1X_packed(size_t nBlocks, void* dOut, size_t outCapacity, size_t* dOffsets, size_t* dCSizes,
                                     const void* const* dSrcs, const size_t* dSrcSizes,
                                     unsigned maxSymbolValue, unsigned tableLog, void* stream);
/* Packed decompress (Huff0, 4X and 1X): every block of a buffer the packed compress above wrote, located by its offsets -- the
 * recipe above without building the descriptor arrays.  Per block b, with L = dOffsets[b+1] - dOffsets[b] and n = dDstSizes[b]
 * (the regenerated size, not a capacity):
 *   n == 0 and L == 0: the result is 0 and nothing is written (an empty block as the packed compress stores it);
 *   otherwise exactly what FSEB200_HUF_decompress_blocks (1X: FSEB200_HUF_decompress1X_blocks) returns for dCSrcs[b] = dIn +
 *   dOffsets[b], dCSrcSizes[b] = L and dDstSizes[b] = n: a raw copy at L == n, RLE at L == 1, the decoders' limit verdicts, and
 *   the reference's weight-12 exception above.
 * So every block the packed compress stored with a value that is not an error decodes back to its source, but for that exception.
 * All arrays and buffers are in DEVICE memory; the calls are asynchronous on `stream`, the host never reads the arrays, and the
 * only memory they take is stream-ordered scratch of 16 bytes per block.
 * Contract: dIn must be readable up to the end of the 32-byte sector that holds each block's last byte; no destination may
 * overlap another destination, dIn or the arrays, and dResults overlaps no other array.
 * Return value: 0 (also for nBlocks == 0, which launches nothing and writes nothing); srcSize_wrong if nBlocks > 0xFFFFFFFF
 * or a pointer is NULL while nBlocks > 0; generic if a launch fails. */
size_t FSEB200_HUF_decompress_packed(size_t nBlocks, void* const* dDsts, const size_t* dDstSizes, size_t* dResults,
                                     const void* dIn, const size_t* dOffsets, void* stream);
size_t FSEB200_HUF_decompress1X_packed(size_t nBlocks, void* const* dDsts, const size_t* dDstSizes, size_t* dResults,
                                       const void* dIn, const size_t* dOffsets, void* stream);

/* Tier 1, packed chains of table reuse (Huff0, 4X and 1X): FSEB200_HUF_compress{4X,1X}_repeat_chains with every block stored back
 * to back in one buffer, as the packed calls above store blocks, and one kind byte per block -- a stream a caller can write, send
 * or move as it is: bytes, nBlocks + 1 offsets and nBlocks kinds are all its decoder needs, and no header is named by a pointer.
 * Kinds are numbered as zstd numbers its literal block types:
 *   0 raw (n bytes of source), 1 RLE (one byte), 2 compressed with its own tree header, 3 compressed with the stream's previous
 *   table and no header ("treeless"), 4 nothing stored.
 * Chain geometry (dChainStarts, nChains + 1 entries), the per-block dSrcs / dSrcSizes / dPreferRepeat, the per-chain in-out state
 * (dCTables, dRepeats, dChainHeaders, dChainHeaderSizes), the asynchrony and the argument verdicts are those of
 * FSEB200_HUF_compress{4X,1X}_repeat_chains, and each chain runs the loop documented there with dDstCapacities[b] =
 * HUF_compressBound(n) (n = dSrcSizes[b]), so no value is ever "does not fit its destination".  Per block b, with r its value:
 *   dCSizes[b]  = r, except for a block that does not fit dOut (below).
 *   stored length L[b] = that of FSEB200_HUF_compress_packed: r for r >= 2, 1 for r == 1 (the byte the reference leaves at dst[0]:
 *                 src[0] for RLE), n (a raw copy) for r == 0, 0 for an error.  L[b] <= n, so sum(n) + 32 bytes of slack always fits.
 *   dKinds[b]   = 0 for r == 0; 1 for r == 1; for r >= 2, 2 if the stream's flag is 0 after the step (a new table, its header
 *                 first) and 3 if it is not (the old table, no header: what the chain call reports as dHeaderSizes[b] != 0);
 *                 4 when dCSizes[b] is an error.  (A 1X block coded with the old table into a single byte also has r == 1, as in
 *                 the reference, whose decoders read a 1-byte block as RLE.)
 *   dOffsets    the packed calls' rule: the exclusive prefix sum of L, dOffsets[nBlocks] the total, written in full even when
 *                 blocks do not fit.
 *   capacity    block b is stored at dOut + dOffsets[b] only if dOffsets[b] + L[b] <= outCapacity; otherwise dCSizes[b] =
 *                 dstSize_tooSmall and dKinds[b] = 4.  Nothing outside [dOut, dOut + min(total, outCapacity)) is ever written.
 * Per-chain state on return:
 *   if dOffsets[nBlocks] <= outCapacity: what the loop leaves (table, flag), and the chain header (dOut + dOffsets[j], L[j]) for the
 *     chain's last kind-2 block j, or as it came in if the chain has none;
 *   otherwise every per-chain entry exactly as it came in, so the same call can be repeated with a buffer of dOffsets[nBlocks]
 *     bytes.  Storage is monotone in offset order: when the total does not fit, the blocks that are stored are exactly those
 *     before the first that does not, so a stored kind-3 block's header (the last kind-2 block before it in its chain, or the
 *     chain's entry header) is stored too; and since the state is left as it came in, no later call can be handed a header
 *     that was never stored.
 * Malformed chain geometry (as for the chain calls): every dCSizes[b] is srcSize_wrong, every dKinds[b] is 4, and nothing else is
 * written -- no byte of dOut, no offset, table, flag or header.
 * Contract: that of FSEB200_HUF_compress{4X,1X}_repeat_chains and of the packed calls; dKinds overlaps no other array.
 * Return value: 0 (also for nBlocks == 0, which launches nothing and writes nothing); srcSize_wrong, the device untouched, for
 * nBlocks or nChains above 0xFFFFFFFF or a NULL array while nBlocks > 0; generic if a launch fails. */
size_t FSEB200_HUF_compress4X_repeat_chains_packed(size_t nChains, const size_t* dChainStarts, size_t nBlocks,
                                                   void* dOut, size_t outCapacity, size_t* dOffsets, size_t* dCSizes, unsigned char* dKinds,
                                                   const void* const* dSrcs, const size_t* dSrcSizes, const int* dPreferRepeat,
                                                   unsigned* const* dCTables, int* dRepeats, const void** dChainHeaders, size_t* dChainHeaderSizes,
                                                   unsigned maxSymbolValue, unsigned tableLog, void* stream);
size_t FSEB200_HUF_compress1X_repeat_chains_packed(size_t nChains, const size_t* dChainStarts, size_t nBlocks,
                                                   void* dOut, size_t outCapacity, size_t* dOffsets, size_t* dCSizes, unsigned char* dKinds,
                                                   const void* const* dSrcs, const size_t* dSrcSizes, const int* dPreferRepeat,
                                                   unsigned* const* dCTables, int* dRepeats, const void** dChainHeaders, size_t* dChainHeaderSizes,
                                                   unsigned maxSymbolValue, unsigned tableLog, void* stream);
/* Packed chains decompress (Huff0, 4X and 1X): every block of a buffer the calls above wrote, from its offsets and kinds.  Per block
 * b of chain c, with L = dOffsets[b+1] - dOffsets[b], n = dDstSizes[b] (the regenerated size) and p = dIn + dOffsets[b]:
 *   n above 128 KB: srcSize_wrong, whatever the kind (the repeat decoders' limit);
 *   kind 0: L == n: the block is copied and the result is n (n == 0 included); otherwise corruption_detected;
 *   kind 1: L == 1: n copies of p[0], the result n; otherwise corruption_detected;
 *   kind 2: exactly what FSEB200_HUF_decompress{4X,1X}_repeat_blocks gives for (p, L) with header size 0;
 *   kind 3: exactly what that call gives with the header (dIn + dOffsets[j], L[j]), j the last kind-2 block before b in chain c,
 *           or (dChainHeaders[c], dChainHeaderSizes[c]) if there is none -- corruption_detected if that size is 0;
 *   any other kind: corruption_detected.
 * Malformed chain geometry makes every result srcSize_wrong, and nothing else is written.  So every block the calls above stored
 * with a value that is not an error decodes back to its source, but for the weight-12 exception of the packed calls, and the
 * kind-3 blocks that take their table from such a block.  dChainHeaders / dChainHeaderSizes are what the chains entered the
 * compress call with; a chain cut into several calls enters the next with a header inside the previous call's buffer.
 * All arrays and buffers are in DEVICE memory; the calls are asynchronous on `stream`, the host never reads the arrays, and the
 * only memory they take is stream-ordered scratch of about 50 bytes per block.
 * Contract: that of FSEB200_HUF_decompress_packed (dIn, and every header, readable up to the end of the 32-byte sector that holds
 * its last byte; no destination overlaps another destination, dIn, a header or the arrays; dResults overlaps no other array).
 * Return value: 0 (also for nBlocks == 0, which launches nothing and writes nothing); srcSize_wrong if nBlocks or nChains is
 * above 0xFFFFFFFF or a pointer is NULL while nBlocks > 0; generic if a launch fails. */
size_t FSEB200_HUF_decompress4X_repeat_packed(size_t nChains, const size_t* dChainStarts, size_t nBlocks,
                                              void* const* dDsts, const size_t* dDstSizes, size_t* dResults,
                                              const void* dIn, const size_t* dOffsets, const unsigned char* dKinds,
                                              const void* const* dChainHeaders, const size_t* dChainHeaderSizes, void* stream);
size_t FSEB200_HUF_decompress1X_repeat_packed(size_t nChains, const size_t* dChainStarts, size_t nBlocks,
                                              void* const* dDsts, const size_t* dDstSizes, size_t* dResults,
                                              const void* dIn, const size_t* dOffsets, const unsigned char* dKinds,
                                              const void* const* dChainHeaders, const size_t* dChainHeaderSizes, void* stream);

/* Tier 1, chains of table reuse whose blocks each choose one or four streams (Huff0): the chain and packed-chain calls above, with
 * one more per-block array, dSingleStream (unsigned char).  dSingleStream[b] == 0 codes step b of the loop with HUF_compress4X_repeat,
 * any other value with HUF_compress1X_repeat -- the value is taken literally, as dPreferRepeat is.  zstd's literal coder makes
 * that choice per section (one stream below 256 bytes) and both forms share the stream's table, flag and tree header: a header
 * written by a 4X block is read by HUF_readDTableX1 exactly as one written by a 1X block.  Every other rule is that of the 4X / 1X
 * call the mixed call stands for:
 *   FSEB200_HUF_compress_mixed_repeat_chains          FSEB200_HUF_compress{4X,1X}_repeat_chains, the form per block;
 *   FSEB200_HUF_decompress_mixed_repeat_blocks        per block exactly FSEB200_HUF_decompress{4X,1X}_repeat_blocks in its form,
 *                                                     so the chain call's output decodes in one call;
 *   FSEB200_HUF_compress_mixed_repeat_chains_packed   FSEB200_HUF_compress{4X,1X}_repeat_chains_packed: capacity HUF_compressBound(n)
 *                                                     for both forms, the same kinds (2 own header, 3 treeless, whatever the form),
 *                                                     offsets, capacity rule and state write-back;
 *   FSEB200_HUF_decompress_mixed_repeat_packed        FSEB200_HUF_decompress{4X,1X}_repeat_packed, the form from the flag; a kind-3
 *                                                     block's header is the last kind-2 block of its chain before it, whatever that
 *                                                     block's form, else the chain's entry header.
 * The form is not part of the kind byte: zstd carries it in the literal section header, apart from the block type, and the kinds
 * keep zstd's numbering.  A mixed packed stream is therefore its bytes, offsets, kinds and the per-block dSingleStream flags.
 * Argument verdicts are those of the 4X / 1X calls; a NULL dSingleStream while nBlocks > 0 is srcSize_wrong, the device untouched. */
size_t FSEB200_HUF_compress_mixed_repeat_chains(size_t nChains, const size_t* dChainStarts, size_t nBlocks,
                                                void* const* dDsts, const size_t* dDstCapacities, size_t* dCSizes,
                                                const void* const* dSrcs, const size_t* dSrcSizes, const int* dPreferRepeat,
                                                const unsigned char* dSingleStream,
                                                unsigned* const* dCTables, int* dRepeats, const void** dChainHeaders, size_t* dChainHeaderSizes,
                                                const void** dHeaders, size_t* dHeaderSizes,
                                                unsigned maxSymbolValue, unsigned tableLog, void* stream);
size_t FSEB200_HUF_decompress_mixed_repeat_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstSizes, size_t* dResults,
                                                  const void* const* dCSrcs, const size_t* dCSrcSizes,
                                                  const void* const* dHeaders, const size_t* dHeaderSizes,
                                                  const unsigned char* dSingleStream, void* stream);
size_t FSEB200_HUF_compress_mixed_repeat_chains_packed(size_t nChains, const size_t* dChainStarts, size_t nBlocks,
                                                       void* dOut, size_t outCapacity, size_t* dOffsets, size_t* dCSizes, unsigned char* dKinds,
                                                       const void* const* dSrcs, const size_t* dSrcSizes, const int* dPreferRepeat,
                                                       const unsigned char* dSingleStream,
                                                       unsigned* const* dCTables, int* dRepeats, const void** dChainHeaders, size_t* dChainHeaderSizes,
                                                       unsigned maxSymbolValue, unsigned tableLog, void* stream);
size_t FSEB200_HUF_decompress_mixed_repeat_packed(size_t nChains, const size_t* dChainStarts, size_t nBlocks,
                                                  void* const* dDsts, const size_t* dDstSizes, size_t* dResults,
                                                  const void* dIn, const size_t* dOffsets, const unsigned char* dKinds,
                                                  const unsigned char* dSingleStream,
                                                  const void* const* dChainHeaders, const size_t* dChainHeaderSizes, void* stream);

/* Tier 1, packed chains under zstd's literal-coding policy (Huff0): FSEB200_HUF_compress_mixed_repeat_chains_packed with the
 * decisions zstd's literal coder (ZSTD_compressLiterals, zstd 1.5) takes around each HUF_compress{4X,1X}_repeat call made on the
 * device from the state the chain carries: the form, the size below which no coding is attempted, the raw and RLE fallbacks,
 * and the rollback of the stream's state when a block is not stored coded.  The arguments are the mixed call's, except that
 * dSingleStream is an output (one form flag per block, written for every block) and minLiterals, minGainLog follow tableLog.
 * The rule, per chain, block after block, with the state (T, F, H) read from the per-chain entries at the start, n = dSrcSizes[b]
 * and minGain(n) = (n >> minGainLog) + 2:
 *   single[b] = n < 256 || (F == 2 && n < 1024)                              -> dSingleStream[b]
 *   n > 128 KB:                           value srcSize_wrong, kind 4, state unchanged   (the decoders' limit, zstd's block limit)
 *   else n < (F == 2 ? 6 : minLiterals):  value 0, kind 0 (raw), state unchanged          (not attempted)
 *   else: on copies T', F' of T, F
 *     v = HUF_compress{1X if single[b] else 4X}_repeat(dst, HUF_compressBound(n), src, n, maxSymbolValue, tableLog, wksp,
 *                                                     sizeof wksp, T', &F', dPreferRepeat[b], 0);  the value is v, and
 *     isError(v) || v == 0 || v >= n - minGain(n)  (size_t: when n < minGain(n) the difference wraps and rejects nothing):
 *                                             kind 0 (raw), state unchanged;
 *     else v == 1:                            kind 1 (RLE) if n >= 8 or all n bytes are equal, else kind 0 (raw: a 1X block of
 *                                             at most 7 symbols coded with the old table can fit in one byte); state unchanged;
 *     else F' != 0:                           kind 3 (coded with the stream's table T, no header), state unchanged;
 *     else:                                   kind 2 (its own tree header), state := (T', 1, this block's stored bytes).
 * HUF_compress_internal saves a new table and sets the flag to none before its last compressibility test, so without the rollback a
 * block that ends up raw or RLE would still have replaced the stream's table; zstd restores the previous table and flag in that
 * case, as this rule does.  zstd 1.5 sets (minLiterals, minGainLog) by strategy (ZSTD_minLiteralsToCompress, ZSTD_minGain): (64, 6)
 * below btopt, (16, 7) for btultra, (8, 8) for btultra2; minLiterals may be any value, 0 included, and minGainLog must be 1 .. 31.
 * zstd derives dPreferRepeat from its strategy and n; here it stays a per-block input.  Byte equality with libzstd is not claimed:
 * later zstd versions also change how the table is built (optimal depth, sampling of incompressible input), and the reference this
 * library follows has no counterpart for that; the bytes of a coded block are those of the reference's HUF_compress{4X,1X}_repeat.
 * Stored length: n for kind 0, 1 for kind 1 (src[0]), v for kinds 2 and 3, 0 for kind 4 -- so at most n, and sum(n) + 32 bytes of
 * slack always fits.  Offsets, the capacity rule (a block that does not fit outCapacity gets dstSize_tooSmall and kind 4) and the
 * state write-back (only if dOffsets[nBlocks] <= outCapacity; otherwise every per-chain entry as it came in) are those of the packed
 * chain calls; a table is written only if a kind-2 block committed one, and the chain header is that of the chain's last kind-2
 * block.  Malformed chain geometry gives every value srcSize_wrong and every kind 4, and nothing else is written (dSingleStream
 * included).  The stream is what the mixed packed calls read: FSEB200_HUF_decompress_mixed_repeat_packed decodes (dOut, dOffsets,
 * dKinds, dSingleStream) with the headers the chains entered with.
 * Contract: that of FSEB200_HUF_compress_mixed_repeat_chains_packed; dSingleStream overlaps no other array.
 * Return value: 0 (also for nBlocks == 0, which launches nothing and writes nothing); srcSize_wrong, the device untouched, for
 * nBlocks or nChains above 0xFFFFFFFF, a NULL array or minGainLog outside 1 .. 31 while nBlocks > 0; generic if a launch fails. */
size_t FSEB200_HUF_compress_literals_chains_packed(size_t nChains, const size_t* dChainStarts, size_t nBlocks,
                                                   void* dOut, size_t outCapacity, size_t* dOffsets, size_t* dCSizes, unsigned char* dKinds,
                                                   const void* const* dSrcs, const size_t* dSrcSizes, const int* dPreferRepeat,
                                                   unsigned char* dSingleStream,
                                                   unsigned* const* dCTables, int* dRepeats, const void** dChainHeaders, size_t* dChainHeaderSizes,
                                                   unsigned maxSymbolValue, unsigned tableLog, unsigned minLiterals, unsigned minGainLog,
                                                   void* stream);

/* Tier 1, per-block descriptors (FSE, FSE-U16): the same argument shape for the two FSE codecs -- e.g. the FSE-coded blocks of
 * an .fse frame body, packed back to back behind their block headers.  All six arrays and every buffer they point to are in
 * DEVICE memory; the call is asynchronous on `stream` and the host never reads the arrays (no copy, no synchronize).
 *   compress:   dCSizes[b] = exactly what FSE_compress2(dDsts[b], dDstCapacities[b], dSrcs[b], dSrcSizes[b], maxSymbolValue,
 *               tableLog) (U16: FSE_compressU16) returns: 0, 1, a size or an error code; bytes [0, dCSizes[b]) are the
 *               reference's.  Per-block verdicts come from the kernels: a bad maxSymbolValue / tableLog gives the reference's
 *               error, and a capacity above 0xFFFFFF00 acts as 0xFFFFFF00.
 *   decompress: dResults[b] = exactly what FSE_decompress(dDsts[b], dDstCapacities[b], dCSrcs[b], dCSrcSizes[b]) (U16:
 *               FSE_decompressU16) returns, sizes taken literally: cSize 0 or 1 is corruption_detected (U16: cSize < 2 is
 *               srcSize_wrong), not "stored", and an error code in dCSrcSizes is not passed through.  Bytes [0, result) are the
 *               reference's.
 * Units follow the reference's functions: for U16, dSrcSizes (compress), dDstCapacities and dResults (decompress) count 16-bit
 * symbols; compressed sizes and capacities are always bytes.
 * Limits, per block, as the one-block calls of this library: FSE sources, capacities and compressed sizes above 2^30 bytes
 * give srcSize_wrong, and so do U16 blocks of more than 2^29 symbols.  A U16 block whose symbols sit at an odd address (the
 * compress source, the decompress destination) gives GENERIC and nothing is written for it; compressed bytes may sit anywhere.
 * Contract: no destination may overlap another destination, any source or the arrays (sources may overlap each other), and
 * the output array (dCSizes / dResults) may not overlap the other arrays: the kernels read the sizes again after writing it.  Each
 * compressed input must be readable up to the end of the 32-byte-aligned sector that holds its last byte (blocks packed back
 * to back meet this when the buffer has 32 bytes of slack).  Bytes of [dst, dst + capacity) beyond the returned size are
 * unspecified; nothing outside the destinations is written.
 * Return value: 0 (also for nBlocks == 0, which launches nothing); srcSize_wrong if nBlocks > 0xFFFFFFFF or an array is NULL
 * while nBlocks > 0; generic if a launch fails. */
size_t FSEB200_FSE_compress_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstCapacities, size_t* dCSizes,
                                   const void* const* dSrcs, const size_t* dSrcSizes,
                                   unsigned maxSymbolValue, unsigned tableLog, void* stream);
size_t FSEB200_FSE_decompress_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstCapacities, size_t* dResults,
                                     const void* const* dCSrcs, const size_t* dCSrcSizes, void* stream);
size_t FSEB200_FSEU16_compress_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstCapacities, size_t* dCSizes,
                                      const void* const* dSrcs, const size_t* dSrcSizes,
                                      unsigned maxSymbolValue, unsigned tableLog, void* stream);
size_t FSEB200_FSEU16_decompress_blocks(size_t nBlocks, void* const* dDsts, const size_t* dDstCapacities, size_t* dResults,
                                        const void* const* dCSrcs, const size_t* dCSrcSizes, void* stream);

/* Tier 1, per-block descriptors with packed output (FSE, FSE-U16): the blocks given by dSrcs / dSrcSizes are compressed and
 * stored back to back in one buffer, each at an offset the call computes on the device, raw and RLE blocks included; the
 * *_decompress_packed calls regenerate every block from that buffer and its offsets.  Let u be the unit (1 for FSE, 2 for
 * U16) and, per block b, n = dSrcSizes[b] (U16: symbols).
 *   dCSizes[b]  = exactly what FSE_compress2(dst, FSE_compressBound(n), src, n, maxSymbolValue, tableLog) returns (U16:
 *                 FSE_compressU16(dst, FSE_compressBound(2n), ...)): 0, 1, a size or an error code -- except for a block
 *                 that does not fit the workspace or the output (below).
 *   stored length L[b]: dCSizes[b] >= 2: dCSizes[b], the reference's compressed bytes; 1: u, the symbol src[0] as it lies in
 *                 memory (RLE); 0: u * n, a raw copy of the source (0 bytes for an empty block); an error code: 0, nothing.
 *                 L[b] <= u * n always (FSE answers 0 once the output reaches n - 1 bytes, U16 at 2(n - 1), and U16 returns
 *                 n itself for n <= 1), so an outCapacity of u * sum(n) always holds every block; add 32 bytes of slack for
 *                 the decoders' sector reads.
 *   dOffsets    has nBlocks + 1 entries: dOffsets[b] = L[0] + ... + L[b-1], dOffsets[nBlocks] = the total.  It is written in
 *                 full even when blocks do not fit, so a too-small call still tells the size it needs.
 *   capacity    block b is stored at dOut + dOffsets[b] only if dOffsets[b] + L[b] <= outCapacity; otherwise dCSizes[b] =
 *                 dstSize_tooSmall and nothing is written for it (a block whose value is an error code keeps it).  Nothing
 *                 outside [dOut, dOut + min(total, outCapacity)) is ever written.
 *   workspace   an FSE block's size is known only once it is coded, so each block is first coded into a staging slot of
 *                 FSE_compressBound(u * n) bytes in dWork; the slots are laid out back to back in block order.  A block the
 *                 limits below settle takes no slot.  Block b is coded only if its slot ends at or before workSize;
 *                 otherwise dCSizes[b] = workSpace_tooSmall and nothing is stored for it.  FSEB200_FSE_packed_workspace gives
 *                 a size that never runs short; dWork beyond workSize is never touched.
 * Limits, as the descriptor calls above: an FSE source above 2^30 bytes and a U16 source above 2^29 symbols give
 * srcSize_wrong, a U16 source at an odd address GENERIC.
 * Decompress, per block b, with L = dOffsets[b+1] - dOffsets[b] and n = dDstSizes[b] (the regenerated size, U16: symbols;
 * not a capacity):
 *   1. the descriptor decoder's limit and alignment verdicts come first: L or n above the limits gives srcSize_wrong, a U16
 *      destination at an odd address GENERIC, and nothing is written;
 *   2. L == u * n: a raw copy; the result is n (n == 0 included);
 *   3. otherwise L == u: RLE, n copies of the unit at dIn + dOffsets[b]; the result is n;
 *   4. otherwise exactly what FSEB200_FSE{,U16}_decompress_blocks returns for source dIn + dOffsets[b], cSize L and
 *      capacity n -- for L == 0 (a block whose value was an error) corruption_detected, U16 srcSize_wrong.
 *   Rules 2 and 3 never capture a compressed block: an FSE one has 2 <= L < n - 1, and a U16 one is never 2 or 2n bytes long.
 * All arrays and buffers are in DEVICE memory; the calls are asynchronous on `stream` and the host never reads the arrays.
 * Contract: compress: dOut, dOffsets, dCSizes and dWork overlap no source and no other array; sources may overlap each other.
 * Decompress: dIn must be readable up to the end of the 32-byte sector that holds each block's last byte; no destination may
 * overlap another destination, dIn or the arrays.
 * Return value: 0 (also for nBlocks == 0, which launches nothing and writes nothing); srcSize_wrong if nBlocks > 0xFFFFFFFF
 * or a pointer is NULL while nBlocks > 0; generic if a launch fails. */
size_t FSEB200_FSE_compress_packed(size_t nBlocks, void* dOut, size_t outCapacity, size_t* dOffsets, size_t* dCSizes,
                                   const void* const* dSrcs, const size_t* dSrcSizes, unsigned maxSymbolValue, unsigned tableLog,
                                   void* dWork, size_t workSize, void* stream);
size_t FSEB200_FSEU16_compress_packed(size_t nBlocks, void* dOut, size_t outCapacity, size_t* dOffsets, size_t* dCSizes,
                                      const void* const* dSrcs, const size_t* dSrcSizes, unsigned maxSymbolValue, unsigned tableLog,
                                      void* dWork, size_t workSize, void* stream);
/* Host-side, no device work: srcBytes + (srcBytes >> 7) + 524 * nBlocks, at least the sum of FSE_compressBound over any batch
 * of nBlocks blocks of srcBytes source bytes in all (U16: 2 * sum(n)). */
size_t FSEB200_FSE_packed_workspace(size_t nBlocks, size_t srcBytes);
size_t FSEB200_FSE_decompress_packed(size_t nBlocks, void* const* dDsts, const size_t* dDstSizes, size_t* dResults,
                                     const void* dIn, const size_t* dOffsets, void* stream);
size_t FSEB200_FSEU16_decompress_packed(size_t nBlocks, void* const* dDsts, const size_t* dDstSizes, size_t* dResults,
                                        const void* dIn, const size_t* dOffsets, void* stream);

/* Table reuse across blocks (lib/huf.h:191 per block; the shape programs/bench.c:610-633 and HUF_compress4X_repeat,
 * lib/huf_compress.c:664-712, reduce to when the previous table is kept): every block of the batch is coded with ONE
 * caller-supplied table -- dCTable = 256 HUF_CElt cells in DEVICE memory, the layout HUF_buildCTable produces.
 * dCSizes[b] = what HUF_compress4X_usingCTable returns for block b (6 + the four streams, no tree header; 0 if it cannot). */
size_t FSEB200_HUF_compress4X_usingCTable_batch(void* dCBuf, size_t slot, size_t* dCSizes, const void* dSrc, size_t srcTotal,
                                                size_t blockSize, const unsigned* dCTable, void* stream);

/* Tier 1b -- the same batches on HOST buffers (pinned or pageable): chunks are copied in, processed and
 * copied out on alternating CUDA streams so that PCIe transfers overlap the kernels.
 * codec: 0 = FSE, 1 = HUF, 2 = FSE-U16.  Synchronous.  Raw / RLE blocks (cSize 0 / 1) are regenerated from
 * hOrig on the host exactly as programs/bench.c:393-402 does. */
size_t FSEB200_compress_host(int codec, void* hCBuf, size_t slot, size_t* hCSizes, const void* hSrc, size_t srcTotal,
                             size_t blockSize, unsigned maxSymbolValue, unsigned tableLog);
size_t FSEB200_decompress_host(int codec, void* hDst, size_t dstTotal, size_t blockSize, const void* hCBuf, size_t slot,
                               const size_t* hCSizes, size_t* hResults, const void* hOrig);

/* Tier 1b, packed -- blocks of any size on HOST buffers through the packed device calls above.  The slot form keeps nothing for
 * a raw block and needs hOrig to regenerate raw and RLE blocks; these calls produce and read the packed device stream instead --
 * one buffer plus nBlocks + 1 offsets, raw and RLE blocks stored in place -- which decodes without the original.
 * codec: 0 = FSE, 1 = Huff0 4X, 2 = FSE-U16, 3 = Huff0 1X.  Synchronous.  All pointers are host pointers, pinned or pageable,
 * with no alignment required.  Let u = 1 (U16: 2) and n_b = hSrcSizes[b] / hDstSizes[b] (U16: symbols).  Blocks lie back to back:
 * block b of the source starts at hSrc + u * (n_0 + ... + n_{b-1}), and decompress writes block b at the same place in hDst.
 *   compress:   hCSizes, hOffsets (nBlocks + 1 entries) and hOut[0, min(total, outCapacity)) are byte for byte what the matching
 *               device packed call (FSEB200_FSE_compress_packed, FSEB200_HUF_compress_packed, FSEB200_FSEU16_compress_packed,
 *               FSEB200_HUF_compress1X_packed) gives for the same blocks at the same outCapacity, with the blocks on the device
 *               at an even address and, for FSE, a workspace of FSEB200_FSE_packed_workspace: workSpace_tooSmall never appears.
 *               Nothing outside the stored blocks is written to hOut; outCapacity = u * sum(n) always holds them all.
 *   decompress: hResults equals the device packed decompress's (FSEB200_{FSE,HUF,FSEU16}_decompress_packed,
 *               FSEB200_HUF_decompress1X_packed) for the same stream; for a block whose result is not an error, [0, result)
 *               holds the regenerated symbols, and the bytes of a block whose result is an error are unspecified.  Nothing
 *               outside [hDst, hDst + u * sum(n)) is written.  Exactly [hIn + hOffsets[0], hIn + hOffsets[nBlocks]) is read --
 *               no slack is needed.  Offsets that decrease anywhere give srcSize_wrong.
 * The batch is cut into chunks of blocks by a byte budget (FSEB200_HOST_PACKED_CHUNK_BYTES, default 64 MiB; a block counts its
 * bytes plus 512, and one above the budget is a chunk of its own) that overlap their copies and kernels on alternating streams;
 * only stored bytes cross PCIe.  Calls from several host threads are serialised per device.
 * Return value: 0 (also for nBlocks == 0, which writes nothing); srcSize_wrong for a bad codec, nBlocks > 0xFFFFFFFF or a NULL
 * pointer while nBlocks > 0; generic if a CUDA call fails. */
size_t FSEB200_compress_host_packed(int codec, void* hOut, size_t outCapacity, size_t* hOffsets, size_t* hCSizes,
                                    const void* hSrc, const size_t* hSrcSizes, size_t nBlocks,
                                    unsigned maxSymbolValue, unsigned tableLog);
size_t FSEB200_decompress_host_packed(int codec, void* hDst, const size_t* hDstSizes, size_t* hResults,
                                      const void* hIn, const size_t* hOffsets, size_t nBlocks);

/* Tier 1b, packed chains of table reuse (Huff0) -- FSEB200_HUF_compress{4X,1X}_repeat_chains_packed and
 * FSEB200_HUF_decompress{4X,1X}_repeat_packed on HOST buffers, so that a host program keeps its literal blocks and its streams'
 * state in host memory and gets the stream it writes out (bytes, nBlocks + 1 offsets, nBlocks kinds) in one call.
 * codec: 1 = Huff0 4X, 3 = Huff0 1X (the host packed numbering).  Synchronous.  All pointers are host pointers, pinned or pageable,
 * with no alignment required: hChainStarts (nChains + 1 entries), the per-block arrays, the per-chain state -- hCTables[c] (256
 * HUF_CElt cells), hRepeats[c], hChainHeaders[c] / hChainHeaderSizes[c] -- and every header.  Blocks lie back to back: block b of
 * the source starts at hSrc + n_0 + ... + n_{b-1}, and decompress writes block b at the same place in hDst.
 *   compress:   hCSizes, hKinds, hOffsets and hOut[0, min(total, outCapacity)) are byte for byte what the matching device call
 *               gives for the same chains, the same entry state and the same outCapacity, and so is every table (all 256 cells),
 *               flag and chain header on return; a header the device call would point at dOut + dOffsets[j] is hOut +
 *               hOffsets[j] here.  Its rules carry over unchanged: the capacity rule, the state left as it came in when the total
 *               does not fit, and for malformed chain geometry only srcSize_wrong values and kind 4, with no offset written.
 *               Nothing outside the stored blocks is written to hOut; outCapacity = sum(n) always holds them all.
 *   decompress: hResults equals the device call's for the same stream and entry headers; [0, result) of each block holds its
 *               bytes.  Exactly [hIn + hOffsets[0], hIn + hOffsets[nBlocks]) of the stream is read, and of an entry header (one
 *               that a kind-3 block of its chain needs) at most its first 128 bytes -- all a tree header can take.  Offsets that
 *               decrease anywhere give srcSize_wrong; malformed chain geometry makes every result srcSize_wrong.
 * The batch is cut into chunks by the packed host calls' byte budget (FSEB200_HOST_PACKED_CHUNK_BYTES), chain boundaries ignored,
 * and each chunk runs the device call on its own part of the chains.  At most one chain crosses each chunk boundary: compress
 * carries its state on the device from one chunk's call to the next, which waits for it while its copies still overlap, and
 * decompress gives a chunk the crossing chain's last tree header from the stream before it.  The calls share the packed host
 * calls' streams and are serialised per device with them and with the frame calls.
 * Return value: 0 (also for nBlocks == 0, which writes nothing); srcSize_wrong, before any device work, for a bad codec, nBlocks or
 * nChains above 0xFFFFFFFF, or a NULL pointer while nBlocks > 0; generic if a CUDA call fails. */
size_t FSEB200_compress_host_repeat_chains_packed(int codec, size_t nChains, const size_t* hChainStarts, size_t nBlocks,
                                                  void* hOut, size_t outCapacity, size_t* hOffsets, size_t* hCSizes, unsigned char* hKinds,
                                                  const void* hSrc, const size_t* hSrcSizes, const int* hPreferRepeat,
                                                  unsigned* const* hCTables, int* hRepeats, const void** hChainHeaders, size_t* hChainHeaderSizes,
                                                  unsigned maxSymbolValue, unsigned tableLog);
size_t FSEB200_decompress_host_repeat_packed(int codec, size_t nChains, const size_t* hChainStarts, size_t nBlocks,
                                             void* hDst, const size_t* hDstSizes, size_t* hResults,
                                             const void* hIn, const size_t* hOffsets, const unsigned char* hKinds,
                                             const void* const* hChainHeaders, const size_t* hChainHeaderSizes);
/* The same pair for chains whose blocks each choose their form (FSEB200_HUF_compress_mixed_repeat_chains_packed /
 * FSEB200_HUF_decompress_mixed_repeat_packed): hSingleStream[b] (0 4X, else 1X, per block) in place of the codec, and every rule
 * above unchanged -- chunking, the crossing chain's state, the entry headers (a tree header does not depend on the form of the
 * block that wrote it) and the capacity rule.  A NULL hSingleStream while nBlocks > 0 gives srcSize_wrong before any device work. */
size_t FSEB200_compress_host_mixed_repeat_chains_packed(size_t nChains, const size_t* hChainStarts, size_t nBlocks,
                                                        void* hOut, size_t outCapacity, size_t* hOffsets, size_t* hCSizes, unsigned char* hKinds,
                                                        const void* hSrc, const size_t* hSrcSizes, const int* hPreferRepeat,
                                                        const unsigned char* hSingleStream,
                                                        unsigned* const* hCTables, int* hRepeats, const void** hChainHeaders, size_t* hChainHeaderSizes,
                                                        unsigned maxSymbolValue, unsigned tableLog);
size_t FSEB200_decompress_host_mixed_repeat_packed(size_t nChains, const size_t* hChainStarts, size_t nBlocks,
                                                   void* hDst, const size_t* hDstSizes, size_t* hResults,
                                                   const void* hIn, const size_t* hOffsets, const unsigned char* hKinds,
                                                   const unsigned char* hSingleStream,
                                                   const void* const* hChainHeaders, const size_t* hChainHeaderSizes);
/* FSEB200_HUF_compress_literals_chains_packed on host buffers, through the same pipeline: hSingleStream is an output (written for
 * every block, as the device call writes it) and every other rule is the mixed compress's above.  The rolled-back state of the
 * chain that crosses a chunk boundary stays on the device between the chunks' calls, so the output, the forms and the state are
 * byte for byte what one device call over the whole batch gives.  The stream decodes with FSEB200_decompress_host_mixed_repeat_packed.
 * Argument verdicts (NULL pointers, sizes, minGainLog outside 1 .. 31) come before any device work. */
size_t FSEB200_compress_host_literals_chains_packed(size_t nChains, const size_t* hChainStarts, size_t nBlocks,
                                                    void* hOut, size_t outCapacity, size_t* hOffsets, size_t* hCSizes, unsigned char* hKinds,
                                                    const void* hSrc, const size_t* hSrcSizes, const int* hPreferRepeat,
                                                    unsigned char* hSingleStream,
                                                    unsigned* const* hCTables, int* hRepeats, const void** hChainHeaders, size_t* hChainHeaderSizes,
                                                    unsigned maxSymbolValue, unsigned tableLog, unsigned minLiterals, unsigned minGainLog);

/* Tier 1b, frames -- the self-describing .fse format of the reference's file tool (programs/fileio.c:266-626) on HOST buffers:
 *   frame   = LE32 magic (0x183E2309 FSE, 0x183E3309 Huff0), 1 byte block-size id (block = 1 KB << id, id <= 6),
 *             { block header, payload }*, 3-byte trailer
 *   header  = 1 byte { type:2 (0 compressed, 1 raw, 2 RLE, 3 trailer), full:1, 0:5 }, then the regenerated size rSize (2 bytes,
 *             big endian) unless the block is full (rSize = block size), then the compressed size cSize (2 bytes, big endian)
 *             if it is compressed; the payload is cSize compressed bytes, rSize raw bytes, or the 1 byte of an RLE block
 *   trailer = type 3 in the top 2 bits, then the 22 bits (XXH32(data, seed 0) >> 5), big endian.
 * Synchronous; host pointers, pinned or pageable, at any alignment.  They run through the packed host pipeline above (its chunks
 * and FSEB200_HOST_PACKED_CHUNK_BYTES budget) and are serialised per device with the packed host calls.
 *   compress:   codec 0 = FSE, 1 = Huff0.  Returns the frame size; the frame is byte for byte what the reference's writer,
 *               FIO_compressFilename, writes at that block-size id (its `fse -e` / `fse -h` command line writes id 5; its -B
 *               option sets the benchmark's block size): ceil(srcSize / block) blocks and no empty one, each
 *               coded as FSE_compress / HUF_compress code it, i.e. at (maxSymbolValue 255, tableLog 11); a value of 0 makes a raw
 *               block, 1 an RLE block.  An empty input gives the 8-byte frame of header and trailer.  The trailer's checksum is
 *               computed on the device for a short input, on a host thread while the chunks run on the device for a longer one
 *               (the batches' threshold below).  frameCapacity >= FSEB200_frame_compressBound
 *               always suffices; a frame that does not fit gives dstSize_tooSmall, and nothing past frameCapacity is written.
 *               srcSize_wrong for a bad codec, blockSizeId > 6, or a NULL pointer with srcSize > 0 (hSrc) or frameCapacity > 0
 *               (hFrame); the error value of a block, should one occur, stops the call as it stops the reference's tool.
 *   compressBound: the size of the frame with every block raw, which no frame of srcSize bytes exceeds; srcSize_wrong for
 *               blockSizeId > 6.  Host-side only.
 *   decompress: returns what `fse -d` writes, in bytes, and hDst holds exactly those bytes.  A block is dispatched by the type in
 *               its header: a compressed block goes to FSE_decompress / HUF_decompress (as FSEB200_FSE_decompress_blocks /
 *               FSEB200_HUF_decompress_blocks) with capacity rSize and contributes what they return -- FSE may return less than
 *               rSize --, a raw block contributes its payload, an RLE block rSize copies of its byte.  Bytes after the trailer
 *               are never read.  A failure returns the verdict at the first point, in frame order, where the reference's tool
 *               stops; hDst's contents are then unspecified:
 *                 too few bytes for a header, a size field, a payload plus the next header byte, or the trailer: srcSize_wrong;
 *                 an unknown magic number (zlibh frames included) or a block-size id above 6: GENERIC;
 *                 a compressed block the decoder rejects: its error code;
 *                 a checksum mismatch: corruption_detected;
 *                 a block that would overrun the reference's buffers -- rSize above the block size for a compressed or RLE
 *                 block, a payload above block size + 4 bytes: corruption_detected;
 *                 output beyond dstCapacity: dstSize_tooSmall, with nothing written past dstCapacity.
 *               srcSize_wrong also for a NULL hFrame with frameSize > 0 or a NULL hDst with dstCapacity > 0.
 *   decompress_bound: the sum of the headers' rSize -- an upper bound on decompress's result, equal to it unless an FSE block
 *               decodes short -- or the verdict of the header walk (the structural verdicts above).  Host-side only.
 *   batches:    many frames in one call, each exactly what the one-frame call gives for it, through one chunk pipeline: a
 *               chunk holds many small frames (a frame that fits the chunk budget is never split), and the checksums of frames
 *               of up to DEVICE_HASH_MAX bytes (csrc/host_pipeline.cu) are computed on the device in one kernel per chunk --
 *               longer frames are hashed on host threads, one per frame up to the core count.  Host pointers, pinned or pageable, at any alignment; synchronous; serialised
 *               per device with the packed host calls.  Return value: 0 (also for nFrames == 0, which writes nothing);
 *               srcSize_wrong for a bad codec, blockSizeId > 6, nFrames > 0xFFFFFFFF, or a NULL pointer while nFrames > 0 (hSrc
 *               may be NULL when every size is 0); generic if a CUDA call fails.
 *   compress_host_batch: frame f's source is hSrcSizes[f] bytes at hSrc + hSrcSizes[0] + ... + hSrcSizes[f - 1].
 *               hResults[f] is what FSEB200_frame_compress_host(codec, blockSizeId, buf, FSEB200_frame_compressBound(n_f,
 *               blockSizeId), src_f, n_f) returns -- the frame size or that call's error -- except that a frame is stored, at
 *               hOut + hOffsets[f], only if it ends at or before outCapacity; otherwise its result is dstSize_tooSmall.  hOffsets
 *               (nFrames + 1 entries) is the prefix sum of the frame sizes, an error frame counting 0, written in full even when
 *               frames do not fit, so hOffsets[nFrames] is the capacity the batch needs.  Nothing outside the stored frames is
 *               written; the sum of FSEB200_frame_compressBound over the frames always suffices.  (One exception: a frame above
 *               the chunk budget that ends in an error value -- which the coders do not return here, coding every block with
 *               room for it -- may leave its first pieces written where it would have been stored.)
 *   decompress_host_batch: frame f is hIn[hOffsets[f], hOffsets[f + 1]); its output region starts at hDst plus the sum of the
 *               earlier capacities and holds hDstCapacities[f] bytes.  hResults[f] is what FSEB200_frame_decompress_host(region,
 *               capacity, frame, size) returns for it: every verdict above, frame by frame.  A failing frame does not stop the
 *               others, and the bytes of its region are then unspecified.  Nothing outside the regions is written, and only the
 *               frames' bytes are read.  Offsets that decrease give srcSize_wrong for the whole call.
 * FSEB200_XXH32 is the library's XXH32 (the public xxHash specification), the hash behind the trailer. */
size_t   FSEB200_frame_compressBound(size_t srcSize, unsigned blockSizeId);
size_t   FSEB200_frame_compress_host(int codec, unsigned blockSizeId, void* hFrame, size_t frameCapacity,
                                     const void* hSrc, size_t srcSize);
size_t   FSEB200_frame_decompress_bound(const void* hFrame, size_t frameSize);
size_t   FSEB200_frame_decompress_host(void* hDst, size_t dstCapacity, const void* hFrame, size_t frameSize);
size_t   FSEB200_frame_compress_host_batch(int codec, unsigned blockSizeId, size_t nFrames,
                                           void* hOut, size_t outCapacity, size_t* hOffsets, size_t* hResults,
                                           const void* hSrc, const size_t* hSrcSizes);
size_t   FSEB200_frame_decompress_host_batch(size_t nFrames, void* hDst, const size_t* hDstCapacities, size_t* hResults,
                                             const void* hIn, const size_t* hOffsets);
unsigned FSEB200_XXH32(const void* src, size_t srcSize, unsigned seed);

/* Tier 1, frames on DEVICE memory: the frame batches above for data already on the GPU.  Geometry on the host, bytes on the
 * device: arguments starting with h are host arrays, read only during the call; arguments starting with d are device memory, at
 * any byte alignment.  Per frame, each call gives exactly what the matching host call gives for the same frames -- every result
 * value, offset, verdict and stored byte, and the capacity rule -- so only the differences are stated here.
 *   compress_device: as FSEB200_frame_compress_host_batch.  Frame f's source is hSrcSizes[f] bytes at dSrc + hSrcSizes[0] + ...
 *               + hSrcSizes[f - 1]; dOffsets (nFrames + 1 entries) and dResults are written on the device.  A frame is stored,
 *               at dOut + dOffsets[f], only if it ends at or before outCapacity; otherwise its result is dstSize_tooSmall.
 *               Nothing outside the stored frames is written (the host call's exception for frames that span chunks does not
 *               apply: there are no chunks).  An empty source gives the 8-byte frame; the blocks are coded at (255, 11).
 *               Fully asynchronous on `stream`: the host never reads device memory and never waits for the device.  The block
 *               layout is uploaded from a pinned host image of the library's.  The checksums run on a second stream that the
 *               library keeps for `stream`, forked from it and joined back into it by events on the device, so everything the
 *               call does is ordered by `stream` and calls on different streams do not wait for each other.  (The packed
 *               coders keep per-stream scratch whose growth synchronises that stream and frees device memory, as the device
 *               packed calls do: the first calls on a stream, or a larger batch than before, may wait.)
 *   decompress_device: as FSEB200_frame_decompress_host_batch.  Frame f is dIn[hOffsets[f], hOffsets[f + 1]); its region starts
 *               at dDst plus the earlier capacities and holds hDstCapacities[f] bytes.  A failing frame leaves its region
 *               unspecified and does not stop the others; nothing outside the regions is written.  The call SYNCHRONISES
 *               `stream` once: after the header walk on the device, to learn how many blocks to launch.  Everything after it
 *               is enqueued, and dResults is valid when the stream reaches it.  (As in compress, the decoders' per-stream
 *               scratch synchronises the stream again, and frees device memory, when it grows.)  dIn must be readable up to the end
 *               of the 32-byte sector that holds the last frame's last byte (every cudaMalloc and torch allocation is).
 *   decompress_bound_device: synchronous; the header walk alone, writing FSEB200_frame_decompress_bound's value (or verdict)
 *               for each frame to hBounds.
 * Checksums: every frame is hashed on the device by one kernel, four lanes per frame, whatever its length.  One frame's hash
 * is a serial chain, measured at about 0.5 GB/s on an H100 80GB HBM3 at 700 W (DESIGN.md 5b): a single large frame is bound by
 * it, and runs several times slower than through the host batch calls, which hash such frames on host threads.
 * Scratch, all stream-ordered (cudaMallocAsync on `stream`), no chunking: compress, the source's size plus 32 bytes for the
 * packed blocks, FSEB200_FSE_packed_workspace(blocks, source size) for FSE, about 6 words per block and 6 per frame;
 * decompress, 5 words per compressed block, 3 per raw or RLE block and 2 per block, 19 words per frame, and the nominal output
 * of every frame with compressed blocks whose nominal output passes its capacity (it decodes there and its true bytes are
 * then copied in).  That nominal output is what the frame's block headers claim, up to 64 KiB per 3-byte header, so a
 * malformed or hostile frame with a small capacity can ask for far more scratch than its size; when the allocation fails
 * the whole call returns generic, where the host batch call would give that frame its verdict.  A caller decoding untrusted
 * frames can run FSEB200_frame_decompress_bound_device first and reject frames whose bound passes its capacity by too much.  Calls on different streams or host threads may run at once; they take no lock the host calls hold.
 * Return value: 0 (also for nFrames == 0, which launches nothing); srcSize_wrong for a bad codec, blockSizeId > 6, nFrames >
 * 0xFFFFFFFF, more than 0xFFFFFFFF blocks, a NULL pointer while nFrames > 0 (dSrc may be NULL when every size is 0), or
 * offsets that decrease (decompress, bound); these checks touch no device.  generic if a CUDA call fails. */
size_t FSEB200_frame_compress_device(int codec, unsigned blockSizeId, size_t nFrames,
                                     void* dOut, size_t outCapacity, size_t* dOffsets, size_t* dResults,
                                     const void* dSrc, const size_t* hSrcSizes, void* stream);
size_t FSEB200_frame_decompress_bound_device(size_t nFrames, size_t* hBounds,
                                             const void* dIn, const size_t* hOffsets, void* stream);
size_t FSEB200_frame_decompress_device(size_t nFrames, void* dDst, const size_t* hDstCapacities, size_t* dResults,
                                       const void* dIn, const size_t* hOffsets, void* stream);

/* Measurement inputs generated directly in device memory: byte i of the output equals byte
 * (streamOffset + i) of the reference generator's stream (programs/probaGenerator.c:95-126 with
 * probability p, seed 1; programs/fuzzerU16.c:107-134 with the given start / p / seed). */
size_t FSEB200_probagen(void* dDst, size_t nBytes, size_t streamOffset, double p, void* stream);
size_t FSEB200_genU16(void* dDst, size_t nSymbols, size_t streamOffset, unsigned start, double p, unsigned seed, void* stream);
int    FSEB200_device_count(void);

/* ------------------------------------------------------------------------------------------------
 * Tier 2 -- the reference API, host pointers.
 * ------------------------------------------------------------------------------------------------ */
/* lib/fse.h:43-105 */
unsigned    FSE_versionNumber(void);
size_t      FSE_compress(void* dst, size_t dstCapacity, const void* src, size_t srcSize);
size_t      FSE_compress2(void* dst, size_t dstCapacity, const void* src, size_t srcSize,
                          unsigned maxSymbolValue, unsigned tableLog);
size_t      FSE_decompress(void* dst, size_t dstCapacity, const void* cSrc, size_t cSrcSize);
size_t      FSE_compressBound(size_t size);
unsigned    FSE_isError(size_t code);
const char* FSE_getErrorName(size_t code);
/* lib/fse.h:135-247 (detailed API) */
unsigned    FSE_optimalTableLog(unsigned maxTableLog, size_t srcSize, unsigned maxSymbolValue);
unsigned    FSE_optimalTableLog_internal(unsigned maxTableLog, size_t srcSize, unsigned maxSymbolValue, unsigned minus);
size_t      FSE_normalizeCount(short* normalizedCounter, unsigned tableLog, const unsigned* count,
                               size_t srcSize, unsigned maxSymbolValue);
size_t      FSE_NCountWriteBound(unsigned maxSymbolValue, unsigned tableLog);
size_t      FSE_writeNCount(void* buffer, size_t bufferSize, const short* normalizedCounter,
                            unsigned maxSymbolValue, unsigned tableLog);
size_t      FSE_readNCount(short* normalizedCounter, unsigned* maxSymbolValuePtr, unsigned* tableLogPtr,
                           const void* rBuffer, size_t rBuffSize);
unsigned*   FSE_createCTable(unsigned maxSymbolValue, unsigned tableLog);
void        FSE_freeCTable(unsigned* ct);
size_t      FSE_buildCTable(unsigned* ct, const short* normalizedCounter, unsigned maxSymbolValue, unsigned tableLog);
unsigned*   FSE_createDTable(unsigned tableLog);
void        FSE_freeDTable(unsigned* dt);
size_t      FSE_buildDTable(unsigned* dt, const short* normalizedCounter, unsigned maxSymbolValue, unsigned tableLog);
/* lib/hist.h:30-75 */
size_t      HIST_count(unsigned* count, unsigned* maxSymbolValuePtr, const void* src, size_t srcSize);
unsigned    HIST_isError(size_t code);
size_t      HIST_count_wksp(unsigned* count, unsigned* maxSymbolValuePtr, const void* src, size_t srcSize,
                            void* workSpace, size_t workSpaceSize);
size_t      HIST_countFast(unsigned* count, unsigned* maxSymbolValuePtr, const void* src, size_t srcSize);
size_t      HIST_countFast_wksp(unsigned* count, unsigned* maxSymbolValuePtr, const void* src, size_t srcSize,
                                void* workSpace, size_t workSpaceSize);
unsigned    HIST_count_simple(unsigned* count, unsigned* maxSymbolValuePtr, const void* src, size_t srcSize);
/* lib/huf.h:54-98 */
size_t      HUF_compress(void* dst, size_t dstCapacity, const void* src, size_t srcSize);
size_t      HUF_compress2(void* dst, size_t dstCapacity, const void* src, size_t srcSize,
                          unsigned maxSymbolValue, unsigned tableLog);
size_t      HUF_compress4X_wksp(void* dst, size_t dstCapacity, const void* src, size_t srcSize,
                                unsigned maxSymbolValue, unsigned tableLog, void* workSpace, size_t wkspSize);
size_t      HUF_decompress(void* dst, size_t originalSize, const void* cSrc, size_t cSrcSize);
size_t      HUF_compressBound(size_t size);
unsigned    HUF_isError(size_t code);
const char* HUF_getErrorName(size_t code);
/* lib/huf.h:155-280 (static-linking tier used by fullbench / the north star).
 * HUF_CElt is {U16 val; BYTE nbBits} in a 4-byte cell (lib/huf_compress.c:106-109); HUF_DTable is U32[]
 * (lib/huf.h:144-149). */
unsigned    HUF_optimalTableLog(unsigned maxTableLog, size_t srcSize, unsigned maxSymbolValue);
size_t      HUF_buildCTable(unsigned* CTable, const unsigned* count, unsigned maxSymbolValue, unsigned maxNbBits);
size_t      HUF_writeCTable(void* dst, size_t maxDstSize, const unsigned* CTable, unsigned maxSymbolValue, unsigned huffLog);
size_t      HUF_readStats(unsigned char* huffWeight, size_t hwSize, unsigned* rankStats, unsigned* nbSymbolsPtr,
                          unsigned* tableLogPtr, const void* src, size_t srcSize);
size_t      HUF_readDTableX1(unsigned* DTable, const void* src, size_t srcSize);
size_t      HUF_readDTableX2(unsigned* DTable, const void* src, size_t srcSize);   /* double-symbol table image (huf_decompress.c:551-649) */
unsigned    HUF_selectDecoder(size_t dstSize, size_t cSrcSize);
size_t      HUF_decompress4X1(void* dst, size_t dstSize, const void* cSrc, size_t cSrcSize);
size_t      HUF_decompress4X2(void* dst, size_t dstSize, const void* cSrc, size_t cSrcSize);
/* Payload coding with a caller-built table image (lib/fse.h:222,247 ; lib/huf.h:191,203,277).  The images are the
 * reference's own ABI layouts (FSE_CTable fse.h:295,483-486 ; FSE_DTable fse.h:296,565-575 ; HUF_CElt huf_compress.c:106-109 ;
 * HUF_DTable single-symbol huf_decompress.c:101,116), e.g. as produced by FSE_buildCTable / FSE_buildDTable /
 * HUF_buildCTable / HUF_readDTableX1 above or by the CPU library.  Single synchronous calls on host buffers, <= 16 MiB. */
/* CTable inspection helpers (lib/huf.h:196-199,221) */
unsigned    HUF_getNbBits(const void* symbolTable, unsigned symbolValue);
size_t      HUF_estimateCompressedSize(const unsigned* CTable, const unsigned* count, unsigned maxSymbolValue);
int         HUF_validateCTable(const unsigned* CTable, const unsigned* count, unsigned maxSymbolValue);
/* constant-pattern tables for stored / single-symbol blocks (lib/fse.h:330-345) */
size_t      FSE_buildCTable_raw(unsigned* ct, unsigned nbBits);
size_t      FSE_buildCTable_rle(unsigned* ct, unsigned char symbolValue);
size_t      FSE_buildDTable_raw(unsigned* dt, unsigned nbBits);
size_t      FSE_buildDTable_rle(unsigned* dt, unsigned char symbolValue);
size_t      FSE_compress_usingCTable(void* dst, size_t dstCapacity, const void* src, size_t srcSize, const unsigned* ct);
size_t      FSE_decompress_usingDTable(void* dst, size_t dstCapacity, const void* cSrc, size_t cSrcSize, const unsigned* dt);
size_t      HUF_compress4X_usingCTable(void* dst, size_t dstSize, const void* src, size_t srcSize, const unsigned* CTable);
size_t      HUF_decompress4X_usingDTable(void* dst, size_t maxDstSize, const void* cSrc, size_t cSrcSize, const unsigned* DTable);
size_t      HUF_decompress4X1_usingDTable(void* dst, size_t maxDstSize, const void* cSrc, size_t cSrcSize, const unsigned* DTable);
size_t      HUF_decompress4X2_usingDTable(void* dst, size_t maxDstSize, const void* cSrc, size_t cSrcSize, const unsigned* DTable);
size_t      HUF_decompress1X2_usingDTable(void* dst, size_t maxDstSize, const void* cSrc, size_t cSrcSize, const unsigned* DTable);
/* single-stream Huff0 (lib/huf.h:288-320) */
size_t      HUF_compress1X(void* dst, size_t dstSize, const void* src, size_t srcSize, unsigned maxSymbolValue, unsigned tableLog);
size_t      HUF_compress1X_usingCTable(void* dst, size_t dstSize, const void* src, size_t srcSize, const unsigned* CTable);
size_t      HUF_decompress1X1(void* dst, size_t dstSize, const void* cSrc, size_t cSrcSize);
size_t      HUF_decompress1X_usingDTable(void* dst, size_t maxDstSize, const void* cSrc, size_t cSrcSize, const unsigned* DTable);
size_t      HUF_decompress1X1_usingDTable(void* dst, size_t maxDstSize, const void* cSrc, size_t cSrcSize, const unsigned* DTable);
/* lib/huf.h:194-208,291-300: table reuse, one block per call.  `repeat` points to a HUF_repeat (an int: none 0, check 1, valid 2).
 * A batch of one through FSEB200_HUF_compress{4X,1X}_repeat_blocks; hufTable holds 256 cells, as the reference saves 256. */
size_t      HUF_compress4X_repeat(void* dst, size_t dstSize, const void* src, size_t srcSize, unsigned maxSymbolValue, unsigned tableLog,
                                  void* workSpace, size_t wkspSize, unsigned* hufTable, int* repeat, int preferRepeat, int bmi2);
size_t      HUF_compress1X_repeat(void* dst, size_t dstSize, const void* src, size_t srcSize, unsigned maxSymbolValue, unsigned tableLog,
                                  void* workSpace, size_t wkspSize, unsigned* hufTable, int* repeat, int preferRepeat, int bmi2);
/* lib/huf.h:231,304,329,333 */
size_t      HUF_readCTable(unsigned* CTable, unsigned* maxSymbolValuePtr, const void* src, size_t srcSize, unsigned* hasZeroWeights);
size_t      HUF_decompress1X2(void* dst, size_t dstSize, const void* cSrc, size_t cSrcSize);
size_t      HUF_decompress1X_usingDTable_bmi2(void* dst, size_t maxDstSize, const void* cSrc, size_t cSrcSize, const unsigned* DTable, int bmi2);
size_t      HUF_decompress4X_usingDTable_bmi2(void* dst, size_t maxDstSize, const void* cSrc, size_t cSrcSize, const unsigned* DTable, int bmi2);
/* lib/fseU16.h:75-79 */
size_t      FSE_compressU16(void* dst, size_t dstCapacity, const unsigned short* src, size_t srcSize,
                            unsigned maxSymbolValue, unsigned tableLog);
size_t      FSE_decompressU16(unsigned short* dst, size_t dstCapacity, const void* cSrc, size_t cSrcSize);
/* lib/fseU16.c:121-145 (not in fseU16.h; programs/fuzzerU16.c:257 declares it `extern`): histogram of 16-bit symbols on the GPU.
 * *maxSymbolValuePtr in: largest symbol `count` has room for; out: largest symbol present.  Returns the largest count. */
size_t      FSE_countU16(unsigned* count, unsigned* maxSymbolValuePtr, const unsigned short* src, size_t srcSize);

#ifdef __cplusplus
}
#endif
#endif /* FSE_B200_H */
