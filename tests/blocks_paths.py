"""Host-side predicates for the per-block descriptor calls (FSEB200_HUF_compress_blocks / _decompress_blocks): which path each
block, and each stream of it, takes.  They restate the guards of the descriptor instantiations one to one:

  decode (csrc/huf_decode.cu)   block kind (HUF_decompress on the literal sizes, then the table budgets of paths.py), and per
                                stream the head decode: a stream whose output segment starts off a 32-byte boundary decodes the
                                (-start) & 31 symbols up to it one at a time, then whole 32-symbol iterations, then a tail --
                                when at least one sector is left after the head and the block is not hard; else every symbol
                                one at a time;
  encode (csrc/huf_encode.cu)   the plan kernel's histogram choice and the emit kernel's group width, per block address.

The GPU tests assert with them that their fixtures reach the paths they claim; tests/test_blocks_model.py pins them on the CPU."""
from collections import Counter

from helpers import is_error
from paths import ROWS_A, ROWS_B, block_rows

HUF_BLOCK_MAX = 128 * 1024


def decode_kind(cblock, csize, dst_size, rows=(ROWS_A, ROWS_B)):
    """'raw' | 'rle' | 'error' | 'A' | 'B' | 'hard' for one block of the descriptor decoder (cblock: its compressed bytes)"""
    rows_a, rows_b = rows
    if dst_size == 0 or dst_size > HUF_BLOCK_MAX or csize > dst_size:
        return "error"
    if csize == dst_size:
        return "raw"
    if csize == 1:
        return "rle"
    r = block_rows(cblock[:csize]) if csize else None
    if r is None:
        return "error"
    if r <= rows_a:
        return "A"
    return "B" if rows_b > rows_a and r <= rows_b else "hard"


def stream_paths(kind, dst_size, dst_addr):
    """per stream of a Huffman block: (head symbols, fast 32-symbol iterations, tail symbols)"""
    seg = (dst_size + 3) // 4
    out = []
    for k in range(4):
        seg_len = seg if k < 3 else dst_size - 3 * seg
        mis = (-(dst_addr + k * seg)) % 32
        if kind != "hard" and seg_len >= mis + 32:
            it = (seg_len - mis) >> 5
            out.append((mis, it, seg_len - mis - 32 * it))
        else:
            out.append((0, 0, seg_len))
    return out


def decode_paths(cblocks, csizes, dst_sizes, dst_addrs, rows=(ROWS_A, ROWS_B)):
    """per block: {'kind', 'streams'} (streams only for the table kinds A, B and hard)"""
    res = []
    for c, cs, n, a in zip(cblocks, csizes, dst_sizes, dst_addrs):
        kind = decode_kind(c, int(cs), int(n), rows)
        res.append({"kind": kind, "streams": stream_paths(kind, int(n), int(a)) if kind in ("A", "B", "hard") else []})
    return res


def stream_kind(head, it, tail):
    """'head+fast' | 'fast' (aligned start) | 'symbol' (no fast iteration)"""
    if not it:
        return "symbol"
    return "head+fast" if head else "fast"


def summarize(paths):
    kinds = Counter(p["kind"] for p in paths)
    streams = Counter(stream_kind(*s) for p in paths for s in p["streams"])
    return kinds, streams


def plan_histogram(src_addr, n):
    """'pipelined' (16-byte aligned source, whole 2 KB segment batches) or 'scalar' -- huf_plan_kernel's choice"""
    seg = (n + 3) // 4
    return "pipelined" if src_addr % 16 == 0 and seg % 2048 == 0 and n == 4 * seg and n else "scalar"


def emit_groups(src_addr, n):
    """per stream of a block the emit kernel codes: 'g256' (8-byte aligned segment end), 'g128' (word aligned) or 'bytes'"""
    seg = (n + 3) // 4
    out = []
    for k in range(4):
        end = src_addr + ((k + 1) * seg if k < 3 else n)
        out.append("g256" if end % 8 == 0 else ("g128" if end % 4 == 0 else "bytes"))
    return out


def expected_decode_verdict(ref_result, csize, dst_size):
    """this library's HUF_decompress value from the reference's: its documented answers for dstSize > 128 KB (srcSize_wrong)
    and for a Huffman block with dstSize < 6 (corruption_detected, DESIGN 2)"""
    if dst_size == 0:
        return ref_result
    if dst_size > HUF_BLOCK_MAX:
        return 2 ** 64 - 3
    if dst_size < 6 and csize not in (1, dst_size) and csize < dst_size and not is_error(ref_result):
        return 2 ** 64 - 4
    return ref_result
