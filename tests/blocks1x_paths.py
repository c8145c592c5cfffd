"""Host-side predicates for the single-stream descriptor calls (FSEB200_HUF_compress1X_blocks / _decompress1X_blocks): which
path each block takes.  They restate the guards of the 1X instantiations one to one:

  decode (csrc/huf_decode.cu, NS = 1)   the block kind is that of the 4X descriptor decoder (HUF_decompress1X_DCtx has the
                                        same size rules and the table is the same); the block's ONE stream covers the whole
                                        output: (-start) & 31 head symbols, whole 32-symbol iterations, a tail -- when at
                                        least one sector is left after the head and the block is not hard; else every symbol
                                        one at a time.  Pass A holds G = 64 blocks per CTA and five CTAs per SM;
  encode (csrc/huf_encode.cu, NS = 1)   the plan kernel's histogram choice (unchanged) and the emit kernel's group width for
                                        the one segment, the whole block.

The GPU tests assert with them that their fixtures reach the paths they claim; tests/test_blocks1x_model.py pins them on the CPU."""
from blocks_paths import decode_kind, stream_kind, summarize            # noqa: F401  (re-exported for the 1X tests)
from paths import ROWS_A, ROWS_B, G

PASS_A_CTAS_PER_SM = 5                   # 1X pass A: 306 rows x 128 B + 2 KB ring + 1.25 KB facts + 2 KB staging = 44.5 KB per CTA


def stream_paths_1x(kind, dst_size, dst_addr):
    """the one stream of a Huffman block: [(head symbols, fast 32-symbol iterations, tail symbols)]"""
    mis = (-dst_addr) % 32
    if kind != "hard" and dst_size >= mis + 32:
        it = (dst_size - mis) >> 5
        return [(mis, it, dst_size - mis - 32 * it)]
    return [(0, 0, dst_size)]


def decode_paths_1x(cblocks, csizes, dst_sizes, dst_addrs, rows=(ROWS_A, ROWS_B)):
    """per block: {'kind', 'streams'} (streams only for the table kinds A, B and hard)"""
    res = []
    for c, cs, n, a in zip(cblocks, csizes, dst_sizes, dst_addrs):
        kind = decode_kind(c, int(cs), int(n), rows)
        res.append({"kind": kind, "streams": stream_paths_1x(kind, int(n), int(a)) if kind in ("A", "B", "hard") else []})
    return res


def pass_a_spread_1x(nblocks, sms):
    """(blocks per CTA, rounds) of the 1X pass A: launch_huf_decode's grid shape with five CTAs per SM"""
    slots = PASS_A_CTAS_PER_SM * sms
    if nblocks * 5 <= slots * G * 4:
        return G, 1
    rounds = (nblocks + slots * G - 1) // (slots * G)
    return max(1, min(G, (nblocks + slots * rounds - 1) // (slots * rounds))), rounds


def emit_group_1x(src_addr, n):
    """the emit kernel's group width for the block's one stream: 'g256' (8-byte aligned end), 'g128' (word aligned) or 'bytes'"""
    end = src_addr + n
    return "g256" if end % 8 == 0 else ("g128" if end % 4 == 0 else "bytes")
