"""Host-side predicates that say which code path of a batch kernel a block (or a stream of it) takes, for a given batch and
buffer placement.  They restate the guards of the kernels one to one:

  Huff0 decode (csrc/huf_decode.cu)   block kind (launch loop), the table split of setup_block and its row budget per pass,
                                      the fast loop's alignment guard (`fastOk`), the pass-A spread (`gEff`);
  Huff0 encode (csrc/huf_encode.cu)   the plan kernel's histogram choice, the emit kernel's group width and its first piece;
  FSE / U16   (csrc/fse_codec.cu)     the encoder's kernel choice, the decoder's check-free loop guard (`al4`, `sameHi`).

The GPU tests use them to assert, before they touch the GPU, that their inputs reach the paths they claim to cover, and
tests/test_paths.py pins those claims on the CPU.  Tree headers are read with the compiled reference's HUF_readStats, or with
the oracle port's restatement of it when the reference library is absent."""
import ctypes as C
from collections import Counter

import numpy as np

from helpers import is_error, load_port, load_ref, ptr, REF_SO
import os

G = 64                                   # block columns per CTA of the Huff0 decoder
ROWS_A, ROWS_B = 306, 808                # default row budgets of its two passes (FSEB200_HUFD_ROWS / _ROWS_B)
MIN_ROWS = 160
RING_BYTES, FACTS_BYTES, STAGE_BYTES = 8 * 256 * 4, 1280, 8 * 32 * 32
HUF_MAX_TLOG = 12


def smem_bytes(rows, staged):
    """hufd::smem_bytes: table rows of 128 B + stream ring + per-block facts (+ output staging in pass A)"""
    return rows * 2 * G + RING_BYTES + FACTS_BYTES + (STAGE_BYTES if staged else 0)


def max_rows(optin_bytes, staged):
    """the most table rows a pass can have under a per-block shared-memory opt-in limit"""
    return (optin_bytes - smem_bytes(0, staged)) // (2 * G)


def row_budgets(req_a=None, req_b=None, optin_bytes=232448):
    """(rowsA, rowsB) as launch_huf_decode clamps the requested values (None = default); 232,448 B is the H100's opt-in limit"""
    a = ROWS_A if req_a is None else req_a
    b = ROWS_B if req_b is None else req_b
    return max(MIN_ROWS, min(a, max_rows(optin_bytes, True))), min(b, max_rows(optin_bytes, False))


# ---- the unified table of setup_block -----------------------------------------------------------------------------------

def rank_end_of(rank_stats, tl):
    """end (exclusive) of weight w's range in tableLog-bit index space, w = 0 .. tl (weight w covers 2^(w-1) cells a symbol)"""
    out, acc = [0] * (tl + 2), 0
    for w in range(1, tl + 1):
        acc += rank_stats[w] << (w - 1)
        out[w] = acc
    return out


def split_candidates(rank_end, tl):
    """the splits setup_block tries, in its order: (M, CUT, rows) for a first level of M bits, 4 <= M < tableLog, M <= 10"""
    for m in range(min(10, tl - 1), 3, -1):
        g = 1 << (tl - m)
        cut = (rank_end[tl - m] + g - 1) & ~(g - 1)       # windows that start a code longer than m bits, rounded up to a group
        yield m, cut, cut + (1 << m) - (cut >> (tl - m))


def table_rows(rank_end, tl):
    """(rows, M, CUT) of the table setup_block builds: the main-only table unless a split is strictly smaller"""
    best = (1 << tl, tl, 0)
    for m, cut, rows in split_candidates(rank_end, tl):
        if rows < best[0]:
            best = (rows, m, cut)
    return best


# ---- tree headers ---------------------------------------------------------------------------------------------------

def _read_stats_fn():
    if os.path.exists(REF_SO):
        return load_ref().HUF_readStats
    return load_port().orc_huf_read_stats


def read_stats(cblock):
    """HUF_readStats over a compressed block: (header bytes, tableLog, rankStats[0..12]) or None on an error verdict"""
    c = np.ascontiguousarray(cblock, dtype=np.uint8)
    wts = np.zeros(260, np.uint8)
    rs = (C.c_uint32 * 16)()
    nsym, tl = C.c_uint32(0), C.c_uint32(0)
    h = _read_stats_fn()(ptr(wts), 256, rs, C.byref(nsym), C.byref(tl), ptr(c), len(c))
    if is_error(h):
        return None
    return int(h), int(tl.value), list(rs)[:HUF_MAX_TLOG + 1]


def block_rows(cblock):
    """rows of the decoder's table for one Huffman block, or None when its tree header is rejected"""
    st = read_stats(cblock)
    if st is None or st[0] >= len(cblock):
        return None
    h, tl, rs = st
    return table_rows(rank_end_of(rs, tl), tl)[0]


def stream_offsets(cblock):
    """byte offsets of the four streams of a Huffman block from its start (tree header + 6-byte jump table)"""
    st = read_stats(cblock)
    if st is None:                  # a header HUF_readStats rejects (a 1-bit code at tableLog 12): offsets are still hSize + ...
        return None
    h = st[0]
    l1, l2, l3 = (int(cblock[h + 2 * k]) | (int(cblock[h + 2 * k + 1]) << 8) for k in range(3))
    return [h + 6, h + 6 + l1, h + 6 + l1 + l2, h + 6 + l1 + l2 + l3]


def _blocks(total, block):
    return (total + block - 1) // block


def _blen(total, block, b):
    return min(block, total - b * block)


# ---- Huff0 decode ---------------------------------------------------------------------------------------------------

def huf_decode_paths(cbuf, cs, total, block, slot, out_addr, rows=(ROWS_A, ROWS_B), have_orig=True):
    """Per block, the path the batch decoder (HUF_decompress semantics) takes: a dict with
         kind     'raw' | 'rle' | 'error' | 'A' (pass A table) | 'B' (deferred to pass B) | 'hard' (canonical-code search),
         rows     table rows (Huffman blocks),
         streams  per stream (fast 32-symbol iterations, per-symbol count) for Huffman blocks, [] otherwise.
       `out_addr` is the address (or any value congruent to it mod 32) the batch's output starts at."""
    rows_a, rows_b = rows
    two_pass = rows_b > rows_a
    res = []
    for b in range(_blocks(total, block)):
        n = _blen(total, block, b)
        c = int(cs[b])
        ent = {"kind": None, "rows": None, "streams": []}
        if is_error(c):
            ent["kind"] = "error"
        elif c == 0:
            ent["kind"] = "raw" if have_orig else "error"
        elif n == 0 or c > n:
            ent["kind"] = "error"
        elif c == n:
            ent["kind"] = "raw"
        elif c == 1:
            ent["kind"] = "rle"
        else:
            r = block_rows(cbuf[b * slot: b * slot + c])
            if r is None:
                ent["kind"] = "error"
            else:
                ent["rows"] = r
                if r <= rows_a:
                    ent["kind"] = "A"
                elif two_pass and r <= rows_b:
                    ent["kind"] = "B"
                else:
                    ent["kind"] = "hard"
                seg = (n + 3) // 4
                for k in range(4):
                    seg_len = seg if k < 3 else n - 3 * seg
                    fast = ent["kind"] != "hard" and (out_addr + b * block + k * seg) % 32 == 0
                    it = seg_len >> 5 if fast else 0
                    ent["streams"].append((it, seg_len - 32 * it))
        res.append(ent)
    return res


def pass_a_spread(nblocks, sms, per_sm=4):
    """(blocks per CTA, rounds) of pass A (launch_huf_decode's grid shape; four CTAs per SM at the default budget)"""
    slots = per_sm * sms
    if nblocks * 5 <= slots * G * 4:
        return G, 1
    rounds = (nblocks + slots * G - 1) // (slots * G)
    return max(1, min(G, (nblocks + slots * rounds - 1) // (slots * rounds))), rounds


def warps_with_both_stream_kinds(paths, g_eff=G):
    """pass-A warps (one stream index, the even or the odd columns of one CTA) holding a fast-loop stream and a per-symbol one"""
    n = 0
    for c0 in range(0, len(paths), g_eff):
        cols = paths[c0: c0 + g_eff]
        for parity in (0, 1):
            for k in range(4):
                kinds = set()
                for p in cols[parity::2]:
                    if p["kind"] == "A":
                        it, rest = p["streams"][k]
                        kinds.add("fast" if it else "symbol")
                n += kinds == {"fast", "symbol"}
    return n


def summarize(paths):
    """counts of block kinds and of stream kinds ('fast', 'fast+tail', 'symbol')"""
    kinds = Counter(p["kind"] for p in paths)
    streams = Counter()
    for p in paths:
        for it, rest in p["streams"]:
            streams["symbol" if not it else ("fast+tail" if rest else "fast")] += 1
    return kinds, streams


# ---- Huff0 encode ---------------------------------------------------------------------------------------------------

def huf_plan_histogram(src_addr, total, block):
    """per block: 'pipelined' (aligned block of whole 2 KB segment batches) or 'scalar' (warp_hist_range)"""
    out = []
    for b in range(_blocks(total, block)):
        n = _blen(total, block, b)
        seg = (n + 3) // 4
        ok = (src_addr + b * block) % 16 == 0 and seg % 2048 == 0 and n == 4 * seg
        out.append("pipelined" if ok else "scalar")
    return out


def huf_emit_paths(src_addr, cbuf_addr, cbuf, cs, total, block, slot):
    """per compressed Huffman block (cs > 1), per stream: (group kind, first piece partial) where group kind is
    'g256' (8-byte aligned segment end), 'g128' (word aligned) or 'bytes', and the first piece is partial when the stream's
    start is not 16-byte aligned in the destination"""
    out = {}
    for b in range(_blocks(total, block)):
        c = int(cs[b])
        if is_error(c) or c <= 1:
            continue
        n = _blen(total, block, b)
        offs = stream_offsets(cbuf[b * slot: b * slot + c])
        if offs is None:
            continue
        seg = (n + 3) // 4
        s = src_addr + b * block
        per = []
        for k in range(4):
            seg_end = (k + 1) * seg if k < 3 else n
            kind = "g256" if (s + seg_end) % 8 == 0 else ("g128" if (s + seg_end) % 4 == 0 else "bytes")
            per.append((kind, (cbuf_addr + b * slot + offs[k]) % 16 != 0))
        out[b] = per
    return out


# ---- FSE / U16 ------------------------------------------------------------------------------------------------------

def fse_encode_kernel(src_addr, total, block):
    """per block: 'chain' (chain-warp kernel: full blocks, block size a multiple of 64, 16-byte aligned source) or 'warp'"""
    fast = block >= 64 and block % 64 == 0 and src_addr % 16 == 0
    n_full = total // block if fast else 0
    return ["chain" if b < n_full else "warp" for b in range(_blocks(total, block))]


def fse_decode_exact(out_addr, cbuf_addr, total, block, slot, wide=False):
    """per block: (output misaligned for the check-free loop, slot or output straddles a 2^32 address boundary)"""
    res = []
    for b in range(_blocks(total, block)):
        n = _blen(total, block, b)
        o = out_addr + b * block
        c = cbuf_addr + b * slot
        low = c & ~15
        same_hi = ((o + n) >> 32) == (o >> 32) and ((c + slot + 16) >> 32) == (low >> 32)
        res.append((o % (8 if wide else 4) != 0, not same_hi))
    return res


# ---- fixtures -------------------------------------------------------------------------------------------------------

# A dyadic distribution (count = 32768 * 2^-length, tableLog 12) whose code has more than 808 table rows at every split M:
# code length -> number of symbols.  The tightest split (M = 9) needs 813 rows, so its blocks stay hard in pass B.
HARD_LENGTHS = {2: 3, 5: 1, 6: 1, 7: 3, 8: 8, 9: 33, 10: 85, 11: 1, 12: 2}


def hard_block(rng, n=32768):
    """one block of n bytes with the HARD_LENGTHS histogram (32 KB: 12-bit codes need tableLog 12), symbols shuffled"""
    syms = rng.permutation(256)[:sum(HARD_LENGTHS.values())]
    parts, i = [], 0
    for ln, k in sorted(HARD_LENGTHS.items()):
        for _ in range(k):
            parts.append(np.full(n >> ln, syms[i], np.uint8))
            i += 1
    v = np.concatenate(parts)
    assert len(v) == n
    return rng.permutation(v).astype(np.uint8)
