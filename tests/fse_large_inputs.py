"""Inputs of the large-block FSE / FSE-U16 tests: blocks from 1 MiB up to the 2^30-byte limit (FSE_BLOCK_MAX), built with numpy
from fixed seeds, so that tests/test_gpu_fse_large.py (-m gpu) and tests/test_fse_large_inputs.py (CPU) build the same bytes.

  uniform_bytes    2^30 + 64 bytes, 64 equally likely symbols: about 6 bits per symbol, so a 2^30-byte block codes to a stream
                   longer than 2^32 bits.  Blocks are views of it (a block at +1 is 2^30 - 1 bytes long).
  uniform_u16      2^29 + 8 symbols, uniform over 0..286: about 8.16 bits per symbol, a 2^29-symbol stream passes 2^32 bits.
  m2_block         2^30 bytes whose histogram sends FSE_normalizeCount to its second method with -1 cells at tableLog 12
                   (table_logs.m2_counts at n = 2^30), laid out by a bijective scramble of the index.
  threshold_buffer 2^30 bytes over 256 symbols whose 32 most frequent occur exactly 2^23 = 2^30 >> 7 times each.  Windows of it
                   (THRESHOLD_WINDOWS) put the most frequent count exactly at n >> 7 (coded) and one below it (stored raw by
                   the `maxCount < n >> 7` early exit).
  random_bytes     2^30 random bytes: a raw block (FSE stores it verbatim)."""
import numpy as np

from table_logs import fit_counts, m2_counts

N = 1 << 30                       # FSE_BLOCK_MAX
U16_N = N // 2                    # symbols
SCRAMBLE = 2654435761             # odd: i -> SCRAMBLE * i mod 2^30 is a bijection
TOP = 32                          # the threshold buffer's most frequent symbols
# (offset, bytes, most frequent count == n >> 7) of the threshold buffer's windows; the first two are coded, the third raw
THRESHOLD_WINDOWS = [(0, N, True), (0, N - 191, True), (64, N - 64, False)]
BATCH_BLOCK = (1 << 29) + 64      # uniform batch: 9 blocks, the 9th (ragged) starts past 2^32
BATCH_TAIL = (1 << 20) + 37
BATCH_TOTAL = 8 * BATCH_BLOCK + BATCH_TAIL


def uniform_bytes():
    return np.frombuffer(np.random.default_rng(0x5E1).bytes(N + 64), np.uint8) & np.uint8(63)


def uniform_u16():
    return np.random.default_rng(0x5E2).integers(0, 287, U16_N + 8, dtype=np.uint16)


def random_bytes():
    return np.frombuffer(np.random.default_rng(0x5E3).bytes(N), np.uint8)


def scrambled(symbols, counts):
    """N bytes: counts[i] copies of symbols[i], index i holding position SCRAMBLE * i mod N of the sorted run (the symbol is
    found from the run's cumulative counts rather than gathered from a 1 GiB run)"""
    import torch
    counts = np.asarray(counts, np.int64)
    assert counts.sum() == N
    ends = torch.from_numpy(np.cumsum(counts))
    syms = torch.from_numpy(np.asarray(symbols, np.uint8))
    out = torch.empty(N, dtype=torch.uint8)
    step = 1 << 24
    for i0 in range(0, N, step):
        j = torch.arange(i0, i0 + step, dtype=torch.int64).mul_(SCRAMBLE).bitwise_and_(N - 1)
        out[i0: i0 + step] = syms[torch.bucketize(j, ends, right=True)]
    return out.numpy()


def m2_histogram():
    """(counts, symbols) of m2_block"""
    return m2_counts(np.random.default_rng(0x5E4), N, 12, 255)


def m2_block():
    return scrambled(*m2_histogram()[::-1])


def threshold_parts():
    """(top symbols, other symbols, the others' counts): 32 symbols of 2^23 each, 224 sharing the rest geometrically"""
    rng = np.random.default_rng(0x5E5)
    top = np.sort(rng.choice(256, TOP, replace=False))
    rest = np.setdiff1d(np.arange(256), top)
    rc = fit_counts(0.992 ** np.arange(256 - TOP), N - TOP * (N >> 7))
    return top, rest, rc


def threshold_buffer():
    """the top symbols 2^23 times each, the scrambled layout rearranged by swaps with the middle so that the first 64 bytes hold
    each top symbol twice and the last 192 bytes 128 other symbols, then each top symbol twice.  So [0, N) holds every top
    symbol 2^23 times, [0, N - 191) and [64, N - 64) 2^23 - 2 times, against n >> 7 = 2^23, 2^23 - 2 and 2^23 - 1."""
    top, rest, rc = threshold_parts()
    out = scrambled(np.concatenate([top, rest]), np.concatenate([np.full(TOP, N >> 7), rc]))
    rng = np.random.default_rng(0x5E6)
    head = rng.permutation(np.repeat(top, 2))
    tail = np.concatenate([rng.permutation(rest[:128]), rng.permutation(np.repeat(top, 2))])
    pos = np.concatenate([np.arange(64), np.arange(N - 192, N)])
    pool = np.arange(1 << 20, (1 << 20) + (1 << 22))              # swap partners, far from both ends
    free = {int(s): list(pool[out[pool] == s]) for s in np.unique(np.concatenate([head, tail]))}
    for p, s in zip(pos, np.concatenate([head, tail])):
        q = free[int(s)].pop()
        out[q], out[p] = out[p], s
    return out


def batch_block(base, b, n):
    """block b of the uniform batch: the first n bytes of `base` (uniform_bytes) XOR b -- still 64 symbols, different bytes"""
    return base[:n] ^ np.uint8(b)


def packed_small():
    """the small compressible blocks that follow the four raw 2^30-byte blocks of the packed test"""
    from helpers import probagen
    rng = np.random.default_rng(0x5E7)
    return [probagen(int(n), 0.3) for n in rng.integers(1000, 200000, 60)]


def fbound(nbytes):
    return 512 + nbytes + (nbytes >> 7) + 4 + 8        # FSE_compressBound (lib/fse.h:290-292)


def header(lib, c, wide):
    """(header bytes, tableLog) of a compressed FSE / FSE-U16 block, read by the reference's FSE_readNCount"""
    import ctypes as C
    from helpers import is_error, ptr
    norm = (C.c_short * 300)()
    msv, tl = C.c_uint(286 if wide else 255), C.c_uint(0)
    h = lib.FSE_readNCount(norm, C.byref(msv), C.byref(tl), ptr(np.ascontiguousarray(c[:600])), min(len(c), 600))
    assert not is_error(h), h
    return int(h), tl.value


def ref_compress(lib, src, wide, cap=None):
    """(value, compressed bytes) of FSE_compress2 / FSE_compressU16 (msv 255 / 0, tableLog 12) at `cap` (default: the bound)"""
    from helpers import is_error, ptr
    n = len(src)
    cap = fbound(src.nbytes) if cap is None else cap
    buf = np.zeros(cap + 8, np.uint8)
    v = int((lib.FSE_compressU16 if wide else lib.FSE_compress2)(ptr(buf), cap, ptr(np.ascontiguousarray(src)), n, 0 if wide else 255, 12))
    return v, (buf[:v] if v > 1 and not is_error(v) else np.zeros(0, np.uint8))     # (not a view: the buffer may hold a cut stream)
