"""CPU checks of the large-block fixtures (tests/fse_large_inputs.py) of tests/test_gpu_fse_large.py: every block reaches what
that test claims for it -- its encode kernel (fse_blocks_paths.encode_route), its decode path (decode_path on the compiled
reference's block), a stream longer than 2^32 bits (8 * (cSize - header) > 2^32), FSE_normalizeCount's second method with -1
cells, both sides of the `maxCount < n >> 7` early exit, and offsets above 2^32.  Addresses are the GPU test's placements
relative to an allocation aligned to 2^32 (the GPU test asserts the same predicates on its real addresses)."""
import os
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import fse_large_inputs as L                                                    # noqa: E402
from helpers import REF_SO, load_ref                                             # noqa: E402
from fse_blocks_paths import decode_path, encode_route                          # noqa: E402
from fse_packed_paths import layout, slots, workspace                           # noqa: E402
from table_logs import normalize_method                                         # noqa: E402

BASE = 1 << 44                      # an allocation aligned to 2^32: no view below 4 GiB straddles a 2^32 address


def _ref():
    if not os.path.exists(REF_SO):
        pytest.skip("needs the compiled reference (oracle/_ref)")
    return load_ref()


def stream_bits(lib, c, wide):
    return 8 * (len(c) - L.header(lib, c, wide)[0])


def test_byte_blocks():
    """2^30 bytes at a 16-aligned source: the CTA encoder; 2^30 - 1 at +1: the warp encoder; both streams pass 2^32 bits; the
    first decodes on the windowed path into an aligned output and on the exact path at an output = 1 mod 4"""
    lib = _ref()
    S = L.uniform_bytes()
    assert encode_route(BASE, L.N, False) == "cta" and encode_route(BASE + 1, L.N - 1, False) == "warp"
    with ThreadPoolExecutor(2) as ex:
        (v1, c1), (v2, c2) = ex.map(lambda a: L.ref_compress(lib, S[a[0]: a[0] + a[1]], False), [(0, L.N), (1, L.N - 1)])
    assert v1 > 1 and v2 > 1 and stream_bits(lib, c1, False) > 1 << 32 and stream_bits(lib, c2, False) > 1 << 32
    h, tl = L.header(lib, c1, False)
    assert tl == 12
    assert decode_path(c1, v1, h, tl, BASE, BASE + (1 << 31), L.N, False) == "windowed"
    assert decode_path(c1, v1, h, tl, BASE + 1, BASE + (1 << 31), L.N, False) == "exact"


def test_second_method_block():
    """the m2 block's histogram: -1 cells and the second method of FSE_normalizeCount at tableLog 12, its most frequent count
    above n >> 7; the scramble keeps the histogram; the reference codes it"""
    lib = _ref()
    c, syms = L.m2_histogram()
    h = np.zeros(256, np.int64)
    h[syms] = c
    assert normalize_method(h, L.N, 255, 12) == (True, True)
    assert h.max() >= L.N >> 7 and (h == 1).sum() > 16
    M = L.m2_block()
    assert np.array_equal(np.bincount(M, minlength=256), h)
    v, cb = L.ref_compress(lib, M, False)
    assert v > 1 and L.header(lib, cb, False)[1] == 12


def test_threshold_windows():
    """the threshold buffer's windows: the most frequent count exactly n >> 7 in the first two (coded, on the CTA and the warp
    encoder) and one below it in the third (stored raw: value 0)"""
    lib = _ref()
    E = L.threshold_buffer()
    assert len(E) == L.N
    windows = [E[o: o + n] for o, n, _ in L.THRESHOLD_WINDOWS]
    for w, (o, n, at) in zip(windows, L.THRESHOLD_WINDOWS):
        best = int(np.bincount(w, minlength=256).max())
        assert best == (n >> 7) if at else best == (n >> 7) - 1, (o, n, best)
    assert [encode_route(BASE + o, n, False) for o, n, _ in L.THRESHOLD_WINDOWS] == ["cta", "warp", "cta"]
    with ThreadPoolExecutor(3) as ex:
        vals = [v for v, _ in ex.map(lambda w: L.ref_compress(lib, w, False), windows)]
    assert vals[0] > 1 and vals[1] > 1 and vals[2] == 0, vals


def test_u16_blocks():
    """2^29 U16 symbols at a 16-aligned source: the CTA encoder; 2^29 - 1 at +2: the warp encoder; both streams pass 2^32 bits;
    an output = 0 mod 8 decodes on the windowed path, one = 2 mod 8 on the exact path"""
    lib = _ref()
    U = L.uniform_u16()
    assert encode_route(BASE, L.U16_N, True) == "cta" and encode_route(BASE + 2, L.U16_N - 1, True) == "warp"
    with ThreadPoolExecutor(2) as ex:
        (v1, c1), (v2, c2) = ex.map(lambda a: L.ref_compress(lib, U[a[0]: a[0] + a[1]], True), [(0, L.U16_N), (1, L.U16_N - 1)])
    assert v1 > 1 and v2 > 1 and stream_bits(lib, c1, True) > 1 << 32 and stream_bits(lib, c2, True) > 1 << 32
    h, tl = L.header(lib, c1, True)
    assert decode_path(c1, v1, h, tl, BASE, BASE + (1 << 31), L.U16_N, True) == "windowed"
    assert decode_path(c1, v1, h, tl, BASE + 2, BASE + (1 << 31), L.U16_N, True) == "exact"


def test_batch_offsets():
    """the uniform batch: full blocks of 2^29 + 64 bytes (a whole number of 64-byte groups: the CTA encoder), a ragged 9th block
    (the warp encoder) whose source, slot and output offsets pass 2^32"""
    assert L.BATCH_BLOCK % 64 == 0 and encode_route(BASE + 8 * L.BATCH_BLOCK, L.BATCH_TAIL, False) == "warp"
    assert L.BATCH_TOTAL // L.BATCH_BLOCK == 8 and L.BATCH_TOTAL % L.BATCH_BLOCK == L.BATCH_TAIL
    assert 8 * L.BATCH_BLOCK > 1 << 32 and 8 * L.fbound(L.BATCH_BLOCK) > 1 << 32


def test_packed_offsets():
    """the packed test: four raw 2^30-byte blocks, then the small ones, whose stored offsets, staging slots and the workspace
    pass 2^32"""
    lib = _ref()
    from fse_packed_paths import ref_value
    R = L.random_bytes()
    assert ref_value(lib, R, False, 255, 12)[0] == 0
    small = L.packed_small()
    vals = [ref_value(lib, s, False, 255, 12)[0] for s in small]
    assert all(v > 1 for v in vals)
    sizes = [L.N] * 4 + [len(s) for s in small]
    total = sum(sizes)
    offs, final, _ = layout([0] * 4 + vals, sizes, total + 32, False)
    assert offs[4] == 4 * L.N == 1 << 32 and min(offs[5:]) > 1 << 32 and final[4:] == vals
    work = workspace(len(sizes), total)
    so, coded = slots([BASE] * len(sizes), sizes, False, work)
    assert work > 1 << 32 and all(coded) and min(so[4:]) > 1 << 32
