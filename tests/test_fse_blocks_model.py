"""CPU-only checks of the host-side models of the FSE / FSE-U16 descriptor calls (tests/fse_blocks_paths.py), on hand-computed
cases and on random block placements: the encoder routing, the CTA group counts, the decoder's windowed-vs-exact choice with
sameHi from the block's own extent, and the decoder's read range against the readable sectors."""
import random

import numpy as np

from fse_blocks_paths import (ERR_GENERIC, ERR_SRC_WRONG, FSE_BLOCK_MAX, cta_groups, decode_path, encode_route, read_range,
                              readable_range, same_hi)


def test_encode_route():
    assert encode_route(0, 32768, False) == "cta" and encode_route(16, 64, False) == "cta"
    assert encode_route(8, 32768, False) == "warp" and encode_route(0, 32769, False) == "warp" and encode_route(0, 0, False) == "warp"
    assert encode_route(0, 1, False) == "warp"                        # FSE_compress2's own n <= 1 verdict, after its parameter checks
    assert encode_route(0, FSE_BLOCK_MAX, False) == "cta" and encode_route(0, FSE_BLOCK_MAX + 1, False) == ERR_SRC_WRONG
    # U16: sizes in symbols, bytes decide the kernel
    assert encode_route(0, 32, True) == "cta" and encode_route(0, 16, True) == "warp" and encode_route(2, 16384, True) == "warp"
    assert encode_route(3, 16384, True) == ERR_GENERIC and encode_route(3, 0, True) == ERR_GENERIC
    assert encode_route(0, 1, True) == 1 and encode_route(0, 0, True) == 0
    assert encode_route(0, FSE_BLOCK_MAX // 2, True) == "cta" and encode_route(0, FSE_BLOCK_MAX // 2 + 1, True) == ERR_SRC_WRONG


def test_cta_groups():
    assert cta_groups([32768] * 16) == ([512] * 16, 512)
    assert cta_groups([64, 4096, 65536]) == ([1, 64, 1024], 1024)
    assert cta_groups([]) == ([], 0)


def test_same_hi_uses_the_block_extent():
    base = 5 << 32
    assert same_hi(base, 32768, base + 100, 5000)
    assert not same_hi(base, 32768, base - 64, 61)                    # the last word reaches past the 4 GiB boundary
    assert same_hi(base, 32768, base - 64, 60)                        # ... and this one ends on it
    assert not same_hi(base - 8, 32768, base + 100, 5000)             # output straddles


def test_decode_path():
    blk = np.zeros(200, np.uint8); blk[-1] = 0x80                    # end mark in bit 7: used = 1
    # bytes, tl 12: used 1 + 12 -> at 192 - 8 - 1 = 183, used 5; + 12 -> at 181, used 1; (181 - 24) // 6 = 26 chunks
    assert decode_path(blk, 200, 8, 12, 0, 1000, 1000, False) == "windowed"
    assert decode_path(blk, 200, 8, 12, 2, 1000, 1000, False) == "exact"     # output not word aligned
    assert decode_path(blk, 200, 8, 12, 0, 1000, 3, False) == "exact"        # fewer than 4 output slots
    assert decode_path(blk, 40, 8, 12, 0, 1000, 1000, False) == "exact"      # too short for a chunk
    assert decode_path(blk, 200, 8, 12, 4, 1000, 1000, True) == "exact"      # U16 needs 8-byte aligned output
    assert decode_path(blk, 200, 8, 12, 8, 1000, 1000, True) == "windowed"
    b0 = blk.copy(); b0[-1] = 0
    assert decode_path(b0, 200, 8, 12, 0, 1000, 1000, False) == "exact"


def test_read_range_inside_readable_sectors():
    rng = random.Random(5)
    for _ in range(20000):
        c = rng.randrange(0, 1 << 40)
        n = rng.choice([0, 1, 2, 3, 4, 5, 7, 8, 31, 32, 33, rng.randrange(0, 1 << 20)])
        lo, hi = read_range(c, n)
        rlo, rhi = readable_range(c, n)
        assert rlo <= lo and hi <= rhi, (c, n)
        assert hi >= c + n
    assert read_range(33, 3) == (32, 36) and readable_range(33, 3) == (32, 64)
    assert read_range(61, 3) == (48, 64) and read_range(61, 4) == (48, 68) and readable_range(61, 4) == (32, 96)
