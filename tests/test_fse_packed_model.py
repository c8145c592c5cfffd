"""CPU-only checks of the packed FSE / FSE-U16 host model (tests/fse_packed_paths.py), no GPU code involved:

  * the stored-length, staging-slot, offset, capacity and decode rules on hand-computed cases;
  * against the compiled reference, the facts the stored format rests on, over constant, two-symbol, skewed, random and
    probagen contents, sizes 0-16, every residue mod 4, 64, 4099, 32 KB, 128 KB and 1 MiB, and tableLogs 5 and 12:
    a stored block is never longer than u * n; no FSE compressed block has a value of 1 or >= n - 1; no U16 compressed block
    is 2 or 2n bytes long -- so the decode rules "L == u * n is raw" and "L == u is RLE" never capture a compressed block;
  * the packed image the model builds from the reference regenerates every block through the decode rule;
  * FSEB200_FSE_packed_workspace's formula covers the sum of FSE_compressBound over random batches."""
import numpy as np
import pytest

from helpers import gen_u16, have_ref, is_error, load_ref, probagen
from fse_packed_paths import (ERR_CORRUPT, ERR_DST_TOO_SMALL, ERR_GENERIC, ERR_SRC_WRONG, ERR_WKSP_TOO_SMALL, FSE_BLOCK_MAX,
                              decode_rule, fbound, image, layout, ref_unpack, ref_value, slots, stored_len, values, workspace)

CODECS = [False, True]
CODEC_IDS = ["FSE", "U16"]


def _ref():
    if not have_ref():
        pytest.skip("needs the compiled reference (oracle/_ref)")
    lib = load_ref()
    if lib is None:
        pytest.skip("needs the compiled reference (oracle/_ref)")
    return lib


def test_stored_length():
    assert stored_len(0, 0, False) == 0 and stored_len(0, 0, True) == 0      # empty blocks
    assert stored_len(0, 500, False) == 500 and stored_len(0, 500, True) == 1000
    assert stored_len(1, 500, False) == 1 and stored_len(1, 500, True) == 2  # RLE: the unit
    assert stored_len(1, 1, True) == 2                                       # U16 n == 1 returns n itself: RLE, 2 bytes
    assert stored_len(321, 500, True) == 321
    assert stored_len(ERR_SRC_WRONG, 2 ** 31, False) == 0


def test_slots_and_workspace_verdicts():
    # block 1 is a U16 source at an odd address and block 3 is above the limit: neither takes a slot
    addrs, sizes = [0, 1, 2, 4, 8], [100, 50, 0, FSE_BLOCK_MAX // 2 + 1, 3]
    need = fbound(200) + fbound(0) + fbound(6)
    offs, coded = slots(addrs, sizes, True, need)
    assert offs == [0, None, fbound(200), None, fbound(200) + fbound(0)] and coded == [True, False, True, False, True]
    _, coded = slots(addrs, sizes, True, need - 1)
    assert coded == [True, False, True, False, False]                        # one byte short: the last coded block only
    got = values([7, 7, 0, 7, 9], addrs, sizes, True, need - 1)
    assert got == [7, ERR_GENERIC, 0, ERR_SRC_WRONG, ERR_WKSP_TOO_SMALL]
    assert values([7, 0], [0, 0], [10, 20], False, 0) == [ERR_WKSP_TOO_SMALL] * 2
    assert workspace(3, 1000) == 1000 + 7 + 3 * 524


def test_offsets_and_capacity_rule():
    vals = [100, 0, 1, ERR_SRC_WRONG, 0, 50]
    sizes = [400, 30, 9, 2 ** 31, 0, 80]
    offs, final, fits = layout(vals, sizes, 10 ** 9, True)
    assert offs == [0, 100, 160, 162, 162, 162, 212]
    assert final == vals and fits == [True, True, True, False, True, True]
    offs2, final2, _ = layout(vals, sizes, 211, True)
    assert offs2 == offs and final2 == vals[:5] + [ERR_DST_TOO_SMALL]
    _, final3, _ = layout(vals, sizes, 0, False)
    assert final3 == [ERR_DST_TOO_SMALL] * 3 + [ERR_SRC_WRONG] + [ERR_DST_TOO_SMALL] * 2


def test_decode_rule():
    assert decode_rule(10, 10, 0, False) == "raw" and decode_rule(20, 10, 0, True) == "raw"
    assert decode_rule(0, 0, 0, False) == "raw" and decode_rule(0, 0, 0, True) == "raw"
    assert decode_rule(1, 10, 0, False) == "rle" and decode_rule(2, 10, 0, True) == "rle"
    assert decode_rule(1, 1, 0, False) == "raw" and decode_rule(2, 1, 0, True) == "raw"
    assert decode_rule(0, 10, 0, False) == "decode" and decode_rule(1, 10, 0, True) == "decode"
    assert decode_rule(5, 10, 1, True) == "limit" and decode_rule(2, 10, 1, True) == "limit"
    assert decode_rule(FSE_BLOCK_MAX + 1, 10, 0, False) == "limit"
    assert decode_rule(5, FSE_BLOCK_MAX // 2 + 1, 0, True) == "limit"


def test_empty_stored_length_decodes_to_the_reference_verdict():
    lib = _ref()
    assert ref_unpack(lib, np.zeros(8, np.uint8), 0, 10, False) == (ERR_CORRUPT, None)
    assert ref_unpack(lib, np.zeros(8, np.uint8), 0, 10, True) == (ERR_SRC_WRONG, None)
    assert ref_unpack(lib, np.zeros(8, np.uint8), 3, 10, True, dst_addr=1) == (ERR_GENERIC, None)


SIZES = list(range(0, 17)) + [64, 1021, 1022, 1023, 1024, 4097, 4098, 4099, 4100, 32768, 131072, 1 << 20]


def contents(rng, n, wide):
    """constant, two symbols, skewed, random, probagen"""
    if wide:
        two = np.where(rng.random(n) < 0.7, 40, 280).astype(np.uint16)
        return [np.full(n, int(rng.integers(0, 287)), np.uint16), two, gen_u16(n, 240, 0.8, int(rng.integers(1, 1000))),
                rng.integers(0, 287, n).astype(np.uint16), gen_u16(n, 240, 0.3, int(rng.integers(1, 1000)))]
    off = int(rng.integers(0, 4096))
    two = np.where(rng.random(n) < 0.7, 65, 200).astype(np.uint8)
    return [np.full(n, int(rng.integers(0, 256)), np.uint8), two, probagen(off + n, 0.80)[off:],
            rng.integers(0, 256, n, dtype=np.uint8), probagen(off + n, 0.14)[off:]]


@pytest.mark.parametrize("wide", CODECS, ids=CODEC_IDS)
@pytest.mark.parametrize("tl", [5, 12])
def test_stored_format_facts(wide, tl):
    lib = _ref()
    u = 2 if wide else 1
    rng = np.random.default_rng(21 + tl + wide)
    kinds = set()
    for n in SIZES:
        for src in contents(rng, n, wide):
            v, st = ref_value(lib, src, wide, 0 if wide else 255, tl)
            assert not is_error(v), (n, v)
            assert len(st) == stored_len(v, n, wide) <= u * n, (n, v)
            if v >= 2:                                                      # a compressed block
                if wide:
                    assert v != 2 and v != 2 * n, (n, v)
                else:
                    assert v < n - 1, (n, v)
                assert decode_rule(v, n, 0, wide) == "decode"
            kinds.add(0 if v == 0 else 1 if v == 1 else "size")
    assert kinds == {0, 1, "size"}


@pytest.mark.parametrize("wide", CODECS, ids=CODEC_IDS)
def test_packed_image_round_trip(wide):
    lib = _ref()
    rng = np.random.default_rng(22 + wide)
    srcs = []
    for n in [0, 1, 2, 3, 11, 64, 200, 4099, 32768] + [int(x) for x in rng.integers(1, 20000, 25)]:
        srcs.append(contents(rng, n, wide)[len(srcs) % 5])
    sizes = [len(s) for s in srcs]
    ref = [ref_value(lib, s, wide, 0 if wide else 255, 12) for s in srcs]
    vals, stored = [r[0] for r in ref], [r[1] for r in ref]
    assert {0, 1} <= set(vals) and any(v > 1 for v in vals)
    u = 2 if wide else 1
    img, written, offs, final = image(vals, stored, sizes, u * sum(sizes), wide)
    assert final == vals and offs[-1] <= u * sum(sizes) and bool(written.all())
    padded = np.concatenate([img, np.zeros(64, np.uint8)])
    for b, n in enumerate(sizes):
        r, out = ref_unpack(lib, padded[offs[b]:], offs[b + 1] - offs[b], n, wide)
        assert r == n and np.array_equal(out, np.ascontiguousarray(srcs[b]).view(np.uint8)), (b, n, vals[b], r)


def test_workspace_covers_the_bounds():
    rng = np.random.default_rng(23)
    for _ in range(200):
        k = int(rng.integers(1, 400))
        sizes = [int(x) for x in rng.integers(0, int(rng.choice([130, 5000, 1 << 20])), k)]
        for wide in CODECS:
            nb = [(2 if wide else 1) * n for n in sizes]
            assert workspace(k, sum(nb)) >= sum(fbound(x) for x in nb)
