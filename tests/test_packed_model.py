"""CPU-only checks of the packed Huff0 compress's host model (tests/packed_paths.py), no GPU code involved:

  * the stored-length, offset and capacity rules on hand-computed cases;
  * against the compiled reference: a stored block is never longer than its source (HUF_compress2 and HUF_compress1X at
    HUF_compressBound(n)), so an output of sum(n) bytes always holds every block -- over the test contents and over sizes
    0-16, 128 KB and every residue mod 4;
  * the packed image the model builds from the reference decodes, block by block, with the reference's own decoders."""
import numpy as np
import pytest

from helpers import have_ref, is_error, load_ref, probagen
from packed_paths import ERR_DST_TOO_SMALL, stored_len, layout, ref_values, image, ref_decode

ERR_SRC_WRONG = 2 ** 64 - 3


def _ref():
    if not have_ref():
        pytest.skip("needs the compiled reference (oracle/_ref)")
    lib = load_ref()
    if lib is None:
        pytest.skip("needs the compiled reference (oracle/_ref)")
    return lib


def test_stored_length():
    assert stored_len(0, 0) == 0                      # empty block
    assert stored_len(0, 500) == 500                  # not compressible: a raw copy
    assert stored_len(1, 500) == 1                    # RLE: the byte
    assert stored_len(321, 500) == 321
    assert stored_len(ERR_SRC_WRONG, 200000) == 0


def test_offsets_and_capacity_rule():
    vals = [100, 0, 1, ERR_SRC_WRONG, 0, 50]
    sizes = [400, 30, 9, 200000, 0, 80]
    offs, final, fits = layout(vals, sizes, 10 ** 9)
    assert offs == [0, 100, 130, 131, 131, 131, 181]
    assert final == vals and fits == [True, True, True, False, True, True]
    # total - 1: only the last block is cut; the offsets stay the full prefix sum
    offs2, final2, fits2 = layout(vals, sizes, 180)
    assert offs2 == offs and final2 == vals[:5] + [ERR_DST_TOO_SMALL] and fits2[:5] == fits[:5] and not fits2[5]
    # cut inside the raw block: it and everything after it that has bytes; the error keeps its code; the empty block at
    # offset 131 fits a capacity of 131, not one of 120
    _, final3, _ = layout(vals, sizes, 120)
    assert final3 == [100, ERR_DST_TOO_SMALL, ERR_DST_TOO_SMALL, ERR_SRC_WRONG, ERR_DST_TOO_SMALL, ERR_DST_TOO_SMALL]
    _, final4, _ = layout(vals, sizes, 131)
    assert final4 == [100, 0, 1, ERR_SRC_WRONG, 0, ERR_DST_TOO_SMALL]
    _, final5, fits5 = layout(vals, sizes, 0)
    assert final5 == [ERR_DST_TOO_SMALL] * 3 + [ERR_SRC_WRONG] + [ERR_DST_TOO_SMALL] * 2 and not any(fits5)


def contents(rng, n):
    """the test contents: probagen P02 / P14 / P80, random, constant, two symbols"""
    off = int(rng.integers(0, 4096))
    two = np.where(rng.random(n) < 0.7, 65, 200).astype(np.uint8)
    return [probagen(off + n, 0.02)[off:], probagen(off + n, 0.14)[off:], probagen(off + n, 0.80)[off:],
            rng.integers(0, 256, n, dtype=np.uint8), np.full(n, int(rng.integers(0, 256)), np.uint8), two]


BOUND_SIZES = list(range(0, 17)) + [1021, 1022, 1023, 1024, 4097, 4098, 4099, 4100, 32765, 32766, 32767, 32768,
                                    131069, 131070, 131071, 131072]


@pytest.mark.parametrize("onex", [False, True], ids=["4X", "1X"])
def test_stored_length_never_exceeds_the_source(onex):
    lib = _ref()
    rng = np.random.default_rng(11)
    kinds = set()
    for n in BOUND_SIZES:
        srcs = contents(rng, n)
        vals, stored = ref_values(lib, srcs, 255, 12, onex)
        for s, v, st in zip(srcs, vals, stored):
            assert not is_error(v), (n, v)
            assert len(st) == stored_len(v, n) <= n, (n, v)
            kinds.add(0 if v == 0 else 1 if v == 1 else "size")
    assert kinds == {0, 1, "size"}


@pytest.mark.parametrize("onex", [False, True], ids=["4X", "1X"])
def test_packed_image_decodes_with_the_reference(onex):
    lib = _ref()
    rng = np.random.default_rng(12)
    srcs = []
    for n in [0, 1, 2, 11, 12, 13, 200, 4099, 32768, 131072, 131073] + [int(x) for x in rng.integers(1, 20000, 20)]:
        srcs.append(contents(rng, n)[len(srcs) % 6])
    sizes = [len(s) for s in srcs]
    vals, stored = ref_values(lib, srcs, 255, 12, onex)
    assert vals[sizes.index(131073)] == ERR_SRC_WRONG
    img, written, offs, final = image(vals, stored, sizes, sum(sizes))
    assert final == vals and offs[-1] <= sum(sizes) and bool(written.all())
    for b, r in enumerate(ref_decode(lib, img, offs, sizes, vals, onex)):
        if r is None:
            assert sizes[b] == 0 or is_error(vals[b])
            continue
        assert r[0] == sizes[b] and np.array_equal(r[1], srcs[b]), (b, sizes[b], vals[b], r[0])
