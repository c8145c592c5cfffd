"""CPU-side checks of the packed Huff0 chain calls on host buffers (FSEB200_compress_host_repeat_chains_packed /
FSEB200_decompress_host_repeat_packed): the header declares them, the library exports them, and every verdict the host settles
before any device work -- bad arguments, nBlocks == 0, malformed chain geometry -- is answered without a GPU, writing only what
the device calls would write."""
import re
import subprocess

import numpy as np
import pytest

from helpers import declared_arity

CALLS = {"FSEB200_compress_host_repeat_chains_packed": 18, "FSEB200_decompress_host_repeat_packed": 12}
ERR_SRC_WRONG = 2 ** 64 - 3
FILL = 0x7777777777777777


def test_header_declares_the_host_chain_calls():
    decl = declared_arity()
    assert {n: decl.get(n) for n in CALLS} == CALLS


def test_library_exports_the_host_chain_calls():
    from finitestateentropy_b200 import _build
    exported = subprocess.check_output(["nm", "-D", "--defined-only", _build.build_lib()]).decode()
    for name in CALLS:
        assert re.search(r" T %s$" % name, exported, flags=re.M), name


class Batch:
    """host arrays of a 3-block, 2-chain batch, every word filled with FILL, so that any write shows"""

    def __init__(self):
        self.starts = np.array([0, 2, 3], np.uint64)
        self.sizes = np.array([5, 6, 7], np.uint64)
        self.src = np.arange(18, dtype=np.uint8)
        self.prefer = np.zeros(3, np.int32)
        self.out = np.full(64, 0x77, np.uint8)
        self.offsets = np.full(4, FILL, np.uint64)
        self.values = np.full(3, FILL, np.uint64)
        self.kinds = np.full(3, 0x77, np.uint8)
        self.tables = np.full((2, 256), 0x77777777, np.uint32)
        self.table_ptrs = np.array([self.tables[c].ctypes.data for c in range(2)], np.uint64)
        self.flags = np.full(2, 0x77777777, np.int32)
        self.hdr = np.full(2, FILL, np.uint64)
        self.hdr_sizes = np.full(2, FILL, np.uint64)
        self.dst = np.full(18, 0x77, np.uint8)
        self.results = np.full(3, FILL, np.uint64)
        self.packed_offsets = np.array([0, 5, 6, 13], np.uint64)

    def snapshot(self):
        return {k: v.copy() for k, v in self.__dict__.items()}

    def compress(self, codec=1, n_chains=2, starts=None, n_blocks=3, null=None):
        import finitestateentropy_b200 as fb
        starts = self.starts if starts is None else starts
        args = [starts, self.out, self.offsets, self.values, self.kinds, self.src, self.sizes, self.prefer, self.table_ptrs,
                self.flags, self.hdr, self.hdr_sizes]
        p = [a.ctypes.data for a in args]
        if null is not None:
            p[null] = None
        return fb.lib().FSEB200_compress_host_repeat_chains_packed(codec, n_chains, p[0], n_blocks, p[1], 64, p[2], p[3], p[4], p[5],
                                                                   p[6], p[7], p[8], p[9], p[10], p[11], 255, 11)

    def decompress(self, codec=1, n_chains=2, starts=None, n_blocks=3, offsets=None, null=None):
        import finitestateentropy_b200 as fb
        starts = self.starts if starts is None else starts
        offsets = self.packed_offsets if offsets is None else offsets
        args = [starts, self.dst, self.sizes, self.results, self.out, offsets, self.kinds, self.hdr, self.hdr_sizes]
        p = [a.ctypes.data for a in args]
        if null is not None:
            p[null] = None
        return fb.lib().FSEB200_decompress_host_repeat_packed(codec, n_chains, p[0], n_blocks, p[1], p[2], p[3], p[4], p[5], p[6],
                                                              p[7], p[8])


def _same(a, b):
    return all(np.array_equal(a[k], b[k]) for k in a)


def test_argument_verdicts_write_nothing():
    """a codec other than 1 and 3, nBlocks or nChains above 2^32 - 1, any NULL pointer: srcSize_wrong; nBlocks == 0: 0"""
    x = Batch()
    before = x.snapshot()
    for codec in (-1, 0, 2, 4, 100):
        assert x.compress(codec=codec) == ERR_SRC_WRONG
        assert x.decompress(codec=codec) == ERR_SRC_WRONG
    for codec in (1, 3):
        assert x.compress(codec=codec, n_blocks=1 << 32) == ERR_SRC_WRONG
        assert x.decompress(codec=codec, n_blocks=1 << 32) == ERR_SRC_WRONG
        assert x.compress(codec=codec, n_chains=1 << 32) == ERR_SRC_WRONG
        assert x.decompress(codec=codec, n_chains=1 << 32) == ERR_SRC_WRONG
        for k in range(12):
            assert x.compress(codec=codec, null=k) == ERR_SRC_WRONG, k
        for k in range(9):
            assert x.decompress(codec=codec, null=k) == ERR_SRC_WRONG, k
        assert x.compress(codec=codec, n_blocks=0) == 0
        assert x.decompress(codec=codec, n_blocks=0) == 0
        assert x.decompress(codec=codec, offsets=np.array([0, 5, 4, 13], np.uint64)) == ERR_SRC_WRONG
        assert _same(before, x.snapshot())
    import finitestateentropy_b200 as fb
    L = fb.lib()
    assert L.FSEB200_compress_host_repeat_chains_packed(1, 0, None, 0, None, 0, None, None, None, None, None, None, None, None, None,
                                                        None, 255, 11) == 0
    assert L.FSEB200_decompress_host_repeat_packed(3, 0, None, 0, None, None, None, None, None, None, None, None) == 0


@pytest.mark.parametrize("codec", [1, 3])
@pytest.mark.parametrize("starts", [[1, 2, 3], [0, 2, 2], [0, 3, 2], [0, 2, 4]])
def test_malformed_geometry_gives_only_verdicts_and_kinds(codec, starts):
    """a first start above 0, a last start other than nBlocks, a decreasing start: every value srcSize_wrong and kind 4 (compress),
    every result srcSize_wrong (decompress); no offset, output byte or state word written"""
    x = Batch()
    before = x.snapshot()
    st = np.array(starts, np.uint64)
    assert x.compress(codec=codec, starts=st) == 0
    assert (x.values == ERR_SRC_WRONG).all() and (x.kinds == 4).all()
    after = x.snapshot()
    for k in before:
        if k not in ("values", "kinds"):
            assert np.array_equal(before[k], after[k]), k
    x.kinds[:] = 2
    assert x.decompress(codec=codec, starts=st) == 0
    assert (x.results == ERR_SRC_WRONG).all()
    assert (x.dst == 0x77).all()
    # no chains at all for a non-empty batch is malformed too
    y = Batch()
    assert y.compress(codec=codec, n_chains=0, starts=np.zeros(1, np.uint64)) == 0
    assert (y.values == ERR_SRC_WRONG).all() and (y.kinds == 4).all() and (y.offsets == FILL).all()


def test_python_wrappers_check_their_arguments():
    import torch
    import finitestateentropy_b200 as fb
    src = torch.zeros(100, dtype=torch.uint8)
    tabs, reps = torch.zeros((1, 256), dtype=torch.int32), torch.zeros(1, dtype=torch.int32)
    hp, hs = torch.zeros(1, dtype=torch.int64), torch.zeros(1, dtype=torch.int64)
    pr = torch.zeros(2, dtype=torch.int32)
    with pytest.raises(KeyError):
        fb.host_compress_repeat_chains_packed(src, [10, 10], [0, 2], pr, tabs, reps, hp, hs, codec="fse")
    with pytest.raises(AssertionError):
        fb.host_compress_repeat_chains_packed(src, [60, 50], [0, 2], pr, tabs, reps, hp, hs)          # sizes beyond the source
    with pytest.raises(AssertionError):
        fb.host_compress_repeat_chains_packed(src, [10, 10], [0, 1, 2], pr, tabs, reps, hp, hs)       # 2 chains, 1 table
    with pytest.raises(AssertionError):
        fb.host_compress_repeat_chains_packed(src, [10, 10], [0, 2], pr[:1], tabs, reps, hp, hs)      # a prefer flag per block
    with pytest.raises(AssertionError):
        fb.host_decompress_repeat_packed(src, torch.tensor([0, 10]), torch.zeros(2, dtype=torch.uint8), [0, 2], [10, 10], hp, hs)
