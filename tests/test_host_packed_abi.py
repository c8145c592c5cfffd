"""CPU-side checks of the packed Huff0 decompress and the packed host-buffer calls: the header declares them, the library exports
them, and the host calls' argument checks -- which answer before any device work -- return srcSize_wrong or 0 without a GPU."""
import ctypes as C
import re
import subprocess

import numpy as np

from helpers import declared_arity

NEW_CALLS = ("FSEB200_HUF_decompress_packed", "FSEB200_HUF_decompress1X_packed",
             "FSEB200_compress_host_packed", "FSEB200_decompress_host_packed")
ERR_SRC_WRONG = 2 ** 64 - 3


def test_header_declares_the_packed_host_calls():
    decl = declared_arity()
    arity = {"FSEB200_HUF_decompress_packed": 7, "FSEB200_HUF_decompress1X_packed": 7,
             "FSEB200_compress_host_packed": 10, "FSEB200_decompress_host_packed": 7}
    assert {n: decl.get(n) for n in NEW_CALLS} == arity


def test_library_exports_the_packed_host_calls():
    from finitestateentropy_b200 import _build
    path = _build.build_lib()
    exported = subprocess.check_output(["nm", "-D", "--defined-only", path]).decode()
    for name in NEW_CALLS:
        assert re.search(r" T %s$" % name, exported, flags=re.M), name


def test_host_packed_argument_checks():
    """bad codec, nBlocks above 2^32 - 1, a NULL pointer, decreasing offsets: srcSize_wrong; nBlocks == 0: 0, nothing written"""
    import finitestateentropy_b200 as fb
    L = fb.lib()
    buf = np.full(64, 7, np.uint64)
    p = buf.ctypes.data
    enc, dec = L.FSEB200_compress_host_packed, L.FSEB200_decompress_host_packed
    for codec in (-1, 4, 100):
        assert enc(codec, p, 64, p, p, p, p, 1, 255, 12) == ERR_SRC_WRONG
        assert dec(codec, p, p, p, p, p, 1) == ERR_SRC_WRONG
    for codec in range(4):
        assert enc(codec, p, 64, p, p, p, p, 1 << 32, 255, 12) == ERR_SRC_WRONG
        assert dec(codec, p, p, p, p, p, 1 << 32) == ERR_SRC_WRONG
        for k in range(5):
            args = [p] * 5
            args[k] = None
            assert enc(codec, args[0], 64, args[1], args[2], args[3], args[4], 1, 255, 12) == ERR_SRC_WRONG
            assert dec(codec, args[0], args[1], args[2], args[3], args[4], 1) == ERR_SRC_WRONG
        assert enc(codec, p, 64, p, p, p, p, 0, 255, 12) == 0
        assert dec(codec, p, p, p, p, p, 0) == 0
        assert enc(codec, None, 0, None, None, None, None, 0, 255, 12) == 0
        offs = np.array([0, 5, 4, 9], np.uint64)
        assert dec(codec, p, p, p, p, offs.ctypes.data, 3) == ERR_SRC_WRONG
    assert (buf == 7).all()
    for fn in (L.FSEB200_HUF_decompress_packed, L.FSEB200_HUF_decompress1X_packed):
        assert fn(0, None, None, None, None, None, None) == 0
        for k in range(5):
            args = [p] * 5
            args[k] = None
            assert fn(1, args[0], args[1], args[2], args[3], args[4], None) == ERR_SRC_WRONG
        assert fn(1 << 32, p, p, p, p, p, None) == ERR_SRC_WRONG


def test_python_wrappers_check_their_arguments():
    import pytest
    import torch
    import finitestateentropy_b200 as fb
    src = torch.zeros(100, dtype=torch.uint8)
    with pytest.raises(KeyError):
        fb.host_compress_packed(src, [10], "lz4")
    with pytest.raises(AssertionError):
        fb.host_compress_packed(src, [60, 50], "huf")                    # sizes beyond the source
    with pytest.raises(AssertionError):
        fb.host_compress_packed(src, [30, 30], "fseu16")                 # 120 bytes of symbols
    with pytest.raises(AssertionError):
        fb.host_decompress_packed(src, torch.tensor([0, 10]), [10, 10], "fse")   # offsets: n + 1 entries
    with pytest.raises(AssertionError):
        fb.host_decompress_packed(src, torch.tensor([0, 200]), [10], "fse")      # beyond the packed buffer
