"""CPU-side checks of the .fse frame calls on device memory (FSEB200_frame_{compress,decompress}_device and
FSEB200_frame_decompress_bound_device): declarations and exports, the argument verdicts, which touch no device, and the Python
wrappers' argument checks.  The header walk these calls run on the device is the one the host calls run: test_frame_abi.py and
test_frame_batch_abi.py check its verdicts through FSEB200_frame_decompress_bound and the batch calls."""
import re
import subprocess

import numpy as np
import pytest

from helpers import declared_arity
from test_frame_abi import ERR, MAGIC

DEVICE_CALLS = {"FSEB200_frame_compress_device": 10, "FSEB200_frame_decompress_bound_device": 5,
                "FSEB200_frame_decompress_device": 7}
POISON = 0x5A


def _lib():
    import finitestateentropy_b200 as fb
    return fb.lib()


def _words(values):
    return np.array(values, dtype=np.uint64)


def test_header_declares_and_library_exports_the_device_calls():
    decl = declared_arity()
    assert {n: decl.get(n) for n in DEVICE_CALLS} == DEVICE_CALLS
    from finitestateentropy_b200 import _build
    exported = subprocess.check_output(["nm", "-D", "--defined-only", _build.build_lib()]).decode()
    for name in DEVICE_CALLS:
        assert re.search(r" T %s$" % name, exported, flags=re.M), name


def test_compress_argument_verdicts():
    """bad codec, id above 6, nFrames above 2^32 - 1, a NULL pointer while nFrames > 0, a NULL source with a non-empty frame:
    srcSize_wrong and nothing written; nFrames == 0 returns 0.  The pointers stand in for device buffers: nothing may touch them."""
    L = _lib()
    out, offs, res = np.full(64, POISON, np.uint8), np.full(3, 7, np.uint64), np.full(2, 7, np.uint64)
    src, sizes = np.full(100, 1, np.uint8), _words([60, 40])
    args = [out.ctypes.data, 64, offs.ctypes.data, res.ctypes.data, src.ctypes.data, sizes.ctypes.data, None]
    for codec in (-1, 2, 7):
        assert L.FSEB200_frame_compress_device(codec, 5, 2, *args) == ERR["srcSize_wrong"]
    for bid in (7, 255, 2 ** 31):
        assert L.FSEB200_frame_compress_device(0, bid, 2, *args) == ERR["srcSize_wrong"]
    assert L.FSEB200_frame_compress_device(0, 5, 2 ** 32, *args) == ERR["srcSize_wrong"]
    for i in (0, 2, 3, 4, 5):
        bad = list(args)
        bad[i] = None
        assert L.FSEB200_frame_compress_device(1, 5, 2, *bad) == ERR["srcSize_wrong"], i
    assert L.FSEB200_frame_compress_device(0, 5, 0, None, 0, None, None, None, None, None) == 0
    assert L.FSEB200_frame_compress_device(1, 6, 0, *args) == 0
    assert (out == POISON).all() and (offs == 7).all() and (res == 7).all()


@pytest.mark.parametrize("call", ["decompress", "bound"])
def test_decompress_and_bound_argument_verdicts(call):
    """nFrames above 2^32 - 1, a NULL pointer while nFrames > 0, decreasing offsets: srcSize_wrong for the call and nothing
    written; nFrames == 0 returns 0"""
    L = _lib()
    frame = np.frombuffer(MAGIC["fse"] + b"\x05\xc0\x00\x00" * 2, np.uint8).copy()
    dst, caps, res = np.full(16, POISON, np.uint8), _words([8, 8]), np.full(2, 7, np.uint64)
    offs = _words([0, 8, 8])
    if call == "decompress":
        fn = L.FSEB200_frame_decompress_device
        args = [dst.ctypes.data, caps.ctypes.data, res.ctypes.data, frame.ctypes.data, offs.ctypes.data]
    else:
        fn = L.FSEB200_frame_decompress_bound_device
        args = [res.ctypes.data, frame.ctypes.data, offs.ctypes.data]
    assert fn(2 ** 32, *args, None) == ERR["srcSize_wrong"]
    for i in range(len(args)):
        bad = list(args)
        bad[i] = None
        assert fn(2, *bad, None) == ERR["srcSize_wrong"], i
    for o in ([0, 8, 7], [1, 0, 8], [0, 9, 8]):
        d = _words(o)
        assert fn(2, *args[:-1], d.ctypes.data, None) == ERR["srcSize_wrong"], o
    assert fn(0, *[None] * len(args), None) == 0
    assert fn(0, *args, None) == 0
    assert (dst == POISON).all() and (res == 7).all()


def test_python_wrappers_reject_cpu_tensors_and_wrong_dtypes():
    """the dtype is checked before the device, so a CPU tensor of the wrong dtype fails on its dtype and one of the right dtype
    on its device"""
    import torch
    import finitestateentropy_b200 as fb
    src = torch.zeros(100, dtype=torch.uint8)
    with pytest.raises(AssertionError, match="device"):
        fb.frame_compress_device(src, [50, 50])
    with pytest.raises(AssertionError, match="dtype"):
        fb.frame_compress_device(src.to(torch.int16), [50, 50])
    with pytest.raises(AssertionError, match="int32"):
        fb.frame_compress_device(src, torch.tensor([50, 50], dtype=torch.int32))
    with pytest.raises(KeyError):
        fb.frame_compress_device(src, [50, 50], codec="zlibh")
    frames = torch.zeros(16, dtype=torch.uint8)
    with pytest.raises(AssertionError, match="device"):
        fb.frame_decompress_device(frames, [0, 8, 16])
    with pytest.raises(AssertionError, match="dtype"):
        fb.frame_decompress_device(frames.to(torch.int32), [0, 8, 16])
    with pytest.raises(AssertionError, match="int32"):
        fb.frame_decompress_device(frames, torch.tensor([0, 8, 16], dtype=torch.int32))
