"""CPU-side checks of the .fse frame batch calls (FSEB200_frame_{compress,decompress}_host_batch): declarations and exports,
the argument verdicts, batches that need no device work (empty frames, frames the header walk rejects) against the one-frame
calls, and the Python wrappers' argument checks."""
import os
import re
import subprocess

import numpy as np
import pytest

from helpers import declared_arity
from test_frame_abi import _frame, _stored_frames, ERR, MAGIC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BATCH_CALLS = {"FSEB200_frame_compress_host_batch": 9, "FSEB200_frame_decompress_host_batch": 6}
POISON = 0x5A


def _lib():
    import finitestateentropy_b200 as fb
    return fb.lib()


def _words(values):
    return np.array(values, dtype=np.uint64)


def test_header_declares_and_library_exports_the_batch_calls():
    decl = declared_arity()
    assert {n: decl.get(n) for n in BATCH_CALLS} == BATCH_CALLS
    from finitestateentropy_b200 import _build
    exported = subprocess.check_output(["nm", "-D", "--defined-only", _build.build_lib()]).decode()
    for name in BATCH_CALLS:
        assert re.search(r" T %s$" % name, exported, flags=re.M), name


def test_compress_argument_verdicts():
    """bad codec, id above 6, nFrames above 2^32 - 1, a NULL pointer while nFrames > 0: srcSize_wrong and nothing written;
    nFrames == 0 returns 0 and writes nothing, even with NULL pointers"""
    L = _lib()
    src, out = np.full(100, 1, np.uint8), np.full(64, POISON, np.uint8)
    sizes, offs, res = _words([60, 40]), np.full(3, 7, np.uint64), np.full(2, 7, np.uint64)
    args = [out.ctypes.data, 64, offs.ctypes.data, res.ctypes.data, src.ctypes.data, sizes.ctypes.data]
    for codec in (-1, 2, 7):
        assert L.FSEB200_frame_compress_host_batch(codec, 5, 2, *args) == ERR["srcSize_wrong"]
    for bid in (7, 255, 2 ** 31):
        assert L.FSEB200_frame_compress_host_batch(0, bid, 2, *args) == ERR["srcSize_wrong"]
    assert L.FSEB200_frame_compress_host_batch(0, 5, 2 ** 32, *args) == ERR["srcSize_wrong"]
    for i in (0, 2, 3, 4, 5):
        bad = list(args)
        bad[i] = None
        assert L.FSEB200_frame_compress_host_batch(1, 5, 2, *bad) == ERR["srcSize_wrong"], i
    assert L.FSEB200_frame_compress_host_batch(0, 5, 0, None, 0, None, None, None, None) == 0
    assert L.FSEB200_frame_compress_host_batch(0, 5, 0, *args) == 0
    assert (out == POISON).all() and (offs == 7).all() and (res == 7).all()


@pytest.mark.parametrize("codec", ["fse", "huf"])
def test_empty_frames_need_no_device(codec):
    """frames of 0 bytes with a NULL source: 8-byte frames equal to the one-frame call's, the capacity rule on each, and the
    decompress of the batch -- all without device work"""
    L = _lib()
    cid = 0 if codec == "fse" else 1
    for bid in (0, 5, 6):
        one = np.full(16, POISON, np.uint8)
        assert L.FSEB200_frame_compress_host(cid, bid, one.ctypes.data, 16, None, 0) == 8
        sizes, offs, res = _words([0] * 4), np.zeros(5, np.uint64), np.zeros(4, np.uint64)
        out = np.full(32 + 16, POISON, np.uint8)
        for cap, stored in ((32, 4), (31, 3), (8, 1), (7, 0)):
            out[:] = POISON
            r = L.FSEB200_frame_compress_host_batch(cid, bid, 4, out.ctypes.data, cap, offs.ctypes.data, res.ctypes.data, None,
                                                    sizes.ctypes.data)
            assert r == 0
            assert offs.tolist() == [0, 8, 16, 24, 32]
            assert res.tolist() == [8] * stored + [ERR["dstSize_tooSmall"]] * (4 - stored)
            assert out[:8 * stored].tobytes() == one[:8].tobytes() * stored and (out[8 * stored:] == POISON).all(), cap
        frames = np.concatenate([one[:8]] * 3)
        dst, caps, res = np.full(8, POISON, np.uint8), _words([0, 5, 0]), np.zeros(3, np.uint64)
        fo = _words([0, 8, 16, 24])
        assert L.FSEB200_frame_decompress_host_batch(3, dst.ctypes.data, caps.ctypes.data, res.ctypes.data, frames.ctypes.data,
                                                     fo.ctypes.data) == 0
        assert res.tolist() == [0, 0, 0] and (dst == POISON).all()


def test_decompress_argument_verdicts():
    """nFrames above 2^32 - 1, a NULL pointer while nFrames > 0, decreasing offsets: srcSize_wrong for the call and nothing
    written; nFrames == 0 returns 0"""
    L = _lib()
    frame = np.frombuffer(MAGIC["fse"] + b"\x05\xc0\x00\x00" * 2, np.uint8).copy()
    dst, caps, res = np.full(16, POISON, np.uint8), _words([8, 8]), np.full(2, 7, np.uint64)
    offs = _words([0, 8, 8])
    args = [dst.ctypes.data, caps.ctypes.data, res.ctypes.data, frame.ctypes.data, offs.ctypes.data]
    assert L.FSEB200_frame_decompress_host_batch(2 ** 32, *args) == ERR["srcSize_wrong"]
    for i in range(5):
        bad = list(args)
        bad[i] = None
        assert L.FSEB200_frame_decompress_host_batch(2, *bad) == ERR["srcSize_wrong"], i
    for o in ([0, 8, 7], [1, 0, 8], [0, 9, 8]):
        d = _words(o)
        assert L.FSEB200_frame_decompress_host_batch(2, *args[:4], d.ctypes.data) == ERR["srcSize_wrong"], o
    assert L.FSEB200_frame_decompress_host_batch(0, None, None, None, None, None) == 0
    assert (dst == POISON).all() and (res == 7).all()


def _single(frame, cap):
    L = _lib()
    f = np.frombuffer(frame + b"\x00", np.uint8)
    dst = np.full(cap + 1, POISON, np.uint8)
    return L.FSEB200_frame_decompress_host(dst.ctypes.data if cap else None, cap, f.ctypes.data if frame else None, len(frame))


def test_walk_rejected_frames_get_their_single_call_verdicts():
    """a batch of frames the header walk settles (truncations at every point, unknown magic, zlibh, ids 7 and 255, a capacity
    below the stored blocks' sizes): each gets exactly the one-frame call's verdict, no device work runs, and no byte of the
    output is written"""
    L = _lib()
    frames = [f for name, f in _stored_frames() if name != "good"]
    good = dict(_stored_frames())["good"]
    frames += [good[:-2], good[:-1]]
    caps = [4096] * (len(frames) - 2) + [2223, 2224]
    frames += [good]
    caps += [100]                                                   # below the 2224 bytes its blocks regenerate
    want = [_single(f, c) for f, c in zip(frames, caps)]
    assert all(w in (ERR["srcSize_wrong"], ERR["GENERIC"], ERR["dstSize_tooSmall"]) for w in want), want
    blob = np.frombuffer(b"".join(frames) + b"\x00", np.uint8)
    offs = _words(np.concatenate([[0], np.cumsum([len(f) for f in frames])]))
    total = sum(caps)
    dst = np.full(total + 64, POISON, np.uint8)
    res = np.zeros(len(frames), np.uint64)
    c = _words(caps)
    assert L.FSEB200_frame_decompress_host_batch(len(frames), dst.ctypes.data, c.ctypes.data, res.ctypes.data, blob.ctypes.data,
                                                 offs.ctypes.data) == 0
    assert res.tolist() == want
    assert (dst == POISON).all()


def test_python_wrappers_check_their_arguments():
    import torch
    import finitestateentropy_b200 as fb
    src = torch.zeros(100, dtype=torch.uint8)
    with pytest.raises(KeyError):
        fb.frame_compress_batch(src, [50, 50], codec="zlibh")
    with pytest.raises(AssertionError):
        fb.frame_compress_batch(src, [50, 50], block_size_id=7)
    with pytest.raises(AssertionError):
        fb.frame_compress_batch(src, [60, 50])                      # more bytes than src holds
    with pytest.raises(AssertionError):
        fb.frame_compress_batch(src.to(torch.int16), [50, 50])
    with pytest.raises(AssertionError):
        fb.frame_compress_batch(src, [-1, 50])                      # a negative size would reach C as a huge size_t
    frames, offsets, results = fb.frame_compress_batch(src, [])
    assert frames.numel() == 0 and offsets.tolist() == [0] and results.numel() == 0
    frames, offsets, results = fb.frame_compress_batch(src, [0, 0, 0], codec="huf", block_size_id=2)
    assert offsets.tolist() == [0, 8, 16, 24] and results.tolist() == [8, 8, 8]
    assert frames[:4].numpy().tobytes() == MAGIC["huf"] and frames[4] == 2
    with pytest.raises(AssertionError):
        fb.frame_decompress_batch(frames, [0, 16, 8, 24])           # decreasing
    with pytest.raises(AssertionError):
        fb.frame_decompress_batch(frames, [0, 8, 16, 25])           # past the frames
    with pytest.raises(AssertionError):
        fb.frame_decompress_batch(frames, offsets, capacities=[0, 0])
    out, res = fb.frame_decompress_batch(frames, offsets)
    assert out.numel() == 0 and res.tolist() == [0, 0, 0]
    bad = torch.from_numpy(np.frombuffer(_frame("fse", 7, []), np.uint8).copy())
    out, res = fb.frame_decompress_batch(bad, [0, bad.numel()])
    assert res.tolist() == [ERR["GENERIC"] - 2 ** 64]                 # int64: the error code's two's complement
