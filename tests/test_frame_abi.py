"""CPU-side checks of the .fse frame calls (FSEB200_frame_*): the header declares them and the library exports them; the argument
verdicts; the structural verdicts the header walk settles before any device work (magic, block-size id, truncation, blocks past
the reference's buffers), against the reference CLI's exit codes where it is built; FSEB200_frame_compressBound against the
all-raw frame; and the library's XXH32 against the trailers the reference CLI writes."""
import os
import re
import subprocess

import numpy as np
import pytest

from helpers import declared_arity

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "fse_ref")
NEW_CALLS = {"FSEB200_frame_compressBound": 2, "FSEB200_frame_compress_host": 6,
             "FSEB200_frame_decompress_bound": 2, "FSEB200_frame_decompress_host": 4}
ERR = {name: 2 ** 64 - code for name, code in
       (("GENERIC", 1), ("dstSize_tooSmall", 2), ("srcSize_wrong", 3), ("corruption_detected", 4))}
MAGIC = {"fse": b"\x09\x23\x3e\x18", "huf": b"\x09\x33\x3e\x18", "zlibh": b"\x09\x43\x3e\x18"}
# the reference tool's exit code -> the frame call's verdict (fileio.c:495-606)
EXIT_VERDICT = {30: "srcSize_wrong", 34: "srcSize_wrong", 35: "srcSize_wrong", 36: "srcSize_wrong", 38: "srcSize_wrong",
                43: "srcSize_wrong", 31: "GENERIC", 32: "GENERIC", 44: "corruption_detected"}


def _lib():
    import finitestateentropy_b200 as fb
    return fb.lib()


def test_header_declares_the_frame_calls():
    decl = declared_arity()
    assert {n: decl.get(n) for n in NEW_CALLS} == NEW_CALLS


def test_library_exports_the_frame_calls():
    from finitestateentropy_b200 import _build
    path = _build.build_lib()
    exported = subprocess.check_output(["nm", "-D", "--defined-only", path]).decode()
    for name in list(NEW_CALLS) + ["FSEB200_XXH32"]:
        assert re.search(r" T %s$" % name, exported, flags=re.M), name


def _buf(n, fill=0x5A):
    return np.full(n, fill, np.uint8)


def test_compress_argument_verdicts():
    """bad codec, id above 6, NULL pointers with sizes above 0: srcSize_wrong; a capacity below 8: dstSize_tooSmall; nothing
    written in either case"""
    L = _lib()
    src, out = _buf(100, 1), _buf(64)
    s, o = src.ctypes.data, out.ctypes.data
    for codec in (-1, 2, 7):
        assert L.FSEB200_frame_compress_host(codec, 5, o, 64, s, 100) == ERR["srcSize_wrong"]
    for bid in (7, 8, 255, 2 ** 31):
        assert L.FSEB200_frame_compress_host(0, bid, o, 64, s, 100) == ERR["srcSize_wrong"]
        assert L.FSEB200_frame_compressBound(100, bid) == ERR["srcSize_wrong"]
    assert L.FSEB200_frame_compress_host(0, 5, o, 64, None, 100) == ERR["srcSize_wrong"]
    assert L.FSEB200_frame_compress_host(1, 5, None, 64, s, 100) == ERR["srcSize_wrong"]
    for cap in range(8):
        assert L.FSEB200_frame_compress_host(0, 5, o, cap, s, 100) == ERR["dstSize_tooSmall"]
    assert L.FSEB200_frame_compress_host(0, 5, None, 0, s, 100) == ERR["dstSize_tooSmall"]
    assert (out == 0x5A).all()


@pytest.mark.parametrize("codec", ["fse", "huf"])
def test_empty_input_is_header_and_trailer(codec):
    """no block, no device work: magic, id, and the checksum of nothing (XXH32 of no bytes, seed 0, is 0x02CC5D05)"""
    L = _lib()
    out = _buf(16)
    for bid in range(7):
        r = L.FSEB200_frame_compress_host(0 if codec == "fse" else 1, bid, out.ctypes.data, 8, None, 0)
        assert r == 8
        crc = (0x02CC5D05 >> 5) & 0x3FFFFF
        assert out[:8].tobytes() == MAGIC[codec] + bytes([bid, 0xC0 | crc >> 16, (crc >> 8) & 0xFF, crc & 0xFF])
        assert (out[8:] == 0x5A).all()
        assert L.FSEB200_frame_decompress_bound(out.ctypes.data, 8) == 0
        dst = _buf(4)
        assert L.FSEB200_frame_decompress_host(dst.ctypes.data, 0, out.ctypes.data, 8) == 0
        assert (dst == 0x5A).all()
    assert L.FSEB200_XXH32(None, 0, 0) == 0x02CC5D05


def test_compress_bound_is_the_all_raw_frame():
    """at every id, for sizes of 0 to 3 blocks plus every residue: 8 bytes of frame, 1 + block per full block and 3 + n for the
    partial one -- what a raw block takes, and at least what a compressed (n - 2 bytes at most, 5 of header) or RLE block takes"""
    L = _lib()
    for bid in range(7):
        bs = 1024 << bid
        n = np.arange(0, 4 * bs + 1, dtype=np.int64)
        full, r = n // bs, n % bs
        raw = 8 + full * (1 + bs) + np.where(r > 0, 3 + r, 0)
        worst_coded = 8 + full * (3 + bs - 2) + np.where(r > 1, 5 + r - 2, np.where(r > 0, 3 + r, 0))
        got = np.array([L.FSEB200_frame_compressBound(int(x), bid) for x in n], dtype=np.int64)
        assert np.array_equal(got, raw), bid
        assert (got >= worst_coded).all(), bid


def _frame(codec, bid, blocks, trailer=b"\xc0\x00\x00"):
    """a hand-made frame: blocks are (type, rSize or None for full, cSize or None, payload bytes)"""
    out = bytearray(MAGIC[codec] + bytes([bid]))
    for t, r, c, payload in blocks:
        out.append(t << 6 | (0x20 if r is None else 0))
        if r is not None:
            out += bytes([r >> 8, r & 0xFF])
        if t == 0:
            out += bytes([c >> 8, c & 0xFF])
        out += payload
    return bytes(out + trailer)


def _stored_frames():
    """frames of raw and RLE blocks only, valid and not: every verdict is settled by the header walk"""
    raw = bytes(range(200))
    good = _frame("fse", 0, [(1, 200, None, raw), (2, 1000, None, b"\x07"), (1, None, None, bytes(1024)), (2, 0, None, b"\x01")])
    yield "good", good
    for cut in range(len(good)):
        yield "cut%d" % cut, good[:cut]
    yield "magic", b"\x00\x23\x3e\x18\x05\xc0\x00\x00"
    yield "zlibh", MAGIC["zlibh"] + b"\x05\xc0\x00\x00"
    yield "id7", MAGIC["huf"] + b"\x07\xc0\x00\x00"
    yield "id255", MAGIC["fse"] + b"\xff\xc0\x00\x00"


def _verdicts(frame, cap):
    L = _lib()
    f = np.frombuffer(frame + b"\x00", np.uint8)                   # a non-NULL pointer also for the empty frame
    dst = _buf(cap + 64)
    bound = L.FSEB200_frame_decompress_bound(f.ctypes.data, len(frame))
    r = L.FSEB200_frame_decompress_host(dst.ctypes.data, cap, f.ctypes.data, len(frame))
    assert (dst[cap:] == 0x5A).all()
    return bound, r


def test_structural_verdicts_of_stored_frames():
    """magic, id and every truncation point of a frame of raw and RLE blocks: the walk's verdict from both calls, without
    device work (the trailer of `good` is deliberately wrong, so only the checksum step needs the device)"""
    L = _lib()
    for name, frame in _stored_frames():
        if name == "good":
            f = np.frombuffer(frame, np.uint8)
            assert L.FSEB200_frame_decompress_bound(f.ctypes.data, len(frame)) == 200 + 1000 + 1024
            continue
        bound, r = _verdicts(frame, 4096)
        want = ERR["GENERIC"] if name in ("magic", "zlibh", "id7", "id255") else ERR["srcSize_wrong"]
        assert bound == want and r == want, (name, bound, r)
    # a truncation after a valid block with a too-small capacity: frame order puts the capacity first
    good = dict(_stored_frames())["good"]
    assert _verdicts(good[:-2], 2223)[1] == ERR["dstSize_tooSmall"]
    assert _verdicts(good[:-2], 2224)[1] == ERR["srcSize_wrong"]


@pytest.mark.skipif(not os.path.exists(REF), reason="fse_ref not built")
def test_structural_verdicts_match_the_reference_tool(tmp_path):
    """the reference CLI (on the CPU) stops on the same frames with the exit codes the verdicts map from (it decodes zlibh
    frames, which the library refuses as an unknown magic number)"""
    for name, frame in _stored_frames():
        if name in ("good", "zlibh"):
            continue
        p = tmp_path / ("%s.fse" % name)
        p.write_bytes(frame)
        rc = subprocess.run([REF, "-f", "-d", str(p), str(tmp_path / "o")], capture_output=True, timeout=60).returncode
        assert ERR[EXIT_VERDICT[rc]] == _verdicts(frame, 4096)[1], (name, rc)


def test_blocks_past_the_reference_buffers_are_corruption():
    """rSize above the block size for a compressed or RLE block, a payload longer than block + 4: corruption_detected from the
    walk, before any device work (the reference's tool overruns its buffers on these, fileio.c:509-510)"""
    bs = 1024
    for blocks in ([(2, bs + 1, None, b"\x01")],
                   [(0, bs + 1, 10, bytes(10))],
                   [(1, bs + 5, None, bytes(bs + 5))],
                   [(0, 100, bs + 5, bytes(bs + 5))],
                   [(1, 10, None, bytes(10)), (2, 2000, None, b"\x01")]):
        frame = _frame("fse", 0, blocks)
        bound, r = _verdicts(frame, 1 << 16)
        assert bound == r == ERR["corruption_detected"], blocks[-1][:3]
    # a raw block up to block + 4 bytes is what the reference accepts: the bound counts it
    assert _verdicts(_frame("fse", 0, [(1, bs + 4, None, bytes(bs + 4))]), 0)[0] == bs + 4


def test_decompress_argument_verdicts():
    L = _lib()
    f = np.frombuffer(MAGIC["fse"] + b"\x05\xc0\x00\x00", np.uint8)
    dst = _buf(8)
    assert L.FSEB200_frame_decompress_host(dst.ctypes.data, 8, None, 8) == ERR["srcSize_wrong"]
    assert L.FSEB200_frame_decompress_host(None, 8, f.ctypes.data, 8) == ERR["srcSize_wrong"]
    assert L.FSEB200_frame_decompress_bound(None, 8) == ERR["srcSize_wrong"]
    assert L.FSEB200_frame_decompress_bound(None, 0) == ERR["srcSize_wrong"]
    assert L.FSEB200_frame_decompress_host(None, 0, None, 0) == ERR["srcSize_wrong"]


@pytest.mark.skipif(not os.path.exists(REF), reason="fse_ref not built")
def test_xxh32_matches_the_reference_trailers(tmp_path):
    """the 22 trailer bits the reference CLI writes equal (FSEB200_XXH32(data, 0) >> 5), over lengths around the 16-byte stripe
    and larger inputs"""
    L = _lib()
    rng = np.random.default_rng(5)
    for n in list(range(1, 70)) + [1000, 4096, 100003]:
        data = rng.integers(0, 256, n, dtype=np.uint8)
        src, dst = tmp_path / "in.bin", tmp_path / "in.fse"
        data.tofile(src)
        subprocess.run([REF, "-f", "-e", str(src), str(dst)], check=True, capture_output=True, timeout=60)
        t = dst.read_bytes()[-3:]
        want = (t[0] & 0x3F) << 16 | t[1] << 8 | t[2]
        assert (L.FSEB200_XXH32(data.ctypes.data, n, 0) >> 5) & 0x3FFFFF == want, n


def test_python_wrappers_check_their_arguments():
    import torch
    import finitestateentropy_b200 as fb
    with pytest.raises(KeyError):
        fb.frame_compress(torch.zeros(10, dtype=torch.uint8), codec="zlibh")
    with pytest.raises(RuntimeError):
        fb.frame_compress(torch.zeros(10, dtype=torch.uint8), block_size_id=7)
    with pytest.raises(AssertionError):
        fb.frame_compress(torch.zeros(10, dtype=torch.int32))
    with pytest.raises(RuntimeError, match="GENERIC"):
        fb.frame_decompress(torch.frombuffer(bytearray(MAGIC["zlibh"] + b"\x05\xc0\x00\x00"), dtype=torch.uint8))
    assert fb.frame_compress(torch.zeros(0, dtype=torch.uint8), codec="huf").numel() == 8
