"""The .fse frame batch calls on the GPU (FSEB200_frame_{compress,decompress}_host_batch): every frame of a batch equals the
one-frame call's frame and verdict, byte for byte, with the capacity rule, guard bytes around every output, the device checksum
kernel at lengths around its stripe and tile sizes and on both sides of the host-hash threshold, many frames per chunk and
frames across chunks, odd buffer addresses, two threads, and the file tool's -m mode against the reference CLI."""
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
from helpers import probagen                                                        # noqa: E402
from test_gpu_frame import (REF, ERR, POISON, _is_err, _lib, _need_ref, build_frame, code_block, coded, hand_frames, host,  # noqa: E402
                            ref_frame, ref_tool, want_frame)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(HERE)
CODEC_ID = {"fse": 0, "huf": 1}
GUARD = 32
DEVICE_HASH_MAX = 1 << 20                                           # host_pipeline.cu: longer frames are hashed on the host


def single_compress(data, codec, bid):
    L = _lib()
    src = host(data)
    cap = L.FSEB200_frame_compressBound(len(data), bid)
    out = host(bytes(cap))
    r = L.FSEB200_frame_compress_host(CODEC_ID[codec], bid, out.data_ptr(), cap, src.data_ptr() if len(data) else None, len(data))
    assert not _is_err(r), r
    return out.numpy()[:r].tobytes()


def single_decompress(frame, cap):
    L = _lib()
    f = host(frame)
    out = host(bytes(cap))
    r = L.FSEB200_frame_decompress_host(out.data_ptr() if cap else None, cap, f.data_ptr() if len(frame) else None, len(frame))
    return r, (out.numpy()[:r].tobytes() if not _is_err(r) else None)


def batch_compress(datas, codec, bid, cap=None, pinned=False, off=0):
    """(results, offsets, out bytes, guard bytes intact) of one batch call on the frames `datas`"""
    L = _lib()
    sizes = np.array([len(d) for d in datas], np.uint64)
    src = host(b"".join(bytes(d) for d in datas), pinned, off)
    need = sum(L.FSEB200_frame_compressBound(len(d), bid) for d in datas)
    cap = need if cap is None else cap
    out = host(bytes([POISON]) * (cap + 2 * GUARD), pinned, (off + 3) % 16)
    offs = np.zeros(len(datas) + 1, np.uint64)
    res = np.zeros(len(datas), np.uint64)
    r = L.FSEB200_frame_compress_host_batch(CODEC_ID[codec], bid, len(datas), out.data_ptr() + GUARD, cap, offs.ctypes.data,
                                            res.ctypes.data, src.data_ptr() if src.numel() else None, sizes.ctypes.data)
    assert r == 0, r
    o = out.numpy()
    return [int(x) for x in res], [int(x) for x in offs], o[GUARD: GUARD + cap].tobytes(), bool((o[:GUARD] == POISON).all() and (o[GUARD + cap:] == POISON).all())


def batch_decompress(frames, caps, pinned=False, off=0):
    """(results, outputs per frame, every byte outside the successful outputs untouched) of one batch call.  Every frame is
    followed by an empty one (srcSize_wrong from the header walk, which writes nothing) whose region is GUARD guard bytes, so a
    write past a region's capacity shows."""
    L = _lib()
    n = len(frames)
    blob = host(b"".join(frames) + b"\x00", pinned, off)
    ends = np.cumsum([len(f) for f in frames]).astype(np.uint64)
    offs = np.zeros(2 * n + 1, np.uint64)
    offs[1::2], offs[2::2] = ends, ends
    slots = np.zeros(2 * n, np.uint64)
    slots[0::2], slots[1::2] = caps, GUARD
    out = host(bytes([POISON]) * (int(slots.sum()) + GUARD), pinned, (off + 5) % 16)
    res = np.zeros(2 * n, np.uint64)
    r = L.FSEB200_frame_decompress_host_batch(2 * n, out.data_ptr() + GUARD, slots.ctypes.data, res.ctypes.data, blob.data_ptr(),
                                              offs.ctypes.data)
    assert r == 0, r
    assert all(int(x) == ERR["srcSize_wrong"] for x in res[1::2])
    o = out.numpy()
    starts = GUARD + np.concatenate([[0], np.cumsum(slots)[:-1]])[0::2].astype(np.int64)
    results = [int(x) for x in res[0::2]]
    mask = np.ones(len(o), bool)
    for f, v in enumerate(results):
        s = int(starts[f])
        mask[s: s + (caps[f] if _is_err(v) else v)] = False          # a failed frame's region is unspecified
    outs = [None if _is_err(v) else o[int(starts[f]): int(starts[f]) + v].tobytes() for f, v in enumerate(results)]
    return results, outs, bool((o[mask] == POISON).all())


def sizes_for(bid, rng):
    bs = 1024 << bid
    s = [0, 1, 15, 16, 17, bs - 1, bs, bs + 1, 3 * bs, 1000]
    s += [int(x) for x in rng.integers(0, 3 << 20, 4)]
    return s


def data_for(n, i, rng):
    kind = i % 4
    if kind == 0:
        return probagen(n, 0.14)
    if kind == 1:
        return probagen(n, 0.8)
    if kind == 2:
        return rng.integers(0, 256, n, dtype=np.uint8)
    return np.full(n, 7, np.uint8)


@pytest.mark.parametrize("bid", [0, 3, 5, 6])
def test_compress_equals_the_single_call(bid):
    rng = np.random.default_rng(10 + bid)
    for codec in ("fse", "huf"):
        datas = [data_for(n, i, rng) for i, n in enumerate(sizes_for(bid, rng))]
        want = [single_compress(d, codec, bid) for d in datas]
        res, offs, out, ok = batch_compress(datas, codec, bid)
        assert ok and res == [len(w) for w in want], (codec, bid)
        assert offs == [0] + list(np.cumsum([len(w) for w in want])), (codec, bid)
        for f, w in enumerate(want):
            assert out[offs[f]: offs[f + 1]] == w, (codec, bid, f)
        # one byte short of the total: the last frame fits nowhere, the offsets stay, nothing else is written
        res2, offs2, out2, ok2 = batch_compress(datas, codec, bid, cap=offs[-1] - 1)
        assert ok2 and offs2 == offs and res2 == res[:-1] + [ERR["dstSize_tooSmall"]], (codec, bid)
        assert out2[:offs[-2]] == out[:offs[-2]] and set(out2[offs[-2]:]) <= {POISON}
        # a capacity in the middle: frames that end past it are dstSize_tooSmall and nothing of them is written
        mid = offs[len(offs) // 2] + 3
        res3, offs3, out3, ok3 = batch_compress(datas, codec, bid, cap=mid)
        assert ok3 and offs3 == offs
        for f in range(len(datas)):
            assert res3[f] == (res[f] if offs[f + 1] <= mid else ERR["dstSize_tooSmall"]), (codec, bid, f)
        last = max(offs[f + 1] for f in range(len(datas)) if offs[f + 1] <= mid)
        assert out3[:last] == out[:last] and set(out3[last:]) <= {POISON}


def test_compress_sample_equals_the_reference_tool(tmp_path):
    _need_ref()
    rng = np.random.default_rng(5)
    for codec in ("fse", "huf"):
        for bid in (0, 5, 6):
            datas = [probagen(70000, 0.2), rng.integers(0, 256, 5000, dtype=np.uint8), probagen(1 << bid << 10, 0.5)]
            res, offs, out, ok = batch_compress(datas, codec, bid)
            for f, d in enumerate(datas):
                assert out[offs[f]: offs[f + 1]] == want_frame(d, codec, bid, str(tmp_path)), (codec, bid, f)


def mixed_frames(tmp):
    """(frame, capacity) pairs: ours, the reference tool's, hand-made frames of both codecs, capacities one byte short"""
    p = probagen(300000, 0.3)
    out = []
    for codec in ("fse", "huf"):
        ours = single_compress(p[:150000], codec, 4)
        out += [(ours, 150000), (ours, 149999)]
        if os.path.exists(REF):
            out.append((ref_frame(p[1000:90000], codec, 5, tmp), 89000))
        for what, frame in hand_frames(codec):
            out.append((frame, 1 << 15))
    v, comp = code_block("fse", p[:900])
    out.append((build_frame("fse", 0, [coded("fse", p[:1024], full=True), (0, 1000, None, comp), (2, 30, None, b"\x03")],
                            data=bytes(p[:1024]) + bytes(p[:900]) + b"\x03" * 30), 4096))
    out.append((build_frame("fse", 0, [(1, 10, None, bytes(range(10))), (2, 1024, None, b"\x05")]), 1033))   # overrun, stored
    out.append((b"\x09\x43\x3e\x18\x05\xc0\x00\x00", 100))                                                 # zlibh
    out.append((b"\x00\x23\x3e\x18\x05\xc0\x00\x00", 100))                                                 # magic
    return out


def test_decompress_mixed_batch_equals_the_single_call(tmp_path):
    pairs = mixed_frames(str(tmp_path))
    frames, caps = [f for f, _ in pairs], [c for _, c in pairs]
    want = [single_decompress(f, c) for f, c in pairs]
    assert len({r for r, _ in want}) > 4
    res, outs, ok = batch_decompress(frames, caps)
    assert ok
    for f, (r, data) in enumerate(want):
        assert res[f] == r and outs[f] == data, f
    # pinned, odd addresses: the same
    assert batch_decompress(frames, caps, pinned=True, off=3)[:2] == (res, outs)


def test_checksums_around_stripes_tiles_and_the_threshold():
    """frames of 0-70 bytes and around the kernel's 992-byte round, device-hashed, and just below and above the host-hash
    threshold: every trailer is FSEB200_XXH32's; the decompress checks them back"""
    L = _lib()
    rng = np.random.default_rng(1)
    lens = list(range(71)) + [991, 992, 993, 1007, 1008, 1009, 1983, 1984, 1985, 5000, 65536 + 13]
    for codec in ("fse", "huf"):
        datas = [rng.integers(0, 256, n, dtype=np.uint8) if n % 2 else probagen(n, 0.3) for n in lens]
        datas += [probagen(DEVICE_HASH_MAX, 0.5), probagen(DEVICE_HASH_MAX + 1, 0.5)]
        res, offs, out, ok = batch_compress(datas, codec, 2, off=1)
        assert ok
        for f, d in enumerate(datas):
            fr = out[offs[f]: offs[f + 1]]
            buf = np.frombuffer(bytes(d) + b"\x00", np.uint8)
            crc = (L.FSEB200_XXH32(buf.ctypes.data, len(d), 0) >> 5) & 0x3FFFFF
            assert fr[-3:] == bytes([0xC0 | crc >> 16, (crc >> 8) & 0xFF, crc & 0xFF]), (codec, f, len(d))
        frames = [out[offs[f]: offs[f + 1]] for f in range(len(datas))]
        r2, outs, ok = batch_decompress(frames, [len(d) for d in datas], off=7)
        assert ok and r2 == [len(d) for d in datas] and outs == [bytes(d) for d in datas], codec
        # a wrong trailer on every frame: corruption_detected on each
        bad = [fr[:-1] + bytes([fr[-1] ^ 1]) for fr in frames]
        assert batch_decompress(bad, [len(d) for d in datas])[0] == [ERR["corruption_detected"]] * len(datas)


def test_ten_thousand_tiny_frames_and_two_threads():
    rng = np.random.default_rng(2)
    sizes = [int(x) for x in rng.integers(0, 300, 10000)]
    datas = [probagen(n, 0.3) for n in sizes]
    for codec in ("fse", "huf"):
        res, offs, out, ok = batch_compress(datas, codec, 0, pinned=True, off=5)
        assert ok and not any(_is_err(r) for r in res)
        for f in range(0, 10000, 997):
            assert out[offs[f]: offs[f + 1]] == single_compress(datas[f], codec, 0), f
        r2, outs, ok = batch_decompress([out[offs[f]: offs[f + 1]] for f in range(10000)], sizes, pinned=False, off=1)
        assert ok and r2 == sizes and outs == [bytes(d) for d in datas]
    errors = []

    def work(i):
        try:
            codec = ("fse", "huf")[i % 2]
            ds = [probagen(50000 + 1000 * j + i, 0.2 + 0.1 * (j % 5)) for j in range(40)]
            for _ in range(2):
                res, offs, out, ok = batch_compress(ds, codec, 5, pinned=i % 2 == 0)
                assert ok and [out[offs[f]: offs[f + 1]] for f in range(3)] == [single_compress(d, codec, 5) for d in ds[:3]]
                r2, outs, ok = batch_decompress([out[offs[f]: offs[f + 1]] for f in range(len(ds))], [len(d) for d in ds])
                assert ok and outs == [bytes(d) for d in ds]
        except BaseException as e:                                  # reported by the main thread
            errors.append(e)
    threads = [threading.Thread(target=work, args=(i,)) for i in range(4)]
    threads.append(threading.Thread(target=lambda: [single_compress(probagen(3_000_000, 0.3), "fse", 5) for _ in range(3)]))
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors


def test_python_wrappers_round_trip():
    import torch
    import finitestateentropy_b200 as fb
    sizes = [0, 5, 70000, 1 << 20, 33]
    src = torch.from_numpy(probagen(sum(sizes), 0.2))
    for codec in ("fse", "huf"):
        frames, offsets, results = fb.frame_compress_batch(src, sizes, codec=codec, block_size_id=4)
        at = 0
        for f, n in enumerate(sizes):
            one = fb.frame_compress(src[at: at + n], codec=codec, block_size_id=4)
            assert torch.equal(frames[int(offsets[f]): int(offsets[f + 1])], one) and int(results[f]) == one.numel()
            at += n
        out, res = fb.frame_decompress_batch(frames, offsets)
        assert res.tolist() == sizes and torch.equal(out, src)


def test_chunk_budgets():
    """in child processes at small FSEB200_HOST_PACKED_CHUNK_BYTES budgets: frames across chunk boundaries, many frames per
    chunk, frames above the budget among small ones"""
    for budget in (20000, 3 * (32768 + 512) + 100, 1 << 20):
        env = dict(os.environ, FSEB200_HOST_PACKED_CHUNK_BYTES=str(budget))
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child"], env=env, capture_output=True, text=True, timeout=1200)
        assert r.returncode == 0 and "child ok" in r.stdout, (budget, r.stdout[-2000:], r.stderr[-4000:])


def _child():
    rng = np.random.default_rng(77)
    sizes = [100, 0, 7000, 300000, 16, 40000, 1 << 20, 5, 2 << 20, 90000] + [int(x) for x in rng.integers(0, 5000, 50)]
    datas = [data_for(n, i, rng) for i, n in enumerate(sizes)]
    for codec in ("fse", "huf"):
        for bid in (0, 5):
            want = [single_compress(d, codec, bid) for d in datas]
            res, offs, out, ok = batch_compress(datas, codec, bid, off=1)
            assert ok and [out[offs[f]: offs[f + 1]] for f in range(len(datas))] == want, (codec, bid)
            res2, _, out2, ok2 = batch_compress(datas, codec, bid, cap=offs[-1] - 1)
            assert ok2 and res2[-1] == ERR["dstSize_tooSmall"] and out2[:offs[-2]] == out[:offs[-2]]
            mid = offs[7] - 1                                       # the 1 MiB frame spans chunks and does not fit
            res3, _, out3, ok3 = batch_compress(datas, codec, bid, cap=mid)
            assert ok3 and res3[6] == ERR["dstSize_tooSmall"] and out3[:offs[6]] == out[:offs[6]] and set(out3[offs[6]:]) <= {POISON}
            r2, outs, ok = batch_decompress(want, sizes, pinned=True, off=3)
            assert ok and r2 == sizes and outs == [bytes(d) for d in datas], (codec, bid)
            r3, _, ok = batch_decompress(want, [max(n - 1, 0) for n in sizes])
            assert ok and r3 == [ERR["dstSize_tooSmall"] if n else 0 for n in sizes]
    print("child ok")


def test_file_tool_many_files(tmp_path):
    _need_ref()
    tool = os.path.join(ROOT, "programs", "_bin", "fse_b200_file")
    rng = np.random.default_rng(4)
    datas = [probagen(100000, 0.2), rng.integers(0, 256, 3000, dtype=np.uint8), probagen(40000, 0.7), np.full(1, 3, np.uint8)]
    for codec, flag in (("fse", "-e"), ("huf", "-h")):
        names = []
        for i, d in enumerate(datas):
            p = str(tmp_path / ("%s%d.bin" % (codec, i)))
            d.tofile(p)
            names.append(p)
        subprocess.run([tool, "-m", flag] + names, check=True, capture_output=True, timeout=300)
        for p, d in zip(names, datas):
            got = open(p + ".fse", "rb").read()
            assert got == ref_frame(d, codec, 5, str(tmp_path)), p
            rc, back, err = ref_tool(["-d", p + ".fse"], str(tmp_path))
            assert rc == 0 and back == d.tobytes(), (p, err[-300:])
            os.remove(p)
        subprocess.run([tool, "-d", "-m"] + [p + ".fse" for p in names], check=True, capture_output=True, timeout=300)
        for p, d in zip(names, datas):
            assert open(p, "rb").read() == d.tobytes(), p


if __name__ == "__main__" and "--child" in sys.argv:
    _child()
