"""The .fse frame calls on device memory (FSEB200_frame_{compress,decompress}_device, FSEB200_frame_decompress_bound_device)
on the GPU: every frame, offset and result equals the host batch call's (FSEB200_frame_{compress,decompress}_host_batch) byte for
byte, with the capacity rule and guard bytes around every output, frames above the device-hash threshold and the host chunk
budget, the mixed decompress batch of reference, hand-made and malformed frames, odd addresses, many frames, and ordering on a
non-default stream and from two threads."""
import os
import sys
import threading

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
from helpers import probagen                                                        # noqa: E402
from test_gpu_frame import ERR, POISON, _is_err, _lib, want_frame, _need_ref         # noqa: E402
from test_gpu_frame_batch import (CODEC_ID, GUARD, batch_compress, batch_decompress, data_for, mixed_frames,  # noqa: E402
                                  sizes_for)

pytestmark = pytest.mark.gpu


def _torch():
    import torch
    return torch


def dev(data, off=0):
    """data on the device at `off` bytes past a 256-byte aligned start; (the view, the whole buffer)"""
    torch = _torch()
    b = np.frombuffer(bytes(data), np.uint8)
    buf = torch.full((len(b) + off + 64,), POISON, dtype=torch.uint8, device="cuda")
    if len(b):
        buf[off: off + len(b)] = torch.from_numpy(b.copy()).cuda()
    return buf[off: off + len(b)], buf


def device_compress(datas, codec, bid, cap=None, off=0, stream=None):
    """(results, offsets, out bytes, guard bytes intact) of one FSEB200_frame_compress_device call"""
    torch = _torch()
    L = _lib()
    sizes = np.array([len(d) for d in datas], np.uint64)
    src, _ = dev(b"".join(bytes(d) for d in datas), off)
    need = sum(L.FSEB200_frame_compressBound(len(d), bid) for d in datas)
    cap = need if cap is None else cap
    out = torch.full((cap + 2 * GUARD + 16,), POISON, dtype=torch.uint8, device="cuda")
    o0 = GUARD + (off + 3) % 16
    offs = torch.full((len(datas) + 1,), -1, dtype=torch.int64, device="cuda")
    res = torch.full((len(datas),), -1, dtype=torch.int64, device="cuda")
    s = stream or torch.cuda.current_stream()
    torch.cuda.current_stream().synchronize()                      # the buffers above were filled on the current stream
    r = L.FSEB200_frame_compress_device(CODEC_ID[codec], bid, len(datas), out.data_ptr() + o0, cap, offs.data_ptr(), res.data_ptr(),
                                        src.data_ptr() if src.numel() else None, sizes.ctypes.data, s.cuda_stream)
    assert r == 0, r
    s.synchronize()
    o = out.cpu().numpy()
    u = lambda t: [int(x) % (1 << 64) for x in t.cpu().tolist()]                  # noqa: E731
    return u(res), u(offs), o[o0: o0 + cap].tobytes(), bool((o[:o0] == POISON).all() and (o[o0 + cap:] == POISON).all())


def device_decompress(frames, caps, off=0):
    """(results, outputs per frame, every byte outside the frames' regions untouched), laid out as batch_decompress lays out the
    host call: every frame is followed by an empty one whose region is GUARD guard bytes.  Inside a region, bytes past the
    result are unspecified (a frame decodes its blocks where their headers put them before moving them down)"""
    torch = _torch()
    L = _lib()
    n = len(frames)
    blob, _ = dev(b"".join(frames) + b"\x00" * 32, off)
    ends = np.cumsum([len(f) for f in frames]).astype(np.uint64)
    offs = np.zeros(2 * n + 1, np.uint64)
    offs[1::2], offs[2::2] = ends, ends
    slots = np.zeros(2 * n, np.uint64)
    slots[0::2], slots[1::2] = caps, GUARD
    o0 = GUARD + (off + 5) % 16
    out = torch.full((int(slots.sum()) + 2 * GUARD + 16,), POISON, dtype=torch.uint8, device="cuda")
    res = torch.zeros(2 * n, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream()
    r = L.FSEB200_frame_decompress_device(2 * n, out.data_ptr() + o0, slots.ctypes.data, res.data_ptr(), blob.data_ptr(), offs.ctypes.data,
                                          s.cuda_stream)
    assert r == 0, r
    s.synchronize()
    res = [int(x) % (1 << 64) for x in res.cpu().tolist()]
    assert all(x == ERR["srcSize_wrong"] for x in res[1::2])
    o = out.cpu().numpy()
    starts = o0 + np.concatenate([[0], np.cumsum(slots)[:-1]])[0::2].astype(np.int64)
    results = res[0::2]
    mask = np.ones(len(o), bool)
    for f, v in enumerate(results):
        st = int(starts[f])
        mask[st: st + caps[f]] = False
    outs = [None if _is_err(v) else o[int(starts[f]): int(starts[f]) + v].tobytes() for f, v in enumerate(results)]
    return results, outs, bool((o[mask] == POISON).all())


@pytest.mark.parametrize("bid", [0, 3, 5, 6])
def test_compress_equals_the_host_batch(bid):
    rng = np.random.default_rng(20 + bid)
    for codec in ("fse", "huf"):
        datas = [data_for(n, i, rng) for i, n in enumerate(sizes_for(bid, rng) + [0, 2 * (1024 << bid)])]
        want = batch_compress(datas, codec, bid)
        got = device_compress(datas, codec, bid, off=bid)
        assert want[3] and got[3]
        assert got[0] == want[0] and got[1] == want[1], (codec, bid)
        assert got[2][:want[1][-1]] == want[2][:want[1][-1]], (codec, bid)


def test_compress_sample_equals_the_reference_tool(tmp_path):
    _need_ref()
    rng = np.random.default_rng(6)
    for codec in ("fse", "huf"):
        for bid in (0, 5, 6):
            datas = [probagen(70000, 0.2), rng.integers(0, 256, 5000, dtype=np.uint8), np.full(3000, 9, np.uint8)]
            res, offs, out, ok = device_compress(datas, codec, bid, off=1)
            assert ok
            for f, d in enumerate(datas):
                assert out[offs[f]: offs[f + 1]] == want_frame(d, codec, bid, str(tmp_path)), (codec, bid, f)


def test_capacity_at_every_frame_end():
    """outCapacity at every frame's end, one byte below it, and 0: the frames that end past it are dstSize_tooSmall and none of
    their bytes, nor any guard byte, is written; the offsets stay the full prefix sums"""
    rng = np.random.default_rng(3)
    datas = [data_for(n, i, rng) for i, n in enumerate([5000, 0, 1, 40000, 70000, 7, 33000])]
    for codec in ("fse", "huf"):
        res, offs, full, ok = device_compress(datas, codec, 4)
        assert ok and not any(_is_err(r) for r in res)
        for cap in sorted({0} | {e for o in offs[1:] for e in (o, o - 1)}):
            want = batch_compress(datas, codec, 4, cap=cap)
            r2, o2, out, ok2 = device_compress(datas, codec, 4, cap=cap, off=cap % 7)
            assert ok2 and r2 == want[0] and o2 == offs, (codec, cap)
            for f in range(len(datas)):
                piece = out[offs[f]: min(offs[f + 1], cap)]
                if offs[f + 1] <= cap:
                    assert piece == full[offs[f]: offs[f + 1]], (codec, cap, f)
                else:
                    assert set(piece) <= {POISON}, (codec, cap, f)


def test_large_frames():
    """frames of 2 MiB, 64 MiB and 300 MiB -- above the 1 MiB device-hash threshold and the 64 MiB host chunk budget of the host
    calls -- equal the host call's frames and round-trip"""
    torch = _torch()
    import finitestateentropy_b200 as fb
    sizes = [2 << 20, 64 << 20, 300 << 20]
    data = probagen(sum(sizes), 0.3)
    for codec in ("fse", "huf"):
        want, woffs, wres = fb.frame_compress_batch(torch.from_numpy(data), sizes, codec=codec)
        src = torch.from_numpy(data).cuda()
        out, offs, res = fb.frame_compress_device(src, sizes, codec=codec)
        torch.cuda.synchronize()
        assert offs.cpu().tolist() == woffs.tolist() and res.cpu().tolist() == wres.tolist(), codec
        assert torch.equal(out[: int(woffs[-1])].cpu(), want), codec
        back, r = fb.frame_decompress_device(out, offs.cpu())
        torch.cuda.synchronize()
        assert r.cpu().tolist() == sizes and torch.equal(back, src), codec
        del out, back


def test_decompress_mixed_batch_equals_the_host_batch(tmp_path):
    pairs = mixed_frames(str(tmp_path))
    frames, caps = [f for f, _ in pairs], [c for _, c in pairs]
    want, wouts, wok = batch_decompress(frames, caps)
    assert wok and len(set(want)) > 4
    for off in (0, 3):
        got, outs, ok = device_decompress(frames, caps, off=off)
        assert ok, off
        assert got == want, off
        assert outs == wouts, off


def test_bound_equals_the_host_bound(tmp_path):
    L = _lib()
    torch = _torch()
    frames = [f for f, _ in mixed_frames(str(tmp_path))] + [b"", b"\x09\x23"]
    blob, _ = dev(b"".join(frames) + b"\x00" * 32, 1)
    offs = np.concatenate([[0], np.cumsum([len(f) for f in frames])]).astype(np.uint64)
    got = np.zeros(len(frames), np.uint64)
    assert L.FSEB200_frame_decompress_bound_device(len(frames), got.ctypes.data, blob.data_ptr(), offs.ctypes.data,
                                                   torch.cuda.current_stream().cuda_stream) == 0
    for f, fr in enumerate(frames):
        b = np.frombuffer(fr + b"\x00", np.uint8)
        assert int(got[f]) == L.FSEB200_frame_decompress_bound(b.ctypes.data if fr else None, len(fr)), f


def test_odd_addresses_round_trip():
    rng = np.random.default_rng(8)
    datas = [data_for(n, i, rng) for i, n in enumerate([100, 0, 33000, 70001, 5])]
    for codec in ("fse", "huf"):
        want = device_compress(datas, codec, 5)
        for off in (1, 3, 7, 13):
            got = device_compress(datas, codec, 5, off=off)
            assert got == want, (codec, off)
            frames = [got[2][got[1][f]: got[1][f + 1]] for f in range(len(datas))]
            r, outs, ok = device_decompress(frames, [len(d) for d in datas], off=off)
            assert ok and r == [len(d) for d in datas] and outs == [bytes(d) for d in datas], (codec, off)


def test_ten_thousand_tiny_frames_and_a_gib_of_64_kib_frames():
    torch = _torch()
    import finitestateentropy_b200 as fb
    rng = np.random.default_rng(9)
    sizes = [int(x) for x in rng.integers(0, 300, 10000)]
    data = probagen(sum(sizes), 0.3)
    for codec in ("fse", "huf"):
        src = torch.from_numpy(data).cuda()
        out, offs, res = fb.frame_compress_device(src, sizes, codec=codec, block_size_id=0)
        want, woffs, wres = fb.frame_compress_batch(torch.from_numpy(data), sizes, codec=codec, block_size_id=0)
        assert offs.cpu().tolist() == woffs.tolist() and torch.equal(out[: int(woffs[-1])].cpu(), want)
        back, r = fb.frame_decompress_device(out, offs.cpu(), capacities=sizes)
        assert r.cpu().tolist() == sizes and torch.equal(back, src), codec
    n = 16384
    big = torch.from_numpy(probagen(1 << 26, 0.14)).cuda().repeat(n >> 10)
    for codec in ("huf", "fse"):
        out, offs, res = fb.frame_compress_device(big, [1 << 16] * n, codec=codec)
        back, r = fb.frame_decompress_device(out, offs.cpu(), capacities=[1 << 16] * n)
        assert bool((r == (1 << 16)).all()) and torch.equal(back, big), codec
        del out, back


def test_stream_ordering_and_two_threads():
    """the source made by a torch op on a non-default stream right before the compress, the frames decoded and compared on that
    stream after it, with no synchronisation in between; then two host threads on two streams at once"""
    torch = _torch()
    import finitestateentropy_b200 as fb
    base = torch.from_numpy(probagen(3 << 20, 0.2)).cuda()
    sizes = [1 << 20, 5000, (1 << 20) + 3, 0, 900000]
    want = fb.frame_compress_batch(base[: sum(sizes)].cpu() ^ 0x11, sizes, codec="fse")
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(st):
        src = base[: sum(sizes)] ^ 0x11                             # queued on st: the compress must wait for it
        out, offs, res = fb.frame_compress_device(src, sizes, codec="fse")
        head = out[: int(want[1][-1])].clone()                      # on st, after the compress
        back, r = fb.frame_decompress_device(out, want[1], capacities=sizes)
        same = torch.equal(back, src)
    st.synchronize()
    assert torch.equal(head.cpu(), want[0]) and offs.cpu().tolist() == want[1].tolist() and same
    assert r.cpu().tolist() == sizes

    errors = []

    def work(i):
        try:
            s = torch.cuda.Stream()
            codec = ("fse", "huf")[i % 2]
            datas = [probagen(40000 + 977 * j + i, 0.2 + 0.1 * (j % 5)) for j in range(30)]
            w = batch_compress(datas, codec, 5)
            for _ in range(3):
                got = device_compress(datas, codec, 5, off=i, stream=s)
                assert got[:3] == w[:3]
        except BaseException as e:                                  # reported by the main thread
            errors.append(e)
    threads = [threading.Thread(target=work, args=(i,)) for i in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors


def test_short_blocks_move_down_across_settle_tiles():
    """frames of about 700 blocks whose FSE blocks at 0, 300 and 650 decode 100 bytes short, so every later block moves down in
    place -- across the settle kernel's 256-block tiles -- or, at capacities between the true and the nominal size, is copied in
    from scratch; capacities at the true size, one byte below, between, at and past the nominal size.  Results, bytes and the
    guard bytes around every region equal the host batch call's."""
    from test_gpu_frame import build_frame, code_block, coded
    rng = np.random.default_rng(12)
    p = probagen(1 << 20, 0.3)
    blocks, data = [], bytearray()
    for i in range(700):
        chunk = p[1024 * i: 1024 * (i + 1)]
        if i in (0, 300, 650):                                     # rSize 1000, FSE bytes of 900: decodes 900
            v, comp = code_block("fse", chunk[:900])
            blocks.append((0, 1000, None, comp))
            data += bytes(chunk[:900])
        elif i % 7 == 3:
            blocks.append((1, None, None, bytes(rng.integers(0, 256, 1024, dtype=np.uint8))))
            data += blocks[-1][3]
        elif i % 11 == 5:
            blocks.append((2, 200, None, b"\x07"))
            data += b"\x07" * 200
        else:
            blocks.append(coded("fse", chunk, full=True))
            data += bytes(chunk)
    frame = build_frame("fse", 0, blocks, data=bytes(data))
    true = len(data)
    nominal = true + 300
    caps = [true, true - 1, true + 150, nominal - 1, nominal, nominal + 77]
    frames = [frame] * len(caps)
    want, wouts, wok = batch_decompress(frames, caps)
    assert wok and want == [true, ERR["dstSize_tooSmall"]] + [true] * 4, want
    for off in (0, 5):
        got, outs, ok = device_decompress(frames, caps, off=off)
        assert ok and got == want and outs == wouts, off


def test_all_empty_frames_through_the_wrapper():
    """a batch of empty frames (every frame 0 bytes) gets the batch wrapper's per-frame verdicts"""
    torch = _torch()
    import finitestateentropy_b200 as fb
    frames = torch.zeros(0, dtype=torch.uint8)
    want_out, want = fb.frame_decompress_batch(frames, [0, 0, 0])
    out, res = fb.frame_decompress_device(frames.cuda(), [0, 0, 0])
    assert res.cpu().tolist() == want.tolist() and out.numel() == want_out.numel() == 0
