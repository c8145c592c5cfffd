""".fse frame calls (FSEB200_frame_{compress,decompress}_host and the Python frame_compress / frame_decompress) on the GPU
(-m gpu), checked against the reference's own command-line tool (oracle/_ref/fse_ref, compiled from the unmodified sources):

- frames byte-identical to `fse_ref -f -e/-h` at id 5 (the only id its command line writes) and to the reference
  writer's layout of the reference library's blocks at ids 0-6, over probagen inputs, mixed raw / RLE / partial inputs, sizes
  0-40 and every multiple of the block size +-1, random bytes and 256 MiB of P14; each side decodes the other's frames;
- hand-made frames (blocks coded with the compiled reference library) compared with `fse_ref -d` on the output bytes or on the
  verdict its exit code maps to: non-full interior blocks, rSize 0 of each type, compressed-type blocks with cSize == rSize and
  cSize == 1, an FSE block whose header claims more symbols than it holds, every truncation point, payload bit flips, bytes
  after the trailer; blocks past the reference's buffers (corruption_detected; the reference is never run on them);
- capacities one byte short, with canaries; pinned and pageable buffers at odd addresses; two threads at once; a child process
  at small FSEB200_HOST_PACKED_CHUNK_BYTES budgets (many chunks, a block above the budget, short FSE blocks across chunks).

Run as a script (`python tests/test_gpu_frame.py --child`) it repeats the round trips under the environment it was started with."""
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

from helpers import probagen, load_ref                                             # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(HERE)
REF = os.path.join(ROOT, "oracle", "_ref", "fse_ref")
CODEC_FLAG = {"fse": "-e", "huf": "-h"}
CODEC_ID = {"fse": 0, "huf": 1}
MAGIC = {"fse": b"\x09\x23\x3e\x18", "huf": b"\x09\x33\x3e\x18"}
ERR = {name: 2 ** 64 - code for name, code in
       (("GENERIC", 1), ("dstSize_tooSmall", 2), ("srcSize_wrong", 3), ("corruption_detected", 4))}
# the reference tool's exit code -> the verdict of FSEB200_frame_decompress_host (39: the decoder's own error, by name)
EXIT_VERDICT = {30: "srcSize_wrong", 34: "srcSize_wrong", 35: "srcSize_wrong", 36: "srcSize_wrong", 38: "srcSize_wrong",
                43: "srcSize_wrong", 31: "GENERIC", 32: "GENERIC", 44: "corruption_detected"}
POISON = 0x5A
CANARY = 64


def _need_ref():
    if not os.path.exists(REF):
        pytest.skip("fse_ref not built")


def _lib():
    import finitestateentropy_b200 as fb
    return fb.lib()


def _is_err(r):
    return r > 2 ** 64 - 10


def ref_tool(args, tmp):
    """runs fse_ref; (exit code, output bytes or None, stderr)"""
    out = os.path.join(tmp, "ref.out")
    if os.path.exists(out):
        os.remove(out)
    r = subprocess.run([REF, "-f"] + args + [out], capture_output=True, timeout=600)
    data = open(out, "rb").read() if r.returncode == 0 else None
    return r.returncode, data, r.stderr.decode(errors="replace")


def ref_frame(data, codec, bid, tmp):
    src = os.path.join(tmp, "src.bin")
    np.asarray(data, np.uint8).tofile(src)
    rc, frame, err = ref_tool([CODEC_FLAG[codec], "-B%d" % bid, src], tmp)
    assert rc == 0, err[-500:]
    return frame


def want_frame(data, codec, bid, tmp):
    """the frame the reference's writer (FIO_compressFilename) makes at block-size id `bid`: its tool's own output at id 5, the
    only id its command line writes (its -B option sets the benchmark's block size); at the other ids the same layout of the
    blocks the compiled reference library codes, with the checksum the reference tool verifies when it decodes the frame"""
    if bid == 5:
        return ref_frame(data, codec, bid, tmp)
    bs = 1024 << bid
    blocks = [coded(codec, data[i: i + bs], full=len(data) - i >= bs) for i in range(0, len(data), bs)]
    return build_frame(codec, bid, blocks, data=bytes(data))


def host(data, pinned=False, off=0):
    """data as a CPU uint8 tensor view at byte offset `off` of its allocation (pinned or pageable)"""
    import torch
    buf = torch.empty(len(data) + off + 16, dtype=torch.uint8, pin_memory=pinned)
    buf.fill_(POISON)
    v = buf[off: off + len(data)]
    if len(data):
        v.copy_(torch.from_numpy(np.frombuffer(bytes(data), np.uint8).copy()))
    return v


def frame_compress(data, codec, bid, cap=None, pinned=False, off=0):
    """(result, frame bytes, canary intact) of FSEB200_frame_compress_host at capacity cap (default: the bound)"""
    L = _lib()
    src = host(data, pinned, off)
    bound = L.FSEB200_frame_compressBound(len(data), bid)
    cap = bound if cap is None else cap
    out = host(bytes([POISON]) * (cap + CANARY), pinned, (off + 3) % 16)
    r = L.FSEB200_frame_compress_host(CODEC_ID[codec], bid, out.data_ptr(), cap, src.data_ptr() if len(data) else None, len(data))
    o = out.numpy()
    return r, (o[:r].tobytes() if not _is_err(r) else None), bool((o[cap:] == POISON).all())


def frame_decompress(frame, cap=None, pinned=False, off=0):
    """(result, output bytes, canary intact) of FSEB200_frame_decompress_host at capacity cap (default: the bound, or 1 MiB
    when the walk fails)"""
    L = _lib()
    f = host(frame, pinned, off)
    fp = f.data_ptr()
    if cap is None:
        bound = L.FSEB200_frame_decompress_bound(fp, len(frame))
        cap = 1 << 20 if _is_err(bound) else bound
    out = host(bytes([POISON]) * (cap + CANARY), pinned, (off + 5) % 16)
    r = L.FSEB200_frame_decompress_host(out.data_ptr(), cap, fp, len(frame))
    o = out.numpy()
    return r, (o[:r].tobytes() if not _is_err(r) else None), bool((o[cap:] == POISON).all())


def inputs(bid):
    rng = np.random.default_rng(100 + bid)
    bs = 1024 << bid
    yield "p20", probagen(1048575, 0.20)
    yield "p80", probagen(300000, 0.80)
    yield "p14", probagen(200000, 0.14)
    yield "mixed", np.concatenate([probagen(bs * 3, 0.14), rng.integers(0, 256, bs * 2, dtype=np.uint8),
                                   np.full(bs * 2 + 777 % bs, 7, np.uint8), probagen(5000, 0.3), np.full(3, 9, np.uint8)])
    yield "random", rng.integers(0, 256, 5 * bs + 123, dtype=np.uint8)
    for n in range(1, 41):
        yield "n%d" % n, probagen(n, 0.3)
    for k in (1, 2, 3):
        for d in (-1, 0, 1):
            yield "%dbs%+d" % (k, d), probagen(k * bs + d, 0.14)


@pytest.mark.parametrize("bid", range(7))
def test_frames_match_the_reference_tool_and_cross_decode(tmp_path, bid):
    _need_ref()
    tmp = str(tmp_path)
    for codec in ("fse", "huf"):
        for name, data in inputs(bid):
            want = want_frame(data, codec, bid, tmp)
            r, got, ok = frame_compress(data, codec, bid)
            assert ok and got == want, (codec, bid, name, r, len(want))
            r, back, ok = frame_decompress(want)                    # the reference's frame through ours
            assert ok and back == data.tobytes(), (codec, bid, name, r)
            p = os.path.join(tmp, "ours.fse")
            open(p, "wb").write(got)
            rc, out, err = ref_tool(["-d", p], tmp)                 # ours through the reference
            assert rc == 0 and out == data.tobytes(), (codec, bid, name, rc, err[-300:])
    r, got, ok = frame_compress(b"", "fse", bid)                    # the reference's tool dies on an empty input
    assert r == 8 and ok and frame_decompress(got)[:2] == (0, b"")


def test_256_mib_across_many_chunks(tmp_path):
    _need_ref()
    import finitestateentropy_b200 as fb
    import torch
    data = probagen(256 << 20, 0.14)
    for codec in ("huf", "fse"):
        want = ref_frame(data, codec, 5, str(tmp_path))
        got = fb.frame_compress(torch.from_numpy(data), codec=codec, block_size_id=5)
        assert got.numpy().tobytes() == want, codec
        back = fb.frame_decompress(got)
        assert torch.equal(back, torch.from_numpy(data)), codec


# ---- hand-made frames -------------------------------------------------------------------------------------------------------
def code_block(codec, data):
    """the compiled reference's FSE_compress / HUF_compress of one block: (value, compressed bytes)"""
    R = load_ref()
    cap = 2 * len(data) + 1024
    dst = np.zeros(cap, np.uint8)
    src = np.frombuffer(bytes(data), np.uint8).copy() if len(data) else np.zeros(1, np.uint8)
    fn = R.FSE_compress if codec == "fse" else R.HUF_compress
    v = fn(dst.ctypes.data, cap, src.ctypes.data, len(data))
    return v, (dst[:v].tobytes() if v > 1 and not _is_err(v) else b"")


def build_frame(codec, bid, blocks, data=None):
    """blocks: (type, rSize or None for full, cSize or None, payload); the trailer is the checksum of `data` (default: the
    concatenation the blocks regenerate when none decodes short)"""
    L = _lib()
    out = bytearray(MAGIC[codec] + bytes([bid]))
    regen = bytearray()
    bs = 1024 << bid
    for t, r, c, payload in blocks:
        out.append(t << 6 | (0x20 if r is None else 0))
        if r is not None:
            out += bytes([r >> 8, r & 0xFF])
        if t == 0:
            out += bytes([(len(payload) if c is None else c) >> 8, (len(payload) if c is None else c) & 0xFF])
        out += payload
        regen += payload if t == 1 else bytes(payload[:1]) * (bs if r is None else r) if t == 2 else b""
    if data is None:
        data = bytes(regen)
    buf = np.frombuffer(bytes(data) + b"\x00", np.uint8)
    crc = (L.FSEB200_XXH32(buf.ctypes.data, len(data), 0) >> 5) & 0x3FFFFF
    return bytes(out + bytes([0xC0 | crc >> 16, (crc >> 8) & 0xFF, crc & 0xFF]))


def coded(codec, data, full=False):
    """a block header tuple for `data` as the format's writer would store it"""
    v, comp = code_block(codec, data)
    r = None if full else len(data)
    if v == 0:
        return (1, r, None, bytes(data))
    if v == 1:
        return (2, r, None, bytes(data[:1]))
    return (0, r, None, comp)


def compare_with_ref(frame, tmp, what):
    """ours against `fse_ref -d` on output bytes, or on the verdict its exit code maps to"""
    p = os.path.join(tmp, "hand.fse")
    open(p, "wb").write(frame)
    rc, want, err = ref_tool(["-d", p], tmp)
    r, got, ok = frame_decompress(frame)
    assert ok, what
    if rc == 0:
        assert got == want, (what, r)
    elif rc == 39:                                                   # the decoder's error: same name
        assert _is_err(r), (what, r, err[-200:])
        name = _lib().FSE_getErrorName(r).decode()
        assert name in err, (what, name, err[-200:])
    else:
        assert rc in EXIT_VERDICT and r == ERR[EXIT_VERDICT[rc]], (what, rc, r, err[-200:])
    return rc


def hand_frames(codec):
    bs = 1024
    p = probagen(20000, 0.2)
    yield "non-full interior", build_frame(codec, 0, [coded(codec, p[:700]), coded(codec, p[700:1724], full=True),
                                                      coded(codec, p[1724:1725]), coded(codec, np.full(300, 4, np.uint8)),
                                                      coded(codec, p[2000:2900]), (1, 13, None, bytes(range(13)))])
    yield "rSize 0 raw", build_frame(codec, 0, [coded(codec, p[:500]), (1, 0, None, b""), coded(codec, p[500:900])])
    yield "rSize 0 rle", build_frame(codec, 0, [(2, 0, None, b"\x09"), coded(codec, p[:900])])
    v, comp = code_block(codec, p[:900])
    yield "rSize 0 compressed", build_frame(codec, 0, [(0, 0, None, comp)], data=b"")
    yield "cSize == rSize", build_frame(codec, 0, [(0, 300, None, bytes(p[3000:3300]))], data=bytes(p[3000:3300]))
    yield "cSize == 1", build_frame(codec, 0, [(0, 300, None, b"\x41")], data=b"\x41" * 300)
    yield "cSize == 1, rSize 1", build_frame(codec, 0, [(0, 1, None, b"\x41")], data=b"\x41")
    # a block whose header claims 100 symbols more than it holds (FSE returns the count it decoded)
    yield "short", build_frame(codec, 0, [coded(codec, p[:400]), (0, 900 + 100, None, comp), coded(codec, p[900:1300])],
                               data=bytes(p[:400]) + bytes(p[:900]) + bytes(p[900:1300]))
    good = build_frame(codec, 0, [coded(codec, p[:bs], full=True), coded(codec, p[bs:bs + 600]), (2, 40, None, b"\x05"),
                                  coded(codec, np.frombuffer(os.urandom(0) + bytes(range(256)) * 2, np.uint8))])
    yield "good", good
    yield "trailing garbage", good + b"\x00garbage\xff" * 3
    for cut in range(len(good)):
        yield "cut %d" % cut, good[:cut]
    rng = np.random.default_rng(9)
    for pos in rng.integers(5, len(good) - 3, 40):
        bad = bytearray(good)
        bad[int(pos)] ^= 1 << int(rng.integers(0, 8))
        yield "flip %d" % pos, bytes(bad)


@pytest.mark.parametrize("codec", ["fse", "huf"])
def test_hand_made_frames_match_the_reference_tool(tmp_path, codec):
    _need_ref()
    L = _lib()
    seen = set()
    for what, frame in hand_frames(codec):
        f = np.frombuffer(frame + b"\x00", np.uint8)
        if L.FSEB200_frame_decompress_bound(f.ctypes.data, len(frame)) == ERR["corruption_detected"]:
            assert frame_decompress(frame)[0] == ERR["corruption_detected"], what   # past the reference's buffers
            continue
        seen.add(compare_with_ref(frame, str(tmp_path), what))
    assert 0 in seen and 38 in seen and 44 in seen, seen


def test_fse_short_block_regenerates_what_it_decodes(tmp_path):
    """FSE_decompress returns the symbols it decoded, which may be fewer than the header's rSize; the frame carries exactly
    those bytes (and the checksum over them), in one chunk and block by block"""
    _need_ref()
    p = probagen(5000, 0.2)
    v, comp = code_block("fse", p[:900])
    frame = build_frame("fse", 0, [coded("fse", p[:1024], full=True), (0, 1000, None, comp), coded("fse", p[1024:2048], full=True)],
                        data=bytes(p[:1024]) + bytes(p[:900]) + bytes(p[1024:2048]))
    assert compare_with_ref(frame, str(tmp_path), "short") == 0
    r, out, ok = frame_decompress(frame)
    assert r == 1024 + 900 + 1024 and ok
    # the tool: it writes what the call returns
    tool = os.path.join(ROOT, "programs", "_bin", "fse_b200_file")
    fp, op = str(tmp_path / "s.fse"), str(tmp_path / "s.out")
    open(fp, "wb").write(frame)
    subprocess.run([tool, "-d", fp, op], check=True, capture_output=True, timeout=120)
    assert open(op, "rb").read() == out


def test_blocks_past_the_reference_buffers_after_coded_blocks():
    p = probagen(3000, 0.2)
    for codec in ("fse", "huf"):
        for tail in ((2, 1025, None, b"\x01"), (0, 1025, None, b"\x00\x01"), (1, 1029, None, bytes(1029))):
            frame = build_frame(codec, 0, [coded(codec, p[:1024], full=True), coded(codec, p[1024:1500]), tail])
            assert frame_decompress(frame)[0] == ERR["corruption_detected"], (codec, tail[:2])
        # ... but a decoder error before them comes first, in frame order (FSE: a tableLog of 20; Huff0: rSize 0)
        first = (0, 500, None, b"\x0f\xff\xff\xff\x00") if codec == "fse" else (0, 0, None, b"\x12\x34")
        alone = frame_decompress(build_frame(codec, 0, [first]))[0]
        assert _is_err(alone) and alone != ERR["corruption_detected"], (codec, alone)
        assert frame_decompress(build_frame(codec, 0, [first, (2, 1025, None, b"\x01")]))[0] == alone, codec


@pytest.mark.parametrize("codec", ["fse", "huf"])
def test_capacities_one_byte_short(codec):
    data = np.concatenate([probagen(100000, 0.3), np.full(5000, 1, np.uint8), np.random.default_rng(3).integers(0, 256, 7000, dtype=np.uint8)])
    r, frame, ok = frame_compress(data, codec, 4)
    assert not _is_err(r) and ok
    for cap in (8, 9, r // 2, r - 4, r - 3, r - 1):
        rr, _, ok = frame_compress(data, codec, 4, cap=cap)
        assert rr == ERR["dstSize_tooSmall"] and ok, (cap, rr)
    assert frame_compress(data, codec, 4, cap=r)[:2] == (r, frame)
    for cap in (0, 1, len(data) // 2, len(data) - 1):
        rr, _, ok = frame_decompress(frame, cap=cap)
        assert rr == ERR["dstSize_tooSmall"] and ok, (cap, rr)
    assert frame_decompress(frame, cap=len(data))[:2] == (len(data), data.tobytes())


def test_pinned_and_pageable_at_odd_addresses():
    data = np.concatenate([probagen(150001, 0.14), np.full(40000, 3, np.uint8)])
    frames = set()
    for pinned in (False, True):
        for off in (0, 1, 3, 7):
            for codec in ("fse", "huf"):
                r, frame, ok = frame_compress(data, codec, 3, pinned=pinned, off=off)
                assert ok and not _is_err(r)
                frames.add((codec, frame))
                assert frame_decompress(frame, pinned=pinned, off=off)[1:] == (data.tobytes(), True)
    assert len(frames) == 2


def test_two_threads_at_once():
    jobs = [(codec, probagen(3_000_000 + 7 * i, [0.14, 0.5, 0.8][i % 3])) for i, codec in enumerate(["fse", "huf"] * 3)]
    errors = []

    def work(codec, data):
        try:
            for _ in range(2):
                r, frame, ok = frame_compress(data, codec, 5, pinned=codec == "huf")
                assert ok and not _is_err(r)
                assert frame_decompress(frame)[1] == data.tobytes()
        except BaseException as e:                                      # reported by the main thread
            errors.append(e)
    threads = [threading.Thread(target=work, args=j) for j in jobs]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors


def test_chunk_budgets():
    """in child processes at small FSEB200_HOST_PACKED_CHUNK_BYTES budgets: many chunks, blocks above the budget"""
    _need_ref()
    for budget in (3 * (32768 + 512) + 100, 20000, 250001):
        env = dict(os.environ, FSEB200_HOST_PACKED_CHUNK_BYTES=str(budget))
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child"], env=env, capture_output=True, text=True, timeout=1200)
        assert r.returncode == 0 and "child ok" in r.stdout, (budget, r.stdout[-2000:], r.stderr[-4000:])


def _child():
    import tempfile
    tmp = tempfile.mkdtemp()
    rng = np.random.default_rng(77)
    data = np.concatenate([probagen(32768 * 9 + 5, 0.14), rng.integers(0, 256, 70000, dtype=np.uint8), np.full(50000, 2, np.uint8)])
    for codec in ("fse", "huf"):
        for bid in (0, 5, 6):
            want = want_frame(data, codec, bid, tmp)
            r, got, ok = frame_compress(data, codec, bid, pinned=bid == 5, off=1)
            assert ok and got == want, (codec, bid, r)
            assert frame_decompress(want, pinned=bid == 6, off=3)[1:] == (data.tobytes(), True), (codec, bid)
    # short FSE blocks scattered over many chunks: block by block copies at their true offsets
    p = probagen(64 * 1024, 0.2)
    blocks, regen = [], b""
    for i in range(40):
        part = p[i * 1500: i * 1500 + 1400]
        v, comp = code_block("fse", part)
        assert v > 1, i
        if i % 3 == 0:
            blocks.append((0, 1400 + 24, None, comp)); regen += bytes(part)
        else:
            blocks.append(coded("fse", part)); regen += bytes(part)
    frame = build_frame("fse", 1, blocks, data=regen)
    assert frame_decompress(frame)[1] == regen
    # a verdict with chunks still in flight, past chunk 4 at each budget of test_chunk_budgets (a 1 KB block weighs 1.5-2 KB):
    # the decoder's (block 1200 coded with tableLog 20, which FSE_readNCount rejects) and a frame capacity that runs out
    big = probagen(1600 * 1024, 0.2)
    blocks = [coded("fse", big[i: i + 1024], full=True) for i in range(0, len(big), 1024)]
    t, r, c, payload = blocks[1200]
    assert t == 0
    blocks[1200] = (t, r, c, bytes([payload[0] | 0x0F]) + payload[1:])
    assert compare_with_ref(build_frame("fse", 0, blocks, data=big), tmp, "tableLog 20 at block 1200") == 39
    for codec in ("fse", "huf"):
        r, frame, ok = frame_compress(big, codec, 0)
        assert ok and not _is_err(r), codec
        rr, _, ok = frame_compress(big, codec, 0, cap=r * 3 // 4)
        assert rr == ERR["dstSize_tooSmall"] and ok, (codec, rr)
    print("child ok")


if __name__ == "__main__" and "--child" in sys.argv:
    _child()
