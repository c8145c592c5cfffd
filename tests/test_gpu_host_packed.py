"""Packed host-buffer calls (FSEB200_compress_host_packed / FSEB200_decompress_host_packed) on the GPU (-m gpu), for FSE, Huff0
4X, Huff0 1X and FSE-U16, against the device packed calls on the same blocks: offsets, values and the whole output capacity
byte for byte (both buffers poisoned alike), sentinels around hOut and hDst untouched, the decompress results equal to the
device packed decompress's, and every stored block regenerated from the stream alone.  Layouts: uniform 32 KB blocks, ragged
blocks from 0 to the codec's maximum, all-raw and all-RLE batches; capacities 0, one byte below a block's end, at it, and the
total; pinned and pageable tensors at odd host offsets; two host threads at once.  The Huff0 values are also checked against
the compiled reference.

Run as a script (`python tests/test_gpu_host_packed.py --child`) it repeats the round trips under the environment it was
started with: test_chunk_budgets starts it with small FSEB200_HOST_PACKED_CHUNK_BYTES budgets."""
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

from helpers import gen_u16, is_error                                             # noqa: E402
from packed_paths import ref_values                                               # noqa: E402
from test_gpu_blocks import POISON, CANARY, content, _ref, _u64, _dev64           # noqa: E402

pytestmark = pytest.mark.gpu

CODECS = ["fse", "huf", "huf1x", "fseu16"]
UNIT = {"fse": 1, "huf": 1, "huf1x": 1, "fseu16": 2}
MAX_BLOCK = {"fse": 1 << 18, "huf": 1 << 17, "huf1x": 1 << 17, "fseu16": 1 << 17}   # symbols; a 2^30-byte FSE block: test_gpu_fse_large.py
UNIT_MSV = {"fse": 255, "huf": 255, "huf1x": 255, "fseu16": 0}                  # the Python calls' default maxSymbolValue
BLOCK_OVERHEAD = 512                                                              # what a block adds to a chunk's weight


def blocks(codec, kind, seed, count=48):
    """(source bytes, sizes in symbols) of a batch: "uniform" 32 KB blocks, "ragged" 0 .. the codec's maximum, "raw" (random
    content; U16 symbols below 287 -- a U16 block is never raw, its symbols hold at most log2(287) bits of 16), "rle"."""
    rng = np.random.default_rng(seed)
    u = UNIT[codec]
    if kind == "uniform":
        sizes = [32768 // u] * count
    elif kind == "ragged":
        sizes = [0, 1, 2, MAX_BLOCK[codec], 0] + [int(x) for x in rng.integers(0, MAX_BLOCK[codec] + 1, count - 5)]
    else:
        sizes = [int(x) for x in rng.integers(64, 40000 // u, count)]
    parts = []
    for i, n in enumerate(sizes):
        if kind == "raw":
            parts.append(rng.integers(0, 256, n, dtype=np.uint8) if u == 1 else rng.integers(0, 287, n, dtype=np.uint16).view(np.uint8))
        elif kind == "rle":
            parts.append(np.full(n, (i * 37) & 0xFF, np.uint8) if u == 1 else np.full(n, 1 + i % 286, np.uint16).view(np.uint8))
        elif u == 2:
            parts.append(gen_u16(n, 240, [0.1, 0.5, 0.9][i % 3], seed + i).view(np.uint8) if i % 7 else
                         rng.integers(0, 65536, n, dtype=np.uint16).view(np.uint8))
        else:
            parts.append(content(rng, n, i))
    return np.concatenate(parts + [np.zeros(0, np.uint8)]), sizes


def device_compress(codec, data, sizes, cap):
    """the device packed call on the blocks back to back at an even address, into a poisoned buffer of `cap` bytes:
    (offsets, values, output bytes)"""
    import torch
    import finitestateentropy_b200 as fb
    u = UNIT[codec]
    L = fb.lib()
    src = torch.from_numpy(np.concatenate([data, np.zeros(64, np.uint8)])).cuda()
    starts = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64) * u
    sp, sn = _dev64([src.data_ptr() + int(s) for s in starts]), _dev64(sizes)
    arena = torch.full((cap + 2 * CANARY,), POISON, dtype=torch.uint8, device="cuda")
    offsets = torch.empty(len(sizes) + 1, dtype=torch.int64, device="cuda")
    cs = torch.empty(len(sizes), dtype=torch.int64, device="cuda")
    args = (len(sizes), arena.data_ptr() + CANARY, cap, offsets.data_ptr(), cs.data_ptr(), sp.data_ptr(), sn.data_ptr())
    stream = torch.cuda.current_stream().cuda_stream
    if codec in ("fse", "fseu16"):
        work = torch.empty(fb.fse_packed_workspace(len(sizes), u * sum(sizes)), dtype=torch.uint8, device="cuda")
        fn = L.FSEB200_FSEU16_compress_packed if codec == "fseu16" else L.FSEB200_FSE_compress_packed
        r = fn(*args, UNIT_MSV[codec], 12, work.data_ptr(), work.numel(), stream)
    else:
        fn = L.FSEB200_HUF_compress1X_packed if codec == "huf1x" else L.FSEB200_HUF_compress_packed
        r = fn(*args, UNIT_MSV[codec], 12, stream)
    assert r == 0, r
    torch.cuda.synchronize()
    a = arena.cpu().numpy()
    assert bool((a[:CANARY] == POISON).all()) and bool((a[CANARY + cap:] == POISON).all())
    return _u64(offsets), _u64(cs), a[CANARY: CANARY + cap]


def device_decompress(codec, packed, offsets, sizes):
    import torch
    import finitestateentropy_b200 as fb
    u = UNIT[codec]
    dev = torch.from_numpy(np.concatenate([packed, np.zeros(64, np.uint8)])).cuda()
    dst = torch.empty(u * sum(sizes) + 64, dtype=torch.uint8, device="cuda")
    starts = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64) * u
    fn = {"fse": fb.fse_decompress_packed, "fseu16": fb.fseu16_decompress_packed,
          "huf": fb.huf_decompress_packed, "huf1x": fb.huf_decompress1x_packed}[codec]
    res = fn(dev, torch.from_numpy(offsets.view(np.int64).copy()).cuda(), _dev64([dst.data_ptr() + int(s) for s in starts]), _dev64(sizes))
    torch.cuda.synchronize()
    return _u64(res)


def host_buffer(n, pinned, off, fill=POISON):
    """a CPU uint8 view of n bytes at host offset `off` inside CANARY sentinel bytes on each side: (arena, view)"""
    import torch
    arena = torch.full((n + off + 2 * CANARY,), fill, dtype=torch.uint8)
    if pinned:
        arena = arena.pin_memory()
    return arena, arena[CANARY + off: CANARY + off + n]


def host_round_trip(codec, data, sizes, cap=None, pinned=False, off=1, want=None):
    """compress on host memory against the device call at `cap`, then (for the full capacity) decompress against the device's
    results and the source.  Returns (packed bytes, offsets, values), or None when the stream does not fit `cap`."""
    import torch
    import finitestateentropy_b200 as fb
    u = UNIT[codec]
    total_src = u * sum(sizes)
    cap = total_src + 32 if cap is None else cap
    want_offs, want_cs, want_out = device_compress(codec, data, sizes, cap) if want is None else want
    sarena, src = host_buffer(len(data), pinned, off + 2)
    src.copy_(torch.from_numpy(data))
    oarena, out = host_buffer(cap, pinned, off)
    _, offsets, cs = fb.host_compress_packed(src, sizes, codec, out=out)
    got_offs, got_cs = offsets.numpy().view(np.uint64), cs.numpy().view(np.uint64)
    assert np.array_equal(got_offs, want_offs), (codec, cap)
    bad = [(b, int(got_cs[b]), int(want_cs[b])) for b in range(len(sizes)) if got_cs[b] != want_cs[b]]
    assert not bad, (codec, cap, bad[:8])
    o = oarena.numpy()
    assert np.array_equal(o[CANARY + off: CANARY + off + cap], want_out), (codec, cap)
    assert bool((o[:CANARY + off] == POISON).all()) and bool((o[CANARY + off + cap:] == POISON).all()), "sentinels around hOut"
    assert np.array_equal(src.numpy(), data)
    total = int(got_offs[-1])
    if total > cap:
        return None
    # decompress from a buffer that ends exactly at the stream's end, without the original
    packed = o[CANARY + off: CANARY + off + total].copy()
    iarena, inp = host_buffer(total, pinned, off + 4)
    inp.copy_(torch.from_numpy(packed))
    darena, dst = host_buffer(total_src, pinned, off)
    _, res = fb.host_decompress_packed(inp, offsets, sizes, codec, out=dst)
    want_res = device_decompress(codec, packed, got_offs, sizes)
    r = res.numpy().view(np.uint64)
    assert np.array_equal(r, want_res), (codec, [(b, int(r[b]), int(want_res[b])) for b in range(len(sizes)) if r[b] != want_res[b]][:8])
    d = darena.numpy()
    assert bool((d[:CANARY + off] == POISON).all()) and bool((d[CANARY + off + total_src:] == POISON).all()), "sentinels around hDst"
    start = 0
    for b, n in enumerate(sizes):
        if not is_error(int(got_cs[b])) and not is_error(int(r[b])):
            assert int(r[b]) == n, (codec, b, n, int(r[b]))
            assert np.array_equal(d[CANARY + off + start: CANARY + off + start + u * n], data[start: start + u * n]), (codec, b)
        elif not is_error(int(got_cs[b])):
            assert codec in ("huf", "huf1x"), (codec, b)                # only the reference's weight-12 exception
        start += u * n
    return packed, got_offs, got_cs


# ---- tests ----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("codec", CODECS)
@pytest.mark.parametrize("kind", ["uniform", "ragged", "raw", "rle"])
def test_round_trip(codec, kind):
    data, sizes = blocks(codec, kind, seed=801 + CODECS.index(codec))
    _, _, cs = host_round_trip(codec, data, sizes, pinned=kind in ("uniform", "raw"), off=1 if kind != "rle" else 3)
    if kind == "raw" and codec != "fseu16":
        assert all(int(v) == 0 for v in cs)
    if kind == "rle":
        assert all(int(v) == 1 for v in cs)


@pytest.mark.parametrize("codec", CODECS)
def test_capacities(codec):
    """outCapacity 0, one byte below a block's end, exactly at it, and at the total: values, offsets and bytes as the device's"""
    data, sizes = blocks(codec, "ragged", seed=811 + CODECS.index(codec), count=24)
    want = device_compress(codec, data, sizes, UNIT[codec] * sum(sizes) + 32)
    offs = want[0]
    mid = next(b for b in range(len(sizes) // 2, len(sizes)) if offs[b + 1] > offs[b] + 1)
    end = int(offs[mid + 1])
    for cap in (0, end - 1, end, int(offs[-1])):
        w = device_compress(codec, data, sizes, cap)
        host_round_trip(codec, data, sizes, cap=cap, pinned=cap % 2 == 0, off=5, want=w)


def test_huf_values_match_the_reference():
    lib = _ref()
    for codec in ("huf", "huf1x"):
        data, sizes = blocks(codec, "ragged", seed=821, count=40)
        _, _, cs = host_round_trip(codec, data, sizes)
        starts = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        vals, _ = ref_values(lib, [data[starts[b]: starts[b + 1]] for b in range(len(sizes))], 255, 12, codec == "huf1x")
        assert [int(v) for v in cs] == vals


def test_two_threads():
    """two host threads call the packed pair on different data at once: both give what one thread alone gives -- the device
    packed decompress's results, every block regenerated but for the reference's weight-12 exception"""
    import torch
    import finitestateentropy_b200 as fb
    jobs = [("huf", blocks("huf", "uniform", 831, 200)), ("fse", blocks("fse", "ragged", 832, 60))]
    alone = {}
    for codec, (data, sizes) in jobs:
        out, offsets, cs = fb.host_compress_packed(torch.from_numpy(data), sizes, codec)
        dst, res = fb.host_decompress_packed(out, offsets, sizes, codec)
        alone[codec] = (out, offsets, cs, res)
        want = device_decompress(codec, out[: int(offsets[-1])].numpy(), offsets.numpy().view(np.uint64), sizes)
        assert np.array_equal(res.numpy().view(np.uint64), want), codec
        assert codec == "huf" or res.tolist() == sizes
    errors = []

    def work(codec, data, sizes):
        try:
            for _ in range(3):
                out, offsets, cs = fb.host_compress_packed(torch.from_numpy(data), sizes, codec)
                dst, res = fb.host_decompress_packed(out, offsets, sizes, codec)
                w = alone[codec]
                assert torch.equal(offsets, w[1]) and torch.equal(cs, w[2]) and torch.equal(res, w[3]), codec
                assert torch.equal(out[: int(offsets[-1])], w[0][: int(offsets[-1])]), codec
                start = 0
                for n, x in zip(sizes, res.tolist()):
                    assert x != n or np.array_equal(dst.numpy()[start: start + n], data[start: start + n]), codec
                    start += n
        except BaseException as e:                                      # reported by the main thread
            errors.append(e)
    threads = [threading.Thread(target=work, args=(c, d, s)) for c, (d, s) in jobs]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors


def test_chunk_budgets():
    """in child processes at small FSEB200_HOST_PACKED_CHUNK_BYTES budgets: block edges before, at and after chunk edges, and
    blocks larger than the budget"""
    _ref()
    for budget in (3 * (32768 + BLOCK_OVERHEAD), 100000, 300001):
        env = dict(os.environ, FSEB200_HOST_PACKED_CHUNK_BYTES=str(budget))
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child"], env=env, capture_output=True, text=True, timeout=1200)
        assert r.returncode == 0 and "child ok" in r.stdout, (budget, r.stdout[-2000:], r.stderr[-4000:])


def _child():
    import torch
    budget = int(os.environ["FSEB200_HOST_PACKED_CHUNK_BYTES"])
    for codec in CODECS:
        u = UNIT[codec]
        data, sizes = blocks(codec, "uniform", seed=841, count=20)           # 32 KB blocks: at budget 3 * 33,280 an edge per 3
        host_round_trip(codec, data, sizes, pinned=True, off=1)
        # edges before, at and after the budget, and a block of 2.5 budgets
        cut = budget // 3 - BLOCK_OVERHEAD
        sz = [cut, cut, budget - 2 * (cut + BLOCK_OVERHEAD) - BLOCK_OVERHEAD, cut + 1, cut - 1, 5, (5 * budget) // 2, 0, cut]
        sz = [max(0, s) // u for s in sz]
        data, _ = blocks(codec, "ragged", seed=842, count=len(sz))
        rng = np.random.default_rng(843)
        parts = [data[:u * n] if u * n <= len(data) else rng.integers(0, 256, u * n, dtype=np.uint8) for n in sz]
        host_round_trip(codec, np.concatenate(parts), sz, pinned=False, off=7)
        data, sizes = blocks(codec, "ragged", seed=844, count=30)
        host_round_trip(codec, data, sizes, cap=u * sum(sizes) // 3, pinned=True, off=3)
        torch.cuda.empty_cache()
    print("child ok")


if __name__ == "__main__" and "--child" in sys.argv:
    _child()
