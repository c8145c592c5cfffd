"""Single-stream per-block descriptor calls (FSEB200_HUF_compress1X_blocks / FSEB200_HUF_decompress1X_blocks) against the
compiled reference's HUF_compress1X / HUF_decompress1X_DCtx, block by block (-m gpu): ragged sizes, sources anywhere
(overlapping too), every capacity and parameter verdict, packed compressed inputs and outputs at odd offsets, malformed
blocks, the head decode at every residue, a batch of two pass-A rounds, the decoder's row budgets and the calls' own argument
checks.  The block contents and layouts are those of tests/test_gpu_blocks.py (imported).

Run as a script (`python tests/test_gpu_blocks_1x.py --child`) it repeats subsets of the ragged tests under the environment it
was started with: test_knobs_1x starts it with FSEB200_HUFD_ROWS / _ROWS_B set."""
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from helpers import is_error, probagen, ptr                                       # noqa: E402
from blocks_paths import plan_histogram, HUF_BLOCK_MAX                           # noqa: E402
from blocks1x_paths import decode_paths_1x, summarize, stream_kind, pass_a_spread_1x, emit_group_1x   # noqa: E402
from test_gpu_blocks import (POISON, CANARY, ERR_SRC_WRONG, SPECIAL_SIZES, content, ragged_sources, hbound,   # noqa: E402
                             _ref, _u64, _dev64)

pytestmark = pytest.mark.gpu

DTABLE_X2_MAX = 12 * 0x01000001                     # HUF_CREATE_STATIC_DTABLEX2(dctx, HUF_TABLELOG_MAX) header


# ---- reference side ---------------------------------------------------------------------------------------------------------

def ref_compress1x(lib, host, offs, sizes, caps, msv, tl):
    """HUF_compress1X per block on the host: (values, compressed bytes); a capacity above the bound runs at the bound"""
    vals, outs = [], []
    for o, n, cap in zip(offs, sizes, caps):
        c = min(cap, hbound(n))
        buf = np.zeros(c + 8, np.uint8)
        src = np.ascontiguousarray(host[o: o + n])
        v = lib.HUF_compress1X(ptr(buf), c, ptr(src), n, msv, tl)
        vals.append(v)
        outs.append(buf[: v] if (not is_error(v) and v >= 1) else buf[:0])
    return vals, outs


def ref_decode1x(lib, blocks, csizes, dsizes):
    """expected (value, bytes) per block: HUF_decompress1X_DCtx on a fresh X2-sized table, and this library's documented
    srcSize_wrong for dstSize > 128 KB; also the number of blocks only the double-symbol decoder accepts"""
    vals, outs, x2_only = [], [], 0
    for c, k, n in zip(blocks, csizes, dsizes):
        if n > HUF_BLOCK_MAX:
            vals.append(ERR_SRC_WRONG); outs.append(None); continue
        tmp = np.concatenate([c, np.zeros(64, np.uint8)])
        o = np.zeros(n + 64, np.uint8)
        dt = np.zeros(1 + 4096, np.uint32)
        dt[0] = DTABLE_X2_MAX
        v = lib.HUF_decompress1X_DCtx(ptr(dt), ptr(o), n, ptr(tmp), k)
        if not is_error(v) and 1 < k < n:
            o2 = np.zeros(n + 64, np.uint8)
            x2_only += bool(is_error(lib.HUF_decompress1X1(ptr(o2), n, ptr(tmp), k)))
        vals.append(v); outs.append(None if is_error(v) else o[:n].copy())
    return vals, outs, x2_only


def capacities_1x(rng, sizes, ref_at_bound):
    """0, 1, 7, 8, 9 (around the one stream's 8-byte rule), 16, 17, result - 1, 2^40, the bound"""
    caps = []
    for i, (n, r) in enumerate(zip(sizes, ref_at_bound)):
        k = i % 11
        fixed = {1: 0, 2: 1, 3: 7, 4: 8, 5: 9, 6: 16, 7: 17, 9: 2 ** 40}
        if k in fixed: caps.append(fixed[k])
        elif k == 8 and not is_error(r) and r > 1: caps.append(r - 1)
        else: caps.append(hbound(n))
    return caps


# ---- GPU side ---------------------------------------------------------------------------------------------------------------

def run_compress1x(host, offs, sizes, caps, msv, tl):
    """the 1X descriptor compress on the GPU: (values, per-block bytes, destination arena intact outside the destinations)"""
    import torch
    import finitestateentropy_b200 as fb
    src = torch.from_numpy(host).cuda()
    regions = [min(c, hbound(n)) for c, n in zip(caps, sizes)]
    rng = np.random.default_rng(len(sizes))
    gaps = [int(g) for g in rng.integers(1, 40, len(sizes))]
    doffs, cur = [], CANARY
    for r, g in zip(regions, gaps):
        doffs.append(cur); cur += r + g
    darena = torch.full((cur + CANARY,), POISON, dtype=torch.uint8, device="cuda")
    base_s, base_d = src.data_ptr(), darena.data_ptr()
    cs = torch.full((len(sizes),), -7, dtype=torch.int64, device="cuda")
    fb.huf_compress1x_blocks(_dev64([base_s + o for o in offs]), _dev64(sizes), _dev64([base_d + o for o in doffs]), _dev64(caps),
                             csizes=cs, max_symbol_value=msv, table_log=tl)
    torch.cuda.synchronize()
    got = _u64(cs)
    d = darena.cpu().numpy()
    allowed = np.zeros(len(d), bool)
    for o, r in zip(doffs, regions):
        allowed[o: o + r] = True
    untouched = bool((d[~allowed] == POISON).all())
    blocks = [d[o: o + (int(v) if not is_error(int(v)) else 0)] for o, v in zip(doffs, got)]
    assert torch.equal(src.cpu(), torch.from_numpy(host))                # sources are read only
    return got, blocks, untouched


def check_compress1x(lib, host, offs, sizes, caps, msv, tl):
    want, want_b = ref_compress1x(lib, host, offs, sizes, caps, msv, tl)
    got, got_b, untouched = run_compress1x(host, offs, sizes, caps, msv, tl)
    bad = [(b, sizes[b], caps[b], int(got[b]), int(want[b])) for b in range(len(sizes)) if got[b] != want[b]]
    assert not bad, (msv, tl, bad[:8])
    for b in range(len(sizes)):
        assert np.array_equal(got_b[b], want_b[b]), (msv, tl, b, sizes[b])
    assert untouched, "bytes outside the destinations were written"
    return want


def run_decode1x_packed(blocks, csizes, dsizes, want_outs, c_odd=1, d_odd=3):
    """compressed blocks back to back at an odd offset, outputs back to back at an odd offset (starting out as the complement
    of the expected bytes): (results, outputs, canaries intact, output addresses)"""
    import torch
    import finitestateentropy_b200 as fb
    coffs = CANARY + c_odd + np.concatenate([[0], np.cumsum(csizes)[:-1]]).astype(np.int64)
    chost = np.full(CANARY + c_odd + sum(csizes) + 32 + CANARY, POISON, np.uint8)
    for o, c, k in zip(coffs, blocks, csizes):
        chost[o: o + k] = c[:k]
    doffs = CANARY + d_odd + np.concatenate([[0], np.cumsum(dsizes)[:-1]]).astype(np.int64)
    dhost = np.full(CANARY + d_odd + sum(dsizes) + CANARY, POISON, np.uint8)
    for o, n, w in zip(doffs, dsizes, want_outs):
        if w is not None:
            dhost[o: o + n] = ~w
    carena = torch.from_numpy(chost).cuda(); darena = torch.from_numpy(dhost).cuda()
    res = torch.full((len(blocks),), -7, dtype=torch.int64, device="cuda")
    out_addrs = darena.data_ptr() + doffs
    fb.huf_decompress1x_blocks(_dev64(carena.data_ptr() + coffs), _dev64(csizes), _dev64(out_addrs), _dev64(dsizes), results=res)
    torch.cuda.synchronize()
    d = darena.cpu().numpy()
    end = doffs[-1] + dsizes[-1] if len(dsizes) else CANARY
    intact = bool((d[:CANARY] == POISON).all()) and bool((d[end:] == POISON).all())
    assert torch.equal(carena.cpu(), torch.from_numpy(chost))
    return _u64(res), [d[o: o + n] for o, n in zip(doffs, dsizes)], intact, out_addrs


def check_decode1x(lib, blocks, csizes, dsizes):
    want, want_o, x2_only = ref_decode1x(lib, blocks, csizes, dsizes)
    got, got_o, intact, addrs = run_decode1x_packed(blocks, csizes, dsizes, want_o)
    bad = [(b, csizes[b], dsizes[b], int(got[b]), int(want[b])) for b in range(len(blocks)) if got[b] != want[b]]
    assert not bad, bad[:8]
    for b in range(len(blocks)):
        if want_o[b] is not None:
            assert np.array_equal(got_o[b], want_o[b]), (b, csizes[b], dsizes[b])
    assert intact, "bytes outside the destinations were written"
    return want, x2_only, addrs


# ---- fixtures ---------------------------------------------------------------------------------------------------------------

def ragged_compress1x_check(seed, count, subset_every):
    rng = np.random.default_rng(seed)
    host, offs, sizes = ragged_sources(rng, count)
    assert set(SPECIAL_SIZES) <= set(sizes)
    lib = _ref()
    at_bound, _ = ref_compress1x(lib, host, offs, sizes, [hbound(n) for n in sizes], 255, 12)
    caps = capacities_1x(rng, sizes, at_bound)
    want = check_compress1x(lib, host, offs, sizes, caps, 255, 12)
    assert {"pipelined", "scalar"} <= {plan_histogram(o, n) for o, n in zip(offs, sizes)}
    assert {"g256", "g128", "bytes"} <= {emit_group_1x(o, n) for o, n in zip(offs, sizes)}
    kinds = {0 if v == 0 else 1 if v == 1 else "err" if is_error(int(v)) else "size" for v in want}
    assert kinds == {0, 1, "err", "size"}, kinds
    sub = list(range(0, len(sizes), subset_every))
    s_off, s_n, s_cap = [offs[i] for i in sub], [sizes[i] for i in sub], [caps[i] for i in sub]
    for msv, tl in ((255, 11), (0, 0), (200, 12), (255, 13), (256, 12)):
        w = check_compress1x(lib, host, s_off, s_n, s_cap, msv, tl)
        if msv == 200:
            assert any(int(v) == 2 ** 64 - 7 for v in w)                  # maxSymbolValue_tooSmall on bytes above 200


def packed_decode1x_fixture(seed, count):
    """(lib, compressed blocks, cSizes, dstSizes): 1X blocks of the GPU's and the reference's, truncated and bit-flipped ones,
    and every size case of HUF_decompress1X_DCtx, including dstSize > 128 KB"""
    import torch
    import finitestateentropy_b200 as fb
    rng = np.random.default_rng(seed)
    lib = _ref()
    sizes = [int(x) for x in rng.integers(6, HUF_BLOCK_MAX + 1, count // 2)] + \
            [int(rng.choice((8192, 32768, 4099, 777, 40, 13))) for _ in range(count - count // 2)]
    datas = [content(rng, n, i if i % 9 not in (6, 7) else 1) for i, n in enumerate(sizes)]   # compressible kinds only
    host = np.concatenate(datas + [np.zeros(64, np.uint8)])
    offs = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
    _, want_b = ref_compress1x(lib, host, offs, sizes, [hbound(n) for n in sizes], 255, 12)
    src = torch.from_numpy(host).cuda()
    dst = torch.zeros(sum(hbound(n) for n in sizes) + 64, dtype=torch.uint8, device="cuda")
    doffs = np.concatenate([[0], np.cumsum([hbound(n) for n in sizes])[:-1]]).astype(np.int64)
    cs = fb.huf_compress1x_blocks(_dev64(src.data_ptr() + offs), _dev64(sizes), _dev64(dst.data_ptr() + doffs),
                                  _dev64([hbound(n) for n in sizes]))
    gcs = _u64(cs); gd = dst.cpu().numpy()
    blocks, csizes, dsizes = [], [], []
    for i, n in enumerate(sizes):
        c = want_b[i] if i % 2 == 0 else gd[doffs[i]: doffs[i] + int(gcs[i])]
        c = np.array(c, np.uint8)
        if len(c) < 2:
            continue
        mode = i % 4
        k = len(c)
        if mode == 1:
            k = int(rng.integers(2, len(c)))                                  # truncated
        elif mode == 2:
            for _ in range(int(rng.integers(1, 4))):
                c[int(rng.integers(0, len(c)))] ^= int(rng.integers(1, 256))  # bit-flipped
        blocks.append(c[:k]); csizes.append(k); dsizes.append(n)
    d0 = datas[0]
    w0 = want_b[0]
    extra = [(d0[:0], 0, 500), (d0[:1], 1, 300), (d0[:300], 300, 300), (d0[:301], 301, 300), (d0[:40], 40, 0),
             (w0[:3], 3, 5), (w0[:2], 2, 4), (d0[:5], 5, 5), (d0[:1], 1, 3), (w0, len(w0), 131073),
             (w0, len(w0), 200000), (w0[:12], 12, 5), (w0, len(w0), sizes[0] - 1), (w0, len(w0), sizes[0] + 1)]
    for size in SPECIAL_SIZES:                                                # the size cases, each with a compressed block of its own
        if size >= 13:
            d = content(rng, size, 1)
            c = np.zeros(hbound(size), np.uint8)
            v = lib.HUF_compress1X(ptr(c), len(c), ptr(d), size, 255, 12)
            if 1 < v < size:
                extra.append((c[:v], int(v), size))
        extra.append((w0[: min(len(w0), 4)], min(len(w0), 4), size))
    for c, k, n in extra:
        blocks.append(np.array(c, np.uint8)); csizes.append(k); dsizes.append(n)
    return lib, blocks, csizes, dsizes


# ---- tests ------------------------------------------------------------------------------------------------------------------

def test_ragged_compress_1x():
    ragged_compress1x_check(seed=111, count=2000, subset_every=10)


def test_packed_decode_1x():
    lib, blocks, csizes, dsizes = packed_decode1x_fixture(seed=212, count=900)
    want, x2_only, addrs = check_decode1x(lib, blocks, csizes, dsizes)
    assert x2_only > 0                              # streams only the double-symbol decoder accepts
    kinds, streams = summarize(decode_paths_1x(blocks, csizes, dsizes, addrs))
    assert {"raw", "rle", "error", "A", "B", "hard"} <= set(kinds), kinds
    assert streams["head+fast"] and streams["symbol"] and streams["fast"], streams
    assert any(int(v) == ERR_SRC_WRONG and n > HUF_BLOCK_MAX for v, n in zip(want, dsizes))


@pytest.mark.parametrize("p,kind", [(0.14, "A"), (0.05, "B")])
def test_head_decode_every_residue_1x(p, kind):
    """blocks of 32,771 symbols, block b's output at residue b mod 32: its one stream decodes (-b) & 31 head symbols"""
    import torch
    import finitestateentropy_b200 as fb
    lib = _ref()
    n = 32771
    data = [probagen(n + 97 * i, p)[97 * i:] for i in range(64)]
    blocks, csizes = [], []
    for d in data:
        c = np.zeros(hbound(n), np.uint8)
        k = lib.HUF_compress1X(ptr(c), len(c), ptr(d), n, 255, 12)
        assert 1 < k < n
        blocks.append(c[:k]); csizes.append(k)
    darena = torch.zeros(64 * 65536 + 4096, dtype=torch.uint8, device="cuda")
    base = (darena.data_ptr() + 31) & ~31
    addrs = [base + b * 65536 + (b % 32) for b in range(64)]
    paths = decode_paths_1x(blocks, csizes, [n] * 64, addrs)
    assert all(q["kind"] == kind for q in paths), summarize(paths)
    heads = {s[0] for q in paths for s in q["streams"] if stream_kind(*s) == "head+fast"}
    assert heads == set(range(1, 32))
    csrc = torch.from_numpy(np.concatenate(blocks + [np.zeros(64, np.uint8)])).cuda()
    coffs = np.concatenate([[0], np.cumsum(csizes)[:-1]]).astype(np.int64)
    res = fb.huf_decompress1x_blocks(_dev64(csrc.data_ptr() + coffs), _dev64(csizes), _dev64(addrs), _dev64([n] * 64))
    torch.cuda.synchronize()
    assert (_u64(res) == n).all()
    out = darena.cpu().numpy()
    for b in range(64):
        o = addrs[b] - darena.data_ptr()
        assert np.array_equal(out[o: o + n], data[b]), b


def test_large_batch_two_rounds_1x():
    """44,000+ small ragged 1X blocks (two pass-A rounds of the 1X decoder on 132 SMs) plus deferred and hard blocks"""
    import torch
    rng = np.random.default_rng(313)
    sizes = [int(x) for x in rng.integers(64, 3000, 64000)] + [32768] * 300
    order = rng.permutation(len(sizes))
    sizes = [sizes[i] for i in order]
    lib = _ref()
    host, offs, sizes = ragged_sources(rng, len(sizes), sizes)
    want = check_compress1x(lib, host, offs, sizes, [hbound(n) for n in sizes], 255, 12)
    idx = [i for i, v in enumerate(want) if 1 < int(v) and not is_error(int(v))]
    cblocks = []
    for i in idx:
        d = np.ascontiguousarray(host[offs[i]: offs[i] + sizes[i]])
        c = np.zeros(hbound(sizes[i]), np.uint8)
        assert lib.HUF_compress1X(ptr(c), len(c), ptr(d), sizes[i], 255, 12) == want[i]
        cblocks.append(c[: int(want[i])])
    cs = [int(want[i]) for i in idx]; ds = [sizes[i] for i in idx]
    assert len(idx) >= 43000 and pass_a_spread_1x(len(idx), torch.cuda.get_device_properties(0).multi_processor_count)[1] >= 2
    _, _, addrs = check_decode1x(lib, cblocks, cs, ds)
    kinds, _ = summarize(decode_paths_1x(cblocks, cs, ds, addrs))
    assert kinds["B"] and kinds["A"] > 40000, kinds


def test_knobs_1x():
    """the single-pass decoder at the smallest row budget, in a child process"""
    _ref()
    e = dict(os.environ, FSEB200_HUFD_ROWS="160", FSEB200_HUFD_ROWS_B="0")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child"], env=e, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0 and "child ok" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])


def test_arguments_and_wrappers_1x():
    import torch
    import finitestateentropy_b200 as fb
    L = fb.lib()
    assert L.FSEB200_HUF_compress1X_blocks(0, None, None, None, None, None, 255, 12, None) == 0
    assert L.FSEB200_HUF_decompress1X_blocks(0, None, None, None, None, None, None) == 0
    a = _dev64([0])
    p = a.data_ptr()
    for k in range(5):
        args = [p] * 5
        args[k] = None
        assert L.FSEB200_HUF_compress1X_blocks(1, *args, 255, 12, None) == ERR_SRC_WRONG
        assert L.FSEB200_HUF_decompress1X_blocks(1, *args, None) == ERR_SRC_WRONG
    assert L.FSEB200_HUF_compress1X_blocks(1 << 32, p, p, p, p, p, 255, 12, None) == ERR_SRC_WRONG
    assert L.FSEB200_HUF_decompress1X_blocks(1 << 32, p, p, p, p, p, None) == ERR_SRC_WRONG
    cs = torch.full((4,), -7, dtype=torch.int64, device="cuda")
    assert L.FSEB200_HUF_compress1X_blocks(0, p, p, cs.data_ptr(), p, p, 255, 12, None) == 0
    assert L.FSEB200_HUF_decompress1X_blocks(0, p, p, cs.data_ptr(), p, p, None) == 0
    torch.cuda.synchronize()
    assert (cs == -7).all()
    # the Python wrappers on views, on a side stream; 1X and 4X blocks of the same data differ (no jump table)
    data = [torch.from_numpy(probagen(n, 0.14)).cuda() for n in (1000, 32768, 4099)]
    srcs, n = fb.block_pointers(data)
    dsts = [torch.zeros(hbound(int(k)), dtype=torch.uint8, device="cuda") for k in n.tolist()]
    dp, dc = fb.block_pointers(dsts)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        csz = fb.huf_compress1x_blocks(srcs, n, dp, dc)
        csz4 = fb.huf_compress_blocks(srcs, n, dp, dc, csizes=torch.empty_like(csz))
        outs = [torch.zeros_like(d) for d in data]
        op, on = fb.block_pointers(outs)
    s.synchronize()
    # the same header and bits: 4X adds the 6-byte jump table and up to 4 bytes of padding of its four streams
    assert all(6 <= d <= 10 for d in (csz4 - csz).tolist()), (csz4.tolist(), csz.tolist())
    with torch.cuda.stream(s):
        csz = fb.huf_compress1x_blocks(srcs, n, dp, dc)
        res = fb.huf_decompress1x_blocks(dp, csz, op, on)
    s.synchronize()
    assert res.tolist() == n.tolist() and all(torch.equal(o, d) for o, d in zip(outs, data))


def _child():
    ragged_compress1x_check(seed=414, count=400, subset_every=7)
    lib, blocks, csizes, dsizes = packed_decode1x_fixture(seed=515, count=300)
    check_decode1x(lib, blocks, csizes, dsizes)
    print("child ok")


if __name__ == "__main__" and "--child" in sys.argv:
    _child()
