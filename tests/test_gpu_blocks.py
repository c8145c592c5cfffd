"""Per-block descriptor calls (FSEB200_HUF_compress_blocks / FSEB200_HUF_decompress_blocks) against the compiled reference,
block by block (-m gpu): ragged sizes, sources anywhere (overlapping too), every capacity and parameter verdict, packed
compressed inputs and outputs at odd offsets, malformed blocks, the head decode at every residue, equivalence with the uniform
calls, a batch of two pass-A rounds, the decoder's row budgets, and the call's own argument checks.

Run as a script (`python tests/test_gpu_blocks.py --child`) it repeats subsets of the ragged tests under the environment it
was started with: test_knobs starts it with FSEB200_HUFD_ROWS / _ROWS_B set."""
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from helpers import REF_SO, is_error, load_ref, probagen, ptr, zoo        # noqa: E402
from paths import hard_block, pass_a_spread                             # noqa: E402
from blocks_paths import (decode_paths, summarize, plan_histogram, expected_decode_verdict, stream_kind,   # noqa: E402
                          HUF_BLOCK_MAX)

pytestmark = pytest.mark.gpu

POISON = 0x5A
CANARY = 4096
ERR_SRC_WRONG = 2 ** 64 - 3


def hbound(n):
    return 129 + n + (n >> 8) + 8                   # HUF_compressBound (lib/huf.h:131-133)


def _ref():
    if not os.path.exists(REF_SO):
        pytest.skip("needs the compiled reference (oracle/_ref)")
    return load_ref()


def _u64(t):
    return t.cpu().numpy().view(np.uint64)


def _dev64(a):
    import torch
    return torch.from_numpy(np.asarray(a, dtype=np.uint64).view(np.int64).copy()).cuda()


# ---- fixtures -------------------------------------------------------------------------------------------------------------

SPECIAL_SIZES = [0, 1, 11, 12, 13, 31, 32, 33, 127, 128, 129, 4099, 32768, 65537, 131071, 131072, 131073]


def content(rng, n, i):
    """block content by index: probagen P 0.02 / 0.14 / 0.30 / 0.80, the fuzzers' zoo, constant, random, the hard histogram"""
    k = i % 9
    if k < 4:
        off = int(rng.integers(0, 1 << 12))
        return probagen(off + n, [0.02, 0.14, 0.30, 0.80][k])[off:]
    if k == 4 or k == 5:
        return zoo(rng, n)
    if k == 6:
        return np.full(n, int(rng.integers(0, 256)), np.uint8)
    if k == 7:
        return rng.integers(0, 256, n, dtype=np.uint8)
    return hard_block(rng, 32768)[:n] if n <= 32768 else np.concatenate([hard_block(rng, 32768)] * ((n + 32767) // 32768))[:n]


def ragged_sources(rng, count, sizes=None):
    """(host arena, offsets, sizes): block contents at random byte offsets of one arena (sizes that are multiples of 8 KiB at
    16-byte aligned ones); about one block in 20 is a window that overlaps other blocks' bytes"""
    if sizes is None:
        sizes = SPECIAL_SIZES + [int(x) for x in rng.integers(1, HUF_BLOCK_MAX + 1, count - len(SPECIAL_SIZES))]
    parts, offs, cur = [], [], CANARY
    for i, n in enumerate(sizes):
        if i > 20 and rng.random() < 0.05 and cur - CANARY > n + 64:
            offs.append(int(rng.integers(CANARY, cur - n)))           # inside earlier blocks
            continue
        gap = int(rng.integers(0, 64))
        if n and n % 8192 == 0:
            gap += -(cur + gap) % 16                                  # 16-byte aligned: the plan kernel's pipelined histogram
        parts.append(np.full(gap, POISON, np.uint8)); cur += gap
        offs.append(cur)
        parts.append(content(rng, n, i)); cur += n
    host = np.concatenate([np.full(CANARY, POISON, np.uint8)] + parts + [np.full(CANARY + 64, POISON, np.uint8)])
    return host, offs, [int(s) for s in sizes]


def ref_compress(lib, host, offs, sizes, caps, msv, tl):
    """HUF_compress2 per block on the host: (values, compressed bytes); a capacity above the bound runs at the bound (same verdict)"""
    vals, outs = [], []
    for o, n, cap in zip(offs, sizes, caps):
        c = min(cap, hbound(n))
        buf = np.zeros(c + 8, np.uint8)
        src = np.ascontiguousarray(host[o: o + n])
        v = lib.HUF_compress2(ptr(buf), c, ptr(src), n, msv, tl)
        vals.append(v)
        outs.append(buf[: v] if (not is_error(v) and v >= 1) else buf[:0])
    return vals, outs


def capacities(rng, sizes, ref_at_bound):
    caps = []
    for i, (n, r) in enumerate(zip(sizes, ref_at_bound)):
        k = i % 10
        if k == 4: caps.append(0)
        elif k == 5: caps.append(1)
        elif k == 6: caps.append(16)
        elif k == 7: caps.append(17)
        elif k == 8 and not is_error(r) and r > 1: caps.append(r - 1)
        elif k == 9: caps.append(2 ** 40)
        else: caps.append(hbound(n))
    return caps


def run_compress(host, offs, sizes, caps, msv, tl):
    """the descriptor compress on the GPU: (values, per-block bytes, destination arena intact outside the destinations)"""
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
    fb.huf_compress_blocks(_dev64([base_s + o for o in offs]), _dev64(sizes), _dev64([base_d + o for o in doffs]), _dev64(caps),
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


def check_compress(lib, host, offs, sizes, caps, msv, tl):
    want, want_b = ref_compress(lib, host, offs, sizes, caps, msv, tl)
    got, got_b, untouched = run_compress(host, offs, sizes, caps, msv, tl)
    bad = [(b, sizes[b], caps[b], int(got[b]), int(want[b])) for b in range(len(sizes)) if got[b] != want[b]]
    assert not bad, (msv, tl, bad[:8])
    for b in range(len(sizes)):
        assert np.array_equal(got_b[b], want_b[b]), (msv, tl, b, sizes[b])
    assert untouched, "bytes outside the destinations were written"
    return want


def ragged_compress_fixture(seed, count):
    rng = np.random.default_rng(seed)
    host, offs, sizes = ragged_sources(rng, count)
    lib = _ref()
    at_bound, _ = ref_compress(lib, host, offs, sizes, [hbound(n) for n in sizes], 255, 12)
    return lib, host, offs, sizes, capacities(rng, sizes, at_bound)


def ragged_compress_check(seed, count, subset_every):
    lib, host, offs, sizes, caps = ragged_compress_fixture(seed, count)
    want = check_compress(lib, host, offs, sizes, caps, 255, 12)
    assert {"pipelined", "scalar"} <= {plan_histogram(o, n) for o, n in zip(offs, sizes)}     # offsets relative to an aligned arena
    kinds = {0 if v == 0 else 1 if v == 1 else "err" if is_error(int(v)) else "size" for v in want}
    assert kinds == {0, 1, "err", "size"}, kinds
    sub = list(range(0, len(sizes), subset_every))
    s_off, s_n, s_cap = [offs[i] for i in sub], [sizes[i] for i in sub], [caps[i] for i in sub]
    for msv, tl in ((255, 11), (0, 0), (200, 12), (255, 13), (256, 12)):
        w = check_compress(lib, host, s_off, s_n, s_cap, msv, tl)
        if msv == 200:
            assert any(int(v) == 2 ** 64 - 7 for v in w)                  # maxSymbolValue_tooSmall on bytes above 200


def packed_decode_fixture(seed, count):
    """(compressed blocks, cSizes, dstSizes, originals or None): Huffman blocks of the GPU's and the reference's, truncated and
    bit-flipped ones, and every size case of HUF_decompress"""
    import torch
    import finitestateentropy_b200 as fb
    rng = np.random.default_rng(seed)
    lib = _ref()
    sizes = [int(x) for x in rng.integers(6, HUF_BLOCK_MAX + 1, count // 2)] + [int(rng.choice((8192, 32768, 4099, 777))) for _ in range(count - count // 2)]
    datas = [content(rng, n, i if i % 9 not in (6, 7) else 1) for i, n in enumerate(sizes)]   # compressible kinds only
    host = np.concatenate(datas + [np.zeros(64, np.uint8)])
    offs = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
    _, want_b = ref_compress(lib, host, offs, sizes, [hbound(n) for n in sizes], 255, 12)
    # the GPU's own compressed blocks for the odd-indexed ones
    src = torch.from_numpy(host).cuda()
    dst = torch.zeros(sum(hbound(n) for n in sizes) + 64, dtype=torch.uint8, device="cuda")
    doffs = np.concatenate([[0], np.cumsum([hbound(n) for n in sizes])[:-1]]).astype(np.int64)
    cs = fb.huf_compress_blocks(_dev64(src.data_ptr() + offs), _dev64(sizes), _dev64(dst.data_ptr() + doffs), _dev64([hbound(n) for n in sizes]))
    gcs = _u64(cs); gd = dst.cpu().numpy()
    blocks, csizes, dsizes, origs = [], [], [], []
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
        blocks.append(c[:k]); csizes.append(k); dsizes.append(n); origs.append(datas[i] if mode in (0, 3) else None)
    d0 = datas[0]
    extra = [(d0[:0], 0, 500), (d0[:1], 1, 300), (d0[:300], 300, 300), (d0[:301], 301, 300), (d0[:40], 40, 0),
             (want_b[0][:3], 3, 5), (want_b[0][:2], 2, 4), (d0[:5], 5, 5), (d0[:1], 1, 3), (want_b[0], len(want_b[0]), 131073),
             (want_b[0], len(want_b[0]), 200000), (want_b[0][:12], 12, 5)]
    for c, k, n in extra:
        blocks.append(np.array(c, np.uint8)); csizes.append(k); dsizes.append(n); origs.append(None)
    return lib, blocks, csizes, dsizes


def ref_decode(lib, blocks, csizes, dsizes):
    """expected (value, bytes) per block: the reference's HUF_decompress, with this library's documented answers"""
    vals, outs, x2_only = [], [], 0
    for c, k, n in zip(blocks, csizes, dsizes):
        if n > HUF_BLOCK_MAX:
            vals.append(ERR_SRC_WRONG); outs.append(None); continue
        tmp = np.concatenate([c, np.zeros(64, np.uint8)])
        o = np.zeros(n + 64, np.uint8)
        v = lib.HUF_decompress(ptr(o), n, ptr(tmp), k)
        if not is_error(v) and 1 < k < n:
            o2 = np.zeros(n + 64, np.uint8)
            x2_only += bool(is_error(lib.HUF_decompress4X1(ptr(o2), n, ptr(tmp), k)))
        v = expected_decode_verdict(v, k, n)
        vals.append(v); outs.append(None if is_error(v) else o[:n].copy())
    return vals, outs, x2_only


def run_decode_packed(blocks, csizes, dsizes, want_outs, c_odd=1, d_odd=3):
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
    fb.huf_decompress_blocks(_dev64(carena.data_ptr() + coffs), _dev64(csizes), _dev64(out_addrs), _dev64(dsizes), results=res)
    torch.cuda.synchronize()
    d = darena.cpu().numpy()
    end = doffs[-1] + dsizes[-1] if len(dsizes) else CANARY
    intact = bool((d[:CANARY] == POISON).all()) and bool((d[end:] == POISON).all())
    assert torch.equal(carena.cpu(), torch.from_numpy(chost))
    return _u64(res), [d[o: o + n] for o, n in zip(doffs, dsizes)], intact, out_addrs


def check_decode(lib, blocks, csizes, dsizes, **kw):
    want, want_o, x2_only = ref_decode(lib, blocks, csizes, dsizes)
    got, got_o, intact, addrs = run_decode_packed(blocks, csizes, dsizes, want_o, **kw)
    bad = [(b, csizes[b], dsizes[b], int(got[b]), int(want[b])) for b in range(len(blocks)) if got[b] != want[b]]
    assert not bad, bad[:8]
    for b in range(len(blocks)):
        if want_o[b] is not None:
            assert np.array_equal(got_o[b], want_o[b]), (b, csizes[b], dsizes[b])
    assert intact, "bytes outside the destinations were written"
    return want, x2_only, addrs


# ---- tests ----------------------------------------------------------------------------------------------------------------

def test_ragged_compress():
    ragged_compress_check(seed=101, count=3000, subset_every=10)


def test_packed_decode():
    lib, blocks, csizes, dsizes = packed_decode_fixture(seed=202, count=900)
    want, x2_only, addrs = check_decode(lib, blocks, csizes, dsizes)
    assert x2_only > 0                              # streams only the double-symbol decoder accepts
    paths = decode_paths(blocks, csizes, dsizes, addrs)
    kinds, streams = summarize(paths)
    assert {"raw", "rle", "error", "A", "B", "hard"} <= set(kinds), kinds
    assert streams["head+fast"] and streams["symbol"] and streams["fast"], streams


@pytest.mark.parametrize("p,kind", [(0.14, "A"), (0.05, "B")])
def test_head_decode_every_residue(p, kind):
    """segments of 8,193 symbols: a block's four streams start at residues r, r+1, r+2, r+3 mod 32 of its output offset r"""
    lib = _ref()
    n = 4 * 8193
    data = [probagen(n + 97 * i, p)[97 * i:] for i in range(64)]
    blocks, csizes = [], []
    for d in data:
        c = np.zeros(hbound(n), np.uint8)
        k = lib.HUF_compress2(ptr(c), len(c), ptr(d), n, 255, 12)
        assert 1 < k < n
        blocks.append(c[:k]); csizes.append(k)
    # output b at offset (b % 32) mod 32: each block in its own 64 KiB-aligned window of the output arena
    import torch
    import finitestateentropy_b200 as fb
    darena = torch.zeros(64 * 65536 + 4096, dtype=torch.uint8, device="cuda")
    base = (darena.data_ptr() + 31) & ~31
    addrs = [base + b * 65536 + (b % 32) for b in range(64)]
    paths = decode_paths(blocks, csizes, [n] * 64, addrs)
    assert all(q["kind"] == kind for q in paths), summarize(paths)
    heads = {s[0] for q in paths for s in q["streams"] if stream_kind(*s) == "head+fast"}
    assert heads == set(range(1, 32))
    csrc = torch.from_numpy(np.concatenate(blocks + [np.zeros(64, np.uint8)])).cuda()
    coffs = np.concatenate([[0], np.cumsum(csizes)[:-1]]).astype(np.int64)
    res = fb.huf_decompress_blocks(_dev64(csrc.data_ptr() + coffs), _dev64(csizes), _dev64(addrs), _dev64([n] * 64))
    torch.cuda.synchronize()
    assert (_u64(res) == n).all()
    out = darena.cpu().numpy()
    for b in range(64):
        o = addrs[b] - darena.data_ptr()
        assert np.array_equal(out[o: o + n], data[b]), b


def test_uniform_layout_equivalence():
    """64 MiB of P14 through the uniform calls and through the descriptor calls at ptr = base + b * blockSize"""
    import torch
    import finitestateentropy_b200 as fb
    block, total = 32768, 64 << 20
    slot = fb.compress_bound(block)
    src = torch.from_numpy(probagen(total, 0.14)).cuda()
    nb = total // block
    cbuf, cs = fb.huf_compress_batch(src, block, slot)
    cbuf2 = torch.zeros_like(cbuf)
    b = np.arange(nb, dtype=np.int64)
    cs2 = fb.huf_compress_blocks(_dev64(src.data_ptr() + b * block), _dev64([block] * nb), _dev64(cbuf2.data_ptr() + b * slot), _dev64([slot] * nb))
    torch.cuda.synchronize()
    assert torch.equal(cs, cs2)
    sizes = cs.cpu().numpy()
    mask = torch.from_numpy((np.arange(slot)[None, :] < sizes[:, None]).reshape(-1)).cuda()
    assert torch.equal(cbuf[: nb * slot][mask], cbuf2[: nb * slot][mask])
    out, res = fb.huf_decompress_batch(cbuf, cs, total, block, slot)
    out2 = torch.empty_like(out)
    res2 = fb.huf_decompress_blocks(_dev64(cbuf.data_ptr() + b * slot), cs, _dev64(out2.data_ptr() + b * block), _dev64([block] * nb))
    torch.cuda.synchronize()
    assert torch.equal(res, res2) and torch.equal(out, out2) and torch.equal(out, src)


def test_large_batch_two_rounds():
    """44,000+ small ragged blocks (two pass-A rounds on 132 SMs) plus deferred and hard blocks, against the reference"""
    import torch
    rng = np.random.default_rng(303)
    sizes = [int(x) for x in rng.integers(64, 3000, 64000)] + [32768] * 300      # ~45,000 of them compress to Huffman blocks
    order = rng.permutation(len(sizes))
    sizes = [sizes[i] for i in order]
    lib = _ref()
    host, offs, sizes = ragged_sources(rng, len(sizes), sizes)
    want = check_compress(lib, host, offs, sizes, [hbound(n) for n in sizes], 255, 12)
    idx = [i for i, v in enumerate(want) if 1 < int(v) and not is_error(int(v))]
    blocks = [np.ascontiguousarray(host[offs[i]: offs[i] + sizes[i]]) for i in idx]
    cblocks = []
    for i, d in zip(idx, blocks):
        c = np.zeros(hbound(sizes[i]), np.uint8)
        assert lib.HUF_compress2(ptr(c), len(c), ptr(d), sizes[i], 255, 12) == want[i]
        cblocks.append(c[: int(want[i])])
    cs = [int(want[i]) for i in idx]; ds = [sizes[i] for i in idx]
    assert len(idx) >= 44000 and pass_a_spread(len(idx), torch.cuda.get_device_properties(0).multi_processor_count)[1] >= 2
    _, _, addrs = check_decode(lib, cblocks, cs, ds)
    kinds, streams = summarize(decode_paths(cblocks, cs, ds, addrs))
    assert kinds["B"] and kinds["A"] > 40000, kinds


def test_knobs():
    """the single-pass decoder at the smallest row budget, in a child process"""
    _ref()
    e = dict(os.environ, FSEB200_HUFD_ROWS="160", FSEB200_HUFD_ROWS_B="0")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child"], env=e, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0 and "child ok" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])


def test_arguments_and_wrappers():
    import ctypes as C
    import torch
    import finitestateentropy_b200 as fb
    L = fb.lib()
    assert L.FSEB200_HUF_compress_blocks(0, None, None, None, None, None, 255, 12, None) == 0
    assert L.FSEB200_HUF_decompress_blocks(0, None, None, None, None, None, None) == 0
    a = _dev64([0])
    p = a.data_ptr()
    for k in range(5):
        args = [p] * 5
        args[k] = None
        assert L.FSEB200_HUF_compress_blocks(1, *args, 255, 12, None) == ERR_SRC_WRONG
        assert L.FSEB200_HUF_decompress_blocks(1, *args, None) == ERR_SRC_WRONG
    assert L.FSEB200_HUF_compress_blocks(1 << 32, p, p, p, p, p, 255, 12, None) == ERR_SRC_WRONG
    assert L.FSEB200_HUF_decompress_blocks(1 << 32, p, p, p, p, p, None) == ERR_SRC_WRONG
    # nBlocks == 0 writes nothing
    cs = torch.full((4,), -7, dtype=torch.int64, device="cuda")
    assert L.FSEB200_HUF_compress_blocks(0, p, p, cs.data_ptr(), p, p, 255, 12, None) == 0
    assert L.FSEB200_HUF_decompress_blocks(0, p, p, cs.data_ptr(), p, p, None) == 0
    torch.cuda.synchronize()
    assert (cs == -7).all()
    # the Python wrappers on views, on a side stream
    data = [torch.from_numpy(probagen(n, 0.14)).cuda() for n in (1000, 32768, 4099)]
    srcs, n = fb.block_pointers(data)
    assert n.tolist() == [1000, 32768, 4099] and srcs.dtype == torch.int64 and srcs.is_cuda
    dsts = [torch.zeros(hbound(int(k)), dtype=torch.uint8, device="cuda") for k in n.tolist()]
    dp, dc = fb.block_pointers(dsts)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        csz = fb.huf_compress_blocks(srcs, n, dp, dc)
        outs = [torch.zeros_like(d) for d in data]
        op, on = fb.block_pointers(outs)
        res = fb.huf_decompress_blocks(dp, csz, op, on)
    s.synchronize()
    assert res.tolist() == n.tolist() and all(torch.equal(o, d) for o, d in zip(outs, data))


def _child():
    ragged_compress_check(seed=404, count=400, subset_every=7)
    lib, blocks, csizes, dsizes = packed_decode_fixture(seed=505, count=300)
    check_decode(lib, blocks, csizes, dsizes)
    print("child ok")


if __name__ == "__main__" and "--child" in sys.argv:
    _child()
