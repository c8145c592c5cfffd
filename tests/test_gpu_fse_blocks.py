"""Per-block descriptor calls for FSE and FSE-U16 (FSEB200_FSE{,U16}_{compress,decompress}_blocks) against the compiled
reference, block by block (-m gpu): ragged sizes at random (and overlapping) source offsets, every capacity and parameter
verdict, packed compressed inputs at odd offsets, malformed blocks, the U16 units and alignment verdict, equivalence with the
uniform calls, a batch of several waves of both encoders, the 2^30 limit on a real allocation, the EK=8 knob and the calls'
own argument checks.  Destinations start out as poison with canaries between them; nothing outside them may change.

Run as a script (`python tests/test_gpu_fse_blocks.py --child`) it repeats the ragged compress tests under the environment it
was started with: test_knob starts it with FSEB200_ENC_EK=8."""
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from helpers import gen_u16, is_error, probagen, ptr, zoo                 # noqa: E402
from test_gpu_blocks import CANARY, POISON, _dev64, _ref, _u64           # noqa: E402
from gpu_common import header_only_u16                                  # noqa: E402
from fse_blocks_paths import (ERR_GENERIC, ERR_SRC_WRONG, FSE_BLOCK_MAX, cta_groups, decode_path, encode_route,   # noqa: E402
                              read_range, readable_range)

pytestmark = pytest.mark.gpu

ERR_CORRUPT = 2 ** 64 - 4
ERR_MSV_SMALL = 2 ** 64 - 7
ERR_TLOG_LARGE = 2 ** 64 - 5
SPECIAL = [0, 1, 2, 3, 63, 64, 65, 127, 128, 4099, 32768, 65536, 131072, 1 << 20]


def fbound(nbytes):
    return 512 + nbytes + (nbytes >> 7) + 4 + 8        # FSE_compressBound (lib/fse.h:290-292)


class Codec:
    """byte FSE or FSE-U16: element width, the reference's calls and this library's wrappers"""
    def __init__(self, wide):
        self.wide, self.w = wide, (2 if wide else 1)

    def content(self, rng, n, i):
        if self.wide:
            k = i % 5
            if k == 3:
                return np.full(n, int(rng.integers(0, 287)), np.uint16)
            if k == 4:
                return rng.integers(0, 287, n).astype(np.uint16)
            return gen_u16(n, 240, [0.2, 0.5, 0.8][k], int(rng.integers(1, 1000)))
        k = i % 7
        if k < 4:
            off = int(rng.integers(0, 1 << 12))
            return probagen(off + n, [0.02, 0.14, 0.30, 0.80][k])[off:]
        if k == 4:
            return zoo(rng, n)
        if k == 5:
            return np.full(n, int(rng.integers(0, 256)), np.uint8)
        return rng.integers(0, 256, n, dtype=np.uint8)

    def ref_compress(self, lib, src, n, cap, msv, tl):
        buf = np.zeros(cap + 8, np.uint8)
        f = lib.FSE_compressU16 if self.wide else lib.FSE_compress2
        v = f(ptr(buf), cap, ptr(src), n, msv, tl)
        return v, buf[: v] if not is_error(v) and v > 1 else buf[:0]

    def ref_decompress(self, lib, c, k, cap):
        if self.wide and header_only_u16(np.asarray(c, np.uint8), k):
            return ERR_CORRUPT, None            # the reference dereferences NULL on an empty stream; this library's answer (DESIGN 2)
        tmp = np.concatenate([np.asarray(c, np.uint8)[:k], np.zeros(64, np.uint8)])
        o = np.zeros(cap * self.w + 64, np.uint8)
        f = lib.FSE_decompressU16 if self.wide else lib.FSE_decompress
        v = f(ptr(o), cap, ptr(tmp), k)
        return v, (None if is_error(v) else o[: v * self.w].copy())

    def compress(self, *a, **kw):
        import finitestateentropy_b200 as fb
        return (fb.fseu16_compress_blocks if self.wide else fb.fse_compress_blocks)(*a, **kw)

    def decompress(self, *a, **kw):
        import finitestateentropy_b200 as fb
        return (fb.fseu16_decompress_blocks if self.wide else fb.fse_decompress_blocks)(*a, **kw)


BYTES, U16 = Codec(False), Codec(True)


# ---- compress ---------------------------------------------------------------------------------------------------------------

def ragged_sources(cd, rng, sizes):
    """(host arena bytes, byte offsets): blocks at random offsets (U16: even ones), sizes of whole 64-byte groups mostly at
    16-byte aligned offsets; about one block in 20 is a window overlapping earlier blocks"""
    parts, offs, cur = [], [], CANARY
    for i, n in enumerate(sizes):
        nb = n * cd.w
        if i > 20 and rng.random() < 0.05 and cur - CANARY > nb + 64:
            offs.append(int(rng.integers(CANARY, cur - nb)) & ~(cd.w - 1))
            continue
        gap = int(rng.integers(0, 64)) * cd.w
        if nb and nb % 64 == 0 and rng.random() < 0.8:
            gap += -(cur + gap) % 16
        parts.append(np.full(gap, POISON, np.uint8)); cur += gap
        offs.append(cur)
        parts.append(cd.content(rng, n, i).view(np.uint8)); cur += nb
    host = np.concatenate([np.full(CANARY, POISON, np.uint8)] + parts + [np.full(CANARY + 64, POISON, np.uint8)])
    return host, offs


def ref_values(cd, lib, host, offs, sizes, caps, msv, tl):
    vals, outs = [], []
    for o, n, cap in zip(offs, sizes, caps):
        src = np.ascontiguousarray(host[o: o + n * cd.w])
        if cd.wide:
            src = src.view(np.uint16)
        v, b = cd.ref_compress(lib, src, n, min(cap, fbound(n * cd.w)), msv, tl)
        vals.append(v); outs.append(b)
    return vals, outs


def run_compress(cd, host, offs, sizes, caps, msv, tl):
    import torch
    src = torch.from_numpy(host).cuda()
    regions = [min(c, fbound(n * cd.w)) for c, n in zip(caps, sizes)]
    rng = np.random.default_rng(len(sizes))
    doffs, cur = [], CANARY
    for r in regions:
        doffs.append(cur); cur += r + int(rng.integers(1, 40))
    darena = torch.full((cur + CANARY,), POISON, dtype=torch.uint8, device="cuda")
    cs = torch.full((len(sizes),), -7, dtype=torch.int64, device="cuda")
    cd.compress(_dev64([src.data_ptr() + o for o in offs]), _dev64(sizes), _dev64([darena.data_ptr() + o for o in doffs]), _dev64(caps),
                csizes=cs, max_symbol_value=msv, table_log=tl)
    torch.cuda.synchronize()
    got = _u64(cs)
    d = darena.cpu().numpy()
    allowed = np.zeros(len(d), bool)
    for o, r in zip(doffs, regions):
        allowed[o: o + r] = True
    assert (d[~allowed] == POISON).all(), "bytes outside the destinations were written"
    assert torch.equal(src.cpu(), torch.from_numpy(host))
    return got, [d[o: o + (int(v) if not is_error(int(v)) else 0)] for o, v in zip(doffs, got)], src.data_ptr()


def header_cut_u16(cblock, cs):
    """a value of FSE_compressU16 that ends inside its own table header: at some capacities below the bound the reference
    returns such a size, whose bytes depend on the capacity and decode to nothing"""
    import ctypes as C
    norm = (C.c_short * 512)()
    msv, tl = C.c_uint(511), C.c_uint(0)
    c = np.concatenate([np.asarray(cblock, np.uint8)[:cs], np.zeros(8, np.uint8)])
    h = _ref().FSE_readNCount(norm, C.byref(msv), C.byref(tl), ptr(c), cs)
    return is_error(h) or h > cs


def one_block_u16(host, o, n, cap, msv, tl):
    """this library's own one-block FSE_compressU16 (host pointers): (value, bytes)"""
    import finitestateentropy_b200 as fb
    f = fb.lib().FSE_compressU16
    src = np.ascontiguousarray(host[o: o + 2 * n])
    buf = np.zeros(cap + 8, np.uint8)
    v = f(ptr(buf), cap, ptr(src), n, msv, tl)
    return v, buf[:v]


def check_compress(cd, lib, host, offs, sizes, caps, msv, tl):
    want, want_b = ref_values(cd, lib, host, offs, sizes, caps, msv, tl)
    got, got_b, base = run_compress(cd, host, offs, sizes, caps, msv, tl)
    bad = [(b, sizes[b], caps[b], int(got[b]), int(want[b])) for b in range(len(sizes)) if got[b] != want[b]]
    assert not bad, (cd.wide, msv, tl, bad[:8])
    for b in range(len(sizes)):
        if int(want[b]) > 1 and not is_error(int(want[b])) and not np.array_equal(got_b[b], want_b[b]):
            # only a U16 value cut inside the reference's own header may differ, and then it is the one-block call's bytes
            assert cd.wide and header_cut_u16(want_b[b], int(want[b])), (cd.wide, msv, tl, b, sizes[b])
            v, one = one_block_u16(host, offs[b], sizes[b], min(caps[b], fbound(2 * sizes[b])), msv, tl)
            assert v == want[b] and np.array_equal(got_b[b], one), (msv, tl, b, sizes[b])
    return want, want_b, base


def capacities(cd, rng, sizes, at_bound):
    caps = []
    for i, (n, r) in enumerate(zip(sizes, at_bound)):
        k = i % 10
        if k == 4: caps.append(0)
        elif k == 5: caps.append(1)
        elif k == 6: caps.append(16)
        elif k == 7 and not is_error(r) and r > 1: caps.append(r - 1)
        elif k == 8: caps.append(2 ** 40)
        else: caps.append(fbound(n * cd.w))
    return caps


def ragged_compress_check(cd, seed, count, subset_every):
    rng = np.random.default_rng(seed)
    lib = _ref()
    special = [s // cd.w for s in SPECIAL] if cd.wide else SPECIAL
    sizes = special + [int(x) for x in rng.integers(1, 131072 // cd.w + 1, count - len(special))]
    sizes += [64 // cd.w * int(x) for x in rng.integers(1, 512, count // 4)]           # whole 64-byte groups: the CTA kernel
    host, offs = ragged_sources(cd, rng, sizes)
    at_bound, _ = ref_values(cd, lib, host, offs, sizes, [fbound(n * cd.w) for n in sizes], 0 if cd.wide else 255, 12)
    caps = capacities(cd, rng, sizes, at_bound)
    want, _, base = check_compress(cd, lib, host, offs, sizes, caps, 0 if cd.wide else 255, 12)
    kinds = {0 if v == 0 else 1 if v == 1 else "err" if is_error(int(v)) else "size" for v in want}
    assert kinds >= {0, 1, "size"}, kinds
    routes = [encode_route(base + o, n, cd.wide) for o, n in zip(offs, sizes)]
    assert min(routes.count("cta"), routes.count("warp")) > count // 10
    cta_sizes = {n for r, n in zip(routes, sizes) if r == "cta"}
    assert len(set(cta_groups([n * cd.w for n in cta_sizes])[0])) > 16       # a CTA of 16 holds blocks of different sizes
    sub = list(range(0, len(sizes), subset_every))
    s_off, s_n, s_cap = [offs[i] for i in sub], [sizes[i] for i in sub], [caps[i] for i in sub]
    params = ((0, 11), (0, 0), (0, 14), (100, 12), (300, 12)) if cd.wide else ((255, 11), (255, 0), (255, 13), (100, 12), (0, 12))
    for msv, tl in params:
        w, _, _ = check_compress(cd, lib, host, s_off, s_n, s_cap, msv, tl)
        if msv == 100:
            assert any(int(v) == ERR_MSV_SMALL for v in w)
        if tl in (13, 14):
            assert any(int(v) == ERR_TLOG_LARGE for v in w)


def test_ragged_compress_bytes():
    ragged_compress_check(BYTES, seed=11, count=800, subset_every=9)


def test_ragged_compress_u16():
    ragged_compress_check(U16, seed=12, count=600, subset_every=9)


# ---- decompress -------------------------------------------------------------------------------------------------------------

def decode_fixture(cd, seed, count):
    """(blocks, cSizes, capacities): compressed blocks of the reference's and the GPU's, truncated and bit-flipped ones, exact,
    larger, one-short and zero capacities, and the literal small cSizes"""
    import torch
    rng = np.random.default_rng(seed)
    lib = _ref()
    sizes = [int(x) for x in rng.integers(2, 131072 // cd.w + 1, count)]
    datas = [cd.content(rng, n, i if i % (5 if cd.wide else 7) < 4 else 1) for i, n in enumerate(sizes)]
    host = np.concatenate([d.view(np.uint8) for d in datas] + [np.zeros(64, np.uint8)])
    offs = np.concatenate([[0], np.cumsum([n * cd.w for n in sizes])[:-1]]).astype(np.int64)
    _, want_b = ref_values(cd, lib, host, offs, sizes, [fbound(n * cd.w) for n in sizes], 0 if cd.wide else 255, 12)
    src = torch.from_numpy(host).cuda()
    bounds = [fbound(n * cd.w) for n in sizes]
    dst = torch.zeros(sum(bounds) + 64, dtype=torch.uint8, device="cuda")
    doffs = np.concatenate([[0], np.cumsum(bounds)[:-1]]).astype(np.int64)
    gcs = _u64(cd.compress(_dev64(src.data_ptr() + offs), _dev64(sizes), _dev64(dst.data_ptr() + doffs), _dev64(bounds),
                           max_symbol_value=0 if cd.wide else 255, table_log=12))
    gd = dst.cpu().numpy()
    blocks, csizes, caps = [], [], []
    for i, n in enumerate(sizes):
        c = np.array(want_b[i] if i % 2 == 0 else gd[doffs[i]: doffs[i] + int(gcs[i])], np.uint8)
        if len(c) < 2:
            continue
        k, cap = len(c), n
        mode = i % 8
        if mode == 1:
            k = int(rng.integers(1, len(c)))                              # truncated
        elif mode == 2:
            for _ in range(int(rng.integers(1, 4))):
                c[int(rng.integers(0, len(c)))] ^= int(rng.integers(1, 256))   # bit-flipped
        elif mode == 3:
            cap = n + int(rng.integers(1, 1000))                          # larger
        elif mode == 4:
            cap = n - 1                                                   # one short
        elif mode == 5 and i % 16 == 5:
            cap = 0
        blocks.append(c[:k]); csizes.append(k); caps.append(cap)
    c0 = blocks[0]
    for k, cap in ((0, 100), (1, 100), (0, 0), (1, 1), (2, 100), (3, 50)):
        blocks.append(c0[:k].copy()); csizes.append(k); caps.append(cap)
    return lib, blocks, csizes, caps


def run_decode_packed(cd, blocks, csizes, caps, c_odd=1, d_off=None):
    """compressed blocks back to back from an odd offset with 32 bytes of slack; outputs back to back (U16: at even offsets)"""
    import torch
    d_off = cd.w * 3 if d_off is None else d_off
    coffs = CANARY + c_odd + np.concatenate([[0], np.cumsum(csizes)[:-1]]).astype(np.int64)
    chost = np.full(CANARY + c_odd + sum(csizes) + 32, POISON, np.uint8)
    for o, c, k in zip(coffs, blocks, csizes):
        chost[o: o + k] = c[:k]
    doffs = CANARY + d_off + np.concatenate([[0], np.cumsum([c * cd.w for c in caps])[:-1]]).astype(np.int64)
    dhost = np.full(CANARY + d_off + sum(caps) * cd.w + CANARY, POISON, np.uint8)
    carena = torch.from_numpy(chost).cuda(); darena = torch.from_numpy(dhost).cuda()
    res = torch.full((len(blocks),), -7, dtype=torch.int64, device="cuda")
    cd.decompress(_dev64(carena.data_ptr() + coffs), _dev64(csizes), _dev64(darena.data_ptr() + doffs), _dev64(caps), results=res)
    torch.cuda.synchronize()
    d = darena.cpu().numpy()
    end = int(doffs[-1]) + caps[-1] * cd.w
    assert (d[:CANARY] == POISON).all() and (d[end:] == POISON).all(), "bytes outside the destinations were written"
    assert torch.equal(carena.cpu(), torch.from_numpy(chost))
    return _u64(res), [d[o: o + c * cd.w] for o, c in zip(doffs, caps)], carena.data_ptr() + coffs, darena.data_ptr() + doffs


def check_decode(cd, lib, blocks, csizes, caps, **kw):
    want = [cd.ref_decompress(lib, c, k, cap) for c, k, cap in zip(blocks, csizes, caps)]
    got, outs, caddrs, daddrs = run_decode_packed(cd, blocks, csizes, caps, **kw)
    bad = [(b, csizes[b], caps[b], int(got[b]), int(w[0])) for b, w in enumerate(want) if got[b] != w[0]]
    assert not bad, (cd.wide, bad[:8])
    for b, (v, o) in enumerate(want):
        if o is not None:
            assert np.array_equal(outs[b][: len(o)], o), (cd.wide, b, csizes[b], caps[b])
    return [w[0] for w in want], caddrs, daddrs


def decode_paths_of(cd, lib, blocks, csizes, caps, caddrs, daddrs):
    import ctypes as C
    paths = []
    for c, k, cap, ca, da in zip(blocks, csizes, caps, caddrs, daddrs):
        lo, hi = read_range(int(ca), k)
        rlo, rhi = readable_range(int(ca), k)
        assert rlo <= lo and hi <= rhi
        if k < 2:
            continue
        norm = (C.c_short * 300)()
        msv, tl = C.c_uint(286 if cd.wide else 255), C.c_uint(0)
        tmp = np.concatenate([c[:k], np.zeros(8, np.uint8)])
        h = lib.FSE_readNCount(norm, C.byref(msv), C.byref(tl), ptr(tmp), k)
        if is_error(h) or h >= k or tl.value > (13 if cd.wide else 12):
            continue
        paths.append(decode_path(c, k, h, tl.value, int(da), int(ca), cap, cd.wide))
    return paths


@pytest.mark.parametrize("cd", [BYTES, U16], ids=["fse", "u16"])
def test_packed_decode(cd):
    lib, blocks, csizes, caps = decode_fixture(cd, seed=21 + cd.wide, count=500)
    want, caddrs, daddrs = check_decode(cd, lib, blocks, csizes, caps)
    kinds = {"err" if is_error(int(v)) else "size" for v in want}
    assert kinds == {"err", "size"}
    assert ERR_CORRUPT in [int(v) for v in want]
    small = want[-6:]
    if cd.wide:
        assert [int(v) for v in small[:4]] == [ERR_SRC_WRONG] * 4           # cSize < 2 (fseU16.c:317)
    else:
        assert [int(v) for v in small[:4]] == [ERR_CORRUPT] * 4             # cSize 0 / 1 are not "stored"
    paths = decode_paths_of(cd, lib, blocks, csizes, caps, caddrs, daddrs)
    assert paths.count("windowed") > 50 and paths.count("exact") > 20, (paths.count("windowed"), paths.count("exact"))


@pytest.mark.parametrize("cd", [BYTES, U16], ids=["fse", "u16"])
def test_packed_decode_aligned_outputs(cd):
    """outputs at 8-byte aligned offsets: the windowed loop for U16 blocks"""
    lib, blocks, csizes, caps = decode_fixture(cd, seed=31 + cd.wide, count=200)
    caps = [(c + 3) & ~3 for c in caps]
    _, caddrs, daddrs = check_decode(cd, lib, blocks, csizes, caps, c_odd=7, d_off=8)
    assert "windowed" in decode_paths_of(cd, lib, blocks, csizes, caps, caddrs, daddrs)


def test_u16_odd_addresses():
    """a U16 block whose symbols sit at an odd address gets GENERIC and nothing is written for it"""
    import torch
    sym = gen_u16(5000, 240, 0.5, 3)
    src = torch.zeros(2 * 5000 + 64, dtype=torch.uint8, device="cuda")
    src[1: 1 + 10000].copy_(torch.from_numpy(sym.view(np.uint8)))
    dst = torch.full((20000,), POISON, dtype=torch.uint8, device="cuda")
    for n in (0, 1, 5000):
        cs = U16.compress(_dev64([src.data_ptr() + 1]), _dev64([n]), _dev64([dst.data_ptr()]), _dev64([20000]))
        torch.cuda.synchronize()
        assert int(_u64(cs)[0]) == ERR_GENERIC and bool((dst == POISON).all())
    good = torch.from_numpy(sym.view(np.uint8).copy()).cuda()
    cs = U16.compress(_dev64([good.data_ptr()]), _dev64([5000]), _dev64([dst.data_ptr() + 1]), _dev64([19000]))   # compressed bytes: any address
    torch.cuda.synchronize()
    k = int(_u64(cs)[0])
    assert 1 < k < 10000
    out = torch.full((10016,), POISON, dtype=torch.uint8, device="cuda")
    res = U16.decompress(_dev64([dst.data_ptr() + 1]), _dev64([k]), _dev64([out.data_ptr() + 3]), _dev64([5000]))
    torch.cuda.synchronize()
    assert int(_u64(res)[0]) == ERR_GENERIC and bool((out == POISON).all())
    res = U16.decompress(_dev64([dst.data_ptr() + 1]), _dev64([k]), _dev64([out.data_ptr() + 2]), _dev64([5000]))
    torch.cuda.synchronize()
    assert int(_u64(res)[0]) == 5000 and np.array_equal(out.cpu().numpy()[2: 10002].view(np.uint16), sym)


# ---- equivalence, scale, limits ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("cd", [BYTES, U16], ids=["fse", "u16"])
def test_uniform_layout_equivalence(cd):
    """64 MiB of the bench inputs (FSE P80, U16 p50) through the uniform calls and the descriptor calls at base + b * blockSize"""
    import torch
    import finitestateentropy_b200 as fb
    block, total = 32768, 64 << 20
    nb = total // block
    if cd.wide:
        host = gen_u16(total // 2, 240, 0.5, 1).view(np.uint8)
        slot, msv = 32768, 0
        cbuf, cs = fb.fseu16_compress_batch(torch.from_numpy(host).cuda(), block, slot, msv, 12)
    else:
        host = probagen(total, 0.80)
        slot, msv = fb.compress_bound(block), 255
        cbuf, cs = fb.fse_compress_batch(torch.from_numpy(host).cuda(), block, slot, msv, 12)
    src = torch.from_numpy(host).cuda()
    b = np.arange(nb, dtype=np.int64)
    cbuf2 = torch.zeros_like(cbuf)
    cs2 = cd.compress(_dev64(src.data_ptr() + b * block), _dev64([block // cd.w] * nb), _dev64(cbuf2.data_ptr() + b * slot),
                      _dev64([slot] * nb), max_symbol_value=msv, table_log=12)
    torch.cuda.synchronize()
    assert torch.equal(cs, cs2)
    sizes = cs.cpu().numpy()
    assert (sizes > 1).all()
    mask = torch.from_numpy((np.arange(slot)[None, :] < sizes[:, None]).reshape(-1)).cuda()
    assert torch.equal(cbuf[: nb * slot][mask], cbuf2[: nb * slot][mask])
    dec = fb.fseu16_decompress_batch if cd.wide else fb.fse_decompress_batch
    out, res = dec(cbuf, cs, total, block, slot)
    out2 = torch.empty_like(out)
    res2 = cd.decompress(_dev64(cbuf.data_ptr() + b * slot), cs, _dev64(out2.data_ptr() + b * block), _dev64([block // cd.w] * nb))
    torch.cuda.synchronize()
    assert torch.equal(res // cd.w, res2) and torch.equal(out, out2) and torch.equal(out, src)


def test_large_mixed_batch():
    """40,000 blocks: several waves of both encode kernels, CTAs of mixed sizes, then all of them decoded back to back"""
    import torch
    rng = np.random.default_rng(41)
    lib = _ref()
    sizes = [64 * int(x) for x in rng.integers(1, 40, 20000)] + [int(x) for x in rng.integers(2, 2500, 20000)]
    sizes = [sizes[i] for i in rng.permutation(len(sizes))]
    host, offs = ragged_sources(BYTES, rng, sizes)
    want, outs, base = check_compress(BYTES, lib, host, offs, sizes, [fbound(n) for n in sizes], 255, 12)
    routes = [encode_route(base + o, n, False) for o, n in zip(offs, sizes)]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert routes.count("cta") > 4 * 16 * sms and routes.count("warp") > 4 * 12 * sms, (routes.count("cta"), routes.count("warp"))
    idx = [i for i, v in enumerate(want) if 1 < int(v) and not is_error(int(v))]
    check_decode(BYTES, lib, [outs[i] for i in idx], [int(want[i]) for i in idx], [sizes[i] for i in idx])


def test_limit_on_a_real_allocation():
    """2^30 + 2 bytes: srcSize_wrong for a 2^30 + 1-byte source, capacity and cSize, and for 2^29 + 1 U16 symbols, with no read
    outside the allocation"""
    import torch
    big = torch.zeros(FSE_BLOCK_MAX + 2, dtype=torch.uint8, device="cuda")
    dst = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    p, d = big.data_ptr(), dst.data_ptr()
    cs = BYTES.compress(_dev64([p, p]), _dev64([FSE_BLOCK_MAX + 1, 1000]), _dev64([d, d + 4096]), _dev64([1 << 20, 2000]))
    cs16 = U16.compress(_dev64([p]), _dev64([FSE_BLOCK_MAX // 2 + 1]), _dev64([d]), _dev64([1 << 20]))
    res = BYTES.decompress(_dev64([p, d]), _dev64([FSE_BLOCK_MAX + 1, 10]), _dev64([d + 8192, p]), _dev64([100, FSE_BLOCK_MAX + 1]))
    res16 = U16.decompress(_dev64([d]), _dev64([10]), _dev64([p]), _dev64([FSE_BLOCK_MAX // 2 + 1]))
    torch.cuda.synchronize()
    assert _u64(cs).tolist() == [ERR_SRC_WRONG, 1] and _u64(cs16).tolist() == [ERR_SRC_WRONG]
    assert _u64(res).tolist() == [ERR_SRC_WRONG, ERR_SRC_WRONG] and _u64(res16).tolist() == [ERR_SRC_WRONG]


def test_knob():
    """FSEB200_ENC_EK=8 (eight blocks per chain-warp CTA) in a child process"""
    _ref()
    e = dict(os.environ, FSEB200_ENC_EK="8")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child"], env=e, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0 and "child ok" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])


def test_arguments_and_wrappers():
    import torch
    import finitestateentropy_b200 as fb
    L = fb.lib()
    p = _dev64([0]).data_ptr()
    for codec in ("FSE", "FSEU16"):
        comp, dec = getattr(L, "FSEB200_%s_compress_blocks" % codec), getattr(L, "FSEB200_%s_decompress_blocks" % codec)
        assert comp(0, None, None, None, None, None, 255, 12, None) == 0 and dec(0, None, None, None, None, None, None) == 0
        for k in range(5):
            args = [p] * 5
            args[k] = None
            assert comp(1, *args, 255, 12, None) == ERR_SRC_WRONG and dec(1, *args, None) == ERR_SRC_WRONG
        assert comp(1 << 32, p, p, p, p, p, 255, 12, None) == ERR_SRC_WRONG and dec(1 << 32, p, p, p, p, p, None) == ERR_SRC_WRONG
        cs = torch.full((4,), -7, dtype=torch.int64, device="cuda")
        assert comp(0, p, p, cs.data_ptr(), p, p, 255, 12, None) == 0 and dec(0, p, p, cs.data_ptr(), p, p, None) == 0
        torch.cuda.synchronize()
        assert (cs == -7).all()
    # the wrappers on views, on a side stream; U16 sizes are symbols (block_pointers gives bytes)
    s = torch.cuda.Stream()
    for cd in (BYTES, U16):
        data = [torch.from_numpy((gen_u16(n, 240, 0.5, 2).view(np.uint8) if cd.wide else probagen(n, 0.5)).copy()).cuda()
                for n in (1000, 32768, 4099)]
        srcs, nbytes = fb.block_pointers(data)
        n = nbytes // cd.w
        dsts = [torch.zeros(fbound(int(k)), dtype=torch.uint8, device="cuda") for k in nbytes.tolist()]
        dp, dc = fb.block_pointers(dsts)
        with torch.cuda.stream(s):
            csz = cd.compress(srcs, n, dp, dc)
            outs = [torch.zeros_like(d) for d in data]
            op, _ = fb.block_pointers(outs)
            res = cd.decompress(dp, csz, op, n)
        s.synchronize()
        assert res.tolist() == n.tolist() and all(torch.equal(o, d) for o, d in zip(outs, data)), (cd.wide, res.tolist())


def _child():
    ragged_compress_check(BYTES, seed=51, count=300, subset_every=7)
    ragged_compress_check(U16, seed=52, count=300, subset_every=7)
    print("child ok")


if __name__ == "__main__" and "--child" in sys.argv:
    _child()
