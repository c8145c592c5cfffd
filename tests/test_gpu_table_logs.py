"""Every codec at every tableLog and maxSymbolValue it accepts, against the compiled reference.

CPU (no mark): the step-by-step FSE oracle of tests/table_logs.py is pinned against the reference's FSE_compress2 /
FSE_compressU16 on every request those can take safely (not raised, a workspace layout that fits) and against the oracle port on every request; the host
restatement of the Huff0 depth limiter is pinned against HUF_buildCTable; and the sweep's inputs are shown to reach the depth
limiter's branches, Huffman codes of 1 to 4 bits, FSE's -1 cells and second normalization method at every tableLog 5..12, and
the raw-weights tree header.

GPU (-m gpu): every compress entry point (uniform batch, per-block descriptors, one-block host calls) at tableLog 0..15, 255,
2^32-1 and maxSymbolValue 0, top-1, top, top+1, 254..256, 286, 287, 767, 768, 4095, 5632, 5633, 2^32-1, compared with the reference (or
the step-by-step oracle where the reference's block call is unsafe): return values, bytes [0, cSize), poisoned destinations with canaries;
then every decoder on those blocks and on the reference's, on truncated / bit-flipped blocks at tableLog 5..8 and on FSE-U16
streams whose header says tableLog 13."""
import ctypes as C
import functools
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from helpers import have_ref, is_error, load_port, load_ref, ptr, zoo, rand_size, gen_u16   # noqa: E402
import table_logs as T                                                                   # noqa: E402
from paths import read_stats                                                             # noqa: E402

needs_ref = pytest.mark.skipif(not have_ref(), reason="compiled reference (oracle/_ref) unavailable")

TOP = 15                                 # the largest symbol of most sweep blocks (small enough for maxNbBits / tableLog 5)
HUF_N, FSE_N, U16_N = 16384, 32768, 32768     # symbols per block: the smallest sizes at which tableLog 12 is not lowered


@functools.lru_cache(maxsize=None)
def huf_fixture():
    """built once per process and shared, hence a tuple"""
    rng = np.random.default_rng(41)
    return tuple(T.shaped_blocks(rng, HUF_N, TOP) + T.limiter_blocks(rng, HUF_N, TOP) + T.raw_weight_blocks(rng, HUF_N))


@functools.lru_cache(maxsize=None)
def fse_fixture():
    rng = np.random.default_rng(42)
    return tuple(T.shaped_blocks(rng, FSE_N, TOP) + T.m2_blocks(rng, FSE_N, TOP))


@functools.lru_cache(maxsize=None)
def u16_fixture():
    rng = np.random.default_rng(43)
    return tuple(T.shaped_blocks(rng, U16_N, TOP, wide=True) + T.m2_blocks(rng, U16_N, TOP, wide=True))


# ---- CPU: the step-by-step oracle ----------------------------------------------------------------------------------------------

def _pin_inputs(wide, count=120):
    rng = np.random.default_rng(7 + wide)
    out = []
    for i in range(count):
        n = rand_size(rng, 40000)
        if wide:
            out.append(gen_u16(n + 50, 240, float(rng.uniform(0.05, 0.9)), i + 1)[50:] if i % 3 else
                       rng.integers(0, int(rng.integers(1, 288)), n).astype(np.uint16))
        else:
            out.append(zoo(rng, n))
    blocks = u16_fixture() if wide else fse_fixture()
    return out + [b[: int(rng.integers(2, len(b) + 1))] for b in blocks[::3]]


def _pin_params(rng, top):
    tls = T.TABLE_LOGS
    msvs = T.msv_values(top)
    return [(int(rng.choice(msvs)), int(rng.choice(tls))) for _ in range(6)] + [(255, int(rng.integers(1, 13))), (T.M32, 12),
                                                                             (int(rng.integers(256, 768)), 12)]


@needs_ref
@pytest.mark.parametrize("wide", [False, True], ids=["fse", "u16"])
def test_steps_equal_reference_block_call_when_not_raised(wide):
    """the step-by-step oracle equals FSE_compress2 / FSE_compressU16 on every request those take safely: not raised and
    (bytes) with a workspace layout that fits, which includes maxSymbolValue 2^32-1 (the workspace test wraps it to 0)"""
    ref = load_ref()
    rng = np.random.default_rng(11 + wide)
    seen = {"plain": 0, "raised": 0}
    for d in _pin_inputs(wide):
        n = len(d)
        for msv, tl in _pin_params(rng, int(d.max()) if n else 0):
            cap = T.bound(n * (2 if wide else 1))
            if not T.ref_call_safe(ref, d, msv, tl, wide):
                seen["raised"] += 1
                continue                                # the reference's block call may fault here: never called
            seen["plain"] += 1
            want = (T.u16_steps if wide else T.fse_steps)(ref, cap, d, msv, tl)
            buf = np.zeros(cap + 16, np.uint8)
            v = (ref.FSE_compressU16 if wide else ref.FSE_compress2)(ptr(buf), cap, ptr(d), n, msv & T.M32, tl & T.M32)
            assert v == want[0], (n, msv, tl, v, want[0])
            if v > 1 and not is_error(v):
                assert bytes(buf[:v]) == want[1], (n, msv, tl)
    assert seen["plain"] > 200 and seen["raised"] > 100, seen


@needs_ref
@pytest.mark.parametrize("wide", [False, True], ids=["fse", "u16"])
def test_steps_equal_port_on_every_request(wide):
    """the step-by-step oracle equals the oracle port's orc_fse_compress2 / orc_fse_compress_u16 on every request, raised ones too"""
    ref, port = load_ref(), load_port()
    rng = np.random.default_rng(21 + wide)
    raised = 0
    for d in _pin_inputs(wide, 80):
        n = len(d)
        for msv, tl in _pin_params(rng, int(d.max()) if n else 0):
            cap = T.bound(n * (2 if wide else 1))
            want = (T.u16_steps if wide else T.fse_steps)(ref, cap, d, msv, tl)
            buf = np.zeros(cap + 16, np.uint8)
            v = (port.orc_fse_compress_u16 if wide else port.orc_fse_compress2)(ptr(buf), cap, ptr(d), n, msv & T.M32, tl & T.M32)
            assert v == want[0], (n, msv, tl, v, want[0])
            if v > 1 and not is_error(v):
                assert bytes(buf[:v]) == want[1], (n, msv, tl)
                raised += n > 0 and T.raised(ref, d, msv, tl)
    assert raised > 30


@needs_ref
def test_ncount_writer_equals_reference():
    """the host NCount writer (used for tableLog-13 headers, which the linked FSE_writeNCount refuses) equals FSE_writeNCount"""
    ref = load_ref()
    rng = np.random.default_rng(5)
    for it in range(300):
        k = int(rng.integers(2, 287))
        hist = (rng.pareto(1.0, k) * 50).astype(np.int64) + (rng.random(k) < 0.7)
        hist[-1] = max(hist[-1], 1)
        n = int(hist.sum())
        tl = int(rng.integers(5, 13))
        if n < 2 or hist.max() == n:
            continue
        tl = ref.FSE_optimalTableLog(tl, n, k - 1)
        norm = (C.c_short * 300)()
        cnt = (T.U * 300)(*map(int, hist))
        if is_error(ref.FSE_normalizeCount(norm, tl, cnt, n, k - 1)):
            continue
        buf = np.zeros(600, np.uint8)
        h = ref.FSE_writeNCount(ptr(buf), 600, norm, k - 1, tl)
        assert T.write_ncount(list(norm), k - 1, tl) == bytes(buf[:h]), (it, tl)


# ---- CPU: the depth limiter and the inputs' coverage ----------------------------------------------------------------------------

def _hist(block, size):
    return np.bincount(block, minlength=size)


@needs_ref
def test_depth_limiter_restatement_equals_reference():
    """huf_limit_trace's code lengths equal HUF_buildCTable's at every maxNbBits the tree fits"""
    ref = load_ref()
    for b in list(huf_fixture()) + [x[:HUF_N // 3] for x in huf_fixture()]:
        h = _hist(b, 256)
        msv = int(np.nonzero(h)[0].max())
        if (h > 0).sum() < 2:
            continue
        cnt = (T.U * 256)(*map(int, h))
        for mb in range(1, 13):
            if (1 << mb) < (h > 0).sum():
                continue                                # the tree cannot fit: the reference loops
            ct = np.zeros(256, np.uint32)
            r = ref.HUF_buildCTable(ptr(ct), cnt, msv, mb)
            lengths, _ = T.huf_limit_trace(h, msv, mb)
            assert list((ct[:msv + 1] >> 16) & 0xFF) == lengths, (msv, mb)
            assert r == max(lengths) or is_error(r)


def huf_branches_per_max_bits(blocks):
    """{maxNbBits: set of branch signatures} over the blocks compressed at every requested tableLog of the sweep (the
    maxNbBits HUF_compress2 builds with is HUF_optimalTableLog(request))"""
    ref = load_ref()
    out = {}
    for b in blocks:
        h = _hist(b, 256)
        top = int(np.nonzero(h)[0].max())
        if (h > 0).sum() < 2:
            continue
        for tl in range(1, 13):
            for msv in (top, 255):
                mb = ref.HUF_optimalTableLog(tl, len(b), msv)
                if (1 << mb) < (h > 0).sum():
                    continue
                _, br = T.huf_limit_trace(h, top, mb)
                sig = "none" if br == {"none"} else "repay_only" if br == {"repay"} else \
                      "giveback_new_rank1" if "giveback_new_rank1" in br else "giveback" if "giveback" in br else "?"
                out.setdefault(mb, set()).add(sig)
    return out


@needs_ref
def test_inputs_reach_parameter_dependent_paths():
    ref = load_ref()
    hb = huf_fixture()
    got = huf_branches_per_max_bits(hb)
    for mb in range(5, 13):
        assert {"none", "repay_only", "giveback", "giveback_new_rank1"} <= got.get(mb, set()), (mb, got.get(mb))
    longest = set()
    for b in hb:
        h = _hist(b, 256)
        if (h > 0).sum() >= 2:
            longest.add(max(T.huf_limit_trace(h, int(np.nonzero(h)[0].max()), 12)[0]))
    assert {1, 2, 3, 4} <= longest, longest
    # FSE: -1 cells and the second normalization method at every tableLog 5..12, bytes and U16
    for blocks, size in ((fse_fixture(), 256), (u16_fixture(), 287)):
        minus1, m2 = set(), set()
        for b in blocks:
            h = _hist(b, size)
            top = int(np.nonzero(h)[0].max())
            if h.max() == len(b):
                continue
            for tl in range(1, 13):
                t = ref.FSE_optimalTableLog(tl, len(b), top)
                a, m = T.normalize_method(h, len(b), top, t)
                if a: minus1.add(t)
                if m: m2.add(t)
        assert set(range(5, 13)) <= minus1 and set(range(5, 13)) <= m2, (size, sorted(minus1), sorted(m2))
    # raw-weights tree headers: a compressed block at 128 symbols, GENERIC at 192 (raw weights above 128 symbols)
    verdicts = []
    for b in T.raw_weight_blocks(np.random.default_rng(1), HUF_N):
        buf = np.zeros(T.bound(HUF_N), np.uint8)
        verdicts.append(ref.HUF_compress2(ptr(buf), len(buf), ptr(b), HUF_N, 255, 11))
    assert not is_error(verdicts[0]) and verdicts[0] > 1 and verdicts[1] == T.ERR_GENERIC, verdicts


# ---- GPU: the sweep ----------------------------------------------------------------------------------------------------------

PARAMS = [(tl, msv) for tl in T.TABLE_LOGS for msv in T.msv_values(TOP)]
# the one-block host calls run every tableLog at three maxSymbolValue values and every maxSymbolValue at three tableLogs
HOST_PARAMS = sorted({(tl, msv) for tl in T.TABLE_LOGS for msv in (0, TOP, 255)} |
                     {(tl, msv) for tl in (0, 5, 12) for msv in T.msv_values(TOP)})
FIXTURE = {"huf": (huf_fixture, 1), "huf1x": (huf_fixture, 1), "fse": (fse_fixture, 1), "u16": (u16_fixture, 2)}


def _host_sigs(lib, names):
    sz, vp, u = C.c_size_t, C.c_void_p, C.c_uint
    for name in names:
        f = getattr(lib, name)
        f.restype = sz
        f.argtypes = [vp, sz, vp, sz, u, u] if "compress" in name and "decompress" not in name else \
                     ([vp, vp, sz, vp, sz] if name.endswith("DCtx") else [vp, sz, vp, sz])
    return lib


def _ref_lib():
    ref = load_ref()
    return _host_sigs(ref, ["HUF_compress1X", "HUF_decompress1X1", "HUF_decompress1X_DCtx"])


def expect(codec, ref, data, cap, msv, tl):
    """(value, bytes the block keeps) of the reference for one block: its block call, or the step-by-step oracle where that
    call is not safe (FSE / U16 requests that are raised or whose workspace layout overflows)"""
    wide = codec == "u16"
    if codec in ("fse", "u16") and not T.ref_call_safe(ref, data, msv, tl, wide):
        return (T.u16_steps if wide else T.fse_steps)(ref, cap, data, msv, tl)
    fn = {"huf": ref.HUF_compress2, "huf1x": ref.HUF_compress1X, "fse": ref.FSE_compress2, "u16": ref.FSE_compressU16}[codec]
    buf = np.zeros(cap + 16, np.uint8)
    v = fn(ptr(buf), cap, ptr(data), len(data), msv, tl)
    keep = 0 if is_error(v) else (v if v > 1 or codec.startswith("huf") else 0)
    return v, bytes(buf[:keep])


def ref_decode(codec, ref, c, n):
    """(value, output) of the reference's decoder for one compressed block of n symbols"""
    w = 2 if codec == "u16" else 1
    tmp = np.concatenate([np.frombuffer(bytes(c), np.uint8), np.zeros(64, np.uint8)])
    o = np.zeros(n * w + 64, np.uint8)
    if codec == "huf1x":
        dt = np.zeros(1 + 4096, np.uint32); dt[0] = 12 * 0x01000001
        v = ref.HUF_decompress1X_DCtx(ptr(dt), ptr(o), n, ptr(tmp), len(c))
    else:
        v = {"huf": ref.HUF_decompress, "fse": ref.FSE_decompress, "u16": ref.FSE_decompressU16}[codec](ptr(o), n, ptr(tmp), len(c))
    return v, (None if is_error(v) else o[: v * w].copy())


class Seen:
    """what the sweep contains: effective tableLog per codec, raised requests, verdicts"""
    def __init__(self):
        self.tl, self.raised, self.verdicts = {}, 0, set()

    def note(self, codec, ref, data, msv, tl, v, b):
        self.verdicts.add((codec, v if is_error(v) else "size" if v > 1 else v))
        if is_error(v) or v < 2:
            return
        if codec.startswith("huf"):
            st = read_stats(np.frombuffer(b, np.uint8))
            if st is not None:
                self.tl.setdefault(codec, set()).add(st[1])
        else:
            norm = (C.c_short * 300)()
            m, t = T.U(286 if codec == "u16" else 255), T.U(0)
            hb = np.concatenate([np.frombuffer(b, np.uint8), np.zeros(8, np.uint8)])
            if not is_error(ref.FSE_readNCount(norm, C.byref(m), C.byref(t), ptr(hb), len(b))):
                self.tl.setdefault(codec, set()).add(t.value)
            self.raised += codec == "fse" and T.raised(ref, data, msv, tl)


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("codec", ["huf", "fse", "u16"])
def test_uniform_batch_every_parameter(codec):
    """*_compress_batch at every (tableLog, maxSymbolValue) of the sweep into poisoned slots pre-filled with the complement of
    the expected bytes, then *_decompress_batch on its own slots, against the reference"""
    import torch
    import finitestateentropy_b200 as fb
    from gpu_common import CANARY, POISON, cpu_decompress
    ref = _ref_lib()
    make, w = FIXTURE[codec]
    blocks = make()
    block = len(blocks[0]) * w
    data = np.concatenate([b.view(np.uint8) for b in blocks])
    nb, slot = len(blocks), T.bound(block)
    enc = {"huf": fb.huf_compress_batch, "fse": fb.fse_compress_batch, "u16": fb.fseu16_compress_batch}[codec]
    dec = {"huf": fb.huf_decompress_batch, "fse": fb.fse_decompress_batch, "u16": fb.fseu16_decompress_batch}[codec]
    src_a = torch.full((len(data) + 2 * CANARY,), POISON, dtype=torch.uint8, device="cuda")
    src = src_a[CANARY: CANARY + len(data)]
    src.copy_(torch.from_numpy(data))
    c_a = torch.full((nb * slot + 2 * CANARY,), POISON, dtype=torch.uint8, device="cuda")
    c_v = c_a[CANARY: CANARY + nb * slot]
    o_a = torch.full((len(data) + 2 * CANARY,), POISON, dtype=torch.uint8, device="cuda")
    o_v = o_a[CANARY: CANARY + len(data)]
    seen, decoded = Seen(), set()
    for tl, msv in PARAMS:
        want_cs = np.zeros(nb, np.uint64)
        want_c = np.zeros(nb * slot, np.uint8)
        for i, b in enumerate(blocks):
            v, bb = expect(codec, ref, b, slot, msv, tl)
            want_cs[i] = v
            want_c[i * slot: i * slot + len(bb)] = np.frombuffer(bb, np.uint8)
            seen.note(codec, ref, b, msv, tl, v, bb)
        c_v.copy_(torch.from_numpy(~want_c).cuda())
        cs = torch.full((nb,), -7, dtype=torch.int64, device="cuda")
        enc(src, block, slot, msv, tl, cbuf=c_v, csizes=cs)
        got_cs = cs.cpu().numpy().view(np.uint64)
        assert np.array_equal(got_cs, want_cs), (codec, tl, msv, [(i, int(got_cs[i]), int(want_cs[i])) for i in range(nb) if got_cs[i] != want_cs[i]][:5])
        got_c = c_v.cpu().numpy()
        for i in range(nb):
            k = 0 if is_error(int(want_cs[i])) else int(want_cs[i]) if (want_cs[i] > 1 or codec == "huf") else 0
            assert np.array_equal(got_c[i * slot: i * slot + k], want_c[i * slot: i * slot + k]), (codec, tl, msv, i)
        key = want_c.tobytes() + want_cs.tobytes()
        if hash(key) in decoded:
            continue
        decoded.add(hash(key))
        want_out, want_res = cpu_decompress(codec, want_c, want_cs, data, block=block, slot=slot)
        o_v.copy_(torch.from_numpy(~want_out).cuda())
        res = torch.full((nb,), -7, dtype=torch.int64, device="cuda")
        dec(c_v, cs, len(data), block, slot, out=o_v, results=res, orig=src)
        got_res = res.cpu().numpy().view(np.uint64)
        got_out = o_v.cpu().numpy()
        for i in range(nb):
            if is_error(int(want_cs[i])):
                continue
            assert got_res[i] == want_res[i], (codec, tl, msv, i, int(got_res[i]), int(want_res[i]))
            if not is_error(int(want_res[i])):
                assert np.array_equal(got_out[i * block: (i + 1) * block], want_out[i * block: (i + 1) * block]), (codec, tl, msv, i)
    torch.cuda.synchronize()
    for a, k in ((src_a, len(data)), (c_a, nb * slot), (o_a, len(data))):
        assert bool((a[:CANARY] == POISON).all()) and bool((a[CANARY + k:] == POISON).all()), (codec, "canary")
    assert set(range(5, 13)) <= seen.tl[codec], (codec, sorted(seen.tl[codec]))
    if codec == "fse":
        assert seen.raised > 0 and ("fse", T.ERR_WKSP_SMALL) in seen.verdicts
    if codec == "huf":
        assert ("huf", T.ERR_GENERIC) in seen.verdicts


def _corrupt_set(rng, codec, ref, blocks, sizes):
    """truncated and bit-flipped copies of the blocks whose header says tableLog 5 to 8"""
    out = []
    for c, n in zip(blocks, sizes):
        if len(c) < 4:
            continue
        if codec.startswith("huf"):
            st = read_stats(np.asarray(c, np.uint8))
            t = None if st is None else st[1]
        else:
            norm = (C.c_short * 300)()
            m, tt = T.U(286), T.U(0)
            hb = np.concatenate([np.asarray(c, np.uint8), np.zeros(8, np.uint8)])
            t = None if is_error(ref.FSE_readNCount(norm, C.byref(m), C.byref(tt), ptr(hb), len(c))) else tt.value
        if t is None or not 5 <= t <= 8:
            continue
        for mode in range(3):
            b = np.array(c, np.uint8)
            if mode == 0:
                b = b[: int(rng.integers(1, len(b)))]
            else:
                for _ in range(mode):
                    b[int(rng.integers(0, len(b)))] ^= 1 << int(rng.integers(0, 8))
            out.append((b, n))
    return out


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("codec", ["huf", "huf1x", "fse", "u16"])
def test_descriptors_every_parameter(codec):
    """the per-block descriptor compress at every (tableLog, maxSymbolValue) of the sweep, blocks at ragged offsets into
    poisoned destinations with gaps; then the descriptor decoder on every distinct block the sweep produced, the reference's
    bytes, truncated / bit-flipped blocks at tableLog 5..8 and (U16) streams whose header says tableLog 13"""
    import test_gpu_blocks as B4
    import test_gpu_blocks_1x as B1
    import test_gpu_fse_blocks as BF
    ref = _ref_lib()
    make, w = FIXTURE[codec]
    blocks = make()
    rng = np.random.default_rng(77)
    parts, offs, cur = [], [], B4.CANARY
    for b in blocks:
        gap = int(rng.integers(0, 40)) * w
        parts.append(np.full(gap, B4.POISON, np.uint8)); cur += gap
        offs.append(cur)
        parts.append(b.view(np.uint8)); cur += len(b) * w
    host = np.concatenate([np.full(B4.CANARY, B4.POISON, np.uint8)] + parts + [np.full(B4.CANARY + 64, B4.POISON, np.uint8)])
    sizes = [len(b) for b in blocks]
    caps = [T.bound(n * w) for n in sizes]
    seen, distinct = Seen(), {}
    cd = BF.U16 if codec == "u16" else BF.BYTES
    for tl, msv in PARAMS:
        want = [expect(codec, ref, b, cap, msv, tl) for b, cap in zip(blocks, caps)]
        if codec == "huf":
            got, got_b, untouched = B4.run_compress(host, offs, sizes, caps, msv, tl)
        elif codec == "huf1x":
            got, got_b, untouched = B1.run_compress1x(host, offs, sizes, caps, msv, tl)
        else:
            got, got_b, _ = BF.run_compress(cd, host, offs, sizes, caps, msv, tl)
            untouched = True                           # run_compress asserts it
        bad = [(i, int(got[i]), int(v)) for i, (v, _) in enumerate(want) if got[i] != v]
        assert not bad, (codec, tl, msv, bad[:6])
        for i, (v, bb) in enumerate(want):
            assert bytes(got_b[i][: len(bb)]) == bb, (codec, tl, msv, i)
            seen.note(codec, ref, blocks[i], msv, tl, v, bb)
            if len(bb) > 1:
                distinct.setdefault(bb, sizes[i])
        assert untouched, "bytes outside the destinations were written"
    assert set(range(5, 13)) <= seen.tl[codec], (codec, sorted(seen.tl[codec]))
    # decode: every distinct compressed block, corrupted ones at small tables, and tableLog-13 U16 streams
    cblocks = [np.frombuffer(b, np.uint8).copy() for b in distinct]
    dsizes = list(distinct.values())
    for b, n in _corrupt_set(rng, codec, ref, cblocks, dsizes):
        cblocks.append(b); dsizes.append(n)
    if codec == "u16":
        for b in blocks[::4]:
            if len(np.unique(b)) > 1:
                cblocks.append(T.u16_tl13_stream(ref, b)); dsizes.append(len(b))
    csz = [len(c) for c in cblocks]
    if codec == "huf":
        B4.check_decode(ref, cblocks, csz, dsizes)
    elif codec == "huf1x":
        B1.check_decode1x(ref, cblocks, csz, dsizes)
    else:
        want, _, _ = BF.check_decode(cd, ref, cblocks, csz, dsizes)
        if codec == "u16":
            n13 = sum(1 for b in blocks[::4] if len(np.unique(b)) > 1)
            assert n13 > 5 and all(not is_error(int(v)) for v in want[-n13:])   # the reference decodes them


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("codec", ["huf", "huf1x", "fse", "u16"])
def test_one_block_host_calls(codec):
    """HUF_compress2 / HUF_compress1X / FSE_compress2 / FSE_compressU16 of this library (host pointers, one block a call) at
    every tableLog and every maxSymbolValue, then its HUF_decompress / HUF_decompress1X1 / FSE_decompress / FSE_decompressU16 on
    the result, each against the reference; destinations are poisoned beyond the capacity"""
    import finitestateentropy_b200 as fb
    ref = _ref_lib()
    L = _host_sigs(fb.lib(), ["HUF_compress2", "HUF_compress1X", "FSE_compress2", "FSE_compressU16",
                              "HUF_decompress", "HUF_decompress1X1", "FSE_decompress", "FSE_decompressU16"])
    enc = {"huf": L.HUF_compress2, "huf1x": L.HUF_compress1X, "fse": L.FSE_compress2, "u16": L.FSE_compressU16}[codec]
    dec = {"huf": L.HUF_decompress, "huf1x": L.HUF_decompress1X1, "fse": L.FSE_decompress, "u16": L.FSE_decompressU16}[codec]
    make, w = FIXTURE[codec]
    blocks = make()[::4]
    done = set()
    for tl, msv in HOST_PARAMS:
        for i, b in enumerate(blocks):
            cap = T.bound(len(b) * w)
            v, bb = expect(codec, ref, b, cap, msv, tl)
            buf = np.full(cap + 64, 0x5A, np.uint8)
            got = enc(ptr(buf), cap, ptr(b), len(b), msv, tl)
            assert got == v, (codec, tl, msv, i, got, v)
            assert bytes(buf[: len(bb)]) == bb and (buf[cap:] == 0x5A).all(), (codec, tl, msv, i)
            if len(bb) < 2 or bb in done:
                continue
            done.add(bb)
            if codec == "huf1x":
                o = np.zeros(len(b) + 64, np.uint8)
                tmp = np.concatenate([np.frombuffer(bb, np.uint8), np.zeros(64, np.uint8)])
                wv = ref.HUF_decompress1X1(ptr(o), len(b), ptr(tmp), len(bb))
                wo = None if is_error(wv) else o[: len(b)].copy()
            else:
                wv, wo = ref_decode(codec, ref, bb, len(b))
            out = np.full(len(b) * w + 64, 0x5A, np.uint8)
            src = np.concatenate([np.frombuffer(bb, np.uint8), np.zeros(64, np.uint8)])
            gv = dec(ptr(out), len(b), ptr(src), len(bb))
            assert gv == wv, (codec, tl, msv, i, gv, wv)
            assert (out[len(b) * w:] == 0x5A).all()
            if wo is not None:
                assert np.array_equal(out[: len(wo)], wo), (codec, tl, msv, i)
