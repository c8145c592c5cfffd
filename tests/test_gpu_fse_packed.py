"""Packed FSE and FSE-U16 (FSEB200_FSE{,U16}_{compress,decompress}_packed) against the compiled reference (-m gpu): the whole
output buffer, the offsets and the values are compared with the packed image the host model (tests/fse_packed_paths.py) builds
from FSE_compress2 / FSE_compressU16 at FSE_compressBound, with poisoned canaries around dOut and around dWork at workSize.
Layouts: 32 KB bench blocks, ragged 1 B - 128 KiB with overlapping sources, the special sizes, all-raw, all-RLE and mixed;
every output offset mod 16 the copy branches on; capacities that cut the stream; workspaces at the bound, one byte short, the
helper's size and 0; bad parameters and the limits; offsets above 2^32; the round trip and malformed stored lengths through the
decompress call, with destination canaries; the Python wrappers and the calls' argument checks.

Run as a script (`python tests/test_gpu_fse_packed.py --child`) it repeats a ragged subset under the environment it was started
with: test_knob starts it with FSEB200_ENC_EK=8."""
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from helpers import gen_u16, is_error, probagen                                           # noqa: E402
from test_gpu_blocks import CANARY, POISON, _dev64, _ref, _u64                            # noqa: E402
from test_gpu_fse_blocks import BYTES, SPECIAL, U16, ragged_sources                       # noqa: E402
from fse_packed_paths import (ERR_DST_TOO_SMALL, ERR_GENERIC, ERR_SRC_WRONG, ERR_WKSP_TOO_SMALL, FSE_BLOCK_MAX,   # noqa: E402
                              decode_rule, fbound, image, limit_value, ref_unpack, ref_value, slots, stored_len, values, workspace)

pytestmark = pytest.mark.gpu

CODECS = [BYTES, U16]
CODEC_IDS = ["FSE", "U16"]
OUT_OFFSETS = [0, 1, 4, 8, 16, 32, 64, 96]


def _msv(cd):
    return 0 if cd.wide else 255


def reference(cd, host, offs, sizes, msv=None, tl=12):
    """(values, stored bytes) per block from the reference; the limits' verdicts for blocks they settle"""
    lib = _ref()
    msv = _msv(cd) if msv is None else msv
    vals, stored = [], []
    for o, n in zip(offs, sizes):
        lv = limit_value(o, n, cd.wide)
        if lv is not None:
            vals.append(lv); stored.append(np.zeros(0, np.uint8))
            continue
        src = host[o: o + n * cd.w]
        v, st = ref_value(lib, src.view(np.uint16) if cd.wide else src, cd.wide, msv, tl)
        vals.append(v); stored.append(st)
    return vals, stored


def coded_bytes(cd, offs, sizes):
    return sum(n * cd.w for o, n in zip(offs, sizes) if limit_value(o, n, cd.wide) is None)


def run_packed(cd, src, offs, sizes, cap, out_off, work_size, msv, tl):
    """the packed compress on the GPU into a poisoned arena (dOut at out_off from a 512-byte aligned start) with a poisoned
    workspace arena: (offsets, values, output arena, dOut's index).  Nothing beyond dWork + workSize may change."""
    import torch
    import finitestateentropy_b200 as fb
    arena = torch.full((CANARY + 512 + 96 + cap + CANARY,), POISON, dtype=torch.uint8, device="cuda")
    o = ((arena.data_ptr() + CANARY + 511) & ~511) + out_off - arena.data_ptr()
    warena = torch.full((CANARY + 512 + work_size + CANARY,), POISON, dtype=torch.uint8, device="cuda")
    wo = ((warena.data_ptr() + CANARY + 511) & ~511) + 3 - warena.data_ptr()
    offsets = torch.full((len(sizes) + 1,), -7, dtype=torch.int64, device="cuda")
    cs = torch.full((len(sizes),), -7, dtype=torch.int64, device="cuda")
    sp, sn = _dev64([src.data_ptr() + x for x in offs]), _dev64(sizes)
    fn = fb.lib().FSEB200_FSEU16_compress_packed if cd.wide else fb.lib().FSEB200_FSE_compress_packed
    r = fn(len(sizes), arena.data_ptr() + o, cap, offsets.data_ptr(), cs.data_ptr(), sp.data_ptr(), sn.data_ptr(), msv, tl,
           warena.data_ptr() + wo, work_size, torch.cuda.current_stream().cuda_stream)
    assert r == 0, r
    torch.cuda.synchronize()
    w = warena.cpu().numpy()
    assert bool((w[:wo] == POISON).all()) and bool((w[wo + work_size:] == POISON).all()), "dWork beyond workSize was touched"
    return _u64(offsets), _u64(cs), arena, o


def check_packed(cd, host, offs, sizes, ref, cap=None, out_off=0, work=None, msv=None, tl=12, src=None):
    """the GPU's offsets, values and whole output buffer against the model's; nothing written outside the stored blocks.
    Returns (offsets, final values, output arena, dOut's index, the model's image)."""
    import torch
    msv = _msv(cd) if msv is None else msv
    nbytes = coded_bytes(cd, offs, sizes)
    cap = nbytes if cap is None else cap
    work = workspace(len(sizes), nbytes) if work is None else work
    vals = values(ref[0], offs, sizes, cd.wide, work)
    stored = [s if int(v) == int(r) else s[:0] for s, v, r in zip(ref[1], vals, ref[0])]
    img, written, want_offs, want_final = image(vals, stored, sizes, cap, cd.wide)
    src = torch.from_numpy(host).cuda() if src is None else src
    got_offs, got_cs, arena, o = run_packed(cd, src, offs, sizes, cap, out_off, work, msv, tl)
    assert [int(x) for x in got_offs] == want_offs, (cd.wide, cap, out_off, work)
    bad = [(b, sizes[b], int(got_cs[b]), want_final[b]) for b in range(len(sizes)) if int(got_cs[b]) != want_final[b]]
    assert not bad, (cd.wide, cap, out_off, work, bad[:8])
    a = arena.cpu().numpy()
    end = min(want_offs[-1], cap)
    region = a[o: o + end]
    assert np.array_equal(region[written], img[written]), (cd.wide, cap, out_off)
    assert bool((region[~written] == POISON).all()), "bytes of a block that does not fit were written"
    assert bool((a[:o] == POISON).all()) and bool((a[o + end:] == POISON).all()), "bytes outside the packed blocks were written"
    assert torch.equal(src.cpu(), torch.from_numpy(host))               # sources are read only
    return want_offs, want_final, arena, o, img


def unpack(cd, packed, offsets, sizes, dst_odd=()):
    """the packed decompress of every block into a poisoned destination arena (block b at an odd address if b in dst_odd):
    (results, arena bytes, destination indices)"""
    import torch
    import finitestateentropy_b200 as fb
    regions = [n * cd.w if n * cd.w <= FSE_BLOCK_MAX else 0 for n in sizes]
    doffs, cur = [], CANARY
    for b, r in enumerate(regions):
        cur += cur & 1                                                  # arena indices have the parity of the addresses
        doffs.append(cur + (1 if b in dst_odd else 0))
        cur = doffs[-1] + r + 32
    darena = torch.full((cur + CANARY,), POISON, dtype=torch.uint8, device="cuda")
    res = torch.full((len(sizes),), -7, dtype=torch.int64, device="cuda")
    fn = fb.fseu16_decompress_packed if cd.wide else fb.fse_decompress_packed
    fn(packed, offsets, _dev64([darena.data_ptr() + d for d in doffs]), _dev64(sizes), results=res)
    torch.cuda.synchronize()
    return _u64(res), darena.cpu().numpy(), doffs


def check_unpack(cd, packed_np, packed_dev, offs_list, sizes, host=None, src_offs=None, dst_odd=()):
    """the decompress call on a packed buffer against ref_unpack block by block.  Nothing is written outside the destinations,
    nor for a block the decoder did not run on; a block it rejects may leave bytes in its own destination.  Returns the results."""
    import torch
    lib = _ref()
    offsets = torch.tensor(offs_list, dtype=torch.int64, device="cuda")
    got, d, doffs = unpack(cd, packed_dev, offsets, sizes, dst_odd)
    pad = np.concatenate([packed_np, np.zeros(64, np.uint8)])
    allowed = np.zeros(len(d), bool)
    for b, n in enumerate(sizes):
        L = offs_list[b + 1] - offs_list[b]
        want, out = ref_unpack(lib, pad[offs_list[b]:] if L <= FSE_BLOCK_MAX else pad[:0], L, n, cd.wide, doffs[b])
        assert int(got[b]) == want, (cd.wide, b, n, L, int(got[b]), want)
        if out is not None:
            assert np.array_equal(d[doffs[b]: doffs[b] + len(out)], out), (cd.wide, b, n, L)
            if host is not None:
                assert np.array_equal(out, host[src_offs[b]: src_offs[b] + n * cd.w]), (cd.wide, b)
            allowed[doffs[b]: doffs[b] + len(out)] = True
        elif L > 0 and decode_rule(L, n, doffs[b], cd.wide) == "decode":
            allowed[doffs[b]: doffs[b] + n * cd.w] = True
    assert bool((d[~allowed] == POISON).all()), "bytes outside the regenerated blocks were written"
    return got


def round_trip(cd, host, offs, sizes, want_offs, final, arena, o, img):
    """the decompress call on the GPU's packed buffer and on the model's image (uploaded): every block regenerates its source,
    with the result n, except those whose value is an error (nothing stored: L == 0)"""
    import torch
    end = want_offs[-1]
    assert len(img) == end
    for packed in (arena[o: o + end + 32], torch.from_numpy(np.concatenate([img, np.zeros(32, np.uint8)])).cuda()):
        got = check_unpack(cd, img, packed, want_offs, sizes, host, offs)
        for b, n in enumerate(sizes):
            if not is_error(final[b]):
                assert int(got[b]) == n, (cd.wide, b, n, final[b], int(got[b]))


def layout_check(cd, host, offs, sizes, kinds=None, out_off=0):
    ref = reference(cd, host, offs, sizes)
    if kinds is not None:
        got = {0 if v == 0 else 1 if v == 1 else "err" if is_error(v) else "size" for v in ref[0]}
        assert got >= kinds, got
    want_offs, final, arena, o, img = check_packed(cd, host, offs, sizes, ref, out_off=out_off)
    round_trip(cd, host, offs, sizes, want_offs, final, arena, o, img)
    return ref, want_offs, final


def back_to_back(cd, datas):
    """sources back to back (U16: even offsets), with canaries"""
    parts, offs, cur = [np.full(CANARY, POISON, np.uint8)], [], CANARY
    for d in datas:
        offs.append(cur); parts.append(d.view(np.uint8)); cur += d.nbytes
    parts.append(np.full(CANARY + 64, POISON, np.uint8))
    return np.concatenate(parts), offs


def ragged_fixture(cd, seed, count):
    rng = np.random.default_rng(seed)
    special = [s // cd.w for s in SPECIAL] if cd.wide else SPECIAL
    sizes = special + [int(x) for x in rng.integers(1, 131072 // cd.w + 1, count - len(special))]
    host, offs = ragged_sources(cd, rng, sizes)
    return host, offs, sizes


# ---- tests ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("cd", CODECS, ids=CODEC_IDS)
def test_bench_layout(cd):
    """64 blocks of 32 KB of the bench's input (FSE: probagen P80; U16: generateU16(240, 0.5))"""
    if cd.wide:
        data = gen_u16(64 * 16384, 240, 0.5, 1)
    else:
        data = probagen(64 * 32768, 0.80)
    host, offs = back_to_back(cd, [data])
    offs = [offs[0] + i * 32768 for i in range(64)]
    sizes = [32768 // cd.w] * 64
    ref, _, _ = layout_check(cd, host, offs, sizes)
    assert all(v > 1 and not is_error(v) for v in ref[0])


@pytest.mark.parametrize("cd", CODECS, ids=CODEC_IDS)
def test_ragged(cd):
    """special sizes and ragged ones of 1 B - 128 KiB, overlapping sources, mixed contents; the round trip; capacities"""
    host, offs, sizes = ragged_fixture(cd, 701 + cd.wide, 500)
    ref, want_offs, final = layout_check(cd, host, offs, sizes, kinds={0, 1, "size"})
    total = want_offs[-1]
    lens = [stored_len(v, n, cd.wide) for v, n in zip(ref[0], sizes)]
    src = None
    comp = [b for b in range(len(sizes)) if ref[0][b] > 1 and not is_error(ref[0][b])]
    cuts = [total - 1, 0, want_offs[comp[len(comp) // 2]] + lens[comp[len(comp) // 2]] // 2]
    raw = [b for b in range(len(sizes)) if ref[0][b] == 0 and lens[b] > 2]
    if raw:
        cuts.append(want_offs[raw[0]] + lens[raw[0]] // 2)
    for cap in cuts:
        _, fin, _, _, _ = check_packed(cd, host, offs, sizes, ref, cap=cap, out_off=cap % 16, src=src)
        assert (ERR_DST_TOO_SMALL in fin) == (cap < total), cap


@pytest.mark.parametrize("cd", CODECS, ids=CODEC_IDS)
def test_special_sizes(cd):
    """every special size of the descriptor tests with five contents each"""
    rng = np.random.default_rng(703 + cd.wide)
    special = [s // cd.w for s in SPECIAL] if cd.wide else SPECIAL
    datas = [cd.content(rng, n, i) for n in special for i in range(5)]
    host, offs = back_to_back(cd, datas)
    layout_check(cd, host, offs, [len(d) for d in datas])


def test_all_raw():
    """FSE: random bytes, every block raw (the copy from the source); U16: random 16-bit words, every block
    maxSymbolValue_tooSmall (nothing stored)"""
    rng = np.random.default_rng(704)
    sizes = [int(x) for x in rng.integers(1, 40000, 120)] + [0, 1, 2, 31, 32, 33]
    datas = [rng.integers(0, 256, n, dtype=np.uint8) for n in sizes]
    host, offs = back_to_back(BYTES, datas)
    ref, want_offs, _ = layout_check(BYTES, host, offs, sizes)
    assert all(v in (0, 1) for v in ref[0]) and ref[0].count(0) >= len(sizes) - 2 and want_offs[-1] > sum(sizes) - 8
    wdatas = [rng.integers(0, 65536, n).astype(np.uint16) for n in sizes]
    host, offs = back_to_back(U16, wdatas)
    ref, want_offs, _ = layout_check(U16, host, offs, sizes)
    assert all(is_error(v) for v, n in zip(ref[0], sizes) if n > 1) and want_offs[-1] == 2 * sum(n for n in sizes if n <= 1)


@pytest.mark.parametrize("cd", CODECS, ids=CODEC_IDS)
def test_all_rle(cd):
    rng = np.random.default_rng(705)
    sizes = [int(x) for x in rng.integers(2, 70000 // cd.w, 150)]
    datas = [np.full(n, int(rng.integers(0, 287 if cd.wide else 256)), np.uint16 if cd.wide else np.uint8) for n in sizes]
    host, offs = back_to_back(cd, datas)
    ref, want_offs, _ = layout_check(cd, host, offs, sizes)
    assert all(v == 1 for v in ref[0]) and want_offs[-1] == cd.w * len(sizes)


@pytest.mark.parametrize("cd", CODECS, ids=CODEC_IDS)
def test_mixed(cd):
    """raw, RLE, empty, one-symbol and compressed blocks interleaved, every content kind of the descriptor tests"""
    rng = np.random.default_rng(706)
    datas = []
    for i in range(300):
        n = int(rng.choice([0, 1, 2, 3, 64, 100, 4099, int(rng.integers(1, 131072 // cd.w))]))
        datas.append(cd.content(rng, n, i))
    host, offs = back_to_back(cd, datas)
    layout_check(cd, host, offs, [len(d) for d in datas], kinds={1, "size"})


@pytest.mark.parametrize("cd", CODECS, ids=CODEC_IDS)
def test_output_offsets(cd):
    """dOut at 0, 1, 4, 8, 16, 32, 64 and 96 from a 512-byte aligned start: every block's alignment changes with it"""
    import torch
    host, offs, sizes = ragged_fixture(cd, 707 + cd.wide, 120)
    ref = reference(cd, host, offs, sizes)
    src = torch.from_numpy(host).cuda()
    for off in OUT_OFFSETS:
        check_packed(cd, host, offs, sizes, ref, out_off=off, src=src)


@pytest.mark.parametrize("cd", CODECS, ids=CODEC_IDS)
def test_workspace_sizes(cd):
    """workSize at exactly the slots' sum, one byte short (workSpace_tooSmall for the last coded block only), the helper's
    value, a cut in the middle and 0; dWork beyond workSize is never touched"""
    import torch
    import finitestateentropy_b200 as fb
    host, offs, sizes = ragged_fixture(cd, 709 + cd.wide, 100)
    ref = reference(cd, host, offs, sizes)
    src = torch.from_numpy(host).cuda()
    exact = sum(fbound(n * cd.w) for o, n in zip(offs, sizes) if limit_value(o, n, cd.wide) is None)
    helper = int(fb.lib().FSEB200_FSE_packed_workspace(len(sizes), coded_bytes(cd, offs, sizes)))
    assert helper == fb.fse_packed_workspace(len(sizes), coded_bytes(cd, offs, sizes)) >= exact
    for work in (exact, exact - 1, helper, exact // 2, 0):
        _, fin, _, _, _ = check_packed(cd, host, offs, sizes, ref, work=work, src=src)
        _, coded = slots(offs, sizes, cd.wide, work)
        short = [b for b in range(len(sizes)) if fin[b] == ERR_WKSP_TOO_SMALL]
        assert short == [b for b in range(len(sizes)) if not coded[b] and limit_value(offs[b], sizes[b], cd.wide) is None]
        if work == exact - 1:
            assert short == [max(b for b in range(len(sizes)) if limit_value(offs[b], sizes[b], cd.wide) is None)]
        if work >= exact:
            assert not short


@pytest.mark.parametrize("cd", CODECS, ids=CODEC_IDS)
def test_parameters_and_limits(cd):
    """bad and unusual maxSymbolValue / tableLog (the reference's verdicts; error blocks store nothing), a U16 source at an
    odd address (GENERIC), and the 2^30 limit claimed by size over an overlapping source, which takes no slot"""
    import torch
    host, offs, sizes = ragged_fixture(cd, 711 + cd.wide, 60)
    src = torch.from_numpy(host).cuda()
    params = ((0, 11), (0, 0), (100, 12), (0, 14)) if cd.wide else ((255, 11), (0, 0), (200, 12), (255, 13), (256, 12))
    for msv, tl in params:
        ref = reference(cd, host, offs, sizes, msv, tl)
        check_packed(cd, host, offs, sizes, ref, msv=msv, tl=tl, out_off=1, src=src)
    # the limit: a block claiming 2^30 + 1 bytes (U16: 2^29 + 1 symbols) over the first source; U16: odd source addresses
    offs2 = list(offs) + [offs[0], offs[3]]
    sizes2 = list(sizes) + [FSE_BLOCK_MAX // cd.w + 1, 7]
    if cd.wide:
        offs2 += [offs[5] + 1, offs[6] + 3]
        sizes2 += [40, 1]
    order = list(np.random.default_rng(1).permutation(len(sizes2)))
    offs2, sizes2 = [offs2[i] for i in order], [sizes2[i] for i in order]
    ref = reference(cd, host, offs2, sizes2)
    assert ERR_SRC_WRONG in ref[0] and (ERR_GENERIC in ref[0]) == cd.wide
    want_offs, final, arena, o, img = check_packed(cd, host, offs2, sizes2, ref, src=src)
    exact = sum(fbound(n * cd.w) for oo, n in zip(offs2, sizes2) if limit_value(oo, n, cd.wide) is None)
    check_packed(cd, host, offs2, sizes2, ref, work=exact, src=src)    # the settled blocks take no slot


def test_offsets_above_4gib():
    """33,000 raw 128 KB FSE blocks that all read one random 128 KB source: offsets above 2^32, every block stored past 4 GiB;
    then the last blocks decoded from there"""
    import torch
    import finitestateentropy_b200 as fb
    n, count = 131072, 33000
    data = np.random.default_rng(712).integers(0, 256, n, dtype=np.uint8)
    assert ref_value(_ref(), data, False, 255, 12)[0] == 0
    src = torch.from_numpy(data).cuda()
    total = n * count
    assert total > 2 ** 32
    arena = torch.full((total + 2 * CANARY,), POISON, dtype=torch.uint8, device="cuda")
    out = arena[CANARY: CANARY + total]
    ptrs, sizes = _dev64([src.data_ptr()] * count), _dev64([n] * count)
    _, offsets, cs = fb.fse_compress_packed(ptrs, sizes, out=out)
    torch.cuda.synchronize()
    want = torch.arange(count + 1, dtype=torch.int64, device="cuda") * n
    assert torch.equal(offsets, want) and bool((cs == 0).all())
    blocks = out.view(count, n)
    assert bool((blocks == src).all())
    assert bool((arena[:CANARY] == POISON).all()) and bool((arena[CANARY + total:] == POISON).all())
    k = 40
    dst = torch.zeros(k * n, dtype=torch.uint8, device="cuda")
    dp = _dev64(dst.data_ptr() + n * np.arange(k))
    res = fb.fse_decompress_packed(out, offsets[-k - 1:].contiguous(), dp, sizes[:k].contiguous())
    torch.cuda.synchronize()
    assert bool((res == n).all()) and bool((dst.view(k, n) == src).all())


@pytest.mark.parametrize("cd", CODECS, ids=CODEC_IDS)
def test_decode_rules(cd):
    """malformed stored lengths that hit each decode rule -- raw, RLE, L == 0, truncated and bit-flipped compressed blocks,
    L and n above the limits -- and (U16) destinations at odd addresses, with destination canaries"""
    import torch
    rng = np.random.default_rng(713 + cd.wide)
    lib = _ref()
    pieces, sizes, odd = [], [], []
    for i in range(60):
        n = int(rng.integers(2, 5000))
        d = cd.content(rng, n, i % 3)
        v, st = ref_value(lib, d, cd.wide, _msv(cd), 12)
        mode = i % 10
        if mode == 0:
            piece = d.view(np.uint8).copy()                             # raw
        elif mode == 1:
            piece = d.view(np.uint8)[: cd.w].copy()                     # RLE of the first unit
        elif mode == 2:
            piece = np.zeros(0, np.uint8)                               # L == 0
        elif mode == 3 and v > 2 and not is_error(v):
            piece = st[: int(rng.integers(1, v))].copy()                # truncated
        elif mode == 4 and v > 2 and not is_error(v):
            piece = st.copy()
            piece[int(rng.integers(0, v))] ^= int(rng.integers(1, 256))  # bit-flipped
        elif mode == 5:
            piece = d.view(np.uint8)[: cd.w * n - 1].copy()             # one byte short of raw
        elif mode == 6 and cd.wide:
            piece = st.copy() if v > 1 and not is_error(v) else d.view(np.uint8).copy()
            odd.append(len(sizes))                                      # an odd destination
        else:
            piece = st.copy() if v > 1 and not is_error(v) else d.view(np.uint8)[: cd.w].copy()
        pieces.append(piece); sizes.append(n)
    sizes.append(FSE_BLOCK_MAX // cd.w + 1); pieces.append(np.zeros(5, np.uint8))   # n above the limit
    offs = [0]
    for p in pieces:
        offs.append(offs[-1] + len(p))
    packed = np.concatenate(pieces + [np.zeros(0, np.uint8)])
    dev = torch.from_numpy(np.concatenate([packed, np.zeros(32, np.uint8)])).cuda()
    got = check_unpack(cd, packed, dev, offs, sizes, dst_odd=set(odd))
    if cd.wide:
        assert all(int(got[b]) == ERR_GENERIC for b in odd) and odd
    assert int(got[-1]) == ERR_SRC_WRONG
    # L above the limit: a stored length of 2^30 + 1 over the same buffer (the decoder settles it without reading)
    got = check_unpack(cd, packed[:0], dev, [0, FSE_BLOCK_MAX + 1], [10])
    assert int(got[0]) == ERR_SRC_WRONG


def test_wrappers_and_arguments():
    import torch
    import finitestateentropy_b200 as fb
    L = fb.lib()
    a = _dev64([0, 0])
    p = a.data_ptr()
    for name in ("FSE", "FSEU16"):
        enc, dec = getattr(L, "FSEB200_%s_compress_packed" % name), getattr(L, "FSEB200_%s_decompress_packed" % name)
        assert enc(0, None, 0, None, None, None, None, 255, 12, None, 0, None) == 0
        assert dec(0, None, None, None, None, None, None) == 0
        for k in range(6):
            args = [p] * 6
            args[k] = None
            assert enc(1, args[0], 100, args[1], args[2], args[3], args[4], 255, 12, args[5], 100, None) == ERR_SRC_WRONG
        for k in range(5):
            args = [p] * 5
            args[k] = None
            assert dec(1, *args, None) == ERR_SRC_WRONG
        assert enc(1 << 32, p, 100, p, p, p, p, 255, 12, p, 100, None) == ERR_SRC_WRONG
        assert dec(1 << 32, p, p, p, p, p, None) == ERR_SRC_WRONG
        t = torch.full((4,), -7, dtype=torch.int64, device="cuda")
        assert enc(0, p, 100, t.data_ptr(), t.data_ptr(), p, p, 255, 12, p, 100, None) == 0      # writes nothing
        assert dec(0, p, p, t.data_ptr(), p, t.data_ptr(), None) == 0
        torch.cuda.synchronize()
        assert (t == -7).all()
    assert L.FSEB200_FSE_packed_workspace(3, 1000) == workspace(3, 1000) == fb.fse_packed_workspace(3, 1000)
    # the Python wrappers on views, on a side stream, allocating the output and the workspace
    lib = _ref()
    s = torch.cuda.Stream()
    for cd in CODECS:
        rng = np.random.default_rng(714)
        hs = [cd.content(rng, n, i) for i, n in enumerate([1000, 300, 777, 16384, 0, 1])]
        hs[1] = np.full(300, 7, hs[1].dtype)
        data = [torch.from_numpy(x.view(np.uint8).copy()).cuda() for x in hs]
        srcs, nb = fb.block_pointers(data)
        n = nb // cd.w
        enc = fb.fseu16_compress_packed if cd.wide else fb.fse_compress_packed
        dec = fb.fseu16_decompress_packed if cd.wide else fb.fse_decompress_packed
        with torch.cuda.stream(s):
            out, offsets, cs = enc(srcs, n)
            outs = [torch.zeros_like(d) for d in data]
            op, _ = fb.block_pointers(outs)
            res = dec(out, offsets, op, n)
        s.synchronize()
        assert out.numel() == int(nb.sum()) + 32 and offsets.numel() == 7 and cs.numel() == 6
        vals = [ref_value(lib, x, cd.wide, _msv(cd), 12)[0] for x in hs]
        assert [int(v) for v in _u64(cs)] == vals and vals[1] == 1
        assert res.tolist() == n.tolist() and all(torch.equal(o, d) for o, d in zip(outs, data))
        with pytest.raises(AssertionError):
            enc(srcs, n, offsets=torch.empty(6, dtype=torch.int64, device="cuda"))


def test_knob():
    """the packed compress with FSEB200_ENC_EK=8 (eight blocks per CTA of the chain-warp encoder), in a child process"""
    _ref()
    e = dict(os.environ, FSEB200_ENC_EK="8")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child"], env=e, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0 and "child ok" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])


def _child():
    for cd in CODECS:
        host, offs, sizes = ragged_fixture(cd, 715 + cd.wide, 200)
        layout_check(cd, host, offs, sizes)
    print("child ok")


if __name__ == "__main__" and "--child" in sys.argv:
    _child()
