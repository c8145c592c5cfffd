"""Packed Huff0 compress (FSEB200_HUF_compress_packed / FSEB200_HUF_compress1X_packed) against the compiled reference (-m gpu):
the whole output buffer is compared with the packed image the host model (tests/packed_paths.py) builds from HUF_compress2 /
HUF_compress1X at HUF_compressBound(n), with the offsets and values exact and poisoned canaries around it.  Ragged, small-block
and special-size layouts with overlapping sources, every output offset mod 16 the kernels branch on, capacities that cut the
stream, bad parameters, a batch of more than one plan round, a total above 4 GiB, the round trip through packed_pointers and
the descriptor decoders, and the calls' argument checks.  Block contents and layouts are those of tests/test_gpu_blocks.py."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from helpers import is_error                                                      # noqa: E402
from packed_paths import ERR_DST_TOO_SMALL, ref_values, image, stored_len, ref_decode           # noqa: E402
from test_gpu_blocks import POISON, CANARY, ERR_SRC_WRONG, ragged_sources, _ref, _u64, _dev64   # noqa: E402

pytestmark = pytest.mark.gpu

FORMATS = [False, True]
FORMAT_IDS = ["4X", "1X"]
OUT_OFFSETS = [0, 1, 4, 8, 16, 32, 64, 96]


def _lib():
    return _ref()


def fixture(seed, count, sizes=None):
    rng = np.random.default_rng(seed)
    host, offs, sizes = ragged_sources(rng, count, sizes)
    return host, offs, sizes


def reference(lib, host, offs, sizes, onex, msv=255, tl=12):
    return ref_values(lib, [host[o: o + n] for o, n in zip(offs, sizes)], msv, tl, onex)


def run_packed(onex, src, offs, sizes, cap, out_off, msv=255, tl=12):
    """the packed compress on the GPU into a poisoned arena, dOut at out_off from a 512-byte aligned start: (offsets, values,
    arena on the device, dOut's index in the arena)"""
    import torch
    import finitestateentropy_b200 as fb
    arena = torch.full((CANARY + 512 + 96 + cap + CANARY,), POISON, dtype=torch.uint8, device="cuda")
    o = ((arena.data_ptr() + CANARY + 511) & ~511) + out_off - arena.data_ptr()
    offsets = torch.full((len(sizes) + 1,), -7, dtype=torch.int64, device="cuda")
    cs = torch.full((len(sizes),), -7, dtype=torch.int64, device="cuda")
    sp, sn = _dev64([src.data_ptr() + x for x in offs]), _dev64(sizes)
    fn = fb.lib().FSEB200_HUF_compress1X_packed if onex else fb.lib().FSEB200_HUF_compress_packed
    r = fn(len(sizes), arena.data_ptr() + o, cap, offsets.data_ptr(), cs.data_ptr(), sp.data_ptr(), sn.data_ptr(), msv, tl,
           torch.cuda.current_stream().cuda_stream)
    assert r == 0, r
    torch.cuda.synchronize()
    return _u64(offsets), _u64(cs), arena, o


def check_packed(onex, host, offs, sizes, ref, cap=None, out_off=0, msv=255, tl=12, src=None):
    """the GPU's offsets, values and whole output buffer against the model's; nothing written outside the stored blocks"""
    import torch
    vals, stored = ref
    cap = sum(sizes) if cap is None else cap
    img, written, want_offs, want_final = image(vals, stored, sizes, cap)
    src = torch.from_numpy(host).cuda() if src is None else src
    got_offs, got_cs, arena, o = run_packed(onex, src, offs, sizes, cap, out_off, msv, tl)
    assert [int(x) for x in got_offs] == want_offs, (onex, cap, out_off)
    bad = [(b, sizes[b], int(got_cs[b]), want_final[b]) for b in range(len(sizes)) if int(got_cs[b]) != want_final[b]]
    assert not bad, (onex, cap, out_off, bad[:8])
    a = arena.cpu().numpy()
    end = min(want_offs[-1], cap)
    region = a[o: o + end]
    assert np.array_equal(region[written], img[written]), (onex, cap, out_off)
    assert bool((region[~written] == POISON).all()), "bytes of a block that does not fit were written"
    assert bool((a[:o] == POISON).all()) and bool((a[o + end:] == POISON).all()), "bytes outside the packed blocks were written"
    assert torch.equal(src.cpu(), torch.from_numpy(host))               # sources are read only
    return want_offs, want_final, arena, o


def round_trip(lib, onex, host, offs, sizes, want_offs, final, arena, o):
    """packed_pointers + the descriptor decoder on every non-empty block without an error: the reference decoder's verdict on
    the same packed bytes, and the source wherever that decodes (the reference cannot decode a few of its own blocks: a code of
    length 1 at tableLog 12 is written as weight 12, which HUF_readStats rejects, entropy_common.c:191)"""
    import torch
    import finitestateentropy_b200 as fb
    out = arena[o: o + want_offs[-1]]
    want = ref_decode(lib, out.cpu().numpy(), want_offs, sizes, final, onex)
    ptrs, lens = fb.packed_pointers(out, torch.tensor(want_offs, dtype=torch.int64, device="cuda"))
    keep = [b for b in range(len(sizes)) if sizes[b] and not is_error(final[b])]
    assert keep
    idx = torch.tensor(keep, dtype=torch.int64, device="cuda")
    kn = [sizes[b] for b in keep]
    dst = torch.zeros(sum(kn) + 1, dtype=torch.uint8, device="cuda")
    doffs = np.concatenate([[0], np.cumsum(kn)[:-1]]).astype(np.int64)
    dec = fb.huf_decompress1x_blocks if onex else fb.huf_decompress_blocks
    res = dec(ptrs[idx].contiguous(), lens[idx].contiguous(), _dev64(dst.data_ptr() + doffs), _dev64(kn))
    torch.cuda.synchronize()
    got = [int(x) for x in _u64(res)]
    assert got == [want[b][0] for b in keep], (onex, [(b, g, want[b][0]) for b, g in zip(keep, got) if g != want[b][0]][:8])
    assert sum(g == n for g, n in zip(got, kn)) >= 0.9 * len(kn)
    d = dst.cpu().numpy()
    for b, do, n in zip(keep, doffs, kn):
        if want[b][0] == n:
            assert np.array_equal(d[do: do + n], host[offs[b]: offs[b] + n]), (onex, b, n)


def ragged_check(onex, seed, count):
    lib = _lib()
    host, offs, sizes = fixture(seed, count)
    ref = reference(lib, host, offs, sizes, onex)
    kinds = {0 if v == 0 else 1 if v == 1 else "err" if is_error(v) else "size" for v in ref[0]}
    assert kinds == {0, 1, "err", "size"}, kinds
    want_offs, final, arena, o = check_packed(onex, host, offs, sizes, ref)
    round_trip(lib, onex, host, offs, sizes, want_offs, final, arena, o)
    total = want_offs[-1]
    raw = next(b for b in range(len(sizes)) if ref[0][b] == 0 and sizes[b] > 2)
    check_packed(onex, host, offs, sizes, ref, cap=want_offs[raw] + sizes[raw] // 2, out_off=1)
    check_packed(onex, host, offs, sizes, ref, cap=total - 1, out_off=4)


# ---- tests ----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("onex", FORMATS, ids=FORMAT_IDS)
def test_ragged(onex):
    """special sizes (0, 1, 11, 12, 128 KB, 128 KB + 1, ...) and ragged ones up to 128 KB + 1, overlapping sources; round trip"""
    ragged_check(onex, seed=601, count=1200)


@pytest.mark.parametrize("onex", FORMATS, ids=FORMAT_IDS)
def test_small_blocks(onex):
    lib = _lib()
    rng = np.random.default_rng(602)
    host, offs, sizes = fixture(602, 3000, [int(x) for x in rng.integers(1, 4097, 3000)])
    ref = reference(lib, host, offs, sizes, onex)
    want_offs, final, arena, o = check_packed(onex, host, offs, sizes, ref, out_off=8)
    round_trip(lib, onex, host, offs, sizes, want_offs, final, arena, o)


@pytest.mark.parametrize("onex", FORMATS, ids=FORMAT_IDS)
def test_output_offsets(onex):
    """dOut at 0, 1, 4, 8, 16, 32, 64 and 96 from a 512-byte aligned start: every block's alignment changes with it"""
    import torch
    lib = _lib()
    host, offs, sizes = fixture(603, 300)
    ref = reference(lib, host, offs, sizes, onex)
    src = torch.from_numpy(host).cuda()
    for off in OUT_OFFSETS:
        check_packed(onex, host, offs, sizes, ref, out_off=off, src=src)


@pytest.mark.parametrize("onex", FORMATS, ids=FORMAT_IDS)
def test_capacities(onex):
    """outCapacity at the total, the total - 1, cut inside a raw block, cut inside a compressed block, and 0"""
    import torch
    lib = _lib()
    host, offs, sizes = fixture(604, 300)
    ref = reference(lib, host, offs, sizes, onex)
    vals = ref[0]
    lens = [stored_len(v, n) for v, n in zip(vals, sizes)]
    starts = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    total = int(starts[-1])
    raw = [b for b in range(len(sizes)) if vals[b] == 0 and lens[b] > 2]
    comp = [b for b in range(len(sizes)) if vals[b] > 1 and not is_error(vals[b])]
    src = torch.from_numpy(host).cuda()
    for cap in (total, total - 1, int(starts[raw[len(raw) // 2]]) + lens[raw[len(raw) // 2]] // 2,
                int(starts[comp[len(comp) // 2]]) + lens[comp[len(comp) // 2]] // 2, int(starts[comp[3]]) + 1, 0):
        _, final, _, _ = check_packed(onex, host, offs, sizes, ref, cap=cap, out_off=cap % 16, src=src)
        assert (ERR_DST_TOO_SMALL in final) == (cap < total), cap


@pytest.mark.parametrize("onex", FORMATS, ids=FORMAT_IDS)
def test_parameters(onex):
    """bad and unusual maxSymbolValue / tableLog: the reference's verdicts, error blocks store nothing"""
    import torch
    lib = _lib()
    host, offs, sizes = fixture(605, 200)
    src = torch.from_numpy(host).cuda()
    for msv, tl in ((255, 11), (0, 0), (200, 12), (255, 13), (256, 12)):
        ref = reference(lib, host, offs, sizes, onex, msv, tl)
        _, final, _, _ = check_packed(onex, host, offs, sizes, ref, msv=msv, tl=tl, out_off=1, src=src)
        if msv == 200:
            assert any(v == 2 ** 64 - 7 for v in final)                 # maxSymbolValue_tooSmall on bytes above 200
        if tl == 13 or msv == 256:
            assert all(is_error(v) or n == 0 for v, n in zip(final, sizes))


@pytest.mark.parametrize("onex", FORMATS, ids=FORMAT_IDS)
def test_large_batch(onex):
    """20,000 small blocks: more than one round of plan CTAs on 132 SMs (12,672 blocks) and ten scan tiles"""
    lib = _lib()
    rng = np.random.default_rng(606)
    host, offs, sizes = fixture(606, 20000, [int(x) for x in rng.integers(1, 3000, 20000)])
    ref = reference(lib, host, offs, sizes, onex)
    want_offs, final, arena, o = check_packed(onex, host, offs, sizes, ref, out_off=64)
    round_trip(lib, onex, host, offs, sizes, want_offs, final, arena, o)


def test_total_above_4gib():
    """33,000 raw 128 KB blocks that all read one random 128 KB source: offsets above 2^32, every block placed past 4 GiB"""
    import torch
    import finitestateentropy_b200 as fb
    lib = _lib()
    n, count = 131072, 33000
    data = np.random.default_rng(607).integers(0, 256, n, dtype=np.uint8)
    for onex in FORMATS:
        vals, _ = ref_values(lib, [data], 255, 12, onex)
        assert vals == [0]
    src = torch.from_numpy(data).cuda()
    total = n * count
    assert total > 2 ** 32
    arena = torch.full((total + 2 * CANARY,), POISON, dtype=torch.uint8, device="cuda")
    out = arena[CANARY: CANARY + total]
    ptrs, sizes = _dev64([src.data_ptr()] * count), _dev64([n] * count)
    want = torch.arange(count + 1, dtype=torch.int64, device="cuda") * n
    for onex in FORMATS:
        fn = fb.huf_compress1x_packed if onex else fb.huf_compress_packed
        _, offsets, cs = fn(ptrs, sizes, out=out)
        torch.cuda.synchronize()
        assert torch.equal(offsets, want) and int(offsets[-1]) > 2 ** 32
        assert bool((cs == 0).all())
        blocks = out.view(count, n)
        first_past = int((2 ** 32 + n - 1) // n)
        for b in (first_past - 1, first_past, first_past + 1, count - 2, count - 1):
            assert torch.equal(blocks[b], src), (onex, b)
        assert bool((blocks == src).all())
        assert bool((arena[:CANARY] == POISON).all()) and bool((arena[CANARY + total:] == POISON).all())
        out[:n].fill_(POISON)
        out[-n:].fill_(POISON)


def test_arguments_and_wrappers():
    import torch
    import finitestateentropy_b200 as fb
    from helpers import probagen
    L = fb.lib()
    a = _dev64([0, 0])
    p = a.data_ptr()
    for fn in (L.FSEB200_HUF_compress_packed, L.FSEB200_HUF_compress1X_packed):
        assert fn(0, None, 0, None, None, None, None, 255, 12, None) == 0
        for k in range(5):
            args = [p] * 5
            args[k] = None
            assert fn(1, args[0], 100, args[1], args[2], args[3], args[4], 255, 12, None) == ERR_SRC_WRONG
        assert fn(1 << 32, p, 100, p, p, p, p, 255, 12, None) == ERR_SRC_WRONG
        # nBlocks == 0 writes nothing, not even dOffsets[0]
        offs = torch.full((4,), -7, dtype=torch.int64, device="cuda")
        assert fn(0, p, 100, offs.data_ptr(), offs.data_ptr(), p, p, 255, 12, None) == 0
        torch.cuda.synchronize()
        assert (offs == -7).all()
    # the Python wrappers on views, on a side stream, allocating the output
    lib = _lib()
    data = [torch.from_numpy(x).cuda() for x in (probagen(1000, 0.14), np.full(300, 7, np.uint8),
                                                 np.random.default_rng(1).integers(0, 256, 777, dtype=np.uint8), probagen(32768, 0.3))]
    srcs, n = fb.block_pointers(data)
    s = torch.cuda.Stream()
    for onex in FORMATS:
        enc = fb.huf_compress1x_packed if onex else fb.huf_compress_packed
        dec = fb.huf_decompress1x_blocks if onex else fb.huf_decompress_blocks
        with torch.cuda.stream(s):
            out, offsets, cs = enc(srcs, n)
            ptrs, lens = fb.packed_pointers(out, offsets)
            outs = [torch.zeros_like(d) for d in data]
            op, on = fb.block_pointers(outs)
            res = dec(ptrs, lens, op, on)
        s.synchronize()
        assert out.numel() == sum(n.tolist()) + 32 and offsets.numel() == 5 and cs.numel() == 4
        vals, _ = ref_values(lib, [d.cpu().numpy() for d in data], 255, 12, onex)
        assert [int(v) for v in _u64(cs)] == vals and vals[1] == 1 and vals[2] == 0
        assert res.tolist() == n.tolist() and all(torch.equal(o, d) for o, d in zip(outs, data))
        with pytest.raises(AssertionError):
            enc(srcs, n, offsets=torch.empty(4, dtype=torch.int64, device="cuda"))
