"""CPU-side checks of the mixed-form Huff0 chain calls (FSEB200_HUF_compress_mixed_repeat_chains[_packed],
FSEB200_HUF_decompress_mixed_repeat_{blocks,packed}): declarations and exports, the argument verdicts, which touch no device, the
Python wrappers' argument checks, and -- on the compiled reference alone -- the claims the calls rest on: a kind-3 block decodes with
the header its chain resolves to whatever form wrote that header, and the case set reaches every input where the form changes the
bytes."""
import re
import subprocess
from collections import Counter

import numpy as np
import pytest
import torch

from helpers import is_error, ptr, load_ref, declared_arity
from huf_repeat_cases import main_configs
from huf_chain_cases import chain_header
from huf_chain_packed_cases import resolve_headers
from huf_mixed_chain_cases import mixed_chains, ref_mixed_chain, expected_mixed, form_counts, pattern_flags, PATTERNS

CALLS = {"FSEB200_HUF_compress_mixed_repeat_chains": 19, "FSEB200_HUF_decompress_mixed_repeat_blocks": 10,
         "FSEB200_HUF_compress_mixed_repeat_chains_packed": 19, "FSEB200_HUF_decompress_mixed_repeat_packed": 13,
         "FSEB200_compress_host_mixed_repeat_chains_packed": 18, "FSEB200_decompress_host_mixed_repeat_packed": 12}
WRAPPERS = ("huf_compress_mixed_repeat_chains", "huf_decompress_mixed_repeat_blocks", "huf_compress_mixed_repeat_chains_packed",
            "huf_decompress_mixed_repeat_packed", "host_compress_mixed_repeat_chains_packed", "host_decompress_mixed_repeat_packed")
SRC_WRONG = (1 << 64) - 3


def _lib():
    import finitestateentropy_b200 as fb
    return fb.lib()


def _ref():
    ref = load_ref()
    if ref is None:
        pytest.skip("compiled reference not available")
    return ref


def test_header_declares_and_library_exports_the_calls():
    decl = declared_arity()
    assert {n: decl.get(n) for n in CALLS} == CALLS
    from finitestateentropy_b200 import _build
    exported = subprocess.check_output(["nm", "-D", "--defined-only", _build.build_lib()]).decode()
    for name in CALLS:
        assert re.search(r" T %s$" % name, exported, flags=re.M), name
    import finitestateentropy_b200 as fb
    for name in WRAPPERS:
        assert callable(getattr(fb, name)), name


def test_argument_verdicts_without_a_device():
    """nBlocks == 0 returns 0 and launches nothing; nBlocks or nChains above 2^32 - 1, or a NULL array (dSingleStream included)
    while nBlocks > 0, gives srcSize_wrong.  Host buffers stand in for device arrays: nothing may touch them."""
    L = _lib()
    words = [np.full(4, 7, np.uint64) for _ in range(16)]
    a = [w.ctypes.data for w in words]

    def chains(arr, nc, nb):         # starts, dsts, caps, csizes, srcs, sizes, prefer, single, tables, flags, chdrs, chsizes, hdrs, hsizes
        return L.FSEB200_HUF_compress_mixed_repeat_chains(nc, arr[0], nb, *arr[1:14], 255, 11, None)

    def blocks(arr, nc, nb):         # dsts, sizes, results, csrcs, csizes, hdrs, hsizes, single
        return L.FSEB200_HUF_decompress_mixed_repeat_blocks(nb, *arr[0:8], None)

    def packed(arr, nc, nb):         # starts, out, offsets, csizes, kinds, srcs, sizes, prefer, single, tables, flags, chdrs, chsizes
        return L.FSEB200_HUF_compress_mixed_repeat_chains_packed(nc, arr[0], nb, arr[1], 1 << 20, *arr[2:13], 255, 11, None)

    def unpack(arr, nc, nb):         # starts, dsts, sizes, results, in, offsets, kinds, single, chdrs, chsizes
        return L.FSEB200_HUF_decompress_mixed_repeat_packed(nc, arr[0], nb, *arr[1:10], None)

    for call, n_arrays, has_chains in ((chains, 14, True), (blocks, 8, False), (packed, 13, True), (unpack, 10, True)):
        assert call([None] * n_arrays, 1, 0) == 0
        assert call(a[:n_arrays], 2 ** 32, 0) == 0
        assert call(a[:n_arrays], 1, 2 ** 32) == SRC_WRONG
        if has_chains:
            assert call(a[:n_arrays], 2 ** 32, 2) == SRC_WRONG
        for i in range(n_arrays):
            bad = list(a[:n_arrays])
            bad[i] = None
            assert call(bad, 1, 2) == SRC_WRONG, (call.__name__, i)
    for w in words:
        assert (w == 7).all()


def test_host_argument_verdicts_before_any_device_work():
    """the host pair: nBlocks == 0 returns 0; nBlocks or nChains above 2^32 - 1, or a NULL pointer (hSingleStream included) while
    nBlocks > 0, gives srcSize_wrong, and nothing is written"""
    L = _lib()
    words = [np.full(4, 7, np.uint64) for _ in range(14)]
    a = [w.ctypes.data for w in words]

    def comp(arr, nc, nb):          # starts, out, offsets, csizes, kinds, src, sizes, prefer, single, tables, flags, chdrs, chsizes
        return L.FSEB200_compress_host_mixed_repeat_chains_packed(nc, arr[0], nb, arr[1], 64, *arr[2:13], 255, 11)

    def decomp(arr, nc, nb):        # starts, dst, sizes, results, in, offsets, kinds, single, chdrs, chsizes
        return L.FSEB200_decompress_host_mixed_repeat_packed(nc, arr[0], nb, *arr[1:10])

    for call, n_arrays in ((comp, 13), (decomp, 10)):
        assert call([None] * n_arrays, 1, 0) == 0
        assert call(a[:n_arrays], 1, 2 ** 32) == SRC_WRONG
        assert call(a[:n_arrays], 2 ** 32, 2) == SRC_WRONG
        for i in range(n_arrays):
            bad = list(a[:n_arrays])
            bad[i] = None
            assert call(bad, 1, 2) == SRC_WRONG, (call.__name__, i)
    for w in words:
        assert (w == 7).all()


def test_host_wrappers_check_dtypes():
    import finitestateentropy_b200 as fb
    src = torch.zeros(64, dtype=torch.uint8)
    st = torch.tensor([0, 2], dtype=torch.int64)
    pr = torch.zeros(2, dtype=torch.int32)
    tabs, flags = torch.zeros(1, 256, dtype=torch.int32), torch.zeros(1, dtype=torch.int32)
    hp, hs = torch.zeros(1, dtype=torch.int64), torch.zeros(1, dtype=torch.int64)
    for single in (torch.zeros(2, dtype=torch.int32), torch.zeros(3, dtype=torch.uint8)):
        with pytest.raises(AssertionError):
            fb.host_compress_mixed_repeat_chains_packed(src, [4, 4], st, pr, single, tabs, flags, hp, hs)
        with pytest.raises(AssertionError):
            fb.host_decompress_mixed_repeat_packed(src, torch.tensor([0, 1, 2]), torch.zeros(2, dtype=torch.uint8), single, st, [4, 4],
                                                   hp, hs)


def test_wrappers_check_dtypes_and_devices():
    import finitestateentropy_b200 as fb
    c64, c32 = torch.zeros(2, dtype=torch.int64), torch.zeros(2, dtype=torch.int32)
    st = torch.tensor([0, 2], dtype=torch.int64)
    one64, one32 = torch.zeros(1, dtype=torch.int64), torch.zeros(1, dtype=torch.int32)
    u8, s8 = torch.zeros(64, dtype=torch.uint8), torch.zeros(2, dtype=torch.uint8)
    if not torch.cuda.is_available():
        with pytest.raises(AssertionError):        # host tensors are refused before anything else
            fb.huf_compress_mixed_repeat_chains_packed(st, c64, c64, c32, s8, one64, one32, one64, one64, out=u8)
        with pytest.raises(AssertionError):
            fb.huf_decompress_mixed_repeat_blocks(c64, c64, c64, c64, c64, c64, s8)
        return
    g = lambda t: t.cuda()
    args = [g(st), g(c64), g(c64), g(c32), g(s8), g(one64), g(one32), g(one64), g(one64)]
    for i, wrong in ((4, g(c32)), (4, g(torch.zeros(3, dtype=torch.uint8))), (4, s8), (3, g(c64)), (6, g(one64))):
        bad = list(args)
        bad[i] = wrong
        with pytest.raises(AssertionError):
            fb.huf_compress_mixed_repeat_chains_packed(*bad, out=g(u8))
    with pytest.raises(AssertionError):
        fb.huf_compress_mixed_repeat_chains(g(st), g(c64), g(c64), g(c64), g(c64), g(c32), g(c32), g(one64), g(one32), g(one64),
                                            g(one64))
    with pytest.raises(AssertionError):
        fb.huf_decompress_mixed_repeat_blocks(g(c64), g(c64), g(c64), g(c64), g(c64), g(c64), g(torch.zeros(2, dtype=torch.int8)))
    with pytest.raises(AssertionError):
        fb.huf_decompress_mixed_repeat_packed(g(st), g(u8), g(torch.zeros(3, dtype=torch.int64)), g(s8), g(c64), g(one64),
                                              g(one64), g(c64), g(c64))


def test_flag_patterns():
    sizes = [32768, 5, 300, 255, 256, 1, 1024]
    assert pattern_flags("all0", sizes) == [0] * 7 and pattern_flags("all1", sizes) == [1] * 7
    assert pattern_flags("alt", sizes) == [0, 1, 0, 1, 0, 1, 0]
    assert pattern_flags("every3", sizes) == [1, 0, 0, 1, 0, 0, 1]
    assert pattern_flags("size", sizes) == [0, 1, 0, 1, 0, 1, 0]
    r = pattern_flags("random", list(range(200)))
    assert set(r) >= {0, 1, 7, 255} and r == pattern_flags("random", list(range(200)))
    assert len(PATTERNS) == 6


def test_cross_form_headers_decode_on_the_reference():
    """for every kind-3 block of the case set: HUF_readDTableX1 on the header its chain resolves to (the last kind-2 block before
    it, of either form, or the chain's entry header), then HUF_decompress{4X1,1X1}_usingDTable in the block's own form, regenerates
    its source -- on the compiled reference, not on this library.  Also counts the inputs where the form changes the bytes."""
    ref = _ref()
    seen, counts = Counter(), Counter()
    for msv, tlog in main_configs():
        chains = mixed_chains(ref, msv, tlog)
        want = [ref_mixed_chain(ref, ch, msv, tlog) for ch in chains]
        vals, kinds, blobs, flags, starts = expected_mixed(want, chains)
        heads = resolve_headers(kinds, starts)
        b = 0
        for c, ch in enumerate(chains):
            entry, real = chain_header(ref, ch)
            for i, blk in enumerate(ch["blocks"]):
                if kinds[b] == 3:
                    h = heads[b]
                    if h[0] == "block":
                        hdr = blobs[h[1]]
                        seen["cross" if (flags[h[1]] != 0) != (flags[b] != 0) else "same_form"] += 1
                    else:
                        hdr = entry
                    if h[0] == "block" or real:
                        dt = np.zeros(4097, np.uint32)
                        dt[0] = 11 * 0x01000001                                     # HUF_CREATE_STATIC_DTABLEX1(DT, HUF_TABLELOG_MAX)
                        hs = ref.HUF_readDTableX1(ptr(dt), ptr(hdr), len(hdr))
                        n = len(blk["src"])
                        out = np.zeros(n + 64, np.uint8)
                        fn = ref.HUF_decompress1X1_usingDTable if flags[b] else ref.HUF_decompress4X1_usingDTable
                        if not is_error(hs):
                            r = fn(ptr(out), n, ptr(blobs[b]), len(blobs[b]), ptr(dt))
                            assert r == n and (out[:n] == blk["src"]).all(), (ch["name"], i)
                            seen["decoded"] += 1
                        else:
                            seen["weight12"] += 1                                   # the reference's own exception
                b += 1
        counts.update(form_counts(ref, chains, want, msv, tlog))
    assert seen["decoded"] and seen["cross"] and seen["same_form"], dict(seen)
    for key in ("x1_reads_x4", "x4_reads_x1", "old_tiny_1x", "old_one_byte_1x", "saved_zero_then_more"):
        assert counts[key], (key, dict(counts))
