"""CPU-side checks of the packed Huff0 chain calls (FSEB200_HUF_compress{4X,1X}_repeat_chains_packed,
FSEB200_HUF_decompress{4X,1X}_repeat_packed): declarations and exports, the argument verdicts, which touch no device, the Python
wrappers' argument checks, and the decoder's header resolution (kinds + chain starts + entry headers) against the header the
reference loop codes every block with, on the chains test_gpu_huf_repeat_packed.py runs."""
import re
import subprocess
from collections import Counter

import numpy as np
import pytest
import torch

from helpers import load_ref, declared_arity
from huf_repeat_cases import main_configs
from huf_chain_cases import ref_chain
from huf_chain_packed_cases import packed_chains, expected, resolve_headers

COMPRESS = {"FSEB200_HUF_compress4X_repeat_chains_packed": 18, "FSEB200_HUF_compress1X_repeat_chains_packed": 18}
DECOMPRESS = {"FSEB200_HUF_decompress4X_repeat_packed": 12, "FSEB200_HUF_decompress1X_repeat_packed": 12}
SRC_WRONG = (1 << 64) - 3


def _lib():
    import finitestateentropy_b200 as fb
    return fb.lib()


def test_header_declares_and_library_exports_the_calls():
    decl = declared_arity()
    calls = dict(COMPRESS, **DECOMPRESS)
    assert {n: decl.get(n) for n in calls} == calls
    from finitestateentropy_b200 import _build
    exported = subprocess.check_output(["nm", "-D", "--defined-only", _build.build_lib()]).decode()
    for name in calls:
        assert re.search(r" T %s$" % name, exported, flags=re.M), name
    import finitestateentropy_b200 as fb
    for name in ("huf_compress_repeat_chains_packed", "huf_compress1x_repeat_chains_packed", "huf_decompress_repeat_packed",
                 "huf_decompress1x_repeat_packed"):
        assert callable(getattr(fb, name)), name


def test_argument_verdicts_without_a_device():
    """nBlocks == 0 returns 0 and launches nothing (NULL arrays and a huge nChains included); nBlocks or nChains above 2^32 - 1,
    or a NULL array while nBlocks > 0, gives srcSize_wrong.  Host buffers stand in for device arrays: nothing may touch them."""
    L = _lib()
    words = [np.full(4, 7, np.uint64) for _ in range(13)]
    arrays = [w.ctypes.data for w in words]
    for name in COMPRESS:
        fn = getattr(L, name)

        def call(n_chains, n_blocks, arr):           # arr: starts, out, offsets, csizes, kinds, srcs, sizes, prefer, tables, flags, hdrs, hsizes
            return fn(n_chains, arr[0], n_blocks, arr[1], 1 << 20, *arr[2:12], 255, 11, None)

        assert call(1, 0, [None] * 12) == 0
        assert call(2 ** 32, 0, arrays) == 0
        assert call(1, 2 ** 32, arrays) == SRC_WRONG
        assert call(2 ** 32, 2, arrays) == SRC_WRONG
        for i in range(12):
            bad = list(arrays[:12])
            bad[i] = None
            assert call(1, 2, bad) == SRC_WRONG, (name, i)
    for name in DECOMPRESS:
        fn = getattr(L, name)

        def call(n_chains, n_blocks, arr):           # arr: starts, dsts, dst sizes, results, in, offsets, kinds, hdrs, hsizes
            return fn(n_chains, arr[0], n_blocks, *arr[1:9], None)

        assert call(1, 0, [None] * 9) == 0
        assert call(2 ** 32, 0, arrays) == 0
        assert call(1, 2 ** 32, arrays) == SRC_WRONG
        assert call(2 ** 32, 2, arrays) == SRC_WRONG
        for i in range(9):
            bad = list(arrays[:9])
            bad[i] = None
            assert call(1, 2, bad) == SRC_WRONG, (name, i)
    for w in words:
        assert (w == 7).all()


def test_wrappers_check_dtypes_and_devices():
    import finitestateentropy_b200 as fb
    c64 = torch.zeros(2, dtype=torch.int64)
    c32 = torch.zeros(2, dtype=torch.int32)
    st = torch.tensor([0, 2], dtype=torch.int64)
    one64, one32 = torch.zeros(1, dtype=torch.int64), torch.zeros(1, dtype=torch.int32)
    u8 = torch.zeros(64, dtype=torch.uint8)
    for fn in (fb.huf_compress_repeat_chains_packed, fb.huf_compress1x_repeat_chains_packed):
        with pytest.raises(AssertionError):
            fn(st, c64, c64, c32, one64, one32, one64, one64, out=u8)
    for fn in (fb.huf_decompress_repeat_packed, fb.huf_decompress1x_repeat_packed):
        with pytest.raises(AssertionError):
            fn(st, u8, torch.zeros(3, dtype=torch.int64), torch.zeros(2, dtype=torch.uint8), one64, one64, c64, c64)
    if torch.cuda.is_available():
        g = lambda t: t.cuda()
        args = [g(st), g(c64), g(c64), g(c32), g(one64), g(one32), g(one64), g(one64)]
        for i, wrong in ((3, g(c64)), (5, g(one64)), (4, g(one32)), (0, g(st).int()), (1, g(c32)), (6, g(c64))):
            bad = list(args)
            bad[i] = wrong
            with pytest.raises(AssertionError):
                fb.huf_compress_repeat_chains_packed(*bad, out=g(u8))
        with pytest.raises(AssertionError):
            fb.huf_compress_repeat_chains_packed(*args, out=g(u8), kinds=g(c64))
        dargs = [g(st), g(u8), g(torch.zeros(3, dtype=torch.int64)), g(torch.zeros(2, dtype=torch.uint8)), g(one64), g(one64),
                 g(c64), g(c64)]
        for i, wrong in ((3, g(c64)), (1, g(c64)), (4, g(one32)), (0, g(st).int()), (2, g(c64))):
            bad = list(dargs)
            bad[i] = wrong
            with pytest.raises(AssertionError):
                fb.huf_decompress_repeat_packed(*bad)


def test_kinds_and_chain_starts_name_the_loops_header_for_every_block():
    """the decoder's resolution, restated on the reference loop's kinds, names the header the loop coded every block with; and
    the chains reach every kind, kind 3 as a chain's first block (the entry header) and a raw block after a saved table"""
    ref = load_ref()
    if ref is None:
        pytest.skip("compiled reference not available")
    seen = Counter()
    for four in (True, False):
        for msv, tlog in main_configs():
            chains = packed_chains(ref, four, msv, tlog)
            want = [ref_chain(ref, four, ch, msv, tlog) for ch in chains]
            vals, kinds, _, starts = expected(want, chains)
            got = resolve_headers(kinds, starts)
            b = 0
            for c, (per, _) in enumerate(want):
                saved_before = False
                for i, (r, _, h) in enumerate(per):
                    k = kinds[b]
                    seen["kind%d" % k] += 1
                    if k == 3:
                        token = ("chain", c) if h == ("chain",) else ("block", starts[c] + h[1])
                        assert got[b] == token, (chains[c]["name"], i)
                        if i == 0:
                            seen["kind3_first"] += 1
                    else:
                        assert got[b] is None
                    if k == 0 and saved_before and vals[b] == 0 and len(chains[c]["blocks"][i]["src"]):
                        seen["raw_after_saved"] += 1
                    if k == 2:
                        saved_before = True
                    b += 1
    for want_key in ("kind0", "kind1", "kind2", "kind3", "kind4", "kind3_first", "raw_after_saved"):
        assert seen[want_key], (want_key, sorted(seen.items()))
