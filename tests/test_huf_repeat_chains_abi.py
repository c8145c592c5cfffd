"""CPU-side checks of the Huff0 chain calls (FSEB200_HUF_compress{4X,1X}_repeat_chains): declarations and exports, the argument
verdicts, which touch no device, the Python wrappers' argument checks, and the reference's decision order restated along the
chains test_gpu_huf_repeat_chains.py runs, to show that blocks in the middle of a chain reach every outcome."""
import re
import subprocess
from collections import Counter

import numpy as np
import pytest
import torch

from test_huf_repeat_abi import trace
from huf_repeat_cases import main_configs, bound
from huf_chain_cases import mid_chains, drift_chains
from helpers import is_error, load_ref, declared_arity

CALLS = {"FSEB200_HUF_compress4X_repeat_chains": 18, "FSEB200_HUF_compress1X_repeat_chains": 18}
SRC_WRONG = (1 << 64) - 3


def _lib():
    import finitestateentropy_b200 as fb
    return fb.lib()


def test_header_declares_and_library_exports_the_calls():
    decl = declared_arity()
    assert {n: decl.get(n) for n in CALLS} == CALLS
    from finitestateentropy_b200 import _build
    exported = subprocess.check_output(["nm", "-D", "--defined-only", _build.build_lib()]).decode()
    for name in CALLS:
        assert re.search(r" T %s$" % name, exported, flags=re.M), name


def test_argument_verdicts_without_a_device():
    """nBlocks == 0 returns 0 and launches nothing (NULL arrays and a huge nChains included); nBlocks or nChains above 2^32 - 1,
    or a NULL array while nBlocks > 0, gives srcSize_wrong.  Host buffers stand in for device arrays: nothing may touch them."""
    L = _lib()
    words = [np.full(4, 7, np.uint64) for _ in range(13)]
    for name in CALLS:
        fn = getattr(L, name)
        arrays = [w.ctypes.data for w in words]

        def call(n_chains, n_blocks, arr):
            return fn(n_chains, arr[0], n_blocks, *arr[1:], 255, 11, None)

        assert call(1, 0, [None] * 13) == 0
        assert call(1, 0, arrays) == 0
        assert call(2 ** 32, 0, arrays) == 0
        assert call(1, 2 ** 32, arrays) == SRC_WRONG
        assert call(2 ** 32, 2, arrays) == SRC_WRONG
        for i in range(13):
            bad = list(arrays)
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
    for fn in (fb.huf_compress_repeat_chains, fb.huf_compress1x_repeat_chains):
        with pytest.raises(AssertionError):
            fn(st, c64, c64, c64, c64, c32, one64, one32, one64, one64)
    if torch.cuda.is_available():
        g = lambda t: t.cuda()
        args = [g(st), g(c64), g(c64), g(c64), g(c64), g(c32), g(one64), g(one32), g(one64), g(one64)]
        for i, wrong in ((5, g(c64)), (7, g(one64)), (6, g(one32)), (0, g(st).int()), (6, g(c64)), (1, g(c32))):
            bad = list(args)
            bad[i] = wrong
            with pytest.raises(AssertionError):
                fb.huf_compress_repeat_chains(*bad)


def walk(ref, four, chain, msv, tlog):
    """the chain's blocks through trace() with the state carried as the reference loop carries it: [(position, outcome, value)]"""
    from huf_repeat_cases import ref_repeat
    T, F = chain["table"].copy(), chain["flag"]
    out = []
    for i, blk in enumerate(chain["blocks"]):
        outcome, value, flag_t = trace(ref, four, blk["src"], blk["cap"], msv, tlog, T, F, blk["prefer"])
        r, _, F2, T2 = ref_repeat(ref, four, blk["src"], blk["cap"], msv, tlog, T, F, blk["prefer"])
        if value is not None:
            assert (value % (1 << 64), flag_t) == (r % (1 << 64), F2), (chain["name"], i, outcome)
        out.append((i, outcome, r, blk))
        T, F = T2, F2
        if not is_error(r) and r >= 2 and F == 0:
            F = 1
    return out


def test_mid_chain_blocks_reach_every_outcome():
    ref = load_ref()
    if ref is None:
        pytest.skip("compiled reference not available")
    seen = Counter()
    for four in (True, False):
        for msv, tlog in main_configs():
            chains = mid_chains(ref, four, msv, tlog) + drift_chains(ref)
            for ch in chains:
                for i, outcome, r, blk in walk(ref, four, ch, msv, tlog):
                    if i == 0:
                        continue
                    seen[outcome] += 1
                    n, cap = len(blk["src"]), blk["cap"]
                    if outcome == "arguments":
                        seen["arguments:" + ("cap0" if cap == 0 and n else "big" if n > 128 * 1024 else "other")] += 1
                    if outcome.startswith("hist:msv_too_small") and (msv, tlog) == (200, 11):
                        seen["msv_too_small@200,11"] += 1
                    if outcome.startswith("new:saved") and r == 0:
                        seen["new_table_saved_then_0"] += 1
                    if ch["name"].startswith("mid:") and i == 1 and cap != bound(n):
                        seen["capacity:%s" % ch["name"].split("/")[2]] += 1     # zero, exact (the size at a larger one), under
    for want in ("new:saved", "old:estimate", "old:estimate:equal", "new:saved:just_above_the_estimate_edge",
                 "new:saved:after_failed_validation", "old:prefer_valid", "hist:rle", "hist:incompressible",
                 "new:header_too_large", "old:header_too_large", "arguments:cap0", "capacity:zero", "arguments:big", "msv_too_small@200,11",
                 "new_table_saved_then_0", "capacity:exact", "capacity:under"):
        assert any(k == want or k.startswith(want + ":") for k in seen), (want, sorted(seen))
