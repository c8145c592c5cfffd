"""CPU-side checks of the Huff0 table-reuse calls (FSEB200_HUF_{compress,decompress}{4X,1X}_repeat_blocks): declarations and
exports, the argument verdicts, which touch no device, the Python wrappers' argument checks, and the reference's decision order
(huf_compress.c:653-724) restated on the host from the compiled reference's table-level calls, to show that the inputs
test_gpu_huf_repeat.py runs reach every outcome of it."""
import ctypes as C
import re
import subprocess
from collections import Counter

import numpy as np
import pytest
import torch

from helpers import ptr, is_error, load_ref, declared_arity
from huf_repeat_cases import main_cases, main_configs, U

CALLS = {"FSEB200_HUF_compress4X_repeat_blocks": 12, "FSEB200_HUF_compress1X_repeat_blocks": 12,
         "FSEB200_HUF_decompress4X_repeat_blocks": 9, "FSEB200_HUF_decompress1X_repeat_blocks": 9}
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
    """nBlocks == 0 returns 0 and launches nothing (NULL arrays included); nBlocks above 2^32 - 1 or a NULL array while
    nBlocks > 0 gives srcSize_wrong.  The host buffers stand in for device arrays: nothing may touch them."""
    L = _lib()
    words = [np.full(4, 7, np.uint64) for _ in range(9)]
    for name in ("FSEB200_HUF_compress4X_repeat_blocks", "FSEB200_HUF_compress1X_repeat_blocks"):
        fn = getattr(L, name)
        args = [w.ctypes.data for w in words[:8]]
        assert fn(0, *[None] * 8, 255, 11, None) == 0
        assert fn(0, *args, 255, 11, None) == 0
        assert fn(2 ** 32, *args, 255, 11, None) == SRC_WRONG
        for i in range(8):
            bad = list(args)
            bad[i] = None
            assert fn(2, *bad, 255, 11, None) == SRC_WRONG, (name, i)
    for name in ("FSEB200_HUF_decompress4X_repeat_blocks", "FSEB200_HUF_decompress1X_repeat_blocks"):
        fn = getattr(L, name)
        args = [w.ctypes.data for w in words[:7]]
        assert fn(0, *[None] * 7, None) == 0
        assert fn(0, *args, None) == 0
        assert fn(2 ** 32, *args, None) == SRC_WRONG
        for i in range(7):
            bad = list(args)
            bad[i] = None
            assert fn(2, *bad, None) == SRC_WRONG, (name, i)
    for w in words:
        assert (w == 7).all()


def test_wrappers_check_dtypes_and_devices():
    import finitestateentropy_b200 as fb
    cpu64 = torch.zeros(2, dtype=torch.int64)
    cpu32 = torch.zeros(2, dtype=torch.int32)
    for fn in (fb.huf_compress_repeat_blocks, fb.huf_compress1x_repeat_blocks):
        with pytest.raises(AssertionError):
            fn(cpu64, cpu64, cpu64, cpu64, cpu64, cpu32, cpu32)
    for fn in (fb.huf_decompress_repeat_blocks, fb.huf_decompress1x_repeat_blocks):
        with pytest.raises(AssertionError):
            fn(cpu64, cpu64, cpu64, cpu64, cpu64, cpu64)
    if torch.cuda.is_available():                                           # wrong dtypes on the device
        g64, g32 = cpu64.cuda(), cpu32.cuda()
        with pytest.raises(AssertionError):
            fb.huf_compress_repeat_blocks(g64, g64, g64, g64, g64, g64, g32)   # flags must be int32
        with pytest.raises(AssertionError):
            fb.huf_compress_repeat_blocks(g64, g64, g64, g64, g32, g32, g32)   # table pointers must be int64
        with pytest.raises(AssertionError):
            fb.huf_decompress_repeat_blocks(g64, g64, g64, g64, g64, g32)


def trace(ref, four, src, cap, msv, tlog, table, flag, prefer):
    """HUF_compress_internal's decision order from the reference's table-level calls: (outcome, value, flag out)"""
    n = len(src)
    coder = ref.HUF_compress4X_usingCTable if four else ref.HUF_compress1X_usingCTable
    out = np.zeros(2 * n + 1024, np.uint8)

    def old_table(how):                                                     # HUF_compressCTable_internal at ostart
        c = coder(ptr(out), cap, ptr(src), n, ptr(table))
        assert not is_error(c)
        if c == 0:
            return how + ":zero_capacity", 0, flag
        if c >= n - 1:
            return how + ":zero_ratio", 0, flag
        return how, c, flag

    if not n or not cap or n > 128 * 1024 or tlog > 12 or msv > 255:
        return "arguments", None, flag
    msv, tlog = msv or 255, tlog or 11
    if prefer and flag == 2:
        return old_table("old:prefer_valid")
    cnt = (U * 256)()
    m = U(msv)
    largest = ref.HIST_count(cnt, C.byref(m), ptr(src), n)
    if is_error(largest):
        return "hist:msv_too_small", largest, flag
    if largest == n:
        return "hist:rle", 1, flag
    if largest <= (n >> 7) + 4:
        return "hist:incompressible", 0, flag
    failed, edge = False, ""
    if flag == 1 and not ref.HUF_validateCTable(ptr(table), cnt, m.value):
        flag, failed = 0, True
    if prefer and flag != 0:
        return old_table("old:prefer_flag")
    ct = np.zeros(256, np.uint32)
    bits = ref.HUF_buildCTable(ptr(ct), cnt, m.value, ref.HUF_optimalTableLog(tlog, n, m.value))
    assert not is_error(bits)
    hdr = np.zeros(256, np.uint8)
    h = ref.HUF_writeCTable(ptr(hdr), cap, ptr(ct), m.value, bits)
    if is_error(h):
        return "header_error", h, flag
    if flag != 0:
        old = ref.HUF_estimateCompressedSize(ptr(table), cnt, m.value)
        new = ref.HUF_estimateCompressedSize(ptr(ct), cnt, m.value)
        if old <= h + new:
            return old_table("old:estimate:equal" if old == h + new else "old:estimate")
        if h + 12 >= n:
            return old_table("old:header_too_large")
        if old == h + new + 1:
            edge = ":just_above_the_estimate_edge"
    if h + 12 >= n:
        return "new:header_too_large", 0, flag
    c = coder(ptr(out), cap - h, ptr(src), n, ptr(ct))
    tag = "new:saved" + (":after_failed_validation" if failed else "") + edge
    if c == 0 or h + c >= n - 1:
        return tag, 0, 0
    return tag, h + c, 0


def test_gpu_inputs_reach_every_outcome_of_the_decision_order():
    ref = load_ref()
    if ref is None:
        pytest.skip("compiled reference not available")
    seen = Counter()
    for four in (True, False):
        for msv, tlog in main_configs():
            for c in main_cases(ref, four, msv, tlog):
                outcome, value, flag_out = trace(ref, four, c["src"], c["cap"], msv, tlog, c["table"], c["flag"], c["prefer"])
                if value is not None:                                       # the restatement agrees with the reference
                    assert (value % (1 << 64), flag_out) == (c["r"] % (1 << 64), c["flag_out"]), (outcome, c["bname"], c["tname"])
                key = outcome.split(":")
                seen[outcome] += 1
                seen["%s|flag=%d|prefer=%d" % (key[0] + ":" + key[1] if len(key) > 1 else key[0], c["flag"], c["prefer"])] += 1
                if c["prefer"] and c["flag"] == 2 and (c["bname"].startswith(("rle", "rand")) or c["bname"] == "high_32768"):
                    seen["prefer_valid_skips_hist_exits:" + outcome] += 1
    for want in ("old:prefer_valid", "old:prefer_flag", "old:estimate", "old:estimate:equal", "new:saved:just_above_the_estimate_edge",
                 "new:saved:after_failed_validation", "new:saved",
                 "old:header_too_large", "new:header_too_large", "hist:rle|flag=1|prefer=0", "hist:incompressible|flag=1|prefer=0",
                 "hist:msv_too_small|flag=1|prefer=0"):
        assert any(k == want or k.startswith(want + ":") for k in seen), (want, sorted(seen))
    assert seen["old:header_too_large"] > 0, sorted(seen)                 # taken by that exit alone, and not 0 either way
    assert any(k.startswith("old:") and k.endswith(":zero_capacity") for k in seen), sorted(seen)
    assert any(k.startswith("old:") and k.endswith(":zero_ratio") for k in seen), sorted(seen)
    hist_under_prefer_valid = [k for k in seen if k.startswith("hist:") and "|flag=2|prefer=1" in k]
    assert not hist_under_prefer_valid
    assert seen["prefer_valid_skips_hist_exits:old:prefer_valid"] + sum(
        v for k, v in seen.items() if k.startswith("prefer_valid_skips_hist_exits:old:prefer_valid:")) > 0
