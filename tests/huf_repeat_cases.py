"""Inputs of the Huff0 table-reuse tests (FSEB200_HUF_{compress,decompress}{4X,1X}_repeat_blocks) and the reference's per-block
function values on them.  test_huf_repeat_abi.py restates the reference's decision order on these inputs and checks that they
reach every outcome; test_gpu_huf_repeat.py runs them through the library and compares with the reference."""
import ctypes as C
import itertools

import numpy as np

from helpers import ptr, probagen, is_error

U = C.c_uint
FLAGS = (0, 1, 2, 3, -1)
PREFERS = (0, 1)
SIZES = (0, 1, 5, 11, 12, 4099, 32768, 131072, 131073)
WKSP_WORDS = 1600                                    # HUF_WORKSPACE_SIZE_U32 (6 KB + 256 bytes)
HUGE_CAP = 1 << 33


def bound(n):
    return 129 + n + (n >> 8) + 8


def room(n, cap):
    """bytes of destination a block can be written into at capacity `cap` (more is never touched: <= 12 bits per symbol)"""
    return min(cap, 2 * n + 1024)


def ref_table(ref, data, tlog=12):
    cnt = (U * 256)()
    m = U(255)
    ref.HIST_count(cnt, C.byref(m), ptr(data), len(data))
    ct = np.zeros(256, np.uint32)
    r = ref.HUF_buildCTable(ptr(ct), cnt, m.value, ref.HUF_optimalTableLog(tlog, len(data), m.value))
    assert not is_error(r)
    return ct


def table_header(ref, ct):
    """HUF_writeCTable of a table: what a block that introduced it starts with"""
    nb = (ct >> 16) & 0xFF
    msv = int(np.nonzero(nb)[0].max())
    out = np.zeros(256, np.uint8)
    h = ref.HUF_writeCTable(ptr(out), 256, ptr(ct), msv, int(nb.max()))
    assert not is_error(h)
    return out[:h].copy()


def tables(ref):
    """name -> 256-cell table: the blocks' own distribution, another one over every symbol (with padding bytes set), one lacking
    symbols the blocks use, all zero, the first read back through HUF_readCTable, and 12-bit codes for every symbol"""
    rng = np.random.default_rng(5)
    same = ref_table(ref, probagen(65536, 0.14))
    w = 1.0 / np.arange(1, 257) ** 1.1
    other = ref_table(ref, rng.permutation(256).astype(np.uint8)[rng.choice(256, 65536, p=w / w.sum())]) | np.uint32(0xA5000000)
    lacking = ref_table(ref, probagen(65536, 0.5))
    hdr = table_header(ref, same)
    back = np.zeros(256, np.uint32)
    m, z = U(255), U(0)
    assert not is_error(ref.HUF_readCTable(ptr(back), C.byref(m), ptr(hdr), len(hdr), C.byref(z)))
    long12 = np.arange(256, dtype=np.uint32) | np.uint32(12 << 16)        # every code 12 bits long: codable, not a Huffman table
    return {"same": same, "other": other, "lacking": lacking, "zero": np.zeros(256, np.uint32), "readback": back, "long": long12}


def blocks():
    """(name, data): every size the plan kernel branches on, RLE, random bytes, another distribution, symbols up to 255"""
    rng = np.random.default_rng(7)
    p14 = probagen(1 << 18, 0.14)
    out = [("p14_%d" % n, p14[1000:1000 + n].copy()) for n in SIZES]
    out += [("rle_4099", np.full(4099, 3, np.uint8)), ("rle_32768", np.full(32768, 200, np.uint8)),
            ("rand_32768", rng.integers(0, 256, 32768, dtype=np.uint8)), ("rand_12", rng.integers(0, 256, 12, dtype=np.uint8)),
            ("p40_32768", probagen(32768, 0.40)), ("high_32768", np.concatenate([p14[:32000], np.full(768, 251, np.uint8)])),
            ("wide_40", np.concatenate([np.zeros(20, np.uint8), rng.integers(1, 200, 20, dtype=np.uint8)])),
            ("tiny_16", np.array([0] * 8 + [10, 60, 110, 160, 199, 30, 90, 140], np.uint8))]
    return out


def ref_repeat(ref, four, src, cap, msv, tlog, table, flag, prefer):
    """the reference's HUF_compress{4X,1X}_repeat on copies of (table, flag), with a zeroed workspace: (value, bytes, flag, table)"""
    n = len(src)
    dst = np.zeros(room(n, cap) + 64, np.uint8)
    ct = table.copy()
    rep = C.c_int(flag)
    wk = np.zeros(WKSP_WORDS, np.uint32)
    fn = ref.HUF_compress4X_repeat if four else ref.HUF_compress1X_repeat
    r = fn(ptr(dst), cap, ptr(src) if n else ptr(np.zeros(1, np.uint8)), n, msv, tlog, ptr(wk), WKSP_WORDS * 4, ptr(ct),
           C.byref(rep), prefer, 0)
    nbytes = 0 if is_error(r) else int(r)
    return int(r), dst[:nbytes].copy(), rep.value, ct


def estimate_edge_table(ref, src, msv, tlog, cap, extra_bytes=0):
    """an old table for `src` whose HUF_estimateCompressedSize is exactly hSize + that of the table the block builds (+ extra_bytes):
    the new table's codes, some lengthened until the estimates meet.  Codable (each val fits its length), not a prefix code."""
    n = len(src)
    cnt = (U * 256)()
    m = U(msv or 255)
    ref.HIST_count(cnt, C.byref(m), ptr(src), n)
    ct = np.zeros(256, np.uint32)
    bits = ref.HUF_buildCTable(ptr(ct), cnt, m.value, ref.HUF_optimalTableLog(tlog or 11, n, m.value))
    assert not is_error(bits)
    hdr = np.zeros(256, np.uint8)
    h = ref.HUF_writeCTable(ptr(hdr), cap, ptr(ct), m.value, bits)
    assert not is_error(h)
    count = np.array(cnt[:256], np.int64)
    nb = ((ct >> 16) & 0xFF).astype(np.int64)
    target = 8 * (h + (int((nb * count).sum()) >> 3) + extra_bytes)          # the old estimate's bits must be in [target, target + 7]
    need = target - int((nb * count).sum())
    reach = {0: None}                                                       # bits added -> (symbol, previous sum): a bounded knapsack
    for s_ in np.nonzero(count)[0]:
        for _ in range(12 - int(nb[s_])):
            for tot in sorted(reach, reverse=True):
                t2 = tot + int(count[s_])
                if t2 <= need + 7 and t2 not in reach:
                    reach[t2] = (s_, tot)
    tot = min(t for t in reach if t >= need)
    assert tot <= need + 7, (need, tot)
    while tot:
        s_, tot = reach[tot]
        nb[s_] += 1
    old = (ct & 0xFFFF) | (nb.astype(np.uint32) << 16)
    assert ref.HUF_estimateCompressedSize(ptr(old), cnt, m.value) == h + ref.HUF_estimateCompressedSize(ptr(ct), cnt, m.value) + extra_bytes
    return old


def main_cases(ref, four, msv, tlog):
    """every flag x prefer x table x block, at capacities cycling through the bound, above 2^32, 0, the reference's exact size and
    one under it.  Returns a list of dicts with the inputs and the reference's function value."""
    tabs = tables(ref)
    nb = (tabs["other"] >> 16) & 0xFF
    rare = np.argsort(-nb[:200].astype(np.int64), kind="stable")[:11].astype(np.uint8)   # the longest codes of "other"
    extra = [("rare_40", np.concatenate([np.full(20, rare[0], np.uint8), np.resize(rare[1:], 20)]))]
    out = []
    kinds = ("bound", "huge", "zero", "exact", "under", "bound")
    for i, (flag, prefer, (tname, tab), (bname, src)) in enumerate(itertools.product(FLAGS, PREFERS, tabs.items(), blocks() + extra)):
        kind = kinds[i % len(kinds)]
        cap = bound(len(src))
        if kind == "huge":
            cap = HUGE_CAP
        elif kind == "zero":
            cap = 0
        elif kind in ("exact", "under"):
            r0 = ref_repeat(ref, four, src, cap, msv, tlog, tab, flag, prefer)[0]
            if not is_error(r0) and r0 >= 2:
                cap = r0 if kind == "exact" else r0 - 1
        r, data, flag_out, tab_out = ref_repeat(ref, four, src, cap, msv, tlog, tab, flag, prefer)
        out.append(dict(src=src, cap=cap, table=tab, flag=flag, prefer=prefer, tname=tname, bname=bname, kind=kind,
                        r=r, data=data, flag_out=flag_out, table_out=tab_out, msv=msv, tlog=tlog))
    # both sides of the estimate comparison's edge (oldEst <= hSize + newEst keeps the old table): equal, and one byte above;
    # and a 20-byte block whose header is too large (hSize + 12 >= n) and whose old table is one byte worse by the estimate,
    # yet codes it (1X) in fewer than n - 1 bytes: only the hSize + 12 >= n exit keeps the old table there
    edge20 = np.array([0, 0, 55, 0, 20, 0, 0, 0, 0, 0, 50, 22, 196, 0, 0, 0, 0, 0, 0, 0], np.uint8)
    for extra_bytes, tname, src in ((0, "edge_equal", dict(blocks())["p14_32768"]), (1, "edge_above", dict(blocks())["p14_32768"]),
                                    (1, "edge_above", edge20)):
        tab = estimate_edge_table(ref, src, msv, tlog, bound(len(src)), extra_bytes)
        for flag in (1, 3):
            r, data, flag_out, tab_out = ref_repeat(ref, four, src, bound(len(src)), msv, tlog, tab, flag, 0)
            out.append(dict(src=src, cap=bound(len(src)), table=tab, flag=flag, prefer=0, tname=tname, bname="edge_%d" % len(src),
                            kind="bound", r=r, data=data, flag_out=flag_out, table_out=tab_out, msv=msv, tlog=tlog))
    return out


def main_configs():
    """(maxSymbolValue, tableLog) of the main batches: the defaults, a declared maxSymbolValue below some blocks' symbols"""
    return ((255, 12), (200, 11))
