"""Oracles and inputs of tests/test_gpu_table_logs.py: every codec at every tableLog and maxSymbolValue it accepts.

  fse_steps / u16_steps   FSE_compress2 / FSE_compressU16 done one reference function at a time (HIST_count, the early exits,
                          FSE_optimalTableLog, FSE_normalizeCount, FSE_writeNCount, FSE_buildCTable, the stream writer, the
                          compressibility test).  The reference's own block functions lay their table and scratch out for the
                          REQUESTED tableLog and maxSymbolValue, and can fault when FSE_optimalTableLog raises the request or
                          when the requested CTable alone exceeds the workspace; such requests are answered by these instead
                          (`ref_call_safe`).
  huf_limit_trace         HUF_buildCTable's sort, tree and HUF_setMaxHeight restated on the host, with the branches the depth
                          limiter takes (lib/huf_compress.c:215-291).
  normalize_method        which of FSE_normalizeCount's two methods a histogram takes and whether it has -1 cells.
  u16_tl13_stream         an FSE-U16 stream whose header says tableLog 13 (the linked FSE_normalizeCount / FSE_writeNCount stop
                          at 12): a plain normalization, a host NCount writer, FSE_buildCTableU16 and the reference's
                          single-state U16 stream writer.

Only the compiled reference library (oracle/_ref) is used, never the reference's source tree."""
import ctypes as C

import numpy as np

from helpers import is_error, ptr

U = C.c_uint
M32 = (1 << 32) - 1


def err(code):
    return 2 ** 64 - code


ERR_GENERIC, ERR_TLOG_LARGE, ERR_MSV_LARGE, ERR_WKSP_SMALL = (err(c) for c in (1, 5, 6, 8))
TABLE_LOGS = list(range(16)) + [255, M32]
FSE_WKSP_BYTES = 14340          # sizeof(fseWkspMax_t) of FSE_compress2 (lib/fse_compress.c:679-685) on x86-64


def msv_values(top):
    """the requested maxSymbolValue values of the sweep around a fixture whose blocks mostly top out at `top` (767 and 768:
    the last value byte FSE refuses with workSpace_tooSmall at tableLog 12 and the first whose CTable exceeds the workspace)"""
    return [0, top - 1, top, top + 1, 254, 255, 256, 286, 287, 767, 768, 4095, 5632, 5633, M32]


def bound(n):
    return 512 + n + (n >> 7) + 4 + 8


# ---- FSE step by step -------------------------------------------------------------------------------------------------------

def fse_wksp_fits(msv, tl):
    """FSE_compress_wksp's `wkspSize < FSE_WKSP_SIZE_U32(tableLog, maxSymbolValue)` test with the REQUESTED values, as compiled:
    unsigned 32-bit arithmetic (maxSymbolValue 2^32-1 wraps the symbol term to 0) against a size in bytes.  tableLog 0 shifts
    by -1, which the compiled reference answers with tableLog_tooLarge."""
    if tl == 0:
        return False
    need = (1 + (1 << (tl - 1)) + (((msv + 1) & M32) * 2 & M32) + 1024) & M32
    return FSE_WKSP_BYTES >= need


def raised(ref, data, msv, tl):
    """True unless FSE_optimalTableLog(tl, n, actual max) <= tl and the requested maxSymbolValue is at least the actual maximum"""
    n = len(data)
    top = int(data.max()) if n else 0
    return not (ref.FSE_optimalTableLog(tl & M32, n, top) <= tl and msv >= top)


def scratch_bytes(msv, tl):
    """bytes FSE_compress_wksp leaves for its scratch after a CTable sized for the REQUESTED tableLog and maxSymbolValue
    (lib/fse_compress.c:641-643, FSE_CTABLE_SIZE_U32 in unsigned 32-bit arithmetic); negative where the size_t subtraction
    wraps and the scratch lies past the 14,340-byte stack workspace"""
    return FSE_WKSP_BYTES - 4 * ((1 + (1 << (tl - 1)) + (((msv + 1) & M32) * 2 & M32)) & M32)


def wksp_too_small(msv, tl):
    """HIST_count_wksp refuses a scratch of 0 to 4095 bytes with workSpace_tooSmall (hist.c:168), before anything is written:
    at tableLog 12, maxSymbolValue 256 to 767"""
    return tl <= 12 and fse_wksp_fits(msv, tl) and 0 <= scratch_bytes(msv, tl) < 4096


def layout_overflows(msv, tl):
    """the requested CTable alone exceeds the workspace (tableLog 12: maxSymbolValue 768 up to 5632, the largest the workspace
    test lets through): the scratch size wraps and the reference's block call runs past its stack"""
    return tl <= 12 and fse_wksp_fits(msv, tl) and scratch_bytes(msv, tl) < 0


def ref_call_safe(ref, data, msv, tl, wide=False):
    """whether the reference's FSE_compress2 / FSE_compressU16 may be called: a request that is not raised and (bytes) whose
    workspace layout fits, or (bytes) one refused with workSpace_tooSmall before its layout is used.  Everything else is
    answered by fse_steps / u16_steps."""
    if len(data) == 0:
        return False
    if wide:
        return not raised(ref, data, msv, tl)
    return wksp_too_small(msv, tl) or not (raised(ref, data, msv, tl) or layout_overflows(msv, tl))


def _norm_write_ctable(ref, count, n, msv, tl, cap, wide):
    """steps 4 to 6: (header bytes or error, norm, CTable words)"""
    norm = (C.c_short * 300)()
    r = ref.FSE_normalizeCount(norm, tl, count, n, msv)
    if is_error(r):
        return r, None, None
    hdr = np.zeros(max(cap, 0) + 600, np.uint8)
    h = ref.FSE_writeNCount(ptr(hdr), cap, norm, msv, tl)
    if is_error(h):
        return h, None, None
    ct = np.zeros(1 + 4096 + 2 * 300, np.uint32)
    e = (ref.FSE_buildCTableU16 if wide else ref.FSE_buildCTable)(ptr(ct), norm, msv, tl)
    if is_error(e):
        return e, None, None
    return hdr[:h].copy(), norm, ct


def fse_steps(ref, cap, data, msv, tl):
    """FSE_compress2 (bytes) one reference function at a time: (value, bytes [0, value))"""
    data = np.ascontiguousarray(data, np.uint8)
    n = len(data)
    if tl > 12 or not fse_wksp_fits(msv, tl):
        return ERR_TLOG_LARGE, b""
    if n <= 1:
        return 0, b""
    if wksp_too_small(msv, tl):
        return ERR_WKSP_SMALL, b""
    msv = msv or 255
    tl = tl or 11
    count = (U * 256)()
    m = U(min(msv, 255))
    mx = ref.HIST_count(count, C.byref(m), ptr(data), n)                 # step 1
    if is_error(mx):
        return mx, b""
    if mx == n:                                                          # step 2
        return 1, b""
    if mx == 1 or mx < (n >> 7):
        return 0, b""
    msv = m.value
    tl = ref.FSE_optimalTableLog(tl, n, msv)                             # step 3
    hdr, norm, ct = _norm_write_ctable(ref, count, n, msv, tl, cap, False)   # steps 4-6
    if norm is None:
        return hdr, b""
    body = np.zeros(cap - len(hdr) + 16, np.uint8)
    cs = ref.FSE_compress_usingCTable(ptr(body), cap - len(hdr), ptr(data), n, ptr(ct))   # step 7
    if is_error(cs):
        return cs, b""
    if cs == 0:
        return 0, b""
    total = len(hdr) + cs
    if total >= n - 1:                                                   # step 8
        return 0, b""
    return total, bytes(hdr) + bytes(body[:cs])


def _u16_sigs(ref):
    ref.FSE_countU16.restype = C.c_size_t
    ref.FSE_countU16.argtypes = [C.POINTER(U), C.POINTER(U), C.c_void_p, C.c_size_t]
    ref.FSE_compressU16_usingCTable.restype = C.c_size_t
    ref.FSE_compressU16_usingCTable.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]


def u16_steps(ref, cap, data, msv, tl):
    """FSE_compressU16 (lib/fseU16.c:203-251) one reference function at a time: (value, bytes [0, value))"""
    _u16_sigs(ref)
    data = np.ascontiguousarray(data, np.uint16)
    n = len(data)
    if n <= 1:
        return n, b""
    msv = msv or 286
    tl = tl or 12
    if msv > 286:
        return ERR_MSV_LARGE, b""
    if tl > 13:
        return ERR_TLOG_LARGE, b""
    count = (U * 300)()
    m = U(msv)
    mx = ref.FSE_countU16(count, C.byref(m), ptr(data), n)               # step 1
    if is_error(mx):
        return mx, b""
    if mx == n:                                                          # step 2
        return 1, b""
    msv = m.value
    tl = ref.FSE_optimalTableLog(tl, n, msv)                             # step 3
    hdr, norm, ct = _norm_write_ctable(ref, count, n, msv, tl, cap, True)    # steps 4-6
    if norm is None:
        return hdr, b""
    assert cap - len(hdr) > 8                                            # below that the writer's init error is ignored
    body = np.zeros(cap - len(hdr) + 16, np.uint8)
    cs = ref.FSE_compressU16_usingCTable(ptr(body), cap - len(hdr), ptr(data), n, ptr(ct))   # step 7
    total = len(hdr) + cs
    if total >= (n - 1) * 2:                                             # step 8
        return 0, b""
    return total, bytes(hdr) + bytes(body[:cs])


# ---- NCount writer and tableLog-13 U16 streams --------------------------------------------------------------------------------

def write_ncount(norm, msv, tl):
    """FSE_writeNCount (lib/fse_compress.c:193-283) on an unlimited buffer, for any tableLog 5..15"""
    out = bytearray()
    bs, bc = (tl - 5), 4
    remaining, threshold, nb = (1 << tl) + 1, 1 << tl, tl + 1
    sym, prev0 = 0, False
    while sym <= msv and remaining > 1:
        if prev0:
            start = sym
            while sym <= msv and not norm[sym]:
                sym += 1
            if sym > msv:
                break
            while sym >= start + 24:
                start += 24
                bs += 0xFFFF << bc
                out += bytes([bs & 0xFF, (bs >> 8) & 0xFF]); bs >>= 16
            while sym >= start + 3:
                start += 3
                bs += 3 << bc; bc += 2
            bs += (sym - start) << bc; bc += 2
            if bc > 16:
                out += bytes([bs & 0xFF, (bs >> 8) & 0xFF]); bs >>= 16; bc -= 16
        cnt = int(norm[sym]); sym += 1
        mx = (2 * threshold - 1) - remaining
        remaining -= abs(cnt)
        cnt += 1
        if cnt >= threshold:
            cnt += mx
        bs += cnt << bc
        bc += nb - (cnt < mx)
        prev0 = cnt == 1
        assert remaining >= 1
        while remaining < threshold:
            nb -= 1; threshold >>= 1
        if bc > 16:
            out += bytes([bs & 0xFF, (bs >> 8) & 0xFF]); bs >>= 16; bc -= 16
    assert remaining == 1
    out += bytes([bs & 0xFF, (bs >> 8) & 0xFF])
    return bytes(out[: len(out) - 2 + (bc + 7) // 8])


def plain_norm(hist, tl):
    """every present symbol at least 1 cell, the rest by largest remainder: a valid distribution over 2^tl cells"""
    hist = np.asarray(hist, np.int64)
    cells = 1 << tl
    present = hist > 0
    assert present.sum() <= cells
    extra = cells - int(present.sum())
    share = hist * extra / hist.sum()
    norm = present.astype(np.int64) + np.floor(share).astype(np.int64)
    left = cells - int(norm.sum())
    order = np.argsort(-(share - np.floor(share)), kind="stable")
    norm[order[:left]] += 1
    assert norm.sum() == cells and (norm[present] > 0).all()
    return [int(x) for x in norm]


def u16_tl13_stream(ref, data, tl=13):
    """an FSE-U16 block whose header says tableLog `tl` (13): FSE_buildCTableU16 on a plain normalization, the host NCount
    writer and the single-state stream writer"""
    data = np.ascontiguousarray(data, np.uint16)
    hist = np.bincount(data)
    msv = len(hist) - 1
    norm = plain_norm(hist, tl)
    ct = np.zeros(1 + (1 << (tl - 1)) + 2 * 300, np.uint32)
    nrm = (C.c_short * 300)(*norm)
    assert ref.FSE_buildCTableU16(ptr(ct), nrm, msv, tl) == 0
    hdr = write_ncount(norm, msv, tl)
    _u16_sigs(ref)
    body = np.zeros(bound(2 * len(data)) + 16, np.uint8)
    cs = ref.FSE_compressU16_usingCTable(ptr(body), bound(2 * len(data)), ptr(data), len(data), ptr(ct))
    assert 0 < cs and not is_error(cs)
    return np.concatenate([np.frombuffer(hdr, np.uint8), body[:cs]])


# ---- Huff0 depth limiter -------------------------------------------------------------------------------------------------------

NONE = 0xF0F0F0F0


def huf_limit_trace(count, msv, max_bits):
    """HUF_buildCTable_wksp's sort, tree and HUF_setMaxHeight on the host: (code length per symbol 0..msv, branches), branches
    a subset of {'none', 'repay', 'giveback', 'giveback_new_rank1'}: no limiting; the debt-repayment loop; its overshoot given
    back from the rank-1 position; the give-back creating a rank-1 position when there is none"""
    count = [int(c) for c in count[:msv + 1]]
    max_bits = max_bits or 11
    # HUF_sort: decreasing order, buckets by highbit(count+1), insertion inside a bucket
    hb = lambda v: v.bit_length() - 1
    base = [0] * 32
    for c in count:
        base[hb(c + 1)] += 1
    for r in range(30, 0, -1):
        base[r - 1] += base[r]
    cur = base[:]
    node_c, node_b = [0] * 512, [0] * 512
    for s, c in enumerate(count):
        r = hb(c + 1) + 1
        p = cur[r]; cur[r] += 1
        while p > base[r] and c > node_c[p - 1]:
            node_c[p], node_b[p] = node_c[p - 1], node_b[p - 1]
            p -= 1
        node_c[p], node_b[p] = c, s
    last = msv
    while node_c[last] == 0:
        last -= 1
    START = 256
    parent = [0] * 512
    low_s, root, low_n = last, START + last - 1, START
    node_c[START] = node_c[low_s] + node_c[low_s - 1]
    parent[low_s] = parent[low_s - 1] = START
    nb = START + 1
    low_s -= 2
    for k in range(nb, root + 1):
        node_c[k] = 1 << 30
    cnt = lambda i: (1 << 31) if i < 0 else node_c[i]
    while nb <= root:
        n1 = low_s if cnt(low_s) < cnt(low_n) else low_n
        if n1 == low_s: low_s -= 1
        else: low_n += 1
        n2 = low_s if cnt(low_s) < cnt(low_n) else low_n
        if n2 == low_s: low_s -= 1
        else: low_n += 1
        node_c[nb] = node_c[n1] + node_c[n2]
        parent[n1] = parent[n2] = nb
        nb += 1
    bits = [0] * 512
    for k in range(root - 1, START - 1, -1):
        bits[k] = bits[parent[k]] + 1
    for k in range(last + 1):
        bits[k] = bits[parent[k]] + 1
    branches = set()
    largest = bits[last]
    if largest <= max_bits:
        branches.add("none")
    else:
        total = 0
        base_cost = 1 << (largest - max_bits)
        n = last
        while bits[n] > max_bits:
            total += base_cost - (1 << (largest - bits[n]))
            bits[n] = max_bits
            n -= 1
        while bits[n] == max_bits:
            n -= 1
        total >>= largest - max_bits
        rank_last = [NONE] * 14
        cb = max_bits
        for p in range(n, -1, -1):
            if bits[p] >= cb:
                continue
            cb = bits[p]
            rank_last[max_bits - cb] = p
        while total > 0:
            branches.add("repay")
            dec = total.bit_length()
            while dec > 1:
                hi, lo = rank_last[dec], rank_last[dec - 1]
                if hi == NONE:
                    dec -= 1
                    continue
                if lo == NONE or node_c[hi] <= 2 * node_c[lo]:
                    break
                dec -= 1
            while dec <= 12 and rank_last[dec] == NONE:
                dec += 1
            total -= 1 << (dec - 1)
            if rank_last[dec - 1] == NONE:
                rank_last[dec - 1] = rank_last[dec]
            bits[rank_last[dec]] += 1
            if rank_last[dec] == 0:
                rank_last[dec] = NONE
            else:
                rank_last[dec] -= 1
                if bits[rank_last[dec]] != max_bits - dec:
                    rank_last[dec] = NONE
        while total < 0:
            if rank_last[1] == NONE:
                branches.add("giveback_new_rank1")
                while bits[n] == max_bits:
                    n -= 1
                bits[n + 1] -= 1
                rank_last[1] = n + 1
                total += 1
                continue
            branches.add("giveback")
            bits[rank_last[1] + 1] -= 1
            rank_last[1] += 1
            total += 1
    lengths = [0] * (msv + 1)
    for k in range(msv + 1):
        lengths[node_b[k]] = bits[k] if k <= last else 0
    return lengths, branches


def normalize_method(count, n, msv, tl):
    """(-1 cells present, second method taken) of FSE_normalizeCount's first pass (lib/fse_compress.c:445-476), for a
    histogram that is not RLE and a tableLog it accepts"""
    rtb = [0, 473195, 504333, 520860, 550000, 700000, 750000, 830000]
    scale = 62 - tl
    step = (1 << 62) // n
    vstep = 1 << (scale - 20)
    still = 1 << tl
    low = n >> tl
    largest, largest_p, norm, minus1 = 0, 0, {}, False
    for s in range(msv + 1):
        c = int(count[s])
        if c == 0:
            continue
        if c <= low:
            minus1 = True
            still -= 1
            norm[s] = -1
            continue
        prob = (c * step) >> scale
        if prob < 8:
            prob += ((c * step) - (prob << scale)) > vstep * rtb[prob]
        if prob > largest_p:
            largest_p, largest = prob, s
        norm[s] = prob
        still -= prob
    return minus1, -still >= (norm.get(largest, 0) >> 1)


# ---- inputs --------------------------------------------------------------------------------------------------------------------

def from_counts(rng, counts, symbols):
    """a shuffled block with counts[i] copies of symbols[i]"""
    v = np.repeat(np.asarray(symbols, np.int64), np.asarray(counts, np.int64))
    return rng.permutation(v)


def fit_counts(counts, n):
    """counts scaled to sum to n, every one at least 1 (the remainder on the largest)"""
    c = np.maximum(1, np.floor(np.asarray(counts, np.float64) * n / float(np.sum(counts)))).astype(np.int64)
    c[int(np.argmax(c))] += n - int(c.sum())
    assert c.min() >= 1 and c.sum() == n
    return c


def shaped_blocks(rng, n, top, wide=False):
    """blocks of n symbols whose histograms reach the depth limiter's branches, FSE's -1 cells and second normalization method,
    and Huffman codes of 1 to 4 bits: Fibonacci-like and geometric counts over alphabets of 2 to 256 (U16: 286) symbols mapped
    below or onto `top` (the largest symbol of most blocks), flat small alphabets, and a few zoo-like blocks"""
    hi = 286 if wide else 255
    blocks = []

    def symbols(k):
        if k <= top + 1:                        # the block's largest symbol is top
            return np.concatenate([np.sort(rng.choice(top, k - 1, replace=False)), [top]])
        return np.sort(rng.choice(hi + 1, k, replace=False))

    for k in (7, 9, 12, 14, 16, 20, 24, 30, 32):                                      # Fibonacci-like: deepest trees
        f = [1, 1]
        while len(f) < k:
            f.append(f[-1] + f[-2] + int(rng.integers(0, 2)))
        blocks.append(from_counts(rng, fit_counts(f, n) if sum(f) > n else np.array(f[:-1] + [f[-1] + n - sum(f)]), symbols(k)))
    for k in (6, 10, 16, 24, 32, 48, 64, 100, 128, 200, 256) + ((286,) if wide else ()):   # geometric
        for q in (0.55, 0.7, 0.85):
            c = np.floor(1e6 * q ** np.arange(k)) + 1
            blocks.append(from_counts(rng, fit_counts(c, n), symbols(k)))
    for k in (2, 3, 4, 5, 8, 11, 16):                                                 # flat: codes of 1 to 4 bits
        blocks.append(from_counts(rng, fit_counts(np.ones(k), n), symbols(k)))
    for k in (40, 90, 180):                                                           # one dominant symbol over many rare ones
        c = np.ones(k) * max(1, n // (k * 40)) + rng.integers(0, 3, k)
        c[0] = n
        blocks.append(from_counts(rng, fit_counts(c, n), symbols(k)))
    if not wide:
        blocks.append(rng.integers(0, 256, n))                                        # noise: raw
    blocks.append(np.full(n, top))                                                    # RLE
    dt = np.uint16 if wide else np.uint8
    return [np.ascontiguousarray(b.astype(dt)) for b in blocks]


def limiter_blocks(rng, n, top):
    """for every maxNbBits 5..12, a block whose tree the depth limiter gives back on from an existing rank-1 position and one
    where the give-back has to create it: a seeded search over Pareto, geometric and Fibonacci-like counts (at most 16 symbols,
    onto 0..top, where HUF_optimalTableLog must keep a request of 5 to 8; up to 64 symbols above)"""
    out = []
    for mb in range(5, 13):
        for want in ("giveback", "giveback_new_rank1"):
            for it in range(20000):
                k = int(rng.integers(3, 17 if mb <= 8 else 65))
                kind = it % 3
                if kind == 0:
                    c = np.floor(1e6 * float(rng.uniform(0.3, 0.8)) ** np.arange(k)) + 1
                elif kind == 1:
                    c = rng.pareto(float(rng.uniform(0.3, 1.5)), k) * 100 + 1
                else:
                    f = [1, 1]
                    while len(f) < k:
                        f.append(f[-1] + f[-2] + int(rng.integers(0, 3)))
                    c = np.array(f, float) * float(rng.uniform(1, 3))
                c = fit_counts(c, n)
                syms = np.concatenate([np.arange(k - 1), [top]]) if k <= top + 1 else np.sort(rng.choice(256, k, replace=False))
                h = np.zeros(256, np.int64)
                h[syms] = c
                _, br = huf_limit_trace(h, int(syms.max()), mb)
                if want in br and (want == "giveback_new_rank1" or "giveback_new_rank1" not in br):
                    out.append(from_counts(rng, c, syms).astype(np.uint8))
                    break
            else:
                raise AssertionError("no input found for %s at maxNbBits %d" % (want, mb))
    return out


def m2_blocks(rng, n, top, wide=False):
    """for every tableLog 5..12, a block that FSE_normalizeCount sends to its second method at that tableLog: half its symbols
    share the block evenly, the other half occur once and take a whole cell each (-1), so the first method overshoots by about
    half a cell per rare symbol while its largest share is small.  Symbols stay below 2^(tl-1) (tableLog 5: onto 0..top), so
    FSE_optimalTableLog keeps the request."""
    out = []
    for tl in range(5, 13):
        k = min(1 << (tl - 1), 287 if wide else 256)
        for it in range(100):
            k2 = k // 2 + int(rng.integers(0, k // 4 + 1))
            k1 = k - k2
            c = np.concatenate([np.ones(k1) * ((n - k2) // k1) + rng.integers(-3, 4, k1), np.ones(k2)]).astype(np.int64)
            c[0] += n - int(c.sum())
            syms = np.concatenate([np.arange(k - 1), [top]]) if k <= top + 1 else np.arange(k)
            h = np.zeros(int(syms.max()) + 1, np.int64)
            h[syms] = c
            if normalize_method(h, n, int(syms.max()), tl)[1]:
                out.append(from_counts(rng, c, syms).astype(np.uint16 if wide else np.uint8))
                break
        else:
            raise AssertionError("no input found for the second method at tableLog %d" % tl)
    return out


def raw_weight_blocks(rng, n):
    """Huff0 blocks whose tree has one code length for all but one symbol (their weights compress to RLE, so HUF_writeCTable
    writes them raw): k symbols of one count plus symbol k holding a quarter of the block, k = 128, 192, 224"""
    out = []
    for k in (128, 192, 224):
        big = n // 4
        a = (n - big) // k
        c = [a] * k + [n - a * k]
        out.append(np.ascontiguousarray(from_counts(rng, c, range(k + 1)).astype(np.uint8)))
    return out
