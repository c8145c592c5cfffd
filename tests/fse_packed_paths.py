"""Host model of the packed FSE / FSE-U16 calls (FSEB200_FSE{,U16}_{compress,decompress}_packed, include/fse_b200.h), built from
the compiled reference's FSE_compress2 / FSE_compressU16 at FSE_compressBound and its decoders:

  values       the reference's value per block at FSE_compressBound(u * n), and the bytes the packed buffer holds for it;
  slots        the staging slots in the workspace: their offsets, and which blocks are coded (the rest: workSpace_tooSmall);
  layout       the stored lengths' offsets and the capacity rule;  image: the packed buffer as the call writes it;
  decode_rule  which of the decompress call's four rules settles a block;  ref_unpack: the regenerated blocks.

u is the unit: 1 for FSE, 2 for U16 (whose sizes count 16-bit symbols).  Used by tests/test_fse_packed_model.py (CPU) and
tests/test_gpu_fse_packed.py (the GPU calls against it)."""
import numpy as np

from gpu_common import header_only_u16
from helpers import is_error, ptr

FSE_BLOCK_MAX = 1 << 30
ERR_GENERIC = 2 ** 64 - 1
ERR_DST_TOO_SMALL = 2 ** 64 - 2
ERR_SRC_WRONG = 2 ** 64 - 3
ERR_CORRUPT = 2 ** 64 - 4
ERR_WKSP_TOO_SMALL = 2 ** 64 - 8


def unit(wide):
    return 2 if wide else 1


def fbound(nbytes):
    return 512 + nbytes + (nbytes >> 7) + 4 + 8        # FSE_compressBound (lib/fse.h:290-292)


def workspace(n_blocks, src_bytes):
    """FSEB200_FSE_packed_workspace"""
    return src_bytes + (src_bytes >> 7) + 524 * n_blocks


def limit_value(src_addr, n, wide):
    """the value the batch tier's limits settle for a block (it takes no staging slot), or None"""
    if wide and src_addr & 1:
        return ERR_GENERIC
    if n * unit(wide) > FSE_BLOCK_MAX:
        return ERR_SRC_WRONG
    return None


def ref_value(lib, src, wide, msv, tl):
    """(value, stored bytes) of one block: FSE_compress2 (U16: FSE_compressU16) at FSE_compressBound(u * n), and what the
    packed buffer holds for it -- the compressed bytes, the unit src[0] for RLE, the source for a raw block, nothing for an error"""
    raw = np.ascontiguousarray(src).view(np.uint8)
    n = len(raw) // unit(wide)
    cap = fbound(len(raw))
    buf = np.zeros(cap + 8, np.uint8)
    f = lib.FSE_compressU16 if wide else lib.FSE_compress2
    v = int(f(ptr(buf), cap, ptr(raw), n, msv, tl))
    L = stored_len(v, n, wide)
    if is_error(v):
        return v, raw[:0].copy()
    return v, (buf[:v].copy() if v > 1 else raw[:L].copy())


def stored_len(v, n, wide):
    """bytes block b takes in the packed buffer: the compressed size, u for RLE, u * n for a raw copy, nothing for an error"""
    v = int(v)
    if is_error(v):
        return 0
    return v if v > 1 else (unit(wide) if v == 1 else unit(wide) * n)


def slots(addrs, sizes, wide, work_size):
    """(slot offsets, coded): block b's staging slot starts at the exclusive prefix sum of FSE_compressBound(u * n) over the
    blocks that take one (None for a block the limits settle); it is coded only if its slot ends at or before work_size"""
    offs, coded, cur = [], [], 0
    for a, n in zip(addrs, sizes):
        if limit_value(a, n, wide) is not None:
            offs.append(None)
            coded.append(False)
            continue
        offs.append(cur)
        cur += fbound(unit(wide) * n)
        coded.append(cur <= work_size)
    return offs, coded


def values(vals, addrs, sizes, wide, work_size):
    """the values the compress call reports before its capacity rule: the limits' verdicts, workSpace_tooSmall for a block whose
    slot does not fit, the reference's value for the others (vals[b])"""
    _, coded = slots(addrs, sizes, wide, work_size)
    out = []
    for v, a, n, c in zip(vals, addrs, sizes, coded):
        lv = limit_value(a, n, wide)
        out.append(lv if lv is not None else (int(v) if c else ERR_WKSP_TOO_SMALL))
    return out


def layout(vals, sizes, out_capacity, wide):
    """(offsets [n + 1], final values, fits): the exclusive prefix sum of the stored lengths, and the capacity rule -- a block
    whose value is not an error and whose bytes end past out_capacity gets dstSize_tooSmall and is not written"""
    lens = [stored_len(v, n, wide) for v, n in zip(vals, sizes)]
    offs = [0]
    for L in lens:
        offs.append(offs[-1] + L)
    final, fits = [], []
    for b, v in enumerate(vals):
        ok = is_error(int(v)) or offs[b] + lens[b] <= out_capacity
        fits.append(ok and not is_error(int(v)))
        final.append(int(v) if ok else ERR_DST_TOO_SMALL)
    return offs, final, fits


def image(vals, stored, sizes, out_capacity, wide):
    """(image, written, offsets, final values): bytes [0, min(total, out_capacity)) of the packed buffer as the model writes it;
    `written` marks the bytes that belong to a stored block"""
    offs, final, fits = layout(vals, sizes, out_capacity, wide)
    end = min(offs[-1], out_capacity)
    img = np.zeros(end, np.uint8)
    written = np.zeros(end, bool)
    for b, s in enumerate(stored):
        if fits[b]:
            assert len(s) == offs[b + 1] - offs[b], (b, len(s))
            img[offs[b]: offs[b] + len(s)] = s
            written[offs[b]: offs[b] + len(s)] = True
    return img, written, offs, final


def decode_rule(L, n, dst_addr, wide):
    """'limit' (the decoder's own verdict), 'raw', 'rle' or 'decode' for a block of stored length L regenerating n units"""
    u = unit(wide)
    if (wide and dst_addr & 1) or L > FSE_BLOCK_MAX or n * u > FSE_BLOCK_MAX:
        return "limit"
    if L == u * n:
        return "raw"
    return "rle" if L == u else "decode"


def ref_unpack(lib, buf, L, n, wide, dst_addr=0):
    """(result, regenerated bytes or None) of the decompress call for one block: buf holds its L stored bytes (and more)"""
    u = unit(wide)
    rule = decode_rule(L, n, dst_addr, wide)
    if rule == "limit":
        return (ERR_GENERIC if wide and dst_addr & 1 else ERR_SRC_WRONG), None
    c = np.asarray(buf, np.uint8)
    if rule == "raw":
        return n, c[: u * n].copy()
    if rule == "rle":
        return n, np.tile(c[:u], n)
    if wide and header_only_u16(c, L):                # the reference dereferences NULL there; this library's answer (DESIGN 2)
        return ERR_CORRUPT, None
    tmp = np.concatenate([c[:L], np.zeros(64, np.uint8)])
    o = np.zeros(u * n + 64, np.uint8)
    f = lib.FSE_decompressU16 if wide else lib.FSE_decompress
    r = int(f(ptr(o), n, ptr(tmp), L))
    return r, (None if is_error(r) else o[: u * r].copy())
