"""Host model of the packed Huff0 compress (FSEB200_HUF_compress_packed / FSEB200_HUF_compress1X_packed, include/fse_b200.h):
the stored length of a block from its compress value, the offsets, the capacity rule, and the packed image built from the
compiled reference's HUF_compress2 / HUF_compress1X at HUF_compressBound(n).  Used by tests/test_packed_model.py (CPU) and
tests/test_gpu_packed.py (the GPU calls against it)."""

import numpy as np

from helpers import is_error, ptr

ERR_DST_TOO_SMALL = 2 ** 64 - 2


def hbound(n):
    return 129 + n + (n >> 8) + 8                   # HUF_compressBound (lib/huf.h:131-133)


def stored_len(v, n):
    """bytes block b takes in the packed buffer: the compressed size, the RLE byte, a raw copy (0: n bytes), nothing for an error"""
    v = int(v)
    return 0 if is_error(v) else (v if v else n)


def layout(vals, sizes, out_capacity):
    """(offsets [n + 1], final values, fits): the exclusive prefix sum of the stored lengths, and the capacity rule -- a block
    whose value is not an error and whose bytes end past out_capacity gets dstSize_tooSmall and is not written"""
    lens = [stored_len(v, n) for v, n in zip(vals, sizes)]
    offs = [0]
    for L in lens:
        offs.append(offs[-1] + L)
    final, fits = [], []
    for b, v in enumerate(vals):
        ok = is_error(int(v)) or offs[b] + lens[b] <= out_capacity
        fits.append(ok and not is_error(int(v)))
        final.append(int(v) if ok else ERR_DST_TOO_SMALL)
    return offs, final, fits


def ref_values(lib, srcs, msv, tl, onex=False):
    """(values, stored bytes) per block: HUF_compress2 (onex: HUF_compress1X) at HUF_compressBound(n), and the bytes the packed
    buffer holds for it -- the compressed bytes, src[0] for RLE, the source for a raw block, nothing for an error"""
    fn = lib.HUF_compress1X if onex else lib.HUF_compress2
    vals, stored = [], []
    for s in srcs:
        n = len(s)
        buf = np.zeros(hbound(n) + 8, np.uint8)
        src = np.ascontiguousarray(s, dtype=np.uint8)
        v = int(fn(ptr(buf), hbound(n), ptr(src), n, msv, tl))
        vals.append(v)
        L = stored_len(v, n)
        stored.append(buf[:L].copy() if v > 1 and not is_error(v) else (src[:1].copy() if v == 1 else src[:L].copy()))
    return vals, stored


def image(vals, stored, sizes, out_capacity):
    """(image, written, offsets, final values): bytes [0, min(total, out_capacity)) of the packed buffer as the model writes it;
    `written` marks the bytes that belong to a stored block (the others -- blocks that do not fit -- are never written)"""
    offs, final, fits = layout(vals, sizes, out_capacity)
    end = min(offs[-1], out_capacity)
    img = np.zeros(end, np.uint8)
    written = np.zeros(end, bool)
    for b, s in enumerate(stored):
        if fits[b]:
            img[offs[b]: offs[b] + len(s)] = s
            written[offs[b]: offs[b] + len(s)] = True
    return img, written, offs, final


def ref_decode(lib, img, offs, sizes, vals, onex=False):
    """the reference's decoder on every non-empty, non-error block of a packed image: the recipe of the header comment"""
    outs = []
    for b, n in enumerate(sizes):
        v = int(vals[b])
        if n == 0 or is_error(v):
            outs.append(None)
            continue
        L = offs[b + 1] - offs[b]
        c = np.concatenate([img[offs[b]: offs[b] + L], np.zeros(64, np.uint8)])
        o = np.zeros(n + 64, np.uint8)
        if onex:
            dt = np.zeros(1 + 4096, np.uint32)
            dt[0] = 12 * 0x01000001                     # HUF_CREATE_STATIC_DTABLEX2(dctx, HUF_TABLELOG_MAX)
            r = int(lib.HUF_decompress1X_DCtx(ptr(dt), ptr(o), n, ptr(c), L))
        else:
            r = int(lib.HUF_decompress(ptr(o), n, ptr(c), L))
        outs.append((r, o[:n].copy()))
    return outs
