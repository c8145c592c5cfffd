"""Helpers for the -m gpu suite: CPU-side compression with the checker (compiled reference when it
travelled with the snapshot, else the oracle port) into the bench.c slot layout."""
import ctypes as C
import os

import numpy as np

from helpers import load_port, load_ref, ptr, REF_SO, is_error

BLOCK = 32768
SLOT = 512 + BLOCK + (BLOCK >> 7) + 4 + 8
CODEC = {"fse": 0, "huf": 1, "u16": 2}


def checker():
    """(library, is_reference).  Never reads /root/reference at test time: only a prebuilt .so."""
    if os.path.exists(REF_SO):
        return load_ref(), True
    return load_port(), False


def cpu_compress(codec, data, block=BLOCK, slot=None, msv=255, tl=12, threads=0):
    data = np.ascontiguousarray(data)
    slot = slot or (512 + block + (block >> 7) + 12)
    nb = (len(data) + block - 1) // block
    cbuf = np.zeros(nb * slot + 64, np.uint8)
    cs = np.zeros(nb, np.uint64)
    lib, isref = checker()
    if isref:
        lib.refshim_compress_blocks(CODEC[codec], ptr(data), len(data), block, ptr(cbuf), slot, ptr(cs), msv, tl,
                                    threads or (os.cpu_count() or 1))
    else:
        lib.orc_compress_blocks(CODEC[codec], ptr(data), len(data), block, ptr(cbuf), slot, ptr(cs), msv, tl)
    return cbuf, cs, slot


POISON = 0x5A      # fills every byte around the views a placed check hands to the GPU
CANARY = 4096      # poisoned bytes checked on each side of each view


def arena(nbytes):
    """a poisoned device buffer with CANARY bytes of room on each side of nbytes (the view starts at CANARY + offset)"""
    import torch
    return torch.full((nbytes + 2 * CANARY + 128,), POISON, dtype=torch.uint8, device="cuda")


def header_only_u16(cblock, cs):
    """an FSE-U16 block whose compressed size is its table header alone (what FSE_compressU16 returns when the stream does
    not fit its dstCapacity)"""
    if cs <= 1 or is_error(cs):
        return False
    norm = (C.c_short * 512)()
    msv, tl = C.c_uint(511), C.c_uint(0)
    c = np.ascontiguousarray(cblock[:cs])
    h = load_ref().FSE_readNCount(norm, C.byref(msv), C.byref(tl), ptr(c), cs)
    return not is_error(h) and h == cs


def placed_check(codec, data, block, slot, want, src, cbuf, out, msv=255, tl=12):
    """Encode `data` from src = (arena, index) into the slots at cbuf = (arena, index), decode those slots and the reference's
    (`want` = cpu_compress output at the same block / slot) into out = (arena, index), and compare everything with the
    compiled reference: return values, bytes [0, cSize) of every slot, decoded bytes, and CANARY poisoned bytes on both sides
    of every view.  The compressed views start out holding the complement of the reference's bytes and the output views the
    complement of the expected output, so a dropped store cannot pass by finding the right byte already there."""
    import torch
    import finitestateentropy_b200 as fb
    enc = {"huf": fb.huf_compress_batch, "fse": fb.fse_compress_batch, "u16": fb.fseu16_compress_batch}[codec]
    dec = {"huf": fb.huf_decompress_batch, "fse": fb.fse_decompress_batch, "u16": fb.fseu16_decompress_batch}[codec]
    data = np.ascontiguousarray(data).view(np.uint8)
    n = len(data)
    nb = (n + block - 1) // block
    want_c, want_cs = want
    empty = [b for b in range(nb) if codec == "u16" and header_only_u16(want_c[b * slot: (b + 1) * slot], int(want_cs[b]))]
    cs_ref = want_cs.copy()
    cs_ref[empty] = 0                              # the reference's FSE_decompressU16 dereferences NULL on an empty stream ...
    want_out, want_res = cpu_decompress(codec, want_c, cs_ref, data, block=block, slot=slot)
    want_res[empty] = 2 ** 64 - 4                  # ... where the batch decoder reports corruption_detected (DESIGN 2)
    (sa, si), (ca, ci), (oa, oi) = src, cbuf, out
    views = [(sa, si, n), (ca, ci, nb * slot), (oa, oi, n)]
    for j, (a, i, k) in enumerate(views):
        assert CANARY <= i and i + k + CANARY <= a.numel()
        for a2, i2, k2 in views[:j]:                # views and their canaries are disjoint
            assert a2 is not a or i + k + CANARY <= i2 - CANARY or i2 + k2 + CANARY <= i - CANARY
        a[i - CANARY: i].fill_(POISON)              # the canaries belong to this check alone (an arena may serve several)
        a[i + k: i + k + CANARY].fill_(POISON)
    s_v = sa[si: si + n]
    s_v.copy_(torch.from_numpy(data))
    c_v = ca[ci: ci + nb * slot]
    o_v = oa[oi: oi + n]
    not_c = torch.from_numpy(~want_c[:nb * slot]).cuda()
    not_out = torch.from_numpy(~want_out).cuda()
    cs = torch.full((nb,), -7, dtype=torch.int64, device="cuda")
    res = torch.full((nb,), -7, dtype=torch.int64, device="cuda")
    c_v.copy_(not_c)
    enc(s_v, block, slot, msv, tl, cbuf=c_v, csizes=cs)
    got_cs = cs.cpu().numpy().view(np.uint64)
    assert np.array_equal(got_cs, want_cs), (codec, block, slot, [(b, int(got_cs[b]), int(want_cs[b])) for b in range(nb) if got_cs[b] != want_cs[b]][:5])
    got_c = c_v.cpu().numpy().reshape(nb, slot) if nb * slot else np.zeros((nb, slot), np.uint8)
    ref_c = want_c[:nb * slot].reshape(nb, slot)
    sizes = want_cs.astype(np.int64)
    sizes[want_cs > np.uint64(1 << 62)] = 0
    if codec != "huf":
        sizes[sizes == 1] = 0                      # FSE / U16 store nothing for an RLE verdict
    mask = np.arange(slot, dtype=np.int64)[None, :] < sizes[:, None]
    bad = (got_c != ref_c) & mask
    assert not bad.any(), (codec, block, slot, "compressed bytes differ in block", int(np.argwhere(bad)[0][0]))
    # decode the GPU's slots in place, then the reference's slots (copied over them)
    for label in ("own", "reference"):
        if label == "reference":
            c_v.copy_(torch.from_numpy(want_c[:nb * slot]).cuda())
            cs.copy_(torch.from_numpy(want_cs.view(np.int64)).cuda())
        o_v.copy_(not_out)
        res.fill_(-7)
        dec(c_v, cs, n, block, slot, out=o_v, results=res, orig=s_v)
        got_res = res.cpu().numpy().view(np.uint64)
        keep = np.array([not is_error(int(c)) for c in want_cs])
        assert np.array_equal(got_res[keep], want_res[keep]), (codec, label, block, slot,
                                                               [(b, int(got_res[b]), int(want_res[b])) for b in range(nb) if keep[b] and got_res[b] != want_res[b]][:5])
        got_out = o_v.cpu().numpy()
        for b in range(nb):
            if keep[b] and not is_error(int(want_res[b])):
                m = min(block, n - b * block)
                assert np.array_equal(got_out[b * block: b * block + m], want_out[b * block: b * block + m]), (codec, label, block, slot, b)
    torch.cuda.synchronize()
    for a, i, k in views:
        assert bool((a[i - CANARY: i] == POISON).all()) and bool((a[i + k: i + k + CANARY] == POISON).all()), (codec, "canary")
    return got_cs


def cpu_decompress(codec, cbuf, cs, orig, block=BLOCK, slot=None, threads=0):
    orig = np.ascontiguousarray(orig)
    slot = slot or (512 + block + (block >> 7) + 12)
    nb = (len(orig) + block - 1) // block
    out = np.zeros(len(orig), np.uint8)
    res = np.zeros(nb, np.uint64)
    lib, isref = checker()
    if isref:
        lib.refshim_decompress_blocks(CODEC[codec], ptr(out), ptr(orig), len(orig), block, ptr(cbuf), slot, ptr(cs), ptr(res),
                                      threads or (os.cpu_count() or 1))
    else:
        lib.orc_decompress_blocks(CODEC[codec], ptr(out), ptr(orig), len(orig), block, ptr(cbuf), slot, ptr(cs), ptr(res))
    return out, res
