"""The .fse frame calls (FSEB200_frame_compress_host / FSEB200_frame_decompress_host) on pinned host buffers, on one GPU, against
what they replace and what bounds them:

  p14_huf   1 GiB of probagen P14 as a Huff0 frame, 32 KB blocks (-B5)
  p80_fse   1 GiB of probagen P80 as an FSE frame, 32 KB blocks

and, per input, in the same run:
  frame          the frame calls, compress and decompress
  slot_layout    the path the file tool took before the frame calls: the slot call (FSEB200_compress_host at (255, 11)), the
                 frame laid out on the host from its slots (numpy), then XXH32 over the input -- compress only
  xxh32          FSEB200_XXH32 over the GiB alone: the host checksum every frame carries, the format's floor
  fse_ref        the reference's tool (oracle/_ref/fse_ref, one thread) on a file of the GiB under a temporary directory,
                 file I/O included: `-h`/`-e -B5` and `-d`

Every call is synchronous and timed with a host clock; within a run the variants alternate, and each figure is the median over
--runs runs in ms per GiB of source.  Every frame must be byte-identical to the reference tool's, and every decoded GiB equal to
the source.  Prints one JSON line with the GPU's name, power limit and SM clocks.

    python scripts/frame_bench.py --runs 5
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
GIB = 1 << 30
BID = 5
BLOCK = 1024 << BID
REF = os.path.join(ROOT, "oracle", "_ref", "fse_ref")

from host_packed_bench import gpu_info                              # noqa: E402


def timed(fn):
    t = time.perf_counter()
    r = fn()
    return (time.perf_counter() - t) * 1e3, r


def slot_layout(L, np, src, codec, cbuf, cs):
    """the frame as the file tool used to write it: slot call, layout from the slots on the host, then the checksum"""
    n = src.size
    nb = (n + BLOCK - 1) // BLOCK
    slot = L.FSE_compressBound(BLOCK)
    r = L.FSEB200_compress_host(codec, cbuf.ctypes.data, slot, cs.ctypes.data, src.ctypes.data, n, BLOCK, 255, 11)
    assert r == 0, r
    c = cs[:nb].astype(np.int64)
    ins = np.full(nb, BLOCK, np.int64)
    ins[-1] = n - (nb - 1) * BLOCK
    full = ins == BLOCK
    typ = np.where(c == 0, 1, np.where(c == 1, 2, 0))
    hdr = 1 + np.where(full, 0, 2) + np.where(typ == 0, 2, 0)
    pay = np.where(typ == 1, ins, np.where(typ == 2, 1, c))
    parts = [np.frombuffer(b"\x09\x33\x3e\x18" if codec else b"\x09\x23\x3e\x18", np.uint8), np.array([BID], np.uint8)]
    slots = cbuf[: nb * slot].reshape(nb, slot)
    for b in range(nb):
        h = [typ[b] << 6 | (0x20 if full[b] else 0)]
        if not full[b]:
            h += [ins[b] >> 8, ins[b] & 0xFF]
        if typ[b] == 0:
            h += [c[b] >> 8, c[b] & 0xFF]
        parts.append(np.array(h, np.uint8))
        parts.append(src[b * BLOCK: b * BLOCK + pay[b]] if typ[b] else slots[b, : pay[b]])
    crc = (L.FSEB200_XXH32(src.ctypes.data, n, 0) >> 5) & 0x3FFFFF
    parts.append(np.array([0xC0 | crc >> 16, (crc >> 8) & 0xFF, crc & 0xFF], np.uint8))
    assert int(hdr.sum() + pay.sum()) + 8 == sum(p.size for p in parts)
    return np.concatenate(parts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--gib", type=float, default=1.0)
    args = ap.parse_args()
    import numpy as np
    import torch
    import finitestateentropy_b200 as fb
    from helpers import probagen
    L = fb.lib()
    n = int(args.gib * GIB)
    out = {"bench": "frame", "runs": args.runs, "bytes": n, "block_size_id": BID}
    out.update(gpu_info())
    tmp = tempfile.mkdtemp()
    for name, p, codec in (("p14_huf", 0.14, 1), ("p80_fse", 0.80, 0)):
        src = torch.empty(n, dtype=torch.uint8, pin_memory=True).numpy()
        src[:] = probagen(n, p)
        cap = L.FSEB200_frame_compressBound(n, BID)
        frame = torch.empty(cap, dtype=torch.uint8, pin_memory=True).numpy()
        dst = torch.empty(n, dtype=torch.uint8, pin_memory=True).numpy()
        nb = (n + BLOCK - 1) // BLOCK
        cbuf = torch.empty(nb * L.FSE_compressBound(BLOCK) + 64, dtype=torch.uint8, pin_memory=True).numpy()
        cs = np.zeros(nb, np.uint64)
        path, fpath, opath = os.path.join(tmp, "in.bin"), os.path.join(tmp, "in.fse"), os.path.join(tmp, "out.bin")
        src.tofile(path)
        t = {k: [] for k in ("frame_c", "frame_d", "slot_layout_c", "xxh32", "ref_c", "ref_d")}
        size = None
        for _ in range(args.runs):
            ms, size = timed(lambda: L.FSEB200_frame_compress_host(codec, BID, frame.ctypes.data, cap, src.ctypes.data, n))
            t["frame_c"].append(ms)
            ms, r = timed(lambda: L.FSEB200_frame_decompress_host(dst.ctypes.data, n, frame.ctypes.data, size))
            assert r == n and np.array_equal(dst, src), (name, r)
            t["frame_d"].append(ms)
            ms, old = timed(lambda: slot_layout(L, np, src, codec, cbuf, cs))
            assert old.size == size and np.array_equal(old, frame[:size]), name
            t["slot_layout_c"].append(ms)
            ms, _ = timed(lambda: L.FSEB200_XXH32(src.ctypes.data, n, 0))
            t["xxh32"].append(ms)
            if os.path.exists(REF):
                ms, _ = timed(lambda: subprocess.run([REF, "-f", "-q", "-h" if codec else "-e", "-B%d" % BID, path, fpath], check=True,
                                                     capture_output=True))
                t["ref_c"].append(ms)
                ms, _ = timed(lambda: subprocess.run([REF, "-f", "-q", "-d", fpath, opath], check=True, capture_output=True))
                t["ref_d"].append(ms)
        if os.path.exists(REF):
            assert open(fpath, "rb").read() == frame[:size].tobytes(), name
        scale = GIB / n
        out[name] = {k: round(statistics.median(v) * scale, 1) for k, v in t.items() if v}
        out[name]["frame_bytes"] = int(size)
        out[name]["frame_c_minus_xxh32"] = round(out[name]["frame_c"] - out[name]["xxh32"], 1)
        out[name]["frame_d_minus_xxh32"] = round(out[name]["frame_d"] - out[name]["xxh32"], 1)
        for f in (path, fpath, opath):
            if os.path.exists(f):
                os.remove(f)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
