"""Batches of .fse frames on pinned host buffers, on one GPU: one batch call (FSEB200_frame_{compress,decompress}_host_batch)
against a loop of one-frame calls (FSEB200_frame_{compress,decompress}_host) over the same frames.

  64k_p14_huf    16,384 frames of 64 KiB of probagen P14, Huff0   (checksums on the device)
  64k_p80_fse    16,384 frames of 64 KiB of probagen P80, FSE     (checksums on the device)
  1m_p14_huf     1,024 frames of 1 MiB of probagen P14, Huff0     (checksums on the device)
  256m_p14_huf   4 frames of 256 MiB of probagen P14, Huff0       (above the device-hash threshold: host threads)

Blocks of 32 KB (-B5).  Every call is synchronous and timed with a host clock; within a run the loop and the batch alternate,
and each figure is the median over --runs runs in ms per GiB of source.  Every batch frame must equal the loop's, and every
decoded byte the source.  Prints one JSON line with the GPU's name, power limit and SM clocks.

    python scripts/frame_batch_bench.py --runs 5
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
GIB = 1 << 30
BID = 5

from host_packed_bench import gpu_info                              # noqa: E402

WORKLOADS = (("64k_p14_huf", 16384, 64 << 10, 0.14, 1), ("64k_p80_fse", 16384, 64 << 10, 0.80, 0),
             ("1m_p14_huf", 1024, 1 << 20, 0.14, 1), ("256m_p14_huf", 4, 256 << 20, 0.14, 1))


def timed(fn):
    t = time.perf_counter()
    r = fn()
    return (time.perf_counter() - t) * 1e3, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--only", default=None, help="comma-separated workload names")
    args = ap.parse_args()
    import numpy as np
    import torch
    import finitestateentropy_b200 as fb
    from helpers import probagen
    L = fb.lib()
    out = {"bench": "frame_batch", "runs": args.runs, "block_size_id": BID}
    out.update(gpu_info())

    def pinned(n):
        return torch.empty(n, dtype=torch.uint8, pin_memory=True).numpy()

    for name, nf, fsize, p, codec in WORKLOADS:
        if args.only and name not in args.only.split(","):
            continue
        n = nf * fsize
        src = pinned(n)
        src[:] = probagen(n, p)
        bound = L.FSEB200_frame_compressBound(fsize, BID)
        cap = nf * bound
        frames, loop_frames, dst = pinned(cap), pinned(cap), pinned(n)
        sizes = np.full(nf, fsize, np.uint64)
        caps = np.full(nf, fsize, np.uint64)
        offs = np.zeros(nf + 1, np.uint64)
        res = np.zeros(nf, np.uint64)
        lens = np.zeros(nf, np.int64)
        s0, f0, l0, d0 = src.ctypes.data, frames.ctypes.data, loop_frames.ctypes.data, dst.ctypes.data

        def loop_c():
            for f in range(nf):                                     # frame f in its own bound-sized slot
                lens[f] = L.FSEB200_frame_compress_host(codec, BID, l0 + f * bound, bound, s0 + f * fsize, fsize)

        def loop_d():
            o = offs.tolist()
            for f in range(nf):
                r = L.FSEB200_frame_decompress_host(d0 + f * fsize, fsize, f0 + o[f], o[f + 1] - o[f])
                assert r == fsize, (name, f, r)

        def batch_c():
            r = L.FSEB200_frame_compress_host_batch(codec, BID, nf, f0, cap, offs.ctypes.data, res.ctypes.data, s0, sizes.ctypes.data)
            assert r == 0 and not any(fb.is_error(int(x)) for x in res[:4]), r

        def batch_d():
            r = L.FSEB200_frame_decompress_host_batch(nf, d0, caps.ctypes.data, res.ctypes.data, f0, offs.ctypes.data)
            assert r == 0 and (res == fsize).all(), (name, r)

        t = {k: [] for k in ("loop_c", "batch_c", "loop_d", "batch_d")}
        for run in range(args.runs):
            for k, fn in (("loop_c", loop_c), ("batch_c", batch_c), ("loop_d", loop_d), ("batch_d", batch_d)):
                dst[:] = 0
                ms, _ = timed(fn)
                t[k].append(ms)
                if k.endswith("_d"):
                    assert np.array_equal(dst, src), (name, k)
            if run == 0:
                o = offs.tolist()
                assert all(o[f + 1] - o[f] == lens[f] for f in range(nf)), name
                assert all(np.array_equal(frames[o[f]: o[f + 1]], loop_frames[f * bound: f * bound + lens[f]]) for f in range(nf)), name
        scale = GIB / n
        out[name] = {k: round(statistics.median(v) * scale, 1) for k, v in t.items()}
        out[name]["spread"] = {k: [round(min(v) * scale, 1), round(max(v) * scale, 1)] for k, v in t.items()}
        out[name]["frames"] = nf
        out[name]["frame_bytes"] = int(offs[-1])
        del src, frames, loop_frames, dst
    print(json.dumps(out))


if __name__ == "__main__":
    main()
