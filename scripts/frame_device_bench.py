"""Batches of .fse frames in device memory, on one GPU: the device calls (FSEB200_frame_{compress,decompress}_device) against
the host batch calls (FSEB200_frame_{compress,decompress}_host_batch) on pinned host copies of the same bytes.

  64k_p14_huf    16,384 frames of 64 KiB of probagen P14, Huff0
  64k_p80_fse    16,384 frames of 64 KiB of probagen P80, FSE
  1m_p14_huf     1,024 frames of 1 MiB of probagen P14, Huff0
  256m_p14_huf   4 frames of 256 MiB of probagen P14, Huff0
  1g_p14_huf     1 frame of 1 GiB of probagen P14, Huff0

Blocks of 32 KB (-B5).  The device calls are timed with CUDA events on the current stream (the decompress synchronises it
once, inside the window), the host calls with a host clock around the synchronous call.  Within a run the four alternate, and
each figure is the median over --runs runs in ms per GiB of source; `walk` is FSEB200_frame_decompress_bound_device alone, the
header walk with its one synchronisation.  In every run the device frames, offsets and results must equal the host call's,
and every decoded byte the source.  Prints one JSON line with the GPU's name, power limit and SM clocks.

    python scripts/frame_device_bench.py --runs 5
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
             ("1m_p14_huf", 1024, 1 << 20, 0.14, 1), ("256m_p14_huf", 4, 256 << 20, 0.14, 1), ("1g_p14_huf", 1, 1 << 30, 0.14, 1))


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
    assert torch.cuda.is_available(), "the device calls need a GPU"
    out = {"bench": "frame_device", "runs": args.runs, "block_size_id": BID}
    out.update(gpu_info())
    stream = torch.cuda.current_stream()
    sp = stream.cuda_stream

    def pinned(n):
        return torch.empty(n, dtype=torch.uint8, pin_memory=True)

    for name, nf, fsize, p, codec in WORKLOADS:
        if args.only and name not in args.only.split(","):
            continue
        n = nf * fsize
        hsrc = pinned(n)
        hsrc.numpy()[:] = probagen(n, p)
        cap = nf * L.FSEB200_frame_compressBound(fsize, BID)
        hframes, hdst = pinned(cap), pinned(n)
        sizes = np.full(nf, fsize, np.uint64)
        caps = np.full(nf, fsize, np.uint64)
        hoffs, hres = np.zeros(nf + 1, np.uint64), np.zeros(nf, np.uint64)
        dsrc = hsrc.cuda()
        dframes = torch.empty(cap + 32, dtype=torch.uint8, device="cuda")
        ddst = torch.empty(n, dtype=torch.uint8, device="cuda")
        doffs = torch.empty(nf + 1, dtype=torch.int64, device="cuda")
        dres = torch.empty(nf, dtype=torch.int64, device="cuda")
        bounds = np.zeros(nf, np.uint64)

        def host_c():
            r = L.FSEB200_frame_compress_host_batch(codec, BID, nf, hframes.data_ptr(), cap, hoffs.ctypes.data, hres.ctypes.data,
                                                    hsrc.data_ptr(), sizes.ctypes.data)
            assert r == 0, r

        def host_d():
            r = L.FSEB200_frame_decompress_host_batch(nf, hdst.data_ptr(), caps.ctypes.data, hres.ctypes.data, hframes.data_ptr(),
                                                      hoffs.ctypes.data)
            assert r == 0 and (hres == fsize).all(), (name, r)

        def dev_c():
            r = L.FSEB200_frame_compress_device(codec, BID, nf, dframes.data_ptr(), cap, doffs.data_ptr(), dres.data_ptr(),
                                                dsrc.data_ptr(), sizes.ctypes.data, sp)
            assert r == 0, r

        def dev_d():
            r = L.FSEB200_frame_decompress_device(nf, ddst.data_ptr(), caps.ctypes.data, dres.data_ptr(), dframes.data_ptr(),
                                                  hoffs.ctypes.data, sp)
            assert r == 0, r

        def walk():
            r = L.FSEB200_frame_decompress_bound_device(nf, bounds.ctypes.data, dframes.data_ptr(), hoffs.ctypes.data, sp)
            assert r == 0 and (bounds == fsize).all(), r

        def host_timed(fn):
            torch.cuda.synchronize()
            t = time.perf_counter()
            fn()
            return (time.perf_counter() - t) * 1e3

        def dev_timed(fn):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record(stream)
            fn()
            b.record(stream)
            b.synchronize()
            return a.elapsed_time(b)

        # warm-up: every call once at this shape
        host_c(); dev_c(); walk(); host_d(); dev_d()
        torch.cuda.synchronize()
        t = {k: [] for k in ("host_c", "dev_c", "host_d", "dev_d", "walk")}
        for run in range(args.runs):
            hdst.zero_(); ddst.zero_()
            t["host_c"].append(host_timed(host_c))
            t["dev_c"].append(dev_timed(dev_c))
            total = int(hoffs[-1])
            assert doffs.cpu().numpy().astype(np.uint64).tolist() == hoffs.tolist(), name
            assert (dres.cpu().numpy() == hres.astype(np.int64)).all(), name
            assert torch.equal(dframes[:total].cpu(), hframes[:total]), name
            t["walk"].append(host_timed(walk))
            t["host_d"].append(host_timed(host_d))
            t["dev_d"].append(dev_timed(dev_d))
            assert bool((dres == fsize).all()), name
            assert torch.equal(hdst, hsrc) and torch.equal(ddst, dsrc), name
        scale = GIB / n
        out[name] = {k: round(statistics.median(v) * scale, 2) for k, v in t.items()}
        out[name]["spread"] = {k: [round(min(v) * scale, 2), round(max(v) * scale, 2)] for k, v in t.items()}
        out[name]["frames"] = nf
        out[name]["frame_bytes"] = int(hoffs[-1])
        del hsrc, hframes, hdst, dsrc, dframes, ddst
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
