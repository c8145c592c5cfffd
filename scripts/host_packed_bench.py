"""The packed host-buffer pair (FSEB200_compress_host_packed + FSEB200_decompress_host_packed) against the slot-based pair
(FSEB200_compress_host + FSEB200_decompress_host) on pinned host buffers, on one GPU.

  p14_huf     1 GiB of probagen P14 in 32 KB blocks, Huff0 4X (255, 12)
  p80_fse     1 GiB of probagen P80 in 32 KB blocks, FSE (255, 12)
  ragged_huf  the P14 GiB cut into seeded sizes uniform in [1 KiB, 128 KiB], Huff0 4X: packed pair only (the slot form takes
              one block size)
  ragged_fse  the same cut of the P80 GiB, FSE: packed pair only
  random_huf  1 GiB of random bytes in 32 KB blocks, every block raw, Huff0 4X.  The packed compress copies the whole GiB back
              down because it stores the raw blocks; the slot compress copies nothing for them and its decompress rebuilds them
              from the original -- a cost of a stream that stands on its own, not a like-for-like comparison.

Every call is synchronous and timed with a host clock; within a run the slot pair and the packed pair alternate, and each
figure is the median over --runs runs in ms per GiB of source.  The bytes each call moved across PCIe (H2D, D2H) are counted
from the calls' rules and the sizes they returned.  The decoded bytes must equal the source in every run.  Prints one JSON
line with the GPU's name, power limit and SM clocks.

    python scripts/host_packed_bench.py --runs 5
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GIB = 1 << 30
BLOCK = 32768
SLOT_CHUNK_BLOCKS = 2048                    # FSEB200_HOST_CHUNK_BLOCKS default
PACKED_CHUNK_BYTES = 64 << 20               # FSEB200_HOST_PACKED_CHUNK_BYTES default
BLOCK_OVERHEAD = 512


def gpu_info():
    import torch
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.check_output(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm,clocks.sm",
                                     "--format=csv,noheader"], text=True).strip()
        info["power_limit"], info["sm_clock_max"], info["sm_clock"] = [x.strip() for x in q.split(",")]
    except (OSError, subprocess.CalledProcessError) as e:
        info["nvidia_smi"] = repr(e)
    return info


def ragged_sizes(total, seed=7):
    import numpy as np
    rng = np.random.default_rng(seed)
    sizes = rng.integers(1024, 128 * 1024 + 1, total // 1024)
    ends = np.cumsum(sizes)
    k = int(np.searchsorted(ends, total))
    sizes = sizes[: k + 1].copy()
    sizes[-1] -= int(ends[k] - total)
    if sizes[-1] < 1024:
        sizes[-2] += sizes[-1]
        sizes = sizes[:-1]
    return sizes.astype(np.uint64)


def slot_bytes(cs, slot, total, n):
    """(H2D, D2H) of the slot compress and the slot decompress: the source up, the used width of each chunk's slots down (and
    back up, +16 bytes), the sizes and results"""
    import numpy as np
    h2d_c, d2h_c, h2d_d, d2h_d = total, 8 * n, 8 * n, total + 8 * n
    ok = cs < np.uint64(2 ** 64 - 9)
    for b0 in range(0, n, SLOT_CHUNK_BLOCKS):
        c = cs[b0: b0 + SLOT_CHUNK_BLOCKS]
        m = int(c[ok[b0: b0 + SLOT_CHUNK_BLOCKS]].max(initial=0))
        d2h_c += min((m + 63) & ~63, slot) * len(c)
        h2d_d += min((m + 16 + 63) & ~63, slot) * len(c)
    return (h2d_c, d2h_c), (h2d_d, d2h_d)


def packed_bytes(sizes, offsets):
    """(H2D, D2H) of the packed compress and decompress: the source and two words per block up, the stored bytes and the
    offsets and values down; the packed bytes and three words per block (+1 per chunk) up, the blocks and results down"""
    n, total, stored = len(sizes), int(sizes.sum()), int(offsets[-1])
    chunks, w = 1, 0
    for s in sizes.tolist():
        if w and w + s + BLOCK_OVERHEAD > PACKED_CHUNK_BYTES:
            chunks, w = chunks + 1, 0
        w += s + BLOCK_OVERHEAD
    dchunks, w = 1, 0
    for s, L in zip(sizes.tolist(), (offsets[1:] - offsets[:-1]).tolist()):       # the decompress weighs stored bytes too
        if w and w + s + L + BLOCK_OVERHEAD > PACKED_CHUNK_BYTES:
            dchunks, w = dchunks + 1, 0
        w += s + L + BLOCK_OVERHEAD
    return (total + 16 * n, stored + 16 * n + 8 * chunks), (stored + 24 * n + 8 * dchunks, total + 8 * n)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--gib", type=float, default=1.0)
    args = ap.parse_args()
    import numpy as np
    import torch
    import finitestateentropy_b200 as fb
    torch.cuda.set_device(0)
    L = fb.lib()
    total = int(args.gib * GIB) // BLOCK * BLOCK
    slot = fb.compress_bound(BLOCK)

    def pinned(n, dtype=torch.uint8):
        return torch.empty(max(n, 1), dtype=dtype).pin_memory()

    def source(kind):
        d = torch.empty(total, dtype=torch.uint8, device="cuda")
        if kind == "random":
            g = torch.Generator(device="cuda"); g.manual_seed(11)
            d = torch.randint(0, 256, (total,), dtype=torch.uint8, device="cuda", generator=g)
        else:
            assert L.FSEB200_probagen(d.data_ptr(), total, 0, {"p14": 0.14, "p80": 0.80}[kind], torch.cuda.current_stream().cuda_stream) == 0
        h = pinned(total)
        h[:total].copy_(d)
        torch.cuda.synchronize()
        return h

    cases = [("p14_huf", "p14", 1, False), ("ragged_huf", "p14", 1, True), ("p80_fse", "p80", 0, False),
             ("ragged_fse", "p80", 0, True), ("random_huf", "random", 1, False)]
    res = {"info": gpu_info(), "gib": total / GIB, "runs": args.runs, "cases": {}}
    src, src_kind = None, None
    for name, kind, codec, ragged in cases:
        if kind != src_kind:
            src = None                                                   # one source GiB pinned at a time
            src, src_kind = source(kind), kind
        sizes = ragged_sizes(total) if ragged else np.full(total // BLOCK, BLOCK, np.uint64)
        n = len(sizes)
        hsizes = torch.from_numpy(sizes.view(np.int64).copy())
        out, offs, cs = pinned(total + 32), torch.empty(n + 1, dtype=torch.int64), torch.empty(n, dtype=torch.int64)
        dst, results = pinned(total), torch.empty(n, dtype=torch.int64)
        if not ragged:
            cbuf, scs, sres = pinned(n * slot), torch.empty(n, dtype=torch.int64), torch.empty(n, dtype=torch.int64)

        def slot_pair():
            t0 = time.perf_counter()
            assert L.FSEB200_compress_host(codec, cbuf.data_ptr(), slot, scs.data_ptr(), src.data_ptr(), total, BLOCK, 255, 12) == 0
            t1 = time.perf_counter()
            assert L.FSEB200_decompress_host(codec, dst.data_ptr(), total, BLOCK, cbuf.data_ptr(), slot, scs.data_ptr(),
                                             sres.data_ptr(), src.data_ptr()) == 0
            t2 = time.perf_counter()
            assert torch.equal(dst[:total], src[:total]), (name, "slot")
            return t1 - t0, t2 - t1

        def packed_pair():
            t0 = time.perf_counter()
            assert L.FSEB200_compress_host_packed(codec, out.data_ptr(), out.numel(), offs.data_ptr(), cs.data_ptr(), src.data_ptr(),
                                                  hsizes.data_ptr(), n, 255, 12) == 0
            t1 = time.perf_counter()
            assert L.FSEB200_decompress_host_packed(codec, dst.data_ptr(), hsizes.data_ptr(), results.data_ptr(), out.data_ptr(),
                                                    offs.data_ptr(), n) == 0
            t2 = time.perf_counter()
            assert torch.equal(dst[:total], src[:total]) and torch.equal(results, hsizes), (name, "packed")
            return t1 - t0, t2 - t1

        pairs = ([("slot", slot_pair)] if not ragged else []) + [("packed", packed_pair)]
        for _, f in pairs:
            f()                                                          # warm-up: allocations, modules
        times = {k: ([], []) for k, _ in pairs}
        for _ in range(args.runs):
            for k, f in pairs:
                dst.fill_(0)
                c, d = f()
                times[k][0].append(c); times[k][1].append(d)
        per_gib = GIB / total * 1e3
        row = {"blocks": n}
        for k, (c, d) in times.items():
            row[k + "_compress_ms"] = round(statistics.median(c) * per_gib, 3)
            row[k + "_decompress_ms"] = round(statistics.median(d) * per_gib, 3)
            row[k + "_compress_range"] = [round(min(c) * per_gib, 3), round(max(c) * per_gib, 3)]
            row[k + "_decompress_range"] = [round(min(d) * per_gib, 3), round(max(d) * per_gib, 3)]
        offsets = offs.numpy().view(np.uint64)
        (pc_h2d, pc_d2h), (pd_h2d, pd_d2h) = packed_bytes(sizes, offsets)
        row["packed_bytes"] = {"compress_h2d": pc_h2d, "compress_d2h": pc_d2h, "decompress_h2d": pd_h2d, "decompress_d2h": pd_d2h}
        row["packed_stream_bytes"] = int(offsets[-1])
        if not ragged:
            (sc_h2d, sc_d2h), (sd_h2d, sd_d2h) = slot_bytes(scs.numpy().view(np.uint64), slot, total, n)
            row["slot_bytes"] = {"compress_h2d": sc_h2d, "compress_d2h": sc_d2h, "decompress_h2d": sd_h2d, "decompress_d2h": sd_d2h}
            assert np.array_equal(scs.numpy(), cs.numpy()), name                # both forms give the reference's values
        res["cases"][name] = row
        print(name, json.dumps(row), file=sys.stderr, flush=True)
        del out, dst
        if not ragged:
            del cbuf
    print(json.dumps(res))


if __name__ == "__main__":
    main()
