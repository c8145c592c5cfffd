"""The packed Huff0 chain pair on host buffers (FSEB200_compress_host_repeat_chains_packed + FSEB200_decompress_host_repeat_packed)
against the packed host pair (FSEB200_compress_host_packed + FSEB200_decompress_host_packed, Huff0 4X) on the same pinned bytes,
on one GPU: 1 GiB of probagen P14 in 32 KB blocks, cut into 32,768 chains of 1 block, 1,024 of 32, 32 of 1,024 and 1 of 32,768.
Every chain enters with no table (flag none, header size 0); no block prefers the old table; (maxSymbolValue, tableLog) =
(255, 12).  The single-chain shape runs the serial decision stage of the device chain call (DESIGN 4.2) over every block, one
chunk after another, since each chunk's call waits for the previous chunk's state.

Every call is synchronous and timed with a host clock; within a run the two pairs alternate, and each figure is the median over
--runs runs in ms per GiB of source, with the range.  The decoded bytes must equal the source in every run.  Prints one JSON line
with the GPU's name, power limit and SM clocks.

    python scripts/host_chain_bench.py --runs 5
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
GIB = 1 << 30
BLOCK = 32768
SHAPES = (32768, 1024, 32, 1)                                       # chains per GiB


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    args = ap.parse_args()
    import numpy as np
    import torch
    import finitestateentropy_b200 as fb
    from host_packed_bench import gpu_info
    torch.cuda.set_device(0)
    L = fb.lib()
    total, n = GIB, GIB // BLOCK

    def pinned(k, dtype=torch.uint8):
        return torch.empty(k, dtype=dtype).pin_memory()

    d = torch.empty(total, dtype=torch.uint8, device="cuda")
    assert L.FSEB200_probagen(d.data_ptr(), total, 0, 0.14, torch.cuda.current_stream().cuda_stream) == 0
    src = pinned(total)
    src.copy_(d)
    torch.cuda.synchronize()
    del d
    sizes = torch.full((n,), BLOCK, dtype=torch.int64)
    prefer = torch.zeros(n, dtype=torch.int32)
    out, offs, cs, kinds = pinned(total + 32), torch.empty(n + 1, dtype=torch.int64), torch.empty(n, dtype=torch.int64), \
        torch.empty(n, dtype=torch.uint8)
    dst, results = pinned(total), torch.empty(n, dtype=torch.int64)

    def packed_pair():
        t0 = time.perf_counter()
        assert L.FSEB200_compress_host_packed(1, out.data_ptr(), out.numel(), offs.data_ptr(), cs.data_ptr(), src.data_ptr(),
                                              sizes.data_ptr(), n, 255, 12) == 0
        t1 = time.perf_counter()
        assert L.FSEB200_decompress_host_packed(1, dst.data_ptr(), sizes.data_ptr(), results.data_ptr(), out.data_ptr(),
                                                offs.data_ptr(), n) == 0
        t2 = time.perf_counter()
        assert torch.equal(dst, src) and torch.equal(results, sizes), "packed"
        return t1 - t0, t2 - t1

    res = {"info": gpu_info(), "gib": total / GIB, "runs": args.runs, "block": BLOCK, "shapes": {}}
    for n_chains in SHAPES:
        per = n // n_chains
        starts = torch.arange(0, n + 1, per, dtype=torch.int64)
        tables = torch.zeros((n_chains, 256), dtype=torch.int32)
        table_ptrs = torch.tensor([tables.data_ptr() + 1024 * c for c in range(n_chains)], dtype=torch.int64)
        flags = torch.zeros(n_chains, dtype=torch.int32)
        hdr, hdr_sizes = torch.zeros(n_chains, dtype=torch.int64), torch.zeros(n_chains, dtype=torch.int64)
        entry_hdr, entry_sizes = hdr.clone(), hdr_sizes.clone()

        def chain_pair():
            tables.zero_(); flags.zero_(); hdr.zero_(); hdr_sizes.zero_()            # every run from the same entry state
            t0 = time.perf_counter()
            assert L.FSEB200_compress_host_repeat_chains_packed(
                1, n_chains, starts.data_ptr(), n, out.data_ptr(), out.numel(), offs.data_ptr(), cs.data_ptr(), kinds.data_ptr(),
                src.data_ptr(), sizes.data_ptr(), prefer.data_ptr(), table_ptrs.data_ptr(), flags.data_ptr(), hdr.data_ptr(),
                hdr_sizes.data_ptr(), 255, 12) == 0
            t1 = time.perf_counter()
            assert L.FSEB200_decompress_host_repeat_packed(1, n_chains, starts.data_ptr(), n, dst.data_ptr(), sizes.data_ptr(),
                                                           results.data_ptr(), out.data_ptr(), offs.data_ptr(), kinds.data_ptr(),
                                                           entry_hdr.data_ptr(), entry_sizes.data_ptr()) == 0
            t2 = time.perf_counter()
            assert torch.equal(dst, src) and torch.equal(results, sizes), ("chains", n_chains)
            return t1 - t0, t2 - t1

        pairs = (("chains", chain_pair), ("packed", packed_pair))
        for _, f in pairs:
            f()                                                          # warm-up: allocations, modules
        times = {k: ([], []) for k, _ in pairs}
        for _ in range(args.runs):
            for k, f in pairs:
                dst.fill_(0)
                c, dd = f()
                times[k][0].append(c); times[k][1].append(dd)
        chain_pair()                                                     # the counts below are the chain call's
        per_gib = GIB / total * 1e3
        k = kinds.numpy()
        row = {"chains": n_chains, "blocks_per_chain": per, "stream_bytes": int(offs[-1]),
               "kinds": {str(x): int((k == x).sum()) for x in range(5) if (k == x).any()}}
        for name, (c, dd) in times.items():
            row[name + "_compress_ms"] = round(statistics.median(c) * per_gib, 3)
            row[name + "_decompress_ms"] = round(statistics.median(dd) * per_gib, 3)
            row[name + "_compress_range"] = [round(min(c) * per_gib, 3), round(max(c) * per_gib, 3)]
            row[name + "_decompress_range"] = [round(min(dd) * per_gib, 3), round(max(dd) * per_gib, 3)]
        res["shapes"][str(n_chains)] = row
        print(n_chains, json.dumps(row), file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
