"""Huff0 table reuse (FSEB200_HUF_{compress,decompress}4X_repeat_blocks) against the descriptor calls without it
(FSEB200_HUF_{compress,decompress}_blocks), on one GPU, in one process.

1 GiB of probagen P14 in 32 KB blocks, one block per stream (every block its own table and flag).  Cases, each alternated with
the plain descriptor call of the same blocks, run by run:
  none      every flag none: the plain path plus the flag and table loads, and every table saved;
  check     flag check, prefer 0, a table built from the same distribution: validation and the estimate comparison;
  valid     flag valid, prefer 1: no tree is built, no header is written;
  mix       none / check / valid by block, prefer by block;
  dec_own   decode of blocks with their own headers (the `none` output) against FSEB200_HUF_decompress_blocks;
  dec_ext   decode of header-less blocks (the `valid` output) with external headers.
Prints one JSON line: the GPU's name and power limit, and per case the median and range in ms per GiB of source bytes."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import finitestateentropy_b200 as fb  # noqa: E402

GIB = 1 << 30
BLOCK = 32768


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--gib", type=float, default=1.0)
    args = ap.parse_args()
    from helpers import load_ref
    from huf_repeat_cases import ref_table, table_header
    import numpy as np
    n = int(args.gib * GIB) // BLOCK * BLOCK
    nb = n // BLOCK
    L = fb.lib()
    src = torch.empty(n, dtype=torch.uint8, device="cuda")
    assert L.FSEB200_probagen(src.data_ptr(), n, 0, 0.14, torch.cuda.current_stream().cuda_stream) == 0
    sample = src[:65536].cpu().numpy()
    ref = load_ref()
    if ref is None:
        raise SystemExit("the compiled reference (oracle/_ref) builds the check table and its header")
    table = ref_table(ref, sample)
    hdr = table_header(ref, table)
    cap = fb.compress_bound(BLOCK)
    ar = torch.arange(nb, dtype=torch.int64, device="cuda")
    sp, ss = ar * BLOCK + src.data_ptr(), torch.full((nb,), BLOCK, dtype=torch.int64, device="cuda")
    dst = torch.empty(nb * cap, dtype=torch.uint8, device="cuda")
    dp, dc = ar * cap + dst.data_ptr(), torch.full((nb,), cap, dtype=torch.int64, device="cuda")
    tabs_init = torch.from_numpy(np.tile(table, nb).view(np.int32)).cuda()
    tabs = tabs_init.clone()
    tp = ar * 1024 + tabs.data_ptr()
    cs = torch.empty(nb, dtype=torch.int64, device="cuda")
    flags = torch.empty(nb, dtype=torch.int32, device="cuda")
    setups = {"none": (0, 0), "check": (1, 0), "valid": (2, 1)}

    def compress_case(name):
        if name == "mix":
            f0 = (ar % 3).to(torch.int32)
            p0 = ((ar // 3) % 2).to(torch.int32)
        else:
            f, p = setups[name]
            f0 = torch.full((nb,), f, dtype=torch.int32, device="cuda")
            p0 = torch.full((nb,), p, dtype=torch.int32, device="cuda")
        tabs.copy_(tabs_init); flags.copy_(f0)
        return timed(lambda: fb.huf_compress_repeat_blocks(sp, ss, dp, dc, tp, flags, p0, csizes=cs, max_symbol_value=255, table_log=11))

    def plain():
        return timed(lambda: fb.huf_compress_blocks(sp, ss, dp, dc, csizes=cs, max_symbol_value=255, table_log=11))

    out = torch.empty(n, dtype=torch.uint8, device="cuda")
    op = ar * BLOCK + out.data_ptr()
    res = torch.empty(nb, dtype=torch.int64, device="cuda")
    hdr_dev = torch.from_numpy(np.concatenate([hdr, np.zeros(64, np.uint8)])).cuda()
    zeros = torch.zeros(nb, dtype=torch.int64, device="cuda")
    results = {}
    scale = GIB / n

    def add(key, ms):
        results.setdefault(key, []).append(ms * scale)

    hp = torch.full((nb,), hdr_dev.data_ptr(), dtype=torch.int64, device="cuda")
    hs = torch.full((nb,), len(hdr), dtype=torch.int64, device="cuda")
    for name in ("none", "check", "valid", "mix"):                         # warm-up of every shape, both decoders included
        compress_case(name)
    plain()
    compress_case("none")
    fb.huf_decompress_blocks(dp, cs, op, ss, results=res)
    fb.huf_decompress_repeat_blocks(dp, cs, op, ss, zeros, zeros, results=res)
    compress_case("valid")
    fb.huf_decompress_repeat_blocks(dp, cs, op, ss, hp, hs, results=res)
    torch.cuda.synchronize()
    for _ in range(args.runs):
        for name in ("none", "check", "valid", "mix"):
            add("plain_compress_blocks", plain())
            add("repeat_" + name, compress_case(name))
        compress_case("none")                                               # own headers everywhere
        own_c = cs.clone()
        add("plain_decompress_blocks", timed(lambda: fb.huf_decompress_blocks(dp, own_c, op, ss, results=res)))
        assert bool((res == BLOCK).all()) and torch.equal(out, src)
        add("repeat_dec_own", timed(lambda: fb.huf_decompress_repeat_blocks(dp, own_c, op, ss, zeros, zeros, results=res)))
        assert bool((res == BLOCK).all()) and torch.equal(out, src)
        compress_case("valid")                                              # header-less everywhere
        ext_c = cs.clone()
        add("repeat_dec_ext", timed(lambda: fb.huf_decompress_repeat_blocks(dp, ext_c, op, ss, hp, hs, results=res)))
        assert bool((res == BLOCK).all()) and torch.equal(out, src)
    summary = {k: {"median": round(sorted(v)[len(v) // 2], 2), "min": round(min(v), 2), "max": round(max(v), 2)} for k, v in results.items()}
    print(json.dumps({"gpu": gpu_info(), "bytes": n, "block": BLOCK, "runs": args.runs, "ms_per_gib": summary}))


if __name__ == "__main__":
    main()
