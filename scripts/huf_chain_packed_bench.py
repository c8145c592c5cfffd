"""Packed Huff0 chains (FSEB200_HUF_compress4X_repeat_chains_packed / FSEB200_HUF_decompress4X_repeat_packed) against the
pointer-based chain calls on the same inputs, on one GPU.

1 GiB of probagen P14 in 32 KB blocks, cut into chains of equal length: 32,768 chains x 1 block, 1,024 x 32, 32 x 1,024 and
1 x 32,768.  Every chain starts with no table (flag none) and prefer 0.  Alternated run by run:
  compress  packed chain call against FSEB200_HUF_compress4X_repeat_chains (slots of HUF_compressBound);
  decode    packed decode (offsets + kinds) against FSEB200_HUF_decompress4X_repeat_blocks on the header arrays the chain call
            reported, over the blocks coded with a table (the packed decode also regenerates the raw and RLE ones).
Every shape is warmed up; the packed call's values are checked against the chain call's, and both decoders' output against the
source, once per shape.  Prints one JSON line: the GPU's name and power limit, and per case the median and range in ms per GiB of
source bytes."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import finitestateentropy_b200 as fb  # noqa: E402

GIB = 1 << 30
BLOCK = 32768
SHAPES = ((32768, 1), (1024, 32), (32, 1024), (1, 32768))                 # (chains, blocks per chain)


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
    n = int(args.gib * GIB) // BLOCK * BLOCK
    nb = n // BLOCK
    L = fb.lib()
    src = torch.empty(n, dtype=torch.uint8, device="cuda")
    assert L.FSEB200_probagen(src.data_ptr(), n, 0, 0.14, torch.cuda.current_stream().cuda_stream) == 0
    cap = fb.compress_bound(BLOCK)
    ar = torch.arange(nb, dtype=torch.int64, device="cuda")
    sp, ss = ar * BLOCK + src.data_ptr(), torch.full((nb,), BLOCK, dtype=torch.int64, device="cuda")
    dst = torch.empty(nb * cap, dtype=torch.uint8, device="cuda")
    dp, dc = ar * cap + dst.data_ptr(), torch.full((nb,), cap, dtype=torch.int64, device="cuda")
    pr = torch.zeros(nb, dtype=torch.int32, device="cuda")
    tabs = torch.zeros(nb * 256, dtype=torch.int32, device="cuda")
    cs, hp, hs = (torch.empty(nb, dtype=torch.int64, device="cuda") for _ in range(3))
    out = torch.empty(n + 32, dtype=torch.uint8, device="cuda")
    off = torch.empty(nb + 1, dtype=torch.int64, device="cuda")
    pcs = torch.empty(nb, dtype=torch.int64, device="cuda")
    kinds = torch.empty(nb, dtype=torch.uint8, device="cuda")
    back = torch.empty(n, dtype=torch.uint8, device="cuda")
    bp = ar * BLOCK + back.data_ptr()
    res = torch.empty(nb, dtype=torch.int64, device="cuda")
    scale = GIB / n
    results = {}

    def add(key, ms):
        results.setdefault(key, []).append(ms * scale)

    class Shape:
        def __init__(self, nch, per):
            self.nch, self.per = nch, per
            self.starts = torch.arange(0, nch + 1, dtype=torch.int64, device="cuda") * per
            self.tp = torch.arange(nch, dtype=torch.int64, device="cuda") * 1024 + tabs.data_ptr()
            self.rep = torch.zeros(nch, dtype=torch.int32, device="cuda")
            self.chp = torch.zeros(nch, dtype=torch.int64, device="cuda")
            self.chs = torch.zeros(nch, dtype=torch.int64, device="cuda")
            self.zp = torch.zeros(nch, dtype=torch.int64, device="cuda")   # entry headers of the decode: none

        def reset(self):
            tabs.zero_(); self.rep.zero_(); self.chp.zero_(); self.chs.zero_()

        def chain(self):
            self.reset()
            return timed(lambda: fb.huf_compress_repeat_chains(self.starts, sp, ss, dp, dc, pr, self.tp, self.rep, self.chp, self.chs,
                                                               csizes=cs, hdr_ptrs=hp, hdr_sizes=hs, max_symbol_value=255, table_log=11))

        def packed(self):
            self.reset()
            return timed(lambda: fb.huf_compress_repeat_chains_packed(self.starts, sp, ss, pr, self.tp, self.rep, self.chp, self.chs,
                                                                      out=out, offsets=off, csizes=pcs, kinds=kinds,
                                                                      max_symbol_value=255, table_log=11))

        def decode_blocks(self):                                        # the coded blocks (every block of these shapes)
            return timed(lambda: fb.huf_decompress_repeat_blocks(dp, cs, bp, ss, hp, hs, results=res))

        def decode_packed(self):
            return timed(lambda: fb.huf_decompress_repeat_packed(self.starts, out, off, kinds, self.zp, self.zp, bp, ss, results=res))

    shapes = [Shape(c, p) for c, p in SHAPES if c * p == nb]
    for sh in shapes:                                                     # warm-up and checks
        sh.chain(); sh.packed()
        assert torch.equal(cs, pcs), (sh.nch, sh.per)
        assert bool((cs >= 2).all()), "every block of P14 is coded"           # error codes are negative as int64
        back.zero_(); sh.decode_blocks()
        assert torch.equal(res, ss) and torch.equal(back, src)
        back.zero_(); sh.decode_packed()
        assert torch.equal(res, ss) and torch.equal(back, src)
    torch.cuda.synchronize()
    for _ in range(args.runs):
        for sh in shapes:
            tag = "%dx%d" % (sh.nch, sh.per)
            add("compress_packed_" + tag, sh.packed())
            add("compress_chains_" + tag, sh.chain())
            add("decode_packed_" + tag, sh.decode_packed())
            add("decode_blocks_" + tag, sh.decode_blocks())
    summary = {k: {"median": round(sorted(v)[len(v) // 2], 2), "min": round(min(v), 2), "max": round(max(v), 2)} for k, v in results.items()}
    print(json.dumps({"gpu": gpu_info(), "bytes": n, "block": BLOCK, "runs": args.runs, "ms_per_gib": summary}))


if __name__ == "__main__":
    main()
