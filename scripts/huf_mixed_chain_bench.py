"""Mixed-form Huff0 chains (FSEB200_HUF_compress_mixed_repeat_chains_packed / FSEB200_HUF_decompress_mixed_repeat_packed) on one
GPU, in ms per GiB of source bytes, median and range over alternated runs.

uniform  1 GiB of probagen P14 as 32 chains x 1,024 blocks of 32 KB, every chain starting with no table, prefer 0.  The mixed
         calls with every flag 0 against the 4X packed chain calls, and with every flag 1 against the 1X ones (compress and
         decode).  The results must be the same; the check runs once per case.
ragged   about 1 GiB of a literal-like stream: 32 chains of 32 KB P14 blocks with 1-4 sections of 1-1,024 bytes between them, each
         section 1X when it is shorter than 256 bytes (zstd's rule) and every 32 KB block 4X, prefer on every other block.  One
         mixed call against today's workaround: the 4X / 1X packed chain calls, one per run of same-form blocks (the chains' k-th
         runs of one form share a call), with the chains' state carried from call to call, and the same for the decode.  Every
         block of both is checked against its source once.
Prints one JSON line: the GPU's name and power limit read in the same run, and per case the median and range."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import finitestateentropy_b200 as fb  # noqa: E402

GIB = 1 << 30
BLOCK = 32768
CHAINS = 32


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


def p14(n, seed):
    L = fb.lib()
    src = torch.empty(n, dtype=torch.uint8, device="cuda")
    assert L.FSEB200_probagen(src.data_ptr(), n, seed, 0.14, torch.cuda.current_stream().cuda_stream) == 0
    return src


class Stream:
    """blocks (sizes, flags) of CHAINS equal chains laid out back to back in one source buffer, and the chains' state"""

    def __init__(self, sizes, flags, prefer):
        self.nb = len(sizes)
        n = int(sum(sizes))
        self.src = p14(n, 1)
        self.n = n
        sz = np.asarray(sizes, np.int64)
        st = np.concatenate([[0], np.cumsum(sz)])
        self.sizes_h, self.flags_h = sz, np.asarray(flags, np.uint8)
        self.sp = torch.from_numpy(st[:-1]).cuda() + self.src.data_ptr()
        self.ss = torch.from_numpy(sz).cuda()
        self.pr = torch.from_numpy(np.asarray(prefer, np.int32)).cuda()
        self.sg = torch.from_numpy(self.flags_h).cuda()
        per = self.nb // CHAINS
        self.starts_h = np.array([c * per for c in range(CHAINS)] + [self.nb], np.int64)
        self.starts = torch.from_numpy(self.starts_h).cuda()
        self.tabs = torch.zeros(CHAINS * 256, dtype=torch.int32, device="cuda")
        self.tp = torch.arange(CHAINS, dtype=torch.int64, device="cuda") * 1024 + self.tabs.data_ptr()
        self.rep = torch.zeros(CHAINS, dtype=torch.int32, device="cuda")
        self.chp = torch.zeros(CHAINS, dtype=torch.int64, device="cuda")
        self.chs = torch.zeros(CHAINS, dtype=torch.int64, device="cuda")
        self.zp = torch.zeros(CHAINS, dtype=torch.int64, device="cuda")
        self.out = torch.empty(n + 32, dtype=torch.uint8, device="cuda")
        self.out_runs = None                                                # the workaround's buffer (plan_runs)
        self.off = torch.empty(self.nb + 1, dtype=torch.int64, device="cuda")
        self.cs = torch.empty(self.nb, dtype=torch.int64, device="cuda")
        self.kinds = torch.empty(self.nb, dtype=torch.uint8, device="cuda")
        self.back = torch.empty(n, dtype=torch.uint8, device="cuda")
        self.bp = torch.from_numpy(st[:-1]).cuda() + self.back.data_ptr()
        self.res = torch.empty(self.nb, dtype=torch.int64, device="cuda")

    def reset(self):
        self.tabs.zero_(); self.rep.zero_(); self.chp.zero_(); self.chs.zero_()

    def mixed(self):
        self.reset()
        return timed(lambda: fb.huf_compress_mixed_repeat_chains_packed(
            self.starts, self.sp, self.ss, self.pr, self.sg, self.tp, self.rep, self.chp, self.chs, out=self.out,
            offsets=self.off, csizes=self.cs, kinds=self.kinds, max_symbol_value=255, table_log=11))

    def mixed_decode(self):
        return timed(lambda: fb.huf_decompress_mixed_repeat_packed(self.starts, self.out, self.off, self.kinds, self.sg,
                                                                   self.zp, self.zp, self.bp, self.ss, results=self.res))

    def uniform(self, four):
        self.reset()
        fn = fb.huf_compress_repeat_chains_packed if four else fb.huf_compress1x_repeat_chains_packed
        return timed(lambda: fn(self.starts, self.sp, self.ss, self.pr, self.tp, self.rep, self.chp, self.chs, out=self.out,
                                offsets=self.off, csizes=self.cs, kinds=self.kinds, max_symbol_value=255, table_log=11))

    def uniform_decode(self, four):
        fn = fb.huf_decompress_repeat_packed if four else fb.huf_decompress1x_repeat_packed
        return timed(lambda: fn(self.starts, self.out, self.off, self.kinds, self.zp, self.zp, self.bp, self.ss,
                                results=self.res))

    # ---- today's workaround: one 4X / 1X call per run of same-form blocks ----
    def plan_runs(self):
        """calls: (four, block indices, chain starts of the call, out slice start, slice length); runs of chain c in order"""
        runs = []
        for c in range(CHAINS):
            b0, b1 = int(self.starts_h[c]), int(self.starts_h[c + 1])
            f = self.flags_h[b0:b1] != 0
            cut = np.nonzero(np.diff(f.astype(np.int8)))[0] + 1
            edges = np.concatenate([[0], cut, [b1 - b0]])
            runs.append([(bool(not f[edges[i]]), b0 + edges[i], b0 + edges[i + 1]) for i in range(len(edges) - 1)])
        calls, pos = [], 0
        for k in range(max(len(r) for r in runs)):
            for four in (True, False):
                idx, st = [], [0]
                for c in range(CHAINS):
                    if k < len(runs[c]) and runs[c][k][0] == four:
                        idx += range(runs[c][k][1], runs[c][k][2])
                    st.append(len(idx))
                if not idx:
                    continue
                ln = int(self.sizes_h[idx].sum()) + 32
                ix = torch.tensor(idx, dtype=torch.int64, device="cuda")
                calls.append(dict(four=four, ix=ix, st=torch.tensor(st, dtype=torch.int64, device="cuda"), o=pos, ln=ln,
                                  off=torch.empty(len(idx) + 1, dtype=torch.int64, device="cuda"),
                                  sp=self.sp[ix], ss=self.ss[ix], pr=self.pr[ix], bp=self.bp[ix],
                                  cs=torch.empty(len(idx), dtype=torch.int64, device="cuda"),
                                  kinds=torch.empty(len(idx), dtype=torch.uint8, device="cuda"),
                                  res=torch.empty(len(idx), dtype=torch.int64, device="cuda")))
                pos += ln
        self.out_runs = torch.empty(pos, dtype=torch.uint8, device="cuda")
        self.calls = calls
        # the entry headers of each call, for the decode: the chains' headers before it (recorded once, untimed)
        self.reset()
        for cl in calls:
            cl["chp"], cl["chs"] = self.chp.clone(), self.chs.clone()
            self._run_one(cl)
        torch.cuda.synchronize()

    def _run_one(self, cl):
        fn = fb.huf_compress_repeat_chains_packed if cl["four"] else fb.huf_compress1x_repeat_chains_packed
        fn(cl["st"], cl["sp"], cl["ss"], cl["pr"], self.tp, self.rep, self.chp, self.chs, out=self.out_runs[cl["o"]:cl["o"] + cl["ln"]],
           offsets=cl["off"], csizes=cl["cs"], kinds=cl["kinds"], max_symbol_value=255, table_log=11)

    def runs_compress(self):
        self.reset()

        def go():
            for cl in self.calls:
                self._run_one(cl)
        return timed(go)

    def runs_decode(self):
        def go():
            for cl in self.calls:
                fn = fb.huf_decompress_repeat_packed if cl["four"] else fb.huf_decompress1x_repeat_packed
                fn(cl["st"], self.out_runs[cl["o"]:cl["o"] + cl["ln"]], cl["off"], cl["kinds"], cl["chp"], cl["chs"], cl["bp"], cl["ss"],
                   results=cl["res"])
        return timed(go)


def ragged_sizes(total, seed=7):
    rng = np.random.default_rng(seed)
    sizes, flags, prefer = [], [], []
    while sum(sizes) < total:
        sizes.append(BLOCK); flags.append(0); prefer.append(len(sizes) % 2)
        for _ in range(int(rng.integers(1, 5))):
            n = int(rng.integers(1, 1025))
            sizes.append(n); flags.append(int(n < 256)); prefer.append(len(sizes) % 2)
    keep = len(sizes) // CHAINS * CHAINS
    return sizes[:keep], flags[:keep], prefer[:keep]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--gib", type=float, default=1.0)
    args = ap.parse_args()
    results = {}

    def add(key, ms, nbytes):
        results.setdefault(key, []).append(ms * GIB / nbytes)

    nb = int(args.gib * GIB) // BLOCK // CHAINS * CHAINS
    uni = Stream([BLOCK] * nb, [0] * nb, [0] * nb)
    for four in (True, False):                                              # warm-up and checks
        uni.sg.fill_(0 if four else 1)
        uni.mixed(); a = (uni.off.clone(), uni.cs.clone(), uni.kinds.clone(), uni.out[:uni.n].clone())
        uni.uniform(four)
        assert torch.equal(a[0], uni.off) and torch.equal(a[1], uni.cs) and torch.equal(a[2], uni.kinds)
        assert torch.equal(a[3], uni.out[:uni.n])
        uni.back.zero_(); uni.mixed_decode()
        assert torch.equal(uni.res, uni.ss) and torch.equal(uni.back, uni.src)
        uni.uniform_decode(four)
    sizes, flags, prefer = ragged_sizes(int(args.gib * GIB))
    rag = Stream(sizes, flags, prefer)
    rag.plan_runs()
    rag.back.zero_(); rag.runs_decode()
    runs_back = rag.back.clone()
    rag.mixed()
    assert bool((rag.cs >= 0).all())                                        # no error codes (they are negative as int64)
    assert torch.equal(torch.cat([c["cs"] for c in rag.calls]), rag.cs[torch.cat([c["ix"] for c in rag.calls])])
    rag.back.zero_(); rag.mixed_decode()
    assert torch.equal(rag.res, rag.ss)
    byte_start = torch.from_numpy(np.concatenate([[0], np.cumsum(rag.sizes_h)])[:-1]).cuda()
    for back in (rag.back, runs_back):                                      # every block regenerates, but a 1X block coded into
        bad = (back != rag.src).nonzero().flatten()                         # one byte, which the decoders read as RLE
        blk = torch.searchsorted(byte_start, bad, right=True) - 1
        assert bool((rag.cs[blk] == 1).all() & (rag.sg[blk] != 0).all())
    torch.cuda.synchronize()
    for _ in range(args.runs):
        for four, tag in ((True, "all0_vs_4X"), (False, "all1_vs_1X")):
            uni.sg.fill_(0 if four else 1)
            add("uniform_compress_mixed_" + tag, uni.mixed(), uni.n)
            add("uniform_compress_existing_" + tag, uni.uniform(four), uni.n)
            add("uniform_decode_mixed_" + tag, uni.mixed_decode(), uni.n)
            add("uniform_decode_existing_" + tag, uni.uniform_decode(four), uni.n)
        add("ragged_compress_mixed", rag.mixed(), rag.n)
        add("ragged_compress_runs", rag.runs_compress(), rag.n)
        add("ragged_decode_mixed", rag.mixed_decode(), rag.n)
        add("ragged_decode_runs", rag.runs_decode(), rag.n)
    summary = {k: {"median": round(sorted(v)[len(v) // 2], 3), "min": round(min(v), 3), "max": round(max(v), 3)} for k, v in results.items()}
    print(json.dumps({"gpu": gpu_info(), "uniform": {"bytes": uni.n, "chains": CHAINS, "blocks": uni.nb},
                      "ragged": {"bytes": rag.n, "chains": CHAINS, "blocks": rag.nb, "workaround_calls": len(rag.calls),
                                 "blocks_1x": int(np.count_nonzero(rag.flags_h))},
                      "runs": args.runs, "ms_per_gib": summary}))


if __name__ == "__main__":
    main()
