"""Huff0 chains of table reuse (FSEB200_HUF_compress4X_repeat_chains) against what a caller does without them, on one GPU.

1 GiB of probagen P14 in 32 KB blocks, cut into chains of equal length: 32,768 chains x 1 block, 1,024 x 32, 32 x 1,024 and
1 x 32,768.  Every chain starts with no table (flag none) and prefer 0, so each block builds a tree, checks the previous table and
compares the estimates.  Baselines, alternated with the chain call run by run:
  blocks   (1-block shape) FSEB200_HUF_compress4X_repeat_blocks over the same blocks, one block per stream;
  loop     (longer shapes) one FSEB200_HUF_compress4X_repeat_blocks call per step of the chains, with the per-stream flag and
           header bookkeeping between steps done by torch ops on the device (INTEGRATION.md B before the chain call existed).
Every shape is warmed up, and the chain call's values are checked against the loop's once per shape.  A separate profiled pass
gives the kernels' own device time per call (plan, the chains' decisions, emit).
Prints one JSON line: the GPU's name and power limit, and per case the median and range in ms per GiB of source bytes."""
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
    scale = GIB / n
    results, kernels = {}, {}

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
            # per step s, the blocks c * per + s of every chain c (contiguous, as the per-block call takes them)
            self.steps = [tuple(t.view(nch, per)[:, s].contiguous() for t in (sp, ss, dp, dc, pr)) for s in range(per)] if per > 1 else None
            self.cs_steps = [torch.empty(nch, dtype=torch.int64, device="cuda") for _ in range(per)] if per > 1 else None

        def reset(self):
            tabs.zero_(); self.rep.zero_(); self.chp.zero_(); self.chs.zero_()

        def chain(self):
            self.reset()
            return timed(lambda: fb.huf_compress_repeat_chains(self.starts, sp, ss, dp, dc, pr, self.tp, self.rep, self.chp, self.chs,
                                                               csizes=cs, hdr_ptrs=hp, hdr_sizes=hs, max_symbol_value=255, table_log=11))

        def baseline(self):
            self.reset()
            if self.per == 1:
                return timed(lambda: fb.huf_compress_repeat_blocks(sp, ss, dp, dc, self.tp, self.rep, pr, csizes=cs,
                                                                   max_symbol_value=255, table_log=11))

            def loop():
                H, HS = self.chp, self.chs
                for s, (a, b_, c_, d_, p_) in enumerate(self.steps):
                    r = fb.huf_compress_repeat_blocks(a, b_, c_, d_, self.tp, self.rep, p_, csizes=self.cs_steps[s],
                                                      max_symbol_value=255, table_log=11)
                    fresh = (r >= 2) & (self.rep == 0)                      # carries a new table: its header, flag check
                    H = torch.where(fresh, c_, H)
                    HS = torch.where(fresh, r, HS)
                    self.rep.masked_fill_(fresh, 1)
                self.chp.copy_(H); self.chs.copy_(HS)
            return timed(loop)

    shapes = [Shape(c, p) for c, p in SHAPES if c * p == nb]
    for sh in shapes:                                                     # warm-up, and the chain call equals the loop
        sh.chain()
        got = cs.clone()
        sh.baseline()
        want = cs if sh.per == 1 else torch.stack(sh.cs_steps, 1).reshape(-1)
        assert torch.equal(got, want), (sh.nch, sh.per)
    torch.cuda.synchronize()
    for _ in range(args.runs):
        for sh in shapes:
            tag = "%dx%d" % (sh.nch, sh.per)
            add("chains_" + tag, sh.chain())
            add(("blocks_" if sh.per == 1 else "loop_") + tag, sh.baseline())
    from torch.profiler import profile, ProfilerActivity
    for sh in shapes:                                                     # kernel device time of one chain call
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            sh.chain()
            torch.cuda.synchronize()
        per = {}
        for ev in prof.key_averages():
            for k in ("huf_plan_kernel", "huf_chain_check_kernel", "huf_chain_kernel", "huf_emit_kernel"):
                if k in ev.key:
                    per[k] = per.get(k, 0.0) + ev.device_time_total / 1000.0 * scale
        kernels["%dx%d" % (sh.nch, sh.per)] = {k: round(v, 3) for k, v in per.items()}
    summary = {k: {"median": round(sorted(v)[len(v) // 2], 2), "min": round(min(v), 2), "max": round(max(v), 2)} for k, v in results.items()}
    print(json.dumps({"gpu": gpu_info(), "bytes": n, "block": BLOCK, "runs": args.runs, "ms_per_gib": summary,
                      "kernel_ms_per_gib": kernels}))


if __name__ == "__main__":
    main()
