"""Packed Huff0 chains under zstd's literal-coding policy (FSEB200_HUF_compress_literals_chains_packed) on one GPU, in ms per GiB of
source bytes, median and range over alternated runs.

The stream is about 1 GiB of a literal-like stream: 32 chains of 32 KB P14 blocks with 1-4 sections of 1-1,024 bytes between them,
prefer on every other block, every chain starting with no table; (minLiterals, minGainLog) = (64, 6), zstd's below btopt.
  policy   one FSEB200_HUF_compress_literals_chains_packed call.
  mixed    one FSEB200_HUF_compress_mixed_repeat_chains_packed call with zstd's size rule as the forms (1X below 256 bytes): the
           same coding work without the policy, so the difference is what the policy costs.
  loop     what a caller without the policy call has to write: per step (the k-th block of every chain), the 4X and the 1X
           *_repeat_blocks call on copies of the chains' state, and torch ops for the form, the thresholds, the kind and the
           rollback -- on the first SLICE_STEPS steps of every chain, scaled to ms per GiB of that slice.
The policy call's values and kinds are checked once against the loop's on the slice, and its stream is decoded once through
FSEB200_HUF_decompress_mixed_repeat_packed with the forms it wrote.
Prints one JSON line: the GPU's name and power limit read in the same run, and per case the median and range."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import finitestateentropy_b200 as fb  # noqa: E402
from huf_mixed_chain_bench import GIB, CHAINS, Stream, ragged_sizes, timed, gpu_info  # noqa: E402

MIN_LIT, MIN_GAIN_LOG = 64, 6
SLICE_STEPS = 128


class Policy(Stream):
    def __init__(self, sizes, prefer):
        super().__init__(sizes, [int(n < 256) for n in sizes], prefer)
        self.forms = torch.empty(self.nb, dtype=torch.uint8, device="cuda")

    def policy(self):
        self.reset()
        return timed(lambda: fb.huf_compress_literals_chains_packed(
            self.starts, self.sp, self.ss, self.pr, self.tp, self.rep, self.chp, self.chs, out=self.out, offsets=self.off,
            csizes=self.cs, kinds=self.kinds, single_stream=self.forms, max_symbol_value=255, table_log=11,
            min_literals=MIN_LIT, min_gain_log=MIN_GAIN_LOG))

    def policy_decode(self):
        return timed(lambda: fb.huf_decompress_mixed_repeat_packed(self.starts, self.out, self.off, self.kinds, self.forms,
                                                                   self.zp, self.zp, self.bp, self.ss, results=self.res))

    def prepare_loop(self, steps):
        """per step k < steps: the k-th block of every chain, and both forms' destinations and state copies"""
        per = self.nb // CHAINS
        self.steps = min(steps, per)
        self.step_ix = [torch.tensor([c * per + k for c in range(CHAINS)], dtype=torch.int64, device="cuda") for k in range(self.steps)]
        self.loop_bytes = int(sum(int(self.ss[ix].sum()) for ix in self.step_ix))
        caps = 129 + self.ss + (self.ss >> 8) + 8
        self.dst = [torch.empty(int(caps.sum()) + 64, dtype=torch.uint8, device="cuda") for _ in range(2)]
        self.dp = [(torch.cumsum(caps, 0) - caps) + d.data_ptr() for d in self.dst]
        self.caps = caps
        self.ltabs = [torch.zeros(CHAINS * 256, dtype=torch.int32, device="cuda") for _ in range(3)]   # state, 4X copy, 1X copy
        self.ltp = [torch.arange(CHAINS, dtype=torch.int64, device="cuda") * 1024 + t.data_ptr() for t in self.ltabs]
        self.lcs = [torch.empty(self.nb, dtype=torch.int64, device="cuda") for _ in range(2)]
        src = self.src.cpu().numpy()
        st = np.concatenate([[0], np.cumsum(self.sizes_h)])
        equal = [bool(n and (src[a:a + n] == src[a]).all()) if n < 8 else False for a, n in zip(st[:-1], self.sizes_h)]
        self.equal = torch.tensor(equal, dtype=torch.bool, device="cuda")         # the all-equal test on blocks below 8 bytes
        self.lval = torch.empty(self.nb, dtype=torch.int64, device="cuda")
        self.lkind = torch.empty(self.nb, dtype=torch.uint8, device="cuda")

    def loop(self):
        T = self.ltabs[0].view(CHAINS, 256)
        F = torch.zeros(CHAINS, dtype=torch.int32, device="cuda")

        def go():
            T.zero_(); F.zero_()
            for ix in self.step_ix:
                n, pr = self.ss[ix], self.pr[ix]
                reps = []
                for j, fn in enumerate((fb.huf_compress_repeat_blocks, fb.huf_compress1x_repeat_blocks)):
                    self.ltabs[1 + j].copy_(self.ltabs[0])
                    r = F.clone()
                    fn(self.sp[ix], n, self.dp[j][ix], self.caps[ix], self.ltp[1 + j], r, pr, csizes=self.lcs[j][:CHAINS],
                       max_symbol_value=255, table_log=11)
                    reps.append(r)
                single = (n < 256) | ((F == 2) & (n < 1024))
                tried = (n <= 128 * 1024) & (n >= torch.where(F == 2, 6, MIN_LIT))
                v = torch.where(single, self.lcs[1][:CHAINS], self.lcs[0][:CHAINS])
                fs = torch.where(single, reps[1], reps[0])
                err = (v < 0) & (v >= -120)                                   # error codes, as int64
                gain = (n >> MIN_GAIN_LOG) + 2                                # size_t: n < gain rejects nothing
                raw = err | (v == 0) | (~err & (v >= n - gain) & (n >= gain))
                rle = ~raw & (v == 1) & ((n >= 8) | self.equal[ix])
                kind = torch.where(raw | (v == 1), torch.where(rle, 1, 0), torch.where(fs != 0, 3, 2))
                kind = torch.where(tried, kind, 0)
                kind = torch.where(n > 128 * 1024, 4, kind)
                commit = kind == 2
                T.copy_(torch.where(commit[:, None], torch.where(single[:, None], self.ltabs[2].view(CHAINS, 256),
                                                                 self.ltabs[1].view(CHAINS, 256)), T))
                F.copy_(torch.where(commit, 1, F))
                self.lval[ix] = torch.where(tried, v, 0)
                self.lkind[ix] = kind.to(torch.uint8)
        return timed(go)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--gib", type=float, default=1.0)
    ap.add_argument("--steps", type=int, default=SLICE_STEPS)
    args = ap.parse_args()
    results = {}

    def add(key, ms, nbytes):
        results.setdefault(key, []).append(ms * GIB / nbytes)

    sizes, flags, prefer = ragged_sizes(int(args.gib * GIB))
    s = Policy(sizes, prefer)
    s.prepare_loop(args.steps)
    s.policy()                                                              # warm-up and checks
    s.back.zero_(); s.policy_decode()
    torch.cuda.synchronize()
    kinds = s.kinds.cpu().numpy()
    back_ok = (s.back == s.src)
    byte_start = torch.from_numpy(np.concatenate([[0], np.cumsum(s.sizes_h)])[:-1]).cuda()
    bad = (~back_ok).nonzero().flatten()
    blk = torch.searchsorted(byte_start, bad, right=True) - 1
    assert bool((s.kinds[blk] == 1).all()), "only RLE by the n >= 8 rule may differ"   # no other block fails to regenerate
    assert torch.equal(s.res[torch.from_numpy(kinds != 4).cuda()], s.ss[torch.from_numpy(kinds != 4).cuda()])
    s.loop()
    ix = torch.cat(s.step_ix)
    assert torch.equal(s.lkind[ix], s.kinds[ix]), "the loop's kinds"
    assert torch.equal(s.lval[ix], s.cs[ix]), "the loop's values"
    s.mixed()
    torch.cuda.synchronize()
    for _ in range(args.runs):
        add("policy_compress", s.policy(), s.n)
        add("mixed_size_rule_compress", s.mixed(), s.n)
        add("policy_decode", s.policy_decode(), s.n)
        add("loop_compress_slice", s.loop(), s.loop_bytes)
    summary = {k: {"median": round(sorted(v)[len(v) // 2], 3), "min": round(min(v), 3), "max": round(max(v), 3)}
               for k, v in results.items()}
    print(json.dumps({"gpu": gpu_info(), "bytes": s.n, "chains": CHAINS, "blocks": s.nb,
                      "kinds": {str(k): int((kinds == k).sum()) for k in range(5)},
                      "blocks_1x": int(s.forms.sum().item()), "loop_slice": {"steps": s.steps, "bytes": s.loop_bytes},
                      "runs": args.runs, "ms_per_gib": summary}))


if __name__ == "__main__":
    main()
