"""FSEB200_HUF_compress{4X,1X}_repeat_chains against the reference loop (-m gpu).

Per chain, HUF_compress{4X,1X}_repeat block after block with the stream's (table, flag, header) carried: every value, the bytes,
every final table word, flag and chain header, and every block's header.  Chains: empty ones, single blocks (which also equal
FSEB200_HUF_compress{4X,1X}_repeat_blocks), every single-block input in the middle of a chain, drifting distributions under every
incoming flag and several prefer patterns, and one chain of 4,096 x 32 KB blocks.  Guard bytes around every buffer and array;
malformed chain geometry; chains cut into two calls; and a round trip through one FSEB200_HUF_decompress{4X,1X}_repeat_blocks
call, which the reference's HUF_readDTableX1 + HUF_decompress{4X,1X}1_usingDTable agrees with."""
import numpy as np
import pytest
import torch

from helpers import is_error
from huf_repeat_cases import main_configs, room
from huf_chain_cases import ref_chain, single_chains, mid_chains, drift_chains, empty_chains, long_chain, chain_header
from huf_chain_harness import Arena, ref_decode, _ref, _dev, _view, _guards_ok, SRC_WRONG
import finitestateentropy_b200 as fb

pytestmark = pytest.mark.gpu


class Run:
    """the chains' buffers on the device: sources, destinations (the complement of the expected bytes, canaries around), tables
    (canaries around), chain headers, and the per-chain state arrays with guards"""

    def __init__(self, ref, four, chains, msv, tlog):
        self.ref, self.four, self.chains, self.msv, self.tlog = ref, four, chains, msv, tlog
        self.want = [ref_chain(ref, four, ch, msv, tlog) for ch in chains]
        self.blocks = [(c, i) for c, ch in enumerate(chains) for i in range(len(ch["blocks"]))]
        srcs, dsts, hdrs = Arena(), Arena(), Arena()
        for k, (c, i) in enumerate(self.blocks):
            blk = self.chains[c]["blocks"][i]
            srcs.add(blk["src"], skew=k % 3)
            fill = np.full(room(len(blk["src"]), blk["cap"]), 0x33, np.uint8)
            exp = self.want[c][0][i][1]
            fill[:len(exp)] = ~exp
            dsts.add(fill, skew=(k * 5) % 7)
        self.hdr_blobs = [chain_header(ref, ch) for ch in chains]
        for blob, _ in self.hdr_blobs:
            hdrs.add(blob)
        self.srcs, self.dsts, self.hdrs = srcs.upload(), dsts.upload(), hdrs.upload()
        words = 256 + 64
        tab = np.full(64 + len(chains) * words, 0xC7C7C7C7, np.uint32)
        self.toff = [64 + c * words + (c % 4) for c in range(len(chains))]
        for o, ch in zip(self.toff, chains):
            tab[o:o + 256] = ch["table"]
        self.tab_host = tab
        self.tab = torch.from_numpy(tab.view(np.int32)).cuda()
        n = len(self.blocks)
        self.sp = torch.tensor([srcs.ptr(k) for k in range(n)] or [0], dtype=torch.int64, device="cuda")[:n]
        self.ss = torch.tensor([len(self.chains[c]["blocks"][i]["src"]) for c, i in self.blocks] or [0], dtype=torch.int64, device="cuda")[:n]
        self.dp = torch.tensor([dsts.ptr(k) for k in range(n)] or [0], dtype=torch.int64, device="cuda")[:n]
        caps = np.array([self.chains[c]["blocks"][i]["cap"] for c, i in self.blocks], np.uint64)
        self.dc = torch.from_numpy(caps.view(np.int64)).cuda()
        self.pr = torch.tensor([self.chains[c]["blocks"][i]["prefer"] for c, i in self.blocks] or [0], dtype=torch.int32, device="cuda")[:n]
        self.ctp = _dev([self.tab.data_ptr() + 4 * o for o in self.toff])
        self.rep = _dev([ch["flag"] for ch in chains], torch.int32)
        self.chp = _dev([hdrs.ptr(c) for c in range(len(chains))])
        self.chs = _dev([len(b) for b, _ in self.hdr_blobs])
        self.cs = _dev([0xAB] * n)
        self.hp = _dev([0xAB] * n)
        self.hs = _dev([0xAB] * n)
        self.first = [sum(len(ch["blocks"]) for ch in chains[:c]) for c in range(len(chains))]

    def call(self, parts=None, starts=None, stream=None):
        """one call over the blocks parts[c] = (lo, hi) of each chain c (all of them by default); `starts` overrides the geometry"""
        parts = parts or [(0, len(ch["blocks"])) for ch in self.chains]
        idx, st = [], [0]
        for c, (lo, hi) in enumerate(parts):
            idx += [self.first[c] + i for i in range(lo, hi)]
            st.append(len(idx))
        if starts is not None:
            st = starts
        ix = torch.tensor(idx or [0], dtype=torch.int64, device="cuda")[:len(idx)]
        cs, hp, hs = _dev([0xCD] * len(idx)), _dev([0xCD] * len(idx)), _dev([0xCD] * len(idx))
        fn = fb.huf_compress_repeat_chains if self.four else fb.huf_compress1x_repeat_chains
        sv = _dev(st)
        with torch.cuda.stream(stream or torch.cuda.current_stream()):
            fn(_view(sv), self.sp[ix], self.ss[ix], self.dp[ix], self.dc[ix], self.pr[ix], _view(self.ctp), _view(self.rep),
               _view(self.chp), _view(self.chs), csizes=_view(cs), hdr_ptrs=_view(hp), hdr_sizes=_view(hs),
               max_symbol_value=self.msv, table_log=self.tlog)
        torch.cuda.synchronize()
        for t in (cs, hp, hs, sv, self.ctp, self.rep, self.chp, self.chs):
            assert _guards_ok(t)
        if starts is None:
            _view(self.cs)[ix] = _view(cs)
            _view(self.hp)[ix] = _view(hp)
            _view(self.hs)[ix] = _view(hs)
        return _view(cs), _view(hp), _view(hs)

    def state(self):
        out = self.dsts.dev.cpu().numpy()
        tabs = self.tab.cpu().numpy().view(np.uint32)
        return dict(out=out, tabs=tabs.copy(), rep=_view(self.rep).cpu().numpy(), chp=_view(self.chp).cpu().numpy().view(np.uint64),
                    chs=_view(self.chs).cpu().numpy(), cs=_view(self.cs).cpu().numpy().view(np.uint64),
                    hp=_view(self.hp).cpu().numpy().view(np.uint64), hs=_view(self.hs).cpu().numpy())

    def header_value(self, c, h):
        """(pointer, size) of a reference-loop header token in chain c"""
        if h is None:
            return 0, 0
        if h[0] == "chain":
            return self.hdrs.ptr(c), len(self.hdr_blobs[c][0])
        k = self.first[c] + h[1]
        return self.dsts.ptr(k), self.want[c][0][h[1]][0]

    def check(self):
        s = self.state()
        assert self.dsts.canaries_intact(s["out"])
        assert (self.srcs.dev.cpu().numpy() == self.srcs.host).all()
        gaps = np.ones(len(s["tabs"]), bool)
        for o in self.toff:
            gaps[o:o + 256] = False
        assert (s["tabs"][gaps] == 0xC7C7C7C7).all()
        for c, ch in enumerate(self.chains):
            per, (T, F, H) = self.want[c]
            for i, (r, data, h) in enumerate(per):
                k = self.first[c] + i
                what = (ch["name"], i, int(s["cs"][k]), r % (1 << 64))
                assert int(s["cs"][k]) == r % (1 << 64), what
                o = self.dsts.offs[k]
                assert (s["out"][o:o + len(data)] == data).all(), what
                assert (int(s["hp"][k]), int(s["hs"][k])) == self.header_value(c, h), what
            t = s["tabs"][self.toff[c]:self.toff[c] + 256]
            if (T == ch["table"]).all():
                assert (t == ch["table"]).all(), ch["name"]
            else:
                assert (t == (T & 0x00FFFFFF)).all(), ch["name"]
            assert int(s["rep"][c]) == F, ch["name"]
            assert (int(s["chp"][c]), int(s["chs"][c])) == self.header_value(c, H), ch["name"]
        return s


@pytest.mark.parametrize("four", [True, False], ids=["4X", "1X"])
def test_single_block_chains_match_the_reference_and_repeat_blocks(four):
    ref = _ref()
    for msv, tlog in main_configs():
        chains = single_chains(ref, four, msv, tlog)
        chains = chains[:40] + empty_chains(2) + chains[40:]
        run = Run(ref, four, chains, msv, tlog)
        run.call(stream=torch.cuda.Stream())
        s = run.check()
        # the same inputs through the per-block call
        nb = len(run.blocks)
        tab2 = torch.from_numpy(run.tab_host.view(np.int32)).cuda()
        tp = torch.tensor([tab2.data_ptr() + 4 * run.toff[c] for c, _ in run.blocks], dtype=torch.int64, device="cuda")
        fl = torch.tensor([chains[c]["flag"] for c, _ in run.blocks], dtype=torch.int32, device="cuda")
        dst2 = torch.zeros_like(run.dsts.dev)
        dp2 = run.dp - run.dsts.dev.data_ptr() + dst2.data_ptr()
        fn = fb.huf_compress_repeat_blocks if four else fb.huf_compress1x_repeat_blocks
        cs2 = fn(run.sp, run.ss, dp2, run.dc, tp, fl, run.pr, max_symbol_value=msv, table_log=tlog).cpu().numpy().view(np.uint64)
        assert nb and (cs2 == s["cs"]).all()
        out2 = dst2.cpu().numpy()
        for k in range(nb):
            r = int(cs2[k])
            if not is_error(r) and r:
                o = run.dsts.offs[k]
                assert (out2[o:o + r] == s["out"][o:o + r]).all(), k
        assert (tab2.cpu().numpy().view(np.uint32) == s["tabs"]).all()


@pytest.mark.parametrize("four", [True, False], ids=["4X", "1X"])
def test_mid_chain_and_drifting_chains_match_the_reference_loop(four):
    ref = _ref()
    for msv, tlog in main_configs():
        chains = mid_chains(ref, four, msv, tlog) + empty_chains(1) + drift_chains(ref) + empty_chains(2)
        run = Run(ref, four, chains, msv, tlog)
        run.call()
        run.check()


@pytest.mark.parametrize("four", [True, False], ids=["4X", "1X"])
def test_split_calls_give_what_one_call_gives(four):
    ref = _ref()
    msv, tlog = 255, 12
    chains = drift_chains(ref)[::3] + mid_chains(ref, four, msv, tlog)[::7]
    one = Run(ref, four, chains, msv, tlog)
    one.call()
    a = one.check()
    two = Run(ref, four, chains, msv, tlog)
    mids = [len(ch["blocks"]) // 2 for ch in chains]
    two.call(parts=[(0, m) for m in mids])
    two.call(parts=[(m, len(ch["blocks"])) for m, ch in zip(mids, chains)])
    b = two.check()
    for k in ("cs", "hs", "rep", "chs"):
        assert (a[k] == b[k]).all(), k


@pytest.mark.parametrize("four", [True, False], ids=["4X", "1X"])
def test_malformed_chain_starts_write_nothing_but_the_verdicts(four):
    ref = _ref()
    chains = drift_chains(ref)[:6]
    run = Run(ref, four, chains, 255, 12)
    nb = len(run.blocks)
    before = run.state()
    good = [0] + [sum(len(ch["blocks"]) for ch in chains[:c + 1]) for c in range(len(chains))]
    bad_first = [1] + good[1:]
    bad_last = good[:-1] + [nb - 1]
    decrease = list(good)
    decrease[3] = decrease[2] - 1
    for st in (bad_first, bad_last, decrease):
        cs, hp, hs = run.call(starts=st)
        assert (cs.cpu().numpy().view(np.uint64) == SRC_WRONG).all()
        assert (hp.cpu().numpy() == 0xCD).all() and (hs.cpu().numpy() == 0xCD).all()
        after = run.state()
        assert (after["out"] == before["out"]).all()
        assert (after["tabs"] == before["tabs"]).all()
        for k in ("rep", "chp", "chs", "hp", "hs"):
            assert (after[k] == before[k]).all(), k


@pytest.mark.parametrize("four", [True, False], ids=["4X", "1X"])
def test_round_trip_through_one_header_decode_call(four):
    ref = _ref()
    msv, tlog = 255, 11                                                    # tables the X1 decoders' 11-bit DTable holds
    chains = drift_chains(ref) + [long_chain(ref, 512)]
    run = Run(ref, four, chains, msv, tlog)
    run.call()
    s = run.check()
    ks, hdr_bytes = [], []
    for c, ch in enumerate(chains):
        per = run.want[c][0]
        for i, (r, data, h) in enumerate(per):
            if is_error(r) or r < 2:
                continue
            if h is not None and h[0] == "chain" and not run.hdr_blobs[c][1]:
                continue                                                    # a stand-in header: the table has none
            ks.append(run.first[c] + i)
            hdr_bytes.append(None if h is None else run.hdr_blobs[c][0] if h[0] == "chain" else per[h[1]][1])
    assert len(ks) > 100 and any(h is not None for h in hdr_bytes) and any(h is None for h in hdr_bytes)
    ix = torch.tensor(ks, dtype=torch.int64, device="cuda")
    n = run.ss[ix]
    back = torch.full((int(n.sum()) + 64,), 0x5A, dtype=torch.uint8, device="cuda")
    bp = torch.cumsum(n, 0) - n + back.data_ptr()
    fn = fb.huf_decompress_repeat_blocks if four else fb.huf_decompress1x_repeat_blocks
    res = fn(run.dp[ix], _view(run.cs)[ix], bp, n, _view(run.hp)[ix], _view(run.hs)[ix]).cpu().numpy().view(np.uint64)
    out = back.cpu().numpy()
    off = 0
    for j, k in enumerate(ks):
        c, i = run.blocks[k]
        src = chains[c]["blocks"][i]["src"]
        assert int(res[j]) == len(src), (chains[c]["name"], i)
        assert (out[off:off + len(src)] == src).all(), (chains[c]["name"], i)
        data = run.want[c][0][i][1]
        assert ref_decode(ref, four, data, len(src), hdr_bytes[j])[0] == len(src), (chains[c]["name"], i)
        off += len(src)


@pytest.mark.parametrize("four", [True, False], ids=["4X", "1X"])
def test_one_chain_of_4096_blocks(four):
    ref = _ref()
    chains = [long_chain(ref, 4096)] + empty_chains(1)
    run = Run(ref, four, chains, 255, 11)
    run.call()
    run.check()
    per = run.want[0][0]
    assert sum(1 for r, _, h in per if h is not None) > 4000 and sum(1 for r, _, h in per if h is None) >= 1
