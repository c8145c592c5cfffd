"""FSEB200_HUF_compress{4X,1X}_repeat_chains_packed and FSEB200_HUF_decompress{4X,1X}_repeat_packed (-m gpu).

Compress, against the reference loop (HUF_compress{4X,1X}_repeat per block at HUF_compressBound, the stream's state carried):
every value, stored block at its offset, kind, final table word, flag and chain header, on single-block, mid-chain, drifting and
4,096-block chains; against FSEB200_HUF_compress{4X,1X}_repeat_chains on the same inputs; capacities one below, at and one above
the end of several blocks; chains cut into two calls; malformed geometry; a non-default stream.
Decompress: the round trip, FSEB200_HUF_decompress{4X,1X}_repeat_blocks on the derived header arrays and the compiled
reference's decoders on a sample; every verdict of its own (raw and RLE lengths, kind 3 without a header, unknown kinds, sizes
above 128 KB, malformed geometry); an odd dIn; canaries around every destination."""
import numpy as np
import pytest
import torch

from helpers import is_error
from huf_repeat_cases import main_configs
from huf_chain_cases import single_chains, drift_chains, empty_chains, long_chain
from huf_chain_packed_cases import at_bound, packed_chains, resolve_headers
from huf_chain_harness import (PLAIN, PackedChains, Arena, decode, ref_decode, regenerable, _ref, _t, _u64, _view, FILL, SRC_WRONG,
                               CORRUPT, TOO_SMALL)
import finitestateentropy_b200 as fb

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("four", [True, False], ids=["4X", "1X"])
def test_compress_matches_the_reference_loop_and_the_chain_call(four):
    ref = _ref()
    for msv, tlog in main_configs():
        chains = at_bound(single_chains(ref, four, msv, tlog))[::3] + empty_chains(1) + packed_chains(ref, four, msv, tlog)
        run = PackedChains(PLAIN[four], ref, chains, msv, tlog)
        res = run.call(stream=torch.cuda.Stream())
        run.check_one_call(res)
        _, out, off, cs, kinds, _ = res
        # the pointer-based chain call on the same inputs at capacities HUF_compressBound
        n = len(run.blocks)
        run2 = PackedChains.__new__(PackedChains)
        run2.__dict__.update(run.__dict__)
        run2.reset()
        caps = np.array([129 + int(x) + (int(x) >> 8) + 8 for x in run.ss.cpu().numpy()], np.uint64)
        dst = Arena()
        for k in range(n):
            dst.add(np.zeros(int(caps[k]), np.uint8), skew=k % 5)
        dst.upload()
        dp = torch.tensor([dst.ptr(k) for k in range(n)], dtype=torch.int64, device="cuda")
        fn = fb.huf_compress_repeat_chains if four else fb.huf_compress1x_repeat_chains
        cs2, hp2, hs2 = fn(_t(run.starts), run.sp, run.ss, dp, _t(caps), run.pr, _view(run2.ctp), _view(run2.rep), _view(run2.chp),
                           _view(run2.chs), max_symbol_value=msv, table_log=tlog)
        cs2, hs2 = _u64(cs2), _u64(hs2)
        assert (cs2 == cs).all()
        coded = np.array([not is_error(int(v)) and int(v) >= 2 for v in cs2])
        assert ((kinds == 3) == (coded & (hs2 != 0))).all()
        h2 = dst.dev.cpu().numpy()
        ho = out.cpu().numpy()
        for k in range(n):
            r = int(cs[k])
            if not is_error(r) and r >= 1:
                assert (ho[int(off[k]):int(off[k]) + r] == h2[dst.offs[k]:dst.offs[k] + r]).all(), k
        s1, s2 = run.state(), run2.state()
        assert (s1["tabs"] == s2["tabs"]).all() and (s1["rep"] == s2["rep"]).all() and (s1["chs"] == s2["chs"]).all()
        ptr_of = {dst.ptr(k): out.data_ptr() + int(off[k]) for k in range(n)}
        for c in range(len(chains)):
            p2 = int(s2["chp"][c])
            assert int(s1["chp"][c]) == ptr_of.get(p2, p2), c


@pytest.mark.parametrize("four", [True, False], ids=["4X", "1X"])
def test_one_chain_of_4096_blocks(four):
    ref = _ref()
    chains = at_bound([long_chain(ref, 4096)]) + empty_chains(1)
    run = PackedChains(PLAIN[four], ref, chains, 255, 11)
    run.check_one_call(run.call())
    assert run.kinds.count(3) > 4000 and run.kinds.count(2) >= 1


@pytest.mark.parametrize("four", [True, False], ids=["4X", "1X"])
def test_capacity_at_block_ends(four):
    ref = _ref()
    chains = packed_chains(ref, four, 255, 12)[::5]
    run = PackedChains(PLAIN[four], ref, chains, 255, 12)
    whole = run.call()
    run.check_one_call(whole)
    ends = whole[2]
    total = int(ends[-1])
    for k in (1, len(ends) // 3, len(ends) // 2, len(ends) - 2):
        for cap in (int(ends[k]) - 1, int(ends[k]), int(ends[k]) + 1):
            if cap < 1 or cap >= total:                                   # an empty `out` has no address
                continue
            run.reset()
            before = run.state()
            buf, out, off, cs, kinds, idx = run.call(cap=cap)
            assert (off == ends).all()
            host = buf.cpu().numpy()
            o0 = out.data_ptr() - buf.data_ptr()
            assert (host[:o0] == FILL).all() and (host[o0 + cap:] == FILL).all()
            for b in range(len(idx)):
                want = run.vals[b]
                if is_error(want):
                    assert int(cs[b]) == want and kinds[b] == 4
                elif int(ends[b + 1]) <= cap:
                    assert int(cs[b]) == want and kinds[b] == run.kinds[b]
                    assert (host[o0 + int(off[b]):o0 + int(off[b + 1])] == run.blobs[b]).all()
                else:
                    assert int(cs[b]) == TOO_SMALL and kinds[b] == 4, (b, cap)
            after = run.state()
            for key in before:
                assert (before[key] == after[key]).all(), key
            run.check_one_call(run.call(cap=int(off[-1])))                # the same call at the size it asked for


@pytest.mark.parametrize("four", [True, False], ids=["4X", "1X"])
def test_split_calls_give_one_calls_result_and_decode(four):
    ref = _ref()
    msv, tlog = 255, 11
    chains = at_bound(drift_chains(ref))[::3]                              # entry tables that are Huffman tables: they decode
    one = PackedChains(PLAIN[four], ref, chains, msv, tlog)
    whole = one.call()
    one.check_one_call(whole)
    two = PackedChains(PLAIN[four], ref, chains, msv, tlog)
    mids = [len(ch["blocks"]) // 2 for ch in chains]
    a = two.call(parts=[(0, m) for m in mids])
    entry = (_view(two.chp).clone(), _view(two.chs).clone())               # the second part's entry headers: inside a's buffer
    b = two.call(parts=[(m, len(ch["blocks"])) for m, ch in zip(mids, chains)])
    s1, s2 = one.state(), two.state()
    for k in ("tabs", "rep", "chs"):
        assert (s1[k] == s2[k]).all(), k
    got = {}
    for buf, out, off, cs, kinds, idx in (a, b):
        host = out.cpu().numpy()
        for j, k in enumerate(idx):
            got[k] = (int(cs[j]), int(kinds[j]), host[int(off[j]):int(off[j + 1])])
    for k in range(len(one.blocks)):
        assert got[k][0] == one.vals[k] and (got[k][2] == one.blobs[k]).all(), k
    # the second part decodes from its own buffer with the entry headers the first call left
    _, out, off, cs, kinds, idx = b
    st = [0]
    for m, ch in zip(mids, chains):
        st.append(st[-1] + len(ch["blocks"]) - m)
    sizes = [int(one.ss[k]) for k in idx]
    res, regions = decode(PLAIN[four], _t(st), out, _t(off), _t(kinds, torch.uint8), entry[0], entry[1], sizes)
    ok = 0
    heads = resolve_headers(kinds, st)
    sub = [None] * len(one.blocks)
    for j, k in enumerate(idx):
        sub[k] = heads[j]
    entry_ptr = entry[0].cpu().numpy()
    for j, k in enumerate(idx):
        c, i = one.blocks[k]
        if not regenerable(one, k, sub, lambda c: int(entry_ptr[c]) == two.hdrs.ptr(c) and not two.hdr_blobs[c][1]):
            continue
        src = chains[c]["blocks"][i]["src"]
        assert int(res[j]) == len(src) and (regions[j] == src).all(), (chains[c]["name"], i)
        ok += 1
    assert ok > 20


@pytest.mark.parametrize("four", [True, False], ids=["4X", "1X"])
def test_round_trip_and_agreement_with_the_header_decoders(four):
    ref = _ref()
    msv, tlog = 255, 11                                                    # tables the X1 decoders' 11-bit DTable holds
    chains = at_bound(drift_chains(ref)) + [long_chain(ref, 512)]         # entry tables that are Huffman tables: they decode
    run = PackedChains(PLAIN[four], ref, chains, msv, tlog)
    res0 = run.call()
    run.reset()
    _, out, off, cs, kinds, idx = res0
    sizes = [int(x) for x in run.ss.cpu().numpy()]
    res, regions = decode(PLAIN[four], _t(run.starts), out, _t(off), _t(kinds, torch.uint8), _view(run.chp), _view(run.chs), sizes,
                          expect=[chains[c]["blocks"][i]["src"] for c, i in run.blocks])
    heads = resolve_headers(kinds, run.starts)
    n_ok = 0
    for k, (c, i) in enumerate(run.blocks):
        if not regenerable(run, k, heads, lambda c: not run.hdr_blobs[c][1]):
            continue
        src = chains[c]["blocks"][i]["src"]
        assert int(res[k]) == len(src) and (regions[k] == src).all(), (chains[c]["name"], i, kinds[k])
        n_ok += 1
    assert n_ok > 500
    # the Huffman kinds through FSEB200_HUF_decompress{4X,1X}_repeat_blocks with the derived header arrays
    hk = [k for k in range(len(kinds)) if kinds[k] in (2, 3)]
    hp, hs = [], []
    for k in hk:
        h = heads[k]
        if h is None:
            hp.append(0); hs.append(0)
        elif h[0] == "chain":
            hp.append(run.hdrs.ptr(h[1])); hs.append(len(run.hdr_blobs[h[1]][0]))
        else:
            hp.append(out.data_ptr() + int(off[h[1]])); hs.append(int(off[h[1] + 1] - off[h[1]]))
    back = torch.zeros(sum(sizes[k] for k in hk) + 64, dtype=torch.uint8, device="cuda")
    nn = torch.tensor([sizes[k] for k in hk], dtype=torch.int64, device="cuda")
    bp = torch.cumsum(nn, 0) - nn + back.data_ptr()
    fn = fb.huf_decompress_repeat_blocks if four else fb.huf_decompress1x_repeat_blocks
    cp = _t([out.data_ptr() + int(off[k]) for k in hk])
    cz = _t([int(off[k + 1] - off[k]) for k in hk])
    r2 = _u64(fn(cp, cz, bp, nn, _t(hp), _t(hs)))
    assert (r2 == res[hk]).all()
    host = out.cpu().numpy()
    for j in range(0, len(hk), 37):                                       # the compiled reference on a sample
        k = hk[j]
        blob = host[int(off[k]):int(off[k + 1])]
        hdr = None if hs[j] == 0 else (host[int(off[heads[k][1]]):int(off[heads[k][1] + 1])] if heads[k][0] == "block"
                                       else run.hdr_blobs[heads[k][1]][0])
        assert ref_decode(ref, four, blob, sizes[k], hdr)[0] == int(res[k]), k


@pytest.mark.parametrize("four", [True, False], ids=["4X", "1X"])
def test_decoder_verdicts(four):
    """raw with L != n, RLE with L != 1, kind 3 without a header, kinds 4 and 200, sizes above 128 KB, malformed chain starts,
    an odd dIn; canaries around every destination"""
    rng = np.random.default_rng(3)
    raw = rng.integers(0, 256, 300, dtype=np.uint8)
    blobs = [raw[:100], raw[100:101], raw[101:150], raw[150:152], raw[152:160], raw[160:170], raw[170:180], raw[180:300],
             np.zeros(0, np.uint8), raw[0:1]]
    kinds = [0, 1, 0, 1, 3, 4, 200, 0, 0, 1]
    sizes = [100, 77, 50, 5, 64, 10, 10, 200 * 1024, 0, 200 * 1024]
    want = [100, 77, CORRUPT, CORRUPT, CORRUPT, CORRUPT, CORRUPT, SRC_WRONG, 0, SRC_WRONG]
    lens = [len(b) for b in blobs]
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    flat = np.concatenate(blobs)
    for skew in (0, 1, 7):
        buf = torch.full((len(flat) + 64 + skew,), 0x11, dtype=torch.uint8, device="cuda")
        buf[skew:skew + len(flat)] = torch.from_numpy(flat).cuda()
        packed = buf[skew:skew + len(flat) + 32]
        st = _t([0, 4, len(blobs)])
        res, regions = decode(PLAIN[four], st, packed, _t(offs), _t(kinds, torch.uint8), _t([0, 0]), _t([0, 0]), sizes)
        assert list(res) == want, (skew, list(res))
        assert (regions[0] == blobs[0]).all() and (regions[1] == blobs[1][0]).all()
        for j in (2, 3, 4, 5, 6, 7, 9):
            assert (regions[j] == 0x5A).all(), j
    for bad in ([1, 4, len(blobs)], [0, 4, len(blobs) - 1], [0, 5, 4]):
        res, regions = decode(PLAIN[four], _t(bad), packed, _t(offs), _t(kinds, torch.uint8), _t([0, 0]), _t([0, 0]), sizes)
        assert (res == SRC_WRONG).all()
        assert all((r == 0x5A).all() for r in regions)


@pytest.mark.parametrize("four", [True, False], ids=["4X", "1X"])
def test_malformed_compress_geometry_writes_only_verdicts_and_kinds(four):
    ref = _ref()
    chains = packed_chains(ref, four, 255, 12)[:6]
    run = PackedChains(PLAIN[four], ref, chains, 255, 12)
    nb = len(run.blocks)
    good = run.starts
    before = run.state()
    for st in ([1] + good[1:], good[:-1] + [nb - 1], good[:3] + [good[2] - 1] + good[4:]):
        buf, out, off, cs, kinds, _ = run.call(starts=st)
        assert (cs == SRC_WRONG).all() and (kinds == 4).all()
        assert (off == 0xCD).all()
        assert (buf.cpu().numpy() == FILL).all()
        after = run.state()
        for k in before:
            assert (before[k] == after[k]).all(), k


@pytest.mark.parametrize("four", [True, False], ids=["4X", "1X"])
def test_both_calls_are_ordered_on_a_side_stream(four):
    ref = _ref()
    chains = at_bound(drift_chains(ref))[:12]
    run = PackedChains(PLAIN[four], ref, chains, 255, 11)
    s = torch.cuda.Stream()
    sizes = [int(x) for x in run.ss.cpu().numpy()]
    saved = run.srcs.dev.clone()
    with torch.cuda.stream(s):
        run.srcs.dev.zero_()                                               # work before: the sources are written back on s
        torch.cuda._sleep(20_000_000)
        run.srcs.dev.copy_(saved)
        fn = fb.huf_compress_repeat_chains_packed if four else fb.huf_compress1x_repeat_chains_packed
        out, off, cs, kinds = fn(_t(run.starts), run.sp, run.ss, run.pr, _view(run.ctp), _view(run.rep), _view(run.chp),
                                 _view(run.chs), out=torch.empty(sum(sizes) + 32, dtype=torch.uint8, device="cuda"),
                                 max_symbol_value=255, table_log=11)
        kinds_copy = kinds.clone()                                         # work after, on s
    s.synchronize()
    assert (_u64(cs) == np.array(run.vals, np.uint64)).all() and list(kinds_copy.cpu().numpy()) == run.kinds
    run.reset()
    dst = torch.full((sum(sizes) + 64,), 0x5A, dtype=torch.uint8, device="cuda")
    nn = torch.tensor(sizes, dtype=torch.int64, device="cuda")
    dp = torch.cumsum(nn, 0) - nn + dst.data_ptr()
    fn = fb.huf_decompress_repeat_packed if four else fb.huf_decompress1x_repeat_packed
    with torch.cuda.stream(s):
        torch.cuda._sleep(20_000_000)
        res = fn(_t(run.starts), out, off, kinds, _view(run.chp), _view(run.chs), dp, nn)
        back = dst.clone()
    s.synchronize()
    r = _u64(res)
    host = back.cpu().numpy()
    o = 0
    heads = resolve_headers(run.kinds, run.starts)
    for k, (c, i) in enumerate(run.blocks):
        src = chains[c]["blocks"][i]["src"]
        if regenerable(run, k, heads, lambda c: not run.hdr_blobs[c][1]):
            assert int(r[k]) == len(src) and (host[o:o + len(src)] == src).all(), k
        o += len(src)
