"""FSEB200_HUF_compress_mixed_repeat_chains[_packed] and FSEB200_HUF_decompress_mixed_repeat_{blocks,packed} (-m gpu): chains whose
blocks each choose one stream or four.

Compress, against the per-block-form reference loop (huf_mixed_chain_cases.py): every value, stored block, kind, offset, final
table, flag and chain header, and the unpacked call's dHeaders / dHeaderSizes, at both main configurations, on the chain tests'
chains under six flag patterns, ragged literal-like chains and the built cross-form chains; all-0 flags against the 4X calls and
all-1 flags against the 1X calls byte for byte; capacities at block ends; a chain cut into two calls; malformed geometry; a side
stream; one chain of 4,096 blocks with alternating flags.
Decompress: the round trip; per-block verdicts equal to the 4X / 1X header decoders, with the flags as written and flipped; the
decoder's own verdicts; the packed decoder against the blocks decoder on the derived header arrays."""
import numpy as np
import pytest
import torch

from helpers import is_error
from huf_repeat_cases import main_configs
from huf_chain_cases import drift_chains
from huf_chain_packed_cases import at_bound, resolve_headers
from huf_mixed_chain_cases import mixed_chains, ragged_chains, with_flags, long_mixed_chain, built_chains
from huf_chain_harness import (MIXED, PackedChains, decode, ref_decode, regenerable, _ref, _t, _u64, _view, FILL, SRC_WRONG, CORRUPT,
                               TOO_SMALL)
import finitestateentropy_b200 as fb

pytestmark = pytest.mark.gpu


def _token_ptrs(run, dst, c, h, cs):
    if h is None:
        return (0, 0)
    if h[0] == "chain":
        return (run.hdrs.ptr(c), len(run.hdr_blobs[c][0]))
    k = run.first[c] + h[1]
    return (dst.ptr(k), int(cs[k]))


@pytest.mark.parametrize("msv,tlog", main_configs())
def test_compress_matches_the_reference_loop(msv, tlog):
    """packed and unpacked mixed calls against the per-block-form loop: values, bytes, kinds, offsets, state, block headers"""
    ref = _ref()
    run = PackedChains(MIXED, ref, mixed_chains(ref, msv, tlog), msv, tlog)
    assert len(set(run.flags)) >= 3
    run.check_one_call(run.call(stream=torch.cuda.Stream()))
    run.reset()
    dst, cs, hp, hs = run.unpacked()
    assert (cs == np.array(run.vals, np.uint64)).all()
    host = dst.dev.cpu().numpy()
    k = 0
    for c, (per, (T, F, H)) in enumerate(run.want):
        for i, (r, data, h) in enumerate(per):
            if not is_error(r) and r >= 1:
                assert (host[dst.offs[k]:dst.offs[k] + r] == data).all(), (run.chains[c]["name"], i)
            assert (int(hp[k]), int(hs[k])) == _token_ptrs(run, dst, c, h, cs), (run.chains[c]["name"], i)
            k += 1
    s = run.state()
    for c, ch in enumerate(run.chains):
        _, (T, F, H) = run.want[c]
        t = s["tabs"][run.toff[c]:run.toff[c] + 256]
        assert (t == (ch["table"] if (T == ch["table"]).all() else T & 0x00FFFFFF)).all(), ch["name"]
        assert int(s["rep"][c]) == F
        assert (int(s["chp"][c]), int(s["chs"][c])) == _token_ptrs(run, dst, c, H, cs), ch["name"]


@pytest.mark.parametrize("flag", [0, 1])
def test_uniform_flags_equal_the_4x_and_1x_calls(flag):
    """all-0 flags give the 4X calls' results byte for byte, all-1 flags the 1X calls', packed and unpacked, and their decoders"""
    ref = _ref()
    pattern = "all%d" % flag
    chains = with_flags(at_bound(drift_chains(ref))[::2] + ragged_chains(seed=9), pattern)
    four = flag == 0
    for msv, tlog in main_configs():
        run = PackedChains(MIXED, ref, chains, msv, tlog)
        a = run.call()
        sa = run.state()
        run.reset()
        b = run.call(fn=fb.huf_compress_repeat_chains_packed if four else fb.huf_compress1x_repeat_chains_packed)
        sb = run.state()
        assert (a[0].cpu().numpy() == b[0].cpu().numpy()).all()
        for j in (2, 3, 4):
            assert (a[j] == b[j]).all()
        for key in ("tabs", "rep", "chs"):
            assert (sa[key] == sb[key]).all(), key
        pa = {a[1].data_ptr() + int(o): j for j, o in enumerate(a[2])}
        pb = {b[1].data_ptr() + int(o): j for j, o in enumerate(b[2])}
        assert [pa.get(int(p), int(p)) for p in sa["chp"]] == [pb.get(int(p), int(p)) for p in sb["chp"]]
        # the decoders on the same buffer
        sizes = [int(x) for x in run.ss.cpu().numpy()]
        run.reset()
        _, out, off, cs, kinds, _ = a
        nn = torch.tensor(sizes, dtype=torch.int64, device="cuda")
        d1 = torch.zeros(sum(sizes) + 64, dtype=torch.uint8, device="cuda")
        d2 = torch.zeros_like(d1)
        fn = fb.huf_decompress_repeat_packed if four else fb.huf_decompress1x_repeat_packed
        r1 = fb.huf_decompress_mixed_repeat_packed(_t(run.starts), out, _t(off), _t(kinds, torch.uint8), run.sg, _view(run.chp),
                                                   _view(run.chs), torch.cumsum(nn, 0) - nn + d1.data_ptr(), nn)
        r2 = fn(_t(run.starts), out, _t(off), _t(kinds, torch.uint8), _view(run.chp), _view(run.chs),
                torch.cumsum(nn, 0) - nn + d2.data_ptr(), nn)
        torch.cuda.synchronize()
        assert (_u64(r1) == _u64(r2)).all() and torch.equal(d1, d2)
        # unpacked
        run.reset()
        dst1, cs1, hp1, hs1 = run.unpacked()
        s1 = run.state()
        run.reset()
        dst2, cs2, hp2, hs2 = run.unpacked(fb.huf_compress_repeat_chains if four else fb.huf_compress1x_repeat_chains)
        s2 = run.state()
        assert (cs1 == cs2).all() and (hs1 == hs2).all()
        assert (dst1.dev.cpu().numpy() == dst2.dev.cpu().numpy()).all()
        m1 = {dst1.ptr(k): k for k in range(len(run.blocks))}
        m2 = {dst2.ptr(k): k for k in range(len(run.blocks))}
        assert [m1.get(int(p), int(p)) for p in hp1] == [m2.get(int(p), int(p)) for p in hp2]
        for key in ("tabs", "rep", "chs"):
            assert (s1[key] == s2[key]).all(), key


def _header_arrays(run, out, off, kinds, heads, hk):
    hp, hs = [], []
    for k in hk:
        h = heads[k]
        if h is None:
            hp.append(0); hs.append(0)
        elif h[0] == "chain":
            hp.append(run.hdrs.ptr(h[1])); hs.append(len(run.hdr_blobs[h[1]][0]))
        else:
            hp.append(out.data_ptr() + int(off[h[1]])); hs.append(int(off[h[1] + 1] - off[h[1]]))
    return hp, hs


def test_round_trip_and_verdicts_of_both_forms():
    """the packed decoder regenerates every stored block (but for the weight-12 exception); its verdicts equal the mixed blocks
    decoder's on the derived header arrays, which equal the 4X decoder's for flag-0 blocks and the 1X decoder's otherwise -- also
    with every flag flipped, where a coded block gets the other form's verdict; the compiled reference agrees on a sample"""
    ref = _ref()
    msv, tlog = 255, 11
    chains = with_flags(at_bound(drift_chains(ref)) + ragged_chains(seed=4), "random", seed=3) + built_chains(ref)
    run = PackedChains(MIXED, ref, chains, msv, tlog)
    _, out, off, cs, kinds, _ = run.call()
    run.reset()
    sizes = [int(x) for x in run.ss.cpu().numpy()]
    res, regions = decode(MIXED, _t(run.starts), out, _t(off), _t(kinds, torch.uint8), run.sg, _view(run.chp), _view(run.chs), sizes)
    heads = resolve_headers(kinds, run.starts)
    n_ok = 0
    for k, (c, i) in enumerate(run.blocks):
        if not regenerable(run, k, heads, lambda c: not run.hdr_blobs[c][1]):
            continue
        src = chains[c]["blocks"][i]["src"]
        assert int(res[k]) == len(src) and (regions[k] == src).all(), (chains[c]["name"], i, kinds[k], run.flags[k])
        n_ok += 1
    assert n_ok > 200
    hk = [k for k in range(len(kinds)) if kinds[k] in (2, 3)]
    hp, hs = _header_arrays(run, out, off, kinds, heads, hk)
    nn = torch.tensor([sizes[k] for k in hk], dtype=torch.int64, device="cuda")
    cp, cz = _t([out.data_ptr() + int(off[k]) for k in hk]), _t([int(off[k + 1] - off[k]) for k in hk])
    flags = np.array([run.flags[k] for k in hk], np.uint8)
    got = {}
    for name, fn in (("4X", fb.huf_decompress_repeat_blocks), ("1X", fb.huf_decompress1x_repeat_blocks)):
        back = torch.zeros(int(nn.sum()) + 64, dtype=torch.uint8, device="cuda")
        got[name] = _u64(fn(cp, cz, torch.cumsum(nn, 0) - nn + back.data_ptr(), nn, _t(hp), _t(hs)))
    for flip in (False, True):
        f = (flags == 0).astype(np.uint8) * 5 if flip else flags
        back = torch.zeros(int(nn.sum()) + 64, dtype=torch.uint8, device="cuda")
        r = _u64(fb.huf_decompress_mixed_repeat_blocks(cp, cz, torch.cumsum(nn, 0) - nn + back.data_ptr(), nn, _t(hp), _t(hs),
                                                       torch.from_numpy(f).cuda()))
        assert (r == np.where(f != 0, got["1X"], got["4X"])).all(), flip
        if not flip:
            assert (r == res[hk]).all()
    assert (got["1X"] != got["4X"]).any()
    host = out.cpu().numpy()
    for j in range(0, len(hk), 29):
        k = hk[j]
        blob = host[int(off[k]):int(off[k + 1])]
        hdr = None if hs[j] == 0 else (host[int(off[heads[k][1]]):int(off[heads[k][1] + 1])] if heads[k][0] == "block"
                                       else run.hdr_blobs[heads[k][1]][0])
        assert ref_decode(ref, run.flags[k] == 0, blob, sizes[k], hdr)[0] == int(res[k]), k


def test_decoder_verdicts():
    """raw with L != n, RLE with L != 1, kind 3 with an entry header of size 0, kinds 4 and 200, sizes above 128 KB, malformed
    chain starts, an odd dIn, under both flags; canaries around every destination"""
    rng = np.random.default_rng(3)
    raw = rng.integers(0, 256, 300, dtype=np.uint8)
    blobs = [raw[:100], raw[100:101], raw[101:150], raw[150:152], raw[152:160], raw[160:170], raw[170:180], raw[180:300],
             np.zeros(0, np.uint8), raw[0:1], raw[0:9]]
    kinds = [0, 1, 0, 1, 3, 4, 200, 0, 0, 1, 3]
    sizes = [100, 77, 50, 5, 64, 10, 10, 200 * 1024, 0, 200 * 1024, 64]
    want = [100, 77, CORRUPT, CORRUPT, CORRUPT, CORRUPT, CORRUPT, SRC_WRONG, 0, SRC_WRONG, CORRUPT]
    lens = [len(b) for b in blobs]
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    flat = np.concatenate(blobs)
    for skew in (0, 1, 7):
        for pat in (0, 1, 2):
            flags = _t([(i + pat) % 2 if pat < 2 else 1 for i in range(len(blobs))], torch.uint8)
            buf = torch.full((len(flat) + 64 + skew,), 0x11, dtype=torch.uint8, device="cuda")
            buf[skew:skew + len(flat)] = torch.from_numpy(flat).cuda()
            packed = buf[skew:skew + len(flat) + 32]
            st = _t([0, 4, len(blobs)])
            res, regions = decode(MIXED, st, packed, _t(offs), _t(kinds, torch.uint8), flags, _t([0, 0]), _t([0, 0]), sizes)
            assert list(res) == want, (skew, pat, list(res))
            assert (regions[0] == blobs[0]).all() and (regions[1] == blobs[1][0]).all()
            for j in (2, 3, 4, 5, 6, 7, 9, 10):
                assert (regions[j] == 0x5A).all(), j
    for bad in ([1, 4, len(blobs)], [0, 4, len(blobs) - 1], [0, 5, 4]):
        res, regions = decode(MIXED, _t(bad), packed, _t(offs), _t(kinds, torch.uint8), flags, _t([0, 0]), _t([0, 0]), sizes)
        assert (res == SRC_WRONG).all()
        assert all((r == 0x5A).all() for r in regions)


def test_capacity_at_block_ends():
    ref = _ref()
    chains = with_flags(at_bound(drift_chains(ref))[::5] + ragged_chains(seed=2, n_chains=1), "size")
    run = PackedChains(MIXED, ref, chains, 255, 12)
    whole = run.call()
    run.check_one_call(whole)
    ends = whole[2]
    total = int(ends[-1])
    for k in range(1, len(ends) - 1, max(1, len(ends) // 7)):
        for cap in (int(ends[k]) - 1, int(ends[k]), int(ends[k]) + 1):
            if cap < 1 or cap >= total:
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
    run.reset()
    run.check_one_call(run.call(cap=total))


def test_split_calls_carry_the_state_and_decode():
    ref = _ref()
    msv, tlog = 255, 11
    chains = with_flags(at_bound(drift_chains(ref))[::3] + ragged_chains(seed=6, n_chains=2), "alt")
    one = PackedChains(MIXED, ref, chains, msv, tlog)
    one.check_one_call(one.call())
    two = PackedChains(MIXED, ref, chains, msv, tlog)
    mids = [len(ch["blocks"]) // 2 for ch in chains]
    a = two.call(parts=[(0, m) for m in mids])
    entry = (_view(two.chp).clone(), _view(two.chs).clone())
    b = two.call(parts=[(m, len(ch["blocks"])) for m, ch in zip(mids, chains)])
    s1, s2 = one.state(), two.state()
    for k in ("tabs", "rep", "chs"):
        assert (s1[k] == s2[k]).all(), k
    got = {}
    for buf, out, off, cs, kinds, idx in (a, b):
        host = out.cpu().numpy()
        for j, k in enumerate(idx):
            got[k] = (int(cs[j]), host[int(off[j]):int(off[j + 1])])
    for k in range(len(one.blocks)):
        assert got[k][0] == one.vals[k] and (got[k][1] == one.blobs[k]).all(), k
    _, out, off, cs, kinds, idx = b
    st = [0]
    for m, ch in zip(mids, chains):
        st.append(st[-1] + len(ch["blocks"]) - m)
    sizes = [int(one.ss[k]) for k in idx]
    res, regions = decode(MIXED, _t(st), out, _t(off), _t(kinds, torch.uint8), one.sg[torch.tensor(idx, device="cuda")],
                          entry[0], entry[1], sizes)
    heads = resolve_headers(kinds, st)
    sub = [None] * len(one.blocks)
    for j, k in enumerate(idx):
        sub[k] = heads[j]
    entry_ptr = entry[0].cpu().numpy()
    ok = 0
    for j, k in enumerate(idx):
        c, i = one.blocks[k]
        if not regenerable(one, k, sub, lambda c: int(entry_ptr[c]) == two.hdrs.ptr(c) and not two.hdr_blobs[c][1]):
            continue
        src = chains[c]["blocks"][i]["src"]
        assert int(res[j]) == len(src) and (regions[j] == src).all(), (chains[c]["name"], i)
        ok += 1
    assert ok > 20


def test_malformed_geometry_writes_only_verdicts_and_kinds():
    ref = _ref()
    chains = with_flags(at_bound(drift_chains(ref))[:6], "alt")
    run = PackedChains(MIXED, ref, chains, 255, 12)
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


def test_both_calls_are_ordered_on_a_side_stream():
    ref = _ref()
    chains = with_flags(at_bound(drift_chains(ref))[:12], "every3")
    run = PackedChains(MIXED, ref, chains, 255, 11)
    s = torch.cuda.Stream()
    sizes = [int(x) for x in run.ss.cpu().numpy()]
    saved = run.srcs.dev.clone()
    with torch.cuda.stream(s):
        run.srcs.dev.zero_()
        torch.cuda._sleep(20_000_000)
        run.srcs.dev.copy_(saved)
        out, off, cs, kinds = fb.huf_compress_mixed_repeat_chains_packed(
            _t(run.starts), run.sp, run.ss, run.pr, run.sg, _view(run.ctp), _view(run.rep), _view(run.chp), _view(run.chs),
            out=torch.empty(sum(sizes) + 32, dtype=torch.uint8, device="cuda"), max_symbol_value=255, table_log=11)
        kinds_copy = kinds.clone()
    s.synchronize()
    assert (_u64(cs) == np.array(run.vals, np.uint64)).all() and list(kinds_copy.cpu().numpy()) == run.kinds
    run.reset()
    dst = torch.full((sum(sizes) + 64,), 0x5A, dtype=torch.uint8, device="cuda")
    nn = torch.tensor(sizes, dtype=torch.int64, device="cuda")
    dp = torch.cumsum(nn, 0) - nn + dst.data_ptr()
    with torch.cuda.stream(s):
        torch.cuda._sleep(20_000_000)
        res = fb.huf_decompress_mixed_repeat_packed(_t(run.starts), out, off, kinds, run.sg, _view(run.chp), _view(run.chs), dp, nn)
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


def test_one_chain_of_4096_blocks_with_alternating_flags():
    ref = _ref()
    chains = at_bound([long_mixed_chain(ref, 4096)])
    run = PackedChains(MIXED, ref, chains, 255, 11)
    res = run.call()
    run.check_one_call(res)
    assert run.kinds.count(3) > 4000 and run.kinds.count(2) >= 1
    run.reset()
    _, out, off, cs, kinds, _ = res
    sizes = [int(x) for x in run.ss.cpu().numpy()]
    r, regions = decode(MIXED, _t(run.starts), out, _t(off), _t(kinds, torch.uint8), run.sg, _view(run.chp), _view(run.chs), sizes)
    for k, (c, i) in enumerate(run.blocks):
        src = chains[c]["blocks"][i]["src"]
        assert int(r[k]) == len(src) and (regions[k] == src).all(), k
