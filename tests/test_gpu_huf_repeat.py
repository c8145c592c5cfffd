"""FSEB200_HUF_{compress,decompress}{4X,1X}_repeat_blocks against the compiled reference (-m gpu).

Compress: per block, HUF_compress{4X,1X}_repeat's return value, bytes, flag and all 256 table words, for every flag and prefer
value, six kinds of table and tables at both sides of the estimate edge, every block size the plan kernel branches on, five
kinds of capacity, odd addresses and batches of several 32-block plan groups; then 64 streams carried through 8 batch calls the
way a zstd-style literal coder carries them.
Decompress: everything the chains produced (header-less blocks read their header from the block of the same batch that carried
it), and the verdicts of HUF_decompress{4X,1X}1_DCtx / HUF_readDTableX1 + HUF_decompress{4X,1X}1_usingDTable on malformed blocks
and headers, streams too long to be consumed included."""
import numpy as np
import pytest
import torch

from helpers import ptr, probagen, is_error
from huf_repeat_cases import main_cases, main_configs, tables, table_header, ref_repeat, bound, room
from huf_chain_harness import Arena, ref_decode, _ref, _u64
import finitestateentropy_b200 as fb

pytestmark = pytest.mark.gpu
ERR = {name: (1 << 64) - code for code, name in fb.ERROR_NAMES.items()}
BIG = 128 * 1024


def _i64(vals, dev="cuda"):
    return torch.tensor(np.array(vals, dtype=np.uint64).view(np.int64), dtype=torch.int64, device=dev)


def gpu_compress(four, cases, msv, tlog, stream=None):
    """runs the cases as one batch; returns (values, destination regions, flags, tables) and checks every canary"""
    srcs, dsts = Arena(), Arena()
    for i, c in enumerate(cases):
        srcs.add(c["src"], skew=i % 3)
        n = len(c["src"])
        fill = np.full(room(n, c["cap"]), 0x33, np.uint8)
        fill[:len(c["data"])] = ~c["data"]                                  # the complement of the expected bytes
        dsts.add(fill, skew=(i * 5) % 7)
    srcs.upload(); dsts.upload()
    words = 256 + 64
    tab_host = np.full(64 + len(cases) * words, 0xC7C7C7C7, np.uint32)
    toff = [64 + i * words + (i % 4) for i in range(len(cases))]           # 4-byte aligned, not 16-byte aligned
    for o, c in zip(toff, cases):
        tab_host[o:o + 256] = c["table"]
    tab_dev = torch.from_numpy(tab_host.view(np.int32)).cuda()
    dev = "cuda"
    sp = _i64([srcs.ptr(i) for i in range(len(cases))]); ss = _i64([len(c["src"]) for c in cases])
    dp = _i64([dsts.ptr(i) for i in range(len(cases))]); dc = _i64([c["cap"] for c in cases])
    tp = _i64([tab_dev.data_ptr() + 4 * o for o in toff])
    fl = torch.tensor([c["flag"] for c in cases], dtype=torch.int32, device=dev)
    pr = torch.tensor([c["prefer"] for c in cases], dtype=torch.int32, device=dev)
    fn = fb.huf_compress_repeat_blocks if four else fb.huf_compress1x_repeat_blocks
    with torch.cuda.stream(stream or torch.cuda.current_stream()):
        cs = fn(sp, ss, dp, dc, tp, fl, pr, max_symbol_value=msv, table_log=tlog)
    torch.cuda.synchronize()
    out = dsts.dev.cpu().numpy()
    assert dsts.canaries_intact(out)
    assert (srcs.dev.cpu().numpy() == srcs.host).all()
    tabs = tab_dev.cpu().numpy().view(np.uint32)
    gaps = np.ones(len(tabs), bool)
    for o in toff:
        gaps[o:o + 256] = False
    assert (tabs[gaps] == 0xC7C7C7C7).all()
    regions = [out[o:o + len(p)] for o, p in zip(dsts.offs, dsts.parts)]
    return _u64(cs), regions, fl.cpu().numpy(), [tabs[o:o + 256] for o in toff]


def check_against_ref(cases, got):
    vals, regions, flags, tabs = got
    for i, c in enumerate(cases):
        what = (i, c["tname"], c["bname"], c["flag"], c["prefer"], c["kind"], c["cap"])
        assert int(vals[i]) == c["r"] % (1 << 64), what
        assert (regions[i][:len(c["data"])] == c["data"]).all(), what
        assert int(flags[i]) == c["flag_out"], what
        if (c["table_out"] == c["table"]).all():
            assert (tabs[i] == c["table"]).all(), what                    # not written
        else:
            assert (tabs[i] == (c["table_out"] & 0x00FFFFFF)).all(), what  # saved: the reference's padding byte is its workspace's
            assert not (tabs[i] >> 24).any(), what


@pytest.mark.parametrize("four", [True, False], ids=["4X", "1X"])
def test_every_flag_table_block_and_capacity_matches_the_reference(four):
    ref = _ref()
    side = torch.cuda.Stream()
    for msv, tlog in main_configs():
        cases = main_cases(ref, four, msv, tlog)
        assert len(cases) % 32 != 0 and len(cases) > 3 * 32
        check_against_ref(cases, gpu_compress(four, cases, msv, tlog, stream=side))


@pytest.mark.parametrize("four", [True, False], ids=["4X", "1X"])
def test_bad_max_symbol_value_and_table_log(four):
    ref = _ref()
    tabs = tables(ref)
    src = probagen(32768, 0.14)
    for msv, tlog in ((256, 11), (255, 13), (0, 0)):
        cases = []
        for flag in (0, 1, 2):
            for prefer in (0, 1):
                r, data, f, t = ref_repeat(ref, four, src, bound(len(src)), msv, tlog, tabs["same"], flag, prefer)
                cases.append(dict(src=src, cap=bound(len(src)), table=tabs["same"], flag=flag, prefer=prefer, tname="same",
                                  bname="p14", kind="bound", r=r, data=data, flag_out=f, table_out=t))
        check_against_ref(cases, gpu_compress(four, cases, msv, tlog))


def _chain(ref, four, n_streams=64, steps=8):
    """n_streams streams x steps batch calls; the library and the reference loop carry (table, flag) alike.  Returns the blocks
    in step order with what a decoder needs: (source, compressed bytes, header), the header being None (the block's own),
    ("block", j) (the start of produced block j, the stream's last block that carried a table) or ("bytes", a table's header)."""
    tabs = tables(ref)
    rng = np.random.default_rng(11)
    pool = probagen(1 << 22, 0.14)
    # a stream that starts valid gets a table over every symbol: a valid flag on a table lacking a symbol codes it in 0 bits
    st_tab = [tabs["other"].copy() if s % 4 == 0 else np.zeros(256, np.uint32) for s in range(n_streams)]
    st_flag = [2 if s % 4 == 0 else 0 for s in range(n_streams)]
    st_hdr = [("bytes", table_header(ref, tabs["other"])) if s % 4 == 0 else None for s in range(n_streams)]
    dev_tab = [t.copy() for t in st_tab]
    dev_flag = list(st_flag)
    produced = []
    for step in range(steps):
        if step == 4:
            st_flag = [1 if f else 0 for f in st_flag]                     # mid-chain reset to check
            dev_flag = list(st_flag)
        cases = []
        for s in range(n_streams):
            n = int(rng.choice([32768, 4099, 700, 20000]))
            if (s + step) % 5 == 0:
                src = probagen(n, float(rng.choice([0.05, 0.3, 0.6])))
            else:
                o = int(rng.integers(0, len(pool) - n))
                src = pool[o:o + n].copy()
            prefer = s % 2
            r, data, f, t = ref_repeat(ref, four, src, bound(n), 255, 11, st_tab[s], st_flag[s], prefer)
            cases.append(dict(src=src, cap=bound(n), table=dev_tab[s], flag=dev_flag[s], prefer=prefer, tname="chain",
                              bname="s%d_t%d" % (s, step), kind="bound", r=r, data=data, flag_out=f, table_out=t))
        vals, regions, flags, gtabs = gpu_compress(four, cases, 255, 11)
        check_against_ref(cases, (vals, regions, flags, gtabs))
        for s, c in enumerate(cases):
            r = c["r"]
            if not is_error(r) and r >= 2:
                if c["flag_out"] != 0:
                    produced.append((c["src"], c["data"], st_hdr[s]))     # old table: no header
                else:
                    produced.append((c["src"], c["data"], None))
                    st_hdr[s] = ("block", len(produced) - 1)                # the block that last carried a table
            if is_error(r) or r < 2:
                if not (c["table_out"] == c["table"]).all():
                    st_hdr[s] = ("bytes", table_header(ref, c["table_out"]))   # saved by a block stored raw: no block carries it
            st_tab[s], dev_tab[s] = c["table_out"], gtabs[s].copy()
            nxt = c["flag_out"]
            if not is_error(r) and r >= 2 and nxt == 0:
                nxt = 1                                                     # a new table was written: check it next time
            st_flag[s] = dev_flag[s] = nxt
    return produced


def gpu_decompress(four, blobs, dst_sizes, hdrs, expect=None):
    """blobs: compressed inputs (the first len(dst_sizes) are decoded); hdrs[b] = None (own header) or (blob index, size) --
    headers point into the same buffer.
    Returns the results and the destination regions; checks the canaries."""
    srcs, dsts = Arena(), Arena()
    for i, b in enumerate(blobs):
        srcs.add(b, skew=i % 2)
    for i, n in enumerate(dst_sizes):
        fill = np.full(n, 0x5A, np.uint8)
        if expect is not None and expect[i] is not None:
            fill[:len(expect[i])] = ~expect[i]
        dsts.add(fill, skew=(3 * i) % 5)
    srcs.upload(); dsts.upload()
    nb = len(dst_sizes)
    cp = _i64([srcs.ptr(i) for i in range(nb)]); csz = _i64([len(blobs[i]) for i in range(nb)])
    dp = _i64([dsts.ptr(i) for i in range(nb)]); dsz = _i64(dst_sizes)
    hp = _i64([srcs.ptr(h[0]) if h else 0 for h in hdrs]); hs = _i64([h[1] if h else 0 for h in hdrs])
    fn = fb.huf_decompress_repeat_blocks if four else fb.huf_decompress1x_repeat_blocks
    res = fn(cp, csz, dp, dsz, hp, hs)
    torch.cuda.synchronize()
    out = dsts.dev.cpu().numpy()
    assert dsts.canaries_intact(out)
    return _u64(res), [out[o:o + len(p)] for o, p in zip(dsts.offs, dsts.parts)]


@pytest.mark.parametrize("four", [True, False], ids=["4X", "1X"])
def test_chains_match_the_reference_loop_and_decode_back(four):
    ref = _ref()
    produced = _chain(ref, four)
    assert any(h is not None for _, _, h in produced) and any(h is None for _, _, h in produced)
    # a header is the start of the block of the same batch that carried the table (so headers overlap each other and other
    # blocks' compressed bytes), sized by that block's compressed size; a table no block carried is a separate blob
    blobs = [d for _, d, _ in produced]
    hdrs = []
    for _, _, h in produced:
        if h is None:
            hdrs.append(None)
        elif h[0] == "block":
            hdrs.append((h[1], len(blobs[h[1]])))
        else:
            blobs.append(h[1])
            hdrs.append((len(blobs) - 1, len(h[1])))
    assert sum(1 for h in produced if h[2] is not None and h[2][0] == "block") > 16
    res, regions = gpu_decompress(four, blobs, [len(s) for s, _, _ in produced], hdrs, expect=[s for s, _, _ in produced])
    for b, (src, data, h) in enumerate(produced):
        assert int(res[b]) == len(src), b
        assert (regions[b] == src).all(), b
        hb = None if h is None else (produced[h[1]][1] if h[0] == "block" else h[1])
        assert int(res[b]) == ref_decode(ref, four, data, len(src), hb)[0], b


@pytest.mark.parametrize("four", [True, False], ids=["4X", "1X"])
def test_malformed_blocks_and_headers_give_the_reference_verdicts(four):
    ref = _ref()
    tabs = tables(ref)
    hdr = table_header(ref, tabs["same"])
    src = probagen(32768, 0.14)
    fn = ref.HUF_compress4X_usingCTable if four else ref.HUF_compress1X_usingCTable
    pay = np.zeros(40000, np.uint8)
    pay = pay[:fn(ptr(pay), len(pay), ptr(src), len(src), ptr(tabs["same"]))].copy()   # a header-less block
    own = ref_repeat(ref, four, src, bound(len(src)), 255, 11, np.zeros(256, np.uint32), 0, 0)[1]   # a block with its header
    own_h = int(ref.HUF_readDTableX1(ptr(np.array([11 * 0x01000001] + [0] * 4096, np.uint32)), ptr(own), len(own)))
    flip = pay.copy(); flip[len(flip) // 2] ^= 0x10
    flip_own = own.copy(); flip_own[own_h + 100] ^= 0x04
    bad_hdr = hdr.copy(); bad_hdr[0] = 255
    bad_hdr2 = hdr.copy(); bad_hdr2[len(hdr) // 2] ^= 0xFF
    cases = [   # (blob, dstSize, header blob or None, header size)
        (pay, 32768, hdr, len(hdr)), (own, 32768, None, 0),
        (pay[:-1], 32768, hdr, len(hdr)), (pay[:len(pay) // 2], 32768, hdr, len(hdr)), (flip, 32768, hdr, len(hdr)),
        (own[:-1], 32768, None, 0), (own[:own_h + 5], 32768, None, 0), (flip_own, 32768, None, 0), (own[:own_h], 32768, None, 0),
        (pay, 32768, bad_hdr, len(bad_hdr)), (pay, 32768, bad_hdr2, len(bad_hdr2)), (pay, 32768, hdr, 1), (pay, 32768, hdr, 5),
        (pay, 32768, hdr, len(hdr) - 1), (pay, 32768, own, len(own)), (pay, 32768, own, own_h),
        (pay[:9], 32768, hdr, len(hdr)), (pay[:5], 32768, hdr, len(hdr)), (pay[:1], 32768, hdr, len(hdr)),
        (pay[:0], 32768, hdr, len(hdr)), (own[:9], 32768, None, 0),
        (pay, 32767, hdr, len(hdr)), (pay, 32769, hdr, len(hdr)), (pay, 0, hdr, len(hdr)), (own, 0, None, 0),
    ]
    if not four:
        cases += [(pay, 5, hdr, len(hdr)), (own, 5, None, 0)]
    # a compressed size no decode can consume exactly (the last stream longer than 2^20 bytes), last byte set or 0
    rng = np.random.default_rng(3)
    for base, h, hsz in ((pay, hdr, len(hdr)), (own, None, 0)):
        tail = rng.integers(1, 256, (3 << 20) // 2, dtype=np.uint8)
        long_ = np.concatenate([base, tail])
        cases.append((long_, 32768, h, hsz))
        zero_end = long_.copy(); zero_end[-1] = 0
        cases.append((zero_end, 32768, h, hsz))
    blobs, hdrs = [c[0] for c in cases], []
    for c in cases:
        if c[2] is None:
            hdrs.append(None)
        else:
            blobs.append(c[2])
            hdrs.append((len(blobs) - 1, c[3]))
    nb = len(cases)
    res, regions = gpu_decompress(four, blobs, [c[1] for c in cases], hdrs)
    for b, (blob, n, h, hs) in enumerate(cases):
        want, data = ref_decode(ref, four, blob, n, None if h is None else h[:hs])
        assert int(res[b]) == want, (b, int(res[b]), want)
        if not is_error(want):
            assert (regions[b] == data).all(), b                           # a flipped payload bit may still decode
    # documented deviations: dstSize above 128 KB, and a 4X dstSize below 6
    dev_cases = [(pay, BIG + 1, "srcSize_wrong"), (own, BIG + 1, "srcSize_wrong")]
    if four:
        dev_cases += [(pay, 5, "corruption_detected")]
    res, _ = gpu_decompress(four, [c[0] for c in dev_cases] + [hdr], [c[1] for c in dev_cases],
                            [(len(dev_cases), len(hdr)) if c[0] is pay else None for c in dev_cases])
    for b, (_, _, name) in enumerate(dev_cases):
        assert int(res[b]) == ERR[name], b


def test_one_gib_batch_block_by_block():
    ref = _ref()
    tabs = tables(ref)
    n, blk = 1 << 30, 32768
    nb = n // blk
    data = probagen(n, 0.14)
    src_dev = torch.from_numpy(data).cuda()
    cap = bound(blk)
    dst_dev = torch.zeros(nb * cap, dtype=torch.uint8, device="cuda")
    tab_dev = torch.from_numpy(np.tile(tabs["same"], nb).view(np.int32)).cuda()
    flags = np.array([(b % 3) for b in range(nb)], np.int32)
    prefer = np.array([(b // 3) % 2 for b in range(nb)], np.int32)
    base = src_dev.data_ptr()
    sp = torch.arange(nb, dtype=torch.int64, device="cuda") * blk + base
    ss = torch.full((nb,), blk, dtype=torch.int64, device="cuda")
    dp = torch.arange(nb, dtype=torch.int64, device="cuda") * cap + dst_dev.data_ptr()
    dc = torch.full((nb,), cap, dtype=torch.int64, device="cuda")
    tp = torch.arange(nb, dtype=torch.int64, device="cuda") * 1024 + tab_dev.data_ptr()
    fl = torch.from_numpy(flags).cuda(); pr = torch.from_numpy(prefer).cuda()
    cs = _u64(fb.huf_compress_repeat_blocks(sp, ss, dp, dc, tp, fl, pr, max_symbol_value=255, table_log=11))
    out = dst_dev.cpu().numpy()
    fl_out = fl.cpu().numpy()
    tab_out = tab_dev.cpu().numpy().view(np.uint32).reshape(nb, 256)
    hdr_blob = table_header(ref, tabs["same"])
    for b in range(nb):
        r, d, f, t = ref_repeat(ref, True, data[b * blk:(b + 1) * blk], cap, 255, 11, tabs["same"], int(flags[b]), int(prefer[b]))
        assert int(cs[b]) == r % (1 << 64), b
        assert (out[b * cap:b * cap + len(d)] == d).all(), b
        assert int(fl_out[b]) == f, b
        assert (tab_out[b] == (t & 0x00FFFFFF)).all(), b
    # decode every block: own headers where the block carries one, the table's header otherwise
    hdr_dev = torch.from_numpy(np.concatenate([hdr_blob, np.zeros(64, np.uint8)])).cuda()
    carries = (fl_out == 0)
    hp = torch.from_numpy(np.where(carries, 0, hdr_dev.data_ptr()).astype(np.int64)).cuda()
    hs = torch.from_numpy(np.where(carries, 0, len(hdr_blob)).astype(np.int64)).cuda()
    back = torch.empty(n, dtype=torch.uint8, device="cuda")
    bp = torch.arange(nb, dtype=torch.int64, device="cuda") * blk + back.data_ptr()
    csz = torch.from_numpy(cs.view(np.int64)).cuda()
    res = _u64(fb.huf_decompress_repeat_blocks(dp, csz, bp, ss, hp, hs))
    assert (cs >= 2).all()
    assert (res == blk).all()
    assert torch.equal(back, src_dev)
