"""The harness the Huff0 table-reuse GPU tests share: device arenas with canaries and guard words, the compiled reference's
decoders, one packed-chain run for every call form (4X, 1X, mixed, the literal policy), the packed decoders, and the host-buffer
calls compared with the device calls.  A form (`PLAIN[four]`, `MIXED`, `literals(min_literals, min_gain_log)`) names the
reference loop, the wrappers and whether the per-block form flags go into the call, come out of it or are absent."""
import numpy as np
import pytest
import torch

from helpers import ptr, is_error, load_ref
from huf_repeat_cases import bound
from huf_chain_cases import ref_chain, chain_header
from huf_chain_packed_cases import expected, resolve_headers
from huf_mixed_chain_cases import ref_mixed_chain, expected_mixed
from huf_literals_chain_cases import ref_literals_chain, expected_literals
from test_gpu_blocks import CANARY                      # the sentinel bytes host_buffer puts on each side of a host view
from test_gpu_host_packed import host_buffer
import finitestateentropy_b200 as fb

ARENA_CANARY, PAD = 0xC7, 4096                          # an Arena's canary byte, and how many of them around each region
G = 8                                                   # guard words around every array
GUARD = -0x3838383838383839                             # 0xC7C7... as int64
EDGE, FILL = 64, 0xC7                                   # guard bytes around the packed buffer
SRC_WRONG, CORRUPT, TOO_SMALL = (1 << 64) - 3, (1 << 64) - 4, (1 << 64) - 2
BLOCK_OVERHEAD = 512                                    # what a block adds to a host chunk's weight


def _ref():
    ref = load_ref()
    if ref is None:
        pytest.skip("compiled reference not available")
    return ref


def _u64(t):
    return t.cpu().numpy().view(np.uint64)


def _t(vals, dtype=torch.int64):
    if dtype == torch.uint8:
        return torch.tensor(np.asarray(vals, np.uint8), dtype=torch.uint8, device="cuda")
    return torch.tensor(np.array(vals, np.uint64).view(np.int64), dtype=torch.int64, device="cuda")


def _dev(vals, dtype=torch.int64):
    a = np.array(vals, dtype=np.uint64).view(np.int64) if dtype == torch.int64 else np.array(vals, np.int32)
    t = torch.full((len(a) + 2 * G,), GUARD if dtype == torch.int64 else -0x38383839, dtype=dtype, device="cuda")
    t[G:G + len(a)] = torch.from_numpy(a).cuda()
    return t


def _view(t):
    return t[G:t.numel() - G]


def _guards_ok(t):
    v = t.cpu().numpy()
    g = GUARD if t.dtype == torch.int64 else -0x38383839
    return bool((v[:G] == g).all() and (v[-G:] == g).all())


class Arena:
    """one device byte buffer: regions at chosen misalignments, PAD canary bytes around each"""

    def __init__(self):
        self.parts, self.offs, self.size = [], [], PAD

    def add(self, data, skew=0):
        self.size += skew
        self.offs.append(self.size)
        self.parts.append(np.asarray(data, np.uint8))
        self.size += len(data) + PAD
        self.size = (self.size + 15) & ~15
        return len(self.offs) - 1

    def upload(self):
        host = np.full(self.size, ARENA_CANARY, np.uint8)
        for o, p in zip(self.offs, self.parts):
            host[o:o + len(p)] = p
        self.host = host
        self.dev = torch.from_numpy(host).cuda()
        return self

    def ptr(self, i):
        return self.dev.data_ptr() + self.offs[i]

    def canaries_intact(self, out):
        mask = np.ones(self.size, bool)
        for o, p in zip(self.offs, self.parts):
            mask[o:o + len(p)] = False
        return bool((out[mask] == ARENA_CANARY).all())


def ref_decode(ref, four, blob, n, hdr):
    dt = np.zeros(1 + 4096, np.uint32)
    dt[0] = 11 * 0x01000001                                                # HUF_CREATE_STATIC_DTABLEX1(DT, HUF_TABLELOG_MAX)
    dst = np.zeros(n + 64, np.uint8)
    src = blob if len(blob) else np.zeros(1, np.uint8)
    if hdr is None:
        fn = ref.HUF_decompress4X1_DCtx if four else ref.HUF_decompress1X1_DCtx
        return int(fn(ptr(dt), ptr(dst), n, ptr(src), len(blob))) % (1 << 64), dst[:n]
    h = ref.HUF_readDTableX1(ptr(dt), ptr(hdr), len(hdr))
    if is_error(h):
        return int(h) % (1 << 64), dst[:n]
    fn = ref.HUF_decompress4X1_usingDTable if four else ref.HUF_decompress1X1_usingDTable
    return int(fn(ptr(dst), n, ptr(src), len(blob), ptr(dt))) % (1 << 64), dst[:n]


# ---- call forms -----------------------------------------------------------------------------------------------------------

class Form:
    """one form of the packed chain calls: the reference loop `model(ref, chain, msv, tlog)` and its `expected` per-block model;
    the device compress and decompress, the pointer-form compress (`unpacked`) and the host pair; `flags`: the per-block form
    flags go "in", come "out" or are absent (None); `kw` the compress calls' extra arguments, `host_kw` the host calls';
    `kept(per, T, table)` whether a chain's final table is expected to be its entry table, unwritten"""

    def __init__(self, model, expected, compress, decompress, host_compress, host_decompress, kept, unpacked=None, flags=None,
                 four=None, kw=None, host_kw=None):
        self.model, self.expected, self.compress, self.decompress = model, expected, compress, decompress
        self.host_compress, self.host_decompress, self.kept, self.unpacked = host_compress, host_decompress, kept, unpacked
        self.flags, self.four, self.kw, self.host_kw = flags, four, kw or {}, host_kw or {}


def _same_table(per, T, table):
    return (T == table).all()


PLAIN = {four: Form(lambda ref, ch, msv, tlog, four=four: ref_chain(ref, four, ch, msv, tlog), expected,
                    fb.huf_compress_repeat_chains_packed if four else fb.huf_compress1x_repeat_chains_packed,
                    fb.huf_decompress_repeat_packed if four else fb.huf_decompress1x_repeat_packed,
                    fb.host_compress_repeat_chains_packed, fb.host_decompress_repeat_packed, _same_table,
                    unpacked=fb.huf_compress_repeat_chains if four else fb.huf_compress1x_repeat_chains, four=four,
                    host_kw=dict(codec="huf" if four else "huf1x"))
         for four in (True, False)}
MIXED = Form(ref_mixed_chain, expected_mixed, fb.huf_compress_mixed_repeat_chains_packed, fb.huf_decompress_mixed_repeat_packed,
             fb.host_compress_mixed_repeat_chains_packed, fb.host_decompress_mixed_repeat_packed, _same_table,
             unpacked=fb.huf_compress_mixed_repeat_chains, flags="in")


def literals(min_lit, min_gain_log):
    """the literal-policy form; its stream decodes with the mixed decoders and the forms the call wrote"""
    return Form(lambda ref, ch, msv, tlog: ref_literals_chain(ref, ch, msv, tlog, min_lit, min_gain_log), expected_literals,
                fb.huf_compress_literals_chains_packed, fb.huf_decompress_mixed_repeat_packed, fb.host_compress_literals_chains_packed,
                fb.host_decompress_mixed_repeat_packed, lambda per, T, table: not any(x["kind"] == 2 for x in per), flags="out",
                kw=dict(min_literals=min_lit, min_gain_log=min_gain_log))


def _flagged(head, flags, tail):
    """a call's positional arguments: the per-block form flags, when given, go between head and tail"""
    return head + ((flags,) if flags is not None else ()) + tail


class PackedChains:
    """the chains' sources, tables, entry headers and per-chain state on the device, and calls of one form's packed compress"""

    def __init__(self, form, ref, chains, msv, tlog):
        self.form, self.ref, self.four, self.chains, self.msv, self.tlog = form, ref, form.four, chains, msv, tlog
        self.want = [form.model(ref, ch, msv, tlog) for ch in chains]
        self.vals, self.kinds, self.blobs, *flags, self.starts = form.expected(self.want, chains)
        self.flags = flags[0] if flags else None
        self.blocks = [(c, i) for c, ch in enumerate(chains) for i in range(len(ch["blocks"]))]
        self.first = self.starts[:-1]
        srcs, hdrs = Arena(), Arena()
        for k, (c, i) in enumerate(self.blocks):
            srcs.add(chains[c]["blocks"][i]["src"], skew=k % 3)
        self.hdr_blobs = [chain_header(ref, ch) for ch in chains]
        for blob, _ in self.hdr_blobs:
            hdrs.add(blob)
        self.srcs, self.hdrs = srcs.upload(), hdrs.upload()
        n = len(self.blocks)
        self.sizes = [len(chains[c]["blocks"][i]["src"]) for c, i in self.blocks]
        self.sp = torch.tensor([srcs.ptr(k) for k in range(n)] or [0], dtype=torch.int64, device="cuda")[:n]
        self.ss = torch.tensor(self.sizes or [0], dtype=torch.int64, device="cuda")[:n]
        self.pr = torch.tensor([chains[c]["blocks"][i]["prefer"] for c, i in self.blocks] or [0], dtype=torch.int32, device="cuda")[:n]
        self.sg = torch.tensor(self.flags or [0], dtype=torch.uint8, device="cuda")[:n] if form.flags == "in" else None
        self.reset()

    def reset(self):
        """the per-chain state as the chains enter"""
        words = 256 + 64
        tab = np.full(64 + len(self.chains) * words, 0xC7C7C7C7, np.uint32)
        self.toff = [64 + c * words + (c % 4) for c in range(len(self.chains))]
        for o, ch in zip(self.toff, self.chains):
            tab[o:o + 256] = ch["table"]
        self.tab = torch.from_numpy(tab.view(np.int32)).cuda()
        self.ctp = _dev([self.tab.data_ptr() + 4 * o for o in self.toff])
        self.rep = _dev([ch["flag"] for ch in self.chains], torch.int32)
        self.chp = _dev([self.hdrs.ptr(c) for c in range(len(self.chains))])
        self.chs = _dev([len(b) for b, _ in self.hdr_blobs])

    def state(self):
        return dict(tabs=self.tab.cpu().numpy().view(np.uint32).copy(), rep=_view(self.rep).cpu().numpy(),
                    chp=_u64(_view(self.chp)), chs=_view(self.chs).cpu().numpy())

    def call(self, cap=None, parts=None, starts=None, stream=None, skew=3, fn=None):
        """one packed call over blocks parts[c] = (lo, hi) of each chain (all by default) into a buffer of `cap` bytes (the sum of
        the sources + 32 by default) with EDGE guard bytes around it and guards around the kinds and the forms the call writes;
        `fn`, a 4X or 1X packed compress, runs in place of the form's call on the same inputs.  Returns (buf, out view, offsets,
        csizes, kinds, [forms written,] idx)."""
        parts = parts or [(0, len(ch["blocks"])) for ch in self.chains]
        idx, st = [], [0]
        for c, (lo, hi) in enumerate(parts):
            idx += [self.first[c] + i for i in range(lo, hi)]
            st.append(len(idx))
        if starts is not None:
            st = starts
        ix = torch.tensor(idx or [0], dtype=torch.int64, device="cuda")[:len(idx)]
        if cap is None:
            cap = int(self.ss[ix].sum()) + 32
        buf = torch.full((cap + 2 * EDGE + skew,), FILL, dtype=torch.uint8, device="cuda")
        out = buf[EDGE + skew:EDGE + skew + cap]
        off, cs = _dev([0xCD] * (len(idx) + 1)), _dev([0xCD] * len(idx))
        guarded = [torch.full((len(idx) + 16,), 0xEE, dtype=torch.uint8, device="cuda")
                   for _ in range(2 if self.form.flags == "out" and fn is None else 1)]
        sv = _dev(st)
        kw = dict(self.form.kw if fn is None else {}, out=out, offsets=_view(off), csizes=_view(cs), kinds=guarded[0][8:8 + len(idx)],
                  max_symbol_value=self.msv, table_log=self.tlog)
        if len(guarded) > 1:
            kw["single_stream"] = guarded[1][8:8 + len(idx)]
        call, flags = (self.form.compress, self.sg[ix] if self.sg is not None else None) if fn is None else (fn, None)
        with torch.cuda.stream(stream or torch.cuda.current_stream()):
            call(*_flagged((_view(sv), self.sp[ix], self.ss[ix], self.pr[ix]), flags,
                           (_view(self.ctp), _view(self.rep), _view(self.chp), _view(self.chs))), **kw)
        torch.cuda.synchronize()
        for t in (off, cs, sv, self.ctp, self.rep, self.chp, self.chs):
            assert _guards_ok(t)
        got = [g.cpu().numpy() for g in guarded]
        for g in got:
            assert (g[:8] == 0xEE).all() and (g[-8:] == 0xEE).all()
        return (buf, out, _u64(_view(off)), _u64(_view(cs))) + tuple(g[8:8 + len(idx)] for g in got) + (idx,)

    def check_one_call(self, res):
        """a whole-batch call that fits: values, kinds, written forms, offsets, stored bytes, guards, and each chain's final
        table, flag and header"""
        buf, out, off, cs, kinds, *forms, idx = res
        n = len(idx)
        forms = forms[0] if forms else None
        assert n == len(self.vals)
        bad = [k for k in range(n) if int(cs[k]) != self.vals[k] or kinds[k] != self.kinds[k]
               or (forms is not None and forms[k] != self.flags[k])]
        assert not bad, [(self.chains[self.blocks[k][0]]["name"], self.blocks[k][1], int(cs[k]), self.vals[k], int(kinds[k]),
                          self.kinds[k]) + ((int(forms[k]), self.flags[k]) if forms is not None else ()) for k in bad[:6]]
        lens = [len(b) for b in self.blobs]
        assert list(off) == list(np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)), "offsets"
        host = buf.cpu().numpy()
        o0 = out.data_ptr() - buf.data_ptr()
        for k in range(n):
            assert (host[o0 + int(off[k]):o0 + int(off[k + 1])] == self.blobs[k]).all(), (k, self.blocks[k])
        assert (host[:o0] == FILL).all() and (host[o0 + int(off[n]):] == FILL).all()
        s = self.state()
        for c, ch in enumerate(self.chains):
            per, (T, F, H) = self.want[c]
            t = s["tabs"][self.toff[c]:self.toff[c] + 256]
            assert (t == (ch["table"] if self.form.kept(per, T, ch["table"]) else T & 0x00FFFFFF)).all(), ch["name"]
            assert int(s["rep"][c]) == F, ch["name"]
            if H[0] == "chain":
                hv = (self.hdrs.ptr(c), len(self.hdr_blobs[c][0]))
            else:
                k = self.first[c] + H[1]
                hv = (out.data_ptr() + int(off[k]), int(cs[k]))
            assert (int(s["chp"][c]), int(s["chs"][c])) == hv, ch["name"]
        return s

    def unpacked(self, fn=None):
        """the pointer-form chain call (the form's, or `fn`, a 4X / 1X one, on the same inputs) at capacities HUF_compressBound:
        (dst arena, csizes, hdr ptrs, hdr sizes)"""
        n = len(self.blocks)
        caps = np.array([bound(int(x)) for x in self.ss.cpu().numpy()], np.uint64)
        dst = Arena()
        for k in range(n):
            dst.add(np.zeros(int(caps[k]), np.uint8), skew=k % 5)
        dst.upload()
        dp = torch.tensor([dst.ptr(k) for k in range(n)], dtype=torch.int64, device="cuda")
        call, flags = (self.form.unpacked, self.sg) if fn is None else (fn, None)
        cs, hp, hs = call(*_flagged((_t(self.starts), self.sp, self.ss, dp, _t(caps), self.pr), flags,
                                    (_view(self.ctp), _view(self.rep), _view(self.chp), _view(self.chs))),
                          max_symbol_value=self.msv, table_log=self.tlog)
        torch.cuda.synchronize()
        return dst, _u64(cs), _u64(hp), _u64(hs)


def regenerable(run, k, heads, entry_is_stand_in=None):
    """whether block k must decode back to its source: stored (kind 0 to 3), not an RLE byte over unequal bytes (a 1X block the
    reference coded into a single byte, or the policy's n >= 8 rule: the decoders read that as RLE too), and not a kind-3 block
    whose entry header is a stand-in (its table has none; by default, a chain header that is not a real one)"""
    c, i = run.blocks[k]
    src, kind = run.chains[c]["blocks"][i]["src"], run.kinds[k]
    if kind == 4 or (kind == 1 and not (src == run.blobs[k][0]).all()):
        return False
    stand_in = entry_is_stand_in or (lambda c: not run.hdr_blobs[c][1])
    return not (heads[k] is not None and heads[k][0] == "chain" and stand_in(c))


def decode(form, starts, packed, offsets, kinds, *args, expect=None, stream=None):
    """the form's packed decoder into destinations with canaries around each; `args` are the decoder's arguments after the kinds
    -- the form flags if it takes them, the chain headers -- and the destination sizes.  Returns (results, regenerated regions)."""
    *flags_and_headers, sizes = args
    dsts = Arena()
    for i, n in enumerate(sizes):
        fill = np.full(n, 0x5A, np.uint8)
        if expect is not None and expect[i] is not None:
            fill[:len(expect[i])] = ~expect[i]
        dsts.add(fill, skew=(3 * i) % 5)
    dsts.upload()
    dp = torch.tensor([dsts.ptr(i) for i in range(len(sizes))] or [0], dtype=torch.int64, device="cuda")[:len(sizes)]
    dsz = torch.tensor(np.array(sizes, np.uint64).view(np.int64), dtype=torch.int64, device="cuda")
    res = torch.full((len(sizes) + 16,), -1, dtype=torch.int64, device="cuda")
    with torch.cuda.stream(stream or torch.cuda.current_stream()):
        form.decompress(starts, packed, offsets, kinds, *flags_and_headers, dp, dsz, results=res[8:8 + len(sizes)])
    torch.cuda.synchronize()
    r = res.cpu().numpy()
    assert (r[:8] == -1).all() and (r[-8:] == -1).all()
    host = dsts.dev.cpu().numpy()
    assert dsts.canaries_intact(host)
    return r[8:8 + len(sizes)].view(np.uint64), [host[o:o + len(p)] for o, p in zip(dsts.offs, dsts.parts)]


# ---- host buffers ---------------------------------------------------------------------------------------------------------

def _sources(run):
    return [run.chains[c]["blocks"][i]["src"] for c, i in run.blocks]


def _host_flags(run):
    """the run's per-block form flags as a CPU tensor, or None for a form without them"""
    return torch.tensor(run.flags, dtype=torch.uint8) if run.form.flags else None


class HostState:
    """the chains' entry state in host memory: tables, flags and entry headers (host copies of the device run's)"""

    def __init__(self, run):
        self.tables = torch.from_numpy(np.stack([np.asarray(ch["table"], np.uint32) for ch in run.chains]).view(np.int32).copy())
        self.flags = torch.tensor([ch["flag"] for ch in run.chains], dtype=torch.int32)
        self.blobs = [np.ascontiguousarray(b, np.uint8) for b, _ in run.hdr_blobs]
        self.entry = [b.ctypes.data for b in self.blobs]
        self.hp = torch.tensor(self.entry, dtype=torch.int64)
        self.hs = torch.tensor([len(b) for b in self.blobs], dtype=torch.int64)


def host_compress(run, cap, pinned, off):
    """the form's host call on the run's chains, sources and output at host offsets `off` + 2 and `off`: (out arena, out view,
    offsets, values, kinds, [forms written,] state)"""
    srcs = _sources(run)
    data = np.concatenate(srcs + [np.zeros(0, np.uint8)])
    _, src = host_buffer(len(data), pinned, off + 2)
    src.copy_(torch.from_numpy(data))
    oarena, out = host_buffer(cap, pinned, off, fill=FILL)
    st = HostState(run)
    prefer = torch.tensor([run.chains[c]["blocks"][i]["prefer"] for c, i in run.blocks], dtype=torch.int32)
    flags = _host_flags(run) if run.form.flags == "in" else None
    res = run.form.host_compress(*_flagged((src, [len(s) for s in srcs], run.starts, prefer), flags,
                                           (st.tables, st.flags, st.hp, st.hs)),
                                 out=out, max_symbol_value=run.msv, table_log=run.tlog, **run.form.kw, **run.form.host_kw)
    _, offs, cs, kinds, *forms, _ = res
    assert np.array_equal(src.numpy(), data)
    return ((oarena, out, offs.numpy().view(np.uint64).copy(), cs.numpy().view(np.uint64).copy(), kinds.numpy().copy())
            + tuple(f.numpy().copy() for f in forms) + (st,))


def compare_compress(run, cap, pinned=True, off=1):
    """the host call against the device call at capacity `cap`, both from the chains' entry state: returns the host's (out view,
    offsets, values, kinds, [forms written])"""
    run.reset()
    _, dout, doff, dcs, dkinds, *dforms, _ = run.call(cap=cap)
    dstate = run.state()
    oarena, out, offs, cs, kinds, *forms, st = host_compress(run, cap, pinned, off)
    assert np.array_equal(cs, dcs), [(b, int(cs[b]), int(dcs[b])) for b in range(len(cs)) if cs[b] != dcs[b]][:8]
    assert np.array_equal(kinds, dkinds)
    assert np.array_equal(offs, doff)
    for f, d in zip(forms, dforms):
        assert np.array_equal(f, d)
    assert np.array_equal(out.numpy(), dout.cpu().numpy()), cap
    o = oarena.numpy()
    assert (o[:CANARY + off] == FILL).all() and (o[CANARY + off + cap:] == FILL).all(), "sentinels around hOut"
    tabs = st.tables.numpy().view(np.uint32)
    for c in range(len(run.chains)):
        assert np.array_equal(tabs[c], dstate["tabs"][run.toff[c]:run.toff[c] + 256]), c
    assert np.array_equal(st.flags.numpy(), dstate["rep"])
    hp, hs = st.hp.numpy().view(np.uint64), st.hs.numpy().view(np.uint64)
    for c in range(len(run.chains)):
        dp = int(dstate["chp"][c])
        want = st.entry[c] if dp == run.hdrs.ptr(c) else out.data_ptr() + (dp - dout.data_ptr())
        assert (int(hp[c]), int(hs[c])) == (want, int(dstate["chs"][c])), c
    if int(offs[-1]) > cap:                                               # the state exactly as it came in
        fresh = HostState(run)
        assert torch.equal(st.tables, fresh.tables) and torch.equal(st.flags, fresh.flags)
        assert st.entry == list(hp) and torch.equal(st.hs, fresh.hs)
    return (out, offs, cs, kinds) + tuple(forms)


def entry_headers(run, variants=False):
    """per chain: (header bytes, whether its table decodes).  With variants, every fifth chain enters with its header followed by
    72 bytes of padding (above 128 bytes in all) and every fifth with a header of size 0"""
    out = []
    for c, (blob, real) in enumerate(run.hdr_blobs):
        blob = np.asarray(blob, np.uint8)
        if variants and c % 5 == 1:
            blob = np.concatenate([blob, np.arange(72 + max(0, 60 - len(blob)), dtype=np.uint8)])
            assert len(blob) > 128
        elif variants and c % 5 == 3:
            blob, real = np.zeros(0, np.uint8), False
        out.append((blob, real))
    return out


def compare_decompress(run, out, offs, kinds, pinned=True, off=3, variants=False):
    """the form's host decompress of the host stream against the device decoder on the same bytes and entry headers, and every
    block the reference loop says decodes regenerated"""
    srcs = _sources(run)
    sizes = [len(s) for s in srcs]
    total = int(offs[-1])
    packed = out.numpy()[:total].copy()
    _, inp = host_buffer(total, pinned, off + 4)
    inp.copy_(torch.from_numpy(packed))
    heads = entry_headers(run, variants)
    hblobs = [np.ascontiguousarray(b) for b, _ in heads]
    hp = torch.tensor([b.ctypes.data for b in hblobs], dtype=torch.int64)
    hs = torch.tensor([len(b) for b in hblobs], dtype=torch.int64)
    darena, dst = host_buffer(sum(sizes), pinned, off, fill=FILL)
    flags = _host_flags(run)
    _, res = run.form.host_decompress(*_flagged((inp, torch.from_numpy(offs.view(np.int64).copy()), torch.from_numpy(kinds.copy())),
                                                flags, (run.starts, sizes, hp, hs)), out=dst, **run.form.host_kw)
    r = res.numpy().view(np.uint64)
    dh = Arena()
    for b, _ in heads:
        dh.add(b, skew=1)
    dh.upload()
    dev_in = torch.from_numpy(np.concatenate([packed, np.zeros(64, np.uint8)])).cuda()
    want, _ = decode(run.form, *_flagged((_t(run.starts), dev_in, _t(offs), _t(kinds, torch.uint8)),
                                         None if flags is None else flags.cuda(),
                                         (_t([dh.ptr(c) for c in range(len(heads))]), _t([len(b) for b, _ in heads]), sizes)))
    assert np.array_equal(r, want), [(b, int(r[b]), int(want[b])) for b in range(len(r)) if r[b] != want[b]][:8]
    d = darena.numpy()
    assert (d[:CANARY + off] == FILL).all() and (d[CANARY + off + sum(sizes):] == FILL).all(), "sentinels around hDst"
    # a kind-3 block decodes from its chain's entry header only if that header is a real one whose table the decoders accept:
    # the mid-chain inputs' entry tables probe the encoder's edges, and the reference's decoders reject some of them
    rh = resolve_headers(kinds, run.starts)
    stand_in = [not real or run.chains[c]["name"].startswith("mid:") for c, (_, real) in enumerate(heads)]
    start, n_ok = 0, 0
    for k, s in enumerate(srcs):
        if regenerable(run, k, rh, lambda c: stand_in[c]):
            assert int(r[k]) == len(s) and np.array_equal(d[CANARY + off + start: CANARY + off + start + len(s)], s), k
            n_ok += 1
        start += len(s)
    return r, n_ok


def _first_blocks(weights, budget):
    """the first block of every chunk, as the host pipeline cuts a batch of these block weights at `budget`"""
    out, w = [0], 0
    for b, x in enumerate(weights):
        if b > out[-1] and w + x > budget:
            out.append(b)
            w = 0
        w += x
    return out
