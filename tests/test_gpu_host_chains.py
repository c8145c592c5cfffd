"""Packed Huff0 chains on host buffers (FSEB200_compress_host_repeat_chains_packed / FSEB200_decompress_host_repeat_packed) on the
GPU (-m gpu), 4X and 1X, against the device calls on the same chains (FSEB200_HUF_compress{4X,1X}_repeat_chains_packed,
FSEB200_HUF_decompress{4X,1X}_repeat_packed): values, kinds, offsets, the whole output capacity byte for byte (both buffers
poisoned alike), every table word, flag and chain header; the decompress results equal to the device decoder's for the same stream
and entry headers, and every block the reference loop says decodes regenerated from the host stream alone.  Also capacities 0,
one byte short of a block's end and the exact total; entry flags none / check / valid; entry headers above 128 bytes and of size 0;
pinned and pageable buffers at odd offsets; two host threads at once.

Run as a script (`python tests/test_gpu_host_chains.py --child`) it repeats the comparisons under the environment it was started
with: test_chunk_budgets starts it with small FSEB200_HOST_PACKED_CHUNK_BYTES budgets, where chains span two and many chunks, a
chunk boundary falls right after a kind-2 block, and chunks open with kind-3 blocks whose header lies chunks back."""
import json
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import torch                                                                       # noqa: E402

from test_gpu_blocks import CANARY                                                 # noqa: E402
from huf_chain_cases import drift_chains, long_chain, empty_chains                 # noqa: E402
from huf_chain_packed_cases import at_bound, packed_chains, resolve_headers        # noqa: E402
from test_gpu_huf_repeat import Arena                                              # noqa: E402
from test_gpu_huf_repeat_packed import Packed, decode, regenerable, _t, _ref, FILL  # noqa: E402
from test_gpu_host_packed import host_buffer                                       # noqa: E402
import finitestateentropy_b200 as fb                                               # noqa: E402

pytestmark = pytest.mark.gpu
CODEC = {True: "huf", False: "huf1x"}
BLOCK_OVERHEAD = 512                                                                # what a block adds to a chunk's weight


def _sources(run):
    return [run.chains[c]["blocks"][i]["src"] for c, i in run.blocks]


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
    """the host call on the run's chains, sources and output at host offsets `off` + 2 and `off`: (out arena, out view, offsets,
    values, kinds, state)"""
    srcs = _sources(run)
    data = np.concatenate(srcs + [np.zeros(0, np.uint8)])
    _, src = host_buffer(len(data), pinned, off + 2)
    src.copy_(torch.from_numpy(data))
    oarena, out = host_buffer(cap, pinned, off, fill=FILL)
    st = HostState(run)
    prefer = torch.tensor([run.chains[c]["blocks"][i]["prefer"] for c, i in run.blocks], dtype=torch.int32)
    _, offs, cs, kinds, _ = fb.host_compress_repeat_chains_packed(src, [len(s) for s in srcs], run.starts, prefer, st.tables, st.flags,
                                                                  st.hp, st.hs, codec=CODEC[run.four], out=out,
                                                                  max_symbol_value=run.msv, table_log=run.tlog)
    assert np.array_equal(src.numpy(), data)
    return oarena, out, offs.numpy().view(np.uint64).copy(), cs.numpy().view(np.uint64).copy(), kinds.numpy().copy(), st


def compare_compress(run, cap, pinned=True, off=1):
    """the host call against the device call at capacity `cap`, both from the chains' entry state: returns the host's (out view,
    offsets, values, kinds)"""
    run.reset()
    _, dout, doff, dcs, dkinds, _ = run.call(cap=cap)
    dstate = run.state()
    oarena, out, offs, cs, kinds, st = host_compress(run, cap, pinned, off)
    assert np.array_equal(cs, dcs), [(b, int(cs[b]), int(dcs[b])) for b in range(len(cs)) if cs[b] != dcs[b]][:8]
    assert np.array_equal(kinds, dkinds)
    assert np.array_equal(offs, doff)
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
    return out, offs, cs, kinds


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
    """the host decompress of the host stream against the device decoder on the same bytes and entry headers, and every block the
    reference loop says decodes regenerated"""
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
    _, res = fb.host_decompress_repeat_packed(inp, torch.from_numpy(offs.view(np.int64).copy()), torch.from_numpy(kinds.copy()),
                                              run.starts, sizes, hp, hs, codec=CODEC[run.four], out=dst)
    r = res.numpy().view(np.uint64)
    dh = Arena()
    for b, _ in heads:
        dh.add(b, skew=1)
    dh.upload()
    dev_in = torch.from_numpy(np.concatenate([packed, np.zeros(64, np.uint8)])).cuda()
    want, _ = decode(run.four, _t(run.starts), dev_in, _t(offs), _t(kinds, torch.uint8), _t([dh.ptr(c) for c in range(len(heads))]),
                     _t([len(b) for b, _ in heads]), sizes)
    assert np.array_equal(r, want), [(b, int(r[b]), int(want[b])) for b in range(len(r)) if r[b] != want[b]][:8]
    d = darena.numpy()
    assert (d[:CANARY + off] == FILL).all() and (d[CANARY + off + sum(sizes):] == FILL).all(), "sentinels around hDst"
    # a kind-3 block decodes from its chain's entry header only if that header is a real one whose table the decoders accept:
    # the mid-chain inputs' entry tables probe the encoder's edges, and the reference's decoders reject some of them
    rh = resolve_headers(kinds, run.starts)
    stand_in = [not real or not run.chains[c]["name"].startswith(("drift", "long")) for c, (_, real) in enumerate(heads)]
    start, n_ok = 0, 0
    for k, s in enumerate(srcs):
        if regenerable(run, k, rh, lambda c: stand_in[c]):
            assert int(r[k]) == len(s) and np.array_equal(d[CANARY + off + start: CANARY + off + start + len(s)], s), k
            n_ok += 1
        start += len(s)
    return r, n_ok


# ---- tests ----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("four", [True, False], ids=["4X", "1X"])
@pytest.mark.parametrize("pinned", [True, False], ids=["pinned", "pageable"])
def test_matches_the_device_calls(four, pinned):
    ref = _ref()
    msv, tlog = (255, 11) if pinned else (200, 11)
    chains = packed_chains(ref, four, msv, tlog)[::2] + empty_chains(1) + at_bound([long_chain(ref, 300)])
    run = Packed(ref, four, chains, msv, tlog)
    out, offs, cs, kinds = compare_compress(run, sum(len(s) for s in _sources(run)) + 32, pinned=pinned, off=1 if pinned else 5)
    assert list(kinds) == run.kinds
    _, n_ok = compare_decompress(run, out, offs, kinds, pinned=pinned, off=3 if pinned else 7)
    assert n_ok > 300


@pytest.mark.parametrize("four", [True, False], ids=["4X", "1X"])
def test_capacities(four):
    """outCapacity 0, one byte short of a block's end, and the exact total: values, kinds, offsets, bytes and state as the device
    call's -- the state as it came in below the total"""
    ref = _ref()
    chains = at_bound(drift_chains(ref))[::4]
    run = Packed(ref, four, chains, 255, 12)
    _, offs, cs, kinds = compare_compress(run, sum(len(s) for s in _sources(run)) + 32)
    mid = next(b for b in range(len(offs) // 2, len(offs) - 1) if offs[b + 1] > offs[b] + 1)
    for cap in (int(offs[mid + 1]) - 1, int(offs[-1])):
        compare_compress(run, cap, pinned=cap % 2 == 0, off=3)
    # capacity 0 (a zero-length tensor has no address to give the device call): the device rule -- a block is stored only if
    # its offset plus its length is at most the capacity -- keeps only the values of the zero-length blocks at offset 0, and the
    # state as it came in
    _, out0, offs0, cs0, kinds0, st = host_compress(run, 0, False, 3)
    assert np.array_equal(offs0, offs)
    error = np.array([fb.is_error(int(v)) for v in cs])
    stored = (offs[1:] == 0) & ~error
    assert (~stored & ~error).any()
    assert [int(v) for v in cs0] == [int(cs[b]) if stored[b] or error[b] else (1 << 64) - 2 for b in range(len(cs))]
    assert np.array_equal(kinds0, np.where(stored, kinds, 4))
    fresh = HostState(run)
    assert torch.equal(st.tables, fresh.tables) and torch.equal(st.flags, fresh.flags) and torch.equal(st.hs, fresh.hs)
    assert st.hp.tolist() == st.entry


@pytest.mark.parametrize("four", [True, False], ids=["4X", "1X"])
def test_entry_flags_and_headers(four):
    """every entry flag (none, check, valid and two invalid ones) over three entry tables, the stream decoded with entry headers
    as given, longer than 128 bytes, and of size 0 (kind 3 from it: corruption_detected, as the device decoder says)"""
    ref = _ref()
    chains = at_bound(drift_chains(ref))
    assert {ch["flag"] for ch in chains} >= {0, 1, 2}
    run = Packed(ref, four, chains, 255, 11)
    out, offs, _, kinds = compare_compress(run, sum(len(s) for s in _sources(run)) + 32, pinned=False, off=1)
    r, n_ok = compare_decompress(run, out, offs, kinds, pinned=False, off=1, variants=True)
    assert n_ok > 100
    heads = resolve_headers(kinds, run.starts)
    assert any(h == ("chain", c) for h in heads for c in range(len(chains)) if c % 5 == 3), "a kind-3 block reads a size-0 header"
    assert any(h == ("chain", c) for h in heads for c in range(len(chains)) if c % 5 == 1), "a kind-3 block reads a long header"


def test_two_threads():
    """two host threads run the pair on different chains at once: both give what one thread alone gives"""
    ref = _ref()
    runs = [Packed(ref, True, at_bound(drift_chains(ref))[::3], 255, 11), Packed(ref, False, at_bound([long_chain(ref, 200)]), 255, 11)]
    alone = []
    for run in runs:
        out, offs, cs, kinds, st = host_compress(run, sum(len(s) for s in _sources(run)) + 32, True, 1)[1:]
        alone.append((out.numpy()[:int(offs[-1])].copy(), offs, cs, kinds, st.tables.clone(), st.flags.clone()))
    errors = []

    def work(i):
        try:
            run = runs[i]
            for _ in range(3):
                out, offs, cs, kinds, st = host_compress(run, sum(len(s) for s in _sources(run)) + 32, i == 0, 1 + i)[1:]
                w = alone[i]
                assert np.array_equal(offs, w[1]) and np.array_equal(cs, w[2]) and np.array_equal(kinds, w[3])
                assert np.array_equal(out.numpy()[:int(offs[-1])], w[0])
                assert torch.equal(st.tables, w[4]) and torch.equal(st.flags, w[5])
                compare_decompress(run, out, offs, kinds, pinned=i == 1, off=2)
        except BaseException as e:                                       # reported by the main thread
            errors.append(e)
    threads = [threading.Thread(target=work, args=(i,)) for i in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors


def _first_blocks(weights, budget):
    """the first block of every chunk, as the host pipeline cuts a batch of these block weights at `budget`"""
    out, w = [0], 0
    for b, x in enumerate(weights):
        if b > out[-1] and w + x > budget:
            out.append(b)
            w = 0
        w += x
    return out


def _shapes(run, offs, kinds, budget):
    """which of the chunk shapes the budget produced: a chain across two chunks and across many (compress cut); a boundary right
    after a kind-2 block and a chunk opening with a kind-3 block whose header lies chunks back (both cuts)"""
    srcs = _sources(run)
    starts = run.starts
    chain_of = np.searchsorted(np.asarray(starts[:-1]), np.arange(len(srcs)), side="right") - 1
    heads = resolve_headers(kinds, starts)
    seen = set()
    for name, weights in (("compress", [len(s) + BLOCK_OVERHEAD for s in srcs]),
                          ("decompress", [len(s) + int(offs[b + 1] - offs[b]) + BLOCK_OVERHEAD for b, s in enumerate(srcs)])):
        firsts = _first_blocks(weights, budget)
        chunk_of = np.searchsorted(np.asarray(firsts), np.arange(len(srcs)), side="right") - 1
        for c in range(len(starts) - 1):
            if starts[c + 1] > starts[c] and name == "compress":
                span = chunk_of[starts[c + 1] - 1] - chunk_of[starts[c]] + 1
                seen |= {"spans 2"} if span == 2 else {"spans many"} if span > 2 else set()
        for b0 in firsts[1:]:
            if kinds[b0 - 1] == 2 and chain_of[b0 - 1] == chain_of[b0]:
                seen.add("edge after kind 2 (%s)" % name)
            h = heads[b0]
            if h is not None and h[0] == "block" and chunk_of[h[1]] < chunk_of[b0]:
                seen.add("opens with kind 3 (%s)" % name)
    return seen


def test_chunk_budgets():
    """in child processes at small FSEB200_HOST_PACKED_CHUNK_BYTES budgets: every chunk shape _shapes names occurs"""
    _ref()
    seen = set()
    for budget in (3 * (32768 + BLOCK_OVERHEAD), 40000, 250001):
        env = dict(os.environ, FSEB200_HOST_PACKED_CHUNK_BYTES=str(budget))
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child"], env=env, capture_output=True, text=True, timeout=1800)
        assert r.returncode == 0 and "child ok" in r.stdout, (budget, r.stdout[-2000:], r.stderr[-4000:])
        seen |= set(json.loads(r.stdout.split("child ok", 1)[1]))
    want = {"spans 2", "spans many", "edge after kind 2 (compress)", "edge after kind 2 (decompress)",
            "opens with kind 3 (compress)", "opens with kind 3 (decompress)"}
    assert seen >= want, want - seen


def _child():
    ref = _ref()
    budget = int(os.environ["FSEB200_HOST_PACKED_CHUNK_BYTES"])
    seen = set()
    for four in (True, False):
        chains = at_bound(drift_chains(ref))[::6] + empty_chains(1) + at_bound([long_chain(ref, 96)])
        run = Packed(ref, four, chains, 255, 11)
        total = sum(len(s) for s in _sources(run))
        out, offs, cs, kinds = compare_compress(run, total + 32, pinned=four, off=1)
        compare_decompress(run, out, offs, kinds, pinned=not four, off=5, variants=True)
        seen |= _shapes(run, offs, kinds, budget)
        compare_compress(run, int(offs[len(offs) // 2]) - 1, pinned=True, off=3)   # a capacity that ends mid-batch
        torch.cuda.empty_cache()
    print("child ok" + json.dumps(sorted(seen)))


if __name__ == "__main__" and "--child" in sys.argv:
    _child()
