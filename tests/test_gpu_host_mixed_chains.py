"""Mixed-form packed Huff0 chains on host buffers (FSEB200_compress_host_mixed_repeat_chains_packed /
FSEB200_decompress_host_mixed_repeat_packed) on the GPU (-m gpu), against the device calls on the same chains and flags
(FSEB200_HUF_compress_mixed_repeat_chains_packed, FSEB200_HUF_decompress_mixed_repeat_packed): values, kinds, offsets, the whole
output capacity byte for byte, every table word, flag and chain header; decompress results equal to the device decoder's and every
block the reference loop says decodes regenerated.  Pinned and pageable buffers at odd offsets, a capacity that ends mid-batch, two
host threads at once.

Run as a script (`python tests/test_gpu_host_mixed_chains.py --child`) it repeats the comparisons under the environment it was
started with: test_chunk_budgets starts it with small FSEB200_HOST_PACKED_CHUNK_BYTES budgets, where a chunk opens with a kind-3
block whose header is a kind-2 block of the other form in an earlier chunk."""
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
from huf_chain_cases import drift_chains                                           # noqa: E402
from huf_chain_packed_cases import at_bound, resolve_headers                       # noqa: E402
from huf_mixed_chain_cases import with_flags, ragged_chains, long_mixed_chain, built_chains   # noqa: E402
from test_gpu_huf_repeat import Arena                                              # noqa: E402
from test_gpu_huf_repeat_packed import regenerable, _t, _ref, FILL                 # noqa: E402
from test_gpu_huf_mixed_chains import Mixed, decode_mixed                          # noqa: E402
from test_gpu_host_packed import host_buffer                                       # noqa: E402
from test_gpu_host_chains import HostState, _sources, _first_blocks, BLOCK_OVERHEAD   # noqa: E402
import finitestateentropy_b200 as fb                                               # noqa: E402

pytestmark = pytest.mark.gpu


def _chains(ref, n_drift=6, seed=0):
    return (with_flags(at_bound(drift_chains(ref))[::n_drift] + ragged_chains(seed=seed, n_chains=2, n_big=4), "size")
            + built_chains(ref)[:2] + at_bound([long_mixed_chain(ref, 64)]))


def host_compress(run, cap, pinned, off):
    srcs = _sources(run)
    data = np.concatenate(srcs + [np.zeros(0, np.uint8)])
    _, src = host_buffer(len(data), pinned, off + 2)
    src.copy_(torch.from_numpy(data))
    oarena, out = host_buffer(cap, pinned, off, fill=FILL)
    st = HostState(run)
    prefer = torch.tensor([run.chains[c]["blocks"][i]["prefer"] for c, i in run.blocks], dtype=torch.int32)
    single = torch.tensor(run.flags, dtype=torch.uint8)
    _, offs, cs, kinds, _ = fb.host_compress_mixed_repeat_chains_packed(src, [len(s) for s in srcs], run.starts, prefer, single,
                                                                        st.tables, st.flags, st.hp, st.hs, out=out,
                                                                        max_symbol_value=run.msv, table_log=run.tlog)
    assert np.array_equal(src.numpy(), data)
    return oarena, out, offs.numpy().view(np.uint64).copy(), cs.numpy().view(np.uint64).copy(), kinds.numpy().copy(), st


def compare_compress(run, cap, pinned=True, off=1):
    run.reset()
    _, dout, doff, dcs, dkinds, _ = run.call(cap=cap)
    dstate = run.state()
    oarena, out, offs, cs, kinds, st = host_compress(run, cap, pinned, off)
    assert np.array_equal(cs, dcs) and np.array_equal(kinds, dkinds) and np.array_equal(offs, doff)
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
    return out, offs, cs, kinds


def compare_decompress(run, out, offs, kinds, pinned=True, off=3):
    srcs = _sources(run)
    sizes = [len(s) for s in srcs]
    total = int(offs[-1])
    packed = out.numpy()[:total].copy()
    _, inp = host_buffer(total, pinned, off + 4)
    inp.copy_(torch.from_numpy(packed))
    hblobs = [np.ascontiguousarray(b, np.uint8) for b, _ in run.hdr_blobs]
    hp = torch.tensor([b.ctypes.data for b in hblobs], dtype=torch.int64)
    hs = torch.tensor([len(b) for b in hblobs], dtype=torch.int64)
    darena, dst = host_buffer(sum(sizes), pinned, off, fill=FILL)
    single = torch.tensor(run.flags, dtype=torch.uint8)
    _, res = fb.host_decompress_mixed_repeat_packed(inp, torch.from_numpy(offs.view(np.int64).copy()), torch.from_numpy(kinds.copy()),
                                                    single, run.starts, sizes, hp, hs, out=dst)
    r = res.numpy().view(np.uint64)
    dh = Arena()
    for b in hblobs:
        dh.add(b, skew=1)
    dh.upload()
    dev_in = torch.from_numpy(np.concatenate([packed, np.zeros(64, np.uint8)])).cuda()
    want, _ = decode_mixed(_t(run.starts), dev_in, _t(offs), _t(kinds, torch.uint8), run.sg, _t([dh.ptr(c) for c in range(len(hblobs))]),
                           _t([len(b) for b in hblobs]), sizes)
    assert np.array_equal(r, want), [(b, int(r[b]), int(want[b])) for b in range(len(r)) if r[b] != want[b]][:8]
    d = darena.numpy()
    assert (d[:CANARY + off] == FILL).all() and (d[CANARY + off + sum(sizes):] == FILL).all(), "sentinels around hDst"
    rh = resolve_headers(kinds, run.starts)
    start, n_ok = 0, 0
    for k, s in enumerate(srcs):
        if regenerable(run, k, rh, lambda c: not run.hdr_blobs[c][1]):
            assert int(r[k]) == len(s) and np.array_equal(d[CANARY + off + start: CANARY + off + start + len(s)], s), k
            n_ok += 1
        start += len(s)
    return r, n_ok


@pytest.mark.parametrize("pinned", [True, False], ids=["pinned", "pageable"])
def test_matches_the_device_calls(pinned):
    ref = _ref()
    msv, tlog = (255, 11) if pinned else (200, 11)
    run = Mixed(ref, _chains(ref, 2, seed=1 if pinned else 2), msv, tlog)
    total = sum(len(s) for s in _sources(run))
    out, offs, cs, kinds = compare_compress(run, total + 32, pinned=pinned, off=1 if pinned else 5)
    assert list(kinds) == run.kinds
    _, n_ok = compare_decompress(run, out, offs, kinds, pinned=pinned, off=3 if pinned else 7)
    assert n_ok > 100
    compare_compress(run, int(offs[len(offs) // 2]) - 1, pinned=not pinned, off=3)   # a capacity that ends mid-batch


def test_two_threads():
    """two host threads run the mixed pair on different chains at once: both give what one thread alone gives"""
    ref = _ref()
    runs = [Mixed(ref, _chains(ref, 3, seed=3), 255, 11), Mixed(ref, at_bound([long_mixed_chain(ref, 200)]), 255, 11)]
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


def _cross_form_openings(run, offs, kinds, budget):
    """chunks (compress and decompress cuts) that open with a kind-3 block whose header is a kind-2 block of the other form in an
    earlier chunk"""
    srcs = _sources(run)
    heads = resolve_headers(kinds, run.starts)
    seen = set()
    for name, weights in (("compress", [len(s) + BLOCK_OVERHEAD for s in srcs]),
                          ("decompress", [len(s) + int(offs[b + 1] - offs[b]) + BLOCK_OVERHEAD for b, s in enumerate(srcs)])):
        firsts = _first_blocks(weights, budget)
        chunk_of = np.searchsorted(np.asarray(firsts), np.arange(len(srcs)), side="right") - 1
        for b0 in firsts[1:]:
            h = heads[b0]
            if h is not None and h[0] == "block" and chunk_of[h[1]] < chunk_of[b0] and (run.flags[h[1]] != 0) != (run.flags[b0] != 0):
                seen.add("opens with a kind-3 block of the other form (%s)" % name)
    return seen


def test_chunk_budgets():
    """in child processes at small FSEB200_HOST_PACKED_CHUNK_BYTES budgets: chains cross chunks, and a chunk opens with a kind-3
    block whose entry header comes from a block of the other form"""
    _ref()
    seen = set()
    for budget in (3 * (32768 + 512), 40000, 70001):
        env = dict(os.environ, FSEB200_HOST_PACKED_CHUNK_BYTES=str(budget))
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child"], env=env, capture_output=True, text=True, timeout=1800)
        assert r.returncode == 0 and "child ok" in r.stdout, (budget, r.stdout[-2000:], r.stderr[-4000:])
        seen |= set(json.loads(r.stdout.split("child ok", 1)[1]))
    want = {"opens with a kind-3 block of the other form (compress)", "opens with a kind-3 block of the other form (decompress)"}
    assert seen >= want, want - seen


def _child():
    ref = _ref()
    budget = int(os.environ["FSEB200_HOST_PACKED_CHUNK_BYTES"])
    run = Mixed(ref, _chains(ref, 6, seed=5), 255, 11)
    total = sum(len(s) for s in _sources(run))
    out, offs, cs, kinds = compare_compress(run, total + 32, pinned=True, off=1)
    compare_decompress(run, out, offs, kinds, pinned=False, off=5)
    seen = _cross_form_openings(run, offs, kinds, budget)
    print("child ok" + json.dumps(sorted(seen)))


if __name__ == "__main__" and "--child" in sys.argv:
    _child()
