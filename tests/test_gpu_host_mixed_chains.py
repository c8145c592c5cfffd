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

from huf_chain_cases import drift_chains                                           # noqa: E402
from huf_chain_packed_cases import at_bound, resolve_headers                       # noqa: E402
from huf_mixed_chain_cases import with_flags, ragged_chains, long_mixed_chain, built_chains   # noqa: E402
from huf_chain_harness import (MIXED, PackedChains, host_compress, compare_compress, compare_decompress, _sources,  # noqa: E402
                               _first_blocks, _ref, BLOCK_OVERHEAD)

pytestmark = pytest.mark.gpu


def _chains(ref, n_drift=6, seed=0):
    return (with_flags(at_bound(drift_chains(ref))[::n_drift] + ragged_chains(seed=seed, n_chains=2, n_big=4), "size")
            + built_chains(ref)[:2] + at_bound([long_mixed_chain(ref, 64)]))


@pytest.mark.parametrize("pinned", [True, False], ids=["pinned", "pageable"])
def test_matches_the_device_calls(pinned):
    ref = _ref()
    msv, tlog = (255, 11) if pinned else (200, 11)
    run = PackedChains(MIXED, ref, _chains(ref, 2, seed=1 if pinned else 2), msv, tlog)
    total = sum(len(s) for s in _sources(run))
    out, offs, cs, kinds = compare_compress(run, total + 32, pinned=pinned, off=1 if pinned else 5)
    assert list(kinds) == run.kinds
    _, n_ok = compare_decompress(run, out, offs, kinds, pinned=pinned, off=3 if pinned else 7)
    assert n_ok > 100
    compare_compress(run, int(offs[len(offs) // 2]) - 1, pinned=not pinned, off=3)   # a capacity that ends mid-batch


def test_two_threads():
    """two host threads run the mixed pair on different chains at once: both give what one thread alone gives"""
    ref = _ref()
    runs = [PackedChains(MIXED, ref, _chains(ref, 3, seed=3), 255, 11),
            PackedChains(MIXED, ref, at_bound([long_mixed_chain(ref, 200)]), 255, 11)]
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
    run = PackedChains(MIXED, ref, _chains(ref, 6, seed=5), 255, 11)
    total = sum(len(s) for s in _sources(run))
    out, offs, cs, kinds = compare_compress(run, total + 32, pinned=True, off=1)
    compare_decompress(run, out, offs, kinds, pinned=False, off=5)
    seen = _cross_form_openings(run, offs, kinds, budget)
    print("child ok" + json.dumps(sorted(seen)))


if __name__ == "__main__" and "--child" in sys.argv:
    _child()
