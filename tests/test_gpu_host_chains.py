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

from huf_chain_cases import drift_chains, long_chain, empty_chains                 # noqa: E402
from huf_chain_packed_cases import at_bound, packed_chains, resolve_headers        # noqa: E402
from huf_chain_harness import (PLAIN, PackedChains, HostState, host_compress, compare_compress, compare_decompress,  # noqa: E402
                               _sources, _first_blocks, _ref, BLOCK_OVERHEAD)
import finitestateentropy_b200 as fb                                               # noqa: E402

pytestmark = pytest.mark.gpu


# ---- tests ----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("four", [True, False], ids=["4X", "1X"])
@pytest.mark.parametrize("pinned", [True, False], ids=["pinned", "pageable"])
def test_matches_the_device_calls(four, pinned):
    ref = _ref()
    msv, tlog = (255, 11) if pinned else (200, 11)
    chains = packed_chains(ref, four, msv, tlog)[::2] + empty_chains(1) + at_bound([long_chain(ref, 300)])
    run = PackedChains(PLAIN[four], ref, chains, msv, tlog)
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
    run = PackedChains(PLAIN[four], ref, chains, 255, 12)
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
    run = PackedChains(PLAIN[four], ref, chains, 255, 11)
    out, offs, _, kinds = compare_compress(run, sum(len(s) for s in _sources(run)) + 32, pinned=False, off=1)
    r, n_ok = compare_decompress(run, out, offs, kinds, pinned=False, off=1, variants=True)
    assert n_ok > 100
    heads = resolve_headers(kinds, run.starts)
    assert any(h == ("chain", c) for h in heads for c in range(len(chains)) if c % 5 == 3), "a kind-3 block reads a size-0 header"
    assert any(h == ("chain", c) for h in heads for c in range(len(chains)) if c % 5 == 1), "a kind-3 block reads a long header"


def test_two_threads():
    """two host threads run the pair on different chains at once: both give what one thread alone gives"""
    ref = _ref()
    runs = [PackedChains(PLAIN[True], ref, at_bound(drift_chains(ref))[::3], 255, 11),
            PackedChains(PLAIN[False], ref, at_bound([long_chain(ref, 200)]), 255, 11)]
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
        run = PackedChains(PLAIN[four], ref, chains, 255, 11)
        total = sum(len(s) for s in _sources(run))
        out, offs, cs, kinds = compare_compress(run, total + 32, pinned=four, off=1)
        compare_decompress(run, out, offs, kinds, pinned=not four, off=5, variants=True)
        seen |= _shapes(run, offs, kinds, budget)
        compare_compress(run, int(offs[len(offs) // 2]) - 1, pinned=True, off=3)   # a capacity that ends mid-batch
        torch.cuda.empty_cache()
    print("child ok" + json.dumps(sorted(seen)))


if __name__ == "__main__" and "--child" in sys.argv:
    _child()
