"""The literal-policy Huff0 chain compress on host buffers (FSEB200_compress_host_literals_chains_packed) on the GPU (-m gpu), against
the device call on the same chains (FSEB200_HUF_compress_literals_chains_packed): values, kinds, form flags, offsets, the whole
output capacity byte for byte, every table word, flag and chain header; the round trip through
FSEB200_decompress_host_mixed_repeat_packed with the forms the call wrote.  Pinned and pageable buffers at odd offsets, and a
capacity that ends mid-batch.

Run as a script (`python tests/test_gpu_host_literals_chains.py --child`) it repeats the comparison under the environment it was
started with: test_chunk_budgets starts it with small FSEB200_HOST_PACKED_CHUNK_BYTES budgets, where a chain crosses a chunk
boundary right after a block whose step the policy rolled back."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import torch                                                                       # noqa: E402

from huf_chain_packed_cases import at_bound, resolve_headers                       # noqa: E402
from huf_literals_chain_cases import literal_chains, built_chains, long_literal_chain   # noqa: E402
from huf_chain_harness import (PackedChains, literals, compare_compress, regenerable, host_buffer, _sources,  # noqa: E402
                               _first_blocks, _ref, BLOCK_OVERHEAD, CANARY, FILL)
import finitestateentropy_b200 as fb                                               # noqa: E402

pytestmark = pytest.mark.gpu


def _chains(ref, step=9):
    return literal_chains(ref, 255, 11)[::step] + built_chains(ref) + at_bound([long_literal_chain(ref, 96)])


def host_round_trip(run, out, offs, kinds, forms, pinned=False, off=3):
    """FSEB200_decompress_host_mixed_repeat_packed with the written forms: every regenerable block comes back"""
    srcs = _sources(run)
    sizes = [len(s) for s in srcs]
    total = int(offs[-1])
    _, inp = host_buffer(total, pinned, off + 4)
    inp.copy_(torch.from_numpy(out.numpy()[:total].copy()))
    hblobs = [np.ascontiguousarray(b, np.uint8) for b, _ in run.hdr_blobs]
    hp = torch.tensor([b.ctypes.data for b in hblobs], dtype=torch.int64)
    hs = torch.tensor([len(b) for b in hblobs], dtype=torch.int64)
    darena, dst = host_buffer(sum(sizes), pinned, off, fill=FILL)
    _, res = fb.host_decompress_mixed_repeat_packed(inp, torch.from_numpy(offs.view(np.int64).copy()), torch.from_numpy(kinds.copy()),
                                                    torch.from_numpy(forms.copy()), run.starts, sizes, hp, hs, out=dst)
    r = res.numpy().view(np.uint64)
    d = darena.numpy()
    assert (d[:CANARY + off] == FILL).all() and (d[CANARY + off + sum(sizes):] == FILL).all(), "sentinels around hDst"
    heads = resolve_headers(kinds, run.starts)
    start, n_ok = 0, 0
    for k, s in enumerate(srcs):
        if regenerable(run, k, heads) and int(r[k]) == len(s):
            assert np.array_equal(d[CANARY + off + start: CANARY + off + start + len(s)], s), k
            n_ok += 1
        start += len(s)
    return n_ok


@pytest.mark.parametrize("pinned", [True, False], ids=["pinned", "pageable"])
def test_matches_the_device_call(pinned):
    ref = _ref()
    run = PackedChains(literals(*((64, 6) if pinned else (8, 8))), ref, _chains(ref, 5 if pinned else 7), 255 if pinned else 200,
                       11)
    total = sum(len(s) for s in _sources(run))
    out, offs, cs, kinds, forms = compare_compress(run, total + 32, pinned=pinned, off=1 if pinned else 5)
    assert list(kinds) == run.kinds and list(forms) == run.flags
    assert host_round_trip(run, out, offs, kinds, forms, pinned=not pinned) > 100
    compare_compress(run, int(offs[len(offs) // 2]) - 1, pinned=not pinned, off=3)   # a capacity that ends mid-batch


def _rolled_back_crossings(run, budget):
    """chunk boundaries (compress cuts) that fall right after a block the policy stored raw or RLE after an attempt, inside its
    chain, with a later block of that chain coded"""
    srcs = _sources(run)
    firsts = _first_blocks([len(s) + BLOCK_OVERHEAD for s in srcs], budget)
    seen = 0
    for b0 in firsts[1:]:
        c, i = run.blocks[b0]
        if i > 0 and run.kinds[b0 - 1] in (0, 1) and len(srcs[b0 - 1]) >= run.form.kw["min_literals"] and run.kinds[b0] in (2, 3):
            seen += 1
    return seen


def test_chunk_budgets():
    """in child processes at small FSEB200_HOST_PACKED_CHUNK_BYTES budgets: chains cross chunks, and a chunk opens right after a
    rolled-back block of its chain"""
    _ref()
    seen = 0
    for budget in (3 * (32768 + 512), 40000, 70001):
        env = dict(os.environ, FSEB200_HOST_PACKED_CHUNK_BYTES=str(budget))
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child"], env=env, capture_output=True, text=True, timeout=1800)
        assert r.returncode == 0 and "child ok" in r.stdout, (budget, r.stdout[-2000:], r.stderr[-4000:])
        seen += json.loads(r.stdout.split("child ok", 1)[1])
    assert seen, "no chunk opens right after a rolled-back block"


def _child():
    ref = _ref()
    budget = int(os.environ["FSEB200_HOST_PACKED_CHUNK_BYTES"])
    run = PackedChains(literals(8, 8), ref, _chains(ref, 11), 255, 11)
    total = sum(len(s) for s in _sources(run))
    out, offs, cs, kinds, forms = compare_compress(run, total + 32, pinned=True, off=1)
    host_round_trip(run, out, offs, kinds, forms, pinned=False, off=5)
    print("child ok" + json.dumps(_rolled_back_crossings(run, budget)))


if __name__ == "__main__" and "--child" in sys.argv:
    _child()
