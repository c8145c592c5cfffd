"""Inputs and models of the packed Huff0 chain tests (FSEB200_HUF_compress{4X,1X}_repeat_chains_packed and
FSEB200_HUF_decompress{4X,1X}_repeat_packed): the chain tests' chains at the packed calls' capacity HUF_compressBound, the stored
lengths and kinds the reference loop implies, and a model of the decoder's header resolution (a scan of kind-2 counts and a
search over the chain starts, as huf_packed.cu does it).  test_huf_repeat_packed_abi.py checks the model against the reference
loop; test_gpu_huf_repeat_packed.py runs the chains through the library."""
import numpy as np

from helpers import is_error
from huf_repeat_cases import bound
from huf_chain_cases import ref_chain, mid_chains, drift_chains, long_chain


def at_bound(chains):
    """the chains with every block's capacity HUF_compressBound(n), the only capacity the packed calls use"""
    return [dict(ch, blocks=[dict(b, cap=bound(len(b["src"]))) for b in ch["blocks"]]) for ch in chains]


def packed_chains(ref, four, msv, tlog, n_long=0):
    out = at_bound(mid_chains(ref, four, msv, tlog) + drift_chains(ref))
    if n_long:
        out.append(long_chain(ref, n_long))
    return out


def kind_of(r, h):
    """the kind of a block from the reference loop's value and header token"""
    if is_error(r):
        return 4
    if r < 2:
        return r
    return 2 if h is None else 3


def stored(r, data, src):
    """the bytes a block takes in the packed buffer"""
    if is_error(r):
        return np.zeros(0, np.uint8)
    return data if r else src


def expected(want, chains):
    """per block, in call order: (value, kind, stored bytes), and the chain starts"""
    vals, kinds, blobs, starts = [], [], [], [0]
    for (per, _), ch in zip(want, chains):
        for (r, data, h), blk in zip(per, ch["blocks"]):
            vals.append(r % (1 << 64))
            kinds.append(kind_of(r, h))
            blobs.append(stored(r, data, blk["src"]))
        starts.append(len(vals))
    return vals, kinds, blobs, starts


def resolve_headers(kinds, starts):
    """per block: None (not kind 3), ("chain", c) (the chain's entry header) or ("block", j) (the last kind-2 block before it in
    its chain) -- from the kinds and chain starts alone, the way the decoder derives them"""
    kinds = np.asarray(kinds)
    new = kinds == 2
    count = np.concatenate([[0], np.cumsum(new)])[:-1]                      # kind-2 blocks before each block
    pos = np.nonzero(new)[0]
    st = np.asarray(starts)
    out = []
    for b, k in enumerate(kinds):
        if k != 3:
            out.append(None)
            continue
        c = int(np.searchsorted(st[:-1], b, side="right")) - 1             # the last chain whose start is <= b
        if count[b] > count[st[c]]:
            out.append(("block", int(pos[count[b] - 1])))
        else:
            out.append(("chain", c))
    return out
