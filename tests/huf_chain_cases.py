"""Inputs of the Huff0 chain tests (FSEB200_HUF_compress{4X,1X}_repeat_chains) and the reference loop they must equal: per chain,
HUF_compress{4X,1X}_repeat block after block with the stream's (table, flag, header) carried as include/fse_b200.h states it.
test_huf_repeat_chains_abi.py restates the decision order on these chains and checks that mid-chain blocks reach every outcome;
test_gpu_huf_repeat_chains.py runs them through the library."""
import numpy as np

from helpers import probagen, is_error
from huf_repeat_cases import blocks, tables, table_header, ref_repeat, main_cases, bound, FLAGS

PREFIX = "rle_4099"          # a block whose verdict (RLE, or the old table under prefer + valid) leaves the state as it is


def ref_chain(ref, four, chain, msv, tlog):
    """the reference loop over one chain: chain = dict(table, flag, blocks=[dict(src, cap, prefer)]).  Returns the per-block
    results [(r, bytes, header)] and the final (table, flag, header); a header is None, ("chain",) (the chain's incoming one) or
    ("block", i) (block i of this chain, r_i bytes)."""
    T, F, H = chain["table"].copy(), chain["flag"], ("chain",)
    out = []
    for i, blk in enumerate(chain["blocks"]):
        r, data, F, T = ref_repeat(ref, four, blk["src"], blk["cap"], msv, tlog, T, F, blk["prefer"])
        coded = not is_error(r) and r >= 2
        out.append((r, data, H if coded and F != 0 else None))
        if coded and F == 0:
            F, H = 1, ("block", i)
    return out, (T, F, H)


def _blk(src, prefer=0, cap=None):
    return dict(src=src, cap=bound(len(src)) if cap is None else cap, prefer=prefer)


def single_chains(ref, four, msv, tlog):
    """every input of the single-block table-reuse tests as a chain of one block"""
    return [dict(table=c["table"], flag=c["flag"], blocks=[_blk(c["src"], c["prefer"], c["cap"])], name="one:%s/%s/%s/f%d/p%d" % (
        c["bname"], c["tname"], c["kind"], c["flag"], c["prefer"])) for c in main_cases(ref, four, msv, tlog)]


def mid_chains(ref, four, msv, tlog):
    """the same inputs in the middle of a chain: a block that leaves the state alone, the input, then a 32 KB P14 block whose
    decision reads the state the input left"""
    pre = dict(blocks())[PREFIX]
    follow = dict(blocks())["p14_32768"]
    return [dict(table=c["table"], flag=c["flag"], name="mid:" + c["name"][4:],
                 blocks=[_blk(pre), c["blocks"][0], _blk(follow, prefer=i % 2)])
            for i, c in enumerate(single_chains(ref, four, msv, tlog))]


def drift_chains(ref):
    """chains whose distribution drifts (P14 -> P40 -> random -> RLE -> P14), for every incoming flag, four prefer patterns and
    three tables, with a capacity under a block's size, an empty block and one above 128 KB along the way"""
    b = dict(blocks())
    tabs = tables(ref)
    seq = ["p14_32768", "p14_32768", "p40_32768", "p40_32768", "rand_32768", "rle_32768", "p14_32768", "p14_4099", "high_32768",
           "p14_0", "p14_131073", "p14_32768", "wide_40", "p14_32768"]
    pats = {"none": lambda i: 0, "all": lambda i: 1, "odd": lambda i: i % 2, "every3": lambda i: int(i % 3 == 0)}
    out = []
    for flag in FLAGS:
        for pname, pat in pats.items():
            for tname in ("same", "other", "zero"):
                blks = [_blk(b[name], pat(i), 3000 if i == 8 else None) for i, name in enumerate(seq)]
                out.append(dict(table=tabs[tname], flag=flag, blocks=blks, name="drift:%s/f%d/%s" % (tname, flag, pname)))
    return out


def empty_chains(n):
    return [dict(table=np.zeros(256, np.uint32), flag=f, blocks=[], name="empty") for f in (0, 2)][:n]


def long_chain(ref, nblocks=4096, blk=32768):
    """one chain of nblocks x 32 KB P14 blocks (prefer every fifth block), starting with no table"""
    data = probagen(nblocks * blk, 0.14)
    return dict(table=np.zeros(256, np.uint32), flag=0, name="long",
                blocks=[_blk(data[i * blk:(i + 1) * blk], int(i % 5 == 4)) for i in range(nblocks)])


def chain_header(ref, chain):
    """the incoming header a chain is given: its table's HUF_writeCTable bytes where the table has one, else a stand-in (the
    compressor only passes it on)"""
    t = chain["table"]
    nb = (t >> 16) & 0xFF
    try:
        if nb.any() and nb.max() <= 11:
            return table_header(ref, t), True
    except AssertionError:
        pass
    return np.arange(40, dtype=np.uint8), False
