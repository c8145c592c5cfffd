"""Inputs and the reference loop of the mixed-form Huff0 chain tests (FSEB200_HUF_compress_mixed_repeat_chains[_packed],
FSEB200_HUF_decompress_mixed_repeat_{blocks,packed}): chains whose blocks each choose one stream or four, and the loop those calls
must equal -- per chain, block b coded by HUF_compress4X_repeat when its flag is 0 and by HUF_compress1X_repeat otherwise, the
stream's (table, flag, header) carried from block to block whatever the form.

The chains are the chain tests' chains (huf_chain_cases.py) under six flag patterns, ragged literal-like chains of 1-1,024-byte
sections between 32 KB blocks, and a few built chains for the inputs where a kernel that ignored the flag, or used the wrong form,
would give different bytes.  test_huf_mixed_chains_abi.py checks these claims against the compiled reference;
test_gpu_huf_mixed_chains.py runs them through the library."""
import numpy as np

from helpers import probagen, is_error
from huf_repeat_cases import ref_repeat, ref_table, table_header, blocks, bound
from huf_chain_cases import mid_chains, drift_chains, long_chain
from huf_chain_packed_cases import at_bound

PATTERNS = ("all0", "all1", "alt", "every3", "size", "random")


def pattern_flags(name, sizes, seed=0):
    """per-block singleStream flags of a pattern: all 4X, all 1X, alternating, every third 1X, zstd's size rule (one stream below
    256 bytes), or seeded random bytes (any non-zero value means 1X)"""
    n = len(sizes)
    if name == "all0":
        return [0] * n
    if name == "all1":
        return [1] * n
    if name == "alt":
        return [i % 2 for i in range(n)]
    if name == "every3":
        return [int(i % 3 == 0) for i in range(n)]
    if name == "size":
        return [int(s < 256) for s in sizes]
    rng = np.random.default_rng(1000 + seed)
    return [int(v) for v in rng.choice([0, 0, 1, 7, 255], n)]


def with_flags(chains, name, seed=0):
    """the chains with every block's `single` flag set by pattern `name` over the call's blocks in order"""
    sizes = [len(b["src"]) for ch in chains for b in ch["blocks"]]
    flags = iter(pattern_flags(name, sizes, seed))
    return [dict(ch, name="%s/%s" % (ch["name"], name), blocks=[dict(b, single=next(flags)) for b in ch["blocks"]]) for ch in chains]


def ref_mixed_chain(ref, chain, msv, tlog):
    """ref_chain (huf_chain_cases.py) with block b in the form its flag names: [(r, bytes, header)] and the final (table, flag,
    header); a header is None, ("chain",) or ("block", i)"""
    T, F, H = chain["table"].copy(), chain["flag"], ("chain",)
    out = []
    for i, blk in enumerate(chain["blocks"]):
        r, data, F, T = ref_repeat(ref, blk["single"] == 0, blk["src"], blk["cap"], msv, tlog, T, F, blk["prefer"])
        coded = not is_error(r) and r >= 2
        out.append((r, data, H if coded and F != 0 else None))
        if coded and F == 0:
            F, H = 1, ("block", i)
    return out, (T, F, H)


def _blk(src, single, prefer=0, cap=None):
    return dict(src=np.asarray(src, np.uint8), cap=bound(len(src)) if cap is None else cap, prefer=prefer, single=single)


def ragged_chains(seed=0, n_chains=3, n_big=6):
    """literal-like streams: 32 KB P14 blocks with runs of 1-1,024-byte sections of P14 / P40 / random / RLE bytes between them,
    prefer on every other section, flags unset (with_flags sets them)"""
    rng = np.random.default_rng(seed)
    p14, p40 = probagen(1 << 20, 0.14), probagen(1 << 18, 0.40)
    out = []
    for c in range(n_chains):
        blks = []
        for k in range(n_big):
            o = int(rng.integers(0, len(p14) - 32768))
            blks.append(dict(src=p14[o:o + 32768].copy(), prefer=k % 2))
            for j in range(int(rng.integers(1, 5))):
                n = int(rng.integers(1, 1025))
                kind = int(rng.integers(0, 4))
                if kind == 0:
                    o = int(rng.integers(0, len(p14) - n)); src = p14[o:o + n].copy()
                elif kind == 1:
                    o = int(rng.integers(0, len(p40) - n)); src = p40[o:o + n].copy()
                elif kind == 2:
                    src = rng.integers(0, 256, n, dtype=np.uint8)
                else:
                    src = np.full(n, int(rng.integers(0, 256)), np.uint8)
                blks.append(dict(src=src, prefer=(j + k) % 2))
        for b in blks:
            b["cap"] = bound(len(b["src"]))
        out.append(dict(table=np.zeros(256, np.uint32), flag=0, blocks=blks, name="ragged%d" % c))
    return out


def built_chains(ref):
    """chains built for the inputs where the form changes the bytes (see form_counts)"""
    b = dict(blocks())
    p14 = probagen(1 << 18, 0.14)
    same = ref_table(ref, probagen(65536, 0.14))
    top = np.argsort(-np.bincount(p14[:65536], minlength=256), kind="stable")[:2].astype(np.uint8)
    out = [
        # a 4X block saves a table, then 1X old-table blocks read its header; and the reverse
        dict(table=np.zeros(256, np.uint32), flag=0, name="x4_then_x1",
             blocks=[_blk(b["p14_32768"], 0), _blk(b["p14_4099"], 1, prefer=1), _blk(p14[5000:5700], 1, prefer=1)]),
        dict(table=np.zeros(256, np.uint32), flag=0, name="x1_then_x4",
             blocks=[_blk(b["p14_32768"], 1), _blk(b["p14_4099"], 0, prefer=1), _blk(p14[9000:41768], 0, prefer=1)]),
        # a valid table and prefer: tiny old-table blocks (4X: 0 below 12 bytes; 1X codes them, into one byte for 3 symbols)
        dict(table=same, flag=2, name="tiny_old",
             blocks=[_blk(p14[100:108], 1, prefer=1), _blk(p14[200:208], 0, prefer=1), _blk([top[0], top[1], top[0]], 1, prefer=1),
                     _blk([top[0]] * 3, 1, prefer=1), _blk([top[1], top[0]], 1, prefer=1), _blk([top[0], top[0], top[1], top[0]], 1, prefer=1),
                     _blk(p14[300:311], 1, prefer=1), _blk([top[0], top[1], top[0]], 0, prefer=1)]),
    ]
    # a new table saved by a block whose value is 0 in its form (and not in the other), then a block that reads that state
    for n in (24, 32, 40, 48, 64, 80, 96, 128):
        for form in (0, 1):
            for o in range(0, 4000, 97):
                src = p14[o:o + n]
                r, _, F, T = ref_repeat(ref, form == 0, src, bound(n), 255, 11, np.zeros(256, np.uint32), 0, 0)
                if r != 0 or not T.any():
                    continue
                r2, _, _, _ = ref_repeat(ref, form != 0, src, bound(n), 255, 11, np.zeros(256, np.uint32), 0, 0)
                if r2 >= 2:
                    out.append(dict(table=np.zeros(256, np.uint32), flag=0, name="saved_zero_x%d_%d" % (1 if form else 4, n),
                                    blocks=[_blk(src, form), _blk(b["p14_4099"], 1 - form, prefer=1), _blk(b["p14_32768"], form)]))
                    break
            if len(out) > 5:
                break
        if len(out) > 5:
            break
    return out


def mixed_chains(ref, msv, tlog, patterns=PATTERNS):
    """the GPU test's chains: the chain tests' mid-chain and drifting chains at HUF_compressBound under every pattern, the ragged
    chains under every pattern, and the built chains as they are"""
    out = []
    for i, p in enumerate(patterns):
        base = at_bound(mid_chains(ref, i % 2 == 0, msv, tlog) + drift_chains(ref)) + ragged_chains(seed=i)
        out += with_flags(base, p, seed=i)
    return out + built_chains(ref)


def long_mixed_chain(ref, nblocks=4096):
    """one chain of nblocks 32 KB P14 blocks with alternating flags"""
    ch = long_chain(ref, nblocks)
    return dict(ch, blocks=[dict(b, single=i % 2) for i, b in enumerate(ch["blocks"])], name="long_alt")


def expected_mixed(want, chains):
    """per block in call order: (value, kind, stored bytes, flag), and the chain starts (huf_chain_packed_cases.expected)"""
    from huf_chain_packed_cases import kind_of, stored
    vals, kinds, blobs, flags, starts = [], [], [], [], [0]
    for (per, _), ch in zip(want, chains):
        for (r, data, h), blk in zip(per, ch["blocks"]):
            vals.append(r % (1 << 64))
            kinds.append(kind_of(r, h))
            blobs.append(stored(r, data, blk["src"]))
            flags.append(blk["single"])
        starts.append(len(vals))
    return vals, kinds, blobs, flags, starts


def form_counts(ref, chains, want, msv, tlog):
    """how often the chains reach each input where a flag-blind or wrong-form coder gives different bytes"""
    seen = dict(x1_reads_x4=0, x4_reads_x1=0, old_tiny_1x=0, old_one_byte_1x=0, saved_zero_then_more=0)
    for ch, (per, _) in zip(chains, want):
        T, F = ch["table"].copy(), ch["flag"]
        blks = ch["blocks"]
        for i, ((r, data, h), blk) in enumerate(zip(per, blks)):
            one = blk["single"] != 0
            n = len(blk["src"])
            if h is not None and h[0] == "block":
                src_form = blks[h[1]]["single"] != 0
                if one and not src_form:
                    seen["x1_reads_x4"] += 1
                if src_form and not one:
                    seen["x4_reads_x1"] += 1
            if one and h is not None and 2 <= n < 12:
                seen["old_tiny_1x"] += 1
            if one and r == 1 and not (blk["src"] == data[0]).all():
                seen["old_one_byte_1x"] += 1
            r_, _, F2, T2 = ref_repeat(ref, not one, blk["src"], blk["cap"], msv, tlog, T, F, blk["prefer"])
            assert r_ == r
            if r == 0 and F2 == 0 and (T2 != T).any() and i + 1 < len(blks):
                other, _, _, _ = ref_repeat(ref, one, blk["src"], blk["cap"], msv, tlog, T, F, blk["prefer"])
                if other != r:
                    seen["saved_zero_then_more"] += 1
            T, F = T2, F2
            if not is_error(r) and r >= 2 and F == 0:
                F = 1
    return seen
