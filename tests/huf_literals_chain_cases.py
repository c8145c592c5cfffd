"""Inputs and the reference loop of the literal-policy Huff0 chain tests (FSEB200_HUF_compress_literals_chains_packed and its host
form): per chain, the rule include/fse_b200.h states -- the form from the stream's flag, the size threshold, HUF_compress{1X,4X}_repeat
on copies of the state (ref_repeat, i.e. the compiled reference), the raw / RLE / minimum-gain fallbacks, and a commit of the step's
table and flag only for a block stored with its own header.

The chains are the chain tests' mid-chain and drifting chains with entry flags 0, 1 and 2, the ragged literal-like chains of
huf_mixed_chain_cases.py, and built chains, one per rule, each of which gives other bytes or another state when its rule is left
out (see BUILT_CLAIMS).  test_huf_literals_chains_abi.py checks those claims and the round trip on the compiled reference;
test_gpu_huf_literals_chains.py and test_gpu_host_literals_chains.py run the chains through the library."""
import numpy as np

from helpers import probagen, is_error
from huf_repeat_cases import ref_repeat, ref_table, bound
from huf_chain_cases import mid_chains, drift_chains, long_chain
from huf_chain_packed_cases import at_bound
from huf_mixed_chain_cases import ragged_chains, ref_mixed_chain

SRC_WRONG = (1 << 64) - 3
HUF_BLOCK_MAX = 128 * 1024
POLICIES = ((64, 6), (8, 8), (1, 1))           # (minLiterals, minGainLog): zstd below btopt, btultra2, and the smallest


def min_gain(n, min_gain_log):
    return (n >> min_gain_log) + 2


def literal_kind(v, n, src, fs, min_gain_log):
    """the kind of an attempted block from the repeat call's value v and the step's flag after it"""
    if is_error(v) or v == 0 or v >= (n - min_gain(n, min_gain_log)) % (1 << 64):
        return 0
    if v == 1:
        return 1 if n >= 8 or (src == src[0]).all() else 0
    return 3 if fs != 0 else 2


def ref_literals_chain(ref, chain, msv, tlog, min_lit, min_gain_log):
    """the policy loop over one chain.  Returns per block dict(r, kind, single, data (the stored bytes), hdr (a kind-3 block's
    header token: ("chain",) or ("block", i)), and the final (table, flag, header)."""
    T, F, H = chain["table"].copy(), chain["flag"], ("chain",)
    out = []
    for i, blk in enumerate(chain["blocks"]):
        src = blk["src"]
        n = len(src)
        single = int(n < 256 or (F == 2 and n < 1024))
        hdr = None
        if n > HUF_BLOCK_MAX:
            r, kind, data = SRC_WRONG, 4, np.zeros(0, np.uint8)
        elif n < (6 if F == 2 else min_lit):
            r, kind, data = 0, 0, src
        else:
            r, code, fs, ts = ref_repeat(ref, not single, src, bound(n), msv, tlog, T, F, blk["prefer"])
            r %= 1 << 64
            kind = literal_kind(r, n, src, fs, min_gain_log)
            data = src if kind == 0 else src[:1] if kind == 1 else code
            if kind == 3:
                hdr = H
            if kind == 2:
                T, F, H = ts, 1, ("block", i)
        out.append(dict(r=r, kind=kind, single=single, data=data, hdr=hdr))
    return out, (T, F, H)


def expected_literals(want, chains):
    """per block in call order: values, kinds, stored bytes, forms; and the chain starts"""
    vals, kinds, blobs, flags, starts = [], [], [], [], [0]
    for per, _ in want:
        for x in per:
            vals.append(x["r"]); kinds.append(x["kind"]); blobs.append(x["data"]); flags.append(x["single"])
        starts.append(len(vals))
    return vals, kinds, blobs, flags, starts


def _blk(src, prefer=0):
    src = np.asarray(src, np.uint8)
    return dict(src=src, cap=bound(len(src)), prefer=prefer)


def _skewed(rng, n, probs):
    """n bytes drawn from symbols 0 .. len(probs) - 1 with these probabilities"""
    p = np.asarray(probs, np.float64)
    return rng.choice(len(p), n, p=p / p.sum()).astype(np.uint8)


def _find(candidates, ok):
    for c in candidates:
        if ok(c):
            return c
    raise AssertionError("no input meets the rule")


def built_chains(ref, msv=255, tlog=11):
    """chains built for one rule each, with the (minLiterals, minGainLog) at which BUILT_CLAIMS holds for them"""
    rng = np.random.default_rng(11)
    p14, p40 = probagen(1 << 18, 0.14), probagen(1 << 16, 0.40)
    same = ref_table(ref, probagen(65536, 0.14))
    follow = p14[50000:50000 + 4099]
    out = []

    # a 0 return that saved a table: the entry table is valid, the block's own table is better by the estimate, but its streams
    # do not beat n - 1; with the rollback the next block (prefer) codes with the entry table
    def saved_zero(src):
        r, _, fs, ts = ref_repeat(ref, True, src, bound(len(src)), msv, tlog, same, 1, 0)
        return r == 0 and fs == 0 and (ts != same).any()
    cands = (np.concatenate([rng.integers(0, 256, k, dtype=np.uint8), p40[o:o + n - k]])
             for n in (1024, 1500, 2000, 3000) for k in range(n // 2, n, n // 16) for o in (0, 7000))
    out.append(dict(table=same, flag=1, name="rollback_saved_zero", policy=(64, 6),
                    blocks=[_blk(_find(cands, saved_zero)), _blk(follow, prefer=1)]))

    # a failed validation (flag 1 -> 0) whose block then ends raw (hSize + 12 >= n): rolled back, the next block (prefer) keeps
    # the entry table
    lacking = ref_table(ref, p14[:30000] & 0x7F)                       # no symbol above 127
    def failed_validation(src):
        r, _, fs, ts = ref_repeat(ref, False, src, bound(len(src)), msv, tlog, lacking, 1, 0)
        return r == 0 and fs == 0 and (ts == lacking).all()
    cands = (np.concatenate([(p14[o:o + n - 4] & 0x7F), [200, 201, 202, 203]]).astype(np.uint8)
             for n in (24, 32, 40, 48, 56, 64) for o in range(0, 3000, 101))
    out.append(dict(table=lacking, flag=1, name="rollback_failed_validation", policy=(8, 8),
                    blocks=[_blk(_find(cands, failed_validation)), _blk(p14[70000:71000] & 0x7F, prefer=1)]))

    # the minimum gain: coded with its own table into fewer than n - 1 bytes, but not below n - minGain(n)
    def gain_rejected(src):
        n = len(src)
        r = ref_repeat(ref, n >= 256, src, bound(n), msv, tlog, np.zeros(256, np.uint32), 0, 0)[0]
        return not is_error(r) and 2 <= r < n - 1 and r >= n - min_gain(n, 6)
    cands = (np.concatenate([rng.integers(0, 256, k, dtype=np.uint8), p40[o:o + n - k]])
             for n in (300, 600, 1000, 2000, 4000) for k in range(n // 2, n, max(1, n // 40)) for o in (0, 3000))
    out.append(dict(table=np.zeros(256, np.uint32), flag=0, name="min_gain", policy=(64, 6),
                    blocks=[_blk(_find(cands, gain_rejected)), _blk(follow)]))

    # flag 2: the form switches at 256 and 1024 while the flag lasts (old table, prefer), then a block commits a table of its own
    # and the flag becomes 1, after which 256 .. 1023 bytes are 4X again
    out.append(dict(table=same, flag=2, name="flag2_forms", policy=(64, 6),
                    blocks=[_blk(p14[1000:1255], 1), _blk(p14[2000:2256], 1), _blk(p14[3000:4023], 1), _blk(p14[5000:6024], 1),
                            _blk(p40[:32768]), _blk(p14[7000:7300], 1), _blk(p40[40000:40600])]))

    # the size threshold: 6 bytes under flag 2 (5 not attempted, 6 coded with the old table), minLiterals under flag 0
    top = np.argsort(-np.bincount(p14[:65536], minlength=256), kind="stable")[:2].astype(np.uint8)
    sk = _skewed(rng, 64, [0.7, 0.3])
    out.append(dict(table=same, flag=2, name="threshold_6", policy=(64, 6),
                    blocks=[_blk([top[0], top[1], top[0], top[0], top[1]], 1), _blk([top[0], top[1], top[0], top[0], top[1], top[0]], 1)]))
    out.append(dict(table=np.zeros(256, np.uint32), flag=0, name="threshold_min_literals", policy=(64, 6),
                    blocks=[_blk(sk[:63]), _blk(sk)]))

    # a 1X block of 6 symbols coded with the old table into one byte (five 1-bit codes, one 2-bit code): raw, not RLE
    one_bit = ref_table(ref, _skewed(rng, 8192, [0.55, 0.25] + [0.2 / 30] * 30))
    out.append(dict(table=one_bit, flag=2, name="one_byte_1x", policy=(64, 6),
                    blocks=[_blk([0, 0, 1, 0, 0, 0], 1), _blk([0] * 7, 1)]))

    # above 128 KB: srcSize_wrong and nothing stored, also where the raw fallback would store it
    out.append(dict(table=same, flag=2, name="above_128k", policy=(64, 6),
                    blocks=[_blk(p14[:HUF_BLOCK_MAX + 1], 1), _blk(p14[:HUF_BLOCK_MAX], 1), _blk(p14[:HUF_BLOCK_MAX + 7])]))

    # 0 and 1 bytes with minLiterals 0: the minimum-gain difference wraps and rejects nothing, so one byte is RLE (two are raw)
    out.append(dict(table=np.zeros(256, np.uint32), flag=0, name="wrap", policy=(0, 6),
                    blocks=[_blk([]), _blk([9]), _blk([7, 7]), _blk(follow)]))
    return out


def plain_mixed_chain(ref, chain, msv, tlog):
    """the plain mixed loop (flags by zstd's size rule) over the chain"""
    ch = dict(chain, blocks=[dict(b, single=int(len(b["src"]) < 256)) for b in chain["blocks"]])
    return ref_mixed_chain(ref, ch, msv, tlog)


def claim_holds(name, pol, mix):
    """does the built chain `name` show its rule: pol = ref_literals_chain's result, mix = the plain mixed loop's"""
    (per, (T, F, _)), (mper, (mT, mF, _)) = pol, mix
    kinds = [x["kind"] for x in per]
    if name == "rollback_saved_zero":             # the 0 return kept the entry state, and the next block reads it
        return kinds == [0, 3] and mper[1][2] is None and F == 1 and (mT != T).any()
    if name == "rollback_failed_validation":
        return kinds == [0, 3] and mper[1][2] is None and mF != 0 and F == 1
    if name == "min_gain":
        return kinds[0] == 0 and mper[0][0] >= 2 and per[0]["r"] == mper[0][0]
    if name == "flag2_forms":
        singles = [x["single"] for x in per]
        return (singles == [1, 1, 1, 0, 0, 0, 0] and kinds[:4] == [3, 3, 3, 3] and kinds[4] == 2 and F == 1
                and any(x[1].tobytes() != y["data"].tobytes() for x, y in zip(mper[1:3], per[1:3])))
    if name == "threshold_6":
        return per[0]["r"] == 0 and kinds[0] == 0 and mper[0][0] >= 2 and kinds[1] in (2, 3) and per[1]["r"] >= 2
    if name == "threshold_min_literals":
        return per[0]["r"] == 0 and mper[0][0] >= 2 and per[1]["r"] >= 2
    if name == "one_byte_1x":
        return per[0]["r"] == 1 and kinds == [0, 1] and mper[0][0] == 1
    if name == "above_128k":
        return kinds[0] == 4 and kinds[2] == 4 and per[0]["r"] == SRC_WRONG and kinds[1] != 4
    if name == "wrap":                            # 1 byte: 1 < (1 - 3) wrapped, RLE; 2 bytes: 1 >= 2 - 2, raw
        return kinds[:3] == [0, 1, 0] and per[1]["r"] == 1 and per[2]["r"] == 1
    raise KeyError(name)


BUILT_CLAIMS = ("rollback_saved_zero", "rollback_failed_validation", "min_gain", "flag2_forms", "threshold_6",
                "threshold_min_literals", "one_byte_1x", "above_128k", "wrap")


def literal_chains(ref, msv, tlog, seed=0):
    """the GPU tests' chains: mid-chain and drifting chains with entry flags 0, 1, 2, ragged chains, and the built chains"""
    base = [c for c in at_bound(mid_chains(ref, seed % 2 == 0, msv, tlog)[::3] + drift_chains(ref)) if c["flag"] in (0, 1, 2)]
    rag = []
    for f, ch in enumerate(ragged_chains(seed=seed)):
        rag.append(dict(ch, flag=f % 3, table=ref_table(ref, probagen(65536, 0.14)) if f % 3 else ch["table"]))
    return base + rag + built_chains(ref)


def long_literal_chain(ref, nblocks=4096):
    """one chain of nblocks blocks: 32 KB P14 blocks with a short section between every two"""
    ch = long_chain(ref, nblocks // 2)
    p40 = probagen(1 << 16, 0.40)
    blks = []
    for i, b in enumerate(ch["blocks"]):
        n = 1 + (i * 97) % 1200
        blks += [b, dict(src=p40[i % 4000:i % 4000 + n].copy(), cap=bound(n), prefer=i % 2)]
    return dict(ch, blocks=blks, name="long_literals")

