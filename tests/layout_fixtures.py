"""Inputs of tests/test_gpu_layouts.py and tests/knob_child.py, and the coverage each must have (checked on the CPU with the
predicates of tests/paths.py, by those tests before they run and by tests/test_paths.py without a GPU)."""
import numpy as np

from helpers import probagen, gen_u16, zoo, is_error
from gpu_common import cpu_compress
import paths as P

STRIDES = ["bound", "x128", "odd", "tight"]
MSV_TL = {"huf": {"msv": 255, "tl": 12}, "fse": {"msv": 255, "tl": 12}, "u16": {"msv": 0, "tl": 12}}


def bound(n):
    return 512 + n + (n >> 7) + 4 + 8               # FSE_compressBound


def offsets(codec):
    """byte offsets of the views from a 512-byte aligned start; U16 views hold unsigned shorts, so its offsets are even"""
    return [0, 2, 4, 8, 16, 32, 64, 96] if codec == "u16" else [0, 1, 4, 8, 16, 32, 64, 96]


def block_size(codec, kind):
    """32 KB, or a size whose Huff0 segments and FSE outputs are not aligned (U16: even, 4 mod 8)"""
    return 32768 if kind == "aligned" else (4100 if codec == "u16" else 4099)


def _probe(n, p, off):
    return probagen(off + n, p)[off:]


def layout_data(codec, block):
    """a few dozen blocks of the probagen inputs (the P blocks, first), wide flat alphabets, hard blocks, raw / RLE blocks
    and a ragged last block"""
    rng = np.random.default_rng(block * 7 + len(codec))
    nb = 24 if block == 32768 else 96
    if codec == "u16":
        parts = [gen_u16(block // 2, 240, [0.5, 0.2, 0.8][i % 3], 1 + i).view(np.uint8) for i in range(nb // 2)]
        parts += [rng.integers(0, 287, block // 2).astype(np.uint16).view(np.uint8) for _ in range(nb // 4)]
        parts += [np.full(block // 2, 77, np.uint16).view(np.uint8)]
        parts += [gen_u16(block // 2, 240, 0.3, 99).view(np.uint8) for _ in range(nb // 4)]
        parts.append(gen_u16(block // 4 + 1, 240, 0.5, 7).view(np.uint8))
        return np.concatenate(parts)
    ps = (0.14, 0.80) if codec == "huf" else (0.80, 0.14)
    parts = [_probe(block, ps[i % 2], 1000 * i) for i in range(nb // 2)]
    parts += [_probe(block, 0.02, 777 * i) for i in range(nb // 8)]
    if codec == "huf" and block == 32768:
        parts += [P.hard_block(rng) for _ in range(3)]
    parts += [rng.integers(0, 256, block, dtype=np.uint8), np.full(block, 9, np.uint8)]
    while len(parts) < nb:
        parts.append(zoo(rng, block))
    parts.append(_probe(block // 3 + 5, 0.2, 5))
    return np.concatenate(parts)


def _p_blocks(codec, block):
    """indices of the probagen / genU16 blocks at the start of layout_data"""
    return range((24 if block == 32768 else 96) // 2)


def slot_for(codec, data, block, stride):
    b = bound(block)
    if stride == "bound":
        return b
    if stride == "x128":
        return (b + 127) // 128 * 128 + 128
    if stride == "odd":
        return b + (2 if codec == "u16" else 1)      # U16: even, 2 mod 4
    _, cs, _ = cpu_compress(codec, data, block=block, slot=b, **MSV_TL[codec])
    top = sorted(int(cs[i]) for i in _p_blocks(codec, block))[len(_p_blocks(codec, block)) // 2:]
    t = top[len(top) // 2] + 12                       # about half of the largest P blocks no longer fit (a writer keeps 8 bytes spare)
    return t + (t & 1) if codec == "u16" else t


def assert_layout_coverage(codec, data, block, slot, want, stride):
    """what one row of the placement matrix (one codec, block size and stride, every offset) must reach"""
    cbuf, cs = want
    n = len(data)
    offs = offsets(codec)
    if stride == "tight":
        _, cs_b, _ = cpu_compress(codec, data, block=block, slot=bound(block), **MSV_TL[codec])
        pb = list(_p_blocks(codec, block))
        lost = sum(1 for i in pb if cs_b[i] != cs[i])    # no longer fit: 0 (U16: the header size alone)
        close = sum(1 for i in pb if 1 < int(cs[i]) and not is_error(int(cs[i])) and slot - int(cs[i]) <= 64)
        assert slot < bound(block) and lost >= 2 and close >= 2, (lost, close)
    if codec == "huf":
        kinds, streams = P.Counter(), P.Counter()
        for o in offs:
            k, s = P.summarize(P.huf_decode_paths(cbuf, cs, n, block, slot, o))
            kinds += k
            streams += s
        want_kinds = {"A", "raw", "rle"} | ({"hard"} if block == 32768 else set())
        if stride != "tight" or block != 32768:        # P02 blocks of 32 KB do not fit the tight stride
            want_kinds.add("B")
        assert want_kinds <= set(kinds), kinds
        assert streams["symbol"] > 0 and streams["fast"] + streams["fast+tail"] > 0, streams
        if block != 32768:
            assert P.warps_with_both_stream_kinds(P.huf_decode_paths(cbuf, cs, n, block, slot, 0)) > 0
        hist = [h for o in offs for h in P.huf_plan_histogram(o, n, block)]
        assert "scalar" in hist and ("pipelined" in hist or block != 32768)
        emit = [e for o, oc in zip(offs, offs[3:] + offs[:3]) for per in P.huf_emit_paths(o, oc, cbuf, cs, n, block, slot).values() for e in per]
        assert {"g256", "g128", "bytes"} <= {e[0] for e in emit} and {True, False} <= {e[1] for e in emit}
    else:
        wide = codec == "u16"
        enc = [k for o in offs for k in P.fse_encode_kernel(o, n, block)]
        assert "warp" in enc and ("chain" in enc or block % 64)
        ex = [e[0] for o in offs for e in P.fse_decode_exact(o, 0, n, block, slot, wide)]
        assert True in ex and False in ex


def x2_data(rng, block):
    return np.concatenate([zoo(rng, block) if i % 3 else probagen(block, [0.14, 0.2, 0.3][i % 9 // 3]) for i in range(200)])


def corrupt(rng, cbuf, cs, slot):
    """truncate or bit-flip some compressed blocks in place (the fuzzers' corruption modes)"""
    for b in range(len(cs)):
        if cs[b] < 2:
            continue
        c = cbuf[b * slot: b * slot + int(cs[b])]
        mode = int(rng.integers(0, 3))
        if mode == 0:
            cs[b] = int(rng.integers(2, int(cs[b])))
        elif mode == 1:
            for _ in range(int(rng.integers(1, 4))):
                c[int(rng.integers(0, len(c)))] ^= int(rng.integers(1, 256))
    return cbuf, cs


def boundary_data(codec):
    """8 MiB: P14 for Huff0, P80 for FSE, genU16(240, 0.5) for U16"""
    if codec == "u16":
        return gen_u16(4 << 20, 240, 0.50, 1).view(np.uint8)
    return probagen(8 << 20, 0.14 if codec == "huf" else 0.80)


def regime_data(sms, block=4096):
    """>= 1.3 x (4 x SMs x 64) blocks: P14, P02 (tables too large for pass A: deferred), P05 and zoo blocks interleaved"""
    nb = int(1.3 * 4 * sms * 64) + 1000
    rng = np.random.default_rng(5)
    p14 = probagen(nb // 8 * 3 * block + block, 0.14)
    p02 = probagen(nb // 8 * 2 * block + block, 0.02)
    p05 = probagen(nb // 8 * 2 * block + block, 0.05)
    zz = [zoo(rng, block) for _ in range(61)]
    out = np.empty(nb * block, np.uint8)
    i14 = i02 = i05 = 0
    for b in range(nb):
        r = b % 8
        if r < 3:
            src, i14 = p14[i14 * block:(i14 + 1) * block], i14 + 1
        elif r < 5:
            src, i02 = p02[i02 * block:(i02 + 1) * block], i02 + 1
        elif r < 7:
            src, i05 = p05[i05 * block:(i05 + 1) * block], i05 + 1
        else:
            src = zz[b % 61]
        out[b * block:(b + 1) * block] = src
    return out, nb


def assert_regime_coverage(data, block, slot, want, sms):
    cbuf, cs = want
    nb = len(cs)
    g_eff, rounds = P.pass_a_spread(nb, sms)
    assert g_eff < P.G and rounds >= 2, (g_eff, rounds)
    kinds, _ = P.summarize(P.huf_decode_paths(cbuf, cs, len(data), block, slot, 0))
    assert kinds["B"] >= 5000 and kinds["A"] >= 10000 and kinds["raw"] + kinds["rle"] > 0, kinds
