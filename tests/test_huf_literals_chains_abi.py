"""CPU-side checks of the literal-policy Huff0 chain compress (FSEB200_HUF_compress_literals_chains_packed and
FSEB200_compress_host_literals_chains_packed): declarations and exports, the argument verdicts, which touch no device, and -- on the
compiled reference alone -- the claims the case set rests on: each built chain's policy loop differs from the plain mixed loop
(flags by the size rule) in the way it claims, and every block the policy loop stores with a value that is not an error decodes
back to its source with the reference's decoders (but for the weight-12 exception)."""
import re
import subprocess
from collections import Counter

import numpy as np
import pytest
import torch

from helpers import is_error, ptr, load_ref, declared_arity
from huf_chain_cases import chain_header
from huf_chain_packed_cases import resolve_headers
from huf_literals_chain_cases import (ref_literals_chain, expected_literals, built_chains, literal_chains, plain_mixed_chain,
                                      claim_holds, BUILT_CLAIMS, POLICIES)

CALLS = {"FSEB200_HUF_compress_literals_chains_packed": 21, "FSEB200_compress_host_literals_chains_packed": 20}
WRAPPERS = ("huf_compress_literals_chains_packed", "host_compress_literals_chains_packed")
SRC_WRONG = (1 << 64) - 3


def _lib():
    import finitestateentropy_b200 as fb
    return fb.lib()


def _ref():
    ref = load_ref()
    if ref is None:
        pytest.skip("compiled reference not available")
    return ref


def test_header_declares_and_library_exports_the_calls():
    decl = declared_arity()
    assert {n: decl.get(n) for n in CALLS} == CALLS
    from finitestateentropy_b200 import _build
    exported = subprocess.check_output(["nm", "-D", "--defined-only", _build.build_lib()]).decode()
    for name in CALLS:
        assert re.search(r" T %s$" % name, exported, flags=re.M), name
    import finitestateentropy_b200 as fb
    for name in WRAPPERS:
        assert callable(getattr(fb, name)), name


def test_argument_verdicts_without_a_device():
    """nBlocks == 0 returns 0 and touches nothing; nBlocks or nChains above 2^32 - 1, a NULL array (dSingleStream included) or
    minGainLog outside 1 .. 31 while nBlocks > 0 gives srcSize_wrong.  Host buffers stand in for device arrays (device call) and
    for the host call's arrays: nothing may touch them."""
    L = _lib()
    words = [np.full(4, 7, np.uint64) for _ in range(14)]
    a = [w.ctypes.data for w in words]

    def dev(arr, nc, nb, mgl=6):     # starts, out, offsets, csizes, kinds, srcs, sizes, prefer, single, tables, flags, chdrs, chsizes
        return L.FSEB200_HUF_compress_literals_chains_packed(nc, arr[0], nb, arr[1], 1 << 20, *arr[2:13], 255, 11, 64, mgl, None)

    def host(arr, nc, nb, mgl=6):
        return L.FSEB200_compress_host_literals_chains_packed(nc, arr[0], nb, arr[1], 64, *arr[2:13], 255, 11, 64, mgl)

    for call in (dev, host):
        assert call([None] * 13, 1, 0) == 0
        assert call(a[:13], 1, 2 ** 32) == SRC_WRONG
        assert call(a[:13], 2 ** 32, 2) == SRC_WRONG
        for mgl in (0, 32, 1 << 31):
            assert call(a[:13], 1, 2, mgl) == SRC_WRONG, (call.__name__, mgl)
        for i in range(13):
            bad = list(a[:13])
            bad[i] = None
            assert call(bad, 1, 2) == SRC_WRONG, (call.__name__, i)
    for w in words:
        assert (w == 7).all()


def test_wrappers_check_dtypes():
    import finitestateentropy_b200 as fb
    src = torch.zeros(64, dtype=torch.uint8)
    st = torch.tensor([0, 2], dtype=torch.int64)
    tabs, flags = torch.zeros(1, 256, dtype=torch.int32), torch.zeros(1, dtype=torch.int32)
    hp, hs = torch.zeros(1, dtype=torch.int64), torch.zeros(1, dtype=torch.int64)
    for pr in (torch.zeros(2, dtype=torch.int64), torch.zeros(3, dtype=torch.int32)):
        with pytest.raises(AssertionError):
            fb.host_compress_literals_chains_packed(src, [4, 4], st, pr, tabs, flags, hp, hs)
    c64, c32 = torch.zeros(2, dtype=torch.int64), torch.zeros(2, dtype=torch.int32)
    one64, one32 = torch.zeros(1, dtype=torch.int64), torch.zeros(1, dtype=torch.int32)
    with pytest.raises(AssertionError):            # host tensors are refused by the device wrapper
        fb.huf_compress_literals_chains_packed(st, c64, c64, c32, one64, one32, one64, one64, out=src)


def test_built_chains_show_their_rules():
    """each built chain, at its (minLiterals, minGainLog), gives what its rule claims against the plain mixed loop; together they
    cover every rule"""
    ref = _ref()
    chains = built_chains(ref)
    assert sorted(ch["name"] for ch in chains) == sorted(BUILT_CLAIMS)
    for ch in chains:
        ml, mgl = ch["policy"]
        pol = ref_literals_chain(ref, ch, 255, 11, ml, mgl)
        assert claim_holds(ch["name"], pol, plain_mixed_chain(ref, ch, 255, 11)), ch["name"]


def _decode(ref, hdr, n, single, payload=None):
    """HUF_readDTableX1 on hdr, then the block's form on payload (by default what follows the header in hdr): (regenerated bytes,
    value), or (None, the header's error) -- the reference's weight-12 exception"""
    dt = np.zeros(4097, np.uint32)
    dt[0] = 11 * 0x01000001                                             # HUF_CREATE_STATIC_DTABLEX1(DT, HUF_TABLELOG_MAX)
    hs = ref.HUF_readDTableX1(ptr(dt), ptr(hdr), len(hdr))
    if is_error(hs):
        return None, hs
    if payload is None:
        payload = hdr[hs:]
    out = np.zeros(n + 64, np.uint8)
    fn = ref.HUF_decompress1X1_usingDTable if single else ref.HUF_decompress4X1_usingDTable
    r = fn(ptr(out), n, ptr(payload), len(payload), ptr(dt))
    return out[:n], r


@pytest.mark.parametrize("policy", POLICIES[:2], ids=["64_6", "8_8"])
def test_the_loops_stream_decodes_on_the_reference(policy):
    """every stored block of the policy loop's stream decodes to its source: raw and RLE directly, kind 2 with its own header,
    kind 3 with the header of the last kind-2 block of its chain or the chain's entry header (HUF_readDTableX1, then the block's
    form); the reference's weight-12 exception aside"""
    ref = _ref()
    ml, mgl = policy
    chains = literal_chains(ref, 255, 11)
    want = [ref_literals_chain(ref, ch, 255, 11, ml, mgl) for ch in chains]
    vals, kinds, blobs, flags, starts = expected_literals(want, chains)
    heads = resolve_headers(kinds, starts)
    seen = Counter()
    b = 0
    for ch in chains:
        entry, real = chain_header(ref, ch)
        for blk in ch["blocks"]:
            src, k, blob = blk["src"], kinds[b], blobs[b]
            n = len(src)
            seen["kind%d" % k] += 1
            seen["single" if flags[b] else "four"] += k in (2, 3)
            if k == 0:
                assert len(blob) == n and (blob == src).all()
            elif k == 1:                                            # n >= 8 is RLE by the rule; only a table declared valid
                assert len(blob) == 1 and blob[0] == src[0]          # that lacks the block's symbols codes it into one byte
                seen["rle" if (src == blob[0]).all() else "rle_by_rule"] += 1
                assert (src == blob[0]).all() or n >= 8
            elif k == 2:
                got, r = _decode(ref, blob, n, flags[b])
                if got is None:
                    seen["weight12"] += 1
                else:
                    assert r == n and (got == src).all(), (ch["name"], b)
            elif k == 3:
                h = heads[b]
                hdr = blobs[h[1]] if h[0] == "block" else entry
                if h[0] == "block" or real:
                    got, r = _decode(ref, hdr, n, flags[b], blob)
                    if got is None:
                        seen["weight12"] += 1
                    else:
                        assert r == n and (got == src).all(), (ch["name"], b)
                        seen["decoded3"] += 1
            b += 1
    assert seen["kind0"] and seen["kind1"] and seen["kind2"] and seen["decoded3"] and seen["kind4"], dict(seen)
    assert seen["single"] and seen["four"], dict(seen)
