"""Packed Huff0 decompress (FSEB200_HUF_decompress_packed / FSEB200_HUF_decompress1X_packed) on the GPU (-m gpu): on the output
of the packed compress -- compressed, raw, RLE, empty, error (L = 0) and weight-12-exception blocks, blocks above 128 KB -- and on
hand-made streams (n = 0 with L > 0, L > n), every result equals the descriptor decoder's on the derived pointers
(dIn + dOffsets[b], dOffsets[b+1] - dOffsets[b]) but for empty blocks, which give 0; every block the compress stored without an
error decodes to its source, but for the reference's own exception, which the compiled reference rejects too; and nothing is
written outside the destinations."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from helpers import is_error                                                      # noqa: E402
from packed_paths import ref_values, image, ref_decode                            # noqa: E402
from test_gpu_blocks import POISON, CANARY, ragged_sources, _ref, _u64, _dev64    # noqa: E402

pytestmark = pytest.mark.gpu

FORMATS = [False, True]
FORMAT_IDS = ["4X", "1X"]


def weight12_block():
    """20,000 bytes whose Huffman tree at tableLog 12 gives one symbol a 1-bit code: the reference writes weight 12 for it and
    its own decoder rejects the block"""
    fib = [1, 1]
    while len(fib) < 14:
        fib.append(fib[-1] + fib[-2])
    s = np.concatenate([np.full(c, i, np.uint8) for i, c in enumerate([5000] + fib)])
    np.random.default_rng(0).shuffle(s)
    return np.resize(s, 20000)


def decode_both(onex, packed, offsets, sizes):
    """the packed decompress and the descriptor decoder on the derived pointers, each into its own poisoned arena (destinations
    32 bytes apart): (packed results, descriptor results, packed arena, descriptor arena, destination indices)"""
    import torch
    import finitestateentropy_b200 as fb
    doffs, cur = [], CANARY
    for n in sizes:
        doffs.append(cur)
        cur += min(n, 1 << 18) + 32
    arenas = [torch.full((cur + CANARY,), POISON, dtype=torch.uint8, device="cuda") for _ in range(2)]
    dsz = _dev64(sizes)
    offs_dev = torch.tensor(offsets, dtype=torch.int64, device="cuda")
    dec_packed = fb.huf_decompress1x_packed if onex else fb.huf_decompress_packed
    dec_blocks = fb.huf_decompress1x_blocks if onex else fb.huf_decompress_blocks
    got = dec_packed(packed, offs_dev, _dev64([arenas[0].data_ptr() + d for d in doffs]), dsz)
    ptrs, lens = fb.packed_pointers(packed, offs_dev)
    want = dec_blocks(ptrs.contiguous(), lens.contiguous(), _dev64([arenas[1].data_ptr() + d for d in doffs]), dsz)
    torch.cuda.synchronize()
    return _u64(got), _u64(want), arenas[0].cpu().numpy(), arenas[1].cpu().numpy(), doffs


def check_against_descriptors(onex, packed, offsets, sizes):
    got, want, a, b, doffs = decode_both(onex, packed, offsets, sizes)
    for i, n in enumerate(sizes):
        L = offsets[i + 1] - offsets[i]
        w = 0 if n == 0 and L == 0 else int(want[i])
        assert int(got[i]) == w, (onex, i, n, L, int(got[i]), w)
        if not is_error(w) and w:
            assert np.array_equal(a[doffs[i]: doffs[i] + w], b[doffs[i]: doffs[i] + w]), (onex, i)
    # nothing outside the destinations: the gaps between them stay poisoned
    mask = np.ones(len(a), bool)
    for d, n in zip(doffs, sizes):
        mask[d: d + min(n, 1 << 18)] = False
    assert bool((a[mask] == POISON).all()), "bytes outside the destinations were written"
    return got, a, doffs


@pytest.mark.parametrize("onex", FORMATS, ids=FORMAT_IDS)
def test_packed_compress_round_trip(onex):
    """the packed compress's own buffer: compressed, raw, RLE, empty, error and weight-12 blocks, blocks above 128 KB; the
    buffer ends 32 bytes after the last block"""
    import torch
    import finitestateentropy_b200 as fb
    lib = _ref()
    rng = np.random.default_rng(701)
    host, offs, sizes = ragged_sources(rng, 500)
    w12 = weight12_block()
    host = np.concatenate([host, w12])
    offs, sizes = offs + [len(host) - len(w12)], sizes + [len(w12)]
    vals, stored = ref_values(lib, [host[o: o + n] for o, n in zip(offs, sizes)], 255, 12, onex)
    src = torch.from_numpy(host).cuda()
    sp, sn = _dev64([src.data_ptr() + o for o in offs]), _dev64(sizes)
    enc = fb.huf_compress1x_packed if onex else fb.huf_compress_packed
    out, offsets, cs = enc(sp, sn)
    torch.cuda.synchronize()
    offsets = [int(x) for x in _u64(offsets)]
    final = [int(x) for x in _u64(cs)]
    assert final == vals
    kinds = {"empty" if n == 0 else 0 if v == 0 else 1 if v == 1 else "err" if is_error(v) else "size" for v, n in zip(vals, sizes)}
    assert kinds == {"empty", 0, 1, "err", "size"}, kinds
    assert any(n > 131072 and is_error(v) for v, n in zip(vals, sizes))
    packed = out[: offsets[-1] + 32].clone()                            # ends 32 bytes after the last block
    got, a, doffs = check_against_descriptors(onex, packed, offsets, sizes)
    img, _, _, _ = image(vals, stored, sizes, offsets[-1])
    ref = ref_decode(lib, img, offsets, sizes, vals, onex)
    undecodable = 0
    for b, (n, v) in enumerate(zip(sizes, vals)):
        if is_error(v):
            continue
        if n == 0:
            assert int(got[b]) == 0
            continue
        assert int(got[b]) == ref[b][0], (onex, b, n, int(got[b]), ref[b][0])
        if int(got[b]) == n:
            assert np.array_equal(a[doffs[b]: doffs[b] + n], host[offs[b]: offs[b] + n]), (onex, b)
        else:
            undecodable += 1
    assert is_error(int(got[-1])) and undecodable >= 1                  # the weight-12 block


@pytest.mark.parametrize("onex", FORMATS, ids=FORMAT_IDS)
def test_hand_made_streams(onex):
    """stored lengths the packed compress never writes: n = 0 with L > 0, L > n, L == n raw copies and L == 1 RLE of any byte,
    L == 0 with n > 0, n above 128 KB, and compressed blocks taken from the compress"""
    import torch
    import finitestateentropy_b200 as fb
    rng = np.random.default_rng(702)
    host, offs, sizes = ragged_sources(rng, 60, [3000, 9000, 40000, 77, 131072] * 12)
    src = torch.from_numpy(host).cuda()
    enc = fb.huf_compress1x_packed if onex else fb.huf_compress_packed
    out, offsets, cs = enc(_dev64([src.data_ptr() + o for o in offs]), _dev64(sizes))
    torch.cuda.synchronize()
    o = [int(x) for x in _u64(offsets)]
    comp = out.cpu().numpy()
    pieces, dst = [], []
    for b in range(len(sizes)):
        L = o[b + 1] - o[b]
        k = b % 8
        if k == 0:
            pieces.append(comp[o[b]: o[b + 1]]); dst.append(sizes[b])               # as compressed
        elif k == 1:
            pieces.append(comp[o[b]: o[b] + 7]); dst.append(0)                       # n = 0, L > 0
        elif k == 2:
            pieces.append(comp[o[b]: o[b + 1]]); dst.append(max(L - 5, 1))            # L > n
        elif k == 3:
            pieces.append(rng.integers(0, 256, 1000, dtype=np.uint8)); dst.append(1000)   # raw copy
        elif k == 4:
            pieces.append(np.array([b & 0xFF], np.uint8)); dst.append(5000)          # RLE
        elif k == 5:
            pieces.append(np.zeros(0, np.uint8)); dst.append(300)                    # L = 0, n > 0
        elif k == 6:
            pieces.append(comp[o[b]: o[b + 1]]); dst.append(131073)                  # n above 128 KB
        else:
            pieces.append(np.zeros(0, np.uint8)); dst.append(0)                      # empty
    packed_np = np.concatenate(pieces)
    offsets = [0] + [int(x) for x in np.cumsum([len(p) for p in pieces])]
    packed = torch.from_numpy(np.concatenate([packed_np, np.zeros(32, np.uint8)])).cuda()
    got, a, doffs = check_against_descriptors(onex, packed, offsets, dst)
    for b in range(len(dst)):
        if b % 8 == 3:
            assert int(got[b]) == 1000 and np.array_equal(a[doffs[b]: doffs[b] + 1000], pieces[b])
        if b % 8 == 4:
            assert int(got[b]) == 5000 and bool((a[doffs[b]: doffs[b] + 5000] == (b & 0xFF)).all())
        if b % 8 == 7:
            assert int(got[b]) == 0


def test_python_wrappers_on_a_side_stream():
    import torch
    import finitestateentropy_b200 as fb
    from helpers import probagen
    data = [torch.from_numpy(x).cuda() for x in (probagen(1000, 0.14), np.full(300, 7, np.uint8), np.zeros(0, np.uint8),
                                                 np.random.default_rng(1).integers(0, 256, 777, dtype=np.uint8))]
    s = torch.cuda.Stream()
    for onex in FORMATS:
        enc = fb.huf_compress1x_packed if onex else fb.huf_compress_packed
        dec = fb.huf_decompress1x_packed if onex else fb.huf_decompress_packed
        sp = _dev64([d.data_ptr() if d.numel() else data[0].data_ptr() for d in data])
        sn = _dev64([d.numel() for d in data])
        with torch.cuda.stream(s):
            out, offsets, _ = enc(sp, sn)
            outs = [torch.zeros(max(d.numel(), 1), dtype=torch.uint8, device="cuda") for d in data]
            res = dec(out, offsets, _dev64([x.data_ptr() for x in outs]), sn)
        s.synchronize()
        assert res.tolist() == [d.numel() for d in data]
        assert all(torch.equal(x[: d.numel()], d) for x, d in zip(outs, data))
        with pytest.raises(AssertionError):
            dec(out, offsets[:-1], _dev64([x.data_ptr() for x in outs]), sn)
