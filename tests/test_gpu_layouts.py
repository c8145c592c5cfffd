"""The batch codecs at every buffer placement, slot stride and batch size their kernels branch on (-m gpu).

Every check goes through gpu_common.placed_check: GPU encode and decode (its own slots and the reference's) against the
compiled reference, with poisoned views and canaries.  Before a check touches the GPU it asserts with the predicates of
tests/paths.py that its input reaches the kernel paths it is there for; tests/test_paths.py pins the same fixtures on the CPU."""
import numpy as np
import pytest
import torch

from helpers import ptr, is_error, probagen
from gpu_common import checker, cpu_compress, arena, placed_check, CANARY, POISON
import layout_fixtures as F
import paths as P
import finitestateentropy_b200 as fb

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _needs_reference():
    if not checker()[1]:
        pytest.skip("compares against the compiled reference")


def _views(codec, data, block, slot, offs):
    """fresh poisoned arenas, one per view, at the given offsets from a 512-byte aligned start"""
    n = len(data)
    nb = (n + block - 1) // block
    out = []
    for k, o in zip((n, nb * slot, n), offs):
        a = arena(k + 128)
        assert a.data_ptr() % 512 == 0
        out.append((a, CANARY + o))
    return out


@pytest.mark.parametrize("codec", ["huf", "fse", "u16"])
@pytest.mark.parametrize("block", ["aligned", "ragged"])
@pytest.mark.parametrize("stride", F.STRIDES)
def test_placement_and_stride_matrix(codec, block, stride):
    """every offset in F.offsets(codec) for src, cbuf and out (rotated against each other), at one slot stride"""
    blk = F.block_size(codec, block)
    data = F.layout_data(codec, blk)
    slot = F.slot_for(codec, data, blk, stride)
    want = cpu_compress(codec, data, block=blk, slot=slot, **F.MSV_TL[codec])[:2]
    F.assert_layout_coverage(codec, data, blk, slot, want, stride)
    offs = F.offsets(codec)
    for i in range(len(offs)):
        o = (offs[i], offs[(i + 3) % len(offs)], offs[(i + 5) % len(offs)])
        placed_check(codec, data, blk, slot, want, *_views(codec, data, blk, slot, o), **F.MSV_TL[codec])
    torch.cuda.empty_cache()


@pytest.mark.parametrize("out_off,odd_slot", [(64, True), (1, True)])
def test_x2_verdicts_at_other_placements(out_off, odd_slot):
    """truncated / bit-flipped Huff0 blocks (the reference's HUF_decompress picks X1 or X2) at a non-default output offset and an
    odd slot stride: same verdicts and bytes, nothing written outside the output view"""
    lib, _ = checker()
    rng = np.random.default_rng(12 + out_off)
    block = 8192
    data = F.x2_data(rng, block)
    slot = fb.compress_bound(block) + 1
    cbuf, cs = F.corrupt(rng, *cpu_compress("huf", data, block=block, slot=slot)[:2], slot)
    nb = len(cs)
    want = np.zeros(nb, np.uint64)
    want_out = np.zeros(len(data), np.uint8)
    for b in range(nb):
        if cs[b] < 2:
            want[b] = block
            want_out[b * block:(b + 1) * block] = data[b * block:(b + 1) * block]
            continue
        tmp = np.concatenate([cbuf[b * slot: b * slot + int(cs[b])], np.zeros(32, np.uint8)])
        o = np.zeros(block + 8, np.uint8)
        want[b] = lib.HUF_decompress(ptr(o), block, ptr(tmp), int(cs[b]))
        want_out[b * block:(b + 1) * block] = o[:block]
    paths = P.huf_decode_paths(cbuf, cs, len(data), block, slot, out_off)
    kinds, streams = P.summarize(paths)
    assert streams["fast"] + streams["fast+tail"] > 100 if out_off % 32 == 0 else streams["symbol"] > 100, streams
    assert sum(is_error(int(x)) for x in want) > 10
    a = arena(len(data) + 128)
    o_v = a[CANARY + out_off: CANARY + out_off + len(data)]
    o_v.copy_(torch.from_numpy(~want_out).cuda())
    c_a = arena(nb * slot + 128)
    c_v = c_a[CANARY + 3: CANARY + 3 + nb * slot]
    c_v.copy_(torch.from_numpy(cbuf[:nb * slot]).cuda())
    out, res = fb.huf_decompress_batch(c_v, torch.from_numpy(cs.view(np.int64)).cuda(), len(data), block, slot, out=o_v,
                                       orig=torch.from_numpy(data).cuda())
    res = res.cpu().numpy().view(np.uint64)
    bad = [(b, int(res[b]), int(want[b])) for b in range(nb) if res[b] != want[b]]
    assert not bad, bad[:10]
    got = o_v.cpu().numpy()
    for b in range(nb):
        if not is_error(int(want[b])):
            assert np.array_equal(got[b * block:(b + 1) * block], want_out[b * block:(b + 1) * block]), b
    assert bool((a[:CANARY + out_off] == POISON).all()) and bool((a[CANARY + out_off + len(data):] == POISON).all())


def test_across_a_4gib_address_boundary():
    """one allocation of 4 GiB + 64 MiB; per codec, the output view and then the compressed view (and the source) straddle the
    2^32-aligned address inside it, so the FSE / U16 decoders' `sameHi` guard sends those blocks to the exact path"""
    size = (4 << 30) + (64 << 20)
    torch.cuda.reset_peak_memory_stats()
    try:
        big = torch.empty(size, dtype=torch.uint8, device="cuda")
    except RuntimeError as exc:          # torch.OutOfMemoryError is a RuntimeError
        pytest.skip("no room for a 4 GiB + 64 MiB buffer on this device: %s" % str(exc).splitlines()[0])
    try:
        big.fill_(POISON)
        base = big.data_ptr()
        x = ((base + (16 << 20)) + (1 << 32) - 1) >> 32 << 32           # a 2^32 boundary with >= 16 MiB on both sides
        assert base + (16 << 20) <= x <= base + size - (16 << 20)
        xi = x - base
        far = xi - (512 << 20) if xi > (600 << 20) else xi + (512 << 20)   # views that do not straddle, away from x
        for codec in ("huf", "fse", "u16"):
            block = 32768
            data = F.boundary_data(codec)
            n = len(data)
            slot = fb.compress_bound(block)
            nb = (n + block - 1) // block
            want = cpu_compress(codec, data, block=block, slot=slot, **F.MSV_TL[codec])[:2]
            mid = lambda k: xi - (k // 2) // 512 * 512 - 2                # a view of k bytes centred on x (even: U16 contract)
            # 1) output straddles
            oi = mid(n)
            ex = P.fse_decode_exact(base + oi, base + far, n, block, slot, wide=codec == "u16")
            assert sum(e[1] for e in ex) >= 1
            placed_check(codec, data, block, slot, want, (big, far + (64 << 20)), (big, far), (big, oi), **F.MSV_TL[codec])
            # 2) compressed slots straddle: several blocks on each side, one slot across
            ci = mid(nb * slot)
            ex = P.fse_decode_exact(base + far, base + ci, n, block, slot, wide=codec == "u16")
            assert sum(e[1] for e in ex) >= 1
            crossing = [b for b in range(nb) if (base + ci + b * slot) >> 32 != (base + ci + (b + 1) * slot - 1) >> 32]
            assert len(crossing) == 1 and 2 < crossing[0] < nb - 2
            placed_check(codec, data, block, slot, want, (big, far + (64 << 20)), (big, ci), (big, far), **F.MSV_TL[codec])
            # 3) the source straddles
            placed_check(codec, data, block, slot, want, (big, mid(n)), (big, far + (32 << 20)), (big, far), **F.MSV_TL[codec])
        peak = torch.cuda.max_memory_allocated()
        print("4 GiB boundary test: peak device memory allocated by torch %.2f GiB" % (peak / 2 ** 30))
    finally:
        del big
        torch.cuda.empty_cache()


def test_huf_batch_spread_over_rounds():
    """a Huff0 batch of >= 1.3 x (4 x SMs x 64) blocks of 4 KB: pass A runs with fewer than 64 blocks per CTA over two or more
    rounds, and thousands of blocks go to one pass-B list; every block compared in full"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    block = 4096
    data, nb = F.regime_data(sms, block)
    slot = fb.compress_bound(block)
    want = cpu_compress("huf", data, block=block, slot=slot)[:2]
    F.assert_regime_coverage(data, block, slot, want, sms)
    placed_check("huf", data, block, slot, want, *_views("huf", data, block, slot, (0, 0, 0)))
    torch.cuda.empty_cache()
