"""Pins the kernel-path predicates of tests/paths.py and the coverage of the GPU layout / knob fixtures on the CPU: each input
the -m gpu tests feed the batch codecs reaches the paths those tests claim for it."""
import numpy as np
import pytest

from gpu_common import checker, cpu_compress
import layout_fixtures as F
import paths as P


def test_row_budget_clamp():
    """the first pass carries 8 KB of output staging: at the H100's 232,448-byte opt-in limit it holds 1678 rows, the second 1742"""
    assert P.smem_bytes(306, True) == 56832 and P.smem_bytes(808, False) == 112896
    assert P.smem_bytes(1700, True) == 235264 > 232448 >= P.smem_bytes(1678, True) and P.smem_bytes(1679, True) > 232448
    assert P.row_budgets() == (306, 808)
    assert P.row_budgets(1700) == (1678, 808) and P.row_budgets(1678) == (1678, 808)
    assert P.row_budgets(None, 1800) == (306, 1742)
    assert P.row_budgets(20, 0) == (160, 0)


def test_hard_distribution_needs_more_rows_than_pass_b():
    """the dyadic HARD_LENGTHS histogram: the compressed blocks' tables need 813 rows at their best split (M = 9)"""
    rng = np.random.default_rng(3)
    data = np.concatenate([P.hard_block(rng) for _ in range(4)])
    cbuf, cs, slot = cpu_compress("huf", data)
    for b in range(4):
        c = cbuf[b * slot: b * slot + int(cs[b])]
        h, tl, rs = P.read_stats(c)
        assert tl == 12
        rows = [r for m, cut, r in P.split_candidates(P.rank_end_of(rs, tl), tl)]
        assert min(rows) == 813 and P.table_rows(P.rank_end_of(rs, tl), tl)[:2] == (813, 9)
    kinds, _ = P.summarize(P.huf_decode_paths(cbuf, cs, len(data), 32768, slot, 0))
    assert kinds == {"hard": 4}


def test_stream_and_encoder_predicates():
    """hand-checked cases of the alignment guards"""
    assert P.fse_decode_exact(3, 0, 100, 100, 200) == [(True, False)]
    assert P.fse_decode_exact((1 << 32) - 52, 0, 100, 100, 200) == [(False, True)]
    assert P.fse_decode_exact(8, (1 << 32) - 100, 100, 100, 200, wide=True) == [(False, True)]
    assert P.fse_encode_kernel(0, 3 * 4096 + 5, 4096) == ["chain"] * 3 + ["warp"]
    assert P.fse_encode_kernel(8, 4096, 4096) == ["warp"]
    assert P.huf_plan_histogram(0, 32768 + 100, 32768) == ["pipelined", "scalar"]
    assert P.huf_plan_histogram(16, 4096, 4096) == ["scalar"]
    assert P.pass_a_spread(1000, 132) == (64, 1)
    assert P.pass_a_spread(44000, 132) == (42, 2)


@pytest.mark.parametrize("codec", ["huf", "fse", "u16"])
@pytest.mark.parametrize("block", ["aligned", "ragged"])
@pytest.mark.parametrize("stride", F.STRIDES)
def test_layout_fixture_coverage(codec, block, stride):
    if not checker()[1]:
        pytest.skip("the fixtures' coverage is stated for the compiled reference's output")
    blk = F.block_size(codec, block)
    data = F.layout_data(codec, blk)
    slot = F.slot_for(codec, data, blk, stride)
    want = cpu_compress(codec, data, block=blk, slot=slot, **F.MSV_TL[codec])[:2]
    F.assert_layout_coverage(codec, data, blk, slot, want, stride)


def test_regime_fixture_coverage():
    """on 132 SMs (the H100 SXM): two pass-A rounds of 42 blocks per CTA, thousands of deferred blocks"""
    if not checker()[1]:
        pytest.skip("the fixtures' coverage is stated for the compiled reference's output")
    data, nb = F.regime_data(132)
    slot = F.bound(4096)
    want = cpu_compress("huf", data, block=4096, slot=slot)[:2]
    F.assert_regime_coverage(data, 4096, slot, want, 132)
