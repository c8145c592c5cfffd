"""CPU-only checks of the per-block descriptor decoder's host-side models (no GPU code involved):

  * the stream ring with a head decode: 0 to 31 single-symbol steps, topped up every 8 symbols as the tail loop does, before
    the fast loop -- the unread count must stay in [1, 8] at every check for the code-length shapes of test_decode_ring_model;
  * the path predicate of tests/blocks_paths.py on hand-computed cases."""
import random

import pytest

from blocks_paths import stream_paths, stream_kind, plan_histogram, emit_groups, expected_decode_verdict
from test_decode_ring_model import MAX_CODE_BITS, run_lane


def run_head(lengths, r0, unread0):
    """the head loop: top_up(4) before symbols 0, 8, 16, 24; returns (r, unread) at the fast loop's first check"""
    r, unread = r0, unread0
    for i, bits in enumerate(lengths):
        if i % 8 == 0:
            assert 1 <= unread <= 8
            if unread <= 4:
                unread += 4
            assert unread >= 5
        old = r
        r += bits
        if (r ^ old) & 32:                                  # one symbol is at most 12 bits: at most one word used up
            assert unread >= 1, "fetch from an empty ring"
            unread -= 1
    return r, unread


@pytest.mark.parametrize("seed", range(8))
def test_ring_with_head_never_runs_dry(seed):
    rng = random.Random(seed)
    n = 32 * 64
    shapes = [
        [MAX_CODE_BITS] * (n + 31),
        [1] * (n + 31),
        [rng.randint(1, MAX_CODE_BITS) for _ in range(n + 31)],
        [MAX_CODE_BITS if (i // 7) & 1 else 1 for i in range(n + 31)],
        [rng.choice((1, 1, 1, 11, 12)) for _ in range(n + 31)],
    ]
    for lengths in shapes:
        for head in range(32):
            for r0 in (0, 1, 17, 31):
                for unread0 in (5, 8):
                    r, unread = run_head(lengths[:head], r0, unread0)
                    assert 1 <= unread <= 8
                    assert 1 <= run_lane(lengths[head: head + n], r, unread) <= 8


def test_stream_paths():
    # 4 x 100 symbols at an aligned start: streams start at 0, 100, 200, 300 (mod 32: 0, 4, 8, 12)
    assert stream_paths("A", 400, 0) == [(0, 3, 4), (28, 2, 8), (24, 2, 12), (20, 2, 16)]
    assert stream_paths("hard", 400, 0) == [(0, 0, 100)] * 4
    # streams of 40 symbols starting at 1, 41, 81, 121: heads of 31, 23, 15, 7; only the last leaves a whole sector
    assert stream_paths("A", 160, 1) == [(0, 0, 40), (0, 0, 40), (0, 0, 40), (7, 1, 1)]
    assert [stream_kind(*s) for s in stream_paths("B", 131072, 3)] == ["head+fast"] * 4
    assert [stream_kind(*s) for s in stream_paths("B", 131072, 0)] == ["fast"] * 4


def test_plan_and_emit_predicates():
    assert plan_histogram(0, 32768) == "pipelined" and plan_histogram(16, 131072) == "pipelined"
    assert plan_histogram(8, 32768) == "scalar" and plan_histogram(0, 32769) == "scalar" and plan_histogram(0, 0) == "scalar"
    assert emit_groups(0, 32768) == ["g256"] * 4
    assert emit_groups(0, 4 * 1001) == ["bytes", "bytes", "bytes", "g128"] and emit_groups(4, 4 * 1003) == ["bytes", "bytes", "bytes", "g256"] and emit_groups(4, 4 * 1000) == ["g128"] * 4


def test_expected_verdicts():
    assert expected_decode_verdict(100000, 5000, 131073) == 2 ** 64 - 3
    assert expected_decode_verdict(5, 3, 5) == 2 ** 64 - 4
    assert expected_decode_verdict(2 ** 64 - 3, 3, 5) == 2 ** 64 - 3
    assert expected_decode_verdict(5, 5, 5) == 5 and expected_decode_verdict(5, 1, 5) == 5
    assert expected_decode_verdict(2 ** 64 - 2, 0, 0) == 2 ** 64 - 2
