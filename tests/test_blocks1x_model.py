"""CPU-only checks of the single-stream (1X) descriptor decoder's host-side models (no GPU code involved):

  * a 1X stream is one whole block, up to 131,072 symbols, four times a 4X segment: the stream ring with a head decode must
    keep its unread count in [1, 8] over that length, and the ring slot the hot loop derives from the never-reduced bit count
    r must be right for the 1X slot stride (64 lanes: 256 bytes) as well as the 4X one (1024 bytes);
  * the path predicate of tests/blocks1x_paths.py on hand-computed cases."""
import random

import pytest

from blocks1x_paths import stream_paths_1x, pass_a_spread_1x, emit_group_1x, stream_kind
from test_blocks_model import run_head
from test_decode_ring_model import MAX_CODE_BITS, run_lane

STREAM_MAX = 128 * 1024


@pytest.mark.parametrize("seed", range(3))
def test_ring_over_a_whole_block_never_runs_dry(seed):
    rng = random.Random(seed)
    shapes = [
        [MAX_CODE_BITS] * STREAM_MAX,
        [1] * STREAM_MAX,
        [rng.randint(1, MAX_CODE_BITS) for _ in range(STREAM_MAX)],
        [rng.choice((1, 1, 1, 11, 12)) for _ in range(STREAM_MAX)],
    ]
    for lengths in shapes:
        for head in (0, 1, 31):
            n = (STREAM_MAX - head) // 32 * 32
            r, unread = run_head(lengths[:head], 17, 5)
            assert 1 <= run_lane(lengths[head: head + n], r, unread) <= 8


@pytest.mark.parametrize("threads", [64, 256])
def test_ring_slot_from_the_bit_count(threads):
    """HUFD_ADVANCE: slot byte offset ((r * (S / 32) + kBase * S) & (7 * S)) == ((kBase + (r >> 5)) & 7) * S, S = threads * 4,
    for every bit count a 131,072-symbol stream of 12-bit codes can reach (u32 arithmetic)"""
    S = threads * 4
    for kbase in range(0, 9):
        for r in list(range(0, 4096)) + list(range(STREAM_MAX * MAX_CODE_BITS - 4096, STREAM_MAX * MAX_CODE_BITS + 64)):
            got = ((r * (S // 32) + kbase * S) & 0xFFFFFFFF) & (7 * S)
            assert got == ((kbase + (r >> 5)) & 7) * S


def test_counters_fit_u32():
    # decoder: expectBits = 8 * (chunkTop - streamStart) < 8 * (128 KB + 32); emit kernel: bitpos < 8 * 15 + 12 * 128 KB + 1
    assert 8 * (STREAM_MAX + 32) < 2 ** 32 and 8 * 15 + MAX_CODE_BITS * STREAM_MAX + 1 < 2 ** 32
    # plan kernel: the four u16 segment counts of a symbol add up to at most 131,072 in u32
    assert 4 * 32768 <= STREAM_MAX < 2 ** 32


def test_stream_paths_1x():
    assert stream_paths_1x("A", 400, 0) == [(0, 12, 16)]
    assert stream_paths_1x("A", 400, 5) == [(27, 11, 21)]
    assert stream_paths_1x("hard", 400, 0) == [(0, 0, 400)]
    assert stream_paths_1x("B", 40, 1) == [(0, 0, 40)]                   # 31 head symbols leave less than a sector
    assert stream_paths_1x("A", 63, 1) == [(31, 1, 0)]
    assert [stream_kind(*s) for s in stream_paths_1x("A", STREAM_MAX, 3)] == ["head+fast"]
    assert [stream_kind(*s) for s in stream_paths_1x("B", STREAM_MAX, 0)] == ["fast"]


def test_pass_a_spread_and_emit_group():
    assert pass_a_spread_1x(100, 132) == (64, 1)
    assert pass_a_spread_1x(5 * 132 * 64 + 1, 132)[1] == 2
    assert emit_group_1x(0, 32768) == "g256" and emit_group_1x(1, 3) == "g128" and emit_group_1x(0, 7) == "bytes"
