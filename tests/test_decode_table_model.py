"""Host-side model of the Huff0 decoder's unified per-block table (finitestateentropy_b200/csrc/huf_decode.cu, setup_block and
HUFD_LOOKUP): rows [0, CUT) hold full-resolution cells for the windows that start a code longer than M bits, rows >= CUT the M-bit
first level minus its never-used head, and the row of window x is min(x, D + (x >> (tableLog - M))) with D = CUT - (CUT >> (tableLog - M)).
Checked here for random canonical codes: every window decodes to the same (length, symbol) as the full 2^tableLog table, for every
split the kernel may pick, and the row count is the one the kernel budgets.  CPU only."""
import random

import pytest

from paths import split_candidates, table_rows


def random_code_lengths(rng, nsym, max_len=12):
    """a complete prefix code with nsym leaves, no code longer than max_len: split random leaves of a one-leaf tree"""
    lengths = [0]
    while len(lengths) < nsym:
        cand = [i for i, n in enumerate(lengths) if n < max_len]
        i = rng.choice(cand) if rng.random() < 0.5 else max(cand, key=lambda j: (lengths[j], rng.random()))   # skewed: deepen the deepest
        lengths[i] += 1
        lengths.append(lengths[i])
    rng.shuffle(lengths)
    return lengths


def full_table(lengths):
    """Huff0's canonical order (lib/huf_decompress.c:151-183): weight ascending = longest codes first, symbols ascending within."""
    tl = max(lengths)
    cells = []
    for w in range(1, tl + 1):                              # weight w <-> length tl + 1 - w, 2^(w-1) cells per symbol
        for s, n in enumerate(lengths):
            if tl + 1 - n == w:
                cells += [(n, s)] * (1 << (w - 1))
    assert len(cells) == 1 << tl
    return tl, cells


@pytest.mark.parametrize("seed", range(12))
def test_unified_table_rows_decode_like_the_full_table(seed):
    rng = random.Random(seed)
    for nsym in (2, 3, 17, 60, 130, 256):
        lengths = random_code_lengths(rng, nsym)
        tl, full = full_table(lengths)
        rank_end = [0] * (tl + 2)                           # end of weight w's range in tableLog-bit index space
        acc = 0
        for w in range(1, tl + 1):
            acc += sum(1 for n in lengths if tl + 1 - n == w) << (w - 1)
            rank_end[w] = acc
        best = 1 << tl
        for m, cut, rows in split_candidates(rank_end, tl):   # the kernel's candidates: first level of m bits, 4 <= m < tableLog
            best = min(best, rows)
            d = cut - (cut >> (tl - m))
            table = [full[r] if r < cut else full[(r - d) << (tl - m)] for r in range(rows)]
            for x in range(1 << tl):
                row = min(x - d, x >> (tl - m)) + d         # the kernel's signed minimum
                assert row == min(x, d + (x >> (tl - m))) and 0 <= row < rows
                assert table[row] == full[x], (nsym, m, x)
        assert best <= 1 << tl and table_rows(rank_end, tl)[0] == best
