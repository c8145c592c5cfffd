"""FSEB200_HUF_compress_literals_chains_packed (-m gpu): packed Huff0 chains under zstd's literal-coding policy, against the policy
loop over the compiled reference (huf_literals_chain_cases.py).

Every value, kind, form flag, offset and stored byte, and every final table, flag and chain header, at both main configurations
and (minLiterals, minGainLog) in {(64, 6), (8, 8), (1, 1)}, on the chain tests' chains with entry flags 0, 1, 2, ragged
literal-like chains and the chains built for each rule; capacities cut at block ends; one chain cut into two calls; malformed
geometry; a side stream; one chain of 4,096 blocks; the round trip through FSEB200_HUF_decompress_mixed_repeat_packed with the
form flags the call wrote."""
import numpy as np
import pytest
import torch

from helpers import is_error
from huf_repeat_cases import main_configs
from huf_chain_packed_cases import at_bound, resolve_headers
from huf_literals_chain_cases import literal_chains, built_chains, long_literal_chain, POLICIES
from huf_chain_harness import (MIXED, PackedChains, literals, decode, regenerable, _ref, _t, _u64, _view, FILL, SRC_WRONG,
                               TOO_SMALL)
import finitestateentropy_b200 as fb

pytestmark = pytest.mark.gpu


def round_trip(run, out, off, kinds, forms, stream=None):
    """the mixed packed decoder with the written forms; every regenerable block comes back.  Returns the count."""
    res, regions = decode(MIXED, _t(run.starts), out, _t(off), _t(kinds, torch.uint8), _t(forms, torch.uint8), _view(run.chp),
                          _view(run.chs), run.sizes, stream=stream)
    heads = resolve_headers(kinds, run.starts)
    ok = 0
    for k, (c, i) in enumerate(run.blocks):
        if not regenerable(run, k, heads):
            continue
        src = run.chains[c]["blocks"][i]["src"]
        if int(res[k]) != len(src) and not is_error(int(res[k])):
            raise AssertionError((run.chains[c]["name"], i))
        if is_error(int(res[k])):
            continue                                                # the weight-12 exception: the decoder refuses the header
        assert (regions[k] == src).all(), (run.chains[c]["name"], i, kinds[k])
        ok += 1
    return ok


@pytest.mark.parametrize("policy", POLICIES, ids=["64_6", "8_8", "1_1"])
@pytest.mark.parametrize("msv,tlog", main_configs())
def test_compress_matches_the_policy_loop(msv, tlog, policy):
    ref = _ref()
    run = PackedChains(literals(*policy), ref, literal_chains(ref, msv, tlog, seed=policy[1]), msv, tlog)
    assert {0, 1, 2, 3, 4} <= set(run.kinds) and set(run.flags) == {0, 1}
    res = run.call(stream=torch.cuda.Stream())
    run.check_one_call(res)
    run.reset()
    _, out, off, cs, kinds, forms, _ = res
    assert round_trip(run, out, off, kinds, forms) > 200


def test_built_chains_at_every_policy():
    """the built chains alone, so that a rule's block is compared at every policy and not only among many chains"""
    ref = _ref()
    for policy in POLICIES + ((0, 6), (16, 7)):
        run = PackedChains(literals(*policy), ref, built_chains(ref), 255, 11)
        res = run.call()
        run.check_one_call(res)
        run.reset()
        round_trip(run, res[1], res[2], res[4], res[5])


def test_capacity_at_block_ends():
    ref = _ref()
    run = PackedChains(literals(8, 8), ref, literal_chains(ref, 255, 11)[::17] + built_chains(ref), 255, 11)
    whole = run.call()
    run.check_one_call(whole)
    ends = whole[2]
    total = int(ends[-1])
    for k in range(1, len(ends) - 1, max(1, len(ends) // 7)):
        for cap in (int(ends[k]) - 1, int(ends[k]), int(ends[k]) + 1):
            if cap < 1 or cap >= total:
                continue
            run.reset()
            before = run.state()
            buf, out, off, cs, kinds, forms, idx = run.call(cap=cap)
            assert (off == ends).all() and list(forms) == run.flags
            host = buf.cpu().numpy()
            o0 = out.data_ptr() - buf.data_ptr()
            assert (host[:o0] == FILL).all() and (host[o0 + cap:] == FILL).all()
            for b in range(len(idx)):
                if run.kinds[b] == 4:
                    assert int(cs[b]) == run.vals[b] and kinds[b] == 4
                elif int(ends[b + 1]) <= cap:
                    assert int(cs[b]) == run.vals[b] and kinds[b] == run.kinds[b]
                    assert (host[o0 + int(off[b]):o0 + int(off[b + 1])] == run.blobs[b]).all()
                else:
                    assert int(cs[b]) == TOO_SMALL and kinds[b] == 4, (b, cap)
            after = run.state()
            for key in before:
                assert (before[key] == after[key]).all(), key
    run.reset()
    run.check_one_call(run.call(cap=total))


def test_split_calls_carry_the_state():
    """each chain cut into two calls right after a block the policy rolled back: the second call's results equal one call's"""
    ref = _ref()
    chains = built_chains(ref)
    one = PackedChains(literals(8, 8), ref, chains, 255, 11)
    one.check_one_call(one.call())
    two = PackedChains(literals(8, 8), ref, chains, 255, 11)
    mids = [max(1, len(ch["blocks"]) // 2) if len(ch["blocks"]) > 1 else 1 for ch in chains]
    rolled = [k for k in range(len(one.blocks)) if one.blocks[k][1] == mids[one.blocks[k][0]] - 1 and one.kinds[k] == 0
              and chains[one.blocks[k][0]]["name"].startswith("rollback")]
    a = two.call(parts=[(0, m) for m in mids])
    b = two.call(parts=[(m, len(ch["blocks"])) for m, ch in zip(mids, chains)])
    s1, s2 = one.state(), two.state()
    for key in ("tabs", "rep", "chs"):
        assert (s1[key] == s2[key]).all(), key
    got = {}
    for buf, out, off, cs, kinds, forms, idx in (a, b):
        host = out.cpu().numpy()
        for j, k in enumerate(idx):
            got[k] = (int(cs[j]), int(kinds[j]), int(forms[j]), host[int(off[j]):int(off[j + 1])])
    for k in range(len(one.blocks)):
        v, kd, f, data = got[k]
        assert (v, kd, f) == (one.vals[k], one.kinds[k], one.flags[k]) and (data == one.blobs[k]).all(), k
    assert rolled, "a chain cut right after a rolled-back block"


def test_malformed_geometry_writes_only_values_and_kinds():
    ref = _ref()
    run = PackedChains(literals(64, 6), ref, built_chains(ref), 255, 12)
    nb = len(run.blocks)
    good = run.starts
    before = run.state()
    for st in ([1] + good[1:], good[:-1] + [nb - 1], good[:3] + [good[2] - 1] + good[4:]):
        buf, out, off, cs, kinds, forms, _ = run.call(starts=st)
        assert (cs == SRC_WRONG).all() and (kinds == 4).all() and (forms == 0xEE).all()
        assert (off == 0xCD).all()
        assert (buf.cpu().numpy() == FILL).all()
        after = run.state()
        for k in before:
            assert (before[k] == after[k]).all(), k


def test_ordered_on_a_side_stream():
    ref = _ref()
    run = PackedChains(literals(64, 6), ref, built_chains(ref) + literal_chains(ref, 255, 11)[::29], 255, 11)
    s = torch.cuda.Stream()
    saved = run.srcs.dev.clone()
    with torch.cuda.stream(s):
        run.srcs.dev.zero_()
        torch.cuda._sleep(20_000_000)
        run.srcs.dev.copy_(saved)
        out, off, cs, kinds, forms = fb.huf_compress_literals_chains_packed(
            _t(run.starts), run.sp, run.ss, run.pr, _view(run.ctp), _view(run.rep), _view(run.chp), _view(run.chs),
            out=torch.empty(sum(run.sizes) + 32, dtype=torch.uint8, device="cuda"), max_symbol_value=255, table_log=11)
        copies = (cs.clone(), kinds.clone(), forms.clone())
    s.synchronize()
    assert (_u64(copies[0]) == np.array(run.vals, np.uint64)).all()
    assert list(copies[1].cpu().numpy()) == run.kinds and list(copies[2].cpu().numpy()) == run.flags
    run.reset()
    assert round_trip(run, out, _u64(off), copies[1].cpu().numpy(), copies[2].cpu().numpy(), stream=s) > 20


def test_one_chain_of_4096_blocks():
    ref = _ref()
    run = PackedChains(literals(64, 6), ref, at_bound([long_literal_chain(ref, 4096)]), 255, 11)
    assert len(run.blocks) == 4096
    res = run.call()
    run.check_one_call(res)
    assert run.kinds.count(3) > 1000 and run.kinds.count(2) >= 1 and run.kinds.count(0) > 100
    run.reset()
    _, out, off, cs, kinds, forms, _ = res
    assert round_trip(run, out, off, kinds, forms) > 3000
