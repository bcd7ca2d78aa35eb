"""ChainPairSerial (raven_b200/csrc/chain.cuh) skips the (diagonal, positions) sort of a
pair whose diagonals all lie within the bandwidth: such a pair is one band. Here, on the
host against ram's Chain, pairs whose diagonal span is exactly the bandwidth (one band)
and one more (two windows), with and without hits far off the diagonal, in shuffled
order, and pairs of fewer than four hits, which form no band."""
import numpy as np
import pytest

from test_chain_host import PARAMS, check, diagonal_run, encode, ours  # noqa: F401 (fixture)

# the first diagonal of each strand's runs (as in test_chain_host.make_pair)
BASE = {0: 10_000_000, 1: 50_000}


def two_diagonals(rng, strand, span, n_each, far=0):
    """n_each hits on each of two diagonals span apart (the second run behind the first
    on the lhs, so that both could chain), plus `far` hits 10 bandwidths off; shuffled"""
    d0 = BASE[strand]
    lp = 1000 + np.cumsum(rng.integers(5, 40, 2 * n_each + far))
    parts = [diagonal_run(lp[:n_each], strand, d0),
             diagonal_run(lp[n_each:2 * n_each], strand, d0 + span)]
    if far:
        parts.append(diagonal_run(lp[2 * n_each:], strand, d0 + 5000))
    l = np.concatenate([q[0] for q in parts])
    r = np.concatenate([q[1] for q in parts])
    order = rng.permutation(l.size)
    return encode(9, strand, l[order], r[order])


@pytest.mark.parametrize("strand", [0, 1])
@pytest.mark.parametrize("prm", PARAMS)
def test_diagonal_span_edge(ours, oracle, prm, strand):
    rng = np.random.default_rng(31 + strand)
    bw = prm["bandwidth"]
    found = 0
    for n_each in (2, 3, 10, 30):
        for span in (0, 1, bw - 1, bw, bw + 1, 2 * bw):
            for far in (0, 4):
                found += check(ours, oracle, prm, *two_diagonals(rng, strand, span, n_each, far))
    assert found > 20


@pytest.mark.parametrize("strand", [0, 1])
def test_fewer_than_four_hits(ours, oracle, strand):
    rng = np.random.default_rng(41 + strand)
    prm = PARAMS[0].values[0]
    for m in (0, 1, 2, 3, 4):
        l, r = diagonal_run(1000 + 30 * np.arange(m), strand, BASE[strand])
        order = rng.permutation(m)
        check(ours, oracle, prm, *encode(9, strand, l[order], r[order]))
