"""The edge between the two pair routes of the chain stage (raven_b200/csrc/map.cu):
GroupChainKernel chains pairs of up to kThreadPairMax = 63 hits one thread per pair,
PairChainKernel the larger ones one CTA per pair. Pairs on both sides of the 48 and 63 hit
class bounds, on both strands, and pairs of those sizes with several bands, merging bands,
gap splits, hits on one diagonal and chains around the length and match thresholds go
through rvn_dist_chain; each read's overlaps, in emission order, are compared with ram's
Chain (oracle)."""
import numpy as np
import pytest

from test_chain_host import DEFAULT, TIGHT, make_pair
from test_gpu_chain_routes import chain_on_gpu, make_read

pytestmark = pytest.mark.gpu

K_THREAD_PAIR_MAX = 63  # kThreadPairMax


def read_of(rng, parts, noise_pairs=10):
    """one read of the given pairs (group, positions) and noise pairs of 1 to 3 hits"""
    rhs = 1000 + len(parts)
    for i in range(noise_pairs):
        parts = parts + [make_pair(rng, int(rng.integers(1, 4)), i & 1, rhs_id=rhs + i,
                                   noise=1.0)]
    g = np.concatenate([q[0] for q in parts])
    p = np.concatenate([q[1] for q in parts])
    order = rng.permutation(g.size)
    return g[order], p[order]


def test_thread_route_edge_both_strands(oracle):
    """48/49 (two thread classes) and 63/64 (thread route / CTA route), each size on both
    strands: one read per size and one read holding all of them."""
    rng = np.random.default_rng(11)
    sizes = (48, 49, 56, K_THREAD_PAIR_MAX, K_THREAD_PAIR_MAX + 1)
    reads = [make_read(rng, 2 * m + 30, [m, m], noise_pairs=10) for m in sizes]
    reads.append(make_read(rng, 2 * sum(sizes) + 200, [m for m in sizes for _ in (0, 1)],
                           noise_pairs=100))
    assert chain_on_gpu(oracle, reads) >= 2 * len(sizes)


@pytest.mark.parametrize("prm", [DEFAULT, TIGHT], ids=["default", "tight"])
def test_thread_route_edge_bands(oracle, prm):
    """Pairs of 49 to 64 hits with several bands (runs on diagonals further apart than the
    bandwidth), bands that merge (runs closer than it), runs whose lhs gaps split a band
    into several overlaps, hits all on one diagonal, and chains just below, at and above
    the chain length and around the matches threshold."""
    rng = np.random.default_rng(12)
    bw = prm["bandwidth"]
    reads = []
    for strand in (0, 1):
        pairs = []
        for m in (49, 56, 63, 64):
            pairs.append(make_pair(rng, m, strand, rhs_id=len(pairs) + 1, runs=3,
                                   spread=3 * bw))                         # separate bands
            pairs.append(make_pair(rng, m, strand, rhs_id=len(pairs) + 1, runs=3,
                                   spread=bw // 3))                        # merging bands
            pairs.append(make_pair(rng, m, strand, rhs_id=len(pairs) + 1, runs=4,
                                   step=prm["gap"] // 8, jitter=0))        # gap splits
            pairs.append(make_pair(rng, m, strand, rhs_id=len(pairs) + 1, jitter=0,
                                   noise=0.0))                             # one diagonal
        reads.append(read_of(rng, pairs))
        near = []
        for m in (49, 63):
            for true in (prm["chain"] - 1, prm["chain"], prm["chain"] + 1):
                near.append(make_pair(rng, m, strand, rhs_id=len(near) + 1,
                                      noise=1 - true / m))
            for step in (prm["matches"] // 24, prm["matches"] // 18, prm["matches"] // 12):
                near.append(make_pair(rng, m, strand, rhs_id=len(near) + 1,
                                      step=max(step, 1), noise=0.0))
        reads.append(read_of(rng, near))
    assert chain_on_gpu(oracle, reads, prm) > 20
