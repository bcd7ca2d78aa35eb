"""Every route a read can take through the chain stage (raven_b200/csrc/map.cu). Crafted
hit sets go through rvn_dist_chain with one part, and each read's overlaps, in emission
order, are compared with ram's Chain (oracle). The reads are built from map.cu's
constants so that they land on both sides of every size class and fallback edge."""
import numpy as np
import pytest
import torch

from raven_b200 import distributed, engine, synth
from test_chain_host import DEFAULT, make_pair

pytestmark = pytest.mark.gpu

K_CHAIN_SMEM_CAP = 65535  # kChainSmemCap
K_SPLIT_MAX_TABLE = 8192  # kSplitMaxTable
K_PAIR_MAX_HITS = 8191    # kPairMaxHits


def make_read(rng, n, pairs, rhs0=1, noise_pairs=None):
    """A read of exactly n hits: pairs of the given sizes (alternating strands), then
    noise_pairs pairs of 1 to 3 random hits (by default as few as fill it up)."""
    parts = [make_pair(rng, m, i & 1, rhs_id=rhs0 + i) for i, m in enumerate(pairs)]
    left = n - sum(pairs)
    noise_pairs = (left + 1) // 2 if noise_pairs is None else noise_pairs
    assert noise_pairs <= left <= 3 * noise_pairs
    sizes = 1 + rng.multivariate_hypergeometric([2] * noise_pairs, left - noise_pairs)
    for i, s in enumerate(sizes):
        parts.append(make_pair(rng, int(s), i & 1, rhs_id=rhs0 + len(pairs) + i, noise=1.0))
    g = np.concatenate([q[0] for q in parts] + [np.zeros(0, np.uint64)])
    p = np.concatenate([q[1] for q in parts] + [np.zeros(0, np.uint64)])
    assert g.size == n
    order = rng.permutation(n)
    return g[order], p[order]


def chain_on_gpu(oracle, reads, prm=DEFAULT):
    """rvn_dist_chain over the reads (read r = query r), against the oracle read by read."""
    n = len(reads)
    eng = engine.Engine(device=0)
    try:
        eng.configure(**prm)
        eng.upload(synth.make_reads(20_000, n, 800, seed=1))
        steps = distributed.CudaSteps(eng, "cuda:0")
        g = np.concatenate([r[0] for r in reads])
        p = np.concatenate([r[1] for r in reads])
        lhs = np.repeat(np.arange(n, dtype=np.uint32), [r[0].size for r in reads])
        dev = lambda a, t: torch.from_numpy(a.view(t)).to("cuda:0")
        steps.chain(dev(g, np.int64), dev(p, np.int64), dev(lhs, np.int32), [g.size], 1, 0, n)
        ovl, _ = steps.overlaps_split(1, 0)
        got = distributed._as_torch(ovl).cpu().numpy().view(np.uint32).reshape(-1, 8)
    finally:
        eng.close()
    oe = oracle.engine(**prm)
    total = 0
    for r, (rg, rp) in enumerate(reads):
        want = oracle.chain(oe, r, rg, rp)
        mine = got[got[:, 0] == r]
        assert np.array_equal(mine, want), f"read {r} ({rg.size} hits)"
        total += want.shape[0]
    assert total == got.shape[0]
    assert np.array_equal(got[:, 0], np.sort(got[:, 0], kind="stable"))
    return total


def test_thread_pair_class_edges(oracle):
    """GroupChainKernel chains pairs of up to kThreadPairMax = 48 hits, one launch per
    class of kPairBounds (8, 16, 24, 32, 48): pairs of 4 (the smallest kept), 8/9, 16/17,
    24/25, 32/33 and 48 hits, one read each, among noise pairs of fewer than 4 hits."""
    rng = np.random.default_rng(1)
    reads = [make_read(rng, m + 40, [m], noise_pairs=20)
             for m in (4, 8, 9, 16, 17, 24, 25, 32, 33, 48)]
    reads.append(make_read(rng, 400, [4, 8, 9, 16, 17, 24, 25, 32, 33, 48], noise_pairs=100))
    assert chain_on_gpu(oracle, reads) > 10


def test_cta_pair_class_edges(oracle):
    """PairChainKernel chains the pairs above kThreadPairMax = 48 hits, one launch per
    class of kPairBounds (63, 127, ..., 4095, kPairMaxHits = 8191): 49, both sides of
    every class edge, and 8191."""
    rng = np.random.default_rng(2)
    sizes = (49, 63, 64, 127, 128, 255, 256, 511, 512, 1023, 1024, 2047, 2048, 4095, 4096,
             K_PAIR_MAX_HITS)
    reads = [make_read(rng, m + 30, [m], noise_pairs=10) for m in sizes]
    assert chain_on_gpu(oracle, reads) >= len(sizes)


def test_split_kernel_widths(oracle):
    """SplitKernel<128, 8> takes reads of up to 2,047 hits (kSplitBounds 2048), and
    SplitKernel<256, 2> the larger ones: reads of 2,046 to 2,049 hits, and of 255/256
    (a smaller table), each of many pairs."""
    rng = np.random.default_rng(3)
    reads = [make_read(rng, n, [40] * (n // 60))
             for n in (255, 256, 2046, 2047, 2048, 2049)]
    assert chain_on_gpu(oracle, reads) > 10


def test_reads_below_four_hits(oracle):
    """Reads of 0 to 3 hits form no band and are chained by no kernel; a read of 4 is."""
    rng = np.random.default_rng(4)
    reads = [make_read(rng, n, [n] if n else []) for n in (0, 1, 2, 3, 4, 0)]
    chain_on_gpu(oracle, reads)


def test_global_memory_path(oracle):
    """ChainKernelGlobal takes a read for each of three reasons, next to reads of the
    split path: more than kChainSmemCap = 65,535 hits; more distinct pairs than the
    kSplitMaxTable = 8,192 entries of SplitKernel's table; one pair of more than
    kPairMaxHits = 8,191 hits in a read that would otherwise be split."""
    rng = np.random.default_rng(5)
    reads = [
        make_read(rng, 1000, [300, 200, 60]),
        make_read(rng, K_CHAIN_SMEM_CAP + 1, [400] * 150),
        make_read(rng, K_CHAIN_SMEM_CAP, [400] * 150),
        make_read(rng, 3000 + K_SPLIT_MAX_TABLE + 500, [500, 300] + [4] * 50,
                  noise_pairs=K_SPLIT_MAX_TABLE + 200),
        make_read(rng, K_PAIR_MAX_HITS + 1 + 700, [K_PAIR_MAX_HITS + 1, 300]),
        make_read(rng, K_PAIR_MAX_HITS + 700, [K_PAIR_MAX_HITS, 300]),
    ]
    assert chain_on_gpu(oracle, reads) > 10


def test_chain_zero_takes_global_path(oracle):
    """chain = 0 sends every read to ChainKernelGlobal."""
    rng = np.random.default_rng(6)
    reads = [make_read(rng, n, [n - 40, 20]) for n in (64, 500, 3000)]
    assert chain_on_gpu(oracle, reads, dict(DEFAULT, chain=0)) > 0
