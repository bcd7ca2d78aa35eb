"""Multiplicities of the bare keys of a tiered index (index.cu): one unstable partition
pass + BareCountKernel (engine option bare_count 1, and cluster size 8 forced) against
two stable radix passes + GroupCountKernel (bare_count 0). Tiers are forced on with
tier_min_records 0. For each case the stage-1 results, stats()["index_keys"] and the
occurrence thresholds filter(f) of the same index are identical over both paths, and
the thresholds match the CPU oracle's Filter where the index holds every read.

Cases: the lambda reads; a small set shaped like the benchmark's (40x coverage of 10 kb
reads); k = 9 (18-bit keys: one bucket, no partition), 11, 13, 15 with w = 5;
near-identical reads and tandem repeats (multiplicities past 255); 70 000 copies of one
read (runs of 65 535 postings and more: the long-run fallback sorts the bare keys
fully); several index batches and flushes."""
import numpy as np
import pytest

from raven_b200 import seqio, synth

pytestmark = pytest.mark.gpu

FREQS = (0.0, 0.0005, 0.001, 0.002, 0.01, 0.5)
PATHS = (0, 1, 8)


def repeat_reads():
    rng = np.random.default_rng(43)
    seqs = []
    for unit_len, copies in ((2000, 300), (1500, 90)):
        unit = rng.integers(0, 4, unit_len, dtype=np.uint8)
        for _ in range(copies):
            s = unit.copy()
            at = rng.integers(0, unit_len, 4)
            s[at] = (s[at] + rng.integers(1, 4, 4)) % 4
            seqs.append(s)
    tile = rng.integers(0, 4, 40, dtype=np.uint8)
    for n in (300, 280, 310):
        seqs.append(np.tile(tile, n))
    seqs += [rng.integers(0, 4, 2000, dtype=np.uint8) for _ in range(60)]
    order = rng.permutation(len(seqs))
    return seqio.pack_codes([seqs[i] for i in order])


def long_run_reads():
    rng = np.random.default_rng(31)
    one = rng.integers(0, 4, 90, dtype=np.uint8)
    return seqio.pack_codes([one] * 70_000 +
                            [rng.integers(0, 4, 400, dtype=np.uint8) for _ in range(50)])


def check_paths(gpu_engine, oracle, rs, k, stage1_freq=0.001, ib=0, qb=0):
    gpu_engine.configure(k=k, w=5)
    gpu_engine.upload(rs)
    gpu_engine.set_option("tier_min_records", 0)
    seen = {}
    try:
        for bare in PATHS:
            gpu_engine.set_option("bare_count", bare)
            got = gpu_engine.find_overlaps_and_create_piles(stage1_freq, 8, False, ib, qb)
            keys = gpu_engine.stats()["index_keys"]
            occ = [gpu_engine.filter(f) for f in FREQS]
            seen[bare] = (got, keys, occ)
    finally:
        gpu_engine.set_option("bare_count", 1)
        gpu_engine.set_option("tier_min_records", 1 << 18)
    for bare in PATHS[1:]:
        for key in ("overlaps", "ovl_off", "pile", "pile_off"):
            assert np.array_equal(seen[bare][0][key], seen[0][0][key]), (bare, key)
        assert seen[bare][0]["num_mapped"] == seen[0][0]["num_mapped"]
        assert seen[bare][1] == seen[0][1], bare
        assert seen[bare][2] == seen[0][2], bare
    if ib == 0:  # the index holds every read: the oracle's engine over all of them
        eng = oracle.engine(k, 5, threads=8)
        oracle.minimize(eng, oracle.reads(rs), 0, rs.n, False)
        assert seen[1][1] == int(oracle.keys(eng)["totals"][0])
        assert seen[1][2] == [oracle.filter(eng, f) for f in FREQS]
    return seen


def test_bare_counts_lambda(gpu_engine, oracle, lambda_reads):
    check_paths(gpu_engine, oracle, lambda_reads, 15)


def test_bare_counts_bench_shaped(gpu_engine, oracle):
    rs = synth.make_reads(1_000_000, 4000, 10_000, seed=5)
    check_paths(gpu_engine, oracle, rs, 15)


@pytest.mark.parametrize("k", [9, 11, 13, 15])
def test_bare_counts_key_widths(gpu_engine, oracle, k):
    rs = synth.make_reads(300_000, 400, 5000, seed=7)
    check_paths(gpu_engine, oracle, rs, k)


def test_bare_counts_repeats(gpu_engine, oracle):
    seen = check_paths(gpu_engine, oracle, repeat_reads(), 15)
    assert any(255 < o < 0xFFFFFFFF for o in seen[1][2]), seen[1][2]


def test_bare_counts_very_long_runs(gpu_engine, oracle):
    seen = check_paths(gpu_engine, oracle, long_run_reads(), 15, stage1_freq=0.5)
    assert seen[1][2][1] > 65_535, seen[1][2]   # f = 0.0005 ranks among the long runs


@pytest.mark.parametrize("ib,qb", [(120_000, 50_000), (250_000, 120_000)])
def test_bare_counts_index_batches(gpu_engine, oracle, ib, qb):
    rs = synth.make_reads(300_000, 400, 5000, seed=11)
    check_paths(gpu_engine, oracle, rs, 15, ib=ib, qb=qb)
    rs = repeat_reads()
    check_paths(gpu_engine, oracle, rs, 15, ib=ib, qb=qb)
