"""Windowed stage 1 (option "stage1_window"): the piles and overlap lists of all reads stay
on the host and each flush brings only the reads it touches to the device. Every result
must be bit-identical to the resident pass and to the oracle: golden files, schedules with
many index batches and flushes (flushes wholly before the batch and flushes that straddle
its first read), kmax 4 / 8 / 32, both -M modes, tiers forced on, the probe path, saturated
piles, the pile regions of TrimAndAnnotatePiles, and the auto mode's choice."""
import json
import os

import numpy as np
import pytest

from raven_b200 import seqio, synth

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
META = json.load(open(os.path.join(HERE, "golden", "lambda_golden.json")))
GOLD = np.load(os.path.join(HERE, "golden", "lambda_golden.npz"))
KEYS = ("overlaps", "ovl_off", "pile", "pile_off")

SCHEDULES = [
    dict(genome_len=80_000, n_reads=300, mean_len=4000, seed=2, kmax=32, ib=0, qb=0),
    dict(genome_len=30_000, n_reads=150, mean_len=3000, seed=3, kmax=8, ib=120_000, qb=50_000),
    dict(genome_len=30_000, n_reads=150, mean_len=3000, seed=4, kmax=4, ib=1 << 40, qb=70_000),
]


@pytest.fixture
def windowed(gpu_engine):
    gpu_engine.set_stage1_window(1)
    try:
        yield gpu_engine
    finally:
        gpu_engine.set_stage1_window(-1, 0)
        gpu_engine.set_option("tier_min_records", 1 << 18)
        gpu_engine.set_option("self_join", 1)
        gpu_engine.configure(k=15, w=5)


def stage1(eng, *args):
    got = eng.find_overlaps_and_create_piles(*args)
    return got, eng.stage1_windowed()


def same(got, want, tag):
    for k in KEYS:
        assert np.array_equal(got[k], want[k]), (tag, k)
    assert got["num_mapped"] == int(np.asarray(want["num_mapped"]).ravel()[0]), tag


@pytest.mark.parametrize("minhash", [False, True])
def test_window_lambda_golden(windowed, lambda_reads, minhash):
    windowed.configure(k=15, w=5)
    windowed.upload(lambda_reads)
    tag = "minhash" if minhash else "plain"
    # one batch, one flush; then many batches and flushes, against the resident pass
    got, win = stage1(windowed, 0.001, 32, minhash)
    assert win
    for k in KEYS:
        assert np.array_equal(got[k], GOLD[f"stage1_{tag}_{k}"]), k
    assert got["num_mapped"] == META[f"stage1_{tag}_num_mapped"]
    got, win = stage1(windowed, 0.001, 16, minhash, 400_000, 150_000)
    assert win
    windowed.set_stage1_window(0)
    want, win = stage1(windowed, 0.001, 16, minhash, 400_000, 150_000)
    assert not win
    same(got, want, tag)


@pytest.mark.parametrize("cfg", SCHEDULES)
def test_window_synthetic_schedules(windowed, oracle, cfg):
    rs = synth.make_reads(cfg["genome_len"], cfg["n_reads"], cfg["mean_len"], seed=cfg["seed"])
    windowed.configure(k=15, w=5)
    windowed.upload(rs)
    for minhash in (False, True):
        got, win = stage1(windowed, 0.001, cfg["kmax"], minhash, cfg["ib"], cfg["qb"])
        assert win
        want = oracle.stage1(oracle.engine(15, 5, threads=4), oracle.reads(rs), 0.001,
                             cfg["kmax"], minhash, cfg["ib"] or 1 << 32, cfg["qb"] or 1 << 30)
        same(got, want, minhash)


def test_window_many_batches_and_flushes(windowed, oracle):
    """Small index and query batches: most flushes lie wholly before their index batch
    (a window of two ranges), others straddle its first read or lie inside it."""
    rs = synth.make_reads(40_000, 200, 3000, seed=17)
    windowed.configure(k=15, w=5)
    windowed.upload(rs)
    for kmax, ib, qb in ((4, 90_000, 40_000), (8, 150_000, 25_000), (32, 60_000, 100_000)):
        got, win = stage1(windowed, 0.001, kmax, False, ib, qb)
        assert win
        want = oracle.stage1(oracle.engine(15, 5, threads=4), oracle.reads(rs), 0.001, kmax,
                             False, ib, qb)
        same(got, want, (kmax, ib, qb))


def test_window_tiers_and_probe_path(windowed, oracle, lambda_reads):
    """The tiered index forced on (tier_min_records 0) and the probe path (self_join 0)."""
    rs = synth.make_reads(30_000, 160, 3000, seed=9)
    for tiers, join in ((0, 1), (1 << 18, 0), (0, 0)):
        windowed.set_option("tier_min_records", tiers)
        windowed.set_option("self_join", join)
        windowed.configure(k=15, w=5)
        windowed.upload(lambda_reads)
        got, win = stage1(windowed, 0.001, 32, False)
        assert win
        for k in KEYS:
            assert np.array_equal(got[k], GOLD[f"stage1_plain_{k}"]), (tiers, join, k)
        windowed.upload(rs)
        for freq, ib, qb in ((0.02, 150_000, 60_000), (0.3, 0, 100_000)):
            got, win = stage1(windowed, freq, 8, False, ib, qb)
            assert win
            want = oracle.stage1(oracle.engine(15, 5, threads=4), oracle.reads(rs), freq, 8,
                                 False, ib or 1 << 32, qb or 1 << 30)
            same(got, want, (tiers, join, freq))


def high_coverage_reads():
    """Twelve copies each of four reads. With chains split at gaps above 3 bases, copies
    overlap in pieces of about 20 bases; a piece shorter than two bins drives the running
    coverage below zero, which the reference's unsigned add turns into a bin clamped at
    65535."""
    rng = np.random.default_rng(5)
    base = [rng.integers(0, 4, int(n), dtype=np.uint8) for n in (2200, 2600, 3100, 3500)]
    seqs = [base[i % 4].copy() for i in range(48)]
    return seqio.pack_codes(seqs)


def test_window_saturated_piles(windowed, oracle):
    rs = high_coverage_reads()
    prm = dict(bandwidth=500, chain=2, matches=15, gap=3)
    windowed.configure(k=15, w=5, **prm)
    windowed.upload(rs)
    for kmax, ib, qb in ((4, 0, 0), (8, 40_000, 15_000)):
        got, win = stage1(windowed, 0.0, kmax, False, ib, qb)
        assert win
        want = oracle.stage1(oracle.engine(15, 5, threads=4, **prm), oracle.reads(rs), 0.0,
                             kmax, False, ib or 1 << 32, qb or 1 << 30)
        same(got, want, (kmax, ib))
        windowed.set_stage1_window(0)
        res, win = stage1(windowed, 0.0, kmax, False, ib, qb)
        assert not win
        same(res, want, (kmax, ib))
        windowed.set_stage1_window(1)
        # one flush leaves the bins clamped; a later flush's wrapped add takes them below
        # 65535 again (65535 + 2^32 - 8), exactly as the reference's unsigned sum does
        assert got["pile"].max() >= 65520
        if qb == 0:
            assert got["pile"].max() == 65535


def test_window_pile_regions(windowed):
    """rvn_stage1_pile_regions after a windowed pass (the piles are on the host and pass
    through the device in chunks) equals the regions after a resident pass."""
    from raven_b200 import engine
    rs = synth.make_reads(40_000, 300, 5000, seed=14)
    windowed.configure(k=15, w=5)
    windowed.upload(rs)
    # a fresh context: its pile buffer holds one window, so the regions take several chunks
    fresh = engine.Engine(device=0)
    try:
        fresh.configure(k=15, w=5)
        fresh.upload(rs)
        fresh.set_stage1_window(1)
        for eng, ib, qb in ((windowed, 0, 0), (fresh, 250_000, 100_000)):
            windowed.set_stage1_window(0)
            windowed.find_overlaps_and_create_piles(0.001, 32, False, ib, qb)
            want = {cov: windowed.stage1_pile_regions(cov) for cov in (4, 1, 9, 30)}
            eng.set_stage1_window(1)
            eng.find_overlaps_and_create_piles(0.001, 32, False, ib, qb)
            assert eng.stage1_windowed()
            for cov, w in want.items():
                got = eng.stage1_pile_regions(cov)
                for k in ("invalid", "begin", "end", "median"):
                    assert np.array_equal(got[k], w[k]), (ib, cov, k)
            assert (got["invalid"] == 0).sum() > 100
        fresh.upload(rs)
        with pytest.raises(RuntimeError):   # a new read set: no stage-1 piles any more
            fresh.stage1_pile_regions(4)
    finally:
        fresh.close()


def test_window_auto_mode(windowed, oracle):
    """Auto (the default) stays resident where the estimate fits, goes windowed under a
    budget that only the windowed pass fits, and stays resident under one that neither
    fits; the same result every time."""
    rs = synth.make_reads(30_000, 150, 3000, seed=3)
    windowed.configure(k=15, w=5)
    windowed.upload(rs)
    windowed.set_stage1_window(-1, 0)
    want, win = stage1(windowed, 0.001, 8, False, 120_000, 50_000)
    assert not win
    fp = windowed.stage1_footprint(8, 120_000, 50_000)
    assert 0 < fp["windowed_device"] < fp["resident"] and fp["windowed_host"] > 0
    windowed.set_stage1_window(-1, (fp["windowed_device"] + fp["resident"]) // 2)
    got, win = stage1(windowed, 0.001, 8, False, 120_000, 50_000)
    assert win
    same(got, want, "auto")
    windowed.set_stage1_window(-1, fp["windowed_device"] // 2)   # neither fits
    got, win = stage1(windowed, 0.001, 8, False, 120_000, 50_000)
    assert not win
    same(got, want, "auto, nothing fits")
    windowed.set_stage1_window(0, 1 << 20)   # forced resident ignores the budget
    got, win = stage1(windowed, 0.001, 8, False, 120_000, 50_000)
    assert not win
    same(got, want, "resident")
    with pytest.raises(ValueError):
        windowed.set_option("stage1_window", 2)
    with pytest.raises(OverflowError):   # rows of max_overlaps records per read
        windowed.set_stage1_window(1)
        windowed.find_overlaps_and_create_piles(0.001, 1 << 20, False)


def test_window_auto_keeps_large_max_overlaps_resident(windowed):
    """A max_overlaps far above what any list holds (no truncation) must not push auto
    into the windowed mode, which cannot take it: 10 k short reads at max_overlaps 2^20
    run resident, with the free memory as the budget and with a tiny one."""
    rs = synth.make_reads(300_000, 10_000, 600, seed=23)
    windowed.configure(k=15, w=5)
    windowed.upload(rs)
    windowed.set_stage1_window(0)
    want, win = stage1(windowed, 0.001, 1 << 20, False)
    assert not win
    fp = windowed.stage1_footprint(1 << 20)
    assert fp["resident"] < 64 << 30   # lists bounded by one overlap per other read
    for budget in (0, 1 << 20):
        windowed.set_stage1_window(-1, budget)
        got, win = stage1(windowed, 0.001, 1 << 20, False)
        assert not win, budget
        same(got, want, budget)
