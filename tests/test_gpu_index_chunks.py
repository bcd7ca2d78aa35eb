"""Chunked index build (option "index_chunk_bases"): every index batch of stage 1 is built
from chunks of reads, sketched twice, without a sketch of the whole batch. Every result
must be bit-identical to the one-shot build and to the oracle: lists, offsets, piles,
num_mapped, the last batch's index records and key count, and the occurrence threshold.
Tiny sets cut into many chunks give the coverage: chunks of one read, of a third of the
batch and larger than the batch; schedules with many batches and flushes; equal values
across chunk boundaries, chunks without minimizers, chunks denser than the sketch's
capacity estimate; every build route (k15 w5 with tiers sketches straight into them); the
auto decision."""
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


@pytest.fixture
def chunked(gpu_engine):
    try:
        yield gpu_engine
    finally:
        gpu_engine.set_index_chunks(-1, 0)
        gpu_engine.set_stage1_window(-1, 0)
        gpu_engine.set_option("tier_min_records", 1 << 18)
        gpu_engine.set_option("self_join", 1)
        gpu_engine.set_option("bare_count", 1)
        gpu_engine.configure(k=15, w=5)


def stage1(eng, chunk, *args):
    """one pass with option index_chunk_bases = chunk: results, the last batch's index
    records, the occurrence threshold, whether it chunked"""
    eng.set_index_chunks(chunk)
    got = eng.find_overlaps_and_create_piles(*args)
    return got, eng.index_records(), eng.stats()["occurrence"], eng.stage1_index_chunked()


def same(a, b, tag):
    got, idx, occ, _ = a
    want, widx, wocc, _ = b
    for k in KEYS:
        assert np.array_equal(got[k], want[k]), (tag, k)
    assert got["num_mapped"] == want["num_mapped"], tag
    assert idx["n_keys"] == widx["n_keys"], tag
    assert np.array_equal(idx["value"], widx["value"]), tag
    assert np.array_equal(idx["origin"], widx["origin"]), tag
    assert occ == wocc, tag


def same_oracle(a, want, tag):
    got = a[0]
    for k in KEYS:
        assert np.array_equal(got[k], want[k]), (tag, k)
    assert got["num_mapped"] == int(np.asarray(want["num_mapped"]).ravel()[0]), tag


@pytest.mark.parametrize("minhash", [False, True])
def test_chunks_lambda_golden(chunked, lambda_reads, minhash):
    chunked.configure(k=15, w=5)
    chunked.upload(lambda_reads)
    tag = "minhash" if minhash else "plain"
    total = int(lambda_reads.lens.sum())
    # tiers off (at this size) and on: k15 w5 then sketches straight into the tiers
    for tiers in (1 << 18, 0):
        chunked.set_option("tier_min_records", tiers)
        one = stage1(chunked, 0, 0.001, 32, minhash)
        assert not one[3]
        for chunk in (1, total // 3, 4 * total):
            got = stage1(chunked, chunk, 0.001, 32, minhash)
            assert got[3], chunk
            for k in KEYS:
                assert np.array_equal(got[0][k], GOLD[f"stage1_{tag}_{k}"]), (tiers, chunk, k)
            assert got[0]["num_mapped"] == META[f"stage1_{tag}_num_mapped"]
            same(got, one, (tag, tiers, chunk))


@pytest.mark.parametrize("ib,qb,kmax", [(120_000, 50_000, 8), (60_000, 100_000, 32),
                                        (150_000, 25_000, 4)])
def test_chunks_schedules(chunked, oracle, ib, qb, kmax):
    """Several index batches and flushes: flushes wholly before a batch and flushes that
    straddle its first read run the probe path between the batch's self-join flushes."""
    rs = synth.make_reads(40_000, 200, 3000, seed=17)
    chunked.configure(k=15, w=5)
    chunked.upload(rs)
    for minhash in (False, True):
        one = stage1(chunked, 0, 0.001, kmax, minhash, ib, qb)
        want = oracle.stage1(oracle.engine(15, 5, threads=4), oracle.reads(rs), 0.001, kmax,
                             minhash, ib, qb)
        same_oracle(one, want, (ib, minhash))
        for chunk in (1, 7_000, ib // 3):
            got = stage1(chunked, chunk, 0.001, kmax, minhash, ib, qb)
            assert got[3]
            same(got, one, (ib, minhash, chunk))


def edge_reads():
    """Copies of a few reads (runs of equal values in every chunk), tandem repeats denser
    than the sketch's capacity estimate (every position a minimizer), and reads shorter
    than k or than k + w - 1 (chunks without minimizers)."""
    rng = np.random.default_rng(31)
    base = [rng.integers(0, 4, int(n), dtype=np.uint8) for n in (2500, 3000, 3600)]
    seqs = []
    for i in range(30):
        seqs.append(base[i % 3].copy())
        if i % 5 == 0:
            seqs.append(np.tile(np.array([0, 1], np.uint8), 1500))   # ACAC...
        if i % 4 == 0:
            seqs.append(rng.integers(0, 4, 10, dtype=np.uint8))       # shorter than k
            seqs.append(rng.integers(0, 4, 17, dtype=np.uint8))       # shorter than k + w - 1
        if i % 7 == 0:
            seqs.append(np.zeros(2000, np.uint8))                     # homopolymer
    return seqio.pack_codes(seqs)


def test_chunks_edges(chunked, oracle):
    rs = edge_reads()
    prm = dict(bandwidth=500, chain=2, matches=15, gap=3)
    chunked.configure(k=15, w=5, **prm)
    chunked.upload(rs)
    chunked.set_option("tier_min_records", 0)   # tiers: the sketch-to-tiers kernel
    for ib, qb in ((0, 0), (30_000, 12_000)):
        one = stage1(chunked, 0, 0.01, 8, False, ib, qb)
        want = oracle.stage1(oracle.engine(15, 5, threads=4, **prm), oracle.reads(rs), 0.01, 8,
                             False, ib or 1 << 32, qb or 1 << 30)
        same_oracle(one, want, ib)
        for chunk in (1, 9, 5_000):
            got = stage1(chunked, chunk, 0.01, 8, False, ib, qb)
            assert got[3]
            same(got, one, (ib, chunk))
    # a short read alone in its chunk, a tandem repeat alone in its chunk
    short = seqio.pack_codes([np.zeros(5, np.uint8)] * 3 +
                             [np.tile(np.array([2, 3], np.uint8), 4000)] * 2)
    chunked.upload(short)
    one = stage1(chunked, 0, 0.001, 8, False)
    got = stage1(chunked, 1, 0.001, 8, False)
    same(got, one, "short")


@pytest.mark.parametrize("k,w", [(15, 5), (15, 10), (19, 10)])
def test_chunks_sketch_routes(chunked, oracle, k, w):
    """k15 w5 (fast sketch), k15 w10 (generic sketch, tiers), k19 w10 (u64, untiered)."""
    rs = synth.make_reads(30_000, 160, 3000, seed=9)
    chunked.configure(k=k, w=w)
    chunked.upload(rs)
    chunked.set_option("tier_min_records", 0)
    for minhash in (False, True):
        one = stage1(chunked, 0, 0.001, 16, minhash, 150_000, 60_000)
        want = oracle.stage1(oracle.engine(k, w, threads=4), oracle.reads(rs), 0.001, 16,
                             minhash, 150_000, 60_000)
        same_oracle(one, want, (k, w, minhash))
        for chunk in (1, 40_000):
            got = stage1(chunked, chunk, 0.001, 16, minhash, 150_000, 60_000)
            assert got[3]
            same(got, one, (k, w, minhash, chunk))


@pytest.mark.parametrize("tiers,bare,join,window", [
    (0, 0, 1, -1), (0, 1, 1, -1), (0, 8, 1, -1), (1 << 18, 1, 1, -1), (0, 1, 0, -1),
    (0, 1, 1, 1), (0, 0, 0, 1)])
def test_chunks_build_routes(chunked, oracle, tiers, bare, join, window):
    """tier_min_records 0 (tiers on) or default (off at this size), bare_count 0 / 1 / 8,
    self_join 0, and the windowed stage 1 together with chunking."""
    rs = synth.make_reads(30_000, 160, 3000, seed=9)
    chunked.configure(k=15, w=5)
    chunked.upload(rs)
    chunked.set_option("tier_min_records", tiers)
    chunked.set_option("bare_count", bare)
    chunked.set_option("self_join", join)
    chunked.set_stage1_window(window)
    for freq, ib, qb in ((0.02, 150_000, 60_000), (0.3, 0, 100_000)):
        one = stage1(chunked, 0, freq, 8, False, ib, qb)
        want = oracle.stage1(oracle.engine(15, 5, threads=4), oracle.reads(rs), freq, 8,
                             False, ib or 1 << 32, qb or 1 << 30)
        same_oracle(one, want, (tiers, bare, join, freq))
        for chunk in (1, 50_000):
            got = stage1(chunked, chunk, freq, 8, False, ib, qb)
            assert got[3]
            if window == 1:
                assert chunked.stage1_windowed()
            same(got, one, (tiers, bare, join, window, freq, chunk))


def test_chunks_auto(chunked):
    """Auto (the default) chunks only when the one-shot pass exceeds the budget; same
    result both times. The estimates: a chunked build saves nothing while a flush is as
    large as the batch (its working set dominates), chunks and flushes far smaller than the
    batch do. Invalid values raise."""
    rs = synth.make_reads(30_000, 150, 3000, seed=3)
    chunked.configure(k=15, w=5)
    chunked.upload(rs)
    chunked.set_index_chunks(-1, 0)
    one = stage1(chunked, -1, 0.001, 8, False, 120_000, 50_000)
    assert not one[3]
    fp = chunked.index_footprint(120_000)   # (with the default query flushes of 2^30 bases)
    assert 0 < fp["chunked"] <= fp["one_shot"]
    s1 = chunked.stage1_footprint(8, 120_000, 50_000)
    chunked.set_index_chunks(1000)   # chunks and flushes far smaller than the batch
    assert chunked.stage1_footprint(8, 120_000, 50_000)["resident"] < s1["resident"]
    pass_one_shot = min(s1["resident"], s1["windowed_device"])
    chunked.set_index_chunks(-1, pass_one_shot - (1 << 10))
    got = chunked.find_overlaps_and_create_piles(0.001, 8, False, 120_000, 50_000)
    assert chunked.stage1_index_chunked()
    same((got, chunked.index_records(), chunked.stats()["occurrence"], True), one, "auto")
    chunked.set_index_chunks(-1, pass_one_shot + (1 << 20))
    got = chunked.find_overlaps_and_create_piles(0.001, 8, False, 120_000, 50_000)
    assert not chunked.stage1_index_chunked()
    same((got, chunked.index_records(), chunked.stats()["occurrence"], False), one, "one-shot")
    with pytest.raises(ValueError):
        chunked.set_option("index_chunk_bases", -2)
    with pytest.raises(ValueError):
        chunked.set_option("index_chunk_budget", -1)
