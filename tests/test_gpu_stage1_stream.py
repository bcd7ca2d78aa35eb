"""Stage-1 results streamed to the host while later flushes run (option "stage1_stream"):
the piles and lists of the reads no later flush touches are copied on a stream of their
own. Option 0 copies everything after the last flush. Both must give identical results:
golden reads, C2-shaped reads with many small query flushes (list buffers reused while
copies are in flight), small index batches (nothing streams before the last batch), kmax
1 / 32 and one above the streamed lists' cap, two calls whose buffers grow, the pile regions
after the call, and the windowed mode, where the option changes nothing."""
import hashlib
import json
import os

import numpy as np
import pytest

from raven_b200 import synth

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
META = json.load(open(os.path.join(HERE, "golden", "lambda_golden.json")))
GOLD = np.load(os.path.join(HERE, "golden", "lambda_golden.npz"))
KEYS = ("overlaps", "ovl_off", "pile", "pile_off")


@pytest.fixture
def eng(gpu_engine):
    gpu_engine.configure(k=15, w=5)
    try:
        yield gpu_engine
    finally:
        gpu_engine.set_option("stage1_stream", 1)
        gpu_engine.set_stage1_window(-1, 0)


def digest(res):
    h = {k: hashlib.sha256(np.ascontiguousarray(res[k]).tobytes()).hexdigest() for k in KEYS}
    h["num_mapped"] = int(res["num_mapped"])
    return h


def both(eng, *args):
    """the call with streaming off, then on: (digest, result of the streamed call)"""
    eng.set_option("stage1_stream", 0)
    want = digest(eng.find_overlaps_and_create_piles(*args))
    # (a resident pass times its tail copies as phase "results")
    assert ("results" in eng.timings()) != eng.stage1_windowed()
    eng.set_option("stage1_stream", 1)
    got = eng.find_overlaps_and_create_piles(*args)
    assert ("results" in eng.timings()) != eng.stage1_windowed()
    assert digest(got) == want, args
    return got


def same_as_oracle(got, want, tag):
    for k in KEYS:
        assert np.array_equal(got[k], want[k]), (tag, k)
    assert got["num_mapped"] == int(np.asarray(want["num_mapped"]).ravel()[0]), tag


def c2_reads(n_reads=1200, seed=20260924):
    """bench.py's C2 model at 1/170 of its size: 10 kb mean reads at 40x"""
    from bench import synth as bench_synth
    return bench_synth.make_reads(seed, n_reads * 10_000 // 40, n_reads, 10_000)


def test_stream_lambda_golden(eng, lambda_reads):
    eng.upload(lambda_reads)
    for minhash in (False, True):
        tag = "minhash" if minhash else "plain"
        got = both(eng, 0.001, 32, minhash)
        for k in KEYS:
            assert np.array_equal(got[k], GOLD[f"stage1_{tag}_{k}"]), (tag, k)
        assert got["num_mapped"] == META[f"stage1_{tag}_num_mapped"]
        both(eng, 0.001, 16, minhash, 0, 60_000)       # many flushes, one batch
        both(eng, 0.001, 16, minhash, 400_000, 150_000)  # many batches and flushes


@pytest.mark.parametrize("kmax", [1, 32, 1000])
def test_stream_many_flushes(eng, oracle, kmax):
    """Flushes of about a tenth of the reads: the lists of a flush are copied from the
    buffer the gather two flushes later writes again. kmax 1000 is above the cap of the
    streamed lists: they go to the host after the last flush, the piles still stream."""
    rs = c2_reads()
    eng.upload(rs)
    qb = int(rs.lens.sum()) // 10
    got = both(eng, 0.001, kmax, False, 0, qb)
    assert len(eng.timings()) and eng.stats()["overlaps"] > 0
    want = oracle.stage1(oracle.engine(15, 5, threads=4), oracle.reads(rs), 0.001, kmax,
                         False, 1 << 32, qb)
    same_as_oracle(got, want, kmax)
    if kmax == 1000:   # nothing truncated: lists longer than kmax 32 keeps
        assert (np.diff(got["ovl_off"].astype(np.int64)) > 32).any()


def test_stream_small_index_batches(eng, oracle):
    """Four index batches: every batch's flushes start at read 0 again, so nothing is
    final before the last batch."""
    rs = c2_reads(900, seed=7)
    eng.upload(rs)
    total = int(rs.lens.sum())
    ib, qb = total // 4 + 1, total // 6
    got = both(eng, 0.001, 32, False, ib, qb)
    want = oracle.stage1(oracle.engine(15, 5, threads=4), oracle.reads(rs), 0.001, 32, False,
                         ib, qb)
    same_as_oracle(got, want, "batches")


def test_stream_buffers_grow(eng, oracle):
    """Two calls on one context, the second over a larger read set: its pinned and device
    buffers grow between the calls, never while a copy is in flight."""
    small, large = c2_reads(300, seed=11), c2_reads(1500, seed=12)
    for rs in (small, large):
        eng.upload(rs)
        qb = int(rs.lens.sum()) // 9
        eng.set_option("stage1_stream", 1)
        got = eng.find_overlaps_and_create_piles(0.001, 32, False, 0, qb)
        want = oracle.stage1(oracle.engine(15, 5, threads=4), oracle.reads(rs), 0.001, 32,
                             False, 1 << 32, qb)
        same_as_oracle(got, want, rs.n)
    both(eng, 0.001, 32, False, 0, int(large.lens.sum()) // 9)


def test_stream_pile_regions(eng):
    """rvn_stage1_pile_regions reads the device piles the streamed call left behind."""
    rs = synth.make_reads(40_000, 300, 5000, seed=14)
    eng.upload(rs)
    regions = {}
    for mode in (0, 1):
        eng.set_option("stage1_stream", mode)
        eng.find_overlaps_and_create_piles(0.001, 32, False, 0, 100_000)
        regions[mode] = {cov: eng.stage1_pile_regions(cov) for cov in (1, 4, 9)}
    for cov, want in regions[0].items():
        for k in ("invalid", "begin", "end", "median"):
            assert np.array_equal(regions[1][cov][k], want[k]), (cov, k)
    assert (regions[1][4]["invalid"] == 0).sum() > 100


def test_stream_windowed(eng, oracle):
    """A windowed pass keeps the results on the host already: the option changes nothing."""
    rs = synth.make_reads(30_000, 150, 3000, seed=3)
    eng.upload(rs)
    eng.set_stage1_window(1)
    got = both(eng, 0.001, 8, False, 120_000, 50_000)
    assert eng.stage1_windowed()
    want = oracle.stage1(oracle.engine(15, 5, threads=4), oracle.reads(rs), 0.001, 8, False,
                         120_000, 50_000)
    same_as_oracle(got, want, "windowed")
    eng.set_stage1_window(0)
    assert digest(eng.find_overlaps_and_create_piles(0.001, 8, False, 120_000, 50_000)) == \
        digest(got)


def test_stream_option_values(eng):
    with pytest.raises(ValueError):
        eng.set_option("stage1_stream", 2)
