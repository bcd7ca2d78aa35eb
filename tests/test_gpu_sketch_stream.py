"""The k=15 w=5 sketch kernel writes each tile's records from shared memory, and
micromizers and thresholds are selected from an on-chip copy of each read's sketch
(global memory for sketches longer than that copy). Bit-exact against the CPU
oracle on benchmark-shaped reads, tile edges, over-dense repeats, long reads and the
asynchronous upload."""
import numpy as np
import pytest

from raven_b200 import seqio, synth

pytestmark = pytest.mark.gpu

K, W = 15, 5
TILE = 2048
STAGE_VALUES = 10240      # u32 values the micromize kernel keeps on chip (40 KB)


def check_sketch(gpu_engine, oracle, rs, minhash_modes=(False, True)):
    gpu_engine.configure(k=K, w=W)
    gpu_engine.upload(rs)
    eng, reads = oracle.engine(K, W), oracle.reads(rs)
    for minhash in minhash_modes:
        got = gpu_engine.sketch(0, rs.n, minhash)
        want = oracle.sketch(eng, reads, 0, rs.n, minhash)
        for key in ("offsets", "value", "origin"):
            assert np.array_equal(got[key], want[key]), (minhash, key)
    return got


def check_stage1(gpu_engine, oracle, rs, ib=0, qb=0, kmax=16):
    gpu_engine.configure(k=K, w=W)
    gpu_engine.upload(rs)
    got = gpu_engine.find_overlaps_and_create_piles(0.001, kmax, False, ib, qb)
    want = oracle.stage1(oracle.engine(K, W, threads=4), oracle.reads(rs), 0.001, kmax,
                         False, ib or 1 << 32, qb or 1 << 30)
    for key in ("overlaps", "ovl_off", "pile", "pile_off"):
        assert np.array_equal(got[key], want[key]), key
    assert got["num_mapped"] == int(want["num_mapped"][0])
    return got


def test_bench_shaped_reads(gpu_engine, oracle):
    from bench import synth as bench_synth
    rs = bench_synth.make_reads(20260924, 5_000_000, 2500, 10_000)
    got = check_sketch(gpu_engine, oracle, rs)
    assert got["value"].size > 0


def tile_edge_reads():
    """k-mer position counts at and around multiples of the tile (2048 j + {0, +-1,
    +-4}) and many reads shorter than a tile, so groups of 4 tiles span reads and
    halos fall on tile and read edges"""
    rng = np.random.default_rng(41)
    L = []
    for j in (1, 2, 3, 5):
        L += [TILE * j + d for d in (-4, -1, 0, 1, 4)]
    L += list(rng.integers(W, TILE, 300))                 # shorter than one tile
    L += [W, W + 1, 3, 2 * TILE - W + 1]
    rng.shuffle(L)
    seqs = [rng.integers(0, 4, int(n) + K - 1, dtype=np.uint8) for n in L]
    return seqio.pack_codes(seqs)


def test_tile_edges(gpu_engine, oracle):
    check_sketch(gpu_engine, oracle, tile_edge_reads())


def repeat_reads():
    """mostly poly-A and dinucleotide repeats: every position of a poly-A tile is a
    minimizer (all windows tie), and the whole set is denser than the sketch's
    first capacity estimate (2.2 / (w + 1) of the positions)"""
    rng = np.random.default_rng(43)
    seqs = []
    for n in (TILE + K - 1, 3 * TILE + 7, 5000, 700, 2 * TILE + K - 1):
        seqs.append(np.zeros(n, np.uint8))                           # poly-A
        seqs.append(np.tile(np.array([0, 1], np.uint8), n // 2))     # (AC)n
        seqs.append(np.tile(np.array([2, 3], np.uint8), n // 2))     # (GT)n
    seqs += [rng.integers(0, 4, 3000, dtype=np.uint8) for _ in range(3)]
    return seqio.pack_codes(seqs)


def test_dense_repeats_retry(gpu_engine, oracle):
    rs = repeat_reads()
    got = check_sketch(gpu_engine, oracle, rs)
    full = gpu_engine.sketch(0, rs.n, False)
    positions = int(sum(int(n) - K + 1 for n in rs.lens if n >= K))
    assert full["value"].size > 2.2 / (W + 1) * positions + 4096   # the retry ran
    # the first poly-A read is one tile, every position a minimizer
    assert int(full["offsets"][1]) == TILE
    assert got["value"].size > 0


def long_reads():
    """a 150 kb read and one with more minimizers than the micromize kernel keeps on
    chip, among ordinary reads"""
    rng = np.random.default_rng(47)
    seqs = [rng.integers(0, 4, n, dtype=np.uint8)
            for n in (150_000, 3 * STAGE_VALUES + 2000, 8000, 12_000, 600)]
    return seqio.pack_codes(seqs)


def test_long_reads_fallback(gpu_engine, oracle):
    rs = long_reads()
    full = check_sketch(gpu_engine, oracle, rs, (False,))
    counts = np.diff(full["offsets"].astype(np.int64))
    assert counts[0] > STAGE_VALUES and counts[1] > STAGE_VALUES
    check_sketch(gpu_engine, oracle, rs, (True,))         # micromizers (kWrite)
    # thresholds (the self-join) of the same long reads, among overlapping reads
    base = synth.make_reads(60_000, 60, 4000, seed=48)
    seqs = [base.codes(i) for i in range(base.n)] + [rs.codes(0), rs.codes(1)]
    check_stage1(gpu_engine, oracle, seqio.pack_codes(seqs))


def test_async_upload_pinned(gpu_engine):
    import torch
    rs = synth.make_reads(200_000, 2400, 4000, seed=53)   # > 1024 reads: chunked
    gpu_engine.configure(k=K, w=W)
    gpu_engine.upload(rs)
    want_sk = gpu_engine.sketch(0, rs.n, False)
    want = gpu_engine.find_overlaps_and_create_piles(0.001, 16, False)

    class Pinned:
        pass

    prs = Pinned()
    words = torch.from_numpy(rs.words.view(np.int64)).pin_memory()
    woff = torch.from_numpy(rs.word_off.view(np.int64)).pin_memory()
    lens = torch.from_numpy(rs.lens.view(np.int32)).pin_memory()
    prs.words = words.numpy().view(np.uint64)
    prs.word_off = woff.numpy().view(np.uint64)
    prs.lens = lens.numpy().view(np.uint32)
    prs.n = rs.n
    gpu_engine.set_option("async_upload", 1)
    try:
        gpu_engine.upload(prs)
        got_sk = gpu_engine.sketch(0, rs.n, False)
        for key in ("offsets", "value", "origin"):
            assert np.array_equal(got_sk[key], want_sk[key]), key
        gpu_engine.upload(prs)
        got = gpu_engine.find_overlaps_and_create_piles(0.001, 16, False)
        for key in ("overlaps", "ovl_off", "pile", "pile_off"):
            assert np.array_equal(got[key], want[key]), key
    finally:
        gpu_engine.set_option("async_upload", 0)


@pytest.mark.parametrize("ib,qb", [(0, 0), (700_000, 0), (400_000, 150_000)])
def test_thresholds_index_batches(gpu_engine, oracle, ib, qb):
    """stage 1 under index batches: the thresholds of each batch's self-join and the
    written micromizers of the earlier batches' probe path"""
    from bench import synth as bench_synth
    rs = bench_synth.make_reads(20260925, 1_000_000, 300, 8000)
    check_stage1(gpu_engine, oracle, rs, ib, qb)
