"""rvn_map in flushes (option "map_flush_bases" forces a size; by default the size comes
from the device memory, at most the reference's 2^30 query bases): the results of any cut
are those of one piece, byte for byte, offsets included, for the flag sets of the three
callers; one flush launches what a single MapRange launches. Then the callers with
chunks and flushes forced on every context of their process (RVN_SET_OPTIONS): the
reference's own stage 1 and stage 2 over the facade, the assembly pin, the polisher."""
import hashlib
import os
import subprocess

import numpy as np
import pytest

from raven_b200 import seqio, synth
from test_gpu_dropin import REF_BIN, assert_reference_assembly, run_dropin, write_vec

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
FLAGS = ((1, 1, 1, 0), (1, 1, 0, 1), (0, 0, 0, 0))   # stage 1, stage 2, the polisher
FORCED = "index_chunk_bases=30000,map_flush_bases=40000"


@pytest.fixture
def eng(gpu_engine):
    try:
        yield gpu_engine
    finally:
        gpu_engine.set_index_chunks(-1, 0)
        gpu_engine.set_option("map_flush_bases", 0)
        gpu_engine.set_option("keep_hits", 0)
        gpu_engine.configure(k=15, w=5)


@pytest.fixture
def forced_env():
    os.environ["RVN_SET_OPTIONS"] = FORCED
    try:
        yield
    finally:
        del os.environ["RVN_SET_OPTIONS"]


def reads_with_loners(seed):
    """overlapping reads with unrelated ones between them: reads without overlaps at the
    edges of flushes, and at both ends of the set"""
    rs = synth.make_reads(40_000, 120, 3000, seed=seed)
    rng = np.random.default_rng(seed)
    seqs = []
    for i in range(rs.n):
        if i % 6 == 0:
            seqs.append(rng.integers(0, 4, 2500, dtype=np.uint8))
        if i % 25 == 3:   # tandem repeats: over-frequent minimizers (filtered positions)
            seqs.append(np.tile(np.array([0, 1, 2], np.uint8), 700))
        seqs.append(rs.codes(i))
    seqs.append(rng.integers(0, 4, 12, dtype=np.uint8))
    return seqio.pack_codes(seqs)


def mapped(eng, flush, first, last, flags):
    eng.set_option("map_flush_bases", flush)
    eng.set_option("reset_stats", 0)
    res = eng.map(first, last, *[bool(f) for f in flags])
    return res, eng.map_flushes(), eng.stats()["kernel_launches"]


@pytest.mark.parametrize("flags", FLAGS)
def test_flush_identity(eng, flags):
    rs = reads_with_loners(21)
    eng.configure(k=15, w=5)
    eng.upload(rs)
    j = 40
    eng.set_index_chunks(0)
    eng.minimize(j, rs.n, False)
    eng.filter(0.001)
    for first, last in ((j, rs.n), (0, j), (0, rs.n), (j + 3, rs.n - 5), (9, 9)):
        bases = int(rs.lens[first:last].sum())
        mapped(eng, 0, first, last, flags)   # (the first map of a range may run the join sweep)
        want, n, launches = mapped(eng, 0, first, last, flags)
        assert n == 0
        one, n, l1 = mapped(eng, 4 * bases + 1, first, last, flags)
        assert n == 0 and l1 == launches      # one flush: the single MapRange, no more
        for flush, flushes in ((4 * bases + 1, 0), (bases // 2 + 1, 2), (bases // 7 + 1, None),
                               (1, last - first)):
            got, n, _ = mapped(eng, flush, first, last, flags)
            if flushes is not None and last - first > 1:
                assert n == flushes, (first, last, flush)
            for key in ("overlaps", "ovl_off", "filt_off", "filtered"):
                assert got[key].dtype == want[key].dtype
                assert got[key].tobytes() == want[key].tobytes(), (first, last, flush, key)
        if last - first > 50:
            assert want["overlaps"].shape[0] > 100
            assert not flags[0] or (np.diff(want["ovl_off"]) == 0).any()
            assert flags[3] == 0 or want["filtered"].size > 0


def test_keep_hits_maps_in_one_piece(eng):
    rs = reads_with_loners(2)
    eng.configure(k=15, w=5)
    eng.upload(rs)
    eng.minimize(0, rs.n, False)
    eng.filter(0.001)
    eng.set_option("keep_hits", 1)
    got, n, _ = mapped(eng, 1, 0, rs.n, (1, 1, 1, 0))
    assert n == 0
    hits = eng.map_hits(rs.n)
    assert hits["hit_off"][-1] == hits["group"].size > 0
    with pytest.raises(ValueError):
        eng.set_option("map_flush_bases", -1)


def same_stage1(got, want):
    for key in ("overlaps", "ovl_off", "pile", "pile_off"):
        assert np.array_equal(got[key], want[key]), key


@pytest.mark.parametrize("minhash", [False, True])
def test_reference_stage1_over_facade_forced(tmp_path, oracle, lambda_reads, forced_env, minhash):
    a, b = run_dropin(tmp_path, lambda_reads, 15, 5, 0.001, 32, minhash)
    want = oracle.stage1(oracle.engine(15, 5, threads=4), oracle.reads(lambda_reads), 0.001, 32,
                         minhash)
    same_stage1(a, want)
    same_stage1(b, want)


def test_reference_stage1_synthetic_forced(tmp_path, oracle, forced_env):
    rs = synth.make_reads(40_000, 150, 3000, seed=13)
    a, b = run_dropin(tmp_path, rs, 15, 5, 0.001, 6, False)
    want = oracle.stage1(oracle.engine(15, 5, threads=4), oracle.reads(rs), 0.001, 6, False)
    same_stage1(a, want)
    same_stage1(b, want)


def test_facade_schedule_forced(tmp_path, oracle, forced_env):
    """several index batches per pass through the facade: same answers, and still one
    batch map per part, however many flushes it took"""
    from test_gpu_facade_batch import Schedule, batches
    rs = synth.make_reads(genome_len=80_000, n_reads=160, mean_len=3000, seed=21)
    bs = batches(rs, int(rs.lens.sum()) // 4)
    for stage1 in (True, False):
        s = Schedule(rs)
        maps = served = 0
        for j, last in bs:
            s.minimize(j, last, stage1)
            s.filter(0.001)
            for k in range(last):
                s.map(k, True, True, stage1, not stage1)
            maps += 1 if j == 0 else 2
            served += last
            s.counters(maps, served, 0)
        s.run(tmp_path, oracle)


def test_assembly_pin_forced(tmp_path, oracle, lambda_reads, forced_env):
    binary = os.path.join(REF_BIN, "assemble_test")
    if not os.path.exists(binary):
        pytest.skip("oracle/_ref/assemble_test not built")
    inp, out = str(tmp_path / "reads.bin"), str(tmp_path / "unitigs.txt")
    with open(inp, "wb") as f:
        write_vec(f, lambda_reads.words.astype(np.uint64))
        write_vec(f, lambda_reads.word_off.astype(np.uint64))
        write_vec(f, lambda_reads.lens.astype(np.uint32))
        write_vec(f, lambda_reads.block_quality.astype(np.uint8))
        write_vec(f, lambda_reads.bq_off.astype(np.uint64))
    subprocess.run([binary, inp, out, "1", "2"], check=True, stderr=subprocess.DEVNULL,
                   timeout=900)
    lines = open(out).read().split("\n")
    names, seqs = lines[0:-1:2], [s.encode() for s in lines[1::2]]
    assert_reference_assembly(names, seqs)
    genome = seqio.ReadSet.load(os.path.join(HERE, "golden", "lambda_genome.npz")).ascii(0)
    rc = seqs[0].translate(bytes.maketrans(b"ACGT", b"TGCA"))[::-1]
    assert oracle.edit_distance(rc, genome) == 1137


def test_stage2_forced_equals_unforced(tmp_path, lambda_reads):
    binary = os.path.join(REF_BIN, "stage2_test")
    if not os.path.exists(binary):
        pytest.skip("oracle/_ref/stage2_test not built")
    inp = str(tmp_path / "reads.bin")
    with open(inp, "wb") as f:
        write_vec(f, lambda_reads.words.astype(np.uint64))
        write_vec(f, lambda_reads.word_off.astype(np.uint64))
        write_vec(f, lambda_reads.lens.astype(np.uint32))
    digests = []
    for forced in (None, FORCED):
        out = str(tmp_path / f"out{len(digests)}.bin")
        env = dict(os.environ)
        if forced:
            env["RVN_SET_OPTIONS"] = forced
        subprocess.run([binary, inp, out, "15", "5", "0.001", "0.8"], check=True, env=env,
                       stderr=subprocess.DEVNULL, timeout=900)
        digests.append(hashlib.sha256(open(out, "rb").read()).hexdigest())
        assert os.path.getsize(out) > 1000
    assert digests[0] == digests[1]


def test_polisher_forced_equals_unforced():
    import sys
    sys.path.insert(0, os.path.dirname(HERE))
    from bench import synth as bsynth
    from raven_b200 import polish
    reads = bsynth.make_reads(77, 60_000, 240, 5000, min_len=1500)
    draft = bsynth.make_contigs(77, 60_000, contig_len=25_000)
    want, st = polish.polish(draft, reads, threads=4)
    assert st["polished_windows"] > 100
    os.environ["RVN_SET_OPTIONS"] = "index_chunk_bases=10000,map_flush_bases=100000"
    try:
        got, _ = polish.polish(draft, reads, threads=4)
    finally:
        del os.environ["RVN_SET_OPTIONS"]
    assert got.names == want.names
    assert [got.ascii(i) for i in range(got.n)] == [want.ascii(i) for i in range(want.n)]
