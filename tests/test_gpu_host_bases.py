"""Packed bases in pinned host memory (option "host_bases"): the sketch kernels read each
read range from a device staging window that the drivers fill from the context's pinned
copy. Every result must be bit-identical to the bases-on-device route on the same context
settings - overlap lists, offsets, piles, num_mapped, map results, sketches - and to the
oracle where the window and chunk tests compare with it: schedules with many index
batches and flushes, resident and windowed stage 1, one-shot and chunked builds, the
self-join and the probe path, tiers, every sketch kernel, rvn_map's flushes and its
external reads, asynchronous uploads; the calls that bring the whole set back to the
device; the auto decision; and the reference's own stage 1 and assembly pin with the
option forced on every context of their process."""
import os
import subprocess

import numpy as np
import pytest

from raven_b200 import engine, seqio, synth
from test_gpu_dropin import REF_BIN, assert_reference_assembly, run_dropin, write_vec

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = np.load(os.path.join(HERE, "golden", "lambda_golden.npz"))
KEYS = ("overlaps", "ovl_off", "pile", "pile_off")


@pytest.fixture
def eng(gpu_engine):
    try:
        yield gpu_engine
    finally:
        gpu_engine.set_host_bases(-1, 0)
        gpu_engine.set_index_chunks(-1, 0)
        gpu_engine.set_stage1_window(-1, 0)
        gpu_engine.set_option("tier_min_records", 1 << 18)
        gpu_engine.set_option("self_join", 1)
        gpu_engine.set_option("map_flush_bases", 0)
        gpu_engine.set_option("async_upload", 0)
        gpu_engine.configure(k=15, w=5)


@pytest.fixture
def host_env():
    os.environ["RVN_SET_OPTIONS"] = "host_bases=1"
    try:
        yield
    finally:
        del os.environ["RVN_SET_OPTIONS"]


def upload(eng, rs, mode):
    eng.set_host_bases(mode)
    eng.upload(rs)
    res = eng.reads_residency()
    assert res["on_host"] == (mode == 1)
    return res


def stage1(eng, *args):
    got = eng.find_overlaps_and_create_piles(*args)
    return got, eng.stats()["occurrence"]


def same(got, want, tag):
    for k in KEYS:
        assert np.array_equal(got[0][k], want[0][k]), (tag, k)
    assert got[0]["num_mapped"] == want[0]["num_mapped"], tag
    assert got[1] == want[1], tag


def same_oracle(got, want, tag):
    for k in KEYS:
        assert np.array_equal(got[0][k], want[k]), (tag, k)
    assert got[0]["num_mapped"] == int(np.asarray(want["num_mapped"]).ravel()[0]), tag


@pytest.mark.parametrize("minhash", [False, True])
def test_lambda_golden(eng, lambda_reads, minhash):
    eng.configure(k=15, w=5)
    tag = "minhash" if minhash else "plain"
    words = lambda_reads.words.size * 8
    for chunk in (0, int(lambda_reads.lens.sum()) // 3):
        eng.set_index_chunks(chunk)
        upload(eng, lambda_reads, 0)
        want = stage1(eng, 0.001, 32, minhash)
        upload(eng, lambda_reads, 1)
        got = stage1(eng, 0.001, 32, minhash)
        same(got, want, (tag, chunk))
        for k in KEYS:
            assert np.array_equal(got[0][k], GOLD[f"stage1_{tag}_{k}"]), (chunk, k)
        res = eng.reads_residency()
        assert res["on_host"]
        if chunk and not minhash:   # two halves of a third of the set each
            assert 0 < res["device_word_bytes"] < words, res
        assert "stage_bases" in eng.timings()


@pytest.mark.parametrize("ib,qb,kmax", [(120_000, 50_000, 8), (60_000, 100_000, 32),
                                        (150_000, 25_000, 4)])
def test_schedules(eng, oracle, ib, qb, kmax):
    """Several index batches and flushes: flushes wholly before a batch and flushes that
    straddle its first read; resident and windowed passes, one-shot and chunked builds,
    self-join and probe path, tiers forced on."""
    rs = synth.make_reads(40_000, 200, 3000, seed=17)
    eng.configure(k=15, w=5)
    eng.set_option("tier_min_records", 0)
    for minhash in (False, True):
        want = oracle.stage1(oracle.engine(15, 5, threads=4), oracle.reads(rs), 0.001, kmax,
                             minhash, ib, qb)
        for window in (0, 1):
            for chunk in (0, 7_000):
                for join in (1, 0):
                    eng.set_stage1_window(window)
                    eng.set_index_chunks(chunk)
                    eng.set_option("self_join", join)
                    tag = (minhash, window, chunk, join)
                    upload(eng, rs, 0)
                    dev = stage1(eng, 0.001, kmax, minhash, ib, qb)
                    upload(eng, rs, 1)
                    got = stage1(eng, 0.001, kmax, minhash, ib, qb)
                    same(got, dev, tag)
                    same_oracle(got, want, tag)


def rc_words(rs, i):
    return seqio.pack_codes([(3 - rs.codes(i)[::-1]).astype(np.uint8)])


@pytest.mark.parametrize("k,w", [(15, 5), (15, 10), (19, 10), (31, 32)])
def test_sketch_routes(eng, oracle, k, w):
    """k15 w5 (SketchFastKernel), k15 w10 (SketchKernel<u32>), k19 w10 and k31 w32
    (SketchKernel<u64>): stage 1, and rvn_minimize / rvn_filter / rvn_map with forced
    chunks and flushes, rvn_map_external of a reverse-complemented read, rvn_sketch."""
    # (31-mers need reads of fewer errors to share seeds)
    err = dict(sub=0.01, ins=0.01, dele=0.01) if k == 31 else {}
    rs = synth.make_reads(30_000, 160, 3000, seed=9, **err)
    eng.configure(k=k, w=w)
    eng.set_option("tier_min_records", 0)
    want = oracle.stage1(oracle.engine(k, w, threads=4), oracle.reads(rs), 0.001, 16, False,
                         150_000, 60_000)
    rc = rc_words(rs, 7)

    def run(mode):
        upload(eng, rs, mode)
        out = {}
        for chunk in (0, 40_000):
            eng.set_index_chunks(chunk)
            out[("s1", chunk)] = stage1(eng, 0.001, 16, False, 150_000, 60_000)
            for minhash in (False, True):
                eng.minimize(40, rs.n, minhash)
                eng.filter(0.001)
                for flush in (0, 20_000):
                    eng.set_option("map_flush_bases", flush)
                    out[("map", chunk, minhash, flush)] = eng.map(0, rs.n, True, True, minhash,
                                                                  not minhash)
                out[("ext", chunk, minhash)] = eng.map_external(
                    rc.words, int(rc.lens[0]), 7, True, True, minhash, not minhash)
            eng.set_option("map_flush_bases", 0)
        out["sketch"] = eng.sketch(3, 90, False)
        return out

    dev, host = run(0), run(1)
    assert eng.reads_residency()["on_host"]
    same_oracle(host[("s1", 0)], want, (k, w))
    for key, d in dev.items():
        h = host[key]
        if key[0] == "s1":
            same(h, d, key)
            continue
        for name in d:
            assert np.array_equal(h[name], d[name]), (k, w, key, name)
    assert dev[("map", 0, False, 0)]["overlaps"].shape[0] > 0


def test_async_upload_and_caller_words(eng):
    """async_upload has nothing to do in host mode; the caller may overwrite its words
    as soon as the upload has returned."""
    rs = synth.make_reads(40_000, 1500, 800, seed=5)
    eng.configure(k=15, w=5)
    upload(eng, rs, 0)
    want = stage1(eng, 0.001, 8, False, 200_000, 100_000)
    eng.set_option("async_upload", 1)
    for chunk in (0, 50_000):
        eng.set_index_chunks(chunk)
        upload(eng, rs, 0)
        same(stage1(eng, 0.001, 8, False, 200_000, 100_000), want, ("async device", chunk))
        own = seqio.ReadSet(rs.words.copy(), rs.word_off, rs.lens)
        upload(eng, own, 1)
        eng._keep[0][:] = 0   # the caller's words, changed right after the upload
        same(stage1(eng, 0.001, 8, False, 200_000, 100_000), want, ("async host", chunk))


def test_calls_that_bring_the_bases_back(eng, lambda_reads):
    """rvn_edit_distance_batch, rvn_stage1_pile_regions + stage 2 and
    rvn_align_breaking_points after a host-mode stage 1 equal the device route's; with a
    budget below the set they return RVN_ERR_LIMIT and the engine stays usable."""
    rs = lambda_reads
    eng.configure(k=15, w=5)
    rng = np.random.default_rng(3)
    n = 200
    a, b = rng.integers(0, rs.n, n), rng.integers(0, rs.n, n)
    la, lb = rs.lens[a], rs.lens[b]
    ab = (rng.random(n) * la * 0.5).astype(np.uint32)
    bb = (rng.random(n) * lb * 0.5).astype(np.uint32)
    al = np.minimum(la - ab, 400).astype(np.uint32)
    bl = np.minimum(lb - bb, 400).astype(np.uint32)
    st = rng.integers(0, 2, n).astype(np.uint8)
    words = rs.words.size * 8

    def run(mode, budget_first):
        upload(eng, rs, mode)
        out = dict(s1=stage1(eng, 0.001, 32, False))
        if budget_first:
            eng.set_host_bases(1, words // 2)
            with pytest.raises(OverflowError):
                eng.edit_distance_batch(a, ab, al, b, bb, bl, st)
            assert eng.reads_residency()["on_host"]
            same(stage1(eng, 0.001, 32, False), out["s1"], "after the refusal")
            eng.set_host_bases(1, 0)
        out["ed"] = eng.edit_distance_batch(a, ab, al, b, bb, bl, st)
        assert not eng.reads_residency()["on_host"]
        out["bp"] = eng.align_breaking_points(a, ab, al, st, b, bb, bl, 500)
        out["regions"] = eng.stage1_pile_regions(4)
        reg = out["regions"]
        end = np.minimum(reg["end"].astype(np.int64) * 16, rs.lens)
        begin = np.minimum(reg["begin"].astype(np.int64) * 16, end)
        out["s2"] = eng.find_overlaps_and_repetitive_regions(0.001, 0.1, rs.n, begin, end)
        return out

    dev = run(0, False)
    host = run(1, True)
    same(host["s1"], dev["s1"], "stage 1")
    assert np.array_equal(host["ed"], dev["ed"])
    for x, y in zip(host["bp"], dev["bp"]):
        assert np.array_equal(x, y)
    for key in dev["regions"]:
        assert np.array_equal(host["regions"][key], dev["regions"][key]), key
    for key in ("overlaps", "ovl_off", "kmer_bits", "kmer_off", "touched"):
        assert np.array_equal(host["s2"][key], dev["s2"][key]), key
    assert host["s2"]["num_mapped"] == dev["s2"]["num_mapped"]
    # the whole set on the device: the next upload decides again
    upload(eng, rs, 1)
    eng.set_host_bases(1, words // 2)
    for call in (lambda: eng.align_breaking_points(a, ab, al, st, b, bb, bl, 500),
                 lambda: eng.kmer_complexity(a, ab, 15)):
        with pytest.raises(OverflowError):
            call()


def test_auto(eng):
    """Small sets stay on the device with the launches of host_bases=0. A set of several
    reference index batches moves to the host when the budget lies between the two
    estimates, and stays on the device below both; the host estimate is the smaller."""
    rs = synth.make_reads(30_000, 150, 3000, seed=3)
    eng.configure(k=15, w=5)
    upload(eng, rs, 0)
    eng.set_option("reset_stats", 0)
    want = stage1(eng, 0.001, 8, False, 120_000, 50_000)
    launches = eng.stats()["kernel_launches"]
    eng.set_host_bases(-1, 0)
    eng.upload(rs)
    assert not eng.reads_residency()["on_host"]
    eng.set_option("reset_stats", 0)
    same(stage1(eng, 0.001, 8, False, 120_000, 50_000), want, "auto")
    assert eng.stats()["kernel_launches"] == launches
    assert "stage_bases" not in eng.timings()

    # 8300 reads of 2^20 bases: three reference index batches (no pass runs on it)
    n, length = 8300, 1 << 20
    big = seqio.ReadSet(np.zeros(n * (length // 32), np.uint64),
                        np.arange(n + 1, dtype=np.uint64) * (length // 32),
                        np.full(n, length, np.uint32))
    e = engine.Engine(device=0)
    try:
        e.set_index_chunks(1 << 30)   # the chunk size of the auto decision's estimate
        est = {}
        for mode in (0, 1):
            e.set_host_bases(mode)
            e.upload(big)
            est[mode] = e.stage1_footprint(32)["windowed_device"]
            dev_bytes = e.reads_residency()["device_word_bytes"]
            assert (dev_bytes == 0) if mode else (dev_bytes >= big.words.size * 8)
        assert est[1] < est[0]
        e.set_host_bases(-1, (est[0] + est[1]) // 2)
        e.upload(big)
        assert e.reads_residency()["on_host"]
        e.set_host_bases(-1, est[1] // 2)
        e.upload(big)
        assert not e.reads_residency()["on_host"]
        with pytest.raises(ValueError):
            e.set_option("host_bases", 2)
        with pytest.raises(ValueError):
            e.set_option("host_bases_budget", -1)
    finally:
        e.close()


@pytest.mark.parametrize("minhash", [False, True])
def test_reference_stage1_over_facade(tmp_path, oracle, lambda_reads, host_env, minhash):
    a, b = run_dropin(tmp_path, lambda_reads, 15, 5, 0.001, 32, minhash)
    want = oracle.stage1(oracle.engine(15, 5, threads=4), oracle.reads(lambda_reads), 0.001, 32,
                         minhash)
    for got in (a, b):
        for key in KEYS:
            assert np.array_equal(got[key], want[key]), key


def test_assembly_pin(tmp_path, oracle, lambda_reads, host_env):
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
