"""rvn_minimize in chunks (option "index_chunk_bases"): the index of every record, built
without a sketch of the whole range, must be the one-shot build's bit for bit: records in
order, key count and occurrence threshold at every frequency, also after rvn_filter has
freed the build's buffers. Maps over it (self-join of the batch's own reads, probes by
earlier reads with micromizers and with full sketches) must return the one-shot results.
k15 w5 sketches straight into the sort's buffers (SketchFastKernel's append mode), the
other (k, w) sketch each chunk and copy it."""
import numpy as np
import pytest

from raven_b200 import seqio, synth

pytestmark = pytest.mark.gpu

FLAGS = ((1, 1, 1, 0), (1, 1, 0, 1), (0, 0, 0, 0))   # stage 1, stage 2, the polisher


@pytest.fixture
def eng(gpu_engine):
    try:
        yield gpu_engine
    finally:
        gpu_engine.set_index_chunks(-1, 0)
        gpu_engine.set_option("map_flush_bases", 0)
        gpu_engine.configure(k=15, w=5)


def reads_with_edges(seed):
    """overlapping reads, plus reads without minimizers and a dense tandem repeat"""
    rs = synth.make_reads(40_000, 120, 3000, seed=seed)
    rng = np.random.default_rng(seed)
    seqs = [rs.codes(i) for i in range(rs.n)]
    seqs.insert(50, rng.integers(0, 4, 10, dtype=np.uint8))
    seqs.insert(51, np.tile(np.array([0, 1], np.uint8), 1200))
    seqs.append(rng.integers(0, 4, 17, dtype=np.uint8))
    return seqio.pack_codes(seqs)


def build(eng, first, last, minhash, chunk, freqs=(0.001, 0.01, 0.0)):
    """minimize + one filter per frequency: chunked?, records, and per frequency the
    threshold (the second and third filter run after the release)"""
    eng.set_index_chunks(chunk)
    eng.set_option("reset_stats", 0)
    eng.minimize(first, last, minhash)
    chunked = eng.minimize_chunked()
    occ = [eng.filter(f) for f in freqs]
    return chunked, eng.index_records(), occ


def same_index(a, b, tag):
    assert a[1]["n_keys"] == b[1]["n_keys"], tag
    assert np.array_equal(a[1]["value"], b[1]["value"]), tag
    assert np.array_equal(a[1]["origin"], b[1]["origin"]), tag
    assert a[2] == b[2], tag


def same_map(a, b, tag):
    for key in ("overlaps", "ovl_off", "filt_off", "filtered"):
        assert np.array_equal(a[key], b[key]), (tag, key)


@pytest.mark.parametrize("minhash", [False, True])
@pytest.mark.parametrize("k,w", [(15, 5), (15, 8), (19, 10), (31, 32)])
def test_index_identity(eng, k, w, minhash):
    rs = reads_with_edges(5)
    eng.configure(k=k, w=w)
    eng.upload(rs)
    total = int(rs.lens.sum())
    for first in (0, 37):
        one = build(eng, first, rs.n, minhash, 0)
        assert not one[0]
        assert one[2][0] != 0xFFFFFFFF and one[2][2] == 0xFFFFFFFF
        # one chunk, two, many, one per read (a chunk smaller than any read)
        for chunk in (4 * total, total // 2, 20_000, 1):
            got = build(eng, first, rs.n, minhash, chunk)
            assert got[0] or minhash, chunk   # (minhash: one sweep, no "sketch_tiers" work)
            same_index(got, one, (k, w, minhash, first, chunk))
    # an empty range
    assert build(eng, 7, 7, minhash, 1)[1]["value"].size == 0


@pytest.mark.parametrize("k,w", [(15, 5), (19, 10)])
def test_map_identity_over_chunked_index(eng, k, w):
    rs = reads_with_edges(11)
    eng.configure(k=k, w=w)
    eng.upload(rs)
    j = 45
    want = {}
    for chunk in (0, 25_000, 1):
        for minhash in (False, True):
            build(eng, j, rs.n, minhash, chunk, freqs=(0.001,))
            for flags in FLAGS:
                # the batch's own reads (flags (1,1,1,0): the self-join), the reads before it
                for rng_ in ((j, rs.n), (0, j), (0, rs.n)):
                    got = eng.map(*rng_, *[bool(f) for f in flags])
                    key = (minhash, flags, rng_)
                    if chunk == 0:
                        want[key] = got
                        continue
                    same_map(got, want[key], (chunk, key))
    assert sum(v["overlaps"].shape[0] for v in want.values()) > 1000
    assert sum(v["filtered"].size for v in want.values()) > 0


def test_filter_again_after_release(eng):
    """an untiered index has no bare keys: any frequency, in any order, after the release"""
    rs = reads_with_edges(3)
    eng.configure(k=15, w=5)
    eng.upload(rs)
    freqs = (0.3, 0.0, 0.001, 0.05)
    one = build(eng, 0, rs.n, False, 0, freqs)
    got = build(eng, 0, rs.n, False, 9_000, freqs)
    assert got[0]
    same_index(got, one, "filters")
    assert len(set(one[2])) >= 3


def test_auto_decision(eng):
    """Auto chunks only when the one-shot estimate exceeds the budget, for rvn_minimize as
    for stage 1; the results are the same either way."""
    rs = synth.make_reads(30_000, 150, 3000, seed=3)
    eng.configure(k=15, w=5)
    eng.upload(rs)
    eng.set_index_chunks(-1, 0)
    fp = eng.minimize_footprint(0, rs.n)
    assert 0 < fp["chunked"] <= fp["one_shot"] and fp["chunk"] == 0
    assert eng.minimize_footprint(10, 10)["one_shot"] < fp["one_shot"]
    one = build(eng, 0, rs.n, False, -1)
    assert not one[0]
    eng.set_index_chunks(-1, fp["one_shot"] - 1)
    assert eng.minimize_footprint(0, rs.n)["chunk"] == 1 << 30
    eng.set_option("reset_stats", 0)
    eng.minimize(0, rs.n)
    assert eng.minimize_chunked()
    got = (True, None, [eng.filter(f) for f in (0.001, 0.01, 0.0)])
    got = (True, eng.index_records(), got[2])
    same_index(got, one, "auto")
    eng.set_index_chunks(-1, fp["one_shot"] + 1)
    assert eng.minimize_footprint(0, rs.n)["chunk"] == 0
    # stage 1 decides with its own estimate through the same budget
    s1 = eng.stage1_footprint(8)
    fit = min(s1["resident"], s1["windowed_device"])
    eng.set_index_chunks(-1, fit - 1)
    eng.find_overlaps_and_create_piles(0.001, 8)
    assert eng.stage1_index_chunked()
    eng.set_index_chunks(-1, fit + (1 << 20))
    eng.find_overlaps_and_create_piles(0.001, 8)
    assert not eng.stage1_index_chunked()
    eng.set_index_chunks(1000)
    assert eng.minimize_footprint(0, rs.n)["chunk"] == 1000
