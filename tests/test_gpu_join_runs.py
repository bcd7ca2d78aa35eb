"""Stage-1 self-join on runs that span many warps of the sweep (map.cu, JoinSweepKernel):
near-identical reads give value runs of 70-120 postings, tandem repeats give runs of
hundreds in which one read holds a segment longer than a warp. Frequency 0 leaves the
occurrence threshold unlimited; the other frequencies put it inside and below those runs.
Bit exact against the CPU oracle, with one and with several index batches and flushes."""
import numpy as np
import pytest

from raven_b200 import seqio

pytestmark = pytest.mark.gpu


def repeat_reads():
    rng = np.random.default_rng(41)
    seqs = []
    for unit_len, copies in ((2000, 120), (1500, 70)):
        unit = rng.integers(0, 4, unit_len, dtype=np.uint8)
        for _ in range(copies):
            s = unit.copy()
            at = rng.integers(0, unit_len, 6)            # a few substitutions per copy
            s[at] = (s[at] + rng.integers(1, 4, 6)) % 4
            seqs.append(s.astype(np.uint8))
    tile = rng.integers(0, 4, 50, dtype=np.uint8)
    for n in (300, 280, 310):                              # tandem repeats
        seqs.append(np.tile(tile, n))
    seqs += [rng.integers(0, 4, 2000, dtype=np.uint8) for _ in range(40)]
    order = rng.permutation(len(seqs))                     # copies spread over the read ids
    return seqio.pack_codes([seqs[i] for i in order])


FREQS = (0.0, 0.002, 0.02, 0.3)


@pytest.mark.parametrize("ib,qb", [(0, 0), (250_000, 120_000)])
def test_stage1_self_join_long_runs(gpu_engine, oracle, ib, qb):
    rs = repeat_reads()
    eng = oracle.engine(15, 5, threads=4)
    reads = oracle.reads(rs)
    gpu_engine.configure(k=15, w=5)
    gpu_engine.upload(rs)
    occ = []
    for freq in FREQS:
        got = gpu_engine.find_overlaps_and_create_piles(freq, 8, False, ib, qb)
        want = oracle.stage1(eng, reads, freq, 8, False, ib or 1 << 32, qb or 1 << 30)
        for k in ("overlaps", "ovl_off", "pile", "pile_off"):
            assert np.array_equal(got[k], want[k]), (freq, k)
        assert got["num_mapped"] == int(want["num_mapped"][0])
        occ.append(gpu_engine.stats()["occurrence"])
    # the thresholds the cases rely on: unlimited, and limited above one warp
    assert occ[0] == 0xFFFFFFFF
    assert any(32 < o < 0xFFFFFFFF for o in occ[1:]), occ
