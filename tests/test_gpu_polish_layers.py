"""racon::Polisher::Polish with its window layers built on the device and the consensus
run in window batches (rvn_polish_windows): the facade (raven_b200.polish) against the
oracle polisher, byte for byte - names, sequences, window and polished-window counts -
over the cases racon's layer rules tell apart: qualities on all, some or no reads, a
piece average exactly at q and just below it, window lengths other than 500, both
strands and read lengths around the 32- and 64-base word and quality blocks, the error
filter, forced window batches, deep windows, and reads flagged is_reverse_complement."""
from __future__ import annotations

import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from raven_b200 import seqio  # noqa: E402

gpu = pytest.mark.gpu

_COMP = np.array([3, 2, 1, 0], np.uint8)


def _mutate(rng, codes, rate):
    """substitutions, insertions and deletions at rate/3 each"""
    out = []
    for c in codes:
        u = rng.random()
        if u < rate / 3:
            continue
        if u < 2 * rate / 3:
            out.append((c + rng.integers(1, 4)) % 4)
        else:
            out.append(c)
            if u < rate:
                out.append(rng.integers(0, 4))
    return np.array(out, np.uint8)


def make_set(seed, genome_len=30_000, n_reads=160, mean_len=3000, err=0.06, contig_len=10_000,
             extra_lens=(1024, 2048, 4096, 1600, 3200, 48, 60)):
    """draft contigs of a random genome and reads sampled from both strands of it, with
    the strand of every read returned; extra_lens adds reads of those lengths (multiples
    of 32 and 64, and reads shorter than 64)"""
    rng = np.random.default_rng(seed)
    genome = rng.integers(0, 4, genome_len).astype(np.uint8)
    lens = list(rng.integers(mean_len // 2, mean_len * 3 // 2, n_reads)) + list(extra_lens)
    reads, strands = [], []
    for i, ln in enumerate(lens):
        b = int(rng.integers(0, genome_len - ln))
        r = _mutate(rng, genome[b:b + ln], err)
        fwd = i % 2 == 0
        if not fwd:
            r = _COMP[r[::-1]]
        reads.append(r)
        strands.append(fwd)
    contigs = [_mutate(rng, genome[b:b + contig_len], 0.01)
               for b in range(0, genome_len, contig_len)]
    return seqio.pack_codes(contigs), seqio.pack_codes(reads), np.array(strands), lens


def with_quality(reads, values, which=None):
    """block qualities: values(i, n_blocks) for the reads in `which` (all when None),
    an empty range for the others"""
    blocks = []
    for i in range(reads.n):
        nb = (int(reads.lens[i]) + 63) // 64
        if which is None or i in which:
            blocks.append(np.asarray(values(i, nb), np.uint8))
        else:
            blocks.append(np.zeros(0, np.uint8))
    reads.block_quality = np.concatenate(blocks)
    reads.bq_off = np.concatenate([[0], np.cumsum([b.size for b in blocks])]).astype(np.uint64)
    return reads


def run_pair(oracle, draft, reads, **kw):
    from raven_b200 import polish
    got, st = polish.polish(draft, reads, threads=4, **kw)
    names, seqs, ost = oracle.polish(draft, reads, threads=8, **kw)
    assert got.names == names
    assert [got.ascii(i) for i in range(got.n)] == seqs
    assert st["windows"] == int(ost[0]) and st["polished_windows"] == int(ost[1])
    return got, st


def coverage_tags(rs):
    return [int(n.split(" RC:i:")[1].split()[0]) for n in rs.names]


class Options:
    """RVN_SET_OPTIONS for the contexts the facade creates inside the block"""

    def __init__(self, value):
        self.value = value

    def __enter__(self):
        os.environ["RVN_SET_OPTIONS"] = self.value

    def __exit__(self, *exc):
        del os.environ["RVN_SET_OPTIONS"]


@pytest.fixture(scope="module")
def base_set():
    return make_set(11)


@gpu
def test_qualities_none_all_some(oracle, base_set):
    draft, reads, strands, lens = base_set
    assert strands.any() and not strands.all()
    lens = np.asarray(reads.lens)
    assert (lens % 64 == 0).any() and (lens % 64 == 32).any() and (lens < 64).any()
    _, st = run_pair(oracle, draft, reads)
    assert st["polished_windows"] > 20
    rng = np.random.default_rng(3)
    all_q = with_quality(reads.subset(range(reads.n)), lambda i, nb: rng.integers(4, 25, nb))
    run_pair(oracle, draft, all_q, q=10.0)
    run_pair(oracle, draft, all_q, q=0.0)
    some = set(range(0, reads.n, 3))
    some_q = with_quality(reads.subset(range(reads.n)), lambda i, nb: rng.integers(4, 25, nb),
                          which=some)
    assert any(some_q.bq_off[i] == some_q.bq_off[i + 1] for i in range(reads.n))
    run_pair(oracle, draft, some_q, q=10.0)


@gpu
def test_average_exactly_at_q_and_just_below(oracle, base_set):
    draft, reads, _, _ = base_set
    q = 10.0
    # every block 10: every piece averages exactly q (an integer sum over its bases / d)
    at_q = with_quality(reads.subset(range(reads.n)), lambda i, nb: np.full(nb, 10))
    for d in (1, 7, 500, 777):
        assert (10 * d) / d == q
    got_at, st_at = run_pair(oracle, draft, at_q, q=q)
    assert st_at["polished_windows"] > 20  # kept: avg < q is false
    # just above q every piece drops: the equal case decides
    got_up, st_up = run_pair(oracle, draft, at_q, q=float(np.nextafter(q, 11.0)))
    assert st_up["polished_windows"] == 0
    # one block of 9 per read: the pieces over it average 10 - k/d, just below q
    below = with_quality(reads.subset(range(reads.n)),
                         lambda i, nb: np.where(np.arange(nb) == nb // 2, 9, 10))
    for k, d in ((1, 800), (64, 600)):
        assert 0 < q - (10 * d - k) / d <= 0.11
    got_below, _ = run_pair(oracle, draft, below, q=q)
    assert coverage_tags(got_below) == coverage_tags(got_at)
    assert [got_below.ascii(i) for i in range(got_below.n)] != \
        [got_at.ascii(i) for i in range(got_at.n)]


@gpu
def test_window_lengths(oracle, base_set):
    draft, reads, _, _ = base_set
    rng = np.random.default_rng(5)
    q_reads = with_quality(reads.subset(range(reads.n)), lambda i, nb: rng.integers(6, 22, nb))
    for w in (200, 137, 1000):
        _, st = run_pair(oracle, draft, reads, w=w)
        assert st["windows"] == sum((int(x) + w - 1) // w for x in draft.lens)
        run_pair(oracle, draft, q_reads, w=w, q=8.0)


@gpu
def test_error_filter_drops_alignments(oracle, base_set):
    draft, reads, _, _ = base_set
    got, _ = run_pair(oracle, draft, reads, e=0.3)
    tight, _ = run_pair(oracle, draft, reads, e=0.01)
    assert sum(coverage_tags(tight)) < sum(coverage_tags(got))
    assert sum(coverage_tags(tight)) > 0


@gpu
def test_forced_window_batches(oracle, base_set):
    from raven_b200 import polish
    draft, reads, _, _ = base_set
    rng = np.random.default_rng(9)
    q_reads = with_quality(reads.subset(range(reads.n)), lambda i, nb: rng.integers(6, 22, nb),
                           which=set(range(0, reads.n, 2)))
    for rs, q in ((reads, 0.0), (q_reads, 8.0)):
        want, st = run_pair(oracle, draft, rs, q=q)
        assert st["window_batches"] == 1  # auto: the whole set fits
        seqs = [want.ascii(i) for i in range(want.n)]
        for size, expect in (("1", st["windows"]), ("60000", None), ("0", 1)):
            with Options(f"poa_batch_bytes={size}"):
                got, gst = polish.polish(draft, rs, q=q, threads=4)
            assert got.names == want.names
            assert [got.ascii(i) for i in range(got.n)] == seqs
            assert gst["polished_windows"] == st["polished_windows"]
            assert gst["wide_windows"] == st["wide_windows"]
            if expect is not None:
                assert gst["window_batches"] == expect
            else:
                # about 500 bases x ~20 layers x 2-3 bytes per window: a few windows each
                assert 1 < gst["window_batches"] < st["windows"]


def concat(a, b):
    """targets first, then the reads: the set the facade uploads"""
    words = np.concatenate([a.words, b.words]).astype(np.uint64)
    woff = np.concatenate([a.word_off[:-1], b.word_off + a.word_off[-1]]).astype(np.uint64)
    return seqio.ReadSet(words, woff, np.concatenate([a.lens, b.lens]).astype(np.uint32))


def facade_alignments(eng, T, S, e=0.3):
    """the facade's alignments: each read's longest overlap (first of equal spans) that
    passes the error filter, in read order"""
    ovl = eng.map(T, T + S, False, False)
    rows, off = ovl["overlaps"], ovl["ovl_off"]
    out = []
    for k in range(S):
        best = None
        for o in rows[int(off[k]):int(off[k + 1])]:
            span = max(int(o[2]) - int(o[1]), int(o[5]) - int(o[4]))
            if best is None or best[0] < span:
                best = (span, o)
        if best is None:
            continue
        o = best[1]
        ql, tl = float(o[2] - o[1]), float(o[5] - o[4])
        if 1 - min(ql, tl) / max(ql, tl) > e:
            continue
        out.append((T + k, int(o[1]), int(o[2] - o[1]), int(o[7]), int(o[3]), int(o[4]),
                    int(o[5] - o[4])))
    return [np.array(c) for c in zip(*out)]


def layer_shapes(lens, T, w, alns, bp_off, bp, bq, bq_off, q):
    """racon's per-slot rules restated: kept layers and their bases per window"""
    first = np.concatenate([[0], np.cumsum([(int(x) + w - 1) // w for x in lens[:T]])])
    cnt = np.zeros(int(first[-1]), np.int64)
    bases = np.zeros(int(first[-1]), np.int64)
    qr, qb0, ql, strand, tr = alns[:5]
    for a in range(qr.size):
        L = int(lens[qr[a]])
        qb = int(qb0[a]) if strand[a] else L - (int(qb0[a]) + int(ql[a]))
        for s in range(int(bp_off[a]), int(bp_off[a + 1])):
            ft, y, lt, z = (int(v) for v in bp[s])
            if ft == 0xFFFFFFFF:
                continue
            fq, lq = qb + y, qb + z
            if not lq - fq >= 0.02 * w:
                continue
            k0, k1 = int(bq_off[qr[a]]), int(bq_off[qr[a] + 1])
            if k1 > k0:
                x = np.arange(fq, lq)
                idx = (L - 1 - x) if not strand[a] else x
                if bq[k0 + (idx >> 6)].astype(np.int64).sum() / (lq - fq) < q:
                    continue
            ws = ft // w * w
            if ft - ws >= lt - ws - 1:
                continue
            cnt[first[tr[a]] + ft // w] += 1
            bases[first[tr[a]] + ft // w] += lq - fq
    return first, cnt, bases


def greedy_batches(need, budget):
    n = i = 0
    while i < len(need):
        j, b = i, 0
        while j < len(need) and (j == i or b + need[j] <= budget):
            b += need[j]
            j += 1
        n, i = n + 1, j
    return n


@gpu
def test_batches_follow_window_shapes(base_set):
    """rvn_polish_windows on the facade's alignments: the polished windows are those the
    restated rules give at least two layers, the batch count is the greedy cut of the
    documented per-window bytes, and every batch size gives the facade's output"""
    from raven_b200 import engine, polish
    draft, reads, _, _ = base_set
    rng = np.random.default_rng(13)
    rs = with_quality(reads.subset(range(reads.n)), lambda i, nb: rng.integers(6, 22, nb),
                      which=set(range(0, reads.n, 2)))
    T, S, w, q = draft.n, rs.n, 500, 8.0
    allr = concat(draft, rs)
    eng = engine.Engine()
    eng.configure(15, 5, 500, 4, 100, 10000)
    eng.upload(allr)
    eng.minimize(0, T)
    eng.filter(0.001)
    alns = facade_alignments(eng, T, S)
    _, bp_off, bp = eng.align_breaking_points(*alns, window=w)
    bq_off = np.concatenate([np.zeros(T, np.uint64), rs.bq_off]).astype(np.uint64)
    first, cnt, bases = layer_shapes(allr.lens, T, w, alns, bp_off, bp, rs.block_quality,
                                     bq_off, q)
    bb = np.array([min(int(allr.lens[t]), (j + 1) * w) - j * w
                   for t in range(T) for j in range(int(first[t + 1] - first[t]))])
    need = [3 * (int(bb[x]) + int(bases[x])) + 20 * (1 + int(cnt[x])) + 64
            for x in range(cnt.size)]
    want, _ = polish.polish(draft, rs, q=q, threads=4)
    results = []
    for budget in (1, 60_000, 150_000, sum(need) - 1, 0):
        eng.set_option("poa_batch_bytes", budget)
        r = eng.polish_windows(alns[0], alns[1], alns[2], alns[3], alns[4], bp_off, bp, T,
                               window=w, block_quality=rs.block_quality, bq_off=bq_off, q=q)
        assert r["batches"] == (greedy_batches(need, budget) if budget else 1), budget
        assert ((r["status"] & 1) == 1).tolist() == (cnt >= 2).tolist()
        results.append(r)
    assert 2 < results[1]["batches"] < cnt.size and results[3]["batches"] == 2
    for r in results:
        assert r["consensus"].tobytes() == results[0]["consensus"].tobytes()
        for t in range(T):
            c0, c1 = r["cons_off"][first[t]], r["cons_off"][first[t + 1]]
            assert r["consensus"][int(c0):int(c1)].tobytes() == want.ascii(t)


@gpu
def test_polish_windows_rejects_offsets_not_from_zero(base_set):
    from raven_b200 import engine
    draft, reads, _, _ = base_set
    eng = engine.Engine()
    eng.configure(15, 5, 500, 4, 100, 10000)
    eng.upload(concat(draft, reads))
    bp = np.full((3, 4), 0xFFFFFFFF, np.uint32)
    with pytest.raises(ValueError, match="bp_off must start at 0"):
        eng.polish_windows([draft.n], [0], [100], [1], [0], [1, 3], bp, draft.n)


@gpu
def test_deep_windows_in_small_batches(oracle):
    from bench import synth as bsynth
    from raven_b200 import polish
    # about 150x over a 20 kb draft: windows past the 16-bit kernels (wide route)
    reads = bsynth.make_reads(401, 20_000, 650, 5000, min_len=1500)
    draft = bsynth.make_contigs(401, 20_000, contig_len=20_000)
    want, st = run_pair(oracle, draft, reads)
    assert st["wide_windows"] > 0
    with Options("poa_batch_bytes=400000"):
        got, gst = polish.polish(draft, reads, threads=4)
    assert [got.ascii(i) for i in range(got.n)] == [want.ascii(i) for i in range(want.n)]
    assert gst["wide_windows"] == st["wide_windows"]
    assert gst["window_batches"] > 3


@gpu
def test_reverse_complement_flagged_objects():
    """targets and reads whose NucleicAcid has is_reverse_complement set (reachable only
    from C++): the facade against the oracle polisher on the same objects"""
    exe = os.path.join(ROOT, "tests", "cpp", "_build", "polish_rc_test")
    assert os.path.exists(exe), "built by __graft_entry__.build()"
    r = subprocess.run([exe, os.path.join(ROOT, "oracle", "liboracle.so")],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "polish_rc_test ok" in r.stdout, r.stdout
