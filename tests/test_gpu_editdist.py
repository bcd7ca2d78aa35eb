"""GPU: batched global edit distance (raven_b200/csrc/editdist.cu) - the
edlibAlign(lhs, rhs, edlibDefaultAlignConfig()).editDistance of the identity filter
(RavenLib/src/construct.cc:176-199,393-416) - against the oracle's textbook
dynamic programme: exact, every band tier, both strands."""
import numpy as np
import pytest

from raven_b200 import seqio, synth

pytestmark = pytest.mark.gpu


def _sub(rs, r, b, n, strand):
    s = rs.codes(r)[b:b + n]
    if not strand:
        s = (3 - s[::-1]).astype(np.uint8)
    return np.frombuffer(b"ACGT", np.uint8)[s].tobytes()


def test_edit_distance_batch_matches_oracle(gpu_engine, oracle):
    rng = np.random.default_rng(5)
    base = rng.integers(0, 4, 9000, dtype=np.uint8)
    seqs = [base]
    # error rates that land in every tier (k = 64, 192, 448, 960) and beyond
    for err in (0.0, 0.002, 0.01, 0.03, 0.06, 0.12, 0.2, 0.35):
        seqs.append(np.asarray(synth.mutate(base, rng, err / 3, err / 3, err / 3), dtype=np.uint8))
    seqs.append((3 - base[::-1]).astype(np.uint8))          # reverse complement
    seqs.append(rng.integers(0, 4, 700, dtype=np.uint8))    # unrelated
    seqs.append(np.zeros(300, np.uint8))
    seqs.append(rng.integers(0, 4, 1, dtype=np.uint8))
    rs = seqio.pack_codes(seqs)
    gpu_engine.configure(15, 5)
    gpu_engine.upload(rs)
    pairs = []
    n0 = len(base)
    for j in range(1, 9):
        pairs.append((0, 0, n0, j, 0, int(rs.lens[j]), 1))
        pairs.append((0, 100, 3000, j, 90, 3100, 1))             # unaligned starts
        pairs.append((j, 17, 4000, 0, 33, 3900, 1))
    pairs.append((0, 0, n0, 9, 0, n0, 0))                         # rhs reverse complemented
    pairs.append((1, 500, 2500, 9, n0 - 3000, 2500, 0))
    pairs.append((0, 0, 63, 1, 0, 64, 1))
    pairs.append((0, 0, 64, 1, 0, 65, 1))
    pairs.append((0, 5, 129, 10, 0, 700, 1))                      # unrelated, unequal
    pairs.append((11, 0, 300, 11, 0, 300, 1))                     # homopolymer with itself
    pairs.append((11, 0, 300, 0, 0, 200, 0))
    pairs.append((12, 0, 1, 12, 0, 1, 0))                         # one base vs its complement
    pairs.append((12, 0, 0, 0, 0, 10, 1))                         # empty lhs
    pairs.append((0, 7, 10, 12, 0, 0, 1))                         # empty rhs
    for _ in range(40):
        a, b = rng.integers(0, 10, 2)
        la, lb = int(rs.lens[a]), int(rs.lens[b])
        na, nb = int(rng.integers(1, min(la, 2500))), int(rng.integers(1, min(lb, 2500)))
        pairs.append((int(a), int(rng.integers(0, la - na + 1)), na, int(b),
                      int(rng.integers(0, lb - nb + 1)), nb, int(rng.integers(0, 2))))
    P = np.array(pairs, dtype=np.int64)
    got = gpu_engine.edit_distance_batch(P[:, 0], P[:, 1], P[:, 2], P[:, 3], P[:, 4], P[:, 5],
                                         P[:, 6])
    want = np.array([oracle.edit_distance(_sub(rs, p[0], p[1], p[2], 1),
                                          _sub(rs, p[3], p[4], p[5], p[6])) for p in pairs],
                    dtype=np.int32)
    assert np.array_equal(got, want)
    # bounded: -1 exactly where the distance exceeds the limit
    for lim in (0, 10, 64, 65, 200, 1000, 5000):
        limit = np.full(len(pairs), lim, dtype=np.int32)
        g = gpu_engine.edit_distance_batch(P[:, 0], P[:, 1], P[:, 2], P[:, 3], P[:, 4], P[:, 5],
                                           P[:, 6], limit)
        assert np.array_equal(g, np.where(want <= lim, want, -1)), lim
    with pytest.raises(ValueError):
        gpu_engine.edit_distance_batch([0], [0], [10**6], [1], [0], [10], [1])


TIER_K = (64, 192, 448, 960)   # kTierK; a tier's CTA holds 128, 128, 64, 64 pairs


def _subs(rng, s, d):
    """d substitutions spread evenly."""
    s = s.copy()
    pos = np.linspace(3, len(s) - 4, d).astype(np.int64)
    s[pos] = (s[pos] + rng.integers(1, 4, d, dtype=np.uint8)) & 3
    return s


def _cut(s, at, d):
    return np.concatenate([s[:at], s[at + d:]])


def test_edit_distance_tier_edges(gpu_engine, oracle):
    """Distances and |m - n| at every tier's k and k + 1, limits around them, block
    lengths 64j - 1 .. 64j + 1, the last read of the upload, HiFi-sized pairs, and
    more than one CTA of pairs in every tier and in the unbanded kernel."""
    rng = np.random.default_rng(8)
    base = rng.integers(0, 4, 16_000, dtype=np.uint8)
    distinct = []   # (lhs, rhs, copies, distance by construction or None)

    for d in (63, 64, 65, 191, 192, 193, 447, 448, 449, 959, 960, 961):
        distinct.append((base[:3000 + d], _cut(base[:3000 + d], 1000, d), 1, d))   # |m - n| = d
        distinct.append((base[:9700], _subs(rng, base[:9700], d), 1, d))           # m == n
    for k in TIER_K:   # |m - n| at k (the tier runs) and at k + 1 (it exits at once)
        for gap in (k, k + 1):
            s = base[2000:4500 + gap]
            distinct.append((s, _subs(rng, _cut(s, 700, gap), 5), 1, None))
    for j in (1, 2, 64):
        for la in (64 * j - 1, 64 * j, 64 * j + 1):
            for lb in (64 * j - 1, 64 * j, 64 * j + 1):
                rhs = np.asarray(synth.mutate(base[500:500 + lb + 8], rng, 0.01, 0.005, 0.005),
                                 dtype=np.uint8)[:lb]
                distinct.append((base[500:500 + la], rhs, 1, None))
    for n, err in ((10_000, 0.001), (12_500, 0.005), (15_000, 0.01), (14_000, 0.003)):
        rhs = np.asarray(synth.mutate(base[:n], rng, err / 3, err / 3, err / 3), dtype=np.uint8)
        distinct.append((base[:n], rhs, 1, None))
    # more than one CTA of pairs in every tier, and in the unbanded kernel
    for d in (30, 150, 300, 700, 1500):
        for x in range(5):
            s = base[x * 1000:x * 1000 + 3000]
            distinct.append((s, _subs(rng, s, d), 30, None))

    seqs, pairs, groups = [], [], []
    for x, (lhs, rhs, copies, _) in enumerate(distinct):
        strand = x % 2
        lp, rp = 1 + x % 63, 2 + (5 * x) % 61
        seqs.append(np.concatenate([rng.integers(0, 4, lp, dtype=np.uint8), lhs,
                                    rng.integers(0, 4, 9, dtype=np.uint8)]))
        r = rhs if strand else (3 - rhs[::-1]).astype(np.uint8)
        seqs.append(np.concatenate([rng.integers(0, 4, rp, dtype=np.uint8), r,
                                    rng.integers(0, 4, 11, dtype=np.uint8)]))
        for _ in range(copies):
            pairs.append((len(seqs) - 2, lp, len(lhs), len(seqs) - 1, rp, len(rhs), strand))
            groups.append(x)
    # the last read of the upload, 64 * 40 + 1 bases, read up to its last base
    last = rng.integers(0, 4, 64 * 40 + 1, dtype=np.uint8)
    other = len(seqs)
    seqs += [base[:2600], last]
    for lr, lb, ll, rr, rb, rl, a, b in (
            (other + 1, 0, len(last), other, 0, 2600, last, base[:2600]),
            (other, 0, 2430, other + 1, 64, len(last) - 64, base[:2430], last[64:]),
            (other + 1, 1, len(last) - 1, other + 1, 0, len(last) - 1, last[1:], last[:-1]),
            (other + 1, 0, len(last), other + 1, 0, len(last), last, last)):
        distinct.append((a, b, 1, None))
        pairs.append((lr, lb, ll, rr, rb, rl, 1))
        groups.append(len(distinct) - 1)
    rs = seqio.pack_codes(seqs)
    gpu_engine.configure(15, 5)
    gpu_engine.upload(rs)

    letters = np.frombuffer(b"ACGT", np.uint8)
    ref = []
    for lhs, rhs, _, d in distinct:
        e = oracle.edit_distance(letters[lhs].tobytes(), letters[rhs].tobytes())
        assert d is None or e == d, (len(lhs), len(rhs), d, e)
        ref.append(e)
    want = np.array([ref[g] for g in groups], dtype=np.int32)
    P = np.array(pairs, dtype=np.int64)
    args = [P[:, i] for i in range(7)]
    # what the pairs were built for: every tier has more than one CTA of pairs
    assert (want > 64).sum() > 128 and (want > 192).sum() > 64 and (want > 960).sum() > 64
    assert np.array_equal(gpu_engine.edit_distance_batch(*args), want)
    for lim in (want - 1, want, want + 1):   # per pair: just below, at, just above
        lim = np.maximum(lim, 0).astype(np.int32)   # (-1 would mean no limit)
        got = gpu_engine.edit_distance_batch(*args, lim)
        assert np.array_equal(got, np.where(want <= lim, want, -1))
    for lim in (100, 500, 2000) + TIER_K + tuple(k + 1 for k in TIER_K):
        got = gpu_engine.edit_distance_batch(*args, np.full(len(P), lim, np.int32))
        assert np.array_equal(got, np.where(want <= lim, want, -1)), lim
