"""Stage 2 at its edges, shared by tests/test_stage2_restatement.py (CPU) and
tests/test_gpu_stage2_edges.py (H100): read sets whose valid regions the test chooses, and
a CPU restatement of rvn_find_overlaps_and_repetitive_regions, flush by flush, from
independent pieces: the oracle's ram (minimize, filter, map and its filtered positions),
the reference's OverlapUpdate as test_gpu_stage2.overlap_update restates it, the textbook
edit distance DP, the reference's double arithmetic for the score and the oracle's
Pile::AddKmers complexity test. Read sets hold reads by id 0..n-1; the call sees the valid
ones in the reference's sorted order (by id), optionally followed by the invalid ones."""
from __future__ import annotations

import dataclasses

import numpy as np

from raven_b200 import seqio, synth
from test_gpu_stage2 import overlap_update

TIER_K = (64, 192, 448, 960)   # the banded tiers; beyond the last, the unbanded kernel
TIER_PHASES = ("myers_k64", "myers_k192", "myers_k448", "myers_k960", "myers_full")
MIN_REGION = 1260              # Pile::FindValidRegion's shortest valid region
# lengths of the unrelated middles of the divergent pairs: their clipped distances land
# in every tier (asserted where they are used)
MIDDLES = (60, 150, 400, 900, 2100)
IDENTITIES = (0.0, 1e-9, 0.5, 0.9, 1.0)
FREQS = (0.0, 0.001, 0.3)
OFF_KW = ((19, 10), (24, 64))  # (24, 64): a long k and wide window of test_gpu_kw_routes


@dataclasses.dataclass
class EdgeSet:
    rs: seqio.ReadSet          # every read, by id
    invalid: np.ndarray        # bool per id
    begin: np.ndarray          # valid region per id, in bases
    end: np.ndarray
    kinds: list                # what each read was built as

    @property
    def valid(self):
        return np.flatnonzero(~self.invalid).astype(np.uint32)

    def upload_ids(self, with_invalid):
        """The reference's sorted order: valid reads by id, then (optionally) the invalid."""
        ids = self.valid
        if with_invalid:
            ids = np.concatenate([ids, np.flatnonzero(self.invalid).astype(np.uint32)])
        return ids

    def region(self):
        return {int(i): (int(self.begin[i]), int(self.end[i])) for i in range(self.rs.n)}


def _rc(s):
    return (3 - s[::-1]).astype(np.uint8)


def edge_reads(seed=7):
    """Overlapping reads of a random genome on both strands, divergent-middle pairs,
    reads shorter than any k used, reads of 511, 512 and 513 bases (the k-mer bitmap
    grows a word at 512), and homopolymer / dinucleotide reads. Ids are shuffled so that
    kinds interleave; two overlapping reads are invalid."""
    rng = np.random.default_rng(seed)
    genome = rng.integers(0, 4, 24_000, dtype=np.uint8)
    seqs, kinds = [], []

    def err(s):
        return synth.mutate(s, rng, 0.003, 0.001, 0.001)

    for _ in range(14):
        ln = int(rng.integers(2000, 4000))
        st = int(rng.integers(0, genome.size - ln))
        s = err(genome[st:st + ln])
        seqs.append(_rc(s) if rng.random() < 0.5 else s)
        kinds.append("genome")
    for n in (511, 512, 513):
        st = int(rng.integers(0, genome.size - n - 64))
        s = genome[st:st + n + 8]
        seqs.append(err(s)[:n])
        kinds.append(f"len{n}")
    for mid in MIDDLES:
        f1 = rng.integers(0, 4, 900, dtype=np.uint8)
        f2 = rng.integers(0, 4, 900, dtype=np.uint8)
        a = np.concatenate([f1, rng.integers(0, 4, mid, dtype=np.uint8), f2])
        b = np.concatenate([err(f1), rng.integers(0, 4, mid, dtype=np.uint8), err(f2)])
        seqs += [a, _rc(b) if mid % 2 else b]
        kinds += [f"mid{mid}", f"mid{mid}"]
    for n in (5, 12):
        seqs.append(rng.integers(0, 4, n, dtype=np.uint8))
        kinds.append("short")
    seqs.append(np.zeros(1500, np.uint8))
    kinds.append("homopolymer")
    seqs.append(np.resize(np.array([0, 1], np.uint8), 1400))
    kinds.append("dinucleotide")
    order = rng.permutation(len(seqs))
    seqs = [seqs[i] for i in order]
    kinds = [kinds[i] for i in order]
    invalid = np.zeros(len(seqs), bool)
    invalid[[i for i, k in enumerate(kinds) if k == "genome"][:2]] = True
    rs = seqio.pack_codes(seqs)
    lens = rs.lens.astype(np.int64)
    return EdgeSet(rs, invalid, np.zeros(rs.n, np.uint32), lens.astype(np.uint32), kinds)


def with_regions(es, oracle, k=15, w=5, aligned=False):
    """The same reads with chosen valid regions: the whole read, the 1260-base minimum,
    and edges that leave a side of some overlap 83, 84 or 85 bases (for `aligned`, in
    whole bins: the side keeps 83-85 bases only where an overlap's end falls so; the
    others still get regions of whole bins)."""
    lens = es.rs.lens.astype(np.int64)
    begin = np.zeros(es.rs.n, np.int64)
    end = lens.copy()
    if aligned:
        end = (lens >> 4) << 4
    base = stage2_overlaps(es, oracle, k, w)
    targets = [83, 84, 85] * 4
    done = set()

    def clipped_min(o, li, b):  # the shorter clipped side with read li's region from b
        reg = {int(i): (int(begin[i]), int(end[i])) for i in range(es.rs.n)}
        reg[li] = (b, reg[li][1])
        c = overlap_update(o, reg)
        return None if c is None else min(c[2] - c[1], c[5] - c[4])

    for o in base:
        o = tuple(int(x) for x in o)
        li, ri, le = o[0], o[3], o[2]
        if not targets or li in done or ri in done or es.kinds[li] != "genome":
            continue
        t = targets[0]
        # the region's first base that leaves the shorter side t bases (83: one past 84)
        keep = 84 if t == 83 else t
        hits = [b for b in range(max(le - keep - 32, 0), le - 64)
                if clipped_min(o, li, b) == keep and not (aligned and (b + (t == 83)) % 16)]
        if not hits:
            continue
        begin[li] = hits[-1] + (t == 83)
        done |= {li, ri}
        targets.pop(0)
    # the 1260-base minimum: on a genome read not clipped above, away from its start
    for i, kd in enumerate(es.kinds):
        if kd == "genome" and i not in done and lens[i] >= MIN_REGION + 400:
            begin[i] = 400
            end[i] = 400 + (MIN_REGION >> 4 << 4 if aligned else MIN_REGION)
            done.add(i)
            break
    return dataclasses.replace(es, begin=begin.astype(np.uint32), end=end.astype(np.uint32))


def stage2_overlaps(es, oracle, k, w, freq=0.001):
    """The map's overlaps of the valid reads over one index (ids translated)."""
    ids = es.upload_ids(False)
    up = es.rs.subset(ids)
    reads = oracle.reads(up)
    eng = oracle.engine(k, w)
    oracle.minimize(eng, reads, 0, up.n, False)
    oracle.filter(eng, freq)
    m = oracle.map(eng, reads, 0, up.n, True, True, False)
    o = m["overlaps"].copy()
    o[:, 0] = ids[o[:, 0]]
    o[:, 3] = ids[o[:, 3]]
    return o


def identity_bound(identity, n):
    """The largest edit distance the filter keeps over a longest side of n bases
    (-1: none): bisection on 1. - ed / n < identity, independent of the device's search."""
    if n == 0:
        return -1
    keeps = lambda e: not (1. - e / n < identity)
    if not keeps(0):
        return -1
    lo, hi = 0, n
    while lo < hi:
        mid = (lo + hi + 1) // 2
        if keeps(mid):
            lo = mid
        else:
            hi = mid - 1
    return lo


def cuts(lens, first, last, chunk):
    """Reads [first, last) cut after each read where the running bases reach `chunk`
    (the reference's batch rule, construct.cc:354-359)."""
    out, bases = [first], 0
    for r in range(first, last):
        bases += int(lens[r])
        if r + 1 != last and bases < chunk:
            continue
        bases = 0
        out.append(r + 1)
    if out[-1] != last:
        out.append(last)
    return out


class Restatement:
    """rvn_find_overlaps_and_repetitive_regions flush by flush on the CPU. Distances are
    computed once per clipped overlap (ed, longest side) and shared by every identity."""

    def __init__(self, oracle):
        self.o = oracle
        self.dist = {}

    def distance(self, up, pos, c):
        key = tuple(int(x) for x in c)
        if key not in self.dist:
            li, lb, le, ri, rb, re_, _, strand = key
            a = up.ascii(pos[li])[lb:le]
            b = np.asarray(up.codes(pos[ri])[rb:re_], np.uint8)
            if not strand:
                b = _rc(b)
            b = np.frombuffer(b"ACGT", np.uint8)[b].tobytes()
            self.dist[key] = (self.o.edit_distance(a, b), max(le - lb, re_ - rb))
        return self.dist[key]

    def run(self, es, k, w, freq, identity, batch_bases=0, flush_bases=0):
        """What the call returns over the valid reads (overlaps, ovl_off, kmers, touched,
        num_mapped), and per flush: its batch, reads, mapped, kept and clipped-away
        counts, and the Myers tiers its pairs reach (TIER_PHASES)."""
        O = self.o
        ids = es.upload_ids(False)
        up = es.rs.subset(ids)
        n, lens = up.n, up.lens
        pos = {int(i): p for p, i in enumerate(ids)}
        reg = es.region()
        reads = O.reads(up)
        kmers = [np.zeros(0, bool) for _ in range(n)]
        rows, ovl_off, flushes, mapped = [], [0] * (n + 1), [], 0
        batches = cuts(lens, 0, n, batch_bases or (1 << 30))
        for bi in range(len(batches) - 1):
            j, i1 = batches[bi], batches[bi + 1]
            for r in range(j, i1):
                ovl_off[r + 1] = len(rows)
            eng = O.engine(k, w)
            O.minimize(eng, reads, j, i1, False)
            O.filter(eng, freq)
            fl = cuts(lens, 0, i1, flush_bases or (1 << 30))
            for fi in range(len(fl) - 1):
                r0, r1 = fl[fi], fl[fi + 1]
                m = O.map(eng, reads, r0, r1, True, True, False)
                filt, foff = m["filtered"], m["filt_off"]
                if filt.size:
                    ri = np.repeat(np.arange(r0, r1, dtype=np.uint32),
                                   np.diff(foff).astype(np.int64))
                    keep = O.kmer_complexity(reads, ri, filt, k)
                    for r in range(r0, r1):
                        a, b = int(foff[r - r0]), int(foff[r - r0 + 1])
                        if a == b:
                            continue
                        if kmers[r].size == 0:
                            kmers[r] = np.zeros((int(lens[r]) >> 4) + 1, bool)
                        kmers[r][filt[a:b][keep[a:b] == 1] >> 4] = True
                ovl = m["overlaps"].astype(np.int64)
                ovl[:, 0] = ids[ovl[:, 0]]
                ovl[:, 3] = ids[ovl[:, 3]]
                batch = [tuple(int(x) for x in o) for o in ovl]
                mapped += len(batch)
                info = dict(batch=bi, reads=(r0, r1), mapped=len(batch), clipped_away=0,
                            pairs=[], tiers=[])
                if identity != 0:
                    kept = []
                    for o in batch:
                        c = overlap_update(o, reg)
                        if c is None:
                            info["clipped_away"] += 1
                            continue
                        ed, longest = self.distance(up, pos, c)
                        lim = max(identity_bound(identity, longest), 0)
                        info["pairs"].append((c, ed, longest, lim))
                        if not (1. - ed / longest < identity):
                            kept.append(c)
                    batch = kept
                    # a pair runs tier t while it is open: beyond every earlier band and
                    # allowed past it by its limit
                    reach = [min(ed, lim) for _, ed, _, lim in info["pairs"]]
                    info["tiers"] = [TIER_PHASES[t] for t in range(5)
                                     if any(x > (TIER_K[t - 1] if t else -1) for x in reach)]
                info["kept"] = len(batch)
                flushes.append(info)
                rows += batch
            ovl_off[i1] = len(rows)
        touched = np.array([x.size > 0 for x in kmers], bool)
        return dict(overlaps=np.array(rows, np.uint32).reshape(-1, 8),
                    ovl_off=np.array(ovl_off, np.uint64), kmers=kmers, touched=touched,
                    num_mapped=mapped, flushes=flushes, batches=len(batches) - 1)


def boundary_identity(restate, es, tier, k=15, w=5):
    """An overlap whose clipped distance lands in `tier` and the identity equal to its
    score, 1 - ed / longest (the largest identity that keeps it)."""
    lo, hi = ((0,) + TIER_K)[tier], (TIER_K + (1 << 30,))[tier]
    r = restate.run(es, k, w, 0.001, 1e-9)
    for f in r["flushes"]:
        for c, ed, n, _ in f["pairs"]:
            if lo < ed <= hi or (tier == 0 and ed == 0):
                return c, 1. - ed / n
    raise AssertionError(f"no overlap in tier {tier}")
