"""Seeded synthetic long reads (host side, numpy): uniform random genome,
reads drawn from both strands with substitution / insertion / deletion errors
(SURVEY.md §8d: ONT 10 % = 3/3/4, HiFi 0.5 % = 0.2/0.15/0.15)."""
from __future__ import annotations

import numpy as np

from . import seqio


def mutate(codes, rng, sub, ins, dele):
    """Apply i.i.d. errors to a uint8 code array."""
    n = len(codes)
    if n == 0 or sub + ins + dele == 0:
        return codes
    u = rng.random(n)
    keep = u >= dele
    is_sub = (u >= dele) & (u < dele + sub)
    out = codes.copy()
    out[is_sub] = (out[is_sub] + rng.integers(1, 4, is_sub.sum(), dtype=np.uint8)) & 3
    is_ins = rng.random(n) < ins
    reps = keep.astype(np.int64) + is_ins
    res = np.repeat(out, reps)
    # the inserted copy gets a random base
    pos = np.cumsum(reps) - 1
    ins_pos = pos[is_ins & (reps > 0)]
    res[ins_pos] = rng.integers(0, 4, len(ins_pos), dtype=np.uint8)
    return res


def make_reads(genome_len=100_000, n_reads=200, mean_len=5000, seed=1, sub=0.03,
               ins=0.03, dele=0.04, min_len=500, genome=None):
    rng = np.random.default_rng(seed)
    if genome is None:
        genome = rng.integers(0, 4, genome_len, dtype=np.uint8)
    genome_len = len(genome)
    seqs = []
    for _ in range(n_reads):
        ln = int(np.clip(rng.normal(mean_len, 0.2 * mean_len), min_len, 5 * mean_len))
        ln = min(ln, genome_len)
        st = int(rng.integers(0, genome_len - ln + 1))
        s = genome[st:st + ln]
        if rng.random() < 0.5:
            s = (3 - s[::-1]).astype(np.uint8)
        seqs.append(mutate(s, rng, sub, ins, dele))
    return seqio.pack_codes(seqs)


def repeat_genome(genome_len=200_000, families=4, family_len=2000, copies=8,
                  tandem_every=5000, tandem_len=120, seed=1, divergence=0.01):
    """A random genome with planted repeats: `families` interspersed families of
    `copies` near-identical copies (substitutions at `divergence`), and a short tandem
    repeat (dinucleotide, trinucleotide or homopolymer run of tandem_len bases) every
    tandem_every bases. Their minimizers are the frequent ones stage 2 filters: the
    families' k-mers pass Pile::AddKmers' complexity test, the tandem repeats' fail it."""
    rng = np.random.default_rng(seed)
    g = rng.integers(0, 4, genome_len, dtype=np.uint8)
    for _ in range(families):
        fam = rng.integers(0, 4, family_len, dtype=np.uint8)
        for _ in range(copies):
            c = fam.copy()
            hit = rng.random(family_len) < divergence
            c[hit] = (c[hit] + rng.integers(1, 4, int(hit.sum()))) % 4
            if rng.random() < 0.5:
                c = (3 - c[::-1]).astype(np.uint8)
            at = int(rng.integers(0, genome_len - family_len))
            g[at:at + family_len] = c
    for at in range(tandem_every // 2, genome_len - tandem_len, tandem_every):
        unit = rng.integers(0, 4, int(rng.integers(1, 4)), dtype=np.uint8)
        g[at:at + tandem_len] = np.resize(unit, tandem_len)
    return g


def random_reads(lengths, seed=1):
    """Unrelated random reads of given lengths (edge-case tests)."""
    rng = np.random.default_rng(seed)
    return seqio.pack_codes([rng.integers(0, 4, n, dtype=np.uint8) for n in lengths])


def make_windows(n_windows=8, backbone_len=500, layers=30, seed=1, sub=0.03, ins=0.03,
                 dele=0.04, backbone_err=0.5, partial=0.3, with_quality=True,
                 min_layers=None):
    """Synthetic racon windows in the flat layout of rvn_poa_batch.

    Every window has a hidden truth; its backbone is a lightly corrupted copy
    (a draft unitig) and its layers are read-like copies of truth segments.
    `partial` of the layers cover only part of the window (begin/end given in
    backbone coordinates, like racon's breaking points)."""
    rng = np.random.default_rng(seed)
    acgt = np.frombuffer(b"ACGT", dtype=np.uint8)
    win_first, seq_off, begins, ends = [0], [0], [], []
    bases, quals, truths = [], [], []
    for _ in range(n_windows):
        truth = rng.integers(0, 4, backbone_len, dtype=np.uint8)
        truths.append(acgt[truth].tobytes())
        bb = mutate(truth, rng, sub * backbone_err, ins * backbone_err, dele * backbone_err)
        seqs = [bb]
        pos = [(0, 0)]
        nl = layers if min_layers is None else int(rng.integers(min_layers, layers + 1))
        for _ in range(nl):
            if rng.random() < partial:
                a = int(rng.integers(0, backbone_len - 40))
                b = int(rng.integers(a + 20, backbone_len))
            else:
                a, b = 0, backbone_len - 1
            seg = mutate(truth[a:b + 1], rng, sub, ins, dele)
            if len(seg) == 0:
                continue
            # backbone coordinates of the segment ends (proportional map)
            ba = min(len(bb) - 2, int(round(a * len(bb) / backbone_len)))
            be = min(len(bb) - 1, max(ba + 1, int(round(b * len(bb) / backbone_len))))
            seqs.append(seg)
            pos.append((ba, be))
        for s, (a, b) in zip(seqs, pos):
            bases.append(acgt[s])
            q = np.full(len(s), 33, np.uint8) if s is seqs[0] else \
                (33 + rng.integers(5, 30, 1 + len(s) // 64).repeat(64)[:len(s)]).astype(np.uint8)
            quals.append(q)
            seq_off.append(seq_off[-1] + len(s))
            begins.append(a)
            ends.append(b)
        win_first.append(win_first[-1] + len(seqs))
    return dict(win_first=np.array(win_first, np.uint32), seq_off=np.array(seq_off, np.uint64),
                bases=np.concatenate(bases), quals=np.concatenate(quals) if with_quality else None,
                seq_begin=np.array(begins, np.uint32), seq_end=np.array(ends, np.uint32),
                truths=truths)
