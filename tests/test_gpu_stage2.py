"""GPU: stage 2 as one device call (rvn_find_overlaps_and_repetitive_regions) against the
reference's own raven::FindOverlapsAndRepetetiveRegions over the ram::MinimizerEngine
facade (oracle/_ref/stage2_call_test): the fast route's end state (every overlap list,
every pile's cereal JSON, kmers_ and its emptiness included) must be the reference's, and
so must the Python call's results once the reference's classification loop has run over
them. Forced smaller batches (option stage2_batch_bases) are checked against the same
schedule built from the single-step entry points (minimize, filter, map, kmer_complexity,
edit_distance_batch)."""
import json
import os
import struct
import subprocess

import numpy as np
import pytest

from raven_b200 import engine, seqio, synth

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
BIN = os.path.join(os.path.dirname(HERE), "oracle", "_ref", "stage2_call_test")
FREQ = 0.001


def write_vec(f, a):
    f.write(struct.pack("<Q", a.size))
    f.write(np.ascontiguousarray(a).tobytes())


def read_vec(f, dt):
    (n,) = struct.unpack("<Q", f.read(8))
    return np.frombuffer(f.read(n * np.dtype(dt).itemsize), dtype=dt).copy()


def run_driver(tmp_path, rs, k, w, identity, all_valid=False):
    if not os.path.exists(BIN):
        pytest.skip("oracle/_ref/stage2_call_test not built (needs the reference tree)")
    inp, out = str(tmp_path / "reads.bin"), str(tmp_path / "out.bin")
    with open(inp, "wb") as f:
        write_vec(f, rs.words.astype(np.uint64))
        write_vec(f, rs.word_off.astype(np.uint64))
        write_vec(f, rs.lens.astype(np.uint32))
    subprocess.run([BIN, inp, out, str(k), str(w), str(FREQ), str(identity),
                    str(int(all_valid))], check=True, stderr=subprocess.DEVNULL, timeout=900)
    res = []
    with open(out, "rb") as f:
        for _ in range(2):
            d = dict(valid=read_vec(f, np.uint32), s=int(read_vec(f, np.uint32)[0]),
                     region=read_vec(f, np.uint32).reshape(-1, 2),
                     overlaps=read_vec(f, np.uint32).reshape(-1, 8),
                     off=read_vec(f, np.uint64))
            d["piles"] = json.loads(read_vec(f, np.uint8).tobytes().decode())
            res.append(d)
    return res


def subset(rs, ids):
    return seqio.pack_codes([rs.codes(int(i)) for i in ids])


# ---- the reference's host logic around the call, restated for the check ----
def overlap_update(o, reg, invalid=frozenset()):
    """raven::OverlapUpdate (overlap_utils.cc:14-60); reg[id] = (begin, end) in bases."""
    li, lb, le, ri, rb, re_, score, strand = (int(x) for x in o)
    if li in invalid or ri in invalid:
        return None
    (pb, pe), (qb, qe) = reg[li], reg[ri]
    if lb >= pe or le <= pb or rb >= qe or re_ <= qb:
        return None
    rbc, rec = (qb - rb if rb < qb else 0), (re_ - qe if re_ > qe else 0)
    lbc, lec = (pb - lb if lb < pb else 0), (le - pe if le > pe else 0)
    nlb = lb + (rbc if strand else rec)
    nle = le - (rec if strand else rbc)
    nrb = rb + (lbc if strand else lec)
    nre = re_ - (lec if strand else lbc)
    if nlb >= pe or nle <= pb or nrb >= qe or nre <= qb:
        return None
    nlb, nle, nrb, nre = max(nlb, pb), min(nle, pe), max(nrb, qb), min(nre, qe)
    if nlb >= nle or nle - nlb < 84 or nrb >= nre or nre - nrb < 84:
        return None
    return (li, nlb, nle, ri, nrb, nre, score, strand)


def overlap_type(o, reg):
    """raven::GetOverlapType (overlap_utils.cc:62-95)."""
    li, lb, le, ri, rb, re_, _, strand = o
    (pb, pe), (qb, qe) = reg[li], reg[ri]
    ll, lb, le = pe - pb, lb - pb, le - pb
    rl = qe - qb
    rb, re_ = (rb - qb, re_ - qb) if strand else (rl - (re_ - qb), rl - (rb - qb))
    over = min(lb, rb) + min(ll - le, rl - re_)
    if le - lb < (le - lb + over) * 0.875 or re_ - rb < (re_ - rb + over) * 0.875:
        return 0
    if lb <= rb and ll - le <= rl - re_:
        return 1
    if rb <= lb and rl - re_ <= ll - le:
        return 2
    return 3 if lb > rb else 4


def classify(rows, reg):
    """construct.cc:430-469 over the call's overlaps: the final overlaps.back() and the
    reads marked contained."""
    out, contained = [], set()
    for o in rows:
        o = overlap_update(o, reg)
        if o is None:
            continue
        t = overlap_type(o, reg)
        if t == 1:
            contained.add(o[0])
        elif t == 2:
            contained.add(o[3])
        elif t >= 3:
            if out and out[-1][0] == o[0] and out[-1][3] == o[3]:
                if max(out[-1][2] - out[-1][1], out[-1][5] - out[-1][4]) < \
                        max(o[2] - o[1], o[5] - o[4]):
                    out[-1] = o
            else:
                out.append(o)
    final = [x for x in (overlap_update(o, reg, frozenset(contained)) for o in out) if x]
    return np.array(final, dtype=np.uint32).reshape(-1, 8), contained


def run_call(rs, ref, k, w, identity, batch_bases=0):
    eng = engine.Engine(device=0)
    eng.configure(k=k, w=w)
    eng.set_option("stage2_batch_bases", batch_bases)
    valid = ref["valid"]
    eng.upload(subset(rs, valid), ids=valid)
    return eng, eng.find_overlaps_and_repetitive_regions(FREQ, identity, ref["s"],
                                                         ref["region"][:, 0], ref["region"][:, 1])


def check_against_reference(rs, k, w, identity, tmp_path, all_valid=False):
    ref, fast = run_driver(tmp_path, rs, k, w, identity, all_valid)
    # the fast route's end state is the reference's, field by field
    for key in ("valid", "region", "overlaps", "off"):
        assert np.array_equal(ref[key], fast[key]), key
    assert ref["s"] == fast["s"]
    assert ref["piles"] == fast["piles"]
    # the Python call, with the reference's classification loop over its results
    _, got = run_call(rs, ref, k, w, identity)
    reg = {int(i): (int(b), int(e)) for i, (b, e) in zip(ref["valid"], ref["region"])}
    final, contained = classify(got["overlaps"], reg)
    want = ref["overlaps"][int(ref["off"][-2]):int(ref["off"][-1])]
    assert np.array_equal(final, want)
    piles = ref["piles"]
    for i, rid in enumerate(ref["valid"]):
        p = piles[str(int(rid))]
        kmers = np.array(p["kmers_"], dtype=bool)
        if got["touched"][i]:
            assert np.array_equal(kmers, got["kmers"][i]), int(rid)
        else:
            assert kmers.size == 0, int(rid)
        assert bool(p["is_contained_"]) == (int(rid) in contained), int(rid)
    return ref, got


@pytest.fixture(scope="module")
def repeat_reads():
    g = synth.repeat_genome(150_000, families=4, copies=8, seed=5)
    return synth.make_reads(genome=g, n_reads=240, mean_len=6000, seed=6, sub=0.01, ins=0.005,
                            dele=0.005)


@pytest.mark.parametrize("identity", [0.0, 0.9, 0.95])
def test_stage2_call_lambda_equals_reference(tmp_path, lambda_reads, identity):
    ref, got = check_against_reference(lambda_reads, 15, 5, identity, tmp_path)
    assert 0 < ref["s"] < lambda_reads.n
    if identity == 0:
        assert got["overlaps"].shape[0] == got["num_mapped"] > 0


@pytest.mark.parametrize("k,w", [(15, 5), (19, 10)])
@pytest.mark.parametrize("identity", [0.0, 0.9, 0.95])
def test_stage2_call_repeats_equals_reference(tmp_path, repeat_reads, k, w, identity):
    ref, got = check_against_reference(repeat_reads, k, w, identity, tmp_path)
    assert 0 < ref["s"] < repeat_reads.n
    ovl = got["overlaps"]
    assert ovl.shape[0] > 0 and set(ovl[:, 7].tolist()) == {0, 1}  # both strands
    assert got["touched"].any()
    if k == 15:
        # a read whose filtered k-mers all fail the complexity test: touched, all zero
        assert any(t and not m.any() for t, m in zip(got["touched"], got["kmers"]))
    if identity != 0:
        assert 0 < ovl.shape[0] < got["num_mapped"]


def test_stage2_call_no_invalid_read_maps_nothing(tmp_path, repeat_reads):
    """construct.cc:343-349: s stays 0 when no pile is invalid, and nothing is mapped."""
    ref, got = check_against_reference(repeat_reads, 15, 5, 0.9, tmp_path, all_valid=True)
    assert ref["s"] == 0 and ref["valid"].size == 0
    assert got["overlaps"].shape[0] == 0 and got["num_mapped"] == 0


def schedule_from_primitives(eng, rs, ref, k, identity, cut):
    """The reference's schedule at batch cut `cut`, built from the single-step calls."""
    s, lens = ref["s"], rs.lens
    reg = {int(i): (int(b), int(e)) for i, (b, e) in zip(ref["valid"], ref["region"])}
    pos = {int(i): n for n, i in enumerate(ref["valid"])}
    kmers = [np.zeros(0, bool) for _ in range(s)]
    rows, ends, clipped_away, nbytes, j = [], [], 0, 0, 0
    for i in range(s):
        nbytes += int(lens[int(ref["valid"][i])])
        if i != s - 1 and nbytes < cut:
            continue
        nbytes = 0
        eng.minimize(j, i + 1)
        eng.filter(FREQ)
        m = eng.map(0, i + 1, True, True, False, True)
        filt, foff = m["filtered"], m["filt_off"]
        reads = np.repeat(np.arange(i + 1, dtype=np.uint32), np.diff(foff).astype(np.int64))
        keep = eng.kmer_complexity(reads, filt, k) if filt.size else np.zeros(0, np.uint8)
        for r in range(i + 1):
            a, b = int(foff[r]), int(foff[r + 1])
            if a == b:
                continue
            if kmers[r].size == 0:
                kmers[r] = np.zeros((int(lens[int(ref["valid"][r])]) >> 4) + 1, bool)
            kmers[r][filt[a:b][keep[a:b] == 1] >> 4] = True
        batch = [tuple(int(x) for x in o) for o in m["overlaps"]]
        if identity != 0:
            upd = [overlap_update(o, reg) for o in batch]
            clipped_away += sum(u is None for u in upd)
            upd = [u for u in upd if u]
            if upd:
                a = np.array(upd, dtype=np.int64)
                dist = eng.edit_distance_batch([pos[x] for x in a[:, 0]], a[:, 1], a[:, 2] - a[:, 1],
                                               [pos[x] for x in a[:, 3]], a[:, 4], a[:, 5] - a[:, 4],
                                               a[:, 7])
                longest = np.maximum(a[:, 2] - a[:, 1], a[:, 5] - a[:, 4])
                ok = [d >= 0 and not (1. - d / n < identity) for d, n in zip(dist, longest)]
                batch = [u for u, x in zip(upd, ok) if x]
            else:
                batch = []
        rows += batch
        ends.append((i, len(rows)))
        j = i + 1
    return np.array(rows, dtype=np.uint32).reshape(-1, 8), ends, kmers, clipped_away


@pytest.mark.parametrize("identity", [0.0, 0.9])
def test_stage2_call_forced_batches(tmp_path, repeat_reads, identity):
    ref, _ = run_driver(tmp_path, repeat_reads, 15, 5, identity)
    cut = int(repeat_reads.lens.astype(np.int64).sum()) // 5
    eng, got = run_call(repeat_reads, ref, 15, 5, identity, batch_bases=cut)
    want, ends, kmers, clipped_away = schedule_from_primitives(eng, repeat_reads, ref, 15,
                                                               identity, cut)
    assert len(ends) >= 3
    assert np.array_equal(got["overlaps"], want)
    want_off, cur, end_at = [0], 0, dict(ends)
    for i in range(ref["s"]):
        cur = end_at.get(i, cur)
        want_off.append(cur)
    assert np.array_equal(got["ovl_off"], np.array(want_off, dtype=np.uint64))
    for i in range(ref["s"]):
        assert bool(got["touched"][i]) == (kmers[i].size > 0)
        if kmers[i].size:
            assert np.array_equal(got["kmers"][i], kmers[i]), i
    if identity != 0:
        assert clipped_away > 0  # overlaps clipped to nothing at a region edge
