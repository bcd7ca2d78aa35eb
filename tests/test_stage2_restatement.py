"""CPU: the stage-2 restatement of stage2_edges.py against the reference's own
raven::FindOverlapsAndRepetetiveRegions (ReferenceStage2.stage2) over the same read sets and
whole-bin valid regions: the final overlaps once the reference's classification loop has
run over the restated ones, every pile's kmers_ and whether it was resized, and the
contained reads. This pins the restatement the GPU edge tests compare the device with,
the identities that sit exactly on an overlap's score included."""
import numpy as np
import pytest

import stage2_edges as E
from test_gpu_stage2 import classify, overlap_update

@pytest.fixture(scope="module")
def ref_stage2():
    import oracle_lib
    if not oracle_lib.ReferenceStage2.available():
        pytest.skip("oracle/_ref/libraven_ref_stage2.so not built (needs the reference tree)")
    return oracle_lib.ReferenceStage2()


@pytest.fixture(scope="module")
def aligned(oracle):
    return E.with_regions(E.edge_reads(), oracle, aligned=True)


@pytest.fixture(scope="module")
def restate(oracle):
    return E.Restatement(oracle)


def check_reference(ref_stage2, es, want, k, w, freq, identity):
    """want (the restatement or the device call) against ReferenceStage2.stage2."""
    ref = ref_stage2.stage2(es.rs, k, w, freq, identity, es.begin >> 4, es.end >> 4, es.invalid)
    assert np.array_equal(ref["valid"], es.valid) and ref["s"] == es.valid.size
    reg = {i: (b << 4, e << 4) for i, (b, e) in
           enumerate(zip((es.begin >> 4).tolist(), (es.end >> 4).tolist()))}
    final, contained = classify(want["overlaps"], reg)
    assert np.array_equal(final, ref["overlaps"])
    assert contained == set(np.flatnonzero(ref["contained"]).tolist())
    for p, rid in enumerate(es.valid):
        assert bool(want["touched"][p]) == bool(ref["touched"][rid]), int(rid)
        if want["touched"][p]:
            assert np.array_equal(want["kmers"][p], ref["kmers"][rid]), int(rid)
    assert not ref["touched"][es.invalid].any()
    return ref


# every identity at raven's k and w, 0 and 0.9 off them
CASES = [(15, 5, f, i) for f in E.FREQS for i in E.IDENTITIES] + \
        [(k, w, f, i) for k, w in E.OFF_KW for f in E.FREQS for i in (0.0, 0.9)]


@pytest.mark.parametrize("k,w,freq,identity", CASES)
def test_restatement_equals_reference(ref_stage2, restate, aligned, k, w, freq, identity):
    want = restate.run(aligned, k, w, freq, identity)
    check_reference(ref_stage2, aligned, want, k, w, freq, identity)
    if freq == 0:
        assert not want["touched"].any()
    if freq == 0.3:
        assert any(m.any() for m in want["kmers"])
    if freq and k == 15:  # homopolymer and dinucleotide reads: touched, every k-mer fails
        for p, rid in enumerate(aligned.valid):
            if aligned.kinds[rid] in ("homopolymer", "dinucleotide"):
                assert want["touched"][p] and not want["kmers"][p].any()


@pytest.mark.parametrize("tier", range(5))
def test_restatement_boundary_identity_equals_reference(ref_stage2, restate, aligned, tier):
    c, score = E.boundary_identity(restate, aligned, tier)
    for identity, kept in ((score, True), (np.nextafter(score, 1.0), False)):
        want = restate.run(aligned, 15, 5, 0.001, identity)
        rows = {tuple(int(x) for x in o) for o in want["overlaps"]}
        assert (tuple(c) in rows) == kept
        check_reference(ref_stage2, aligned, want, 15, 5, 0.001, identity)


def test_regions_reach_their_edges(oracle, aligned):
    """The sets carry what the cases below rely on: clipped sides of exactly 84 and 85
    bases, a side one base short of 84, the 1260-base minimum, whole-bin regions."""
    es = E.with_regions(E.edge_reads(), oracle, aligned=False)
    reg = es.region()
    sides = set()
    short = False
    for o in E.stage2_overlaps(es, oracle, 15, 5):
        o = tuple(int(x) for x in o)
        c = overlap_update(o, reg)
        if c is not None:
            sides.add(min(c[2] - c[1], c[5] - c[4]))
            continue
        wide = dict(reg)
        b, e = reg[o[0]]
        wide[o[0]] = (b - 1, e) if b else (b, e)
        short = short or overlap_update(o, wide) is not None
    assert {84, 85} <= sides and short
    assert E.MIN_REGION in (es.end - es.begin).tolist()
    assert not (aligned.begin % 16).any() and not (aligned.end % 16).any()
    assert ((aligned.end - aligned.begin) == E.MIN_REGION >> 4 << 4).any()
