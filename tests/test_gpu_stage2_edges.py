"""GPU: rvn_find_overlaps_and_repetitive_regions at its edges, bit for bit against the CPU
restatement of stage2_edges.py (overlaps, ovl_off, kmers, touched, num_mapped) and, for
whole-bin regions in one batch, against the reference's own stage 2 (ReferenceStage2.stage2:
final overlaps after the classification loop, kmers_, containment). Every case first
asserts the edge it was built for: valid regions that leave a side of 83, 84 or 85 bases
or the 1260-base minimum, identities exactly on an overlap's score and the next double
above it, the Myers tiers (64, 192, 448, 960, unbanded) that run with a limit inside the
call and the ones a pair's limit stops, several flushes per batch and flushes that map
nothing, batches whose overlaps are all clipped away, chunked index builds, other k and
w, frequencies 0, 0.001 and 0.3, and invalid reads uploaded after the valid ones."""
import numpy as np
import pytest

import stage2_edges as E
from raven_b200 import engine
from test_gpu_stage2 import classify

pytestmark = pytest.mark.gpu

@pytest.fixture(scope="module")
def ref_stage2():
    import oracle_lib
    if not oracle_lib.ReferenceStage2.available():
        pytest.skip("oracle/_ref/libraven_ref_stage2.so not built (needs the reference tree)")
    return oracle_lib.ReferenceStage2()


@pytest.fixture(scope="module")
def restate(oracle):
    return E.Restatement(oracle)


@pytest.fixture(scope="module")
def any_regions(oracle):
    return E.with_regions(E.edge_reads(), oracle, aligned=False)


@pytest.fixture(scope="module")
def aligned(oracle):
    return E.with_regions(E.edge_reads(), oracle, aligned=True)


def run_device(es, k, w, freq, identity, batch=0, flush=0, chunk=-1, with_invalid=False):
    eng = engine.Engine(device=0)
    eng.configure(k=k, w=w)
    eng.set_option("stage2_batch_bases", batch)
    eng.set_option("map_flush_bases", flush)
    eng.set_option("index_chunk_bases", chunk)
    ids = es.upload_ids(with_invalid)
    eng.upload(es.rs.subset(ids), ids=ids)
    v = es.valid
    eng.set_option("reset_stats", 1)
    got = eng.find_overlaps_and_repetitive_regions(freq, identity, v.size, es.begin[v],
                                                   es.end[v])
    got["phases"] = eng.phases()
    eng.close()
    return got


def flush_tiers(phases):
    """The Myers tier phases of each stage2_filter phase (one per flush)."""
    out = []
    for name in phases:
        if name == "stage2_filter":
            out.append([])
        elif name.startswith("myers_") and out:
            out[-1].append(name)
    return out


def check(got, want, identity):
    assert np.array_equal(got["overlaps"], want["overlaps"])
    assert np.array_equal(got["ovl_off"], want["ovl_off"])
    assert got["num_mapped"] == want["num_mapped"]
    assert np.array_equal(got["touched"], want["touched"])
    for p, m in enumerate(want["kmers"]):
        if m.size:
            assert np.array_equal(got["kmers"][p], m), p
    if identity != 0:
        # one filter per flush, and each runs exactly the tiers its pairs reach
        assert flush_tiers(got["phases"]) == [f["tiers"] for f in want["flushes"]]


def check_reference(ref_stage2, es, got, k, w, freq, identity):
    ref = ref_stage2.stage2(es.rs, k, w, freq, identity, es.begin >> 4, es.end >> 4, es.invalid)
    assert ref["s"] == es.valid.size
    reg = es.region()
    final, contained = classify(got["overlaps"], reg)
    assert np.array_equal(final, ref["overlaps"])
    assert contained == set(np.flatnonzero(ref["contained"]).tolist())
    for p, rid in enumerate(es.valid):
        assert bool(got["touched"][p]) == bool(ref["touched"][rid]), int(rid)
        if ref["touched"][rid]:
            assert np.array_equal(got["kmers"][p], ref["kmers"][rid]), int(rid)


@pytest.mark.parametrize("identity", E.IDENTITIES)
@pytest.mark.parametrize("regions", ["any", "aligned"])
def test_stage2_edges_identities(request, ref_stage2, restate, regions, identity):
    es = request.getfixturevalue("any_regions" if regions == "any" else "aligned")
    want = restate.run(es, 15, 5, 0.001, identity)
    got = run_device(es, 15, 5, 0.001, identity)
    if identity == 1e-9:  # every tier runs, the unbanded kernel with a limit
        assert want["flushes"][0]["tiers"] == list(E.TIER_PHASES)
        assert all(lim >= 0 for _, _, _, lim in want["flushes"][0]["pairs"])
    if identity == 0.9:  # limits below the pairs' distances stop them before the 960 tier
        assert "myers_full" not in want["flushes"][0]["tiers"]
        assert any(ed > 960 for _, ed, _, _ in want["flushes"][0]["pairs"])
    check(got, want, identity)
    if regions == "aligned":
        check_reference(ref_stage2, es, got, 15, 5, 0.001, identity)


@pytest.mark.parametrize("tier", range(5))
def test_stage2_edges_boundary_identity(ref_stage2, restate, aligned, tier):
    """identity = 1 - ed / longest of an overlap in each tier keeps it; the next double
    towards 1 drops it. The limit and the keep test agree at the bound."""
    c, score = E.boundary_identity(restate, aligned, tier)
    for identity, kept in ((score, True), (np.nextafter(score, 1.0), False)):
        want = restate.run(aligned, 15, 5, 0.001, identity)
        got = run_device(aligned, 15, 5, 0.001, identity)
        rows = {tuple(int(x) for x in o) for o in got["overlaps"]}
        assert (tuple(c) in rows) == kept
        assert E.TIER_PHASES[tier] in flush_tiers(got["phases"])[0]
        check(got, want, identity)
        check_reference(ref_stage2, aligned, got, 15, 5, 0.001, identity)


SCHEDULES = {  # (batch bases or a fraction of the valid bases, flush bases, index chunk bases)
    "default": (0, 0, -1),
    "batch_one_read": (1, 0, -1),
    "batch_fifth": (0.2, 0, -1),
    "flushes": (0, 1500, -1),
    "chunks": (0, 0, 4000),
    "all": (0.2, 1500, 4000),
}


@pytest.mark.parametrize("identity", [0.0, 0.9])
@pytest.mark.parametrize("name", list(SCHEDULES))
def test_stage2_edges_schedules(ref_stage2, restate, any_regions, aligned, name, identity):
    # one-read batches over the narrow regions: some batch's overlaps all clipped away
    es = any_regions if name == "batch_one_read" else aligned
    bases = int(es.rs.lens[es.valid].astype(np.int64).sum())
    b, f, c = SCHEDULES[name]
    batch = int(b * bases) if isinstance(b, float) else b
    want = restate.run(es, 15, 5, 0.001, identity, batch_bases=batch, flush_bases=f)
    got = run_device(es, 15, 5, 0.001, identity, batch=batch, flush=f, chunk=c)
    fl = want["flushes"]
    if batch:
        assert want["batches"] >= 3
    if name == "batch_one_read" and identity:
        # a batch whose every mapped overlap the regions cut away
        assert any(x["mapped"] > 0 and x["clipped_away"] == x["mapped"] for x in fl)
    if f:
        per_batch = np.bincount([x["batch"] for x in fl])
        assert per_batch.max() >= 3
        assert any(x["mapped"] == 0 for x in fl)  # a flush that maps nothing
    if c > 0:  # every batch's index was built in chunks
        assert got["phases"].count("sketch_tiers") > want["batches"]
    else:
        assert "sketch_tiers" not in got["phases"]
    check(got, want, identity)
    if want["batches"] == 1:
        check_reference(ref_stage2, es, got, 15, 5, 0.001, identity)


@pytest.mark.parametrize("freq", E.FREQS)
@pytest.mark.parametrize("k,w", ((15, 5),) + E.OFF_KW)
def test_stage2_edges_kw_freq(ref_stage2, restate, aligned, k, w, freq):
    want = restate.run(aligned, k, w, freq, 0.9)
    got = run_device(aligned, k, w, freq, 0.9)
    if freq == 0:
        assert not want["touched"].any()
    else:
        assert want["touched"].any()
    if freq == 0.3:
        assert any(m.any() for m in want["kmers"])
    check(got, want, 0.9)
    check_reference(ref_stage2, aligned, got, k, w, freq, 0.9)


@pytest.mark.parametrize("identity", [0.0, 0.9])
@pytest.mark.parametrize("schedule", ["default", "all"])
def test_stage2_edges_invalid_reads_uploaded(restate, any_regions, schedule, identity):
    """n_valid below the uploaded reads: the invalid reads after the valid ones change
    nothing."""
    es = any_regions
    assert es.invalid.any()
    bases = int(es.rs.lens[es.valid].astype(np.int64).sum())
    b, f, c = SCHEDULES[schedule]
    batch = int(b * bases) if isinstance(b, float) else b
    want = restate.run(es, 15, 5, 0.3, identity, batch_bases=batch, flush_bases=f)
    got = [run_device(es, 15, 5, 0.3, identity, batch, f, c, with_invalid=x)
           for x in (False, True)]
    for g in got:
        check(g, want, identity)
