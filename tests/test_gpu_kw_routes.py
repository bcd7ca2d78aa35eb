"""raven -k / -w off the default (15, 5): every sketch, index, map and chain route that
k and w select, bit-exact against the CPU oracle (and the oracle against a naive
minimizer definition and the reference's own construct.cc).

k and w pick kernels, value widths and index layouts, not only constants:
  sketch   k <= 15 and w == 5: SketchFastKernel; k <= 15: SketchKernel<u32>; k >= 16:
           SketchKernel<u64> (also at w == 5); the generic kernels' halo is w - 1
  capacity 2.2 / (w + 1) of the k-mer positions, an exact-size retry when denser
  micro     len / k micromizers; the on-chip stage holds 40 KB of values (10240 u32,
           5120 u64), longer sketches are selected from global memory
  build    k <= 15 with w == 5 sketches straight into the tiers (fused) or appends
           chunks untiered (append); everything else sorts a full sketch (impl)
  tiers    u32 values only (k <= 15)
  bare     bucket partition and group-low split only for 2k > 20; slot_bits =
           max(0, min(15, span_bits - log2(cluster))); hist_shift = max(0, 2k - 10)
  probe    2^16 or more suffix-probe queries are sorted over 2k bits (u32 / u64 keys)
`routes()` restates that arithmetic; the unmarked test checks that the matrix below
takes every route on both sides."""
import numpy as np
import pytest

from raven_b200 import seqio, synth

TILE = 2048
MICRO_STAGE_BYTES = 40 << 10
BARE_BUCKET_BITS, BARE_SLOT_BITS, GROUP_LOW_BITS, CAP_BITS = 10, 15, 10, 10
SORTED_PROBE_MIN = 1 << 16
TIER_MIN_DEFAULT = 1 << 18
HIT_BOUND = 50_000_000     # hits of one map or stage-1 call
HIT_BUDGET = 20_000_000    # predicted hits the frequency is chosen for
KEYS = ("overlaps", "ovl_off", "pile", "pile_off")
HIFI = dict(sub=0.004, ins=0.003, dele=0.003)   # long k and w find overlaps of these

POINTS = [(1, 3), (2, 2), (4, 5), (8, 8), (10, 12), (15, 4), (15, 6), (16, 5), (17, 33),
          (19, 10), (24, 64), (28, 128), (31, 255), (15, 256)]
IDS = [f"k{k}w{w}" for k, w in POINTS]


def routes(k, w, n_records=0, n_queries=0, tier_min=TIER_MIN_DEFAULT, bare_count=1,
           chunked=False, cluster=8):
    """The route every (k, w) takes, for an index batch of n_records records and a map
    call of n_queries suffix-probe queries (sketch.cu, index.cu, map.cu)."""
    k = min(max(k, 1), 31)
    key_bits = 2 * k
    is32 = key_bits <= 30
    fast = is32 and w == 5
    tiered = is32 and n_records >= tier_min
    bare = tiered and bare_count != 0
    partition = bare and key_bits > 2 * BARE_BUCKET_BITS
    span_bits = key_bits - BARE_BUCKET_BITS if partition else key_bits
    log_c = (cluster - 1).bit_length()
    return dict(
        kernel="fast" if fast else ("generic32" if is32 else "generic64"),
        width=32 if is32 else 64,
        halo=w - 1,
        build=("fused" if tiered else "append") if chunked and fast else "impl",
        tiered=tiered,
        partition=partition,
        group_low=tiered and not bare and key_bits > 2 * GROUP_LOW_BITS,
        slot_bits=max(0, min(BARE_SLOT_BITS, span_bits - log_c)) if bare else None,
        hist_shift=max(0, key_bits - CAP_BITS),
        sorted_probe=("u32" if is32 else "u64") if n_queries >= SORTED_PROBE_MIN else None,
        stage_cap=MICRO_STAGE_BYTES // (4 if is32 else 8),
    )


# what each point is in the matrix for: (kernel, tiered bare-count slot_bits)
INTENDED = {
    (1, 3): ("generic32", 0),        # slot table of 0 bits, 2 canonical keys
    (2, 2): ("generic32", 1),        # palindromic k-mers, the narrowest window
    (4, 5): ("fast", 5),             # the fast kernel at tiny k
    (8, 8): ("generic32", 13),
    (10, 12): ("generic32", 15),     # 2k = 20: no bucket partition, no group-low split
    (15, 4): ("generic32", 15),      # w = 4 and w = 6 beside the fast kernel's w = 5
    (15, 6): ("generic32", 15),
    (16, 5): ("generic64", None),    # the first u64 k, at w = 5
    (17, 33): ("generic64", None),   # halo 32: wider than a warp
    (19, 10): ("generic64", None),
    (24, 64): ("generic64", None),
    (28, 128): ("generic64", None),
    (31, 255): ("generic64", None),  # 2k = 62, halo 255
    (15, 256): ("generic32", 15),    # the largest window
}


def test_route_table_covers_both_sides():
    assert set(INTENDED) == set(POINTS)
    seen = {}
    for k, w in POINTS:
        kernel, slot = INTENDED[(k, w)]
        r = routes(k, w, n_records=1, tier_min=0)
        assert r["kernel"] == kernel, (k, w)
        assert r["slot_bits"] == slot, (k, w)
        assert r["tiered"] == (r["width"] == 32), (k, w)
        assert r["partition"] == (r["tiered"] and 2 * k > 20), (k, w)
        variants = [r, routes(k, w, n_records=1), routes(k, w, 1, tier_min=0, bare_count=0),
                    routes(k, w, 1, tier_min=0, chunked=True), routes(k, w, 1, chunked=True),
                    routes(k, w, n_queries=SORTED_PROBE_MIN),
                    routes(k, w, n_queries=SORTED_PROBE_MIN - 1)]
        for v in variants:
            for name, val in v.items():
                seen.setdefault(name, set()).add(val)
    assert seen["kernel"] == {"fast", "generic32", "generic64"}
    assert seen["build"] == {"fused", "append", "impl"}
    for flag in ("tiered", "partition", "group_low"):
        assert seen[flag] == {False, True}, flag
    assert {0, 1, 15, None} <= seen["slot_bits"]
    assert 0 in seen["hist_shift"] and max(seen["hist_shift"]) == 52
    assert seen["sorted_probe"] == {None, "u32", "u64"}
    assert seen["stage_cap"] == {10240, 5120}
    assert {1, 32, 255} <= seen["halo"]   # the narrowest, just past a warp, the widest
    # the edges themselves
    assert routes(15, 5)["kernel"] == "fast" and routes(16, 5)["kernel"] == "generic64"
    assert not routes(10, 12, 1, tier_min=0)["partition"]
    assert routes(11, 12, 1, tier_min=0)["partition"]
    assert routes(5, 3)["hist_shift"] == 0 and routes(6, 3)["hist_shift"] == 2
    assert routes(0, 3) == routes(1, 3) and routes(40, 7) == routes(31, 7)


# ---- read sets ----

def _rng(k, w, salt):
    return np.random.default_rng(100_000 * salt + 1000 * k + w)


def at_rich(rng, n_reads, length, gc=0.005):
    """Reads over A/T with rare C/G: at k <= 4 the A/T keys are few and dense (the
    frequency filter removes them), the C/G keys sparse."""
    seqs = []
    for _ in range(n_reads):
        s = rng.choice(np.array([0, 3], np.uint8), length)
        m = rng.random(length) < gc
        s[m] = rng.choice(np.array([1, 2], np.uint8), int(m.sum()))
        seqs.append(s)
    return seqs


def sketch_reads(k, w):
    """Lengths k+w-2 / k+w-1, reads whose end falls on either side of a tile edge and
    of its halo, dense repeats beyond the capacity estimate and the on-chip micromize
    stage, a long random read."""
    rng = _rng(k, w, 1)
    h = w - 1
    lens = [1, k + w - 2, k + w - 1, k + w, k + w + 1]
    for q in (TILE - h - 1, TILE - h, TILE - 1, TILE, TILE + 1, TILE + h, TILE + h + 1,
              2 * TILE + h, 3 * TILE - h):
        lens.append(max(q, 1) + k - 1)
    seqs = [rng.integers(0, 4, n, dtype=np.uint8) for n in lens]
    for n in (3 * TILE + k + 7, 24_000):
        seqs.append(np.zeros(n, np.uint8))                        # poly-A
        seqs.append(np.tile(np.array([0, 1], np.uint8), n // 2))  # (AC)n
    seqs.append(np.tile(np.array([0, 3], np.uint8), 400))         # (AT)n: palindromes
    seqs.append(rng.integers(0, 4, 40_000, dtype=np.uint8))
    return seqio.pack_codes(seqs)


def naive_reads(k, w):
    rng = _rng(k, w, 2)
    seqs = [rng.integers(0, 4, n, dtype=np.uint8) for n in (k + w - 2, k + w - 1, k + w, 300)]
    seqs.append(np.zeros(k + w + 40, np.uint8))
    seqs.append(np.tile(np.array([0, 3], np.uint8), (k + w + 40) // 2))
    return seqio.pack_codes(seqs)


def overlap_reads(k, w, bases, seed):
    """Overlapping reads of about `bases` bases (A/T-rich unrelated ones for k <= 4)."""
    rng = _rng(k, w, seed)
    if k <= 4:
        return seqio.pack_codes(at_rich(rng, max(1, bases // 1600), 1600))
    n = max(4, bases // 3000)
    return synth.make_reads(max(20_000, bases // 8), n, 3000, seed=int(rng.integers(1 << 30)),
                            **HIFI)


def large_query_bases(k, w):
    """bases whose full sketch holds 2^16 queries or more (the A/T-rich reads of k <= 4
    are sparser: palindromes and long runs of one key)"""
    return int((2.6 if k <= 4 else 1.3) * SORTED_PROBE_MIN * max(1.0, (w + 1) / 2))


# ---- oracle anchors (CPU) ----

@pytest.mark.parametrize("kw", POINTS, ids=IDS)
def test_oracle_sketch_matches_naive_definition(oracle, kw):
    from test_oracle import _numpy_minimizers
    k, w = kw
    rs = naive_reads(k, w)
    eng = oracle.engine(k, w)
    sk = oracle.sketch(eng, oracle.reads(rs), 0, rs.n, False)
    for i in range(rs.n):
        codes = rs.codes(i)
        a, b = int(sk["offsets"][i]), int(sk["offsets"][i + 1])
        got = list(zip(sk["value"][a:b].tolist(), (sk["origin"][a:b] & 0xFFFFFFFF).tolist()))
        assert got == _numpy_minimizers(codes, k, w), (k, w, i)
        assert ((sk["origin"][a:b] >> 32) == i).all()


STAGE1_REF_POINTS = [(8, 8), (15, 6), (16, 5), (17, 33), (31, 255)]


@pytest.mark.parametrize("kw", STAGE1_REF_POINTS, ids=[f"k{k}w{w}" for k, w in STAGE1_REF_POINTS])
def test_oracle_stage1_equals_reference(oracle, reference, kw):
    k, w = kw
    rs = synth.make_reads(40_000, 120, 3000, seed=11 + k, **HIFI)
    for minhash in (False, True):
        a = oracle.stage1(oracle.engine(k, w, threads=4), oracle.reads(rs), 0.001, 16, minhash)
        b = reference.stage1(reference.reads(rs), k, w, 0.001, 16, minhash, 4)
        for key in KEYS + ("occurrences",):
            assert np.array_equal(a[key], b[key]), (k, w, minhash, key)
        assert a["overlaps"].shape[0] > 0


# ---- GPU against the oracle ----

def choose_freq(oracle, eng, candidates=(0.0, 0.0005, 0.002, 0.01, 0.05, 0.2, 0.6, 1.0)):
    """The least filtering frequency whose kept keys give at most HIT_BUDGET hits in a
    self-map (sum of squared counts; the oracle engine holds the index)."""
    counts = oracle.keys(eng)["counts"].astype(np.int64)
    for f in candidates:
        occ = oracle.filter(eng, f)
        if int((counts[counts <= occ] ** 2).sum()) <= HIT_BUDGET:
            return f
    raise AssertionError("no frequency keeps the hits bounded")


def sketch_equal(got, want, tag):
    for key in ("offsets", "value", "origin"):
        assert np.array_equal(got[key], want[key]), (tag, key)


@pytest.mark.gpu
@pytest.mark.parametrize("kw", POINTS, ids=IDS)
def test_sketch_routes(oracle, kw):
    from raven_b200 import engine
    k, w = kw
    rs = sketch_reads(k, w)
    eng = engine.Engine(device=0)   # fresh buffers: the capacity estimate is what counts
    try:
        eng.configure(k=k, w=w)
        eng.upload(rs)
        oeng, reads = oracle.engine(k, w), oracle.reads(rs)
        full = eng.sketch(0, rs.n, False)
        sketch_equal(full, oracle.sketch(oeng, reads, 0, rs.n, False), (k, w, "full"))
        sketch_equal(eng.sketch(0, rs.n, True), oracle.sketch(oeng, reads, 0, rs.n, True),
                     (k, w, "micro"))
        # a sub-range whose first read is not the first tile
        sketch_equal(eng.sketch(3, rs.n - 2, True), oracle.sketch(oeng, reads, 3, rs.n - 2, True),
                     (k, w, "sub"))
    finally:
        eng.close()
    positions = sum(int(n) - k + 1 for n in rs.lens if n >= k)
    if w >= 8:   # the dense repeats overflow the first capacity: the retry ran
        assert full["value"].size > min(1.0, 2.2 / (w + 1)) * positions + 4096
    cnt = np.diff(full["offsets"].astype(np.int64))
    cap = routes(k, w)["stage_cap"]
    # a read whose micromizers are selected from global memory (at k = 1 a read keeps
    # len / 1 micromizers: its whole sketch, nothing is selected)
    assert ((cnt > cap) & (rs.lens.astype(np.int64) // k < cnt)).any() == (k > 1)


def index_reads(k, w):
    """overlapping reads and one poly-A read: a key with 65535 postings or more"""
    rs = overlap_reads(k, w, 120_000, 3)
    seqs = [rs.codes(i) for i in range(rs.n)]
    seqs.append(np.zeros(70_000 + k, np.uint8))
    return seqio.pack_codes(seqs)


@pytest.mark.gpu
@pytest.mark.parametrize("kw", POINTS, ids=IDS)
def test_index_and_filter_routes(gpu_engine, oracle, kw):
    k, w = kw
    rs = index_reads(k, w)
    gpu_engine.configure(k=k, w=w)
    gpu_engine.upload(rs)
    reads = oracle.reads(rs)
    for minhash in (False, True):
        gpu_engine.minimize(0, rs.n, minhash)
        idx = gpu_engine.index_records()
        eng = oracle.engine(k, w, threads=4)
        oracle.minimize(eng, reads, 0, rs.n, minhash)
        keys = oracle.keys(eng)
        v, o = idx["value"], idx["origin"]
        assert v.size == int(keys["totals"][1]) and idx["n_keys"] == int(keys["totals"][0])
        assert (v[1:] >= v[:-1]).all()
        same = v[1:] == v[:-1]
        assert (o[1:][same] > o[:-1][same]).all()
        uv, uc = np.unique(v, return_counts=True)
        assert np.array_equal(uv, keys["values"])
        assert np.array_equal(uc.astype(np.uint32), keys["counts"])
        if not minhash:
            assert int(keys["counts"].max()) >= 65535   # CollectLongRuns
        for f in (0.0005, 0.002, 1e-7, 0.001, 0.01, 0.2, 0.5, 1.0, 0):
            assert gpu_engine.filter(f) == oracle.filter(eng, f), (minhash, f)


def check_map(gpu_engine, oracle, rs, k, w, cases, n_index=None):
    """configure, index reads [0, n_index), map `cases`; hits (keep_hits), filtered
    positions and overlaps against the oracle; the hits of every call bounded. Returns
    the filtered positions of the first case and the query counts."""
    n_index = rs.n if n_index is None else n_index
    gpu_engine.configure(k=k, w=w)
    gpu_engine.upload(rs)
    eng, reads = oracle.engine(k, w, threads=4), oracle.reads(rs)
    oracle.minimize(eng, reads, 0, n_index, False)
    freq = choose_freq(oracle, eng)
    gpu_engine.set_option("keep_hits", 1)
    try:
        gpu_engine.minimize(0, n_index, False)
        assert gpu_engine.filter(freq) == oracle.filter(eng, freq)
        out, queries = None, []
        for (first, last, ae, asym, mh) in cases:
            gpu_engine.set_option("reset_stats", 1)
            got = gpu_engine.map(first, last, ae, asym, mh, want_filtered=True)
            st = gpu_engine.stats()
            assert st["hits"] <= HIT_BOUND
            queries.append((ae, asym, mh, st["query_records"]))
            hits = gpu_engine.map_hits(last - first)
            want = oracle.map(eng, reads, first, last, ae, asym, mh, want_matches=True)
            tag = (k, w, first, last, ae, asym, mh)
            assert np.array_equal(hits["hit_off"], want["match_off"]), tag
            assert st["hits"] == int(want["match_off"][-1])
            for i in range(last - first):
                a, b = int(hits["hit_off"][i]), int(hits["hit_off"][i + 1])
                g = np.stack([hits["group"][a:b], hits["positions"][a:b]], 1)
                x = np.stack([want["match_group"][a:b], want["match_pos"][a:b]], 1)
                assert np.array_equal(g[np.lexsort((g[:, 1], g[:, 0]))],
                                      x[np.lexsort((x[:, 1], x[:, 0]))]), (tag, i)
            for key in ("filt_off", "filtered", "ovl_off", "overlaps"):
                assert np.array_equal(got[key], want[key]), (tag, key)
            if out is None:
                out = got
        # a read outside the index (the last one)
        for j in range(n_index, rs.n):
            wd = rs.words[int(rs.word_off[j]):int(rs.word_off[j + 1])]
            for (ae, asym, mh) in ((True, True, True), (False, False, False)):
                got = gpu_engine.map_external(wd, int(rs.lens[j]), j, ae, asym, mh,
                                              want_filtered=True)
                want = oracle.map(eng, reads, j, j + 1, ae, asym, mh)
                assert np.array_equal(got["overlaps"], want["overlaps"]), (k, w, j, ae, mh)
                assert np.array_equal(got["filtered"], want["filtered"]), (k, w, j, ae, mh)
        return out, queries, reads
    finally:
        gpu_engine.set_option("keep_hits", 0)


@pytest.mark.gpu
@pytest.mark.parametrize("kw", POINTS, ids=IDS)
def test_map_routes(gpu_engine, oracle, kw):
    k, w = kw
    # fewer than 2^16 queries: the probe kernels in query order; all four flag pairs
    rs = overlap_reads(k, w, 60_000, 4)
    n = rs.n - 1
    cases = [(0, n, True, True, False), (0, n, True, False, True), (0, n, False, True, False),
             (0, n, False, False, True), (1, n - 1, True, True, True)]
    got, queries, reads = check_map(gpu_engine, oracle, rs, k, w, cases, n_index=n)
    assert max(q for *_, q in queries) < SORTED_PROBE_MIN
    # Pile::AddKmers' rule at this k on the positions map filtered
    ri = np.repeat(np.arange(n), np.diff(got["filt_off"].astype(np.int64)))
    keep = gpu_engine.kmer_complexity(ri, got["filtered"], k)
    assert np.array_equal(keep, oracle.kmer_complexity(reads, ri, got["filtered"], k))
    # 2^16 queries or more: the suffix probes go through the radix sort over 2k bits
    rs = overlap_reads(k, w, large_query_bases(k, w), 5)
    cases = [(0, rs.n, True, True, False), (0, rs.n, False, False, False)]
    _, queries, _ = check_map(gpu_engine, oracle, rs, k, w, cases)
    assert min(q for *_, q in queries) >= SORTED_PROBE_MIN


def oracle_stage1(oracle, rs, k, w, freq, kmax, minhash, ib=0, qb=0):
    return oracle.stage1(oracle.engine(k, w, threads=4), oracle.reads(rs), freq, kmax, minhash,
                         ib or 1 << 32, qb or 1 << 30)


def stage1_equal(got, want, tag):
    for key in KEYS:
        assert np.array_equal(got[key], want[key]), (tag, key)
    assert got["num_mapped"] == int(np.asarray(want["num_mapped"]).ravel()[0]), tag


@pytest.fixture
def restore(gpu_engine):
    try:
        yield gpu_engine
    finally:
        gpu_engine.set_index_chunks(-1, 0)
        gpu_engine.set_stage1_window(-1, 0)
        gpu_engine.set_option("tier_min_records", TIER_MIN_DEFAULT)
        gpu_engine.set_option("self_join", 1)
        gpu_engine.set_option("bare_count", 1)
        gpu_engine.configure(k=15, w=5)


WINDOW_POINTS = {(16, 5), (15, 6)}


@pytest.mark.gpu
@pytest.mark.parametrize("kw", POINTS, ids=IDS)
def test_stage1_routes(restore, oracle, kw):
    eng = restore
    k, w = kw
    rs = overlap_reads(k, w, 200_000, 6)
    bases = int(rs.lens.astype(np.int64).sum())
    probe = oracle.engine(k, w, threads=4)
    oracle.minimize(probe, oracle.reads(rs), 0, rs.n, False)
    # (an index batch of a few reads has fewer keys: at k <= 4 only the rarest survive
    # in every batch when the frequency is 1)
    freq = 1.0 if k <= 4 else choose_freq(oracle, probe, (0.001, 0.01, 0.05, 0.2, 0.6, 1.0))
    kmax = 8
    eng.configure(k=k, w=w)
    eng.upload(rs)

    def run(minhash, ib=0, qb=0, tiers=TIER_MIN_DEFAULT, join=1, bare=1, chunk=0, window=-1):
        eng.set_option("tier_min_records", tiers)
        eng.set_option("self_join", join)
        eng.set_option("bare_count", bare)
        eng.set_index_chunks(chunk)
        eng.set_stage1_window(window)
        eng.set_option("reset_stats", 1)
        got = eng.find_overlaps_and_create_piles(freq, kmax, minhash, ib, qb)
        assert eng.stats()["hits"] <= HIT_BOUND
        if chunk:
            assert eng.stage1_index_chunked()
        if window == 1:
            assert eng.stage1_windowed()
        return got

    sched = (bases // 3, bases // 7)
    for minhash in (False, True):
        # one index batch: untiered, then tiered (u32) with its thresholds
        want = oracle_stage1(oracle, rs, k, w, freq, kmax, minhash)
        assert len(want["occurrences"]) == 1
        stage1_equal(run(minhash), want, (k, w, minhash))
        stage1_equal(run(minhash, tiers=0), want, (k, w, minhash, "tiers"))
        assert eng.stats()["occurrence"] == int(want["occurrences"][0])
        if not minhash:   # thresholds of other frequencies off the same (tiered) index
            for f in (0.0005, 0.002, 0.2, 1.0):
                assert eng.filter(f) == oracle.filter(probe, f), f
        stage1_equal(run(minhash, chunk=bases // 3), want, (k, w, minhash, "chunked"))
        # several index batches and flushes
        want = oracle_stage1(oracle, rs, k, w, freq, kmax, minhash, *sched)
        assert len(want["occurrences"]) >= 3
        variants = [dict(), dict(join=0), dict(tiers=0), dict(tiers=0, join=0),
                    dict(chunk=bases // 5), dict(tiers=0, chunk=bases // 5)]
        if not minhash:
            variants += [dict(tiers=0, bare=0)]
            if (k, w) in WINDOW_POINTS:
                variants += [dict(window=1), dict(window=1, tiers=0, join=0)]
        for v in variants:
            stage1_equal(run(minhash, *sched, **v), want, (k, w, minhash, v))


# ---- other entry points ----

ENTRY_POINTS = [(16, 5), (15, 6), (17, 33)]
ENTRY_IDS = [f"k{k}w{w}" for k, w in ENTRY_POINTS]


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("kw", ENTRY_POINTS, ids=ENTRY_IDS)
def test_partitioned_run_routes(oracle, kw, world):
    from test_gpu_dist import check, run_virtual
    k, w = kw
    rs = synth.make_reads(60_000, 150, 5000, seed=11 + k, **HIFI)
    for minhash, ib, qb, tiers in ((True, 0, 0, False), (False, 250_000, 90_000, True)):
        want = oracle_stage1(oracle, rs, k, w, 0.001, 16, minhash, ib, qb)
        res = run_virtual(rs, world, 0.001, 16, ib, qb, params=dict(k=k, w=w), minhash=minhash,
                          tiers=tiers)
        check(res, want)
        assert list(res[0]["occurrences"]) == list(want["occurrences"])


@pytest.mark.gpu
@pytest.mark.parametrize("kw", ENTRY_POINTS, ids=ENTRY_IDS)
def test_reference_construct_over_facade_routes(tmp_path, oracle, kw):
    from test_gpu_dropin import run_dropin
    k, w = kw
    rs = synth.make_reads(40_000, 150, 3000, seed=13 + k, **HIFI)
    for minhash in (False, True):
        a, b = run_dropin(tmp_path, rs, k, w, 0.001, 8, minhash)
        want = oracle_stage1(oracle, rs, k, w, 0.001, 8, minhash)
        for got, name in ((a, "construct.cc over the facade"), (b, "batched")):
            for key in KEYS:
                assert np.array_equal(got[key], want[key]), (k, w, minhash, name, key)


# ---- configure ----

@pytest.mark.gpu
def test_configure_clamps_k_and_bounds_w(restore, oracle):
    eng = restore
    rs = synth.make_reads(30_000, 60, 2500, seed=19, **HIFI)
    rs_small = seqio.pack_codes(at_rich(np.random.default_rng(5), 30, 800))

    def results(k, w, reads):
        eng.configure(k=k, w=w)
        eng.upload(reads)
        sk = eng.sketch(0, reads.n, False)
        st = eng.find_overlaps_and_create_piles(0.6 if k <= 1 else 0.001, 8, False)
        return sk, st

    for lo, hi, w, reads in ((0, 1, 3, rs_small), (32, 31, 7, rs), (40, 31, 7, rs)):
        a_sk, a_st = results(lo, w, reads)
        b_sk, b_st = results(hi, w, reads)
        sketch_equal(a_sk, b_sk, (lo, hi))
        stage1_equal(a_st, dict(b_st, num_mapped=[b_st["num_mapped"]]), (lo, hi))
        sketch_equal(b_sk, oracle.sketch(oracle.engine(hi, w), oracle.reads(reads), 0, reads.n,
                                         False), hi)
    assert a_st["overlaps"].shape[0] > 0   # k = 31 finds the overlaps
    eng.configure(k=15, w=256)
    eng.upload(rs)
    assert eng.sketch(0, rs.n, False)["value"].size > 0
    with pytest.raises(ValueError):
        eng.configure(k=15, w=0)
    with pytest.raises(OverflowError):
        eng.configure(k=15, w=257)
