"""Deep POA windows: option "poa_wide" runs the windows past the 16-bit consensus
kernels' limits on PoaKernel<PoaWide> (poa.cu), and racon::Polisher sets it, so a
Polish of a high-coverage read set returns what racon returns instead of failing.

Every case first asserts which side of which limit its windows sit on (host
predicates of test_gpu_poa_edges.py and, for the graph-size limits, the oracle's
cell count); that part runs without a GPU.  The GPU cases compare bit exact with
the CPU oracle (oracle/spoa_graph.cpp + oracle/racon_window.cpp, int32 scalar
fill, no depth limit): consensus letters, offsets, status, coverages, cells.

No window of at most 65000 bases can outgrow 65000 edges: a sequence adds at most
one new edge per pair of consecutive bases, so a window has fewer edges than bases.
Past 65000 bases the host limit sends a window to the wide kernel before any graph
is built; at or below it, the capacity retry reaches the wide kernel through the
int16 guard."""
import os
import sys

import numpy as np
import pytest

from raven_b200 import synth
from test_gpu_poa_edges import (KEYS, MAX_LAYER_BASES, MAX_LAYERS, MAX_WINDOW_BASES,
                                TIE_SCORES, I16_LIMIT, _dims, all_oracle_batches, batch,
                                guard_cases, guard_lhs, kept_layers, per_window, rand_seq,
                                still_usable, substitute, window)

gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------------------
# host predicates
# ---------------------------------------------------------------------------
def flat_dims(b, i):
    """(window bases, longest layer, kept layers) of window i of a flat batch."""
    s0, s1 = int(b["win_first"][i]), int(b["win_first"][i + 1])
    lens = np.diff(b["seq_off"][s0:s1 + 1].astype(np.int64))
    kept = sum(1 for s in range(s0 + 1, s1)
               if lens[s - s0] > 0 and b["seq_begin"][s] != b["seq_end"][s])
    return int(lens.sum()), int(lens[1:].max(initial=0)), kept


def past_host_limits(b, i):
    tot, lmax, kept = flat_dims(b, i)
    return tot > MAX_WINDOW_BASES or lmax > MAX_LAYER_BASES or kept > MAX_LAYERS


def deep_windows(layers, n_windows=2, seed=0, with_quality=True):
    """ONT-like windows, every layer over the whole 500-base backbone."""
    return synth.make_windows(n_windows=n_windows, backbone_len=500, layers=layers,
                              seed=900 + layers + seed, partial=0.0,
                              with_quality=with_quality)


def sub_batch(b, idx):
    """Windows idx (in that order) of a flat batch."""
    wf, so = b["win_first"].astype(np.int64), b["seq_off"].astype(np.int64)
    out = dict(win_first=[0], seq_off=[0], bases=[], quals=[], seq_begin=[], seq_end=[])
    for i in idx:
        s0, s1 = wf[i], wf[i + 1]
        out["win_first"].append(out["win_first"][-1] + s1 - s0)
        for s in range(s0, s1):
            out["seq_off"].append(out["seq_off"][-1] + so[s + 1] - so[s])
        out["bases"].append(b["bases"][so[s0]:so[s1]])
        if b.get("quals") is not None:
            out["quals"].append(b["quals"][so[s0]:so[s1]])
        out["seq_begin"].append(b["seq_begin"][s0:s1])
        out["seq_end"].append(b["seq_end"][s0:s1])
    return dict(win_first=np.array(out["win_first"], np.uint32),
                seq_off=np.array(out["seq_off"], np.uint64),
                bases=np.concatenate(out["bases"]),
                quals=np.concatenate(out["quals"]) if out["quals"] else None,
                seq_begin=np.concatenate(out["seq_begin"]).astype(np.uint32),
                seq_end=np.concatenate(out["seq_end"]).astype(np.uint32))


def limit_cases():
    """(name, scores, window just inside a limit, window just past it)."""
    rng = np.random.default_rng(301)
    out = []
    # window bases: 500 + 129 * 500 = 65000; one more backbone base is past it
    bb = rand_seq(rng, 500)
    full = window(bb, [(substitute(rng, bb, 0.02), 0, 499) for _ in range(129)])
    assert _dims(full)[2] == MAX_WINDOW_BASES
    out.append(("window_bases", {}, full, window(bb + b"A", full["layers"])))
    # kept layers
    bb = rand_seq(rng, 10)
    many = window(bb, [(bb[3:5], 3, 4)] * MAX_LAYERS)
    assert len(kept_layers(many)) == MAX_LAYERS
    out.append(("layers", {}, many, window(bb, many["layers"] + [(bb[3:5], 3, 4)])))
    # layer bases: a layer of 32000 bases is inside the host limit, but never inside the
    # int16 guard (32000 + 2 columns alone): it reaches the wide kernel by the retry
    long_layer = rand_seq(rng, MAX_LAYER_BASES)
    inside = window(bb, [(bb, 0, 9), (long_layer, 0, 9)])
    past = window(bb, [(bb, 0, 9), (long_layer + b"C", 0, 9)])
    assert guard_lhs(rows=10, length=MAX_LAYER_BASES, **TIE_SCORES) > I16_LIMIT
    out.append(("layer_bases", TIE_SCORES, inside, past))
    # the int16 guard, at and one base past it (graph rows pinned by the oracle's cells in
    # test_gpu_poa_edges.test_guard_rows_are_what_the_cases_assume): windows of at most
    # 65000 bases that reach the wide kernel through the capacity retry
    for name, scores, w, _, over in guard_cases():
        if over is not None:
            out.append(("guard_" + name, scores, w, over))
    return out


# ---------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------
@pytest.fixture(scope="module")
def eng():
    from raven_b200 import engine
    e = engine.Engine(device=0)
    yield e
    e.close()


def set_wide(e, mode, budget=0):
    e.set_option("poa_wide", mode)
    e.set_option("poa_scratch_budget", budget)


def check(e, oracle, b, **kw):
    got = e.poa_batch(b, **kw)
    want = oracle.poa_batch(b, threads=8, **kw)
    for k in KEYS:
        assert np.array_equal(got[k], want[k]), k
    assert got["cells"] == int(want["cells"].sum())
    return got


def launches(e):
    r = e.poa_routes()["launches"]
    return r["fast"], r["generic"], r["wide"]


@gpu
@pytest.mark.parametrize("layers", [150, 250, 400])
def test_deep_ont_windows(eng, oracle, layers):
    for with_q in (True, False):
        b = deep_windows(layers, with_quality=with_q)
        nw = b["win_first"].size - 1
        assert all(past_host_limits(b, i) for i in range(nw))
        set_wide(eng, 1)
        for trim in (True, False):
            got = check(eng, oracle, b, trim=trim)
            assert (got["status"] & 1).all()
            r = eng.poa_routes()
            assert (r["fast"], r["generic"], r["wide"]) == (0, 0, nw)
            assert "poa_wide" in eng.timings()
        set_wide(eng, 0)
        with pytest.raises(OverflowError, match="65000 bases"):
            eng.poa_batch(b)
    # the deep consensus is closer to the hidden truth than the draft
    b = deep_windows(layers)
    set_wide(eng, 1)
    got = eng.poa_batch(b)
    set_wide(eng, 0)
    off = got["cons_off"].astype(np.int64)
    for i in range(off.size - 1):
        s0 = int(b["win_first"][i])
        draft = b["bases"][int(b["seq_off"][s0]):int(b["seq_off"][s0 + 1])].tobytes()
        cons = got["consensus"][off[i]:off[i + 1]].tobytes()
        assert oracle.edit_distance(cons, b["truths"][i]) * 5 < \
            oracle.edit_distance(draft, b["truths"][i])


@gpu
def test_both_sides_of_every_limit(eng, oracle):
    for name, scores, inside, past in limit_cases():
        set_wide(eng, 0)
        today = None
        try:
            today = eng.poa_batch(batch([inside]), **scores)
            before = launches(eng)
        except OverflowError:
            pass
        with pytest.raises(OverflowError):
            eng.poa_batch(batch([past]), **scores)
        set_wide(eng, 1)
        got = check(eng, oracle, batch([inside]), **scores)
        if today is not None:   # inside the limit: today's route and result
            assert launches(eng) == before and launches(eng)[2] == 0, name
            assert per_window(got) == per_window(today), name
        else:                   # only the 32000-base layer: the guard sends it on
            assert name == "layer_bases"
            assert launches(eng) == (0, 2, 1)
        got = check(eng, oracle, batch([past]), **scores)
        assert got["status"][0] & 1, name
        assert eng.poa_routes()["wide"] == 1, name
        if name.startswith("guard_"):
            # first and second tier on the narrow kernels, then the wide one
            assert sum(launches(eng)[:2]) == 2, name
        else:
            assert launches(eng)[:2] == (0, 0), name
    set_wide(eng, 0)


@gpu
def test_mixed_batch(eng, oracle):
    shallow = synth.make_windows(n_windows=20, backbone_len=500, layers=30, seed=321)
    deep = deep_windows(150, n_windows=3, seed=1)
    both = synth_concat(shallow, deep)
    ns, nd = shallow["win_first"].size - 1, deep["win_first"].size - 1
    order = np.random.default_rng(322).permutation(ns + nd)
    mixed = sub_batch(both, order)
    set_wide(eng, 0)
    alone = eng.poa_batch(shallow)
    alone_launches = launches(eng)
    set_wide(eng, 1)
    got = check(eng, oracle, mixed)
    r = eng.poa_routes()
    assert r["wide"] == nd and launches(eng)[:2] == alone_launches[:2]
    set_wide(eng, 0)
    a, m = per_window(alone), per_window(got)
    for at, i in enumerate(order):
        if i < ns:
            assert m[at] == a[i], f"shallow window {i}"


def synth_concat(a, b):
    n = a["win_first"].size - 1 + b["win_first"].size - 1
    both = dict(win_first=np.concatenate([a["win_first"], b["win_first"][1:] + a["win_first"][-1]]),
                seq_off=np.concatenate([a["seq_off"], b["seq_off"][1:] + a["seq_off"][-1]]),
                bases=np.concatenate([a["bases"], b["bases"]]),
                quals=np.concatenate([a["quals"], b["quals"]]),
                seq_begin=np.concatenate([a["seq_begin"], b["seq_begin"]]),
                seq_end=np.concatenate([a["seq_end"], b["seq_end"]]))
    assert both["win_first"].size == n + 1
    return both


def poa_module_batches():
    """The window batches of test_gpu_poa.py, as (name, batch, kwargs)."""
    out = []
    for seed in (1, 2, 3):
        out.append((f"ont_{seed}", synth.make_windows(n_windows=24, backbone_len=500, layers=30,
                                                      seed=seed), {}))
    w = synth.make_windows(n_windows=12, backbone_len=300, layers=12, seed=5,
                           with_quality=False, partial=1.0)
    for i, kw in enumerate(({}, dict(m=5, n=-4, g=-8), dict(trim=False), dict(tgs=False))):
        out.append((f"variants_{i}", w, kw))
    out.append(("hifi", synth.make_windows(n_windows=6, backbone_len=500, layers=60, seed=6,
                                           sub=0.002, ins=0.0015, dele=0.0015), {}))
    out.append(("ragged", synth.make_windows(n_windows=16, backbone_len=200, layers=6, seed=7,
                                             min_layers=0), {}))
    out.append(("long", synth.make_windows(n_windows=5, backbone_len=760, layers=14, seed=11),
                {}))
    out.append(("insertions", synth.make_windows(n_windows=3, backbone_len=520, layers=10,
                                                 seed=13, ins=0.12, dele=0.01), {}))
    return out


@gpu
def test_every_window_on_the_wide_kernel(eng):
    """poa_wide=2: the batches of test_gpu_poa.py and test_gpu_poa_edges.py on the wide
    kernel give what the narrow kernels give - one definition, two widths."""
    cases = [(n, b, kw) for n, b, kw in poa_module_batches()]
    cases += [(n, batch(w, q), kw) for n, w, q, kw in all_oracle_batches()]
    for name, b, kw in cases:
        nw = b["win_first"].size - 1
        set_wide(eng, 0)
        narrow = eng.poa_batch(b, **kw)
        assert eng.poa_routes()["wide"] == 0, name
        set_wide(eng, 2)
        wide = eng.poa_batch(b, **kw)
        assert eng.poa_routes()["wide"] == nw, name
        for k in KEYS + ("cells",):
            assert np.array_equal(narrow[k], wide[k]), (name, k)
    set_wide(eng, 0)


@gpu
def test_scratch_budget(eng, oracle):
    b = deep_windows(150, n_windows=1)
    set_wide(eng, 1, budget=1 << 20)
    with pytest.raises(OverflowError, match=r"needs \d+ bytes of scratch"):
        eng.poa_batch(b)
    with pytest.raises(RuntimeError, match="no POA results"):
        eng.poa_routes()
    set_wide(eng, 1)
    check(eng, oracle, b)
    set_wide(eng, 0)
    still_usable(eng, oracle)


def _polish_pair(oracle, draft, reads, q=0.0):
    from raven_b200 import polish
    got, st = polish.polish(draft, reads, q=q, threads=4)
    names, seqs, ost = oracle.polish(draft, reads, q=q, threads=8)
    assert got.names == names
    assert [got.ascii(i) for i in range(got.n)] == seqs
    assert st["windows"] == int(ost[0]) and st["polished_windows"] == int(ost[1])
    assert st["wide_windows"] > 0
    os.environ["RVN_SET_OPTIONS"] = "poa_wide=0"
    try:
        with pytest.raises(RuntimeError, match="65000 bases"):
            polish.polish(draft, reads, q=q, threads=4)
    finally:
        del os.environ["RVN_SET_OPTIONS"]
    return st


@gpu
def test_polisher_at_high_coverage(oracle, lambda_reads):
    sys.path.insert(0, ROOT)
    from bench import synth as bsynth
    from raven_b200 import seqio
    # about 150x over a 20 kb draft
    reads = bsynth.make_reads(401, 20_000, 650, 5000, min_len=1500)
    draft = bsynth.make_contigs(401, 20_000, contig_len=20_000)
    assert reads.bases > 140 * 20_000
    _polish_pair(oracle, draft, reads)
    # the lambda fixture's reads four times over (about 140x) against the lambda genome
    genome = seqio.ReadSet.load(os.path.join(ROOT, "tests", "golden", "lambda_genome.npz"))
    deep = lambda_reads.subset(list(range(lambda_reads.n)) * 4)
    assert deep.bases > 130 * genome.bases
    _polish_pair(oracle, genome, deep)


# ---------------------------------------------------------------------------
# without a GPU
# ---------------------------------------------------------------------------
def test_deep_cases_sit_past_their_limits():
    for layers in (150, 250, 400):
        b = deep_windows(layers)
        for i in range(b["win_first"].size - 1):
            tot, lmax, kept = flat_dims(b, i)
            assert tot > MAX_WINDOW_BASES and lmax <= MAX_LAYER_BASES and kept == layers
    for name, scores, inside, past in limit_cases():
        bi, bp = batch([inside]), batch([past])
        if name in ("window_bases", "layers"):
            assert not past_host_limits(bi, 0) and past_host_limits(bp, 0), name
        elif name == "layer_bases":
            assert flat_dims(bi, 0)[1] == MAX_LAYER_BASES and past_host_limits(bp, 0)
        else:
            assert not past_host_limits(bp, 0), name
