"""POA window consensus at its structural edges: windows built on purpose for
every route of PoaBatch / PoaKernelFast / PoaKernel (poa.cu, poa_fast.cuh),
each compared bit exact with the CPU oracle (oracle/spoa_graph.cpp +
oracle/racon_window.cpp): consensus letters, offsets, status, coverages, cells.

A host predicate (`route`, `is_full`, `guard_lhs`) restates PoaBatch's
arithmetic; every case asserts that its windows sit on the intended side of
the edge before anything is compared.  The unmarked tests at the end run
without a GPU: the same windows through the oracle's scalar and AVX2 fills,
the route assertions, and hand-computed expectations that anchor the oracle."""
import numpy as np
import pytest

gpu = pytest.mark.gpu

# thresholds of poa.cu / poa_fast.cuh as the source has them
K_S = 18                     # DP columns per lane of PoaKernelFast
FAST_COLS = 32 * K_S         # 576: layers of at most 575 bases take the fast kernel
FAST_SMEM_MAX = 220 * 1024   # beyond it a fast-group window runs on PoaKernel
I16_LIMIT = 32000            # amax * (rows + len + 2) above it: LimitError
MAX_LAYERS = 4095
MAX_WINDOW_BASES = 65000
MAX_LAYER_BASES = 32000

LANE_LENGTHS = [1, 2, 17, 18, 19, 35, 36, 37, 557, 558, 559, 574, 575]
GENERIC_LENGTHS = [576, 607, 608, 639]

ACGT = b"ACGT"


# ---------------------------------------------------------------------------
# builder
# ---------------------------------------------------------------------------
def window(backbone, layers, backbone_quals=None):
    """layers: (bases, begin, end[, quals]) in backbone coordinates."""
    out = []
    for l in layers:
        bases, begin, end = l[0], l[1], l[2]
        out.append((bytes(bases), int(begin), int(end), l[3] if len(l) > 3 else None))
    return dict(bb=bytes(backbone), bq=backbone_quals, layers=out)


def _default_quals(n, salt):
    return bytes(33 + 10 + (i * 7 + salt) % 17 for i in range(n))


def batch(windows, with_quality=False):
    """The flat dict Engine.poa_batch and Oracle.poa_batch take."""
    win_first, seq_off, begins, ends, bases, quals = [0], [0], [], [], [], []
    for w in windows:
        seqs = [(w["bb"], 0, 0, w["bq"] if w["bq"] is not None else b"!" * len(w["bb"]))]
        for k, (b, lo, hi, q) in enumerate(w["layers"]):
            seqs.append((b, lo, hi, q if q is not None else _default_quals(len(b), k)))
        for b, lo, hi, q in seqs:
            assert len(q) == len(b)
            bases.append(b)
            quals.append(q)
            seq_off.append(seq_off[-1] + len(b))
            begins.append(lo)
            ends.append(hi)
        win_first.append(win_first[-1] + len(seqs))
    return dict(win_first=np.array(win_first, np.uint32), seq_off=np.array(seq_off, np.uint64),
                bases=np.frombuffer(b"".join(bases), np.uint8).copy(),
                quals=np.frombuffer(b"".join(quals), np.uint8).copy() if with_quality else None,
                seq_begin=np.array(begins, np.uint32), seq_end=np.array(ends, np.uint32))


def rand_seq(rng, n, letters=ACGT):
    return bytes(letters[i] for i in rng.integers(0, len(letters), n))


def substitute(rng, s, rate):
    """Substitutions only: the length stays what the case needs."""
    s = bytearray(s)
    for i in range(len(s)):
        if rng.random() < rate:
            s[i] = ACGT[(ACGT.index(s[i]) + int(rng.integers(1, 4))) % 4]
    return bytes(s)


def shift_one(s, at):
    """One deletion and one insertion, 5 bases apart: same length, two gaps."""
    if len(s) < at + 8:
        return s
    s = bytearray(s)
    del s[at]
    s.insert(at + 5, ACGT[(ACGT.index(s[at + 5]) + 1) % 4])
    return bytes(s)


# ---------------------------------------------------------------------------
# the route a window takes, by PoaBatch's arithmetic
# ---------------------------------------------------------------------------
def kept_layers(w):
    """racon::Window::AddLayer drops a layer without bases or with begin == end."""
    return [l for l in w["layers"] if len(l[0]) > 0 and l[1] != l[2]]


def sequences(w):
    return 1 + len(kept_layers(w))


def _dims(w):
    lmax = max([1] + [len(l[0]) for l in w["layers"]])
    total = len(w["bb"]) + sum(len(l[0]) for l in w["layers"])
    return lmax, max(1, len(w["bb"])), max(1, total)


def fast_group(w):
    return _dims(w)[0] + 1 <= FAST_COLS


def route(windows, tier=0):
    """Per kernel group ('fast' / 'generic' by longest layer): the shape PoaBatch
    gives the launch that holds `windows` at that tier, and the kernel it runs."""
    out = {}
    for name, want in (("fast", True), ("generic", False)):
        mem = [_dims(w) for w in windows if fast_group(w) == want]
        if not mem:
            continue
        lmax, bb, total = (max(d[i] for d in mem) for i in range(3))
        ncap = min(total, 3 * bb + lmax + 64) if tier == 0 else total
        ncap = min(ncap, 65000)
        smem = ((ncap + 15) & ~15) + 4 * ncap + 16
        out[name] = dict(lmax=lmax, ncap=ncap, total=total, smem=smem,
                         width=(lmax + 1 + 31) & ~31,
                         kernel="fast" if want and smem <= FAST_SMEM_MAX else "generic")
    return out


def is_full(w, layer):
    """The layer aligns to the whole graph and not to a sub-graph."""
    L0 = len(w["bb"])
    offset = int(0.01 * L0)
    return layer[1] < offset and layer[2] > L0 - offset


def guard_lhs(m, n, g, rows, length):
    return max(abs(m), abs(n), abs(g)) * (rows + length + 2)


# ---------------------------------------------------------------------------
# comparison
# ---------------------------------------------------------------------------
KEYS = ("cons_off", "consensus", "status", "coverage")


def check(eng, oracle, windows, with_quality=False, **kw):
    b = batch(windows, with_quality)
    got = eng.poa_batch(b, **kw)
    want = oracle.poa_batch(b, threads=8, **kw)
    for k in KEYS:
        assert np.array_equal(got[k], want[k]), k
    assert got["cells"] == int(want["cells"].sum())
    return got


def per_window(res):
    off = res["cons_off"].astype(np.int64)
    return [(res["consensus"][off[i]:off[i + 1]].tobytes(), int(res["status"][i]),
             res["coverage"][off[i]:off[i + 1]].tolist()) for i in range(off.size - 1)]


def still_usable(eng, oracle):
    check(eng, oracle, anchor_windows()[0])


# ---------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------
def lane_windows():
    """Per edge length: a window whose layers all have it, and a window with one
    such layer among short ones.  Returns (windows, lengths)."""
    wins, lens = [], []
    for ell in LANE_LENGTHS + GENERIC_LENGTHS:
        rng = np.random.default_rng(1000 + ell)
        B = max(ell + 7, 40)
        bb = rand_seq(rng, B)
        hi = lambda a: a + max(ell - 1, 1)   # a one-base layer still spans two nodes
        every = []
        for k, a in enumerate((0, 3, 7, 0, 5)):
            s = substitute(rng, bb[a:a + ell], 0.06)
            if k == 3:
                s = shift_one(s, 4)
            every.append((s, a, hi(a)))
        assert all(len(l[0]) == ell for l in every)
        wins.append(window(bb, every))
        mixed = [(substitute(rng, bb[a:a + 20], 0.06), a, a + 19) for a in (0, 9, 15, 18)]
        mixed.insert(2, (substitute(rng, bb[2:2 + ell], 0.06), 2, hi(2)))
        wins.append(window(bb, mixed))
        lens += [ell, ell]
    for w, ell in zip(wins, lens):
        assert fast_group(w) == (ell <= 575)
        r = route([w])
        assert r["fast" if ell <= 575 else "generic"]["kernel"] == ("fast" if ell <= 575 else "generic")
        # the sink column of the fast kernel: lane len / 18, slot len % 18
    assert {(l // K_S, l % K_S) for l in LANE_LENGTHS} >= {
        (0, 1), (0, 17), (1, 0), (1, 1), (1, 17), (2, 0), (31, 0), (31, 16), (31, 17)}
    assert [route([w])["generic"]["width"] for w in wins[2 * len(LANE_LENGTHS)::2]] == [
        608, 608, 640, 640]
    return wins, lens


def graph_windows():
    """Full graph or sub-graph: begin / end around offset = uint32(0.01 * L0).
    Returns (windows, number of layers that take the full graph)."""
    wins, n_full = [], 0
    for L0 in (99, 100, 199, 200):
        rng = np.random.default_rng(2000 + L0)
        bb = rand_seq(rng, L0)
        off = int(0.01 * L0)
        begins = sorted({0, max(off - 1, 0), off, off + 1})
        ends = sorted({L0 - off - 1, min(L0 - off, L0 - 1), min(L0 - off + 1, L0 - 1), L0 - 1})
        for b in begins:
            for e in ends:
                w = window(bb, [(substitute(rng, bb[b:e + 1], 0.08), b, e) for _ in range(4)])
                full = is_full(w, w["layers"][0])
                assert full == (L0 == 200 and b < 2 and e == 199)
                n_full += full
                wins.append(w)
    assert n_full == 2   # only L0 = 200 has a begin and an end that select the full graph
    rng = np.random.default_rng(2999)
    bb = rand_seq(rng, 150)
    # the smallest sub-graph, with layers of its size and with a long layer whose
    # bases almost all become leading or trailing chain
    wins.append(window(bb, [(bb[0:2], 0, 1), (bb[0:2], 0, 1), (bb[1:2] + b"T", 0, 1)]))
    wins.append(window(bb, [(rand_seq(rng, 300), 0, 1), (bb[0:2], 0, 1),
                            (rand_seq(rng, 40) + bb[148:150], 148, 149),
                            (substitute(rng, bb, 0.05), 0, 149)]))
    # layers that end before the next begins
    wins.append(window(bb, [(substitute(rng, bb[a:a + 30], 0.05), a, a + 29)
                            for a in (0, 30, 61, 100, 120)]))
    for w in wins[-3:]:
        assert not any(is_full(w, l) for l in w["layers"])
    return wins, n_full


def plain_windows(seed, n=3, B=100, layers=6):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        bb = rand_seq(rng, B)
        out.append(window(bb, [(shift_one(substitute(rng, bb, 0.05), 10 + 3 * k), 0, B - 1)
                               for k in range(layers)]))
    return out


def divergent_window(seed, n_layers, length, B=50):
    """Unrelated layers over a short backbone: the graph grows by most of every
    layer and outgrows the first capacity tier."""
    rng = np.random.default_rng(seed)
    return window(rand_seq(rng, B), [(rand_seq(rng, length), 0, B - 1) for _ in range(n_layers)])


def tier_windows():
    plain = plain_windows(31)
    big = divergent_window(32, 16, 400)
    r0, r1 = route(plain + [big]), route([big], tier=1)
    assert set(r0) == {"fast"} and r0["fast"]["kernel"] == "fast"
    assert r0["fast"]["ncap"] == 3 * 100 + 400 + 64 < r1["fast"]["ncap"] == 50 + 16 * 400
    assert r1["fast"]["kernel"] == "fast"
    return plain, big


def fallback_windows():
    """Layers of 575 bases (fast group), more than 45,056 bases of them: the retry's
    shared-memory need passes 220 KiB and the window runs on the generic kernel."""
    plain = plain_windows(41)
    big = divergent_window(42, 85, 575)
    assert 45056 < _dims(big)[2] <= MAX_WINDOW_BASES and fast_group(big)
    assert route(plain + [big])["fast"]["kernel"] == "fast"
    r1 = route([big], tier=1)["fast"]
    assert r1["smem"] > FAST_SMEM_MAX and r1["kernel"] == "generic"
    return plain, big


TIE_SCORES = dict(m=1, n=-1, g=-1)   # amax = 1 keeps the deep graph inside int16


def guard_cases():
    """(name, scores, window at or just below the limit, rows seen by each layer,
    the first window above the limit).  rows are what the case is built to give;
    test_guard_rows_are_what_the_cases_assume checks them against the oracle's cells."""
    out = []
    rng = np.random.default_rng(51)

    def match(B, ll):      # layers = a prefix of the backbone: ll matches, B - ll gaps
        bb = rand_seq(rng, B)
        return window(bb, [(bb[:ll], 0, B - 1)] * 2), [B, B]

    def mismatch(B, ll):   # every layer base opens a new node in its column
        return window(b"A" * B, [(b"C" * ll, 0, B - 1)] * 2), [B, B + ll]

    def gaps(B):           # one base against B nodes: B - 1 gaps
        return window(b"A" * B, [(b"A", 0, B - 1)] * 2), [B, B]

    for scores, S in ((dict(m=127, n=-127, g=-127), 249), (dict(m=5, n=-4, g=-8), 3998)):
        amax = max(abs(v) for v in scores.values())
        assert amax * (S + 2) <= I16_LIMIT < amax * (S + 3)
        ll = min(S // 2, 500)   # at most 575: the fast kernel's guard
        fills = [("match", match, (S - ll, ll)),
                 ("match_below", match, (S - ll, ll - 1)),
                 ("mismatch", mismatch, (S - 2 * min(S // 5, 500), min(S // 5, 500))),
                 ("gaps", gaps, (S - 1,))]
        if amax == 8:   # room for a layer beyond 575 bases: the generic kernel's guard
            fills.append(("match_generic", match, (S - 1000, 1000)))
        for name, make, args in fills:
            w, rows = make(*args)
            lhs = max(guard_lhs(rows=r, length=len(l[0]), **scores)
                      for r, l in zip(rows, w["layers"]))
            below = name == "match_below"
            assert lhs == amax * (S + 1 if below else S + 2) <= I16_LIMIT
            if amax == 8 and not below:
                assert lhs == I16_LIMIT
            assert fast_group(w) == (name != "match_generic")
            over = None
            if not below:
                bigger = list(args)
                bigger[-1] += 1   # one more base (a longer layer, or a longer backbone)
                over, orows = make(*bigger)
                olhs = max(guard_lhs(rows=r, length=len(l[0]), **scores)
                           for r, l in zip(orows, over["layers"]))
                assert olhs > I16_LIMIT and olhs - lhs <= 2 * amax
            out.append((f"{name}_{amax}", scores, w, rows, over))
    return out


def simd_limit_cases():
    """The oracle's AVX2 fill keeps int16 by amax * (2 * width + height + 32) <= 32000
    and leaves the rest to the scalar fill: windows on its last admitted size, filled
    so the scores run to the negative end."""
    out = []
    for scores, room in ((dict(m=127, n=-127, g=-127), 251), (dict(m=5, n=-4, g=-8), 4000)):
        ll = min((room - 35) // 5, 500)
        B = room - 35 - 3 * ll            # second layer: height B + ll + 1, width ll + 1
        out.append((scores, window(b"A" * B, [(b"C" * ll, 0, B - 1)] * 2), (B + ll + 1, ll + 1)))
        B = room - 38                     # one base against B nodes and one more
        out.append((scores, window(b"A" * B, [(b"C", 0, B - 1), (b"A", 0, B - 1)]), (B + 2, 2)))
    for scores, w, (height, width) in out:
        amax = max(abs(v) for v in scores.values())
        assert amax * (2 * width + height + 32) <= I16_LIMIT < amax * (2 * width + height + 33)
    return out


def pred_windows():
    """70 layers, each the backbone without the k bases before position P: node P
    collects an in-edge per k, 71 with the backbone's.  No letter before P stands
    twice in a row, which leaves each deletion one best place and no edge to share.
    Then layers that cross P over a predecessor below and above ordinal 63."""
    rng = np.random.default_rng(61)
    B, P, K = 200, 120, 70
    bb = bytearray(rand_seq(rng, B))
    for i in range(P - K - 2, P - 1):   # no letter twice in a row: a deletion cannot slide
        bb[i] = [x for x in b"ACG" if x != bb[i - 1]][int(rng.integers(0, 2))]
    bb[P - 2] = ord("A") if bb[P - 3] != ord("A") else ord("C")
    bb[P - 1:P + 1] = b"GT"
    bb = bytes(bb)
    assert all(bb[i] != bb[i + 1] for i in range(P - K - 3, P))
    cut = lambda k: bb[:P - k] + bb[P:]
    layers = [(cut(k), 0, B - 1) for k in range(1, K + 1)]
    layers += [(cut(10), 0, B - 1), (cut(68), 0, B - 1), (cut(33), 0, B - 1), (cut(64), 0, B - 1)]
    fast = window(bb, layers)
    assert all(is_full(fast, l) for l in layers) and K + 1 > 64
    generic = window(bb, layers + [(rand_seq(rng, 600), 0, B - 1)])
    assert route([fast])["fast"]["kernel"] == "fast" and not fast_group(generic)
    # a column with all four letters: a node with three aligned partners
    bb2 = rand_seq(rng, 120)
    c = 60
    put = lambda ch: bb2[:c] + ch + bb2[c + 1:]
    others = [bytes([x]) for x in ACGT if x != bb2[c]]
    col = [(put(ch), 0, 119) for ch in others]
    col += [(put(ch), 0, 119) for ch in others + [bb2[c:c + 1]] * 2 + others[::-1]]
    col += [(put(ch)[40:80], 40, 79) for ch in others]
    four = window(bb2, col)
    expect_cells = sum((B + 1) * (len(l[0]) + 1) for l in layers)
    return fast, generic, four, expect_cells


def dropped_layer_windows():
    """Layers racon::Window::AddLayer drops (no bases, or begin == end) at the first,
    a middle and the last position.  Returns (windows, expected status)."""
    rng = np.random.default_rng(71)
    B = 100
    bb = rand_seq(rng, B)
    real = lambda b=0, e=B - 1: (substitute(rng, bb[b:e + 1], 0.08), b, e)
    empty = (b"", 0, B - 1)
    point = (bb[10:30], 40, 40)
    outside = (bb[10:30], 5000, 5000)   # dropped before its coordinates are looked at
    wins, status = [], []
    for drops in ([empty], [point], [empty, point, outside]):
        # across `sequences < 3`: one real layer and dropped ones is the backbone
        wins += [window(bb, drops + [real()]), window(bb, [real()] + drops)]
        status += [0, 0]
        # two real layers stay polished wherever the dropped ones sit
        for at in (0, 1, 2):
            l = [real(), real()]
            l[at:at] = drops
            wins.append(window(bb, l))
            status.append(1)
    # across the trimming threshold (sequences - 1) / 2: the ends are covered by the
    # backbone and two layers = 3; six sequences ask for 2, ten would ask for 4
    part = [real(), real(20, 80), (b"", 3, 9), real(20, 80), point, real(20, 80), empty,
            real(), outside]
    wins.append(window(bb, part))
    status.append(1)
    assert sequences(wins[-1]) == 6 and len(part) + 1 == 10
    # every layer dropped
    wins.append(window(bb, [empty, point, outside]))
    status.append(0)
    assert sequences(wins[-1]) == 1
    for w, st in zip(wins, status):
        assert (sequences(w) >= 3) == bool(st)
    return wins, status


def tie_windows():
    """Repeats, copies and equal begins: every DP cell and every weight a tie."""
    rng = np.random.default_rng(81)
    wins = []
    for unit in (b"A", b"AC", b"ACG"):
        bb = (unit * 120)[:120]
        # the same repeat with a unit more or less, whole and partial
        layers = [(bb, 0, 119), ((unit * 120)[:120 - len(unit)], 0, 119),
                  ((unit * 130)[:120 + len(unit)], 0, 119), (bb[:60], 0, 59),
                  (bb[30:90], 30, 89), ((unit * 40)[:60 + len(unit)], 30, 89)]
        wins.append(window(bb, layers))
    bb = rand_seq(rng, 140)
    other = substitute(rng, bb, 0.1)
    wins.append(window(bb, [(bb, 0, 139)] * 4))                       # layers = backbone
    wins.append(window(bb, [(other, 0, 139)] * 5))                    # layers = each other
    a, b, c = (shift_one(substitute(rng, bb[20:120], 0.1), 7 * k) for k in (1, 2, 3))
    wins.append(window(bb, [(a, 20, 119), (b, 20, 119), (c, 20, 119), (a, 20, 119)]))
    wins.append(window(bb, [(c, 20, 119), (a, 20, 119), (a, 20, 119), (b, 20, 119)]))
    return wins


def quality_variants(wins):
    """(windows, with_quality) under each weighting."""
    def requal(w, q, bq):
        return window(w["bb"], [(l[0], l[1], l[2], q * len(l[0])) for l in w["layers"]],
                      bq * len(w["bb"]) if bq else None)
    real_bq = [window(w["bb"], w["layers"], _default_quals(len(w["bb"]), 5)) for w in wins]
    return [("none", wins, False), ("default", wins, True),
            ("all_zero", [requal(w, b"!", b"!") for w in wins], True),
            ("backbone_weighs", real_bq, True)]


def heavy_window():
    """200 layers of quality '~' (weight 93 a base): the largest edge weights."""
    rng = np.random.default_rng(91)
    bb = rand_seq(rng, 100)
    return window(bb, [(substitute(rng, bb, 0.05), 0, 99, b"~" * 100) for _ in range(200)],
                  b"~" * 100)


def chimeric_windows():
    """Coverage below (sequences - 1) / 2 everywhere, at one position, at two."""
    rng = np.random.default_rng(95)
    bb = rand_seq(rng, 240)
    seg = lambda a, b: (bb[a:b + 1], a, b)
    spread = [seg(110, 130), seg(140, 160), seg(170, 190), seg(200, 220)]
    never = window(bb, [seg(a, a + 24) for a in range(0, 200, 25)])
    once = window(bb, [seg(0, 50), seg(50, 100)] + spread)
    twice = window(bb, [seg(0, 51), seg(50, 100)] + spread)
    assert (sequences(never) - 1) // 2 == 4 and (sequences(once) - 1) // 2 == 3
    return [never, once, twice], [3, 3, 1]


def anchor_windows():
    """Windows whose result follows from racon's rules without running anything."""
    rng = np.random.default_rng(99)
    bb = rand_seq(rng, 40)
    layer = bytearray(bb)
    for i in (5, 20, 33):
        layer[i] = ACGT[(ACGT.index(layer[i]) + 1) % 4]
    layer = bytes(layer)
    return [window(bb, [(layer, 0, 39)] * 3), window(bb, [(layer, 0, 39)]), window(bb, [])], layer


def all_oracle_batches():
    """Every batch of this file the oracle can run, as (name, windows, quality, kwargs)."""
    out = [("lane", lane_windows()[0], False, {}), ("graph", graph_windows()[0], False, {})]
    plain, big = tier_windows()
    out.append(("tier", plain + [big], False, {}))
    for name, scores, w, _, _ in guard_cases():
        out.append(("guard_" + name, [w], False, scores))
    fast, generic, four, _ = pred_windows()
    out.append(("pred", [fast, generic, four], False, {}))
    for i, (scores, w, _) in enumerate(simd_limit_cases()):
        out.append((f"simd_limit_{i}", [w], False, scores))
    out.append(("dropped", dropped_layer_windows()[0], False, {}))
    for name, wins, q in quality_variants(tie_windows()):
        out.append(("ties_" + name, wins, q, {}))
        out.append(("ties_notrim_" + name, wins, q, dict(trim=False)))
    out.append(("heavy", [heavy_window()], True, {}))
    out.append(("chimeric", chimeric_windows()[0], False, {}))
    out.append(("anchor", anchor_windows()[0], False, {}))
    return out


# ---------------------------------------------------------------------------
# GPU: every case against the oracle
# ---------------------------------------------------------------------------
@gpu
def test_lane_and_kernel_edges(gpu_engine, oracle):
    wins, lens = lane_windows()
    alone = [per_window(gpu_engine.poa_batch(batch([w])))[0] for w in wins]
    order = np.random.default_rng(5).permutation(len(wins))
    mixed = per_window(check(gpu_engine, oracle, [wins[i] for i in order]))
    for at, i in enumerate(order):
        assert mixed[at] == alone[i], f"layer length {lens[i]}, window {i}"
        assert mixed[at][1] & 1
    # and in the given order, with qualities
    check(gpu_engine, oracle, wins, with_quality=True)


@gpu
def test_full_graph_or_sub_graph(gpu_engine, oracle):
    wins, _ = graph_windows()
    for q in (False, True):
        got = check(gpu_engine, oracle, wins, with_quality=q)
        assert (got["status"] & 1).all()
    check(gpu_engine, oracle, wins, trim=False)


def _launches(eng, oracle, wins, **kw):
    before = eng.stats()["kernel_launches"]
    got = check(eng, oracle, wins, **kw)
    return eng.stats()["kernel_launches"] - before, got


@gpu
def test_capacity_tier_retry(gpu_engine, oracle):
    plain, big = tier_windows()
    base, ref = _launches(gpu_engine, oracle, plain)
    more, got = _launches(gpu_engine, oracle, plain[:2] + [big] + plain[2:])
    assert (base, more) == (1, 2)   # one group; the retry is one more launch
    a, b = per_window(ref), per_window(got)
    assert b[:2] + b[3:] == a       # the windows that fitted are left as they were
    assert b[2][1] & 1


@gpu
def test_fast_group_retry_on_the_generic_kernel(gpu_engine, oracle):
    plain, big = fallback_windows()
    base, ref = _launches(gpu_engine, oracle, plain, **TIE_SCORES)
    more, got = _launches(gpu_engine, oracle, [big] + plain, **TIE_SCORES)
    assert (base, more) == (1, 2)
    assert per_window(got)[1:] == per_window(ref)


@gpu
def test_int16_guard_both_sides(gpu_engine, oracle):
    for name, scores, w, _, over in guard_cases():
        got = check(gpu_engine, oracle, [w], **scores)
        assert got["status"][0] & 1, name
        if over is None:
            continue
        with pytest.raises(OverflowError):
            gpu_engine.poa_batch(batch([over]), **scores)
        # a failed call leaves no results behind, and the engine goes on
        with pytest.raises(RuntimeError, match="no POA results"):
            gpu_engine._check(gpu_engine.lib.rvn_poa_results(gpu_engine.h, None, None, None,
                                                             None, None))
        check(gpu_engine, oracle, [w] + plain_windows(52), **scores)


@gpu
def test_many_predecessors(gpu_engine, oracle):
    fast, generic, four, cells = pred_windows()
    got = check(gpu_engine, oracle, [fast])
    assert got["cells"] == cells   # no layer added a node: every deletion became an edge
    check(gpu_engine, oracle, [generic])
    check(gpu_engine, oracle, [four, fast, generic, four], with_quality=True)
    check(gpu_engine, oracle, [fast, four], **TIE_SCORES)


@gpu
def test_dropped_layers_follow_racon(gpu_engine, oracle):
    wins, status = dropped_layer_windows()
    for q in (False, True):
        got = check(gpu_engine, oracle, wins, with_quality=q)
        assert got["status"].tolist() == status
    # the trimming threshold counts kept sequences only: nothing is trimmed
    w = wins[-2]
    off = got["cons_off"].astype(np.int64)
    assert off[-2] - off[-3] >= len(w["bb"]) - 5
    # alone as well (the all-dropped window is the backbone)
    alone = per_window(check(gpu_engine, oracle, [wins[-1]]))[0]
    assert alone == (wins[-1]["bb"], 0, [0] * len(wins[-1]["bb"]))


@gpu
def test_ties_and_weights(gpu_engine, oracle):
    for name, wins, q in quality_variants(tie_windows()):
        for kw in ({}, dict(trim=False), dict(tgs=False), TIE_SCORES):
            check(gpu_engine, oracle, wins, with_quality=q, **kw)
    # equal begins in two arrival orders: each equals the oracle on its own order
    got = per_window(check(gpu_engine, oracle, tie_windows()[-2:]))
    assert len(got) == 2
    check(gpu_engine, oracle, [heavy_window()], with_quality=True)


@gpu
def test_chimeric_bit(gpu_engine, oracle):
    wins, status = chimeric_windows()
    got = check(gpu_engine, oracle, wins)
    assert got["status"].tolist() == status
    off = got["cons_off"].astype(np.int64)
    assert off[3] - off[2] == 2    # trimmed to the two covered positions
    got = check(gpu_engine, oracle, wins, trim=False)
    assert got["status"].tolist() == [1, 1, 1]


@gpu
def test_letters(gpu_engine, oracle):
    """Upper-case ACGT only.  racon never passes anything else; the oracle would
    give every other byte a column letter of its own (test_oracle_keeps_letter_case)."""
    (w, _, _), layer = anchor_windows()
    for ch in b"NacgtUu-":
        for seq, at in ((0, 0), (0, 39), (1, 0), (2, 17), (3, 39)):
            b = batch([w] + plain_windows(3, n=1))
            b["bases"][int(b["seq_off"][seq]) + at] = ch
            with pytest.raises(ValueError):
                gpu_engine.poa_batch(b)
    still_usable(gpu_engine, oracle)


@gpu
def test_limits_are_clean_errors(gpu_engine, oracle):
    rng = np.random.default_rng(7)
    bb = rand_seq(rng, 10)
    ok = plain_windows(8, n=1)
    # layers: 4,095 pass, 4,096 are over the limit - and reported as that limit
    many = window(bb, [(bb[3:5], 3, 4)] * (MAX_LAYERS + 1))
    with pytest.raises(OverflowError, match="4095 layers"):
        gpu_engine.poa_batch(batch(ok + [many]))
    still_usable(gpu_engine, oracle)
    # dropped layers do not count
    many["layers"][7] = (b"", 3, 4, None)
    got = check(gpu_engine, oracle, [many])
    assert got["status"][0] == 1
    # bases of a window
    full = window(rand_seq(rng, 500), [(rand_seq(rng, 500), 0, 499)] * 129)
    assert _dims(full)[2] == MAX_WINDOW_BASES
    over = window(full["bb"] + b"A", full["layers"])
    with pytest.raises(OverflowError, match="65000 bases"):
        gpu_engine.poa_batch(batch([over] + ok))
    # bases of a layer
    long_layer = window(bb, [(bb, 0, 9), (rand_seq(rng, MAX_LAYER_BASES + 1), 0, 9)])
    assert _dims(long_layer)[2] < MAX_WINDOW_BASES
    with pytest.raises(OverflowError, match="32000 bases"):
        gpu_engine.poa_batch(batch([long_layer]))
    still_usable(gpu_engine, oracle)
    # coordinates: end < backbone length is the documented contract
    for lo, hi in ((0, 10), (5, 4), (3, 11)):
        bad = window(bb, [(bb, 0, 9), (bb, lo, hi)])
        with pytest.raises(ValueError, match="begin and end"):
            gpu_engine.poa_batch(batch(ok + [bad]))
    with pytest.raises(ValueError):
        gpu_engine.poa_batch(batch(ok), g=0)
    still_usable(gpu_engine, oracle)


# ---------------------------------------------------------------------------
# without a GPU
# ---------------------------------------------------------------------------
def test_routes_sit_on_their_edges():
    """Every builder asserts the route of its windows; build them all.  Together:
    fast, generic, tier-1 retry, fast group on the generic kernel, both sides of the
    int16 guard, a node with more than 64 in-edges, full graph and sub-graph."""
    names = [n for n, _, _, _ in all_oracle_batches()]
    assert len(names) == len(set(names))
    fallback_windows()
    assert sum(over is not None for *_, over in guard_cases()) >= 7
    wins, _ = lane_windows()
    assert {route([w]).popitem()[1]["kernel"] for w in wins} == {"fast", "generic"}
    assert graph_windows()[1] > 0


def _oracle_run(oracle, wins, q, simd, **kw):
    oracle.lib.orc_spoa_use_simd(int(simd))
    try:
        return oracle.poa_batch(batch(wins, q), threads=8, **kw)
    finally:
        oracle.lib.orc_spoa_use_simd(0)


def test_oracle_simd_fill_equals_scalar_on_edge_windows(oracle):
    """The oracle's AVX2 int16 fill against its scalar int32 fill on every window of
    this file, the int16 extremes included."""
    for name, wins, q, kw in all_oracle_batches():
        a = _oracle_run(oracle, wins, q, False, **kw)
        b = _oracle_run(oracle, wins, q, True, **kw)
        for k in KEYS + ("cells",):
            assert np.array_equal(a[k], b[k]), (name, k)


def test_guard_rows_are_what_the_cases_assume(oracle):
    """cells = sum of (rows + 1) * (len + 1) over the layers: the oracle's count pins
    the graph sizes the guard cases and the tier cases are built on."""
    for name, scores, w, rows, _ in guard_cases():
        got = _oracle_run(oracle, [w], False, False, **scores)
        want = sum((r + 1) * (len(l[0]) + 1) for r, l in zip(rows, w["layers"]))
        assert int(got["cells"][0]) == want, name
    for scores, w, (height, width) in simd_limit_cases():
        got = _oracle_run(oracle, [w], False, True, **scores)
        first = (len(w["bb"]) + 1) * (len(w["layers"][0][0]) + 1)
        assert int(got["cells"][0]) == first + height * width
    # the divergent windows outgrow tier 0: their mean graph is already beyond it
    for (plain, big), kw in ((tier_windows(), {}), (fallback_windows(), TIE_SCORES)):
        got = _oracle_run(oracle, [big], False, False, **kw)
        n, length = len(big["layers"]), len(big["layers"][0][0])
        mean_rows = int(got["cells"][0]) / (length + 1) / n - 1
        assert mean_rows > route(plain + [big])["fast"]["ncap"]
    fast, _, _, cells = pred_windows()
    assert int(_oracle_run(oracle, [fast], False, False)["cells"][0]) == cells


def test_hand_computed_consensus(oracle):
    (three, one, none), layer = anchor_windows()
    got = per_window(_oracle_run(oracle, [three, one, none], False, False))
    # three equal layers outvote the backbone (weight 0); every consensus base is on
    # the path of the three layers, and of the backbone through its column
    assert got[0] == (layer, 1, [4] * 40)
    # fewer than three sequences: the backbone, unpolished, no coverage
    assert got[1] == (three["bb"], 0, [0] * 40)
    assert got[2] == (three["bb"], 0, [0] * 40)
    # the chimeric cases, from the coverage rule alone
    wins, status = chimeric_windows()
    res = _oracle_run(oracle, wins, False, False)
    assert res["status"].tolist() == status
    assert per_window(res)[2][0] == wins[2]["bb"][50:52]


def test_oracle_keeps_letter_case(oracle):
    """Why rvn_poa_batch rejects lower case and U: spoa codes letters as they come,
    so 'a' is a letter of its own that mismatches 'A' and is printed as 'a'."""
    (three, _, _), layer = anchor_windows()
    low = window(three["bb"], [(layer.lower(), 0, 39)] * 3)
    got = per_window(_oracle_run(oracle, [low], False, False))[0]
    assert got[0] == layer.lower()
