"""Alignment paths and window breaking points (alnpath.cu, rvn_align_breaking_points)
at their edges: pairs built on purpose for the tie rules, the leaf / Hirschberg
boundary, the split-row fallbacks, every column-kernel route, the distance rounds,
the window cuts and the leaf chunking, each compared with the oracle's plain banded
dynamic programme plus edlib's two rules (oracle/nw_path.cpp, orc_nw_path) and with
the product's host edlib (raven_b200/host/edlib.cc).

A host mirror (`plan`) restates AlignBreakingPoints' arithmetic: the prefix estimate,
the band of every distance round, the ring and route of every column task, the leaf
rule and the leaf chunks. The unmarked test asserts that every case sits on the
intended side of its edge; the GPU tests compare the kernels' output with the
oracle, group by group and all groups in one call."""
import numpy as np
import pytest

from raven_b200 import seqio, synth
from test_gpu_alnpath import _expected

gpu = pytest.mark.gpu

ACGT = np.frombuffer(b"ACGT", np.uint8)

# thresholds of alnpath.cu as the source has them
WARP_RING = 24           # kWarpRing: bands of this many blocks run on ColumnsWarpKernel
WARP_STEPS = 16384       # kWarpSteps: so does any task of this many block steps
SMEM_RING = 208          # kSmemRing: ColumnsKernel<true> holds rings up to this size
LEAF_BYTES = 1 << 20     # edlib's traceback data limit: leaf below, Hirschberg split above
PREFIX = 384             # kPrefix: target columns of the prefix estimate
PREFIX_BAND = 96         # kPrefixBand
LEAF_BUDGET = 1 << 29    # 8-byte words of leaf scratch per LeafKernel launch


# ---------------------------------------------------------------------------
# the host mirror
# ---------------------------------------------------------------------------
def blocks(m):
    return (m + 63) // 64


def ring_of(m, k):
    return max(1, min(blocks(m), ((2 * k) >> 6) + 2))


def ring_class(ring):
    c = 3
    while (1 << c) < ring:
        c += 1
    return c


def route(m, cols, k):
    """Kernel of one column task: 'warp' or 'thread<ring class>'."""
    r = ring_of(m, k)
    if r >= WARP_RING or cols * r >= WARP_STEPS:
        return "warp"
    return f"thread{ring_class(r)}"


def is_leaf(m, n):
    return (20 * blocks(m) + 8) * n < LEAF_BYTES


def leaf_words(m, n, score):
    cells = n * ring_of(m, score)
    return 2 * cells + (cells + 1) // 2


def last_column(q, t):
    """D[r][len(t)] for r = 0..len(q): the plain unit-cost programme, column by column."""
    rows = np.arange(len(q) + 1, dtype=np.int64)
    col = rows.copy()
    for c in t:
        nxt = np.empty_like(col)
        nxt[0] = col[0] + 1
        nxt[1:] = np.minimum(col[:-1] + (q != c), col[1:] + 1)
        col = np.minimum.accumulate(nxt - rows) + rows   # vertical steps
    return col


def prefix_estimate(q, t):
    """The mode-1 probe: the smallest D[r][384] if it is <= 96, else -1."""
    best = int(last_column(q[:PREFIX + PREFIX_BAND + 1], t[:PREFIX]).min())
    return best if best <= PREFIX_BAND else -1


def split_row(q, t, best):
    """edlib's Hirschberg split of (q, t): column |t|/2, smallest row in 1..|q|-1 on
    an optimal path, then 0, then |q|."""
    m, half = len(q), len(t) // 2
    fw = last_column(q, t[:half])
    bw = last_column(q[::-1], t[half:][::-1])[::-1]   # bw[r]: q[r:] against t[half:]
    hit = np.flatnonzero(fw + bw == best)
    inner = hit[(hit >= 1) & (hit <= m - 1)]
    if inner.size:
        return int(inner[0])
    return 0 if fw[0] + bw[0] == best else m


def plan(q, t, d):
    """What AlignBreakingPoints does with one pair of distance d at the top level."""
    m, n = len(q), len(t)
    p = dict(m=m, n=n, probe=m >= 4 * PREFIX and n >= 4 * PREFIX, est=None)
    kk = max(64, abs(m - n))
    if p["probe"]:
        p["est"] = prefix_estimate(q, t)
        longest = max(m, n)
        kk = max(kk, (longest * p["est"] * 5 // 4) // PREFIX + 48 if p["est"] >= 0
                 else longest // 4)
    p["rounds"] = []
    while True:
        k = min(kk, m + n)
        p["rounds"].append(k)
        if d <= k:
            break
        kk *= 2
    k0 = p["rounds"][0]
    p["ring"], p["steps"], p["route"] = ring_of(m, k0), n * ring_of(m, k0), route(m, n, k0)
    p["routes"] = {route(m, n, k) for k in p["rounds"]}
    p["root"] = "leaf" if is_leaf(m, n) else "split"
    if p["root"] == "split":
        p["routes"] |= {route(m, n // 2, d), route(m, n - n // 2, d)}
        p["root_route"] = route(m, n // 2, d)
    return p


def leaf_chunks(leaves):
    """LeafKernel launches for leaves (m, n, score): largest first, 2^29 words each."""
    sizes = sorted((n * ring_of(m, s), leaf_words(m, n, s)) for m, n, s in leaves)[::-1]
    chunks, used = [], None
    for _, need in sizes:
        if used is None or used + need > LEAF_BUDGET:
            chunks.append(0)
            used = 0
        used += need
        chunks[-1] += 1
    return chunks


# ---------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------
class Case:
    """One pair: oriented query q against target t (codes), the query read stored
    reverse complemented when strand == 0, both inside random flanks so that
    neither starts at a word boundary. `expect`: facts of plan() the case is for."""

    def __init__(self, group, name, q, t, strand, t_begin, expect=None, d=None,
                 copies=1, split_row=None):
        self.group, self.name = group, name
        self.q = np.ascontiguousarray(q, dtype=np.uint8)
        self.t = np.ascontiguousarray(t, dtype=np.uint8)
        self.strand, self.t_begin = strand, t_begin
        self.expect = expect or {}
        self.d = d                # distance by construction, when it is known
        self.copies = copies
        self.split_row = split_row

    def __repr__(self):
        return f"{self.group}/{self.name}"


def rand(rng, n):
    return rng.integers(0, 4, n, dtype=np.uint8)


def errs(rng, s, e):
    return np.asarray(synth.mutate(s, rng, e / 3, e / 3, e / 3), dtype=np.uint8)


def fit(rng, s, n):
    """s cut or padded with random bases to exactly n."""
    return s[:n] if len(s) >= n else np.concatenate([s, rand(rng, n - len(s))])


def subs(rng, s, d):
    """d substitutions spread evenly."""
    s = s.copy()
    pos = np.linspace(5, len(s) - 6, d).astype(np.int64)
    s[pos] = (s[pos] + rng.integers(1, 4, d, dtype=np.uint8)) & 3
    return s


def ties(rng):
    runs = np.repeat(rand(rng, 700), rng.integers(1, 9, 700))   # homopolymer runs
    ac = np.tile(np.array([0, 1], np.uint8), 1500)
    gac = np.tile(np.array([2, 0, 1], np.uint8), 4000)           # (GAC)n, 12 kb
    unit = np.tile(rand(rng, 300), 30)                            # 300-bp unit x 30
    out = [Case("ties", "homopolymer runs", errs(rng, runs, 0.15), errs(rng, runs, 0.02), 1, 37),
           Case("ties", "(AC)n", errs(rng, ac, 0.12), ac, 0, 5),
           Case("ties", "(GAC)n 12 kb", errs(rng, gac, 0.15), gac, 1, 1001),
           Case("ties", "300-bp unit x30", errs(rng, unit, 0.18), errs(rng, unit, 0.02), 0, 77)]
    # poly-A against poly-A: every path with |m - n| gaps is optimal
    for i, (a, b) in enumerate(((200, 260), (700, 640), (64, 129), (3000, 2900), (9000, 8000))):
        out.append(Case("ties", f"polyA {a} vs {b}", np.zeros(a, np.uint8), np.zeros(b, np.uint8),
                        i % 2, 3 + 64 * i, d=abs(a - b)))
    return out


def leaf_split(rng):
    out = []
    for n in (8191, 8192):   # (20*6 + 8) * 8192 == 2^20
        t = rand(rng, n)
        root = "leaf" if n == 8191 else "split"
        out.append(Case("leaf_split", f"384 in {n}", fit(rng, errs(rng, t[3000:3390], 0.02), 384),
                        t, n % 2, 11, expect=dict(m=384, n=n, root=root)))
        out.append(Case("leaf_split", f"321 unrelated {n}", rand(rng, 321), t, 1 - n % 2, 300,
                        expect=dict(m=321, n=n, root=root)))
    for n in (1783, 1784):   # (20*29 + 8) * 1783 < 2^20 <= 588 * 1784, near the diagonal
        t = rand(rng, n)
        out.append(Case("leaf_split", f"1820 x {n}", fit(rng, errs(rng, t, 0.03), 1820), t, n % 2,
                        41, expect=dict(m=1820, n=n, root="leaf" if n == 1783 else "split")))
    return out


def fallbacks(rng):
    # a G/T query at one end of an A/C target of 40 kb (28 * n >= 2^20 from n = 37,450
    # on): no base of the query matches the rest of the target, so no inner row of
    # the middle column is on an optimal path
    q64 = rand(rng, 64) % 2 + 2
    rest = rand(rng, 40_000 - 64) % 2
    q = rand(rng, 100_000)
    return [
        Case("fallbacks", "64 at the start of 40 kb", q64, np.concatenate([q64, rest]), 1, 13,
             expect=dict(root="split", route="warp"), d=40_000 - 64, split_row=64),
        Case("fallbacks", "64 at the end of 40 kb", q64, np.concatenate([rest, q64]), 0, 13,
             expect=dict(root="split", route="warp"), d=40_000 - 64, split_row=0),
        Case("fallbacks", "100 kb query, 40-base target", q, errs(rng, q[60_000:60_040], 0.1),
             1, 9, expect=dict(root="split", route="warp")),
    ]


def deletion(rng, n, d, at=None):
    """(query, target): the target with one block of d bases removed; distance d."""
    t = rand(rng, n)
    at = (n - d) // 2 if at is None else at
    return np.concatenate([t[:at], t[at + d:]]), t


def insertion(rng, n, d):
    """(query, target): the target with d random bases inserted; distance d."""
    t = rand(rng, n)
    return np.concatenate([t[:n // 2], rand(rng, d), t[n // 2:]]), t


def columns(rng):
    out = []

    def add(name, qt, strand, **expect):
        q, t = qt
        out.append(Case("columns", name, q, t, strand, 19 + len(out), d=abs(len(q) - len(t)),
                        expect=expect))

    add("ring 1", deletion(rng, 150, 100), 1, ring=1, route="thread3")
    add("ring 8", deletion(rng, 1200, 200), 0, ring=8, route="thread3")
    add("ring 9", deletion(rng, 1240, 240), 1, ring=9, route="thread4")
    add("ring 16", insertion(rng, 600, 460), 0, ring=16, route="thread4")
    add("ring 17", insertion(rng, 600, 490), 1, ring=17, route="thread5")
    add("ring 23", insertion(rng, 712, 760), 0, ring=23, route="thread5", steps=16376)
    add("ring 24", insertion(rng, 660, 840), 1, ring=24, route="warp", steps=15840)
    add("steps 16383", deletion(rng, 5461, 5461 - 150), 0, ring=3, steps=16383, route="thread3")
    add("steps 16386", deletion(rng, 5462, 5462 - 150), 1, ring=3, steps=16386, route="warp")
    add("steps 16380", deletion(rng, 4095, 4095 - 200), 0, ring=4, steps=16380, route="thread3")
    add("steps 16384", deletion(rng, 4096, 4096 - 200), 1, ring=4, steps=16384, route="warp")
    # warp kernel: one full strip of 32 blocks, a partial last strip, two and three strips
    for m in (2048, 2049, 4096, 4097):
        t = rand(rng, m + 30)
        out.append(Case("columns", f"warp m={m}", fit(rng, errs(rng, t, 0.1), m), t, m % 2,
                        100 + m, expect=dict(m=m, route="warp", probe=True)))
        q, t = deletion(rng, m + 800, 800, at=1000)
        out.append(Case("columns", f"warp m={m} wide ring", q, t, 1 - m % 2, 3, d=800,
                        expect=dict(m=m, route="warp", rounds=[800])))
    # near the diagonal at low error: the Hirschberg columns run one thread per problem
    t = rand(rng, 4000)
    out.append(Case("columns", "split on threads", subs(rng, t, 200), t, 1, 21, d=200,
                    expect=dict(root="split", root_route="thread3")))
    return out


def rounds(rng):
    out = []
    for d, want in ((64, [64]), (65, [64, 128]), (128, [64, 128]), (129, [64, 128, 256])):
        t = rand(rng, 1500)
        out.append(Case("rounds", f"distance {d}", subs(rng, t, d), t, d % 2, 29 + d, d=d,
                        expect=dict(rounds=want, probe=False)))
    clean = rand(rng, 400)
    out.append(Case("rounds", "clean prefix, unrelated tail",
                    np.concatenate([clean, rand(rng, 2600)]), np.concatenate([clean, rand(rng, 2600)]),
                    0, 7, expect=dict(est=0, rounds=[64, 128, 256, 512, 1024, 2048])))
    rest = rand(rng, 3000)
    out.append(Case("rounds", "unrelated prefix, clean rest",
                    np.concatenate([rand(rng, 400), fit(rng, errs(rng, rest, 0.05), 3000)]),
                    np.concatenate([rand(rng, 400), rest]), 1, 99, expect=dict(est=-1, rounds=[850])))
    out.append(Case("rounds", "band clamped to m+t", rand(rng, 20), rand(rng, 30), 0, 1,
                    expect=dict(rounds=[50])))
    # G/T against A/C: no base matches, distance max(m, n) > |m - n|
    out.append(Case("rounds", "doubling clamped to m+t", rand(rng, 40) % 2 + 2, rand(rng, 1000) % 2,
                    1, 3, d=1000, expect=dict(rounds=[960, 1040])))
    return out


def windows(rng):
    out = []
    for tb in (499, 500, 501):
        t = rand(rng, 1200)
        out.append(Case("windows", f"t_begin {tb}", errs(rng, t, 0.1), t, tb % 2, tb))
    t = rand(rng, 700)
    out.append(Case("windows", "query ends early", errs(rng, t[:300], 0.05), t, 1, 250))
    return out


def leaf_chunks_case(rng):
    """Enough copies of one leaf that their scratch exceeds one launch's budget."""
    t = rand(rng, 8191)
    q = rand(rng, 384)
    return Case("leaf_chunks", "384 x 8191 unrelated", q, t, 0, 45,
                expect=dict(m=384, n=8191, root="leaf", route="warp"))


GROUPS = {"ties": ties, "leaf_split": leaf_split, "fallbacks": fallbacks, "columns": columns,
          "rounds": rounds, "windows": windows}


def build_cases():
    out = []
    for i, (name, make) in enumerate(GROUPS.items()):
        out += make(np.random.default_rng(100 + i))
    return out


def chunk_copies(d):
    """Copies of the leaf-chunk case that need two LeafKernel launches by themselves."""
    return LEAF_BUDGET // leaf_words(384, 8191, d) + 32


# ---------------------------------------------------------------------------
# references
# ---------------------------------------------------------------------------
def oracle_path(oracle, q, t):
    """orc_nw_path as edlib operation codes (0 match, 1 insert, 2 delete)."""
    import ctypes as C
    oracle.lib.orc_nw_path.restype = C.c_int64
    oracle.lib.orc_nw_path.argtypes = [C.c_char_p, C.c_int, C.c_char_p, C.c_int, C.c_char_p]
    sq, st = ACGT[q].tobytes(), ACGT[t].tobytes()
    buf = C.create_string_buffer(len(sq) + len(st) + 1)
    ln = oracle.lib.orc_nw_path(sq, len(sq), st, len(st), buf)
    return buf.raw[:ln].translate(bytes.maketrans(b"MID", bytes([0, 1, 2])))


def path_cost(path, q, t):
    ops = np.frombuffer(path, np.uint8)
    assert int((ops != 2).sum()) == len(q) and int((ops != 1).sum()) == len(t)
    qi = np.cumsum(ops != 2)[ops == 0] - 1
    ti = np.cumsum(ops != 1)[ops == 0] - 1
    return int((ops != 0).sum() + (q[qi] != t[ti]).sum())


@pytest.fixture(scope="module")
def refs(oracle):
    """Per case: (distance, path) of the oracle, checked against the host edlib."""
    import test_oracle
    align = test_oracle._host_edlib()
    cases = build_cases() + [leaf_chunks_case(np.random.default_rng(7))]
    out = {}
    for c in cases:
        path = oracle_path(oracle, c.q, c.t)
        d = path_cost(path, c.q, c.t)
        hd, hpath = align(ACGT[c.q].tobytes(), ACGT[c.t].tobytes(), 2)
        assert hd == d and hpath.replace(b"\x03", b"\x00") == path, c
        if c.d is not None:
            assert d == c.d, c
        out[c.name] = (d, path)
    chunk = cases[-1]
    chunk.copies = chunk_copies(out[chunk.name][0])
    return cases, out


def upload(engine, cases):
    """Reads: per case a flanked query read and a target read; pair arrays (copies
    of a case share its reads)."""
    rng = np.random.default_rng(1)
    seqs, pairs, owner = [], [], []
    for c in cases:
        pad = int(rng.integers(1, 31)) * 2 + 1
        qs = c.q if c.strand else (3 - c.q[::-1]).astype(np.uint8)
        seqs.append(np.concatenate([rand(rng, pad), qs, rand(rng, 17)]))
        seqs.append(np.concatenate([rand(rng, c.t_begin), c.t, rand(rng, 23)]))
        for _ in range(c.copies):
            pairs.append((len(seqs) - 2, pad, len(c.q), c.strand, len(seqs) - 1, c.t_begin,
                          len(c.t)))
            owner.append(c)
    engine.configure(15, 5)
    engine.upload(seqio.pack_codes(seqs))
    return np.array(pairs, dtype=np.int64), owner


def run_and_compare(engine, cases, out, window=500):
    P, owner = upload(engine, cases)
    dist, off, bp = engine.align_breaking_points(P[:, 0], P[:, 1], P[:, 2], P[:, 3], P[:, 4],
                                                 P[:, 5], P[:, 6], window)
    want_rows = {}
    for i, c in enumerate(owner):
        d, path = out[c.name]
        assert dist[i] == d, (c, i)
        if c.name not in want_rows:
            want_rows[c.name] = _expected(path, c.t_begin, len(c.t), window)
        got = bp[int(off[i]):int(off[i + 1])]
        assert np.array_equal(got, want_rows[c.name]), (c, i, window)
    return dist, bp


# ---------------------------------------------------------------------------
# on the GPU
# ---------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("group", list(GROUPS))
def test_group_alone(gpu_engine, refs, group):
    cases, out = refs
    run_and_compare(gpu_engine, [c for c in cases if c.group == group], out)


@gpu
def test_all_groups_in_one_call(gpu_engine, refs):
    """Tasks of all groups share the cost sort, the ring classes and the leaf chunks
    of one call: the same answers as group by group."""
    cases, out = refs
    dist, bp = run_and_compare(gpu_engine, cases, out)
    # the 64-base queries leave most windows of their 40 kb target untouched
    assert (bp == 0xFFFFFFFF).all(axis=1).sum() >= 150


@gpu
@pytest.mark.parametrize("window", [1, 137, 1 << 20])
def test_windows(gpu_engine, refs, window):
    """Every target base its own window; a window larger than any target."""
    cases, out = refs
    run_and_compare(gpu_engine, [c for c in cases if c.group in ("windows", "rounds", "ties")
                                 and len(c.t) <= 12_000], out, window)


@gpu
def test_trace_shows_warp_kernel_and_leaf_chunks(gpu_engine, refs, monkeypatch, capfd):
    cases, out = refs
    monkeypatch.setenv("RVN_ALIGN_TRACE", "1")
    run_and_compare(gpu_engine, [c for c in cases if c.group in ("leaf_chunks", "columns")], out)
    err = capfd.readouterr().err
    wide = [ln for ln in err.splitlines() if "columns:" in ln and "(0 wide)" not in ln]
    chunks = [ln for ln in err.splitlines() if "leaves: chunk" in ln]
    assert wide and len(chunks) >= 2, err
    print("\n".join(wide + chunks))


# ---------------------------------------------------------------------------
# without a GPU
# ---------------------------------------------------------------------------
def test_routes_sit_on_their_edges():
    """Every case's distance, band rounds, ring, route and leaf / split root are what
    it was built for, so that both sides of every edge are reached. Two branches
    cannot be reached and are not aimed at: ColumnsKernel<false> (a task that is not
    wide has ring < 24 <= kSmemRing) and ColumnsWarpKernel's mode 1 (the prefix probe
    has band 96 over 384 columns: ring <= 5, 1920 block steps)."""
    import test_oracle
    align = test_oracle._host_edlib()
    cases = build_cases()
    chunk = leaf_chunks_case(np.random.default_rng(7))
    routes, roots = set(), set()
    for c in cases + [chunk]:
        d = align(ACGT[c.q].tobytes(), ACGT[c.t].tobytes(), 0)[0]
        if c.d is not None:
            assert d == c.d, c
        p = plan(c.q, c.t, d)
        for key, want in c.expect.items():
            assert p[key] == want, (c, key, p[key], want)
        for k in p["rounds"]:
            assert ring_of(len(c.q), k) >= WARP_RING or ring_of(len(c.q), k) < SMEM_RING
        if p["probe"]:
            assert ring_of(len(c.q), PREFIX_BAND) <= 5
            assert route(len(c.q), PREFIX, PREFIX_BAND).startswith("thread")
        if c.split_row is not None:
            assert split_row(c.q, c.t, d) == c.split_row, c
        routes |= p["routes"]
        roots.add(p["root"])
    assert {"warp", "thread3", "thread4", "thread5"} <= routes
    assert roots == {"leaf", "split"}
    # two LeafKernel launches for the copies of one leaf
    d = align(ACGT[chunk.q].tobytes(), ACGT[chunk.t].tobytes(), 0)[0]
    copies = chunk_copies(d)
    assert 4000 < copies < 5000
    assert leaf_chunks([(384, 8191, d)] * copies) == [copies - 32, 32]
