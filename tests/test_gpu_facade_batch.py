"""GPU: the ram::MinimizerEngine facade answers per-read Map calls from one batched
device map of every resident read. Its results must equal the CPU oracle's per-read
Map, and its counters show which path ran.

Two drivers:
- tests/cpp/facade_batch (product only) replays a Minimize / Filter / Map schedule,
  with several index batches per pass and the cases that must leave the batch
  (reverse-complemented views, reads never minimized, reads changed after Minimize).
- oracle/_ref/facade_batch_test (recipe oracle/facade_batch.mk) runs the reference's
  own construct.cc stages over the facade.
build() compiles both."""
import os
import struct
import subprocess

import numpy as np
import pytest

from raven_b200 import seqio, synth

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
DRIVER = os.path.join(HERE, "cpp", "_build", "facade_batch")
REF_DRIVER = os.path.join(os.path.dirname(HERE), "oracle", "_ref", "facade_batch_test")


def write_vec(f, a):
    f.write(struct.pack("<Q", a.size))
    f.write(np.ascontiguousarray(a).tobytes())


def read_vec(f, dt):
    (n,) = struct.unpack("<Q", f.read(8))
    return np.frombuffer(f.read(n * np.dtype(dt).itemsize), dtype=dt).copy()


def write_reads(path, rs):
    with open(path, "wb") as f:
        write_vec(f, rs.words.astype(np.uint64))
        write_vec(f, rs.word_off.astype(np.uint64))
        write_vec(f, rs.lens.astype(np.uint32))


class Schedule:
    """A script for the driver and its replay on the CPU oracle."""

    def __init__(self, rs):
        self.codes = [rs.codes(i) for i in range(rs.n)]
        self.lines = []

    def minimize(self, first, last, minhash):
        self.lines.append(("minimize", first, last, int(minhash)))

    def filter(self, freq):
        self.lines.append(("filter", freq))

    def map(self, i, ae, as_, mh, wf, rc=False):
        self.lines.append(("map_rc" if rc else "map", i, int(ae), int(as_), int(mh), int(wf)))

    def mutate(self, i, src):
        self.lines.append(("mutate", i, src))

    def reset(self, i):
        self.lines.append(("reset", i))

    def counters(self, batch_maps, served, single_maps):
        self.lines.append(("counters", batch_maps, served, single_maps))

    def run(self, tmp_path, oracle, k=15, w=5, threads=4):
        if not os.path.exists(DRIVER):
            pytest.skip("tests/cpp/_build/facade_batch not built")
        rs = seqio.pack_codes(self.codes)
        inp, script, out = (str(tmp_path / n) for n in ("reads.bin", "script.txt", "out.bin"))
        write_reads(inp, rs)
        with open(script, "w") as f:
            for op, *args in self.lines:
                if op == "counters":
                    args = []
                f.write(" ".join(str(a) for a in (op, *args)) + "\n")
        subprocess.run([DRIVER, inp, script, out, str(k), str(w), str(threads)], check=True,
                       timeout=600)
        codes = list(self.codes)
        eng = oracle.engine(k, w, threads=4)
        reads = oracle.reads(rs)
        n_maps = 0
        with open(out, "rb") as f:
            for op, *args in self.lines:
                if op == "minimize":
                    oracle.minimize(eng, reads, *args[:2], bool(args[2]))
                elif op == "filter":
                    oracle.filter(eng, args[0])
                elif op == "mutate":
                    codes[args[0]] = codes[args[1]]
                    reads = oracle.reads(seqio.pack_codes(codes))
                elif op == "counters":
                    got = read_vec(f, np.uint64)
                    assert got.tolist() == args, ("counters after", n_maps, "maps")
                elif op in ("map", "map_rc"):
                    i, ae, as_, mh, wf = args
                    q = reads
                    if op == "map_rc":
                        view = list(codes)
                        view[i] = (3 - codes[i])[::-1]
                        q = oracle.reads(seqio.pack_codes(view))
                    want = oracle.map(eng, q, i, i + 1, bool(ae), bool(as_), bool(mh))
                    ovl = read_vec(f, np.uint32).reshape(-1, 8)
                    filt = read_vec(f, np.uint32)
                    assert np.array_equal(ovl, want["overlaps"]), (op, *args)
                    assert np.array_equal(filt, want["filtered"] if wf else filt[:0]), (op, *args)
                    n_maps += 1
            assert f.read() == b""


def batches(rs, batch_bases):
    """Index batches [j, i + 1) of construct.cc:32-43 with a threshold of batch_bases."""
    out, bases, j = [], 0, 0
    for i in range(rs.n):
        bases += int(rs.lens[i])
        if i != rs.n - 1 and bases < batch_bases:
            continue
        out.append((j, i + 1))
        bases, j = 0, i + 1
    return out


@pytest.fixture(scope="module")
def reads():
    return synth.make_reads(genome_len=80_000, n_reads=160, mean_len=3000, seed=21)


@pytest.mark.parametrize("threads", [1, 16])
@pytest.mark.parametrize("stage", ["overlaps", "repeats"])
def test_pass_of_index_batches(tmp_path, oracle, reads, stage, threads):
    """construct.cc:32-70 (stage 1: minhash maps) and :354-381 (stage 2: filtered
    positions) with index batches small enough for four batches: one device map for
    the first batch, two for each later one, every Map call served."""
    bs = batches(reads, int(reads.lens.sum()) // 4)
    assert len(bs) >= 3
    s = Schedule(reads)
    maps = served = 0
    for j, last in bs:
        s.minimize(j, last, stage == "overlaps")
        s.filter(0.001)
        for k in range(last):
            if stage == "overlaps":
                s.map(k, True, True, True, False)
            else:
                s.map(k, True, True, False, True)
        maps += 1 if j == 0 else 2
        served += last
        s.counters(maps, served, 0)
    s.run(tmp_path, oracle, threads=threads)


def test_reads_that_leave_the_batch(tmp_path, oracle, reads):
    s = Schedule(reads)
    a, b = 60, 110
    s.minimize(0, a, False)
    s.filter(0.001)
    for k in (5, 0, 59, 5):                     # the same read twice: one device map
        s.map(k, True, True, False, True)
    s.counters(1, 4, 0)
    s.filter(0.01)                              # another threshold: a new device map
    s.map(5, True, True, False, True)
    s.counters(2, 5, 0)
    for _ in range(2):                          # flag sets alternating on one read
        s.map(7, True, True, False, False)
        s.map(7, False, False, False, True)
        s.map(7, True, False, True, False)
    s.counters(5, 11, 0)
    s.map(8, False, False, False, False, rc=True)  # a reverse-complemented view
    s.map(a + 3, True, True, False, True)       # a read never minimized
    s.counters(5, 11, 2)
    s.mutate(9, 140)                            # new bases after Minimize: not stale
    s.map(9, True, True, False, True)
    s.map(10, True, True, False, True)
    s.counters(5, 12, 3)
    s.minimize(a, b, False)                     # continues the pass
    s.filter(0.001)
    s.map(0, True, True, False, False)
    s.map(9, True, True, False, False)          # (its kept copy has the old bases)
    s.map(a, True, True, False, False)
    s.counters(7, 14, 4)
    s.minimize(b + 5, 150, True)                # not after the last range: a new pass
    s.filter(0.001)
    s.map(0, True, True, True, False)
    s.map(b + 5, True, True, True, False)
    s.counters(8, 15, 5)
    s.minimize(0, 40, False)                    # the salvage pattern (assemble.cc:754-763)
    s.filter(0.001)
    for k in range(40):
        s.map(k, True, True, False, False)
        s.reset(k)
    s.counters(9, 55, 5)
    s.run(tmp_path, oracle)


def run_reference(tmp_path, rs, minhash, threads):
    if not os.path.exists(REF_DRIVER):
        pytest.skip("oracle/_ref/facade_batch_test not built (needs the reference tree at build time)")
    inp, out = str(tmp_path / "reads.bin"), str(tmp_path / "out.bin")
    write_reads(inp, rs)
    subprocess.run([REF_DRIVER, inp, out, "15", "5", "0.001", str(int(minhash)), str(threads)],
                   check=True, stderr=subprocess.DEVNULL, timeout=900)
    stage2 = lambda f: dict(overlaps=read_vec(f, np.uint32), ovl_off=read_vec(f, np.uint64),
                            piles=read_vec(f, np.uint32), order=read_vec(f, np.uint32))
    with open(out, "rb") as f:
        s1 = dict(overlaps=read_vec(f, np.uint32).reshape(-1, 8), ovl_off=read_vec(f, np.uint64),
                  pile=read_vec(f, np.uint16), pile_off=read_vec(f, np.uint64))
        c1 = read_vec(f, np.uint64).tolist()
        s2 = stage2(f)
        c2 = read_vec(f, np.uint64).tolist()
        (valid,) = read_vec(f, np.uint64).tolist()
        s2_batched = stage2(f)
        assert f.read() == b""
    return s1, c1, s2, c2, valid, s2_batched


@pytest.mark.parametrize("threads", [1, 16])
@pytest.mark.parametrize("data,minhash", [("lambda", False), ("lambda", True),
                                          ("synthetic", False)])
def test_reference_stages_over_facade(tmp_path, oracle, lambda_reads, data, minhash, threads):
    """raven::FindOverlapsAndCreatePiles, then raven::FindOverlapsAndRepetetiveRegions,
    over the facade: stage 1 equals the CPU oracle, stage 2 equals the batched
    replacements, and each stage is one device map with every Map call served."""
    rs = lambda_reads if data == "lambda" else synth.make_reads(40_000, 150, 3000, seed=13)
    s1, c1, s2, c2, valid, s2_batched = run_reference(tmp_path, rs, minhash, threads)
    want = oracle.stage1(oracle.engine(15, 5, threads=4), oracle.reads(rs), 0.001, 32, minhash)
    for key in ("overlaps", "ovl_off", "pile", "pile_off"):
        assert np.array_equal(s1[key], want[key]), key
    assert c1 == [1, rs.n, 0]
    # (stage 2 maps nothing when no read is invalid, construct.cc:343-349)
    assert c2 == ([2, rs.n + valid, 0] if valid < rs.n else c1)
    for key in s2:
        assert np.array_equal(s2[key], s2_batched[key]), key
