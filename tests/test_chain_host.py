"""ram's per-band chain rules have one copy, raven_b200/csrc/chain.cuh, which every
chain kernel calls. Here that header, compiled for the host, chains one (rhs, strand)
pair with ChainPairSerial (what GroupChainKernel runs per thread) and is compared
with ram's Chain in the oracle, overlap for overlap in emission order."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
U64P = C.POINTER(C.c_uint64)
U32P = C.POINTER(C.c_uint32)

DEFAULT = dict(k=15, w=5, bandwidth=500, chain=4, matches=100, gap=10000)
HIFI = dict(DEFAULT, k=19, w=10)
TIGHT = dict(DEFAULT, bandwidth=200, chain=3, matches=60, gap=2000)
PARAMS = [pytest.param(DEFAULT, id="default"), pytest.param(HIFI, id="hifi"),
          pytest.param(TIGHT, id="bw200-chain3-matches60-gap2000")]


def encode(rhs_id, strand, lpos, rpos):
    """Seed hits as seed.cuh's EncodeHit writes them: (group, positions)."""
    lpos = np.asarray(lpos, np.uint64)
    rpos = np.asarray(rpos, np.uint64)
    diag = rpos - lpos + np.uint64(3 << 30) if strand else rpos + lpos
    group = (np.uint64((rhs_id << 1) | int(strand)) << np.uint64(32)) | diag
    return group, (lpos << np.uint64(32)) | rpos


def diagonal_run(lpos, strand, diag, walk=0):
    """Hits at lhs positions lpos along one diagonal, rhs positions off by `walk`."""
    lpos = np.asarray(lpos, np.int64)
    rpos = (lpos + diag if strand else diag - lpos) + walk
    assert (rpos >= 0).all() and (rpos < 1 << 28).all()
    return lpos, rpos


def make_pair(rng, m, strand, rhs_id=7, runs=1, spread=0, noise=0.2, step=40, jitter=2):
    """m distinct hits of one pair: `runs` overlap-like runs with indel jitter, on
    diagonals `spread` apart, and a `noise` share of random hits. Shuffled."""
    n_true = m - int(m * noise)
    ls, rs = [], []
    for i, k in enumerate(np.diff(np.linspace(0, n_true, runs + 1).astype(int))):
        lp = 1000 + 3000 * i + np.cumsum(rng.integers(1, step + 1, k))
        walk = np.cumsum(rng.integers(-jitter, jitter + 1, k))
        l, r = diagonal_run(lp, strand, (50_000 if strand else 10_000_000) + i * spread, walk)
        ls.append(l)
        rs.append(r)
    keys = set(zip(np.concatenate(ls).tolist(), np.concatenate(rs).tolist()))
    while len(keys) < m:
        keys.add((int(rng.integers(0, 1 << 20)), int(rng.integers(0, 1 << 24))))
    keys = np.array(sorted(keys), np.int64)[:m]
    keys = keys[rng.permutation(len(keys))]
    return encode(rhs_id, strand, keys[:, 0], keys[:, 1])


@pytest.fixture(scope="module")
def ours():
    so = os.path.join(HERE, "_chain_host.so")
    src = os.path.join(HERE, "chain_host.cpp")
    hdrs = [os.path.join(HERE, "..", "raven_b200", "csrc", "chain.cuh"),
            os.path.join(HERE, "..", "include", "raven_b200.h")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(map(os.path.getmtime, [src] + hdrs)):
        subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++",
                        src, "-o", so], check=True)
    lib = C.CDLL(so)
    lib.rvn_test_chain_pair.restype = C.c_uint64
    lib.rvn_test_chain_pair.argtypes = [U64P, U64P, C.c_uint32, C.c_uint32, U32P, U32P,
                                        C.c_uint64]
    return lib


def check(ours, oracle, prm, group, positions, lhs_id=3):
    g = np.ascontiguousarray(group, np.uint64)
    p = np.ascontiguousarray(positions, np.uint64)
    cp = np.array([prm[n] for n in ("k", "bandwidth", "chain", "matches", "gap")], np.uint32)
    cap = g.size + 1
    out = np.zeros((cap, 8), np.uint32)
    n = ours.rvn_test_chain_pair(g.ctypes.data_as(U64P), p.ctypes.data_as(U64P), g.size, lhs_id,
                                 cp.ctypes.data_as(U32P), out.ctypes.data_as(U32P), cap)
    want = oracle.chain(oracle.engine(**prm), lhs_id, g, p)
    assert np.array_equal(out[:n], want)
    return n


@pytest.mark.parametrize("strand", [0, 1])
@pytest.mark.parametrize("prm", PARAMS)
def test_pairs_equal_ram(ours, oracle, prm, strand):
    rng = np.random.default_rng(17 + strand)
    bw = prm["bandwidth"]
    found = 0
    for m in (4, 5, 8, 9, 17, 33, 48, 49, 100, 300, 1000, 2500, 6000):
        for runs, spread in ((1, 0), (2, bw // 2), (2, bw), (2, bw + 1), (3, bw - 3), (3, 2 * bw)):
            for noise in (0.0, 0.3):
                found += check(ours, oracle, prm,
                               *make_pair(rng, m, strand, runs=runs, spread=spread, noise=noise))
    assert found > 100


@pytest.mark.parametrize("strand", [0, 1])
@pytest.mark.parametrize("prm", PARAMS)
def test_gap_edges(ours, oracle, prm, strand):
    """A chain whose lhs positions jump by exactly `gap` stays whole; by gap + 1 it
    is cut in two."""
    d = 50_000 if strand else 10_000_000
    counts = []
    for jump in (prm["gap"], prm["gap"] + 1):
        lp = np.r_[np.arange(0, 400, 10), 390 + jump + np.arange(0, 400, 10)] + 1000
        counts.append(check(ours, oracle, prm, *encode(5, strand, *diagonal_run(lp, strand, d))))
    assert counts == [1, 2]


@pytest.mark.parametrize("strand", [0, 1])
@pytest.mark.parametrize("prm", PARAMS)
def test_matches_edge(ours, oracle, prm, strand):
    """Covered bases of exactly `matches` give an overlap, one fewer gives none."""
    d = 50_000 if strand else 10_000_000
    counts = []
    for span in (prm["matches"] - prm["k"], prm["matches"] - prm["k"] - 1):
        lp = np.unique(np.r_[np.arange(0, span, 7), span]) + 2000
        counts.append(check(ours, oracle, prm, *encode(5, strand, *diagonal_run(lp, strand, d))))
    assert counts == [1, 0]
