"""GPU: the radix sort and partition of raven_b200/csrc/radix.cu across PORTIONS, and the
exclusive scan of scan.cu.

A status word of the sort's decoupled look-back counts below 2^30, so an input of more
than (2^30 - 1) / tile tiles runs as several launches per pass, the last tile of each
handing the running end of every bin to the next. Engine option radix_portion_tiles
cuts portions of a few tiles, which brings that handoff to test sizes:

a. every sort instantiation with portions of 1, 2 and 3 tiles, at q * P - 1, q * P and
   q * P + 1 records, with runs of equal keys across every portion boundary, against
   numpy's stable argsort, bit exact, and the launch count of the portion rule;
b. the unstable partition with forced portions: the multiset of every bin and bin_start;
c. the exclusive scan of u32 counts into u64 offsets past 2^32 and past 1024 chunks;
d. stage 1, the index, map and the polisher's window layers with 1-tile portions,
   against the golden files and the CPU oracle;
e. (slow) the default portion plus two tiles and three records, checked on the device.
"""
import threading
import time

import numpy as np
import pytest

from raven_b200 import synth
from test_gpu_bare_counts import FREQS
from test_gpu_overlap import GOLD, META, _check_map

pytestmark = pytest.mark.gpu

TILE = {4: 8192, 8: 4096}   # records per tile by key bytes
MAX_LAUNCHES = 64           # tickets of one sort: passes * portions


@pytest.fixture(scope="module")
def eng():
    from raven_b200 import engine
    e = engine.Engine(device=0)
    yield e
    e.close()


def n_passes(begin_bit, end_bit):
    return -(-max(0, end_bit - begin_bit) // 10)


def portion_tiles(tile, tiles, passes, forced):
    """the portion rule of radix.cu (PortionTiles)"""
    cap = ((1 << 30) - 1) // tile
    want = min(forced, cap) if forced > 0 else cap
    per_pass = MAX_LAUNCHES // passes
    return min(cap, max(want, -(-tiles // per_pass)))


def sort_launches(key_bytes, n, begin_bit, end_bit, forced):
    passes = n_passes(begin_bit, end_bit)
    if n == 0 or passes == 0:
        return 0
    tile = TILE[key_bytes]
    tiles = -(-n // tile)
    return 2 + passes * -(-tiles // portion_tiles(tile, tiles, passes, forced))


def counted(eng, fn):
    """fn's result and the kernel launches it took"""
    eng.set_option("reset_stats", 1)
    out = fn()
    return out, eng.stats()["kernel_launches"]


def stable_ref(keys, vals, begin_bit, end_bit, descending):
    mask = np.uint64((1 << (end_bit - begin_bit)) - 1)
    d = (keys.astype(np.uint64) >> np.uint64(begin_bit)) & mask
    if descending:
        d = mask - d
    order = np.argsort(d, kind="stable")
    return keys[order], None if vals is None else vals[order]


def boundary_runs(keys, period, width, value):
    """a run of `value` across every multiple of `period` inside the array"""
    for b in range(period, keys.size, period):
        keys[max(0, b - width):b + width] = value
    return keys


# (key dtype, value dtype or None, begin_bit, end_bit, descending, bits drawn)
INSTANTIATIONS = {
    "u32_u64": (np.uint32, np.uint64, 0, 30, False, 32),     # the index, bits above ignored
    "u64_u64": (np.uint64, np.uint64, 0, 38, False, 40),     # k = 19: 10, 10, 9, 9 bits
    "u32_u32": (np.uint32, np.uint32, 0, 17, True, 17),      # pair sizes, descending: 9, 8
    "u64_u32": (np.uint64, np.uint32, 14, 37, False, 40),    # begin_bit > 0: 8, 8, 7 bits
    "u32_keys": (np.uint32, None, 3, 29, False, 32),         # bare keys: 9, 9, 8 bits
}


def check_sort(eng, kt, vt, keys, begin_bit, end_bit, desc, forced, rng):
    vals = None if vt is None else rng.integers(0, 1 << 31, keys.size, dtype=np.uint64).astype(vt)
    eng.set_option("radix_portion_tiles", forced)
    try:
        (gk, gv), launches = counted(
            eng, lambda: eng.debug_sort_pairs(keys, vals, begin_bit, end_bit, desc))
    finally:
        eng.set_option("radix_portion_tiles", 0)
    wk, wv = stable_ref(keys, vals, begin_bit, end_bit, desc)
    assert np.array_equal(gk, wk)
    if vt is not None:
        assert np.array_equal(gv, wv)
    assert launches == sort_launches(keys.itemsize, keys.size, begin_bit, end_bit, forced)
    return launches


@pytest.mark.parametrize("inst", list(INSTANTIATIONS))
@pytest.mark.parametrize("forced", [1, 2, 3])
@pytest.mark.parametrize("edge", [-1, 0, 1])
def test_forced_portions_match_stable_numpy(eng, inst, forced, edge):
    kt, vt, b, e, desc, bits = INSTANTIATIONS[inst]
    P = forced * TILE[np.dtype(kt).itemsize]
    n = 3 * P + edge
    rng = np.random.default_rng(forced * 10 + edge + 7)
    keys = rng.integers(0, 1 << bits, n, dtype=np.uint64).astype(kt)
    keys = boundary_runs(keys, P, 900, keys[n // 2])
    launches = check_sort(eng, kt, vt, keys, b, e, desc, forced, rng)
    # the same input in one portion: the portions above took more launches
    assert launches > sort_launches(keys.itemsize, n, b, e, 0)


@pytest.mark.parametrize("inst", list(INSTANTIATIONS))
def test_forced_portions_all_keys_equal(eng, inst):
    kt, vt, b, e, desc, _ = INSTANTIATIONS[inst]
    n = 2 * TILE[np.dtype(kt).itemsize] + 1
    rng = np.random.default_rng(5)
    check_sort(eng, kt, vt, np.full(n, 0x2B5A3F1, kt), b, e, desc, 1, rng)


@pytest.mark.parametrize("kt,vt,end_bit,tiles", [
    (np.uint64, np.uint64, 62, 41),    # 7 passes, 9 portions of 5 tiles: 63 launches
    (np.uint32, np.uint64, 30, 50),    # 3 passes, 17 portions of 3 tiles
    (np.uint32, None, 30, 64),         # 3 passes: 22 portions of 3 tiles would take 66
])
def test_launch_bound_overrides_one_tile_portions(eng, kt, vt, end_bit, tiles):
    n = (tiles - 1) * TILE[np.dtype(kt).itemsize] + 5
    passes = n_passes(0, end_bit)
    pt = portion_tiles(TILE[np.dtype(kt).itemsize], tiles, passes, 1)
    assert pt > 1 and passes * -(-tiles // pt) <= MAX_LAUNCHES
    rng = np.random.default_rng(tiles)
    keys = rng.integers(0, 1 << end_bit, n, dtype=np.uint64).astype(kt)
    keys = boundary_runs(keys, pt * TILE[np.dtype(kt).itemsize], 700, keys[1])
    check_sort(eng, kt, vt, keys, 0, end_bit, False, 1, rng)


def test_option_rejects_negative_portions(eng):
    with pytest.raises(ValueError):
        eng.set_option("radix_portion_tiles", -1)


# ---- b. the unstable partition ----

def check_partition(eng, keys, begin_bit, end_bit, forced):
    width = end_bit - begin_bit
    eng.set_option("radix_portion_tiles", forced)
    try:
        (got, start), launches = counted(
            eng, lambda: eng.debug_partition_keys(keys, begin_bit, end_bit))
    finally:
        eng.set_option("radix_portion_tiles", 0)
    digit = (keys >> np.uint32(begin_bit)) & np.uint32((1 << width) - 1)
    counts = np.bincount(digit, minlength=1024)
    want_start = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.uint32)
    assert np.array_equal(start, want_start)      # n for the digits past the bit range
    assert (start[1 << width:] == keys.size).all()
    gdigit = (got >> np.uint32(begin_bit)) & np.uint32((1 << width) - 1)
    assert (np.diff(gdigit.astype(np.int64)) >= 0).all()
    # every bin holds its keys: the same (digit, key) multiset in (digit, key) order
    assert np.array_equal(got[np.lexsort((got, gdigit))], keys[np.lexsort((keys, digit))])
    tiles = -(-keys.size // TILE[4])
    want = 0 if keys.size == 0 else 2 + -(-tiles // portion_tiles(TILE[4], tiles, 1, forced))
    assert launches == want
    return launches


@pytest.mark.parametrize("width", range(1, 11))
@pytest.mark.parametrize("begin_bit", [0, 5, 22])
def test_partition_forced_portions(eng, width, begin_bit):
    forced = 1 + (width + begin_bit) % 3
    P = forced * TILE[4]
    rng = np.random.default_rng(width * 100 + begin_bit)
    for n in (4 * P - 1, 4 * P + 1):
        keys = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
        keys = boundary_runs(keys, P, 1500, keys[7])
        assert check_partition(eng, keys, begin_bit, begin_bit + width, forced) > 3


def test_partition_edges(eng):
    rng = np.random.default_rng(3)
    check_partition(eng, np.zeros(0, np.uint32), 20, 30, 1)
    check_partition(eng, np.full(3 * TILE[4] + 2, 0xABCDEF, np.uint32), 20, 30, 1)
    # 70 portions of one tile would pass the ticket bound: 2-tile portions
    keys = rng.integers(0, 1 << 30, 70 * TILE[4], dtype=np.uint64).astype(np.uint32)
    assert check_partition(eng, keys, 20, 30, 1) == 2 + 35


# ---- c. the exclusive scan ----

CHUNK = 4096  # counts per CTA of ScanChunkSums; ScanOfSums takes 1024 chunk sums a round


@pytest.mark.parametrize("n", [0, 1, CHUNK - 1, CHUNK, CHUNK + 1, CHUNK * 1024 - 1,
                               CHUNK * 1024, CHUNK * 1024 + 1, CHUNK * 3000 + 7])
def test_exclusive_scan_past_2_32(eng, n):
    rng = np.random.default_rng(n % 1009)
    vals = (np.uint64(0xFFFFFFFF) - rng.integers(0, 16, n, dtype=np.uint64)).astype(np.uint32)
    if n > 10:
        vals[rng.integers(0, n, n // 7)] = rng.integers(0, 1 << 32, n // 7, dtype=np.uint64)
    got = eng.debug_exclusive_scan(vals)
    want = np.concatenate([np.zeros(1, np.uint64), np.cumsum(vals, dtype=np.uint64)])
    assert got.dtype == np.uint64 and np.array_equal(got, want)
    if n > 1:
        assert got[-1] > np.uint64(1 << 32)


# ---- d. the pipeline with 1-tile portions ----

def both_ways(eng, fn):
    """fn with the default portions and with 1-tile portions: both results, and the
    launches of the second are more (the portions ran)"""
    off, n_off = counted(eng, fn)
    eng.set_option("radix_portion_tiles", 1)
    try:
        on, n_on = counted(eng, fn)
    finally:
        eng.set_option("radix_portion_tiles", 0)
    assert n_on > n_off, (n_on, n_off)
    return off, on


STAGE1_KEYS = ("overlaps", "ovl_off", "pile", "pile_off")


@pytest.mark.parametrize("minhash", [False, True])
def test_stage1_lambda_golden(eng, lambda_reads, minhash):
    eng.configure(k=15, w=5)
    eng.upload(lambda_reads)
    _, got = both_ways(eng, lambda: eng.find_overlaps_and_create_piles(0.001, 32, minhash))
    tag = "minhash" if minhash else "plain"
    for k in STAGE1_KEYS:
        assert np.array_equal(got[k], GOLD[f"stage1_{tag}_{k}"]), k
    assert got["num_mapped"] == META[f"stage1_{tag}_num_mapped"]


def test_stage1_multi_batch_schedule(eng, oracle):
    """three index batches and eight query flushes; with minhash the index of a batch
    holds its micromizers only: some 27 000 records, still four tiles"""
    rs = synth.make_reads(80_000, 300, 4000, seed=2)
    ib, qb = 400_000, 150_000
    eng.configure(k=15, w=5)
    eng.upload(rs)
    for minhash in (False, True):
        _, got = both_ways(eng, lambda: eng.find_overlaps_and_create_piles(
            0.001, 8, minhash, ib, qb))
        want = oracle.stage1(oracle.engine(15, 5, threads=4), oracle.reads(rs), 0.001, 8,
                             minhash, ib, qb)
        for k in STAGE1_KEYS:
            assert np.array_equal(got[k], want[k]), (minhash, k)
        assert got["num_mapped"] == int(want["num_mapped"][0])


@pytest.mark.parametrize("bare", [0, 1, 8])
def test_stage1_tiered_bare_keys(eng, oracle, bare):
    """tiers forced on: the bare keys partitioned (bare_count 1, 8) or sorted (0)"""
    rs = synth.make_reads(300_000, 400, 5000, seed=7)
    eng.configure(k=15, w=5)
    eng.upload(rs)
    eng.set_option("tier_min_records", 0)
    eng.set_option("bare_count", bare)
    try:
        def run():
            got = eng.find_overlaps_and_create_piles(0.001, 8, False)
            return got, eng.stats()["index_keys"], [eng.filter(f) for f in FREQS]
        _, (got, n_keys, occ) = both_ways(eng, run)
    finally:
        eng.set_option("bare_count", 1)
        eng.set_option("tier_min_records", 1 << 18)
    o = oracle.engine(15, 5, threads=8)
    reads = oracle.reads(rs)
    want = oracle.stage1(o, reads, 0.001, 8, False, 1 << 32, 1 << 30)
    for k in STAGE1_KEYS:
        assert np.array_equal(got[k], want[k]), k
    o = oracle.engine(15, 5, threads=8)
    oracle.minimize(o, reads, 0, rs.n, False)
    assert n_keys == int(oracle.keys(o)["totals"][0])
    assert occ == [oracle.filter(o, f) for f in FREQS]


@pytest.mark.parametrize("minhash", [False, True])
def test_index_records(eng, oracle, lambda_reads, minhash):
    eng.configure(k=15, w=5)
    eng.upload(lambda_reads)

    def run():
        eng.minimize(0, lambda_reads.n, minhash)
        return eng.index_records()
    off, idx = both_ways(eng, run)
    o = oracle.engine(15, 5, threads=4)
    oracle.minimize(o, oracle.reads(lambda_reads), 0, lambda_reads.n, minhash)
    keys = oracle.keys(o)
    v, org = idx["value"], idx["origin"]
    assert v.size == int(keys["totals"][1]) and idx["n_keys"] == int(keys["totals"][0])
    assert (np.diff(v.astype(np.int64)) >= 0).all()
    same = v[1:] == v[:-1]
    assert (org[1:][same] > org[:-1][same]).all()
    uv, uc = np.unique(v, return_counts=True)
    assert np.array_equal(uv, keys["values"])
    assert np.array_equal(uc.astype(np.uint32), keys["counts"])
    assert np.array_equal(v, off["value"]) and np.array_equal(org, off["origin"])


def test_map_lambda(eng, oracle, lambda_reads):
    n = lambda_reads.n
    eng.set_option("radix_portion_tiles", 1)
    try:
        _check_map(eng, oracle, lambda_reads, 15, 5, 0.001, False,
                   [(0, n, True, True, True), (0, n, True, True, False),
                    (0, n, False, False, False)])
    finally:
        eng.set_option("radix_portion_tiles", 0)
    off, on = both_ways(eng, lambda: eng.map(0, n, True, True, False))
    assert np.array_equal(on["overlaps"], GOLD["map_full_overlaps"])
    assert np.array_equal(off["overlaps"], on["overlaps"])


def test_polish_window_layers(eng, oracle):
    """racon::Polisher::Polish at 90x with 137-base windows: some 20 000 layer slots,
    three tiles, sorted by window on the device (layers.cu)"""
    from raven_b200 import polish
    from test_gpu_polish_layers import Options, concat, facade_alignments, make_set, run_pair
    w = 137
    draft, reads, _, _ = make_set(17, n_reads=900)
    want, _ = run_pair(oracle, draft, reads, w=w)
    with Options("radix_portion_tiles=1"):
        got, _ = polish.polish(draft, reads, w=w, threads=4)
    assert [got.ascii(i) for i in range(got.n)] == [want.ascii(i) for i in range(want.n)]
    T = draft.n
    allr = concat(draft, reads)
    eng.configure(15, 5, 500, 4, 100, 10000)
    eng.upload(allr)
    eng.minimize(0, T)
    eng.filter(0.001)
    alns = facade_alignments(eng, T, reads.n)
    _, bp_off, bp = eng.align_breaking_points(*alns, window=w)
    assert bp_off[-1] > 2 * TILE[4]
    off, on = both_ways(eng, lambda: eng.polish_windows(
        alns[0], alns[1], alns[2], alns[3], alns[4], bp_off, bp, T, window=w))
    assert on["consensus"].tobytes() == off["consensus"].tobytes()
    first = np.concatenate([[0], np.cumsum([(int(x) + w - 1) // w for x in draft.lens])])
    for t in range(T):
        c0, c1 = on["cons_off"][first[t]], on["cons_off"][first[t + 1]]
        assert on["consensus"][int(c0):int(c1)].tobytes() == want.ascii(t)


# ---- e. full size: the default portion + 2 tiles + 3 records, checked on the device ----

def _torch():
    import torch
    return torch


def full_n(key_bytes):
    tile = TILE[key_bytes]
    return ((1 << 30) - 1) // tile * tile + 2 * tile + 3


def need_memory(nbytes):
    torch = _torch()
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip(f"needs {nbytes / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} free")


def buf(nbytes):
    """device bytes of a DevBuf of nbytes (it reserves a sixteenth more)"""
    return nbytes + nbytes // 16 + 64


STEP = 1 << 27


def chunks(n):
    for a in range(0, n, STEP):
        yield a, min(n, a + STEP + 1)   # one record of overlap: pairs across chunks


def full_keys(torch, n, values, shift, run_at):
    """keys of `values` distinct values << shift (30-bit), a heavy run across run_at"""
    k = torch.randint(0, values, (n,), dtype=torch.int32, device="cuda",
                      generator=torch.Generator("cuda").manual_seed(n % 977))
    k <<= shift
    k[run_at - 3 * 8192:run_at + 3 * 8192] = k[0]
    return k


class DevicePeak:
    """the least free device memory seen while the block runs, polled every 2 ms from a
    thread (the library's calls release the GIL)"""

    def __enter__(self):
        torch = _torch()
        self.low, self.total = torch.cuda.mem_get_info()
        self.stop = threading.Event()

        def poll():
            while not self.stop.is_set():
                self.low = min(self.low, torch.cuda.mem_get_info()[0])
                time.sleep(0.002)
        self.thread = threading.Thread(target=poll, daemon=True)
        self.thread.start()
        return self

    def __exit__(self, *exc):
        self.stop.set()
        self.thread.join()


def report(name, n, nbytes, peak):
    torch = _torch()
    print(f"\n[{name}] n={n}: device memory in use at the peak "
          f"{(peak.total - peak.low) / 2**30:.1f} GiB (engine buffers {nbytes / 2**30:.1f} GiB, "
          f"torch peak {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB)")


@pytest.mark.slow
@pytest.mark.parametrize("key_bytes", [4, 8])
def test_full_size_pairs(eng, key_bytes):
    """(u32, u64) - the index - and (u64, u64), in place: a stable permutation"""
    torch = _torch()
    n = full_n(key_bytes)
    kdt = torch.int32 if key_bytes == 4 else torch.int64
    engine_bytes = buf(n * (key_bytes + 8)) + (n // TILE[key_bytes] + 1) * 4096
    need_memory(n * (2 * key_bytes + 8) + engine_bytes + (2 << 30))
    with DevicePeak() as peak:
        torch.cuda.reset_peak_memory_stats()
        P = ((1 << 30) - 1) // TILE[key_bytes] * TILE[key_bytes]
        src = full_keys(torch, n, 1 << 30, 0, P).to(kdt)
        keys = src.clone()
        vals = torch.arange(n, dtype=torch.int64, device="cuda")
        (_, _), launches = counted(eng, lambda: eng.debug_sort_pairs(keys, vals, 0, 30))
        assert launches == sort_launches(key_bytes, n, 0, 30, 0) == 2 + 3 * 2
        for a, b in chunks(n):
            k, v = keys[a:b], vals[a:b]
            assert bool((k[1:] >= k[:-1]).all()), a
            # (payloads the sort did not write are garbage: bounds first, then the gather)
            assert bool(((v >= 0) & (v < n)).all()), a
            assert bool((src[v] == k).all()), a
            same = k[1:] == k[:-1]
            assert bool((v[1:][same] > v[:-1][same]).all()), a
    report(f"pairs {key_bytes}", n, engine_bytes, peak)
    del src, keys, vals
    torch.cuda.empty_cache()


def key_histogram(torch, keys, shift):
    h = torch.zeros(1 << 24, dtype=torch.int64, device="cuda")
    for a in range(0, keys.numel(), STEP):
        h += torch.bincount((keys[a:a + STEP] >> shift).long(), minlength=1 << 24)
    return h


@pytest.mark.slow
def test_full_size_keys_only(eng):
    torch = _torch()
    n = full_n(4)
    engine_bytes = buf(4 * n) + (n // TILE[4] + 1) * 4096
    need_memory(4 * n + engine_bytes + (2 << 30))
    with DevicePeak() as peak:
        torch.cuda.reset_peak_memory_stats()
        keys = full_keys(torch, n, 1 << 24, 6, n - 2 * 8192 - 3)
        want = key_histogram(torch, keys, 6)
        (_, _), launches = counted(eng, lambda: eng.debug_sort_pairs(keys, None, 0, 30))
        assert launches == 2 + 3 * 2
        for a, b in chunks(n):
            k = keys[a:b]
            assert bool((k[1:] >= k[:-1]).all()), a
        assert torch.equal(key_histogram(torch, keys, 6), want)
    report("keys", n, engine_bytes, peak)
    del keys
    torch.cuda.empty_cache()


@pytest.mark.slow
def test_full_size_partition(eng):
    torch = _torch()
    n = full_n(4)
    engine_bytes = buf(4 * n) + (n // TILE[4] + 1) * 4096
    need_memory(4 * n + engine_bytes + (2 << 30))
    with DevicePeak() as peak:
        torch.cuda.reset_peak_memory_stats()
        keys = full_keys(torch, n, 1 << 24, 6, n - 2 * 8192 - 3)
        want = key_histogram(torch, keys, 6)
        (_, start), launches = counted(eng, lambda: eng.debug_partition_keys(keys, 20, 30))
        assert launches == 2 + 2
        counts = want.view(1024, -1).sum(1)   # digit = key >> 20 = (key >> 6) >> 14
        want_start = torch.cumsum(counts, 0) - counts
        assert np.array_equal(start.astype(np.int64), want_start.cpu().numpy())
        for a, b in chunks(n):
            d = keys[a:b] >> 20
            assert bool((d[1:] >= d[:-1]).all()), a
        assert torch.equal(key_histogram(torch, keys, 6), want)
    report("partition", n, engine_bytes, peak)
    del keys
    torch.cuda.empty_cache()
