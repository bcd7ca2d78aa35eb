"""The BGZF member inflate has one copy, raven_b200/csrc/inflate.cuh, which FxInflateKernel
runs one member per warp. Here that header, compiled for the host, inflates raw deflate
streams and is compared with zlib's raw inflate: it must accept exactly the streams zlib
accepts (ending exactly at the end of the input, within the output bound) and give the
same bytes. The slice-wise CRC-32 the kernel uses is compared with zlib.crc32."""
import ctypes as C
import os
import subprocess
import zlib
from collections import Counter

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
MAX = 65536

LBASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99,
         115, 131, 163, 195, 227, 258]
LEXT = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DBASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025,
         1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577]
DEXT = [0, 0, 0, 0] + [e for e in range(1, 14) for _ in (0, 1)]
ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_DIST = [5] * 32
CL_LENS = [4] * 13 + [5] * 6  # a complete code-length code over all 19 symbols


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("inflate") / "_inflate_host.so")
    subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++",
                    os.path.join(HERE, "inflate_host.cpp"), "-o", so], check=True)
    lib = C.CDLL(so)
    lib.rvn_test_inflate.restype = C.c_int64
    lib.rvn_test_inflate.argtypes = [C.c_char_p, C.c_uint64, C.c_void_p, C.c_uint32]
    lib.rvn_test_crc32.restype = C.c_uint32
    lib.rvn_test_crc32.argtypes = [C.c_char_p, C.c_uint32, C.c_uint32]
    return lib


def ours(lib, data, cap=MAX):
    out = C.create_string_buffer(max(cap, 1))
    n = lib.rvn_test_inflate(data, len(data), out, cap)
    return None if n < 0 else out.raw[:n]


def zlibs(data, cap=MAX):
    d = zlib.decompressobj(-15)
    try:
        out = d.decompress(data)
    except zlib.error:
        return None
    if not d.eof or d.unused_data or len(out) > cap:
        return None
    return out


def same(lib, data, cap=MAX):
    want = zlibs(data, cap)
    assert ours(lib, data, cap) == want
    return want is not None


def deflate(data, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, flushes=()):
    co = zlib.compressobj(level, zlib.DEFLATED, -15, 9, strategy)
    out, at = b"", 0
    for pos, mode in flushes:
        out += co.compress(data[at:pos]) + co.flush(mode)
        at = pos
    return out + co.compress(data[at:]) + co.flush()


def fastq(rng, n_bytes):
    out = bytearray()
    i = 0
    while len(out) < n_bytes:
        n = int(rng.integers(50, 400))
        out += b"@read%d ch=%d\n" % (i, i % 7)
        out += bytes(rng.choice(list(b"ACGT"), n)) + b"\n+\n"
        out += bytes(rng.integers(33, 75, n).astype(np.uint8)) + b"\n"
        i += 1
    return bytes(out[:n_bytes])


class Bits:
    def __init__(self):
        self.v, self.n = 0, 0

    def put(self, val, k):
        self.v |= (val & ((1 << k) - 1)) << self.n
        self.n += k

    def huff(self, code, length):  # Huffman codes go most significant bit first
        self.put(int(format(code, "0%db" % length)[::-1], 2) if length else 0, length)

    def align(self):
        self.n = (self.n + 7) // 8 * 8

    def bytes(self):
        return self.v.to_bytes((self.n + 7) // 8, "little")


def canon(lens):
    count = Counter(l for l in lens if l)
    code, first = 0, {}
    for b in range(1, 16):
        code = (code + count.get(b - 1, 0)) << 1
        first[b] = code
    codes = {}
    for s, l in enumerate(lens):
        if l:
            codes[s] = (first[l], l)
            first[l] += 1
    return codes


def tokens_body(w, tokens, lit, dist):
    """tokens: a byte (literal), (length, distance), or ("lit", symbol) / ("dist", length,
    symbol) for symbols a valid encoder never writes"""
    for t in tokens:
        if isinstance(t, int):
            w.huff(*lit[t])
        elif t[0] == "lit":
            w.huff(*lit[t[1]])
        else:
            if t[0] == "dist":
                w.huff(*lit[257]), w.huff(*dist[t[2]])
                continue
            ln, d = t
            i = 28 if ln == 258 else max(k for k in range(28) if LBASE[k] <= ln)
            w.huff(*lit[257 + i])
            w.put(ln - LBASE[i], LEXT[i])
            j = max(k for k in range(30) if DBASE[k] <= d)
            w.huff(*dist[j])
            w.put(d - DBASE[j], DEXT[j])
    w.huff(*lit[256])


def fixed(w, tokens, last=1):
    w.put(last, 1), w.put(1, 2)
    tokens_body(w, tokens, canon(FIXED_LIT), canon(FIXED_DIST))


def stored(w, data, last=1, nlen=None):
    w.put(last, 1), w.put(0, 2)
    w.align()
    w.put(len(data), 16)
    w.put(nlen if nlen is not None else ~len(data) & 0xFFFF, 16)
    for b in data:
        w.put(b, 8)


def dynamic(w, lit_lens, dist_lens, tokens=(), last=1, seq=None, hlit=None, hdist=None,
            cl_lens=CL_LENS):
    """seq: the code-length symbols as (symbol, extra, extra bits); by default one per length"""
    w.put(last, 1), w.put(2, 2)
    w.put(len(lit_lens) - 257 if hlit is None else hlit, 5)
    w.put(len(dist_lens) - 1 if hdist is None else hdist, 5)
    w.put(19 - 4, 4)
    for i in range(19):
        w.put(cl_lens[ORDER[i]], 3)
    clc = canon(cl_lens)
    for sym, extra, k in (seq if seq is not None else [(l, 0, 0) for l in lit_lens + dist_lens]):
        w.huff(*clc[sym])
        w.put(extra, k)
    if tokens is not None:
        tokens_body(w, list(tokens), canon(lit_lens), canon(dist_lens))


def build(*blocks):
    w = Bits()
    for f, *args in blocks:
        f(w, *args)
    return w.bytes()


# a valid dynamic code: literals 'A', 'C', 'G', 'T', '\n', end of block and lengths 3 and 4
def small_lit(extra=()):
    lens = [0] * 259
    for s in b"ACGT\n":
        lens[s] = 3
    lens[256] = lens[257] = lens[258] = 3
    for s, l in extra:
        lens[s] = l
    return lens


STRATEGIES = [
    pytest.param(0, zlib.Z_DEFAULT_STRATEGY, id="stored"),
    pytest.param(1, zlib.Z_DEFAULT_STRATEGY, id="level1"),
    pytest.param(6, zlib.Z_DEFAULT_STRATEGY, id="level6"),
    pytest.param(9, zlib.Z_DEFAULT_STRATEGY, id="level9"),
    pytest.param(6, zlib.Z_FIXED, id="fixed"),
    pytest.param(6, zlib.Z_HUFFMAN_ONLY, id="huffman_only"),
    pytest.param(6, zlib.Z_RLE, id="rle"),
]


@pytest.mark.parametrize("level,strategy", STRATEGIES)
def test_levels_and_strategies(lib, level, strategy):
    rng = np.random.default_rng(level * 10 + strategy)
    for n in (0, 1, 100, 5000, 65280, MAX):
        for data in (fastq(rng, n), rng.integers(0, 256, n).astype(np.uint8).tobytes(),
                     b"A" * n):
            z = deflate(data, level, strategy)
            assert same(lib, z)
            assert ours(lib, z) == data


@pytest.mark.parametrize("mode", [zlib.Z_SYNC_FLUSH, zlib.Z_FULL_FLUSH], ids=["sync", "full"])
def test_flushes_mid_stream(lib, mode):
    rng = np.random.default_rng(mode)
    data = fastq(rng, 60000)
    for k in (1, 3, 17):
        cuts = sorted(set(int(x) for x in rng.integers(0, len(data), k)))
        for level in (1, 6):
            z = deflate(data, level, flushes=[(c, mode) for c in cuts] + [(len(data), mode)])
            assert ours(lib, z) == data
            assert same(lib, z)


def test_output_bound(lib):
    rng = np.random.default_rng(3)
    data = fastq(rng, MAX)
    z = deflate(data, 1)
    assert ours(lib, z, MAX) == data
    assert ours(lib, z, MAX - 1) is None and not same(lib, z, MAX - 1)
    assert ours(lib, deflate(b""), 0) == b""
    assert ours(lib, deflate(data + b"x")) is None  # 65,537 bytes


def test_every_length_and_distance_code_at_both_ends(lib):
    rng = np.random.default_rng(1)
    prefix = rng.integers(0, 256, 32768).astype(np.uint8).tobytes()
    toks = []
    for i in range(29):
        for ln in (LBASE[i], LBASE[i] + (1 << LEXT[i]) - 1):
            toks.append((ln, 1))
            toks.append((ln, 32768))
    for j in range(30):
        for d in (DBASE[j], DBASE[j] + (1 << DEXT[j]) - 1):
            toks.append((3, d))
            toks.append((258, d))
    z = build((stored, prefix, 0), (fixed, toks))
    out = ours(lib, z, 1 << 20)
    assert out is not None and out[:32768] == prefix
    assert same(lib, z, 1 << 20)
    # the same tokens through complete dynamic codes over every length and distance symbol
    z = build((stored, prefix, 0), (dynamic, [8] * 226 + [9] * 60, [4] * 2 + [5] * 28, toks))
    assert ours(lib, z, 1 << 20) == out
    assert same(lib, z, 1 << 20)
    # distance 1 and 32,768 reaching exactly the first byte; one further is too far back
    for d, ok in ((1, True), (32768, True)):
        assert same(lib, build((stored, prefix[-d:], 0), (fixed, [(258, d)]))) == ok
    assert not same(lib, build((stored, prefix[:100], 0), (fixed, [(3, 101)])))
    assert not same(lib, build((fixed, [(3, 1)])))


def test_hand_built_codes(lib):
    ok = lambda z: same(lib, z + b"")  # noqa: E731
    body = list(b"ACGT\nAC") + [(3, 2), (4, 1)]
    assert ok(build((dynamic, small_lit(), [1, 1], body)))
    # over-subscribed literal/length and distance codes, the code-length code
    assert not ok(build((dynamic, small_lit([(ord("N"), 1)]), [1, 1], None)) + b"\0" * 8)
    assert not ok(build((dynamic, small_lit(), [1, 1, 1], None)) + b"\0" * 8)
    assert not ok(build((dynamic, small_lit(), [1, 1], None, 1, None, None, None,
                         [4] * 14 + [5] * 5)) + b"\0" * 8)
    # incomplete: the literal code (not a single 1-bit code), the code-length code
    assert not ok(build((dynamic, small_lit([(ord("N"), 4)])[:258] + [0], [1, 1], None))
                  + b"\0" * 8)
    assert not ok(build((dynamic, small_lit(), [1, 1], None, 1, None, None, None,
                         [4] * 12 + [5] * 7)) + b"\0" * 8)
    # a single 1-bit literal/length code (only the end of block) and a single 1-bit distance
    # code, or none: zlib takes them
    only_end = [0] * 256 + [1]
    assert ok(build((dynamic, only_end, [1], [])))
    assert ok(build((dynamic, small_lit(), [1], list(b"ACG") + [(3, 1)])))
    assert ok(build((dynamic, small_lit(), [0], list(b"ACGT"))))
    # ... but a length with no distance code, or the unused half of a single code, fails
    z = build((dynamic, small_lit(), [0], list(b"AC") + [("lit", 257)]))
    assert not ok(z + b"\0\0")
    w = Bits()
    dynamic(w, small_lit(), [1], None)
    for t in (ord("A"), ord("C")):
        w.huff(*canon(small_lit())[t])
    w.huff(*canon(small_lit())[257])
    w.put(1, 1)  # the distance code '1' has no symbol
    assert not ok(w.bytes() + b"\0\0")
    # missing end of block, too many length / distance codes
    lens = small_lit()
    lens[256], lens[258] = 0, 2
    assert not ok(build((dynamic, lens, [1, 1], None)) + b"\0" * 8)
    lit286 = small_lit() + [0] * (286 - 259)
    assert ok(build((dynamic, lit286, [1, 1], list(b"GATTACA"))))
    assert not ok(build((dynamic, lit286 + [0], [1, 1], None)) + b"\0" * 8)
    assert not ok(build((dynamic, small_lit(), [1] * 2 + [0] * 29, None)) + b"\0" * 8)
    # repeat code 16 first, repeats past the lengths; 17/18 runs that land exactly
    seq = [(16, 0, 2)] + [(l, 0, 0) for l in small_lit() + [1, 1]]
    assert not ok(build((dynamic, small_lit(), [1, 1], None, 1, seq)) + b"\0" * 8)
    lit = small_lit()
    seq = [(l, 0, 0) for l in lit[:258]] + [(2, 0, 0)] + [(16, 3, 2)]
    assert not ok(build((dynamic, lit, [1, 1], None, 1, seq)) + b"\0" * 8)
    seq = [(17, 7, 3), (3, 0, 0), (18, 43, 7), (3, 0, 0), (0, 0, 0), (3, 0, 0), (17, 0, 3),
           (3, 0, 0), (18, 1, 7), (3, 0, 0), (18, 127, 7), (18, 22, 7), (3, 0, 0), (3, 0, 0),
           (3, 0, 0), (1, 0, 0), (1, 0, 0)]
    assert ok(build((dynamic, small_lit(), [1, 1], body, 1, seq)))
    over = seq[:-1] + [(16, 0, 2)]  # the last repeat runs three past the distance lengths
    assert not ok(build((dynamic, small_lit(), [1, 1], None, 1, over)) + b"\0" * 8)
    # fixed-code symbols no valid stream uses: lengths 286 / 287, distances 30 / 31
    for t in (("lit", 286), ("lit", 287)):
        assert not ok(build((fixed, [65, t])) + b"\0\0")
    for d in (30, 31):
        assert not ok(build((fixed, [65, ("dist", 0, d)])) + b"\0\0")
    # block type 3; a stored block whose NLEN is not ~LEN
    w = Bits()
    w.put(1, 1), w.put(3, 2)
    assert not ok(w.bytes() + b"\0" * 4)
    assert ok(build((stored, b"ACGT")))
    assert not ok(build((stored, b"ACGT", 1, 0xFFFF)))
    assert not ok(build((stored, b"ACGT", 1, 4)))
    # empty stored blocks, and a stream that ends before / after its input
    assert ok(build((stored, b"", 0), (stored, b"", 0), (fixed, [65])))
    z = build((fixed, list(b"ACGT")))
    assert not ok(z[:-1]) and not ok(z + b"\0")


MUTATED = [pytest.param(lvl, st, id=i) for lvl, st, i in (
    (1, zlib.Z_DEFAULT_STRATEGY, "level1"), (6, zlib.Z_DEFAULT_STRATEGY, "level6"),
    (9, zlib.Z_FIXED, "fixed"), (6, zlib.Z_HUFFMAN_ONLY, "huffman_only"),
    (0, zlib.Z_DEFAULT_STRATEGY, "stored"))]


@pytest.mark.parametrize("level,strategy", MUTATED)
def test_mutated_streams_match_zlib(lib, level, strategy):
    rng = np.random.default_rng(1000 + level * 7 + strategy)
    data = fastq(rng, 20000)
    z = bytearray(deflate(data, level, strategy,
                          flushes=[(7000, zlib.Z_SYNC_FLUSH)] if level else ()))
    accepted = rejected = 0
    for trial in range(600):
        m = bytearray(z)
        kind = trial % 3
        if kind == 0:
            for _ in range(int(rng.integers(1, 4))):
                bit = int(rng.integers(0, 8 * len(m)))
                m[bit >> 3] ^= 1 << (bit & 7)
        elif kind == 1:
            m = m[:int(rng.integers(0, len(m)))]
        else:
            bit = int(rng.integers(0, min(8 * len(m), 2000)))  # the block headers
            m[bit >> 3] ^= 1 << (bit & 7)
        if same(lib, bytes(m)):
            accepted += 1
        else:
            rejected += 1
    assert rejected > 100


@pytest.mark.parametrize("slices", [1, 2, 7, 32])
def test_crc32_by_slices(lib, slices):
    rng = np.random.default_rng(slices)
    for n in (0, 1, 31, 32, 33, 1000, 65280, MAX):
        data = rng.integers(0, 256, n).astype(np.uint8).tobytes()
        assert lib.rvn_test_crc32(data, n, slices) == zlib.crc32(data)
