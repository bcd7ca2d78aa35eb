"""GPU: BGZF files (the blocked gzip of bgzip and samtools) take the device inflate route of
rvn_reads_upload_files. The oracle is the drop-in parser (tests/cpp/_build/io_test parse),
which reads every file through zlib: a BGZF file must parse to the read set it gives, and
every odd case (foreign members after BGZF ones, trailing bytes, truncation, a damaged
member) must give its result or its message. The BGZF files are written here with zlib."""
import gzip
import os
import struct
import subprocess
import zlib

import numpy as np
import pytest

from raven_b200 import engine
from test_gpu_fastx import (SWEEP, LENGTHS, _check, _fasta, _fastq, _kind,  # noqa: F401
                            _lambda_fastq, _rc, eng, io_test)

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
BGZIP_CUT = 65280  # bgzip's text per member
# bgzip's end-of-file marker: an empty member
EOF_MARKER = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")

pytestmark = pytest.mark.gpu


def deflate(data, level=1, strategy=zlib.Z_DEFAULT_STRATEGY, sync_at=None):
    co = zlib.compressobj(level, zlib.DEFLATED, -15, 9, strategy)
    if sync_at is None:
        return co.compress(data) + co.flush()
    return (co.compress(data[:sync_at]) + co.flush(zlib.Z_SYNC_FLUSH) + co.compress(data[sync_at:])
            + co.flush())


def member(data, level=1, strategy=zlib.Z_DEFAULT_STRATEGY, sync_at=None, crc=None, isize=None,
           other_subfield=False):
    d = deflate(data, level, strategy, sync_at)
    pre = b"XY" + struct.pack("<H", 3) + b"abc" if other_subfield else b""
    xlen = len(pre) + 6
    total = 12 + xlen + len(d) + 8
    return (b"\x1f\x8b\x08\x04\0\0\0\0\0\xff" + struct.pack("<H", xlen) + pre + b"BC"
            + struct.pack("<HH", 2, total - 1) + d
            + struct.pack("<II", zlib.crc32(data) if crc is None else crc,
                          len(data) if isize is None else isize))


def bgzf(text, cuts=None, eof=True, **kw):
    """text as BGZF members cut at `cuts` (default: bgzip's 65,280-byte members)"""
    if cuts is None:
        cuts = list(range(BGZIP_CUT, len(text), BGZIP_CUT))
    bounds = [0] + list(cuts) + [len(text)]
    out = b"".join(member(text[a:b], **kw) for a, b in zip(bounds, bounds[1:]))
    return out + (EOF_MARKER if eof else b"")


def gzip_fname(data):
    """a gzip member with FNAME, as gzip(1) writes it"""
    return (b"\x1f\x8b\x08\x08\0\0\0\0\0\x03reads.fq\0" + deflate(data)
            + struct.pack("<II", zlib.crc32(data), len(data)))


def _write(path, data):
    with open(path, "wb") as f:
        f.write(data)


def _oracle_error(io_test, p):
    out = subprocess.run([io_test, "parse", _kind(p), str(p)], stdout=subprocess.PIPE)
    if out.returncode == 0:
        return None
    assert out.returncode == 3, out.stdout
    return out.stdout.decode().strip().split("invalid_argument: ", 1)[1]


def _same_as_oracle(eng, io_test, p, chunks=(0,)):
    """the oracle's reads, or its message with the context left without a read set"""
    what = _oracle_error(io_test, p)
    if what is None:
        return _check(eng, io_test, [p], chunks)
    for chunk in chunks:
        eng.set_option("fastx_chunk_bytes", chunk)
        with pytest.raises(ValueError) as e:
            eng.upload_files([str(p)])
        assert str(e.value) == f"{what} ({p})", chunk
        assert _rc(eng) == -3
    eng.set_option("fastx_chunk_bytes", 0)
    return what


def _route(eng, p):
    """whether p took the device inflate route"""
    eng.set_option("reset_stats", 1)
    eng.upload_files([str(p)])
    return "fastx_inflate" in eng.timings()


@pytest.mark.parametrize("variant", ["fasta_crlf_blanks_spaces", "fasta_no_last_newline",
                                     "fastq_four_line", "fastq_multi_line_at_plus_crlf",
                                     "fastq_blanks", "fastq_low_high"])
def test_text_edges_every_chunk_size(eng, io_test, tmp_path, variant):
    rng = np.random.default_rng(len(variant) + 7)
    if variant.startswith("fasta"):
        text = _fasta(rng, 37, blanks="blanks" in variant, crlf="crlf" in variant,
                      spaces="spaces" in variant, last_newline="no_last" not in variant)
        p = tmp_path / "r.fa.gz"
    else:
        text = _fastq(rng, wrap=23 if "multi_line" in variant else None, crlf="crlf" in variant,
                      blanks="blanks" in variant, low_high="low_high" in variant,
                      at_plus="at_plus" in variant)
        p = tmp_path / "r.fq.gz"
    # members of 61 text bytes: at chunk sizes up to 61 every piece is one member
    _write(p, bgzf(text, cuts=range(61, len(text), 61)))
    assert _route(eng, p)
    assert _check(eng, io_test, [p], chunks=[0] + SWEEP) == len(LENGTHS)


def test_member_cuts(eng, io_test, tmp_path):
    rng = np.random.default_rng(21)
    text = _fastq(rng, wrap=50, crlf=True) * 40
    crlf = [i + 1 for i in range(len(text) - 1) if text[i:i + 2] == b"\r\n"][::37]
    at = [i for i in range(len(text)) if text[i:i + 1] == b"@"][1::5]
    cuts = sorted(set(crlf + [a + 3 for a in at]))
    p = tmp_path / "cuts.fastq.gz"
    _write(p, bgzf(text, cuts=cuts))
    assert _check(eng, io_test, [p], chunks=(0, 1, 100, 4093)) == 40 * len(LENGTHS)
    # members of exactly 65,536 bytes of text, and an empty member between two
    big = _fastq(rng, wrap=70) * 300
    cuts = list(range(65536, len(big), 65536))
    p = tmp_path / "full.fq.gz"
    _write(p, bgzf(big, cuts=cuts[:2] + [cuts[1]] + cuts[2:]))
    assert _route(eng, p)
    assert _check(eng, io_test, [p], chunks=(0, 65536, 100000)) == 300 * len(LENGTHS)


@pytest.mark.parametrize("level,strategy,sync", [
    (0, zlib.Z_DEFAULT_STRATEGY, None), (1, zlib.Z_DEFAULT_STRATEGY, None),
    (6, zlib.Z_DEFAULT_STRATEGY, 1000), (9, zlib.Z_DEFAULT_STRATEGY, None),
    (6, zlib.Z_FIXED, None), (6, zlib.Z_HUFFMAN_ONLY, 5000), (6, zlib.Z_RLE, None)],
    ids=["stored", "level1", "level6_sync", "level9", "fixed", "huffman_only_sync", "rle"])
def test_block_types(eng, io_test, tmp_path, level, strategy, sync):
    rng = np.random.default_rng(level + 3 * strategy)
    text = _fastq(rng, wrap=80) * 60
    p = tmp_path / "b.fastq"  # (the route follows the bytes, not the name)
    _write(p, bgzf(text, cuts=range(20000, len(text), 20000), level=level, strategy=strategy,
                   sync_at=sync, other_subfield=True))
    assert _route(eng, p)
    assert _check(eng, io_test, [p], chunks=(0, 30000)) == 60 * len(LENGTHS)


def test_eof_marker_only_and_mixed_files(eng, io_test, tmp_path):
    rng = np.random.default_rng(4)
    empty = tmp_path / "empty.fq.gz"
    _write(empty, EOF_MARKER)
    assert _route(eng, empty)
    rs = eng.upload_files([str(empty)])
    assert rs.n == 0 and eng.n_reads == 0
    a, b, c, d, e = (tmp_path / "a.fasta.gz", tmp_path / "b.fq.gz", tmp_path / "c.fastq",
                     tmp_path / "d.fa", tmp_path / "e.fq.gz")
    _write(a, bgzf(_fasta(rng, 60), cuts=[500]))
    _write(b, gzip.compress(_fastq(rng), compresslevel=1))
    _write(c, _fastq(rng, wrap=30))
    _write(d, b"")
    _write(e, bgzf(_fastq(rng, crlf=True), cuts=[999]))
    assert not _route(eng, b)
    assert _check(eng, io_test, [a, b, empty, c, d, e], chunks=(0, 7, 1000)) == 4 * len(LENGTHS)


def _handoff_cases(rng):
    text = _fastq(rng, wrap=60) * 20
    fasta = _fasta(rng, 60) * 20
    body = bgzf(text, cuts=range(3000, len(text), 3000), eof=False)
    more = _fastq(rng)
    last_bsize = body.rfind(b"BC\x02\x00") + 4
    return {
        "gzip_after.fq.gz": body + gzip.compress(more, compresslevel=6),
        "fname_after.fq.gz": body + gzip_fname(more) + EOF_MARKER,
        "text_after.fa.gz": bgzf(fasta, cuts=[4000]) + b"trailing text\n",
        "lone_1f.fq.gz": body + EOF_MARKER + b"\x1f",
        "magic_garbage.fq.gz": body + EOF_MARKER + b"\x1f\x8bxxxxxxxxxxxxxxxxxxxx",
        "cut_in_member.fq.gz": body[:len(body) // 2 + 11],
        "cut_in_member.fa.gz": bgzf(fasta, cuts=range(2000, len(fasta), 2000))[:5000],
        "cut_in_header.fq.gz": body + EOF_MARKER[:9],
        "bsize_past_end.fq.gz": (body[:last_bsize] + struct.pack("<H", 65000)
                                 + body[last_bsize + 2:]),
        "isize_over_64k.fa.gz": bgzf(fasta * 4, cuts=[100000]),
    }


@pytest.mark.parametrize("name", list(_handoff_cases(np.random.default_rng(0))))
def test_handoff_equals_zlib(eng, io_test, tmp_path, name):
    p = tmp_path / name
    _write(p, _handoff_cases(np.random.default_rng(77))[name])
    _same_as_oracle(eng, io_test, p, chunks=(0, 1000))


def test_device_faults(eng, io_test, tmp_path):
    rng = np.random.default_rng(31)
    text = _fastq(rng, wrap=60) * 20
    cuts = list(range(4000, len(text), 4000))
    parts = [text[a:b] for a, b in zip([0] + cuts, cuts + [len(text)])]
    good = tmp_path / "good.fasta"
    _write(good, b">g\nACGT\n")
    unreadable = "[bioparser::Parser::Parse] error: unable to read file"

    def expect_fault(p):
        assert _oracle_error(io_test, p) == unreadable
        eng.upload_files([str(good)])
        with pytest.raises(ValueError) as e:
            eng.upload_files([str(good), str(p)])
        assert str(e.value) == f"{unreadable} ({p})"
        assert _rc(eng) == -3
        assert eng.lib.rvn_reads_parsed(eng.h, None, None, None, None, None, None, None) == -3

    members = [member(x) for x in parts]
    # a flipped bit in the Huffman codes of the second member
    start = len(members[0]) + 18 + 2
    for bit in range(0, 400, 7):
        m = bytearray(b"".join(members) + EOF_MARKER)
        m[start + bit // 8] ^= 1 << (bit % 8)
        p = tmp_path / "flip.fq.gz"
        _write(p, bytes(m))
        if _oracle_error(io_test, p) == unreadable:
            break
    expect_fault(p)
    # a flipped byte inside a stored block: the deflate data stay valid, the CRC does not
    stored = [member(x, level=0) for x in parts]
    m = bytearray(b"".join(stored) + EOF_MARKER)
    m[len(stored[0]) + 18 + 5 + 100] ^= 0x04
    p = tmp_path / "stored_flip.fq.gz"
    _write(p, bytes(m))
    expect_fault(p)
    # a wrong CRC field; a wrong ISIZE, smaller and larger
    for name, kw in (("crc", dict(crc=zlib.crc32(parts[1]) ^ 1)),
                     ("isize_small", dict(isize=len(parts[1]) - 1)),
                     ("isize_large", dict(isize=len(parts[1]) + 1))):
        p = tmp_path / (name + ".fq.gz")
        _write(p, members[0] + member(parts[1], **kw) + b"".join(members[2:]) + EOF_MARKER)
        expect_fault(p)
    eng.upload_files([str(good)])
    assert _rc(eng) == 0


def test_lambda_bgzf_end_to_end(eng, tmp_path, lambda_reads):
    plain = tmp_path / "lambda.fastq"
    _lambda_fastq(lambda_reads, plain)
    p = tmp_path / "lambda.fastq.gz"
    _write(p, bgzf(open(plain, "rb").read()))
    ref = engine.Engine(device=0)
    try:
        ref.configure(k=15, w=5)
        ref.upload(lambda_reads)
        want = ref.find_overlaps_and_create_piles(0.001, 32, False)
    finally:
        ref.close()
    eng.configure(k=15, w=5)
    for host_bases in (0, 1):
        eng.set_host_bases(host_bases)
        eng.set_option("reset_stats", 1)
        rs = eng.upload_files([str(p)], words=True)
        assert {"fastx_read", "fastx_copy", "fastx_inflate", "fastx_parse"} <= set(eng.timings())
        assert np.array_equal(rs.words, lambda_reads.words)
        assert np.array_equal(rs.word_off, lambda_reads.word_off)
        assert np.array_equal(rs.lens, lambda_reads.lens)
        assert np.array_equal(rs.block_quality, lambda_reads.block_quality)
        assert np.array_equal(rs.bq_off, lambda_reads.bq_off)
        assert rs.names == lambda_reads.names
        got = eng.find_overlaps_and_create_piles(0.001, 32, False)
        for k in ("overlaps", "ovl_off", "pile", "pile_off"):
            assert np.array_equal(got[k], want[k]), (host_bases, k)
        assert got["num_mapped"] == want["num_mapped"]
    eng.set_host_bases(-1)


def test_load_sequences_cpp_bgzf(tmp_path, lambda_reads):
    exe = tmp_path / "load_sequences_test"
    subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-I" + os.path.join(ROOT, "include"),
                    "-o", str(exe), os.path.join(HERE, "cpp", "load_sequences_test.cc"),
                    "-L" + os.path.join(ROOT, "raven_b200"), "-lraven_b200", "-lz",
                    "-Wl,-rpath," + os.path.join(ROOT, "raven_b200")], check=True)
    rng = np.random.default_rng(12)
    plain = tmp_path / "l.fastq"
    _lambda_fastq(lambda_reads, plain)
    lq = tmp_path / "l.fastq.gz"
    _write(lq, bgzf(open(plain, "rb").read()))
    fa = tmp_path / "r.fa.gz"
    _write(fa, bgzf(_fasta(rng, 60, blanks=True), cuts=[333]))
    for paths in ([lq], [fa], [fa, lq]):
        out = subprocess.run([str(exe)] + [str(x) for x in paths], stdout=subprocess.PIPE,
                             stderr=subprocess.PIPE)
        assert out.returncode == 0, out.stdout.decode() + out.stderr.decode()
        assert out.stdout.decode().startswith("ok ")
