"""GPU: rvn_reads_upload_files / Engine.upload_files parse FASTA and FASTQ(.gz) text on the
device. The oracle is the drop-in bioparser + biosoup::NucleicAcid (tests/cpp/_build/io_test
parse): ids, names, lengths, words and block qualities must equal it bit for bit, at every
chunk size; errors carry its message and leave the context without a read set."""
import ctypes as C
import gzip
import os
import subprocess

import numpy as np
import pytest

from raven_b200 import engine, seqio

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
IO_TEST = os.path.join(HERE, "cpp", "_build", "io_test")
SWEEP = list(range(1, 65)) + [97, 251, 1021, 4093]

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def io_test():
    subprocess.run(["make", "-C", os.path.join(HERE, "cpp"), "host"], check=True,
                   stdout=subprocess.DEVNULL)
    return IO_TEST


@pytest.fixture(scope="module")
def eng():
    e = engine.Engine(device=0)
    yield e
    e.close()


def _kind(path):
    p = str(path)
    return "fastq" if p.endswith((".fastq", ".fq", ".fastq.gz", ".fq.gz")) else "fasta"


def _oracle(io_test, paths):
    """main.cc's loop over the drop-in parser: (names, ascii sequences, block qualities)"""
    names, seqs, bqs = [], [], []
    for path in paths:
        out = subprocess.run([io_test, "parse", _kind(path), str(path)], check=True,
                             stdout=subprocess.PIPE).stdout
        for line in out.split(b"\n"):
            if not line:
                continue
            _, name, seq, bq = line.split(b"\t")
            names.append(name.decode(errors="surrogateescape"))
            seqs.append(seq)
            bqs.append(np.array([int(x) for x in bq.split(b",") if x], np.uint8))
    return names, seqs, bqs


def _write(path, data, gz=False, members=1):
    if not gz:
        open(path, "wb").write(data)
        return
    with open(path, "wb") as f:  # (several members: a concatenated gzip file)
        cut = [len(data) * i // members for i in range(members + 1)]
        for a, b in zip(cut, cut[1:]):
            f.write(gzip.compress(data[a:b], compresslevel=1))


def _check(eng, io_test, paths, chunks=(0,)):
    names, seqs, bqs = _oracle(io_test, paths)
    want = seqio.pack_ascii(seqs) if seqs else None
    for chunk in chunks:
        eng.set_option("fastx_chunk_bytes", chunk)
        rs = eng.upload_files([str(p) for p in paths], words=True)
        assert rs.n == len(names) == eng.n_reads, chunk
        assert rs.names == names, chunk
        if not names:
            continue
        assert np.array_equal(rs.lens, want.lens), chunk
        assert np.array_equal(rs.word_off, want.word_off), chunk
        assert np.array_equal(rs.words, want.words), chunk
        got_bq = [rs.block_quality[int(rs.bq_off[i]):int(rs.bq_off[i + 1])]
                  for i in range(rs.n)]
        for i, (g, w) in enumerate(zip(got_bq, bqs)):
            assert np.array_equal(g, w), (chunk, i)
    eng.set_option("fastx_chunk_bytes", 0)
    return len(names)


def _seq(rng, n, letters="ACGT"):
    return "".join(rng.choice(list(letters), n)).encode()


LENGTHS = [1, 31, 32, 33, 63, 64, 65, 200, 1000]


def _fasta(rng, width, crlf=False, blanks=False, last_newline=True, spaces=False,
           letters="ACGTacgtRYKMSWBDHVNUu-"):
    nl = b"\r\n" if crlf else b"\n"
    out = bytearray()
    if blanks:
        out += nl + b"\n"
    for i, n in enumerate(LENGTHS):
        s = _seq(rng, n, letters)
        out += b">read%d some\tdescription %d" % (i, i) + nl
        for k in range(0, n, width):
            line = s[k:k + width]
            if spaces and len(line) > 2:
                line = line[:1] + b" \t" + line[1:]
            out += line + nl
        if blanks:
            out += b" \t" + nl + nl
    if not last_newline:
        out = out.rstrip(b"\r\n")
    return bytes(out)


def _qual(rng, n, low_high=False):
    q = rng.integers(33, 127, n).astype(np.uint8)
    if low_high:
        # below '!' (not a space, tab, CR or LF) and above '~', signed-char wrap included
        odd = np.array([1, 2, 8, 11, 12, 31, 127, 128, 200, 255], np.uint8)
        q[rng.integers(0, n, max(1, n // 4))] = rng.choice(odd, max(1, n // 4))
    return q.tobytes()


def _fastq(rng, wrap=None, crlf=False, blanks=False, last_newline=True, spaces=False,
           low_high=False, at_plus=False):
    nl = b"\r\n" if crlf else b"\n"
    out = bytearray()
    if blanks:
        out += nl
    for i, n in enumerate(LENGTHS):
        s = _seq(rng, n, "ACGTacgtN")
        q = bytearray(_qual(rng, n, low_high))
        if at_plus:
            q[0] = ord("@") if i % 2 else ord("+")
        q = bytes(q)
        out += b"@read%d runid=x\tch=%d" % (i, i) + nl
        w = wrap or n
        for k in range(0, n, w):
            line = s[k:k + w]
            if spaces and len(line) > 2:
                line = line[:1] + b"\t " + line[1:]
            out += line + nl
        out += (b"+read%d" % i if i % 3 == 0 else b"+") + nl
        wq = (wrap + 7) if wrap else n
        for k in range(0, n, wq):
            line = q[k:k + wq]
            if spaces and len(line) > 2:
                line = line[:2] + b" " + line[2:]
            out += line + nl
        if blanks:
            out += nl
    if not last_newline:
        out = out.rstrip(b"\r\n")
    return bytes(out)


@pytest.mark.parametrize("width", [1, 60, 80])
def test_fasta_wrapped(eng, io_test, tmp_path, width):
    rng = np.random.default_rng(width)
    p = tmp_path / "r.fasta"
    _write(p, _fasta(rng, width))
    assert _check(eng, io_test, [p], chunks=(0, 13, 4096)) == len(LENGTHS)


@pytest.mark.parametrize("variant", ["blanks", "crlf", "no_last_newline", "spaces",
                                     "crlf_blanks_spaces"])
def test_fasta_text_edges_every_chunk_size(eng, io_test, tmp_path, variant):
    rng = np.random.default_rng(len(variant))
    kw = dict(blanks="blanks" in variant, crlf="crlf" in variant,
              last_newline=variant != "no_last_newline", spaces="spaces" in variant)
    p = tmp_path / "r.fa"
    _write(p, _fasta(rng, 37, **kw))
    assert _check(eng, io_test, [p], chunks=[0] + SWEEP) == len(LENGTHS)


@pytest.mark.parametrize("variant", ["four_line", "multi_line", "crlf", "no_last_newline",
                                     "spaces", "low_high", "at_plus", "blanks",
                                     "multi_line_at_plus_crlf"])
def test_fastq_every_chunk_size(eng, io_test, tmp_path, variant):
    rng = np.random.default_rng(len(variant) + 100)
    kw = dict(wrap=23 if "multi_line" in variant else None, crlf="crlf" in variant,
              last_newline=variant != "no_last_newline", spaces="spaces" in variant,
              low_high=variant == "low_high", at_plus="at_plus" in variant,
              blanks=variant == "blanks")
    p = tmp_path / "r.fastq"
    _write(p, _fastq(rng, **kw))
    assert _check(eng, io_test, [p], chunks=[0] + SWEEP) == len(LENGTHS)


@pytest.mark.parametrize("kind", ["fasta", "fastq"])
def test_long_read(eng, io_test, tmp_path, kind):
    rng = np.random.default_rng(5)
    n = (1 << 20) + 12345
    s = _seq(rng, n)
    if kind == "fasta":
        text = b">long\n" + b"\n".join(s[k:k + 60] for k in range(0, n, 60)) + b"\n>short\nACG\n"
    else:
        text = (b"@long x\n" + s + b"\n+\n" + _qual(rng, n) + b"\n@short\nACG\n+\nIII\n")
    p = tmp_path / ("r." + kind)
    _write(p, text)
    assert _check(eng, io_test, [p], chunks=(0, 65536, 999983)) == 2


@pytest.mark.parametrize("members", [1, 3])
def test_gzip(eng, io_test, tmp_path, members):
    rng = np.random.default_rng(members)
    fq = tmp_path / "r.fq.gz"
    _write(fq, _fastq(rng, wrap=41, blanks=True), gz=True, members=members)
    fa = tmp_path / "r.fasta.gz"
    _write(fa, _fasta(rng, 60, crlf=True), gz=True, members=members)
    assert _check(eng, io_test, [fq], chunks=(0, 7, 333)) == len(LENGTHS)
    assert _check(eng, io_test, [fa], chunks=(0, 7, 333)) == len(LENGTHS)


def test_several_files_with_an_empty_one(eng, io_test, tmp_path):
    rng = np.random.default_rng(9)
    a, b, c, d = (tmp_path / "a.fasta", tmp_path / "b.fastq", tmp_path / "c.fq",
                  tmp_path / "d.fa.gz")
    _write(a, _fasta(rng, 60))
    _write(b, b"")
    _write(c, _fastq(rng))
    _write(d, _fasta(rng, 17, blanks=True), gz=True)
    assert _check(eng, io_test, [a, b, c, d], chunks=(0, 11, 500)) == 3 * len(LENGTHS)
    rs = eng.upload_files([str(b)])
    assert rs.n == 0 and eng.n_reads == 0


def _rc(eng):
    return eng.lib.rvn_minimize(eng.h, 0, 0, 0)


ERRORS = [
    ("lead.fasta", b"ACGT\n>x\nAC\n"),
    ("space_lead.fa", b"\n \n>x\nAC\n"),
    ("noname.fasta", b">x\nAC\n>\nACGT\n"),
    ("spacename.fasta", b"> x\nAC\n"),
    ("nodata.fasta", b">x\n>y\nAC\n"),
    ("nodata_end.fasta", b">x\nAC\n>y\n\n"),
    ("nuc.fasta", b">x\nAC!T\n"),
    ("nuc_before_invalid.fasta", b">x\nACGT\n>y\nNNXN\n>z\n\n"),
    ("short.fastq", b"@x\nACGT\n+\nII\n"),
    ("long.fastq", b"@x\nACGT\n+\nIIIII\n"),
    ("header.fastq", b"@a\nAC\n+\nII\nx\nACGT\n+\nIIII\n"),
    ("space_header.fq", b" \n@x\nACGT\n+\nIIII\n"),
    ("noplus.fastq", b"@x\nACGT\n"),
    ("noname.fastq", b"@\nACGT\n+\nIIII\n"),
    ("nodata.fastq", b"@x\n+\n@y\nAC\n+\nII\n"),
    ("nuc.fastq", b"@x\nAC!T\n+\nIIII\n"),
    ("nuc_first.fastq", b"@x\nACGT\n+\nIIII\n@y\nACXT\n+\nIIII\n@z\nAC\n+\nI\n"),
    ("invalid_first.fq", b"@x\nACGT\n+\nIIII\n@\nACXT\n+\nIIII\n@z\nAX\n+\nI\n"),
]


@pytest.mark.parametrize("name,text", ERRORS, ids=[e[0] for e in ERRORS])
def test_errors_carry_the_dropin_message(eng, io_test, tmp_path, name, text):
    p = tmp_path / name
    _write(p, text)
    out = subprocess.run([io_test, "parse", _kind(p), str(p)], stdout=subprocess.PIPE)
    assert out.returncode == 3
    what = out.stdout.decode().strip().split("invalid_argument: ", 1)[1]
    good = tmp_path / "good.fasta"
    _write(good, b">g\nACGT\n")
    for chunk in (0, 1, 5, 64):
        eng.set_option("fastx_chunk_bytes", chunk)
        eng.upload_files([str(good)])
        with pytest.raises(ValueError) as e:
            eng.upload_files([str(good), str(p)])
        assert str(e.value) == f"{what} ({p})", chunk
        assert _rc(eng) == -3  # RVN_ERR_STATE: no read set
        assert eng.lib.rvn_reads_parsed(eng.h, None, None, None, None, None, None, None) == -3
    eng.set_option("fastx_chunk_bytes", 0)


def test_file_errors(eng, tmp_path):
    good = tmp_path / "good.fq"
    _write(good, b"@g\nACGT\n+\nIIII\n")
    missing = str(tmp_path / "missing.fasta")
    with pytest.raises(ValueError) as e:
        eng.upload_files([str(good), missing])
    assert str(e.value) == "[bioparser::Parser::Create] error: unable to open file " + missing
    assert _rc(eng) == -3
    bad = str(tmp_path / "reads.txt")
    _write(bad, b">x\nACGT\n")
    with pytest.raises(ValueError) as e:
        eng.upload_files([str(good), bad])
    assert str(e.value) == (
        "[raven::CreateParser] error: file " + bad + " has unsupported format extension "
        "(valid extensions: .fasta, .fasta.gz, .fa, .fa.gz, .fastq, .fastq.gz, .fq, .fq.gz)")
    assert _rc(eng) == -3
    # the first failing file in order decides
    broken = tmp_path / "broken.fastq"
    _write(broken, b"@x\nAC\n")
    with pytest.raises(ValueError) as e:
        eng.upload_files([str(broken), bad])
    assert "FastqParser" in str(e.value)
    # a later upload makes a read set again
    eng.upload_files([str(good)])
    assert _rc(eng) == 0


def _lambda_fastq(rs, path):
    out = bytearray()
    for i in range(rs.n):
        bq = rs.block_quality[int(rs.bq_off[i]):int(rs.bq_off[i + 1])]
        q = np.repeat(bq.astype(np.uint16) + 33, 64)[:int(rs.lens[i])].astype(np.uint8)
        out += b"@" + rs.names[i].encode() + b" lambda\n" + rs.ascii(i) + b"\n+\n"
        out += q.tobytes() + b"\n"
    _write(path, bytes(out))


def test_lambda_end_to_end(eng, tmp_path, lambda_reads):
    p = tmp_path / "lambda.fastq"
    _lambda_fastq(lambda_reads, p)
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
        rs = eng.upload_files([str(p)], words=True)
        assert {"fastx_read", "fastx_copy", "fastx_parse"} <= set(eng.timings())
        assert eng.reads_residency()["on_host"] == bool(host_bases)
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


def test_load_sequences_cpp(tmp_path, lambda_reads):
    exe = tmp_path / "load_sequences_test"
    subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-I" + os.path.join(ROOT, "include"),
                    "-o", str(exe), os.path.join(HERE, "cpp", "load_sequences_test.cc"),
                    "-L" + os.path.join(ROOT, "raven_b200"), "-lraven_b200", "-lz",
                    "-Wl,-rpath," + os.path.join(ROOT, "raven_b200")], check=True)
    rng = np.random.default_rng(11)
    fa, fq, gz = tmp_path / "r.fasta", tmp_path / "r.fastq", tmp_path / "l.fastq.gz"
    _write(fa, _fasta(rng, 60, blanks=True))
    _write(fq, _fastq(rng, wrap=30, at_plus=True))
    plain = tmp_path / "l.fastq"
    _lambda_fastq(lambda_reads, plain)
    _write(gz, open(plain, "rb").read(), gz=True, members=2)
    for paths in ([fa], [fq], [gz], [fa, fq, gz]):
        out = subprocess.run([str(exe)] + [str(x) for x in paths], stdout=subprocess.PIPE,
                             stderr=subprocess.PIPE)
        assert out.returncode == 0, out.stdout.decode() + out.stderr.decode()
        assert out.stdout.decode().startswith("ok ")
