"""Reading C2 from FASTQ: the drop-in parser, seqio.parse and Engine.upload_files.

    python profiles/fastx_load.py [--rounds 2] [--reads 200000] [--formats plain,gz,bgzf]
                                  [--skip-seqio] [--out DIR]

C2 is bench.py's seeded read set (200 k reads of 10 kb mean, 2 Gbp). It is written as plain
FASTQ, as `gzip -1` FASTQ and as BGZF FASTQ (level 1, members of 65,280 text bytes as bgzip
cuts them, written by tests/test_gpu_bgzf.py's writer) in a temporary directory, with seeded
qualities. For each file, rounds that alternate the routes:
  dropin        main.cc's loop over the drop-in bioparser + biosoup::NucleicAcid
                (profiles/fastx_load.cc, compiled into the temporary directory)
  upload_files  rvn_reads_upload_files on a fresh context, with its phase split:
                fastx_read (read or inflate that nothing hid), fastx_copy, fastx_inflate
                (BGZF only), fastx_parse
  seqio         seqio.parse, once per file (it takes tens of seconds)
Wall times are host clocks around calls that end when the set is built. The kernels' rate is
their algorithmic bytes (the line index and the pack read the text three times, the words and
block qualities are written once) over fastx_parse, against the H100's 3.35 TB/s; the copy
rate is the bytes copied (the text, or the BGZF file's compressed bytes) over fastx_copy; the
inflate rate is the text bytes over fastx_inflate. Last, the stage-1 result after upload_files
of the plain and the BGZF file must have the sha256 of the one after upload of the same set.

Needs an H100; prints the card's name and power limit with the numbers. The files are read
right after they were written, so they are likely in the page cache.
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from index_chunks import FREQ, GENOME, K, KMAX, MEAN_LEN, READS, SEED, W, card  # noqa: E402

HBM = 3.35e12


def write_fastq(rs, path, seed):
    rng = np.random.default_rng(seed)
    acgt = np.frombuffer(b"ACGT", np.uint8)
    shifts = np.arange(32, dtype=np.uint64) * np.uint64(2)
    with open(path, "wb") as f:
        for a in range(0, rs.n, 1000):
            b = min(rs.n, a + 1000)
            w = rs.words[int(rs.word_off[a]):int(rs.word_off[b])]
            codes = ((w[:, None] >> shifts[None, :]) & np.uint64(3)).astype(np.uint8).reshape(-1)
            for i in range(a, b):
                o = (int(rs.word_off[i]) - int(rs.word_off[a])) * 32
                n = int(rs.lens[i])
                q = rng.integers(33, 75, n, dtype=np.uint8)
                f.write(b"@read%d runid=c2 ch=%d\n" % (i, i % 512))
                f.write(acgt[codes[o:o + n]].tobytes())
                f.write(b"\n+\n")
                f.write(q.tobytes())
                f.write(b"\n")


def write_bgzf(src, path):
    """src as BGZF at level 1, members of 65,280 text bytes, compressed on all cores"""
    from concurrent.futures import ThreadPoolExecutor
    from test_gpu_bgzf import BGZIP_CUT, EOF_MARKER, member
    with open(src, "rb") as f, open(path, "wb") as out, ThreadPoolExecutor() as pool:
        while True:
            block = f.read(BGZIP_CUT * 1024)
            if not block:
                break
            parts = [block[i:i + BGZIP_CUT] for i in range(0, len(block), BGZIP_CUT)]
            for m in pool.map(member, parts):
                out.write(m)
        out.write(EOF_MARKER)


def digest(res):
    h = hashlib.sha256()
    for k in ("overlaps", "ovl_off", "pile", "pile_off"):
        h.update(np.ascontiguousarray(res[k]).tobytes())
    return h.hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--reads", type=int, default=READS)
    ap.add_argument("--formats", default="plain,gz,bgzf")
    ap.add_argument("--skip-seqio", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    from bench import synth
    from raven_b200 import engine, seqio
    torch.cuda.init()
    genome = GENOME * args.reads // READS
    rs = synth.make_reads(SEED, genome, args.reads, MEAN_LEN)
    out = dict(card=card(), reads=rs.n, bases=rs.bases, routes={})
    print("card:", out["card"], "reads:", rs.n, "bases:", rs.bases, flush=True)
    formats = args.formats.split(",")
    tmp = tempfile.mkdtemp(prefix="fastx_load_")
    try:
        plain = os.path.join(tmp, "c2.fastq")
        gz = plain + ".gz"
        bgz = os.path.join(tmp, "c2.bgzf.fastq.gz")
        write_fastq(rs, plain, SEED)
        print("wrote", plain, os.path.getsize(plain), "bytes", flush=True)
        if "gz" in formats and shutil.which("gzip"):
            with open(gz, "wb") as f:
                subprocess.run(["gzip", "-1", "-c", plain], stdout=f, check=True)
        elif "gz" in formats:
            import gzip
            with open(plain, "rb") as src, gzip.open(gz, "wb", compresslevel=1) as dst:
                shutil.copyfileobj(src, dst, 1 << 24)
        if "bgzf" in formats:
            write_bgzf(plain, bgz)
        text = os.path.getsize(plain)
        out.update(text_bytes=text, gz_bytes=os.path.getsize(gz) if "gz" in formats else None,
                   bgzf_bytes=os.path.getsize(bgz) if "bgzf" in formats else None)
        exe = os.path.join(tmp, "fastx_load")
        subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-I" + os.path.join(ROOT, "include"),
                        "-o", exe, os.path.join(ROOT, "profiles", "fastx_load.cc"), "-lz"],
                       check=True)
        kernel_bytes = 3 * text + rs.words.size * 8 + (rs.bases + 63) // 64
        for name, path in (("plain", plain), ("gz", gz), ("bgzf", bgz)):
            if name not in formats:
                continue
            rec = dict(dropin_s=[], upload_files_s=[], phases=[])
            for _ in range(args.rounds):
                t0 = time.perf_counter()
                got = subprocess.run([exe, path], check=True, stdout=subprocess.PIPE).stdout
                rec["dropin_s"].append(time.perf_counter() - t0)
                assert int(got.split()[0]) == rs.n, got
                eng = engine.Engine(device=0)
                try:
                    t0 = time.perf_counter()
                    parsed = eng.upload_files([path])
                    rec["upload_files_s"].append(time.perf_counter() - t0)
                    tm = eng.timings()
                finally:
                    eng.close()
                assert parsed.n == rs.n and np.array_equal(parsed.lens, rs.lens)
                ph = {k: tm.get(k, 0.0)
                      for k in ("fastx_read", "fastx_copy", "fastx_inflate", "fastx_parse")}
                ph["kernel_TBps"] = kernel_bytes / (ph["fastx_parse"] * 1e-3) / 1e12
                ph["kernel_share_of_hbm"] = kernel_bytes / (ph["fastx_parse"] * 1e-3) / HBM
                copied = os.path.getsize(path) if name == "bgzf" else text
                ph["copy_GBps"] = copied / (ph["fastx_copy"] * 1e-3) / 1e9
                if ph["fastx_inflate"]:
                    ph["inflate_GBps"] = text / (ph["fastx_inflate"] * 1e-3) / 1e9
                rec["phases"].append(ph)
                print(name, "dropin %.2f s" % rec["dropin_s"][-1],
                      "upload_files %.2f s" % rec["upload_files_s"][-1],
                      {k: round(v, 3) for k, v in ph.items()}, flush=True)
            if not args.skip_seqio:
                t0 = time.perf_counter()
                s = seqio.parse(path)
                rec["seqio_s"] = time.perf_counter() - t0
                assert s.n == rs.n
                print(name, "seqio %.2f s" % rec["seqio_s"], flush=True)
            out["routes"][name] = rec
        # the stage-1 result after upload_files is the one after upload of the same set
        digests = []
        sources = [None, plain] + ([bgz] if "bgzf" in formats else [])
        for src in sources:
            eng = engine.Engine(device=0)
            try:
                eng.configure(K, W)
                if src is None:
                    eng.upload(rs)
                else:
                    eng.upload_files([src])
                digests.append(digest(eng.find_overlaps_and_create_piles(FREQ, KMAX, False)))
            finally:
                eng.close()
        out["stage1_sha256"] = digests
        print("stage-1 sha256 upload / upload_files (plain, bgzf):", *digests, flush=True)
        assert len(set(digests)) == 1
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "fastx_load.json"), "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
