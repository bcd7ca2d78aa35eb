"""Stage-1 and stage-2 times of the reference's own `raven` executable, built
unmodified over the ram::MinimizerEngine facade (oracle/Makefile `_ref/raven`),
on seeded synthetic ONT reads (bench/synth, the benchmark's C2 read model).

Each run is `raven -t T -p 0 reads.fasta`; the times are the reference's own
stderr lines ("minimized ...", "mapped sequences", "mapped valid sequences"),
and the run is stopped once stage 2 has printed its map time. With --baseline,
the runs alternate between that binary (e.g. `_ref/raven` built from an earlier
commit by the same recipe) and the current one. Beside them, the batched
replacements on the same reads: `_ref/dropin_test` part B (stage 1) and
`_ref/stage2_test` mode 1 (stage 2), whose "(GPU)" lines are reported.

The card's name and power limit are read at the start of the run. Output: a
table on stdout; --out DIR also writes facade_cli_stages.json there.
  usage: python profiles/facade_cli_stages.py [--reads 20000 200000] [--rounds 2]
             [--baseline PATH] [--threads 16] [--timeout 900] [--out DIR]"""
import argparse
import json
import os
import re
import shutil
import struct
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF_BIN = os.path.join(ROOT, "oracle", "_ref")
SEED = 20260924  # bench.py's
LINE = re.compile(r"\[raven::Graph::Construct\] (.*?) ?([0-9.]+)s$")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       check=True, stdout=subprocess.PIPE, text=True).stdout
    return q.strip().split("\n")[0]


def write_inputs(rs, d):
    """reads.fasta for raven, reads.bin (words, offsets, lengths) for the drivers."""
    with open(os.path.join(d, "reads.bin"), "wb") as f:
        for a, dt in ((rs.words, np.uint64), (rs.word_off, np.uint64), (rs.lens, np.uint32)):
            a = np.ascontiguousarray(a, dtype=dt)
            f.write(struct.pack("<Q", a.size))
            f.write(a.tobytes())
    lut = np.frombuffer(b"ACGT", dtype=np.uint8)
    shifts = np.arange(32, dtype=np.uint64) * np.uint64(2)
    with open(os.path.join(d, "reads.fasta"), "wb") as f:
        step = 4096
        for r0 in range(0, rs.n, step):
            r1 = min(rs.n, r0 + step)
            w0, w1 = int(rs.word_off[r0]), int(rs.word_off[r1])
            codes = ((rs.words[w0:w1, None] >> shifts[None, :]) & np.uint64(3)).astype(np.uint8)
            text = lut[codes.reshape(-1)]
            for i in range(r0, r1):
                b = (int(rs.word_off[i]) - w0) * 32
                f.write(b">%d\n" % i)
                f.write(text[b:b + int(rs.lens[i])].tobytes())
                f.write(b"\n")


def run(cmd, cwd, timeout, stop=None):
    """Phase lines of one run, [(what, seconds)], whether it finished, and its wall
    time; stops the process after the first line that contains `stop`, or when
    `timeout` seconds have passed."""
    t0 = time.monotonic()
    p = subprocess.Popen(cmd, cwd=cwd, stdout=subprocess.DEVNULL, stderr=subprocess.PIPE,
                         text=True)
    watchdog = threading.Timer(timeout, p.kill)
    watchdog.start()
    lines, done = [], False
    try:
        for raw in p.stderr:
            m = LINE.search(raw.strip())
            if m:
                lines.append((m.group(1), float(m.group(2))))
                if stop and stop in m.group(1):
                    done = True
                    break
    finally:
        watchdog.cancel()
        if p.poll() is None:
            p.kill()
        p.wait()
    finished = done if stop else p.returncode == 0
    return lines, finished, time.monotonic() - t0


def stages(lines):
    """Reference lines -> seconds of stage 1 (minimize, map) and stage 2 (minimize, map)."""
    out = dict(s1_minimize=0.0, s1_map=0.0, s2_minimize=0.0, s2_map=0.0)
    stage = 1
    for what, s in lines:
        if what.startswith("minimized"):
            out[f"s{stage}_minimize"] += s
        elif what == "mapped sequences":
            out["s1_map"] += s
        elif what == "mapped valid sequences":
            out["s2_map"] += s
        elif what.startswith("removed chimeric"):
            stage = 2
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, nargs="+", default=[20_000, 200_000])
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--baseline", default=None, help="an earlier build of _ref/raven")
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--timeout", type=float, default=900.0, help="seconds per run")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from bench import synth

    raven = os.path.join(REF_BIN, "raven")
    builds = [("current", raven)]
    if a.baseline:
        builds.insert(0, ("baseline", os.path.abspath(a.baseline)))
    result = dict(card=card(), threads=a.threads, sizes=[])
    print("card:", result["card"])
    for n in a.reads:
        genome = max(50_000_000 * n // 200_000, 80_000)  # the C2 coverage
        rs = synth.make_reads(SEED, genome, n, 10_000)
        d = tempfile.mkdtemp(prefix="raven_cli_")
        try:
            write_inputs(rs, d)
            size = dict(reads=n, bases=rs.bases, runs=[])
            for r in range(a.rounds):
                for name, binary in builds:
                    lines, finished, wall = run(
                        [binary, "-t", str(a.threads), "-p", "0", "reads.fasta"], d, a.timeout,
                        stop="mapped valid sequences")
                    # (an unfinished run reports the phases it printed)
                    rec = dict(build=name, round=r, wall_s=round(wall, 1), finished=finished,
                               **stages(lines))
                    size["runs"].append(rec)
                    print(n, rec, flush=True)
            inp = os.path.join(d, "reads.bin")
            lines, _, _ = run([os.path.join(REF_BIN, "dropin_test"), inp, "out.bin", "15", "5",
                               "0.001", "32", "0"], d, a.timeout)
            gpu = [s for what, s in lines if what.endswith("(GPU)")]
            size["batched_stage1_s"] = gpu[0] if gpu else None
            lines, _, _ = run([os.path.join(REF_BIN, "stage2_test"), inp, "out.bin", "15", "5",
                               "0.001", "0"], d, a.timeout)
            gpu = [s for what, s in lines if "valid sequences (GPU)" in what]
            size["batched_stage2_s"] = sum(gpu) if gpu else None
            print(n, "batched replacements: stage 1", size["batched_stage1_s"], "s, stage 2",
                  size["batched_stage2_s"], "s", flush=True)
            result["sizes"].append(size)
        finally:
            shutil.rmtree(d, ignore_errors=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "facade_cli_stages.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
