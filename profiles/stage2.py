"""Stage 2's fast route (raven_b200::FindOverlapsAndRepetetiveRegions over the one device
call rvn_find_overlaps_and_repetitive_regions) timed against the route it replaced (per
batch rvn_minimize / rvn_filter / rvn_map, Pile::AddKmers serially on the host, the
identity filter through rvn_edit_distance_batch), alternating in one process on the same
reads, by oracle/_ref/stage2_time (profiles/stage2_time.cc, built by build() where the
reference tree exists). Only stage 2 is timed; stage 1 and the pile steps before it run
anew before every timed call.

Sets: C2's read model (bench.py: uniform random genome, 40x ONT-like reads of ~10 kb
with 10 % error) on a smaller genome, and a seeded repeat-rich genome of the same size
(raven_b200.synth.repeat_genome: interspersed repeat families and tandem repeats) under
the same read model. Reports the card and its power limit, per route and run the stage-2
seconds, the filtered positions the previous route handed to Pile::AddKmers, and a
digest of the end state (every overlap list, every pile's cereal JSON), which must agree.

  python profiles/stage2.py [--genome 5000000] [--reps 3] [--out DIR]
"""
import argparse
import json
import os
import struct
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
BIN = os.path.join(ROOT, "oracle", "_ref", "stage2_time")


def write_reads(path, rs):
    with open(path, "wb") as f:
        for a, dt in ((rs.words, np.uint64), (rs.word_off, np.uint64), (rs.lens, np.uint32)):
            a = np.ascontiguousarray(a, dtype=dt)
            f.write(struct.pack("<Q", a.size))
            f.write(a.tobytes())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genome", type=int, default=5_000_000)
    ap.add_argument("--coverage", type=int, default=40)
    ap.add_argument("--mean-len", type=int, default=10_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--identity", type=float, default=0.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not os.path.exists(BIN):
        sys.exit("oracle/_ref/stage2_time not built (build() needs the reference tree)")
    from bench import synth as bsynth
    from raven_b200 import synth
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit",
                           "--format=csv,noheader"], stdout=subprocess.PIPE, text=True,
                          check=True).stdout.strip()
    print("card:", card, flush=True)
    n_reads = a.genome * a.coverage // a.mean_len
    sets = {
        "c2_model": lambda: bsynth.make_reads(11, a.genome, n_reads, a.mean_len),
        "repeat_rich": lambda: synth.make_reads(
            genome=synth.repeat_genome(a.genome, families=a.genome // 25_000, copies=12,
                                       family_len=3000, tandem_every=4000, seed=12),
            n_reads=n_reads, mean_len=a.mean_len, seed=13, min_len=2000),
    }
    lines = [f"card: {card}"]
    with tempfile.TemporaryDirectory() as tmp:
        for name, make in sets.items():
            rs = make()
            path = os.path.join(tmp, name + ".bin")
            write_reads(path, rs)
            del rs
            out = subprocess.run([BIN, path, "15", "5", "0.001", str(a.identity), str(a.reps)],
                                 stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True,
                                 check=True).stdout
            runs = [json.loads(x) for x in out.splitlines() if x.startswith("{")]
            digests = {r["digest"] for r in runs}
            prev = [r["seconds"] for r in runs if r["route"] == "previous"]
            new = [r["seconds"] for r in runs if r["route"] == "one_call"]
            summary = (f"{name}: {n_reads} reads, genome {a.genome}, identity {a.identity}: "
                       f"filtered positions {runs[0]['filtered_positions']}, final overlaps "
                       f"{runs[0]['final_overlaps']}; stage 2 previous route "
                       f"{' '.join(f'{x:.3f}' for x in prev)} s, one call "
                       f"{' '.join(f'{x:.3f}' for x in new)} s; digests "
                       f"{'identical' if len(digests) == 1 else 'DIFFER'}")
            print(summary, flush=True)
            lines.append(summary)
            lines += [json.dumps(r) for r in runs]
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "stage2.txt"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
