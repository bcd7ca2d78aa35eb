"""Packed bases on the device against bases in pinned host memory (option "host_bases"):
time per stage-1 pass, the copy time no kernel hid, device memory and digests.

    python profiles/host_bases.py [--rounds 3] [--steps 3] [--large-reads N] [--out DIR]

1. C2, the seeded set of bench.py (200 k reads, 2 Gbp, one index batch), and the same set
   cut into five index batches (bench.py --index-batches 5, whose probe-path flushes stage
   more bytes): rounds that alternate a pass with the bases on the device and one with
   host_bases forced, each in a fresh context. Per round and mode: ms per pass (host clock
   around calls that end in a stream synchronise, after one warm-up pass), phase
   "stage_bases" of the last pass (the copy time no kernel hid), the peak device memory in
   use during the passes (sampled every millisecond from another thread, less what was in
   use before the context), the device bytes of packed words the context holds, and a
   digest of the results, which must be equal.
2. --large-reads N > 0: a seeded set of N reads of 10 kb mean, 40x of a genome sized to
   match, one pass with default arguments (index batches of 2^32 bases, every option
   auto): time, peak device memory, where auto put the bases, and the host's peak
   resident memory.

Needs an H100; prints the card's name and power limit with the numbers. --out DIR also
writes them as DIR/host_bases.json.
"""
from __future__ import annotations

import argparse
import json
import os
import resource
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

from index_chunks import FREQ, GENOME, K, KMAX, MEAN_LEN, READS, SEED, W, PeakMemory, card  # noqa: E402


def run(rs, host, steps, warmup, ib=0):
    """one fresh context: ms per pass, stage_bases of the last pass, peak device bytes,
    device bytes of packed words, residency, digest"""
    import hashlib

    import torch
    from raven_b200 import engine
    torch.cuda.synchronize()
    with PeakMemory() as pm:
        eng = engine.Engine(device=0)
        try:
            eng.configure(K, W)
            eng.set_host_bases(host)
            eng.upload(rs)
            for _ in range(warmup):
                eng.find_overlaps_and_create_piles(FREQ, KMAX, False, ib, fetch=False)
            t = []
            for _ in range(steps):
                t0 = time.perf_counter()
                eng.find_overlaps_and_create_piles(FREQ, KMAX, False, ib, fetch=False)
                t.append((time.perf_counter() - t0) * 1e3)
            tm = eng.timings()
            res = eng.reads_residency()
            r = eng.stage1_results()
            h = hashlib.sha256()
            for k in ("overlaps", "ovl_off", "pile", "pile_off"):
                h.update(r[k].tobytes())
            h.update(str(r["num_mapped"]).encode())
            return dict(ms_per_pass=round(sorted(t)[len(t) // 2], 1),
                        stage_bases_ms=round(tm.get("stage_bases", 0.0), 2),
                        sketch_ms=round(tm.get("sketch", 0.0) + tm.get("sketch_tiers", 0.0), 2),
                        gb_peak=round((pm.peak - pm.base) / 1e9, 2),
                        gb_words=round(res["device_word_bytes"] / 1e9, 3),
                        on_host=res["on_host"], chunked=eng.stage1_index_chunked(),
                        digest=h.hexdigest()[:16])
        finally:
            eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--large-reads", type=int, default=0)
    ap.add_argument("--out", default=None, metavar="DIR")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("host_bases.py needs a CUDA device")
    from bench import synth

    dev = card()
    print(f"card: {dev}", flush=True)
    out = {"card": dev}
    rs = synth.make_reads(SEED, GENOME, READS, MEAN_LEN)
    bases = int(rs.lens.sum())
    print(f"C2: {rs.n} reads, {bases / 1e9:.2f} Gbp", flush=True)
    for name, ib in (("c2", 0), ("c2_5_batches", (bases + 4) // 5)):
        out[name] = []
        for r in range(a.rounds):
            for host in (0, 1):
                e = run(rs, host, a.steps, 1, ib)
                e.update(round=r, mode="host" if host else "device")
                out[name].append(e)
                print(f"  {name} {r} {json.dumps(e)}", flush=True)
        out[name + "_identical"] = len({e["digest"] for e in out[name]}) == 1
        print(f"  {name} results identical: {out[name + '_identical']}", flush=True)
    del rs

    if a.large_reads:
        n = a.large_reads
        rs = synth.make_reads(SEED + 11, n * MEAN_LEN // 40, n, MEAN_LEN)
        gbp = int(rs.lens.sum()) / 1e9
        print(f"large: {rs.n} reads, {gbp:.2f} Gbp", flush=True)
        try:
            e = run(rs, -1, 1, 0)
        except RuntimeError as err:
            e = {"error": str(err)}
        e.update(reads=rs.n, gbp=round(gbp, 2),
                 host_peak_gb=round(resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1e6, 1))
        out["large"] = e
        print(f"  {json.dumps(e)}", flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "host_bases.json"), "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
