"""One-shot against chunked rvn_minimize (option "index_chunk_bases") followed by rvn_filter
and rvn_map of all reads: time per pass, device memory and per-phase times.

    python profiles/minimize_chunks.py [--rounds 3] [--large-reads N] [--out DIR]

1. C2, the seeded set of bench.py (200 k reads, 2 Gbp): rounds that alternate a one-shot
   pass and a pass forced into chunks of 2^30 bases, each in a fresh context: minimize,
   filter, map of every read (stage 1's flags). Per round and mode: ms per pass (host clock
   around calls that end in a stream synchronise), the peak device memory in use during
   the pass (sampled every millisecond from another thread), the memory the context still
   holds afterwards, the per-phase device times, the flushes of the map and a digest of
   the index records' count, the threshold and the map results, which must be equal.
   (Sweep 2 of the untiered chunked build has one route per (k, w); the sketch-then-copy
   route of other parameters cannot be selected at k15 w5, so it is not timed here.)
2. A set with a full 2^32-base index batch and a small second one (--large-reads reads of
   10 kb mean; 0 skips it), default options, in the reference's order: per batch Minimize,
   Filter, map of the earlier reads, map of the batch. Reports that it completes, its peak
   and its time, once.

Needs an H100; prints the card's name and power limit with the numbers. --out DIR also
writes them as DIR/minimize_chunks.json.
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from index_chunks import FREQ, GENOME, K, MEAN_LEN, READS, SEED, W, PeakMemory, card  # noqa: E402

PHASES = ("sketch", "sketch_tiers", "micromize", "index_sort", "index_table", "probe", "expand",
          "map_flush")


def batches(rs, batch_bases):
    out, bases, j = [], 0, 0
    for i in range(rs.n):
        bases += int(rs.lens[i])
        if i != rs.n - 1 and bases < batch_bases:
            continue
        out.append((j, i + 1))
        bases, j = 0, i + 1
    return out


def run(rs, chunk, ib=1 << 32):
    """one fresh context, one pass in the reference's order: ms, peak and held device
    bytes, chunked?, flushes, phases, digest"""
    import torch
    from raven_b200 import engine
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    h = hashlib.sha256()
    with PeakMemory() as pm:
        eng = engine.Engine(device=0)
        try:
            eng.configure(K, W)
            eng.set_index_chunks(chunk)
            eng.upload(rs)
            t0 = time.perf_counter()
            for j, last in batches(rs, ib):
                eng.minimize(j, last, False)
                h.update(str(eng.filter(FREQ)).encode())
                for first, end in ((0, j), (j, last)):
                    if first == end:
                        continue
                    r = eng.map(first, end, True, True, True, False)
                    h.update(r["overlaps"].tobytes())
                    h.update(r["ovl_off"].tobytes())
            ms = (time.perf_counter() - t0) * 1e3
            held = free0 - torch.cuda.mem_get_info()[0]
            tm = eng.timings()
            h.update(str(eng.stats()["index_records"]).encode())
            return dict(ms_per_pass=round(ms, 1), gb_peak=round((pm.peak - pm.base) / 1e9, 2),
                        gb_held=round(held / 1e9, 2), chunked=eng.minimize_chunked(),
                        map_flushes=eng.map_flushes(),
                        phases={p: round(tm[p], 2) for p in PHASES if p in tm},
                        digest=h.hexdigest()[:16])
        finally:
            eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--large-reads", type=int, default=440_000)
    ap.add_argument("--out", default=None, metavar="DIR")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("minimize_chunks.py needs a CUDA device")
    from bench import synth

    dev = card()
    print(f"card: {dev}", flush=True)
    out = {"card": dev, "c2": [], "large": None}
    rs = synth.make_reads(SEED, GENOME, READS, MEAN_LEN)
    print(f"C2: {rs.n} reads, {int(rs.lens.sum()) / 1e9:.2f} Gbp", flush=True)
    run(rs, 0)   # (warm-up: module load, pinned result buffers of the process)
    for r in range(a.rounds):
        for chunk, name in ((0, "one-shot"), (1 << 30, "chunks 2^30")):
            e = run(rs, chunk)
            e.update(round=r, mode=name)
            out["c2"].append(e)
            print(f"  {r} {name:<12} {json.dumps(e)}", flush=True)
    out["c2_identical"] = len({e["digest"] for e in out["c2"]}) == 1
    print(f"  results identical: {out['c2_identical']}", flush=True)
    del rs

    if a.large_reads:
        n = a.large_reads
        rs = synth.make_reads(SEED + 11, n * MEAN_LEN // 40, n, MEAN_LEN)
        gbp = int(rs.lens.sum()) / 1e9
        print(f"large: {rs.n} reads, {gbp:.2f} Gbp, batches {batches(rs, 1 << 32)}", flush=True)
        try:
            e = run(rs, -1)
        except RuntimeError as err:
            e = {"error": str(err)}
        out["large"] = dict(e, reads=rs.n, gbp=round(gbp, 2))
        print(f"  default      {json.dumps(out['large'])}", flush=True)
        out["device_gb"] = round(torch.cuda.mem_get_info()[1] / 1e9, 1)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "minimize_chunks.json"), "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
