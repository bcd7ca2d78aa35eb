"""One-shot against chunked index builds in stage 1 (option "index_chunk_bases"): time per
pass, device memory and per-phase times.

    python profiles/index_chunks.py [--rounds 3] [--steps 3] [--large-reads N] [--out DIR]

1. C2, the seeded set of bench.py (200 k reads, 2 Gbp, one index batch): rounds that
   alternate a one-shot pass and a pass forced into chunks of 2^30 bases, each in a fresh
   context. Per round and mode: ms per pass (host clock around calls that end in a stream
   synchronise, after one warm-up pass), the peak device memory in use during the passes
   (sampled every millisecond from another thread, less what was in use before the
   context), the memory the context still holds afterwards, the per-phase device times of
   the last pass and a digest of the results, which must be equal.
2. A set with a full 2^32-base index batch (--large-reads reads of 10 kb mean, 40x of a
   genome sized to match; 0 skips it), one pass with default arguments (index batches of
   2^32 bases, every option auto): time, peak memory and the modes auto chose. Then the
   same set with chunks of 2^30 and 2^29 bases forced; the digests must be equal.

Needs an H100; prints the card's name and power limit with the numbers. --out DIR also
writes them as DIR/index_chunks.json.
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# the flagship workload of bench.py (C2)
SEED = 20260924
K, W, FREQ, KMAX = 15, 5, 0.001, 32
READS, GENOME, MEAN_LEN = 200_000, 50_000_000, 10_000
PHASES = ("sketch", "sketch_tiers", "micromize", "index_sort", "index_table", "probe",
          "stage1_window")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


class PeakMemory:
    """device memory in use, sampled from another thread while the block runs"""

    def __enter__(self):
        import torch
        self.torch = torch
        self.total = torch.cuda.mem_get_info()[1]
        self.base = self.total - torch.cuda.mem_get_info()[0]
        self.peak = self.base
        self.stop = False
        self.t = threading.Thread(target=self.poll, daemon=True)
        self.t.start()
        return self

    def poll(self):
        while not self.stop:
            used = self.total - self.torch.cuda.mem_get_info()[0]
            self.peak = max(self.peak, used)
            time.sleep(0.001)

    def __exit__(self, *exc):
        self.stop = True
        self.t.join()


def run(rs, chunk, steps, warmup, ib=0):
    """one fresh context: ms per pass, peak and held device bytes, chunked?, windowed?,
    phases of the last pass, digest"""
    import torch
    from raven_b200 import engine
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    with PeakMemory() as pm:
        eng = engine.Engine(device=0)
        try:
            eng.configure(K, W)
            eng.set_index_chunks(chunk)
            eng.upload(rs)
            for _ in range(warmup):
                eng.find_overlaps_and_create_piles(FREQ, KMAX, False, ib, fetch=False)
            t = []
            for _ in range(steps):
                t0 = time.perf_counter()
                eng.find_overlaps_and_create_piles(FREQ, KMAX, False, ib, fetch=False)
                t.append((time.perf_counter() - t0) * 1e3)
            held = free0 - torch.cuda.mem_get_info()[0]
            tm = eng.timings()
            phases = {p: round(tm[p], 2) for p in PHASES if p in tm}
            r = eng.stage1_results()
            h = hashlib.sha256()
            for k in ("overlaps", "ovl_off", "pile", "pile_off"):
                h.update(r[k].tobytes())
            h.update(str(r["num_mapped"]).encode())
            return dict(ms_per_pass=round(sorted(t)[len(t) // 2], 1),
                        gb_peak=round((pm.peak - pm.base) / 1e9, 2),
                        gb_held=round(held / 1e9, 2),
                        chunked=eng.stage1_index_chunked(), windowed=eng.stage1_windowed(),
                        phases=phases, digest=h.hexdigest()[:16])
        finally:
            eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--large-reads", type=int, default=440_000)
    ap.add_argument("--out", default=None, metavar="DIR")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("index_chunks.py needs a CUDA device")
    from bench import synth
    from raven_b200 import engine

    dev = card()
    print(f"card: {dev}", flush=True)
    out = {"card": dev, "c2": [], "large": None}
    rs = synth.make_reads(SEED, GENOME, READS, MEAN_LEN)
    print(f"C2: {rs.n} reads, {int(rs.lens.sum()) / 1e9:.2f} Gbp", flush=True)
    for r in range(a.rounds):
        for chunk, name in ((0, "one-shot"), (1 << 30, "chunks 2^30")):
            e = run(rs, chunk, a.steps, 1)
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
        eng = engine.Engine(device=0)
        try:
            eng.upload(rs)
            fp = {k: round(v / 1e9, 1) for k, v in eng.index_footprint().items()}
            s1 = {k: round(v / 1e9, 1) for k, v in eng.stage1_footprint(KMAX).items()}
        finally:
            eng.close()
        print(f"large: {rs.n} reads, {gbp:.2f} Gbp; index footprint (GB) {fp}, "
              f"stage-1 estimates (GB) {s1}", flush=True)
        out["large"] = {"reads": rs.n, "gbp": round(gbp, 2), "index_footprint_gb": fp,
                        "stage1_estimates_gb": s1, "runs": []}
        for chunk, name in ((-1, "default"), (1 << 30, "chunks 2^30"), (1 << 29, "chunks 2^29")):
            try:
                e = run(rs, chunk, 1, 0)
            except RuntimeError as err:
                e = {"error": str(err)}
            e.update(mode=name)
            out["large"]["runs"].append(e)
            print(f"  {name:<12} {json.dumps(e)}", flush=True)
        digs = {e.get("digest") for e in out["large"]["runs"]}
        out["large"]["identical"] = len(digs) == 1 and None not in digs
        print(f"  results identical: {out['large']['identical']}", flush=True)
        out["device_gb"] = round(torch.cuda.mem_get_info()[1] / 1e9, 1)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "index_chunks.json"), "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
