"""Resident against windowed stage 1 (option "stage1_window"): time per pass and device
memory in use after the call.

    python profiles/stage1_window.py [--rounds 3] [--steps 3] [--large-reads N]
                                     [--large-ib BASES] [--out DIR]

1. C2, the seeded set of bench.py (200 k reads, 2 Gbp): rounds that alternate a resident
   and a forced-windowed pass, each in a fresh context (the device buffers only grow, so
   the memory a context holds after its calls is its peak). Per round and mode: ms per pass
   (host clock around calls that end in a stream synchronise, after one warm-up pass) and
   the device memory the context holds. The results of the two modes are compared.
2. Windowed alone on a larger seeded set (--large-reads reads of 10 kb mean, 40x of a
   genome sized to match; 0 skips it) with index batches of --large-ib bases, one pass
   without warm-up (it includes the first allocation of the pinned host state). The
   resident mode is not run there; the script prints the auto mode's estimates
   (rvn_stage1_footprint) of what each mode would need. (One C2 pass holds about 44 GB for
   its 1.98 Gbp index batch built in one piece, so the default 2^32-base batch fits an 80 GB
   card only built in chunks - option "index_chunk_bases", profiles/index_chunks.py.)

Needs an H100; prints the card's name and power limit with the numbers. --out DIR also
writes them as DIR/stage1_window.json.
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# the flagship workload of bench.py (C2)
SEED = 20260924
K, W, FREQ, KMAX = 15, 5, 0.001, 32
READS, GENOME, MEAN_LEN = 200_000, 50_000_000, 10_000


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def estimates(rs, kmax, ib):
    """the auto mode's estimates (rvn_stage1_footprint) for these reads, in GB"""
    from raven_b200 import engine
    eng = engine.Engine(device=0)
    try:
        eng.upload(rs)
        return {k: round(v / 1e9, 1) for k, v in eng.stage1_footprint(kmax, ib).items()}
    finally:
        eng.close()


def run(rs, mode, steps, warmup, fetch_digest=False, ib=0):
    """one fresh context: (ms per pass, device bytes it holds, windowed?, digest)"""
    import torch
    from raven_b200 import engine
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    eng = engine.Engine(device=0)
    try:
        eng.configure(K, W)
        eng.set_stage1_window(mode)
        eng.upload(rs)
        for _ in range(warmup):
            eng.find_overlaps_and_create_piles(FREQ, KMAX, False, ib, fetch=False)
        t = []
        for _ in range(steps):
            t0 = time.perf_counter()
            eng.find_overlaps_and_create_piles(FREQ, KMAX, False, ib, fetch=False)
            t.append((time.perf_counter() - t0) * 1e3)
        held = free0 - torch.cuda.mem_get_info()[0]
        windowed = eng.stage1_windowed()
        digest = None
        if fetch_digest:
            r = eng.stage1_results()
            h = hashlib.sha256()
            for k in ("overlaps", "ovl_off", "pile", "pile_off"):
                h.update(r[k].tobytes())
            digest = h.hexdigest()[:16]
        return sorted(t)[len(t) // 2], held, windowed, digest
    finally:
        eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--large-reads", type=int, default=1_000_000)
    ap.add_argument("--large-ib", type=int, default=1 << 31)
    ap.add_argument("--out", default=None, metavar="DIR")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("stage1_window.py needs a CUDA device")
    from bench import synth

    dev = card()
    print(f"card: {dev}")
    out = {"card": dev, "c2": [], "large": None}
    rs = synth.make_reads(SEED, GENOME, READS, MEAN_LEN)
    gbp = int(rs.lens.sum()) / 1e9
    est = estimates(rs, KMAX, 0)
    out["c2_estimates_gb"] = est
    print(f"C2: {rs.n} reads, {gbp:.2f} Gbp; estimates (GB) {est}")
    print(f"  {'round':>5} {'mode':<9} {'ms/pass':>9} {'GB held':>8} {'digest':>17}")
    for r in range(a.rounds):
        for mode, name in ((0, "resident"), (1, "windowed")):
            ms, held, win, dig = run(rs, mode, a.steps, 1, fetch_digest=(r == 0))
            assert win == (mode == 1)
            out["c2"].append({"round": r, "mode": name, "ms_per_pass": round(ms, 2),
                              "gb_held": round(held / 1e9, 3), "digest": dig})
            print(f"  {r:>5} {name:<9} {ms:9.1f} {held / 1e9:8.2f} {dig or '':>17}")
    digs = {e["digest"] for e in out["c2"] if e["digest"]}
    print(f"  results identical: {len(digs) == 1}")
    out["c2_identical"] = len(digs) == 1
    del rs

    if a.large_reads:
        n = a.large_reads
        rs = synth.make_reads(SEED + 7, n * MEAN_LEN // 40, n, MEAN_LEN)
        gbp = int(rs.lens.sum()) / 1e9
        est = estimates(rs, KMAX, a.large_ib)
        print(f"large: {rs.n} reads, {gbp:.2f} Gbp, index batches of {a.large_ib} bases",
              flush=True)
        ms, held, win, _ = run(rs, 1, 1, 0, ib=a.large_ib)
        assert win
        total = torch.cuda.mem_get_info()[1]
        out["large"] = {"reads": rs.n, "gbp": round(gbp, 2), "index_batch_bases": a.large_ib,
                        "ms_per_pass": round(ms, 1),
                        "gb_held": round(held / 1e9, 3),
                        "estimates_gb": est,
                        "device_gb": round(total / 1e9, 1)}
        print(f"  windowed: {ms / 1e3:.2f} s per pass, {held / 1e9:.2f} GB held of "
              f"{total / 1e9:.1f} GB; estimates (GB) {est}")
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "stage1_window.json"), "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
