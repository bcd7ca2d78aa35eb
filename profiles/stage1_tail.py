"""Where the last milliseconds of a C2 stage-1 step go: the copies of the results to the
host against the step's kernels.

    python profiles/stage1_tail.py [--warmup 3] [--index-batches 1] [--stream -1|0|1]
                                   [--out DIR]

bench.py's flagship workload (C2, 200 k reads, 1.98 Gbp), resident, on the context and stream
bench.py uses: --warmup warm steps, then one step under torch.profiler (CUDA activities only).
For that step it prints
- every memcpy: direction, bytes, ms, its start relative to the step's first kernel, and the
  share of its time that some kernel runs beside it (0 %: it is serialized behind them);
- the device time of the copies no kernel runs beside (the serialized tail);
- the sum of the engine's phase timings (eng.timings()) and their breakdown;
- the step's time from CUDA events around it on the stream.
--stream sets the engine option "stage1_stream" (-1 leaves it alone: builds without the
option). --out DIR also writes the numbers to DIR/stage1_tail.json.

Needs an H100; prints the card's name and power limit with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# the flagship workload of bench.py (C2)
SEED = 20260924
K, W, FREQ, KMAX = 15, 5, 0.001, 32
READS, GENOME, MEAN_LEN = 200_000, 50_000_000, 10_000


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit",
                              "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def covered(a, b, spans):
    """microseconds of [a, b) that some span of the sorted, merged `spans` covers"""
    t = 0.0
    for s, e in spans:
        if e <= a:
            continue
        if s >= b:
            break
        t += min(b, e) - max(a, s)
    return t


def merge(spans):
    out = []
    for s, e in sorted(spans):
        if out and s <= out[-1][1]:
            out[-1][1] = max(out[-1][1], e)
        else:
            out.append([s, e])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--index-batches", type=int, default=1)
    ap.add_argument("--stream", type=int, default=-1)
    ap.add_argument("--out", default=None, metavar="DIR")
    a = ap.parse_args()

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    if not torch.cuda.is_available():
        raise SystemExit("stage1_tail.py needs a CUDA device")
    from bench import synth
    from raven_b200 import engine

    dev = card()
    rs = synth.make_reads(SEED, GENOME, READS, MEAN_LEN)
    stream = torch.cuda.current_stream()
    eng = engine.Engine(device=0, stream=stream.cuda_stream)
    eng.configure(K, W)
    eng.set_option("async_upload", 1)
    if a.stream >= 0:
        eng.set_option("stage1_stream", a.stream)
    eng.upload(rs)
    ib = 0
    if a.index_batches > 1:
        ib = -(-int(rs.lens.astype(np.uint64).sum()) // a.index_batches)

    def step():
        eng.find_overlaps_and_create_piles(FREQ, KMAX, False, ib, fetch=False)

    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ev0.record(stream)
        step()
        ev1.record(stream)
        torch.cuda.synchronize()
    step_ms = ev0.elapsed_time(ev1)
    phases = eng.timings()
    eng.close()

    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    evs = [e for e in trace.get("traceEvents", []) if e.get("ph") == "X"]
    kernels = [e for e in evs if e.get("cat") == "kernel"]
    copies = [e for e in evs if e.get("cat") == "gpu_memcpy"]
    t0 = min(float(e["ts"]) for e in kernels) if kernels else 0.0
    kspans = merge([(float(e["ts"]), float(e["ts"]) + float(e["dur"])) for e in kernels])
    rows, serial_us = [], 0.0
    for e in sorted(copies, key=lambda e: float(e["ts"])):
        s, d = float(e["ts"]), float(e["dur"])
        under = covered(s, s + d, kspans)
        serial_us += d - under
        rows.append({"name": e["name"], "bytes": int(e.get("args", {}).get("bytes", 0)),
                     "ms": round(d / 1e3, 3), "start_ms": round((s - t0) / 1e3, 3),
                     "under_kernels": round(under / d, 3) if d > 0 else 1.0,
                     "stream": e.get("args", {}).get("stream")})
    last_kernel_ms = (kspans[-1][1] - t0) / 1e3 if kspans else 0.0

    print(f"card: {dev}")
    print(f"C2: {rs.n} reads, {int(rs.lens.sum()) / 1e9:.2f} Gbp, index batches "
          f"{a.index_batches}, stage1_stream {a.stream if a.stream >= 0 else 'unset'}")
    print(f"  {'memcpy':<36} {'stream':>6} {'bytes':>12} {'ms':>8} {'start':>9} {'under':>6}")
    for r in rows:
        if r["bytes"] < 4096:
            continue  # scalars and offsets of the schedule: listed in the JSON only
        print(f"  {r['name'][:36]:<36} {str(r['stream']):>6} {r['bytes']:>12} {r['ms']:8.3f} "
              f"{r['start_ms']:9.2f} {100 * r['under_kernels']:5.0f}%")
    small = [r for r in rows if r["bytes"] < 4096]
    print(f"  + {len(small)} copies under 4 KiB, {sum(r['ms'] for r in small):.3f} ms in all")
    d2h = [r for r in rows if "DtoH" in r["name"]]
    print(f"  D2H: {sum(r['bytes'] for r in d2h) / 1e9:.3f} GB in "
          f"{sum(r['ms'] for r in d2h):.2f} ms; copies no kernel runs beside: "
          f"{serial_us / 1e3:.2f} ms")
    total = sum(phases.values())
    print(f"  phases: {total:.1f} ms in all: " +
          ", ".join(f"{k} {v:.1f}" for k, v in sorted(phases.items(), key=lambda kv: -kv[1])))
    print(f"  step (CUDA events): {step_ms:.1f} ms; last kernel ends at {last_kernel_ms:.1f} ms "
          f"after the first begins")
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "stage1_tail.json"), "w") as f:
            json.dump({"card": dev, "index_batches": a.index_batches, "stream": a.stream,
                       "step_ms": round(step_ms, 3), "phases_ms": phases,
                       "phases_sum_ms": round(total, 3), "serial_copy_ms": round(serial_us / 1e3, 3),
                       "memcpy": rows}, f, indent=1)


if __name__ == "__main__":
    main()
