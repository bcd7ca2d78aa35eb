"""Where the sketch and micromize phases of a stage-1 step go, kernel by kernel.

Builds the C2 read set the way bench.py does (bench/synth.py, same seed and sizes),
runs a few stage-1 steps under torch.profiler (CUDA activities, in a run of its own)
and prints, per kernel of the sketch and micromize phases: ms per step, launches per
step, the bytes the algorithm has to move and those bytes over the kernel time.

    python profiles/sketch_split.py [--steps 3] [--warmup 2] [--out DIR]

Bytes per step (one index batch, so the index holds every sketch record, n):
  SketchFastKernel   the packed reads in (2 bits a base) + 12 B a record out
                     (u32 value, u64 origin)
  MicromizeKernel    4 B a record in (each read's values once) + 12 B a read out
  GatherReadOffsets  8 B a tile-offset lookup + 8 B a read-offset out, per read

The table goes to stdout; --out DIR also writes it as JSON. Needs an H100; prints the
card's name and power limit with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# the flagship workload of bench.py (C2)
SEED = 20260924
K, W, FREQ, KMAX = 15, 5, 0.001, 32
READS, GENOME, MEAN_LEN = 200_000, 50_000_000, 10_000

KERNELS = ("SketchFastKernel", "SketchKernel", "MicromizeKernel", "GatherReadOffsets")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def algorithmic_bytes(name, n, n_reads, word_bytes):
    """bytes a kernel has to move per step (None: not modelled)"""
    if "SketchFastKernel" in name:
        return word_bytes + 12 * n
    if "MicromizeKernel" in name:
        return 4 * n + 12 * n_reads
    if "GatherReadOffsets" in name:
        return 16 * (n_reads + 1)
    return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, metavar="DIR",
                    help="also write the table as DIR/sketch_split.json")
    a = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    if not torch.cuda.is_available():
        raise SystemExit("sketch_split.py needs a CUDA device")
    from bench import synth
    from raven_b200 import engine

    rs = synth.make_reads(SEED, GENOME, READS, MEAN_LEN)
    stream = torch.cuda.current_stream()
    eng = engine.Engine(device=0, stream=stream.cuda_stream)
    eng.configure(K, W)
    eng.upload(rs)

    def step():
        eng.find_overlaps_and_create_piles(FREQ, KMAX, False, 0, fetch=False)

    dev = card()
    print(f"card: {dev}")
    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    eng.set_option("reset_stats", 1)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.steps):
            step()
        torch.cuda.synchronize()
    phases = eng.timings()
    n = int(eng.stats()["index_records"])   # one index batch: every sketch record
    word_bytes = int(rs.words.nbytes)
    per = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        if not any(k in e.name for k in KERNELS):
            continue
        d = per.setdefault(e.name, [0.0, 0])
        d[0] += (e.time_range.end - e.time_range.start) / 1e3
        d[1] += 1
    rows = []
    for name, (ms, cnt) in sorted(per.items(), key=lambda x: -x[1][0]):
        ms_step, launches = ms / a.steps, cnt / a.steps
        b = algorithmic_bytes(name, n, rs.n, word_bytes)
        rate = (b / (ms_step * 1e-3) / 1e12) if b and ms_step > 0 else None
        short = name.replace("(anonymous namespace)::", "").replace("void ", "")
        short = short.replace("unsigned ", "u").replace("rvn::", "").split("(")[0]
        rows.append({"kernel": short, "ms_per_step": round(ms_step, 3),
                     "launches_per_step": launches,
                     "gbytes": None if b is None else round(b / 1e9, 3),
                     "tb_per_s": None if rate is None else round(rate, 3)})
    print(f"\n{a.steps} steps, {rs.n} reads, {word_bytes / 1e9:.3f} GB packed, "
          f"n={n} sketch records")
    print(f"  phases (last step, ms): sketch {phases.get('sketch', 0):.2f}  "
          f"micromize {phases.get('micromize', 0):.2f}")
    print(f"  {'kernel':<44} {'ms/step':>8} {'launch':>6} {'GB':>7} {'TB/s':>6}")
    for r in rows:
        print(f"  {r['kernel'][:44]:<44} {r['ms_per_step']:8.3f} {r['launches_per_step']:6.1f} "
              f"{'' if r['gbytes'] is None else r['gbytes']:>7} "
              f"{'' if r['tb_per_s'] is None else r['tb_per_s']:>6}")
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "sketch_split.json"), "w") as f:
            json.dump({"card": dev, "n": n, "reads": rs.n, "packed_bytes": word_bytes,
                       "phases_ms": phases, "kernels": rows}, f, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
