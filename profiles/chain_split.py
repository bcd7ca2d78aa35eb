"""Where the chain phase of a stage-1 step goes, kernel by kernel and pair size class by class.

Builds the C2 read set the way bench.py does (bench/synth.py, same seed and sizes; --c5:
bench.py's C5 set, HiFi reads at k=19 w=10), runs a few warm stage-1 steps under
torch.profiler (CUDA activities, in a run of its own) and prints, for every kernel of the
chain phase, ms per step and launches per step:

- SplitKernel per instantiation;
- the RadixSortPairs passes of ChainPairs (the descending pair size sort) and of
  OrderPairOverlaps (the overlap key sort), told apart by where they run in the phase;
- GroupChainKernel (a thread per pair) and PairChainKernel (a CTA per pair), per pair
  size class, with the pairs of the class recovered from the launch's grid and shared
  memory;
- GatherOverlapsByIndex, LocateReadOverlaps, ChainKernelGlobal, ReorderOverlaps and the rest.

    python profiles/chain_split.py [--steps 3] [--c5] [--out DIR]

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

# the flagship workload of bench.py (C2), and its C5 set
SEED = 20260924
C2 = dict(seed=SEED, k=15, w=5, reads=200_000, genome=50_000_000, mean=10_000, err={})
C5_READS, C5_MEAN = 30_000, 15_000
C5 = dict(seed=SEED + 5, k=19, w=10, reads=C5_READS, genome=C5_READS * C5_MEAN // 30,
          mean=C5_MEAN, err=dict(sub=0.002, ins=0.0015, dele=0.0015))
FREQ, KMAX = 0.001, 32

def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def pair_chain_smem(npad):
    """PairChainSmem (map.cu): shared memory of one pair of a class of npad slots"""
    n = npad - 1
    nb = n // 4 + 1
    o = 16 * npad + 2 * (n + nb + 2) + 2 * (n + 1) + 2 * 2 * nb
    o = (o + 3) & ~3
    o += 4 * nb
    return (o + 15) & ~15


def npad_of(smem):
    """the largest npad whose PairChainSmem fits in smem bytes (the trace's shared memory
    of a launch holds the kernel's static scalars as well)"""
    fits = [1 << b for b in range(3, 14) if pair_chain_smem(1 << b) <= smem]
    return fits[-1] if fits else None


def short_name(name):
    s = name.replace("(anonymous namespace)::", "").replace("void ", "").replace("rvn::", "")
    return s.replace("unsigned ", "u").split("(")[0]


def classify(evs):
    """rows keyed by label: [total us, launches, pairs] over the chain phases of the trace.
    A chain phase runs from a SplitKernel launch to the next ReorderOverlaps."""
    rows = {}
    in_phase, sorted_pairs = False, False

    def add(label, dur, pairs=0):
        r = rows.setdefault(label, [0.0, 0, 0])
        r[0] += dur
        r[1] += 1
        r[2] += pairs

    for e in evs:
        name, dur = e["name"], float(e["dur"])
        a = e.get("args", {})
        grid, block = a.get("grid", [0, 1, 1]), a.get("block", [0, 1, 1])
        smem = int(a.get("shared memory", 0))
        if "SplitKernel" in name:
            if not in_phase:
                in_phase, sorted_pairs = True, False
            add(short_name(name), dur)
            continue
        if not in_phase:
            continue
        if "SizeClassStarts" in name:
            sorted_pairs = True
        if "Radix" in name or "Onesweep" in name or "PartitionPass" in name:
            which = "OrderPairOverlaps" if sorted_pairs else "ChainPairs"
            add(f"RadixSortPairs[{which}] {short_name(name)}", dur)
        elif "GroupChainKernel" in name:
            threads = block[0]
            bound = smem // (12 * threads) if threads else 0
            add(f"GroupChainKernel <= {bound} hits", dur, grid[0] * threads)
        elif "PairChainKernel" in name:
            npad = npad_of(smem)
            add(f"PairChainKernel <= {npad - 1 if npad else '?'} hits", dur, grid[0])
        else:
            add(short_name(name), dur)
        if "ReorderOverlaps" in name:
            in_phase = False
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--c5", action="store_true", help="bench.py's C5 set (HiFi, k=19 w=10)")
    ap.add_argument("--out", default=None, metavar="DIR",
                    help="also write the tables as DIR/chain_split[_c5].json")
    a = ap.parse_args()

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile

    if not torch.cuda.is_available():
        raise SystemExit("chain_split.py needs a CUDA device")
    from bench import synth
    from raven_b200 import engine

    ws = C5 if a.c5 else C2
    rs = synth.make_reads(ws["seed"], ws["genome"], ws["reads"], ws["mean"], **ws["err"])
    stream = torch.cuda.current_stream()
    eng = engine.Engine(device=0, stream=stream.cuda_stream)
    eng.configure(ws["k"], ws["w"])
    eng.set_option("async_upload", 1)
    eng.upload(rs)

    def step():
        eng.find_overlaps_and_create_piles(FREQ, KMAX, False, 0, fetch=False)

    dev = card()
    print(f"card: {dev}")
    print(f"{'C5' if a.c5 else 'C2'}: {rs.n} reads, "
          f"{int(rs.lens.astype(np.uint64).sum()) / 1e9:.2f} Gbp, k={ws['k']} w={ws['w']}")
    report = {"card": dev, "workload": "c5" if a.c5 else "c2"}
    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    eng.set_option("reset_stats", 1)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.steps):
            step()
        torch.cuda.synchronize()
    phases = eng.timings()
    st = eng.stats()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    kernels = sorted((e for e in trace.get("traceEvents", [])
                      if e.get("ph") == "X" and e.get("cat") == "kernel"),
                     key=lambda e: float(e["ts"]))
    per = classify(kernels)
    rows = []
    for label, (us, cnt, pairs) in sorted(per.items(), key=lambda x: -x[1][0]):
        rows.append({"kernel": label, "ms_per_step": round(us / 1e3 / a.steps, 3),
                     "launches_per_step": cnt / a.steps,
                     "pairs_per_step": pairs // a.steps if pairs else None})
    total = sum(r["ms_per_step"] for r in rows)
    print(f"\n{a.steps} steps; overlaps (last step) {st['overlaps']}")
    print(f"  phase chain (last step, engine timer): {phases.get('chain', 0):.2f} ms; "
          f"kernels below sum to {total:.2f} ms/step")
    print(f"  {'kernel':<62} {'ms/step':>8} {'launch':>6} {'pairs':>9}")
    for r in rows:
        p = "" if r["pairs_per_step"] is None else r["pairs_per_step"]
        print(f"  {r['kernel'][:62]:<62} {r['ms_per_step']:8.3f} "
              f"{r['launches_per_step']:6.1f} {p:>9}")
    report.update({"phases_ms": phases, "kernels": rows, "overlaps": int(st["overlaps"])})
    print("\n(pairs: grid x pairs per CTA of each launch, so up to a CTA's worth above the "
          "class's true count per launch)")
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        name = "chain_split_c5.json" if a.c5 else "chain_split.json"
        with open(os.path.join(a.out, name), "w") as f:
            json.dump(report, f, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
