"""Where the index build of a stage-1 step goes, kernel by kernel.

Builds the C2 read set the way bench.py does (bench/synth.py, same seed and sizes),
runs a few stage-1 steps under torch.profiler (CUDA activities, in a run of its own)
and prints, per kernel of the index_sort and index_table phases: ms per step, launches
per step and algorithmic bytes over time. One table per setting of the engine option
bare_count (0: bare keys sorted by two stable radix passes + GroupCountKernel; 1: one
unstable partition pass + BareCountKernel in clusters of 8 CTAs; 8 or 16:
that cluster size; default: leave the option alone), so the same run compares the two
paths and the cluster sizes.

    python profiles/index_build_split.py [--steps 3] [--bare-count 0,1,8,16] [--out DIR]

The tables go to stdout; --out DIR also writes them as JSON.

Needs an H100; prints the card's name and power limit with the numbers.
"""
from __future__ import annotations

import argparse
import ctypes as C
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

# kernels of the index_sort and index_table phases (substring of the profiler's name)
KERNELS = ("TierCountKernel", "TierScatterKernel", "RadixHistogramKernel", "RadixScanBinsKernel",
           "OnesweepPass", "PartitionPass", "GroupCountKernel", "BareCountKernel",
           "IndexTableKernel", "FillLongGaps")
# (the OnesweepPass and RadixHistogramKernel rows also hold the other sorts of the step,
#  of the queries and the overlaps: their bytes model covers the index build only)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def index_sizes(eng):
    """records of the probe-able tier (n_a), all records (n) and the bit width of the
    largest probe-able value, of the last index build"""
    v, o, n, nk = (C.POINTER(C.c_uint64)(), C.POINTER(C.c_uint64)(), C.c_uint64(0),
                   C.c_uint64(0))
    eng._check(eng.lib.rvn_index_records(eng.h, C.byref(v), C.byref(o), C.byref(n), C.byref(nk)))
    n_a = n.value
    vmax = max(v[n_a - 1], 1) if n_a else 1   # (sorted by value)
    return n_a, int(eng.stats()["index_records"]), int(vmax).bit_length()


def algorithmic_bytes(name, n, n_a, n_b, passes_a):
    """bytes a kernel has to move per index build (None: not modelled)"""
    if "TierCountKernel" in name:
        return 4 * n
    if "TierScatterKernel" in name:          # values + origins of tier A in, both tiers out
        return 4 * n + 8 * n_a + 12 * n_a + 4 * n_b
    if "RadixHistogramKernel<unsigned int>" in name:  # once over tier A, once over the bare keys
        return 4 * (n_a + n_b)
    if "OnesweepPass<unsigned int, unsigned long" in name:
        return passes_a * 24 * n_a
    if "OnesweepPass<unsigned int, unsigned int, false>" in name:
        return 2 * 8 * n_b
    if "PartitionPass" in name:
        return 8 * n_b
    if "GroupCountKernel" in name or "BareCountKernel" in name:
        return 4 * n_b
    if "IndexTableKernel<unsigned int, true>" in name:
        return 4 * n_a
    return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--bare-count", default="0,1,8,16")
    ap.add_argument("--out", default=None, metavar="DIR",
                    help="also write the tables as DIR/index_build_split.json")
    a = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    if not torch.cuda.is_available():
        raise SystemExit("index_build_split.py needs a CUDA device")
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
    report = {"card": dev, "settings": {}}
    for setting in a.bare_count.split(","):
        if setting != "default":      # ("default": leave the option alone)
            eng.set_option("bare_count", int(setting))
        for _ in range(a.warmup):
            step()
        torch.cuda.synchronize()
        eng.set_option("reset_stats", 1)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.steps):
                step()
            torch.cuda.synchronize()
        phases = eng.timings()
        free, total = torch.cuda.mem_get_info()
        n_a, n, bits_a = index_sizes(eng)
        n_b = n - n_a
        passes_a = -(-bits_a // 10)
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
            b = algorithmic_bytes(name, n, n_a, n_b, passes_a)
            rate = (b / (ms_step * 1e-3) / 1e12) if b and ms_step > 0 else None
            short = name.replace("(anonymous namespace)::", "").replace("void ", "")
            short = short.replace("unsigned ", "u").replace("rvn::", "").split("(")[0]
            rows.append({"kernel": short, "ms_per_step": round(ms_step, 3),
                         "launches_per_step": launches,
                         "gbytes": None if b is None else round(b / 1e9, 3),
                         "tb_per_s": None if rate is None else round(rate, 3)})
        print(f"\nbare_count={setting}: {a.steps} steps, n={n} n_a={n_a} n_b={n_b} "
              f"(tier A: {bits_a} bits, {passes_a} passes); device memory in use after the "
              f"steps {(total - free) / 2**30:.2f} GiB")
        print(f"  phases (last step, ms): index_sort {phases.get('index_sort', 0):.2f}  "
              f"index_table {phases.get('index_table', 0):.2f}")
        print(f"  {'kernel':<58} {'ms/step':>8} {'launch':>6} {'GB':>7} {'TB/s':>6}")
        for r in rows:
            print(f"  {r['kernel'][:58]:<58} {r['ms_per_step']:8.3f} {r['launches_per_step']:6.1f} "
                  f"{'' if r['gbytes'] is None else r['gbytes']:>7} "
                  f"{'' if r['tb_per_s'] is None else r['tb_per_s']:>6}")
        report["settings"][setting] = {
            "n": n, "n_a": n_a, "n_b": n_b, "phases_ms": phases, "kernels": rows,
            "device_mem_used_gib": round((total - free) / 2**30, 3)}
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "index_build_split.json"), "w") as f:
            json.dump(report, f, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
