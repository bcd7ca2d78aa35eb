"""Kernel time and result digest of each POA route, to compare two builds of the library
on the same windows (RVN_LIB selects the build).

  fast     bench.py's POA batch: 8192 windows of 500 bases x 30 ONT layers; PoaKernelFast
  generic  700-base windows with 30 full-length layers (every layer 576 to ~800 bases);
           PoaKernel<PoaNarrow>
  wide     profiles/poa_deep.py's 150-layer windows (option "poa_wide"); PoaKernel<PoaWide>

For each route it prints the kernel phase of rvn_poa_batch (timer phase "poa" or
"poa_wide": the launches and their retries, without the copies) as the median, min and max
over --reps calls after one warm-up call, the windows and launches per kernel, and a
sha256 over consensus, consensus offsets, coverage, status and cells. Card name and
power limit first. --json appends the same as one JSON line.

    python profiles/poa_routes.py [--reps 5] [--wide-windows 512] [--json FILE]
"""
import argparse
import hashlib
import importlib.util
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                               "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def bench_module():
    # bench.py, not the bench/ package next to it
    spec = importlib.util.spec_from_file_location("bench_main", os.path.join(ROOT, "bench.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def batches(wide_windows):
    from raven_b200 import synth
    fast, _, _ = bench_module().poa_windows(8192)
    generic = synth.make_windows(n_windows=2048, backbone_len=700, layers=30, seed=6700,
                                 partial=0.0)
    wide = synth.make_windows(n_windows=wide_windows, backbone_len=500, layers=150,
                              seed=7000 + 150, partial=0.0)
    return {"fast": (fast, "poa"), "generic": (generic, "poa"), "wide": (wide, "poa_wide")}


def layer_lengths(w):
    import numpy as np
    lens = np.diff(w["seq_off"].astype(np.int64))
    layer = np.ones(lens.size, bool)
    layer[w["win_first"][:-1]] = False
    return int(lens[layer].min()), int(lens[layer].max())


def digest(r):
    h = hashlib.sha256()
    for k in ("consensus", "cons_off", "coverage", "status"):
        h.update(r[k].tobytes())
    h.update(int(r["cells"]).to_bytes(8, "little"))
    return h.hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--wide-windows", type=int, default=512)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()

    from raven_b200 import _lib, engine

    print("card:", card())
    print("library:", os.path.relpath(_lib.LIB_PATH, ROOT))
    eng = engine.Engine(device=0)
    eng.set_option("poa_wide", 1)
    out = {"card": card(), "library": os.path.relpath(_lib.LIB_PATH, ROOT)}
    for route, (w, phase) in batches(a.wide_windows).items():
        eng.poa_batch(w)  # warm-up: allocations, module load
        ms, sha = [], set()
        for _ in range(a.reps):
            r = eng.poa_batch(w)
            ms.append(eng.timings().get(phase, 0.0))
            sha.add(digest(r))
        routes = eng.poa_routes()
        lo, hi = layer_lengths(w)
        n = w["win_first"].size - 1
        print(f"{route}: {n} windows, layers {lo}-{hi} bases, routes {routes}")
        print(f"  kernel phase ms: median {statistics.median(ms):.2f}, min {min(ms):.2f}, "
              f"max {max(ms):.2f}; cells {r['cells']}")
        print(f"  sha256 {' '.join(sorted(sha))}")
        out[route] = {"ms": ms, "sha256": sorted(sha), "routes": routes, "cells": r["cells"]}
    eng.close()
    if a.json:
        with open(a.json, "a") as f:
            f.write(json.dumps(out) + "\n")


if __name__ == "__main__":
    main()
