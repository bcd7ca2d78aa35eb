"""Deep POA windows on the wide consensus kernel (option "poa_wide", DESIGN.md §5).

Windows of 500 backbone bases with 150 and 300 full-length ONT-like layers
(raven_b200/synth.make_windows, partial=0): every one is past the 65000 bases of the
16-bit kernels and runs on PoaKernel<PoaWide>.  Prints, per depth, windows/s of the
whole rvn_poa_batch call (H2D, kernels, D2H), the wide kernel's phase time, DP cells
and GCUPS, and the CPU oracle (racon::Window + spoa, AVX2 int16 fill with its int32
scalar fill where int16 does not fit) on a sample of the same windows at 16 threads.
Card name and power limit first.

    python profiles/poa_deep.py [--windows 2048] [--oracle-windows 128] [--reps 3]
"""
import argparse
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                               "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=2048)
    ap.add_argument("--oracle-windows", type=int, default=128)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--threads", type=int, default=16)
    a = ap.parse_args()

    import numpy as np
    import oracle_lib
    from raven_b200 import engine, synth
    from test_gpu_poa_deep import sub_batch

    print("card:", card())
    eng = engine.Engine(device=0)
    eng.set_option("poa_wide", 1)
    orc = oracle_lib.Oracle()
    for layers in (150, 300):
        w = synth.make_windows(n_windows=a.windows, backbone_len=500, layers=layers,
                               seed=7000 + layers, partial=0.0)
        eng.poa_batch(w, want_coverage=False)   # warm-up: allocations, module load
        best, kern, cells = None, None, 0
        for _ in range(a.reps):
            t0 = time.perf_counter()
            r = eng.poa_batch(w, want_coverage=False)
            dt = time.perf_counter() - t0
            if best is None or dt < best:
                best, kern, cells = dt, eng.timings().get("poa_wide", 0.0) / 1e3, r["cells"]
        routes = eng.poa_routes()
        ow = sub_batch(w, range(min(a.oracle_windows, a.windows)))
        orc.lib.orc_spoa_use_simd(1)
        try:
            t0 = time.perf_counter()
            o = orc.poa_batch(ow, threads=a.threads)
            odt = time.perf_counter() - t0
        finally:
            orc.lib.orc_spoa_use_simd(0)
        n_o = ow["win_first"].size - 1
        ocells = int(np.asarray(o["cells"]).sum())
        print(f"layers {layers}: {a.windows} windows, routes {routes}")
        print(f"  GPU  call {best:.3f} s = {a.windows / best:.1f} windows/s; wide kernel phase "
              f"{kern:.3f} s; {cells / 1e9:.1f} G cells = {cells / best / 1e9:.1f} GCUPS (call), "
              f"{cells / kern / 1e9:.1f} GCUPS (kernel phase)")
        print(f"  CPU oracle, {a.threads} threads, {n_o} windows: {odt:.2f} s = "
              f"{n_o / odt:.1f} windows/s, {ocells / odt / 1e9:.2f} GCUPS")
    eng.close()


if __name__ == "__main__":
    main()
