"""racon::Polisher::Polish through the facade (raven_b200.polish) on one seeded set: time
per phase, window batches, peak device memory (free memory polled during the call), peak
host memory, the polished-window fraction and the sha256 of the polished output; with
--identity, the identity of sampled contigs to the synthetic genome against the draft's.

  python profiles/polish_scale.py --c3                 # bench.py's C3 set (sha256 checks)
  python profiles/polish_scale.py --genome 440000000 --coverage 50 --quality --identity

Prints one JSON line; the card's name and power limit are part of it. Device memory is the
card's used memory (torch.cuda.mem_get_info), over the whole call and over the part that
rvn_polish_windows runs (its start taken from the phase times)."""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import resource
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit",
                               "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=60).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


class DevicePeak:
    """free device memory polled every 10 ms while the block runs, with the time of each
    poll; the card's free memory also reflects any other process on it"""

    def __enter__(self):
        import torch
        self.torch = torch
        self.free0, self.total = torch.cuda.mem_get_info()
        self.samples = []
        self.stop = False
        self.t = threading.Thread(target=self.poll, daemon=True)
        self.t.start()
        return self

    def poll(self):
        t0 = last = time.perf_counter()
        while not self.stop:
            now = time.perf_counter()
            self.samples.append((now, self.torch.cuda.mem_get_info()[0]))
            if now - last >= 30:  # progress of a long call
                print(f"polish: {now - t0:.0f} s, {(self.total - self.samples[-1][1]) / 1e9:.1f} "
                      "GB in use on the card", file=sys.stderr, flush=True)
                last = now
            time.sleep(0.01)

    def __exit__(self, *exc):
        self.end = time.perf_counter()
        self.stop = True
        self.t.join()

    def peak_used_gb(self, t0=None, t1=None):
        """the most memory in use on the card between t0 and t1 (the whole block: None)"""
        low = min((f for t, f in self.samples
                   if (t0 is None or t >= t0) and (t1 is None or t <= t1)), default=self.free0)
        return round((self.total - low) / 1e9, 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--c3", action="store_true", help="bench.py's C3 set")
    ap.add_argument("--genome", type=int, default=40_000_000)
    ap.add_argument("--coverage", type=float, default=50)
    ap.add_argument("--mean-len", type=int, default=10_000)
    ap.add_argument("--contig-len", type=int, default=50_000)
    ap.add_argument("--quality", action="store_true", help="block qualities on every read")
    ap.add_argument("--identity", action="store_true")
    ap.add_argument("--seed", type=int, default=7)
    a = ap.parse_args()
    from bench import synth
    from raven_b200 import polish
    if a.c3:
        # bench.py's C3 leg at its defaults: seed SEED + 1, 20 k reads over 5 Mbp
        seed, g, n, contig = 20260924 + 1, 5_000_000, 20_000, 1_000_000
    else:
        seed, g, contig = a.seed, a.genome, a.contig_len
        n = int(a.coverage * g / a.mean_len)
    mem = subprocess.run(["free", "-g"], capture_output=True, text=True).stdout
    import torch
    torch.cuda.init()
    t = time.perf_counter()
    reads = synth.make_reads(seed, g, n, a.mean_len)
    draft = synth.make_contigs(seed, g, contig_len=contig)
    if a.quality:
        rng = np.random.default_rng(seed)
        nb = (reads.lens.astype(np.int64) + 63) // 64
        reads.block_quality = rng.integers(6, 22, int(nb.sum())).astype(np.uint8)
        reads.bq_off = np.concatenate([[0], np.cumsum(nb)]).astype(np.uint64)
    t_synth = time.perf_counter() - t
    print(f"synthetic set: {reads.bases / 1e9:.2f} Gbp of reads, {draft.bases / 1e6:.0f} Mbp of "
          f"draft, {t_synth:.0f} s", file=sys.stderr, flush=True)
    threads = os.cpu_count() or 1
    if a.c3:
        polish.polish(draft, reads, threads=threads)  # warm-up, as bench.py's C3 leg
    with DevicePeak() as dp:
        got, st = polish.polish(draft, reads, threads=threads, q=10.0 if a.quality else 0.0)
    ph = st["phases_s"]
    h = hashlib.sha256()
    for i in range(got.n):
        h.update(got.names[i].encode() + b"\n" + got.ascii(i) + b"\n")
    out = {
        "card": card(), "host_memory_before": mem.splitlines()[1] if mem else "",
        "reads": n, "read_bases": int(reads.bases), "draft_bases": int(draft.bases),
        "quality": a.quality, "synth_s": round(t_synth, 1),
        "windows": st["windows"], "polished_windows": st["polished_windows"],
        "polished_fraction": st["polished_windows"] / max(st["windows"], 1),
        "window_batches": st["window_batches"], "wide_windows": st["wide_windows"],
        "seconds": st["seconds"], "poa_seconds": st["poa_seconds"],
        "consensus_windows_per_s": st["polished_windows"] / st["poa_seconds"],
        "phases_s": {k: round(v, 3) for k, v in st["phases_s"].items()},
        "device_peak_used_gb": dp.peak_used_gb(),
        # rvn_polish_windows (layer rules, packing, consensus) runs just before the stitch
        "device_peak_used_layers_and_consensus_gb": dp.peak_used_gb(
            dp.end - ph["stitch"] - ph["pieces"] - ph["pack"] - ph["consensus"],
            dp.end - ph["stitch"]),
        "device_used_before_gb": round((dp.total - dp.free0) / 1e9, 2),
        "host_peak_rss_gb": round(resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1e6, 2),
        "sha256": h.hexdigest(),
    }
    if a.identity:
        import oracle_lib
        O = oracle_lib.Oracle()
        genome = synth.make_contigs(seed, g, contig_len=contig, sub=0, ins=0, dele=0)
        rng = np.random.default_rng(1)
        pick = rng.choice(min(draft.n, got.n), size=min(12, draft.n, got.n), replace=False)
        ed_d = ed_p = tot = 0
        for i in pick:
            ref = genome.ascii(int(i))
            ed_d += O.edit_distance(draft.ascii(int(i)), ref)
            ed_p += O.edit_distance(got.ascii(int(i)), ref)
            tot += len(ref)
        out["identity"] = {"contigs": len(pick), "bases": tot, "draft": 1 - ed_d / tot,
                           "polished": 1 - ed_p / tot}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
