#!/usr/bin/env python3
"""extract_kmer_pairs' pair files on bench.py's workload (BASELINE.json configs[1]), written in one process: the
executable before and after hm_scan_write_pairs (--exe-old: an extract_kmer_pairs built from an older tree, which
lists the pairs to the host and writes them there), alternating, and hetmers.Scan.write_pairs phase by phase
(DESIGN.md §6c).  Three quarters of the plot's pixels carry one of three labels (time_extract.label_pixels).

Prints one JSON line with the card name and power limit; exits 3 unless every arm wrote the same bytes.  Writes only
under a temporary directory (--dir, default the system's).

    python tools/time_scan_write_pairs.py [--nels 2e8] [--runs 2] [--exe-old <path>]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import COV, HET, K, LCUT, PLOIDY, SEED, workload_name  # noqa: E402
from tools import synth  # noqa: E402
from tools.time_extract import label_pixels  # noqa: E402
from tools.time_stream import power_limit  # noqa: E402
from tools.time_write_pairs import LABELS, files_of, write_sma  # noqa: E402


def run_exe(exe, table, sma, out):
    """one executable run -> (wall ms, its HETMERS_STATS line)"""
    env = dict(os.environ, HETMERS_STATS="1")
    t0 = time.perf_counter()
    r = subprocess.run([exe, f"-e{LCUT}", f"-o{out}", table, sma], capture_output=True, text=True, env=env)
    ms = (time.perf_counter() - t0) * 1e3
    if r.returncode != 0:
        raise SystemExit(f"{exe} failed: {r.stderr[-2000:]}")
    stats = None
    for line in r.stderr.splitlines():
        if line.startswith("{"):
            stats = json.loads(line)
    return ms, stats


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nels", type=float, default=2e8)
    ap.add_argument("--runs", type=int, default=2, help="runs of each executable, alternating")
    ap.add_argument("--exe-old", default=None, help="an older extract_kmer_pairs to time against")
    ap.add_argument("--dir", default=None)
    a = ap.parse_args()
    import torch
    from smudgeplot_b200 import fastk, hetmers
    if not torch.cuda.is_available():
        raise SystemExit("time_scan_write_pairs.py needs a CUDA device: the hetmers path has no CPU fallback")
    tmp = tempfile.mkdtemp(prefix="time_scan_write_pairs.", dir=a.dir)
    try:
        G = synth.calibrate_G(K, int(a.nels), PLOIDY, HET, COV, LCUT)
        keys, cnt = synth.synth_table(K, G, PLOIDY, HET, COV, LCUT, SEED, device="cuda")
        table = os.path.join(tmp, "t")
        synth.write_table(table, K, keys, cnt, ibyte=3, nparts=4)
        del keys, cnt
        torch.cuda.empty_cache()
        sma = os.path.join(tmp, "ann.sma")
        arms, same = {}, {}
        with hetmers.Scan(fastk.read_ktab(table, mmap=True)) as sc:
            plot, _ = sc.run()
            write_sma(label_pixels(plot), sma)
            st = None
            for i in range(2):                                   # the first call warms up the kernels
                t0 = time.perf_counter()
                st = sc.write_pairs(sma, os.path.join(tmp, "w"))
                st["wall_ms"] = (time.perf_counter() - t0) * 1e3
            arms["scan_write_pairs"] = st
        want = files_of(os.path.join(tmp, "w"))
        exes = {"new": hetmers.get_binary_path("extract_kmer_pairs")}
        if a.exe_old:
            exes["old"] = a.exe_old
        for name in exes:
            arms[f"exe_{name}"] = {"wall_ms": [], "stats": None}
        for _ in range(a.runs):
            for name, exe in exes.items():
                out = os.path.join(tmp, name)
                ms, stats = run_exe(exe, table, sma, out)
                arms[f"exe_{name}"]["wall_ms"].append(ms)
                arms[f"exe_{name}"]["stats"] = stats
                same[f"exe_{name}"] = files_of(out) == want and same.get(f"exe_{name}", True)
        ok = all(same.values())
        line = {"metric": "ms to write extract_kmer_pairs' files in one process", "unit": "ms",
                "workload": workload_name(1), "nels": fastk.read_ktab(table).nels,
                "gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(),
                "file_bytes": sum(len(v) for v in want.values()), "labels": [f"{x}A{y}B" for x, y in LABELS],
                "arms": arms, "same_bytes_as_scan_write_pairs": same, "ok": ok}
        print(json.dumps(line), flush=True)
        if not ok:
            sys.stderr.write("time_scan_write_pairs.py: the arms wrote different files\n")
            sys.exit(3)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
