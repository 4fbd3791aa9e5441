#!/usr/bin/env python3
"""Scanning a raw FastK table larger than the device budget in one process: conditioned into new table files first
(hetmers.condition_table, then Scan(dst).run()) against conditioned on the way in, into host memory
(Scan.from_ktab(src, L).run(); DESIGN.md §4d).  The table is canonical and untrimmed (counts from 1, one strand),
shaped like bench.py's workload (BASELINE.json configs[1]: k = 31, diploid, het 1 %, coverage 40, L = 12) at --nels
entries, written to a temporary directory under --dir.  The device budget is --budget-frac of what the conditioned
table's in-core scan takes, so both arms stream it.  Per GPU count (1, and 2 where the box has them) the arms
alternate after --warmup rounds, --steps calls each; each call (conditioning, scan creation and one run) is timed
by the wall clock around library calls that synchronise.  The plots must be equal or the run exits 3.  One JSON line
with the card and its power limit, read in the same run.

    python tools/time_scan_from_ktab.py [--nels 2e7] [--steps 3] [--warmup 1] [--budget-frac 0.5] [--dir /tmp]
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import COV, HET, K, LCUT, PLOIDY, SEED  # noqa: E402
from tools import synth  # noqa: E402
from tools.time_condition_gpus import filesystem  # noqa: E402
from tools.time_stream import power_limit  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nels", type=float, default=2e7, help="entries of the canonical untrimmed table")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--budget-frac", type=float, default=0.5,
                    help="device budget as a fraction of the conditioned table's in-core scan")
    ap.add_argument("--dir", default=None, help="where the table files are written (a temporary directory)")
    a = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_scan_from_ktab.py needs a CUDA device: the hetmers path has no CPU fallback")
    from smudgeplot_b200 import _lib, fastk, hetmers
    ngpu = _lib.lib().hm_device_count()
    work = tempfile.mkdtemp(prefix="time_scan_from_ktab.", dir=a.dir)
    try:
        dev = torch.device("cuda", 0)
        G = synth.calibrate_G(K, int(2 * a.nels), PLOIDY, HET, COV, 1)
        keys, cnt = synth.synth_table(K, G, PLOIDY, HET, COV, 1, SEED, device=dev)
        keep = keys <= synth.revcomp_left(keys, K)                     # what FastK writes: the canonical strand
        ku = synth.keys_to_u64_numpy(keys[keep].cpu())
        cn = cnt[keep].cpu().numpy().astype(np.uint16)
        del keys, cnt, keep
        torch.cuda.empty_cache()
        src, dst = os.path.join(work, "src"), os.path.join(work, "dst")
        fastk.write_ktab(src, K, ku, cn, ibyte=3, nparts=4)
        del ku, cn
        n = fastk.read_ktab(src).nels

        # the budget: a fraction of the conditioned table's in-core scan
        hetmers.condition_table(src, dst, LCUT)
        with hetmers.Scan(fastk.read_ktab(dst)) as sc:
            incore = sc.residency()[1]
        budget = int(incore * a.budget_frac)

        def files(g):
            t0 = time.perf_counter()
            cst = hetmers.condition_table(src, dst, LCUT, device_budget=budget, gpus=g)
            t1 = time.perf_counter()
            with hetmers.Scan(fastk.read_ktab(dst, mmap=True), gpus=g) as sc:
                t2 = time.perf_counter()
                plot, _ = sc.run()
                t3 = time.perf_counter()
                streamed = sc.residency()[0]
            return plot, {"ms_condition": (t1 - t0) * 1e3, "ms_open": (t2 - t1) * 1e3, "ms_scan": (t3 - t2) * 1e3,
                          "ms_total": (t3 - t0) * 1e3, "ranges": cst["ranges"], "streamed": streamed,
                          "condition_peak_bytes": cst["peak_bytes"], "bytes_written": cst["bytes_written"],
                          "host_bytes": 0}

        def host(g):
            t0 = time.perf_counter()
            with hetmers.Scan.from_ktab(src, LCUT, gpus=g, device_budget=budget) as sc:
                t1 = time.perf_counter()
                plot, _ = sc.run()
                t2 = time.perf_counter()
                st, streamed = sc.stats["condition"], sc.residency()[0]
            return plot, {"ms_condition": st["ms_total"], "ms_open": (t1 - t0) * 1e3 - st["ms_total"],
                          "ms_scan": (t2 - t1) * 1e3, "ms_total": (t2 - t0) * 1e3, "ranges": st["ranges"],
                          "route": st["route"], "streamed": streamed, "condition_peak_bytes": st["peak_bytes"],
                          "bytes_written": 0, "host_bytes": st["host_bytes"]}

        arms = {"files": files, "host": host}
        results, same = {}, True
        for g in sorted({1, min(2, ngpu)}):
            runs = {name: [] for name in arms}
            plots = {}
            for step in range(a.warmup + a.steps):
                for name, fn in arms.items():
                    plot, r = fn(g)
                    plots[name] = plot
                    if step >= a.warmup:
                        runs[name].append(r)
            same = same and np.array_equal(plots["files"], plots["host"])
            results[f"gpus{g}"] = {"median": {name: {key: sorted(r[key] for r in rs)[len(rs) // 2] for key in rs[0]}
                                              for name, rs in runs.items()}, "runs": runs}
        print(json.dumps({"metric": "raw table -> streamed scan in one process: condition into files then scan, "
                                    "against condition into host memory then scan", "unit": "ms (median)",
                          "nels": n, "k": K, "L": LCUT, "budget": budget, "incore_bytes": incore,
                          "gpu": torch.cuda.get_device_name(dev), "power_limit": power_limit(),
                          "filesystem": filesystem(work), "steps": a.steps, "plots_equal": bool(same),
                          "results": results}))
        if not same:
            sys.exit(3)
    finally:
        shutil.rmtree(work, ignore_errors=True)


if __name__ == "__main__":
    main()
