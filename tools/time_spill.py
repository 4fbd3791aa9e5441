#!/usr/bin/env python3
"""The streamed scan with its candidate records and S list resident on the device against the same scan with them in
host memory (hm_set_list_host_budget, DESIGN.md §4c, *Lists in host memory*), in one process on one GPU.  The table
is trimmed and symmetric, shaped like bench.py's workload (BASELINE.json configs[1]: k = 31, diploid, het 1 %,
coverage 40) at --nels entries.  Both arms stream it in chunks of nels / --chunks entries: the resident arm under a
budget that also holds the whole lists, the spilled arm under the smallest budget whose plan has chunks that large,
where the lists do not fit (the run refuses without a list host budget).  The arms alternate after --warmup rounds,
--steps calls each; a call is one run(), timed by the wall clock around it (it ends in a device synchronise) and
split into pass 1 and pass 2 by the scan's stats.  Medians are reported with the spill stats (flushes, bytes each
way, rounds, partitions), the device peak and the card and power limit read in the same run.  The plots must be
equal or the run exits 3; a spilled arm that did not spill exits 2.

    python tools/time_spill.py [--nels 3e7] [--chunks 128] [--steps 3] [--warmup 1] [--dir /tmp]
"""
import argparse
import ctypes as C
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
from tools.time_stream import power_limit  # noqa: E402


def budget_for_chunk(lib, StreamLayout, n, k, ibyte, chunk):
    """the smallest device budget whose streamed plan has chunks of at least `chunk` entries"""
    lo, hi = 1 << 20, 1 << 40
    lay = StreamLayout()
    while lo < hi:
        mid = (lo + hi) // 2
        if lib.hm_stream_plan(n, k, ibyte, mid, C.byref(lay)) == 0 and lay.chunk >= chunk:
            hi = mid
        else:
            lo = mid + 1
    return lo


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nels", type=float, default=3e7, help="entries of the trimmed, symmetric table")
    ap.add_argument("--chunks", type=int, default=128, help="chunk cap: nels / chunks entries")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--dir", default=None, help="where the table files are written (a temporary directory)")
    a = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_spill.py needs a CUDA device: the hetmers path has no CPU fallback")
    from smudgeplot_b200 import _lib, fastk, hetmers
    L = _lib.lib()
    work = tempfile.mkdtemp(prefix="time_spill.", dir=a.dir)
    try:
        dev = torch.device("cuda", 0)
        G = synth.calibrate_G(K, int(a.nels), PLOIDY, HET, COV, LCUT)
        keys, cnt = synth.synth_table(K, G, PLOIDY, HET, COV, LCUT, SEED, device=dev)
        name = os.path.join(work, "t")
        synth.write_table(name, K, keys, cnt, ibyte=3, nparts=4)
        del keys, cnt
        torch.cuda.empty_cache()
        kt = fastk.read_ktab(name, mmap=True)
        n = kt.nels
        chunk = -(-n // a.chunks)
        tight = budget_for_chunk(L, _lib.StreamLayout, n, K, kt.ibyte, chunk)
        lists = 16 * (n // 2 + 4096) + 8 * (n + 4096)              # the lists' bound: a candidate per 2 entries, an S key each
        roomy = tight + 2 * lists
        os.environ["HETMERS_STREAM"], os.environ["HETMERS_STREAM_CHUNK"] = "1", str(chunk)

        def arm(budget, cap):
            L.hm_set_list_host_budget(cap)
            with hetmers.Scan(kt, device_budget=budget) as sc:
                t0 = time.perf_counter()
                plot, st = sc.run()
                t1 = time.perf_counter()
                sp, res = sc.spill_stats(), sc.residency()
            r = {"ms_run": (t1 - t0) * 1e3, "ms_pass1": st["ms_pass1"], "ms_pass2": st["ms_pass2"],
                 "device_peak": res[1], "chunks": res[2]}
            r.update({key: sp[key] for key in ("flushes", "d2h_bytes", "host_peak_bytes", "rounds", "partitions",
                                               "h2d_bytes", "slice", "part", "ms_flush")})
            r["spill_ms_pass2"] = sp["ms_pass2"]
            return plot, r

        arms = {"resident": lambda: arm(roomy, 0), "spilled": lambda: arm(tight, 1 << 40)}
        runs, plots = {k: [] for k in arms}, {}
        for step in range(a.warmup + a.steps):
            for key, fn in arms.items():
                plots[key], r = fn()
                if step >= a.warmup:
                    runs[key].append(r)
        L.hm_set_list_host_budget(0)
        same = bool(np.array_equal(plots["resident"], plots["spilled"]))
        med = {key: {f: sorted(r[f] for r in rs)[len(rs) // 2] for f in rs[0]} for key, rs in runs.items()}
        print(json.dumps({"metric": "streamed scan, one GPU: lists resident against lists in host memory",
                          "unit": "ms (median)", "nels": n, "k": K, "chunk": chunk, "budget_resident": roomy,
                          "budget_spilled": tight, "gpu": torch.cuda.get_device_name(dev),
                          "power_limit": power_limit(), "steps": a.steps, "plots_equal": same,
                          "ratio_run": med["spilled"]["ms_run"] / med["resident"]["ms_run"],
                          "median": med, "runs": runs}))
        if not same:
            sys.exit(3)
        if med["spilled"]["flushes"] == 0 or med["resident"]["flushes"] != 0:
            sys.exit(2)
    finally:
        os.environ.pop("HETMERS_STREAM", None)
        os.environ.pop("HETMERS_STREAM_CHUNK", None)
        shutil.rmtree(work, ignore_errors=True)


if __name__ == "__main__":
    main()
