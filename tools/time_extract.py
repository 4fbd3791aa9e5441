#!/usr/bin/env python3
"""extract_kmer_pairs' pair listing (hm_scan_extract) on bench.py's workload (BASELINE.json configs[1]), by the default
route -- the strand-symmetric scan's candidates, hm_k_symm_extract -- and by the direct passes (HETMERS_PATH=direct).
Three quarters of the plot's pixels carry a label (as test_gpu_parity.write_labelled_sma labels them).  Prints one
JSON line with the card name and power limit:

  * ms per hm_scan_extract call after a run of the same route, the two routes alternated, `reps` calls each;
  * extract_kernel alone: the mean over `reps` launches (CUDA events) on a layer-A table of the same workload;
  * the records listed and the device bytes each route adds to the scan (computed from the sizes).

Exits 3 unless both routes return identical arrays and the record count equals plot[pix > 0].sum().  Writes
nothing to the tree.

    python tools/time_extract.py [--nels 2e8] [--reps 3]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import COV, HET, K, LCUT, PLOIDY, SEED, workload_name  # noqa: E402
from smudgeplot_b200 import _lib  # noqa: E402
from tools import synth  # noqa: E402
from tools.time_stream import host_records, power_limit  # noqa: E402

REC_DT = np.dtype([("key_hi", "<u8"), ("key_lo", "<u8"), ("smudge", "<u4"), ("pos", "u1"), ("alt", "u1"),
                   ("pad", "<u2")])


def label_pixels(plot):
    """labels 1..3 on the pixels with (sum + min) mod 4 < 3 among those the plot fills (3/4 of them)"""
    pix = np.zeros((_lib.SMAX + 1, _lib.PLOT_W), dtype=np.uint16)
    s, m = np.nonzero(plot[:, :_lib.FMAX] > 0)
    lab = (s + m) % 4
    pix[s[lab < 3], m[lab < 3]] = lab[lab < 3] + 1
    return pix


def extract(L, h, pix):
    out = C.POINTER(_lib.PairRec)()
    n = C.c_int64()
    _lib.check(L.hm_scan_extract(h, pix.ctypes.data, C.byref(out), C.byref(n)))
    arr = np.empty(n.value, dtype=REC_DT)
    if n.value:
        C.memmove(arr.ctypes.data, out, n.value * REC_DT.itemsize)
    libc = C.CDLL(None)
    libc.free.argtypes = [C.c_void_p]
    libc.free(out)
    return arr


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nels", type=float, default=2e8)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_extract.py needs a CUDA device: the hetmers path has no CPU fallback")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    G = synth.calibrate_G(K, int(a.nels), PLOIDY, HET, COV, LCUT)
    keys, cnt = synth.synth_table(K, G, PLOIDY, HET, COV, LCUT, SEED, device=dev)
    n = keys.numel()
    ht, h_rec, h_idx = host_records(torch, dev, keys, cnt)
    L = _lib.lib()

    # ---- hm_scan_extract after a run, the two routes alternated ----
    devs = (C.c_int * 1)(0)
    h = C.c_void_p()
    _lib.check(L.hm_scan_create(C.byref(ht), devs, 1, C.byref(h)))
    plot = np.zeros(_lib.PLOT_CELLS, dtype=np.int64)
    ms = {"symm": [], "direct": []}
    lists = {}
    try:
        _lib.check(L.hm_scan_run(h, plot.ctypes.data, None))
        plot = plot.reshape(_lib.SMAX + 1, _lib.PLOT_W)
        pix = label_pixels(plot)
        p2 = np.zeros(_lib.PLOT_CELLS, dtype=np.int64)
        for r in range(a.reps + 1):                                  # the first round warms both routes up
            for route in ("symm", "direct"):
                if route == "direct":
                    os.environ["HETMERS_PATH"] = "direct"
                try:
                    _lib.check(L.hm_scan_run(h, p2.ctypes.data, None))
                    t0 = time.perf_counter()
                    rec = extract(L, h, pix)
                    dt = (time.perf_counter() - t0) * 1e3
                finally:
                    os.environ.pop("HETMERS_PATH", None)
                if r > 0:
                    ms[route].append(dt)
                lists[route] = rec
                if not np.array_equal(p2.reshape(plot.shape), plot):
                    raise SystemExit(f"time_extract.py: the {route} run gave another plot")
        b = C.c_int64()
        L.hm_scan_residency(h, C.byref(b), None)
        incore = b.value
    finally:
        L.hm_scan_destroy(h)
    del h_rec, h_idx

    # ---- extract_kernel alone (layer A, the same table) ----
    from smudgeplot_b200.device import DeviceTable
    t = DeviceTable(K, keys, cnt.to(torch.int16)).build_index(direct=False)
    t.alloc_symm()
    t.runscan()
    nc, st = t.symm_status()
    d_pix = torch.from_numpy(pix.view(np.int16).reshape(-1).copy()).to(dev)
    d_out = torch.empty(2 * nc * REC_DT.itemsize, dtype=torch.uint8, device=dev)
    d_cnt = torch.zeros(1, dtype=torch.int64, device=dev)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    kms = []
    for r in range(a.reps + 2):
        d_cnt.zero_()
        ev[0].record()
        t.extract(d_pix, d_out, d_cnt, 0, nc)
        ev[1].record()
        torch.cuda.synchronize()
        if r >= 2:
            kms.append(ev[0].elapsed_time(ev[1]))
    kernel_records = int(d_cnt.item())

    nrec = len(lists["symm"])
    want = int(plot[pix > 0].sum())
    same = bool(np.array_equal(lists["symm"], lists["direct"]))
    rb = REC_DT.itemsize
    fpos = L.hm_pick_filter_bits(n)
    symm_bytes = 2 * _lib.PLOT_CELLS + 256 + rb * 2 * nc             # default budget: one slice of 2 records per candidate
    direct_bytes = {"incidence": (n + 4) & ~3, "partners": 4 * (n + 1), "prefix_filter": 4 * L.hm_filter_words(fpos),
                    "pixmap_and_count": 2 * _lib.PLOT_CELLS + 8, "records": rb * nrec}
    line = {"metric": "ms per hm_scan_extract call after a run, symmetric route vs direct passes", "unit": "ms",
            "workload": workload_name(1), "nels": n, "reps": a.reps, "gpu": torch.cuda.get_device_name(0),
            "power_limit": power_limit(), "labelled_pixels": int((pix > 0).sum()),
            "symm": {"ms_per_call": ms["symm"], "mean_ms": sum(ms["symm"]) / len(ms["symm"]),
                     "extract_kernel_ms": sum(kms) / len(kms), "candidates": nc,
                     "device_bytes_added": symm_bytes},
            "direct": {"ms_per_call": ms["direct"], "mean_ms": sum(ms["direct"]) / len(ms["direct"]),
                       "device_bytes_added": sum(direct_bytes.values()), "device_bytes": direct_bytes},
            "records": nrec, "record_bytes": rb * nrec, "in_core_device_bytes": incore,
            "parity": {"routes_equal": same, "records_equal_labelled_plot": nrec == want,
                       "kernel_records": kernel_records == nrec, "status": st,
                       "ok": same and nrec == want and kernel_records == nrec and st == 0}}
    print(json.dumps(line), flush=True)
    if not line["parity"]["ok"]:
        sys.stderr.write("time_extract.py: the routes' pair lists differ, or do not match the labelled plot\n")
        sys.exit(3)


if __name__ == "__main__":
    main()
