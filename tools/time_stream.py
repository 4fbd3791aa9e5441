#!/usr/bin/env python3
"""The streamed symmetric scan (DESIGN.md §4c) against the in-core scan on bench.py's workload (BASELINE.json
configs[1]): ms per hm_hetmers_host call from the same pinned host table, chunks, device bytes and records GB/s
over PCIe, with the card name and power limit.  Prints one JSON line; exits 3 unless the streamed plot equals
the in-core plot.  Writes nothing to the tree.

    python tools/time_stream.py --budget-gb 1.6 [--nels 2e8] [--steps 5] [--warmup 2] [--gpus N]

--gpus N streams over devices 0..N-1, a run-aligned share of the table each (the budget is per GPU); the
in-core scan it is compared with runs on the same devices.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import COV, HET, K, LCUT, PLOIDY, SEED, workload_name  # noqa: E402
from smudgeplot_b200 import _lib  # noqa: E402
from tools import synth  # noqa: E402


def host_records(torch, dev, keys, cnt):
    """the table as FastK records (ibyte 3, one part) + stub index in pinned host memory
    -> (hm_host_table, records, index); the last two must outlive every scan of the table"""
    n = keys.numel()
    kbyte, ibyte = (K + 3) // 4, 3
    pbyte = kbyte - ibyte + 2
    rec = torch.empty((n, pbyte), dtype=torch.uint8, device=dev)
    for j in range(ibyte, kbyte):
        rec[:, j - ibyte] = ((keys >> (56 - 8 * j)) & 0xFF).to(torch.uint8)
    rec[:, pbyte - 2] = (cnt & 0xFF).to(torch.uint8)
    rec[:, pbyte - 1] = ((cnt >> 8) & 0xFF).to(torch.uint8)
    index = torch.cumsum(torch.bincount((keys >> 40) & 0xFFFFFF, minlength=1 << 24), 0)
    h_rec = torch.empty(rec.numel(), dtype=torch.uint8, pin_memory=True)
    h_rec.copy_(rec.view(-1))
    h_idx = torch.empty(1 << 24, dtype=torch.int64, pin_memory=True)
    h_idx.copy_(index)
    del rec, index
    torch.cuda.synchronize()
    part_nels = (C.c_int64 * 1)(n)
    part_rec = (C.c_void_p * 1)(h_rec.data_ptr())
    ht = _lib.HostTable(K, ibyte, 1, LCUT, n, C.cast(h_idx.data_ptr(), C.POINTER(C.c_int64)), part_nels, part_rec,
                        None, None)
    ht._keep = (part_nels, part_rec)
    return ht, h_rec, h_idx


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip() or None
    except OSError:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--budget-gb", type=float, required=True, help="device budget of the streamed scan (GB)")
    ap.add_argument("--nels", type=float, default=2e8)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--gpus", type=int, default=1, help="stream over devices 0..N-1")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_stream.py needs a CUDA device: the hetmers path has no CPU fallback")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    G = synth.calibrate_G(K, int(a.nels), PLOIDY, HET, COV, LCUT)
    keys, cnt = synth.synth_table(K, G, PLOIDY, HET, COV, LCUT, SEED, device=dev)
    n = keys.numel()
    ht, h_rec, h_idx = host_records(torch, dev, keys, cnt)
    del keys, cnt
    torch.cuda.empty_cache()
    L = _lib.lib()
    ng = a.gpus
    if not 1 <= ng <= torch.cuda.device_count():
        raise SystemExit(f"time_stream.py: --gpus {ng} asks for more GPUs than the {torch.cuda.device_count()} visible")
    devs = (C.c_int * ng)(*range(ng))
    budget = int(a.budget_gb * 1e9)

    def timed(stream):
        if stream:                                   # streamed whatever the budget says about the table
            os.environ["HETMERS_STREAM"] = "1"
            L.hm_set_device_budget(budget)
        plot = torch.empty(_lib.PLOT_CELLS, dtype=torch.int64, pin_memory=True)
        st = _lib.ScanStats()
        try:
            for _ in range(max(a.warmup, 1)):
                _lib.check(L.hm_hetmers_host(C.byref(ht), devs, ng, plot.data_ptr(), C.byref(st)))
            t0 = time.perf_counter()
            for _ in range(a.steps):
                _lib.check(L.hm_hetmers_host(C.byref(ht), devs, ng, plot.data_ptr(), C.byref(st)))
            dt = (time.perf_counter() - t0) / a.steps
            h = C.c_void_p()                         # one more scan, kept open to read its residency
            _lib.check(L.hm_scan_create(C.byref(ht), devs, ng, C.byref(h)))
            try:
                p2 = torch.empty(_lib.PLOT_CELLS, dtype=torch.int64)
                _lib.check(L.hm_scan_run(h, p2.data_ptr(), None))
                b, c = C.c_int64(), C.c_int64()
                res = (L.hm_scan_residency(h, C.byref(b), C.byref(c)), b.value, c.value)
            finally:
                L.hm_scan_destroy(h)
        finally:
            os.environ.pop("HETMERS_STREAM", None)
            L.hm_set_device_budget(0)
        return plot.clone(), dt * 1e3, st, res

    plot_in, ms_in, st_in, res_in = timed(False)
    plot_st, ms_st, st_st, res_st = timed(True)
    same = bool(torch.equal(plot_in, plot_st))
    rec_bytes = int(h_rec.numel())
    line = {"metric": "ms per hm_hetmers_host call, streamed vs in core", "unit": "ms",
            "workload": workload_name(1), "nels": n, "steps": a.steps, "warmup": max(a.warmup, 1),
            "gpu": torch.cuda.get_device_name(0), "gpus": ng, "power_limit": power_limit(), "budget_bytes": budget,
            "in_core": {"ms_per_call": ms_in, "device_bytes": res_in[1],
                        "records_gbs": rec_bytes / (ms_in * 1e-3) / 1e9,
                        "last_call_ms": {"load": st_in.ms_h2d_unpack, "pass1": st_in.ms_pass1, "pass2": st_in.ms_pass2}},
            "streamed": {"ms_per_call": ms_st, "streamed": bool(res_st[0]), "chunks": res_st[2], "device_bytes": res_st[1],
                         "records_gbs": rec_bytes / (ms_st * 1e-3) / 1e9,
                         "last_call_ms": {"loads_with_pass1_behind": st_st.ms_records, "pass1_kernels": st_st.ms_pass1,
                                          "s_index_pass2": st_st.ms_index, "pass2": st_st.ms_pass2,
                                          "total_in_call": st_st.ms_total}},
            "ratio_streamed_vs_in_core": ms_st / ms_in,
            "device_bytes_ratio": res_st[1] / max(res_in[1], 1),
            "record_bytes": rec_bytes, "stub_index_bytes": int(h_idx.numel()) * 8,
            "parity": {"plot_streamed_vs_in_core": same, "ok": same and bool(res_st[0])}}
    print(json.dumps(line), flush=True)
    if not line["parity"]["ok"]:
        sys.stderr.write("time_stream.py: the streamed plot differs from the in-core plot\n")
        sys.exit(3)


if __name__ == "__main__":
    main()
