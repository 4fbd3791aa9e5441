#!/usr/bin/env python3
"""Profiling driver: one seeded bench-workload table on cuda:0, a few device-resident scans.
Meant to be wrapped in a profiler such as ncu; prints per-kernel CUDA-event times itself."""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from smudgeplot_b200.device import DeviceTable  # noqa: E402
from tools import synth  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nels", type=float, default=2e8)
    ap.add_argument("--k", type=int, default=31)
    ap.add_argument("--ploidy", type=int, default=2)
    ap.add_argument("--het", type=float, default=0.01)
    ap.add_argument("--cov", type=float, default=40.0)
    ap.add_argument("--L", type=int, default=12)
    ap.add_argument("--seed", type=int, default=2)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--bits", type=int, default=None)
    ap.add_argument("--fbits", type=int, default=None)
    a = ap.parse_args()
    G = synth.calibrate_G(a.k, int(a.nels), a.ploidy, a.het, a.cov, a.L)
    keys, cnt = synth.synth_table(a.k, G, a.ploidy, a.het, a.cov, a.L, a.seed, device="cuda")
    t = DeviceTable(a.k, keys, cnt.to(torch.int16), bits=a.bits, fbits=a.fbits).build_index()
    t.alloc_work()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    for it in range(a.iters):
        t.deg.zero_()
        t.plot.zero_()
        ev[0].record()
        t.pass1()
        ev[1].record()
        t.pass2()
        ev[2].record()
        torch.cuda.synchronize()
        print(f"iter {it}: n={t.n} bits={t.bits} fbits={t.fbits} pass1 {ev[0].elapsed_time(ev[1]):.3f} ms  "
              f"pass2 {ev[1].elapsed_time(ev[2]):.3f} ms  pairs {int(t.plot.sum())}", flush=True)


if __name__ == "__main__":
    main()
