#!/usr/bin/env python3
"""Where runscan_kernel's time goes, on bench.py's workload (BASELINE.json configs[1], one GPU).

For every source tree given, the library is built a second time with RS_PROBE defined, into a temporary
directory (make EXTRA=-DRS_PROBE=1 OBJDIR=... LIBDIR=...; the tree's own build is not touched), and a child
process runs the bench table through that build (HETMERS_LIB):

  full          runscan_kernel as it is, and the clock64() cycles its warps spend per phase (0 staging / TMA
                wait, 1 adjacency bits, 2 classification + task lists, 3 runs of two, 4 longer runs, then step 5:
                5 hand-off between the warps, 6 the global atomics on the list counters until their results
                are back, 7 the copy of the staged records), summed over all warps; `per_warp` is cycles per
                warp and tile.  `cta` is each CTA's lifetime in cycles, split at the moments its window has
                landed and every warp is done with step 4: `to_window`, `steps_1_4` (two or more warps
                running) and `tail` (from then to the CTA's end)
  load_only     every CTA stages its window, then returns: the bound set by the table's bytes
  compute_only  every CTA stages tile blockIdx.x % 64 (which stays in L2) and does the full work: the bound
                set by the kernel's own instructions and latencies
  no_red        the full kernel, but bloom_insert computes the Bloom slot and issues no atomic
  no_stage      the full kernel, but no candidate record is staged or flushed (step 5)
  no_long       the full kernel without step 4 (runs of three or more)
  no_tail       the full kernel, but every warp returns after step 4: nothing is moved out
The gap between `full` and each of the last four is the price of the part that mode takes out.

`records` are sha256 digests of the full kernel's candidate records (key, lo, meta; sorted) and of its listed
run heads (sorted), with their counts: equal digests across trees mean the same records as a multiset.

Times are CUDA events around hm_k_symm_runscan (the header and Bloom clears included, as in bench.py's
roofline.ms_per_launch), the median of `rounds` rounds of `reps` launches, the modes alternated round by round.
`phases` holds every mode's cycles.  Prints one JSON line with the card name and power limit.  Writes nothing
to the trees.

    python tools/time_runscan_phases.py [--tree NAME=DIR ...] [--reps 20] [--rounds 5] [--nels 2e8]

Without --tree it measures this tree as "branch".  A tree must have the RS_PROBE hooks of csrc/hm_symm.cu.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PHASES = ["stage", "adjacency", "classify", "runs_of_two", "longer_runs", "handoff", "list_atomics", "copy"]
LIFE = ["to_window", "steps_1_4", "tail"]
MODES = {"full": 0, "load_only": 1, "compute_only": 2, "no_red": 3, "no_stage": 4, "no_long": 5, "no_tail": 6}


def card():
    """(name, power limit, max SM clock) of device 0, read with nvidia-smi (queries only)"""
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True)
        f = [x.strip() for x in r.stdout.strip().split(",")]
        if len(f) == 3:
            return {"gpu": f[0], "power_limit": f[1], "clocks_max_sm": f[2]}
    except OSError:
        pass
    return {"gpu": None, "power_limit": None, "clocks_max_sm": None}


def build_probe(tree, tmp):
    """the tree's library with RS_PROBE defined, built under tmp -> path of the .so"""
    obj, libdir = os.path.join(tmp, "obj"), os.path.join(tmp, "lib")
    r = subprocess.run(["make", "-C", tree, "-j8", "lib", "EXTRA=-DRS_PROBE=1", f"OBJDIR={obj}", f"LIBDIR={libdir}"],
                       capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout[-4000:] + r.stderr[-4000:])
        raise SystemExit(f"probe build of {tree} failed")
    return os.path.join(libdir, "libhetmers_b200.so")


def child(args):
    """runs inside a process whose HETMERS_LIB is a probe build"""
    import torch

    from bench import COV, HET, K, LCUT, PLOIDY, SEED
    from smudgeplot_b200 import _lib
    from smudgeplot_b200.device import DeviceTable
    from tools import synth

    L = _lib.lib()
    if not hasattr(L, "hm_probe_runscan"):
        raise SystemExit(f"{_lib.LIB_PATH} is not a probe build (no hm_probe_runscan)")
    L.hm_probe_runscan.argtypes = [C.c_int, C.POINTER(C.c_uint64)]
    cycles = (C.c_uint64 * (len(PHASES) + len(LIFE)))()
    dev = torch.device("cuda", 0)
    G = synth.calibrate_G(K, int(args.nels), PLOIDY, HET, COV, LCUT)
    keys, cnt = synth.synth_table(K, G, PLOIDY, HET, COV, LCUT, SEED, device=dev)
    t = DeviceTable(K, keys, cnt.to(torch.int16)).build_index(direct=False)
    if not t.check_symmetric():
        raise SystemExit("the bench table is not symmetric")
    t.alloc_symm()
    tiles = (t.n + 2047) // 2048
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2 * args.reps)]

    def timed(mode):
        _lib.check(L.hm_probe_runscan(mode, None))           # set the mode, clear the cycle sums
        for r in range(args.reps):
            ev[2 * r].record()
            t.runscan(mid_event=ev[2 * r + 1])
        torch.cuda.synchronize()
        return sum(ev[2 * r].elapsed_time(ev[2 * r + 1]) for r in range(args.reps)) / args.reps

    for m in MODES.values():                                 # warm-up, every mode
        timed(m)
    _lib.check(L.hm_probe_runscan(0, None))                 # the full kernel
    records = digests(t, torch)
    ms = {name: [] for name in MODES}
    cyc = {name: [0] * (len(PHASES) + len(LIFE)) for name in MODES}
    for _ in range(args.rounds):
        for name, m in MODES.items():
            ms[name].append(timed(m))
            _lib.check(L.hm_probe_runscan(0, cycles))
            cyc[name] = [a + int(b) for a, b in zip(cyc[name], cycles)]
    _lib.check(L.hm_probe_runscan(0, None))
    warps = args.rounds * args.reps * tiles * 8

    ctas = args.rounds * args.reps * tiles

    def split(c):
        ph, life = c[:len(PHASES)], c[len(PHASES):]
        tot = sum(ph) or 1
        return {"cycles_per_warp": round(tot / warps, 1),
                **{p: {"share": round(x / tot, 4), "per_warp": round(x / warps, 1)} for p, x in zip(PHASES, ph)},
                "cta": {p: round(x / ctas, 1) for p, x in zip(LIFE, life)}}

    out = {"nels": t.n, "tiles": tiles, "reps": args.reps, "rounds": args.rounds, "records": records,
           "ms": {name: round(statistics.median(v), 4) for name, v in ms.items()},
           "ms_range": {name: [round(min(v), 4), round(max(v), 4)] for name, v in ms.items()},
           "phases": {name: split(c) for name, c in cyc.items()}}
    print(json.dumps(out), flush=True)


def digests(t, torch):
    """one full-kernel pass 1 -> sha256 of its sorted candidate records and of its sorted run heads"""
    import hashlib

    import numpy as np
    t.runscan()
    torch.cuda.synchronize()
    lay, w = t.symm_layout, t.symm_work
    hdr = w[lay.off_header: lay.off_header + 24].view(torch.int64).cpu().numpy()
    nc, nr = min(int(hdr[0]), lay.cand_cap), min(int(hdr[2]), lay.runs_cap)

    def words(off, n):
        return w[off: off + 8 * n].view(torch.int64).cpu().numpy().view(np.uint64)
    key = words(lay.off_cand_key, nc)
    lo = words(lay.off_cand_lo, nc) if t.kmer > 32 else np.zeros(nc, np.uint64)
    meta = words(lay.off_cand_meta, nc)
    rec = np.stack([key, lo, meta], axis=1)
    rec = rec[np.lexsort((meta, lo, key))]
    runs = np.sort(words(lay.off_runs, nr))
    return {"cand_n": nc, "cand_sha256": hashlib.sha256(np.ascontiguousarray(rec).tobytes()).hexdigest(),
            "runs_n": nr, "runs_sha256": hashlib.sha256(runs.tobytes()).hexdigest(), "status": int(hdr[1])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tree", action="append", default=[], metavar="NAME=DIR",
                    help="a source tree to measure (repeatable); default: this tree as 'branch'")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--nels", type=float, default=2e8)
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args)
    trees = [tuple(s.split("=", 1)) for s in args.tree] or [("branch", ROOT)]
    out = card()
    out["workload"] = f"bench.py configs[1], {args.nels:g} k-mers, k=31"
    with tempfile.TemporaryDirectory() as tmp:
        libs = {}
        for name, tree in trees:
            libs[name] = build_probe(os.path.abspath(tree), os.path.join(tmp, name))
        for name, _ in trees:
            env = dict(os.environ, HETMERS_LIB=libs[name])
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--reps", str(args.reps),
                                "--rounds", str(args.rounds), "--nels", str(args.nels)],
                               env=env, capture_output=True, text=True)
            if r.returncode != 0:
                sys.stderr.write(r.stdout[-4000:] + r.stderr[-4000:])
                raise SystemExit(f"probe run of {name} failed")
            out[name] = json.loads(r.stdout.strip().splitlines()[-1])
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
