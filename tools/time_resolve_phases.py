#!/usr/bin/env python3
"""Where resolve_kernel's time goes (pass 2 of the symmetric scan), on bench.py's workload (BASELINE.json
configs[1], one GPU).

For every source tree given, the library is built a second time with RESOLVE_PROBE defined, into a temporary
directory (make EXTRA=-DRESOLVE_PROBE=1 OBJDIR=... LIBDIR=...; the tree's own build is not touched), and a child
process runs the bench table through that build (HETMERS_LIB):

  full          resolve_kernel as it is
  records_only  the candidate records are loaded and dropped: the bound the record stream sets
  bloom_only    records and Bloom look-ups; every Bloom hit is taken as not isolated, no exact check

and once more in full with counters on: candidates, Bloom hits on rc x only / rc y only / both, exact checks
that take the general path (has_upper_partner: a bucket of more than 48 keys, or a bucket prefix longer than
the run prefix), and the sizes of the buckets the exact checks scan ("49+": more than 48).

Times are CUDA events around hm_k_symm_resolve alone (each launch after a pass 1 of its own, as in a scan), the
median of `rounds` rounds of `reps` launches, the three modes alternated round by round.  Prints one JSON line
with the card name and power limit.  Writes nothing to the trees.

    python tools/time_resolve_phases.py [--tree NAME=DIR ...] [--lib NAME=SO ...] [--reps 20] [--rounds 5] [--nels 2e8]

Without --tree it measures this tree as "branch".  A tree must have the RESOLVE_PROBE hooks of csrc/hm_symm.cu.
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

from tools.time_runscan_phases import card  # noqa: E402

MODES = {"full": 0, "records_only": 1, "bloom_only": 2}
BINS = 50
NCTR = 5 + BINS


def build_probe(tree, tmp):
    """the tree's library with RESOLVE_PROBE defined, built under tmp -> path of the .so"""
    obj, libdir = os.path.join(tmp, "obj"), os.path.join(tmp, "lib")
    r = subprocess.run(["make", "-C", tree, "-j8", "lib", "EXTRA=-DRESOLVE_PROBE=1", f"OBJDIR={obj}",
                        f"LIBDIR={libdir}"], capture_output=True, text=True)
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
    if not hasattr(L, "hm_probe_resolve"):
        raise SystemExit(f"{_lib.LIB_PATH} is not a probe build (no hm_probe_resolve)")
    L.hm_probe_resolve.argtypes = [C.c_int, C.POINTER(C.c_uint64)]
    ctr = (C.c_uint64 * NCTR)()
    dev = torch.device("cuda", 0)
    G = synth.calibrate_G(K, int(args.nels), PLOIDY, HET, COV, LCUT)
    keys, cnt = synth.synth_table(K, G, PLOIDY, HET, COV, LCUT, SEED, device=dev)
    t = DeviceTable(K, keys, cnt.to(torch.int16)).build_index(direct=False)
    if not t.check_symmetric():
        raise SystemExit("the bench table is not symmetric")
    t.alloc_symm()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2 * args.reps)]

    def timed(mode):
        _lib.check(L.hm_probe_resolve(mode, None))           # set the mode, clear the counts
        for r in range(args.reps):
            t.runscan()
            ev[2 * r].record()
            t.resolve()
            ev[2 * r + 1].record()
        torch.cuda.synchronize()
        return sum(ev[2 * r].elapsed_time(ev[2 * r + 1]) for r in range(args.reps)) / args.reps

    for m in MODES.values():                                 # warm-up, every mode
        timed(m)
    ms = {name: [] for name in MODES}
    for _ in range(args.rounds):
        for name, m in MODES.items():
            ms[name].append(timed(m))
    _lib.check(L.hm_probe_resolve(3, None))                  # one counting launch
    t.runscan()
    t.resolve()
    _lib.check(L.hm_probe_resolve(0, ctr))
    c = [int(v) for v in ctr]
    nc, st = t.symm_status()
    hist = {str(i) if i < BINS - 1 else f"{BINS - 1}+": c[5 + i] for i in range(BINS) if c[5 + i]}
    checked = sum(c[5:])
    out = {"nels": t.n, "candidates_listed": nc, "status": st, "reps": args.reps, "rounds": args.rounds,
           "ms": {name: round(statistics.median(v), 4) for name, v in ms.items()},
           "ms_range": {name: [round(min(v), 4), round(max(v), 4)] for name, v in ms.items()},
           "candidates": c[0], "hits_rcx_only": c[1], "hits_rcy_only": c[2], "hits_both": c[3],
           "hit_share": round((c[1] + c[2] + c[3]) / max(c[0], 1), 4),
           "general_path": c[4], "buckets_checked": checked,
           "bucket_mean": round(sum(i * c[5 + i] for i in range(BINS)) / max(checked, 1), 3),
           "bucket_sizes": hist}
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tree", action="append", default=[], metavar="NAME=DIR",
                    help="a source tree to measure (repeatable); default: this tree as 'branch'")
    ap.add_argument("--lib", action="append", default=[], metavar="NAME=SO",
                    help="a probe build made beforehand (repeatable), measured as NAME instead of building a tree")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--nels", type=float, default=2e8)
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args)
    prebuilt = [tuple(s.split("=", 1)) for s in args.lib]
    trees = [tuple(s.split("=", 1)) for s in args.tree] or ([] if prebuilt else [("branch", ROOT)])
    out = card()
    out["workload"] = f"bench.py configs[1], {args.nels:g} k-mers, k=31"
    with tempfile.TemporaryDirectory() as tmp:
        libs = {}
        for name, tree in trees:
            libs[name] = build_probe(os.path.abspath(tree), os.path.join(tmp, name))
        libs.update((name, os.path.abspath(so)) for name, so in prebuilt)
        for name in libs:
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
