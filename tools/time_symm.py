"""time the strand-symmetric scan against the direct passes on the bench workload (one GPU)

The symmetric scan is timed kernel by kernel: `runscan_ms` (runscan_kernel, with the clearing of the
work-area header and the Bloom filter), `runs_ms` (runs_kernel) and `resolve_ms` (resolve_kernel), each
the mean over `reps` scans bracketed by CUDA events.  `runs_listed` is the number of runs runscan_kernel
left to runs_kernel (header word 2 of the work area)."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from smudgeplot_b200.device import DeviceTable  # noqa: E402
from tools import synth  # noqa: E402


def main():
    nels = float(sys.argv[1]) if len(sys.argv) > 1 else 2e8
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 10
    direct = os.environ.get("NO_DIRECT") is None
    K, P, HET, COV, L, SEED = 31, 2, 0.01, 40.0, 12, 2
    G = synth.calibrate_G(K, int(nels), P, HET, COV, L)
    keys, cnt = synth.synth_table(K, G, P, HET, COV, L, SEED, device="cuda")
    t = DeviceTable(K, keys, cnt.to(torch.int16)).build_index(direct=direct)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    ev[0].record()
    sym = t.check_symmetric()
    ev[1].record()
    torch.cuda.synchronize()
    out = {"nels": t.n, "symmetric": sym, "fingerprint_ms": ev[0].elapsed_time(ev[1])}
    t.alloc_symm()
    res = {}
    for name in (["direct"] if direct else []) + ["symm"]:
        if name == "direct":
            t.alloc_work()
        tms = []
        for r in range(reps + 3):
            t.plot.zero_()
            if name == "direct":
                t.deg.zero_()
            ev[0].record()
            if name == "direct":
                t.pass1()
                ev[1].record()
                ev[2].record()
                t.pass2()
            else:
                t.runscan(mid_event=ev[1])
                ev[2].record()
                t.resolve()
            ev[3].record()
            torch.cuda.synchronize()
            if r >= 3:
                tms.append([ev[i].elapsed_time(ev[i + 1]) for i in range(3)])
        res[name] = t.plot.clone()
        a, b, c = (sum(x[i] for x in tms) / len(tms) for i in range(3))
        if name == "direct":
            out[name] = {"k1_ms": a, "k2_ms": c, "kmers_per_s": t.n / ((a + c) * 1e-3)}
        else:
            out[name] = {"k1_ms": a + b, "k2_ms": c, "runscan_ms": a, "runs_ms": b, "resolve_ms": c,
                         "kmers_per_s": t.n / ((a + b + c) * 1e-3)}
    if direct:
        out["plots_equal"] = bool(torch.equal(res["direct"], res["symm"]))
    out["plot_sum"] = int(res["symm"].sum())
    nc, st = t.symm_status()
    hdr = t.symm_work[t.symm_layout.off_header:t.symm_layout.off_header + 24].view(torch.int64)
    out["candidates"], out["runs_listed"], out["status"] = nc, int(hdr[2]), st
    print(json.dumps(out))


if __name__ == "__main__":
    main()
