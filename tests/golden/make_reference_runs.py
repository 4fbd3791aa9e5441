#!/usr/bin/env python3
"""Regenerate tests/golden/reference_runs/: what the UNMODIFIED reference binaries (oracle/_ref/hetmers and
oracle/_ref/extract_kmer_pairs, built by oracle/Makefile from the reference sources) write for the seeded
tables of tests/test_gpu_parity.py that are too large to store themselves.  The tables are regenerated
by the tests from their seeds (tools/synth.py gives the same table on the CPU and on the GPU), so only
the reference's answers are kept:

  medium_k<k>_s<seed>.smu       test_medium_table_matches_reference_binary
  conditioned_k<k>_s<seed>.smu  test_gpu_conditioning_of_canonical_untrimmed_table (the conditioned table)
  extract.json                  test_extract_matches_reference_binary_and_inprocess_list: per table and
                                smudge, the number and SHA-256 of the sorted lines of <out>.<smudge>.txt

Run from the repository root once oracle/_ref/ is built:   python tests/golden/make_reference_runs.py
"""
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

import oracle_util as ou  # noqa: E402
import test_gpu_parity as tp  # noqa: E402
from smudgeplot_b200 import fastk  # noqa: E402
from tools import synth  # noqa: E402

OUT = os.path.join(HERE, "reference_runs")


def ref_smu(table, e, threads, d):
    r = ou.run_ref(table, os.path.join(d, "ref"), e, threads=threads, verbose=True)
    assert r.returncode == 0 and "trimmed and symmetric" in r.stderr, r.stderr
    return open(os.path.join(d, "ref.smu")).read()


def main():
    if not (ou.have_ref() and ou.have_ref_extract()):
        sys.exit("oracle/_ref/ has no reference binaries: build them first (oracle/Makefile)")
    os.makedirs(OUT, exist_ok=True)
    cores = min(os.cpu_count() or 4, 64)
    for k, target, ploidy, het, cov, L, seed, ref_threads in tp.MEDIUM_CASES:
        with tempfile.TemporaryDirectory() as d:
            G = synth.calibrate_G(k, target, ploidy, het, cov, L)
            keys, cnt = synth.synth_table(k, G, ploidy, het, cov, L, seed)
            name = os.path.join(d, "t")
            synth.write_table(name, k, keys, cnt, ibyte=3, nparts=4)
            smu = ref_smu(name, L, ref_threads or cores, d)
        with open(os.path.join(OUT, ou.reference_run_name("medium", k, seed)), "w") as f:
            f.write(smu)
        print("medium", k, seed, keys.shape[0], "k-mers,", len(smu.splitlines()), "rows")
    for k, G, ploidy, seed, L in tp.CONDITIONING_CASES:
        keys, cnt = synth.synth_table(k, G, ploidy, 0.02, 40, 1, seed)
        ku = synth.keys_to_u64_numpy(keys)
        cn = cnt.numpy().astype(np.uint16)
        canon = tp.canonical_mask(keys, ku, k)
        ck, cc = tp._condition_numpy(ku[canon], cn[canon], k, L, True, True)
        with tempfile.TemporaryDirectory() as d:
            cond = os.path.join(d, "cond")
            fastk.write_ktab(cond, k, ck, cc, ibyte=3, nparts=2)
            smu = ref_smu(cond, L, 4, d)
        with open(os.path.join(OUT, ou.reference_run_name("conditioned", k, seed)), "w") as f:
            f.write(smu)
        print("conditioned", k, seed, len(cc), "k-mers,", len(smu.splitlines()), "rows")
    digests = {}
    for k, G, ploidy, seed, L in tp.EXTRACT_CASES:
        keys, cnt = synth.synth_table(k, G, ploidy, 0.02, 20 * ploidy, L, seed)
        with tempfile.TemporaryDirectory() as d:
            name = os.path.join(d, "t")
            kt = synth.write_table(name, k, keys, cnt, ibyte=3, nparts=3)
            kb, cn = fastk.unpack_host(kt)
            plot, _ = ou.oracle_scan(kb, cn, k)
            sma = os.path.join(d, "ann.sma")
            tp.write_labelled_sma(plot, sma)
            r = ou.run_ref_extract(name, sma, os.path.join(d, "ref"), L, threads=cores)
            assert r.returncode == 0, r.stderr
            digests[f"k{k}_s{seed}"] = ou.pair_digests(ou.sorted_pair_files(os.path.join(d, "ref")))
        print("extract", k, seed, digests[f"k{k}_s{seed}"])
    with open(os.path.join(OUT, "extract.json"), "w") as f:
        json.dump(digests, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
