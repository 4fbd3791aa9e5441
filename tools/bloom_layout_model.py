#!/usr/bin/env python3
"""The symmetric scan's Bloom filter (csrc/hm_symm.cu, bloom_slot / bloom_insert) restated in numpy, and what it
predicts for pass 2 on bench.py's workload (BASELINE.json configs[1]), on the CPU.

The filter holds the set S (table entries with a partner at a position >= k - k/2); pass 2 looks up rc x and rc y
of every candidate pair (x, y) and sends a hit to the exact check.  S is about 1/6 of the table and the filter has
one bit per entry, so it carries c ~ 6 bits per element of S whatever the table's size: its false-positive rate
depends on c and on the layout only.  This builds a seeded bench-workload table scaled down to --nels entries
(tools/synth.py, bench.py's parameters), its S and candidates exactly as pass 1 defines them, and counts the Bloom
hits on rc x only / rc y only / both for each layout:

  word32    the former layout: 2 bits in one 32-bit word
  word64    the layout hm_symm.cu uses: 3 bits in one 64-bit word (one 64-bit atomic per insert)
  sector    a 32-byte sector, 2 bits in each of two of its four 64-bit words (1 or 2 atomics per insert); the
            fewest false positives, but on the H100 its second atomic cost pass 1 far more than pass 2 gained

The counts are also given scaled to 2e8 entries (x 2e8 / n).  Prints one JSON line.

    python tools/bloom_layout_model.py [--nels 4e6] [--seed 2]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SMAX = 1000
LAYOUTS = ("word32", "word64", "sector")
_U32 = np.uint32


def _mul32(a, b):
    return (a.astype(np.uint64) * np.uint64(b) & np.uint64(0xFFFFFFFF)).astype(_U32)


def _umulhi(a, b):
    return ((a.astype(np.uint64) * np.uint64(b)) >> np.uint64(32)).astype(_U32)


def slot_hashes(hi, lo, k):
    """bloom_slot's two 32-bit hashes of left-aligned keys (hi, lo: uint64 arrays; lo unused for k <= 32):
    h of the last k/2 bases (the filter word or sector), g of the first k - k/2 bases (the bits)"""
    hi = np.asarray(hi, dtype=np.uint64)
    Pr = k >> 1
    pup = k - Pr
    if k <= 32:
        sfx = hi >> np.uint64(64 - 2 * k)
    else:
        lo = np.asarray(lo, dtype=np.uint64)
        sr = 128 - 2 * k
        sfx = lo if sr == 0 else (lo >> np.uint64(sr)) | (hi << np.uint64(64 - sr))
    if 2 * Pr < 64:
        sfx = sfx & np.uint64((1 << (2 * Pr)) - 1)
    pfx = hi >> np.uint64(64 - 2 * pup)
    h = _mul32(sfx.astype(_U32) ^ _mul32((sfx >> np.uint64(32)).astype(_U32), 0x85EBCA6B), 0x9E3779B1)
    g = _mul32(pfx.astype(_U32) ^ _mul32((pfx >> np.uint64(32)).astype(_U32), 0xC2B2AE35), 0x27D4EB2F)
    h ^= h >> _U32(15)
    return h, g


def slots(layout, h, g, seg_words):
    """-> list of (index, mask) in uint64 units of the segment (word32: uint32 units), one per word a key sets"""
    hm = _mul32(h, 0x2C1B3C6D)
    if layout == "word32":
        w = _umulhi(hm, seg_words).astype(np.int64)
        m = (_U32(1) << (g >> _U32(27))) | (_U32(1) << ((g >> _U32(22)) & _U32(31)))
        return [(w, m)]
    one = np.uint64(1)
    if layout == "word64":
        w = _umulhi(hm, seg_words >> 1).astype(np.int64)
        m = ((one << (g >> _U32(26)).astype(np.uint64)) | (one << ((g >> _U32(20)) & _U32(63)).astype(np.uint64)) |
             (one << ((g >> _U32(14)) & _U32(63)).astype(np.uint64)))
        return [(w, m)]
    assert layout == "sector"
    g = g ^ (g >> _U32(16))
    s = _umulhi(hm, seg_words >> 3).astype(np.int64) * 4
    w0 = s + (g >> _U32(30)).astype(np.int64)
    w1 = s + ((g >> _U32(28)) & _U32(3)).astype(np.int64)
    m0 = (one << ((g >> _U32(22)) & _U32(63)).astype(np.uint64)) | (one << ((g >> _U32(16)) & _U32(63)).astype(np.uint64))
    m1 = (one << ((g >> _U32(10)) & _U32(63)).astype(np.uint64)) | (one << ((g >> _U32(4)) & _U32(63)).astype(np.uint64))
    return [(w0, m0), (w1, m1)]


def build_filter(layout, hi, lo, k, seg_words):
    """one segment of seg_words uint32 with every key (hi, lo) inserted, as bloom_insert leaves it"""
    h, g = slot_hashes(hi, lo, k)
    f = np.zeros(seg_words if layout == "word32" else seg_words // 2,
                 dtype=np.uint32 if layout == "word32" else np.uint64)
    for w, m in slots(layout, h, g, seg_words):
        np.bitwise_or.at(f, w, m)
    return f if layout == "word32" else f.view(np.uint32)


def test_filter(layout, f, hi, lo, k, seg_words):
    """the look-up of sweep: are all of the key's bits set in segment f (uint32[seg_words])?"""
    h, g = slot_hashes(hi, lo, k)
    fw = f if layout == "word32" else f.view(np.uint64)
    hit = np.ones(len(h), dtype=bool)
    for w, m in slots(layout, h, g, seg_words):
        hit &= (fw[w] & m) == m
    return hit


def seg_words_for(n, bits=1):
    """hm_symm_plan's segment size (one segment)"""
    segw = max((n * bits + 31) // 32, 1024)
    return (segw + 63) & ~63


def revcomp(x, k):
    """reverse complement of left-aligned k-mers, k <= 32 (uint64)"""
    r = np.zeros_like(x)
    v = x >> np.uint64(64 - 2 * k)
    for _ in range(k):
        r = (r << np.uint64(2)) | (np.uint64(3) - (v & np.uint64(3)))
        v = v >> np.uint64(2)
    return r << np.uint64(64 - 2 * k)


def s_and_candidates(keys, cnt, k):
    """pass 1's S (mask) and candidate records (x, p, yb) of a sorted table, k <= 31: every entry's partners
    at the positions >= k/2 found by look-ups in the table"""
    n = len(keys)
    Pr, pup = k // 2, k - k // 2
    H = np.zeros(n, dtype=np.int32)
    U = np.zeros(n, dtype=np.int32)
    part = np.full(n, -1, dtype=np.int64)
    ppos = np.zeros(n, dtype=np.int32)
    c = cnt.astype(np.int64)
    for p in range(Pr, k):
        sh = np.uint64(62 - 2 * p)
        b = (keys >> sh) & np.uint64(3)
        for d in (1, 2, 3):
            y = (keys & ~(np.uint64(3) << sh)) | (((b + np.uint64(d)) & np.uint64(3)) << sh)
            j = np.searchsorted(keys, y)
            jc = np.minimum(j, n - 1)
            ok = (keys[jc] == y) & (c + c[jc] <= SMAX)
            H += ok
            if p >= pup:
                U += ok
            part[ok] = jc[ok]
            ppos[ok] = p
    i = np.arange(n)
    cand = (H == 1) & (part > i)
    cand &= H[np.maximum(part, 0)] == 1
    x = keys[cand]
    p = ppos[cand]
    yb = ((keys[part[cand]] >> (np.uint64(62) - np.uint64(2) * p.astype(np.uint64))) & np.uint64(3)).astype(np.int64)
    return U > 0, x, p, yb


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nels", type=float, default=4e6)
    ap.add_argument("--seed", type=int, default=None, help="table seed (default: bench.py's)")
    args = ap.parse_args()
    from bench import COV, HET, K, LCUT, PLOIDY, SEED
    from tools import synth
    assert K <= 31
    G = synth.calibrate_G(K, int(args.nels), PLOIDY, HET, COV, LCUT)
    keys, cnt = synth.synth_table(K, G, PLOIDY, HET, COV, LCUT, SEED if args.seed is None else args.seed)
    keys = synth.keys_to_u64_numpy(keys)
    cnt = cnt.numpy()
    n = len(keys)
    inS, x, p, yb = s_and_candidates(keys, cnt, K)
    rx = revcomp(x, K)
    sh = np.uint64(62) - np.uint64(2) * (K - 1 - p).astype(np.uint64)
    ry = (rx & ~(np.uint64(3) << sh)) | ((np.uint64(3) - yb.astype(np.uint64)) << sh)
    segw = seg_words_for(n)
    sk = keys[inS]
    scale = 2e8 / n
    out = {"workload": f"bench.py configs[1] (k={K}) scaled to {n} entries", "nels": n, "S": int(inS.sum()),
           "candidates": len(x), "seg_words": segw, "bits_per_S": round(32 * segw / max(int(inS.sum()), 1), 2),
           "rcx_in_S": int(np.isin(rx, sk).sum()), "rcy_in_S": int(np.isin(ry, sk).sum())}
    for lay in LAYOUTS:
        f = build_filter(lay, sk, None, K, segw)
        ha = test_filter(lay, f, rx, None, K, segw)
        hb = test_filter(lay, f, ry, None, K, segw)
        r = {"rcx_only": int((ha & ~hb).sum()), "rcy_only": int((hb & ~ha).sum()), "both": int((ha & hb).sum())}
        r["hit_share"] = round((r["rcx_only"] + r["rcy_only"] + r["both"]) / max(len(x), 1), 4)
        r["fp_per_lookup"] = round((ha.sum() + hb.sum()) / max(2 * len(x), 1), 4)
        r["at_2e8"] = {key: float(f"{r[key] * scale:.3g}") for key in ("rcx_only", "rcy_only", "both")}
        out[lay] = r
    out["candidates_at_2e8"] = float(f"{len(x) * scale:.3g}")
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
