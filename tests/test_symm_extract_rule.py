"""CPU pin of the pair-listing rule of hm_k_symm_extract (csrc/hm_symm.cu, DESIGN.md §4a), against the oracle's
extract_kmer_pairs: on a strand-symmetric table, each isolated candidate pair (x < y, differing at a position
p >= k/2) stands for itself and -- unless it differs at the middle base of an odd k -- for its mirror image
(rc y, rc x), and each is listed as pass2_extract_kernel lists it.  `partial_extract` restates the kernel's
contract in Python (next to oracle_util.partial_runscan / partial_resolve, for any k <= 64); the test requires its
records to be exactly the oracle's lines for a .sma that labels every pixel.  No GPU needed; the GPU tests
(test_gpu_symm_extract.py) compare the kernel with the direct passes."""
import numpy as np
import pytest

import oracle_util as ou
from smudgeplot_b200 import fastk

SMAX = ou.SMAX


def partial_extract(keys, cnt, k: int, pixmap, lo: int = 0, hi=None):
    """what hm_k_symm_extract lists for the candidates of the run-aligned range [lo,hi) of a symmetric table (keys:
    python ints, left aligned in 64 bits for k <= 32 and in 128 bits, (hi word << 64) | lo word, for k > 32).  A
    candidate (x < y, one partner each among positions >= k/2, differing at p with bases bx < by, counts cx, cy)
    that is isolated -- neither rc x nor rc y has a partner at a position >= k - k/2 -- and whose pixel
    (cx+cy, min) has a label gives the pair itself: y with alt bx if cx < cy, else x with alt by, at p; and,
    unless 2p = k-1, its mirror image (u, v) = (rc y, rc x) at k-1-p with counts (cy, cx): v with alt 3-by if
    cy < cx, else u with alt 3-bx.  -> list of (key, label, pos, alt), one per line extract_kmer_pairs writes"""
    keys = [int(x) for x in keys]
    cnt = [int(c) for c in cnt]
    hi = len(keys) if hi is None else hi
    W = 64 if k <= 32 else 128
    pos_of = {x: i for i, x in enumerate(keys)}
    Pr, pup = k // 2, k - k // 2

    def rc(x):
        v, r = x >> (W - 2 * k), 0
        for _ in range(k):
            r = (r << 2) | (3 - (v & 3))
            v >>= 2
        return r << (W - 2 * k)

    def partners(x, cx, p0):
        out = []
        for p in range(p0, k):
            sh = W - 2 - 2 * p
            b = (x >> sh) & 3
            for alt in range(4):
                if alt != b:
                    j = pos_of.get((x & ~(3 << sh)) | (alt << sh))
                    if j is not None and cx + cnt[j] <= SMAX:
                        out.append((j, p))
        return out

    recs = []
    for i in range(lo, hi):
        x, cx = keys[i], cnt[i]
        pr = partners(x, cx, Pr)
        if len(pr) != 1 or pr[0][0] < i:
            continue
        j, p = pr[0]
        y, cy = keys[j], cnt[j]
        if len(partners(y, cy, Pr)) != 1:
            continue
        rx, ry = rc(x), rc(y)
        if partners(rx, cx, pup) or partners(ry, cy, pup):               # rc x or rc y is in S: not isolated
            continue
        lab = int(pixmap[cx + cy][min(cx, cy)])
        if lab == 0:
            continue
        sh = W - 2 - 2 * p
        bx, by = (x >> sh) & 3, (y >> sh) & 3
        recs.append((y, lab, p, bx) if cx < cy else (x, lab, p, by))
        if 2 * p != k - 1:
            q = k - 1 - p
            recs.append((rx, lab, q, 3 - by) if cy < cx else (ry, lab, q, 3 - bx))
    return recs


def pair_line(key: int, k: int, pos: int, alt: int) -> str:
    """extract_kmer_pairs' line for a record (print_het, PloidyList.c:128-165); key as in partial_extract"""
    W = 64 if k <= 32 else 128
    dna = "acgt"
    bases = [(key >> (W - 2 - 2 * p)) & 3 for p in range(k)]
    return "".join(f"({dna[b]}/{dna[alt]})" if p == pos else dna[b] for p, b in enumerate(bases))


def _symmetric_table_any_k(k, n0, counts, seed, palindromes=0):
    """strand-symmetric table for 2 <= k <= 64: keys as python ints left aligned in 64 bits (k <= 32) or 128 bits
    (k > 32), sorted, and their counts (equal for x and rc x).  Partners are planted at random positions;
    `palindromes` (even k) adds k-mers equal to their own reverse complement, with planted partners too.
    counts: "ties" (1..4), "wide" (1..40) or "smax" (around SMAX/2, so that count sums straddle SMAX)."""
    rng = np.random.default_rng(seed)
    W = 64 if k <= 32 else 128

    def rc(x):
        v, r = x >> (W - 2 * k), 0
        for _ in range(k):
            r = (r << 2) | (3 - (v & 3))
            v >>= 2
        return r << (W - 2 * k)

    def rand_kmer():
        v = 0
        for b in rng.integers(0, 4, size=k).tolist():
            v = (v << 2) | b
        return v << (W - 2 * k)

    base = {rand_kmer() for _ in range(n0)}
    for _ in range(palindromes):
        h = rand_kmer() >> (W - k)                                       # the first k/2 bases
        x = h << (W - k)
        base.add(x | (rc(x) >> k))
    vals = sorted(base)
    for x in list(vals)[: len(vals) // 2]:                              # one-substitution partners
        p = int(rng.integers(0, k))
        sh = W - 2 - 2 * p
        base.add(x ^ (int(rng.integers(1, 4)) << sh))
    keys = sorted(base | {rc(x) for x in base})
    canon = sorted({min(x, rc(x)) for x in keys})
    if counts == "ties":
        c = rng.integers(1, 5, size=len(canon))
    elif counts == "wide":
        c = rng.integers(1, 41, size=len(canon))
    else:
        c = rng.choice([1, 2, 498, 499, 500, 501, 502], size=len(canon))
    cc = dict(zip(canon, c.tolist()))
    return keys, np.array([cc[min(x, rc(x))] for x in keys], dtype=np.uint16)


def _label_every_pixel(sma):
    """a .sma that gives every pixel (sum <= SMAX, min <= FMAX) one of five smudges; -> (pixmap, label names)"""
    names = ["1A1B", "2A1B", "2A2B", "3A1B", "3A2B"]
    order, pix = [], np.zeros((ou.SMAX + 1, ou.PLOT_W), dtype=np.uint16)
    with open(sma, "w") as f:
        f.write("covB\tcovA\tfreq\tsmudge\n")
        for s in range(ou.SMAX + 1):
            for m in range(min(s // 2, ou.FMAX) + 1):
                lab = names[(7 * s + m) % 5]
                if lab not in order:
                    order.append(lab)
                pix[s, m] = order.index(lab) + 1
                f.write(f"{m}\t{s - m}\t1\t{lab}\n")
    return pix, order


@pytest.mark.parametrize("k,n0,counts,seed,pal", [(4, 60, "wide", 21, 4), (5, 200, "ties", 22, 0), (7, 150, "ties", 23, 0),
                                                  (11, 1500, "smax", 24, 0), (16, 1200, "ties", 25, 40),
                                                  (21, 1500, "wide", 26, 0), (31, 1500, "smax", 27, 0),
                                                  (32, 1000, "ties", 28, 30), (33, 1000, "smax", 29, 0),
                                                  (40, 1200, "ties", 30, 30), (64, 800, "smax", 31, 20)])
def test_symmetric_pair_listing_equals_the_oracle_extract(k, n0, counts, seed, pal, tmp_path):
    """the listing rule of hm_k_symm_extract (partial_extract: each isolated candidate once, its mirror image
    too unless it differs at the middle base of an odd k) gives exactly extract_kmer_pairs' lines, as the oracle
    (the reference's algorithm restated) writes them for a .sma that labels every pixel"""
    keys, cnt = _symmetric_table_any_k(k, n0, counts, seed, pal)
    kb = (k + 3) // 4
    W = 64 if k <= 32 else 128
    kbytes = np.array([list(x.to_bytes(W // 8, "big")[:kb]) for x in keys], dtype=np.uint8)
    name = str(tmp_path / "t")
    fastk.write_ktab(name, k, kbytes, cnt, ibyte=1, nparts=2)
    pix, order = _label_every_pixel(str(tmp_path / "all.sma"))
    assert ou.oracle_extract(name, 1, str(tmp_path / "all.sma"), str(tmp_path / "ora")) == 0
    want = ou.sorted_pair_files(str(tmp_path / "ora"))
    recs = partial_extract(keys, cnt, k, pix)
    got = {}
    for key, lab, pos, alt in recs:
        got.setdefault(order[lab - 1], []).append(pair_line(key, k, pos, alt))
    got = {lab: sorted(v) for lab, v in got.items()}
    want = {lab: v for lab, v in want.items() if v}                      # (the oracle opens a file per smudge)
    assert got == want, ou.first_pair_difference(got, want)
    assert sum(len(v) for v in want.values()) > 0 or k <= 5
    if k % 2 == 1:                                                       # middle-base pairs are listed once
        assert any(pos == k // 2 for _, _, pos, _ in recs) or k <= 7
