"""CPU tests of the pair-file writing of dist.ShardedScan / StreamedShardedScan.write_pairs (DESIGN.md §6b):
hetmers.read_sma against the extract_kmer_pairs executable (which parses the .sma before it opens the table), the
window plan, a numpy restatement of the file phase applied to the oracle's pair lists, and the host side of the
writing (file creation, offsets, pwrite by gloo ranks, clean-up on failure)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import GOLDEN, ROOT

ORDER = ["smudge", "key_hi", "key_lo", "pos", "alt"]
SMA_GOLDENS = ["dip_k21", "dip_k40", "tet_k32"]
EXE = os.path.join(ROOT, "smudgeplot_b200", "bin", "extract_kmer_pairs")
HEADER = "covB\tcovA\tfreq\tsmudge\n"

CRAFTED = {                                       # name: (file name, text or None = no file)
    "missing": ("missing.sma", None),
    "unparsable": ("u.sma", HEADER + "3 4 5 1A1B\n3 x 5 1A1B\n"),
    "a_below_b": ("ab.sma", HEADER + "3 4 5 1A2B\n"),
    "zero_label": ("z.sma", HEADER + "3 4 5 0A0B\n"),
    "pixel_out_of_range": ("p.sma", HEADER + "400 700 5 1A1B\n"),
    "pixel_below_diagonal": ("q.sma", HEADER + "5 4 5 1A1B\n"),
    "repeated_pixel": ("r.sma", HEADER + "3 4 5 1A1B\n7 9 1 2A1B\n3 4 2 3A1B\n"),
    "trailing_text": ("t.sma", HEADER + "  3\t4 5 2A1B extra words\n8 9 1 1A1Bxyz\n"),
    "header_only": ("h.sma", HEADER),
    "upper_suffix": ("s.SMA", HEADER + "3 4 5 1A1B\n"),
}


def _executable(sma_arg, out, tmp_path):
    return subprocess.run([EXE, f"-o{out}", str(tmp_path / "no_such_table"), sma_arg], capture_output=True, text=True)


@pytest.mark.parametrize("case", sorted(CRAFTED))
def test_read_sma_is_the_executables_parser(case, tmp_path, built):
    """a malformed .sma: the executable's message and exit 1, read_sma raising that message; a valid one, run with
    a missing table: exactly the label files read_sma names are left"""
    from smudgeplot_b200 import hetmers
    fname, text = CRAFTED[case]
    if text is not None:
        with open(tmp_path / fname, "w") as f:
            f.write(text)
    arg = str(tmp_path / fname)                    # (s.SMA: both take <root>.SMA as <root>)
    out = str(tmp_path / "o")
    r = _executable(arg, out, tmp_path)
    assert r.returncode == 1
    try:
        pix, labels = hetmers.read_sma(arg)
    except ValueError as e:
        assert str(e) in r.stderr, (str(e), r.stderr)
        assert "Cannot open k-mer table" not in r.stderr
        return
    assert "Cannot open k-mer table" in r.stderr, r.stderr
    left = sorted(f for f in os.listdir(tmp_path) if f.startswith("o."))
    assert left == sorted(f"o.{a}A{b}B.txt" for a, b in labels)
    if case == "repeated_pixel":                    # the later line wins the pixel; labels keep first appearance
        assert labels == [(1, 1), (2, 1), (3, 1)] and pix[7, 3] == 3 and pix[16, 7] == 2
    if case == "header_only":
        assert labels == [] and not pix.any()


def test_read_sma_on_the_goldens():
    import test_gpu_stream_dist_extract as sde
    from smudgeplot_b200 import hetmers
    for name in SMA_GOLDENS:
        path = os.path.join(GOLDEN, name, name + ".sma")
        pix, labels = hetmers.read_sma(path)
        want, order = sde.read_sma(path)
        assert np.array_equal(pix, want) and [f"{a}A{b}B" for a, b in labels] == order
        assert np.array_equal(hetmers.read_sma(path[:-4])[0], want)


# ------------------------------------------------------------------ the window plan ----------------------------

@pytest.mark.parametrize("world", [1, 2, 3])
@pytest.mark.parametrize("seed", range(4))
def test_window_plan(world, seed):
    """the fewest passes whose windows fit the room, P * world windows, every window within the room"""
    from smudgeplot_b200 import dist as hd
    rng = np.random.default_rng(seed)
    h = rng.integers(0, 30, size=1 << 12) * (rng.random(1 << 12) < 0.5)
    before = np.concatenate([[0], np.cumsum(h)])
    for room in (int(h.max()), 100, 1000, int(h.sum())):
        P, cuts = hd.pair_windows(h, world, room)
        assert len(cuts) == P * world + 1 and cuts[0] == 0 and cuts[-1] == h.size
        assert all(a <= b for a, b in zip(cuts, cuts[1:]))
        assert np.diff(before[cuts]).max() <= room
        if P > 1:                                     # one pass fewer does not fit
            fewer = hd.condition_cuts(h, (P - 1) * world)
            assert np.diff(before[fewer]).max() > room
        assert P >= -(-int(h.sum()) // (room * world))


def test_window_plan_refuses_an_oversized_prefix():
    from smudgeplot_b200 import _lib
    from smudgeplot_b200 import dist as hd
    h = np.zeros(1 << 10, dtype=np.int64)
    h[77] = 500
    h[3] = 20
    with pytest.raises(_lib.HetmersError) as ei:
        hd.pair_windows(h, 2, 499)
    assert ei.value.code == -3 and "prefix 77 holds 500 records" in str(ei.value) and "499" in str(ei.value)
    assert hd.pair_windows(h, 2, 500)[0] == 1
    assert hd.pair_windows(np.zeros(16, dtype=np.int64), 3, 0) == (1, [0, 16, 16, 16])


def test_pairs_room_is_the_largest_window_the_model_allows():
    from smudgeplot_b200 import _lib
    from smudgeplot_b200 import dist as hd
    f = _lib.lib().hm_pairs_bytes
    assert f(21, -1) == -1 and f(0, 5) == -1
    for k in (2, 21, 40, 64):
        assert all(f(k, r) <= f(k, r + 1) for r in range(0, 5000, 7))
        for budget in (f(k, 0) - 1, f(k, 0), 64 << 20, 3 << 30):
            r = hd.pairs_room(k, budget)
            if r < 0:
                assert f(k, 0) > budget
                continue
            assert f(k, r) <= budget < f(k, r + 1)


# ------------------------------------------------------------------ numpy restatement of the file phase ---------

def pair_line(key_hi, key_lo, k, pos, alt):
    dna = "acgt"
    out = []
    for p in range(k):
        b = ((key_hi if p < 32 else key_lo) >> (62 - 2 * (p & 31))) & 3
        out.append(f"({dna[b]}/{dna[alt]})" if p == pos else dna[b])
    return "".join(out) + "\n"


def parse_line(line, k):
    """a print_het line -> (key_hi, key_lo, pos, alt)"""
    i = line.index("(")
    bases = line[:i] + line[i + 1] + line[i + 5:]
    v = ["acgt".index(c) for c in bases]
    hi = sum(b << (62 - 2 * p) for p, b in enumerate(v[:32]))
    lo = sum(b << (62 - 2 * p) for p, b in enumerate(v[32:]))
    return hi, lo, i, "acgt".index(line[i + 3])


def file_phase(rank_recs, k, n_labels, world, room):
    """write_pair_files restated: histogram, plan, per pass route / sort / count / segments -> {label: bytes}"""
    from smudgeplot_b200 import dist as hd
    hb = min(20, 2 * k)
    every = np.concatenate(rank_recs)
    h = np.bincount((every["key_hi"] >> np.uint64(64 - hb)).astype(np.int64), minlength=1 << hb)
    P, cuts = hd.pair_windows(h, world, room)
    files = [bytearray() for _ in range(n_labels + 1)]
    before = np.zeros(n_labels + 1, dtype=np.int64)
    for p in range(P):
        wins, counts = [], []
        for d in range(world):
            lo, hi = cuts[p * world + d], cuts[p * world + d + 1]
            got = [r[((r["key_hi"] >> np.uint64(64 - hb)) >= lo) & ((r["key_hi"] >> np.uint64(64 - hb)) < hi)]
                   for r in rank_recs]
            w = np.sort(np.concatenate(got), order=ORDER)
            wins.append(w)
            counts.append(np.bincount(w["smudge"].astype(np.int64), minlength=n_labels + 1))
        for d, w in enumerate(wins):
            text = "".join(pair_line(int(r["key_hi"]), int(r["key_lo"]), k, int(r["pos"]), int(r["alt"]))
                           for r in w).encode()
            for s, a, nb, off in hd.window_segments(counts, d, before, k + 5):
                f = files[s]
                f.extend(b"\0" * max(0, off + nb - len(f)))
                f[off:off + nb] = text[a:a + nb]
        before += np.sum(counts, axis=0)
    return files


@pytest.mark.parametrize("name", SMA_GOLDENS)
def test_file_phase_restatement_gives_the_golden_files(name, tmp_path):
    """the oracle's lists of the golden tables, split over 1-3 ranks and cut into windows of 1-3 passes: the files
    hold the golden pair files' lines, in the executable's order (smudge, key, position, alternative base)"""
    import oracle_util as ou
    from smudgeplot_b200 import fastk, hetmers
    from smudgeplot_b200.hetmers import PAIR_DTYPE
    path = os.path.join(GOLDEN, name, name)
    k = fastk.read_ktab(path).kmer
    assert ou.oracle_extract(path, 4, path + ".sma", str(tmp_path / "ora")) == 0
    _, labels = hetmers.read_sma(path + ".sma")
    recs = []
    for s, (a, b) in enumerate(labels, 1):
        with open(tmp_path / f"ora.{a}A{b}B.txt") as f:
            for ln in f.read().splitlines():
                hi, lo, pos, alt = parse_line(ln, k)
                recs.append((hi, lo, s, pos, alt, 0))
    recs = np.array(recs, dtype=PAIR_DTYPE)
    np.random.default_rng(1).shuffle(recs)
    ordered = np.sort(recs, order=ORDER)
    want = {s: "".join(pair_line(int(r["key_hi"]), int(r["key_lo"]), k, int(r["pos"]), int(r["alt"]))
                       for r in ordered[ordered["smudge"] == s]).encode() for s in range(1, len(labels) + 1)}
    for s, (a, b) in enumerate(labels, 1):
        with open(os.path.join(GOLDEN, name, f"{name}.pairs.{a}A{b}B.txt")) as f:
            assert sorted(want[s].decode().splitlines()) == sorted(f.read().splitlines())
    for world in (1, 2, 3):
        parts = np.array_split(recs, world)
        for room in (len(recs), len(recs) // 5 + 1):
            files = file_phase(parts, k, len(labels), world, room)
            assert {s: bytes(files[s]) for s in want} == want, (world, room)


# ------------------------------------------------------------------ the host side, with gloo ranks ---------------

def _worker(rank, world, port, d, labels, k, fail_rank, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import torch
        from smudgeplot_b200 import dist as hd
        from test_dist_extract import records
        coll = torch.device("cpu")
        paths = hd.label_paths(os.path.join(d, "o"), labels)
        try:
            files = hd.PairFiles(paths, None, coll)
            recs = records(rank, 500 + 300 * rank, 9)
            recs["smudge"] = recs["smudge"] % len(labels) + 1
            recs["key_lo"] = 0
            recs["pos"] %= k
            w = np.sort(recs, order=ORDER)                 # one pass: this rank's window is its own records
            own = np.bincount(w["smudge"].astype(np.int64), minlength=len(labels) + 1)
            every = torch.zeros((world, len(labels) + 1), dtype=torch.int64)
            every[rank] = torch.from_numpy(own)
            dist.all_reduce(every)
            if rank == fail_rank:                           # its pwrites fail: bad file descriptors
                for fd in files.fds:
                    os.close(fd)
            text = "".join(pair_line(int(r["key_hi"]), 0, k, int(r["pos"]), int(r["alt"])) for r in w).encode()
            for s, a, nb, off in hd.window_segments(every.numpy(), rank, np.zeros(len(labels) + 1, np.int64), k + 5):
                files.write(s, text[a:a + nb], off)
            files.close()
            files.check("writing")
            q.put((rank, ("ok", w.tobytes())))
        except OSError as e:
            q.put((rank, ("error", str(e))))
    finally:
        dist.barrier()
        dist.destroy_process_group()


def _run(world, d, labels, k, fail_rank=-1):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 33900 + (os.getpid() % 2000) + 10 * world + (fail_rank + 1)
    procs = [ctx.Process(target=_worker, args=(r, world, port, d, labels, k, fail_rank, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=300) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    return [res[r] for r in range(world)]


@pytest.mark.parametrize("world", [1, 2, 3])
def test_ranks_write_their_segments(world, tmp_path, built):
    """rank d's window precedes rank d+1's: every file is the ranks' sorted lines of its label in rank order, and an
    existing longer file is truncated first"""
    from smudgeplot_b200.hetmers import PAIR_DTYPE
    labels, k = [(1, 1), (2, 1), (9, 2)], 21
    with open(tmp_path / "o.2A1B.txt", "w") as f:
        f.write("z" * 100_000)
    res = _run(world, str(tmp_path), labels, k)
    assert all(r[0] == "ok" for r in res), res
    wins = [np.frombuffer(r[1], dtype=PAIR_DTYPE) for r in res]
    for s, (a, b) in enumerate(labels, 1):
        want = "".join(pair_line(int(r["key_hi"]), 0, k, int(r["pos"]), int(r["alt"]))
                       for w in wins for r in w[w["smudge"] == s])
        with open(tmp_path / f"o.{a}A{b}B.txt") as f:
            assert f.read() == want


@pytest.mark.parametrize("world,fail_rank", [(1, 0), (2, 1), (3, 0), (3, 2)])
def test_a_failed_write_raises_everywhere_and_leaves_no_file(world, fail_rank, tmp_path, built):
    res = _run(world, str(tmp_path), [(1, 1), (2, 1)], 31, fail_rank)
    assert all(r[0] == "error" and "failed on some rank" in r[1] for r in res), res
    assert not [f for f in os.listdir(tmp_path) if f.startswith("o.")]
