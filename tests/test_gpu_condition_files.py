"""Conditioning to table files on the GPU (hm_scan_condition_files, DESIGN.md §4d): the written table equals the
numpy restatement of trim + symmetrise and the in-core hm_scan_condition, for tables conditioned in one range or
many, from in-core and streamed scans; hetmers then scans the result as trimmed and symmetric."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from conftest import GOLDEN
import oracle_util as ou
from smudgeplot_b200 import _lib, fastk, hetmers
from test_gpu_parity import CONDITIONING_CASES, _condition_numpy, canonical_mask
from tools import synth

pytestmark = pytest.mark.gpu

COND_BIN = os.path.join(os.path.dirname(_lib.BIN_PATH), "condition_kmer_table")


@pytest.fixture(autouse=True)
def _clean_env(monkeypatch, built):
    for var in ("HETMERS_PATH", "HETMERS_STREAM", "HETMERS_STREAM_CHUNK", "HETMERS_DEVICE_BUDGET"):
        monkeypatch.delenv(var, raising=False)
    yield
    _lib.lib().hm_set_device_budget(0)


def table_u64(name):
    kt = fastk.read_ktab(name)
    kb, cn = fastk.unpack_host(kt)
    return fastk.keys_bytes_to_u64(kb), cn, kt


def parts_on_buckets(kt):
    starts = set(np.concatenate([[0], kt.index]).tolist())
    return all(c in starts for c in np.cumsum(kt.part_nels).tolist())


def output_hist(ku, cn, k, L, trim, symm):
    """kept originals + their reverse complements per HM_COND_HIST_BITS-bit key prefix (what pass 0 counts)"""
    hb = min(_lib.COND_HIST_BITS, 2 * k)
    if trim:
        keep = cn >= L
        ku = ku[keep]
    first = ku if ku.ndim == 1 else ku[:, 0]
    h = np.bincount((first >> np.uint64(64 - hb)).astype(np.int64), minlength=1 << hb)
    if symm:
        t = torch.from_numpy(np.ascontiguousarray(ku).view(np.int64))
        if ku.ndim == 2:
            rh, _ = synth.revcomp_long(t[:, 0].contiguous(), t[:, 1].contiguous(), k)
        else:
            rh = synth.revcomp_left(t, k)
        r = rh.numpy().view(np.uint64)
        h = h + np.bincount((r >> np.uint64(64 - hb)).astype(np.int64), minlength=1 << hb)
    return h.astype(np.int64)


def budget_for(hist, n, k, ibyte, ranges, symm=1):
    """the smallest budget (to 1 MB) whose plan has at most `ranges` ranges"""
    L = _lib.lib()
    cuts = np.zeros(len(hist) + 1, dtype=np.int64)
    hb = int(np.log2(len(hist)))

    def nr(b):
        lay = _lib.ConditionLayout()
        rc = L.hm_condition_plan(n, k, ibyte, b, symm, hist.ctypes.data, hb, cuts.ctypes.data, C.byref(lay))
        return lay.n_ranges if rc == 0 else 1 << 40
    lo, hi = 1 << 20, 1 << 36
    while hi - lo > (1 << 20):
        mid = (lo + hi) // 2
        if nr(mid) <= ranges:
            hi = mid
        else:
            lo = mid
    return hi


def held_by_scan(src, L, streamed, monkeypatch, tmp_path):
    """device bytes a scan of src holds, which an explicit budget has to cover besides the call's own"""
    big = 8 << 30
    st = condition(src, str(tmp_path / "held"), L, True, True, big, streamed, monkeypatch)
    fastk.remove_ktab(str(tmp_path / "held"))
    return big - st["budget_bytes"]


def condition(src, dst, L, trim, symm, budget, streamed, monkeypatch):
    if streamed:
        monkeypatch.setenv("HETMERS_STREAM", "1")
    else:
        monkeypatch.delenv("HETMERS_STREAM", raising=False)
    with hetmers.Scan(fastk.read_ktab(src)) as sc:
        assert sc.residency()[0] == streamed
        st = sc.condition_files(dst, L, trim, symm, device_budget=budget)
        assert st["peak_bytes"] <= st["budget_bytes"] <= budget      # what the scan holds comes off the budget
        assert st["passes"] == st["ranges"] + 1
    _lib.lib().hm_set_device_budget(0)
    return st


@pytest.mark.parametrize("k,G,ploidy,seed,L", CONDITIONING_CASES)
def test_canonical_untrimmed_table_to_files(k, G, ploidy, seed, L, tmp_path, monkeypatch):
    keys, cnt = synth.synth_table(k, G, ploidy, 0.02, 40, 1, seed)          # untrimmed: counts from 1
    ku = synth.keys_to_u64_numpy(keys)
    cn = cnt.numpy().astype(np.uint16)
    canon = canonical_mask(keys, ku, k)
    raw = str(tmp_path / "raw")
    fastk.write_ktab(raw, k, ku[canon], cn[canon], ibyte=3, nparts=3)
    ck, cc = _condition_numpy(ku[canon], cn[canon], k, L, True, True)
    with hetmers.Scan(fastk.read_ktab(raw)) as sc:                           # the in-core conditioning
        assert sc.condition(L, True, True) == len(cc)
        k2, c2, _ = sc.download(deg=False)
    assert np.array_equal(k2, ck) and np.array_equal(c2, cc)
    hist = output_hist(ku[canon], cn[canon], k, L, True, True)
    n = int(canon.sum())
    budgets = [8 << 30] + [budget_for(hist, n, k, 3, r) for r in (3, 10)]
    seen = set()
    for streamed in (False, True):
        held = held_by_scan(raw, L, streamed, monkeypatch, tmp_path)
        for b in budgets:
            b = b if b == budgets[0] else b + held
            out = str(tmp_path / f"out{int(streamed)}_{b}")
            st = condition(raw, out, L, True, True, b, streamed, monkeypatch)
            seen.add(st["ranges"])
            gk, gc, kt = table_u64(out)
            assert np.array_equal(gk, ck) and np.array_equal(gc, cc), (streamed, b, st)
            assert st["nels_out"] == len(cc) and kt.nparts == 3 and parts_on_buckets(kt)
            assert kt.minval == L
    assert 1 in seen and max(seen) >= 5
    # hetmers on the result: trimmed and symmetric, streamed under a small budget, the reference's .smu
    env = dict(os.environ, HETMERS_DEVICE_BUDGET=str(budgets[-1]), HETMERS_STREAM="1")
    smu = str(tmp_path / "scan")
    r = subprocess.run([_lib.BIN_PATH, "-v", f"-e{L}", "-T4", f"-o{smu}", out], input="n\n", capture_output=True,
                       text=True, env=env)
    assert r.returncode == 0, r.stderr
    assert "trimmed and symmetric" in r.stderr
    assert open(smu + ".smu").read() == ou.reference_smu("conditioned", k, seed)


def test_trim_only_and_symm_only(golden_meta, tmp_path, monkeypatch):
    for name, (trim, symm) in (("untrimmed", (True, False)), ("asymmetric", (False, True))):
        c = golden_meta["_conditioning"][name]
        src = os.path.join(GOLDEN, "conditioning", name)
        ku, cn, _ = table_u64(src)
        ck, cc = _condition_numpy(ku, cn, 21, c["e"], trim, symm)
        for streamed in (False, True):
            out = str(tmp_path / f"{name}{int(streamed)}")
            condition(src, out, c["e"], trim, symm, 4 << 30, streamed, monkeypatch)
            gk, gc, _ = table_u64(out)
            assert np.array_equal(gk, ck) and np.array_equal(gc, cc), name


@pytest.mark.parametrize("k,ibyte", [(8, 1), (10, 2), (16, 2), (16, 1), (21, 1), (64, 3), (64, 2)])
def test_even_k_palindromes_boundaries_and_k64(k, ibyte, tmp_path, monkeypatch):
    """every k-mer of k = 8 and a random sample of 4^k at k = 10 and 16 (palindromes among them: originals win),
    ranges cut inside stub buckets (2k or 20 prefix bits against 8*ibyte), and k = 64"""
    rng = np.random.default_rng(k * 7 + ibyte)
    if k <= 8:
        x = np.arange(4 ** k, dtype=np.uint64)
    elif k <= 16:
        x = np.unique(rng.integers(0, 4 ** k, size=200_000, dtype=np.uint64))
    if k <= 16:
        ku = (x << np.uint64(64 - 2 * k)).astype(np.uint64)
    else:
        keys, _ = synth.synth_table(k, 40000, 2, 0.02, 30, 1, k)
        ku = synth.keys_to_u64_numpy(keys)
    cn = rng.integers(1, 60, size=len(ku), dtype=np.uint16)
    src = str(tmp_path / "src")
    fastk.write_ktab(src, k, ku, cn, ibyte=ibyte, nparts=2)
    ck, cc = _condition_numpy(ku, cn, k, 5, True, True)
    hist = output_hist(ku, cn, k, 5, True, True)
    b = budget_for(hist, len(ku), k, ibyte, 6)
    for streamed in (False, True):
        out = str(tmp_path / f"out{int(streamed)}")
        held = held_by_scan(src, 5, streamed, monkeypatch, tmp_path)
        st = condition(src, out, 5, True, True, b + held, streamed, monkeypatch)
        gk, gc, kt = table_u64(out)
        assert np.array_equal(gk, ck) and np.array_equal(gc, cc), st
        assert parts_on_buckets(kt) and st["ranges"] >= 2


def test_refusals_leave_no_files_and_the_scan_intact(tmp_path):
    keys, cnt = synth.synth_table(21, 30000, 2, 0.02, 40, 1, 3)
    ku = synth.keys_to_u64_numpy(keys)
    src = str(tmp_path / "src")
    fastk.write_ktab(src, 21, ku, cnt.numpy().astype(np.uint16), ibyte=2, nparts=2)
    dst = str(tmp_path / "dst")
    with hetmers.Scan(fastk.read_ktab(src)) as sc:
        before, _ = sc.run()
        with pytest.raises(_lib.HetmersError) as ei:                  # below one range's working set
            sc.condition_files(dst, 5, True, True, device_budget=20 << 20)
        assert ei.value.code == -3 and "cannot hold one range" in str(ei.value)
        assert not os.path.exists(fastk.stub_path(dst))
        _lib.lib().hm_set_device_budget(0)
        after, _ = sc.run()
        assert np.array_equal(before, after)
        sc.condition(5, True, True)                                     # conditioned in place
        with pytest.raises(_lib.HetmersError) as ei:
            sc.condition_files(dst, 5, True, True)
        assert ei.value.code == -1 and "conditioned in place" in str(ei.value)
    assert sorted(os.listdir(tmp_path)) == sorted([".src.ktab.1", ".src.ktab.2", "src.ktab"])
    # a destination naming the source, however spelled, from a scan of a table read in Python (the C ABI sees no
    # part descriptors there): refused before anything is written, the source's files unchanged
    files = {f: open(tmp_path / f, "rb").read() for f in os.listdir(tmp_path)}
    for mmap in (False, True):
        with hetmers.Scan(fastk.read_ktab(src, mmap=mmap)) as sc:
            for name in (src, src + ".ktab", os.path.join(str(tmp_path), ".", "src")):
                with pytest.raises(_lib.HetmersError) as ei:
                    sc.condition_files(name, 50, True, True)
                assert ei.value.code == -1 and "names the source table" in str(ei.value)
    with pytest.raises(_lib.HetmersError) as ei:
        hetmers.condition_table(src, src + ".ktab", 50)
    assert ei.value.code == -1
    assert {f: open(tmp_path / f, "rb").read() for f in os.listdir(tmp_path)} == files
    r = subprocess.run([COND_BIN, "-e50", src, src], capture_output=True, text=True)  # dst names the source
    assert r.returncode == 1 and "names the source table" in r.stderr
    assert sorted(os.listdir(tmp_path)) == sorted([".src.ktab.1", ".src.ktab.2", "src.ktab"])


def test_prefix_larger_than_a_range_is_refused_after_the_histogram(tmp_path, monkeypatch):
    """a budget that holds the fixed part and a chunk (so the source is read) but not the range one key prefix
    alone needs: HM_ENOMEM from the plan after the histogram pass, still before any file is written"""
    k, n, hb = 31, 2_000_000, _lib.COND_HIST_BITS
    rng = np.random.default_rng(11)
    suf = np.unique(rng.integers(0, 1 << 42, size=n + n // 8, dtype=np.uint64))[:n]
    ku = (np.uint64(0x5A5A5) << np.uint64(44)) | (suf << np.uint64(2))       # one 20-bit prefix for all
    cn = rng.integers(5, 60, size=n, dtype=np.uint16)
    src = str(tmp_path / "src")
    fastk.write_ktab(src, k, ku, cn, ibyte=2, nparts=2)
    hist = output_hist(ku, cn, k, 5, True, True)
    assert hist.max() >= n

    def plan_ok(h, b):
        cuts = np.zeros(len(h) + 1, dtype=np.int64)
        lay = _lib.ConditionLayout()
        return _lib.lib().hm_condition_plan(n, k, 2, b, 1, h.ctypes.data, hb, cuts.ctypes.data, C.byref(lay)) == 0

    zero = np.zeros_like(hist)
    b_fixed = next(b << 20 for b in range(1, 4096) if plan_ok(zero, b << 20))   # fixed part + a chunk fit
    b_range = next(b << 20 for b in range(1, 4096) if plan_ok(hist, b << 20))   # ... and the big prefix
    assert b_range - b_fixed > (48 << 20)
    budget = (b_fixed + b_range) // 2        # the streamed scan holds a few MB of this (plot, fingerprint sums)
    assert plan_ok(zero, budget - (16 << 20)) and not plan_ok(hist, budget)
    monkeypatch.setenv("HETMERS_STREAM", "1")
    dst = str(tmp_path / "dst")
    with hetmers.Scan(fastk.read_ktab(src)) as sc:
        with pytest.raises(_lib.HetmersError) as ei:
            sc.condition_files(dst, 5, True, True, device_budget=budget)
        assert ei.value.code == -3 and "cannot hold one range" in str(ei.value) and str(int(hist.max())) in str(ei.value)
    assert sorted(os.listdir(tmp_path)) == sorted([".src.ktab.1", ".src.ktab.2", "src.ktab"])


def test_condition_kmer_table_executable(tmp_path):
    k, L = 31, 12
    keys, cnt = synth.synth_table(k, 50000, 2, 0.02, 40, 1, 32)
    ku = synth.keys_to_u64_numpy(keys)
    cn = cnt.numpy().astype(np.uint16)
    canon = canonical_mask(keys, ku, k)
    raw = str(tmp_path / "raw")
    fastk.write_ktab(raw, k, ku[canon], cn[canon], ibyte=3, nparts=2)
    out = str(tmp_path / "cond")
    r = subprocess.run([COND_BIN, "-v", f"-e{L}", "-T4", raw, out], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert r.stderr.startswith("\n  The input table is untrimmed and not symmetric\n"
                               f"\n  Trimming k-mers in table with count < {L}\n"
                               "\n  Making trimmed table symmetric\n")
    ck, cc = _condition_numpy(ku[canon], cn[canon], k, L, True, True)
    gk, gc, _ = table_u64(out)
    assert np.array_equal(gk, ck) and np.array_equal(gc, cc)
    # nothing to do: said on stderr, nothing written, exit 0
    again = str(tmp_path / "again")
    r = subprocess.run([COND_BIN, "-v", f"-e{L}", out, again], capture_output=True, text=True)
    assert r.returncode == 0 and "trimmed and symmetric" in r.stderr and "nothing written" in r.stderr
    assert not os.path.exists(fastk.stub_path(again))
    assert hetmers.condition_table(out, again, L) is None
    # argv errors
    for argv, text in (([raw], "Usage"), (["-x", raw, out], "-x is an illegal option"),
                       (["-e0", raw, out], "must be positive"), (["-eZ", raw, out], "is not an integer"),
                       ([str(tmp_path / "none"), out], "Cannot open k-mer table")):
        r = subprocess.run([COND_BIN] + argv, capture_output=True, text=True)
        assert r.returncode == 1 and text in r.stderr, (argv, r.stderr)
    # HETMERS_DEVICE_BUDGET below the smallest range: refused, nothing written
    r = subprocess.run([COND_BIN, f"-e{L}", raw, str(tmp_path / "small")], capture_output=True, text=True,
                       env=dict(os.environ, HETMERS_DEVICE_BUDGET=str(300 << 20), HETMERS_STREAM="1"))
    assert r.returncode == 1 and "cannot hold one range" in r.stderr
    assert not os.path.exists(str(tmp_path / "small.ktab"))


def test_device_memory_is_given_back(tmp_path, monkeypatch):
    monkeypatch.setenv("HETMERS_NO_POOL", "1")
    keys, cnt = synth.synth_table(31, 40000, 2, 0.02, 40, 1, 7)
    src = str(tmp_path / "src")
    fastk.write_ktab(src, 31, synth.keys_to_u64_numpy(keys), cnt.numpy().astype(np.uint16), ibyte=3, nparts=1)
    for streamed in (False, True):
        if streamed:
            monkeypatch.setenv("HETMERS_STREAM", "1")
        with hetmers.Scan(fastk.read_ktab(src)) as sc:
            sc.condition_files(str(tmp_path / "a"), 6, True, True)
            torch.cuda.synchronize()
            before = torch.cuda.mem_get_info(0)[0]
            st = sc.condition_files(str(tmp_path / "b"), 6, True, True, device_budget=2 << 30)
            torch.cuda.synchronize()
            assert torch.cuda.mem_get_info(0)[0] == before
            assert 0 < st["peak_bytes"] <= 2 << 30
            _lib.lib().hm_set_device_budget(0)
