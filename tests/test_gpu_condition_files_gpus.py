"""Conditioning to table files on several GPUs of one process (hm_set_condition_gpus, Scan.condition_files(gpus=n),
HETMERS_GPUS for condition_kmer_table): the files are byte-identical to one GPU's whatever the GPU count and the
ranges, the budget holds on every GPU, and refusals and failures leave no file and the scan usable.  Streamed
scans run their shards on one device listed several times, so every case but the in-core ones runs on one H100."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from conftest import GOLDEN
import oracle_util as ou
from smudgeplot_b200 import _lib, fastk, hetmers
from test_gpu_condition_files import COND_BIN, output_hist, table_u64
from test_gpu_parity import CONDITIONING_CASES, _condition_numpy, canonical_mask
from tools import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _clean_env(monkeypatch, built):
    for var in ("HETMERS_PATH", "HETMERS_STREAM", "HETMERS_STREAM_CHUNK", "HETMERS_DEVICE_BUDGET", "HETMERS_GPUS"):
        monkeypatch.delenv(var, raising=False)
    yield
    _lib.lib().hm_set_device_budget(0)
    _lib.lib().hm_set_condition_gpus(1)


def n_devices():
    return _lib.lib().hm_device_count()


def table_files(name):
    """{file name: bytes} of a table's stub and parts"""
    kt = fastk.read_ktab(name)
    paths = [fastk.stub_path(name)] + [fastk.part_path(name, p) for p in range(1, kt.nparts + 1)]
    return {os.path.basename(p): open(p, "rb").read() for p in paths}


def condition(src, dst, L, trim, symm, devices, gpus, budget, streamed, monkeypatch):
    if streamed:
        monkeypatch.setenv("HETMERS_STREAM", "1")
    else:
        monkeypatch.delenv("HETMERS_STREAM", raising=False)
    with hetmers.Scan(fastk.read_ktab(src), devices=devices) as sc:
        assert sc.residency()[0] == streamed
        st = sc.condition_files(dst, L, trim, symm, device_budget=budget, gpus=gpus)
    _lib.lib().hm_set_device_budget(0)
    g = min(gpus, len(devices))
    assert st["gpus"] == g and len(st["gpu_peak_bytes"]) == g
    assert max(st["gpu_peak_bytes"]) == st["peak_bytes"] <= st["budget_bytes"]        # every GPU within the budget
    assert budget is None or st["budget_bytes"] <= budget
    assert st["passes"] == st["ranges"] + 1
    pbyte = fastk.read_ktab(src).pbyte
    assert st["bytes_read"] == (0 if g > 1 and not streamed else st["passes"] * st["nels_in"] * pbyte)
    return st


def tables():
    """(name, source, L, trim, symm, seed): the conditioning goldens, and seeded canonical untrimmed tables (source
    = their synth_table arguments) whose conditioned .smu the reference wrote"""
    meta = __import__("json").load(open(os.path.join(GOLDEN, "golden.json")))["_conditioning"]
    for name, (trim, symm) in (("untrimmed", (True, False)), ("asymmetric", (False, True))):
        yield name, os.path.join(GOLDEN, "conditioning", name), meta[name]["e"], trim, symm, None
    for k, G, ploidy, seed, L in CONDITIONING_CASES:
        yield f"k{k}", (k, G, ploidy, seed), L, True, True, seed


def make_source(spec, tmp_path):
    if isinstance(spec, str):
        return spec
    k, G, ploidy, seed = spec
    keys, cnt = synth.synth_table(k, G, ploidy, 0.02, 40, 1, seed)          # untrimmed: counts from 1
    ku = synth.keys_to_u64_numpy(keys)
    cn = cnt.numpy().astype(np.uint16)
    canon = canonical_mask(keys, ku, k)
    raw = str(tmp_path / f"raw{k}")
    fastk.write_ktab(raw, k, ku[canon], cn[canon], ibyte=3, nparts=3)
    return raw


def budget_for_ranges(hist, n, k, ibyte, ranges, symm):
    """the smallest planning budget (to 4 KB) whose plan has at most `ranges` ranges"""
    L = _lib.lib()
    cuts = np.zeros(len(hist) + 1, dtype=np.int64)
    hb = int(np.log2(len(hist)))

    def nr(b):
        lay = _lib.ConditionLayout()
        rc = L.hm_condition_plan(n, k, ibyte, b, int(symm), hist.ctypes.data, hb, cuts.ctypes.data, C.byref(lay))
        return lay.n_ranges if rc == 0 else 1 << 40
    lo, hi = 1 << 20, 1 << 36
    while hi - lo > 4096:
        mid = (lo + hi) // 2
        if nr(mid) <= ranges:
            hi = mid
        else:
            lo = mid
    return hi


def named_files(name):
    """table_files(name), the table's own name replaced by "t" (tables of different names compare equal)"""
    return {f.replace(os.path.basename(name), "t"): b for f, b in table_files(name).items()}


def check_gpu_counts(src, L, trim, symm, configs, tmp_path, monkeypatch, streamed, ranges=12):
    """for each (devices, gpus): one range under a large budget (fewer ranges than GPUs), then about `ranges` under
    a small one (several per GPU); every table's files equal the first one's.  -> the last table written"""
    ku, cn, kt = table_u64(src)
    hist = output_hist(ku, cn, kt.kmer, L, trim, symm)
    b = budget_for_ranges(hist, kt.nels, kt.kmer, kt.ibyte, ranges, symm)
    big = 8 << 30
    want, nels = None, None
    for devices, gpus in configs:
        tag = "_".join(map(str, devices))
        one, small = str(tmp_path / f"one{tag}"), str(tmp_path / f"small{tag}")
        st = condition(src, one, L, trim, symm, devices, gpus, big, streamed, monkeypatch)
        assert st["ranges"] == 1
        held = big - st["budget_bytes"]                                # what the scan holds comes off the budget
        st = condition(src, small, L, trim, symm, devices, gpus, b + held, streamed, monkeypatch)
        assert st["budget_bytes"] == b and st["ranges"] >= 2 * gpus
        want = want or named_files(one)
        nels = nels or st["nels_out"]
        assert named_files(one) == want and named_files(small) == want, (devices, gpus)
        assert st["nels_out"] == nels
    return small


@pytest.mark.parametrize("case", [t[0] for t in tables()])
def test_several_gpus_write_the_files_of_one(case, tmp_path, monkeypatch):
    name, spec, L, trim, symm, seed = next(t for t in tables() if t[0] == case)
    src = make_source(spec, tmp_path)
    out = check_gpu_counts(src, L, trim, symm, [([0], 1), ([0, 0], 2), ([0, 0, 0], 3)], tmp_path, monkeypatch, True)
    ku, cn, kt = table_u64(src)
    ck, cc = _condition_numpy(ku, cn, kt.kmer, L, trim, symm)
    gk, gc, _ = table_u64(out)
    assert np.array_equal(gk, ck) and np.array_equal(gc, cc)
    # the conditioned table scans to the reference's / the oracle's plot
    with hetmers.Scan(fastk.read_ktab(out)) as sc:
        plot, _ = sc.run()
    if seed is not None:
        assert hetmers.smu_text(plot) == ou.reference_smu("conditioned", kt.kmer, seed)
    else:
        want_plot, _ = ou.oracle_scan(fastk.keys_u64_to_bytes(ck, kt.kmer), cc, kt.kmer)
        assert np.array_equal(plot, want_plot)


def few_bucket_source(ibyte, nparts, tmp_path):
    """k = 31 entries in a few stub buckets of ibyte bytes, symmetrised into the same buckets: each group's keys
    begin with a prefix P of 4 ibyte bases and end with rc(P), so their reverse complements begin with P too;
    plus a few keys spread over the other buckets"""
    k, rng = 31, np.random.default_rng(ibyte * 10 + nparts)
    p = 4 * ibyte
    groups = []
    for pre, m in ((0b00011011 << (8 * ibyte - 8), 30000), (0b10110001 << (8 * ibyte - 8), 12000)):
        b = rng.integers(0, 4, size=(m, k), dtype=np.int64)
        b[:, :p] = [(pre >> (2 * (p - 1 - i))) & 3 for i in range(p)]
        b[:, k - p:] = 3 - b[:, :p][:, ::-1]
        groups.append(b)
    groups.append(rng.integers(0, 4, size=(2000, k), dtype=np.int64))
    b = np.concatenate(groups)
    ku = np.zeros(len(b), dtype=np.uint64)
    for i in range(k):
        ku |= b[:, i].astype(np.uint64) << np.uint64(62 - 2 * i)
    ku = np.unique(ku)
    src = str(tmp_path / "few")
    fastk.write_ktab(src, k, ku, rng.integers(1, 40, size=len(ku), dtype=np.uint16), ibyte=ibyte, nparts=nparts)
    return src


@pytest.mark.parametrize("ibyte,nparts", [(1, 3), (1, 4), (2, 3), (2, 4)])
def test_ranges_smaller_than_a_stub_bucket(ibyte, nparts, tmp_path, monkeypatch):
    """FastK writes tables with ibyte 1 or 2; a large one under a small budget has many ranges inside one stub
    bucket, so a part cut stays open across several ranges placed by different GPUs"""
    src = few_bucket_source(ibyte, nparts, tmp_path)
    out = check_gpu_counts(src, 5, True, True, [([0], 1), ([0, 0], 2), ([0, 0, 0], 3)], tmp_path, monkeypatch,
                           True, ranges=40)
    ku, cn, kt = table_u64(src)
    ck, cc = _condition_numpy(ku, cn, 31, 5, True, True)
    gk, gc, got = table_u64(out)
    assert np.array_equal(gk, ck) and np.array_equal(gc, cc)
    biggest = int(np.diff(np.concatenate([[0], got.index])).max())
    assert biggest > 8 * len(cc) // 40 and got.nparts == nparts          # a bucket holds many ranges


def test_in_core_scans_on_two_gpus(tmp_path, monkeypatch):
    if n_devices() < 2:
        pytest.skip("needs 2 GPUs")
    for name, spec, L, trim, symm, seed in tables():
        d = tmp_path / name
        d.mkdir()
        src = make_source(spec, d)
        check_gpu_counts(src, L, trim, symm, [([0], 1), ([0, 1], 2)], d, monkeypatch, False)


def test_condition_kmer_table_with_hetmers_gpus(tmp_path):
    if n_devices() < 2:
        pytest.skip("needs 2 GPUs")
    src = make_source((31, 80000, 3, 32), tmp_path)
    outs = {}
    for g in ("1", "2"):
        out = str(tmp_path / f"cond{g}")
        r = subprocess.run([COND_BIN, "-v", "-e12", "-T4", src, out], capture_output=True, text=True,
                           env=dict(os.environ, HETMERS_GPUS=g))
        assert r.returncode == 0, r.stderr
        assert ("2 GPUs)" in r.stderr) == (g == "2")
        outs[g] = list(table_files(out).values())
    assert outs["1"] == outs["2"]


def symmetric_source(tmp_path):
    keys, cnt = synth.synth_table(21, 30000, 2, 0.02, 40, 1, 3)
    src = str(tmp_path / "src")
    fastk.write_ktab(src, 21, synth.keys_to_u64_numpy(keys), cnt.numpy().astype(np.uint16), ibyte=2, nparts=2)
    return src


def test_refusals_leave_no_files_and_the_scan_usable(tmp_path, monkeypatch):
    src = symmetric_source(tmp_path)
    dst = str(tmp_path / "dst")
    monkeypatch.setenv("HETMERS_STREAM", "1")
    with hetmers.Scan(fastk.read_ktab(src), devices=[0, 0]) as sc:
        before, _ = sc.run()
        with pytest.raises(_lib.HetmersError) as ei:                      # below one range's working set
            sc.condition_files(dst, 5, True, True, device_budget=20 << 20, gpus=2)
        assert ei.value.code == -3 and "cannot hold one range" in str(ei.value) and "bytes are fixed" in str(ei.value)
        assert not os.path.exists(fastk.stub_path(dst))
        _lib.lib().hm_set_device_budget(0)
        after, _ = sc.run()
        assert np.array_equal(before, after)
        st = sc.condition_files(dst, 5, True, False, gpus=2)              # and it still conditions
        assert st["gpus"] == 2
    L = _lib.lib()
    L.hm_set_condition_gpus(3)
    with hetmers.Scan(fastk.read_ktab(src), devices=[0, 0]) as sc:
        sc.condition_files(str(tmp_path / "again"), 5, True, False, gpus=2)
    assert L.hm_set_condition_gpus(1) == 3                                # gpus= applies to the call only
    fastk.remove_ktab(str(tmp_path / "again"))
    # a destination naming the source, seen by the C call through the part descriptors hm_table_open keeps
    fastk.remove_ktab(dst)
    files = {f: open(tmp_path / f, "rb").read() for f in os.listdir(tmp_path)}
    L = _lib.lib()
    t, h = C.c_void_p(), C.c_void_p()
    _lib.check(L.hm_table_open(src.encode(), C.byref(t)))
    devs = (C.c_int * 2)(0, 0)
    _lib.check(L.hm_scan_create(L.hm_table_view(t), devs, 2, C.byref(h)))
    L.hm_set_condition_gpus(2)
    st = _lib.ConditionStats()
    rc = L.hm_scan_condition_files(h, 5, 1, 0, (src + ".ktab").encode(), C.byref(st))
    msg = L.hm_last_error().decode()
    L.hm_scan_destroy(h)
    L.hm_table_close(t)
    assert rc == -1 and "names the source table" in msg
    assert {f: open(tmp_path / f, "rb").read() for f in os.listdir(tmp_path)} == files


def test_device_memory_is_given_back(tmp_path, monkeypatch):
    monkeypatch.setenv("HETMERS_NO_POOL", "1")
    monkeypatch.setenv("HETMERS_STREAM", "1")
    src = symmetric_source(tmp_path)
    with hetmers.Scan(fastk.read_ktab(src), devices=[0, 0, 0]) as sc:
        sc.condition_files(str(tmp_path / "a"), 6, True, False, gpus=3)
        torch.cuda.synchronize()
        before = torch.cuda.mem_get_info(0)[0]
        st = sc.condition_files(str(tmp_path / "b"), 6, True, False, device_budget=1 << 30, gpus=3)
        torch.cuda.synchronize()
        assert torch.cuda.mem_get_info(0)[0] == before
        assert 0 < st["peak_bytes"] <= 1 << 30 and st["gpus"] == 3
        with pytest.raises(_lib.HetmersError) as ei:
            sc.condition_files(str(tmp_path / "c"), 6, True, True, device_budget=20 << 20, gpus=3)
        assert ei.value.code == -3
        torch.cuda.synchronize()
        assert torch.cuda.mem_get_info(0)[0] == before
        _lib.lib().hm_set_device_budget(0)
    assert not os.path.exists(str(tmp_path / "c.ktab"))
