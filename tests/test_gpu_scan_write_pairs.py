"""GPU tests of extract_kmer_pairs' pair files written in one process (hetmers.Scan.write_pairs, hm_scan_write_pairs,
DESIGN.md §6c; run with -m gpu): every label file byte for byte what the executable writes, what a numpy formatter
makes of Scan.extract's list, and on the goldens the reference's sorted pair lists -- on both routes, under budgets
that force several passes or refuse the plan, and on several GPUs when the box has them."""
import json
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN
import oracle_util as ou
from smudgeplot_b200 import _lib, fastk, hetmers

pytestmark = pytest.mark.gpu

SMA_GOLDENS = ["dip_k21", "dip_k40", "tet_k32"]


@pytest.fixture(autouse=True)
def _need_gpu(built, monkeypatch):
    if _lib.lib().hm_device_count() < 1:
        pytest.skip("no CUDA device")
    monkeypatch.delenv("HETMERS_PATH", raising=False)
    monkeypatch.delenv("HETMERS_DEVICE_BUDGET", raising=False)
    _lib.lib().hm_set_device_budget(0)
    yield
    _lib.lib().hm_set_device_budget(0)


def numpy_files(recs, k, labels):
    """{label name: bytes}: print_het lines of a sorted record list, formatted in numpy"""
    from tools.time_write_pairs import _lines
    dna = np.frombuffer(b"acgt", dtype=np.uint8)
    return {f"{a}A{b}B": _lines(recs[recs["smudge"] == s], k, dna) if (recs["smudge"] == s).any() else b""
            for s, (a, b) in enumerate(labels, 1)}


def files(out, labels):
    got = {}
    for a, b in labels:
        with open(f"{out}.{a}A{b}B.txt", "rb") as f:
            got[f"{a}A{b}B"] = f.read()
    return got


def conditioned_scan(kt, e, gpus=1):
    """a Scan conditioned as the executable conditions it under -e<e>"""
    sc = hetmers.Scan(kt, gpus=gpus)
    trim, symm = sc.examine(e)
    if not (trim and symm):
        sc.condition(e, not trim, not symm)
    return sc


def check_table(table, sma, e, tmp_path, tag, gpus=1, exe=True):
    """Scan.write_pairs == the executable == numpy of Scan.extract; -> (files, stats)"""
    pix, labels = hetmers.read_sma(sma)
    with conditioned_scan(fastk.read_ktab(table), e, gpus) as sc:
        sc.run()
        recs = sc.extract(pix)
        st = sc.write_pairs(sma, str(tmp_path / f"w{tag}"))
        assert np.array_equal(sc.extract(pix), recs)
    got = files(str(tmp_path / f"w{tag}"), labels)
    assert got == numpy_files(recs, fastk.read_ktab(table).kmer, labels)
    assert st["records"] == len(recs) and st["passes"] >= 1 and st["planned"] == 1
    assert st["lines"] == {n: v.count(b"\n") for n, v in got.items()}
    if exe:
        hetmers.run_extract(table, sma, o=str(tmp_path / f"x{tag}"), e=e)
        assert files(str(tmp_path / f"x{tag}"), labels) == got
    return got, st


@pytest.mark.parametrize("route", ["auto", "direct", "symm"])
@pytest.mark.parametrize("name", SMA_GOLDENS)
def test_goldens(name, route, golden_meta, tmp_path, monkeypatch):
    from test_gpu_parity import _golden_pairs
    if route != "auto":
        monkeypatch.setenv("HETMERS_PATH", route)
    table = os.path.join(GOLDEN, name, name)
    got, st = check_table(table, table + ".sma", golden_meta[name]["e"], tmp_path, name)
    assert st["path"] == {"auto": st["path"], "direct": 1, "symm": 2}[route]
    assert {n: sorted(v.decode().splitlines()) for n, v in got.items()} == _golden_pairs(name)


@pytest.mark.parametrize("case", range(2))
def test_seeded_extract_cases_carry_the_reference_digests(case, tmp_path):
    from test_gpu_parity import EXTRACT_CASES, write_labelled_sma
    from tools import synth
    k, G, ploidy, seed, L = EXTRACT_CASES[case]
    keys, cnt = synth.synth_table(k, G, ploidy, 0.02, 20 * ploidy, L, seed, device="cuda")
    name = str(tmp_path / "t")
    kt = synth.write_table(name, k, keys, cnt, ibyte=3, nparts=3)
    sma = str(tmp_path / "ann.sma")
    with hetmers.Scan(kt) as sc:
        write_labelled_sma(sc.run()[0], sma)
    check_table(name, sma, L, tmp_path, "s")
    assert ou.pair_digests(ou.sorted_pair_files(str(tmp_path / "ws"))) == ou.reference_pair_digests(k, seed)


def seeded_sma(kt, sma):
    from test_gpu_parity import write_labelled_sma
    with hetmers.Scan(kt) as sc:
        return write_labelled_sma(sc.run()[0], sma)


@pytest.mark.parametrize("k", [21, 47, 64])
def test_seeded_tables_on_both_routes(k, tmp_path, monkeypatch):
    from test_gpu_symm_extract import seeded_table
    kt = seeded_table(k, 300 + k, str(tmp_path / "t"))
    seeded_sma(kt, str(tmp_path / "a.sma"))
    got, st = check_table(str(tmp_path / "t"), str(tmp_path / "a.sma"), 1, tmp_path, "a")
    assert st["path"] == 2 and sum(map(len, got.values())) > 0
    monkeypatch.setenv("HETMERS_PATH", "direct")
    got_d, st_d = check_table(str(tmp_path / "t"), str(tmp_path / "a.sma"), 1, tmp_path, "d")
    assert st_d["path"] == 1 and got_d == got


@pytest.fixture(scope="module")
def budget_table(tmp_path_factory):
    from test_gpu_symm_extract import seeded_table
    d = tmp_path_factory.mktemp("budget")
    kt = seeded_table(31, 7, str(d / "t"))
    seeded_sma(kt, str(d / "a.sma"))
    with hetmers.Scan(kt) as sc:
        sc.run()
        pix, labels = hetmers.read_sma(str(d / "a.sma"))
        recs = sc.extract(pix)
        h = sc.pairs_hist(pix)
    return d, kt, recs, h, labels


def test_histogram_sweep_is_hm_k_pairs_hist_of_the_list(budget_table, monkeypatch):
    import torch
    d, kt, recs, h, labels = budget_table
    assert h.sum() == len(recs) > 0
    dev = torch.from_numpy(recs.view(np.uint8).copy()).cuda()
    hk = torch.zeros(h.size, dtype=torch.int64, device="cuda")
    _lib.check(_lib.lib().hm_k_pairs_hist(dev.data_ptr(), len(recs), kt.kmer, hk.data_ptr(), None))
    torch.cuda.synchronize()
    assert np.array_equal(hk.cpu().numpy().astype(np.uint64), h)
    monkeypatch.setenv("HETMERS_PATH", "direct")
    with hetmers.Scan(kt) as sc:
        assert np.array_equal(sc.pairs_hist(hetmers.read_sma(str(d / "a.sma"))[0]), h)


def test_a_budget_forcing_three_passes(budget_table, tmp_path):
    """same bytes in >= 3 passes, peak device bytes within the budget; extract() and run() unchanged after it"""
    d, kt, recs, h, labels = budget_table
    want = numpy_files(recs, kt.kmer, labels)
    L = _lib.lib()
    with hetmers.Scan(kt) as sc:
        plot, _ = sc.run()
        held = sc.residency()[1]
        room = len(recs) // 3 - 1
        budget = held + L.hm_pairs_bytes(kt.kmer, room) + 2 * _lib.PLOT_CELLS + 256
        st = sc.write_pairs(str(d / "a.sma"), str(tmp_path / "w"), device_budget=budget)
        assert st["passes"] >= 3 and st["windows"] == st["passes"]
        assert st["peak_bytes"] <= st["budget"] <= budget
        assert files(str(tmp_path / "w"), labels) == want
        L.hm_set_device_budget(0)
        assert np.array_equal(sc.extract(hetmers.read_sma(str(d / "a.sma"))[0]), recs)
        assert np.array_equal(sc.run()[0], plot)


def test_a_budget_below_the_largest_prefix(budget_table, tmp_path):
    """the plan refuses (-3) before any file is touched; the executable under that budget takes the host writer"""
    d, kt, recs, h, labels = budget_table
    L = _lib.lib()
    big = int(h.max())
    victim = tmp_path / f"w.{labels[0][0]}A{labels[0][1]}B.txt"
    victim.write_bytes(b"x" * 100000)
    with hetmers.Scan(kt) as sc:
        sc.run()
        probe = 16 << 30                                   # what the scan holds: the budget less the call's share
        held = probe - sc.write_pairs(str(d / "a.sma"), str(d / "probe"), device_budget=probe)["budget"]
        incore = sc.residency()[1]
        room0 = L.hm_pairs_bytes(kt.kmer, 0) + 2 * _lib.PLOT_CELLS + 256     # a room of 0 records
        budget = held + room0
        with pytest.raises(_lib.HetmersError) as ei:
            sc.write_pairs(str(d / "a.sma"), str(tmp_path / "w"), device_budget=budget)
        assert ei.value.code == -3 and f"holds {big} records" in str(ei.value)
    assert victim.read_bytes() == b"x" * 100000
    assert sorted(os.listdir(tmp_path)) == [victim.name]
    # the executable's scan must stay in core (its in-core bytes fit) and leave no room for the plan
    env = dict(os.environ, HETMERS_DEVICE_BUDGET=str(max(held, incore) + room0 - 1024), HETMERS_STATS="1")
    out = str(tmp_path / "x")
    r = subprocess.run([hetmers.get_binary_path("extract_kmer_pairs"), "-e1", f"-o{out}", str(d / "t"),
                        str(d / "a.sma")], capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr
    stats = json.loads(r.stderr.strip().splitlines()[-1])
    assert stats["pairs"]["writer"] == "host"
    assert files(out, labels) == numpy_files(recs, kt.kmer, labels)
    env.pop("HETMERS_DEVICE_BUDGET")
    r = subprocess.run([hetmers.get_binary_path("extract_kmer_pairs"), "-e1", f"-o{out}g", str(d / "t"),
                        str(d / "a.sma")], capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr
    stats = json.loads(r.stderr.strip().splitlines()[-1])
    assert stats["pairs"]["writer"] == "gpu" and stats["pairs"]["records"] == len(recs)
    assert files(out + "g", labels) == files(out, labels)


def test_empty_labels_and_truncated_files(budget_table, tmp_path):
    d, kt, recs, h, labels = budget_table
    sma = tmp_path / "e.sma"
    text = (d / "a.sma").read_text() + "0\t1\t1\t9A9B\n"                 # a pixel no pair falls on
    sma.write_text(text)
    pix, labs = hetmers.read_sma(str(sma))
    assert labs[-1] == (9, 9)
    longer = tmp_path / "w.9A9B.txt"
    longer.write_bytes(b"y" * 5000)
    first = tmp_path / f"w.{labs[0][0]}A{labs[0][1]}B.txt"
    first.write_bytes(b"z" * (len(recs) * (kt.kmer + 5) + 12345))
    with hetmers.Scan(kt) as sc:
        st = sc.write_pairs(str(sma), str(tmp_path / "w"))
    assert longer.read_bytes() == b"" and st["lines"]["9A9B"] == 0
    assert files(str(tmp_path / "w"), labs) == numpy_files(recs, kt.kmer, labs)


def test_a_streamed_scan_refuses(budget_table, monkeypatch):
    d, kt, recs, h, labels = budget_table
    monkeypatch.setenv("HETMERS_STREAM", "1")
    with hetmers.Scan(kt) as sc:
        assert sc.residency()[0]
        with pytest.raises(_lib.HetmersError) as ei:
            sc.write_pairs(str(d / "a.sma"), str(d / "never"))
        assert ei.value.code == -6
    assert not any(f.startswith("never") for f in os.listdir(d))


def test_two_gpus(budget_table, tmp_path, monkeypatch):
    if _lib.lib().hm_device_count() < 2:
        pytest.skip("needs 2 GPUs")
    d, kt, recs, h, labels = budget_table
    want = numpy_files(recs, kt.kmer, labels)
    for route in ("symm", "direct"):
        monkeypatch.setenv("HETMERS_PATH", route)
        with hetmers.Scan(kt, gpus=2) as sc:
            sc.run()
            st = sc.write_pairs(str(d / "a.sma"), str(tmp_path / f"w{route}"))
            assert np.array_equal(sc.pairs_hist(hetmers.read_sma(str(d / "a.sma"))[0]), h)
        assert st["windows"] == 2 * st["passes"]
        assert files(str(tmp_path / f"w{route}"), labels) == want
