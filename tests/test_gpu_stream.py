"""GPU tests of the streamed symmetric scan (DESIGN.md §4c; run with -m gpu on an H100): a table that
does not fit the device budget passes through the GPU in run-aligned chunks and must give exactly the
plot of the in-core scan, the goldens and the stored reference runs, whatever the chunk size; what it
cannot do is refused cleanly."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, golden_cases
import oracle_util as ou
from smudgeplot_b200 import _lib, fastk, hetmers
from tools import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _need_gpu(built):
    assert _lib.lib().hm_device_count() >= 1, "these tests need a CUDA device (no CPU fallback exists)"


@pytest.fixture(autouse=True)
def _reset_budget(monkeypatch):
    monkeypatch.delenv("HETMERS_STREAM", raising=False)
    monkeypatch.delenv("HETMERS_STREAM_CHUNK", raising=False)
    yield
    _lib.lib().hm_set_device_budget(0)


def _golden(name):
    return os.path.join(GOLDEN, name, name)


def budget_for_chunk(n, k, ibyte, chunk):
    """the smallest device budget whose streamed plan has chunks of at least `chunk` entries"""
    lo, hi = 1 << 20, 1 << 40
    lay = _lib.StreamLayout()
    while lo < hi:
        mid = (lo + hi) // 2
        if _lib.lib().hm_stream_plan(n, k, ibyte, mid, C.byref(lay)) == 0 and lay.chunk >= chunk:
            hi = mid
        else:
            lo = mid + 1
    return lo


def stream_setup(n, k, ibyte, chunks):
    """(budget, chunk): chunks of about n / chunks entries under a budget that also has room for the resident
    lists of the whole table at their bound (a candidate record per two entries, an S key per entry)"""
    chunk = max(256, -(-n // chunks))
    kw = 2 if k > 32 else 1
    lists = (8 * kw + 8) * (n // 2 + 4096) + 8 * kw * (n + 4096)
    return budget_for_chunk(n, k, ibyte, chunk) + 2 * lists, chunk


def streamed_scan(kt, chunks, monkeypatch, path="auto"):
    """plot of the streamed scan of kt with about `chunks` chunks; -> (plot, stats, residency, budget)"""
    budget, chunk = stream_setup(kt.nels, kt.kmer, kt.ibyte, chunks)
    monkeypatch.setenv("HETMERS_STREAM", "1")
    monkeypatch.setenv("HETMERS_STREAM_CHUNK", str(chunk))
    with hetmers.Scan(kt, device_budget=budget) as sc:
        plot, st = sc.run(path)
        res = sc.residency()
    monkeypatch.delenv("HETMERS_STREAM")
    monkeypatch.delenv("HETMERS_STREAM_CHUNK")
    _lib.lib().hm_set_device_budget(0)
    assert res[0] and res[1] <= budget
    return plot, st, res, budget


def incore_symm(kt):
    with hetmers.Scan(kt) as sc:
        assert sc.residency()[0] is False
        assert sc.is_symmetric()
        plot, st = sc.run("symm")
    assert st["path"] == 2
    return plot


# ------------------------------------------------------------------ goldens through the executable --

@pytest.mark.parametrize("name", golden_cases())
def test_executable_streams_goldens_to_the_reference_smu(name, golden_meta, tmp_path):
    c = golden_meta[name]
    kt = fastk.read_ktab(_golden(name))
    budget, chunk = stream_setup(kt.nels, kt.kmer, kt.ibyte, 5)
    out = str(tmp_path / "out")
    env = dict(os.environ, HETMERS_STREAM="1", HETMERS_STREAM_CHUNK=str(chunk), HETMERS_DEVICE_BUDGET=str(budget),
               HETMERS_STATS="1")
    r = subprocess.run([_lib.BIN_PATH, "-v", f"-e{c['e']}", "-T4", f"-o{out}", _golden(name)],
                       input="n\n", capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr
    assert r.stderr.startswith("\n  The input table is trimmed and symmetric\n"
                               "\n  Starting to count covariant pairs\n")
    st = json.loads([ln for ln in r.stderr.splitlines() if ln.startswith("{")][0])
    assert st["streamed"] is True and st["chunks"] >= 4 and 0 < st["device_bytes"] <= budget
    assert st["path"] == "symmetric"
    assert open(out + ".smu").read() == open(_golden(name) + ".smu").read()


# ------------------------------------------------------------------ stored reference runs ----------

from test_gpu_parity import MEDIUM_CASES  # noqa: E402


@pytest.mark.parametrize("chunks", [8, 64])
@pytest.mark.parametrize("k,target,ploidy,het,cov,L,seed,ref_threads", MEDIUM_CASES)
def test_streamed_medium_tables_match_the_reference_runs(k, target, ploidy, het, cov, L, seed, ref_threads, chunks,
                                                         tmp_path, monkeypatch):
    G = synth.calibrate_G(k, target, ploidy, het, cov, L)
    keys, cnt = synth.synth_table(k, G, ploidy, het, cov, L, seed, device="cuda")
    name = str(tmp_path / "t")
    kt = synth.write_table(name, k, keys, cnt, ibyte=3, nparts=4)
    del keys, cnt
    plot, st, res, _ = streamed_scan(fastk.read_ktab(name, mmap=True), chunks, monkeypatch)
    assert st["path"] == 2 and res[2] >= chunks - 1
    assert hetmers.smu_text(plot) == ou.reference_smu("medium", k, seed)


# ------------------------------------------------------------------ chunk boundaries --------------

def _check_tables(kt, keys, cnt, monkeypatch, chunk_counts=(3, 7, 31)):
    want, _ = ou.oracle_scan(fastk.keys_u64_to_bytes(keys, kt.kmer), cnt, kt.kmer)
    assert np.array_equal(incore_symm(kt), want)
    for chunks in chunk_counts:
        if -(-kt.nels // chunks) < 256:
            continue
        plot, st, res, _ = streamed_scan(kt, chunks, monkeypatch)
        assert np.array_equal(plot, want), chunks


@pytest.mark.parametrize("variant", ["sparse", "dense"])
@pytest.mark.parametrize("k,seed", [(11, 1), (12, 2), (11, 3)])
def test_streamed_dense_small_k_tables(k, seed, variant, tmp_path, monkeypatch):
    """runs of hundreds of entries everywhere: every cut lies next to a long run"""
    from test_gpu_symm import _symmetric_closure
    monkeypatch.setenv("HETMERS_RUNSCAN", variant)
    rng = np.random.default_rng(9100 + seed)
    vals = rng.choice(4 ** k, size=int(4 ** k * 0.05), replace=False).astype(np.uint64) << np.uint64(64 - 2 * k)
    keys, cnt = _symmetric_closure(vals, k, rng, 700)
    kt = fastk.write_ktab(str(tmp_path / "t"), k, keys, cnt, ibyte=1, nparts=2)
    _check_tables(kt, keys, cnt, monkeypatch)


@pytest.mark.parametrize("k,seed", [(31, 1), (21, 3), (32, 4)])
def test_streamed_long_runs_in_a_sparse_table(k, seed, tmp_path, monkeypatch):
    """the long-run tables of test_long_runs_in_a_sparse_table: a 3000-entry run is longer than the small
    chunks, which must grow to hold it"""
    import test_gpu_symm as tg
    rng = np.random.default_rng(8000 + seed)
    Pr = k // 2
    tail_bits = 2 * (k - Pr)
    parts = []
    for run_len in (3000, 700, 130, 66, 65, 64, 63, 40, 9):
        pre = int(rng.integers(0, 4 ** Pr))
        tails = rng.choice(min(4 ** (k - Pr), 1 << 40), size=run_len, replace=False).astype(np.uint64)
        for i in range(0, run_len - 1, 2):
            pos = int(rng.integers(0, k - Pr))
            tails[i + 1] = tails[i] ^ (np.uint64(int(rng.integers(1, 4))) << np.uint64(2 * pos))
        v = (np.uint64(pre) << np.uint64(tail_bits)) | tails
        parts.append(np.unique(v) << np.uint64(64 - 2 * k))
    bg = rng.integers(0, 1 << 62, size=20000, dtype=np.int64).astype(np.uint64)
    bg = (bg >> np.uint64(64 - 2 * k)) << np.uint64(64 - 2 * k) if k < 32 else bg
    parts.append(bg)
    keys, cnt = tg._symmetric_closure(np.concatenate(parts), k, rng, 40)
    kt = fastk.write_ktab(str(tmp_path / "t"), k, keys, cnt, ibyte=3, nparts=2)
    _check_tables(kt, keys, cnt, monkeypatch, chunk_counts=(4, 40))


def test_streamed_tables_made_of_pairs(tmp_path, monkeypatch):
    import test_gpu_symm as tg
    rng = np.random.default_rng(4242)
    k = 31
    base = rng.integers(0, 1 << 62, size=30000, dtype=np.int64).astype(np.uint64)
    base = (base >> np.uint64(2)) << np.uint64(2)
    pos = rng.integers(k // 2, k, size=base.size)
    sh = (np.uint64(62) - np.uint64(2) * pos.astype(np.uint64))
    mate = base ^ (rng.integers(1, 4, size=base.size).astype(np.uint64) << sh)
    keys, cnt = tg._symmetric_closure(np.concatenate([base, mate]), k, rng, 60)
    kt = fastk.write_ktab(str(tmp_path / "t"), k, keys, cnt, ibyte=3, nparts=2)
    _check_tables(kt, keys, cnt, monkeypatch)


@pytest.mark.parametrize("k", [32, 33, 64, 40])
def test_streamed_seeded_tables_long_k(k, tmp_path, monkeypatch):
    keys, cnt = synth.synth_table(k, 40000, 2, 0.02, 40, 4, 500 + k, extra_hom_repeats=1)
    name = str(tmp_path / "t")
    synth.write_table(name, k, keys, cnt, ibyte=2, nparts=3)
    kt = fastk.read_ktab(name)
    kb, cn = fastk.unpack_host(kt)
    want, _ = ou.oracle_scan(kb, cn, k)
    assert np.array_equal(incore_symm(kt), want)
    for chunks in (5, 33):
        plot, st, res, _ = streamed_scan(kt, chunks, monkeypatch)
        assert np.array_equal(plot, want), chunks


@pytest.mark.parametrize("k", [8, 10, 16])
def test_streamed_even_k_with_palindromes(k, tmp_path, monkeypatch):
    """even k: palindromes are their own reverse complement (one entry, one count)"""
    from test_gpu_symm import _symmetric_closure
    rng = np.random.default_rng(77 + k)
    n0 = min(4 ** k // 20, 60000)
    vals = rng.choice(4 ** k, size=n0, replace=False).astype(np.uint64) << np.uint64(64 - 2 * k)
    keys, cnt = _symmetric_closure(vals, k, rng, 300)
    rc = synth.revcomp_left(__import__("torch").from_numpy(keys.view(np.int64).copy()), k).numpy().view(np.uint64)
    assert (rc == keys).sum() > 0 or k > 12
    kt = fastk.write_ktab(str(tmp_path / "t"), k, keys, cnt, ibyte=1, nparts=2)
    _check_tables(kt, keys, cnt, monkeypatch, chunk_counts=(4, 16))


# ------------------------------------------------------------------ examine, conditioning ---------

@pytest.mark.parametrize("name,verdict", [("untrimmed", (False, True)), ("asymmetric", (True, False))])
def test_streamed_examine_and_conditioning_route(name, verdict, golden_meta, tmp_path, monkeypatch):
    c = golden_meta["_conditioning"][name]
    table = os.path.join(GOLDEN, "conditioning", name)
    kt = fastk.read_ktab(table)
    budget, _ = stream_setup(kt.nels, kt.kmer, kt.ibyte, 4)
    monkeypatch.setenv("HETMERS_STREAM", "1")
    with hetmers.Scan(kt, device_budget=budget) as sc:
        assert sc.residency()[0]
        assert sc.examine(c["e"]) == verdict
        with pytest.raises(_lib.HetmersError) as ei:
            sc.condition(c["e"], not verdict[0], not verdict[1])
        assert ei.value.code == -6
    # the executable takes the reference's route: its -v verdict, then the shell-outs to FastK's tools
    env = dict(os.environ, HETMERS_STREAM="1", HETMERS_DEVICE_BUDGET=str(budget))
    env.pop("HETMERS_EXTERNAL_CONDITIONING", None)
    r = subprocess.run([_lib.BIN_PATH, "-v", f"-e{c['e']}", "-T4", f"-o{tmp_path}/o", table],
                       input="n\n", capture_output=True, text=True, cwd=tmp_path, env=env)
    assert r.returncode == 1
    assert c["verbose"][0] in r.stderr
    assert "Command '" in r.stderr and "failed" in r.stderr
    assert not os.path.exists(f"{tmp_path}/o.smu")


def test_condition_refuses_a_budget_it_cannot_fit_before_touching_the_table(golden_meta):
    c = golden_meta["_conditioning"]["untrimmed"]
    kt = fastk.read_ktab(os.path.join(GOLDEN, "conditioning", "untrimmed"))
    with hetmers.Scan(kt) as ref:
        incore = ref.residency()[1]
    with hetmers.Scan(kt, device_budget=incore + 4096) as sc:          # room for the scan, not for conditioning
        assert not sc.residency()[0]
        with pytest.raises(_lib.HetmersError) as ei:
            sc.condition(c["e"], True, True)
        assert ei.value.code == -3
        assert sc.examine(c["e"]) == (False, True)                    # the table is untouched
        sc.run()


# ------------------------------------------------------------------ refusals ----------------------

def test_streamed_asymmetric_table_is_refused(tmp_path, monkeypatch):
    keys, cnt = synth.synth_table(31, 30000, 2, 0.02, 40, 4, 321)
    ku = synth.keys_to_u64_numpy(keys)
    cu = cnt.numpy().astype(np.uint16)
    keep = np.ones(len(ku), dtype=bool)
    keep[len(ku) // 3] = False
    kt = fastk.write_ktab(str(tmp_path / "asym"), 31, ku[keep], cu[keep], ibyte=3, nparts=2)
    budget, _ = stream_setup(kt.nels, 31, 3, 4)
    monkeypatch.setenv("HETMERS_STREAM", "1")
    with hetmers.Scan(kt, device_budget=budget) as sc:
        with pytest.raises(_lib.HetmersError) as ei:
            sc.run()
        assert ei.value.code == -6 and "not strand-symmetric" in str(ei.value)
    env = dict(os.environ, HETMERS_STREAM="1", HETMERS_DEVICE_BUDGET=str(budget))
    out = str(tmp_path / "o")
    # (examine's one-k-mer probe passes this table: it is scanned, and the scan refuses it)
    r = subprocess.run([_lib.BIN_PATH, "-e4", f"-o{out}", str(tmp_path / "asym")],
                       input="n\n", capture_output=True, text=True, env=env)
    assert r.returncode == 1
    assert "not strand-symmetric" in r.stderr or "Command '" in r.stderr
    assert not os.path.exists(out + ".smu")


def test_streamed_scan_refuses_what_needs_the_table_resident(monkeypatch):
    kt = fastk.read_ktab(_golden("dip_k21"))
    monkeypatch.setenv("HETMERS_STREAM", "1")
    budget, _ = stream_setup(kt.nels, kt.kmer, kt.ibyte, 4)
    with hetmers.Scan(kt, device_budget=budget) as sc:
        for call in (lambda: sc.run("direct"), lambda: sc.download(deg=False),
                     lambda: sc.extract(np.zeros(_lib.PLOT_CELLS, dtype=np.uint16))):
            with pytest.raises(_lib.HetmersError) as ei:
                call()
            assert ei.value.code == -6
        plot, st = sc.run()                                  # and the scan still works afterwards
    assert hetmers.smu_text(plot) == open(_golden("dip_k21") + ".smu").read()


def test_extract_executable_refuses_a_streamed_table(golden_meta, tmp_path):
    kt = fastk.read_ktab(_golden("dip_k21"))
    budget, _ = stream_setup(kt.nels, kt.kmer, kt.ibyte, 4)
    env = dict(os.environ, HETMERS_STREAM="1", HETMERS_DEVICE_BUDGET=str(budget))
    r = subprocess.run([os.path.join(os.path.dirname(_lib.BIN_PATH), "extract_kmer_pairs"), "-e4",
                        f"-o{tmp_path}/p", _golden("dip_k21"), _golden("dip_k21") + ".sma"],
                       capture_output=True, text=True, env=env)
    assert r.returncode == 1
    assert "direct passes' arrays" in r.stderr


def test_tables_that_fit_stay_in_core_by_default():
    kt = fastk.read_ktab(_golden("trip_k31"))
    with hetmers.Scan(kt) as sc:
        streamed, dev_bytes, chunks = sc.residency()
        plot, st = sc.run()
    assert streamed is False and chunks == 0 and dev_bytes > 0
    assert hetmers.smu_text(plot) == open(_golden("trip_k31") + ".smu").read()


def test_budget_below_the_in_core_footprint_streams_without_the_switch(monkeypatch):
    """a budget alone (no HETMERS_STREAM) decides: a 2e6-entry table under half of its in-core bytes"""
    keys, cnt = synth.synth_table(31, 1_000_000, 2, 0.01, 40, 8, 31, device="cuda")
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        kt = synth.write_table(os.path.join(d, "t"), 31, keys, cnt, ibyte=2, nparts=2)
        want = incore_symm(kt)
        with hetmers.Scan(kt) as sc:
            incore = sc.residency()[1]
        with hetmers.Scan(kt, device_budget=incore // 2) as sc:
            streamed, dev_bytes, chunks = sc.residency()
            assert streamed
            plot, st = sc.run()
            streamed, dev_bytes, chunks = sc.residency()
        assert chunks >= 2 and dev_bytes <= incore // 2
        assert np.array_equal(plot, want)
