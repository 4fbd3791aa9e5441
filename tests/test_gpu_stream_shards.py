"""GPU tests of the sharded streamed scan (DESIGN.md §4c; run with -m gpu): G shards each stream a run-aligned
share of the table, the Bloom segments cross between the passes and pass 2 checks a Bloom hit in the S list
of the key's owner.  Shards may share a device (devices=[0] * G), so every case here runs on one H100; the
plot must equal the goldens, the stored reference runs, the oracle and the in-core scan."""
import ctypes as C
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


def shard_budget(n, k, ibyte, G, chunk):
    """a per-shard budget whose plan has chunks of at least `chunk` entries (at most a share), with room for the
    resident lists of the whole table at their bound (a candidate record per two entries, an S key per entry)"""
    share = max(1, -(-n // G))
    chunk = min(chunk, share)
    lo, hi = 1 << 20, 1 << 40
    lay = _lib.StreamLayout()
    while lo < hi:
        mid = (lo + hi) // 2
        if _lib.lib().hm_stream_plan_shards(n, k, ibyte, mid, G, C.byref(lay)) == 0 and lay.chunk >= chunk:
            hi = mid
        else:
            lo = mid + 1
    kw = 2 if k > 32 else 1
    return lo + 2 * ((8 * kw + 8) * (n // 2 + 4096) + 8 * kw * (n + 4096))


def sharded_scan(kt, G, chunks_per_shard, monkeypatch, devices=None, path="auto"):
    """plot of the streamed scan of kt over G shards (all on device 0 unless `devices`), about
    `chunks_per_shard` chunks each; -> (plot, stats, residency, budget)"""
    chunk = max(256, -(-kt.nels // (G * chunks_per_shard)))
    budget = shard_budget(kt.nels, kt.kmer, kt.ibyte, G, chunk)
    monkeypatch.setenv("HETMERS_STREAM", "1")
    monkeypatch.setenv("HETMERS_STREAM_CHUNK", str(chunk))
    try:
        with hetmers.Scan(kt, devices=devices or [0] * G, device_budget=budget) as sc:
            plot, st = sc.run(path)
            res = sc.residency()
    finally:
        monkeypatch.delenv("HETMERS_STREAM")
        monkeypatch.delenv("HETMERS_STREAM_CHUNK")
        _lib.lib().hm_set_device_budget(0)
    assert res[0] and res[1] <= budget
    assert st["n_gpus"] == G and st["path"] == 2
    return plot, st, res, budget


def incore_symm(kt):
    with hetmers.Scan(kt) as sc:
        assert sc.residency()[0] is False
        plot, st = sc.run("symm")
    assert st["path"] == 2
    return plot


def host_cuts(keys_hi, k, G):
    """the shard cuts of the rule the library applies: c_r = first run start at or after n*r/G"""
    n = len(keys_hi)
    pfx = keys_hi >> np.uint64(64 - 2 * (k // 2))
    starts = np.concatenate([[0], np.nonzero(pfx[1:] != pfx[:-1])[0] + 1, [n]])
    return [0] + [int(starts[np.searchsorted(starts, n * r // G)]) for r in range(1, G)] + [n]


# ------------------------------------------------------------------ goldens ---------------------------

@pytest.mark.parametrize("G", [2, 3, 4])
@pytest.mark.parametrize("name", golden_cases())
def test_sharded_goldens_equal_the_reference_smu(name, G, monkeypatch):
    kt = fastk.read_ktab(_golden(name))
    plot, st, res, _ = sharded_scan(kt, G, 3, monkeypatch)
    assert res[2] >= 2
    assert hetmers.smu_text(plot) == open(_golden(name) + ".smu").read()


@pytest.mark.parametrize("name", golden_cases())
def test_executable_streams_goldens_over_two_gpus(name, golden_meta, tmp_path):
    if _lib.lib().hm_device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import json
    c = golden_meta[name]
    kt = fastk.read_ktab(_golden(name))
    budget = shard_budget(kt.nels, kt.kmer, kt.ibyte, 2, max(256, kt.nels // 8))
    out = str(tmp_path / "out")
    env = dict(os.environ, HETMERS_STREAM="1", HETMERS_DEVICE_BUDGET=str(budget), HETMERS_GPUS="2", HETMERS_STATS="1")
    r = subprocess.run([_lib.BIN_PATH, "-v", f"-e{c['e']}", "-T4", f"-o{out}", _golden(name)],
                       input="n\n", capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr
    st = json.loads([ln for ln in r.stderr.splitlines() if ln.startswith("{")][0])
    assert st["streamed"] is True and st["n_gpus"] == 2 and st["path"] == "symmetric"
    assert open(out + ".smu").read() == open(_golden(name) + ".smu").read()


# ------------------------------------------------------------------ stored reference runs -------------

from test_gpu_parity import MEDIUM_CASES  # noqa: E402


@pytest.mark.parametrize("k,target,ploidy,het,cov,L,seed,ref_threads", MEDIUM_CASES)
def test_sharded_medium_tables_match_the_reference_runs(k, target, ploidy, het, cov, L, seed, ref_threads, tmp_path,
                                                        monkeypatch):
    Gn = synth.calibrate_G(k, target, ploidy, het, cov, L)
    keys, cnt = synth.synth_table(k, Gn, ploidy, het, cov, L, seed, device="cuda")
    name = str(tmp_path / "t")
    synth.write_table(name, k, keys, cnt, ibyte=3, nparts=4)
    del keys, cnt
    plot, st, res, _ = sharded_scan(fastk.read_ktab(name, mmap=True), 4, 8, monkeypatch)
    assert res[2] >= 4 * 7
    assert hetmers.smu_text(plot) == ou.reference_smu("medium", k, seed)


# ------------------------------------------------------------------ cut stress ------------------------

def _check_shards(kt, keys, cnt, monkeypatch, Gs=(2, 3, 5)):
    want, _ = ou.oracle_scan(fastk.keys_u64_to_bytes(keys, kt.kmer), cnt, kt.kmer)
    assert np.array_equal(incore_symm(kt), want)
    for G in Gs:
        plot, st, res, _ = sharded_scan(kt, G, 4, monkeypatch)
        assert np.array_equal(plot, want), G
    return want


@pytest.mark.parametrize("k,seed", [(11, 1), (12, 2)])
def test_sharded_dense_small_k_tables(k, seed, tmp_path, monkeypatch):
    """runs of hundreds of entries: cuts move far, and with five shards of a tiny table some are empty"""
    from test_gpu_symm import _symmetric_closure
    rng = np.random.default_rng(9300 + seed)
    vals = rng.choice(4 ** k, size=int(4 ** k * 0.05), replace=False).astype(np.uint64) << np.uint64(64 - 2 * k)
    keys, cnt = _symmetric_closure(vals, k, rng, 700)
    kt = fastk.write_ktab(str(tmp_path / "t"), k, keys, cnt, ibyte=1, nparts=2)
    _check_shards(kt, keys, cnt, monkeypatch)


def test_sharded_runs_longer_than_a_share(tmp_path, monkeypatch):
    """k = 3, every k-mer: 4 runs of 16 entries, so with 5 or 16 shards some shards are empty, the last of
    the 5 among them"""
    from test_gpu_symm import _symmetric_closure
    k = 3
    rng = np.random.default_rng(5150)
    vals = np.arange(4 ** k, dtype=np.uint64) << np.uint64(64 - 2 * k)
    keys, cnt = _symmetric_closure(vals, k, rng, 300)
    cuts5, cuts16 = host_cuts(keys, k, 5), host_cuts(keys, k, 16)
    assert cuts5[4] == cuts5[5] == len(keys)
    assert sum(cuts16[r] == cuts16[r + 1] for r in range(16)) >= 8
    kt = fastk.write_ktab(str(tmp_path / "t"), k, keys, cnt, ibyte=1, nparts=1)
    _check_shards(kt, keys, cnt, monkeypatch, Gs=(2, 5, 16))


@pytest.mark.parametrize("k", [8, 10, 16])
def test_sharded_even_k_with_palindromes(k, tmp_path, monkeypatch):
    from test_gpu_symm import _symmetric_closure
    rng = np.random.default_rng(177 + k)
    n0 = min(4 ** k // 20, 60000)
    vals = rng.choice(4 ** k, size=n0, replace=False).astype(np.uint64) << np.uint64(64 - 2 * k)
    keys, cnt = _symmetric_closure(vals, k, rng, 300)
    kt = fastk.write_ktab(str(tmp_path / "t"), k, keys, cnt, ibyte=1, nparts=2)
    _check_shards(kt, keys, cnt, monkeypatch)


@pytest.mark.parametrize("k", [32, 33, 40, 64])
def test_sharded_seeded_tables_long_k(k, tmp_path, monkeypatch):
    """two-word keys (k > 32): shards are owned by the first word"""
    keys, cnt = synth.synth_table(k, 40000, 2, 0.02, 40, 4, 700 + k, extra_hom_repeats=1)
    name = str(tmp_path / "t")
    synth.write_table(name, k, keys, cnt, ibyte=2, nparts=3)
    kt = fastk.read_ktab(name)
    kb, cn = fastk.unpack_host(kt)
    want, _ = ou.oracle_scan(kb, cn, k)
    assert np.array_equal(incore_symm(kt), want)
    for G in (2, 3, 5):
        plot, st, res, _ = sharded_scan(kt, G, 4, monkeypatch)
        assert np.array_equal(plot, want), G


def test_sharded_tables_made_of_pairs(tmp_path, monkeypatch):
    import test_gpu_symm as tg
    rng = np.random.default_rng(4343)
    k = 31
    base = rng.integers(0, 1 << 62, size=30000, dtype=np.int64).astype(np.uint64)
    base = (base >> np.uint64(2)) << np.uint64(2)
    pos = rng.integers(k // 2, k, size=base.size)
    sh = (np.uint64(62) - np.uint64(2) * pos.astype(np.uint64))
    mate = base ^ (rng.integers(1, 4, size=base.size).astype(np.uint64) << sh)
    keys, cnt = tg._symmetric_closure(np.concatenate([base, mate]), k, rng, 60)
    kt = fastk.write_ktab(str(tmp_path / "t"), k, keys, cnt, ibyte=3, nparts=2)
    _check_shards(kt, keys, cnt, monkeypatch)


# ------------------------------------------------------------------ foreign exact checks -------------

FOREIGN_MIN = 1000          # candidate pairs whose rc x has an upper partner in another shard, at least


def test_exact_checks_reach_the_owner_shards_s_list(tmp_path, monkeypatch):
    """Pairs (x, y) one base apart at a high position, with rc x given a partner at an upper position: rc x is
    in S, so (x, y) is not isolated -- but only the S list of rc x's owner says so.  A pass 2 that only looked
    in its own S list would count these pairs, and the plot would differ from the oracle's."""
    import test_gpu_symm as tg
    k, m, G = 31, 4000, 4
    Pr, pup = k // 2, k - k // 2
    rng = np.random.default_rng(6060)
    x = (rng.integers(0, 1 << 62, size=m, dtype=np.int64).astype(np.uint64) >> np.uint64(2)) << np.uint64(2)
    p = rng.integers(Pr, k, size=m).astype(np.uint64)
    y = x ^ (rng.integers(1, 4, size=m).astype(np.uint64) << (np.uint64(62) - np.uint64(2) * p))
    z = tg._rc_u64(x, k)
    q = rng.integers(pup, k, size=m).astype(np.uint64)
    z2 = z ^ (rng.integers(1, 4, size=m).astype(np.uint64) << (np.uint64(62) - np.uint64(2) * q))
    keys, cnt = tg._symmetric_closure(np.concatenate([x, y, z2]), k, rng, 60)
    cuts = host_cuts(keys, k, G)
    owner = lambda v: np.searchsorted(cuts, np.searchsorted(keys, v), side="right") - 1   # noqa: E731
    foreign = int(np.sum(owner(z) != owner(x)))
    assert foreign >= FOREIGN_MIN, foreign
    kt = fastk.write_ktab(str(tmp_path / "t"), k, keys, cnt, ibyte=3, nparts=2)
    want, _ = ou.oracle_scan(fastk.keys_u64_to_bytes(keys, k), cnt, k)
    assert np.array_equal(incore_symm(kt), want)
    plot, st, res, _ = sharded_scan(kt, G, 2, monkeypatch)
    assert np.array_equal(plot, want)


# ------------------------------------------------------------------ capacity --------------------------

def test_shards_scan_a_table_one_budget_cannot_hold(monkeypatch):
    """the budget that runs out of list room on one GPU is enough for each of four shards"""
    import tempfile
    keys, cnt = synth.synth_table(31, 1_000_000, 2, 0.01, 40, 8, 131, device="cuda")
    with tempfile.TemporaryDirectory() as d:
        kt = synth.write_table(os.path.join(d, "t"), 31, keys, cnt, ibyte=2, nparts=2)
        kb, cn = fastk.unpack_host(kt)
        want, _ = ou.oracle_scan(kb, cn, 31)
        chunk = -(-kt.nels // 32)
        monkeypatch.setenv("HETMERS_STREAM", "1")
        monkeypatch.setenv("HETMERS_STREAM_CHUNK", str(chunk))
        with hetmers.Scan(kt, devices=[0] * 4, device_budget=1 << 34) as sc:     # room to spare: the peaks
            sc.run()
            peak4 = sc.residency()[1]
        budget = int(peak4 * 1.05)
        with hetmers.Scan(kt, devices=[0], device_budget=budget) as sc:
            with pytest.raises(_lib.HetmersError) as ei:
                sc.run()
        assert ei.value.code == -3 and "list needs" in str(ei.value)
        with hetmers.Scan(kt, devices=[0] * 4, device_budget=budget) as sc:
            plot, st = sc.run()
            streamed, dev_bytes, chunks = sc.residency()
        assert streamed and dev_bytes <= budget and chunks >= 28
        assert np.array_equal(plot, want)


# ------------------------------------------------------------------ refusals ---------------------------

def test_sharded_scan_refuses_what_needs_the_table_resident(monkeypatch):
    kt = fastk.read_ktab(_golden("dip_k21"))
    monkeypatch.setenv("HETMERS_STREAM", "1")
    budget = shard_budget(kt.nels, kt.kmer, kt.ibyte, 2, 1024)
    with hetmers.Scan(kt, devices=[0, 0], device_budget=budget) as sc:
        assert sc.residency()[0]
        for call in (lambda: sc.run("direct"), lambda: sc.download(deg=False),
                     lambda: sc.extract(np.zeros(_lib.PLOT_CELLS, dtype=np.uint16)),
                     lambda: sc.condition(4, True, False)):
            with pytest.raises(_lib.HetmersError) as ei:
                call()
            assert ei.value.code == -6
        plot, st = sc.run()                                  # and the scan still works afterwards
    assert st["n_gpus"] == 2
    assert hetmers.smu_text(plot) == open(_golden("dip_k21") + ".smu").read()


def test_sharded_asymmetric_table_is_refused_after_the_pass(tmp_path, monkeypatch):
    keys, cnt = synth.synth_table(31, 30000, 2, 0.02, 40, 4, 421)
    ku = synth.keys_to_u64_numpy(keys)
    cu = cnt.numpy().astype(np.uint16)
    keep = np.ones(len(ku), dtype=bool)
    keep[len(ku) // 3] = False
    kt = fastk.write_ktab(str(tmp_path / "asym"), 31, ku[keep], cu[keep], ibyte=3, nparts=2)
    budget = shard_budget(kt.nels, 31, 3, 3, 1024)
    monkeypatch.setenv("HETMERS_STREAM", "1")
    with hetmers.Scan(kt, devices=[0, 0, 0], device_budget=budget) as sc:
        for _ in range(2):
            with pytest.raises(_lib.HetmersError) as ei:
                sc.run()
            assert ei.value.code == -6 and "not strand-symmetric" in str(ei.value)


def test_in_core_scan_refuses_repeated_devices():
    kt = fastk.read_ktab(_golden("trip_k31"))
    with pytest.raises(_lib.HetmersError) as ei:
        hetmers.Scan(kt, devices=[0, 0])
    assert ei.value.code == -1 and "listed twice" in str(ei.value)


# ------------------------------------------------------------------ several GPUs ----------------------

def test_two_gpus_equal_two_shards_on_one(monkeypatch):
    if _lib.lib().hm_device_count() < 2:
        pytest.skip("needs 2 GPUs")
    keys, cnt = synth.synth_table(31, 200_000, 2, 0.01, 40, 4, 77)
    ku = synth.keys_to_u64_numpy(keys)
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        kt = fastk.write_ktab(os.path.join(d, "t"), 31, ku, cnt.numpy().astype(np.uint16), ibyte=2, nparts=2)
        want = incore_symm(kt)
        same, _, _, _ = sharded_scan(kt, 2, 4, monkeypatch)
        two, _, _, _ = sharded_scan(kt, 2, 4, monkeypatch, devices=[0, 1])
    assert np.array_equal(same, want) and np.array_equal(two, want)
