"""GPU parity tests of the strand-symmetric scan (csrc/hm_symm.cu; run with -m gpu on an H100).
The symmetric scan must give the reference's plot on every symmetric table (goldens written by the
unmodified reference binary, the oracle on seeded / dense / long-run tables), the fingerprint must send
every table that is not symmetric to the direct passes, and the sharded form (several GPUs) must not
depend on the cuts."""
import os

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


@pytest.fixture(autouse=True, params=["sparse", "dense"])
def runscan_kernel_variant(request, monkeypatch):
    """pass 1 has two kernels, picked by the mean number of run mates n / 4^(k/2) (the classifying one for
    sparse tables, all-pairs-in-the-run for crowded ones): every test runs with each of them forced"""
    monkeypatch.setenv("HETMERS_RUNSCAN", request.param)
    return request.param


def _golden(name):
    return os.path.join(GOLDEN, name, name)


def _rc_u64(x, k):
    """reverse complement of left-aligned packed k-mers (numpy uint64, k <= 32)"""
    import torch
    t = torch.from_numpy(x.view(np.int64).copy())
    return synth.revcomp_left(t, k).numpy().view(np.uint64)


def _symmetric_closure(vals, k, rng, cmax):
    """sorted unique keys = vals + their reverse complements; counts equal on both strands"""
    keys = np.unique(np.concatenate([vals, _rc_u64(vals, k)]))
    rc = _rc_u64(keys, k)
    canon = np.minimum(keys, rc)
    _, inv = np.unique(canon, return_inverse=True)
    cc = rng.integers(1, cmax + 1, size=inv.max() + 1).astype(np.uint16)
    return keys, cc[inv]


# ------------------------------------------------------------------ goldens -------------------

@pytest.mark.parametrize("name", golden_cases())
def test_symmetric_scan_reproduces_reference_smu(name, golden_meta):
    c = golden_meta[name]
    kt = fastk.read_ktab(_golden(name))
    with hetmers.Scan(kt) as sc:
        assert sc.is_symmetric()                        # every golden table is strand-symmetric
        plot_s, st_s = sc.run("symm")
        plot_a, st_a = sc.run()                         # auto = the symmetric scan
        plot_d, st_d = sc.run("direct")
    assert st_s["path"] == 2 and st_a["path"] == 2 and st_d["path"] == 1
    want = open(_golden(name) + ".smu").read()
    assert hetmers.smu_text(plot_s) == want
    assert np.array_equal(plot_s, plot_d) and np.array_equal(plot_a, plot_d)    # incl. the m=500 column
    assert st_s["nels"] == c["nels"]


# ------------------------------------------------------------------ seeded tables vs oracle ---

from test_gpu_parity import CASES  # noqa: E402


@pytest.mark.parametrize("k,G,ploidy,het,cov,L,seed,ibyte,nparts", CASES)
def test_symmetric_scan_matches_oracle_on_seeded_tables(k, G, ploidy, het, cov, L, seed, ibyte, nparts, tmp_path):
    keys, cnt = synth.synth_table(k, G, ploidy, het, cov, L, seed, extra_hom_repeats=1)
    name = str(tmp_path / "t")
    kt = synth.write_table(name, k, keys, cnt, ibyte=ibyte, nparts=nparts)
    kb, cn = fastk.unpack_host(kt)
    want_plot, _ = ou.oracle_scan(kb, cn, k)
    with hetmers.Scan(fastk.read_ktab(name)) as sc:
        assert sc.is_symmetric()
        plot, st = sc.run("symm")
    assert st["path"] == 2
    assert np.array_equal(plot, want_plot)
    plot2, st2 = hetmers.scan_table(kt)                                 # one-call route takes it too
    assert st2["path"] == 2 and np.array_equal(plot2, want_plot)


# ------------------------------------------------------------------ dense / long runs ---------

@pytest.mark.parametrize("seed", range(10))
def test_dense_symmetric_tables_small_k(seed, tmp_path):
    """tiny k: runs of up to 4^(k - k/2) entries, i.e. far longer than the 64-entry linear scan and the
    2048-entry tile -> the per-candidate look-up path of runscan / resolve; counts around the SMAX gate"""
    rng = np.random.default_rng(7000 + seed)
    k = int(rng.integers(2, 12))
    n0 = max(2, int(4 ** k * float(rng.choice([0.003, 0.01, 0.04, 0.15, 0.4]))))
    cmax = int(rng.choice([6, 40, 520, 700]))
    vals = rng.choice(4 ** k, size=n0, replace=False).astype(np.uint64) << np.uint64(64 - 2 * k)
    keys, cnt = _symmetric_closure(vals, k, rng, cmax)
    if len(keys) < 2:
        pytest.skip("degenerate")
    ibyte = 1 if k < 8 else int(rng.integers(1, 3))
    kt = fastk.write_ktab(str(tmp_path / "t"), k, keys, cnt, ibyte=ibyte, nparts=int(rng.integers(1, 4)))
    want_plot, _ = ou.oracle_scan(fastk.keys_u64_to_bytes(keys, k), cnt, k)
    with hetmers.Scan(kt) as sc:
        assert sc.is_symmetric()
        plot, st = sc.run("symm")
        plot_d, _ = sc.run("direct")
    assert st["path"] == 2
    assert np.array_equal(plot_d, want_plot)
    assert np.array_equal(plot, want_plot)


@pytest.mark.parametrize("k,seed", [(31, 1), (31, 2), (21, 3), (32, 4)])
def test_long_runs_in_a_sparse_table(k, seed, tmp_path):
    """genome-like k with engineered long runs: many entries sharing their first k/2 bases (tandem
    repeats / low-complexity sequence), some longer than the scan cap, one longer than a tile"""
    rng = np.random.default_rng(8000 + seed)
    Pr = k // 2
    tail_bits = 2 * (k - Pr)
    parts = []
    for run_len in (3000, 700, 130, 66, 65, 64, 63, 40, 9):
        pre = int(rng.integers(0, 4 ** Pr))
        tails = rng.choice(min(4 ** (k - Pr), 1 << 40), size=run_len, replace=False).astype(np.uint64)
        # make single-base neighbours likely: half of the tails are one substitution from another tail
        for i in range(0, run_len - 1, 2):
            pos = int(rng.integers(0, k - Pr))
            tails[i + 1] = tails[i] ^ (np.uint64(int(rng.integers(1, 4))) << np.uint64(2 * pos))
        v = (np.uint64(pre) << np.uint64(tail_bits)) | tails
        parts.append(np.unique(v) << np.uint64(64 - 2 * k))
    bg = rng.integers(0, 1 << 62, size=20000, dtype=np.int64).astype(np.uint64)
    bg = (bg >> np.uint64(64 - 2 * k)) << np.uint64(64 - 2 * k) if k < 32 else bg
    parts.append(bg)
    keys, cnt = _symmetric_closure(np.concatenate(parts), k, rng, 40)
    kt = fastk.write_ktab(str(tmp_path / "t"), k, keys, cnt, ibyte=3, nparts=2)
    want_plot, _ = ou.oracle_scan(fastk.keys_u64_to_bytes(keys, k), cnt, k)
    assert want_plot.sum() > 0
    with hetmers.Scan(kt) as sc:
        assert sc.is_symmetric()
        plot, st = sc.run("symm")
    assert st["path"] == 2
    assert np.array_equal(plot, want_plot)


# ------------------------------------------------------------------ the fingerprint -----------

def test_fingerprint_sends_asymmetric_tables_to_the_direct_passes(tmp_path):
    """a table may pass the reference's one-k-mer probe (PloidyPlot.c:1199-1229) without being
    symmetric: the fingerprint looks at every entry, and anything it rejects is scanned directly"""
    import torch
    from smudgeplot_b200.device import DeviceTable
    k = 31
    keys, cnt = synth.synth_table(k, 60000, 2, 0.02, 40, 4, 321, device="cuda")
    c16 = cnt.to(torch.int16)
    t = DeviceTable(k, keys, c16)
    assert t.check_symmetric()
    n = keys.numel()
    # (1) one entry missing, (2) one count off by one, (3) two counts swapped
    drop = torch.ones(n, dtype=torch.bool, device="cuda")
    drop[n // 3] = False
    assert not DeviceTable(k, keys[drop].contiguous(), c16[drop].contiguous()).check_symmetric()
    c2 = c16.clone()
    c2[n // 2] += 1
    assert not DeviceTable(k, keys, c2).check_symmetric()
    c3 = c16.clone()
    i, j = n // 5, n // 5 + 1
    if int(c3[i]) == int(c3[j]):
        c3[j] += 3
    c3[i], c3[j] = c3[j].clone(), c3[i].clone()
    rc = synth.revcomp_left(keys[i:i + 1], k)
    assert int(rc[0]) != int(keys[j])
    assert not DeviceTable(k, keys, c3).check_symmetric()
    # partial sums add up: fingerprint of two halves == fingerprint of the whole
    a = t.fingerprint(0, n // 2) + t.fingerprint(n // 2, n)
    assert torch.equal(a, t.fingerprint())
    # end to end: the asymmetric table goes through the direct passes and matches the oracle
    ku = synth.keys_to_u64_numpy(keys[drop])
    cu = cnt[drop].cpu().numpy().astype(np.uint16)
    kt = fastk.write_ktab(str(tmp_path / "asym"), k, ku, cu, ibyte=3, nparts=2)
    want_plot, _ = ou.oracle_scan(fastk.keys_u64_to_bytes(ku, k), cu, k)
    with hetmers.Scan(kt) as sc:
        assert not sc.is_symmetric()
        plot, st = sc.run()
        with pytest.raises(_lib.HetmersError):
            sc.run("symm")
    assert st["path"] == 1
    assert np.array_equal(plot, want_plot)


# ------------------------------------------------------------------ layer A: shards, widths ---

@pytest.mark.parametrize("k", [25, 40])
def test_sharded_symmetric_scan_is_independent_of_the_cuts(k):
    """what several GPUs do, on one: every shard runs runscan over its run-aligned range into its own
    work area, the Bloom segments are exchanged (the all-gather), every shard resolves its own
    candidates; the summed plot equals the one-shard plot and the direct passes"""
    import torch
    from smudgeplot_b200.device import DeviceTable
    keys, cnt = synth.synth_table(k, 60000, 3, 0.02, 60, 8, 77, device="cuda")
    khi = keys[:, 0].contiguous() if k > 32 else keys
    klo = keys[:, 1].contiguous() if k > 32 else None
    c16 = cnt.to(torch.int16)
    base = DeviceTable(k, khi, c16, keys_lo=klo).build_index()
    want = base.scan("direct").clone()
    assert torch.equal(base.scan("symm"), want)
    b64 = DeviceTable(k, khi, c16, keys_lo=klo, force_idx64=True).build_index(direct=False)
    assert torch.equal(b64.scan("symm"), want)                        # 64-bit bucket offsets
    n = base.n
    for raw in ([0, n // 7, n // 2, n - 3, n], [0, 1, n], [0, n // 3, n // 3 + 1, n]):
        cuts = [0] + [base.align_cut(c) for c in raw[1:-1]] + [n]
        cuts = sorted(set(cuts))
        nseg = len(cuts) - 1
        parts = []
        for r in range(nseg):
            w = DeviceTable(k, khi, c16, keys_lo=klo, bits=base.bits)
            w.bucket = base.bucket
            w.alloc_symm(cuts[r], cuts[r + 1], shards=w.make_symm_shards(cuts, r) if nseg > 1 else None)
            w.plot = torch.zeros_like(want).view(-1)
            w.runscan()
            parts.append(w)
        torch.cuda.synchronize()
        if nseg > 1:                                                   # the all-gather
            for r, w in enumerate(parts):
                for q, v in enumerate(parts):
                    if q != r:
                        w.bloom_view()[q].copy_(v.bloom_view()[q])
        total = torch.zeros_like(want).view(-1)
        ncand = 0
        for w in parts:
            w.resolve()
            nc, st = w.symm_status()
            assert st == 0
            ncand += nc
            total += w.plot
        assert torch.equal(total.view_as(want), want), cuts
        assert ncand > 0


def test_symmetric_scan_repeats_and_bloom_width(monkeypatch):
    """the plot depends neither on the Bloom filter's size nor on what an earlier scan left behind"""
    import torch
    from smudgeplot_b200.device import DeviceTable
    keys, cnt = synth.synth_table(31, 300000, 2, 0.01, 40, 12, 5, device="cuda")
    c16 = cnt.to(torch.int16)
    want = DeviceTable(31, keys, c16).build_index().scan("direct").clone()
    for bits in ("1", "2", "7", "64"):
        monkeypatch.setenv("HETMERS_BLOOM_BITS", bits)
        t = DeviceTable(31, keys, c16).build_index(direct=False)
        assert torch.equal(t.scan("symm"), want), bits
        assert torch.equal(t.scan("symm"), want), bits


def test_tables_made_of_pairs_overflow_the_record_staging(tmp_path):
    """nearly every entry is a member of an isolated pair: ~1000 candidate records per 2048-entry tile, far
    beyond the per-CTA staging area (RS_STAGE = 384) -> the warp-aggregated direct path to the list"""
    rng = np.random.default_rng(4242)
    k = 31
    base = rng.integers(0, 1 << 62, size=30000, dtype=np.int64).astype(np.uint64)
    base = (base >> np.uint64(2)) << np.uint64(2)                      # k = 31: the last two bits are padding
    pos = rng.integers(k // 2, k, size=base.size)                      # partner: one base changed in the back half
    sh = (np.uint64(62) - np.uint64(2) * pos.astype(np.uint64))
    delta = rng.integers(1, 4, size=base.size).astype(np.uint64)
    mate = base ^ (delta << sh)
    keys, cnt = _symmetric_closure(np.concatenate([base, mate]), k, rng, 60)
    kt = fastk.write_ktab(str(tmp_path / "t"), k, keys, cnt, ibyte=3, nparts=2)
    want_plot, want_deg = ou.oracle_scan(fastk.keys_u64_to_bytes(keys, k), cnt, k)
    assert (want_deg == 1).mean() > 0.9
    with hetmers.Scan(kt) as sc:
        assert sc.is_symmetric()
        plot, st = sc.run("symm")
    assert st["path"] == 2
    assert np.array_equal(plot, want_plot)
