"""A scan gives back all the device memory it took, also when a call is refused.  With HETMERS_NO_POOL=1 every
device allocation of the scan driver is a cudaMalloc, so it shows in cudaMemGetInfo: free device memory after
hm_scan_destroy must equal free memory before hm_scan_create, byte for byte.  Each cycle runs once first, so that
what CUDA keeps for the process (lazily loaded kernels, runtime buffers) is in place before the measured cycle.
cudaMemGetInfo counts whole device pages, so a leak smaller than a page can pass unseen; the buffers a scan holds
are larger."""
import os
import re

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from smudgeplot_b200 import _lib, fastk, hetmers
from tools import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _need_gpu(built):
    assert _lib.lib().hm_device_count() >= 1, "these tests need a CUDA device (no CPU fallback exists)"


@pytest.fixture(autouse=True)
def _no_pool(monkeypatch):
    monkeypatch.setenv("HETMERS_NO_POOL", "1")
    for var in ("HETMERS_PATH", "HETMERS_STREAM", "HETMERS_STREAM_CHUNK"):
        monkeypatch.delenv(var, raising=False)
    yield
    _lib.lib().hm_set_device_budget(0)


def free_bytes():
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info(0)[0]


def gives_back(cycle):
    cycle()
    before = free_bytes()
    cycle()
    assert free_bytes() == before


def refused(call, code, text):
    with pytest.raises(_lib.HetmersError) as ei:
        call()
    assert ei.value.code == code and text in str(ei.value)


PIX = np.ones((_lib.SMAX + 1, _lib.PLOT_W), dtype=np.uint16)


def test_in_core_cycle(golden_meta, monkeypatch):
    """create -> examine -> run (both paths) -> extract (both routes) -> condition -> run"""
    e = golden_meta["_conditioning"]["untrimmed"]["e"]
    kt = fastk.read_ktab(os.path.join(GOLDEN, "conditioning", "untrimmed"))

    def cycle():
        with hetmers.Scan(kt) as sc:
            sc.examine(e)
            sc.run("symm")
            sc.run("direct")
            assert len(sc.extract(PIX)) > 0
            monkeypatch.setenv("HETMERS_PATH", "direct")
            assert len(sc.extract(PIX)) > 0
            monkeypatch.delenv("HETMERS_PATH")
            sc.condition(e, True, False)
            sc.run()
    gives_back(cycle)


def test_extract_refused_below_the_floor():
    kt = fastk.read_ktab(os.path.join(GOLDEN, "trip_k31", "trip_k31"))
    with hetmers.Scan(kt) as ref:
        incore = ref.residency()[1]

    def cycle():
        with hetmers.Scan(kt, device_budget=incore + 4096) as sc:
            sc.run()
            refused(lambda: sc.extract(PIX), -3, "device budget")
    gives_back(cycle)


@pytest.fixture(scope="module")
def list_table(tmp_path_factory):
    """the table and budget of test_shards_scan_a_table_one_budget_cannot_hold: one GPU runs out of list room"""
    keys, cnt = synth.synth_table(31, 1_000_000, 2, 0.01, 40, 8, 131, device="cuda")
    kt = synth.write_table(str(tmp_path_factory.mktemp("lt") / "t"), 31, keys, cnt, ibyte=2, nparts=2)
    return kt, -(-kt.nels // 32)


def test_streamed_list_enomem(list_table, monkeypatch):
    kt, chunk = list_table
    monkeypatch.setenv("HETMERS_STREAM", "1")
    monkeypatch.setenv("HETMERS_STREAM_CHUNK", str(chunk))
    with hetmers.Scan(kt, devices=[0] * 4, device_budget=1 << 34) as sc:
        sc.run()
        budget = int(sc.residency()[1] * 1.05)

    def cycle():
        with hetmers.Scan(kt, devices=[0], device_budget=budget) as sc:
            refused(sc.run, -3, "list needs")
    gives_back(cycle)


@pytest.mark.parametrize("shards", [1, 2])
def test_streamed_runs(shards, monkeypatch):
    kt = fastk.read_ktab(os.path.join(GOLDEN, "dip_k21", "dip_k21"))
    want = open(os.path.join(GOLDEN, "dip_k21", "dip_k21") + ".smu").read()
    monkeypatch.setenv("HETMERS_STREAM", "1")
    monkeypatch.setenv("HETMERS_STREAM_CHUNK", "1024")

    def cycle():
        with hetmers.Scan(kt, devices=[0] * shards, device_budget=1 << 34) as sc:
            assert sc.residency()[0]
            sc.examine(4)
            plot, _ = sc.run()
            sc.run()
        assert hetmers.smu_text(plot) == want
    gives_back(cycle)


def test_trimmed_table_is_counted_at_its_allocated_size(tmp_path):
    """conditioning sizes the new arrays for the entries before the trim; the scan counts them at that size, so
    the room extraction sees is the room the budget really leaves.  A refused extraction reports what is held."""
    keys, cnt = synth.synth_table(31, 3000, 2, 0.01, 40, 2, 5)
    kt = synth.write_table(str(tmp_path / "t"), 31, keys, cnt, ibyte=3)
    ethresh = int(np.sort(fastk.unpack_host(kt)[1])[7]) + 1       # drops at least 8 entries (the counts' padding)
    n0 = kt.nels
    with hetmers.Scan(kt) as ref:
        budget = ref.residency()[1]                       # in core, with no room to list pairs after the trim
    err = None
    for attempt in range(2):
        with hetmers.Scan(kt, device_budget=budget) as sc:
            assert not sc.residency()[0]
            try:
                n1 = sc.condition(ethresh, True, False)
            except _lib.HetmersError as e:                # conditioning's own budget check: take what it needs
                m = re.search(r"needs (\d+) device bytes", str(e))
                assert attempt == 0 and m, str(e)
                budget = int(m.group(1))
                continue
            sc.run()
            k1, c1, _ = sc.download(deg=False)
            with pytest.raises(_lib.HetmersError) as ei:
                sc.extract(PIX)
            err = str(ei.value)
            break
    assert 0 < n1 < n0 and err is not None and "device budget" in err
    held = int(re.search(r"beside the scan's (\d+) on GPU", err).group(1))
    with hetmers.Scan(fastk.write_ktab(str(tmp_path / "trimmed"), 31, k1, c1, ibyte=3)) as sc:
        incore1 = sc.residency()[1]                       # the same scan planned for n1 entries
    cap = n0 + 1                                          # keys and counts as the trim allocated them
    assert held == incore1 - 8 * (n1 + 1) - 2 * (n1 + 8) + 8 * cap + 2 * cap
