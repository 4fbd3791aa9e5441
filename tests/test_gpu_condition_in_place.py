"""Conditioning the resident table in place (hm_scan_condition, DESIGN.md §4d): on seeded canonical untrimmed tables
of a few million entries at k = 31 and 40, trim + symmetrise, trim only and symmetrise only give the table and the
plot of the numpy restatement, under the default budget and under one below what the earlier in-place algorithm
needed (the doubled table sorted in one piece), where symmetrising takes several key ranges."""
import re

import numpy as np
import pytest

from smudgeplot_b200 import _lib, fastk, hetmers
from test_gpu_parity import _condition_numpy, canonical_mask
from tools import synth

pytestmark = pytest.mark.gpu

L = 12
MODES = [(True, True), (True, False), (False, True)]          # (trim, symm)


@pytest.fixture(autouse=True)
def _clean_env(monkeypatch, built):
    for var in ("HETMERS_PATH", "HETMERS_STREAM", "HETMERS_STREAM_CHUNK", "HETMERS_DEVICE_BUDGET"):
        monkeypatch.delenv(var, raising=False)
    yield
    _lib.lib().hm_set_device_budget(0)


def old_in_place_bytes(n, k, trim, symm):
    """what the earlier in-place algorithm asked of the budget for n entries: the table arrays and the plot, plus
    the larger of the trim (flags + an n-entry copy) and the symmetrise stage (two 2n-entry tables, flags, the
    sort's permutation pair at k > 32), with CUB's scratch counted as 0"""
    ent = 8 + (8 if k > 32 else 0) + 2
    table = 8 * (n + 1) + (8 * (n + 1) if k > 32 else 0) + 2 * (n + 8) + 8 * _lib.PLOT_CELLS
    t = n + ent * (n + 1) + 8 if trim else 0
    m = 2 * n
    s = 2 * ent * (m + 1) + m + 8 + (8 * m if k > 32 else 0) if symm else 0
    return table + max(t, s)


@pytest.fixture(scope="module", params=[31, 40])
def table(request, tmp_path_factory):
    k = request.param
    G = synth.calibrate_G(k, 7_000_000, 2, 0.02, 40, 1)
    keys, cnt = synth.synth_table(k, G, 2, 0.02, 40, 1, 40 + k, device="cuda")      # untrimmed: counts from 1
    keys, cnt = keys.cpu(), cnt.cpu()
    ku = synth.keys_to_u64_numpy(keys)
    cn = cnt.numpy().astype(np.uint16)
    canon = canonical_mask(keys, ku, k)
    ku, cn = ku[canon], cn[canon]
    assert len(cn) > 2_000_000
    kt = fastk.write_ktab(str(tmp_path_factory.mktemp(f"k{k}") / "raw"), k, ku, cn, ibyte=3, nparts=2)
    want = {}
    for trim, symm in MODES:
        ck, cc = _condition_numpy(ku, cn, k, L, trim, symm)
        with hetmers.Scan(fastk.write_ktab(str(tmp_path_factory.mktemp("want") / "t"), k, ck, cc, ibyte=3)) as sc:
            plot, _ = sc.run()
        want[trim, symm] = ck, cc, plot
    with hetmers.Scan(kt) as sc:
        incore = sc.residency()[1]
    return k, kt, incore, want


def condition(kt, budget, trim, symm):
    with hetmers.Scan(kt, device_budget=budget) as sc:
        assert not sc.residency()[0]
        n = sc.condition(L, trim, symm)
        keys, cnt, _ = sc.download(deg=False)
        plot, _ = sc.run()
    _lib.lib().hm_set_device_budget(0)
    return n, keys, cnt, plot


def needs(kt, budget, trim, symm):
    """(bytes the call needs at least, bytes it needs to condition in one range) from a refusal, or None"""
    with hetmers.Scan(kt, device_budget=budget) as sc:
        try:
            sc.condition(L, trim, symm)
        except _lib.HetmersError as e:
            assert e.code == -3, str(e)
            m = re.search(r"needs (\d+) device bytes \((\d+) in one range\)", str(e))
            assert m, str(e)
            return int(m.group(1)), int(m.group(2))
        finally:
            _lib.lib().hm_set_device_budget(0)
    return None


@pytest.mark.parametrize("trim,symm", MODES)
def test_default_budget(table, trim, symm):
    k, kt, _, want = table
    ck, cc, plot = want[trim, symm]
    n, keys, cnt, got = condition(kt, 0, trim, symm)
    assert n == len(cc)
    assert np.array_equal(keys, ck) and np.array_equal(cnt, cc)
    assert np.array_equal(got, plot)


@pytest.mark.parametrize("trim,symm", MODES)
def test_budget_below_the_doubled_table(table, trim, symm):
    """a budget the in-core scan fits but the doubled table does not, so symmetrising takes several ranges;
    trimming alone takes the least budget that fits both the in-core scan and the call"""
    k, kt, incore, want = table
    ck, cc, plot = want[trim, symm]
    sizes = needs(kt, incore, trim, symm)                 # the scan's own budget, nothing beside it
    if symm:
        assert sizes is not None and sizes[0] < sizes[1]
        least, one = sizes
        budget = least + (one - least) // 4               # below one range over the whole table
        assert incore <= budget < old_in_place_bytes(kt.nels, k, trim, symm)
    elif sizes is None:
        budget = incore                                   # trimming alone: the trimmed copy fits where the index was
    else:
        budget = sizes[0]                                 # ... or takes exactly what the refusal asked for
        assert incore <= budget < old_in_place_bytes(kt.nels, k, trim, symm)
    n, keys, cnt, got = condition(kt, budget, trim, symm)
    assert n == len(cc)
    assert np.array_equal(keys, ck) and np.array_equal(cnt, cc)
    assert np.array_equal(got, plot)
