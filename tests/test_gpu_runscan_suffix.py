"""GPU test of runscan_kernel's in-run pair test at the edges of its word size (run with -m gpu on an H100).
Two members of a run differ only in their last k - k/2 bases, and runscan_kernel tests a pair on those
bases alone: one 32-bit word for k <= 32 (k = 32: exactly 32 bits), one 64-bit word for 32 < k <= 64
(k = 33: the first two-word key, 34 bits; k = 64: exactly 64 bits).  Each case has runs of three to 66
entries straddling tile edges, in the style of test_gpu_symm_runs, and the symmetric scan's plot must equal
both the direct passes' and the oracle's."""
import numpy as np
import pytest

import oracle_util as ou
from smudgeplot_b200 import fastk, hetmers
from test_gpu_symm import _need_gpu  # noqa: F401
from test_gpu_symm_runs import RUN_LENGTHS, RUNS_PER_LENGTH, _symmetric_closure2, run_length_counts, runs_table

pytestmark = pytest.mark.gpu


def runs_table_k64(seed):
    """runs_table for k = 64, where the run prefix and the varying tail are one whole key word each"""
    k = 64
    rng = np.random.default_rng(9300 + seed)
    lens = np.repeat(np.array(list(RUN_LENGTHS)), RUNS_PER_LENGTH)
    pres = np.unique(rng.integers(0, 1 << 64, size=2 * lens.size, dtype=np.uint64))
    pres = rng.permutation(pres)[:lens.size]
    hi_l, lo_l = [], []
    for run_len, pre in zip(lens.tolist(), pres.tolist()):
        tails = np.unique(rng.integers(0, (1 << 64) - 1, size=run_len + 8, dtype=np.uint64, endpoint=True))
        tails = rng.permutation(tails)[:run_len]
        for i in range(0, run_len - 1, 2):
            if rng.random() < 0.5:
                pos = int(rng.integers(0, k // 2))
                tails[i + 1] = tails[i] ^ (np.uint64(int(rng.integers(1, 4))) << np.uint64(2 * pos))
        hi_l.append(np.full(run_len, pre, dtype=np.uint64))
        lo_l.append(tails)
    nbg = 200000
    bh = rng.integers(0, 1 << 64, size=nbg, dtype=np.uint64)
    bl = rng.integers(0, 1 << 64, size=nbg, dtype=np.uint64)
    keys = np.stack([np.concatenate(hi_l + [bh]), np.concatenate(lo_l + [bl])], axis=1)
    return _symmetric_closure2(keys, k, rng, 160)


@pytest.mark.parametrize("k,seed", [(32, 11), (33, 12), (64, 13)])
def test_in_run_pair_test_at_word_edges(k, seed, tmp_path, monkeypatch):
    monkeypatch.setenv("HETMERS_RUNSCAN", "sparse")          # runscan_kernel, whatever the table's density
    keys, cnt = runs_table_k64(seed) if k == 64 else runs_table(k, seed)
    lengths = run_length_counts(keys, k)
    assert all(lengths.get(n, 0) >= RUNS_PER_LENGTH // 2 for n in RUN_LENGTHS), lengths
    kb = fastk.keys_u64_to_bytes(keys, k)
    kt = fastk.write_ktab(str(tmp_path / "t"), k, kb, cnt, ibyte=3, nparts=2)
    want_plot, _ = ou.oracle_scan(kb, cnt, k)
    assert want_plot.sum() > 0
    with hetmers.Scan(kt) as sc:
        assert sc.is_symmetric()
        plot, st = sc.run("symm")
        direct, _ = sc.run("direct")
    assert st["path"] == 2
    assert np.array_equal(plot, direct)
    assert np.array_equal(plot, want_plot)
