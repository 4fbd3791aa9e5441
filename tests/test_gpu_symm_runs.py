"""GPU test of the strand-symmetric scan on runs of three to 66 entries (run with -m gpu on an H100).
runscan_kernel settles every run of up to 65 entries whose head lies in its 2048-entry tile from the
shared-memory window (the tile plus 64 entries on either side) and lists longer runs for runs_kernel, so
runs that straddle a tile edge and the lengths around that limit are where a slip would show.  Both
pass-1 kernels run every case (test_gpu_symm's autouse fixtures)."""
import numpy as np
import pytest
import torch

import oracle_util as ou
from smudgeplot_b200 import fastk, hetmers
from test_gpu_symm import _need_gpu, _symmetric_closure, runscan_kernel_variant  # noqa: F401
from tools import synth

pytestmark = pytest.mark.gpu

RUN_LENGTHS = range(3, 67)
RUNS_PER_LENGTH = 200


def _rc2(hi, lo, k):
    """reverse complements of two-word keys (32 < k <= 64), numpy uint64"""
    a, b = synth.revcomp_long(torch.from_numpy(hi.view(np.int64).copy()), torch.from_numpy(lo.view(np.int64).copy()), k)
    return a.numpy().view(np.uint64), b.numpy().view(np.uint64)


def _symmetric_closure2(keys, k, rng, cmax):
    """_symmetric_closure for two-word keys uint64[n,2]: sorted unique keys and their reverse complements"""
    keys = np.unique(np.concatenate([keys, np.stack(_rc2(keys[:, 0], keys[:, 1], k), axis=1)]), axis=0)
    rh, rl = _rc2(keys[:, 0], keys[:, 1], k)
    fwd = (keys[:, 0] < rh) | ((keys[:, 0] == rh) & (keys[:, 1] <= rl))
    canon = np.where(fwd[:, None], keys, np.stack([rh, rl], axis=1))
    _, inv = np.unique(canon, axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    cc = rng.integers(1, cmax + 1, size=inv.max() + 1).astype(np.uint16)
    return keys, cc[inv]


def runs_table(k, seed):
    """RUNS_PER_LENGTH runs of every length in RUN_LENGTHS (entries sharing their first k/2 bases, half of
    them one substitution from another member) among unrelated entries, closed under reverse complement;
    counts up to 160, so that pairs land both inside and outside the shared-memory plot tile of pass 2.
    Keys: left-aligned uint64[n] (k <= 32) or uint64[n,2] (32 < k <= 64)."""
    rng = np.random.default_rng(9100 + seed)
    Pr = k // 2
    tail_bits = 2 * (k - Pr)                             # <= 64 for k <= 64
    lens = np.repeat(np.array(list(RUN_LENGTHS)), RUNS_PER_LENGTH)
    pres = np.unique(rng.integers(0, 4 ** Pr, size=2 * lens.size, dtype=np.uint64))
    pres = rng.permutation(pres)[:lens.size]
    pre_l, tail_l = [], []
    for run_len, pre in zip(lens.tolist(), pres.tolist()):
        tails = np.unique(rng.integers(0, (1 << tail_bits) - 1, size=run_len + 8, dtype=np.uint64,
                                       endpoint=True))
        tails = rng.permutation(tails)[:run_len]
        for i in range(0, run_len - 1, 2):
            if rng.random() < 0.5:
                pos = int(rng.integers(0, k - Pr))
                tails[i + 1] = tails[i] ^ (np.uint64(int(rng.integers(1, 4))) << np.uint64(2 * pos))
        pre_l.append(np.full(run_len, pre, dtype=np.uint64))
        tail_l.append(tails)
    pre, tail = np.concatenate(pre_l), np.concatenate(tail_l)
    nbg = 200000
    if k <= 32:
        runs = ((pre << np.uint64(tail_bits)) | tail) << np.uint64(64 - 2 * k)
        bg = rng.integers(0, 1 << 62, size=nbg, dtype=np.int64).astype(np.uint64) << np.uint64(2)
        bg = (bg >> np.uint64(64 - 2 * k)) << np.uint64(64 - 2 * k)
        return _symmetric_closure(np.concatenate([runs, bg]), k, rng, 160)
    # the k-mer is pre (2*Pr bits) then tail (tail_bits bits), 2k bits in all, left aligned in two words
    lo_bits = 2 * k - 64                                 # bits of the k-mer in the second word
    hi = (pre << np.uint64(64 - 2 * Pr)) | (tail >> np.uint64(lo_bits))
    lo = (tail & np.uint64((1 << lo_bits) - 1)) << np.uint64(64 - lo_bits)
    bh = rng.integers(0, 1 << 62, size=nbg, dtype=np.int64).astype(np.uint64) << np.uint64(2)
    bl = (rng.integers(0, 1 << 62, size=nbg, dtype=np.int64).astype(np.uint64) >> np.uint64(62 - lo_bits)) \
        << np.uint64(64 - lo_bits)
    keys = np.stack([np.concatenate([hi, bh]), np.concatenate([lo, bl])], axis=1)
    return _symmetric_closure2(keys, k, rng, 160)


def run_length_counts(keys, k):
    """{run length: number of runs} of sorted left-aligned keys"""
    hi = keys if keys.ndim == 1 else keys[:, 0]
    pre = hi >> np.uint64(64 - 2 * (k // 2))
    _, lengths = np.unique(pre, return_counts=True)
    ls, n = np.unique(lengths, return_counts=True)
    return dict(zip(ls.tolist(), n.tolist()))


@pytest.mark.parametrize("k,seed", [(31, 1), (32, 2), (40, 3)])
def test_runs_of_three_to_66_entries_across_tile_edges(k, seed, tmp_path):
    keys, cnt = runs_table(k, seed)
    lengths = run_length_counts(keys, k)
    assert all(lengths.get(n, 0) >= RUNS_PER_LENGTH // 2 for n in RUN_LENGTHS), lengths
    kb = fastk.keys_u64_to_bytes(keys, k)
    kt = fastk.write_ktab(str(tmp_path / "t"), k, kb, cnt, ibyte=3, nparts=2)
    want_plot, _ = ou.oracle_scan(kb, cnt, k)
    with hetmers.Scan(kt) as sc:
        assert sc.is_symmetric()
        plot, st = sc.run("symm")
    assert st["path"] == 2
    assert np.array_equal(plot, want_plot)
