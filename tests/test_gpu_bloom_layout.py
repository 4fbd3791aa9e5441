"""The symmetric scan's Bloom filter after pass 1 (csrc/hm_symm.cu bloom_slot / bloom_insert: 3 bits in one 64-bit
word, DESIGN.md §4a), bit for bit against its numpy restatement in tools/bloom_layout_model.py: every segment holds exactly the set S of its
range (entries with a partner at a position >= k - k/2 and a count sum <= SMAX, oracle_util.partial_runscan's
rule), so no element of S can test negative in pass 2.  Genome-like tables at k = 21 .. 64 in one and in three
segments, and the crowded small-k table of the dense pass-1 kernel (and runs_kernel behind it)."""
import numpy as np
import pytest
import torch

import oracle_util as ou
from smudgeplot_b200 import _lib
from smudgeplot_b200.device import DeviceTable
from tools import bloom_layout_model as blm
from tools import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _need_gpu(built):
    assert _lib.lib().hm_device_count() >= 1, "these tests need a CUDA device (no CPU fallback exists)"


@pytest.fixture(autouse=True)
def _default_filter(monkeypatch):
    monkeypatch.delenv("HETMERS_BLOOM_BITS", raising=False)
    monkeypatch.delenv("HETMERS_RUNSCAN", raising=False)


def _in_s(hi, lo, cnt, k):
    """S membership by partial_runscan's rule, on 128-bit keys (hi << 64 | lo; lo = 0 for k <= 32)"""
    key = [(int(a) << 64) | int(b) for a, b in zip(hi.tolist(), lo.tolist())]
    pos_of = {x: i for i, x in enumerate(key)}
    pup = k - k // 2
    out = np.zeros(len(key), dtype=bool)
    for i, x in enumerate(key):
        cx = int(cnt[i])
        for p in range(pup, k):
            sh = 126 - 2 * p
            b = (x >> sh) & 3
            for alt in range(4):
                j = pos_of.get((x & ~(3 << sh)) | (alt << sh)) if alt != b else None
                if j is not None and cx + int(cnt[j]) <= ou.SMAX:
                    out[i] = True
                    break
            if out[i]:
                break
    return out


def _check_filter(k, khi, klo, cnt, nseg):
    c16 = cnt.to(torch.int16)
    base = DeviceTable(k, khi, c16, keys_lo=klo).build_index(direct=False)
    n = base.n
    cuts = sorted(set([0] + [base.align_cut(n * r // nseg) for r in range(1, nseg)] + [n]))
    assert len(cuts) == nseg + 1
    hi = khi.cpu().numpy().view(np.uint64)
    lo = klo.cpu().numpy().view(np.uint64) if klo is not None else np.zeros_like(hi)
    s = _in_s(hi, lo, cnt.cpu().numpy(), k)
    assert s.sum() > 0
    for r in range(nseg):
        w = DeviceTable(k, khi, c16, keys_lo=klo, bits=base.bits)
        w.bucket = base.bucket
        w.alloc_symm(cuts[r], cuts[r + 1], shards=w.make_symm_shards(cuts, r) if nseg > 1 else None)
        w.runscan()
        nc, st = w.symm_status()
        assert st == 0
        got = w.bloom_view()[r].cpu().numpy().view(np.uint32)
        seg_words = got.size
        m = np.zeros(n, dtype=bool)
        m[cuts[r]:cuts[r + 1]] = True
        m &= s
        want = blm.build_filter("word64", hi[m], lo[m], k, seg_words)
        assert np.array_equal(got, want), (k, nseg, r)
        assert blm.test_filter("word64", got, hi[m], lo[m], k, seg_words).all()


@pytest.mark.parametrize("nseg", [1, 3])
@pytest.mark.parametrize("k", [21, 31, 32, 33, 40, 64])
def test_filter_is_the_restated_layout_over_s(k, nseg):
    keys, cnt = synth.synth_table(k, 8000, 2, 0.02, 40, 4, 600 + k, device="cuda", extra_hom_repeats=1)
    khi = keys[:, 0].contiguous() if k > 32 else keys
    klo = keys[:, 1].contiguous() if k > 32 else None
    _check_filter(k, khi, klo, cnt, nseg)


@pytest.mark.parametrize("route", ["auto", "dense"])
def test_filter_of_the_crowded_small_k_table(route, monkeypatch):
    """a quarter of all 10-mers: the dense pass-1 kernel, its long runs left to runs_kernel"""
    if route == "dense":
        monkeypatch.setenv("HETMERS_RUNSCAN", "dense")
    k = 10
    rng = np.random.default_rng(910)
    vals = rng.choice(4 ** k, size=4 ** k // 8, replace=False).astype(np.uint64) << np.uint64(64 - 2 * k)
    t = torch.from_numpy(vals.view(np.int64).copy())
    keys = np.unique(np.concatenate([vals, synth.revcomp_left(t, k).numpy().view(np.uint64)]))
    canon = np.minimum(keys, synth.revcomp_left(torch.from_numpy(keys.view(np.int64).copy()), k).numpy().view(np.uint64))
    _, inv = np.unique(canon, return_inverse=True)
    cnt = rng.integers(1, 600, size=inv.max() + 1).astype(np.int32)[inv]
    khi = torch.from_numpy(keys.view(np.int64).copy()).cuda()
    _check_filter(k, khi, None, torch.from_numpy(cnt).cuda(), 1)
