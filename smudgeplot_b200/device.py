"""Layer A of the C ABI driven from Python: torch supplies device memory and streams (plumbing
only), every computation is one of our CUDA kernels in libhetmers_b200.so.

`DeviceTable` holds the structure-of-arrays table of DESIGN.md §3 in torch tensors:
    keys  int64[n]   (bit pattern of the left-aligned uint64 packed k-mer, bases 0..31)
    keys_lo int64[n] (bases 32..63, k > 32 only)
    cnt   int16[n]   (bit pattern of the uint16 count)
    deg   uint8[n+]  (the reference's `Pair` incidence array, PloidyPlot.c:163)
    bucket int32/int64[(1<<bits)+1]
    filter int32[2^fbits/32]  (prefix presence bitmap probed by pass 1)
    up    int32/int64[hi-lo]  (upper partner recorded by pass 1)
    plot  int64[1001*501]
"""
from __future__ import annotations

import torch

from . import _lib


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _stream():
    return torch.cuda.current_stream().cuda_stream


class DeviceTable:
    def __init__(self, kmer: int, keys: torch.Tensor, cnt: torch.Tensor, bits: int | None = None,
                 fbits: int | None = None, keys_lo: torch.Tensor | None = None, force_idx64: bool = False):
        assert keys.is_cuda and keys.dtype == torch.int64 and keys.is_contiguous()
        assert (kmer > 32) == (keys_lo is not None), "k > 32 needs the second key word (keys_lo)"
        self.keys_lo = keys_lo
        assert cnt.is_cuda and cnt.dtype == torch.int16 and cnt.is_contiguous()
        self.L = _lib.lib()
        self.kmer = kmer
        self.keys, self.cnt = keys, cnt
        self.n = keys.numel()
        self.device = keys.device
        self.idx64 = int(self.n >= 0xFFFFFFF0 or force_idx64)     # 64-bit offsets (tables >= 2^32 entries)
        self.idx_dtype = torch.int64 if self.idx64 else torch.int32
        self.bits = bits if bits is not None else self.L.hm_pick_bucket_bits(self.n)
        self.fbits = fbits if fbits is not None else self.L.hm_pick_filter_bits(self.n)
        self.bucket = None
        self.filter = None
        self.deg = None
        self.up = None
        self.lo = self.hi = 0
        self.launches = 0
        self.shards = None          # _lib.Shards when the incidence array is sharded over GPUs
        self.deg_ptr = None         # raw device pointer overriding self.deg (IPC-shared allocation)
        self.symmetric = None       # fingerprint verdict (None = not examined yet)
        self.symm_layout = None     # _lib.SymmLayout + work area of the strand-symmetric scan
        self.symm_work = None
        self.symm_shards = None     # _lib.SymmShards when several GPUs share the scan

    # ---- construction -------------------------------------------------------------------
    @classmethod
    def from_records(cls, kmer: int, ibyte: int, records: torch.Tensor, index: torch.Tensor,
                     first: int = 0, n_total: int | None = None, out=None, out_lo=None):
        """Unpack raw FastK part records (uint8[n*pbyte], on the device) holding table ordinals
        [first, first+n) into SoA tensors; `index` is the stub index int64[1<<8*ibyte] on the
        device.  With `out=(keys, cnt)` (full-table tensors) the shard is written in place."""
        L = _lib.lib()
        kbyte = (kmer + 3) >> 2
        pbyte = kbyte - ibyte + 2
        n = records.numel() // pbyte
        lv = klo = None
        if out is None:
            keys = torch.empty(n, dtype=torch.int64, device=records.device)
            cnt = torch.empty(n, dtype=torch.int16, device=records.device)
            kv, cv = keys, cnt
            if kmer > 32:
                klo = lv = torch.empty(n, dtype=torch.int64, device=records.device)
        else:
            keys, cnt = out
            kv, cv = keys[first:first + n], cnt[first:first + n]
            if kmer > 32:
                lv = out_lo[first:first + n]
        with torch.cuda.device(records.device):
            _lib.check(L.hm_k_unpack_records(_ptr(records), n, first, _ptr(index), ibyte, kmer,
                                             _ptr(kv), _ptr(lv), _ptr(cv), _stream()))
        if out is None:
            t = cls(kmer, keys, cnt, keys_lo=klo)
            t.launches += 1
            return t
        return None

    def build_index(self, direct: bool = True):
        """bucket index (both paths) + the prefix filter of the direct search (`direct=False` skips
        the filter: tables that pass the symmetry fingerprint never probe it)"""
        self.bucket = torch.empty((1 << self.bits) + 1, dtype=self.idx_dtype, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.L.hm_k_build_bucket_index(_ptr(self.keys), self.n, self.bits,
                                                      _ptr(self.bucket), self.idx64, _stream()))
        self.launches += 1
        if direct:
            self.build_filter()
        return self

    def build_filter(self):
        self.filter = torch.empty(self.L.hm_filter_words(self.fbits), dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.L.hm_k_build_filter(_ptr(self.keys), self.n, self.fbits, _ptr(self.filter), _stream()))
        self.launches += 1
        return self

    # ---- strand-symmetric scan (csrc/hm_symm.cu) -----------------------------------------
    def fingerprint(self, i0: int = 0, i1: int | None = None, seeds=None) -> torch.Tensor:
        """keyed multiset fingerprints of {(x,cnt)} and {(rc x,cnt)} over entries [i0,i1): int64[4]
        device tensor (sums mod 2^64; partial sums of several ranges / ranks just add up)"""
        import ctypes as C
        i1 = self.n if i1 is None else i1
        sd = (C.c_uint64 * 2)()
        if seeds is None:
            self.L.hm_symm_seeds(sd)
        else:
            sd[0], sd[1] = seeds
        acc = torch.zeros(4, dtype=torch.int64, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.L.hm_k_symm_fingerprint(_ptr(self.keys), _ptr(self.keys_lo), _ptr(self.cnt), i0, i1,
                                                    self.kmer, sd, _ptr(acc), _stream()))
        self.launches += 1
        return acc

    def check_symmetric(self) -> bool:
        """does the table hold rc(x) with count(x) for every x?  (what examine_table's one-k-mer
        probe stands for, PloidyPlot.c:1199-1229, verified for the whole table)"""
        if self.kmer < 2:
            self.symmetric = False
        else:
            a = self.fingerprint().tolist()
            self.symmetric = (a[0] == a[2] and a[1] == a[3])
        return self.symmetric

    def align_cut(self, cut: int) -> int:
        """next run boundary at or after `cut` (a run = entries sharing their first k/2 bases)"""
        import ctypes as C
        out = C.c_int64()
        with torch.cuda.device(self.device):
            _lib.check(self.L.hm_symm_align_cut(_ptr(self.keys), self.n, self.kmer, int(cut), C.byref(out)))
        return int(out.value)

    def make_symm_shards(self, cuts, rank: int):
        """_lib.SymmShards for run-aligned cuts [0, c1, ..., n] as seen from shard `rank`"""
        sh = _lib.SymmShards()
        sh.n_seg, sh.self_ = len(cuts) - 1, rank
        for r, c in enumerate(cuts):
            sh.off[r] = c
        idx = torch.tensor([min(c, self.n - 1) for c in cuts[1:-1]], dtype=torch.int64, device=self.device)
        first = self.keys[idx].tolist() if idx.numel() and self.n else [0] * idx.numel()   # (an empty table: no keys)
        for r, (c, v) in enumerate(zip(cuts[1:-1], first), start=1):
            sh.first_key[r] = (v & 0xFFFFFFFFFFFFFFFF) if c < self.n else 0xFFFFFFFFFFFFFFFF
        return sh

    def alloc_symm(self, lo: int = 0, hi: int | None = None, shards=None):
        """work area of the symmetric scan over [lo,hi); `shards` = _lib.SymmShards for several GPUs"""
        import ctypes as C
        hi = self.n if hi is None else hi
        self.lo, self.hi = lo, hi
        lay = _lib.SymmLayout()
        nseg = shards.n_seg if shards is not None else 1
        _lib.check(self.L.hm_symm_plan(self.n, hi - lo, self.kmer, nseg, C.byref(lay)))
        self.symm_layout, self.symm_shards = lay, shards
        self.symm_work = torch.empty(lay.bytes, dtype=torch.uint8, device=self.device)
        if getattr(self, "plot", None) is None:
            self.plot = torch.zeros(_lib.PLOT_CELLS, dtype=torch.int64, device=self.device)
        return self

    def bloom_view(self) -> torch.Tensor:
        """int32[n_seg, seg_words] view of the Bloom segments inside the work area"""
        lay = self.symm_layout
        return self.symm_work[lay.off_bloom: lay.off_bloom + 4 * lay.seg_words * lay.n_seg].view(torch.int32) \
                   .view(lay.n_seg, lay.seg_words)

    def _symm_shards(self):
        import ctypes as C
        return C.byref(self.symm_shards) if self.symm_shards is not None else None

    def runscan(self, mid_event=None):
        """'pass 1' of the symmetric scan over [lo,hi): runscan kernel, then the kernel for the runs it only
        listed; `mid_event` is recorded between the two (timing of the dominant kernel alone)"""
        import ctypes as C
        args = (_ptr(self.keys), _ptr(self.keys_lo), _ptr(self.cnt), self.n, _ptr(self.bucket), self.bits, self.idx64,
                self.kmer, self.lo, self.hi, _ptr(self.symm_work), C.byref(self.symm_layout), self._symm_shards())
        with torch.cuda.device(self.device):
            _lib.check(self.L.hm_k_symm_runscan(*args, _stream()))
            if mid_event is not None:
                mid_event.record()
            _lib.check(self.L.hm_k_symm_runs(*args, _stream()))
        self.launches += 2

    def resolve(self):
        """'pass 2' of the symmetric scan; accumulates into self.plot"""
        import ctypes as C
        with torch.cuda.device(self.device):
            _lib.check(self.L.hm_k_symm_resolve(_ptr(self.keys), _ptr(self.keys_lo), _ptr(self.cnt), self.n,
                                                _ptr(self.bucket), self.bits, self.idx64, self.kmer,
                                                _ptr(self.symm_work), C.byref(self.symm_layout), self._symm_shards(),
                                                _ptr(self.plot), _stream()))
        self.launches += 1

    def extract(self, pixmap: torch.Tensor, out: torch.Tensor, count: torch.Tensor, c0: int = 0, c1: int | None = None):
        """extract_kmer_pairs from the symmetric scan's work area (after runscan()): the isolated pairs among
        candidates [c0, c1) whose pixel has a label in pixmap (int16[1001*501], device) are appended to `out`
        (uint8[cap * 24] device tensor of hm_pair_rec) and counted in count (int64[1], zeroed by the caller;
        it counts every record, also those beyond cap).  At most two records per candidate."""
        import ctypes as C
        c1 = self.symm_layout.cand_cap if c1 is None else c1
        cap = out.numel() // C.sizeof(_lib.PairRec)
        with torch.cuda.device(self.device):
            _lib.check(self.L.hm_k_symm_extract(_ptr(self.keys), _ptr(self.keys_lo), _ptr(self.cnt), self.n,
                                                _ptr(self.bucket), self.bits, self.idx64, self.kmer,
                                                _ptr(self.symm_work), C.byref(self.symm_layout), self._symm_shards(),
                                                _ptr(pixmap), int(c0), int(c1), _ptr(out), cap, _ptr(count), _stream()))
        self.launches += 1

    def symm_status(self):
        """(candidate pairs, status bits) of the last symmetric scan; synchronises"""
        import ctypes as C
        nc, st = C.c_uint64(), C.c_uint64()
        with torch.cuda.device(self.device):
            _lib.check(self.L.hm_symm_status(_ptr(self.symm_work), C.byref(self.symm_layout), C.byref(nc), C.byref(st),
                                             _stream()))
        return int(nc.value), int(st.value)

    def scan_symm(self):
        """both kernels of the symmetric scan on one GPU; -> plot int64[1001,501] (device tensor).
        Raises if the status word says the table was not symmetric after all."""
        if self.bucket is None:
            self.build_index(direct=False)
        if self.symm_work is None:
            self.alloc_symm()
        self.plot.zero_()
        self.runscan()
        self.resolve()
        nc, st = self.symm_status()
        if st != 0:
            raise _lib.HetmersError(-1, f"symmetric scan: status {st} (1 = a reverse complement is missing, "
                                        f"2 = candidate list overflow); use the direct passes")
        return self.plot.view(_lib.SMAX + 1, _lib.PLOT_W)

    # ---- the two passes -----------------------------------------------------------------
    def alloc_work(self, lo: int = 0, hi: int | None = None):
        hi = self.n if hi is None else hi
        self.lo, self.hi = lo, hi
        self.deg = torch.zeros((self.n + 4) & ~3, dtype=torch.uint8, device=self.device)
        self.up = torch.empty(max(hi - lo, 1), dtype=self.idx_dtype, device=self.device)
        self.plot = torch.zeros(_lib.PLOT_CELLS, dtype=torch.int64, device=self.device)
        return self

    def _deg(self):
        return self.deg_ptr if self.deg_ptr is not None else _ptr(self.deg)

    def _shards(self):
        import ctypes as C
        return C.byref(self.shards) if self.shards is not None else None

    def pass1(self):
        """neighbour search + degree (hm_k_pass1_degree) over [lo,hi); deg must be zero."""
        with torch.cuda.device(self.device):
            _lib.check(self.L.hm_k_pass1_degree(_ptr(self.keys), _ptr(self.keys_lo), _ptr(self.cnt), self.n, _ptr(self.bucket),
                                                self.bits, self.idx64, _ptr(self.filter), self.fbits, self.kmer,
                                                self.lo, self.hi,
                                                self._deg(), _ptr(self.up), self._shards(), _stream()))
        self.launches += 1

    def pass2(self):
        """isolated pairs -> plot (hm_k_pass2_plot) over [lo,hi); accumulates into self.plot."""
        with torch.cuda.device(self.device):
            _lib.check(self.L.hm_k_pass2_plot(_ptr(self.cnt), self._deg(), _ptr(self.up), self.idx64,
                                              self.lo, self.hi, _ptr(self.plot), self._shards(), _stream()))
        self.launches += 1

    def pass2_extract(self, pixmap: torch.Tensor, out: torch.Tensor | None, count: torch.Tensor,
                      lo: int | None = None, hi: int | None = None):
        """extract_kmer_pairs from the direct passes' results (hm_k_pass2_extract, after pass 1 and the exchange of
        the incidence bytes): the isolated pairs of entries [lo, hi) (default: the scan range [self.lo, self.hi))
        whose pixel has a label in pixmap (int16[1001*501], device) are appended to `out` (uint8[cap * 24] device
        tensor of hm_pair_rec; None = count only) and counted in count (int64[1], zeroed by the caller; it counts
        every record, also those beyond cap).  At most one record per entry."""
        import ctypes as C
        lo = self.lo if lo is None else lo
        hi = self.hi if hi is None else hi
        assert self.lo <= lo <= hi <= self.hi, (lo, hi, self.lo, self.hi)
        cap = out.numel() // C.sizeof(_lib.PairRec) if out is not None else 0
        up = _ptr(self.up) + (lo - self.lo) * self.up.element_size()     # up[] is indexed from self.lo
        with torch.cuda.device(self.device):
            _lib.check(self.L.hm_k_pass2_extract(_ptr(self.keys), _ptr(self.keys_lo), _ptr(self.cnt), self._deg(), up,
                                                 self.idx64, lo, hi, _ptr(pixmap), _ptr(out), cap, _ptr(count),
                                                 self._shards(), _stream()))
        self.launches += 1

    def scan(self, path: str = "auto"):
        """one GPU; -> plot int64[1001,501] (device tensor).  path: "auto" = the symmetric scan when the
        fingerprint says the table is strand-symmetric, else the direct passes; "direct" / "symm" force one"""
        if path == "symm" or (path == "auto" and self.kmer >= 2 and
                              (self.symmetric if self.symmetric is not None else self.check_symmetric())):
            return self.scan_symm()
        if self.bucket is None:
            self.build_index()
        if self.filter is None:
            self.build_filter()
        if self.deg is None:
            self.alloc_work()
        else:
            self.deg.zero_()
            self.plot.zero_()
        self.pass1()
        self.pass2()
        return self.plot.view(_lib.SMAX + 1, _lib.PLOT_W)

    # ---- examine_table pieces -----------------------------------------------------------
    def min_count(self, frst: int, last: int) -> int:
        out = torch.full((1,), 0x8000, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.L.hm_k_min_count(_ptr(self.cnt), frst, last, _ptr(out), _stream()))
        self.launches += 1
        return int(out.item())

    def find(self, queries: torch.Tensor, queries_lo: torch.Tensor | None = None) -> torch.Tensor:
        pos = torch.empty(queries.numel(), dtype=torch.int64, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.L.hm_k_find_keys(_ptr(self.keys), _ptr(self.keys_lo), self.n, _ptr(self.bucket), self.bits,
                                             self.idx64, _ptr(queries), _ptr(queries_lo), queries.numel(), _ptr(pos),
                                             _stream()))
        self.launches += 1
        return pos
